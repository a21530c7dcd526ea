// hts_io.h — host-side readers: BAI linear index + stats bin, .crai, .fai, and a BGZF writer; the BAM header type (the
// BAM reader itself is bam_feed.h).  Written from the SAM/BAM spec (SURVEY.md Appendix D); replaces what the reference
// gets from github.com/biogo/hts (indexcov/indexcov.go:514).
#pragma once
#include <stdint.h>
#include <string>
#include <utility>
#include <vector>

namespace glhts {

struct RefInfo {
    std::string name;
    int64_t length = 0;
    int64_t offset = 0, line_bases = 0, line_width = 0;   // .fai columns 3-5 (0 when the source has none, e.g. a BAM header)
};

// byte offset of 0-based base p of a FASTA record, relative to the record's first base (faidx `position`)
inline int64_t fasta_position(const RefInfo& r, int64_t p) { return r.line_bases > 0 ? p / r.line_bases * r.line_width + p % r.line_bases : p; }

// ---------------------------------------------------------------------------------------------- BGZF
// BGZF writer (indexcov's *.bed.gz, indexcov.go:248-257): 64 KB blocks, ModTime 0, OS 0xff, EOF block.
class BgzfWriter {
public:
    explicit BgzfWriter(const std::string& path);
    ~BgzfWriter();
    bool ok() const { return f_ != nullptr; }
    void write(const char* p, size_t n);
    void close();
private:
    void flush_batch();                              // deflates the pending 64 KB blocks on all cores, writes them in order
    void* f_ = nullptr;
    std::vector<uint8_t> buf_;                       // pending uncompressed bytes (up to kBatchBlocks blocks)
};

// ---------------------------------------------------------------------------------------------- BAM
struct BamHeader {
    std::string text;
    std::vector<RefInfo> refs;
    std::vector<std::string> sample_names() const;      // distinct @RG SM values, in order of appearance
};

// ---------------------------------------------------------------------------------------------- BAI / CSI
struct BaiIndex {
    std::vector<std::vector<uint64_t>> ioffsets;         // per reference: linear index (16 KB tiles; rebuilt from the bins' loffsets
                                                         // for a CSI, see bai_read)
    std::vector<uint64_t> mapped, unmapped;              // stats pseudo-bin 0x924a (indexcov/types.go:19,33-43; its CSI equivalent)
    std::vector<uint8_t> has_stats;
    uint64_t n_no_coor = 0;
    std::vector<uint64_t> ref_beg, ref_end;              // virtual-offset range of the reference's records (min chunk begin /
                                                         // max chunk end over its bins; 0 = no records)
    int min_shift = 14, depth = 5;                       // binning geometry: a BAI is (14, 5); a CSI says its own
    bool is_csi = false;
};
// One reference's binning index (SAM spec 5.2): the chunks of every bin but the stats pseudo-bin, bins in ascending order;
// bin[i]'s chunks are [cb, ce)[first[i] .. first[i+1]).
struct BaiBins {
    std::vector<uint32_t> bin, first;
    std::vector<uint64_t> cb, ce;
};
// Reads a BAI (raw, magic "BAI\1") or a CSI (BGZF, "CSI\1" once inflated; CSIv1 spec), told apart by their first bytes.
// bins (may be null): also keep every reference's binning index.  Most callers only want the linear index and the stats
// bin, and a WGS index's chunks are several MB, so they are dropped unless asked for.  A CSI has no linear index: ioffsets
// is rebuilt at 16 KB tiles from the bins' loffsets (hts_io.cpp, csi_linear), so every linear-index reader works on both.
std::string bai_read(const std::string& path, BaiIndex& out, std::vector<BaiBins>* bins = nullptr);
// The index files of a BAM in lookup order: x.bam.bai, x.bai (x.bam only), x.bam.csi, x.csi (x.bam only).  A BAM with
// both a BAI and a CSI uses its BAI.
std::vector<std::string> index_candidates(const std::string& bam_path);
// The virtual-offset ranges a query of intervals [beg[i], end[i]) on one reference has to read, as htslib's index query
// (hts_itr_query) picks them: the chunks of every bin reg2bins (SAM spec 5.3, over depth + 1 levels of 2^min_shift-base
// leaves) names for an interval, less those that end at or before min_off, the linear-index offset of the interval's first
// 16 KB tile (past the linear index: its last entry), and those that begin at or after max_off, the first chunk of the
// nearest bin with chunks to the right of the interval (htslib's walk: right along the leaves, up to the parent at a first
// child).  A bin several intervals name keeps the chunks any of them would keep between its smallest min_off and its
// largest max_off.  Sorted by begin, overlapping or touching ranges merged.  Empty intervals name no bins.
void bai_region_chunks(const BaiBins& bins, const std::vector<uint64_t>& lin, int min_shift, int depth, const int64_t* beg,
                       const int64_t* end, int64_t n, std::vector<std::pair<uint64_t, uint64_t>>& out);

// ---------------------------------------------------------------------------------------------- CRAI
// .crai (gzip'd text, 6 tab columns) -> per reference slices; sizes = the 16 KB pseudo-tiles indexcov uses for
// CRAM (indexcov/crai/crai.go:56-192).  crai_make_sizes returns false where the reference panics.
struct CraiSlices { std::vector<int64_t> start, span; std::vector<int32_t> bytes; };
std::string crai_read(const std::string& path, std::vector<CraiSlices>& out);
bool crai_make_sizes(const int64_t* start, const int64_t* span, const int32_t* bytes, int64_t n, std::vector<int64_t>& sizes);

// ---------------------------------------------------------------------------------------------- FAI
std::string fai_read(const std::string& path, std::vector<RefInfo>& out);

}  // namespace glhts
