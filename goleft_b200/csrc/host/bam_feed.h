// bam_feed.h — the BAM reader: header, index, and the two ways through the records.
//   BamFile::stream  every record from the first to EOF, in file order (no index needed): bam_decode_segments (an unindexed
//                    `goleft depth` / multidepth input) and bam_covstats_sample.
//   BamFile::decode  the index-guided, parallel feeder of `goleft depth`.
// decode replaces what the reference gets from its `samtools depth -Q q -r chr:b-e` children (depth/depth.go:45,116,152):
// only the BGZF blocks of the requested reference range are read (BAI linear index -> record-aligned virtual offsets),
// the range is cut into units at those offsets, and every pool thread inflates AND parses its own units — no serial
// record walk.  Each unit yields its M/=/X blocks already in start order (the parser knows the read position, so the
// second block of a deletion read waits in a tiny pending list until the stream has passed it); the units are then
// assembled into the engine's packed8 words (short reads) or sorted int32 arrays (long reads) by seg_pack.h.
#pragma once
#include <stdint.h>
#include <functional>
#include <string>
#include <vector>
#include "hts_io.h"

namespace glhts {

struct DecodeStats {
    int64_t n_records = 0, n_pass = 0;          // records seen / passing the samtools-depth filter
    int64_t bytes_in = 0, bytes_out = 0;        // compressed bytes read, bytes inflated
    double inflate_s = 0, parse_s = 0;          // summed over the workers
    double wall_s = 0;                          // of the whole call
    int units = 0;
};

struct ContigSegs {
    int format = 0;                             // 8: packed8 words, 32: (start,end) sorted by start, 0: nothing decoded
    std::vector<int32_t> anchors; std::vector<uint8_t> ds, len; int64_t n_blocks = 0;
    std::vector<int32_t> start, end; int64_t n = 0;
    int64_t n_pieces = 0; int32_t max_len = 0;
};

class BamFile {
public:
    BamFile() {}
    ~BamFile();
    BamFile(const BamFile&) = delete;
    // opens path and parses its header; with_index: also loads the first index of index_candidates(path) that reads (a BAI
    // or a CSI), and has_index tells whether one was found
    std::string open(const std::string& path, bool with_index = true);
    bool has_index = false;
    BamHeader header;
    BaiIndex bai;
    std::string path, index_path;               // index_path: the .bai or .csi that was loaded
    // M/=/X blocks of the records of reference `tid` that pass the samtools-depth filter (glbam::depth_counts) and can
    // overlap [beg, end).  want: 0 = choose (packed8 unless the blocks are long), 8, 32.  Needs the index.
    std::string decode(int tid, int64_t beg, int64_t end, int min_mapq, int threads, int want, ContigSegs& out, DecodeStats* st);
    // fn(r, bs) for every record from the first to EOF, in file order, on the calling thread (r: the record after its
    // block_size field, bs: block_size); fn returns false to stop.  The file is read in 32 MB compressed chunks whose
    // BGZF members are inflated on `threads` threads of the library's pool (0 = all of it), so it must not be called from
    // a pool task.
    std::string stream(int threads, const std::function<bool(const uint8_t*, uint32_t)>& fn);
    int fd() const { return fd_; }
    int64_t file_size() const { return size_; }
    int64_t rec_member() const { return rec_member_; }
    uint32_t rec_skip() const { return rec_skip_; }
private:
    int fd_ = -1;
    int64_t size_ = 0;
    int64_t rec_member_ = 0;                    // the first record: the file offset of its BGZF member and its offset
    uint32_t rec_skip_ = 0;                     // in that member's inflated bytes (may be the member's whole size)
};

// What `samtools depth -Q q` counts (SURVEY.md §8a D0, glbam::depth_counts / depth_blocks) from every record of the file.
struct SegmentSet {
    BamHeader header;
    std::vector<std::vector<int32_t>> start, end;        // per reference id, in record order
    int64_t n_records = 0, n_pass = 0;
};
std::string bam_decode_segments(const std::string& path, int min_mapq, int threads, int only_tid, SegmentSet& out);
std::string bam_read_header(const std::string& path, BamHeader& out);

// covstats (covstats/covstats.go:122-173): the sampled per-record values
struct CovstatsSample {
    std::vector<int32_t> read_len, insert, tmpl;
    int64_t n_unmapped = 0, k = 0, n_bad = 0, n_dup = 0, n_proper = 0;
    int64_t n_read = 0;                          // records up to and including the last one looked at, the skipped ones too
};
std::string bam_covstats_sample(BamFile& f, int n, int skip, CovstatsSample& out);

}  // namespace glhts

struct gl_ctx;
// the C ABI's opaque BAM handle (feeder_api.cpp, bamgpu.cu).  cs_pf: the ctx whose covstats prefetch reads this file.
// bins: the index's binning section, read again from index_path on the first region query (bins_read), so that only
// handles that query pay for it.
struct gl_bam {
    glhts::BamFile f; glhts::ContigSegs segs; glhts::CovstatsSample cs; gl_ctx* cs_pf = nullptr;
    std::vector<glhts::BaiBins> bins; bool bins_read = false;
};
// The virtual-offset ranges that hold every record of reference tid overlapping one of the intervals [beg[i], end[i])
// (glhts::bai_region_chunks over b's index).  "" or an error: no index, or its binning section cannot be read.
std::string gl_bam_plan_regions(gl_bam& b, int tid, const int64_t* beg, const int64_t* end, int64_t n,
                                std::vector<std::pair<uint64_t, uint64_t>>& out);
// covstats.cu: join and forget ctx's covstats prefetch, if any
void cs_prefetch_drop(gl_ctx* ctx);
