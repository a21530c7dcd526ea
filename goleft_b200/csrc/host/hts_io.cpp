// hts_io.cpp — BAI / CSI / CRAI / FAI readers, the BAM header's sample names and a BGZF writer (see hts_io.h).
#include "hts_io.h"
#include <stdio.h>
#include <string.h>
#include <zlib.h>
#include <algorithm>
#include <atomic>
#include <thread>

namespace glhts {

namespace {

inline uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
inline int32_t rdi32(const uint8_t* p) { return (int32_t)rd32(p); }
inline uint64_t rd64(const uint8_t* p) { return (uint64_t)rd32(p) | ((uint64_t)rd32(p + 4) << 32); }

}  // namespace

// ---------------------------------------------------------------------------------------------- writer
namespace {
constexpr size_t kBlockIn = 0xff00;                  // uncompressed bytes per BGZF block
constexpr size_t kBatchBlocks = 256;                 // 16 MB of text per parallel deflate round

// one BGZF member (indexcov.go:248-257: ModTime 0, OS 0xff); out must hold 64 KB + 64
size_t bgzf_deflate_block(const uint8_t* in, size_t n, uint8_t* out) {
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    deflateInit2(&zs, 6, Z_DEFLATED, -15, 8, Z_DEFAULT_STRATEGY);
    zs.next_in = const_cast<Bytef*>(in);
    zs.avail_in = (uInt)n;
    zs.next_out = out + 18;
    zs.avail_out = 0x10000 + 64 - 18 - 8;
    deflate(&zs, Z_FINISH);
    const size_t clen = zs.total_out;
    deflateEnd(&zs);
    const uint8_t hdr[18] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0, 0};
    memcpy(out, hdr, 18);
    const size_t bsize = 18 + clen + 8;
    out[16] = (uint8_t)((bsize - 1) & 0xff);
    out[17] = (uint8_t)((bsize - 1) >> 8);
    const uint32_t crc = (uint32_t)crc32(crc32(0L, Z_NULL, 0), in, (uInt)n);
    const uint32_t isz = (uint32_t)n;
    for (int i = 0; i < 4; i++) { out[18 + clen + i] = (uint8_t)(crc >> (8 * i)); out[22 + clen + i] = (uint8_t)(isz >> (8 * i)); }
    return bsize;
}
}  // namespace

BgzfWriter::BgzfWriter(const std::string& path) { f_ = fopen(path.c_str(), "wb"); buf_.reserve(kBlockIn * kBatchBlocks); }
BgzfWriter::~BgzfWriter() { close(); }

void BgzfWriter::flush_batch() {
    FILE* f = static_cast<FILE*>(f_);
    if (!f || buf_.empty()) return;
    const size_t nblk = (buf_.size() + kBlockIn - 1) / kBlockIn;
    std::vector<std::vector<uint8_t>> outs(nblk);
    std::vector<size_t> lens(nblk, 0);
    std::atomic<size_t> next(0);
    auto work = [&]() {
        for (;;) {
            const size_t i = next.fetch_add(1);
            if (i >= nblk) break;
            const size_t off = i * kBlockIn, n = std::min(kBlockIn, buf_.size() - off);
            outs[i].resize(0x10000 + 64);
            lens[i] = bgzf_deflate_block(buf_.data() + off, n, outs[i].data());
        }
    };
    const size_t nt = std::min<size_t>(nblk, std::max(1u, std::thread::hardware_concurrency()));
    std::vector<std::thread> pool;
    for (size_t t = 1; t < nt; t++) pool.emplace_back(work);
    work();
    for (auto& t : pool) t.join();
    for (size_t i = 0; i < nblk; i++) fwrite(outs[i].data(), 1, lens[i], f);
    buf_.clear();
}

void BgzfWriter::write(const char* p, size_t n) {
    while (n) {
        const size_t room = kBlockIn * kBatchBlocks - buf_.size();
        const size_t k = std::min(room, n);
        buf_.insert(buf_.end(), p, p + k);
        p += k; n -= k;
        if (buf_.size() == kBlockIn * kBatchBlocks) flush_batch();
    }
}

void BgzfWriter::close() {
    FILE* f = static_cast<FILE*>(f_);
    if (!f) return;
    flush_batch();
    uint8_t eof_block[0x10000 + 64];
    const size_t n = bgzf_deflate_block(nullptr, 0, eof_block);      // empty block = BGZF EOF marker
    fwrite(eof_block, 1, n, f);
    fclose(f);
    f_ = nullptr;
}

// ---------------------------------------------------------------------------------------------- BAM
std::vector<std::string> BamHeader::sample_names() const {
    std::vector<std::string> names;
    size_t p = 0;
    while (p < text.size()) {
        size_t e = text.find('\n', p);
        if (e == std::string::npos) e = text.size();
        if (e - p >= 3 && text.compare(p, 3, "@RG") == 0) {
            size_t q = p;
            while (q < e) {
                size_t t = text.find('\t', q);
                if (t == std::string::npos || t > e) t = e;
                if (t - q > 3 && text.compare(q, 3, "SM:") == 0) {
                    std::string sm = text.substr(q + 3, t - q - 3);
                    if (std::find(names.begin(), names.end(), sm) == names.end()) names.push_back(sm);
                }
                q = t + 1;
            }
        }
        p = e + 1;
    }
    return names;
}

// ---------------------------------------------------------------------------------------------- BAI / CSI
namespace {

// the BAI layout (SAM spec 5.2), b starting with its magic
std::string bai_parse(const std::vector<uint8_t>& b, const std::string& path, BaiIndex& out, std::vector<BaiBins>* bins) {
    out.min_shift = 14; out.depth = 5; out.is_csi = false;
    size_t off = 4;
    const int32_t n_ref = rdi32(b.data() + off); off += 4;
    if (n_ref < 0) return "corrupt BAI: " + path;
    out.ioffsets.assign((size_t)n_ref, {});
    out.mapped.assign((size_t)n_ref, 0);
    out.unmapped.assign((size_t)n_ref, 0);
    out.has_stats.assign((size_t)n_ref, 0);
    out.ref_beg.assign((size_t)n_ref, 0);
    out.ref_end.assign((size_t)n_ref, 0);
    if (bins) bins->assign((size_t)n_ref, BaiBins());
    for (int32_t r = 0; r < n_ref; r++) {
        if (off + 4 > b.size()) return "truncated BAI: " + path;
        const int32_t n_bin = rdi32(b.data() + off); off += 4;
        std::vector<std::pair<uint32_t, size_t>> at;                       // (bin, offset of its chunk list) when bins are kept
        for (int32_t k = 0; k < n_bin; k++) {
            if (off + 8 > b.size()) return "truncated BAI: " + path;
            const uint32_t bin = rd32(b.data() + off);
            const int32_t n_chunk = rdi32(b.data() + off + 4);
            off += 8;
            if (n_chunk < 0 || off + 16 * (size_t)n_chunk > b.size()) return "truncated BAI: " + path;
            if (bin == 0x924a && n_chunk == 2) {                           // StatsDummyBin, indexcov/types.go:19
                out.mapped[r] = rd64(b.data() + off + 16);
                out.unmapped[r] = rd64(b.data() + off + 24);
                out.has_stats[r] = 1;
            } else {
                if (bins) at.emplace_back(bin, off - 4);
                for (int32_t c = 0; c < n_chunk; c++) {
                    const uint64_t cb = rd64(b.data() + off + 16 * (size_t)c), ce = rd64(b.data() + off + 16 * (size_t)c + 8);
                    if (out.ref_beg[r] == 0 || cb < out.ref_beg[r]) out.ref_beg[r] = cb;
                    if (ce > out.ref_end[r]) out.ref_end[r] = ce;
                }
            }
            off += 16 * (size_t)n_chunk;
        }
        if (bins) {
            BaiBins& B = (*bins)[(size_t)r];
            std::sort(at.begin(), at.end());
            for (const auto& bo : at) {
                const int32_t n_chunk = rdi32(b.data() + bo.second);
                B.bin.push_back(bo.first);
                B.first.push_back((uint32_t)B.cb.size());
                for (int32_t c = 0; c < n_chunk; c++) {
                    B.cb.push_back(rd64(b.data() + bo.second + 4 + 16 * (size_t)c));
                    B.ce.push_back(rd64(b.data() + bo.second + 12 + 16 * (size_t)c));
                }
            }
            B.first.push_back((uint32_t)B.cb.size());
        }
        if (off + 4 > b.size()) return "truncated BAI: " + path;
        const int32_t n_intv = rdi32(b.data() + off); off += 4;
        if (n_intv < 0 || off + 8 * (size_t)n_intv > b.size()) return "truncated BAI: " + path;
        out.ioffsets[r].resize((size_t)n_intv);
        for (int32_t k = 0; k < n_intv; k++) out.ioffsets[r][k] = rd64(b.data() + off + 8 * (size_t)k);
        off += 8 * (size_t)n_intv;
    }
    out.n_no_coor = (off + 8 <= b.size()) ? rd64(b.data() + off) : 0;
    return "";
}

// a BGZF file (concatenated gzip members) inflated whole; false when a member is malformed or cut short
bool gunzip_all(const std::vector<uint8_t>& in, std::vector<uint8_t>& out) {
    z_stream zs;
    memset(&zs, 0, sizeof zs);
    if (inflateInit2(&zs, 15 + 16) != Z_OK) return false;
    zs.next_in = const_cast<Bytef*>(in.data());
    zs.avail_in = (uInt)in.size();
    uint8_t buf[1 << 16];
    bool ok = true;
    for (;;) {
        zs.next_out = buf;
        zs.avail_out = sizeof buf;
        const int rc = inflate(&zs, Z_NO_FLUSH);
        out.insert(out.end(), buf, buf + (sizeof buf - zs.avail_out));
        if (rc == Z_STREAM_END) {
            if (zs.avail_in == 0) break;
            if (inflateReset(&zs) != Z_OK) { ok = false; break; }
        } else if (rc != Z_OK) {                                           // Z_BUF_ERROR: the input ends inside a member
            ok = false;
            break;
        }
    }
    inflateEnd(&zs);
    return ok;
}

inline int64_t bin_first(int level) { return ((int64_t(1) << (3 * level)) - 1) / 7; }   // the first bin of a level (CSIv1)

// No BAM record starts at or past 2^31 (positions are int32): bins whose first base lies there take no part in the linear
// index, which keeps it at most 2^17 entries whatever the geometry.
constexpr int64_t kBamPosEnd = int64_t(1) << 31;

// The 16 KB linear index of one reference of a CSI, rebuilt from its bins' loffsets.  bots: (the bin's first tile at
// 2^min_shift granularity, its loffset) of every real bin with loffset != 0.
//   F[x] = the smallest loffset of the bins whose first tile is x; a tile no bin starts in takes the value of the nearest
//   known tile to its left, leading unknown tiles the first known value; F has max x + 1 entries.
//   min_shift <= 14: lin[t] = F[t << (14 - min_shift)], ceil(|F| / 2^(14 - min_shift)) entries;
//   min_shift >  14: lin[t] = F[t >> (min_shift - 14)], |F| << (min_shift - 14) entries (at most 2^17).
// Why this is safe: an indexer that follows htslib fills its 2^min_shift-tile linear index (every tile a record overlaps
// takes the first such record; gaps take the value on their left) and sets each bin's loffset to that index at the bin's
// first tile.  So F equals that filled index at every tile some bin starts in, and is never above it elsewhere, because the
// filled index does not decrease.  Every entry is therefore a record start at or before the first record that overlaps the
// tile: the host feeder, the device decode and the region planner may start there (and cut parse units there) without
// dropping a record.  With min_shift > 14 one wide tile's value stands for each 16 KB tile inside it: still such a bound.
std::vector<uint64_t> csi_linear(std::vector<std::pair<int64_t, uint64_t>>& bots, int min_shift) {
    std::vector<uint64_t> lin;
    if (bots.empty()) return lin;
    std::sort(bots.begin(), bots.end());
    size_t m = 0;
    for (size_t i = 0; i < bots.size(); i++)                          // one entry per tile: sorted, so the first is the smallest
        if (m == 0 || bots[i].first != bots[m - 1].first) bots[m++] = bots[i];
    bots.resize(m);
    const int64_t n_f = bots.back().first + 1;
    size_t j = 0;                                                      // F at increasing tiles x: a walk over bots
    auto F = [&](int64_t x) -> uint64_t {
        while (j + 1 < bots.size() && bots[j + 1].first <= x) j++;
        return bots[j].first <= x ? bots[j].second : bots[0].second;
    };
    if (min_shift <= 14) {
        const int s = 14 - min_shift;
        const int64_t n = (n_f + (int64_t(1) << s) - 1) >> s;
        lin.resize((size_t)n);
        for (int64_t t = 0; t < n; t++) lin[(size_t)t] = F(t << s);
    } else {
        const int d = min_shift - 14;
        const int64_t cap = kBamPosEnd >> 14;
        const int64_t n = d >= 17 ? cap : std::min<int64_t>(n_f << d, cap);
        lin.resize((size_t)n);
        for (int64_t t = 0; t < n; t++) lin[(size_t)t] = F(t >> d);
    }
    return lin;
}

// the CSIv1 layout, b inflated and starting with its magic:
//   "CSI\1" min_shift:i32 depth:i32 l_aux:i32 aux[l_aux] n_ref:i32
//   per ref: n_bin:i32, per bin: bin:u32 loffset:u64 n_chunk:i32 (beg:u64 end:u64)[n_chunk];  [n_no_coor:u64]
// The stats pseudo-bin ((1 << (3 depth + 3)) - 1) / 7 + 1 holds (ref_beg, ref_end), (mapped, unmapped), as BAI's 0x924a.
std::string csi_parse(const std::vector<uint8_t>& b, const std::string& path, BaiIndex& out, std::vector<BaiBins>* bins) {
    const std::string trunc = "truncated CSI: " + path, bad = "corrupt CSI: " + path;
    if (b.size() < 16 || memcmp(b.data(), "CSI\1", 4) != 0) return "not a BAI or CSI file: " + path;
    const int32_t min_shift = rdi32(b.data() + 4), depth = rdi32(b.data() + 8), l_aux = rdi32(b.data() + 12);
    // bin numbers up to the pseudo-bin fit 32 bits for depth <= 10, and the addressable range 2^(min_shift + 3 depth) an int64
    if (min_shift < 0 || depth < 0 || depth > 10 || min_shift + 3 * depth > 62)
        return "unsupported CSI geometry (min_shift " + std::to_string(min_shift) + ", depth " + std::to_string(depth) + "): " + path;
    if (l_aux < 0) return bad;
    size_t off = 16;
    if (off + (size_t)l_aux + 4 > b.size()) return trunc;
    off += (size_t)l_aux;                                              // a tabix header: read past, not used
    const int32_t n_ref = rdi32(b.data() + off); off += 4;
    if (n_ref < 0) return bad;
    out.min_shift = min_shift; out.depth = depth; out.is_csi = true;
    out.ioffsets.assign((size_t)n_ref, {});
    out.mapped.assign((size_t)n_ref, 0);
    out.unmapped.assign((size_t)n_ref, 0);
    out.has_stats.assign((size_t)n_ref, 0);
    out.ref_beg.assign((size_t)n_ref, 0);
    out.ref_end.assign((size_t)n_ref, 0);
    if (bins) bins->assign((size_t)n_ref, BaiBins());
    const int64_t n_real = bin_first(depth + 1);                      // bins 0 .. n_real - 1 are real
    const uint32_t stats_bin = (uint32_t)(n_real + 1);
    for (int32_t r = 0; r < n_ref; r++) {
        if (off + 4 > b.size()) return trunc;
        const int32_t n_bin = rdi32(b.data() + off); off += 4;
        if (n_bin < 0) return bad;
        std::vector<std::pair<uint32_t, size_t>> at;                   // (bin, offset of its chunk list) when bins are kept
        std::vector<std::pair<int64_t, uint64_t>> bots;
        for (int32_t k = 0; k < n_bin; k++) {
            if (off + 16 > b.size()) return trunc;
            const uint32_t bin = rd32(b.data() + off);
            const uint64_t loff = rd64(b.data() + off + 4);
            const int32_t n_chunk = rdi32(b.data() + off + 12);
            off += 16;
            if (n_chunk < 0 || off + 16 * (size_t)n_chunk > b.size()) return trunc;
            if (bin == stats_bin && n_chunk == 2) {
                out.mapped[r] = rd64(b.data() + off + 16);
                out.unmapped[r] = rd64(b.data() + off + 24);
                out.has_stats[r] = 1;
            } else if ((int64_t)bin < n_real) {
                if (bins) at.emplace_back(bin, off - 4);
                for (int32_t c = 0; c < n_chunk; c++) {
                    const uint64_t cb = rd64(b.data() + off + 16 * (size_t)c), ce = rd64(b.data() + off + 16 * (size_t)c + 8);
                    if (out.ref_beg[r] == 0 || cb < out.ref_beg[r]) out.ref_beg[r] = cb;
                    if (ce > out.ref_end[r]) out.ref_end[r] = ce;
                }
                int l = 0;
                while (l < depth && (int64_t)bin >= bin_first(l + 1)) l++;
                const int64_t bot = ((int64_t)bin - bin_first(l)) << (3 * (depth - l));
                if (loff != 0 && (bot << min_shift) < kBamPosEnd) bots.emplace_back(bot, loff);
            }                                                          // other ids (a pseudo-bin of another shape) are no bins
            off += 16 * (size_t)n_chunk;
        }
        if (bins) {
            BaiBins& B = (*bins)[(size_t)r];
            std::sort(at.begin(), at.end());
            for (const auto& bo : at) {
                const int32_t n_chunk = rdi32(b.data() + bo.second);
                B.bin.push_back(bo.first);
                B.first.push_back((uint32_t)B.cb.size());
                for (int32_t c = 0; c < n_chunk; c++) {
                    B.cb.push_back(rd64(b.data() + bo.second + 4 + 16 * (size_t)c));
                    B.ce.push_back(rd64(b.data() + bo.second + 12 + 16 * (size_t)c));
                }
            }
            B.first.push_back((uint32_t)B.cb.size());
        }
        out.ioffsets[r] = csi_linear(bots, min_shift);
    }
    out.n_no_coor = (off + 8 <= b.size()) ? rd64(b.data() + off) : 0;
    return "";
}

}  // namespace

std::string bai_read(const std::string& path, BaiIndex& out, std::vector<BaiBins>* bins) {
    FILE* f = fopen(path.c_str(), "rb");
    if (!f) return "cannot open " + path;
    std::vector<uint8_t> b;
    uint8_t tmp[1 << 16];
    size_t got;
    while ((got = fread(tmp, 1, sizeof tmp, f)) > 0) b.insert(b.end(), tmp, tmp + got);
    fclose(f);
    if (b.size() >= 8 && memcmp(b.data(), "BAI\1", 4) == 0) return bai_parse(b, path, out, bins);
    if (b.size() < 2 || b[0] != 0x1f || b[1] != 0x8b) return "not a BAI or CSI file: " + path;
    std::vector<uint8_t> raw;
    if (!gunzip_all(b, raw)) return "truncated or corrupt CSI: " + path;
    return csi_parse(raw, path, out, bins);
}

std::vector<std::string> index_candidates(const std::string& p) {
    const bool bam = p.size() > 4 && p.compare(p.size() - 4, 4, ".bam") == 0;
    const std::string stem = bam ? p.substr(0, p.size() - 4) : std::string();
    std::vector<std::string> c;
    c.push_back(p + ".bai");
    if (bam) c.push_back(stem + ".bai");
    c.push_back(p + ".csi");
    if (bam) c.push_back(stem + ".csi");
    return c;
}

void bai_region_chunks(const BaiBins& bins, const std::vector<uint64_t>& lin, int min_shift, int depth, const int64_t* beg,
                       const int64_t* end, int64_t n, std::vector<std::pair<uint64_t, uint64_t>>& out) {
    out.clear();
    // the bins cover [0, 2^(min_shift + 3 depth)) (BAI: 2^29); no BAM record starts at or past 2^31
    const int64_t kMax = std::min<int64_t>(int64_t(1) << (min_shift + 3 * depth), kBamPosEnd);
    const int64_t kBins = bin_first(depth + 1) + 1;                    // the stats pseudo-bin and up are not bins (BAI: 37450)
    const int64_t kLeaf = bin_first(depth);                            // the first leaf (BAI: 4681)
    auto find = [&](int64_t k) -> int64_t {                            // index of bin k with chunks, or -1
        const auto it = std::lower_bound(bins.bin.begin(), bins.bin.end(), (uint32_t)k);
        if (it == bins.bin.end() || *it != (uint32_t)k) return -1;
        const size_t j = (size_t)(it - bins.bin.begin());
        return bins.first[j + 1] > bins.first[j] ? (int64_t)j : -1;
    };
    // (bin, min_off, max_off) for every interval that names the bin; a bin keeps the loosest cut (smallest min_off,
    // largest max_off)
    struct Named { uint32_t bin; uint64_t lo, hi; };
    std::vector<Named> named;
    for (int64_t i = 0; i < n; i++) {
        const int64_t b = std::max<int64_t>(beg[i], 0), e = std::min<int64_t>(end[i], kMax);
        if (e <= b) continue;
        const uint64_t min_off = lin.empty() ? 0 : lin[(size_t)std::min<int64_t>(b >> 14, (int64_t)lin.size() - 1)];
        // max_off: the first chunk of the nearest bin with chunks to the right of the interval (its records start at or
        // after e, and so does every record after them); moving right, a first child goes up to its parent
        uint64_t max_off = UINT64_MAX;
        for (int64_t k = kLeaf + ((e - 1) >> min_shift) + 1;; k++) {
            if (k >= kBins) k = 0;
            while (k % 8 == 1) k = (k - 1) >> 3;
            if (k == 0) break;
            const int64_t j = find(k);
            if (j < 0) continue;
            max_off = *std::min_element(bins.cb.begin() + bins.first[(size_t)j], bins.cb.begin() + bins.first[(size_t)j + 1]);
            break;
        }
        for (int l = 0; l <= depth; l++) {                             // reg2bins: every level, the bins [b, e - 1] touches
            const int shift = min_shift + 3 * (depth - l);
            for (int64_t k = bin_first(l) + (b >> shift); k <= bin_first(l) + ((e - 1) >> shift); k++)
                named.push_back(Named{(uint32_t)k, min_off, max_off});
        }
    }
    std::sort(named.begin(), named.end(), [](const Named& x, const Named& y) { return x.bin < y.bin; });
    for (size_t a = 0; a < named.size();) {
        size_t z = a;
        uint64_t lo = UINT64_MAX, hi = 0;
        for (; z < named.size() && named[z].bin == named[a].bin; z++) { lo = std::min(lo, named[z].lo); hi = std::max(hi, named[z].hi); }
        const int64_t j = find(named[a].bin);
        a = z;
        if (j < 0) continue;
        for (uint32_t c = bins.first[(size_t)j]; c < bins.first[(size_t)j + 1]; c++)
            if (bins.ce[c] > lo && bins.cb[c] < hi && bins.ce[c] > bins.cb[c]) out.emplace_back(bins.cb[c], bins.ce[c]);
    }
    std::sort(out.begin(), out.end());
    size_t m = 0;
    for (size_t i = 0; i < out.size(); i++) {
        if (m > 0 && out[i].first <= out[m - 1].second) out[m - 1].second = std::max(out[m - 1].second, out[i].second);
        else out[m++] = out[i];
    }
    out.resize(m);
}

// ---------------------------------------------------------------------------------------------- CRAI
std::string crai_read(const std::string& path, std::vector<CraiSlices>& out) {
    gzFile f = gzopen(path.c_str(), "rb");
    if (!f) return "cannot open " + path;
    std::string text;
    char buf[1 << 16];
    int n;
    while ((n = gzread(f, buf, sizeof buf)) > 0) text.append(buf, (size_t)n);
    gzclose(f);
    size_t p = 0;
    int iline = 1;
    while (p < text.size()) {
        size_t e = text.find('\n', p);
        if (e == std::string::npos) break;                      // ReadString returns io.EOF: an unterminated last line is dropped
        std::string line = text.substr(p, e - p);
        p = e + 1;
        while (!line.empty() && isspace((unsigned char)line.back())) line.pop_back();
        size_t b = 0;
        while (b < line.size() && isspace((unsigned char)line[b])) b++;
        line = line.substr(b);
        long long v[6];
        int nf = 0;
        size_t q = 0;
        bool bad = false;
        while (true) {
            size_t t = line.find('\t', q);
            std::string tok = line.substr(q, t == std::string::npos ? std::string::npos : t - q);
            if (nf < 6) {
                char* endp = nullptr;
                v[nf] = strtoll(tok.c_str(), &endp, 10);
                if (tok.empty() || *endp) bad = true;
            }
            nf++;
            if (t == std::string::npos) break;
            q = t + 1;
        }
        if (nf != 6) return "crai: expected 6 fields in index, got " + std::to_string(nf) + " at line " + std::to_string(iline);
        if (bad) return "crai: unable to parse line " + std::to_string(iline);
        if (v[0] == -1) continue;                               // unmapped (crai.go:147-150)
        if (v[0] < 0) return "crai: bad seqID at line " + std::to_string(iline);
        if ((size_t)v[0] >= out.size()) out.resize((size_t)v[0] + 1);
        if (v[2] < 0) break;                                    // negative alnSpan: "breaking early" (crai.go:164-167)
        out[(size_t)v[0]].start.push_back(v[1]);
        out[(size_t)v[0]].span.push_back(v[2]);
        out[(size_t)v[0]].bytes.push_back((int32_t)v[5]);
        iline++;
    }
    return "";
}

bool crai_make_sizes(const int64_t* start_in, const int64_t* span_in, const int32_t* bytes, int64_t n, std::vector<int64_t>& sizes) {
    const int64_t TW = 16384;
    sizes.clear();
    int64_t last_start = 0, last_val = 0;
    for (int64_t s = 0; s < n; s++) {
        int64_t st = start_in[s], sp = span_in[s];
        bool first = true;
        while (last_start < st - TW) {                          // back-fill the gap before this slice
            sizes.push_back(first ? last_val : 0);
            if (first) last_val = 0;
            first = false;
            last_start += TW;
        }
        if (st - last_start > TW) return false;                 // "tilewidth logic error"
        while (st - last_start < -TW) { st += TW; sp -= TW; }   // a long read of the previous slice reached into this one
        if (sp <= 0) continue;
        const int64_t per_base = (int64_t)(100000 * (double)bytes[s] / (double)sp);
        const int64_t n_tiles = (int64_t)((double)sp / (double)TW);
        if (n_tiles == 0 && st - last_start < TW) { last_val = per_base; continue; }
        sizes.insert(sizes.end(), (size_t)n_tiles, per_base);
        const int64_t cmp = (st + sp) / TW;
        if ((int64_t)sizes.size() > cmp + 1 || cmp < (int64_t)sizes.size() - 1) return false;   // "logic error"
        last_start += TW * n_tiles;
        last_val = per_base;
    }
    return true;
}

// ---------------------------------------------------------------------------------------------- FAI
std::string fai_read(const std::string& path, std::vector<RefInfo>& out) {
    FILE* f = fopen(path.c_str(), "r");
    if (!f) return "cannot open " + path;
    char line[1 << 16];
    while (fgets(line, sizeof line, f)) {
        char* t1 = strchr(line, '\t');
        if (!t1) continue;
        RefInfo ri;
        ri.name.assign(line, (size_t)(t1 - line));
        ri.length = atoll(t1 + 1);
        long long off = 0, lb = 0, lw = 0;
        if (sscanf(t1 + 1, "%*d\t%lld\t%lld\t%lld", &off, &lb, &lw) == 3) { ri.offset = off; ri.line_bases = lb; ri.line_width = lw; }
        out.push_back(ri);
    }
    fclose(f);
    return "";
}

}  // namespace glhts
