// bamgpu.cu — the whole `samtools depth` child on the GPU: BGZF inflate (inflate.cu) + BAM record parse + the
// flag/MAPQ filter + CIGAR walk, for one reference sequence of an indexed BAM.  Only COMPRESSED bytes cross PCIe; the
// M/=/X blocks come out as int32 (start, end) arrays resident in HBM, in BAM order, and go straight into the depth kernels.
// Replaces the decode half of depth/depth.go:45,116,152 (and this library's host feeder, whose zlib inflate is the CLI's
// wall clock).
//
//   host      compressed byte range of the reference from the BAI (min chunk begin .. max chunk end), parallel pread into
//             pinned memory, a hop over the BGZF headers for the member table, the linear-index offsets as record-aligned
//             unit starts
//   K_inflate one warp per BGZF member (inflate.cu)
//   K_parse   one thread per unit (the records between two consecutive linear-index offsets): pass 1 counts the blocks of
//             the passing records, a scan places the units, pass 2 writes (start, end)
// Anything unexpected (a member the inflater rejects, a malformed record) makes the call return GL_ESTATE and the caller
// uses the host feeder for that reference.
#include "gl_common.cuh"
#include "ll_scan.cuh"
#include "host/bam_cigar.h"
#include "host/bam_feed.h"
#include "host/thread_pool.h"
#include <unistd.h>
#include <string.h>
#include <chrono>

extern "C" int gl_bgzf_inflate_device(gl_ctx* ctx, const uint8_t* d_comp, const int64_t* d_comp_off, const int64_t* d_out_off, int64_t n_blocks,
                                      uint8_t* d_out, int32_t* d_status);

namespace {

// a block [b0, b1) meets one of the n_iv merged, sorted intervals [iv_s[k], iv_e[k]) (n_iv < 0: no interval filter)
__device__ __forceinline__ bool meets_intervals(int b0, int b1, const int* __restrict__ iv_s, const int* __restrict__ iv_e, int n_iv) {
    if (n_iv < 0) return true;
    int lo = 0, hi = n_iv;                                             // the first interval ending after b0
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (iv_e[mid] > b0) hi = mid; else lo = mid + 1;
    }
    return lo < n_iv && iv_s[lo] < b1;
}

// one thread per unit: records in [unit_beg[u], unit_end[u]) of the inflated stream.  kEmit = false: count the M/=/X blocks
// of the passing records that meet the intervals; kEmit = true: write them at seg_off[u].  Filter and walk are
// glbam::depth_counts / depth_blocks, as on the host; both passes apply the same interval test, so they agree.
template <bool kEmit>
__global__ void __launch_bounds__(128) bam_parse_kernel(const unsigned char* __restrict__ data, const long long* __restrict__ unit_beg,
                                                       const long long* __restrict__ unit_end, int n_units, int tid_want, int min_mapq,
                                                       const int* __restrict__ iv_s, const int* __restrict__ iv_e, int n_iv,
                                                       long long* __restrict__ seg_cnt, const long long* __restrict__ seg_off,
                                                       int* __restrict__ start, int* __restrict__ end, unsigned long long* __restrict__ stats /* records, pass, maxlen, error */) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n_units) return;
    long long p = unit_beg[u];
    const long long pe = unit_end[u];
    long long n_seg = 0, out = kEmit ? seg_off[u] : 0;
    unsigned long long n_rec = 0, n_pass = 0;
    int maxlen = 0;
    bool bad = false;
    while (p + 36 <= pe) {
        const unsigned char* r = data + p + 4;
        const unsigned bs = glbam::ld_u32(data + p);
        if (bs < 32 || p + 4 + (long long)bs > pe) { bad = true; break; }       // corrupt size, or a record crossing a unit edge (the index lied)
        const int rtid = (int)glbam::ld_u32(r);
        p += 4 + (long long)bs;
        if (rtid != tid_want) { if (rtid > tid_want || rtid < 0) break; continue; }
        n_rec++;
        if (!glbam::depth_counts(r, bs, min_mapq)) continue;
        n_pass++;
        glbam::depth_blocks(r, bs, [&](int b0, int b1) {
            if (!meets_intervals(b0, b1, iv_s, iv_e, n_iv)) return;
            if (kEmit) { start[out] = b0; end[out] = b1; out++; }
            n_seg++;
            maxlen = max(maxlen, b1 - b0);
        });
    }
    if (!kEmit) {
        seg_cnt[u] = n_seg;
        if (n_rec) atomicAdd(stats + 0, n_rec);
        if (n_pass) atomicAdd(stats + 1, n_pass);
        if (maxlen) atomicMax(stats + 2, (unsigned long long)maxlen);
        if (bad) atomicAdd(stats + 3, 1ull);
    }
}

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

inline uint16_t rd16(const uint8_t* p) { return (uint16_t)(p[0] | (p[1] << 8)); }
inline uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }

using VRange = std::pair<uint64_t, uint64_t>;

// Members whose headers start within kGap compressed bytes of each other are read (and inflated) as one span: a gap that
// small costs less than another pread and another hop.
constexpr int64_t kGap = 65536;

// The body of both device decodes: the records of reference tid in the virtual-offset ranges (sorted, disjoint), parsed on
// the device.  iv_s / iv_e: the merged, sorted intervals a block must meet (filter = false: every block).
//   read   the members each range needs — from the one holding vb to the one holding the last byte before ve (ve on a member
//          start names a member that may not be needed: the range ends with the member before it) — as spans of nearby
//          members, parallel preads into pinned memory, then a hop over the BGZF headers that packs the members of the
//          set back to back (the member table); a member two ranges share is inflated once
//   units  each range is cut at the linear-index offsets inside it (record starts): one parse thread per unit
int decode_ranges(gl_ctx* ctx, glhts::BamFile& F, int32_t tid, const std::vector<VRange>& ranges, bool filter, const std::vector<int32_t>& iv_s,
                  const std::vector<int32_t>& iv_e, int32_t min_mapq, const int32_t** d_start, const int32_t** d_end, int64_t* n,
                  gl_bam_segments* stats, double t_wall, const char* who) {
    const std::vector<uint64_t>& lin = F.bai.ioffsets[(size_t)tid];
    // ---- member spans [a, b): a member whose header starts in one is read; spans closer than kGap are joined
    std::vector<std::pair<int64_t, int64_t>> spans;
    for (const VRange& r : ranges) {
        const int64_t a = (int64_t)(r.first >> 16), b = (int64_t)(r.second >> 16) + ((r.second & 0xffff) ? 1 : 0);
        if (b <= a || r.second <= r.first) continue;
        if (!spans.empty() && a <= spans.back().second + kGap) spans.back().second = std::max(spans.back().second, b);
        else spans.emplace_back(a, b);
    }
    if (spans.empty()) return GL_OK;
    // bytes [a, b - 1 + 65536 + 64) of each span hold its members (a member is at most 64 KB)
    std::vector<int64_t> span_len(spans.size()), span_at(spans.size() + 1, 0);
    for (size_t i = 0; i < spans.size(); i++) {
        span_len[i] = std::max<int64_t>(0, std::min<int64_t>(F.file_size(), spans[i].second - 1 + 65536 + 64) - spans[i].first);
        span_at[i + 1] = span_at[i] + span_len[i];
    }
    const size_t nbytes = (size_t)span_at.back();
    GL_CHECK(gl_pinned_reserve(ctx, nbytes + 256, nbytes + nbytes / 8 + (size_t(1) << 20)));
    uint8_t* h = static_cast<uint8_t*>(ctx->pack_pinned);
    {
        const int64_t piece = int64_t(8) << 20;
        std::vector<std::pair<size_t, int64_t>> jobs;                  // (span, offset in it)
        for (size_t i = 0; i < spans.size(); i++)
            for (int64_t o = 0; o < span_len[i]; o += piece) jobs.emplace_back(i, o);
        std::atomic<bool> bad(false);
        const int fd = F.fd();
        glhost::ThreadPool::global().run((int64_t)jobs.size(), [&](int64_t k, int) {
            const size_t i = jobs[(size_t)k].first;
            int64_t off = jobs[(size_t)k].second, left = std::min<int64_t>(piece, span_len[i] - off);
            while (left > 0) {
                const ssize_t got = pread(fd, h + span_at[i] + off, (size_t)left, spans[i].first + off);
                if (got <= 0) { bad = true; return; }
                off += got; left -= got;
            }
        });
        if (bad) return gl_fail(ctx, GL_ESTATE, "%s: read failed", who);
    }
    // ---- member table: the members of the set, packed back to back at the front of h
    std::vector<int64_t> comp_off(1, 0), out_off(1, 0), mem_file, mem_size;
    for (size_t i = 0; i < spans.size(); i++) {
        const size_t len = (size_t)span_len[i];
        const uint8_t* s = h + span_at[i];
        size_t q = 0;
        while (q + 18 <= len && spans[i].first + (int64_t)q < spans[i].second) {
            if (s[q] != 0x1f || s[q + 1] != 0x8b || s[q + 2] != 8 || !(s[q + 3] & 4) || s[q + 12] != 'B' || s[q + 13] != 'C')
                return gl_fail(ctx, GL_ESTATE, "%s: unexpected BGZF header layout", who);
            const size_t bs = (size_t)rd16(s + q + 16) + 1;
            if (q + bs > len) break;
            const uint32_t isize = rd32(s + q + bs - 4);
            if (isize > 65536) return gl_fail(ctx, GL_ESTATE, "%s: bad ISIZE", who);
            uint8_t* dst = h + comp_off.back();
            if (dst != s + q) memmove(dst, s + q, bs);                  // dst <= s + q: the packed table never overtakes the hop
            mem_file.push_back(spans[i].first + (int64_t)q);
            mem_size.push_back((int64_t)bs);
            comp_off.push_back(comp_off.back() + (int64_t)bs);
            out_off.push_back(out_off.back() + isize);
            q += bs;
        }
    }
    const int64_t n_blocks = (int64_t)comp_off.size() - 1;
    if (n_blocks == 0) return GL_OK;
    const int64_t inflated = out_off.back();
    // virtual offset -> position in the inflated stream of the set.  at_end: v ends a range, so a v on a member start is the
    // end of the member before it, which must be in the set and end where v's member begins.
    auto stream_pos = [&](uint64_t v, bool at_end) -> int64_t {
        const int64_t c = (int64_t)(v >> 16), w = (int64_t)(v & 0xffff);
        if (at_end && w == 0) {
            const auto it = std::lower_bound(mem_file.begin(), mem_file.end(), c);
            if (it == mem_file.begin()) return -1;
            const size_t m = (size_t)(it - mem_file.begin()) - 1;
            return mem_file[m] + mem_size[m] == c ? out_off[m + 1] : -1;
        }
        const auto it = std::lower_bound(mem_file.begin(), mem_file.end(), c);
        if (it == mem_file.end() || *it != c) return -1;
        const size_t m = (size_t)(it - mem_file.begin());
        return w <= out_off[m + 1] - out_off[m] ? out_off[m] + w : -1;
    };
    // ---- units: each range from vb to ve, cut at the distinct linear-index offsets inside it (record-aligned)
    std::vector<int64_t> unit_beg, unit_end;
    for (const VRange& r : ranges) {
        if (r.second <= r.first) continue;
        const int64_t p0 = stream_pos(r.first, false), p1 = stream_pos(r.second, true);
        if (p0 < 0 || p1 < 0 || p1 < p0 || p1 > inflated) return gl_fail(ctx, GL_ESTATE, "%s: index offsets do not land on members", who);
        std::vector<int64_t> cut(1, p0);
        uint64_t prev = r.first;
        for (auto it = std::upper_bound(lin.begin(), lin.end(), r.first); it != lin.end() && *it < r.second; ++it) {
            const uint64_t v = *it;
            if (v <= prev) continue;
            const int64_t p = stream_pos(v, false);
            if (p < 0) return gl_fail(ctx, GL_ESTATE, "%s: index offsets do not land on members", who);
            if (p > cut.back()) cut.push_back(p);
            prev = v;
        }
        if (p1 > cut.back()) cut.push_back(p1); else cut.back() = p1;
        for (size_t k = 0; k + 1 < cut.size(); k++) { unit_beg.push_back(cut[k]); unit_end.push_back(cut[k + 1]); }
    }
    if (unit_beg.empty()) return GL_OK;
    const int n_units = (int)unit_beg.size();
    const int n_iv = filter ? (int)iv_s.size() : -1;
    // ---- device buffers (ctx-owned, grow-only): compressed | tables | inflated | unit tables | intervals | segments
    auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
    const size_t n_ivs = filter ? iv_s.size() : 0;
    const size_t used = (size_t)comp_off.back();
    const size_t tab_bytes = al((size_t)(n_blocks + 1) * 8) * 2 + al((size_t)n_blocks * 4) + al((size_t)(n_units + 2) * 8) * 4 +
                             al(n_ivs * 4 + 4) * 2 + al(64);
    GL_CHECK(gl_buf_reserve(ctx, ctx->bam_comp, al(used) + tab_bytes));
    GL_CHECK(gl_buf_reserve(ctx, ctx->bam_out, (size_t)inflated + 256));
    char* dbase = static_cast<char*>(ctx->bam_comp.p);
    uint8_t* d_comp = reinterpret_cast<uint8_t*>(dbase);
    char* q = dbase + al(used);
    int64_t* d_coff = reinterpret_cast<int64_t*>(q); q += al((size_t)(n_blocks + 1) * 8);
    int64_t* d_ooff = reinterpret_cast<int64_t*>(q); q += al((size_t)(n_blocks + 1) * 8);
    int32_t* d_stat = reinterpret_cast<int32_t*>(q); q += al((size_t)n_blocks * 4);
    long long* d_ubeg = reinterpret_cast<long long*>(q); q += al((size_t)(n_units + 2) * 8);
    long long* d_uend = reinterpret_cast<long long*>(q); q += al((size_t)(n_units + 2) * 8);
    long long* d_cnt = reinterpret_cast<long long*>(q); q += al((size_t)(n_units + 2) * 8);
    long long* d_off = reinterpret_cast<long long*>(q); q += al((size_t)(n_units + 2) * 8);
    int32_t* d_ivs = reinterpret_cast<int32_t*>(q); q += al(n_ivs * 4 + 4);
    int32_t* d_ive = reinterpret_cast<int32_t*>(q); q += al(n_ivs * 4 + 4);
    unsigned long long* d_stats = reinterpret_cast<unsigned long long*>(q);
    GL_CUDA(ctx, cudaMemcpyAsync(d_comp, h, used, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(d_coff, comp_off.data(), (size_t)(n_blocks + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(d_ooff, out_off.data(), (size_t)(n_blocks + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(d_ubeg, unit_beg.data(), (size_t)n_units * 8, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(d_uend, unit_end.data(), (size_t)n_units * 8, cudaMemcpyHostToDevice, ctx->stream));
    if (n_ivs) {
        GL_CUDA(ctx, cudaMemcpyAsync(d_ivs, iv_s.data(), n_ivs * 4, cudaMemcpyHostToDevice, ctx->stream));
        GL_CUDA(ctx, cudaMemcpyAsync(d_ive, iv_e.data(), n_ivs * 4, cudaMemcpyHostToDevice, ctx->stream));
    }
    GL_CUDA(ctx, cudaMemsetAsync(d_stats, 0, 64, ctx->stream));
    cudaEvent_t ev[4];
    for (auto& e : ev) GL_CUDA(ctx, cudaEventCreate(&e));
    GL_CUDA(ctx, cudaEventRecord(ev[0], ctx->stream));
    GL_CHECK(gl_bgzf_inflate_device(ctx, d_comp, d_coff, d_ooff, n_blocks, static_cast<uint8_t*>(ctx->bam_out.p), d_stat));
    GL_CUDA(ctx, cudaEventRecord(ev[1], ctx->stream));
    {
        gl_prof_scope prof(ctx, "bam_parse_count_kernel");
        bam_parse_kernel<false><<<(unsigned)((n_units + 127) / 128), 128, 0, ctx->stream>>>(static_cast<const unsigned char*>(ctx->bam_out.p), d_ubeg, d_uend,
                                                                                          n_units, tid, min_mapq, d_ivs, d_ive, n_iv, d_cnt, nullptr,
                                                                                          nullptr, nullptr, d_stats);
        GL_LAUNCHED(ctx, 1);
    }
    ll_scan_kernel<<<1, 1024, 0, ctx->stream>>>(d_cnt, d_off, n_units);
    GL_LAUNCHED(ctx, 1);
    unsigned long long hst[4] = {0, 0, 0, 0};
    long long total = 0;
    std::vector<int32_t> st_host((size_t)n_blocks);
    GL_CUDA(ctx, cudaMemcpyAsync(hst, d_stats, 32, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(&total, d_off + n_units, 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(st_host.data(), d_stat, (size_t)n_blocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int32_t sb : st_host) if (sb != 0) { for (auto& e : ev) cudaEventDestroy(e); return gl_fail(ctx, GL_ESTATE, "%s: a BGZF member was rejected by the device inflater (status %d)", who, sb); }
    if (hst[3] != 0) { for (auto& e : ev) cudaEventDestroy(e); return gl_fail(ctx, GL_ESTATE, "%s: malformed BAM record", who); }
    GL_CHECK(gl_buf_reserve(ctx, ctx->bam_seg, al((size_t)std::max<long long>(total, 1) * 4) * 2));
    int32_t* ds = static_cast<int32_t*>(ctx->bam_seg.p);
    int32_t* de = reinterpret_cast<int32_t*>(static_cast<char*>(ctx->bam_seg.p) + al((size_t)std::max<long long>(total, 1) * 4));
    GL_CUDA(ctx, cudaEventRecord(ev[2], ctx->stream));
    if (total > 0) {
        gl_prof_scope prof(ctx, "bam_parse_emit_kernel");
        bam_parse_kernel<true><<<(unsigned)((n_units + 127) / 128), 128, 0, ctx->stream>>>(static_cast<const unsigned char*>(ctx->bam_out.p), d_ubeg, d_uend,
                                                                                         n_units, tid, min_mapq, d_ivs, d_ive, n_iv, nullptr, d_off,
                                                                                         ds, de, d_stats);
        GL_LAUNCHED(ctx, 1);
    }
    GL_CUDA(ctx, cudaEventRecord(ev[3], ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    float ms_inf = 0, ms_p1 = 0, ms_p2 = 0;
    cudaEventElapsedTime(&ms_inf, ev[0], ev[1]);
    cudaEventElapsedTime(&ms_p1, ev[1], ev[2]);
    cudaEventElapsedTime(&ms_p2, ev[2], ev[3]);
    for (auto& e : ev) cudaEventDestroy(e);
    *d_start = ds; *d_end = de; *n = total;
    if (stats) {
        stats->format = 32; stats->units = n_units; stats->max_len = (int32_t)hst[2]; stats->n = total;
        stats->n_records = (int64_t)hst[0]; stats->n_pass = (int64_t)hst[1];
        stats->bytes_in = (int64_t)used; stats->bytes_out = inflated;
        stats->inflate_s = ms_inf * 1e-3; stats->parse_s = (ms_p1 + ms_p2) * 1e-3; stats->wall_s = now_s() - t_wall;
    }
    return GL_OK;
}

// the index's virtual-offset range of reference tid's records: GL_OK with *has = false when it has none
int ref_range(gl_ctx* ctx, const glhts::BamFile& F, int32_t tid, VRange& r, bool& has, const char* who) {
    const std::vector<uint64_t>& lin = F.bai.ioffsets[(size_t)tid];
    r.first = tid < (int)F.bai.ref_beg.size() ? F.bai.ref_beg[(size_t)tid] : 0;
    r.second = tid < (int)F.bai.ref_end.size() ? F.bai.ref_end[(size_t)tid] : 0;
    has = false;
    if (r.first == 0 || r.second <= r.first) {
        for (uint64_t v : lin) if (v) return gl_fail(ctx, GL_ESTATE, "%s: the index has no chunk range for this reference", who);
        return GL_OK;
    }
    has = true;
    return GL_OK;
}

}  // namespace

extern "C" {

// The segments of reference `tid` (whole reference) decoded on the device.  On success *d_start / *d_end point into
// ctx-owned device memory (valid until the next gl_bam_decode_device on this ctx) and hold *n segments in BAM order;
// stats (may be NULL): same fields as gl_bam_decode (inflate_s = device time of K_inflate, parse_s = of the two K_parse
// passes).  GL_ESTATE: this reference cannot be done on the device (no index, a member the inflater rejects, ...): use
// gl_bam_decode.
int gl_bam_decode_device(gl_ctx* ctx, gl_bam* b, int32_t tid, int32_t min_mapq, const int32_t** d_start, const int32_t** d_end, int64_t* n,
                         gl_bam_segments* stats) {
    GL_CHECK(gl_use(ctx));
    if (!b || !d_start || !d_end || !n) return gl_fail(ctx, GL_EINVAL, "gl_bam_decode_device: null argument");
    *d_start = *d_end = nullptr; *n = 0;
    if (stats) memset(stats, 0, sizeof *stats);
    const double t_wall = now_s();
    glhts::BamFile& F = b->f;
    if (!F.has_index || F.fd() < 0) return gl_fail(ctx, GL_ESTATE, "gl_bam_decode_device: no index");
    if (tid < 0 || tid >= (int)F.header.refs.size() || tid >= (int)F.bai.ioffsets.size()) return GL_OK;
    VRange whole;
    bool has = false;
    GL_CHECK(ref_range(ctx, F, tid, whole, has, "gl_bam_decode_device"));
    if (!has) return GL_OK;
    static const std::vector<int32_t> none;
    return decode_ranges(ctx, F, tid, {whole}, false, none, none, min_mapq, d_start, d_end, n, stats, t_wall, "gl_bam_decode_device");
}

// The segments of reference `tid` whose blocks meet the intervals [beg[i], end[i]), decoded on the device from the
// members the index's bin query names (include/goleft_b200.h).
int gl_bam_decode_device_regions(gl_ctx* ctx, gl_bam* b, int32_t tid, const int64_t* beg, const int64_t* end, int64_t n,
                                 int32_t min_mapq, const int32_t** d_start, const int32_t** d_end, int64_t* n_seg,
                                 gl_bam_segments* stats) {
    const char* who = "gl_bam_decode_device_regions";
    GL_CHECK(gl_use(ctx));
    if (!b || !d_start || !d_end || !n_seg || n < 0 || (n > 0 && (!beg || !end))) return gl_fail(ctx, GL_EINVAL, "%s: bad argument", who);
    *d_start = *d_end = nullptr; *n_seg = 0;
    if (stats) memset(stats, 0, sizeof *stats);
    const double t_wall = now_s();
    glhts::BamFile& F = b->f;
    if (!F.has_index || F.fd() < 0) return gl_fail(ctx, GL_ESTATE, "%s: no index", who);
    if (tid < 0 || tid >= (int)F.header.refs.size()) return gl_fail(ctx, GL_EINVAL, "%s: tid %d is not in the header", who, tid);
    if (tid >= (int)F.bai.ioffsets.size()) return GL_OK;
    // the intervals as the blocks see them (int32 coordinates), merged and sorted
    std::vector<std::pair<int64_t, int64_t>> iv;
    for (int64_t i = 0; i < n; i++) {
        const int64_t s = std::max<int64_t>(beg[i], 0), e = std::min<int64_t>(end[i], INT32_MAX);
        if (e > s) iv.emplace_back(s, e);
    }
    if (iv.empty()) return GL_OK;
    std::sort(iv.begin(), iv.end());
    std::vector<int32_t> iv_s, iv_e;
    for (const auto& x : iv) {
        if (!iv_e.empty() && x.first <= iv_e.back()) iv_e.back() = std::max<int32_t>(iv_e.back(), (int32_t)x.second);
        else { iv_s.push_back((int32_t)x.first); iv_e.push_back((int32_t)x.second); }
    }
    VRange whole;
    bool has = false;
    GL_CHECK(ref_range(ctx, F, tid, whole, has, who));
    if (!has) return GL_OK;
    std::vector<VRange> ranges;
    const std::vector<int64_t> pb(iv_s.begin(), iv_s.end()), pe(iv_e.begin(), iv_e.end());
    if (!gl_bam_plan_regions(*b, tid, pb.data(), pe.data(), (int64_t)pb.size(), ranges).empty())
        return gl_fail(ctx, GL_ESTATE, "%s: cannot read the index's bins", who);
    if (ranges.empty()) return GL_OK;
    int64_t covered = 0;                                               // compressed bytes the ranges span
    for (const VRange& r : ranges) covered += (int64_t)(r.second >> 16) - (int64_t)(r.first >> 16);
    if (2 * covered >= (int64_t)(whole.second >> 16) - (int64_t)(whole.first >> 16)) ranges.assign(1, whole);
    return decode_ranges(ctx, F, tid, ranges, true, iv_s, iv_e, min_mapq, d_start, d_end, n_seg, stats, t_wall, who);
}

}  // extern "C"
