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

// one thread per unit: records in [unit_pos[u], unit_pos[u+1]) of the inflated stream.  kEmit = false: count the M/=/X blocks of
// the passing records; kEmit = true: write them at seg_off[u].  Filter and walk are glbam::depth_counts / depth_blocks, as
// on the host.
template <bool kEmit>
__global__ void __launch_bounds__(128) bam_parse_kernel(const unsigned char* __restrict__ data, const long long* __restrict__ unit_pos, int n_units,
                                                       int tid_want, int min_mapq, long long* __restrict__ seg_cnt, const long long* __restrict__ seg_off,
                                                       int* __restrict__ start, int* __restrict__ end, unsigned long long* __restrict__ stats /* records, pass, maxlen, error */) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n_units) return;
    long long p = unit_pos[u];
    const long long pe = unit_pos[u + 1];
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
    const std::vector<uint64_t>& lin = F.bai.ioffsets[(size_t)tid];
    const uint64_t vbeg = tid < (int)F.bai.ref_beg.size() ? F.bai.ref_beg[(size_t)tid] : 0;
    const uint64_t vend = tid < (int)F.bai.ref_end.size() ? F.bai.ref_end[(size_t)tid] : 0;
    if (vbeg == 0 || vend <= vbeg) {
        if (lin.empty()) return GL_OK;
        bool any = false;
        for (uint64_t v : lin) if (v) { any = true; break; }
        if (!any) return GL_OK;
        return gl_fail(ctx, GL_ESTATE, "gl_bam_decode_device: the index has no chunk range for this reference");
    }
    // ---- compressed bytes [c0, c1): from the member holding the first record to the end of the member holding the last
    const int64_t c0 = (int64_t)(vbeg >> 16);
    int64_t c1 = std::min<int64_t>(F.file_size(), (int64_t)(vend >> 16) + 65536 + 64);
    const size_t nbytes = (size_t)(c1 - c0);
    GL_CHECK(gl_pinned_reserve(ctx, nbytes + 256, nbytes + nbytes / 8 + (size_t(1) << 20)));
    uint8_t* h = static_cast<uint8_t*>(ctx->pack_pinned);
    const double t_read = now_s();
    {
        const int64_t piece = int64_t(8) << 20;
        const int64_t n_pieces = ((int64_t)nbytes + piece - 1) / piece;
        std::atomic<bool> bad(false);
        const int fd = F.fd();
        glhost::ThreadPool::global().run(n_pieces, [&](int64_t k, int) {
            int64_t off = k * piece, left = std::min<int64_t>(piece, (int64_t)nbytes - off);
            while (left > 0) {
                const ssize_t got = pread(fd, h + off, (size_t)left, c0 + off);
                if (got <= 0) { bad = true; return; }
                off += got; left -= got;
            }
        });
        if (bad) return gl_fail(ctx, GL_ESTATE, "gl_bam_decode_device: read failed");
    }
    const double read_s = now_s() - t_read;
    // ---- member table (a hop over the headers), stopping after the member that holds the last record
    std::vector<int64_t> comp_off(1, 0), out_off(1, 0);
    {
        const int64_t last_c = (int64_t)(vend >> 16) - c0;
        size_t q = 0;
        while (q + 18 <= nbytes) {
            if (h[q] != 0x1f || h[q + 1] != 0x8b || h[q + 2] != 8 || !(h[q + 3] & 4) || h[q + 12] != 'B' || h[q + 13] != 'C')
                return gl_fail(ctx, GL_ESTATE, "gl_bam_decode_device: unexpected BGZF header layout");
            const size_t bs = (size_t)rd16(h + q + 16) + 1;
            if (q + bs > nbytes) break;
            const uint32_t isize = rd32(h + q + bs - 4);
            if (isize > 65536) return gl_fail(ctx, GL_ESTATE, "gl_bam_decode_device: bad ISIZE");
            const bool is_last = (int64_t)q >= last_c;
            q += bs;
            comp_off.push_back((int64_t)q);
            out_off.push_back(out_off.back() + isize);
            if (is_last) break;
        }
    }
    const int64_t n_blocks = (int64_t)comp_off.size() - 1;
    if (n_blocks == 0) return GL_OK;
    const int64_t inflated = out_off.back();
    auto stream_pos = [&](uint64_t v) -> int64_t {                     // virtual offset -> position in the inflated stream of this range
        const int64_t c = (int64_t)(v >> 16) - c0;
        const auto it = std::lower_bound(comp_off.begin(), comp_off.end(), c);
        if (it == comp_off.end() || *it != c) return -1;
        const size_t blk = (size_t)(it - comp_off.begin());
        if (blk >= (size_t)n_blocks) return (v & 0xffff) == 0 ? inflated : -1;
        return out_off[blk] + (int64_t)(v & 0xffff);
    };
    // ---- units: the distinct linear-index offsets inside the range are record-aligned
    std::vector<int64_t> unit_pos;
    {
        const int64_t p0 = stream_pos(vbeg), p1 = stream_pos(vend);
        if (p0 < 0 || p1 < 0 || p1 < p0 || p1 > inflated) return gl_fail(ctx, GL_ESTATE, "gl_bam_decode_device: index offsets do not land on members");
        unit_pos.push_back(p0);
        uint64_t prev = vbeg;
        for (uint64_t v : lin) {
            if (v <= prev || v >= vend) continue;
            const int64_t p = stream_pos(v);
            if (p < 0) return gl_fail(ctx, GL_ESTATE, "gl_bam_decode_device: index offsets do not land on members");
            if (p > unit_pos.back()) unit_pos.push_back(p);
            prev = v;
        }
        if (p1 > unit_pos.back()) unit_pos.push_back(p1); else unit_pos.back() = p1;
        if (unit_pos.size() < 2) return GL_OK;
    }
    const int n_units = (int)unit_pos.size() - 1;
    // ---- device buffers (ctx-owned, grow-only): compressed | tables | inflated | unit tables | segments
    auto al = [](size_t x) { return (x + 255) & ~size_t(255); };
    const size_t tab_bytes = al((size_t)(n_blocks + 1) * 8) * 2 + al((size_t)n_blocks * 4) + al((size_t)(n_units + 2) * 8) * 3 + al(64);
    GL_CHECK(gl_buf_reserve(ctx, ctx->bam_comp, al(nbytes) + tab_bytes));
    GL_CHECK(gl_buf_reserve(ctx, ctx->bam_out, (size_t)inflated + 256));
    char* dbase = static_cast<char*>(ctx->bam_comp.p);
    uint8_t* d_comp = reinterpret_cast<uint8_t*>(dbase);
    char* q = dbase + al(nbytes);
    int64_t* d_coff = reinterpret_cast<int64_t*>(q); q += al((size_t)(n_blocks + 1) * 8);
    int64_t* d_ooff = reinterpret_cast<int64_t*>(q); q += al((size_t)(n_blocks + 1) * 8);
    int32_t* d_stat = reinterpret_cast<int32_t*>(q); q += al((size_t)n_blocks * 4);
    long long* d_upos = reinterpret_cast<long long*>(q); q += al((size_t)(n_units + 2) * 8);
    long long* d_cnt = reinterpret_cast<long long*>(q); q += al((size_t)(n_units + 2) * 8);
    long long* d_off = reinterpret_cast<long long*>(q); q += al((size_t)(n_units + 2) * 8);
    unsigned long long* d_stats = reinterpret_cast<unsigned long long*>(q);
    const size_t used = (size_t)comp_off.back();
    GL_CUDA(ctx, cudaMemcpyAsync(d_comp, h, used, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(d_coff, comp_off.data(), (size_t)(n_blocks + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(d_ooff, out_off.data(), (size_t)(n_blocks + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(d_upos, unit_pos.data(), (size_t)(n_units + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(d_stats, 0, 64, ctx->stream));
    cudaEvent_t ev[4];
    for (auto& e : ev) GL_CUDA(ctx, cudaEventCreate(&e));
    GL_CUDA(ctx, cudaEventRecord(ev[0], ctx->stream));
    GL_CHECK(gl_bgzf_inflate_device(ctx, d_comp, d_coff, d_ooff, n_blocks, static_cast<uint8_t*>(ctx->bam_out.p), d_stat));
    GL_CUDA(ctx, cudaEventRecord(ev[1], ctx->stream));
    {
        gl_prof_scope prof(ctx, "bam_parse_count_kernel");
        bam_parse_kernel<false><<<(unsigned)((n_units + 127) / 128), 128, 0, ctx->stream>>>(static_cast<const unsigned char*>(ctx->bam_out.p), d_upos, n_units, tid,
                                                                                          min_mapq, d_cnt, nullptr, nullptr, nullptr, d_stats);
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
    for (int32_t sb : st_host) if (sb != 0) { for (auto& e : ev) cudaEventDestroy(e); return gl_fail(ctx, GL_ESTATE, "gl_bam_decode_device: a BGZF member was rejected by the device inflater (status %d)", sb); }
    if (hst[3] != 0) { for (auto& e : ev) cudaEventDestroy(e); return gl_fail(ctx, GL_ESTATE, "gl_bam_decode_device: malformed BAM record"); }
    GL_CHECK(gl_buf_reserve(ctx, ctx->bam_seg, al((size_t)std::max<long long>(total, 1) * 4) * 2));
    int32_t* ds = static_cast<int32_t*>(ctx->bam_seg.p);
    int32_t* de = reinterpret_cast<int32_t*>(static_cast<char*>(ctx->bam_seg.p) + al((size_t)std::max<long long>(total, 1) * 4));
    GL_CUDA(ctx, cudaEventRecord(ev[2], ctx->stream));
    if (total > 0) {
        gl_prof_scope prof(ctx, "bam_parse_emit_kernel");
        bam_parse_kernel<true><<<(unsigned)((n_units + 127) / 128), 128, 0, ctx->stream>>>(static_cast<const unsigned char*>(ctx->bam_out.p), d_upos, n_units, tid,
                                                                                         min_mapq, nullptr, d_off, ds, de, d_stats);
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
        (void)read_s;
    }
    return GL_OK;
}

}  // extern "C"
