// multidepth.cu — `goleft multidepth` (multidepth/multidepth.go) on sm_90a: S samples of one contig -> blocks of sufficient
// coverage with every sample's mean depth.
//
// Pass 1 (count), per sample: the sample's segments go through the depth tile core (depth.cu, any of its paths) with the
//   count epilogue, which writes the sample's (d >= MinCov) and (d > 0) bits; K_md_accum adds them into a per-base uint16
//   counter and ORs them into a per-base site bit.  O(L) state whatever S is; per-base depth never reaches HBM.
// Sites: K_md_classify marks the sufficient sites (site and counter > minSamples), K_md_runs_count / K_md_scan /
//   K_md_runs_write emit the runs of the site classes (absent / insufficient / sufficient) in position order: per 8192-base
//   CTA a count, one exclusive scan over the CTAs, then every CTA writes its runs at its offset.
// Blocks: on the host (host/multidepth.cpp, gl_multidepth_blocks) from the class runs.
// Pass 2 (means), per sample: the tile core's sum epilogue writes, for every (tile, block) pair, Σ d over the block's
//   sufficient sites per 512-base chunk; K_md_pair_sums adds them up per block (exact, int64), K_md_certify decides per cell
//   whether the "%.2f" digits follow from the integers (host/md_cert.h).  Cells it cannot certify (ties among them) take the
//   literal float64 chain of the reference in K_md_walk, over the sample's per-base depth materialised in scratch.
#include "gl_common.cuh"
#include "host/md_cert.h"
#include <string.h>

namespace {

constexpr int kTileBases = 4096;                 // the depth tile core's tile
constexpr int kRunThreads = 256;                 // K_md_runs_*: one 32-base word per thread, 8192 bases per CTA

struct MdState {
    int64_t L = 0, words = 0, tiles = 0;         // contig length, 32-base words and 4096-base tiles covering it
    int32_t S = 0, mincov = 0;
    int64_t min_samples = 0;
    int32_t counted = 0, summed = 0;
    bool sites_done = false;
    int64_t n_runs = 0;
    gl_buf ge, pos, cnt, site, suf, depth, run_s, run_c, cta_cnt, small;
    // blocks
    int64_t nb = 0, n_pairs = 0;
    gl_buf blk, pair_ptr, pair_blk, slots, tmp, sums, q, val, cert, walk_list;
    int64_t walked = 0, certified = 0;
    bool blocks_set = false;
};

MdState* st(gl_ctx* ctx) { return static_cast<MdState*>(ctx->md); }

void md_buf_free(gl_buf& b) {
    if (b.p) cudaFree(b.p);
    b.p = nullptr;
    b.cap = 0;
}

// ------------------------------------------------------------------------------------------------ pass 1
// one 32-base word per thread: site |= pos; cnt[x] += ge bit of x
__global__ void __launch_bounds__(256) md_accum_kernel(const unsigned* __restrict__ ge, const unsigned* __restrict__ pos,
                                                       unsigned short* __restrict__ cnt, unsigned* __restrict__ site, long long words) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= words) return;
    const unsigned g = ge[w], p = pos[w];
    if (p) site[w] |= p;
    if (!g) return;
    uint4* c4 = reinterpret_cast<uint4*>(cnt + w * 32);
#pragma unroll
    for (int j = 0; j < 4; j++) {
        uint4 v = c4[j];
        unsigned* u = reinterpret_cast<unsigned*>(&v);
#pragma unroll
        for (int h = 0; h < 4; h++) {
            const int k = 8 * j + 2 * h;
            u[h] += ((g >> k) & 1u) | (((g >> (k + 1)) & 1u) << 16);   // two uint16 counters per word, < 65536: no carry
        }
        c4[j] = v;
    }
}

// sufficient bit of x = site(x) and cnt[x] > minSamples
__global__ void __launch_bounds__(256) md_classify_kernel(const unsigned short* __restrict__ cnt, const unsigned* __restrict__ site,
                                                          unsigned* __restrict__ suf, long long words, int min_samples) {
    const long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= words) return;
    const unsigned s = site[w];
    unsigned m = 0;
    if (s) {
        const uint4* c4 = reinterpret_cast<const uint4*>(cnt + w * 32);
#pragma unroll
        for (int j = 0; j < 4; j++) {
            const uint4 v = c4[j];
            const unsigned u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int h = 0; h < 4; h++) {
                const int k = 8 * j + 2 * h;
                m |= ((int)(u[h] & 0xffffu) > min_samples ? 1u : 0u) << k;
                m |= ((int)(u[h] >> 16) > min_samples ? 1u : 0u) << (k + 1);
            }
        }
        m &= s;
    }
    suf[w] = m;
}

// run starts of word w: bases whose (site, sufficient) pair differs from the base before (base 0 always starts a run)
__device__ __forceinline__ unsigned md_run_mask(const unsigned* site, const unsigned* suf, long long w, long long L) {
    const unsigned s = site[w], f = suf[w];
    const unsigned ps = (s << 1) | (w > 0 ? site[w - 1] >> 31 : 0u);
    const unsigned pf = (f << 1) | (w > 0 ? suf[w - 1] >> 31 : 0u);
    unsigned m = (s ^ ps) | (f ^ pf);
    if (w == 0) m |= 1u;
    const long long rem = L - w * 32;                         // bases of this word inside the contig
    if (rem < 32) m &= rem <= 0 ? 0u : ((1u << rem) - 1u);
    return m;
}

__global__ void __launch_bounds__(kRunThreads) md_runs_count_kernel(const unsigned* __restrict__ site, const unsigned* __restrict__ suf,
                                                                    long long words, long long L, unsigned* __restrict__ cta_cnt) {
    const long long w = (long long)blockIdx.x * kRunThreads + threadIdx.x;
    const int c = w < words ? __popc(md_run_mask(site, suf, w, L)) : 0;
    __shared__ int s_part[kRunThreads / 32];
    const int v = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int k = 0; k < kRunThreads / 32; k++) t += s_part[k];
        cta_cnt[blockIdx.x] = (unsigned)t;
    }
}

// one CTA: exclusive scan of the per-CTA counts in place, total -> *total
__global__ void __launch_bounds__(1024) md_scan_kernel(unsigned* __restrict__ cnt, long long n, unsigned long long* __restrict__ total) {
    __shared__ unsigned long long s_w[32];
    __shared__ unsigned long long s_base;
    if (threadIdx.x == 0) s_base = 0;
    __syncthreads();
    for (long long b0 = 0; b0 < n; b0 += 1024) {
        const long long i = b0 + threadIdx.x;
        const unsigned long long v = i < n ? cnt[i] : 0;
        unsigned long long inc = v;
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += t;
        }
        if (lane == 31) s_w[warp] = inc;
        __syncthreads();
        unsigned long long wb = 0;
        for (int k = 0; k < warp; k++) wb += s_w[k];
        const unsigned long long base = s_base;
        if (i < n) cnt[i] = (unsigned)(base + wb + inc - v);
        __syncthreads();
        if (threadIdx.x == 1023) s_base = base + wb + inc;
        __syncthreads();
    }
    if (threadIdx.x == 0) *total = s_base;
}

__global__ void __launch_bounds__(kRunThreads) md_runs_write_kernel(const unsigned* __restrict__ site, const unsigned* __restrict__ suf,
                                                                    long long words, long long L, const unsigned* __restrict__ cta_off,
                                                                    int* __restrict__ run_start, unsigned char* __restrict__ run_class) {
    const long long w = (long long)blockIdx.x * kRunThreads + threadIdx.x;
    const unsigned m = w < words ? md_run_mask(site, suf, w, L) : 0u;
    const int c = __popc(m);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    __shared__ int s_w[kRunThreads / 32];
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    int wb = 0;
    for (int k = 0; k < warp; k++) wb += s_w[k];
    long long r = (long long)cta_off[blockIdx.x] + wb + inc - c;
    if (!m) return;
    const unsigned s = site[w], f = suf[w];
    unsigned mm = m;
    while (mm) {
        const int k = __ffs(mm) - 1;
        mm &= mm - 1;
        run_start[r] = (int)(w * 32 + k);
        run_class[r] = (unsigned char)(((s >> k) & 1u) ? (((f >> k) & 1u) ? 2 : 1) : 0);
        r++;
    }
}

// ------------------------------------------------------------------------------------------------ pass 2
// per pair: the eight 512-base chunk slots -> the block's sum for this sample
__global__ void __launch_bounds__(256) md_pair_sums_kernel(const unsigned long long* __restrict__ slots, const int* __restrict__ pair_blk,
                                                           long long n_pairs, unsigned long long* __restrict__ blk_sum) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n_pairs) return;
    const ulonglong2* s2 = reinterpret_cast<const ulonglong2*>(slots + q * 8);
    unsigned long long t = 0;
#pragma unroll
    for (int j = 0; j < 4; j++) { const ulonglong2 v = s2[j]; t += v.x + v.y; }
    if (t) atomicAdd(blk_sum + pair_blk[q], t);
}

// blk: [start | end | sites] x nb (int32, region-relative).  Cell (b, sample) of the row-major block x S outputs.
__global__ void __launch_bounds__(256) md_certify_kernel(const int* __restrict__ blk, long long nb, const unsigned long long* __restrict__ blk_sum,
                                                         int S, int sample, unsigned long long* __restrict__ sums, long long* __restrict__ q,
                                                         unsigned char* __restrict__ cert, int* __restrict__ walk_list,
                                                         unsigned* __restrict__ walk_cnt) {
    const long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nb) return;
    const unsigned long long sum = blk_sum[b];
    const long long c = b * S + sample;
    int64_t v = 0;
    const bool ok = glmd::certify(sum, blk[2 * nb + b], (int64_t)blk[nb + b] - blk[b], &v);
    sums[c] = sum;
    q[c] = ok ? v : 0;
    cert[c] = ok ? 1 : 0;
    if (!ok) walk_list[atomicAdd(walk_cnt, 1u)] = (int)b;
}

// the reference's chain for the listed cells: acc += float64(d)/1000. over the block's sufficient sites in position order,
// then acc/float64(l)*1000 (multidepth.go:268-283); every operation rounded on its own, as Go does on amd64
__global__ void __launch_bounds__(128) md_walk_kernel(const int* __restrict__ blk, long long nb, const int* __restrict__ walk_list,
                                                      const unsigned* __restrict__ walk_cnt, const int* __restrict__ depth,
                                                      const unsigned* __restrict__ suf, int S, int sample, double* __restrict__ val) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *walk_cnt) return;
    const int b = walk_list[i];
    const int s = blk[b], e = blk[nb + b];
    double acc = 0.0;
    for (int x = s; x < e; x++)
        if ((suf[x >> 5] >> (x & 31)) & 1u) acc = __dadd_rn(acc, __ddiv_rn((double)depth[x], 1000.0));
    val[(long long)b * S + sample] = __dmul_rn(__ddiv_rn(acc, (double)(e - s)), 1000.0);
}

// minSamples = int(0.5 + MinSamples * S) (multidepth.go:64) as Go compiles it on amd64 (CVTTSD2SQ): truncation toward
// zero, and NaN, +-Inf and anything outside [-2^63, 2^63) become INT64_MIN.  A C++ cast leaves those inputs undefined.
int64_t md_min_samples(double frac, int32_t S) {
    const double x = 0.5 + frac * (double)S;
    if (!(x >= -9223372036854775808.0 && x < 9223372036854775808.0)) return INT64_MIN;
    return (int64_t)x;
}

int md_need(gl_ctx* ctx, const char* who) {
    GL_CHECK(gl_use(ctx));
    if (!ctx->md) return gl_fail(ctx, GL_ESTATE, "%s: call gl_multidepth_begin first", who);
    return GL_OK;
}

// the open depth region must be the whole contig of the multidepth run
int md_region_ok(gl_ctx* ctx, const char* who) {
    MdState* m = st(ctx);
    if (!ctx->depth_active || ctx->rs != 0 || ctx->re != m->L)
        return gl_fail(ctx, GL_ESTATE, "%s: open the contig with gl_depth_begin(ctx, 0, %lld) and add one sample's segments", who,
                       (long long)m->L);
    return GL_OK;
}

}  // namespace

void md_free(gl_ctx* ctx) {
    MdState* m = st(ctx);
    if (!m) return;
    for (gl_buf* b : {&m->ge, &m->pos, &m->cnt, &m->site, &m->suf, &m->depth, &m->run_s, &m->run_c, &m->cta_cnt, &m->small, &m->blk,
                      &m->pair_ptr, &m->pair_blk, &m->slots, &m->tmp, &m->sums, &m->q, &m->val, &m->cert, &m->walk_list})
        md_buf_free(*b);
    delete m;
    ctx->md = nullptr;
}

extern "C" {

int gl_multidepth_begin(gl_ctx* ctx, int64_t contig_len, int32_t n_samples, int32_t mincov, double min_samples) {
    GL_CHECK(gl_use(ctx));
    if (contig_len <= 0) return gl_fail(ctx, GL_EINVAL, "gl_multidepth_begin: contig length must be > 0");
    if (contig_len >= (int64_t(1) << 30))
        return gl_fail(ctx, GL_ERANGE, "gl_multidepth_begin: contigs of 2^30 bases or more are not supported (length %lld)",
                       (long long)contig_len);
    if (n_samples < 1 || n_samples >= 65536)
        return gl_fail(ctx, GL_ERANGE, "gl_multidepth_begin: %d samples; the per-base counters hold 1 to 65535", n_samples);
    if (!ctx->md) ctx->md = new MdState();
    MdState* m = st(ctx);
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const int64_t tiles = (contig_len + kTileBases - 1) / kTileBases;
    const int64_t bases = tiles * kTileBases;                 // the tile core writes whole tiles
    m->counted = m->summed = 0;
    m->sites_done = m->blocks_set = false;
    m->n_runs = m->nb = m->n_pairs = m->walked = m->certified = 0;
    m->L = contig_len; m->words = bases / 32; m->tiles = tiles;
    m->S = n_samples; m->mincov = mincov;
    m->min_samples = md_min_samples(min_samples, n_samples);
    GL_CHECK(gl_buf_reserve(ctx, m->ge, (size_t)bases / 8));
    GL_CHECK(gl_buf_reserve(ctx, m->pos, (size_t)bases / 8));
    GL_CHECK(gl_buf_reserve(ctx, m->site, (size_t)bases / 8));
    GL_CHECK(gl_buf_reserve(ctx, m->suf, (size_t)bases / 8));
    GL_CHECK(gl_buf_reserve(ctx, m->cnt, (size_t)bases * 2));
    GL_CHECK(gl_buf_reserve(ctx, m->small, 64));
    GL_CUDA(ctx, cudaMemsetAsync(m->site.p, 0, (size_t)bases / 8, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(m->cnt.p, 0, (size_t)bases * 2, ctx->stream));
    return GL_OK;
}

int gl_multidepth_count(gl_ctx* ctx) {
    GL_CHECK(md_need(ctx, "gl_multidepth_count"));
    GL_CHECK(md_region_ok(ctx, "gl_multidepth_count"));
    MdState* m = st(ctx);
    if (m->counted >= m->S) return gl_fail(ctx, GL_ESTATE, "gl_multidepth_count: all %d samples were counted already", m->S);
    gl_md_ep ep;
    ep.mode = 1;
    ep.mincov = m->mincov;
    ep.ge16 = static_cast<unsigned short*>(m->ge.p);
    ep.pos16 = static_cast<unsigned short*>(m->pos.p);
    ctx->md_ep = ep;
    const int rc = depth_reduce_epilogue(ctx, nullptr);
    ctx->md_ep = gl_md_ep();
    GL_CHECK(rc);
    {
        gl_prof_scope prof(ctx, "md_accum_kernel");
        md_accum_kernel<<<(unsigned)((m->words + 255) / 256), 256, 0, ctx->stream>>>(
            static_cast<const unsigned*>(m->ge.p), static_cast<const unsigned*>(m->pos.p), static_cast<unsigned short*>(m->cnt.p),
            static_cast<unsigned*>(m->site.p), m->words);
    }
    GL_LAUNCHED(ctx, 1);
    m->counted++;
    return GL_OK;
}

int gl_multidepth_sites(gl_ctx* ctx, int32_t* run_start, uint8_t* run_class, int64_t cap, int64_t* n_runs) {
    GL_CHECK(md_need(ctx, "gl_multidepth_sites"));
    MdState* m = st(ctx);
    if (m->counted != m->S) return gl_fail(ctx, GL_ESTATE, "gl_multidepth_sites: %d of %d samples counted", m->counted, m->S);
    if (!m->sites_done) {
        const long long words = m->words;
        const unsigned ctas = (unsigned)((words + kRunThreads - 1) / kRunThreads);
        GL_CHECK(gl_buf_reserve(ctx, m->cta_cnt, (size_t)ctas * 4));
        {
            // counts lie in [0, 65535]: every threshold below -1 acts as -1, every one above 65535 as 65535
            const int thr = (int)std::max<int64_t>(-1, std::min<int64_t>(m->min_samples, 65535));
            gl_prof_scope prof(ctx, "md_classify_kernel");
            md_classify_kernel<<<(unsigned)((words + 255) / 256), 256, 0, ctx->stream>>>(
                static_cast<const unsigned short*>(m->cnt.p), static_cast<const unsigned*>(m->site.p), static_cast<unsigned*>(m->suf.p),
                words, thr);
        }
        {
            gl_prof_scope prof(ctx, "md_runs_count_kernel");
            md_runs_count_kernel<<<ctas, kRunThreads, 0, ctx->stream>>>(static_cast<const unsigned*>(m->site.p),
                                                                        static_cast<const unsigned*>(m->suf.p), words, m->L,
                                                                        static_cast<unsigned*>(m->cta_cnt.p));
        }
        {
            gl_prof_scope prof(ctx, "md_scan_kernel");
            md_scan_kernel<<<1, 1024, 0, ctx->stream>>>(static_cast<unsigned*>(m->cta_cnt.p), ctas,
                                                        static_cast<unsigned long long*>(m->small.p));
        }
        GL_LAUNCHED(ctx, 3);
        unsigned long long total = 0;
        GL_CUDA(ctx, cudaMemcpyAsync(&total, m->small.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        m->n_runs = (int64_t)total;
        GL_CHECK(gl_buf_reserve(ctx, m->run_s, (size_t)std::max<int64_t>(m->n_runs, 1) * 4));
        GL_CHECK(gl_buf_reserve(ctx, m->run_c, (size_t)std::max<int64_t>(m->n_runs, 1)));
        {
            gl_prof_scope prof(ctx, "md_runs_write_kernel");
            md_runs_write_kernel<<<ctas, kRunThreads, 0, ctx->stream>>>(static_cast<const unsigned*>(m->site.p),
                                                                        static_cast<const unsigned*>(m->suf.p), words, m->L,
                                                                        static_cast<const unsigned*>(m->cta_cnt.p),
                                                                        static_cast<int*>(m->run_s.p), static_cast<unsigned char*>(m->run_c.p));
        }
        GL_LAUNCHED(ctx, 1);
        m->sites_done = true;
    }
    if (n_runs) *n_runs = m->n_runs;
    if (!run_start && !run_class) return GL_OK;
    if (cap < m->n_runs) return gl_fail(ctx, GL_ERANGE, "gl_multidepth_sites: %lld runs, capacity %lld", (long long)m->n_runs, (long long)cap);
    if (m->n_runs > 0) {
        if (run_start) GL_CUDA(ctx, cudaMemcpyAsync(run_start, m->run_s.p, (size_t)m->n_runs * 4, cudaMemcpyDeviceToHost, ctx->stream));
        if (run_class) GL_CUDA(ctx, cudaMemcpyAsync(run_class, m->run_c.p, (size_t)m->n_runs, cudaMemcpyDeviceToHost, ctx->stream));
    }
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_multidepth_set_blocks(gl_ctx* ctx, const int64_t* blk_start, const int64_t* blk_end, const int64_t* blk_sites, int64_t n_blocks) {
    GL_CHECK(md_need(ctx, "gl_multidepth_set_blocks"));
    MdState* m = st(ctx);
    if (!m->sites_done) return gl_fail(ctx, GL_ESTATE, "gl_multidepth_set_blocks: call gl_multidepth_sites first");
    if (n_blocks < 0 || n_blocks >= INT32_MAX || (n_blocks > 0 && (!blk_start || !blk_end || !blk_sites)))
        return gl_fail(ctx, GL_EINVAL, "gl_multidepth_set_blocks: bad argument");
    // blocks as int32 [start | end | sites]; (tile, block) pairs in tile order (counting sort)
    std::vector<int> blk((size_t)n_blocks * 3);
    std::vector<int> ptr((size_t)m->tiles + 1, 0);
    for (int64_t b = 0; b < n_blocks; b++) {
        const int64_t s = blk_start[b], e = blk_end[b], n = blk_sites[b];
        if (s < 0 || e <= s || e > m->L || n < 1 || n > e - s)
            return gl_fail(ctx, GL_EINVAL, "gl_multidepth_set_blocks: block %lld [%lld,%lld) with %lld sites is not inside the contig",
                           (long long)b, (long long)s, (long long)e, (long long)n);
        blk[(size_t)b] = (int)s; blk[(size_t)(n_blocks + b)] = (int)e; blk[(size_t)(2 * n_blocks + b)] = (int)n;
        for (int64_t t = s / kTileBases; t <= (e - 1) / kTileBases; t++) ptr[(size_t)t + 1]++;
    }
    for (int64_t t = 0; t < m->tiles; t++) ptr[(size_t)t + 1] += ptr[(size_t)t];
    const int64_t np = ptr[(size_t)m->tiles];
    std::vector<int> pair((size_t)std::max<int64_t>(np, 1));
    {
        std::vector<int> fill(ptr.begin(), ptr.end() - 1);
        for (int64_t b = 0; b < n_blocks; b++)
            for (int64_t t = blk_start[b] / kTileBases; t <= (blk_end[b] - 1) / kTileBases; t++) pair[(size_t)fill[(size_t)t]++] = (int)b;
    }
    const size_t cells = (size_t)std::max<int64_t>(n_blocks, 1) * m->S;
    GL_CHECK(gl_buf_reserve(ctx, m->blk, std::max<size_t>(blk.size(), 1) * 4));
    GL_CHECK(gl_buf_reserve(ctx, m->pair_ptr, ptr.size() * 4));
    GL_CHECK(gl_buf_reserve(ctx, m->pair_blk, pair.size() * 4));
    GL_CHECK(gl_buf_reserve(ctx, m->slots, (size_t)std::max<int64_t>(np, 1) * 64));
    GL_CHECK(gl_buf_reserve(ctx, m->tmp, (size_t)std::max<int64_t>(n_blocks, 1) * 8));
    GL_CHECK(gl_buf_reserve(ctx, m->walk_list, (size_t)std::max<int64_t>(n_blocks, 1) * 4));
    GL_CHECK(gl_buf_reserve(ctx, m->sums, cells * 8));
    GL_CHECK(gl_buf_reserve(ctx, m->q, cells * 8));
    GL_CHECK(gl_buf_reserve(ctx, m->val, cells * 8));
    GL_CHECK(gl_buf_reserve(ctx, m->cert, cells));
    if (!blk.empty()) GL_CUDA(ctx, cudaMemcpyAsync(m->blk.p, blk.data(), blk.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(m->pair_ptr.p, ptr.data(), ptr.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(m->pair_blk.p, pair.data(), pair.size() * 4, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(m->slots.p, 0, (size_t)std::max<int64_t>(np, 1) * 64, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(m->sums.p, 0, cells * 8, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(m->q.p, 0, cells * 8, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(m->val.p, 0, cells * 8, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(m->cert.p, 0, cells, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));                 // the host tables above go out of scope
    m->nb = n_blocks;
    m->n_pairs = np;
    m->summed = 0;
    m->walked = 0;
    m->certified = 0;
    m->blocks_set = true;
    return GL_OK;
}

int gl_multidepth_sums(gl_ctx* ctx, int32_t sample) {
    GL_CHECK(md_need(ctx, "gl_multidepth_sums"));
    MdState* m = st(ctx);
    if (!m->blocks_set) return gl_fail(ctx, GL_ESTATE, "gl_multidepth_sums: call gl_multidepth_set_blocks first");
    if (sample < 0 || sample >= m->S) return gl_fail(ctx, GL_EINVAL, "gl_multidepth_sums: sample %d out of range [0,%d)", sample, m->S);
    GL_CHECK(md_region_ok(ctx, "gl_multidepth_sums"));
    if (m->nb == 0) { m->summed++; return GL_OK; }
    gl_md_ep ep;
    ep.mode = 2;
    ep.suf = static_cast<const unsigned*>(m->suf.p);
    ep.pair_ptr = static_cast<const int*>(m->pair_ptr.p);
    ep.pair_blk = static_cast<const int*>(m->pair_blk.p);
    ep.blk_start = static_cast<const int*>(m->blk.p);
    ep.blk_end = static_cast<const int*>(m->blk.p) + m->nb;
    ep.slots = static_cast<unsigned long long*>(m->slots.p);
    ctx->md_ep = ep;
    const int rc = depth_reduce_epilogue(ctx, nullptr);
    ctx->md_ep = gl_md_ep();
    GL_CHECK(rc);
    unsigned* walk_cnt = static_cast<unsigned*>(m->small.p) + 8;
    GL_CUDA(ctx, cudaMemsetAsync(m->tmp.p, 0, (size_t)m->nb * 8, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(walk_cnt, 0, 4, ctx->stream));
    {
        gl_prof_scope prof(ctx, "md_pair_sums_kernel");
        md_pair_sums_kernel<<<(unsigned)((m->n_pairs + 255) / 256), 256, 0, ctx->stream>>>(
            static_cast<const unsigned long long*>(m->slots.p), static_cast<const int*>(m->pair_blk.p), m->n_pairs,
            static_cast<unsigned long long*>(m->tmp.p));
    }
    {
        gl_prof_scope prof(ctx, "md_certify_kernel");
        md_certify_kernel<<<(unsigned)((m->nb + 255) / 256), 256, 0, ctx->stream>>>(
            static_cast<const int*>(m->blk.p), m->nb, static_cast<const unsigned long long*>(m->tmp.p), m->S, sample,
            static_cast<unsigned long long*>(m->sums.p), static_cast<long long*>(m->q.p), static_cast<unsigned char*>(m->cert.p),
            static_cast<int*>(m->walk_list.p), walk_cnt);
    }
    GL_LAUNCHED(ctx, 2);
    unsigned n_walk = 0;
    GL_CUDA(ctx, cudaMemcpyAsync(&n_walk, walk_cnt, 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (n_walk > 0) {
        // the cells that could not be certified: this sample's per-base depth, then the literal chain per cell
        GL_CHECK(gl_buf_reserve(ctx, m->depth, (size_t)m->L * 4));
        GL_CHECK(depth_reduce_epilogue(ctx, static_cast<int32_t*>(m->depth.p)));
        {
            gl_prof_scope prof(ctx, "md_walk_kernel");
            md_walk_kernel<<<(n_walk + 127) / 128, 128, 0, ctx->stream>>>(
                static_cast<const int*>(m->blk.p), m->nb, static_cast<const int*>(m->walk_list.p), walk_cnt,
                static_cast<const int*>(m->depth.p), static_cast<const unsigned*>(m->suf.p), m->S, sample, static_cast<double*>(m->val.p));
        }
        GL_LAUNCHED(ctx, 1);
    }
    m->walked += n_walk;
    m->certified += m->nb - (int64_t)n_walk;
    m->summed++;
    return GL_OK;
}

int gl_multidepth_result(gl_ctx* ctx, uint64_t* sums, int64_t* q, double* val, uint8_t* certified) {
    GL_CHECK(md_need(ctx, "gl_multidepth_result"));
    MdState* m = st(ctx);
    if (!m->blocks_set) return gl_fail(ctx, GL_ESTATE, "gl_multidepth_result: call gl_multidepth_set_blocks first");
    const size_t cells = (size_t)m->nb * m->S;
    if (cells > 0) {
        if (sums) GL_CUDA(ctx, cudaMemcpyAsync(sums, m->sums.p, cells * 8, cudaMemcpyDeviceToHost, ctx->stream));
        if (q) GL_CUDA(ctx, cudaMemcpyAsync(q, m->q.p, cells * 8, cudaMemcpyDeviceToHost, ctx->stream));
        if (val) GL_CUDA(ctx, cudaMemcpyAsync(val, m->val.p, cells * 8, cudaMemcpyDeviceToHost, ctx->stream));
        if (certified) GL_CUDA(ctx, cudaMemcpyAsync(certified, m->cert.p, cells, cudaMemcpyDeviceToHost, ctx->stream));
    }
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_multidepth_stats(gl_ctx* ctx, int64_t* n_blocks, int64_t* n_walked, int64_t* n_certified, int64_t* min_samples) {
    GL_CHECK(md_need(ctx, "gl_multidepth_stats"));
    MdState* m = st(ctx);
    if (n_blocks) *n_blocks = m->nb;
    if (n_walked) *n_walked = m->walked;
    if (n_certified) *n_certified = m->certified;
    if (min_samples) *min_samples = m->min_samples;
    return GL_OK;
}

}  // extern "C"
