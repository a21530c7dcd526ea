// dcnv_svd.cu — `goleft dcnv --svd PCT` (DESIGN §1.13): the reference's ZScore.Scale, SVD.Debias{MinVariancePct} and
// ZScore.UnScale (dcnv/scalers/scalers.go:25-56, dcnv/debiaser/debiaser.go:173-200), which its main never reaches, on the
// n-sites x S-samples matrix X after the median normalisation.
//
//   row z-score     m = sum / S, sd = sqrt(sum (x - m)^2 / (S - 1)), z = (x - m) * (1 / sd).  A row whose values are all
//                   equal (every row when S < 2) is excluded: it takes no part and is never written.
//   singular values s = sqrt(eigenvalues of G = Z^T Z), S x S; an eigenvalue <= 1e-12 * lambda_1 counts as 0.
//   count           n = the first index with n >= min(15, rank) or 100 s[n] / sum(s) <= PCT.
//   remove          z' = z - V_n (V_n^T z) for every kept row (= U Sigma' V^T with the first n values zeroed), written back
//                   as max(0, z' sd + m).  n = 0 writes nothing.
//
// Kernels:
//   svd_stats_kernel    one warp per row: m, sd, 1/sd (0 for an excluded row), the kept count and the first bad row.
//   svd_gram_kernel     the upper 64 x 64 tiles of G on the FP64 tensor cores (mma.sync m8n8k4 f64), K along the rows.  The
//                       z-scoring is fused into the fragment loads: a thread's A and B elements of one k4 step come from
//                       the same row, so each needs one (x - m) * r from the staged x.  Writing Z instead would cost one
//                       more 16 B/cell pass, the traffic of the whole projection pass (DESIGN §1.13 has both times).
//                       Deterministic: the rows are cut into chunks whose size depends on (n, S) only; a CTA sums one
//                       (tile, chunk) in row order, one k4 group of rows at a time, into its slot of the workspace W.  A
//                       chunk cut by a streamed row block resumes from W in the next block with the same k4 groups (block
//                       boundaries are multiples of 4), so the bits do not depend on the block size or the SM count.
//   svd_reduce_kernel   G = the chunks' partial tiles added in chunk order, mirrored.
//   svd_project_kernel  one warp per kept row: p = V_n^T z, z' = z - V_n p, unscaled in place.
// The eigenproblem: sym_tridiag (pca.cu) tridiagonalises G on the device; the host counts the eigenvalues above the rank
// threshold with one Sturm count and bisects only those, each on its own pool task (host/pca_eig.cpp), then finds the top
// n vectors by inverse iteration and takes them back through the reflectors.
#include <math.h>
#include <chrono>
#include "gl_common.cuh"
#include "host/pca_eig.h"
#include "sym_eig.cuh"

namespace {

constexpr int kT = 64;                 // Gram tile (samples x samples)
constexpr int kBK = 16;                // rows per pipeline stage
constexpr int kStages = 4;
constexpr int kThreads = 128;          // 4 warps, 2 x 2, 32 x 32 outputs each
constexpr int kPitch = kT + 4;         // doubles per staged row: the 4 rows a k4 step reads land in distinct banks
constexpr int kStageDoubles = 2 * kBK * kPitch + 2 * kBK;
constexpr int kSmem = kStages * kStageDoubles * 8;
constexpr int kMaxRemove = 15;         // debiaser.go:185
constexpr int64_t kMinChunk = 2048;    // rows
constexpr int64_t kTargetCtas = 1024;  // (tile, chunk) pairs the chunking aims for; a constant, not the SM count
constexpr double kRankTol = 1e-12;     // as glpca::kRankTol (DESIGN §1.11)
constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// rows [0, nb) of the block x (row stride ld); row i of the block is row b0 + i of the matrix
__global__ void __launch_bounds__(256) svd_stats_kernel(const double* __restrict__ x, long long ld, long long nb, int S, long long b0,
                                                        double* __restrict__ mean, double* __restrict__ sd, double* __restrict__ rsd,
                                                        unsigned long long* __restrict__ counters) {
    __shared__ unsigned long long kept_sh;
    if (threadIdx.x == 0) kept_sh = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    unsigned long long kept = 0;
    for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < nb; i += ((long long)gridDim.x * blockDim.x) >> 5) {
        const double* row = x + i * ld;
        const double v0 = row[0];
        double s = 0;
        bool same = true, finite = true;
        for (int j = lane; j < S; j += 32) {
            const double v = row[j];
            s += v;
            same &= v == v0;
            finite &= isfinite(v);
        }
        same = __all_sync(kFull, same);
        finite = __all_sync(kFull, finite);
        double m = 0, d = 0, r = 0;
        if (S >= 2 && !same) {
            m = warp_sum(s) / S;
            double q = 0;
            for (int j = lane; j < S; j += 32) {
                const double t = row[j] - m;
                q += t * t;
            }
            d = sqrt(warp_sum(q) / (S - 1));
            r = 1.0 / d;
            if (!finite || !isfinite(m) || !isfinite(d)) {
                if (lane == 0) atomicMin(&counters[1], (unsigned long long)(b0 + i));
                r = 0;
            } else if (!(d > 0) || isinf(r)) {           // deviations that underflow: nothing to scale by
                m = d = r = 0;
            }
        }
        if (lane == 0) {
            mean[b0 + i] = m;
            sd[b0 + i] = d;
            rsd[b0 + i] = r;
            kept += r != 0;
        }
    }
    if (lane == 0 && kept) atomicAdd(&kept_sh, kept);
    __syncthreads();
    if (threadIdx.x == 0 && kept_sh) atomicAdd(&counters[0], kept_sh);
}

__device__ __forceinline__ void cp_async8(uint32_t dst, const void* src, int bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(dst), "l"(src), "r"(bytes));
}

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

// CTA (tile, chunk c_first + blockIdx.y): rows [max(c * cr, b0), min((c + 1) * cr, b1)) of the block x, whose first row is
// row b0 (row stride ld).  tile enumerates the upper triangle of T x T tiles row by row.  W: [chunks][tiles][64 x 64].
__global__ void __launch_bounds__(kThreads) svd_gram_kernel(const double* __restrict__ x, long long ld, int S, long long b0, long long b1,
                                                            const double* __restrict__ mean, const double* __restrict__ rsd, int T,
                                                            int tiles, long long cr, int c_first, double* __restrict__ W) {
    extern __shared__ __align__(16) double smem[];
    int t = blockIdx.x, I = 0;
    while (t >= T - I) { t -= T - I; I++; }
    const int J = I + t;
    const long long c = c_first + blockIdx.y;
    const long long r0 = max(c * cr, b0), r1 = min((c + 1) * cr, b1);
    const int nk = (int)((r1 - r0 + kBK - 1) / kBK);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 1, wn = warp & 1;
    const bool diag = I == J;
    const uint32_t s0 = (uint32_t)__cvta_generic_to_shared(smem);

    auto load = [&](int stage, int kb) {
        const uint32_t sa = s0 + stage * kStageDoubles * 8, sb = sa + kBK * kPitch * 8, sm = sb + kBK * kPitch * 8;
        const long long rb = r0 + (long long)kb * kBK;
#pragma unroll
        for (int h = 0; h < kBK * kT / kThreads; h++) {
            const int e = tid + h * kThreads, rr = e / kT, cc = e % kT;
            const long long row = rb + rr;
            const int ca = I * kT + cc, cb = J * kT + cc;
            const bool ok = row < r1;
            const double* p = x + (row - b0) * ld;
            cp_async8(sa + (rr * kPitch + cc) * 8, ok && ca < S ? p + ca : x, ok && ca < S ? 8 : 0);
            if (!diag) cp_async8(sb + (rr * kPitch + cc) * 8, ok && cb < S ? p + cb : x, ok && cb < S ? 8 : 0);
        }
        if (tid < 2 * kBK) {
            const int rr = tid % kBK;
            const long long row = rb + rr;
            const double* src = tid < kBK ? mean : rsd;
            cp_async8(sm + tid * 8, row < r1 ? src + row : src, row < r1 ? 8 : 0);
        }
    };

    double acc[4][4][2];
    const size_t slot = ((size_t)c * tiles + blockIdx.x) * (kT * kT);
    const int g = lane >> 2, tq = lane & 3;
#pragma unroll
    for (int mi = 0; mi < 4; mi++)
#pragma unroll
        for (int nj = 0; nj < 4; nj++) {
            if (c * cr < b0) {                                   // the chunk began in the previous block: resume its sums
                const double2 v = *reinterpret_cast<const double2*>(&W[slot + (wm * 32 + mi * 8 + g) * kT + wn * 32 + nj * 8 + tq * 2]);
                acc[mi][nj][0] = v.x;
                acc[mi][nj][1] = v.y;
            } else {
                acc[mi][nj][0] = acc[mi][nj][1] = 0;
            }
        }

#pragma unroll
    for (int s = 0; s < kStages - 1; s++) {
        if (s < nk) load(s, s);
        asm volatile("cp.async.commit_group;\n" ::);
    }
    for (int kb = 0; kb < nk; kb++) {
        asm volatile("cp.async.wait_group %0;\n" ::"n"(kStages - 2));
        __syncthreads();
        const int nxt = kb + kStages - 1;
        if (nxt < nk) load(nxt % kStages, nxt);
        asm volatile("cp.async.commit_group;\n" ::);
        const double* sa = smem + (kb % kStages) * kStageDoubles;
        const double* sb = diag ? sa : sa + kBK * kPitch;
        const double* sm = sa + 2 * kBK * kPitch;
        const long long left = r1 - (r0 + (long long)kb * kBK);
        const int groups = (int)min(4LL, (left + 3) / 4);        // k4 groups that hold a row of the range
        for (int q = 0; q < groups; q++) {
            const int kk = q * 4 + tq;
            const double mk = sm[kk], rk = sm[kBK + kk];
            double a[4], b[4];
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const double va = sa[kk * kPitch + wm * 32 + i * 8 + g], vb = sb[kk * kPitch + wn * 32 + i * 8 + g];
                a[i] = rk != 0 ? (va - mk) * rk : 0.0;
                b[i] = rk != 0 ? (vb - mk) * rk : 0.0;
            }
#pragma unroll
            for (int mi = 0; mi < 4; mi++)
#pragma unroll
                for (int nj = 0; nj < 4; nj++) dmma(acc[mi][nj][0], acc[mi][nj][1], a[mi], b[nj]);
        }
    }
    asm volatile("cp.async.wait_group 0;\n" ::);
#pragma unroll
    for (int mi = 0; mi < 4; mi++)
#pragma unroll
        for (int nj = 0; nj < 4; nj++)
            *reinterpret_cast<double2*>(&W[slot + (wm * 32 + mi * 8 + g) * kT + wn * 32 + nj * 8 + tq * 2]) =
                make_double2(acc[mi][nj][0], acc[mi][nj][1]);
}

// G(i, j) = G(j, i) = the chunks' partial sums of the upper entry (i <= j), added in chunk order; one CTA per tile
__global__ void __launch_bounds__(256) svd_reduce_kernel(const double* __restrict__ W, int T, int tiles, int chunks, int S,
                                                         double* __restrict__ G) {
    int t = blockIdx.x, I = 0;
    while (t >= T - I) { t -= T - I; I++; }
    const int J = I + t;
    for (int e = threadIdx.x; e < kT * kT; e += blockDim.x) {
        const int i = I * kT + e / kT, j = J * kT + e % kT;
        if (i >= S || j >= S || i > j) continue;
        const double* w = W + (size_t)blockIdx.x * (kT * kT) + e;
        double s = w[0];
        for (int c = 1; c < chunks; c++) s += w[(size_t)c * tiles * (kT * kT)];
        G[(size_t)i * S + j] = s;
        G[(size_t)j * S + i] = s;
    }
}

// every kept row of the block: z' = z - V_n (V_n^T z), x = max(0, z' sd + m); V is nr x S (row c = component c)
__global__ void __launch_bounds__(256) svd_project_kernel(double* __restrict__ x, long long ld, long long nb, int S, long long b0,
                                                          const double* __restrict__ mean, const double* __restrict__ sd,
                                                          const double* __restrict__ rsd, const double* __restrict__ V, int nr) {
    const int lane = threadIdx.x & 31;
    for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < nb; i += ((long long)gridDim.x * blockDim.x) >> 5) {
        const double r = rsd[b0 + i];
        if (r == 0) continue;
        const double m = mean[b0 + i], d = sd[b0 + i];
        double* row = x + i * ld;
        double p[kMaxRemove];
#pragma unroll
        for (int k = 0; k < kMaxRemove; k++) p[k] = 0;
        for (int j = lane; j < S; j += 32) {
            const double z = (row[j] - m) * r;
#pragma unroll
            for (int k = 0; k < kMaxRemove; k++)
                if (k < nr) p[k] += __ldg(&V[(size_t)k * S + j]) * z;
        }
#pragma unroll
        for (int k = 0; k < kMaxRemove; k++)
            if (k < nr) p[k] = warp_sum(p[k]);
        for (int j = lane; j < S; j += 32) {
            double z = (row[j] - m) * r;
#pragma unroll
            for (int k = 0; k < kMaxRemove; k++)
                if (k < nr) z -= __ldg(&V[(size_t)k * S + j]) * p[k];
            const double v = z * d + m;
            row[j] = v > 0 ? v : 0.0;                          // math.Max(0, v); -0 becomes +0
        }
    }
}

double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// the whole call.  hx: host matrix (streamed through a device block of br rows), or dx: the device matrix (one block).
int svd_run(gl_ctx* ctx, const char* fn, double* hx, double* dx, int64_t n, int64_t ld, int32_t S, double pct, int64_t block_rows,
            double* sv, double* gram, int32_t* n_removed, int64_t* n_kept) {
    double* ph = ctx->svd_phase;
    for (int i = 0; i < 4; i++) ph[i] = 0;
    double t0 = now();
    const int T = (S + kT - 1) / kT, tiles = T * (T + 1) / 2;
    const int64_t nc0 = std::max<int64_t>(1, std::min<int64_t>((n + kMinChunk - 1) / kMinChunk, (kTargetCtas + tiles - 1) / tiles));
    const int64_t cr = ((n + nc0 - 1) / nc0 + kBK - 1) / kBK * kBK;
    const int64_t chunks = (n + cr - 1) / cr;
    const double fixed = 8.0 * (3.0 * (double)n + (double)S * S + (double)chunks * tiles * kT * kT + (kMaxRemove + 4.0) * S) + (1 << 20);
    size_t free_b = 0, total_b = 0;
    GL_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
    if (fixed > 0.9 * (double)free_b)
        return gl_fail(ctx, GL_ENOMEM, "%s: the %d x %d Gram and its workspace (%.0f MB) do not fit in free device memory", fn, S, S, fixed / 1e6);
    int64_t br = n;
    if (hx) {
        if (block_rows == 0) {
            br = (int64_t)std::min<double>((double)n, (0.8 * (double)free_b - fixed) / (8.0 * S));
            if (br < std::min<int64_t>(n, 4)) return gl_fail(ctx, GL_ENOMEM, "%s: no row block of %d samples fits beside the Gram", fn, S);
        } else {
            br = block_rows;
        }
        if (br < n) br = std::max<int64_t>(4, br & ~(int64_t)3);           // block boundaries on k4 groups
        br = std::min(br, n);
    }
    gl_scratch tmp(ctx);
    double *d_stats, *d_G, *d_W, *d_V, *d_blk = dx;
    unsigned long long* d_cnt;
    GL_CHECK(tmp.alloc(d_stats, (size_t)n * 3));
    GL_CHECK(tmp.alloc(d_G, (size_t)S * S));
    GL_CHECK(tmp.alloc(d_W, (size_t)chunks * tiles * kT * kT));
    GL_CHECK(tmp.alloc(d_V, (size_t)kMaxRemove * S));
    GL_CHECK(tmp.alloc(d_cnt, 2));
    if (hx) GL_CHECK(tmp.alloc(d_blk, (size_t)br * S));
    const int64_t ldd = hx ? S : ld;
    double *d_mean = d_stats, *d_sd = d_stats + n, *d_rsd = d_stats + 2 * n;
    const unsigned long long cnt0[2] = {0, ~0ull};
    GL_CUDA(ctx, cudaMemcpyAsync(d_cnt, cnt0, sizeof cnt0, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaFuncSetAttribute(svd_gram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    const unsigned row_blocks = (unsigned)ctx->sm_count * 8;
    auto copy = [&](bool up, int64_t b0, int64_t nb) -> int {               // one block between x and d_blk, timed
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));                   // the kernels before it count as theirs
        const double tc = now();
        if (up) GL_CUDA(ctx, cudaMemcpy2DAsync(d_blk, (size_t)S * 8, hx + b0 * ld, (size_t)ld * 8, (size_t)S * 8, (size_t)nb, cudaMemcpyHostToDevice, ctx->stream));
        else GL_CUDA(ctx, cudaMemcpy2DAsync(hx + b0 * ld, (size_t)ld * 8, d_blk, (size_t)S * 8, (size_t)S * 8, (size_t)nb, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        ph[3] += now() - tc;
        return GL_OK;
    };

    // ---- pass 1: row stats and the Gram's partial tiles, block by block
    for (int64_t b0 = 0; b0 < n; b0 += br) {
        const int64_t nb = std::min(br, n - b0);
        const double* blk = hx ? d_blk : dx + b0 * ld;
        if (hx) GL_CHECK(copy(true, b0, nb));
        {
            gl_prof_scope prof(ctx, "svd_stats_kernel");
            svd_stats_kernel<<<(unsigned)std::min<int64_t>(row_blocks, (nb + 7) / 8), 256, 0, ctx->stream>>>(blk, (long long)ldd, (long long)nb, S,
                                                                                                        (long long)b0, d_mean, d_sd, d_rsd, d_cnt);
        }
        GL_LAUNCHED(ctx, 1);
        const int64_t c_first = b0 / cr, c_last = (b0 + nb - 1) / cr;
        {
            gl_prof_scope prof(ctx, "svd_gram_kernel");
            svd_gram_kernel<<<dim3((unsigned)tiles, (unsigned)(c_last - c_first + 1)), kThreads, kSmem, ctx->stream>>>(
                blk, (long long)ldd, S, (long long)b0, (long long)(b0 + nb), d_mean, d_rsd, T, tiles, (long long)cr, (int)c_first, d_W);
        }
        GL_LAUNCHED(ctx, 1);
    }
    unsigned long long cnt[2];
    GL_CUDA(ctx, cudaMemcpyAsync(cnt, d_cnt, sizeof cnt, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (cnt[1] != ~0ull) return gl_fail(ctx, GL_EINVAL, "%s: row %llu has a non-finite value (or its mean or sd is not finite)", fn, cnt[1]);
    if (n_kept) *n_kept = (int64_t)cnt[0];
    {
        gl_prof_scope prof(ctx, "svd_reduce_kernel");
        svd_reduce_kernel<<<(unsigned)tiles, 256, 0, ctx->stream>>>(d_W, T, tiles, (int)chunks, S, d_G);
    }
    GL_LAUNCHED(ctx, 1);
    if (gram) GL_CUDA(ctx, cudaMemcpyAsync(gram, d_G, (size_t)S * S * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ph[0] = now() - t0 - ph[3];

    // ---- the singular values, the count, the top vectors
    t0 = now();
    SymTridiag tri;
    GL_CHECK(sym_tridiag(ctx, d_G, S, tri));
    std::vector<double> lam((size_t)S, 0.0);
    const int rank = glpca::tridiag_values_above(tri.d.data(), tri.e.data(), S, kRankTol, lam.data());
    std::vector<double> s((size_t)S, 0.0);
    double sum = 0;
    for (int j = 0; j < rank; j++) { s[(size_t)j] = sqrt(lam[(size_t)j]); sum += s[(size_t)j]; }
    int nr = 0;
    while (nr < std::min(kMaxRemove, rank) && 100 * s[(size_t)nr] / sum > pct) nr++;
    if (sv) std::copy(s.begin(), s.end(), sv);
    *n_removed = nr;
    if (nr > 0) {
        std::vector<double> u((size_t)nr * S);
        glpca::tridiag_vectors(tri.d.data(), tri.e.data(), S, lam.data(), nr, u.data());
        tri.back_transform(u.data(), nr);
        GL_CUDA(ctx, cudaMemcpyAsync(d_V, u.data(), u.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    ph[1] = now() - t0;
    if (nr == 0) return GL_OK;                                   // nothing removed: X is left as it was, bit for bit

    // ---- pass 2: the projection, in place; a single host block is still on the device
    t0 = now();
    const double c0 = ph[3];
    for (int64_t b0 = 0; b0 < n; b0 += br) {
        const int64_t nb = std::min(br, n - b0);
        double* blk = hx ? d_blk : dx + b0 * ld;
        if (hx && br < n) GL_CHECK(copy(true, b0, nb));
        {
            gl_prof_scope prof(ctx, "svd_project_kernel");
            svd_project_kernel<<<(unsigned)std::min<int64_t>(row_blocks, (nb + 7) / 8), 256, 0, ctx->stream>>>(
                blk, (long long)ldd, (long long)nb, S, (long long)b0, d_mean, d_sd, d_rsd, d_V, nr);
        }
        GL_LAUNCHED(ctx, 1);
        if (hx) GL_CHECK(copy(false, b0, nb));
    }
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ph[2] = now() - t0 - (ph[3] - c0);
    return GL_OK;
}

int check_args(gl_ctx* ctx, const char* fn, const void* x, int64_t n, int64_t ld, int32_t S, double pct, const void* n_removed) {
    if (!x || !n_removed || n < 1 || S < 1 || ld < S)
        return gl_fail(ctx, GL_EINVAL, "%s: bad argument (n = %lld, ld = %lld, S = %d)", fn, (long long)n, (long long)ld, S);
    if (S > 65535) return gl_fail(ctx, GL_EINVAL, "%s: %d samples; at most 65535", fn, S);
    if (!(pct >= 0) || isinf(pct)) return gl_fail(ctx, GL_EINVAL, "%s: the minimum variance percentage must be finite and >= 0", fn);
    return GL_OK;
}

}  // namespace

extern "C" {

int gl_dcnv_svd(gl_ctx* ctx, double* x, int64_t n, int64_t ld, int32_t S, double min_pct, int64_t block_rows, double* sv,
                double* gram, int32_t* n_removed, int64_t* n_kept) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(check_args(ctx, "gl_dcnv_svd", x, n, ld, S, min_pct, n_removed));
    if (block_rows < 0) return gl_fail(ctx, GL_EINVAL, "gl_dcnv_svd: block_rows < 0");
    return svd_run(ctx, "gl_dcnv_svd", x, nullptr, n, ld, S, min_pct, block_rows, sv, gram, n_removed, n_kept);
}

int gl_dcnv_svd_device(gl_ctx* ctx, double* d_x, int64_t n, int64_t ld, int32_t S, double min_pct, double* sv, double* gram,
                       int32_t* n_removed, int64_t* n_kept) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(check_args(ctx, "gl_dcnv_svd_device", d_x, n, ld, S, min_pct, n_removed));
    if ((uintptr_t)d_x & 7) return gl_fail(ctx, GL_EINVAL, "gl_dcnv_svd_device: d_x is not 8-byte aligned");
    return svd_run(ctx, "gl_dcnv_svd_device", nullptr, d_x, n, ld, S, min_pct, 0, sv, gram, n_removed, n_kept);
}

int gl_dcnv_svd_phases(gl_ctx* ctx, double* t4) {
    if (!ctx || !t4) return gl_fail(ctx, GL_EINVAL, "gl_dcnv_svd_phases: bad argument");
    for (int i = 0; i < 4; i++) t4[i] = ctx->svd_phase[i];
    return GL_OK;
}

}  // extern "C"
