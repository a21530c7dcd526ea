// emdepth.cu — `goleft emdepth` (emdepth/emdepth.go:117-304, stats.go): a cn.mops-style EM per row of an n-rows x S-samples
// float32 depth matrix, then a copy number (CN) and the Log2FC classes of every cell.  DESIGN §1.10.
//
// One warp per row (rows are independent; S <= 65535 samples strided over the lanes, read from global memory / L1):
//   median32     two exact order statistics by a bitwise radix select on the float32 bits (inputs are non-negative, so bit
//                order is value order); an even S takes (b[S/2] + b[S/2+1]) / 2, the reference's off-by-one.
//   EM loop      <= 10 passes: every lane assigns its samples to the 9 bins (the CN2 fast path, then Go's sort.Search with
//                the idx / idx-1 rule; the centres live in shared memory for the search) and sums bin 2 in float64.  The
//                mean must equal Go's sequential mean64: when the bin's non-zero bits span at most 53 (em_core.h sum_exact)
//                every partial sum is exact and the warp's tree sum is that value; otherwise lane 0 sums in sample order.
//                mean(bin 2) == 0 takes the reference's fallback over bins 1..7, literally.
//   Type         SearchFloat64s over the final centres (above the top one: CN 9), then adjustCN's Poisson test o * 0.9 < o2.
//   Log2FC       log2(d / lambda[2]) against -0.8 / 0.4 (Same) and -0.5 / 0.3 (makecnvs).
// Go's amd64 Exp / Log are assembly (Exp uses FMA where the CPU has it), so the reference's last bits depend on the CPU.  The
// Poisson test and the thresholds are decided here with rigorous error bounds that hold for any faithful Log / Lgamma / Exp;
// a cell whose decision falls inside a bound is decided by the device's own functions and counted (gl_emdepth_stats).
#include <math_constants.h>
#include "gl_common.cuh"
#include "host/em_core.h"

namespace {

constexpr int kWarps = 8;                    // rows per CTA
constexpr unsigned kFull = 0xffffffffu;
// float32 bits of 2^62: this and above is rejected, and so is any sign bit, Inf or NaN.  A library policy (DESIGN §1.10):
// the reference itself panics only for some of these (d <= -1.5 off CN 2, int(0.5 + d) overflow).
constexpr uint32_t kBadBits = 0x5e800000u;
// 2^t for the Log2FC thresholds t = -0.8, 0.4 (Same), -0.5, 0.3 (makecnvs)
constexpr double kQm08 = 0.57434917749851755, kQ04 = 1.3195079107728942, kQm05 = 0.70710678118654752, kQ03 = 1.2311444133449163;
constexpr double kRel = 1e-12;               // relative band around 2^t inside which log2 implementations may disagree
constexpr double kLn09 = -0.10536051565782628;   // log(0.9)

// sort.SearchFloat64s(l, d) = sort.Search(9, l[h] >= d), literally (the centres need not be sorted: lambda[0] = 0.01 m)
__device__ __forceinline__ int go_search(const double* l, double d) {
    int i = 0, j = glem::kCN;
    while (i < j) {
        const int h = (i + j) >> 1;
        if (!(l[h] >= d)) i = h + 1;
        else j = h;
    }
    return i;
}

// the bin EMDepth puts depth d in (emdepth.go:152-176)
__device__ __forceinline__ int em_bin(const double* l, double d) {
    if (d > l[1] && d < l[3] && fabs(d - l[2]) < fabs(d - l[1]) && fabs(d - l[2]) < fabs(d - l[3])) return 2;
    const int idx = go_search(l, d);
    if (idx == 0) return 0;
    if (idx == glem::kCN) return glem::kCN - 1;
    return fabs(d - l[idx]) < fabs(d - l[idx - 1]) ? idx : idx - 1;
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// the k-th smallest (0-based) of row[0, S) as float32 bits; all values have the sign bit clear
__device__ __forceinline__ unsigned warp_select(const float* __restrict__ row, int S, unsigned k, int lane) {
    unsigned prefix = 0;
    for (int b = 30; b >= 0; b--) {
        const unsigned hi_mask = ~((2u << b) - 1u);
        unsigned cnt = 0;
        for (int i = lane; i < S; i += 32) {
            const unsigned v = __float_as_uint(row[i]);
            cnt += (v & hi_mask) == prefix && !((v >> b) & 1u);
        }
        cnt = __reduce_add_sync(kFull, cnt);
        if (k >= cnt) { k -= cnt; prefix |= 1u << b; }
    }
    return prefix;
}

// mean64 of bin b under the centres l (shared), exactly as the reference's sequential float64 sum; *cnt = the bin's size
__device__ __forceinline__ double bin_mean(const float* __restrict__ row, int S, const double* l, int b, int lane, int& cnt,
                           unsigned long long* ctr) {
    int c = 0, lo = INT_MAX, hi = INT_MIN;
    double s = 0.0;
    for (int i = lane; i < S; i += 32) {
        const float f = row[i];
        const double d = f;
        if (em_bin(l, d) != b) continue;
        c++;
        s += d;
        int a, z;
        if (glem::f32_span(__float_as_uint(f), a, z)) { lo = min(lo, a); hi = max(hi, z); }
    }
    c = __reduce_add_sync(kFull, c);
    lo = __reduce_min_sync(kFull, lo);
    hi = __reduce_max_sync(kFull, hi);
    s = warp_sum(s);
    if (!glem::sum_exact(lo, hi, c)) {                           // the order matters: sum in sample order
        if (lane == 0) {
            s = 0.0;
            for (int i = 0; i < S; i++) {
                const double d = row[i];
                if (em_bin(l, d) == b) s += d;
            }
            atomicAdd(&ctr[2], 1ull);
        }
        s = __shfl_sync(kFull, s, 0);
    }
    cnt = c;
    return c ? s / (double)c : 0.0;
}

// exponent of pmf(k, mu) = Exp(k Log(mu) - Lgamma(k + 1) - mu) (stats.go:14-23) and a bound on how far any faithful Log and
// Lgamma (within 4 ulp) can move it; returns true when the pmf is NaN (Log(0) * 0)
__device__ __forceinline__ bool pmf_exponent(double k, double mu, double lg, double& v, double& e) {
    if (mu == 0) { v = -CUDART_INF; e = 0; return k == 0; }
    const double t = k * log(mu);
    v = t - lg - mu;
    e = 0x1p-46 * (fabs(t) + fabs(lg) + mu) + 1e-300;
    return false;
}

// adjustCN's test pmf(k, mu1) * 0.9 < pmf(k, mu2) (emdepth.go:293-304); *unc when the bounds do not decide it
__device__ __forceinline__ bool pmf_less(long long k, double mu1, double mu2, bool& unc) {
    const double kd = (double)k, lg = lgamma((double)(k + 1));
    double a, ea, b, eb;
    if (pmf_exponent(kd, mu1, lg, a, ea) | pmf_exponent(kd, mu2, lg, b, eb)) return false;
    const double alo = a - ea, ahi = a + ea, blo = b - eb, bhi = b + eb;
    if (bhi < -750) return false;                                // o2 underflows to 0: o * 0.9 < 0 is false
    if (ahi < -750) {                                            // o is 0: true when o2 is a normal number
        if (blo > -700) return true;
    } else if (alo > -700 && blo > -700 && ahi < 700 && bhi < 700) {
        if (blo - ahi > kLn09 + 1e-12) return true;
        if (bhi - alo < kLn09 - 1e-12) return false;
    }
    unc = true;
    return 0.9 * exp(a) < exp(b);
}

// sign of log2(q) - t, from q against c = 2^t; inside the band the device's log2 decides and *unc is set
__device__ __forceinline__ int fc_side(double q, double c, double t, bool& unc) {
    if (q > c * (1 + kRel)) return 1;
    if (q < c * (1 - kRel)) return -1;
    unc = true;
    const double f = log2(q);
    return f > t ? 1 : (f < t ? -1 : 0);
}

__global__ void __launch_bounds__(kWarps * 32, 2) emdepth_kernel(const float* __restrict__ x, long long n, long long ld, int S,
                                                            uint8_t* __restrict__ cells, double* __restrict__ lam_out,
                                                            unsigned long long* __restrict__ ctr) {
    __shared__ double sh[kWarps][glem::kCN];
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    double* sl = sh[w];
    for (long long r = (long long)blockIdx.x * kWarps + w; r < n; r += (long long)gridDim.x * kWarps) {
        const float* row = x + r * ld;
        bool bad = false;
        for (int i = lane; i < S; i += 32) bad |= __float_as_uint(row[i]) >= kBadBits;
        if (__any_sync(kFull, bad)) {
            if (lane == 0) atomicMin(&ctr[0], (unsigned long long)r);
            continue;
        }
        double m;                                                // median32 (emdepth.go:18-29)
        if (S & 1) {
            m = __uint_as_float(warp_select(row, S, (unsigned)S / 2, lane));
        } else {
            const double lo = __uint_as_float(warp_select(row, S, (unsigned)S / 2, lane));
            const double hi = __uint_as_float(warp_select(row, S, (unsigned)S / 2 + 1, lane));
            m = (lo + hi) / 2;
        }
        double l[glem::kCN], last[glem::kCN];
        l[0] = 0.01 * m;
        l[2] = m;
#pragma unroll
        for (int i = 1; i < glem::kCN; i++)
            if (i != 2) l[i] = l[2] * glem::pow_factor(i);
        last[0] = l[0];
        double sumd = 100, maxd = 100;
        for (int it = 0; it < glem::kMaxIter && sumd > 0.01 && maxd > 0.5; it++) {
#pragma unroll
            for (int i = 1; i < glem::kCN; i++) last[i] = l[i];
            __syncwarp();
            if (lane == 0) {
#pragma unroll
                for (int i = 0; i < glem::kCN; i++) sl[i] = l[i];
            }
            __syncwarp();
            int c2;
            l[2] = bin_mean(row, S, sl, 2, lane, c2, ctr);
            if (l[2] == 0) {                                     // emdepth.go:181-192, bins as assigned above
                double mb[glem::kCN - 1];
                int cb[glem::kCN - 1];
#pragma unroll
                for (int i = 1; i < glem::kCN - 1; i++) mb[i] = bin_mean(row, S, sl, i, lane, cb[i], ctr);
                const double nn = (double)S;
#pragma unroll
                for (int i = 1; i < glem::kCN - 1; i++) {
                    const double pdepth = (double)cb[i] / nn;
                    if (l[i] < 0.01) l[i] = 0.01;
                    l[2] += mb[i] * (2 / (double)i) * pdepth;
                }
            }
#pragma unroll
            for (int i = 1; i < glem::kCN; i++) l[i] = l[2] * ((double)i / 2);
            const double span = l[2] - l[1];
            l[1] -= span / 1.5;
            l[3] += span / 1.5;
            sumd = 0; maxd = 0;                                  // summaxdiff
#pragma unroll
            for (int i = 0; i < glem::kCN; i++) {
                const double d = fabs(l[i] - last[i]);
                sumd += d;
                if (d > maxd) maxd = d;
            }
        }
        __syncwarp();
        if (lane == 0) {
#pragma unroll
            for (int i = 0; i < glem::kCN; i++) sl[i] = l[i];
        }
        __syncwarp();
        if (lam_out && lane < glem::kCN) lam_out[r * glem::kCN + lane] = sl[lane];
        unsigned n_unc = 0;
        for (int i = lane; i < S; i += 32) {
            const double d = row[i];
            bool unc = false;
            const int idx = go_search(sl, d);                    // Type (emdepth.go:272-289)
            int cn = idx == 0 ? 0 : idx == glem::kCN ? glem::kCN : (fabs(d - sl[idx]) < fabs(d - sl[idx - 1]) ? idx : idx - 1);
            if (cn != 2 && cn < glem::kCN && pmf_less((long long)(0.5 + d), sl[cn], l[2], unc)) cn = 2;
            const double q = d / l[2];                           // Log2FC = Log2(q)
            int cls;
            bool outside;
            if (q != q) {
                cls = glem::kNaN;
                outside = true;
            } else {
                const int s08 = fc_side(q, kQm08, -0.8, unc), s04 = fc_side(q, kQ04, 0.4, unc);
                cls = s08 <= 0 ? glem::kLo : (s04 >= 0 ? glem::kHi : glem::kMid);
                outside = !(fc_side(q, kQm05, -0.5, unc) > 0 && fc_side(q, kQ03, 0.3, unc) < 0);
            }
            cells[r * S + i] = glem::cell(cn, cls, outside);
            n_unc += unc;
        }
        n_unc = __reduce_add_sync(kFull, n_unc);
        if (lane == 0 && n_unc) atomicAdd(&ctr[1], (unsigned long long)n_unc);
    }
}

int check_shape(gl_ctx* ctx, const char* fn, int64_t n, int64_t ld, int32_t S) {
    if (n < 0 || S < 1 || ld < S) return gl_fail(ctx, GL_EINVAL, "%s: bad argument", fn);
    if (S == 2) return gl_fail(ctx, GL_EINVAL, "%s: 2 samples: the reference's median32 indexes past the end of 2 values", fn);
    if (S > glem::kMaxSamples) return gl_fail(ctx, GL_EINVAL, "%s: %d samples; at most %d", fn, S, glem::kMaxSamples);
    return GL_OK;
}

// rows [0, n) of d_x; the counters d_ctr[3] are the caller's; rows are named from row0 in messages
int em_block(gl_ctx* ctx, const float* d_x, int64_t n, int64_t ld, int32_t S, uint8_t* d_cells, double* d_lambda,
             unsigned long long* d_ctr, int64_t row0) {
    if (n == 0) return GL_OK;
    GL_CUDA(ctx, cudaMemsetAsync(d_ctr, 0xff, sizeof(unsigned long long), ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(d_ctr + 1, 0, 2 * sizeof(unsigned long long), ctx->stream));
    {
        gl_prof_scope prof(ctx, "emdepth_kernel");
        const unsigned blocks = (unsigned)std::min<long long>((n + kWarps - 1) / kWarps, (long long)ctx->sm_count * 64);
        emdepth_kernel<<<blocks, kWarps * 32, 0, ctx->stream>>>(d_x, (long long)n, (long long)ld, S, d_cells, d_lambda, d_ctr);
    }
    GL_LAUNCHED(ctx, 1);
    unsigned long long h[3];
    GL_CUDA(ctx, cudaMemcpyAsync(h, d_ctr, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h[0] != ~0ull)
        return gl_fail(ctx, GL_EINVAL, "emdepth: row %lld has a negative, non-finite or too large (>= 2^62) value", (long long)(row0 + (int64_t)h[0]));
    ctx->em_rows += n;
    ctx->em_uncertified += (int64_t)h[1];
    ctx->em_sequential += (int64_t)h[2];
    return GL_OK;
}

}  // namespace

extern "C" {

int gl_emdepth_device(gl_ctx* ctx, const float* d_x, int64_t n, int64_t ld, int32_t S, uint8_t* d_cells, double* d_lambda) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(check_shape(ctx, "gl_emdepth_device", n, ld, S));
    if (n > 0 && (!d_x || !d_cells)) return gl_fail(ctx, GL_EINVAL, "gl_emdepth_device: bad argument");
    ctx->em_rows = ctx->em_uncertified = ctx->em_sequential = 0;
    gl_scratch tmp(ctx);
    unsigned long long* d_ctr;
    GL_CHECK(tmp.alloc(d_ctr, 3));
    return em_block(ctx, d_x, n, ld, S, d_cells, d_lambda, d_ctr, 0);
}

int gl_emdepth(gl_ctx* ctx, const float* x, int64_t n, int64_t ld, int32_t S, int64_t block_rows, uint8_t* cells, double* lambda) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(check_shape(ctx, "gl_emdepth", n, ld, S));
    if (block_rows < 0 || (n > 0 && (!x || !cells))) return gl_fail(ctx, GL_EINVAL, "gl_emdepth: bad argument");
    ctx->em_rows = ctx->em_uncertified = ctx->em_sequential = 0;
    if (n == 0) return GL_OK;
    const double per_row = 5.0 * S + (lambda ? 8.0 * glem::kCN : 0.0);   // float32 in, one byte out, the centres
    int64_t br = block_rows;
    if (br == 0) {
        size_t free_b = 0, total_b = 0;
        GL_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
        br = (int64_t)std::min<double>((double)n, 0.8 * (double)free_b / per_row);
        if (br < 1) return gl_fail(ctx, GL_ENOMEM, "gl_emdepth: one row of %d samples does not fit in device memory", S);
    }
    br = std::min(br, n);
    gl_scratch tmp(ctx);
    float* d_x; uint8_t* d_cells; double* d_lam = nullptr; unsigned long long* d_ctr;
    GL_CHECK(tmp.alloc(d_x, (size_t)br * S));
    GL_CHECK(tmp.alloc(d_cells, (size_t)br * S));
    if (lambda) GL_CHECK(tmp.alloc(d_lam, (size_t)br * glem::kCN));
    GL_CHECK(tmp.alloc(d_ctr, 3));
    for (int64_t r0 = 0; r0 < n; r0 += br) {
        const int64_t nb = std::min(br, n - r0);
        GL_CUDA(ctx, cudaMemcpy2DAsync(d_x, (size_t)S * 4, x + r0 * ld, (size_t)ld * 4, (size_t)S * 4, (size_t)nb, cudaMemcpyHostToDevice, ctx->stream));
        GL_CHECK(em_block(ctx, d_x, nb, S, S, d_cells, d_lam, d_ctr, r0));
        GL_CUDA(ctx, cudaMemcpyAsync(cells + r0 * S, d_cells, (size_t)(nb * S), cudaMemcpyDeviceToHost, ctx->stream));
        if (lambda) GL_CUDA(ctx, cudaMemcpyAsync(lambda + r0 * glem::kCN, d_lam, (size_t)nb * glem::kCN * 8, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return GL_OK;
}

int gl_emdepth_stats(gl_ctx* ctx, int64_t* n_rows, int64_t* n_uncertified, int64_t* n_sequential) {
    if (!ctx) return gl_fail(nullptr, GL_EINVAL, "null ctx");
    if (n_rows) *n_rows = ctx->em_rows;
    if (n_uncertified) *n_uncertified = ctx->em_uncertified;
    if (n_sequential) *n_sequential = ctx->em_sequential;
    return GL_OK;
}

int gl_emdepth_factors(double* f9) {
    if (!f9) return GL_EINVAL;
    for (int i = 0; i < glem::kCN; i++) f9[i] = glem::pow_factor(i);
    return GL_OK;
}

}  // extern "C"
