// dcnv.cu — `goleft dcnv` (dcnv/dcnv.go:323-354): GC-debias and median-normalise an n-sites x S-samples depth matrix.
//
// The reference, per sample column c of the matrix with its rows in GC order (inds = Go's argsort of the GC fractions,
// host/dcnv.cpp):
//   Debias (debiaser.go:98-123, Window 9, mid 5) pushes c[0..4] into a moving median of 9, then c[i+5] for i in [5, n-5),
//   and divides row i by max(median, 1) of the window after its pushes.  So c[5..9] are never pushed, and with
//   p = c[0..4] ++ c[10..n-1] row i divides by the median of p[max(0, j-8) .. j], j = clamp(i, 4, max(4, n-6)): the
//   first five rows by the median of p[0..4], the last rows by the final window.  Every window holds values that have not
//   been divided yet, so each (row, sample) is independent.  An even count (6 or 8 values, sorted rows 5 and 7 only)
//   takes (lo + hi) / 2, restating JaderDias/movingmedian (not in the reference tree: UNPINNED).
//   NormalizeBySampleMedian (dcnv.go:108-136), after Unsort: sort the column, k = its leading exact zeros (0 when a
//   value is negative), median = sorted[k + int(0.65 * float64(n - k))], every cell / median.
//
// Kernels (columns [c0, c1) of a row-major matrix with leading dimension ld; the caller streams column blocks):
//   dcnv_debias_kernel  a CTA gathers the p-rows its 64 sorted rows need x 32 samples through inds into shared memory (reads
//                       along samples are coalesced), sorts each window of <= 9 in registers, and writes x / max(med, 1) to
//                       the ORIGINAL row inds[i] (that is Unsort) plus an order-preserving key, column-major, for the select.
//   dcnv_select_kernel  a CTA per sample: zeros and negatives give the rank, then an exact 8-pass radix select over the keys.
//   dcnv_divide_kernel  every cell / its sample's median (__ddiv_rn; the library builds with --fmad=false).
//   fmt_f2_kernel       "%.2f" tokens (host/f2_token.h).
#include <math_constants.h>
#include "gl_common.cuh"
#include "host/f2_token.h"

namespace {

constexpr int kDbRows = 64;        // sorted rows per debias CTA
constexpr int kDbCols = 32;        // samples per debias CTA (one warp across a row)
constexpr int kDbWarps = 8;
constexpr int kSelThreads = 1024;
constexpr unsigned long long kZeroKey = 0x8000000000000000ull;

// order-preserving key of a float64 (-0 and +0 share a key: the reference compares with == 0 and <)
__device__ __forceinline__ unsigned long long f64_key(double v) {
    unsigned long long b = (unsigned long long)__double_as_longlong(v);
    if (b == kZeroKey) b = 0;
    return (b >> 63) ? ~b : (b | kZeroKey);
}

__device__ __forceinline__ double key_f64(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & ~kZeroKey) : ~k));
}

__device__ __forceinline__ void cas(double& a, double& b) { const double lo = fmin(a, b), hi = fmax(a, b); a = lo; b = hi; }

__global__ void __launch_bounds__(kDbCols * kDbWarps) dcnv_debias_kernel(const double* __restrict__ x, long long ld, const long long* __restrict__ inds,
                                                                       long long n, int nc, double* __restrict__ out, long long ld_out,
                                                                       unsigned long long* __restrict__ keys) {
    __shared__ double pv[kDbRows + 8][kDbCols];
    const long long i0 = (long long)blockIdx.x * kDbRows;
    const long long i1 = min(n, i0 + kDbRows) - 1;
    const long long jmax = max(4ll, n - 6);
    const long long q_lo = max(0ll, min(max(i0, 4ll), jmax) - 8);
    const long long q_hi = min(max(i1, 4ll), jmax);
    const int col = blockIdx.y * kDbCols + threadIdx.x;
    const bool ok = col < nc;
    for (long long q = q_lo + threadIdx.y; q <= q_hi; q += kDbWarps) {
        const long long sr = q < 5 ? q : q + 5;                  // p-row q is sorted row sr
        if (ok) pv[q - q_lo][threadIdx.x] = x[inds[sr] * ld + col];
    }
    __syncthreads();
    if (!ok) return;
    for (long long i = i0 + threadIdx.y; i <= i1; i += kDbWarps) {
        const long long j = min(max(i, 4ll), jmax);
        const long long lo = max(0ll, j - 8);
        const int m = (int)(j - lo + 1);                         // 5..9 values
        double w[9];
#pragma unroll
        for (int k = 0; k < 9; k++) w[k] = k < m ? pv[lo - q_lo + k][threadIdx.x] : CUDART_INF;
#pragma unroll
        for (int r = 0; r < 9; r++) {                            // odd-even transposition: 9 rounds sort 9 values
#pragma unroll
            for (int k = r & 1; k + 1 < 9; k += 2) cas(w[k], w[k + 1]);
        }
        double med;
        if (m == 9) med = w[4];
        else if (m == 8) med = __ddiv_rn(__dadd_rn(w[3], w[4]), 2.0);
        else if (m == 7) med = w[3];
        else if (m == 6) med = __ddiv_rn(__dadd_rn(w[2], w[3]), 2.0);
        else med = w[2];
        const long long row = inds[i];
        const double v = __ddiv_rn(x[row * ld + col], fmax(med, 1.0));
        out[row * ld_out + col] = v;
        keys[(long long)col * n + row] = f64_key(v);
    }
}

// medians[c] = the reference's sample median of column c; err = 1 + the first all-zero column (the reference panics there)
__global__ void __launch_bounds__(kSelThreads) dcnv_select_kernel(const unsigned long long* __restrict__ keys, long long n,
                                                                  double* __restrict__ medians, int* __restrict__ err) {
    __shared__ unsigned hist[256];
    __shared__ unsigned n_zero, n_neg;
    __shared__ unsigned long long s_prefix;
    __shared__ long long s_rank;
    const int c = blockIdx.x;
    const unsigned long long* k = keys + (long long)c * n;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { n_zero = 0; n_neg = 0; s_prefix = 0; s_rank = 0; }
    for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0;
    __syncthreads();
    for (int shift = 56; shift >= 0; shift -= 8) {
        const unsigned long long hi_mask = shift == 56 ? 0ull : (~0ull << (shift + 8));
        const unsigned long long prefix = s_prefix;
        unsigned zeros = 0, negs = 0;
        for (long long base = 0; base < n; base += blockDim.x) {      // uniform trip count: every lane reaches the match
            const long long i = base + threadIdx.x;
            const unsigned long long key = i < n ? k[i] : 0ull;
            const bool in = i < n && (key & hi_mask) == prefix;
            if (shift == 56 && i < n) { zeros += key == kZeroKey; negs += key < kZeroKey; }
            const unsigned act = __ballot_sync(0xffffffffu, in);
            if (in) {
                const unsigned d = (unsigned)(key >> shift) & 0xffu;
                const unsigned peers = __match_any_sync(act, d);
                if (lane == __ffs(peers) - 1) atomicAdd(&hist[d], (unsigned)__popc(peers));
            }
        }
        if (shift == 56) {
            zeros = __reduce_add_sync(0xffffffffu, zeros);
            negs = __reduce_add_sync(0xffffffffu, negs);
            if (lane == 0) { atomicAdd(&n_zero, zeros); atomicAdd(&n_neg, negs); }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long long t = s_rank;
            if (shift == 56) {                                   // dcnv.go:118-122
                const long long kz = n_neg ? 0 : (long long)n_zero;
                t = kz + (long long)__dmul_rn(0.65, (double)(n - kz));
                if (kz == n) { atomicMin(err, c + 1); t = -1; }
            }
            if (t >= 0) {
                unsigned long long cum = 0;
                int d = 0;
                for (; d < 255 && cum + hist[d] <= (unsigned long long)t; d++) cum += hist[d];
                s_prefix = prefix | ((unsigned long long)d << shift);
                t -= (long long)cum;
            }
            s_rank = t;
        }
        __syncthreads();
        if (s_rank < 0) break;                                   // all zero: nothing to select
        for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0;
        __syncthreads();
    }
    if (threadIdx.x == 0) medians[c] = s_rank < 0 ? CUDART_NAN : key_f64(s_prefix);
}

__global__ void __launch_bounds__(256) dcnv_divide_kernel(double* __restrict__ out, long long n, int nc, long long ld_out,
                                                         const double* __restrict__ medians) {
    const long long total = n * nc;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long r = t / nc;
        const int c = (int)(t - r * nc);
        double* p = out + r * ld_out + c;
        *p = __ddiv_rn(*p, medians[c]);
    }
}

__global__ void __launch_bounds__(256) fmt_f2_kernel(const double* __restrict__ v, long long n, uint4* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned char t[glf2::kTok];
    glf2::token(v[i], t);
    uint4 w;
    memcpy(&w, t, 16);
    out[i] = w;
}

// the three kernels over columns [c0, c1) of d_x (arguments checked by the caller); an all-zero column is reported as
// column col_name + (its index in the block)
int normalize_block(gl_ctx* ctx, const double* d_x, int64_t n, int64_t ld, const int64_t* d_inds, int32_t c0, int32_t c1,
                    double* d_out, int64_t ld_out, double* d_medians, int64_t col_name) {
    const int nc = c1 - c0;
    gl_scratch tmp(ctx);
    unsigned long long* d_keys; int* d_err;
    GL_CHECK(tmp.alloc(d_keys, (size_t)n * nc));
    GL_CHECK(tmp.alloc(d_err, 1));
    GL_CUDA(ctx, cudaMemsetAsync(d_err, 0x7f, sizeof(int), ctx->stream));
    {
        gl_prof_scope prof(ctx, "dcnv_debias_kernel");
        const dim3 grid((unsigned)((n + kDbRows - 1) / kDbRows), (unsigned)((nc + kDbCols - 1) / kDbCols));
        dcnv_debias_kernel<<<grid, dim3(kDbCols, kDbWarps), 0, ctx->stream>>>(d_x + c0, (long long)ld, reinterpret_cast<const long long*>(d_inds),
                                                                             (long long)n, nc, d_out, (long long)ld_out, d_keys);
    }
    GL_LAUNCHED(ctx, 1);
    {
        gl_prof_scope prof(ctx, "dcnv_select_kernel");
        dcnv_select_kernel<<<(unsigned)nc, kSelThreads, 0, ctx->stream>>>(d_keys, (long long)n, d_medians, d_err);
    }
    GL_LAUNCHED(ctx, 1);
    {
        gl_prof_scope prof(ctx, "dcnv_divide_kernel");
        const long long total = (long long)n * nc;
        const unsigned blocks = (unsigned)std::min<long long>((total + 255) / 256, (long long)ctx->sm_count * 16);
        dcnv_divide_kernel<<<blocks, 256, 0, ctx->stream>>>(d_out, (long long)n, nc, (long long)ld_out, d_medians);
    }
    GL_LAUNCHED(ctx, 1);
    int err = 0;
    GL_CUDA(ctx, cudaMemcpyAsync(&err, d_err, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (err != 0x7f7f7f7f)
        return gl_fail(ctx, GL_ERANGE, "dcnv: sample column %lld is all zero (the reference's median index is out of range)", (long long)(col_name + err - 1));
    return GL_OK;
}

}  // namespace

extern "C" {

int gl_dcnv_normalize_device(gl_ctx* ctx, const double* d_x, int64_t n, int64_t ld, const int64_t* d_inds, int32_t c0, int32_t c1,
                             double* d_out, int64_t ld_out, double* d_medians) {
    GL_CHECK(gl_use(ctx));
    if (!d_x || !d_inds || !d_out || !d_medians || c0 < 0 || c1 <= c0 || ld < c1 || ld_out < c1 - c0)
        return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize_device: bad argument");
    if (n < 5) return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize_device: %lld rows; the moving median needs at least 5", (long long)n);
    if (n > INT32_MAX) return gl_fail(ctx, GL_ERANGE, "gl_dcnv_normalize_device: more than 2^31-1 rows");
    return normalize_block(ctx, d_x, n, ld, d_inds, c0, c1, d_out, ld_out, d_medians, c0);
}

int gl_dcnv_normalize(gl_ctx* ctx, const double* x, int64_t n, int64_t ld, const int64_t* inds, int32_t c0, int32_t c1, int32_t block_cols,
                      double* out, int64_t ld_out, double* medians) {
    GL_CHECK(gl_use(ctx));
    const int nc = c1 - c0;
    if (!x || !inds || !out || !medians || c0 < 0 || nc < 1 || ld < c1 || ld_out < nc || block_cols < 0)
        return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize: bad argument");
    if (n < 5) return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize: %lld rows; the moving median needs at least 5", (long long)n);
    if (n > INT32_MAX) return gl_fail(ctx, GL_ERANGE, "gl_dcnv_normalize: more than 2^31-1 rows");
    {                                                            // the kernels gather through inds: it must be a permutation
        std::vector<uint8_t> seen((size_t)n, 0);
        for (int64_t i = 0; i < n; i++) {
            if (inds[i] < 0 || inds[i] >= n || seen[(size_t)inds[i]]) return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize: inds is not a permutation of [0, n)");
            seen[(size_t)inds[i]] = 1;
        }
    }
    int bw = block_cols;
    if (bw == 0) {                                               // a block's input, output and keys: 24 bytes per cell
        size_t free_b = 0, total_b = 0;
        GL_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
        const double room = 0.8 * (double)free_b - 8.0 * (double)n;
        bw = (int)std::min<double>((double)nc, room / (24.0 * (double)n));
        if (bw < 1) return gl_fail(ctx, GL_ENOMEM, "gl_dcnv_normalize: one sample column of %lld rows does not fit in device memory", (long long)n);
    }
    bw = std::min(bw, nc);
    gl_scratch tmp(ctx);
    int64_t* d_inds; double *d_x, *d_out, *d_med;
    GL_CHECK(tmp.upload(d_inds, inds, (size_t)n));
    GL_CHECK(tmp.alloc(d_x, (size_t)n * bw));
    GL_CHECK(tmp.alloc(d_out, (size_t)n * bw));
    GL_CHECK(tmp.alloc(d_med, (size_t)bw));
    for (int b0 = c0; b0 < c1; b0 += bw) {
        const int nb = std::min(bw, c1 - b0);
        GL_CUDA(ctx, cudaMemcpy2DAsync(d_x, (size_t)nb * 8, x + b0, (size_t)ld * 8, (size_t)nb * 8, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        GL_CHECK(normalize_block(ctx, d_x, n, nb, d_inds, 0, nb, d_out, nb, d_med, b0));
        GL_CUDA(ctx, cudaMemcpy2DAsync(out + (b0 - c0), (size_t)ld_out * 8, d_out, (size_t)nb * 8, (size_t)nb * 8, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaMemcpyAsync(medians + (b0 - c0), d_med, (size_t)nb * 8, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return GL_OK;
}

int gl_format_f2_device(gl_ctx* ctx, const double* d_vals, int64_t n, uint8_t* d_tokens) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || (n > 0 && (!d_vals || !d_tokens)) || ((uintptr_t)d_tokens & 15)) return gl_fail(ctx, GL_EINVAL, "gl_format_f2_device: bad argument");
    if (n == 0) return GL_OK;
    {
        gl_prof_scope prof(ctx, "fmt_f2_kernel");
        fmt_f2_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_vals, (long long)n, reinterpret_cast<uint4*>(d_tokens));
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_format_f2(gl_ctx* ctx, const double* vals, int64_t n, uint8_t* tokens) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || (n > 0 && (!vals || !tokens))) return gl_fail(ctx, GL_EINVAL, "gl_format_f2: bad argument");
    if (n == 0) return GL_OK;
    gl_scratch tmp(ctx);
    double* d_vals; uint8_t* d_tokens;
    GL_CHECK(tmp.upload(d_vals, vals, (size_t)n));
    GL_CHECK(tmp.alloc(d_tokens, (size_t)n * glf2::kTok));
    GL_CHECK(gl_format_f2_device(ctx, d_vals, n, d_tokens));
    GL_CUDA(ctx, cudaMemcpyAsync(tokens, d_tokens, (size_t)n * glf2::kTok, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

}  // extern "C"
