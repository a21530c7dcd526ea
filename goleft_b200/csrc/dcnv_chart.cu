// dcnv_chart.cu — `goleft dcnv`'s depth chart drawn on the GPU (DESIGN §1.9).
//
// Which points (dcnv/dcnv.go asValues, float64 throughout, no thinning): per sample, leading values == 0 are skipped
// (-0.0 is zero, NaN is not); every row i from the first other one on is a vertex x = float64(i) * 16384 (the row index,
// not the row's start: the reference's quirk), y = min(v, 2.5).  The line is stepped, as the page draws it: step i goes
// from (x_i, y_i) across to (x_{i+1}, y_i), then up or down to (x_{i+1}, y_{i+1}).  A step with a NaN or -Inf y at either
// end is not drawn (the page breaks its line there); the y extent is over the other vertices, with -0.0 taken as 0.0.
//
// The image is plot.cu's INDEX IMAGE with plot_rule.cuh's float64 pixel rule: sample k is drawn with index S - k, so
// sample 0 shows on top, as Chart.js 2 draws a chart's datasets last to first.
//
// The matrix is row-major on the host and goes to the device in row blocks (one when it fits).  Select: per block, the
// first non-zero row of each sample (atomicMin of row indices: blocks come in order, so the earliest wins) and then the
// min / max of the plotted y over the block's rows from that row on (atomicMin / atomicMax of order-preserving keys).
// Raster: a CTA owns one sample's steps in one row range.  Every pixel its steps cover gets the same value (S - k), so it
// marks them in a shared-memory bitmap of the data area, skipping the exact test where the bit is already set, and then
// flushes each set bit with one atomicMax into the image.  OR and max do not depend on order, so neither the row blocks
// nor the CTA shape change a bit of the image.
#include "gl_common.cuh"
#include "plot_rule.cuh"
#include "host/thread_pool.h"
#include <float.h>
#include <math.h>
#include <string.h>
#include <mutex>

namespace {

using glplot::draw_segment;
using glplot::p_mul;

constexpr double kCnMax = 2.5;            // dcnv.go:218 cnMax
constexpr double kMult = 16384.0;         // dcnv.go:298 asValues(depth, 16384)
constexpr int kThreads = 256;
constexpr int64_t kRowsPerCta = 8192;
constexpr int64_t kMaxBitmapPx = 48 * 1024 * 8;     // the data area's bitmap fits the default 48 KB of shared memory
constexpr unsigned long long kNone = ~0ull;         // no non-zero row seen yet

__host__ __device__ inline double cap(double v) { return v > kCnMax ? kCnMax : v; }
// a plotted y that is drawn: not NaN, not -Inf (+Inf is capped to 2.5)
__host__ __device__ inline bool drawn_y(double y) { return y >= -DBL_MAX; }

// a monotone uint64 key of a double that is not NaN (-0.0 as 0.0), and back
__host__ __device__ inline unsigned long long okey(double y) {
    if (y == 0.0) y = 0.0;
#ifdef __CUDA_ARCH__
    const unsigned long long u = (unsigned long long)__double_as_longlong(y);
#else
    unsigned long long u;
    memcpy(&u, &y, 8);
#endif
    return (u >> 63) ? ~u : (u | (1ull << 63));
}
inline double okey_inv(unsigned long long k) {
    const unsigned long long u = (k >> 63) ? (k & ~(1ull << 63)) : ~k;
    double y;
    memcpy(&y, &u, 8);
    return y;
}

// the rows of one CTA: [a, b) of [0, n), with at most 65535 CTAs along y
inline int64_t rows_per_cta(int64_t n) { return std::max<int64_t>(kRowsPerCta, (n + 65534) / 65535); }

// blockIdx = (sample k, row range): first[k] = min(first[k], row0 + the first row != 0 of the range)
__global__ void __launch_bounds__(kThreads) dc_first_kernel(const double* __restrict__ X, int64_t row0, int64_t rows, int S, int64_t per,
                                                            unsigned long long* __restrict__ first) {
    __shared__ unsigned long long s_first;
    const int k = blockIdx.x;
    if (first[k] < (unsigned long long)row0) return;                      // found in an earlier block
    if (threadIdx.x == 0) s_first = kNone;
    __syncthreads();
    const int64_t a = (int64_t)blockIdx.y * per, b = min(rows, a + per);
    for (int64_t i = a + threadIdx.x; i < b; i += blockDim.x)
        if (X[i * S + k] != 0.0) { atomicMin(&s_first, (unsigned long long)(row0 + i)); break; }   // NaN != 0: it ends the skip
    __syncthreads();
    if (threadIdx.x == 0 && s_first != kNone) atomicMin(&first[k], s_first);
}

// blockIdx = (sample k, row range): lo[k], hi[k] take the keys of the min and max drawn y over the range's rows >= first[k]
__global__ void __launch_bounds__(kThreads) dc_ext_kernel(const double* __restrict__ X, int64_t row0, int64_t rows, int S, int64_t per,
                                                          const unsigned long long* __restrict__ first, unsigned long long* __restrict__ lo_key,
                                                          unsigned long long* __restrict__ hi_key) {
    __shared__ double s_lo[kThreads / 32], s_hi[kThreads / 32];
    const int k = blockIdx.x;
    const unsigned long long f = first[k];
    if (f >= (unsigned long long)(row0 + rows)) return;                   // no plotted row in this block
    int64_t a = (int64_t)blockIdx.y * per;
    const int64_t b = min(rows, a + per);
    a = max(a, (int64_t)f - row0);
    double lo = INFINITY, hi = -INFINITY;
    for (int64_t i = a + threadIdx.x; i < b; i += blockDim.x) {
        const double y = cap(X[i * S + k]);
        if (drawn_y(y)) { lo = fmin(lo, y); hi = fmax(hi, y); }
    }
    for (int o = 16; o > 0; o >>= 1) { lo = fmin(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = fmax(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    if ((threadIdx.x & 31) == 0) { s_lo[threadIdx.x >> 5] = lo; s_hi[threadIdx.x >> 5] = hi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kThreads / 32; w++) { lo = fmin(lo, s_lo[w]); hi = fmax(hi, s_hi[w]); }
        if (lo <= hi) { atomicMin(&lo_key[k], okey(lo)); atomicMax(&hi_key[k], okey(hi)); }
    }
}

// blockIdx = (sample k, step range): the steps i >= first[k] with rows i and i + 1 both in the block (rows row_lo ..
// row_lo + rows - 1 at X), marked in a shared bitmap of the W x H data area, then flushed into img with index S - k
__global__ void __launch_bounds__(kThreads, 2) dc_raster_kernel(const double* __restrict__ X, int64_t row_lo, int64_t rows, int S, int64_t per,
                                                             const int64_t* __restrict__ first, const double* __restrict__ xf, int W, int H,
                                                             double r, double r2, uint32_t* __restrict__ img) {
    extern __shared__ unsigned int bm[];
    const int k = blockIdx.x;
    const int64_t s1 = min(row_lo + rows - 1, row_lo + (int64_t)blockIdx.y * per + per);
    const int64_t s0 = max(row_lo + (int64_t)blockIdx.y * per, first[k]);
    if (s0 >= s1) return;
    const int words = (W * H + 31) / 32;
    for (int w = threadIdx.x; w < words; w += blockDim.x) bm[w] = 0;
    __syncthreads();
    volatile unsigned int* vbm = bm;
    auto skip = [vbm, W](int i, int j) { const int p = j * W + i; return (vbm[p >> 5] >> (p & 31)) & 1u; };
    auto mark = [W](int i, int j) { const int p = j * W + i; atomicOr(&bm[p >> 5], 1u << (p & 31)); };
    for (int64_t i = s0 + threadIdx.x; i < s1; i += blockDim.x) {
        const double y0 = cap(X[(i - row_lo) * S + k]), y1 = cap(X[(i + 1 - row_lo) * S + k]);
        if (!drawn_y(y0) || !drawn_y(y1)) continue;
        const double x0 = p_mul((double)i, kMult), x1 = p_mul((double)(i + 1), kMult);
        draw_segment(x0, y0, x1, y0, xf, W, H, r, r2, skip, mark);
        draw_segment(x1, y0, x1, y1, xf, W, H, r, r2, skip, mark);
    }
    __syncthreads();
    const uint32_t idx = (uint32_t)(S - k);
    for (int w = threadIdx.x; w < words; w += blockDim.x) {
        for (unsigned int bits = bm[w]; bits; bits &= bits - 1) {
            unsigned int* p = reinterpret_cast<unsigned int*>(img + (int64_t)w * 32 + (__ffs(bits) - 1));
            if (__ldcg(p) < idx) atomicMax(p, idx);
        }
    }
}

int check_args(gl_ctx* ctx, const char* fn, const double* x, int64_t n, int64_t S) {
    if (n < 0 || S < 1 || S > INT32_MAX || (n > 0 && !x)) return gl_fail(ctx, GL_EINVAL, "%s: bad argument", fn);
    return GL_OK;
}

int check_image(gl_ctx* ctx, const char* fn, int32_t W, int32_t H, double r, const void* img) {
    if (W < 1 || H < 1 || (int64_t)W * H > kMaxBitmapPx || !(r > 0) || !img)
        return gl_fail(ctx, GL_EINVAL, "%s: bad image (W %d, H %d, r %g)", fn, W, H, r);
    return GL_OK;
}

// the host mirror of one sample's select
void select_one(const double* x, int64_t n, int64_t S, int64_t k, int64_t& first, double* yext2) {
    int64_t f = 0;
    while (f < n && x[f * S + k] == 0.0) f++;
    double lo = INFINITY, hi = -INFINITY;
    for (int64_t i = f; i < n; i++) {
        double y = cap(x[i * S + k]);
        if (!drawn_y(y)) continue;
        if (y == 0.0) y = 0.0;
        lo = std::min(lo, y); hi = std::max(hi, y);
    }
    first = f; yext2[0] = lo; yext2[1] = hi;
}

}  // namespace

extern "C" {

int gl_dcnv_chart_select_host(const double* x, int64_t n, int64_t S, int64_t* first, double* yext2) {
    GL_CHECK(check_args(nullptr, "gl_dcnv_chart_select_host", x, n, S));
    if (!first || !yext2) return gl_fail(nullptr, GL_EINVAL, "gl_dcnv_chart_select_host: bad argument");
    glhost::ThreadPool::global().run(S, [&](int64_t k, int) { select_one(x, n, S, k, first[k], yext2 + 2 * k); });
    return GL_OK;
}

int gl_dcnv_chart_extent(const int64_t* first, const double* yext2, int64_t n, int64_t S, double* ext4) {
    if (n < 0 || S < 1 || !first || !yext2 || !ext4) return gl_fail(nullptr, GL_EINVAL, "gl_dcnv_chart_extent: bad argument");
    double e[4] = {INFINITY, -INFINITY, INFINITY, -INFINITY};
    for (int64_t k = 0; k < S; k++) {
        if (first[k] >= n) continue;
        e[0] = std::min(e[0], (double)first[k] * kMult);
        e[1] = (double)(n - 1) * kMult;
        if (yext2[2 * k] <= yext2[2 * k + 1]) { e[2] = std::min(e[2], yext2[2 * k]); e[3] = std::max(e[3], yext2[2 * k + 1]); }
    }
    if (e[0] > e[1]) e[0] = e[1] = 0;                                     // no vertex
    if (e[2] > e[3]) e[2] = e[3] = 0;                                     // no drawn y
    memcpy(ext4, e, sizeof e);
    return GL_OK;
}

int gl_dcnv_chart_raster_host(const double* x, int64_t n, int64_t S, const int64_t* first, const double* xf4, int32_t W, int32_t H,
                              double r, uint32_t* img) {
    GL_CHECK(check_args(nullptr, "gl_dcnv_chart_raster_host", x, n, S));
    GL_CHECK(check_image(nullptr, "gl_dcnv_chart_raster_host", W, H, r, img));
    if (!first || !xf4) return gl_fail(nullptr, GL_EINVAL, "gl_dcnv_chart_raster_host: bad argument");
    const size_t px = (size_t)W * H;
    memset(img, 0, px * 4);
    const double r2 = r * r;
    const int64_t per = (int64_t)1 << 18, chunks = std::max<int64_t>(1, (n + per - 1) / per);
    std::mutex mu;
    glhost::ThreadPool::global().run(S * chunks, [&](int64_t t, int) {
        const int64_t k = t / chunks, s0 = std::max((t % chunks) * per, first[k]), s1 = std::min((t % chunks + 1) * per, n - 1);
        if (s0 >= s1) return;
        std::vector<uint8_t> cov(px, 0);
        auto skip = [&](int i, int j) { return cov[(size_t)j * W + i] != 0; };
        auto mark = [&](int i, int j) { cov[(size_t)j * W + i] = 1; };
        for (int64_t i = s0; i < s1; i++) {
            const double y0 = cap(x[i * S + k]), y1 = cap(x[(i + 1) * S + k]);
            if (!drawn_y(y0) || !drawn_y(y1)) continue;
            const double x0 = (double)i * kMult, x1 = (double)(i + 1) * kMult;
            draw_segment(x0, y0, x1, y0, xf4, W, H, r, r2, skip, mark);
            draw_segment(x1, y0, x1, y1, xf4, W, H, r, r2, skip, mark);
        }
        const uint32_t idx = (uint32_t)(S - k);
        std::lock_guard<std::mutex> g(mu);
        for (size_t p = 0; p < px; p++)
            if (cov[p] && img[p] < idx) img[p] = idx;
    });
    return GL_OK;
}

int gl_dcnv_chart(gl_ctx* ctx, const double* x, int64_t n, int64_t S, int64_t block_rows, int32_t W, int32_t H, double r, int64_t* first,
                  double* yext2, double* ext4, uint32_t* img) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(check_args(ctx, "gl_dcnv_chart", x, n, S));
    GL_CHECK(check_image(ctx, "gl_dcnv_chart", W, H, r, img));
    if (block_rows < 0 || !first || !yext2 || !ext4) return gl_fail(ctx, GL_EINVAL, "gl_dcnv_chart: bad argument");
    int64_t br = block_rows;
    if (br == 0) {
        size_t free_b = 0, total_b = 0;
        GL_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
        const double fit = 0.8 * (double)free_b / (8.0 * (double)S) - 1;   // a block holds one row more than it adds
        if (fit < 1) return gl_fail(ctx, GL_ENOMEM, "gl_dcnv_chart: two rows of %lld samples do not fit in device memory", (long long)S);
        br = (int64_t)std::min<double>((double)n, fit);
    }
    br = std::max<int64_t>(1, std::min(br, n));
    const size_t px = (size_t)W * H;
    gl_scratch tmp(ctx);
    double *d_x, *d_xf;
    unsigned long long *d_first, *d_lo, *d_hi;
    uint32_t* d_img;
    GL_CHECK(tmp.alloc(d_x, (size_t)(br + 1) * S));                    // a raster block also holds the row before it
    GL_CHECK(tmp.alloc(d_first, (size_t)S));
    GL_CHECK(tmp.alloc(d_lo, (size_t)S));
    GL_CHECK(tmp.alloc(d_hi, (size_t)S));
    GL_CHECK(tmp.alloc(d_xf, 4));
    GL_CHECK(tmp.alloc(d_img, px));
    GL_CUDA(ctx, cudaMemsetAsync(d_first, 0xFF, (size_t)S * 8, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(d_lo, 0xFF, (size_t)S * 8, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(d_hi, 0, (size_t)S * 8, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(d_img, 0, px * 4, ctx->stream));
    auto upload = [&](int64_t r0, int64_t nr) -> int {
        GL_CUDA(ctx, cudaMemcpyAsync(d_x, x + r0 * S, (size_t)(nr * S) * 8, cudaMemcpyHostToDevice, ctx->stream));
        return GL_OK;
    };
    // ---- select, one pass over the row blocks in order
    for (int64_t r0 = 0; r0 < n; r0 += br) {
        const int64_t nr = std::min(br, n - r0), per = rows_per_cta(nr);
        GL_CHECK(upload(r0, nr));
        const dim3 grid((unsigned)S, (unsigned)((nr + per - 1) / per));
        {
            gl_prof_scope prof(ctx, "dc_first_kernel");
            dc_first_kernel<<<grid, kThreads, 0, ctx->stream>>>(d_x, r0, nr, (int)S, per, d_first);
        }
        {
            gl_prof_scope prof(ctx, "dc_ext_kernel");
            dc_ext_kernel<<<grid, kThreads, 0, ctx->stream>>>(d_x, r0, nr, (int)S, per, d_first, d_lo, d_hi);
        }
        GL_LAUNCHED(ctx, 2);
    }
    std::vector<unsigned long long> f((size_t)S), lo((size_t)S), hi((size_t)S);
    GL_CUDA(ctx, cudaMemcpyAsync(f.data(), d_first, (size_t)S * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(lo.data(), d_lo, (size_t)S * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(hi.data(), d_hi, (size_t)S * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int64_t k = 0; k < S; k++) {
        first[k] = f[k] == kNone ? n : (int64_t)f[k];
        const bool any = lo[k] != kNone;
        yext2[2 * k] = any ? okey_inv(lo[k]) : INFINITY;
        yext2[2 * k + 1] = any ? okey_inv(hi[k]) : -INFINITY;
    }
    GL_CHECK(gl_dcnv_chart_extent(first, yext2, n, S, ext4));
    double xf[4];
    GL_CHECK(gl_plot_transform(ext4, W, H, xf));
    // ---- raster: block b holds its rows and the row before, so every step is drawn by exactly one block
    int64_t* d_fr = reinterpret_cast<int64_t*>(d_first);
    GL_CUDA(ctx, cudaMemcpyAsync(d_fr, first, (size_t)S * 8, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(d_xf, xf, 32, cudaMemcpyHostToDevice, ctx->stream));
    const int smem = (int)((px + 31) / 32 * 4);
    for (int64_t r0 = 0; r0 < n; r0 += br) {
        const int64_t lo_row = r0 > 0 ? r0 - 1 : 0, nr = std::min(r0 + br, n) - lo_row;
        if (nr < 2) continue;
        if (r0 > 0 || br < n) GL_CHECK(upload(lo_row, nr));                 // one block: still on the device from the select
        const int64_t per = rows_per_cta(nr - 1);
        const dim3 grid((unsigned)S, (unsigned)((nr - 1 + per - 1) / per));
        gl_prof_scope prof(ctx, "dc_raster_kernel");
        dc_raster_kernel<<<grid, kThreads, smem, ctx->stream>>>(d_x, lo_row, nr, (int)S, per, d_fr, d_xf, W, H, r, r * r, d_img);
        GL_LAUNCHED(ctx, 1);
    }
    GL_CUDA(ctx, cudaMemcpyAsync(img, d_img, px * 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

}  // extern "C"
