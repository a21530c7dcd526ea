// plot.cu — indexcov's depth and ROC charts drawn on the GPU (DESIGN §1.14).
//
// A chart is first an INDEX IMAGE: one uint32 per pixel of its data area, 0 where no line passes and otherwise the largest
// draw index of the datasets whose line covers the pixel.  Every line is opaque, so the dataset drawn last (the largest
// index) is the one that shows; max is order-free, so the image does not depend on launch shape, scheduling or how the
// samples were split over GPUs (images of sample shards combine by element-wise max).
//
// Which points (indexcov/plot.go asValues + asPng): leading values == 0 are skipped (NaN counts as non-zero); vertex j of
// what is left is x = (first + j * stride) * mult, y = min(v, 2.5).  With n values after the skip, stride is 10 when
// n > 2000, 5 when n > 1000, else 1 (vs.Sample keeps post-skip positions p % stride == 0).  A dataset whose plotted
// vertices hold a NaN is not drawn: the reference skips it when stride is 1 and panics inside gonum otherwise.
//
// The raster rule: a vertex maps to X = (x - xmin) * sx, Y = H - (y - ymin) * sy in data-area pixels (y down); segment AB
// covers pixel (i, j) when the squared distance from (i + 0.5, j + 0.5) to AB is <= r * r, with the clamped projection
// t = clamp(((P - A) . d) / L, 0, 1), d = B - A, L = d . d (the distance to A when L == 0).  Every operation is one float64
// round-to-nearest step in the order written in plot_rule.cuh: explicit _rn intrinsics on the device, plain operations on
// the host (the library is built with --fmad=false and no host FMA), so the host mirror and numpy restate the device bit
// for bit.
#include "gl_common.cuh"
#include "plot_rule.cuh"
#include "host/font5x7.h"
#include "host/thread_pool.h"
#include <zlib.h>
#include <math.h>
#include <string.h>

namespace {

using glplot::draw_segment;
using glplot::p_mul;

constexpr float kCnMax = 2.5f;         // plot.go:63 cnMax
constexpr int kSelThreads = 256;
constexpr int kRasterThreads = 128;

__host__ __device__ inline int64_t sel_stride(int64_t n) { return n > 2000 ? 10 : (n > 1000 ? 5 : 1); }

// vertex sources: a selected series of float32 values, or explicit float64 arrays
struct SeriesSrc {
    const float* vals; const int64_t* off; const int64_t* sel; double mult;
    __host__ __device__ int64_t count(int64_t d) const { return sel[d * 3 + 1]; }
    __host__ __device__ void xy(int64_t d, int64_t j, double& x, double& y) const {
        const int64_t i = sel[d * 3] + j * sel[d * 3 + 2];
        const float v = vals[off[d] + i];
        x = p_mul((double)i, mult);
        y = (double)(v > kCnMax ? kCnMax : v);
    }
};
struct XySrc {
    const double* x; const double* y; const int64_t* ptr;
    __host__ __device__ int64_t count(int64_t d) const { return ptr[d + 1] - ptr[d]; }
    __host__ __device__ void xy(int64_t d, int64_t j, double& xo, double& yo) const { xo = x[ptr[d] + j]; yo = y[ptr[d] + j]; }
};

// one CTA per dataset: first non-zero, stride, plotted count (0 = not drawn) and the y extent of the plotted vertices
__global__ void __launch_bounds__(kSelThreads) pl_select_kernel(const float* __restrict__ vals, const int64_t* __restrict__ off,
                                                                const int64_t* __restrict__ len, int32_t n, int64_t* __restrict__ sel,
                                                                float* __restrict__ yext) {
    __shared__ long long s_first;
    __shared__ int s_nan;
    __shared__ float s_lo[kSelThreads / 32], s_hi[kSelThreads / 32];
    const int64_t d = blockIdx.x;
    const float* v = vals + off[d];
    const long long L = len[d];
    if (threadIdx.x == 0) { s_first = L; s_nan = 0; }
    __syncthreads();
    long long mine = L;
    for (long long i = threadIdx.x; i < L; i += blockDim.x)
        if (v[i] != 0.f) { mine = i; break; }                  // NaN != 0: a NaN ends the skip, as in asValues
    if (mine < L) atomicMin(&s_first, mine);
    __syncthreads();
    const long long first = s_first, nv = L - first, stride = sel_stride(nv), m = (nv + stride - 1) / stride;
    float lo = INFINITY, hi = -INFINITY;
    bool nan = false;
    for (long long j = threadIdx.x; j < m; j += blockDim.x) {
        float y = v[first + j * stride];
        y = y > kCnMax ? kCnMax : y;
        if (y != y) nan = true;
        else { lo = fminf(lo, y); hi = fmaxf(hi, y); }
    }
    if (__syncthreads_or(nan) && threadIdx.x == 0) s_nan = 1;
    for (int o = 16; o > 0; o >>= 1) { lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    if ((threadIdx.x & 31) == 0) { s_lo[threadIdx.x >> 5] = lo; s_hi[threadIdx.x >> 5] = hi; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < kSelThreads / 32; w++) { lo = fminf(lo, s_lo[w]); hi = fmaxf(hi, s_hi[w]); }
        const bool drawn = m > 0 && !s_nan;
        sel[d * 3] = first; sel[d * 3 + 1] = drawn ? m : 0; sel[d * 3 + 2] = stride;
        yext[d * 2] = drawn ? lo : 0.f; yext[d * 2 + 1] = drawn ? hi : 0.f;
    }
}

// One CTA per dataset, one thread per segment.  The plain read before the atomic skips pixels that a later (larger) draw
// index already holds: in the y ~ 1 band most of a cohort's lines land on the same pixels.  A stale read can only be
// smaller than the pixel's value, which costs one atomic and never changes the result.
template <class Src>
__global__ void __launch_bounds__(kRasterThreads) pl_raster_kernel(Src src, const int32_t* __restrict__ chart,
                                                                   const uint32_t* __restrict__ draw, const double* __restrict__ xf,
                                                                   int W, int H, double r, double r2, uint32_t* __restrict__ img) {
    const int64_t d = blockIdx.x;
    const int64_t m = src.count(d);
    if (m < 2) return;
    const double* f = xf + 4 * (int64_t)chart[d];
    const uint32_t idx = draw[d];
    uint32_t* im = img + (int64_t)chart[d] * W * H;
    for (int64_t j = threadIdx.x; j + 1 < m; j += blockDim.x) {
        double x0, y0, x1, y1;
        src.xy(d, j, x0, y0);
        src.xy(d, j + 1, x1, y1);
        draw_segment(x0, y0, x1, y1, f, W, H, r, r2, [&](int i, int jj) {
            unsigned int* p = reinterpret_cast<unsigned int*>(im + (int64_t)jj * W + i);
            if (__ldcg(p) < idx) atomicMax(p, idx);
        });
    }
}

// host mirror of pl_raster_kernel: the charts are independent images, one pool task each
template <class Src>
void raster_host(const Src& src, const int32_t* chart, const uint32_t* draw, int32_t n, const double* xf, int32_t n_charts,
                 int W, int H, double r, uint32_t* img) {
    const double r2 = r * r;
    memset(img, 0, (size_t)n_charts * W * H * 4);
    glhost::ThreadPool::global().run(n_charts, [&](int64_t c, int) {
        uint32_t* im = img + c * W * H;
        for (int32_t d = 0; d < n; d++) {
            if (chart[d] != c) continue;
            const int64_t m = src.count(d);
            const uint32_t idx = draw[d];
            for (int64_t j = 0; j + 1 < m; j++) {
                double x0, y0, x1, y1;
                src.xy(d, j, x0, y0);
                src.xy(d, j + 1, x1, y1);
                draw_segment(x0, y0, x1, y1, xf + 4 * c, W, H, r, r2, [&](int i, int jj) {
                    uint32_t& p = im[(int64_t)jj * W + i];
                    if (p < idx) p = idx;
                });
            }
        }
    });
}

int raster_args(gl_ctx* ctx, const char* fn, const void* a, const void* b, const int32_t* chart, const uint32_t* draw, int32_t n,
                const double* xf, int32_t n_charts, int32_t W, int32_t H, double r, const void* img) {
    if (n < 0 || n_charts < 0 || W < 1 || H < 1 || !(r > 0) || (n > 0 && (!a || !b || !chart || !draw || !xf)) || (n_charts > 0 && !img))
        return gl_fail(ctx, GL_EINVAL, "%s: bad argument", fn);
    return GL_OK;
}

int check_charts_host(const char* fn, const int32_t* chart, int32_t n, int32_t n_charts) {
    for (int32_t d = 0; d < n; d++)
        if (chart[d] < 0 || chart[d] >= n_charts) return gl_fail(nullptr, GL_EINVAL, "%s: chart[%d] = %d out of range", fn, d, chart[d]);
    return GL_OK;
}

template <class Src>
int raster_device(gl_ctx* ctx, const Src& src, const int32_t* d_chart, const uint32_t* d_draw, int32_t n, const double* d_xf,
                  int32_t n_charts, int32_t W, int32_t H, double r, uint32_t* d_img) {
    GL_CUDA(ctx, cudaMemsetAsync(d_img, 0, (size_t)n_charts * W * H * 4, ctx->stream));
    if (n > 0) {
        gl_prof_scope prof(ctx, "pl_raster_kernel");
        pl_raster_kernel<<<(unsigned)n, kRasterThreads, 0, ctx->stream>>>(src, d_chart, d_draw, d_xf, W, H, r, r * r, d_img);
        GL_LAUNCHED(ctx, 1);
    }
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

// ---- the frame
constexpr int kGlyphW = 6;             // 5 columns and a blank one

void put_px(uint8_t* rgb, int CW, int CH, int x, int y, uint8_t c) {
    if (x < 0 || y < 0 || x >= CW || y >= CH) return;
    uint8_t* p = rgb + ((size_t)y * CW + x) * 3;
    p[0] = p[1] = p[2] = c;
}

void text(uint8_t* rgb, int CW, int CH, int x, int y, const char* s, bool vertical) {
    for (int k = 0; s[k]; k++) {
        const unsigned ch = (unsigned char)s[k];
        const uint8_t* g = kFont5x7[(ch >= 0x20 && ch <= 0x7E ? ch : '?') - 0x20];
        for (int c = 0; c < 5; c++)
            for (int rr = 0; rr < 7; rr++)
                if (g[c] >> rr & 1) {
                    if (vertical) put_px(rgb, CW, CH, x + rr, y - (k * kGlyphW + c), 0);   // reads bottom to top
                    else put_px(rgb, CW, CH, x + k * kGlyphW + c, y + rr, 0);
                }
    }
}

int text_w(const std::string& s) { return (int)s.size() * kGlyphW - 1; }

void nice_ticks(double lo, double hi, std::vector<double>& out) {
    out.clear();
    if (!(hi > lo) || !std::isfinite(lo) || !std::isfinite(hi)) return;
    double step = pow(10.0, floor(log10(hi - lo)) - 2);
    for (int it = 0; it < 64; it++) {
        for (double m : {1.0, 2.0, 5.0}) {
            const double s = step * m;
            const double k0 = ceil(lo / s), k1 = floor(hi / s);
            if (k1 - k0 + 1 <= 8) {
                for (double k = k0; k <= k1; k++) out.push_back(k * s);
                return;
            }
        }
        step *= 10;
    }
}

std::string millions(double v) {                       // plot.go:564-577 makeMillions
    char b[64];
    if (v > 2000000) snprintf(b, sizeof b, "%.1fMB", v / 1000000);
    else if (v > 10000) snprintf(b, sizeof b, "%.1fKB", v / 1000);
    else snprintf(b, sizeof b, "%.1f", v);
    std::string s = b;
    if (s.size() >= 4 && s.compare(s.size() - 4, 4, ".0MB") == 0) s = s.substr(0, s.size() - 4) + "MB";
    return s;
}

std::string plain_label(double v, double step) {
    const int dec = step > 0 ? std::max(0, (int)-floor(log10(step) + 1e-9)) : 0;
    char b[64];
    snprintf(b, sizeof b, "%.*f", dec, v == 0 ? 0.0 : v);
    return b;
}

void be32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)(v >> 24); p[1] = (uint8_t)(v >> 16); p[2] = (uint8_t)(v >> 8); p[3] = (uint8_t)v; }

}  // namespace

extern "C" {

int gl_plot_select_device(gl_ctx* ctx, const float* d_vals, const int64_t* d_off, const int64_t* d_len, int32_t n, int64_t* d_sel3,
                          float* d_yext2) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || (n > 0 && (!d_vals || !d_off || !d_len || !d_sel3 || !d_yext2))) return gl_fail(ctx, GL_EINVAL, "gl_plot_select_device: bad argument");
    if (n == 0) return GL_OK;
    {
        gl_prof_scope prof(ctx, "pl_select_kernel");
        pl_select_kernel<<<(unsigned)n, kSelThreads, 0, ctx->stream>>>(d_vals, d_off, d_len, n, d_sel3, d_yext2);
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_plot_select_host(const float* vals, const int64_t* off, const int64_t* len, int32_t n, int64_t* sel3, float* yext2) {
    if (n < 0 || (n > 0 && (!vals || !off || !len || !sel3 || !yext2))) return gl_fail(nullptr, GL_EINVAL, "gl_plot_select_host: bad argument");
    for (int32_t d = 0; d < n; d++) {
        const float* v = vals + off[d];
        int64_t first = 0;
        while (first < len[d] && v[first] == 0.f) first++;
        const int64_t nv = len[d] - first, stride = sel_stride(nv), m = (nv + stride - 1) / stride;
        float lo = INFINITY, hi = -INFINITY;
        bool nan = false;
        for (int64_t j = 0; j < m; j++) {
            float y = v[first + j * stride];
            y = y > kCnMax ? kCnMax : y;
            if (y != y) nan = true;
            else { lo = std::min(lo, y); hi = std::max(hi, y); }
        }
        const bool drawn = m > 0 && !nan;
        sel3[d * 3] = first; sel3[d * 3 + 1] = drawn ? m : 0; sel3[d * 3 + 2] = stride;
        yext2[d * 2] = drawn ? lo : 0.f; yext2[d * 2 + 1] = drawn ? hi : 0.f;
    }
    return GL_OK;
}

int gl_plot_transform(const double* ext4, int32_t W, int32_t H, double* xf4) {
    if (!ext4 || !xf4 || W < 1 || H < 1) return gl_fail(nullptr, GL_EINVAL, "gl_plot_transform: bad argument");
    double x0 = ext4[0], x1 = ext4[1], y0 = ext4[2], y1 = ext4[3];
    if (x0 == x1) { x0 -= 1; x1 += 1; }
    if (y0 == y1) { y0 -= 1; y1 += 1; }
    xf4[0] = x0; xf4[1] = (double)W / (x1 - x0); xf4[2] = y0; xf4[3] = (double)H / (y1 - y0);
    return GL_OK;
}

double gl_plot_line_radius(int32_t n_datasets) {
    const double w = n_datasets > 30 ? 0.65 : 0.8;           // plot.go:508-511, points
    return std::max(0.5, w * 96.0 / 72.0 / 2.0);
}

int gl_plot_raster_series_device(gl_ctx* ctx, const float* d_vals, const int64_t* d_off, const int64_t* d_sel3, double mult,
                                 const int32_t* d_chart, const uint32_t* d_draw, int32_t n, const double* d_xf4, int32_t n_charts,
                                 int32_t W, int32_t H, double r, uint32_t* d_img) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(raster_args(ctx, "gl_plot_raster_series_device", d_vals, d_sel3, d_chart, d_draw, n, d_xf4, n_charts, W, H, r, d_img));
    if (n > 0 && !d_off) return gl_fail(ctx, GL_EINVAL, "gl_plot_raster_series_device: bad argument");
    return raster_device(ctx, SeriesSrc{d_vals, d_off, d_sel3, mult}, d_chart, d_draw, n, d_xf4, n_charts, W, H, r, d_img);
}

int gl_plot_raster_series_host(const float* vals, const int64_t* off, const int64_t* sel3, double mult, const int32_t* chart,
                               const uint32_t* draw, int32_t n, const double* xf4, int32_t n_charts, int32_t W, int32_t H, double r,
                               uint32_t* img) {
    GL_CHECK(raster_args(nullptr, "gl_plot_raster_series_host", vals, sel3, chart, draw, n, xf4, n_charts, W, H, r, img));
    if (n > 0 && !off) return gl_fail(nullptr, GL_EINVAL, "gl_plot_raster_series_host: bad argument");
    GL_CHECK(check_charts_host("gl_plot_raster_series_host", chart, n, n_charts));
    raster_host(SeriesSrc{vals, off, sel3, mult}, chart, draw, n, xf4, n_charts, W, H, r, img);
    return GL_OK;
}

int gl_plot_raster_xy(gl_ctx* ctx, const double* x, const double* y, const int64_t* ptr, const int32_t* chart, const uint32_t* draw,
                      int32_t n, const double* xf4, int32_t n_charts, int32_t W, int32_t H, double r, uint32_t* img) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(raster_args(ctx, "gl_plot_raster_xy", x, y, chart, draw, n, xf4, n_charts, W, H, r, img));
    if (n > 0 && !ptr) return gl_fail(ctx, GL_EINVAL, "gl_plot_raster_xy: bad argument");
    GL_CHECK(check_charts_host("gl_plot_raster_xy", chart, n, n_charts));
    if (n_charts == 0) return GL_OK;
    const int64_t nv = n > 0 ? ptr[n] : 0;
    gl_scratch tmp(ctx);
    double *d_x, *d_y, *d_xf; int64_t* d_ptr; int32_t* d_chart; uint32_t *d_draw, *d_img;
    GL_CHECK(tmp.upload(d_x, x, (size_t)nv));
    GL_CHECK(tmp.upload(d_y, y, (size_t)nv));
    GL_CHECK(tmp.upload(d_ptr, ptr, (size_t)n + 1));
    GL_CHECK(tmp.upload(d_chart, chart, (size_t)n));
    GL_CHECK(tmp.upload(d_draw, draw, (size_t)n));
    GL_CHECK(tmp.upload(d_xf, xf4, (size_t)n_charts * 4));
    GL_CHECK(tmp.alloc(d_img, (size_t)n_charts * W * H));
    GL_CHECK(raster_device(ctx, XySrc{d_x, d_y, d_ptr}, d_chart, d_draw, n, d_xf, n_charts, W, H, r, d_img));
    GL_CUDA(ctx, cudaMemcpyAsync(img, d_img, (size_t)n_charts * W * H * 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_plot_raster_xy_host(const double* x, const double* y, const int64_t* ptr, const int32_t* chart, const uint32_t* draw, int32_t n,
                           const double* xf4, int32_t n_charts, int32_t W, int32_t H, double r, uint32_t* img) {
    GL_CHECK(raster_args(nullptr, "gl_plot_raster_xy_host", x, y, chart, draw, n, xf4, n_charts, W, H, r, img));
    if (n > 0 && !ptr) return gl_fail(nullptr, GL_EINVAL, "gl_plot_raster_xy_host: bad argument");
    GL_CHECK(check_charts_host("gl_plot_raster_xy_host", chart, n, n_charts));
    raster_host(XySrc{x, y, ptr}, chart, draw, n, xf4, n_charts, W, H, r, img);
    return GL_OK;
}

void gl_plot_color(int32_t k, int32_t n_background, uint8_t* rgb3) {
    if (k < n_background) { rgb3[0] = rgb3[1] = rgb3[2] = 180; return; }     // plot.go:98-101
    uint64_t z = (uint64_t)(uint32_t)k + 0x9E3779B97F4A7C15ull;                // splitmix64 of the sample index
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    z ^= z >> 31;
    for (int c = 0; c < 3; c++) rgb3[c] = (uint8_t)(((z >> (8 * c)) & 255) * 220 / 255);   // nothing lighter than 220: lines stay visible on white
}

int gl_plot_ticks(double lo, double hi, double* out, int32_t cap, int32_t* n) {
    if (!n || cap < 0 || (cap > 0 && !out)) return gl_fail(nullptr, GL_EINVAL, "gl_plot_ticks: bad argument");
    std::vector<double> t;
    nice_ticks(lo, hi, t);
    *n = (int32_t)t.size();
    if ((int32_t)t.size() > cap) return gl_fail(nullptr, GL_ERANGE, "gl_plot_ticks: %zu ticks, room for %d", t.size(), cap);
    std::copy(t.begin(), t.end(), out);
    return GL_OK;
}

int gl_plot_millions(double v, char* buf, int32_t cap) {
    const std::string s = millions(v);
    if (!buf || cap < (int32_t)s.size() + 1) return gl_fail(nullptr, GL_ERANGE, "gl_plot_millions: buffer too small");
    memcpy(buf, s.c_str(), s.size() + 1);
    return GL_OK;
}

int gl_plot_text(uint8_t* rgb, int32_t CW, int32_t CH, int32_t x, int32_t y, const char* s, int32_t vertical) {
    if (!rgb || !s || CW < 1 || CH < 1) return gl_fail(nullptr, GL_EINVAL, "gl_plot_text: bad argument");
    text(rgb, CW, CH, x, y, s, vertical != 0);
    return GL_OK;
}

int gl_plot_compose(const uint32_t* img, const uint8_t* palette, int32_t n_pal, int32_t kind, const double* ext4, const char* xtitle,
                    const char* ytitle, uint8_t* rgb) {
    if (!img || !palette || n_pal < 1 || !ext4 || !xtitle || !ytitle || !rgb || kind < GL_PLOT_DEPTH || kind > GL_PLOT_SQUARE)
        return gl_fail(nullptr, GL_EINVAL, "gl_plot_compose: bad argument");
    const bool sq = kind == GL_PLOT_SQUARE;
    const int CW = sq ? GL_PLOT_SQ_CW : GL_PLOT_CW, CH = sq ? GL_PLOT_SQ_CH : GL_PLOT_CH, AX = GL_PLOT_AX, AY = GL_PLOT_AY;
    const int W = sq ? GL_PLOT_SQ_W : GL_PLOT_W, H = sq ? GL_PLOT_SQ_H : GL_PLOT_H;
    memset(rgb, 255, (size_t)CW * CH * 3);
    for (int j = 0; j < H; j++)
        for (int i = 0; i < W; i++) {
            const uint32_t v = img[(size_t)j * W + i];
            if (!v) continue;
            const uint8_t* c = v < (uint32_t)n_pal ? palette + 3 * (size_t)v : palette;
            memcpy(rgb + ((size_t)(AY + j) * CW + AX + i) * 3, c, 3);
        }
    for (int j = AY; j <= AY + H; j++) put_px(rgb, CW, CH, AX - 1, j, 0);
    for (int i = AX - 1; i < AX + W; i++) put_px(rgb, CW, CH, i, AY + H, 0);
    double xf[4];
    GL_CHECK(gl_plot_transform(ext4, W, H, xf));
    std::vector<double> xt, yt;
    nice_ticks(xf[0], xf[0] + W / xf[1], xt);
    if (kind == GL_PLOT_DEPTH) yt = {0.0, 0.5, 1.0, 1.5, 2.0};                  // plot.go:542-549
    else nice_ticks(xf[2], xf[2] + H / xf[3], yt);
    const double xstep = xt.size() > 1 ? xt[1] - xt[0] : 0, ystep = yt.size() > 1 ? yt[1] - yt[0] : 0;
    for (double t : xt) {
        const double X = (t - xf[0]) * xf[1];
        if (!(X >= 0 && X <= W)) continue;
        const int px = AX + std::min(W - 1, (int)X);
        for (int k = 1; k <= 4; k++) put_px(rgb, CW, CH, px, AY + H + k, 0);
        const std::string l = kind == GL_PLOT_DEPTH ? millions(t) : plain_label(t, xstep);
        text(rgb, CW, CH, px - text_w(l) / 2, AY + H + 7, l.c_str(), false);
    }
    for (double t : yt) {
        const double Y = H - (t - xf[2]) * xf[3];
        if (!(Y >= 0 && Y <= H)) continue;
        const int py = AY + std::min(H - 1, (int)Y);
        for (int k = 2; k <= 5; k++) put_px(rgb, CW, CH, AX - k, py, 0);
        char b[64];
        if (kind == GL_PLOT_DEPTH) snprintf(b, sizeof b, "%.1f", t);
        else snprintf(b, sizeof b, "%s", plain_label(t, ystep).c_str());
        text(rgb, CW, CH, AX - 8 - text_w(b), py - 3, b, false);
    }
    text(rgb, CW, CH, AX + W / 2 - text_w(xtitle) / 2, CH - 10, xtitle, false);
    text(rgb, CW, CH, 3, AY + H / 2 + text_w(ytitle) / 2, ytitle, true);
    return GL_OK;
}

int gl_plot_png(const uint8_t* rgb, int32_t W, int32_t H, uint8_t* out, int64_t cap, int64_t* len) {
    if (!rgb || W < 1 || H < 1 || !len || cap < 0 || (cap > 0 && !out)) return gl_fail(nullptr, GL_EINVAL, "gl_plot_png: bad argument");
    const size_t raw_n = (size_t)H * ((size_t)W * 3 + 1);
    const size_t bound = compressBound((uLong)raw_n) + 8 + 25 + 12 + 12;
    if (!out || (size_t)cap < bound) {
        *len = (int64_t)bound;
        return out ? gl_fail(nullptr, GL_ERANGE, "gl_plot_png: %lld bytes of room, %zu needed", (long long)cap, bound) : GL_OK;
    }
    std::vector<uint8_t> raw(raw_n);
    for (int32_t j = 0; j < H; j++) {
        raw[(size_t)j * (W * 3 + 1)] = 0;                                         // filter 0 on every row
        memcpy(&raw[(size_t)j * (W * 3 + 1) + 1], rgb + (size_t)j * W * 3, (size_t)W * 3);
    }
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    uint8_t* p = out;
    memcpy(p, sig, 8); p += 8;
    auto chunk = [&](const char* type, const uint8_t* data, uint32_t n) {
        be32(p, n); memcpy(p + 4, type, 4);
        if (n) memmove(p + 8, data, n);
        be32(p + 8 + n, (uint32_t)crc32(0, p + 4, n + 4));
        p += 12 + n;
    };
    uint8_t ihdr[13];
    be32(ihdr, (uint32_t)W); be32(ihdr + 4, (uint32_t)H);
    ihdr[8] = 8; ihdr[9] = 2; ihdr[10] = ihdr[11] = ihdr[12] = 0;                  // RGB8, deflate, no interlace
    chunk("IHDR", ihdr, 13);
    uLongf zn = (uLongf)(cap - (p - out) - 24);
    if (compress2(p + 8, &zn, raw.data(), (uLong)raw_n, 6) != Z_OK) return gl_fail(nullptr, GL_EINVAL, "gl_plot_png: deflate failed");
    chunk("IDAT", p + 8, (uint32_t)zn);
    chunk("IEND", nullptr, 0);
    *len = p - out;
    return GL_OK;
}

}  // extern "C"
