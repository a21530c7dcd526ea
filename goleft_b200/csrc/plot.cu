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
//
// The vector charts (INDEXCOV_FMT, indexcov/plot.go:527-536) are the same charts in points (72 per inch, 0.75 per pixel):
// vertex (x, y) of a dataset is at Xpt = 0.75 (AX + (x - xmin) sx), Ypt = 0.75 (AY + (H - (y - ymin) sy)), one float64
// round-to-nearest step per operation in that order (EPS: y = 0.75 CH - Ypt), written as printf("%.2f") by the f2 token
// rule (host/f2_token.h).  pl_path_kernel makes every dataset's path text on the device in two passes: the byte length of
// each dataset, then, at the offsets an exclusive scan of those lengths gives, the text itself.
#include "gl_common.cuh"
#include "plot_rule.cuh"
#include "ll_scan.cuh"
#include "host/f2_token.h"
#include "host/font5x7.h"
#include "host/thread_pool.h"
#include <zlib.h>
#include <math.h>
#include <string.h>
#include <array>

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

// ---- path text
constexpr int kPathThreads = 256;
constexpr int kVertexMax = 2 * glf2::kTok + 16;       // the longest vertex token: " L x y" or "x y lineto\n"

// the canvas of a chart kind, in pixels, and the output format
struct Canvas {
    double ax, ay, h, ch;
    bool eps;
};

bool canvas_of(int32_t kind, int32_t fmt, Canvas& cv) {
    if (kind < GL_PLOT_DEPTH || kind > GL_PLOT_SQUARE || (fmt != GL_PLOT_SVG && fmt != GL_PLOT_EPS)) return false;
    const bool sq = kind == GL_PLOT_SQUARE;
    cv = Canvas{(double)GL_PLOT_AX, (double)GL_PLOT_AY, (double)(sq ? GL_PLOT_SQ_H : GL_PLOT_H), (double)(sq ? GL_PLOT_SQ_CH : GL_PLOT_CH),
                fmt == GL_PLOT_EPS};
    return true;
}

// The text of vertex j of dataset d into t (kVertexMax bytes of room): SVG "M x y" (j == 0) or " L x y"; EPS "x y moveto\n"
// or "x y lineto\n".  Returns its length, or 0 when a coordinate is not finite or its "%.2f" does not fit a token.
template <class Src>
__host__ __device__ inline int vertex_text(const Src& src, int64_t d, int64_t j, const double* f, const Canvas& cv, unsigned char* t) {
    using glplot::p_add; using glplot::p_sub;
    double x, y;
    src.xy(d, j, x, y);
    const double X = p_mul(0.75, p_add(cv.ax, p_mul(p_sub(x, f[0]), f[1])));
    double Y = p_mul(0.75, p_add(cv.ay, p_sub(cv.h, p_mul(p_sub(y, f[2]), f[3]))));
    if (cv.eps) Y = p_sub(p_mul(0.75, cv.ch), Y);
    if (!isfinite(X) || !isfinite(Y)) return 0;
    unsigned char tx[glf2::kTok], ty[glf2::kTok];
    const int lx = glf2::token(X, tx), ly = glf2::token(Y, ty);
    if (!lx || !ly) return 0;
    int n = 0;
    auto put = [&](const char* s) { while (*s) t[n++] = (unsigned char)*s++; };
    if (!cv.eps) put(j ? " L " : "M ");
    for (int k = 0; k < lx; k++) t[n++] = tx[k];
    t[n++] = ' ';
    for (int k = 0; k < ly; k++) t[n++] = ty[k];
    if (cv.eps) put(j ? " lineto\n" : " moveto\n");
    return n;
}

// Pass 1 (pos == nullptr): len[d] = the bytes of dataset d's path text, 0 when it is not written (fewer than 2 vertices, as
// the raster draws nothing then, or a vertex vertex_text rejects).  Pass 2: the text at out + pos[d]; no byte is written at
// or past min(pos[d + 1], cap), so a pos that does not match pass 1 cannot write out of bounds.
template <class Src>
__global__ void __launch_bounds__(kPathThreads) pl_path_kernel(Src src, const int32_t* __restrict__ chart, const double* __restrict__ xf,
                                                               Canvas cv, long long* __restrict__ len, const long long* __restrict__ pos,
                                                               unsigned char* __restrict__ out, long long cap) {
    __shared__ long long s_w[kPathThreads / 32];
    const int64_t d = blockIdx.x;
    const int64_t m = src.count(d);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const double* f = xf + 4 * (int64_t)chart[d];
    unsigned char t[kVertexMax];
    if (!pos) {
        long long sum = 0;
        bool bad = false;
        for (int64_t j = threadIdx.x; j < m && m >= 2; j += blockDim.x) {
            const int n = vertex_text(src, d, j, f, cv, t);
            bad |= n == 0;
            sum += n;
        }
        bad = __syncthreads_or(bad);
        for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        if (lane == 0) s_w[warp] = sum;
        __syncthreads();
        if (threadIdx.x == 0) {
            for (int w = 1; w < kPathThreads / 32; w++) sum += s_w[w];
            len[d] = (m < 2 || bad) ? 0 : sum;
        }
        return;
    }
    const long long end = min(pos[d + 1], cap);
    if (pos[d] >= end) return;
    long long base = pos[d];
    for (int64_t j0 = 0; j0 < m; j0 += blockDim.x) {
        const int64_t j = j0 + threadIdx.x;
        const int n = j < m ? vertex_text(src, d, j, f, cv, t) : 0;
        int inc = n;                                   // block-wide exclusive scan of the vertex lengths
        for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += y; }
        __syncthreads();                               // s_w of the previous chunk has been read
        if (lane == 31) s_w[warp] = inc;
        __syncthreads();
        long long at = base + inc - n, tot = 0;
        for (int w = 0; w < kPathThreads / 32; w++) { if (w < warp) at += s_w[w]; tot += s_w[w]; }
        for (int k = 0; k < n && at + k < end; k++) out[at + k] = t[k];
        base += tot;
    }
}

template <class Src>
int path_size_device(gl_ctx* ctx, const Src& src, const int32_t* d_chart, int32_t n, const double* d_xf, const Canvas& cv, int64_t* d_len,
                     int64_t* d_pos) {
    if (n > 0) {
        gl_prof_scope prof(ctx, "pl_path_kernel");
        pl_path_kernel<<<(unsigned)n, kPathThreads, 0, ctx->stream>>>(src, d_chart, d_xf, cv, reinterpret_cast<long long*>(d_len), nullptr,
                                                                      nullptr, 0);
        GL_LAUNCHED(ctx, 1);
    }
    ll_scan_kernel<<<1, 1024, 0, ctx->stream>>>(reinterpret_cast<const long long*>(d_len), reinterpret_cast<long long*>(d_pos), n);
    GL_LAUNCHED(ctx, 1);
    return GL_OK;
}

template <class Src>
int path_emit_device(gl_ctx* ctx, const char* fn, const Src& src, const int32_t* d_chart, int32_t n, const double* d_xf, const Canvas& cv,
                     const int64_t* d_pos, int64_t total, char* d_out, int64_t cap) {
    if (total < 0 || cap < 0 || (cap > 0 && !d_out)) return gl_fail(ctx, GL_EINVAL, "%s: bad argument", fn);
    if (total > cap) return gl_fail(ctx, GL_ERANGE, "%s: path text is %lld bytes, buffer holds %lld", fn, (long long)total, (long long)cap);
    if (n == 0 || total == 0) return GL_OK;
    gl_prof_scope prof(ctx, "pl_path_kernel");
    pl_path_kernel<<<(unsigned)n, kPathThreads, 0, ctx->stream>>>(src, d_chart, d_xf, cv, nullptr, reinterpret_cast<const long long*>(d_pos),
                                                                  reinterpret_cast<unsigned char*>(d_out), (long long)cap);
    GL_LAUNCHED(ctx, 1);
    return GL_OK;
}

// host mirror: one pool task per dataset
template <class Src>
void path_size_host(const Src& src, const int32_t* chart, int32_t n, const double* xf, const Canvas& cv, int64_t* len, int64_t* pos) {
    glhost::ThreadPool::global().run(n, [&](int64_t d, int) {
        const int64_t m = src.count(d);
        unsigned char t[kVertexMax];
        int64_t sum = 0;
        for (int64_t j = 0; j < m && m >= 2; j++) {
            const int k = vertex_text(src, d, j, xf + 4 * chart[d], cv, t);
            if (!k) { sum = 0; break; }
            sum += k;
        }
        len[d] = m < 2 ? 0 : sum;
    });
    pos[0] = 0;
    for (int32_t d = 0; d < n; d++) pos[d + 1] = pos[d] + len[d];
}

template <class Src>
int path_emit_host(const char* fn, const Src& src, const int32_t* chart, int32_t n, const double* xf, const Canvas& cv, const int64_t* pos,
                   char* out, int64_t cap) {
    for (int32_t d = 0; d < n; d++)
        if (pos[d + 1] < pos[d] || pos[0] != 0) return gl_fail(nullptr, GL_EINVAL, "%s: pos is not a scan of the lengths", fn);
    if (pos[n] > cap) return gl_fail(nullptr, GL_ERANGE, "%s: path text is %lld bytes, buffer holds %lld", fn, (long long)pos[n], (long long)cap);
    if (pos[n] > 0 && !out) return gl_fail(nullptr, GL_EINVAL, "%s: bad argument", fn);
    glhost::ThreadPool::global().run(n, [&](int64_t d, int) {
        if (pos[d + 1] == pos[d]) return;
        const int64_t m = src.count(d);
        unsigned char t[kVertexMax];
        int64_t at = pos[d];
        for (int64_t j = 0; j < m; j++) {
            const int k = vertex_text(src, d, j, xf + 4 * chart[d], cv, t);
            for (int i = 0; i < k && at < pos[d + 1]; i++) out[at++] = (char)t[i];
        }
    });
    return GL_OK;
}

int path_args(gl_ctx* ctx, const char* fn, const void* a, const void* b, const void* c, const int32_t* chart, int32_t n, const double* xf,
              int32_t n_charts, int32_t kind, int32_t fmt, Canvas& cv) {
    if (n < 0 || n_charts < 0 || (n > 0 && (!a || !b || !c || !chart || !xf)) || !canvas_of(kind, fmt, cv))
        return gl_fail(ctx, GL_EINVAL, "%s: bad argument", fn);
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

// ---- the vector document (header, frame, paths, trailer)
std::string f2(double v) {
    char b[64];
    snprintf(b, sizeof b, "%.2f", v);
    return b;
}

std::string svg_escape(const char* s) {
    std::string o;
    for (; *s; s++) {
        const unsigned char c = (unsigned char)*s;
        if (c == '&') o += "&amp;";
        else if (c == '<') o += "&lt;";
        else if (c == '>') o += "&gt;";
        else if (c == '"') o += "&quot;";
        else if (c < 0x20) o += '?';                   // not allowed in XML 1.0 text
        else o += (char)c;
    }
    return o;
}

std::string ps_string(const char* s) {
    std::string o = "(";
    for (; *s; s++) {
        const unsigned char c = (unsigned char)*s;
        if (c == '(' || c == ')' || c == '\\') { o += '\\'; o += (char)c; }
        else if (c < 0x20 || c >= 0x7F) { char b[8]; snprintf(b, sizeof b, "\\%03o", c); o += b; }
        else o += (char)c;
    }
    return o + ")";
}

// Everything before the paths: the header, the white page, the axes and ticks as strokes, the labels and titles as text.
// Positions are gl_plot_compose's, in points: the tick values are its ticks at their exact (not pixel-rounded) places.
std::string vector_head(int32_t kind, const Canvas& cv, const double* xf, const char* xtitle, const char* ytitle) {
    const bool sq = kind == GL_PLOT_SQUARE;
    const double W = sq ? GL_PLOT_SQ_W : GL_PLOT_W, CW = sq ? GL_PLOT_SQ_CW : GL_PLOT_CW, H = cv.h, CH = cv.ch, AX = cv.ax, AY = cv.ay;
    const double pw = CW * 0.75, ph = CH * 0.75;
    auto px = [&](double x) { return f2(0.75 * x); };
    auto py = [&](double y) { return f2(cv.eps ? ph - 0.75 * y : 0.75 * y); };
    std::vector<double> xt, yt;
    nice_ticks(xf[0], xf[0] + W / xf[1], xt);
    if (kind == GL_PLOT_DEPTH) yt = {0.0, 0.5, 1.0, 1.5, 2.0};
    else nice_ticks(xf[2], xf[2] + H / xf[3], yt);
    const double xstep = xt.size() > 1 ? xt[1] - xt[0] : 0, ystep = yt.size() > 1 ? yt[1] - yt[0] : 0;
    // (x0, y0)-(x1, y1) strokes and (x, y, anchor: 0 start, 1 middle, 2 end, rotated, text) labels, in pixels
    std::vector<std::array<double, 4>> lines = {{AX, AY, AX, AY + H}, {AX, AY + H, AX + W, AY + H}};
    struct Label { double x, y; int anchor; bool rot; std::string s; };
    std::vector<Label> labels;
    for (double t : xt) {
        const double X = (t - xf[0]) * xf[1];
        if (!(X >= 0 && X <= W)) continue;
        lines.push_back({AX + X, AY + H, AX + X, AY + H + 4});
        labels.push_back({AX + X, AY + H + 14, 1, false, kind == GL_PLOT_DEPTH ? millions(t) : plain_label(t, xstep)});
    }
    for (double t : yt) {
        const double Y = H - (t - xf[2]) * xf[3];
        if (!(Y >= 0 && Y <= H)) continue;
        lines.push_back({AX - 5, AY + Y, AX, AY + Y});
        char b[64];
        if (kind == GL_PLOT_DEPTH) snprintf(b, sizeof b, "%.1f", t);
        else snprintf(b, sizeof b, "%s", plain_label(t, ystep).c_str());
        labels.push_back({AX - 8, AY + Y + 3.5, 2, false, b});
    }
    labels.push_back({AX + W / 2, CH - 3, 1, false, xtitle});
    labels.push_back({10, AY + H / 2, 1, true, ytitle});
    std::string o;
    if (!cv.eps) {
        const std::string w = std::to_string((int)pw), h = std::to_string((int)ph);
        o += "<?xml version=\"1.0\" encoding=\"UTF-8\"?>\n<svg xmlns=\"http://www.w3.org/2000/svg\" version=\"1.1\" width=\"" + w + "pt\" height=\"" + h +
             "pt\" viewBox=\"0 0 " + w + " " + h + "\">\n";
        o += "<rect x=\"0\" y=\"0\" width=\"100%\" height=\"100%\" fill=\"#ffffff\"/>\n";
        for (auto& l : lines)
            o += "<path d=\"M " + px(l[0]) + " " + py(l[1]) + " L " + px(l[2]) + " " + py(l[3]) + "\" stroke=\"#000000\" stroke-width=\"0.75\" fill=\"none\"/>\n";
        static const char* anchor[3] = {"start", "middle", "end"};
        for (auto& l : labels) {
            o += "<text font-family=\"Helvetica, Arial, sans-serif\" font-size=\"7\" fill=\"#000000\" text-anchor=\"" + std::string(anchor[l.anchor]) + "\" ";
            if (l.rot) o += "transform=\"translate(" + px(l.x) + " " + py(l.y) + ") rotate(-90)\" x=\"0\" y=\"0\">";
            else o += "x=\"" + px(l.x) + "\" y=\"" + py(l.y) + "\">";
            o += svg_escape(l.s.c_str()) + "</text>\n";
        }
        return o;
    }
    char b[256];
    snprintf(b, sizeof b, "%%!PS-Adobe-3.0 EPSF-3.0\n%%%%BoundingBox: 0 0 %d %d\n%%%%Creator: goleft indexcov\n%%%%EndComments\n", (int)pw, (int)ph);
    o += b;
    o += "1 setgray newpath 0 0 moveto " + f2(pw) + " 0 lineto " + f2(pw) + " " + f2(ph) + " lineto 0 " + f2(ph) + " lineto closepath fill\n";
    o += "1 setlinejoin 1 setlinecap\n0 setgray 0.75 setlinewidth\n";
    for (auto& l : lines) o += "newpath " + px(l[0]) + " " + py(l[1]) + " moveto " + px(l[2]) + " " + py(l[3]) + " lineto stroke\n";
    o += "/Helvetica findfont 7 scalefont setfont\n";
    for (auto& l : labels) {
        const std::string s = ps_string(l.s.c_str()), shift = l.anchor == 0 ? "" : l.anchor == 1 ? "dup stringwidth pop 2 div neg 0 rmoveto " : "dup stringwidth pop neg 0 rmoveto ";
        if (l.rot) o += "gsave " + px(l.x) + " " + py(l.y) + " translate 90 rotate 0 0 moveto " + s + " " + shift + "show grestore\n";
        else o += px(l.x) + " " + py(l.y) + " moveto " + s + " " + shift + "show\n";
    }
    return o;
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
    return std::max(0.5, gl_plot_line_width(n_datasets) * 96.0 / 72.0 / 2.0);
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

int gl_plot_path_series_size(gl_ctx* ctx, const float* d_vals, const int64_t* d_off, const int64_t* d_sel3, double mult, const int32_t* d_chart,
                             int32_t n, const double* d_xf4, int32_t n_charts, int32_t kind, int32_t fmt, int64_t* d_len, int64_t* d_pos) {
    GL_CHECK(gl_use(ctx));
    Canvas cv;
    GL_CHECK(path_args(ctx, "gl_plot_path_series_size", d_vals, d_off, d_sel3, d_chart, n, d_xf4, n_charts, kind, fmt, cv));
    if ((n > 0 && !d_len) || !d_pos) return gl_fail(ctx, GL_EINVAL, "gl_plot_path_series_size: bad argument");
    return path_size_device(ctx, SeriesSrc{d_vals, d_off, d_sel3, mult}, d_chart, n, d_xf4, cv, d_len, d_pos);
}

int gl_plot_path_series_emit(gl_ctx* ctx, const float* d_vals, const int64_t* d_off, const int64_t* d_sel3, double mult, const int32_t* d_chart,
                             int32_t n, const double* d_xf4, int32_t n_charts, int32_t kind, int32_t fmt, const int64_t* d_pos, int64_t total,
                             char* d_out, int64_t cap) {
    GL_CHECK(gl_use(ctx));
    Canvas cv;
    GL_CHECK(path_args(ctx, "gl_plot_path_series_emit", d_vals, d_off, d_sel3, d_chart, n, d_xf4, n_charts, kind, fmt, cv));
    if (!d_pos) return gl_fail(ctx, GL_EINVAL, "gl_plot_path_series_emit: bad argument");
    return path_emit_device(ctx, "gl_plot_path_series_emit", SeriesSrc{d_vals, d_off, d_sel3, mult}, d_chart, n, d_xf4, cv, d_pos, total, d_out, cap);
}

int gl_plot_path_series_size_host(const float* vals, const int64_t* off, const int64_t* sel3, double mult, const int32_t* chart, int32_t n,
                                  const double* xf4, int32_t n_charts, int32_t kind, int32_t fmt, int64_t* len, int64_t* pos) {
    Canvas cv;
    GL_CHECK(path_args(nullptr, "gl_plot_path_series_size_host", vals, off, sel3, chart, n, xf4, n_charts, kind, fmt, cv));
    if ((n > 0 && !len) || !pos) return gl_fail(nullptr, GL_EINVAL, "gl_plot_path_series_size_host: bad argument");
    GL_CHECK(check_charts_host("gl_plot_path_series_size_host", chart, n, n_charts));
    path_size_host(SeriesSrc{vals, off, sel3, mult}, chart, n, xf4, cv, len, pos);
    return GL_OK;
}

int gl_plot_path_series_emit_host(const float* vals, const int64_t* off, const int64_t* sel3, double mult, const int32_t* chart, int32_t n,
                                  const double* xf4, int32_t n_charts, int32_t kind, int32_t fmt, const int64_t* pos, char* out, int64_t cap) {
    Canvas cv;
    GL_CHECK(path_args(nullptr, "gl_plot_path_series_emit_host", vals, off, sel3, chart, n, xf4, n_charts, kind, fmt, cv));
    if (!pos) return gl_fail(nullptr, GL_EINVAL, "gl_plot_path_series_emit_host: bad argument");
    GL_CHECK(check_charts_host("gl_plot_path_series_emit_host", chart, n, n_charts));
    return path_emit_host("gl_plot_path_series_emit_host", SeriesSrc{vals, off, sel3, mult}, chart, n, xf4, cv, pos, out, cap);
}

int gl_plot_path_xy_size(gl_ctx* ctx, const double* d_x, const double* d_y, const int64_t* d_ptr, const int32_t* d_chart, int32_t n,
                         const double* d_xf4, int32_t n_charts, int32_t kind, int32_t fmt, int64_t* d_len, int64_t* d_pos) {
    GL_CHECK(gl_use(ctx));
    Canvas cv;
    GL_CHECK(path_args(ctx, "gl_plot_path_xy_size", d_x, d_y, d_ptr, d_chart, n, d_xf4, n_charts, kind, fmt, cv));
    if ((n > 0 && !d_len) || !d_pos) return gl_fail(ctx, GL_EINVAL, "gl_plot_path_xy_size: bad argument");
    return path_size_device(ctx, XySrc{d_x, d_y, d_ptr}, d_chart, n, d_xf4, cv, d_len, d_pos);
}

int gl_plot_path_xy_emit(gl_ctx* ctx, const double* d_x, const double* d_y, const int64_t* d_ptr, const int32_t* d_chart, int32_t n,
                         const double* d_xf4, int32_t n_charts, int32_t kind, int32_t fmt, const int64_t* d_pos, int64_t total, char* d_out,
                         int64_t cap) {
    GL_CHECK(gl_use(ctx));
    Canvas cv;
    GL_CHECK(path_args(ctx, "gl_plot_path_xy_emit", d_x, d_y, d_ptr, d_chart, n, d_xf4, n_charts, kind, fmt, cv));
    if (!d_pos) return gl_fail(ctx, GL_EINVAL, "gl_plot_path_xy_emit: bad argument");
    return path_emit_device(ctx, "gl_plot_path_xy_emit", XySrc{d_x, d_y, d_ptr}, d_chart, n, d_xf4, cv, d_pos, total, d_out, cap);
}

int gl_plot_path_xy_size_host(const double* x, const double* y, const int64_t* ptr, const int32_t* chart, int32_t n, const double* xf4,
                              int32_t n_charts, int32_t kind, int32_t fmt, int64_t* len, int64_t* pos) {
    Canvas cv;
    GL_CHECK(path_args(nullptr, "gl_plot_path_xy_size_host", x, y, ptr, chart, n, xf4, n_charts, kind, fmt, cv));
    if ((n > 0 && !len) || !pos) return gl_fail(nullptr, GL_EINVAL, "gl_plot_path_xy_size_host: bad argument");
    GL_CHECK(check_charts_host("gl_plot_path_xy_size_host", chart, n, n_charts));
    path_size_host(XySrc{x, y, ptr}, chart, n, xf4, cv, len, pos);
    return GL_OK;
}

int gl_plot_path_xy_emit_host(const double* x, const double* y, const int64_t* ptr, const int32_t* chart, int32_t n, const double* xf4,
                              int32_t n_charts, int32_t kind, int32_t fmt, const int64_t* pos, char* out, int64_t cap) {
    Canvas cv;
    GL_CHECK(path_args(nullptr, "gl_plot_path_xy_emit_host", x, y, ptr, chart, n, xf4, n_charts, kind, fmt, cv));
    if (!pos) return gl_fail(nullptr, GL_EINVAL, "gl_plot_path_xy_emit_host: bad argument");
    GL_CHECK(check_charts_host("gl_plot_path_xy_emit_host", chart, n, n_charts));
    return path_emit_host("gl_plot_path_xy_emit_host", XySrc{x, y, ptr}, chart, n, xf4, cv, pos, out, cap);
}

double gl_plot_line_width(int32_t n_datasets) {
    return n_datasets > 30 ? 0.65 : 0.8;                      // plot.go:508-511, points
}

int gl_plot_vector_write(const char* path, int32_t kind, int32_t fmt, const double* ext4, const char* xtitle, const char* ytitle, int32_t n,
                         const uint8_t* rgb, double width, const char* const* data, const int64_t* len) {
    Canvas cv;
    double xf[4];
    if (!path || !ext4 || !xtitle || !ytitle || n < 0 || (n > 0 && (!rgb || !data || !len)) || !(width > 0) || !canvas_of(kind, fmt, cv))
        return gl_fail(nullptr, GL_EINVAL, "gl_plot_vector_write: bad argument");
    for (int32_t d = 0; d < n; d++)
        if (len[d] < 0 || (len[d] > 0 && !data[d])) return gl_fail(nullptr, GL_EINVAL, "gl_plot_vector_write: dataset %d: bad text", d);
    const bool sq = kind == GL_PLOT_SQUARE;
    GL_CHECK(gl_plot_transform(ext4, sq ? GL_PLOT_SQ_W : GL_PLOT_W, sq ? GL_PLOT_SQ_H : GL_PLOT_H, xf));
    FILE* f = fopen(path, "wb");
    if (!f) return gl_fail(nullptr, GL_EINVAL, "gl_plot_vector_write: cannot create %s", path);
    bool ok = true;
    auto put = [&](const std::string& s) { ok = ok && fwrite(s.data(), 1, s.size(), f) == s.size(); };
    put(vector_head(kind, cv, xf, xtitle, ytitle));
    const std::string w = f2(width);
    for (int32_t d = 0; d < n; d++) {
        if (len[d] == 0) continue;
        const uint8_t* c = rgb + 3 * (size_t)d;
        char pre[96];
        if (cv.eps) snprintf(pre, sizeof pre, "%.4f %.4f %.4f setrgbcolor %s setlinewidth newpath\n", c[0] / 255.0, c[1] / 255.0, c[2] / 255.0, w.c_str());
        else snprintf(pre, sizeof pre, "<path d=\"");
        put(pre);
        ok = ok && fwrite(data[d], 1, (size_t)len[d], f) == (size_t)len[d];
        if (cv.eps) put("stroke\n");
        else { char post[96]; snprintf(post, sizeof post, "\" stroke=\"#%02x%02x%02x\" stroke-width=\"%s\" fill=\"none\"/>\n", c[0], c[1], c[2], w.c_str()); put(post); }
    }
    put(cv.eps ? "showpage\n%%EOF\n" : "</svg>\n");
    ok = fclose(f) == 0 && ok;
    if (!ok) return gl_fail(nullptr, GL_EINVAL, "gl_plot_vector_write: cannot write %s", path);
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
