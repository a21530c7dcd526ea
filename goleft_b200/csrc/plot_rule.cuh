// plot_rule.cuh — the float64 raster rule of the charts (plot.cu, dcnv_chart.cu; DESIGN §1.14).  See plot.cu's header
// for the rule.  Every operation is one float64 round-to-nearest step in the order written: explicit _rn intrinsics on
// the device, plain operations on the host (the library is built with --fmad=false and no host FMA), so the host mirrors
// and numpy (tests/plot_rule.py) restate the device bit for bit.
#pragma once
#include <math.h>

namespace glplot {

__host__ __device__ inline double p_add(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
__host__ __device__ inline double p_sub(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
__host__ __device__ inline double p_mul(double a, double b) {
#ifdef __CUDA_ARCH__
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
__host__ __device__ inline double p_div(double a, double b) {
#ifdef __CUDA_ARCH__
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// Segment (x0,y0)-(x1,y1) in data coordinates through chart transform f = {xmin, sx, ymin, sy}: plot(i, j) for every
// covered pixel of the W x H data area.  A pixel for which skip(i, j) holds is not tested; callers pass a skip that only
// holds where plot would change nothing.
template <class Skip, class Plot>
__host__ __device__ inline void draw_segment(double x0, double y0, double x1, double y1, const double* f, int W, int H,
                                             double r, double r2, Skip&& skip, Plot&& plot) {
    const double hh = (double)H;
    const double ax = p_mul(p_sub(x0, f[0]), f[1]), ay = p_sub(hh, p_mul(p_sub(y0, f[2]), f[3]));
    const double bx = p_mul(p_sub(x1, f[0]), f[1]), by = p_sub(hh, p_mul(p_sub(y1, f[2]), f[3]));
    const double dx = p_sub(bx, ax), dy = p_sub(by, ay);
    const double L = p_add(p_mul(dx, dx), p_mul(dy, dy));
    // a conservative box: the exact test below decides every pixel in it
    int i0 = (int)floor(fmin(ax, bx) - r) - 1, i1 = (int)ceil(fmax(ax, bx) + r) + 1;
    int j0 = (int)floor(fmin(ay, by) - r) - 1, j1 = (int)ceil(fmax(ay, by) + r) + 1;
    i0 = i0 < 0 ? 0 : i0; j0 = j0 < 0 ? 0 : j0; i1 = i1 > W - 1 ? W - 1 : i1; j1 = j1 > H - 1 ? H - 1 : j1;
    for (int j = j0; j <= j1; j++) {
        const double ey = p_sub((double)j + 0.5, ay);
        for (int i = i0; i <= i1; i++) {
            if (skip(i, j)) continue;
            const double ex = p_sub((double)i + 0.5, ax);
            double qx = ex, qy = ey;
            if (L != 0.0) {
                double t = p_div(p_add(p_mul(ex, dx), p_mul(ey, dy)), L);
                t = t < 0.0 ? 0.0 : (t > 1.0 ? 1.0 : t);
                qx = p_sub(ex, p_mul(t, dx));
                qy = p_sub(ey, p_mul(t, dy));
            }
            if (p_add(p_mul(qx, qx), p_mul(qy, qy)) <= r2) plot(i, j);
        }
    }
}

template <class Plot>
__host__ __device__ inline void draw_segment(double x0, double y0, double x1, double y1, const double* f, int W, int H,
                                             double r, double r2, Plot&& plot) {
    draw_segment(x0, y0, x1, y1, f, W, H, r, r2, [](int, int) { return false; }, plot);
}

}  // namespace glplot
