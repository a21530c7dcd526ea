// pca_eig.cpp — see pca_eig.h.  Host-only and deterministic: the same input gives the same bits.  Only
// tridiag_values_above runs on the host pool, one independent bisection per index.
#include "pca_eig.h"

#include <float.h>
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "../../../include/goleft_b200.h"
#include "thread_pool.h"

namespace glpca {
namespace {

// number of eigenvalues of T below x (Sturm sequence of the LDL^T pivots; a pivot smaller than pivmin is taken as -pivmin)
int count_below(const double* d, const double* e2, int n, double x, double pivmin) {
    int c = 0;
    double q = 1;
    for (int i = 0; i < n; i++) {
        double t = d[i] - x - (i ? e2[i - 1] / q : 0.0);
        if (fabs(t) < pivmin) t = -pivmin;
        c += t < 0;
        q = t;
    }
    return c;
}

double inf_norm(const double* d, const double* e, int n) {
    double nrm = 0;
    for (int i = 0; i < n; i++) nrm = std::max(nrm, fabs(d[i]) + (i ? fabs(e[i - 1]) : 0.0) + (i + 1 < n ? fabs(e[i]) : 0.0));
    return nrm;
}

// what every bisection of one T shares: the squared off-diagonal, the pivot floor and the padded Gershgorin interval
struct Sturm {
    const double* d;
    int n;
    std::vector<double> e2;
    double pivmin, glo, ghi;
    Sturm(const double* d_, const double* e, int n_) : d(d_), n(n_), e2(n_ > 1 ? n_ - 1 : 1, 0.0) {
        double emax2 = 0;
        for (int i = 0; i + 1 < n; i++) { e2[i] = e[i] * e[i]; emax2 = std::max(emax2, e2[i]); }
        pivmin = DBL_MIN * std::max(1.0, emax2);
        glo = d[0], ghi = d[0];                                      // Gershgorin interval
        for (int i = 0; i < n; i++) {
            const double r = (i ? fabs(e[i - 1]) : 0.0) + (i + 1 < n ? fabs(e[i]) : 0.0);
            glo = std::min(glo, d[i] - r);
            ghi = std::max(ghi, d[i] + r);
        }
        const double pad = 4 * DBL_EPSILON * n * std::max(fabs(glo), fabs(ghi)) + 2 * pivmin;
        glo -= pad;
        ghi += pad;
    }
    int below(double x) const { return count_below(d, e2.data(), n, x, pivmin); }
    // the eigenvalue with ascending index t, bisected until no double lies strictly inside (lo, hi)
    double value(int t) const {
        double lo = glo, hi = ghi;
        for (;;) {
            const double mid = lo + 0.5 * (hi - lo);
            if (!(mid > lo && mid < hi)) break;
            if (below(mid) <= t) lo = mid;
            else hi = mid;
        }
        return lo + 0.5 * (hi - lo);
    }
};

}  // namespace

void tridiag_top_values(const double* d, const double* e, int n, int k, double* w) {
    const Sturm st(d, e, n);
    for (int j = 0; j < k; j++) w[j] = st.value(n - 1 - j);           // ascending index of the j-th largest
}

int tridiag_values_above(const double* d, const double* e, int n, double rel, double* w) {
    const Sturm st(d, e, n);
    const double top = st.value(n - 1);
    if (!(top > 0)) return 0;
    const double thr = rel * top;
    const int m = std::max(1, n - st.below(thr));                    // eigenvalues >= thr; the bisection settles the rest
    w[0] = top;
    if (m > 1) glhost::ThreadPool::global().run(m - 1, [&](int64_t j, int) { w[j + 1] = st.value(n - 2 - (int)j); });
    int k = 1;
    while (k < m && w[k] > thr) k++;
    return k;
}

void tridiag_vectors(const double* d, const double* e, int n, const double* w, int k, double* z) {
    const double tnorm = inf_norm(d, e, n);
    memset(z, 0, sizeof(double) * (size_t)n * (size_t)k);
    if (tnorm == 0) {                                                // T = 0: any orthonormal set
        for (int j = 0; j < k; j++) z[(size_t)j * n + j] = 1;
        return;
    }
    const double eps = DBL_EPSILON, ortol = 1e-3 * tnorm, sep = 10 * eps * tnorm, tiny = eps * tnorm;
    constexpr int kSolves = 4;                                       // inverse iteration steps per vector (fixed)
    std::vector<double> u0(n), u1(n), u2(n), mult(n), y(n);
    std::vector<char> swp(n);
    double prev = 0;
    int cluster0 = 0;
    for (int j = 0; j < k; j++) {
        double lam = w[j];
        if (j > 0) {
            if (w[j - 1] - w[j] > ortol) cluster0 = j;
            else if (lam > prev - sep) lam = prev - sep;             // coincident eigenvalues: separate the shifts
        }
        prev = lam;
        // LU of T - lam I with partial pivoting: U has two superdiagonals; row i of L is (mult[i], swap[i])
        double p = d[0] - lam, q = n > 1 ? e[0] : 0.0;
        for (int i = 0; i + 1 < n; i++) {
            const double a = e[i], b = d[i + 1] - lam, c = i + 2 < n ? e[i + 1] : 0.0;
            if (fabs(a) > fabs(p)) {
                const double m = p / a;
                swp[i] = 1; mult[i] = m;
                u0[i] = a; u1[i] = b; u2[i] = c;
                p = q - m * b;
                q = -m * c;
            } else {
                if (p == 0) p = tiny;                                // a == p == 0: the column is already eliminated
                const double m = a / p;
                swp[i] = 0; mult[i] = m;
                u0[i] = p; u1[i] = q; u2[i] = 0;
                p = b - m * q;
                q = c;
            }
        }
        u0[n - 1] = p;
        for (int i = 0; i < n; i++)
            if (fabs(u0[i]) < tiny) u0[i] = u0[i] < 0 ? -tiny : tiny;
        uint64_t s = 0x9E3779B97F4A7C15ull * (uint64_t)(j + 1);     // fixed pseudo-random start
        for (int i = 0; i < n; i++) {
            s = s * 6364136223846793005ull + 1442695040888963407ull;
            y[i] = (double)(int64_t)(s >> 11) * 0x1p-52 - 1.0;
        }
        for (int it = 0; it < kSolves; it++) {
            for (int i = 0; i + 1 < n; i++) {                        // L
                if (swp[i]) { const double t = y[i]; y[i] = y[i + 1]; y[i + 1] = t - mult[i] * y[i]; }
                else y[i + 1] -= mult[i] * y[i];
            }
            for (int i = n - 1; i >= 0; i--) {                       // U
                double t = y[i];
                if (i + 1 < n) t -= u1[i] * y[i + 1];
                if (i + 2 < n) t -= u2[i] * y[i + 2];
                y[i] = t / u0[i];
            }
            for (int c = cluster0; c < j; c++) {                     // re-orthogonalise inside the cluster
                const double* zc = z + (size_t)c * n;
                double dot = 0;
                for (int i = 0; i < n; i++) dot += zc[i] * y[i];
                for (int i = 0; i < n; i++) y[i] -= dot * zc[i];
            }
            double mx = 0;
            for (int i = 0; i < n; i++) mx = std::max(mx, fabs(y[i]));
            if (mx == 0) { y[std::min(j, n - 1)] = 1; mx = 1; }
            for (int i = 0; i < n; i++) y[i] /= mx;
        }
        double nrm = 0;
        for (int i = 0; i < n; i++) nrm += y[i] * y[i];
        nrm = sqrt(nrm);
        double* zj = z + (size_t)j * n;
        for (int i = 0; i < n; i++) zj[i] = y[i] / nrm;
    }
}

void project(const double* lambda, double* u, const double* c, int S, int k, double* proj, double* sv) {
    for (int j = 0; j < k; j++) {
        double* uj = u + (size_t)j * S;
        const bool zero = !(lambda[0] > 0) || !(lambda[j] > kRankTol * lambda[0]);
        sv[j] = zero ? 0.0 : sqrt(lambda[j]);
        if (zero) {
            for (int i = 0; i < S; i++) proj[(size_t)i * k + j] = 0.0;
            continue;
        }
        int imax = 0;                                                // sign rule
        for (int i = 1; i < S; i++)
            if (fabs(uj[i]) > fabs(uj[imax])) imax = i;
        if (uj[imax] < 0)
            for (int i = 0; i < S; i++) uj[i] = -uj[i];
        double cu = 0;
        for (int i = 0; i < S; i++) cu += c[i] * uj[i];
        const double off = cu / sv[j];
        for (int i = 0; i < S; i++) proj[(size_t)i * k + j] = sv[j] * uj[i] + off;
    }
}

}  // namespace glpca

extern "C" int gl_pca_tridiag_top(const double* d, const double* e, int32_t n, int32_t k, double* w, double* z) {
    if (!d || (n > 1 && !e) || !w || n < 1 || k < 1 || k > n) return GL_EINVAL;
    glpca::tridiag_top_values(d, e, n, k, w);
    if (z) glpca::tridiag_vectors(d, e, n, w, k, z);
    return GL_OK;
}

extern "C" int gl_pca_tridiag_above(const double* d, const double* e, int32_t n, double rel, double* w, int32_t* count) {
    if (!d || (n > 1 && !e) || !w || !count || n < 1 || !(rel >= 0) || !(rel < 1)) return GL_EINVAL;
    *count = glpca::tridiag_values_above(d, e, n, rel, w);
    return GL_OK;
}

extern "C" int gl_indexcov_pca_total(const uint8_t* x, int64_t ld, int32_t S, int64_t D, double* total) {
    if (!total || S < 1 || D < 0 || ld < D || (D > 0 && !x)) return GL_EINVAL;
    std::vector<int64_t> sum((size_t)D, 0), sq((size_t)D, 0);
    for (int32_t i = 0; i < S; i++) {
        const uint8_t* row = x + (size_t)i * (size_t)ld;
        for (int64_t j = 0; j < D; j++) { sum[(size_t)j] += row[j]; sq[(size_t)j] += (int64_t)row[j] * row[j]; }
    }
    __int128 acc = 0;
    for (int64_t j = 0; j < D; j++) acc += (__int128)S * sq[(size_t)j] - (__int128)sum[(size_t)j] * sum[(size_t)j];
    *total = (double)acc / (double)S;
    return GL_OK;
}
