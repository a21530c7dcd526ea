/* oracle_emdepth.c — TEST INFRASTRUCTURE ONLY.  A literal, single-threaded restatement of emdepth/emdepth.go (EMDepth,
 * Type, adjustCN, Log2FC) and stats.go (pmf with its Lgamma table), one row at a time, with glibc's pow route, exp, log,
 * lgamma and log2: a full sort for the median, the bins as arrays, sequential float64 means.  The Cache lives in
 * oracle/emdepth.py.  Built with -ffp-contract=off. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define EM_CN 9

/* math.Pow(x, y) for x > 0, y = 1.1 as Go's pow.go computes it, with glibc's exp / log */
static double go_pow(double x, double y) {
    double yi;
    double yf = modf(fabs(y), &yi);
    double a1 = 1.0;
    int ae = 0;
    if (yf != 0) {
        if (yf > 0.5) { yf--; yi++; }
        a1 = exp(yf * log(x));
    }
    int xe;
    double x1 = frexp(x, &xe);
    for (int64_t i = (int64_t)yi; i != 0; i >>= 1) {
        if (xe < -(1 << 12) || (1 << 12) < xe) { ae += xe; break; }
        if (i & 1) { a1 *= x1; ae += xe; }
        x1 *= x1;
        xe <<= 1;
        if (x1 < .5) { x1 += x1; xe--; }
    }
    return ldexp(a1, ae);
}

void orc_em_factors(double* f9) {
    for (int i = 0; i < EM_CN; i++) f9[i] = (i == 0 || i == 2) ? (double)(i / 2) : go_pow((double)i / 2, 1.1);
}

static int cmp_f64(const void* a, const void* b) {
    const double x = *(const double*)a, y = *(const double*)b;
    return x < y ? -1 : x > y;
}

static double go_abs(double a) { return a < 0 ? -a : a; }

static int search(const double* l, double d) {           /* sort.SearchFloat64s */
    int i = 0, j = EM_CN;
    while (i < j) {
        int h = (int)((unsigned)(i + j) >> 1);
        if (!(l[h] >= d)) i = h + 1;
        else j = h;
    }
    return i;
}

static double mean64(const double* a, int n) {
    if (n == 0) return 0;
    double s = 0;
    for (int i = 0; i < n; i++) s += a[i];
    return s / (double)n;
}

static double gammas[1000];
static int gammas_ready;

static double pmf(int64_t k, double mu) {
    if (!gammas_ready) {
        for (int i = 0; i < 1000; i++) gammas[i] = lgamma((double)(i + 1));
        gammas_ready = 1;
    }
    int sign = 1;
    double lg;
    if (k < 1000) lg = gammas[k];
    else { lg = lgamma((double)(k + 1)); sign = signgam; }
    return exp((double)k * log(mu) - (double)sign * lg - mu);
}

static int type_cn(const double* l, float df) {          /* Type + adjustCN */
    const double d = df;
    const int idx = search(l, d);
    int cn;
    if (idx == 0) cn = 0;
    else if (idx == EM_CN) cn = EM_CN;
    else cn = go_abs(d - l[idx]) < go_abs(d - l[idx - 1]) ? idx : idx - 1;
    if (cn != 2 && cn < EM_CN) {
        const int64_t dk = (int64_t)(0.5 + d);
        const double o = pmf(dk, l[cn]), o2 = pmf(dk, l[2]);
        if (o * 0.9 < o2) cn = 2;
    }
    return cn;
}

/* EMDepth of one row; b (S doubles) and bins (9 x S doubles) are scratch */
static void em_row(const float* x, int S, double* l, double* b, double* bins) {
    for (int i = 0; i < S; i++) b[i] = x[i];
    qsort(b, (size_t)S, sizeof(double), cmp_f64);
    const double m = S % 2 == 1 ? b[S / 2] : (b[S / 2] + b[S / 2 + 1]) / 2;
    double last[EM_CN];
    int cnt[EM_CN];
    l[0] = 0.01 * m;
    l[2] = m;
    last[0] = l[0];
    for (int i = 1; i < EM_CN; i++)
        if (i != 2) l[i] = l[2] * go_pow((double)i / 2, 1.1);
    double sumd = 100, maxd = 100;
    for (int iter = 0; iter < 10 && sumd > 0.01 && maxd > 0.5; iter++) {
        for (int i = 1; i < EM_CN; i++) last[i] = l[i];
        for (int i = 0; i < EM_CN; i++) cnt[i] = 0;
        for (int s = 0; s < S; s++) {
            const double d = x[s];
            int bin;
            if (d > l[1] && d < l[3] && go_abs(d - l[2]) < go_abs(d - l[1]) && go_abs(d - l[2]) < go_abs(d - l[3])) {
                bin = 2;
            } else {
                const int idx = search(l, d);
                if (idx == 0) bin = 0;
                else if (idx == EM_CN) bin = idx - 1;
                else bin = go_abs(d - l[idx]) < go_abs(d - l[idx - 1]) ? idx : idx - 1;
            }
            bins[(size_t)bin * S + cnt[bin]++] = d;
        }
        l[2] = mean64(bins + 2 * (size_t)S, cnt[2]);
        if (l[2] == 0) {
            const double n = (double)S;
            for (int i = 1; i < EM_CN - 1; i++) {
                const double pdepth = (double)cnt[i] / n;
                if (l[i] < 0.01) l[i] = 0.01;
                l[2] += mean64(bins + (size_t)i * S, cnt[i]) * (2 / (double)i) * pdepth;
            }
        }
        for (int i = 1; i < EM_CN; i++) l[i] = l[2] * ((double)i / 2);
        const double span = l[2] - l[1];
        l[1] -= span / 1.5;
        l[3] += span / 1.5;
        sumd = 0; maxd = 0;
        for (int i = 0; i < EM_CN; i++) {
            const double d = go_abs(l[i] - last[i]);
            sumd += d;
            if (d > maxd) maxd = d;
        }
    }
}

/* n rows of x (row stride ld) -> cells (n x S: CN | class << 4 | outside << 6), lambda (n x 9, nullable), fc (n x S,
 * nullable).  Returns 0; -1 when S is 0 or 2 (the reference's median indexes out of range); -2 - r when row r holds a value
 * the library rejects (sign bit set, not finite, or >= 2^62). */
int orc_emdepth(const float* x, int64_t n, int64_t ld, int S, uint8_t* cells, double* lambda, double* fc) {
    if (S < 1 || S == 2) return -1;
    for (int64_t r = 0; r < n; r++)
        for (int s = 0; s < S; s++) {
            uint32_t bits;
            memcpy(&bits, x + r * ld + s, 4);
            if (bits >= 0x5e800000u) return (int)(-2 - r);
        }
    double* b = malloc(sizeof(double) * (size_t)S);
    double* bins = malloc(sizeof(double) * (size_t)S * EM_CN);
    for (int64_t r = 0; r < n; r++) {
        const float* row = x + r * ld;
        double l[EM_CN];
        em_row(row, S, l, b, bins);
        if (lambda) memcpy(lambda + r * EM_CN, l, sizeof l);
        for (int s = 0; s < S; s++) {
            const int cn = type_cn(l, row[s]);
            const double f = log2((double)row[s] / l[2]);
            int cls;
            if (f > -0.8 && f < 0.4) cls = 0;
            else if (f <= -0.8) cls = 1;
            else if (f >= 0.4) cls = 2;
            else cls = 3;
            const int outside = !(f > -0.5 && f < 0.3);
            cells[r * S + s] = (uint8_t)(cn | cls << 4 | outside << 6);
            if (fc) fc[r * S + s] = f;
        }
    }
    free(b);
    free(bins);
    return 0;
}
