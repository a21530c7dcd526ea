/* oracle_cnveval.c — TEST INFRASTRUCTURE ONLY: a literal restatement of cnveval/cnveval.go Evaluate, updatePositive and
 * updateFP (:163-341), with the shared pointer i that steps back one call per truth, the `used` map of each truth copy, the
 * fpfound / tpfound flags that updateFP never resets, and `others` built one sample at a time.  Sorting is Go 1.21's
 * sort.Slice (pdqsort_func, src/sort/zsortfunc.go), restated here over records.
 *
 *   orc_go_sort_calls : the permutation sort.Slice leaves for n (chrom, start) keys in file order
 *   orc_cnveval       : stats[S][3][4] (TP, FP, FN, TN per sample and size class) */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
    int32_t chrom;
    int64_t start, end, cn;
    int64_t id;       /* file index (sort) */
    int counted;
} Rec;

typedef struct { Rec* r; } Data;

static int less(const Data* d, int64_t i, int64_t j) {
    return d->r[i].chrom < d->r[j].chrom || (d->r[i].chrom == d->r[j].chrom && d->r[i].start < d->r[j].start);
}
static void swp(Data* d, int64_t i, int64_t j) { Rec t = d->r[i]; d->r[i] = d->r[j]; d->r[j] = t; }

static int bitlen(uint64_t x) { int n = 0; while (x) { n++; x >>= 1; } return n; }

static void insertionSort(Data* d, int64_t a, int64_t b) {
    for (int64_t i = a + 1; i < b; i++)
        for (int64_t j = i; j > a && less(d, j, j - 1); j--) swp(d, j, j - 1);
}

static void siftDown(Data* d, int64_t lo, int64_t hi, int64_t first) {
    int64_t root = lo;
    for (;;) {
        int64_t child = 2 * root + 1;
        if (child >= hi) return;
        if (child + 1 < hi && less(d, first + child, first + child + 1)) child++;
        if (!less(d, first + root, first + child)) return;
        swp(d, first + root, first + child);
        root = child;
    }
}

static void heapSort(Data* d, int64_t a, int64_t b) {
    int64_t first = a, lo = 0, hi = b - a;
    for (int64_t i = (hi - 1) / 2; i >= 0; i--) siftDown(d, i, hi, first);
    for (int64_t i = hi - 1; i >= 0; i--) { swp(d, first, first + i); siftDown(d, lo, i, first); }
}

static int64_t partition(Data* d, int64_t a, int64_t b, int64_t pivot, int* already) {
    swp(d, a, pivot);
    int64_t i = a + 1, j = b - 1;
    while (i <= j && less(d, i, a)) i++;
    while (i <= j && !less(d, j, a)) j--;
    if (i > j) { swp(d, j, a); *already = 1; return j; }
    swp(d, i, j); i++; j--;
    for (;;) {
        while (i <= j && less(d, i, a)) i++;
        while (i <= j && !less(d, j, a)) j--;
        if (i > j) break;
        swp(d, i, j); i++; j--;
    }
    swp(d, j, a);
    *already = 0;
    return j;
}

static int64_t partitionEqual(Data* d, int64_t a, int64_t b, int64_t pivot) {
    swp(d, a, pivot);
    int64_t i = a + 1, j = b - 1;
    for (;;) {
        while (i <= j && !less(d, a, i)) i++;
        while (i <= j && less(d, a, j)) j--;
        if (i > j) break;
        swp(d, i, j); i++; j--;
    }
    return i;
}

static int partialInsertionSort(Data* d, int64_t a, int64_t b) {
    const int maxSteps = 5, shortestShifting = 50;
    int64_t i = a + 1;
    for (int j = 0; j < maxSteps; j++) {
        while (i < b && !less(d, i, i - 1)) i++;
        if (i == b) return 1;
        if (b - a < shortestShifting) return 0;
        swp(d, i, i - 1);
        if (i - a >= 2)
            for (int64_t k = i - 1; k >= 1; k--) { if (!less(d, k, k - 1)) break; swp(d, k, k - 1); }
        if (b - i >= 2)
            for (int64_t k = i + 1; k < b; k++) { if (!less(d, k, k - 1)) break; swp(d, k, k - 1); }
    }
    return 0;
}

static void breakPatterns(Data* d, int64_t a, int64_t b) {
    int64_t length = b - a;
    if (length >= 8) {
        uint64_t random = (uint64_t)length;
        uint64_t modulus = (uint64_t)1 << bitlen((uint64_t)length);
        int64_t idx = a + (length / 4) * 2 - 1;
        for (int i = 0; i < 3; i++) {
            random ^= random << 13; random ^= random >> 7; random ^= random << 17;
            int64_t other = (int64_t)(random & (modulus - 1));
            if (other >= length) other -= length;
            swp(d, idx - 1 + i, a + other);
        }
    }
}

static void order2(Data* d, int64_t* a, int64_t* b, int* swaps) {
    if (less(d, *b, *a)) { (*swaps)++; int64_t t = *a; *a = *b; *b = t; }
}

static int64_t median(Data* d, int64_t a, int64_t b, int64_t c, int* swaps) {
    order2(d, &a, &b, swaps);
    order2(d, &b, &c, swaps);
    order2(d, &a, &b, swaps);
    return b;
}

static int64_t medianAdjacent(Data* d, int64_t a, int* swaps) { return median(d, a - 1, a, a + 1, swaps); }

enum { unknownHint, increasingHint, decreasingHint };

static int64_t choosePivot(Data* d, int64_t a, int64_t b, int* hint) {
    const int64_t shortestNinther = 50;
    const int maxSwaps = 4 * 3;
    int64_t l = b - a;
    int swaps = 0;
    int64_t i = a + l / 4 * 1, j = a + l / 4 * 2, k = a + l / 4 * 3;
    if (l >= 8) {
        if (l >= shortestNinther) {
            i = medianAdjacent(d, i, &swaps);
            j = medianAdjacent(d, j, &swaps);
            k = medianAdjacent(d, k, &swaps);
        }
        j = median(d, i, j, k, &swaps);
    }
    if (swaps == 0) *hint = increasingHint;
    else if (swaps == maxSwaps) *hint = decreasingHint;
    else *hint = unknownHint;
    return j;
}

static void reverseRange(Data* d, int64_t a, int64_t b) {
    for (int64_t i = a, j = b - 1; i < j; i++, j--) swp(d, i, j);
}

static void pdqsort_func(Data* d, int64_t a, int64_t b, int limit) {
    const int64_t maxInsertion = 12;
    int wasBalanced = 1, wasPartitioned = 1;
    for (;;) {
        int64_t length = b - a;
        if (length <= maxInsertion) { insertionSort(d, a, b); return; }
        if (limit == 0) { heapSort(d, a, b); return; }
        if (!wasBalanced) { breakPatterns(d, a, b); limit--; }
        int hint;
        int64_t pivot = choosePivot(d, a, b, &hint);
        if (hint == decreasingHint) {
            reverseRange(d, a, b);
            pivot = (b - 1) - (pivot - a);
            hint = increasingHint;
        }
        if (wasBalanced && wasPartitioned && hint == increasingHint)
            if (partialInsertionSort(d, a, b)) return;
        if (a > 0 && !less(d, a - 1, pivot)) {
            a = partitionEqual(d, a, b, pivot);
            continue;
        }
        int already = 0;
        int64_t mid = partition(d, a, b, pivot, &already);
        wasPartitioned = already;
        int64_t left = mid - a, right = b - mid, balanceThreshold = length / 8;
        if (left < right) {
            wasBalanced = left >= balanceThreshold;
            pdqsort_func(d, a, mid, limit);
            a = mid + 1;
        } else {
            wasBalanced = right >= balanceThreshold;
            pdqsort_func(d, mid + 1, b, limit);
            b = mid;
        }
    }
}

/* sort.Slice(x, less by (chrom, start)) */
static void sort_slice(Rec* r, int64_t n) {
    Data d = {r};
    pdqsort_func(&d, 0, n, bitlen((uint64_t)n));
}

void orc_go_sort_calls(const int32_t* chrom, const int64_t* start, int64_t n, int64_t* perm) {
    Rec* r = (Rec*)calloc((size_t)(n > 0 ? n : 1), sizeof(Rec));
    for (int64_t i = 0; i < n; i++) { r[i].chrom = chrom[i]; r[i].start = start[i]; r[i].id = i; }
    sort_slice(r, n);
    for (int64_t i = 0; i < n; i++) perm[i] = r[i].id;
    free(r);
}

/* ---------------------------------------------------------------- Evaluate */
static int size_class(int64_t s, int64_t e) {
    int64_t l = e - s;
    if (l < 20000) return 0;
    if (l < 100000) return 1;
    return 2;
}

static int sameCN(int64_t a, int64_t b) {
    if (a > 2) a = 3;
    if (b > 2) b = 3;
    return a == b;
}

static double poverlap(const Rec* a, const Rec* b) {
    if (a->chrom != b->chrom) return 0;
    double la = (double)(a->end - a->start), lb = (double)(b->end - b->start);
    double total = la < lb ? la : lb;                      /* math.Min: lengths are never NaN */
    int64_t ovl = (a->end < b->end ? a->end : b->end) - (a->start > b->start ? a->start : b->start);
    if (ovl < 0) return 0;
    return (double)ovl / total;
}

enum { TP = 0, FP = 1, FN = 2, TN = 3 };

static void updatePositive(uint64_t* st, Rec* truths, int64_t nt, Rec* cnvs, int64_t nc, double po) {
    if (nc == 0) return;
    int64_t i = 0;
    for (int64_t ti = 0; ti < nt; ti++) {
        const Rec* t = &truths[ti];
        int found = 0, used = 0;                           /* t.used: a fresh map on each loop copy */
        uint64_t* val = st + size_class(t->start, t->end) * 4;
        for (; i < nc && (cnvs[i].chrom < t->chrom || (cnvs[i].chrom == t->chrom && cnvs[i].end < t->start)); i++) {}
        if (i > 0) i--;
        for (int64_t k = i; k < nc; k++) {
            Rec* cnv = &cnvs[k];
            if (cnv->chrom > t->chrom || (t->chrom == cnv->chrom && cnv->start > t->end)) break;
            if (poverlap(cnv, t) >= po && sameCN(cnv->cn, t->cn)) {
                if (!used) {
                    val[TP]++;
                    cnv->counted = 1;
                    found = 1;
                    used = 1;
                }
            }
        }
        if (!found) val[FN]++;
    }
    for (int64_t k = 0; k < nc; k++)
        if (!cnvs[k].counted) st[size_class(cnvs[k].start, cnvs[k].end) * 4 + FP]++;
}

static void updateFP(uint64_t* st, Rec* others, int64_t no, Rec* cnvs, int64_t nc, Rec* truths, int64_t nt, double po) {
    if (nc == 0 || no == 0) return;
    int64_t i = 0;
    for (int64_t oi = 0; oi < no; oi++) {
        const Rec* o = &others[oi];
        uint64_t* val = st + size_class(o->start, o->end) * 4;
        for (; i < nc && (cnvs[i].chrom < o->chrom || (cnvs[i].chrom == o->chrom && cnvs[i].end < o->start)); i++) {}
        if (i > 0) i--;
        int tpfound = 0, fpfound = 0, found = 0;
        for (int64_t k = i; k < nc; k++) {
            Rec* cnv = &cnvs[k];
            if (cnv->chrom > o->chrom || (o->chrom == cnv->chrom && cnv->start > o->end)) break;
            if (poverlap(cnv, o) >= po && sameCN(cnv->cn, o->cn)) {
                fpfound = 1;
                for (int64_t j = 0; j < nt; j++) {
                    const Rec* t = &truths[j];
                    if (t->chrom != cnv->chrom) continue;
                    if (poverlap(cnv, t) >= po && sameCN(cnv->cn, t->cn)) { tpfound = 1; break; }
                }
            }
            if (fpfound && !tpfound) {
                val[FP]++;
                found = 1;
                cnv->counted = 1;
            }
        }
        if (!(found || tpfound)) val[TN]++;
    }
}

/* calls in file order (sample, chrom, start, end, cn); truths in file order with samples t_mem_sample[t_mem_ptr[t] ..
 * t_mem_ptr[t+1]); stats[S * 12] is overwritten */
void orc_cnveval(int32_t S, const int32_t* c_sample, const int32_t* c_chrom, const int64_t* c_start, const int64_t* c_end,
                 const int64_t* c_cn, int64_t n_calls, const int32_t* t_chrom, const int64_t* t_start, const int64_t* t_end,
                 const int64_t* t_cn, int64_t n_truths, const int64_t* t_mem_ptr, const int32_t* t_mem_sample, double po,
                 uint64_t* stats) {
    memset(stats, 0, (size_t)S * 12 * sizeof(uint64_t));
    int64_t n_mem = n_truths > 0 ? t_mem_ptr[n_truths] : 0;
    Rec* cn = (Rec*)calloc((size_t)(n_calls + 1), sizeof(Rec));
    Rec* own = (Rec*)calloc((size_t)(n_mem + 1), sizeof(Rec));
    Rec* oth = (Rec*)calloc((size_t)(n_truths + 1), sizeof(Rec));
    for (int32_t s = 0; s < S; s++) {
        int64_t nc = 0, nt = 0, no = 0;
        for (int64_t t = 0; t < n_truths; t++) {
            Rec r = {t_chrom[t], t_start[t], t_end[t], t_cn[t], t, 0};
            int in = 0;
            for (int64_t k = t_mem_ptr[t]; k < t_mem_ptr[t + 1]; k++)
                if (t_mem_sample[k] == s) { own[nt++] = r; in = 1; }     /* truthBySample: once per listing */
            if (!in) oth[no++] = r;                                    /* truthWithoutSample: notin */
        }
        for (int64_t i = 0; i < n_calls; i++)
            if (c_sample[i] == s) { Rec r = {c_chrom[i], c_start[i], c_end[i], c_cn[i], i, 0}; cn[nc++] = r; }
        sort_slice(own, nt);
        sort_slice(cn, nc);
        uint64_t* st = stats + (int64_t)s * 12;
        updatePositive(st, own, nt, cn, nc, po);
        sort_slice(oth, no);
        updateFP(st, oth, no, cn, nc, own, nt, po);
    }
    free(cn); free(own); free(oth);
}
