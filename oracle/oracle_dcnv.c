/* oracle_dcnv.c — TEST INFRASTRUCTURE: a plain C restatement of dcnv/dcnv.go main() (:323-354) after the text is parsed
 * (oracle/dcnv.py parses it and takes the GC through orc_faidx_stats).  Written to be obviously literal, not fast:
 *   - sort.Sort (go 1.21 pdqsort, src/sort/zsortinterface.go) over an Interface of Less / Swap callbacks, as
 *     floats.Argsort drives it (gonum v0.14.0);
 *   - GeneralDebiaser.Debias replayed push by push over a 9-slot FIFO whose median sorts a copy of the window
 *     (JaderDias/movingmedian semantics: even count -> (lo + hi) / 2; UNPINNED, its source is not in the reference tree);
 *   - SampleMedians with a full sort per sample, NormalizeBySampleMedian, and "%.2f" through snprintf. */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------ sort.Sort */
typedef struct {
    int (*less)(void* self, int64_t i, int64_t j);
    void (*swap)(void* self, int64_t i, int64_t j);
    void* self;
} GoSort;

#define LESS(i, j) d->less(d->self, (i), (j))
#define SWAP(i, j) d->swap(d->self, (i), (j))

static int go_bits_len(uint64_t x) { int n = 0; for (; x; x >>= 1) n++; return n; }

static void go_insertion_sort(GoSort* d, int64_t a, int64_t b) {
    for (int64_t i = a + 1; i < b; i++)
        for (int64_t j = i; j > a && LESS(j, j - 1); j--) SWAP(j, j - 1);
}

static void go_sift_down(GoSort* d, int64_t lo, int64_t hi, int64_t first) {
    int64_t root = lo;
    for (;;) {
        int64_t child = 2 * root + 1;
        if (child >= hi) return;
        if (child + 1 < hi && LESS(first + child, first + child + 1)) child++;
        if (!LESS(first + root, first + child)) return;
        SWAP(first + root, first + child);
        root = child;
    }
}

static void go_heap_sort(GoSort* d, int64_t a, int64_t b) {
    int64_t first = a, lo = 0, hi = b - a;
    for (int64_t i = (hi - 1) / 2; i >= 0; i--) go_sift_down(d, i, hi, first);
    for (int64_t i = hi - 1; i >= 0; i--) { SWAP(first, first + i); go_sift_down(d, lo, i, first); }
}

static int64_t go_partition(GoSort* d, int64_t a, int64_t b, int64_t pivot, int* already) {
    SWAP(a, pivot);
    int64_t i = a + 1, j = b - 1;
    while (i <= j && LESS(i, a)) i++;
    while (i <= j && !LESS(j, a)) j--;
    if (i > j) { SWAP(j, a); *already = 1; return j; }
    SWAP(i, j); i++; j--;
    for (;;) {
        while (i <= j && LESS(i, a)) i++;
        while (i <= j && !LESS(j, a)) j--;
        if (i > j) break;
        SWAP(i, j); i++; j--;
    }
    SWAP(j, a);
    *already = 0;
    return j;
}

static int64_t go_partition_equal(GoSort* d, int64_t a, int64_t b, int64_t pivot) {
    SWAP(a, pivot);
    int64_t i = a + 1, j = b - 1;
    for (;;) {
        while (i <= j && !LESS(a, i)) i++;
        while (i <= j && LESS(a, j)) j--;
        if (i > j) break;
        SWAP(i, j); i++; j--;
    }
    return i;
}

static int go_partial_insertion_sort(GoSort* d, int64_t a, int64_t b) {
    int64_t i = a + 1;
    for (int k = 0; k < 5; k++) {                    /* maxSteps */
        while (i < b && !LESS(i, i - 1)) i++;
        if (i == b) return 1;
        if (b - a < 50) return 0;                    /* shortestShifting */
        SWAP(i, i - 1);
        if (i - a >= 2) {
            for (int64_t j = i - 1; j >= 1; j--) { if (!LESS(j, j - 1)) break; SWAP(j, j - 1); }
        }
        if (b - i >= 2) {
            for (int64_t j = i + 1; j < b; j++) { if (!LESS(j, j - 1)) break; SWAP(j, j - 1); }
        }
    }
    return 0;
}

static void go_break_patterns(GoSort* d, int64_t a, int64_t b) {
    int64_t length = b - a;
    if (length >= 8) {
        uint64_t r = (uint64_t)length;
        uint64_t modulus = (uint64_t)1 << go_bits_len((uint64_t)length);
        int64_t idx = a + (length / 4) * 2 - 1;
        for (int i = 0; i < 3; i++) {
            r ^= r << 13; r ^= r >> 7; r ^= r << 17;  /* xorshift.Next */
            int64_t other = (int64_t)(r & (modulus - 1));
            if (other >= length) other -= length;
            SWAP(idx - 1 + i, a + other);
        }
    }
}

static void go_order2(GoSort* d, int64_t* a, int64_t* b, int* swaps) {
    if (LESS(*b, *a)) { (*swaps)++; int64_t t = *a; *a = *b; *b = t; }
}

static int64_t go_median(GoSort* d, int64_t a, int64_t b, int64_t c, int* swaps) {
    go_order2(d, &a, &b, swaps);
    go_order2(d, &b, &c, swaps);
    go_order2(d, &a, &b, swaps);
    return b;
}

/* hint: 0 unknown, 1 increasing, 2 decreasing */
static int64_t go_choose_pivot(GoSort* d, int64_t a, int64_t b, int* hint) {
    int64_t l = b - a;
    int swaps = 0;
    int64_t i = a + l / 4 * 1, j = a + l / 4 * 2, k = a + l / 4 * 3;
    if (l >= 8) {
        if (l >= 50) {                               /* shortestNinther: medianAdjacent */
            i = go_median(d, i - 1, i, i + 1, &swaps);
            j = go_median(d, j - 1, j, j + 1, &swaps);
            k = go_median(d, k - 1, k, k + 1, &swaps);
        }
        j = go_median(d, i, j, k, &swaps);
    }
    *hint = swaps == 0 ? 1 : (swaps == 12 ? 2 : 0);
    return j;
}

static void go_pdqsort(GoSort* d, int64_t a, int64_t b, int limit) {
    int was_balanced = 1, was_partitioned = 1;
    for (;;) {
        int64_t length = b - a;
        if (length <= 12) { go_insertion_sort(d, a, b); return; }
        if (limit == 0) { go_heap_sort(d, a, b); return; }
        if (!was_balanced) { go_break_patterns(d, a, b); limit--; }
        int hint;
        int64_t pivot = go_choose_pivot(d, a, b, &hint);
        if (hint == 2) {
            for (int64_t i = a, j = b - 1; i < j; i++, j--) SWAP(i, j);   /* reverseRange */
            pivot = (b - 1) - (pivot - a);
            hint = 1;
        }
        if (was_balanced && was_partitioned && hint == 1) {
            if (go_partial_insertion_sort(d, a, b)) return;
        }
        if (a > 0 && !LESS(a - 1, pivot)) {
            a = go_partition_equal(d, a, b, pivot);
            continue;
        }
        int already;
        int64_t mid = go_partition(d, a, b, pivot, &already);
        was_partitioned = already;
        int64_t left = mid - a, right = b - mid, thr = length / 8;
        if (left < right) {
            was_balanced = left >= thr;
            go_pdqsort(d, a, mid, limit);
            a = mid + 1;
        } else {
            was_balanced = right >= thr;
            go_pdqsort(d, mid + 1, b, limit);
            b = mid;
        }
    }
}

static void go_sort(GoSort* d, int64_t n) {
    if (n <= 1) return;
    go_pdqsort(d, 0, n, go_bits_len((uint64_t)n));
}

typedef struct { double* s; int64_t* inds; } Argsort;
static int as_less(void* p, int64_t i, int64_t j) { Argsort* a = (Argsort*)p; return a->s[i] < a->s[j]; }
static void as_swap(void* p, int64_t i, int64_t j) {
    Argsort* a = (Argsort*)p;
    double t = a->s[i]; a->s[i] = a->s[j]; a->s[j] = t;
    int64_t u = a->inds[i]; a->inds[i] = a->inds[j]; a->inds[j] = u;
}

/* floats.Argsort: inds = the permutation; v is left as it was */
void orc_go_argsort(const double* v, int64_t n, int64_t* inds) {
    double* s = (double*)malloc((size_t)(n > 0 ? n : 1) * sizeof(double));
    memcpy(s, v, (size_t)n * sizeof(double));
    for (int64_t i = 0; i < n; i++) inds[i] = i;
    Argsort a = {s, inds};
    GoSort d = {as_less, as_swap, &a};
    go_sort(&d, n);
    free(s);
}

/* ------------------------------------------------------------------ GeneralDebiaser.Debias, literally */
typedef struct { double q[9]; int head, count; } MovingMedian;

static void mm_push(MovingMedian* m, double v) {
    if (m->count == 9) { m->q[m->head] = v; m->head = (m->head + 1) % 9; }
    else m->q[(m->head + m->count++) % 9] = v;
}

static double mm_median(const MovingMedian* m) {
    double w[9];
    int c = m->count;
    for (int i = 0; i < c; i++) w[i] = m->q[(m->head + i) % 9];
    for (int i = 1; i < c; i++)
        for (int j = i; j > 0 && w[j] < w[j - 1]; j--) { double t = w[j]; w[j] = w[j - 1]; w[j - 1] = t; }
    if (c % 2 == 0) return (w[c / 2 - 1] + w[c / 2]) / 2;
    return w[c / 2];
}

/* col: one sample's values in GC order, divided in place.  -1 where the reference panics (n < 5). */
int orc_dcnv_debias(double* col, int64_t n) {
    if (n < 5) return -1;
    MovingMedian mm = {{0}, 0, 0};
    const int64_t mid = (9 - 1) / 2 + 1;
    for (int64_t i = 0; i < mid; i++) mm_push(&mm, col[i]);
    for (int64_t i = 0; i < mid; i++) col[i] /= fmax(mm_median(&mm), 1);
    int64_t i;
    for (i = mid; i < n - mid; i++) {
        mm_push(&mm, col[i + mid]);
        col[i] /= fmax(mm_median(&mm), 1);
    }
    for (; i < n; i++) col[i] /= fmax(mm_median(&mm), 1);
    return 0;
}

static int cmp_f64(const void* a, const void* b) {
    double x = *(const double*)a, y = *(const double*)b;
    return x < y ? -1 : (x > y ? 1 : 0);
}

/* SampleMedians for one column: -1 where the reference panics (all zero) */
int orc_dcnv_sample_median(const double* col, int64_t n, double* med) {
    double* s = (double*)malloc((size_t)(n > 0 ? n : 1) * sizeof(double));
    memcpy(s, col, (size_t)n * sizeof(double));
    qsort(s, (size_t)n, sizeof(double), cmp_f64);
    int64_t k = 0;
    while (k < n && s[k] == 0) k++;
    int rc = -1;
    if (k < n) { *med = s[k + (int64_t)(0.65 * (double)(n - k))]; rc = 0; }
    free(s);
    return rc;
}

/* Sort + Debias + Unsort + NormalizeBySampleMedian on the n x S row-major matrix x (rows in position order), in place.
 * Returns 0, -1 (n < 5) or -2 - c (sample c is all zero). */
int orc_dcnv_matrix(double* x, int64_t n, int64_t S, const double* gc, int64_t* inds_out, double* medians) {
    if (n < 5) return -1;
    int64_t* inds = (int64_t*)malloc((size_t)n * sizeof(int64_t));
    double* col = (double*)malloc((size_t)n * sizeof(double));
    orc_go_argsort(gc, n, inds);
    if (inds_out) memcpy(inds_out, inds, (size_t)n * sizeof(int64_t));
    int rc = 0;
    for (int64_t c = 0; c < S && rc == 0; c++) {
        for (int64_t i = 0; i < n; i++) col[i] = x[inds[i] * S + c];          /* Sort: tmp row ai = mat row inds[ai] */
        orc_dcnv_debias(col, n);
        for (int64_t i = 0; i < n; i++) x[inds[i] * S + c] = col[i];          /* Unsort */
    }
    for (int64_t c = 0; c < S && rc == 0; c++) {
        for (int64_t i = 0; i < n; i++) col[i] = x[i * S + c];
        if (orc_dcnv_sample_median(col, n, &medians[c]) != 0) { rc = -2 - (int)c; break; }
    }
    if (rc == 0)
        for (int64_t i = 0; i < n; i++)
            for (int64_t c = 0; c < S; c++) x[i * S + c] /= medians[c];
    free(inds); free(col);
    return rc;
}

/* fmt.Sprintf("%.2f", v): C's digits, Go's spellings of the non-finite values */
static int go_f2(double v, char* out, int cap) {
    if (isnan(v)) return snprintf(out, (size_t)cap, "NaN");
    if (isinf(v)) return snprintf(out, (size_t)cap, v > 0 ? "+Inf" : "-Inf");
    return snprintf(out, (size_t)cap, "%.2f", v);
}

/* the rows of depth.bed after the header: label \t start \t end (\t %.2f)*S \n.  *out is malloc'ed (orc_free). */
typedef struct { char* p; size_t len, cap; } Text;

static void text_add(Text* t, const char* s, int n) {
    if (t->len + (size_t)n + 1 > t->cap) {
        while (t->len + (size_t)n + 1 > t->cap) t->cap = t->cap ? 2 * t->cap : 4096;
        t->p = (char*)realloc(t->p, t->cap);
    }
    memcpy(t->p + t->len, s, (size_t)n);
    t->len += (size_t)n;
}

int orc_dcnv_rows(const char* label, const int64_t* starts, const int64_t* ends, const double* x, int64_t n, int64_t S, char** out, int64_t* out_len) {
    Text t = {NULL, 0, 0};
    char tok[400];
    text_add(&t, "", 0);
    for (int64_t i = 0; i < n; i++) {
        text_add(&t, tok, snprintf(tok, sizeof tok, "%s\t%lld\t%lld", label, (long long)starts[i], (long long)ends[i]));
        for (int64_t c = 0; c < S; c++) {
            tok[0] = '\t';
            text_add(&t, tok, 1 + go_f2(x[i * S + c], tok + 1, (int)sizeof tok - 1));
        }
        text_add(&t, "\n", 1);
    }
    *out = t.p;
    *out_len = (int64_t)t.len;
    return 0;
}

/* how many 16-byte "%.2f" tokens differ from snprintf (an empty token must be a value whose text is longer than 16) */
int64_t orc_f2_mismatches(const double* v, int64_t n, const uint8_t* tokens, int64_t* first_bad) {
    int64_t bad = 0;
    char want[400];
    *first_bad = -1;
    for (int64_t i = 0; i < n; i++) {
        int k = go_f2(v[i], want, sizeof want);
        const uint8_t* t = tokens + i * 16;
        int ok;
        if (t[0] == 0) ok = k > 16;
        else ok = k <= 16 && memcmp(t, want, (size_t)k) == 0 && (k == 16 || t[k] == 0);
        if (!ok) { if (*first_bad < 0) *first_bad = i; bad++; }
    }
    return bad;
}
