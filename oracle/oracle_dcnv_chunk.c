/* oracle_dcnv_chunk.c — TEST INFRASTRUCTURE: a plain C restatement of ChunkDebiaser.Debias (dcnv/debiaser/debiaser.go:
 * 125-170) for `goleft dcnv --chunk W`, with the driver DESIGN §1.9 defines: Sort (the rows AND their GC values in GC order),
 * Debias, Unsort, then NormalizeBySampleMedian as oracle_dcnv.c has it.  Written to be obviously literal, not fast: the
 * chunk cuts are Go's loop over the sorted values, and each (sample, chunk) median is a full qsort of a copy of the chunk,
 * the leading-zero loop and sorted[(len - k) / 2]. */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

void orc_go_argsort(const double* v, int64_t n, int64_t* inds);                  /* oracle_dcnv.c */
int orc_dcnv_sample_median(const double* col, int64_t n, double* med);            /* oracle_dcnv.c */

static int cmp_f64(const void* a, const void* b) {
    double x = *(const double*)a, y = *(const double*)b;
    return x < y ? -1 : (x > y ? 1 : 0);
}

/* debiaser.go:133-141 over vals (the GC values in sorted order): slices[0 .. *n_slices) into slices (room for n + 1) */
void orc_dcnv_chunk_slices(const double* vals, int64_t n, double w, int64_t* slices, int64_t* n_slices) {
    int64_t m = 1;
    slices[0] = 0;
    double v0 = vals[0];
    for (int64_t i = 0; i < n; i++) {
        if (vals[i] - v0 > w) {
            v0 = vals[i];
            slices[m++] = i;
        }
    }
    slices[m++] = n;
    *n_slices = m;
}

/* ChunkDebiaser.Debias on the n x S row-major matrix x, rows in sorted order, in place; slices[0 .. n_slices) as above */
void orc_dcnv_chunk_debias(double* x, int64_t n, int64_t S, const int64_t* slices, int64_t n_slices) {
    double* col = (double*)malloc((size_t)(n > 0 ? n : 1) * sizeof(double));
    double* sub = (double*)malloc((size_t)(n > 0 ? n : 1) * sizeof(double));
    for (int64_t c = 0; c < S; c++) {
        for (int64_t i = 0; i < n; i++) col[i] = x[i * S + c];
        for (int64_t s = 1; s < n_slices; s++) {
            int64_t si = slices[s - 1], ei = slices[s];
            memcpy(sub, col + si, (size_t)(ei - si) * sizeof(double));
            qsort(sub, (size_t)(ei - si), sizeof(double), cmp_f64);
            int64_t k = 0;
            for (; k < ei - si && sub[k] == 0; k++) {
            }
            double median = sub[(ei - si - k) / 2];
            if (median > 0)
                for (int64_t j = si; j < ei; j++) col[j] /= median;
        }
        for (int64_t i = 0; i < n; i++) x[i * S + c] = col[i];
    }
    free(col);
    free(sub);
}

/* Sort + ChunkDebiaser.Debias + Unsort + NormalizeBySampleMedian on the n x S row-major matrix x (rows in position order),
 * in place.  inds_out (n) and slices_out (room for n + 1; *n_slices) may be NULL.  Returns 0, -1 (n < 1) or -2 - c (sample
 * c is all zero). */
int orc_dcnv_chunk_matrix(double* x, int64_t n, int64_t S, const double* gc, double w, int64_t* inds_out, int64_t* slices_out,
                          int64_t* n_slices_out, double* medians) {
    if (n < 1) return -1;
    int64_t* inds = (int64_t*)malloc((size_t)n * sizeof(int64_t));
    int64_t* slices = (int64_t*)malloc((size_t)(n + 1) * sizeof(int64_t));
    double* vals = (double*)malloc((size_t)n * sizeof(double));
    double* tmp = (double*)malloc((size_t)n * (size_t)S * sizeof(double));
    double* col = (double*)malloc((size_t)n * sizeof(double));
    orc_go_argsort(gc, n, inds);
    for (int64_t i = 0; i < n; i++) vals[i] = gc[inds[i]];
    for (int64_t i = 0; i < n; i++) memcpy(tmp + i * S, x + inds[i] * S, (size_t)S * sizeof(double));     /* Sort */
    int64_t n_slices;
    orc_dcnv_chunk_slices(vals, n, w, slices, &n_slices);
    orc_dcnv_chunk_debias(tmp, n, S, slices, n_slices);
    for (int64_t i = 0; i < n; i++) memcpy(x + inds[i] * S, tmp + i * S, (size_t)S * sizeof(double));     /* Unsort */
    if (inds_out) memcpy(inds_out, inds, (size_t)n * sizeof(int64_t));
    if (slices_out) memcpy(slices_out, slices, (size_t)n_slices * sizeof(int64_t));
    if (n_slices_out) *n_slices_out = n_slices;
    int rc = 0;
    for (int64_t c = 0; c < S; c++) {
        for (int64_t i = 0; i < n; i++) col[i] = x[i * S + c];
        if (orc_dcnv_sample_median(col, n, &medians[c]) != 0) { rc = -2 - (int)c; break; }
    }
    if (rc == 0)
        for (int64_t i = 0; i < n; i++)
            for (int64_t c = 0; c < S; c++) x[i * S + c] /= medians[c];
    free(inds); free(slices); free(vals); free(tmp); free(col);
    return rc;
}
