// dcnv.cpp — the host-only parts of `goleft dcnv` (dcnv/dcnv.go, dcnv/debiaser/debiaser.go):
//
//   gl_go_argsort_f64 : the permutation gonum's floats.Argsort leaves in inds (GeneralDebiaser.Sort, debiaser.go:56-76).
//                       floats.Argsort (gonum v0.14.0) is sort.Sort over an adaptor whose Less compares the values and whose
//                       Swap moves a value and its index together.  sort.Sort is unstable, and rows of one window size share
//                       a few hundred GC values, so the order inside a tie decides which depths share a median window: the
//                       permutation has to be Go's own.  go.mod says go 1.21.5, whose sort.Sort is pattern-defeating
//                       quicksort, restated in go_sort.h.  PARITY UNPINNED until the reference goldens exist.
//   gl_dcnv_chunk_slices : ChunkDebiaser's chunks (debiaser.go:133-141) over the GC-sorted rows, as CSR offsets for
//                       gl_dcnv_normalize_chunked (`dcnv --chunk W`).  A sequential scan: each cut depends on the last.
//   gl_format_f2_host : the host mirror of fmt_f2_kernel (host/f2_token.h).
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../../include/goleft_b200.h"
#include "f2_token.h"
#include "go_sort.h"

namespace {

// the sort.Interface of floats.Argsort's adaptor, over plain arrays
struct ArgsortData {
    double* v;
    int64_t* ind;
    bool less(int64_t i, int64_t j) const { return v[i] < v[j]; }
    void swap(int64_t i, int64_t j) {
        const double t = v[i]; v[i] = v[j]; v[j] = t;
        const int64_t u = ind[i]; ind[i] = ind[j]; ind[j] = u;
    }
};

}  // namespace

extern "C" {

int gl_go_argsort_f64(const double* v, int64_t n, int64_t* inds) {
    if (n < 0 || (n > 0 && (!v || !inds))) return GL_EINVAL;
    std::vector<double> w(v, v + n);                           // floats.Argsort sorts its argument too; the caller's stays
    for (int64_t i = 0; i < n; i++) inds[i] = i;
    if (n <= 1) return GL_OK;
    ArgsortData d{w.data(), inds};
    glsort::go_sort(d, n);
    return GL_OK;
}

int gl_dcnv_chunk_slices(const double* gc_sorted, int64_t n, double w, int64_t* ptr, int64_t cap, int64_t* n_chunks) {
    if (!gc_sorted || n < 1 || !n_chunks || !(w > 0) || w == INFINITY || cap < 0 || (cap > 0 && !ptr)) return GL_EINVAL;
    int64_t nc = 0;
    double v0 = gc_sorted[0];
    for (int64_t i = 0; i < n; i++) {                           // debiaser.go:133-141
        if (gc_sorted[i] - v0 > w) {
            v0 = gc_sorted[i];
            if (ptr && nc + 1 < cap) ptr[nc + 1] = i;
            nc++;
        }
    }
    *n_chunks = nc + 1;
    if (!ptr) return GL_OK;
    if (cap < nc + 2) return GL_ERANGE;
    ptr[0] = 0;
    ptr[nc + 1] = n;
    return GL_OK;
}

int gl_format_f2_host(const double* vals, int64_t n, uint8_t* tokens) {
    if (n < 0 || (n > 0 && (!vals || !tokens))) return GL_EINVAL;
    for (int64_t i = 0; i < n; i++) glf2::token(vals[i], tokens + i * glf2::kTok);
    return GL_OK;
}

}  // extern "C"
