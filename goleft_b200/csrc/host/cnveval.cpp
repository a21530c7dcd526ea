// cnveval.cpp — the host-only part of `goleft cnveval` (cnveval/cnveval.go):
//
//   gl_cnveval_order : the permutation Go 1.21's sort.Slice leaves when Evaluate sorts one sample's calls, given in file
//                      order, by (chrom, start) (cnveval.go:199-201).  sort.Slice is unstable and calls often share a start,
//                      and the order inside such a tie decides which call a truth counts and where an FP run stops
//                      (DESIGN §1.12), so the permutation has to be Go's own: go_sort.h.  PARITY UNPINNED until the
//                      reference goldens exist.
#include <stdint.h>
#include <vector>

#include "../../../include/goleft_b200.h"
#include "go_sort.h"

namespace {

// sort.Slice's lessSwap over (chrom rank, start) keys; the swap carries the file index along
struct CallKeys {
    int32_t* chrom;
    int64_t* start;
    int64_t* perm;
    bool less(int64_t i, int64_t j) const { return chrom[i] < chrom[j] || (chrom[i] == chrom[j] && start[i] < start[j]); }
    void swap(int64_t i, int64_t j) {
        const int32_t c = chrom[i]; chrom[i] = chrom[j]; chrom[j] = c;
        const int64_t s = start[i]; start[i] = start[j]; start[j] = s;
        const int64_t p = perm[i]; perm[i] = perm[j]; perm[j] = p;
    }
};

}  // namespace

extern "C" {

int gl_cnveval_order(const int32_t* chrom, const int64_t* start, int64_t n, int64_t* perm) {
    if (n < 0 || (n > 0 && (!chrom || !start || !perm))) return GL_EINVAL;
    std::vector<int32_t> c(chrom, chrom + n);
    std::vector<int64_t> s(start, start + n);
    for (int64_t i = 0; i < n; i++) perm[i] = i;
    CallKeys d{c.data(), s.data(), perm};
    glsort::go_sort(d, n);
    return GL_OK;
}

}  // extern "C"
