// dcnv.cpp — the host-only parts of `goleft dcnv` (dcnv/dcnv.go, dcnv/debiaser/debiaser.go):
//
//   gl_go_argsort_f64 : the permutation gonum's floats.Argsort leaves in inds (GeneralDebiaser.Sort, debiaser.go:56-76).
//                       floats.Argsort (gonum v0.14.0) is sort.Sort over an adaptor whose Less compares the values and whose
//                       Swap moves a value and its index together.  sort.Sort is unstable, and rows of one window size share
//                       a few hundred GC values, so the order inside a tie decides which depths share a median window: the
//                       permutation has to be Go's own.  go.mod says go 1.21.5, whose sort.Sort is pattern-defeating
//                       quicksort (src/sort/zsortinterface.go, sort.go).  It is restated here from Go's published source:
//                       insertion sort up to 12 elements, median-of-three / Tukey ninther pivots with the swap-count hint,
//                       breakPatterns with the length-seeded xorshift, partialInsertionSort, partitionEqual, and heapsort
//                       once bits.Len(n) bad partitions have been made.  PARITY UNPINNED until the reference goldens exist.
//   gl_format_f2_host : the host mirror of fmt_f2_kernel (host/f2_token.h).
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../../include/goleft_b200.h"
#include "f2_token.h"

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

enum SortedHint { kUnknownHint, kIncreasingHint, kDecreasingHint };

int bits_len(uint64_t x) { int n = 0; while (x) { n++; x >>= 1; } return n; }

void insertion_sort(ArgsortData& d, int64_t a, int64_t b) {
    for (int64_t i = a + 1; i < b; i++)
        for (int64_t j = i; j > a && d.less(j, j - 1); j--) d.swap(j, j - 1);
}

void sift_down(ArgsortData& d, int64_t lo, int64_t hi, int64_t first) {
    int64_t root = lo;
    for (;;) {
        int64_t child = 2 * root + 1;
        if (child >= hi) return;
        if (child + 1 < hi && d.less(first + child, first + child + 1)) child++;
        if (!d.less(first + root, first + child)) return;
        d.swap(first + root, first + child);
        root = child;
    }
}

void heap_sort(ArgsortData& d, int64_t a, int64_t b) {
    const int64_t first = a, lo = 0, hi = b - a;
    for (int64_t i = (hi - 1) / 2; i >= 0; i--) sift_down(d, i, hi, first);
    for (int64_t i = hi - 1; i >= 0; i--) { d.swap(first, first + i); sift_down(d, lo, i, first); }
}

// data[newpivot] = p; data[i] < p left of it, data[j] >= p right of it
int64_t partition(ArgsortData& d, int64_t a, int64_t b, int64_t pivot, bool& already) {
    d.swap(a, pivot);
    int64_t i = a + 1, j = b - 1;
    while (i <= j && d.less(i, a)) i++;
    while (i <= j && !d.less(j, a)) j--;
    if (i > j) { d.swap(j, a); already = true; return j; }
    d.swap(i, j); i++; j--;
    for (;;) {
        while (i <= j && d.less(i, a)) i++;
        while (i <= j && !d.less(j, a)) j--;
        if (i > j) break;
        d.swap(i, j); i++; j--;
    }
    d.swap(j, a);
    already = false;
    return j;
}

// data[a:b] holds nothing smaller than data[pivot]: the elements equal to it first, then the greater ones
int64_t partition_equal(ArgsortData& d, int64_t a, int64_t b, int64_t pivot) {
    d.swap(a, pivot);
    int64_t i = a + 1, j = b - 1;
    for (;;) {
        while (i <= j && !d.less(a, i)) i++;
        while (i <= j && d.less(a, j)) j--;
        if (i > j) break;
        d.swap(i, j); i++; j--;
    }
    return i;
}

bool partial_insertion_sort(ArgsortData& d, int64_t a, int64_t b) {
    const int kMaxSteps = 5, kShortestShifting = 50;
    int64_t i = a + 1;
    for (int step = 0; step < kMaxSteps; step++) {
        while (i < b && !d.less(i, i - 1)) i++;
        if (i == b) return true;
        if (b - a < kShortestShifting) return false;
        d.swap(i, i - 1);
        if (i - a >= 2)
            for (int64_t j = i - 1; j >= 1; j--) { if (!d.less(j, j - 1)) break; d.swap(j, j - 1); }
        if (b - i >= 2)
            for (int64_t j = i + 1; j < b; j++) { if (!d.less(j, j - 1)) break; d.swap(j, j - 1); }
    }
    return false;
}

void break_patterns(ArgsortData& d, int64_t a, int64_t b) {
    const int64_t length = b - a;
    if (length < 8) return;
    uint64_t random = (uint64_t)length;                      // xorshift(length)
    const uint64_t modulus = uint64_t(1) << bits_len((uint64_t)length);
    const int64_t idx = a + (length / 4) * 2 - 1;
    for (int i = 0; i < 3; i++) {
        random ^= random << 13; random ^= random >> 7; random ^= random << 17;
        int64_t other = (int64_t)(random & (modulus - 1));
        if (other >= length) other -= length;
        d.swap(idx - 1 + i, a + other);
    }
}

void order2(ArgsortData& d, int64_t& a, int64_t& b, int& swaps) {
    if (d.less(b, a)) { swaps++; const int64_t t = a; a = b; b = t; }
}

int64_t median3(ArgsortData& d, int64_t a, int64_t b, int64_t c, int& swaps) {
    order2(d, a, b, swaps);
    order2(d, b, c, swaps);
    order2(d, a, b, swaps);
    return b;
}

int64_t choose_pivot(ArgsortData& d, int64_t a, int64_t b, SortedHint& hint) {
    const int64_t kShortestNinther = 50;
    const int kMaxSwaps = 4 * 3;
    const int64_t l = b - a;
    int swaps = 0;
    int64_t i = a + l / 4 * 1, j = a + l / 4 * 2, k = a + l / 4 * 3;
    if (l >= 8) {
        if (l >= kShortestNinther) {
            i = median3(d, i - 1, i, i + 1, swaps);
            j = median3(d, j - 1, j, j + 1, swaps);
            k = median3(d, k - 1, k, k + 1, swaps);
        }
        j = median3(d, i, j, k, swaps);
    }
    hint = swaps == 0 ? kIncreasingHint : (swaps == kMaxSwaps ? kDecreasingHint : kUnknownHint);
    return j;
}

void reverse_range(ArgsortData& d, int64_t a, int64_t b) {
    for (int64_t i = a, j = b - 1; i < j; i++, j--) d.swap(i, j);
}

void pdqsort(ArgsortData& d, int64_t a, int64_t b, int limit) {
    const int64_t kMaxInsertion = 12;
    bool was_balanced = true, was_partitioned = true;
    for (;;) {
        const int64_t length = b - a;
        if (length <= kMaxInsertion) { insertion_sort(d, a, b); return; }
        if (limit == 0) { heap_sort(d, a, b); return; }
        if (!was_balanced) { break_patterns(d, a, b); limit--; }
        SortedHint hint;
        int64_t pivot = choose_pivot(d, a, b, hint);
        if (hint == kDecreasingHint) {
            reverse_range(d, a, b);
            pivot = (b - 1) - (pivot - a);
            hint = kIncreasingHint;
        }
        if (was_balanced && was_partitioned && hint == kIncreasingHint && partial_insertion_sort(d, a, b)) return;
        if (a > 0 && !d.less(a - 1, pivot)) {                  // many duplicates: split off the run equal to the pivot
            a = partition_equal(d, a, b, pivot);
            continue;
        }
        bool already = false;
        const int64_t mid = partition(d, a, b, pivot, already);
        was_partitioned = already;
        const int64_t left = mid - a, right = b - mid, balance = length / 8;
        if (left < right) {
            was_balanced = left >= balance;
            pdqsort(d, a, mid, limit);
            a = mid + 1;
        } else {
            was_balanced = right >= balance;
            pdqsort(d, mid + 1, b, limit);
            b = mid;
        }
    }
}

}  // namespace

extern "C" {

int gl_go_argsort_f64(const double* v, int64_t n, int64_t* inds) {
    if (n < 0 || (n > 0 && (!v || !inds))) return GL_EINVAL;
    std::vector<double> w(v, v + n);                           // floats.Argsort sorts its argument too; the caller's stays
    for (int64_t i = 0; i < n; i++) inds[i] = i;
    if (n <= 1) return GL_OK;
    ArgsortData d{w.data(), inds};
    pdqsort(d, 0, n, bits_len((uint64_t)n));
    return GL_OK;
}

int gl_format_f2_host(const double* vals, int64_t n, uint8_t* tokens) {
    if (n < 0 || (n > 0 && (!vals || !tokens))) return GL_EINVAL;
    for (int64_t i = 0; i < n; i++) glf2::token(vals[i], tokens + i * glf2::kTok);
    return GL_OK;
}

}  // extern "C"
