// go_sort.h — Go 1.21's pattern-defeating quicksort (src/sort/zsortinterface.go, zsortfunc.go), restated from Go's
// published source over any D with `bool less(int64_t, int64_t)` and `void swap(int64_t, int64_t)`.  sort.Sort and
// sort.Slice run this same algorithm: insertion sort up to 12 elements, median-of-three / Tukey ninther pivots with the
// swap-count hint, breakPatterns with the length-seeded xorshift, partialInsertionSort, partitionEqual, and heapsort once
// bits.Len(n) bad partitions have been made.  It is unstable, and callers that restate a reference's tie order depend on it
// step for step:
//   gl_go_argsort_f64 (dcnv.cpp)   floats.Argsort = sort.Sort over (value, index)
//   gl_cnveval_order (cnveval.cpp) cnveval's sort.Slice of one sample's calls by (chrom, start)
#pragma once
#include <stdint.h>

namespace glsort {

enum SortedHint { kUnknownHint, kIncreasingHint, kDecreasingHint };

inline int bits_len(uint64_t x) { int n = 0; while (x) { n++; x >>= 1; } return n; }

template <class D> void insertion_sort(D& d, int64_t a, int64_t b) {
    for (int64_t i = a + 1; i < b; i++)
        for (int64_t j = i; j > a && d.less(j, j - 1); j--) d.swap(j, j - 1);
}

template <class D> void sift_down(D& d, int64_t lo, int64_t hi, int64_t first) {
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

template <class D> void heap_sort(D& d, int64_t a, int64_t b) {
    const int64_t first = a, lo = 0, hi = b - a;
    for (int64_t i = (hi - 1) / 2; i >= 0; i--) sift_down(d, i, hi, first);
    for (int64_t i = hi - 1; i >= 0; i--) { d.swap(first, first + i); sift_down(d, lo, i, first); }
}

// data[newpivot] = p; data[i] < p left of it, data[j] >= p right of it
template <class D> int64_t partition(D& d, int64_t a, int64_t b, int64_t pivot, bool& already) {
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
template <class D> int64_t partition_equal(D& d, int64_t a, int64_t b, int64_t pivot) {
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

template <class D> bool partial_insertion_sort(D& d, int64_t a, int64_t b) {
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

template <class D> void break_patterns(D& d, int64_t a, int64_t b) {
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

template <class D> void order2(D& d, int64_t& a, int64_t& b, int& swaps) {
    if (d.less(b, a)) { swaps++; const int64_t t = a; a = b; b = t; }
}

template <class D> int64_t median3(D& d, int64_t a, int64_t b, int64_t c, int& swaps) {
    order2(d, a, b, swaps);
    order2(d, b, c, swaps);
    order2(d, a, b, swaps);
    return b;
}

template <class D> int64_t choose_pivot(D& d, int64_t a, int64_t b, SortedHint& hint) {
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

template <class D> void reverse_range(D& d, int64_t a, int64_t b) {
    for (int64_t i = a, j = b - 1; i < j; i++, j--) d.swap(i, j);
}

template <class D> void pdqsort(D& d, int64_t a, int64_t b, int limit) {
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

// sort.Sort / sort.Slice over d[0, n)
template <class D> void go_sort(D& d, int64_t n) {
    if (n > 1) pdqsort(d, 0, n, bits_len((uint64_t)n));
}

}  // namespace glsort
