// covstats.h — the tail of BamStats (covstats/covstats.go:57-89,175-218), shared by the device sampler (covstats.cu), the host
// sampler and gl_covstats_tail.  The reference sorts the sampled insert sizes / template lengths / read lengths and reads
// order statistics off the sorted slices.  Here the multiset is a histogram: the k-th smallest value is a search in its
// running count, madFilter's cut is a count, and meanStd's float64 accumulation visits the values in ascending order with
// their multiplicities — the same sequence of additions as over the sorted slice, so the results are bit-identical
// without a sort.
#pragma once
#include <stdint.h>
#include <algorithm>
#include <string>
#include <vector>
#include "../../../include/goleft_b200.h"

int gl_fail(gl_ctx* ctx, int code, const char* fmt, ...);      // gl_ctx.cu

namespace glcs {

constexpr long long kMaxHistRange = 1LL << 22;               // a wider multiset is kept as a sorted array

struct SortedCounts {
    int32_t lo = 0;
    std::vector<uint64_t> cum;                               // cum[i] = how many values are <= lo + i
    std::vector<int32_t> sorted;                             // when the value range is too wide for a histogram
    size_t n = 0;
    // hist[i] = how many values equal lo + i (taken over; it becomes the running count)
    void from_hist(int32_t lo_, std::vector<uint64_t>&& hist) {
        lo = lo_; cum = std::move(hist); sorted.clear();
        for (size_t i = 1; i < cum.size(); i++) cum[i] += cum[i - 1];
        n = cum.empty() ? 0 : (size_t)cum.back();
    }
    void from_values(const int32_t* v, size_t nv) {
        cum.clear(); sorted.assign(v, v + nv); n = nv;
        std::sort(sorted.begin(), sorted.end());
    }
    // the multiset of host values: a histogram counted on the device (gl_bincount_i32) when there is a context and the
    // range allows, the sorted array otherwise
    int build(gl_ctx* ctx, const int32_t* v, size_t nv);
    int32_t kth(size_t k) const {                            // k-th smallest, 0-based
        if (!sorted.empty()) return sorted[k];
        return lo + (int32_t)(std::upper_bound(cum.begin(), cum.end(), (uint64_t)k) - cum.begin());
    }
    size_t count_le(long long v) const {
        if (!sorted.empty()) return (size_t)(std::upper_bound(sorted.begin(), sorted.end(), v, [](long long a, int32_t b) { return a < (long long)b; }) - sorted.begin());
        if (v < lo) return 0;
        const long long i = v - lo;
        return (size_t)(i >= (long long)cum.size() ? cum.back() : cum[(size_t)i]);
    }
    template <class F> void for_first(size_t m, F f) const { // the m smallest values, ascending, with multiplicity
        if (!sorted.empty()) { for (size_t i = 0; i < m; i++) f(sorted[i]); return; }
        size_t done = 0;
        for (size_t i = 0; i < cum.size() && done < m; i++) {
            const size_t c = std::min<size_t>((size_t)(cum[i] - (i ? cum[i - 1] : 0)), m - done);
            for (size_t k = 0; k < c; k++) f(lo + (int32_t)i);
            done += c;
        }
    }
};

void mean_std(const SortedCounts& a, size_t n, double& mean, double& sd);     // covstats.go:78-89 over the n smallest
size_t mad_filter(const SortedCounts& a, int nmads);                          // covstats.go:57-76: how many values are kept

// covstats.go:175-218 from the three multisets and the counters already in *io (n_unmapped, k, n_bad, n_dup, n_proper):
// fills every Stats field, n_read_len, n_insert and h_len, and H.  GL_EINVAL: 1 or 2 inserts (madFilter indexes past
// the slice); GL_ERANGE: H's length is negative (Go's makeslice panics).
int tail(gl_ctx* ctx, const SortedCounts& rl, const SortedCounts& ins, const SortedCounts& tm, gl_covstats* io, std::vector<double>& H);
// copies H out under the two-call convention: io->h_len is set either way, GL_ERANGE when h_cap is too small
int put_hist(gl_ctx* ctx, const std::vector<double>& H, double* out, int64_t h_cap);

}  // namespace glcs
