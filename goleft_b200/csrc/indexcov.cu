// indexcov.cu — `goleft indexcov` arithmetic on sm_90a, plus the small covstats / depthwed kernels.
//
//   I1  ic_sizes_batch_kernel  BAI linear-index virtual offsets -> per-tile sizes, one warp per (sample, reference)
//                                                                                      (indexcov/types.go:45-82)
//   I2+I3 ic_cohort2_kernel ONE kernel, a CTA per sample: the 98th percentile and the capped weighted median, exactly, from
//                           the brackets a sorted strided sample gives and one pass over the tiles (small samples: a full
//                           sort; brackets that fail: a range-adaptive histogram select), then normalised depth
//                                                                                      (indexcov.go:83-151)
//   I4+I5 ic_counts_kernel  per (sample, chromosome) segment: 70-slot histogram + in/out/hi/low counters
//                                                                            (indexcov.go:170-177,1050-1078)
//   I6  fmt_g3_kernel       float32 -> the bytes of "%.3g", exact (integer arithmetic), 10-byte tokens
//                                                                              (indexcov.go:678-680,1038-1048)
//   I7  ic_xnorm_kernel     cross-sample normalisation, sequential in tile j, parallel over samples, with the
//                           float64 mean reproduced bit-exactly (order-free when provably exact, else ordered)
//   V2  bincount_kernel     shared-memory privatised histogram (covstats/covstats.go:202-217)
//   W1  depthwed_kernel     int(0.5+mean), group-sum, sample-major -> row-major transpose (depthwed.go:93-157)
//
// Floating point follows Go on amd64: no fused multiply-add (the library is compiled with --fmad=false and
// the hot expressions use the explicit _rn intrinsics), float64 division rounded to float32 exactly once.
#include "gl_common.cuh"
#include <string.h>

namespace {

constexpr unsigned kFull = 0xffffffffu;

// ------------------------------------------------------------------------------------------------ I2 + I3
// Selection without a sort: ic_cohort2_kernel's exact fallback.  Both selects of Index.init are "smallest value v with
// F(v) > target", where F(v) = sum over x <= v of w(x):  w = 1 gives the k-th smallest (target = k), w = min(x, cap)
// gives the capped weighted median (target = total/2).  The answer is bracketed by [lo,hi]; each level histograms the candidates
// into kSelBins equal-width bins over the CURRENT range (not over radix digits: tile sizes of one sample share
// their leading bytes, a digit histogram would put every shared-memory atomic on one bin), picks the bin where
// the running weight crosses the target, and shrinks [lo,hi] to the min/max of that bin's members.  The width
// drops by >= kSelBins per level, so 64-bit values need at most 7 levels; real data takes 3.
constexpr int kSelBins = 1024;

struct SelSmem {
    unsigned long long w[kSelBins];
    long long red_lo[32], red_hi[32];
    long long bcast[3];
};

__device__ __forceinline__ int sel_bin(long long x, long long lo, double scale) {
    const int b = (int)((double)(unsigned long long)(x - lo) * scale);      // monotone in x
    return b < kSelBins - 1 ? b : kSelBins - 1;
}

// block-wide min / max of the values in [flo,fhi] whose bin at (lo,scale) equals `bin` (bin < 0: every value in range)
__device__ void block_minmax(const long long* __restrict__ v, long long n, long long flo, long long fhi, long long lo, double scale,
                             int bin, SelSmem& sm, long long& out_lo, long long& out_hi) {
    long long mn = 0x7fffffffffffffffll, mx = -0x7fffffffffffffffll - 1;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const long long x = v[i];
        if (x >= flo && x <= fhi && (bin < 0 || sel_bin(x, lo, scale) == bin)) { mn = min(mn, x); mx = max(mx, x); }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { mn = min(mn, __shfl_xor_sync(kFull, mn, o)); mx = max(mx, __shfl_xor_sync(kFull, mx, o)); }
    if ((threadIdx.x & 31) == 0) { sm.red_lo[threadIdx.x >> 5] = mn; sm.red_hi[threadIdx.x >> 5] = mx; }
    __syncthreads();
    mn = 0x7fffffffffffffffll; mx = -0x7fffffffffffffffll - 1;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) { mn = min(mn, sm.red_lo[w]); mx = max(mx, sm.red_hi[w]); }
    __syncthreads();
    out_lo = mn; out_hi = mx;
}

template <bool kWeighted>
__device__ long long block_select(const long long* __restrict__ v, long long n, long long cap, long long target, long long lo,
                                  long long hi, SelSmem& sm) {
    long long below = 0;                                   // F just below lo
    while (lo < hi) {
        const double scale = (double)kSelBins / ((double)(unsigned long long)(hi - lo) + 1.0);
        for (int i = threadIdx.x; i < kSelBins; i += blockDim.x) sm.w[i] = 0;
        __syncthreads();
        for (long long i = threadIdx.x; i < n; i += blockDim.x) {
            const long long x = v[i];
            if (x >= lo && x <= hi) {
                const unsigned long long w = kWeighted ? (unsigned long long)min(x, cap) : 1ull;
                if (w) atomicAdd(&sm.w[sel_bin(x, lo, scale)], w);
            }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long long acc = below;
            int b = 0;
            for (; b < kSelBins - 1; b++) {
                if (acc + (long long)sm.w[b] > target) break;
                acc += (long long)sm.w[b];
            }
            sm.bcast[0] = b;
            sm.bcast[1] = acc;
        }
        __syncthreads();
        const int bin = (int)sm.bcast[0];
        below = sm.bcast[1];
        __syncthreads();
        long long nlo, nhi;
        block_minmax(v, n, lo, hi, lo, scale, bin, sm, nlo, nhi);
        if (nlo > nhi) return lo;                          // cannot happen when F(max) > target; keeps the loop finite
        lo = nlo;
        hi = nhi;
    }
    return lo;
}

// ic_cohort2_kernel: the two order statistics of Index.init (indexcov.go:111-124).  The sample's tiles are streamed TWICE
// instead of the ~17 times of the selects above, and no shared-memory histogram (64-bit shared atomics are a CAS loop on
// sm_90) is involved:
//   small samples (n <= 8192): all tiles sorted in shared memory (bitonic), Index.init done literally.
//   large samples: a strided sample of 8192 tiles is sorted in shared memory; it brackets the 98th-percentile element
//     (n98) and the capped weighted median (med) by VALUE:  [lo98, hi98] around sample rank 0.98 K (+-64 ranks, > 5 sigma)
//     and [loM, hiM] around the sample's own capped weighted median (+-136 ranks, 3 sigma).  One pass over the tiles then
//     sums what lies below / between the brackets, counts what lies above, and collects the tiles INSIDE the brackets into
//     two small shared-memory lists (warp-aggregated appends); the lists are sorted and the exact answers read off them:
//       n98   = cand98[k98 - #{s < lo98}],
//       total = sum(s < loM) + sum(candM) + sum(hiM < s < lo98) + sum(min(cand98, n98)) + n98 * #{s > hi98},
//       med   = first candM value whose running sum (from sum(s < loM)) exceeds total/2.
//     Every step is verified (rank inside the list, brackets disjoint, lists not overflowing); on any failure — heavy ties,
//     a pathological order — the sample falls back to the range-adaptive select above, so the result is always exact.
//   A last pass writes float32(float64(size)/med).  Traffic: 2 reads of 8 B + 1 write of 4 B per tile.
constexpr int kC2Threads = 1024;
constexpr int kC2Unroll = 8;                         // 8-byte loads in flight per thread in the streaming passes
constexpr int kC2Sample = 8192;
constexpr int kC2CandM = 8192;
constexpr int kC2Cand98 = 4096;
constexpr long long kI64Max = 0x7fffffffffffffffll;

struct C2Smem {
    long long samp[kC2Sample];
    long long candM[kC2CandM];
    long long cand98[kC2Cand98];
};

// ascending bitonic sort of a[0..n2), n2 a power of two, by the whole block (blockDim.x a multiple of 32).
// A compare-exchange at distance j < 256 pairs two elements of the same 256-element chunk: warp w owns the chunks w, w + W, ...
// and runs all those stages on its own with __syncwarp between them; only the stages with j >= 256 (15 of the 91 for 8192
// elements) are block-wide.  Every stage visits the n2/2 pairs directly (pair p -> i = p with a zero inserted at bit log2 j).
__device__ void block_bitonic(long long* a, int n2) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    auto cex = [&](int i, int j, int k) {
        const int ixj = i | j;
        const bool up = (i & k) == 0;
        const long long x = a[i], y = a[ixj];
        if ((x > y) == up) { a[i] = y; a[ixj] = x; }
    };
    for (int k = 2; k <= n2; k <<= 1) {
        int j = k >> 1;
        for (; j >= 256; j >>= 1) {                          // block-wide stages
            for (int p = threadIdx.x; p < (n2 >> 1); p += blockDim.x) cex(((p & ~(j - 1)) << 1) | (p & (j - 1)), j, k);
            __syncthreads();
        }
        // the remaining stages of this k (j = min(k/2, 128) .. 1) stay inside 256-element chunks
        for (int c = warp; c * 256 < n2; c += W) {
            const int base = c * 256, m = min(256, n2 - base);             // m < 256 only when n2 < 256
            for (int jj = j; jj > 0; jj >>= 1) {
                for (int p = lane; p < (m >> 1); p += 32) cex(base + (((p & ~(jj - 1)) << 1) | (p & (jj - 1))), jj, k);
                __syncwarp();
            }
        }
        __syncthreads();
    }
}

__device__ __forceinline__ int next_pow2(int n) { int p = 1; while (p < n) p <<= 1; return p; }

// block-wide sum of one long long per thread (result to every thread); red has blockDim/32 slots
__device__ long long block_sum(long long v, long long* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    long long t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += red[w];
    __syncthreads();
    return t;
}

// in-place inclusive prefix sum of a[0..m), m <= 8 * blockDim.x
__device__ void block_prefix(long long* a, int m, long long* red) {
    const int per = (m + (int)blockDim.x - 1) / (int)blockDim.x;
    const int b = threadIdx.x * per, e = min(m, b + per);
    long long loc = 0;
    for (int i = b; i < e; i++) loc += a[i];
    long long inc = loc;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long t = __shfl_up_sync(kFull, inc, o); if (lane >= o) inc += t; }
    if (lane == 31) red[warp] = inc;
    __syncthreads();
    long long base = inc - loc;
    for (int w = 0; w < warp; w++) base += red[w];
    __syncthreads();
    for (int i = b; i < e; i++) { base += a[i]; a[i] = base; }
    __syncthreads();
}

__device__ __forceinline__ void warp_append(long long* list, int cap, int* counter, int* overflow, bool take, long long x) {
    const unsigned m = __ballot_sync(kFull, take);
    if (m == 0) return;
    const int lane = threadIdx.x & 31;
    int base = 0;
    if (lane == __ffs(m) - 1) base = atomicAdd(counter, __popc(m));
    base = __shfl_sync(kFull, base, __ffs(m) - 1);
    if (take) {
        const int at = base + __popc(m & ((1u << lane) - 1u));
        if (at < cap) list[at] = x; else *overflow = 1;
    }
}

__global__ void __launch_bounds__(kC2Threads, 1) ic_cohort2_kernel(const long long* __restrict__ sizes, const long long* __restrict__ sample_ptr,
                                                                     int S, double* __restrict__ medians, float* __restrict__ depth_out,
                                                                     unsigned* __restrict__ fallback_count) {
    extern __shared__ __align__(16) unsigned char c2_raw[];
    C2Smem& sm = *reinterpret_cast<C2Smem*>(c2_raw);
    __shared__ long long s_red[kC2Threads / 32];
    __shared__ long long s_b[8];
    __shared__ int s_cnt[4];
    const int tid = threadIdx.x;
    for (int smp = blockIdx.x; smp < S; smp += gridDim.x) {
        const long long a = sample_ptr[smp], n = sample_ptr[smp + 1] - a;
        const long long* v = sizes + a;
        if (n <= 0) { if (tid == 0) medians[smp] = 0.0; continue; }
        const long long k98 = (long long)(0.98 * (double)n);                     // indexcov.go:111
        long long med = 0;
        bool ok = true;
        if (n <= kC2Sample) {
            // ---- everything fits: sort and follow Index.init literally
            const int n2 = next_pow2((int)n);
            for (int i = tid; i < n2; i += kC2Threads) sm.samp[i] = i < n ? v[i] : kI64Max;
            __syncthreads();
            block_bitonic(sm.samp, n2);
            const long long n98 = sm.samp[k98];
            for (int i = tid; i < (int)n; i += kC2Threads) sm.candM[i] = min(sm.samp[i], n98);
            __syncthreads();
            block_prefix(sm.candM, (int)n, s_red);
            const long long total = sm.candM[n - 1];
            // first i with cumsum[i] > total/2 (sort.Search); when none (total == 0) the clamp picks the last element
            int lo = 0, hi = (int)n;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (sm.candM[mid] > total / 2) hi = mid; else lo = mid + 1; }
            med = sm.samp[min(lo, (int)n - 1)];
            __syncthreads();
        } else {
            // ---- sorted sample -> brackets
            for (int i = tid; i < kC2Sample; i += kC2Threads) sm.samp[i] = v[(long long)(((__int128)i * n) / kC2Sample)];
            __syncthreads();
            block_bitonic(sm.samp, kC2Sample);
            const int p98 = (int)(((__int128)k98 * kC2Sample) / n);
            const long long cap_est = sm.samp[p98];
            for (int i = tid; i < kC2Sample; i += kC2Threads) sm.candM[i] = min(sm.samp[i], cap_est);
            __syncthreads();
            block_prefix(sm.candM, kC2Sample, s_red);
            if (tid == 0) {
                const long long tot = sm.candM[kC2Sample - 1];
                int lo = 0, hi = kC2Sample;
                while (lo < hi) { const int mid = (lo + hi) >> 1; if (sm.candM[mid] > tot / 2) hi = mid; else lo = mid + 1; }
                const int pM = min(lo, kC2Sample - 1);
                s_b[0] = sm.samp[max(0, pM - 136)];                                            // loM
                s_b[1] = sm.samp[min(kC2Sample - 1, pM + 136)];                                // hiM
                s_b[2] = sm.samp[max(0, p98 - 64)];                                            // lo98
                s_b[3] = p98 + 64 < kC2Sample ? sm.samp[p98 + 64] : kI64Max;                   // hi98
                s_cnt[0] = s_cnt[1] = s_cnt[2] = 0;
            }
            __syncthreads();
            const long long loM = s_b[0], hiM = s_b[1], lo98 = s_b[2], hi98 = s_b[3];
            ok = hiM < lo98;                                                       // brackets must not touch
            long long sum_lo = 0, sum_mid = 0, cnt_above = 0, vmax = 0;
            if (ok) {
                // kC2Unroll loads per thread are issued before any of them is used: one CTA per SM has only 32 warps, and with one
                // 8-byte load per warp in flight the pass ran at DRAM latency (1 TB/s over the chip), not at bandwidth
                const long long n_round = (n + kC2Unroll * kC2Threads - 1) / (kC2Unroll * kC2Threads) * (kC2Unroll * kC2Threads);
                for (long long base = 0; base < n_round; base += kC2Unroll * kC2Threads) {
                    long long xs[kC2Unroll];
#pragma unroll
                    for (int u = 0; u < kC2Unroll; u++) {
                        const long long i = base + (long long)u * kC2Threads + tid;
                        xs[u] = i < n ? __ldg(v + i) : 0;
                    }
#pragma unroll
                    for (int u = 0; u < kC2Unroll; u++) {
                        const long long x = xs[u];
                        const bool live = base + (long long)u * kC2Threads + tid < n;
                        const bool inM = live && x >= loM && x <= hiM, in98 = live && x >= lo98 && x <= hi98;
                        if (live) {
                            vmax = max(vmax, x);
                            if (x < loM) sum_lo += x;
                            else if (x > hiM && x < lo98) sum_mid += x;
                            else if (x > hi98) cnt_above++;
                        }
                        warp_append(sm.candM, kC2CandM, &s_cnt[0], &s_cnt[2], inM, x);
                        warp_append(sm.cand98, kC2Cand98, &s_cnt[1], &s_cnt[2], in98, x);
                    }
                }
                sum_lo = block_sum(sum_lo, s_red);
                sum_mid = block_sum(sum_mid, s_red);
                cnt_above = block_sum(cnt_above, s_red);
                {                                                                   // block max
                    long long m = vmax;
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(kFull, m, o));
                    if ((tid & 31) == 0) s_red[tid >> 5] = m;
                    __syncthreads();
                    m = 0;
                    for (int w = 0; w < kC2Threads / 32; w++) m = max(m, s_red[w]);
                    __syncthreads();
                    vmax = m;
                }
                ok = s_cnt[2] == 0;
            }
            long long n98 = 0, total = 0;
            if (ok) {
                const int nM = s_cnt[0], n9 = s_cnt[1];
                const long long below98 = n - n9 - cnt_above;                       // #{s < lo98}
                const long long idx = k98 - below98;
                ok = idx >= 0 && idx < n9;
                if (ok) {
                    const int n92 = next_pow2(max(n9, 1));
                    for (int i = n9 + tid; i < n92; i += kC2Threads) sm.cand98[i] = kI64Max;
                    const int nM2 = next_pow2(max(nM, 1));
                    for (int i = nM + tid; i < nM2; i += kC2Threads) sm.candM[i] = kI64Max;
                    __syncthreads();
                    block_bitonic(sm.cand98, n92);
                    block_bitonic(sm.candM, nM2);
                    n98 = sm.cand98[idx];
                    long long part = 0;
                    for (int i = tid; i < n9; i += kC2Threads) part += min(sm.cand98[i], n98);
                    long long partM = 0;
                    for (int i = tid; i < nM; i += kC2Threads) partM += sm.candM[i];
                    part = block_sum(part, s_red);
                    partM = block_sum(partM, s_red);
                    total = sum_lo + partM + sum_mid + part + n98 * cnt_above;
                    if (total == 0) med = vmax;                                     // cumsum never exceeds 0: the clamp picks the largest
                    else {
                        const long long target = total / 2;
                        // running sums of candM on top of sum_lo, in samp[] (the sample is no longer needed)
                        for (int i = tid; i < nM; i += kC2Threads) sm.samp[i] = sm.candM[i];
                        __syncthreads();
                        block_prefix(sm.samp, nM, s_red);
                        if (tid == 0) {
                            int lo = 0, hi = nM;
                            while (lo < hi) { const int mid = (lo + hi) >> 1; if (sum_lo + sm.samp[mid] > target) hi = mid; else lo = mid + 1; }
                            // the answer must be INSIDE the list: below it the running sum is still <= target, and it is reached
                            s_cnt[3] = (sum_lo <= target && lo < nM) ? lo : -1;
                        }
                        __syncthreads();
                        ok = s_cnt[3] >= 0;
                        if (ok) med = sm.candM[s_cnt[3]];
                    }
                }
            }
            __syncthreads();
            if (!ok) {
                // ---- exact fallback: the range-adaptive select (uses the same shared memory)
                SelSmem& sel = *reinterpret_cast<SelSmem*>(c2_raw);
                if (tid == 0 && fallback_count) atomicAdd(fallback_count, 1u);
                long long vmin, vmx;
                block_minmax(v, n, -kI64Max - 1, kI64Max, 0, 0.0, -1, sel, vmin, vmx);
                const long long f98 = block_select<false>(v, n, 0, k98, vmin, vmx, sel);
                long long part = 0;
                for (long long i = tid; i < n; i += kC2Threads) part += min(v[i], f98);
                const long long tot = block_sum(part, s_red);
                med = (tot == 0) ? vmx : block_select<true>(v, n, f98, tot / 2, vmin, vmx, sel);
                __syncthreads();
            }
        }
        const double dm = (double)med;
        if (tid == 0) medians[smp] = dm;
        // depth = float32(float64(o)/median), capped at 50000                    (indexcov.go:129-151)
        if (depth_out) {
            float* out = depth_out + a;
            for (long long base = 0; base < n; base += kC2Unroll * kC2Threads) {
                long long xs[kC2Unroll];
#pragma unroll
                for (int u = 0; u < kC2Unroll; u++) {
                    const long long i = base + (long long)u * kC2Threads + tid;
                    xs[u] = i < n ? __ldg(v + i) : 0;
                }
#pragma unroll
                for (int u = 0; u < kC2Unroll; u++) {
                    const long long i = base + (long long)u * kC2Threads + tid;
                    float d = (med == 0) ? 0.0f : __double2float_rn(__ddiv_rn((double)xs[u], dm));
                    if (d > 50000.0f) d = 50000.0f;
                    if (i < n) out[i] = d;
                }
            }
        }
        __syncthreads();
    }
}

// I1 for a whole cohort in one launch: one warp per (sample, reference) descriptor, sizes = consecutive differences of the
// reference's linear-index virtual offsets (indexcov/types.go:60-78)
__global__ void __launch_bounds__(256) ic_sizes_batch_kernel(const unsigned long long* __restrict__ voff, const long long* __restrict__ d_voff_off,
                                                            const int* __restrict__ d_n_intv, const long long* __restrict__ d_size_off,
                                                            long long n_desc, long long* __restrict__ sizes, int* __restrict__ neg_flag) {
    const long long w = ((long long)blockIdx.x * 256 + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (w >= n_desc) return;
    const long long a = d_voff_off[w], o = d_size_off[w];
    const int n = d_n_intv[w];
    for (int k = lane; k + 1 < n; k += 32) {
        const long long d = (long long)voff[a + k + 1] - (long long)voff[a + k];
        if (d < 0) *neg_flag = 1;
        sizes[o + k] = d;
    }
}

__global__ void __launch_bounds__(256) ic_normalize_kernel(const long long* __restrict__ sizes, long long n, double median,
                                                          float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float d = __double2float_rn(__ddiv_rn((double)sizes[i], median));
    if (d > 50000.0f) d = 50000.0f;
    out[i] = d;
}

// ------------------------------------------------------------------------------------------------ I4 + I5
// one CTA per segment (a sample's tiles on one chromosome)
// seg_len == null: segment seg = [seg_ptr[seg], seg_ptr[seg+1]) (CSR); else [seg_ptr[seg], seg_ptr[seg] + seg_len[seg]) —
// the (sample, chromosome) slices of a cohort's depth array are not contiguous per chromosome
__global__ void __launch_bounds__(256) ic_counts_kernel(const float* __restrict__ depth, const long long* __restrict__ seg_ptr,
                                                       const long long* __restrict__ seg_len,
                                                       const long long* __restrict__ longest, int n_seg,
                                                       int* __restrict__ counts70, long long* __restrict__ bins4) {
    __shared__ int s_cnt[GL_INDEXCOV_SLOTS];
    __shared__ int s_bin[4];
    const int seg = blockIdx.x;
    if (seg >= n_seg) return;
    for (int i = threadIdx.x; i < GL_INDEXCOV_SLOTS; i += blockDim.x) s_cnt[i] = 0;
    if (threadIdx.x < 4) s_bin[threadIdx.x] = 0;
    __syncthreads();
    const long long a = seg_ptr[seg], n = seg_len ? seg_len[seg] : seg_ptr[seg + 1] - a;
    const float K = 46.66666793823242f;                      // float32(70 * float32(2/3)), indexcov.go:153-157,175
    int b_out = 0, b_low = 0, b_hi = 0, b_in = 0;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const float d = depth[a + i];
        const float v = __fadd_rn(__fmul_rn(d, K), 0.5f);
        int slot = __float2int_rz(v);                       // Go int(f): truncation
        slot = slot < GL_INDEXCOV_SLOTS ? (slot < 0 ? 0 : slot) : GL_INDEXCOV_SLOTS - 1;
        atomicAdd(&s_cnt[slot], 1);
        const float c = d > 8.0f ? 8.0f : d;                // MaxCN clip, :694-697
        if (c < 0.85f || c > 1.15f) {                       // counter.count, :1053-1066
            b_out++;
            if (c > 1.15f) b_hi++;
            else if (c < 0.15f) b_low++;
        } else {
            b_in++;
        }
    }
    b_out = __reduce_add_sync(kFull, b_out); b_low = __reduce_add_sync(kFull, b_low);
    b_hi = __reduce_add_sync(kFull, b_hi); b_in = __reduce_add_sync(kFull, b_in);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&s_bin[0], b_out); atomicAdd(&s_bin[1], b_low); atomicAdd(&s_bin[2], b_hi); atomicAdd(&s_bin[3], b_in);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < GL_INDEXCOV_SLOTS; i += blockDim.x) counts70[(size_t)seg * GL_INDEXCOV_SLOTS + i] = s_cnt[i];
    if (threadIdx.x == 0) {
        const long long miss = longest ? max(0ll, longest[seg] - n) : 0;   // c.out += n - i; c.low += n - i  (:1076-1077)
        bins4[(size_t)seg * 4 + 0] = s_bin[0] + miss;
        bins4[(size_t)seg * 4 + 1] = s_bin[1] + miss;
        bins4[(size_t)seg * 4 + 2] = s_bin[2];
        bins4[(size_t)seg * 4 + 3] = s_bin[3];
    }
}

// ------------------------------------------------------------------------------------------------ I7
// One CTA; threads own samples (i = tid, tid+blockDim, ...).  For every tile j the float64 mean over
// samples of d[j], d[j-1], d[j+1] must equal the reference's sequential sum bit for bit.  A float64 sum of
// float32 addends is exact — hence order-free — when (max exponent + log2(count) + 1) - (min ulp exponent)
// <= 52; the block checks that per tile and otherwise thread 0 redoes the sum in the reference's order.
constexpr int kXnThreads = 1024;

__device__ __forceinline__ int f32_ulp_exp(float v) {       // exponent of the unit in the last place
    int e = (int)((__float_as_uint(v) >> 23) & 0xff);
    return (e == 0 ? 1 : e) - 127 - 23;
}

__global__ void __launch_bounds__(kXnThreads) ic_xnorm_kernel(float* __restrict__ depths, const int* __restrict__ lens, int S, int T,
                                                             int max_len) {
    __shared__ double s_sum[kXnThreads / 32];
    __shared__ int s_cnt[kXnThreads / 32], s_emax[kXnThreads / 32], s_emin[kXnThreads / 32];
    __shared__ double s_m;
    __shared__ int s_skip;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int j = 0; j < max_len; j++) {
        double part = 0;
        int cnt = 0, emax = -1000, emin = 1000;
        for (int i = tid; i < S; i += kXnThreads) {
            const int len = lens[i];
            if (len > j) {
                const float* d = depths + (size_t)i * T;
                float a = d[j];
                part += (double)a; cnt++;
                if (a != 0) { emax = max(emax, f32_ulp_exp(a) + 24); emin = min(emin, f32_ulp_exp(a)); }
                if (j > 0) { a = d[j - 1]; part += (double)a; cnt++; if (a != 0) { emax = max(emax, f32_ulp_exp(a) + 24); emin = min(emin, f32_ulp_exp(a)); } }
                if (j < len - 1) { a = d[j + 1]; part += (double)a; cnt++; if (a != 0) { emax = max(emax, f32_ulp_exp(a) + 24); emin = min(emin, f32_ulp_exp(a)); } }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(kFull, part, o);
        cnt = __reduce_add_sync(kFull, cnt);
        emax = __reduce_max_sync(kFull, emax);
        emin = __reduce_min_sync(kFull, emin);
        if (lane == 0) { s_sum[warp] = part; s_cnt[warp] = cnt; s_emax[warp] = emax; s_emin[warp] = emin; }
        __syncthreads();
        if (tid == 0) {
            double m = 0; int n = 0, ex = -1000, en = 1000;
            for (int w = 0; w < kXnThreads / 32; w++) { m += s_sum[w]; n += s_cnt[w]; ex = max(ex, s_emax[w]); en = min(en, s_emin[w]); }
            int lg = 0;
            while ((1 << lg) < n) lg++;
            const bool exact = (en == 1000) || (ex + lg + 1 - en <= 52);
            if (!exact) {                                   // reproduce the reference's order (indexcov.go:566-574)
                m = 0;
                for (int i = 0; i < S; i++) {
                    const int len = lens[i];
                    if (len > j) {
                        const float* d = depths + (size_t)i * T;
                        m += (double)d[j];
                        if (j > 0) m += (double)d[j - 1];
                        if (j < len - 1) m += (double)d[j + 1];
                    }
                }
            }
            int skip = n < 3 * S - 4;                       // :577
            if (!skip) {
                m = __ddiv_rn(m, (double)n);
                if (m < 0.1) skip = 1;
            }
            s_m = m;
            s_skip = skip;
        }
        __syncthreads();
        if (!s_skip) {
            const float m32 = __double2float_rn(s_m);
            for (int i = tid; i < S; i += kXnThreads) {
                const int len = lens[i];
                if (len > j) {
                    float* d = depths + (size_t)i * T;
                    float x = __fdiv_rn(d[j], m32);
                    if (j > 2 && j < len - 3) {
                        float a = __fadd_rn(d[j - 3], d[j - 2]);
                        a = __fadd_rn(a, d[j - 1]);
                        a = __fadd_rn(a, x);
                        a = __fadd_rn(a, __fdiv_rn(d[j + 1], m32));
                        a = __fadd_rn(a, __fdiv_rn(d[j + 2], m32));
                        a = __fadd_rn(a, __fdiv_rn(d[j + 3], m32));
                        x = __fmul_rn(0.14285714924335479736328125f, a);
                    }
                    d[j] = x;
                }
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ V2
constexpr int kBinSmem = 8192;
__global__ void __launch_bounds__(256) bincount_kernel(const int* __restrict__ v, long long n, int lo, int hi,
                                                      unsigned long long* __restrict__ hist) {
    __shared__ unsigned s_h[kBinSmem];
    const long long nb = (long long)hi - lo;                       // up to 2^32 - 1: the width and x - lo need 64 bits
    const bool priv = nb <= kBinSmem;
    if (priv) {
        for (int i = threadIdx.x; i < nb; i += blockDim.x) s_h[i] = 0;
        __syncthreads();
    }
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int x = v[i];
        if (x >= lo && x < hi) {
            const long long b = (long long)x - lo;
            if (priv) atomicAdd(&s_h[b], 1u);
            else atomicAdd(&hist[b], 1ull);
        }
    }
    if (priv) {
        __syncthreads();
        for (int i = threadIdx.x; i < nb; i += blockDim.x)
            if (s_h[i]) atomicAdd(&hist[i], (unsigned long long)s_h[i]);
    }
}

// ------------------------------------------------------------------------------------------------ W1
// Go's int(0.5 + dep) (depthwed.go:103) as amd64 compiles it (CVTTSD2SQ): truncation toward zero, and NaN, +-Inf and
// anything outside [-2^63, 2^63) become INT64_MIN.  __double2ll_rz leaves those inputs undefined (the H100 clamps +Inf and
// 0.5 + dep >= 2^63 to INT64_MAX), so they are sorted out first.  Returned as the two's-complement bits, for wrapping sums.
__device__ __forceinline__ unsigned long long go_int_half_up(double mean) {
    const double x = __dadd_rn(0.5, mean);
    if (!(x >= -9223372036854775808.0 && x < 9223372036854775808.0)) return 0x8000000000000000ull;
    return (unsigned long long)__double2ll_rz(x);
}

// means: S x R sample-major.  Group g sums rows [grp[g], grp[g+1]) of int(0.5+mean); out is n_out x S
// row-major.  A 32x32 tile goes through shared memory so both the reads and the writes are coalesced.  The sums wrap
// modulo 2^64 as Go's int additions do (taken unsigned: signed overflow is undefined in C++).
__global__ void __launch_bounds__(256) depthwed_kernel(const double* __restrict__ means, int S, long long R,
                                                      const long long* __restrict__ grp, long long n_out, int simple,
                                                      long long* __restrict__ out) {
    __shared__ unsigned long long s_t[32][33];
    const long long g0 = (long long)blockIdx.x * 32;
    const int s0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;       // 32 x 8
    for (int k = ty; k < 32; k += 8) {                             // k: sample inside the tile, tx: group
        const int s = s0 + k;
        const long long g = g0 + tx;
        unsigned long long acc = 0;
        if (s < S && g < n_out) {
            const long long a = simple ? g : grp[g], b = simple ? g + 1 : grp[g + 1];
            for (long long r = a; r < b; r++) acc += go_int_half_up(means[(size_t)s * R + r]);
        }
        s_t[k][tx] = acc;
    }
    __syncthreads();
    for (int k = ty; k < 32; k += 8) {                             // k: group inside the tile, tx: sample
        const long long g = g0 + k;
        const int s = s0 + tx;
        if (s < S && g < n_out) out[(size_t)g * S + s] = (long long)s_t[tx][k];
    }
}

// The same at the width BASELINE budgets (4 B in + 4 B out per cell): the reference rounds when it PARSES a line
// (depthwed.go:103 d.depth = int(0.5 + dep)), so the matrix that travels is int32.  Group sums are taken in 64 bits; a sum
// that does not fit int32 raises *overflow and the caller reruns on the int64 path.  Groups [g_begin, g_end) only: the
// caller walks the rows in chunks so that the all-gather of one chunk overlaps the aggregation of the next.
__global__ void __launch_bounds__(256) depthwed_i32_kernel(const int* __restrict__ depth, int S, long long R, const long long* __restrict__ grp,
                                                          long long g_begin, long long g_end, int simple, int* __restrict__ out,
                                                          int* __restrict__ overflow) {
    __shared__ int s_t[32][33];
    const long long g0 = g_begin + (long long)blockIdx.x * 32;
    const int s0 = blockIdx.y * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;       // 32 x 8
    for (int k = ty; k < 32; k += 8) {                             // k: sample inside the tile, tx: group
        const int s = s0 + k;
        const long long g = g0 + tx;
        long long acc = 0;
        if (s < S && g < g_end) {
            const long long a = simple ? g : grp[g], b = simple ? g + 1 : grp[g + 1];
            for (long long r = a; r < b; r++) acc += depth[(size_t)s * R + r];
            if (acc > 2147483647ll || acc < -2147483648ll) *overflow = 1;
        }
        s_t[k][tx] = (int)acc;
    }
    __syncthreads();
    for (int k = ty; k < 32; k += 8) {                             // k: group inside the tile, tx: sample
        const long long g = g0 + k;
        const int s = s0 + tx;
        if (s < S && g < g_end) out[(size_t)(g - g_begin) * S + s] = s_t[tx][k];
    }
}

// W1 fused with its collective: the aggregation kernel stores every output row straight into the row-major n-sites x
// n-samples matrix of EVERY GPU — its own and, through NVLink peer mappings, the other ranks' — so the matrix is assembled
// while it is computed and no separate all-gather pass (and no block re-assembly on the receiving side) exists.
// dst[d] = base of rank d's matrix (row stride `row_stride` ints); this rank owns columns [col_off, col_off + S).
// A warp stores 32 consecutive samples of one row (128 B), one store per destination; the destinations are visited in a
// per-block rotated order so that all NVLink links carry traffic all the time.  Stores to a peer are complete when the
// kernel is; the ranks then meet at a host barrier.
struct WedPeers { int* dst[16]; };
// A CTA takes 32 rows (groups) x 128 samples.  Phase 1 reads the sample-major input coalesced along the rows (one warp
// instruction = 32 consecutive rows of one sample) and parks the group sums in shared memory; phase 2 stores them
// row-major with 16-BYTE stores: a lane owns 4 consecutive samples of one row, a warp instruction covers 512 B of it —
// NVLink likes wide stores (4-byte stores reached a quarter of the link rate).  `vec` (decided on the host) says every
// destination is 16-byte aligned and row_stride and col_off are multiples of 4 (callers pad the per-rank width to a
// multiple of 4); otherwise scalar stores.
__global__ void __launch_bounds__(256) depthwed_i32_p2p_kernel(const int* __restrict__ depth, int S, long long R, const long long* __restrict__ grp,
                                                              long long g_begin, long long g_end, int simple, WedPeers peers, int world,
                                                              long long row_stride, int col_off, int vec, int* __restrict__ overflow) {
    __shared__ __align__(16) int s_t[32][132];                     // [row][sample], padded: 132 keeps int4 alignment and spreads banks
    const long long g0 = g_begin + (long long)blockIdx.x * 32;
    const int s0 = blockIdx.y * 128;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;       // 32 lanes x 8 warps
    for (int k = ty; k < 128; k += 8) {                            // k: sample inside the tile, tx: row
        const int s = s0 + k;
        const long long g = g0 + tx;
        long long acc = 0;
        if (s < S && g < g_end) {
            const long long a = simple ? g : grp[g], b = simple ? g + 1 : grp[g + 1];
            for (long long r = a; r < b; r++) acc += depth[(size_t)s * R + r];
            if (acc > 2147483647ll || acc < -2147483648ll) *overflow = 1;
        }
        s_t[tx][k] = (int)acc;
    }
    __syncthreads();
    const int rot = (int)((blockIdx.x + blockIdx.y) % (unsigned)world);
    for (int k = ty; k < 32; k += 8) {                             // k: row inside the tile, tx: 4 consecutive samples
        const long long g = g0 + k;
        const int s = s0 + 4 * tx;
        if (g >= g_end || s >= S) continue;
        const size_t at = (size_t)g * (size_t)row_stride + (size_t)(col_off + s);
        const int4 v = *reinterpret_cast<const int4*>(&s_t[k][4 * tx]);
        for (int d = 0; d < world; d++) {
            int dd = d + rot; if (dd >= world) dd -= world;
            int* dst = peers.dst[dd] + at;
            if (vec && s + 3 < S) *reinterpret_cast<int4*>(dst) = v;
            else {
                dst[0] = v.x;
                if (s + 1 < S) dst[1] = v.y;
                if (s + 2 < S) dst[2] = v.z;
                if (s + 3 < S) dst[3] = v.w;
            }
        }
    }
}

// ------------------------------------------------------------------------------------------------ I6
// float32 -> the bytes of Go's fmt "%.3g" (== C printf "%.3g" of the same value), exactly: the three significant
// digits come from integer arithmetic on mantissa * 10^k (128-bit), rounded half-to-even on the exact binary
// value, never from floating-point scaling.  Output: 10-byte tokens, bytes [0..len) = text, byte 9 = len
// (len 0 = "format this one on the host": magnitudes outside [1e-15, 1e15), not seen in normalised depths).
__device__ __forceinline__ unsigned __int128 pow10_u128(int k) {
    unsigned __int128 r = 1;
    for (int i = 0; i < k; i++) r *= 10;
    return r;
}

// round_half_even( m * 2^e2 * 10^k ) for 0 <= result < 2^63
__device__ __forceinline__ unsigned long long scaled_round(unsigned m, int e2, int k) {
    unsigned __int128 num = m, den = 1;
    if (k >= 0) num *= pow10_u128(k); else den *= pow10_u128(-k);
    if (e2 >= 0) num <<= e2; else den <<= -e2;
    unsigned __int128 q = num / den, r = num % den;
    const unsigned __int128 twice = r * 2;
    if (twice > den || (twice == den && (q & 1))) q++;
    return (unsigned long long)q;
}

__constant__ unsigned long long c_p10[13] = {1ull, 10ull, 100ull, 1000ull, 10000ull, 100000ull, 1000000ull, 10000000ull, 100000000ull,
                                              1000000000ull, 10000000000ull, 100000000000ull, 1000000000000ull};

// the same value in 64-bit arithmetic when everything fits (normalised depths are 1e-3 .. 1e3: k in [0, 5], a power-of-two
// denominator -> a multiply, a shift and a compare); false: take scaled_round
__device__ __forceinline__ bool scaled_round_fast(unsigned m, int e2, int k, unsigned long long& N) {
    if (k >= 0) {
        if (k > 11 || e2 >= 0 || e2 <= -64) return false;
        const unsigned long long num = (unsigned long long)m * c_p10[k];            // < 2^24 * 10^11 < 2^61
        const int sh = -e2;
        const unsigned long long q = num >> sh, rem = num & ((1ull << sh) - 1ull), half = 1ull << (sh - 1);
        N = q + ((rem > half || (rem == half && (q & 1ull))) ? 1ull : 0ull);
        return true;
    }
    if (-k > 12) return false;
    unsigned long long den = c_p10[-k], num = m;
    if (e2 >= 0) { if (e2 > 39) return false; num <<= e2; }
    else { const int sh = -e2; if (sh >= 62 || den > (0x3fffffffffffffffull >> sh)) return false; den <<= sh; }
    const unsigned long long q = num / den, r = num - q * den;                     // den < 2^62: 2 r does not overflow
    N = q + ((2ull * r > den || (2ull * r == den && (q & 1ull))) ? 1ull : 0ull);
    return true;
}

__device__ __forceinline__ unsigned long long scaled_round_any(unsigned m, int e2, int k) {
    unsigned long long N;
    return scaled_round_fast(m, e2, k, N) ? N : scaled_round(m, e2, k);
}

// One value per thread; the 10-byte tokens of a CTA are put together in shared memory and leave as 16-byte stores (a thread
// writing its own 10 bytes issued ten strided byte stores: the kernel ran at 6 % of HBM bandwidth).
__global__ void __launch_bounds__(256) fmt_g3_kernel(const float* __restrict__ v, long long n, unsigned char* __restrict__ out) {
    __shared__ __align__(16) unsigned char s_tok[256 * 10];
    const long long i0 = (long long)blockIdx.x * 256;
    const long long i = i0 + threadIdx.x;
    unsigned char t[10];
#pragma unroll
    for (int k = 0; k < 10; k++) t[k] = 0;
    const float f = i < n ? v[i] : 0.0f;
    const unsigned bits = __float_as_uint(f);
    const bool neg = bits >> 31;
    const unsigned ex = (bits >> 23) & 0xff, frac = bits & 0x7fffff;
    int len = 0;
    if (ex == 0xff) {                                            // Go: "+Inf" "-Inf" "NaN"
        if (frac) { t[0] = 'N'; t[1] = 'a'; t[2] = 'N'; len = 3; }
        else { t[0] = neg ? '-' : '+'; t[1] = 'I'; t[2] = 'n'; t[3] = 'f'; len = 4; }
    } else if (ex == 0 && frac == 0) {
        if (neg) t[len++] = '-';
        t[len++] = '0';
    } else {
        const unsigned m = ex ? (frac | 0x800000u) : frac;
        const int e2 = ex ? (int)ex - 150 : -149;
        // floor(log10 |f|): for normal numbers from the binary exponent E (2^E <= |f| < 2^(E+1)): floor(E log10 2) is the answer or
        // one less (corrected below by the digits themselves); subnormals take the floating-point estimate
        int e10 = ex ? (((int)ex - 127) * 78913) >> 18 : (int)floor(log10((double)fabsf(f)));
        if (e10 < -16 || e10 >= 15) {
            len = 0;                                             // host formats it
        } else {
            unsigned long long N = scaled_round_any(m, e2, 2 - e10);
            if (N < 100) { e10--; N = scaled_round_any(m, e2, 2 - e10); }          // estimate one too high
            else if (N > 1000) { e10++; N = scaled_round_any(m, e2, 2 - e10); }    // one too low
            if (N >= 1000) { N = 100; e10++; }                                     // 999.5.. rounds up to the next decade
            if (e10 < -15) len = 0;                              // below 1e-15 after all: the host's
            else {
            const unsigned Nu = (unsigned)N;
            const int d1 = (int)(Nu / 100u), d2 = (int)(Nu / 10u % 10u), d3 = (int)(Nu % 10u);
            const int nd = d3 ? 3 : (d2 ? 2 : 1);                // significant digits after stripping zeros
            const int dig[3] = {d1, d2, d3};
            if (neg) t[len++] = '-';
            if (e10 < -4 || e10 >= 3) {                          // %e form, exponent at least two digits
                t[len++] = (unsigned char)('0' + d1);
                if (nd > 1) { t[len++] = '.'; t[len++] = (unsigned char)('0' + d2); if (nd > 2) t[len++] = (unsigned char)('0' + d3); }
                t[len++] = 'e';
                t[len++] = e10 < 0 ? '-' : '+';
                const int ae = e10 < 0 ? -e10 : e10;
                t[len++] = (unsigned char)('0' + ae / 10);
                t[len++] = (unsigned char)('0' + ae % 10);
            } else if (e10 >= 0) {                               // d[.d[d]] with the point after e10+1 digits
                for (int k = 0; k < 3; k++) {
                    if (k <= e10 || k < nd) {
                        if (k == e10 + 1) t[len++] = '.';
                        t[len++] = (unsigned char)('0' + dig[k]);
                    }
                }
            } else {                                             // 0.000ddd
                t[len++] = '0'; t[len++] = '.';
                for (int z = 0; z < -e10 - 1; z++) t[len++] = '0';
                for (int k = 0; k < nd; k++) t[len++] = (unsigned char)('0' + dig[k]);
            }
            }
        }
    }
    t[9] = (unsigned char)len;
    unsigned short* st = reinterpret_cast<unsigned short*>(s_tok + threadIdx.x * 10);
#pragma unroll
    for (int k = 0; k < 5; k++) st[k] = (unsigned short)(t[2 * k] | (t[2 * k + 1] << 8));
    __syncthreads();
    const long long live = min((long long)256, n - i0);         // tokens of this CTA that exist
    unsigned char* o = out + i0 * 10;
    if (live == 256 && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
        if (threadIdx.x < 160) reinterpret_cast<uint4*>(o)[threadIdx.x] = reinterpret_cast<const uint4*>(s_tok)[threadIdx.x];
    } else {
        for (long long j = threadIdx.x; j < live * 10; j += 256) o[j] = s_tok[j];
    }
}

// indexsplit (indexsplit/indexsplit.go:92-115): cohort data per 16 KB tile = sum over the samples, IN PATH ORDER, of
// float64(size)/1e9.  One thread per (reference, tile): the float64 adds run in the reference's order, so the result is
// bit-identical; consecutive tiles of one sample are consecutive in memory, so every pass over the samples is coalesced.
// ptr[s*(R+1)+r] = offset of sample s's tiles of reference r in `sizes` (a sample with fewer references repeats its end).
__global__ void __launch_bounds__(256) indexsplit_sum_kernel(const long long* __restrict__ sizes, const long long* __restrict__ ptr,
                                                            int S, int R, const long long* __restrict__ out_ptr, double* __restrict__ out) {
    const int r = blockIdx.y;
    const long long j = (long long)blockIdx.x * 256 + threadIdx.x;
    const long long n = out_ptr[r + 1] - out_ptr[r];
    if (j >= n) return;
    double acc = 0.0;
    for (int s = 0; s < S; s++) {
        const long long a = ptr[(size_t)s * (R + 1) + r], b = ptr[(size_t)s * (R + 1) + r + 1];
        if (j < b - a) acc += (double)sizes[a + j] / 1000000000.0;
    }
    out[out_ptr[r] + j] = acc;
}

}  // namespace

// hist[x - lo] = how many of the n device values equal x, for x in [lo, hi); queued on ctx->stream
int gl_bincount_device(gl_ctx* ctx, const int32_t* d_v, int64_t n, int32_t lo, int32_t hi, unsigned long long* d_hist) {
    GL_CUDA(ctx, cudaMemsetAsync(d_hist, 0, (size_t)((int64_t)hi - lo) * 8, ctx->stream));
    if (n) {
        const unsigned grid = (unsigned)std::min<int64_t>((n + 255) / 256, (int64_t)ctx->sm_count * 8);
        {
            gl_prof_scope prof(ctx, "bincount_kernel");
            bincount_kernel<<<grid, 256, 0, ctx->stream>>>(d_v, n, lo, hi, d_hist);
        }
        GL_LAUNCHED(ctx, 1);
    }
    return GL_OK;
}

extern "C" {

int gl_indexcov_sizes(gl_ctx* ctx, const uint64_t* voff, const int64_t* ref_ptr, int32_t n_refs, int64_t* sizes,
                      int64_t* size_ptr) {
    GL_CHECK(gl_use(ctx));
    if (n_refs < 0 || !ref_ptr || !size_ptr || (n_refs > 0 && !voff)) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_sizes: bad argument");
    std::vector<int64_t> voff_off, size_off;                       // one gl_indexcov_sizes_batch_device descriptor per
    std::vector<int32_t> n_intv;                                   // reference with >= 2 entries
    size_ptr[0] = 0;
    for (int32_t r = 0; r < n_refs; r++) {
        const int64_t ni = ref_ptr[r + 1] - ref_ptr[r];
        if (ni < 0) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_sizes: ref_ptr not monotone");
        if (ni > INT32_MAX) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_sizes: reference %d has more than %d entries", r, INT32_MAX);
        size_ptr[r + 1] = size_ptr[r] + (ni >= 2 ? ni - 1 : 0);     // types.go:68-72
        if (ni >= 2) { voff_off.push_back(ref_ptr[r]); n_intv.push_back((int32_t)ni); size_off.push_back(size_ptr[r]); }
    }
    const int64_t total_v = ref_ptr[n_refs], total_s = size_ptr[n_refs];
    if (total_s == 0) return GL_OK;
    if (!sizes) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_sizes: null sizes");
    gl_scratch tmp(ctx);
    uint64_t* d_voff; int64_t *d_voff_off, *d_size_off, *d_sizes; int32_t* d_n_intv;
    GL_CHECK(tmp.upload(d_voff, voff, (size_t)total_v));
    GL_CHECK(tmp.upload(d_voff_off, voff_off.data(), voff_off.size()));
    GL_CHECK(tmp.upload(d_n_intv, n_intv.data(), n_intv.size()));
    GL_CHECK(tmp.upload(d_size_off, size_off.data(), size_off.size()));
    GL_CHECK(tmp.alloc(d_sizes, (size_t)total_s));
    GL_CHECK(gl_indexcov_sizes_batch_device(ctx, d_voff, d_voff_off, d_n_intv, d_size_off, (int64_t)n_intv.size(), d_sizes));
    GL_CUDA(ctx, cudaMemcpyAsync(sizes, d_sizes, (size_t)total_s * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_indexcov_cohort_device(gl_ctx* ctx, const int64_t* d_sizes, const int64_t* d_sample_ptr, int32_t S,
                              double* d_medians, float* d_depth_out) {
    GL_CHECK(gl_use(ctx));
    if (S < 0 || !d_sizes || !d_sample_ptr || !d_medians) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_cohort_device: bad argument");
    if (S == 0) return GL_OK;
    if (!ctx->cohort_attr_set) {                              // per device (a function attribute belongs to the device it was set on)
        GL_CUDA(ctx, cudaFuncSetAttribute(ic_cohort2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(C2Smem)));
        ctx->cohort_attr_set = true;
    }
    GL_CHECK(gl_buf_reserve(ctx, ctx->misc, 64));
    GL_CUDA(ctx, cudaMemsetAsync(ctx->misc.p, 0, 4, ctx->stream));
    {
        gl_prof_scope prof(ctx, "ic_cohort2_kernel");
        const unsigned grid = (unsigned)std::min<int64_t>((int64_t)S, (int64_t)ctx->sm_count);
        ic_cohort2_kernel<<<grid, kC2Threads, sizeof(C2Smem), ctx->stream>>>(reinterpret_cast<const long long*>(d_sizes),
                                                                              reinterpret_cast<const long long*>(d_sample_ptr), S, d_medians,
                                                                              d_depth_out, static_cast<unsigned*>(ctx->misc.p));
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaMemcpyAsync(&ctx->cohort_fallbacks, ctx->misc.p, 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

// how many samples of the last gl_indexcov_cohort* call took the exact fallback select instead of the bracketed path
int gl_indexcov_cohort_fallbacks(gl_ctx* ctx, int32_t* n) {
    if (!ctx || !n) return gl_fail(ctx, GL_EINVAL, "null argument");
    *n = (int32_t)ctx->cohort_fallbacks;
    return GL_OK;
}

// I1 for every sample at once (one launch): voff = all samples' linear-index virtual offsets concatenated; descriptor d
// says reference d's n_intv[d] entries start at voff_off[d] and its n_intv[d]-1 sizes go to size_off[d] (device pointers).
int gl_indexcov_sizes_batch_device(gl_ctx* ctx, const uint64_t* d_voff, const int64_t* d_voff_off, const int32_t* d_n_intv,
                                   const int64_t* d_size_off, int64_t n_desc, int64_t* d_sizes) {
    GL_CHECK(gl_use(ctx));
    if (n_desc < 0 || (n_desc > 0 && (!d_voff || !d_voff_off || !d_n_intv || !d_size_off || !d_sizes))) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_sizes_batch_device: bad argument");
    if (n_desc == 0) return GL_OK;
    GL_CHECK(gl_buf_reserve(ctx, ctx->misc, 64));
    GL_CUDA(ctx, cudaMemsetAsync(static_cast<char*>(ctx->misc.p) + 16, 0, 4, ctx->stream));
    {
        gl_prof_scope prof(ctx, "ic_sizes_batch_kernel");
        ic_sizes_batch_kernel<<<(unsigned)((n_desc * 32 + 255) / 256), 256, 0, ctx->stream>>>(
            reinterpret_cast<const unsigned long long*>(d_voff), reinterpret_cast<const long long*>(d_voff_off), d_n_intv,
            reinterpret_cast<const long long*>(d_size_off), n_desc, reinterpret_cast<long long*>(d_sizes), reinterpret_cast<int*>(static_cast<char*>(ctx->misc.p) + 16));
    }
    GL_LAUNCHED(ctx, 1);
    int neg = 0;
    GL_CUDA(ctx, cudaMemcpyAsync(&neg, static_cast<char*>(ctx->misc.p) + 16, 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (neg) return gl_fail(ctx, GL_ERANGE, "gl_indexcov_sizes_batch: expected positive change in vOffset");   // types.go:75-77
    return GL_OK;
}

int gl_indexcov_cohort(gl_ctx* ctx, const int64_t* sizes, const int64_t* sample_ptr, int32_t S, double* medians,
                       float* depth_out) {
    GL_CHECK(gl_use(ctx));
    if (S < 0 || !sample_ptr || !medians) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_cohort: bad argument");
    if (S == 0) return GL_OK;
    const int64_t total = sample_ptr[S];
    if (total > 0 && !sizes) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_cohort: null sizes");
    gl_scratch tmp(ctx);
    int64_t *d_sizes, *d_ptr; double* d_med; float* d_depth = nullptr;
    GL_CHECK(tmp.upload(d_sizes, sizes, (size_t)total));
    GL_CHECK(tmp.upload(d_ptr, sample_ptr, (size_t)S + 1));
    GL_CHECK(tmp.alloc(d_med, (size_t)S));
    if (depth_out) GL_CHECK(tmp.alloc(d_depth, (size_t)total));
    GL_CHECK(gl_indexcov_cohort_device(ctx, d_sizes, d_ptr, S, d_med, d_depth));
    GL_CUDA(ctx, cudaMemcpyAsync(medians, d_med, (size_t)S * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (depth_out && total) GL_CUDA(ctx, cudaMemcpyAsync(depth_out, d_depth, (size_t)total * 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_indexcov_scale(gl_ctx* ctx, const int64_t* sizes, int64_t n, int64_t* median_out) {
    if (n <= 0 || !sizes || !median_out) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_scale: needs at least one tile (indexcov.go:100-102)");
    const int64_t ptr[2] = {0, n};
    double m = 0;
    GL_CHECK(gl_indexcov_cohort(ctx, sizes, ptr, 1, &m, nullptr));
    *median_out = (int64_t)m;
    return GL_OK;
}

int gl_indexcov_normalize(gl_ctx* ctx, const int64_t* sizes, int64_t n, double median, float* depth_out) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || (n > 0 && (!sizes || !depth_out))) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_normalize: bad argument");
    if (n == 0) return GL_OK;
    if (median == 0.0) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_normalize: median is 0 (the reference returns no depths, indexcov.go:140-142)");
    gl_scratch tmp(ctx);
    int64_t* d_sizes; float* d_depth;
    GL_CHECK(tmp.upload(d_sizes, sizes, (size_t)n));
    GL_CHECK(tmp.alloc(d_depth, (size_t)n));
    {
        gl_prof_scope prof(ctx, "ic_normalize_kernel");
        ic_normalize_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(reinterpret_cast<const long long*>(d_sizes), n, median, d_depth);
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaMemcpyAsync(depth_out, d_depth, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_indexcov_counts_batch_device(gl_ctx* ctx, const float* d_depth, const int64_t* d_seg_ptr, const int64_t* d_longest,
                                    int32_t n_seg, int32_t* d_counts70, int64_t* d_bins4) {
    GL_CHECK(gl_use(ctx));
    if (n_seg < 0 || !d_seg_ptr || !d_counts70 || !d_bins4) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_counts_batch_device: bad argument");
    if (n_seg == 0) return GL_OK;
    {
        gl_prof_scope prof(ctx, "ic_counts_kernel");
        ic_counts_kernel<<<(unsigned)n_seg, 256, 0, ctx->stream>>>(d_depth, reinterpret_cast<const long long*>(d_seg_ptr), nullptr,
                                                                   reinterpret_cast<const long long*>(d_longest), n_seg, d_counts70,
                                                                   reinterpret_cast<long long*>(d_bins4));
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

// I4+I5 for arbitrary slices of a device-resident depth array: every (chromosome, sample) pair of a cohort in one launch
int gl_indexcov_counts_segs_device(gl_ctx* ctx, const float* d_depth, const int64_t* d_seg_start, const int64_t* d_seg_len,
                                   const int64_t* d_longest, int32_t n_seg, int32_t* d_counts70, int64_t* d_bins4) {
    GL_CHECK(gl_use(ctx));
    if (n_seg < 0 || !d_seg_start || !d_seg_len || !d_counts70 || !d_bins4) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_counts_segs_device: bad argument");
    if (n_seg == 0) return GL_OK;
    {
        gl_prof_scope prof(ctx, "ic_counts_kernel");
        ic_counts_kernel<<<(unsigned)n_seg, 256, 0, ctx->stream>>>(d_depth, reinterpret_cast<const long long*>(d_seg_start),
                                                                   reinterpret_cast<const long long*>(d_seg_len),
                                                                   reinterpret_cast<const long long*>(d_longest), n_seg, d_counts70,
                                                                   reinterpret_cast<long long*>(d_bins4));
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_indexcov_counts_batch(gl_ctx* ctx, const float* depth, const int64_t* seg_ptr, const int64_t* longest, int32_t n_seg,
                             int32_t* counts70, int64_t* bins4) {
    GL_CHECK(gl_use(ctx));
    if (n_seg < 0 || !seg_ptr || !counts70 || !bins4) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_counts_batch: bad argument");
    if (n_seg == 0) return GL_OK;
    const int64_t total = seg_ptr[n_seg];
    gl_scratch tmp(ctx);
    float* d_depth; int64_t *d_ptr, *d_longest = nullptr, *d_bins; int32_t* d_counts;
    GL_CHECK(tmp.upload(d_depth, depth, (size_t)total));
    GL_CHECK(tmp.upload(d_ptr, seg_ptr, (size_t)n_seg + 1));
    if (longest) GL_CHECK(tmp.upload(d_longest, longest, (size_t)n_seg));
    GL_CHECK(tmp.alloc(d_counts, (size_t)n_seg * GL_INDEXCOV_SLOTS));
    GL_CHECK(tmp.alloc(d_bins, (size_t)n_seg * 4));
    GL_CHECK(gl_indexcov_counts_batch_device(ctx, d_depth, d_ptr, d_longest, n_seg, d_counts, d_bins));
    GL_CUDA(ctx, cudaMemcpyAsync(counts70, d_counts, (size_t)n_seg * GL_INDEXCOV_SLOTS * 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(bins4, d_bins, (size_t)n_seg * 32, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_indexcov_counts(gl_ctx* ctx, const float* depth, int64_t n, int32_t counts[GL_INDEXCOV_SLOTS]) {
    if (n < 0 || !counts) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_counts: bad argument");
    const int64_t ptr[2] = {0, n};
    int32_t c[GL_INDEXCOV_SLOTS];
    int64_t b[4];
    GL_CHECK(gl_indexcov_counts_batch(ctx, depth, ptr, nullptr, 1, c, b));
    for (int i = 0; i < GL_INDEXCOV_SLOTS; i++) counts[i] += c[i];            // counts[...]++ accumulates, indexcov.go:175
    return GL_OK;
}

int gl_indexcov_bins(gl_ctx* ctx, const float* depth, int64_t n, int64_t longest, int64_t out4[4]) {
    if (n < 0 || !out4) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_bins: bad argument");
    const int64_t ptr[2] = {0, n};
    int32_t c[GL_INDEXCOV_SLOTS];
    int64_t b[4];
    GL_CHECK(gl_indexcov_counts_batch(ctx, depth, ptr, &longest, 1, c, b));
    for (int i = 0; i < 4; i++) out4[i] += b[i];
    return GL_OK;
}

int gl_indexcov_xnorm(gl_ctx* ctx, float* depths, const int32_t* lens, int32_t S, int32_t T) {
    GL_CHECK(gl_use(ctx));
    if (S < 0 || T < 0 || (S > 0 && (!depths || !lens))) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_xnorm: bad argument");
    if (S < 5 || T == 0) return GL_OK;                                          // indexcov.go:551
    int32_t max_len = 0;
    for (int32_t i = 0; i < S; i++) {
        if (lens[i] < 0 || lens[i] > T) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_xnorm: lens[%d] out of range", i);
        if (lens[i] > max_len) max_len = lens[i];
    }
    gl_scratch tmp(ctx);
    float* d_depths; int32_t* d_lens;
    GL_CHECK(tmp.upload(d_depths, depths, (size_t)S * T));
    GL_CHECK(tmp.upload(d_lens, lens, (size_t)S));
    {
        gl_prof_scope prof(ctx, "ic_xnorm_kernel");
        ic_xnorm_kernel<<<1, kXnThreads, 0, ctx->stream>>>(d_depths, d_lens, S, T, max_len);
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaMemcpyAsync(depths, d_depths, (size_t)S * T * 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_format_g3_device(gl_ctx* ctx, const float* d_vals, int64_t n, uint8_t* d_tokens) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || (n > 0 && (!d_vals || !d_tokens))) return gl_fail(ctx, GL_EINVAL, "gl_format_g3_device: bad argument");
    if (n == 0) return GL_OK;
    {
        gl_prof_scope prof(ctx, "fmt_g3_kernel");
        fmt_g3_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_vals, n, d_tokens);
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_format_g3(gl_ctx* ctx, const float* vals, int64_t n, uint8_t* tokens) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || (n > 0 && (!vals || !tokens))) return gl_fail(ctx, GL_EINVAL, "gl_format_g3: bad argument");
    if (n == 0) return GL_OK;
    gl_scratch tmp(ctx);
    float* d_vals; uint8_t* d_tokens;
    GL_CHECK(tmp.upload(d_vals, vals, (size_t)n));
    GL_CHECK(tmp.alloc(d_tokens, (size_t)n * 10));
    GL_CHECK(gl_format_g3_device(ctx, d_vals, n, d_tokens));
    GL_CUDA(ctx, cudaMemcpyAsync(tokens, d_tokens, (size_t)n * 10, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_indexsplit_accumulate(gl_ctx* ctx, const int64_t* sizes, const int64_t* ptr, int32_t S, int32_t R, const int64_t* out_ptr, double* out) {
    GL_CHECK(gl_use(ctx));
    if (S < 0 || R < 0 || !out_ptr || (S > 0 && R > 0 && !ptr)) return gl_fail(ctx, GL_EINVAL, "gl_indexsplit_accumulate: bad argument");
    if (R == 0) return GL_OK;
    const int64_t n_out = out_ptr[R] - out_ptr[0];
    int64_t max_len = 0;
    for (int32_t r = 0; r < R; r++) {
        if (out_ptr[r + 1] < out_ptr[r]) return gl_fail(ctx, GL_EINVAL, "gl_indexsplit_accumulate: out_ptr not monotone");
        max_len = std::max<int64_t>(max_len, out_ptr[r + 1] - out_ptr[r]);
    }
    if (n_out == 0 || out_ptr[0] != 0) return n_out == 0 ? GL_OK : gl_fail(ctx, GL_EINVAL, "gl_indexsplit_accumulate: out_ptr[0] must be 0");
    if (!out || (S > 0 && !sizes)) return gl_fail(ctx, GL_EINVAL, "gl_indexsplit_accumulate: bad argument");
    const int64_t n_in = S > 0 ? ptr[(size_t)(S - 1) * (R + 1) + R] : 0;
    for (int32_t s = 0; s < S; s++)
        for (int32_t r = 0; r < R; r++) {
            const int64_t a = ptr[(size_t)s * (R + 1) + r], b = ptr[(size_t)s * (R + 1) + r + 1];
            if (a < 0 || b < a || b > n_in || b - a > out_ptr[r + 1] - out_ptr[r]) return gl_fail(ctx, GL_EINVAL, "gl_indexsplit_accumulate: ptr out of range (sample %d, ref %d)", s, r);
        }
    if (R > 65535) return gl_fail(ctx, GL_ERANGE, "gl_indexsplit_accumulate: more than 65535 references");
    gl_scratch tmp(ctx);
    int64_t *d_sizes, *d_ptr, *d_out_ptr; double* d_out;
    GL_CHECK(tmp.upload(d_sizes, sizes, (size_t)n_in));
    GL_CHECK(tmp.upload(d_ptr, ptr, (size_t)S * (R + 1)));
    GL_CHECK(tmp.upload(d_out_ptr, out_ptr, (size_t)R + 1));
    GL_CHECK(tmp.alloc(d_out, (size_t)n_out));
    {
        gl_prof_scope prof(ctx, "indexsplit_sum_kernel");
        indexsplit_sum_kernel<<<dim3((unsigned)((max_len + 255) / 256), (unsigned)R), 256, 0, ctx->stream>>>(
            reinterpret_cast<const long long*>(d_sizes), reinterpret_cast<const long long*>(d_ptr), S, R,
            reinterpret_cast<const long long*>(d_out_ptr), d_out);
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaMemcpyAsync(out, d_out, (size_t)n_out * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_bincount_i32(gl_ctx* ctx, const int32_t* v, int64_t n, int32_t lo, int32_t hi, uint64_t* hist) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || hi <= lo || !hist || (n > 0 && !v)) return gl_fail(ctx, GL_EINVAL, "gl_bincount_i32: bad argument");
    const int64_t nb = (int64_t)hi - lo;
    gl_scratch tmp(ctx);
    int32_t* d_v; unsigned long long* d_hist;
    GL_CHECK(tmp.upload(d_v, v, (size_t)n));
    GL_CHECK(tmp.alloc(d_hist, (size_t)nb));
    GL_CHECK(gl_bincount_device(ctx, d_v, n, lo, hi, d_hist));
    GL_CUDA(ctx, cudaMemcpyAsync(hist, d_hist, (size_t)nb * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

}  // extern "C"

// groups of consecutive rows per output line (depthwed.go:117-157): sequential in the row order, O(R) on the host
template <class Pos>
static int64_t depthwed_groups(int64_t R, const Pos* starts, const Pos* ends, const int32_t* chrom_id, int64_t size,
                               std::vector<int64_t>& grp) {
    grp.clear();
    int64_t r = 0;
    while (r < R) {
        grp.push_back(r);
        const int32_t chrom = chrom_id[r];
        const int64_t st = starts[r];
        int64_t en = ends[r];
        r++;
        while (r < R && en - st < size && chrom_id[r] == chrom) { en = ends[r]; r++; }
    }
    grp.push_back(R);
    return (int64_t)grp.size() - 1;
}

// a depthwed column (int64 group sums) narrowed to int32; *overflow = 1 when a sum does not fit
__global__ void __launch_bounds__(256) depthwed_narrow_kernel(const long long* __restrict__ col, long long n, int* __restrict__ out,
                                                             int* __restrict__ overflow) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const long long v = col[i];
    if (v > 2147483647ll || v < -2147483648ll) *overflow = 1;
    out[i] = (int)v;
}

extern "C" {

int gl_depthwed_plan(const int64_t* starts, const int64_t* ends, const int32_t* chrom_id, int64_t R, int64_t size, int64_t* grp_first,
                     int64_t* out_start, int64_t* out_end, int32_t* out_chrom, int64_t cap, int64_t* n_groups) {
    if (R < 0 || size <= 0 || !n_groups || (R > 0 && (!starts || !ends || !chrom_id)))
        return gl_fail(nullptr, GL_EINVAL, "gl_depthwed_plan: bad argument");
    std::vector<int64_t> grp;
    const int64_t ng = depthwed_groups(R, starts, ends, chrom_id, size, grp);
    *n_groups = ng;
    if (ng > cap) return gl_fail(nullptr, GL_ERANGE, "gl_depthwed_plan: %lld groups > cap %lld", (long long)ng, (long long)cap);
    for (int64_t g = 0; g <= ng; g++) {
        if (grp_first) grp_first[g] = grp[g];
        if (g == ng) break;
        if (out_start) out_start[g] = starts[grp[g]];
        if (out_end) out_end[g] = ends[grp[g + 1] - 1];
        if (out_chrom) out_chrom[g] = chrom_id[grp[g]];
    }
    return GL_OK;
}

int gl_depthwed_column_i32(gl_ctx* ctx, const int64_t* d_col, int64_t n_groups, int32_t* d_col32, int32_t* d_overflow) {
    GL_CHECK(gl_use(ctx));
    if (n_groups < 0 || !d_overflow || (n_groups > 0 && (!d_col || !d_col32))) return gl_fail(ctx, GL_EINVAL, "gl_depthwed_column_i32: bad argument");
    GL_CUDA(ctx, cudaMemsetAsync(d_overflow, 0, 4, ctx->stream));
    if (n_groups == 0) return GL_OK;
    {
        gl_prof_scope prof(ctx, "depthwed_narrow_kernel");
        depthwed_narrow_kernel<<<(unsigned)((n_groups + 255) / 256), 256, 0, ctx->stream>>>(reinterpret_cast<const long long*>(d_col), n_groups,
                                                                                             d_col32, d_overflow);
    }
    GL_LAUNCHED(ctx, 1);
    return GL_OK;
}

int gl_depthwed_aggregate_device(gl_ctx* ctx, const double* d_means, int32_t S, int64_t R, const int64_t* d_grp, int64_t n_out,
                                 int64_t* d_out) {
    GL_CHECK(gl_use(ctx));
    if (S <= 0 || R < 0 || n_out < 0 || !d_means || !d_out) return gl_fail(ctx, GL_EINVAL, "gl_depthwed_aggregate_device: bad argument");
    if (n_out == 0) return GL_OK;
    dim3 grid((unsigned)((n_out + 31) / 32), (unsigned)((S + 31) / 32));
    {
        gl_prof_scope prof(ctx, "depthwed_kernel");
        depthwed_kernel<<<grid, 256, 0, ctx->stream>>>(d_means, S, R, reinterpret_cast<const long long*>(d_grp), n_out, d_grp ? 0 : 1,
                                                       reinterpret_cast<long long*>(d_out));
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

// int32 form (depthwed.go:103 rounds at parse time): d_depth S x R sample-major; the groups [g_begin, g_end) of d_grp (NULL:
// one row per output line) go to d_out[(g - g_begin) * S + s].  ASYNCHRONOUS on the ctx stream (gl_sync / a later
// synchronous call waits); *d_overflow (device int, zeroed by the caller) is set when a group sum does not fit int32.
int gl_depthwed_aggregate_i32_device(gl_ctx* ctx, const int32_t* d_depth, int32_t S, int64_t R, const int64_t* d_grp, int64_t g_begin,
                                     int64_t g_end, int32_t* d_out, int32_t* d_overflow) {
    GL_CHECK(gl_use(ctx));
    if (S <= 0 || R < 0 || g_begin < 0 || g_end < g_begin || !d_depth || !d_out || !d_overflow)
        return gl_fail(ctx, GL_EINVAL, "gl_depthwed_aggregate_i32_device: bad argument");
    if (g_end == g_begin) return GL_OK;
    dim3 grid((unsigned)((g_end - g_begin + 31) / 32), (unsigned)((S + 31) / 32));
    {
        gl_prof_scope prof(ctx, "depthwed_i32_kernel");
        depthwed_i32_kernel<<<grid, 256, 0, ctx->stream>>>(d_depth, S, R, reinterpret_cast<const long long*>(d_grp), g_begin, g_end, d_grp ? 0 : 1,
                                                           d_out, d_overflow);
    }
    GL_LAUNCHED(ctx, 1);
    return GL_OK;
}

// fused aggregate + all-gather over peer memory: d_dst[d] = rank d's full matrix (device pointers valid on this device:
// its own allocation and gl_ipc_open / peer-enabled pointers of the others).  ASYNCHRONOUS on the ctx stream.
int gl_depthwed_aggregate_i32_p2p(gl_ctx* ctx, const int32_t* d_depth, int32_t S, int64_t R, const int64_t* d_grp, int64_t g_begin, int64_t g_end,
                                  int32_t* const* d_dst, int32_t world, int64_t row_stride, int32_t col_off, int32_t* d_overflow) {
    GL_CHECK(gl_use(ctx));
    if (S <= 0 || R < 0 || g_begin < 0 || g_end < g_begin || !d_depth || !d_dst || world < 1 || world > 16 || row_stride < (int64_t)col_off + S || col_off < 0 || !d_overflow)
        return gl_fail(ctx, GL_EINVAL, "gl_depthwed_aggregate_i32_p2p: bad argument");
    if (g_end == g_begin) return GL_OK;
    WedPeers peers;
    for (int d = 0; d < 16; d++) peers.dst[d] = d < world ? d_dst[d] : nullptr;
    for (int d = 0; d < world; d++) if (!peers.dst[d]) return gl_fail(ctx, GL_EINVAL, "gl_depthwed_aggregate_i32_p2p: null destination %d", d);
    // 16-byte stores only where every one of them is aligned: a 4-sample group starts at a multiple of 4 ints from
    // each destination's base
    bool vec = ((row_stride | (int64_t)col_off) & 3) == 0;
    for (int d = 0; d < world; d++) vec = vec && (reinterpret_cast<uintptr_t>(peers.dst[d]) & 15) == 0;
    dim3 grid((unsigned)((g_end - g_begin + 31) / 32), (unsigned)((S + 127) / 128));
    {
        gl_prof_scope prof(ctx, "depthwed_i32_p2p_kernel");
        depthwed_i32_p2p_kernel<<<grid, 256, 0, ctx->stream>>>(d_depth, S, R, reinterpret_cast<const long long*>(d_grp), g_begin, g_end, d_grp ? 0 : 1,
                                                               peers, world, row_stride, col_off, vec ? 1 : 0, d_overflow);
    }
    GL_LAUNCHED(ctx, 1);
    return GL_OK;
}

// host form: depth S x R int32 (already int(0.5 + mean)); GL_ERANGE with *n_out set when out_cap is too small, and
// GL_ERANGE with *n_out = -1 when a group sum overflows int32 (use gl_depthwed_aggregate)
int gl_depthwed_aggregate_i32(gl_ctx* ctx, const int32_t* depth, int32_t S, int64_t R, const int32_t* starts, const int32_t* ends,
                              const int32_t* chrom_id, int64_t size, int32_t* out_start, int32_t* out_end, int32_t* out_chrom,
                              int32_t* out, int64_t out_cap, int64_t* n_out) {
    GL_CHECK(gl_use(ctx));
    if (S <= 0 || R < 0 || !depth || !starts || !ends || !chrom_id || !n_out || size <= 0)
        return gl_fail(ctx, GL_EINVAL, "gl_depthwed_aggregate_i32: bad argument");
    std::vector<int64_t> grp;
    const int64_t ng = depthwed_groups(R, starts, ends, chrom_id, size, grp);
    *n_out = ng;
    if (ng > out_cap) return gl_fail(ctx, GL_ERANGE, "gl_depthwed_aggregate_i32: %lld rows > cap %lld", (long long)ng, (long long)out_cap);
    if (ng == 0) return GL_OK;
    for (int64_t g = 0; g < ng; g++) {
        out_start[g] = starts[grp[g]];
        out_end[g] = ends[grp[g + 1] - 1];
        out_chrom[g] = chrom_id[grp[g]];
    }
    gl_scratch tmp(ctx);
    int32_t *d_depth, *d_out, *d_ovf; int64_t* d_grp;
    GL_CHECK(tmp.upload(d_depth, depth, (size_t)S * R));
    GL_CHECK(tmp.upload(d_grp, grp.data(), (size_t)ng + 1));
    GL_CHECK(tmp.alloc(d_out, (size_t)ng * S));
    GL_CHECK(tmp.alloc(d_ovf, 1));
    GL_CUDA(ctx, cudaMemsetAsync(d_ovf, 0, 4, ctx->stream));
    GL_CHECK(gl_depthwed_aggregate_i32_device(ctx, d_depth, S, R, d_grp, 0, ng, d_out, d_ovf));
    int ovf = 0;
    GL_CUDA(ctx, cudaMemcpyAsync(out, d_out, (size_t)ng * S * 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(&ovf, d_ovf, 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (ovf) { *n_out = -1; return gl_fail(ctx, GL_ERANGE, "gl_depthwed_aggregate_i32: a group sum does not fit int32"); }
    return GL_OK;
}

int gl_depthwed_aggregate(gl_ctx* ctx, const double* means, int32_t S, int64_t R, const int32_t* starts, const int32_t* ends,
                          const int32_t* chrom_id, int64_t size, int32_t* out_start, int32_t* out_end, int32_t* out_chrom,
                          int64_t* out, int64_t out_cap, int64_t* n_out) {
    GL_CHECK(gl_use(ctx));
    if (S <= 0 || R < 0 || !means || !starts || !ends || !chrom_id || !n_out || size <= 0)
        return gl_fail(ctx, GL_EINVAL, "gl_depthwed_aggregate: bad argument");
    std::vector<int64_t> grp;
    const int64_t ng = depthwed_groups(R, starts, ends, chrom_id, size, grp);
    *n_out = ng;
    if (ng > out_cap) return gl_fail(ctx, GL_ERANGE, "gl_depthwed_aggregate: %lld rows > cap %lld", (long long)ng, (long long)out_cap);
    if (ng == 0) return GL_OK;
    for (int64_t g = 0; g < ng; g++) {
        out_start[g] = starts[grp[g]];
        out_end[g] = ends[grp[g + 1] - 1];
        out_chrom[g] = chrom_id[grp[g]];
    }
    gl_scratch tmp(ctx);
    double* d_means; int64_t *d_grp, *d_out;
    GL_CHECK(tmp.upload(d_means, means, (size_t)S * R));
    GL_CHECK(tmp.upload(d_grp, grp.data(), (size_t)ng + 1));
    GL_CHECK(tmp.alloc(d_out, (size_t)ng * S));
    GL_CHECK(gl_depthwed_aggregate_device(ctx, d_means, S, R, d_grp, ng, d_out));
    GL_CUDA(ctx, cudaMemcpyAsync(out, d_out, (size_t)ng * S * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

}  // extern "C"
