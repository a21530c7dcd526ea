// dcnv.cu — `goleft dcnv` (dcnv/dcnv.go:323-354): GC-debias and median-normalise an n-sites x S-samples depth matrix.
//
// The reference, per sample column c of the matrix with its rows in GC order (inds = Go's argsort of the GC fractions,
// host/dcnv.cpp):
//   Debias (debiaser.go:98-123, Window 9, mid 5) pushes c[0..4] into a moving median of 9, then c[i+5] for i in [5, n-5),
//   and divides row i by max(median, 1) of the window after its pushes.  So c[5..9] are never pushed, and with
//   p = c[0..4] ++ c[10..n-1] row i divides by the median of p[max(0, j-8) .. j], j = clamp(i, 4, max(4, n-6)): the
//   first five rows by the median of p[0..4], the last rows by the final window.  Every window holds values that have not
//   been divided yet, so each (row, sample) is independent.  An even count (6 or 8 values, sorted rows 5 and 7 only)
//   takes (lo + hi) / 2, restating JaderDias/movingmedian (not in the reference tree: UNPINNED).
//   NormalizeBySampleMedian (dcnv.go:108-136), after Unsort: sort the column, k = its leading exact zeros (0 when a
//   value is negative), median = sorted[k + int(0.65 * float64(n - k))], every cell / median.
//
// Kernels (columns [c0, c1) of a row-major matrix with leading dimension ld; the caller streams column blocks):
//   dcnv_debias_kernel  a CTA gathers the p-rows its 64 sorted rows need x 32 samples through inds into shared memory (reads
//                       along samples are coalesced), sorts each window of <= 9 in registers, and writes x / max(med, 1) to
//                       the ORIGINAL row inds[i] (that is Unsort) plus an order-preserving key, column-major, for the select.
//   dcnv_select_kernel  a CTA per sample: zeros and negatives give the rank, then an exact 8-pass radix select over the keys.
//   dcnv_divide_kernel  every cell / its sample's median (__ddiv_rn; the library builds with --fmad=false).
//   fmt_f2_kernel       "%.2f" tokens (host/f2_token.h).
//
// `dcnv --chunk W` replaces the moving median with ChunkDebiaser.Debias (debiaser.go:125-170) over the GC-sorted rows, cut
// into chunks [ptr[j], ptr[j+1]) by gl_dcnv_chunk_slices (DESIGN §1.9): each (sample, chunk) divides by
// sorted[(len - k) / 2] of its own values (k = leading exact zeros, 0 when a value is negative) when that is > 0.
//   dcnv_chunk_keys_kernel    gathers the sorted rows through inds (a shared-memory tile, coalesced along samples) and writes
//                             their keys column-major in sorted order, so every chunk is a contiguous run of each column.
//   dcnv_chunk_select_*       the exact order statistic of every (sample, chunk), bucketed by the chunk's length: a thread
//                             sorts <= 16 keys in registers; a warp (<= 1024 rows), a 256-thread CTA (<= 65536) or a
//                             1024-thread CTA runs the 8 x 8-bit radix select, whose first pass also counts zeros and
//                             negatives.  The divisor (the median when > 0, else 1, which leaves x's bits as they are) goes
//                             to div[chunk * nc + sample].
//   dcnv_chunk_divide_kernel  x / div to the ORIGINAL row inds[i] (that is Unsort), plus the keys of the results for the
//                             sample median, which then runs as above (dcnv_select_kernel, dcnv_divide_kernel).
#include <math_constants.h>
#include "gl_common.cuh"
#include "host/f2_token.h"

namespace {

constexpr int kDbRows = 64;        // sorted rows per debias CTA
constexpr int kDbCols = 32;        // samples per debias CTA (one warp across a row)
constexpr int kDbWarps = 8;
constexpr int kSelThreads = 1024;
constexpr unsigned long long kZeroKey = 0x8000000000000000ull;

// order-preserving key of a float64 (-0 and +0 share a key: the reference compares with == 0 and <)
__device__ __forceinline__ unsigned long long f64_key(double v) {
    unsigned long long b = (unsigned long long)__double_as_longlong(v);
    if (b == kZeroKey) b = 0;
    return (b >> 63) ? ~b : (b | kZeroKey);
}

__device__ __forceinline__ double key_f64(unsigned long long k) {
    return __longlong_as_double((long long)((k >> 63) ? (k & ~kZeroKey) : ~k));
}

__device__ __forceinline__ void cas(double& a, double& b) { const double lo = fmin(a, b), hi = fmax(a, b); a = lo; b = hi; }

__global__ void __launch_bounds__(kDbCols * kDbWarps) dcnv_debias_kernel(const double* __restrict__ x, long long ld, const long long* __restrict__ inds,
                                                                       long long n, int nc, double* __restrict__ out, long long ld_out,
                                                                       unsigned long long* __restrict__ keys) {
    __shared__ double pv[kDbRows + 8][kDbCols];
    const long long i0 = (long long)blockIdx.x * kDbRows;
    const long long i1 = min(n, i0 + kDbRows) - 1;
    const long long jmax = max(4ll, n - 6);
    const long long q_lo = max(0ll, min(max(i0, 4ll), jmax) - 8);
    const long long q_hi = min(max(i1, 4ll), jmax);
    const int col = blockIdx.y * kDbCols + threadIdx.x;
    const bool ok = col < nc;
    for (long long q = q_lo + threadIdx.y; q <= q_hi; q += kDbWarps) {
        const long long sr = q < 5 ? q : q + 5;                  // p-row q is sorted row sr
        if (ok) pv[q - q_lo][threadIdx.x] = x[inds[sr] * ld + col];
    }
    __syncthreads();
    if (!ok) return;
    for (long long i = i0 + threadIdx.y; i <= i1; i += kDbWarps) {
        const long long j = min(max(i, 4ll), jmax);
        const long long lo = max(0ll, j - 8);
        const int m = (int)(j - lo + 1);                         // 5..9 values
        double w[9];
#pragma unroll
        for (int k = 0; k < 9; k++) w[k] = k < m ? pv[lo - q_lo + k][threadIdx.x] : CUDART_INF;
#pragma unroll
        for (int r = 0; r < 9; r++) {                            // odd-even transposition: 9 rounds sort 9 values
#pragma unroll
            for (int k = r & 1; k + 1 < 9; k += 2) cas(w[k], w[k + 1]);
        }
        double med;
        if (m == 9) med = w[4];
        else if (m == 8) med = __ddiv_rn(__dadd_rn(w[3], w[4]), 2.0);
        else if (m == 7) med = w[3];
        else if (m == 6) med = __ddiv_rn(__dadd_rn(w[2], w[3]), 2.0);
        else med = w[2];
        const long long row = inds[i];
        const double v = __ddiv_rn(x[row * ld + col], fmax(med, 1.0));
        out[row * ld_out + col] = v;
        keys[(long long)col * n + row] = f64_key(v);
    }
}

// medians[c] = the reference's sample median of column c; err = 1 + the first all-zero column (the reference panics there)
__global__ void __launch_bounds__(kSelThreads) dcnv_select_kernel(const unsigned long long* __restrict__ keys, long long n,
                                                                  double* __restrict__ medians, int* __restrict__ err) {
    __shared__ unsigned hist[256];
    __shared__ unsigned n_zero, n_neg;
    __shared__ unsigned long long s_prefix;
    __shared__ long long s_rank;
    const int c = blockIdx.x;
    const unsigned long long* k = keys + (long long)c * n;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) { n_zero = 0; n_neg = 0; s_prefix = 0; s_rank = 0; }
    for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0;
    __syncthreads();
    for (int shift = 56; shift >= 0; shift -= 8) {
        const unsigned long long hi_mask = shift == 56 ? 0ull : (~0ull << (shift + 8));
        const unsigned long long prefix = s_prefix;
        unsigned zeros = 0, negs = 0;
        for (long long base = 0; base < n; base += blockDim.x) {      // uniform trip count: every lane reaches the match
            const long long i = base + threadIdx.x;
            const unsigned long long key = i < n ? k[i] : 0ull;
            const bool in = i < n && (key & hi_mask) == prefix;
            if (shift == 56 && i < n) { zeros += key == kZeroKey; negs += key < kZeroKey; }
            const unsigned act = __ballot_sync(0xffffffffu, in);
            if (in) {
                const unsigned d = (unsigned)(key >> shift) & 0xffu;
                const unsigned peers = __match_any_sync(act, d);
                if (lane == __ffs(peers) - 1) atomicAdd(&hist[d], (unsigned)__popc(peers));
            }
        }
        if (shift == 56) {
            zeros = __reduce_add_sync(0xffffffffu, zeros);
            negs = __reduce_add_sync(0xffffffffu, negs);
            if (lane == 0) { atomicAdd(&n_zero, zeros); atomicAdd(&n_neg, negs); }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            long long t = s_rank;
            if (shift == 56) {                                   // dcnv.go:118-122
                const long long kz = n_neg ? 0 : (long long)n_zero;
                t = kz + (long long)__dmul_rn(0.65, (double)(n - kz));
                if (kz == n) { atomicMin(err, c + 1); t = -1; }
            }
            if (t >= 0) {
                unsigned long long cum = 0;
                int d = 0;
                for (; d < 255 && cum + hist[d] <= (unsigned long long)t; d++) cum += hist[d];
                s_prefix = prefix | ((unsigned long long)d << shift);
                t -= (long long)cum;
            }
            s_rank = t;
        }
        __syncthreads();
        if (s_rank < 0) break;                                   // all zero: nothing to select
        for (int b = threadIdx.x; b < 256; b += blockDim.x) hist[b] = 0;
        __syncthreads();
    }
    if (threadIdx.x == 0) medians[c] = s_rank < 0 ? CUDART_NAN : key_f64(s_prefix);
}

__global__ void __launch_bounds__(256) dcnv_divide_kernel(double* __restrict__ out, long long n, int nc, long long ld_out,
                                                         const double* __restrict__ medians) {
    const long long total = n * nc;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const long long r = t / nc;
        const int c = (int)(t - r * nc);
        double* p = out + r * ld_out + c;
        *p = __ddiv_rn(*p, medians[c]);
    }
}

__global__ void __launch_bounds__(256) fmt_f2_kernel(const double* __restrict__ v, long long n, uint4* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned char t[glf2::kTok];
    glf2::token(v[i], t);
    uint4 w;
    memcpy(&w, t, 16);
    out[i] = w;
}

// ---------------------------------------------------------------- dcnv --chunk
constexpr int kChThr = 16;           // chunks of <= 16 rows: one thread each
constexpr int kChWarp = 1024;        // <= 1024 rows: one warp each
constexpr int kChCta = 65536;        // <= 65536 rows: a 256-thread CTA; longer chunks a 1024-thread CTA
constexpr int kChWarpsPerCta = 8;

__device__ __forceinline__ double chunk_divisor(unsigned long long key) {
    const double m = key_f64(key);
    return m > 0 ? m : 1.0;                                      // x / 1.0 is x, bit for bit: the chunk is left as it is
}

// the sorted rows' keys, column-major: keys[c * n + i] = key of x[inds[i], c]
__global__ void __launch_bounds__(kDbCols * kDbWarps) dcnv_chunk_keys_kernel(const double* __restrict__ x, long long ld, const long long* __restrict__ inds,
                                                                           long long n, int nc, unsigned long long* __restrict__ keys) {
    __shared__ double tile[kDbRows][kDbCols + 1];
    const long long i0 = (long long)blockIdx.x * kDbRows;
    const int col = blockIdx.y * kDbCols + threadIdx.x;
    for (int r = threadIdx.y; r < kDbRows; r += kDbWarps)
        if (col < nc && i0 + r < n) tile[r][threadIdx.x] = x[inds[i0 + r] * ld + col];
    __syncthreads();
    for (int c = threadIdx.y; c < kDbCols && blockIdx.y * kDbCols + c < nc; c += kDbWarps)
        for (int r = threadIdx.x; r < kDbRows; r += 32)
            if (i0 + r < n) keys[(long long)(blockIdx.y * kDbCols + c) * n + i0 + r] = f64_key(tile[r][c]);
}

// one thread per (sample, chunk of <= kChThr rows): a bitonic network over the keys padded with ~0 (above every finite key)
__global__ void __launch_bounds__(256) dcnv_chunk_select_thread_kernel(const unsigned long long* __restrict__ keys, long long n,
                                                                       const long long* __restrict__ ptr, const int* __restrict__ tasks,
                                                                       long long n_tasks, int nc, double* __restrict__ div) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_tasks * nc) return;
    const int col = (int)(t / n_tasks);
    const int ch = tasks[t - (long long)col * n_tasks];
    const long long a = ptr[ch];
    const int len = (int)(ptr[ch + 1] - a);
    const unsigned long long* k = keys + (long long)col * n + a;
    unsigned long long v[kChThr];
    int zeros = 0, negs = 0;
#pragma unroll
    for (int j = 0; j < kChThr; j++) {
        v[j] = j < len ? k[j] : ~0ull;
        zeros += v[j] == kZeroKey;
        negs += v[j] < kZeroKey;
    }
#pragma unroll
    for (int size = 2; size <= kChThr; size <<= 1) {
#pragma unroll
        for (int stride = size / 2; stride > 0; stride >>= 1) {
#pragma unroll
            for (int i = 0; i < kChThr; i++) {
                const int l = i ^ stride;
                if (l > i) {
                    const unsigned long long lo = min(v[i], v[l]), hi = max(v[i], v[l]);
                    const bool up = (i & size) == 0;
                    v[i] = up ? lo : hi;
                    v[l] = up ? hi : lo;
                }
            }
        }
    }
    const int r = (len - (negs ? 0 : zeros)) / 2;                // debiaser.go:160-163: the index is into the whole chunk
    unsigned long long m = v[0];
#pragma unroll
    for (int j = 1; j < kChThr; j++) if (j == r) m = v[j];
    div[(long long)ch * nc + col] = chunk_divisor(m);
}

struct ChunkSel {
    unsigned hist[256];
    unsigned n_zero, n_neg;
    unsigned long long prefix;
    long long rank;
};

// the key of sorted[(len - k) / 2] of k[0, len), by a group of B threads (B = 32: one warp; else the whole CTA), t = the
// thread's index in the group.  The 8 x 8-bit passes of dcnv_select_kernel; one warp scans the histogram (8 bins a lane).
template <int B>
__device__ unsigned long long chunk_group_select(const unsigned long long* __restrict__ k, long long len, ChunkSel& s, int t) {
    const int lane = threadIdx.x & 31;
    auto sync = [] { if (B == 32) __syncwarp(); else __syncthreads(); };
    if (t == 0) { s.n_zero = 0; s.n_neg = 0; s.prefix = 0; s.rank = 0; }
    for (int b = t; b < 256; b += B) s.hist[b] = 0;
    sync();
    for (int shift = 56; shift >= 0; shift -= 8) {
        const unsigned long long hi_mask = shift == 56 ? 0ull : (~0ull << (shift + 8));
        const unsigned long long prefix = s.prefix;
        unsigned zeros = 0, negs = 0;
        for (long long base = 0; base < len; base += B) {        // uniform trip count: every lane reaches the match
            const long long i = base + t;
            const unsigned long long key = i < len ? k[i] : 0ull;
            const bool in = i < len && (key & hi_mask) == prefix;
            if (shift == 56 && i < len) { zeros += key == kZeroKey; negs += key < kZeroKey; }
            const unsigned act = __ballot_sync(0xffffffffu, in);
            if (in) {
                const unsigned d = (unsigned)(key >> shift) & 0xffu;
                const unsigned peers = __match_any_sync(act, d);
                if (lane == __ffs(peers) - 1) atomicAdd(&s.hist[d], (unsigned)__popc(peers));
            }
        }
        if (shift == 56) {
            zeros = __reduce_add_sync(0xffffffffu, zeros);
            negs = __reduce_add_sync(0xffffffffu, negs);
            if (lane == 0) { atomicAdd(&s.n_zero, zeros); atomicAdd(&s.n_neg, negs); }
        }
        sync();
        if (t < 32) {
            long long r = s.rank;
            if (shift == 56) r = (len - (s.n_neg ? 0 : (long long)s.n_zero)) / 2;
            unsigned h[8], sum = 0;
#pragma unroll
            for (int j = 0; j < 8; j++) { h[j] = s.hist[8 * lane + j]; sum += h[j]; }
            unsigned inc = sum;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned u = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += u;
            }
            long long cum = inc - sum;
            if (cum <= r && r < (long long)inc) {                // exactly one lane: the candidates outnumber the rank
                int d = 8 * lane;
#pragma unroll
                for (int j = 0; j < 7; j++)
                    if (d == 8 * lane + j && cum + h[j] <= r) { cum += h[j]; d++; }
                s.prefix = prefix | ((unsigned long long)d << shift);
                s.rank = r - cum;
            }
        }
        sync();
        for (int b = t; b < 256; b += B) s.hist[b] = 0;
        sync();
    }
    return s.prefix;
}

// one warp per (sample, chunk of kChThr + 1 .. kChWarp rows)
__global__ void __launch_bounds__(32 * kChWarpsPerCta) dcnv_chunk_select_warp_kernel(const unsigned long long* __restrict__ keys, long long n,
                                                                                     const long long* __restrict__ ptr, const int* __restrict__ tasks,
                                                                                     long long n_tasks, int nc, double* __restrict__ div) {
    __shared__ ChunkSel sel[kChWarpsPerCta];
    const int w = threadIdx.x >> 5;
    const long long t = (long long)blockIdx.x * kChWarpsPerCta + w;
    if (t >= n_tasks * nc) return;                               // whole warps: the select syncs a warp only
    const int col = (int)(t / n_tasks);
    const int ch = tasks[t - (long long)col * n_tasks];
    const long long a = ptr[ch];
    const unsigned long long m = chunk_group_select<32>(keys + (long long)col * n + a, ptr[ch + 1] - a, sel[w], threadIdx.x & 31);
    if ((threadIdx.x & 31) == 0) div[(long long)ch * nc + col] = chunk_divisor(m);
}

// one B-thread CTA per (sample, chunk)
template <int B>
__global__ void __launch_bounds__(B, 1) dcnv_chunk_select_cta_kernel(const unsigned long long* __restrict__ keys, long long n,
                                                                  const long long* __restrict__ ptr, const int* __restrict__ tasks,
                                                                  long long n_tasks, int nc, double* __restrict__ div) {
    __shared__ ChunkSel sel;
    const long long t = blockIdx.x;
    const int col = (int)(t / n_tasks);
    const int ch = tasks[t - (long long)col * n_tasks];
    const long long a = ptr[ch];
    const unsigned long long m = chunk_group_select<B>(keys + (long long)col * n + a, ptr[ch + 1] - a, sel, threadIdx.x);
    if (threadIdx.x == 0) div[(long long)ch * nc + col] = chunk_divisor(m);
}

// sorted row i of every sample / its chunk's divisor, written to row inds[i]; keys[c * n + i] = the result's key
__global__ void __launch_bounds__(kDbCols * kDbWarps) dcnv_chunk_divide_kernel(const double* __restrict__ x, long long ld, const long long* __restrict__ inds,
                                                                             long long n, int nc, const long long* __restrict__ ptr, int n_chunks,
                                                                             const double* __restrict__ div, double* __restrict__ out, long long ld_out,
                                                                             unsigned long long* __restrict__ keys) {
    __shared__ double tile[kDbRows][kDbCols + 1];
    __shared__ int s_ch[kDbRows];
    const long long i0 = (long long)blockIdx.x * kDbRows;
    const int tid = threadIdx.y * kDbCols + threadIdx.x;
    if (tid < kDbRows && i0 + tid < n) {                         // the chunk of sorted row i0 + tid: last j with ptr[j] <= i
        const long long i = i0 + tid;
        int lo = 0, hi = n_chunks - 1;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (ptr[mid] <= i) lo = mid; else hi = mid - 1;
        }
        s_ch[tid] = lo;
    }
    __syncthreads();
    const int col = blockIdx.y * kDbCols + threadIdx.x;
    for (int r = threadIdx.y; r < kDbRows; r += kDbWarps) {
        if (col >= nc || i0 + r >= n) continue;
        const long long row = inds[i0 + r];
        const double v = __ddiv_rn(x[row * ld + col], div[(long long)s_ch[r] * nc + col]);
        out[row * ld_out + col] = v;
        tile[r][threadIdx.x] = v;
    }
    __syncthreads();
    for (int c = threadIdx.y; c < kDbCols && blockIdx.y * kDbCols + c < nc; c += kDbWarps)
        for (int r = threadIdx.x; r < kDbRows; r += 32)
            if (i0 + r < n) keys[(long long)(blockIdx.y * kDbCols + c) * n + i0 + r] = f64_key(tile[r][c]);
}

// the chunks on the device: ptr (n_chunks + 1 offsets) and the chunk numbers of each length bucket, concatenated
struct ChunkPlan {
    const long long* d_ptr = nullptr;
    const int* d_tasks = nullptr;
    int n_chunks = 0;
    long long off[5] = {};                                       // bucket b is d_tasks[off[b], off[b + 1])
};

// checks chunk_ptr (host) and buckets its chunks by length
int chunk_buckets(gl_ctx* ctx, const char* fn, const int64_t* chunk_ptr, int64_t n_chunks, int64_t n, std::vector<int>& tasks, long long off[5]) {
    if (!chunk_ptr || n_chunks < 1 || n_chunks > n || chunk_ptr[0] != 0 || chunk_ptr[n_chunks] != n)
        return gl_fail(ctx, GL_EINVAL, "%s: chunk_ptr must run from 0 to n in 1 .. n chunks", fn);
    for (int64_t j = 0; j < n_chunks; j++)
        if (chunk_ptr[j + 1] <= chunk_ptr[j]) return gl_fail(ctx, GL_EINVAL, "%s: chunk %lld is empty or reversed", fn, (long long)j);
    const int64_t lim[4] = {kChThr, kChWarp, kChCta, INT64_MAX};
    tasks.clear();
    tasks.reserve((size_t)n_chunks);
    for (int b = 0; b < 4; b++) {
        off[b] = (long long)tasks.size();
        for (int64_t j = 0; j < n_chunks; j++) {
            const int64_t len = chunk_ptr[j + 1] - chunk_ptr[j];
            if (len <= lim[b] && (b == 0 || len > lim[b - 1])) tasks.push_back((int)j);
        }
    }
    off[4] = (long long)tasks.size();
    return GL_OK;
}

// select + divide by the sample medians over the keys of d_out's columns [0, nc); checks the error flag
int sample_normalize(gl_ctx* ctx, const unsigned long long* d_keys, int64_t n, int nc, double* d_out, int64_t ld_out, double* d_medians,
                     int* d_err, int64_t col_name) {
    {
        gl_prof_scope prof(ctx, "dcnv_select_kernel");
        dcnv_select_kernel<<<(unsigned)nc, kSelThreads, 0, ctx->stream>>>(d_keys, (long long)n, d_medians, d_err);
    }
    GL_LAUNCHED(ctx, 1);
    {
        gl_prof_scope prof(ctx, "dcnv_divide_kernel");
        const long long total = (long long)n * nc;
        const unsigned blocks = (unsigned)std::min<long long>((total + 255) / 256, (long long)ctx->sm_count * 16);
        dcnv_divide_kernel<<<blocks, 256, 0, ctx->stream>>>(d_out, (long long)n, nc, (long long)ld_out, d_medians);
    }
    GL_LAUNCHED(ctx, 1);
    int err = 0;
    GL_CUDA(ctx, cudaMemcpyAsync(&err, d_err, sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (err != 0x7f7f7f7f)
        return gl_fail(ctx, GL_ERANGE, "dcnv: sample column %lld is all zero (the reference's median index is out of range)", (long long)(col_name + err - 1));
    return GL_OK;
}

// the chunk debias and the sample median over columns [c0, c1) of d_x (arguments checked by the caller)
int chunked_block(gl_ctx* ctx, const double* d_x, int64_t n, int64_t ld, const int64_t* d_inds, const ChunkPlan& P, int32_t c0, int32_t c1,
                  double* d_out, int64_t ld_out, double* d_medians, int64_t col_name) {
    const int nc = c1 - c0;
    gl_scratch tmp(ctx);
    unsigned long long* d_keys; int* d_err; double* d_div;
    GL_CHECK(tmp.alloc(d_keys, (size_t)n * nc));
    GL_CHECK(tmp.alloc(d_div, (size_t)P.n_chunks * nc));
    GL_CHECK(tmp.alloc(d_err, 1));
    GL_CUDA(ctx, cudaMemsetAsync(d_err, 0x7f, sizeof(int), ctx->stream));
    const long long* inds = reinterpret_cast<const long long*>(d_inds);
    const dim3 tiles((unsigned)((n + kDbRows - 1) / kDbRows), (unsigned)((nc + kDbCols - 1) / kDbCols));
    {
        gl_prof_scope prof(ctx, "dcnv_chunk_keys_kernel");
        dcnv_chunk_keys_kernel<<<tiles, dim3(kDbCols, kDbWarps), 0, ctx->stream>>>(d_x + c0, (long long)ld, inds, (long long)n, nc, d_keys);
    }
    GL_LAUNCHED(ctx, 1);
    for (int b = 0; b < 4; b++) {
        const long long nt = P.off[b + 1] - P.off[b];
        if (nt == 0) continue;
        const int* tasks = P.d_tasks + P.off[b];
        const long long work = nt * nc;
        if (b == 0) {
            gl_prof_scope prof(ctx, "dcnv_chunk_select_thread_kernel");
            dcnv_chunk_select_thread_kernel<<<(unsigned)((work + 255) / 256), 256, 0, ctx->stream>>>(d_keys, (long long)n, P.d_ptr, tasks, nt, nc, d_div);
        } else if (b == 1) {
            gl_prof_scope prof(ctx, "dcnv_chunk_select_warp_kernel");
            dcnv_chunk_select_warp_kernel<<<(unsigned)((work + kChWarpsPerCta - 1) / kChWarpsPerCta), 32 * kChWarpsPerCta, 0, ctx->stream>>>(
                d_keys, (long long)n, P.d_ptr, tasks, nt, nc, d_div);
        } else if (b == 2) {
            gl_prof_scope prof(ctx, "dcnv_chunk_select_cta_kernel<256>");
            dcnv_chunk_select_cta_kernel<256><<<(unsigned)work, 256, 0, ctx->stream>>>(d_keys, (long long)n, P.d_ptr, tasks, nt, nc, d_div);
        } else {
            gl_prof_scope prof(ctx, "dcnv_chunk_select_cta_kernel<1024>");
            dcnv_chunk_select_cta_kernel<1024><<<(unsigned)work, 1024, 0, ctx->stream>>>(d_keys, (long long)n, P.d_ptr, tasks, nt, nc, d_div);
        }
        GL_LAUNCHED(ctx, 1);
    }
    {
        gl_prof_scope prof(ctx, "dcnv_chunk_divide_kernel");
        dcnv_chunk_divide_kernel<<<tiles, dim3(kDbCols, kDbWarps), 0, ctx->stream>>>(d_x + c0, (long long)ld, inds, (long long)n, nc, P.d_ptr,
                                                                                   P.n_chunks, d_div, d_out, (long long)ld_out, d_keys);
    }
    GL_LAUNCHED(ctx, 1);
    return sample_normalize(ctx, d_keys, n, nc, d_out, ld_out, d_medians, d_err, col_name);
}

// the three kernels over columns [c0, c1) of d_x (arguments checked by the caller); an all-zero column is reported as
// column col_name + (its index in the block)
int normalize_block(gl_ctx* ctx, const double* d_x, int64_t n, int64_t ld, const int64_t* d_inds, int32_t c0, int32_t c1,
                    double* d_out, int64_t ld_out, double* d_medians, int64_t col_name) {
    const int nc = c1 - c0;
    gl_scratch tmp(ctx);
    unsigned long long* d_keys; int* d_err;
    GL_CHECK(tmp.alloc(d_keys, (size_t)n * nc));
    GL_CHECK(tmp.alloc(d_err, 1));
    GL_CUDA(ctx, cudaMemsetAsync(d_err, 0x7f, sizeof(int), ctx->stream));
    {
        gl_prof_scope prof(ctx, "dcnv_debias_kernel");
        const dim3 grid((unsigned)((n + kDbRows - 1) / kDbRows), (unsigned)((nc + kDbCols - 1) / kDbCols));
        dcnv_debias_kernel<<<grid, dim3(kDbCols, kDbWarps), 0, ctx->stream>>>(d_x + c0, (long long)ld, reinterpret_cast<const long long*>(d_inds),
                                                                             (long long)n, nc, d_out, (long long)ld_out, d_keys);
    }
    GL_LAUNCHED(ctx, 1);
    return sample_normalize(ctx, d_keys, n, nc, d_out, ld_out, d_medians, d_err, col_name);
}

}  // namespace

extern "C" {

int gl_dcnv_normalize_device(gl_ctx* ctx, const double* d_x, int64_t n, int64_t ld, const int64_t* d_inds, int32_t c0, int32_t c1,
                             double* d_out, int64_t ld_out, double* d_medians) {
    GL_CHECK(gl_use(ctx));
    if (!d_x || !d_inds || !d_out || !d_medians || c0 < 0 || c1 <= c0 || ld < c1 || ld_out < c1 - c0)
        return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize_device: bad argument");
    if (n < 5) return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize_device: %lld rows; the moving median needs at least 5", (long long)n);
    if (n > INT32_MAX) return gl_fail(ctx, GL_ERANGE, "gl_dcnv_normalize_device: more than 2^31-1 rows");
    return normalize_block(ctx, d_x, n, ld, d_inds, c0, c1, d_out, ld_out, d_medians, c0);
}

int gl_dcnv_normalize(gl_ctx* ctx, const double* x, int64_t n, int64_t ld, const int64_t* inds, int32_t c0, int32_t c1, int32_t block_cols,
                      double* out, int64_t ld_out, double* medians) {
    GL_CHECK(gl_use(ctx));
    const int nc = c1 - c0;
    if (!x || !inds || !out || !medians || c0 < 0 || nc < 1 || ld < c1 || ld_out < nc || block_cols < 0)
        return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize: bad argument");
    if (n < 5) return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize: %lld rows; the moving median needs at least 5", (long long)n);
    if (n > INT32_MAX) return gl_fail(ctx, GL_ERANGE, "gl_dcnv_normalize: more than 2^31-1 rows");
    {                                                            // the kernels gather through inds: it must be a permutation
        std::vector<uint8_t> seen((size_t)n, 0);
        for (int64_t i = 0; i < n; i++) {
            if (inds[i] < 0 || inds[i] >= n || seen[(size_t)inds[i]]) return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize: inds is not a permutation of [0, n)");
            seen[(size_t)inds[i]] = 1;
        }
    }
    int bw = block_cols;
    if (bw == 0) {                                               // a block's input, output and keys: 24 bytes per cell
        size_t free_b = 0, total_b = 0;
        GL_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
        const double room = 0.8 * (double)free_b - 8.0 * (double)n;
        bw = (int)std::min<double>((double)nc, room / (24.0 * (double)n));
        if (bw < 1) return gl_fail(ctx, GL_ENOMEM, "gl_dcnv_normalize: one sample column of %lld rows does not fit in device memory", (long long)n);
    }
    bw = std::min(bw, nc);
    gl_scratch tmp(ctx);
    int64_t* d_inds; double *d_x, *d_out, *d_med;
    GL_CHECK(tmp.upload(d_inds, inds, (size_t)n));
    GL_CHECK(tmp.alloc(d_x, (size_t)n * bw));
    GL_CHECK(tmp.alloc(d_out, (size_t)n * bw));
    GL_CHECK(tmp.alloc(d_med, (size_t)bw));
    for (int b0 = c0; b0 < c1; b0 += bw) {
        const int nb = std::min(bw, c1 - b0);
        GL_CUDA(ctx, cudaMemcpy2DAsync(d_x, (size_t)nb * 8, x + b0, (size_t)ld * 8, (size_t)nb * 8, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        GL_CHECK(normalize_block(ctx, d_x, n, nb, d_inds, 0, nb, d_out, nb, d_med, b0));
        GL_CUDA(ctx, cudaMemcpy2DAsync(out + (b0 - c0), (size_t)ld_out * 8, d_out, (size_t)nb * 8, (size_t)nb * 8, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaMemcpyAsync(medians + (b0 - c0), d_med, (size_t)nb * 8, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return GL_OK;
}

int gl_dcnv_normalize_chunked_device(gl_ctx* ctx, const double* d_x, int64_t n, int64_t ld, const int64_t* d_inds, const int64_t* chunk_ptr,
                                     int64_t n_chunks, int32_t c0, int32_t c1, double* d_out, int64_t ld_out, double* d_medians) {
    GL_CHECK(gl_use(ctx));
    if (!d_x || !d_inds || !d_out || !d_medians || c0 < 0 || c1 <= c0 || ld < c1 || ld_out < c1 - c0 || n < 1)
        return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize_chunked_device: bad argument");
    if (n > INT32_MAX) return gl_fail(ctx, GL_ERANGE, "gl_dcnv_normalize_chunked_device: more than 2^31-1 rows");
    std::vector<int> tasks;
    ChunkPlan P;
    GL_CHECK(chunk_buckets(ctx, "gl_dcnv_normalize_chunked_device", chunk_ptr, n_chunks, n, tasks, P.off));
    gl_scratch tmp(ctx);
    int64_t* d_ptr; int* d_tasks;
    GL_CHECK(tmp.upload(d_ptr, chunk_ptr, (size_t)n_chunks + 1));
    GL_CHECK(tmp.upload(d_tasks, tasks.data(), tasks.size()));
    P.d_ptr = reinterpret_cast<const long long*>(d_ptr);
    P.d_tasks = d_tasks;
    P.n_chunks = (int)n_chunks;
    return chunked_block(ctx, d_x, n, ld, d_inds, P, c0, c1, d_out, ld_out, d_medians, c0);
}

int gl_dcnv_normalize_chunked(gl_ctx* ctx, const double* x, int64_t n, int64_t ld, const int64_t* inds, const int64_t* chunk_ptr, int64_t n_chunks,
                              int32_t c0, int32_t c1, int32_t block_cols, double* out, int64_t ld_out, double* medians) {
    GL_CHECK(gl_use(ctx));
    const int nc = c1 - c0;
    if (!x || !inds || !out || !medians || c0 < 0 || nc < 1 || ld < c1 || ld_out < nc || block_cols < 0 || n < 1)
        return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize_chunked: bad argument");
    if (n > INT32_MAX) return gl_fail(ctx, GL_ERANGE, "gl_dcnv_normalize_chunked: more than 2^31-1 rows");
    {                                                            // the kernels gather through inds: it must be a permutation
        std::vector<uint8_t> seen((size_t)n, 0);
        for (int64_t i = 0; i < n; i++) {
            if (inds[i] < 0 || inds[i] >= n || seen[(size_t)inds[i]]) return gl_fail(ctx, GL_EINVAL, "gl_dcnv_normalize_chunked: inds is not a permutation of [0, n)");
            seen[(size_t)inds[i]] = 1;
        }
    }
    std::vector<int> tasks;
    ChunkPlan P;
    GL_CHECK(chunk_buckets(ctx, "gl_dcnv_normalize_chunked", chunk_ptr, n_chunks, n, tasks, P.off));
    int bw = block_cols;
    if (bw == 0) {                                               // a block's input, output, keys and chunk divisors
        size_t free_b = 0, total_b = 0;
        GL_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
        const double room = 0.8 * (double)free_b - 8.0 * (double)n - 12.0 * (double)(n_chunks + 1);
        bw = (int)std::min<double>((double)nc, room / (24.0 * (double)n + 8.0 * (double)n_chunks));
        if (bw < 1) return gl_fail(ctx, GL_ENOMEM, "gl_dcnv_normalize_chunked: one sample column of %lld rows does not fit in device memory", (long long)n);
    }
    bw = std::min(bw, nc);
    gl_scratch tmp(ctx);
    int64_t *d_inds, *d_ptr; int* d_tasks; double *d_x, *d_out, *d_med;
    GL_CHECK(tmp.upload(d_inds, inds, (size_t)n));
    GL_CHECK(tmp.upload(d_ptr, chunk_ptr, (size_t)n_chunks + 1));
    GL_CHECK(tmp.upload(d_tasks, tasks.data(), tasks.size()));
    GL_CHECK(tmp.alloc(d_x, (size_t)n * bw));
    GL_CHECK(tmp.alloc(d_out, (size_t)n * bw));
    GL_CHECK(tmp.alloc(d_med, (size_t)bw));
    P.d_ptr = reinterpret_cast<const long long*>(d_ptr);
    P.d_tasks = d_tasks;
    P.n_chunks = (int)n_chunks;
    for (int b0 = c0; b0 < c1; b0 += bw) {
        const int nb = std::min(bw, c1 - b0);
        GL_CUDA(ctx, cudaMemcpy2DAsync(d_x, (size_t)nb * 8, x + b0, (size_t)ld * 8, (size_t)nb * 8, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        GL_CHECK(chunked_block(ctx, d_x, n, nb, d_inds, P, 0, nb, d_out, nb, d_med, b0));
        GL_CUDA(ctx, cudaMemcpy2DAsync(out + (b0 - c0), (size_t)ld_out * 8, d_out, (size_t)nb * 8, (size_t)nb * 8, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaMemcpyAsync(medians + (b0 - c0), d_med, (size_t)nb * 8, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return GL_OK;
}

int gl_format_f2_device(gl_ctx* ctx, const double* d_vals, int64_t n, uint8_t* d_tokens) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || (n > 0 && (!d_vals || !d_tokens)) || ((uintptr_t)d_tokens & 15)) return gl_fail(ctx, GL_EINVAL, "gl_format_f2_device: bad argument");
    if (n == 0) return GL_OK;
    {
        gl_prof_scope prof(ctx, "fmt_f2_kernel");
        fmt_f2_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_vals, (long long)n, reinterpret_cast<uint4*>(d_tokens));
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_format_f2(gl_ctx* ctx, const double* vals, int64_t n, uint8_t* tokens) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || (n > 0 && (!vals || !tokens))) return gl_fail(ctx, GL_EINVAL, "gl_format_f2: bad argument");
    if (n == 0) return GL_OK;
    gl_scratch tmp(ctx);
    double* d_vals; uint8_t* d_tokens;
    GL_CHECK(tmp.upload(d_vals, vals, (size_t)n));
    GL_CHECK(tmp.alloc(d_tokens, (size_t)n * glf2::kTok));
    GL_CHECK(gl_format_f2_device(ctx, d_vals, n, d_tokens));
    GL_CUDA(ctx, cudaMemcpyAsync(tokens, d_tokens, (size_t)n * glf2::kTok, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

}  // extern "C"
