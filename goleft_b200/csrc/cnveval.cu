// cnveval.cu — `goleft cnveval` (cnveval/cnveval.go Evaluate, updatePositive, updateFP): TP / FP / FN / TN of a set of
// CNV calls against a truth set, per sample and size class.  DESIGN §1.12.
//
// The reference walks each sample's sorted calls with a shared pointer and two flags that are never reset; its counts equal
// an order-free form (DESIGN §1.12) built from three positions in the sample's call order: min Q(t), the first call that
// qualifies against truth t; k_tp, the first qualifying call that also qualifies against a truth the sample carries; and
// b(t), the first call past t.  Each is a binary search plus a short scan here, because every sample's calls are grouped in
// Go's sort.Slice order and carry the prefix maximum of End within each (sample, chrom) run.
//   prep       one thread per sample: checks the call layout and builds that prefix maximum (and the same for the sample's
//              carried truths); one thread per truth checks the truths
//   bitset     one thread per membership entry: bit (s, t) of a sample-major bitset
//   tp_any     one thread per call: does some truth the sample carries qualify against it
//   own        one thread per membership entry: TP or FN in the truth's class; marks min Q(t) counted
//   uncounted  one thread per call: FP in the call's own class when it was not counted
//   others     (sample) x (tile of 2048 truths): the sample's calls staged in shared memory (read from global memory when
//              there are more than kSmemCalls), a truth the sample does not carry gives TN, or FP = min(k_tp, b) - min Q;
//              per-class sums reduced in the CTA before one 64-bit atomic each
#include <math.h>
#include <string.h>
#include <cmath>
#include "gl_common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kTileTruths = 2048;                 // truths per CTA of the others pass
constexpr int kSmemCalls = 1024;                  // calls one CTA stages in shared memory (37 KB)
constexpr long long kMaxCoord = 1ll << 62;        // coordinates lie in [0, 2^62): lengths and overlaps fit int64
enum { kTP = 0, kFP = 1, kFN = 2, kTN = 3 };

// sizeClass (cnveval.go:343-352)
__device__ __forceinline__ int size_class(long long s, long long e) {
    const long long l = e - s;
    return l < 20000 ? 0 : (l < 100000 ? 1 : 2);
}

// sameCN (cnveval.go:354-362)
__device__ __forceinline__ long long cn_key(long long cn) { return cn > 2 ? 3 : cn; }

// poverlap(a, b) >= po && sameCN(a.CN, b.CN) for two intervals on one chromosome, in Go's float64 arithmetic
// (cnveval.go:378-389): an IEEE division compared with po, no integer shortcut (it would disagree at ties)
__device__ __forceinline__ bool qualifies(long long as, long long ae, long long acn, long long bs, long long be, long long bcn,
                                          double po) {
    const double total = fmin((double)(ae - as), (double)(be - bs));
    const long long ovl = min(ae, be) - max(as, bs);
    const double r = ovl < 0 ? 0.0 : (double)ovl / total;
    return r >= po && cn_key(acn) == cn_key(bcn);
}

// one sample's calls, in its sort.Slice order
struct Calls {
    const int* chrom;
    const long long *start, *end, *pmax, *cn;
    const uint8_t* tp;
};

// b: the first call past (chr, te) (a greater chrom, or chr with Start > te); *k0: the first call on chr whose prefix-maximum
// End exceeds ts.  Every call that can overlap [ts, te) on chr lies in [k0, b).
__device__ __forceinline__ long long window(const Calls& c, long long n, int chr, long long ts, long long te, long long& k0) {
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long m = (lo + hi) >> 1;
        if (c.chrom[m] < chr) lo = m + 1; else hi = m;
    }
    const long long r0 = lo;
    hi = n;
    while (lo < hi) {
        const long long m = (lo + hi) >> 1;
        if (c.chrom[m] == chr && c.start[m] <= te) lo = m + 1; else hi = m;
    }
    const long long b = lo;
    lo = r0; hi = b;
    while (lo < hi) {
        const long long m = (lo + hi) >> 1;
        if (c.pmax[m] <= ts) lo = m + 1; else hi = m;
    }
    k0 = lo;
    return b;
}

// min Q(t) in [k0, b), or b
__device__ __forceinline__ long long first_q(const Calls& c, long long k0, long long b, long long ts, long long te, long long tcn,
                                             double po) {
    for (long long k = k0; k < b; k++)
        if (qualifies(c.start[k], c.end[k], c.cn[k], ts, te, tcn, po)) return k;
    return b;
}

// the index i with ptr[i] <= x < ptr[i + 1]
__device__ __forceinline__ int owner(const long long* ptr, int S, long long x) {
    int lo = 0, hi = S;
    while (lo < hi) {
        const int m = (lo + hi + 1) >> 1;
        if (ptr[m] <= x) lo = m; else hi = m - 1;
    }
    return lo;
}

__device__ __forceinline__ void flag(unsigned long long* err, long long x) { atomicMin(err, (unsigned long long)x); }

// per sample: the calls' offsets, ranges and (chrom, start) order, and their prefix-maximum End per chrom run
__global__ void prep_calls_kernel(int S, const long long* __restrict__ ptr, long long n_calls, const int* __restrict__ chrom,
                                  const long long* __restrict__ start, const long long* __restrict__ end,
                                  long long* __restrict__ pmax, unsigned long long* err) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const long long a = ptr[s], z = ptr[s + 1];
    if ((s == 0 && a != 0) || (s == S - 1 && z != n_calls) || z < a || a < 0 || z > n_calls) { flag(&err[3], s); return; }
    long long m = 0;
    for (long long k = a; k < z; k++) {
        const int c = chrom[k];
        const long long b = start[k], e = end[k];
        if (c < 0 || b < 0 || e < b || e >= kMaxCoord) { flag(&err[0], k); return; }
        if (k > a && (c < chrom[k - 1] || (c == chrom[k - 1] && b < start[k - 1]))) { flag(&err[0], k); return; }
        m = (k == a || c != chrom[k - 1]) ? e : max(m, e);
        pmax[k] = m;
    }
}

__global__ void check_truths_kernel(long long T, const int* __restrict__ chrom, const long long* __restrict__ start,
                                    const long long* __restrict__ end, unsigned long long* err) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    const int c = chrom[t];
    const long long b = start[t], e = end[t];
    if (c < 0 || b < 0 || e < b || e >= kMaxCoord) flag(&err[1], t);
    else if (t > 0 && (c < chrom[t - 1] || (c == chrom[t - 1] && b < start[t - 1]))) flag(&err[1], t);
}

// per sample: its carried truths (ascending truth indices) and their prefix-maximum End per chrom run
__global__ void prep_members_kernel(int S, const long long* __restrict__ ptr, long long n_mem, const long long* __restrict__ truth,
                                    long long T, const int* __restrict__ chrom, const long long* __restrict__ end,
                                    long long* __restrict__ pmax, unsigned long long* err) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const long long a = ptr[s], z = ptr[s + 1];
    if ((s == 0 && a != 0) || (s == S - 1 && z != n_mem) || z < a || a < 0 || z > n_mem) { flag(&err[3], (long long)S + s); return; }
    long long m = 0;
    for (long long k = a; k < z; k++) {
        const long long t = truth[k];
        if (t < 0 || t >= T || (k > a && t < truth[k - 1])) { flag(&err[2], k); return; }
        m = (k == a || chrom[t] != chrom[truth[k - 1]]) ? end[t] : max(m, end[t]);
        pmax[k] = m;
    }
}

__global__ void bitset_kernel(int S, const long long* __restrict__ ptr, long long n_mem, const long long* __restrict__ truth,
                              long long W, unsigned* __restrict__ bits) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_mem) return;
    const int s = owner(ptr, S, k);
    const long long t = truth[k];
    atomicOr(&bits[(long long)s * W + (t >> 5)], 1u << (t & 31));
}

// tp_any[k]: some truth the call's sample carries qualifies against call k (the reference's tpfound test, cnveval.go:263-271)
__global__ void tp_any_kernel(int S, const long long* __restrict__ c_ptr, long long n_calls, const int* __restrict__ c_chrom,
                              const long long* __restrict__ c_start, const long long* __restrict__ c_end,
                              const long long* __restrict__ c_cn, const long long* __restrict__ m_ptr,
                              const long long* __restrict__ m_truth, const long long* __restrict__ m_pmax,
                              const int* __restrict__ t_chrom, const long long* __restrict__ t_start,
                              const long long* __restrict__ t_end, const long long* __restrict__ t_cn, double po,
                              uint8_t* __restrict__ tp) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_calls) return;
    const int s = owner(c_ptr, S, k);
    const int chr = c_chrom[k];
    const long long cs = c_start[k], ce = c_end[k], ccn = c_cn[k];
    long long lo = m_ptr[s], hi = m_ptr[s + 1];
    const long long z = hi;
    while (lo < hi) {
        const long long m = (lo + hi) >> 1;
        if (t_chrom[m_truth[m]] < chr) lo = m + 1; else hi = m;
    }
    long long r = lo;
    hi = z;
    while (lo < hi) {                                            // the run's prefix maximum is non-decreasing until chr ends
        const long long m = (lo + hi) >> 1;
        if (t_chrom[m_truth[m]] == chr && m_pmax[m] <= cs) lo = m + 1; else hi = m;
    }
    uint8_t any = 0;
    for (r = lo; r < z; r++) {
        const long long t = m_truth[r];
        if (t_chrom[t] != chr || t_start[t] >= ce) break;          // starts ascend: nothing further can overlap
        if (qualifies(cs, ce, ccn, t_start[t], t_end[t], t_cn[t], po)) { any = 1; break; }
    }
    tp[k] = any;
}

// updatePositive's truths loop (cnveval.go:294-329): one membership entry each
__global__ void own_kernel(int S, const long long* __restrict__ m_ptr, long long n_mem, const long long* __restrict__ m_truth,
                           const int* __restrict__ t_chrom, const long long* __restrict__ t_start, const long long* __restrict__ t_end,
                           const long long* __restrict__ t_cn, const long long* __restrict__ c_ptr, Calls c, double po,
                           uint8_t* __restrict__ counted, unsigned long long* __restrict__ stats) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n_mem) return;
    const int s = owner(m_ptr, S, e);
    const long long base = c_ptr[s], n = c_ptr[s + 1] - base;
    if (n == 0) return;                                          // a sample without calls: no TP, no FN
    const long long t = m_truth[e], ts = t_start[t], te = t_end[t];
    Calls cs{c.chrom + base, c.start + base, c.end + base, c.pmax + base, c.cn + base, nullptr};
    long long k0;
    const long long b = window(cs, n, t_chrom[t], ts, te, k0);
    const long long q = first_q(cs, k0, b, ts, te, t_cn[t], po);
    unsigned long long* st = stats + (long long)s * 12 + size_class(ts, te) * 4;
    if (q < b) {
        atomicAdd(&st[kTP], 1ull);
        counted[base + q] = 1;
    } else {
        atomicAdd(&st[kFN], 1ull);
    }
}

// updatePositive's last loop (cnveval.go:330-340)
__global__ void uncounted_kernel(int S, const long long* __restrict__ c_ptr, long long n_calls, const long long* __restrict__ c_start,
                                 const long long* __restrict__ c_end, const uint8_t* __restrict__ counted,
                                 unsigned long long* __restrict__ stats) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_calls || counted[k]) return;
    const int s = owner(c_ptr, S, k);
    atomicAdd(&stats[(long long)s * 12 + size_class(c_start[k], c_end[k]) * 4 + kFP], 1ull);
}

__device__ __forceinline__ unsigned long long warp_sum(unsigned long long v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// updateFP (cnveval.go:231-285) for every (sample with calls, truth it does not carry)
__global__ void __launch_bounds__(kThreads) others_kernel(const long long* __restrict__ c_ptr, Calls g, long long T,
                                                          const int* __restrict__ t_chrom, const long long* __restrict__ t_start,
                                                          const long long* __restrict__ t_end, const long long* __restrict__ t_cn,
                                                          const unsigned* __restrict__ bits, long long W, double po,
                                                          unsigned long long* __restrict__ stats) {
    __shared__ int sh_chrom[kSmemCalls];
    __shared__ long long sh_start[kSmemCalls], sh_end[kSmemCalls], sh_pmax[kSmemCalls], sh_cn[kSmemCalls];
    __shared__ uint8_t sh_tp[kSmemCalls];
    __shared__ unsigned long long sh_sum[6];
    const int s = blockIdx.x;
    const long long base = c_ptr[s], n = c_ptr[s + 1] - base;
    if (n == 0) return;                                          // the whole CTA: a sample without calls counts nothing
    Calls c{g.chrom + base, g.start + base, g.end + base, g.pmax + base, g.cn + base, g.tp + base};
    if (threadIdx.x < 6) sh_sum[threadIdx.x] = 0;
    if (n <= kSmemCalls) {
        for (long long k = threadIdx.x; k < n; k += kThreads) {
            sh_chrom[k] = c.chrom[k]; sh_start[k] = c.start[k]; sh_end[k] = c.end[k];
            sh_pmax[k] = c.pmax[k]; sh_cn[k] = c.cn[k]; sh_tp[k] = c.tp[k];
        }
        c = Calls{sh_chrom, sh_start, sh_end, sh_pmax, sh_cn, sh_tp};
    }
    __syncthreads();
    unsigned long long fp[3] = {0, 0, 0}, tn[3] = {0, 0, 0};
    const unsigned* row = bits + (long long)s * W;
    for (int j = 0; j < kTileTruths / kThreads; j++) {
        const long long o = (long long)blockIdx.y * kTileTruths + j * kThreads + threadIdx.x;
        if (o >= T) break;
        if ((row[o >> 5] >> (o & 31)) & 1u) continue;            // a truth the sample carries is not one of its others
        const long long ts = t_start[o], te = t_end[o], tcn = t_cn[o];
        long long k0;
        const long long b = window(c, n, t_chrom[o], ts, te, k0);
        const long long q = first_q(c, k0, b, ts, te, tcn, po);
        const int cls = size_class(ts, te);
        if (q == b) { tn[cls]++; continue; }
        long long k = q;                                         // k_tp: fpfound and tpfound are never reset
        while (k < b && !(c.tp[k] && qualifies(c.start[k], c.end[k], c.cn[k], ts, te, tcn, po))) k++;
        fp[cls] += (unsigned long long)(k - q);
    }
#pragma unroll
    for (int i = 0; i < 3; i++) {
        const unsigned long long a = warp_sum(fp[i]), b = warp_sum(tn[i]);
        if ((threadIdx.x & 31) == 0) {
            if (a) atomicAdd(&sh_sum[i], a);
            if (b) atomicAdd(&sh_sum[3 + i], b);
        }
    }
    __syncthreads();
    if (threadIdx.x < 6 && sh_sum[threadIdx.x]) {
        const int i = threadIdx.x % 3;
        atomicAdd(&stats[(long long)s * 12 + i * 4 + (threadIdx.x < 3 ? kFP : kTN)], sh_sum[threadIdx.x]);
    }
}

unsigned grid1(long long n) { return (unsigned)std::max<long long>(1, (n + kThreads - 1) / kThreads); }

// one device buffer carved into 16-byte-aligned arrays
struct Carve {
    size_t off = 0;
    template <class T> size_t take(size_t n) { off = (off + 15) & ~size_t(15); const size_t o = off; off += n * sizeof(T); return o; }
};

struct DeviceSet {
    int S; long long n_calls, T, n_mem;
    const long long* c_ptr; const int* c_chrom; const long long *c_start, *c_end, *c_cn;
    const int* t_chrom; const long long *t_start, *t_end, *t_cn;
    const long long *m_ptr, *m_truth;
};

int run(gl_ctx* ctx, const char* fn, const DeviceSet& d, double po, unsigned long long* d_stats) {
    const long long W = (d.T + 31) / 32;
    if ((d.T + kTileTruths - 1) / kTileTruths > 65535) return gl_fail(ctx, GL_EINVAL, "%s: %lld truths; at most %lld", fn, d.T, 65535ll * kTileTruths);
    if (d.S == 0) return GL_OK;
    GL_CUDA(ctx, cudaMemsetAsync(d_stats, 0, (size_t)d.S * 12 * 8, ctx->stream));
    Carve cv;
    const size_t o_err = cv.take<unsigned long long>(4), o_cp = cv.take<long long>((size_t)d.n_calls),
                 o_mp = cv.take<long long>((size_t)d.n_mem), o_tp = cv.take<uint8_t>((size_t)d.n_calls),
                 o_cnt = cv.take<uint8_t>((size_t)d.n_calls), o_bits = cv.take<unsigned>((size_t)(d.S * W));
    gl_scratch tmp(ctx);
    uint8_t* buf;
    GL_CHECK(tmp.alloc(buf, cv.off));
    unsigned long long* err = reinterpret_cast<unsigned long long*>(buf + o_err);
    long long* c_pmax = reinterpret_cast<long long*>(buf + o_cp);
    long long* m_pmax = reinterpret_cast<long long*>(buf + o_mp);
    uint8_t* tp = buf + o_tp;
    uint8_t* counted = buf + o_cnt;
    unsigned* bits = reinterpret_cast<unsigned*>(buf + o_bits);
    GL_CUDA(ctx, cudaMemsetAsync(err, 0xff, 4 * 8, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(counted, 0, (size_t)d.n_calls, ctx->stream));
    GL_CUDA(ctx, cudaMemsetAsync(bits, 0, (size_t)(d.S * W) * 4, ctx->stream));
    {
        gl_prof_scope prof(ctx, "cnveval_prep");
        prep_calls_kernel<<<grid1(d.S), kThreads, 0, ctx->stream>>>(d.S, d.c_ptr, d.n_calls, d.c_chrom, d.c_start, d.c_end, c_pmax, err);
        check_truths_kernel<<<grid1(d.T), kThreads, 0, ctx->stream>>>(d.T, d.t_chrom, d.t_start, d.t_end, err);
    }
    GL_LAUNCHED(ctx, 2);
    unsigned long long h[4];
    GL_CUDA(ctx, cudaMemcpyAsync(h, err, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h[3] != ~0ull) return gl_fail(ctx, GL_EINVAL, "%s: the call offsets of sample %lld are not a CSR of %lld calls", fn, (long long)h[3], d.n_calls);
    if (h[0] != ~0ull)
        return gl_fail(ctx, GL_EINVAL, "%s: call %lld has end < start, a coordinate outside [0, 2^62), a negative chrom rank, or is out of (chrom, start) order in its sample", fn, (long long)h[0]);
    if (h[1] != ~0ull)
        return gl_fail(ctx, GL_EINVAL, "%s: truth %lld has end < start, a coordinate outside [0, 2^62), a negative chrom rank, or is out of (chrom, start) order", fn, (long long)h[1]);
    {
        gl_prof_scope prof(ctx, "cnveval_members");
        prep_members_kernel<<<grid1(d.S), kThreads, 0, ctx->stream>>>(d.S, d.m_ptr, d.n_mem, d.m_truth, d.T, d.t_chrom, d.t_end, m_pmax, err);
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaMemcpyAsync(h, err, sizeof h, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (h[3] != ~0ull) return gl_fail(ctx, GL_EINVAL, "%s: the membership offsets of sample %lld are not a CSR of %lld entries", fn, (long long)h[3] - d.S, d.n_mem);
    if (h[2] != ~0ull) return gl_fail(ctx, GL_EINVAL, "%s: membership entry %lld names no truth or is out of ascending order in its sample", fn, (long long)h[2]);

    const Calls calls{d.c_chrom, d.c_start, d.c_end, c_pmax, d.c_cn, tp};
    {
        gl_prof_scope prof(ctx, "cnveval_bitset");
        if (d.n_mem) bitset_kernel<<<grid1(d.n_mem), kThreads, 0, ctx->stream>>>(d.S, d.m_ptr, d.n_mem, d.m_truth, W, bits);
    }
    {
        gl_prof_scope prof(ctx, "cnveval_tp_any");
        if (d.n_calls)
            tp_any_kernel<<<grid1(d.n_calls), kThreads, 0, ctx->stream>>>(d.S, d.c_ptr, d.n_calls, d.c_chrom, d.c_start, d.c_end, d.c_cn,
                                                                          d.m_ptr, d.m_truth, m_pmax, d.t_chrom, d.t_start, d.t_end,
                                                                          d.t_cn, po, tp);
    }
    {
        gl_prof_scope prof(ctx, "cnveval_own");
        if (d.n_mem)
            own_kernel<<<grid1(d.n_mem), kThreads, 0, ctx->stream>>>(d.S, d.m_ptr, d.n_mem, d.m_truth, d.t_chrom, d.t_start, d.t_end,
                                                                     d.t_cn, d.c_ptr, calls, po, counted, d_stats);
    }
    {
        gl_prof_scope prof(ctx, "cnveval_uncounted");
        if (d.n_calls)
            uncounted_kernel<<<grid1(d.n_calls), kThreads, 0, ctx->stream>>>(d.S, d.c_ptr, d.n_calls, d.c_start, d.c_end, counted, d_stats);
    }
    {
        gl_prof_scope prof(ctx, "cnveval_others");
        if (d.n_calls && d.T) {
            const dim3 grid((unsigned)d.S, (unsigned)((d.T + kTileTruths - 1) / kTileTruths));
            others_kernel<<<grid, kThreads, 0, ctx->stream>>>(d.c_ptr, calls, d.T, d.t_chrom, d.t_start, d.t_end, d.t_cn, bits, W, po, d_stats);
        }
    }
    GL_LAUNCHED(ctx, 5);
    return GL_OK;
}

bool po_ok(double po) { return std::isnan(po) || (po > 0 && po <= 1); }

}  // namespace

extern "C" {

int gl_cnveval_device(gl_ctx* ctx, int32_t S, const int64_t* d_c_ptr, int64_t n_calls, const int32_t* d_c_chrom, const int64_t* d_c_start,
                      const int64_t* d_c_end, const int64_t* d_c_cn, int64_t n_truths, const int32_t* d_t_chrom, const int64_t* d_t_start,
                      const int64_t* d_t_end, const int64_t* d_t_cn, const int64_t* d_m_ptr, int64_t n_mem, const int64_t* d_m_truth,
                      double po, uint64_t* d_stats) {
    GL_CHECK(gl_use(ctx));
    if (S < 0 || n_calls < 0 || n_truths < 0 || n_mem < 0 || (S > 0 && (!d_c_ptr || !d_m_ptr || !d_stats)) ||
        (n_calls > 0 && (!d_c_chrom || !d_c_start || !d_c_end || !d_c_cn)) ||
        (n_truths > 0 && (!d_t_chrom || !d_t_start || !d_t_end || !d_t_cn)) || (n_mem > 0 && !d_m_truth))
        return gl_fail(ctx, GL_EINVAL, "gl_cnveval_device: bad argument");
    if (!po_ok(po)) return gl_fail(ctx, GL_EINVAL, "gl_cnveval_device: minimum overlap %g is outside (0, 1]", po);
    const DeviceSet d{S, n_calls, n_truths, n_mem,
                      reinterpret_cast<const long long*>(d_c_ptr), d_c_chrom, reinterpret_cast<const long long*>(d_c_start),
                      reinterpret_cast<const long long*>(d_c_end), reinterpret_cast<const long long*>(d_c_cn),
                      d_t_chrom, reinterpret_cast<const long long*>(d_t_start), reinterpret_cast<const long long*>(d_t_end),
                      reinterpret_cast<const long long*>(d_t_cn), reinterpret_cast<const long long*>(d_m_ptr),
                      reinterpret_cast<const long long*>(d_m_truth)};
    return run(ctx, "gl_cnveval_device", d, po, reinterpret_cast<unsigned long long*>(d_stats));
}

int gl_cnveval(gl_ctx* ctx, int32_t S, const int32_t* c_sample, const int32_t* c_chrom, const int64_t* c_start, const int64_t* c_end,
               const int64_t* c_cn, int64_t n_calls, const int32_t* t_chrom, const int64_t* t_start, const int64_t* t_end,
               const int64_t* t_cn, int64_t n_truths, const int64_t* t_mem_ptr, const int32_t* t_mem_sample, double po,
               uint64_t* stats) {
    GL_CHECK(gl_use(ctx));
    if (S < 0 || n_calls < 0 || n_truths < 0 || (S > 0 && !stats) ||
        (n_calls > 0 && (!c_sample || !c_chrom || !c_start || !c_end || !c_cn)) ||
        (n_truths > 0 && (!t_chrom || !t_start || !t_end || !t_cn || !t_mem_ptr)))
        return gl_fail(ctx, GL_EINVAL, "gl_cnveval: bad argument");
    if (!po_ok(po)) return gl_fail(ctx, GL_EINVAL, "gl_cnveval: minimum overlap %g is outside (0, 1]", po);
    // the value policy (DESIGN §1.12), named by input position
    for (int64_t i = 0; i < n_calls; i++) {
        if (c_sample[i] < 0 || c_sample[i] >= S) return gl_fail(ctx, GL_EINVAL, "gl_cnveval: call %lld names sample %d of %d", (long long)i, c_sample[i], S);
        if (c_chrom[i] < 0 || c_start[i] < 0 || c_end[i] < c_start[i] || c_end[i] >= kMaxCoord)
            return gl_fail(ctx, GL_EINVAL, "gl_cnveval: call %lld (%lld-%lld) has end < start or a coordinate outside [0, 2^62)", (long long)i,
                           (long long)c_start[i], (long long)c_end[i]);
    }
    const int64_t n_mem = n_truths > 0 ? t_mem_ptr[n_truths] : 0;
    if (n_truths > 0 && (t_mem_ptr[0] != 0 || n_mem < 0 || (n_mem > 0 && !t_mem_sample))) return gl_fail(ctx, GL_EINVAL, "gl_cnveval: bad membership offsets");
    for (int64_t t = 0; t < n_truths; t++) {
        if (t_chrom[t] < 0 || t_start[t] < 0 || t_end[t] < t_start[t] || t_end[t] >= kMaxCoord)
            return gl_fail(ctx, GL_EINVAL, "gl_cnveval: truth %lld (%lld-%lld) has end < start or a coordinate outside [0, 2^62)", (long long)t,
                           (long long)t_start[t], (long long)t_end[t]);
        if (t_mem_ptr[t + 1] < t_mem_ptr[t] || t_mem_ptr[t + 1] > n_mem) return gl_fail(ctx, GL_EINVAL, "gl_cnveval: bad membership offsets");
        for (int64_t k = t_mem_ptr[t]; k < t_mem_ptr[t + 1]; k++)
            if (t_mem_sample[k] < 0 || t_mem_sample[k] >= S)
                return gl_fail(ctx, GL_EINVAL, "gl_cnveval: truth %lld names sample %d of %d", (long long)t, t_mem_sample[k], S);
    }

    // truths by (chrom, start) (their order inside a tie does not change any count); memberships sample-major, ascending
    std::vector<int64_t> to((size_t)n_truths);
    for (int64_t t = 0; t < n_truths; t++) to[(size_t)t] = t;
    std::stable_sort(to.begin(), to.end(), [&](int64_t a, int64_t b) {
        return t_chrom[a] < t_chrom[b] || (t_chrom[a] == t_chrom[b] && t_start[a] < t_start[b]); });
    std::vector<int32_t> tc((size_t)n_truths);
    std::vector<int64_t> tsv((size_t)n_truths), tev((size_t)n_truths), tcn((size_t)n_truths);
    std::vector<int64_t> m_ptr((size_t)S + 1, 0), m_truth((size_t)n_mem);
    for (int64_t k = 0; k < n_mem; k++) m_ptr[(size_t)t_mem_sample[k] + 1]++;
    for (int32_t s = 0; s < S; s++) m_ptr[(size_t)s + 1] += m_ptr[(size_t)s];
    {
        std::vector<int64_t> fill(m_ptr.begin(), m_ptr.end() - 1);
        for (int64_t r = 0; r < n_truths; r++) {
            const int64_t t = to[(size_t)r];
            tc[(size_t)r] = t_chrom[t]; tsv[(size_t)r] = t_start[t]; tev[(size_t)r] = t_end[t]; tcn[(size_t)r] = t_cn[t];
            for (int64_t k = t_mem_ptr[t]; k < t_mem_ptr[t + 1]; k++) m_truth[(size_t)fill[(size_t)t_mem_sample[k]]++] = r;
        }
    }
    // calls grouped by sample in file order, then each sample in Go's sort.Slice order
    std::vector<int64_t> c_ptr((size_t)S + 1, 0), grp((size_t)n_calls);
    for (int64_t i = 0; i < n_calls; i++) c_ptr[(size_t)c_sample[i] + 1]++;
    for (int32_t s = 0; s < S; s++) c_ptr[(size_t)s + 1] += c_ptr[(size_t)s];
    {
        std::vector<int64_t> fill(c_ptr.begin(), c_ptr.end() - 1);
        for (int64_t i = 0; i < n_calls; i++) grp[(size_t)fill[(size_t)c_sample[i]]++] = i;
    }
    std::vector<int32_t> cc((size_t)n_calls), kc;
    std::vector<int64_t> csv((size_t)n_calls), cev((size_t)n_calls), ccn((size_t)n_calls), ks, perm;
    for (int32_t s = 0; s < S; s++) {
        const int64_t a = c_ptr[(size_t)s], n = c_ptr[(size_t)s + 1] - a;
        kc.resize((size_t)n); ks.resize((size_t)n); perm.resize((size_t)n);
        for (int64_t j = 0; j < n; j++) { kc[(size_t)j] = c_chrom[grp[(size_t)(a + j)]]; ks[(size_t)j] = c_start[grp[(size_t)(a + j)]]; }
        gl_cnveval_order(kc.data(), ks.data(), n, perm.data());
        for (int64_t j = 0; j < n; j++) {
            const int64_t i = grp[(size_t)(a + perm[(size_t)j])];
            cc[(size_t)(a + j)] = c_chrom[i]; csv[(size_t)(a + j)] = c_start[i]; cev[(size_t)(a + j)] = c_end[i]; ccn[(size_t)(a + j)] = c_cn[i];
        }
    }

    Carve cv;
    const size_t o_cptr = cv.take<int64_t>((size_t)S + 1), o_cc = cv.take<int32_t>((size_t)n_calls), o_cs = cv.take<int64_t>((size_t)n_calls),
                 o_ce = cv.take<int64_t>((size_t)n_calls), o_ccn = cv.take<int64_t>((size_t)n_calls), o_tc = cv.take<int32_t>((size_t)n_truths),
                 o_ts = cv.take<int64_t>((size_t)n_truths), o_te = cv.take<int64_t>((size_t)n_truths), o_tcn = cv.take<int64_t>((size_t)n_truths),
                 o_mptr = cv.take<int64_t>((size_t)S + 1), o_mt = cv.take<int64_t>((size_t)n_mem), o_st = cv.take<uint64_t>((size_t)S * 12);
    std::vector<uint8_t> host(cv.off);
    auto put = [&](size_t off, const void* p, size_t bytes) { if (bytes) memcpy(host.data() + off, p, bytes); };
    put(o_cptr, c_ptr.data(), c_ptr.size() * 8);
    put(o_cc, cc.data(), cc.size() * 4); put(o_cs, csv.data(), csv.size() * 8); put(o_ce, cev.data(), cev.size() * 8); put(o_ccn, ccn.data(), ccn.size() * 8);
    put(o_tc, tc.data(), tc.size() * 4); put(o_ts, tsv.data(), tsv.size() * 8); put(o_te, tev.data(), tev.size() * 8); put(o_tcn, tcn.data(), tcn.size() * 8);
    put(o_mptr, m_ptr.data(), m_ptr.size() * 8); put(o_mt, m_truth.data(), m_truth.size() * 8);
    gl_scratch tmp(ctx);
    uint8_t* dev;
    GL_CHECK(tmp.upload(dev, host.data(), host.size()));
    auto at = [&](size_t off) { return reinterpret_cast<const long long*>(dev + off); };
    const DeviceSet d{S, n_calls, n_truths, n_mem, at(o_cptr), reinterpret_cast<const int*>(dev + o_cc), at(o_cs), at(o_ce), at(o_ccn),
                      reinterpret_cast<const int*>(dev + o_tc), at(o_ts), at(o_te), at(o_tcn), at(o_mptr), at(o_mt)};
    unsigned long long* d_stats = reinterpret_cast<unsigned long long*>(dev + o_st);
    GL_CHECK(run(ctx, "gl_cnveval", d, po, d_stats));
    if (S > 0) GL_CUDA(ctx, cudaMemcpyAsync(stats, d_stats, (size_t)S * 12 * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

}  // extern "C"
