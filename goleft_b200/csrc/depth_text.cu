// depth_text.cu — the text half of `goleft depth` on the device: the rows the reference callback writes with
//   fmt.Sprintf("%s\t%d\t%d\t%.4g%s\n", chrom, s, e, mean(depthCache, e-s), stats)      depth/depth.go:301,337,357
//   fmt.Sprintf("%s\t%d\t%d\t%s\n", chrom, start, end, class)                            depth/depth.go:312,316,324,346,349
// are produced as bytes by three small kernels from the window sums / class runs the reduce left in HBM, so only
// finished BED text crosses PCIe (about 28 B per window instead of 8 B + a host sprintf per window).
//
//   K_rows   one thread per row: the variable part "\t<s>\t<e>\t<%.4g mean | CLASS>\n" into a 48-byte slot
//            (byte 47 = length) + the row lengths summed per 256-row block
//   K_scan   one CTA: exclusive scan of the block sums -> byte offset of every block, total length
//   K_emit   one CTA per 256 rows: CTA scan of the row lengths, rows assembled in shared memory, coalesced copy out
//
// mean(depthCache, e-s) (depth.go:181-189) adds the ints as float64 (exact below 2^53) and divides by float64(e-s):
// one IEEE division.  "%.4g" of that double is made exactly: the four significant digits are
// round_half_even(q * 10^k) in 128-bit integer arithmetic on q's mantissa, never by floating-point scaling; %e or %f
// form like strconv (exponent < -4 or >= 4 -> %e), trailing zeros stripped.  Checked against printf on every test.
#include "gl_common.cuh"
#include <string.h>

namespace {

constexpr int kSlot = 48;            // bytes per row slot; byte 47 = length of the variable part
constexpr int kRowsPerBlock = 256;
constexpr int kMaxChrom = 64;        // chrom names up to this many bytes are formatted on the device

struct TextParams {
    char chrom[kMaxChrom];
    int cl;                                   // strlen(chrom)
    int mode;                                 // 0: window rows, 1: class rows
    long long n;                              // rows
    // window rows, implicit (row i = window w0+i of [rs,re)) or explicit (row_s != null)
    long long rs, re, w0;
    int W;
    const unsigned long long* win_sum;
    const int* row_s; const int* row_e; const long long* row_sum;
    // class rows: run i = [run_start[i], run_start[i+1] or re) of class run_class[i]
    const int* run_start; const unsigned char* run_class;
    // outputs
    unsigned char* slots;                     // [n * 48]
    unsigned long long* block_off;            // [n_blocks + 1]: K_rows writes the block sums, K_scan turns them into offsets
    unsigned char* out;                       // compact text
};

__device__ __forceinline__ int put_u32(unsigned char* t, int len, unsigned v) {
    unsigned char b[10];
    int n = 0;
    do { b[n++] = (unsigned char)('0' + v % 10u); v /= 10u; } while (v);
    while (n) t[len++] = b[--n];
    return len;
}

__device__ __forceinline__ unsigned __int128 pow10_128(int k) {
    unsigned __int128 r = 1;
    for (int i = 0; i < k; i++) r *= 10;
    return r;
}

// round_half_even(m * 2^e2 * 10^k); the caller keeps m*10^k and 2^-e2 * 10^-k below 2^127
__device__ __forceinline__ unsigned long long scaled_round64(unsigned long long m, int e2, int k) {
    unsigned __int128 num = m, q, r, den;
    if (k >= 0) {
        num *= pow10_128(k);
        if (e2 >= 0) return (unsigned long long)(num << e2);
        den = (unsigned __int128)1 << (-e2);                          // power of two: shift instead of divide
        q = num >> (-e2);
        r = num & (den - 1);
    } else {
        den = pow10_128(-k);
        if (e2 >= 0) num <<= e2; else den <<= -e2;
        q = num / den;
        r = num % den;
    }
    const unsigned __int128 twice = r * 2;
    if (twice > den || (twice == den && (q & 1))) q++;
    return (unsigned long long)q;
}

// The four significant digits of "%.4g" of a finite double 0 < q < 1e15, q >= 1e-15: the text's value is N * 10^(e10-3)
// with 1000 <= N <= 9999.  The text kernel prints them and the depthwed cell kernel rounds them, so both read one rounding.
__device__ __forceinline__ unsigned long long g4_digits(double q, int& e10) {
    const unsigned long long bits = (unsigned long long)__double_as_longlong(q);
    const int ex = (int)((bits >> 52) & 0x7ff);
    const unsigned long long frac = bits & ((1ull << 52) - 1);
    const unsigned long long m = ex ? (frac | (1ull << 52)) : frac;
    const int e2 = ex ? ex - 1075 : -1074;
    e10 = (int)floor(log10(q));
    unsigned long long N = scaled_round64(m, e2, 3 - e10);
    if (N < 1000) { e10--; N = scaled_round64(m, e2, 3 - e10); }            // estimate one too high
    else if (N > 10000) { e10++; N = scaled_round64(m, e2, 3 - e10); }      // one too low
    if (N >= 10000) { N = 1000; e10++; }                                    // 9999.5.. rounds up to the next decade
    return N;
}

// "%.4g" of a finite double 0 <= q < 1e15 (and q == 0 or q >= 1e-15): appends to t, returns the new length
__device__ __forceinline__ int put_g4(unsigned char* t, int len, double q) {
    if (q == 0.0) { t[len++] = '0'; return len; }
    int e10;
    const unsigned long long N = g4_digits(q, e10);
    int dig[4];
    dig[0] = (int)(N / 1000); dig[1] = (int)(N / 100 % 10); dig[2] = (int)(N / 10 % 10); dig[3] = (int)(N % 10);
    const int nd = dig[3] ? 4 : (dig[2] ? 3 : (dig[1] ? 2 : 1));             // significant digits after stripping zeros
    if (e10 < -4 || e10 >= 4) {                                              // %e form, exponent at least two digits
        t[len++] = (unsigned char)('0' + dig[0]);
        if (nd > 1) {
            t[len++] = '.';
            for (int k = 1; k < nd; k++) t[len++] = (unsigned char)('0' + dig[k]);
        }
        t[len++] = 'e';
        t[len++] = e10 < 0 ? '-' : '+';
        const int ae = e10 < 0 ? -e10 : e10;
        t[len++] = (unsigned char)('0' + ae / 10);
        t[len++] = (unsigned char)('0' + ae % 10);
    } else if (e10 >= 0) {                                                   // dddd / d.ddd: the point after e10+1 digits
        for (int k = 0; k < 4; k++) {
            if (k <= e10 || k < nd) {
                if (k == e10 + 1) t[len++] = '.';
                t[len++] = (unsigned char)('0' + dig[k]);
            }
        }
    } else {                                                                 // 0.000dddd
        t[len++] = '0'; t[len++] = '.';
        for (int z = 0; z < -e10 - 1; z++) t[len++] = '0';
        for (int k = 0; k < nd; k++) t[len++] = (unsigned char)('0' + dig[k]);
    }
    return len;
}

__device__ __forceinline__ int put_class(unsigned char* t, int len, int cls) {
    // depth.go:223-234
    const char* nm = cls == GL_NO_COVERAGE ? "NO_COVERAGE" : cls == GL_LOW_COVERAGE ? "LOW_COVERAGE"
                   : cls == GL_CALLABLE ? "CALLABLE" : "EXCESSIVE_COVERAGE";
    for (int k = 0; nm[k]; k++) t[len++] = (unsigned char)nm[k];
    return len;
}

// ------------------------------------------------------------------------------------------------ depthwed cells
// The cell depthwed.go:103 makes of a depth.bed row, int(0.5 + ParseFloat("%.4g" of q)), without the text: the text's value
// is N * 10^(e10-3), so the cell is floor(N * 10^(e10-3) + 1/2) in integers, ties up.  That is exactly what Go computes:
// a value with a fractional part is below 1000 and a multiple of 10^-4 or zero, so 0.5 + it truncates to the same integer.
__device__ __forceinline__ unsigned long long g4_cell(double q) {
    if (q == 0.0) return 0;
    int e10;
    const unsigned long long N = g4_digits(q, e10);
    unsigned long long p = 1;
    for (int k = e10 > 3 ? e10 - 3 : 3 - e10; k > 0; k--) p *= 10;          // 10^|e10-3|, at most 10^19
    return e10 >= 3 ? N * p : (N + p / 2) / p;
}

struct CellParams {
    long long n;                              // windows
    // implicit windows of the last reduce (sum == null): window i = [max(rs, (wb+i)W), min(re, (wb+i+1)W))
    long long rs, re, wb;
    int W;
    const unsigned long long* win_sum;
    const long long* sum; const long long* len;   // explicit windows
    const int* grp_of; long long g0;          // window i adds into col[grp_of[g0 + i]]; grp_of == null: col[i]
    unsigned long long* col;
};

// One thread per window.  Consecutive windows of one group are summed in the warp (a segmented suffix scan over the runs of
// equal group ids) and each run's first lane adds the run's sum with one 64-bit atomic: a group of SIZE/W windows costs
// about SIZE/W/32 atomics per column, not one per window.  Any map is accepted; a group split into several runs gets one
// atomic per run.
__global__ void __launch_bounds__(256) depthwed_cells_kernel(const CellParams p) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    const int lane = threadIdx.x & 31;
    unsigned long long v = 0;
    long long key = -1;
    if (i < p.n) {
        long long sum, len;
        if (p.sum) { sum = p.sum[i]; len = p.len[i]; }
        else {
            sum = (long long)p.win_sum[i];
            len = min(p.re, (p.wb + i + 1) * (long long)p.W) - max(p.rs, (p.wb + i) * (long long)p.W);
        }
        // depth.go:181-189, as bed_rows_kernel: 0 for an empty cache or zero length, else float64 sum / float64(len)
        v = g4_cell((sum <= 0 || len <= 0) ? 0.0 : __ddiv_rn((double)sum, (double)len));
        key = p.grp_of ? (long long)p.grp_of[p.g0 + i] : i;
    }
    const long long knext = __shfl_down_sync(0xffffffffu, key, 1);
    bool ends = lane == 31 || knext != key;                                   // the lane's run ends here
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_down_sync(0xffffffffu, v, o);
        const bool ey = __shfl_down_sync(0xffffffffu, ends, o);
        if (!ends && lane + o < 32) { v += y; ends = ey; }
    }
    const long long kprev = __shfl_up_sync(0xffffffffu, key, 1);
    if (key >= 0 && v != 0 && (lane == 0 || kprev != key)) atomicAdd(p.col + key, v);
}

int launch_cells(gl_ctx* ctx, const CellParams& p) {
    if (p.n <= 0) return GL_OK;
    {
        gl_prof_scope prof(ctx, "depthwed_cells_kernel");
        depthwed_cells_kernel<<<(unsigned)((p.n + 255) / 256), 256, 0, ctx->stream>>>(p);
    }
    GL_LAUNCHED(ctx, 1);
    return GL_OK;
}

__global__ void __launch_bounds__(kRowsPerBlock) bed_rows_kernel(const TextParams p) {
    __shared__ unsigned s_sum[kRowsPerBlock / 32];
    const long long i = (long long)blockIdx.x * kRowsPerBlock + threadIdx.x;
    __align__(16) unsigned char t[kSlot];
    int len = 0;
    if (i < p.n) {
        long long s, e;
        if (p.mode == 0) {
            long long sum;
            if (p.row_s) { s = p.row_s[i]; e = p.row_e[i]; sum = p.row_sum[i]; }
            else {
                s = max(p.rs, (p.w0 + i) * (long long)p.W);
                e = min(p.re, (p.w0 + i + 1) * (long long)p.W);
                sum = (long long)p.win_sum[i];
            }
            t[len++] = '\t'; len = put_u32(t, len, (unsigned)s);
            t[len++] = '\t'; len = put_u32(t, len, (unsigned)e);
            t[len++] = '\t';
            // depth.go:181-189: 0 for an empty cache or zero length, else float64 sum / float64(e - s)
            const double q = (sum <= 0 || e <= s) ? 0.0 : __ddiv_rn((double)sum, (double)(e - s));
            len = put_g4(t, len, q);
        } else {
            s = p.run_start[i];
            e = (i + 1 < p.n) ? (long long)p.run_start[i + 1] : p.re;
            t[len++] = '\t'; len = put_u32(t, len, (unsigned)s);
            t[len++] = '\t'; len = put_u32(t, len, (unsigned)e);
            t[len++] = '\t';
            len = put_class(t, len, p.run_class[i]);
        }
        t[len++] = '\n';
        t[kSlot - 1] = (unsigned char)len;
        uint4* dst = reinterpret_cast<uint4*>(p.slots + i * kSlot);
        const uint4* src = reinterpret_cast<const uint4*>(t);
        dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
        len += p.cl;
    }
    const unsigned w = __reduce_add_sync(0xffffffffu, (unsigned)len);
    if ((threadIdx.x & 31) == 0) s_sum[threadIdx.x >> 5] = w;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned tot = 0;
        for (int k = 0; k < kRowsPerBlock / 32; k++) tot += s_sum[k];
        p.block_off[blockIdx.x] = tot;
    }
}

// exclusive scan of block_off[0..nb) in place; block_off[nb] = total
__global__ void __launch_bounds__(1024) bed_scan_kernel(unsigned long long* __restrict__ v, long long nb) {
    __shared__ unsigned long long s_w[32];
    __shared__ unsigned long long s_carry;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_carry = 0;
    __syncthreads();
    for (long long base = 0; base < nb; base += 1024) {
        const long long i = base + tid;
        const unsigned long long x = i < nb ? v[i] : 0;
        unsigned long long inc = x;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, inc, o);
            if (lane >= o) inc += y;
        }
        if (lane == 31) s_w[warp] = inc;
        __syncthreads();
        unsigned long long wbase = 0;
        for (int k = 0; k < warp; k++) wbase += s_w[k];
        const unsigned long long carry = s_carry;
        if (i < nb) v[i] = carry + wbase + inc - x;
        __syncthreads();
        if (tid == 1023) s_carry = carry + wbase + inc;
        __syncthreads();
    }
    if (tid == 0) v[nb] = s_carry;
}

__global__ void __launch_bounds__(kRowsPerBlock) bed_emit_kernel(const TextParams p) {
    extern __shared__ unsigned char s_text[];                      // up to 256 * (cl + 47) bytes
    __shared__ unsigned s_w[kRowsPerBlock / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const long long i = (long long)blockIdx.x * kRowsPerBlock + tid;
    __align__(16) unsigned char t[kSlot];
    int vlen = 0, len = 0;
    if (i < p.n) {
        const uint4* src = reinterpret_cast<const uint4*>(p.slots + i * kSlot);
        uint4* dst = reinterpret_cast<uint4*>(t);
        dst[0] = src[0]; dst[1] = src[1]; dst[2] = src[2];
        vlen = t[kSlot - 1];
        len = vlen + p.cl;
    }
    unsigned inc = (unsigned)len;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    unsigned off = inc - (unsigned)len, total = 0;
    for (int k = 0; k < kRowsPerBlock / 32; k++) { if (k < warp) off += s_w[k]; total += s_w[k]; }
    if (i < p.n) {
        unsigned char* o = s_text + off;
        for (int k = 0; k < p.cl; k++) o[k] = (unsigned char)p.chrom[k];
        o += p.cl;
        for (int k = 0; k < vlen; k++) o[k] = t[k];
    }
    __syncthreads();
    unsigned char* g = p.out + p.block_off[blockIdx.x];
    // coalesced copy: bytes up to 16-byte alignment of the destination, then 16-byte words, then the tail
    const unsigned head = min(total, (unsigned)((16 - ((uintptr_t)g & 15)) & 15));
    for (unsigned k = tid; k < head; k += kRowsPerBlock) g[k] = s_text[k];
    const unsigned words = (total - head) / 16;
    for (unsigned k = tid; k < words; k += kRowsPerBlock) {
        const unsigned char* s = s_text + head + k * 16;
        uint4 v;
        unsigned x[4];
#pragma unroll
        for (int j = 0; j < 4; j++) x[j] = (unsigned)s[4 * j] | ((unsigned)s[4 * j + 1] << 8) | ((unsigned)s[4 * j + 2] << 16) | ((unsigned)s[4 * j + 3] << 24);
        v.x = x[0]; v.y = x[1]; v.z = x[2]; v.w = x[3];
        reinterpret_cast<uint4*>(g + head)[k] = v;
    }
    for (unsigned k = head + words * 16 + tid; k < total; k += kRowsPerBlock) g[k] = s_text[k];
}

// runs the three kernels for one row list; the text stays on the device in ctx->text_out[which], *len_out = its length
int format_rows(gl_ctx* ctx, TextParams& p, int which, int64_t* len_out) {
    *len_out = 0;
    if (p.n <= 0) return GL_OK;
    const long long nb = (p.n + kRowsPerBlock - 1) / kRowsPerBlock;
    GL_CHECK(gl_buf_reserve(ctx, ctx->text_slots, (size_t)p.n * kSlot));
    GL_CHECK(gl_buf_reserve(ctx, ctx->text_blk, (size_t)(nb + 1) * 8));
    GL_CHECK(gl_buf_reserve(ctx, ctx->text_out[which], (size_t)p.n * (size_t)(p.cl + (p.mode ? 42 : 33)) + 16));
    p.slots = static_cast<unsigned char*>(ctx->text_slots.p);
    p.block_off = static_cast<unsigned long long*>(ctx->text_blk.p);
    p.out = static_cast<unsigned char*>(ctx->text_out[which].p);
    {
        gl_prof_scope prof(ctx, "bed_rows_kernel");
        bed_rows_kernel<<<(unsigned)nb, kRowsPerBlock, 0, ctx->stream>>>(p);
    }
    GL_LAUNCHED(ctx, 1);
    {
        gl_prof_scope prof(ctx, "bed_scan_kernel");
        bed_scan_kernel<<<1, 1024, 0, ctx->stream>>>(p.block_off, nb);
    }
    GL_LAUNCHED(ctx, 1);
    {
        gl_prof_scope prof(ctx, "bed_emit_kernel");
        bed_emit_kernel<<<(unsigned)nb, kRowsPerBlock, (size_t)kRowsPerBlock * (size_t)(p.cl + kSlot - 1), ctx->stream>>>(p);
    }
    GL_LAUNCHED(ctx, 1);
    return GL_OK;
}

int set_chrom(gl_ctx* ctx, TextParams& p, const char* chrom) {
    if (!chrom) return gl_fail(ctx, GL_EINVAL, "null chrom");
    const size_t cl = strlen(chrom);
    if (cl > (size_t)kMaxChrom) return gl_fail(ctx, GL_ERANGE, "chrom name longer than %d bytes: use gl_depth_format_chunk", kMaxChrom);
    memcpy(p.chrom, chrom, cl);
    p.cl = (int)cl;
    return GL_OK;
}

}  // namespace

extern "C" {

int gl_depth_text(gl_ctx* ctx, const char* chrom, char* depth_bed, int64_t depth_cap, int64_t* depth_len,
                  char* callable_bed, int64_t callable_cap, int64_t* callable_len) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(depth_resolve(ctx));
    if (!ctx->depth_reduced) return gl_fail(ctx, GL_ESTATE, "gl_depth_text: call gl_depth_reduce first");
    if (!depth_len || !callable_len) return gl_fail(ctx, GL_EINVAL, "gl_depth_text: null length pointer");
    const int W = ctx->red.W;
    if (ctx->n_windows > 0 && ctx->rs % W != 0)
        return gl_fail(ctx, GL_EINVAL, "gl_depth_text: region start %lld is not a multiple of the window size (use gl_depth_format_rows)", (long long)ctx->rs);
    if (ctx->red.run_break > 0 && ctx->red.run_break % W != 0)
        return gl_fail(ctx, GL_EINVAL, "gl_depth_text: run_break must be a multiple of the window size");
    TextParams pw, pc;
    memset(&pw, 0, sizeof pw);
    GL_CHECK(set_chrom(ctx, pw, chrom));
    pc = pw;
    // window rows: with rs % W == 0 (and chunks that are multiples of W, depth.go:132) the rows of depth.go:293-305,
    // 329-341 and 351-358 are exactly the genome-aligned windows of the region, each once, in order
    pw.mode = 0;
    pw.n = ctx->n_windows;
    pw.rs = ctx->rs; pw.re = ctx->re; pw.W = W; pw.w0 = ctx->rs / W;
    pw.win_sum = static_cast<const unsigned long long*>(ctx->win_sum_p);
    // the host pointers below may already hold prefetched results; the device copies are what is formatted
    pc.mode = 1;
    pc.n = ctx->n_runs;
    pc.re = ctx->re;
    pc.run_start = static_cast<const int*>(ctx->run_start.p);
    pc.run_class = static_cast<const unsigned char*>(ctx->run_class.p);
    int64_t dummy;
    // class rows first: their slots/offset buffers are reused by the window rows (stream order keeps that safe),
    // the two compact texts live in separate buffers
    const long long nbc = (pc.n + kRowsPerBlock - 1) / kRowsPerBlock, nbw = (pw.n + kRowsPerBlock - 1) / kRowsPerBlock;
    unsigned long long lens[2] = {0, 0};
    GL_CHECK(gl_buf_reserve(ctx, ctx->text_len, 16));
    GL_CHECK(format_rows(ctx, pc, 1, &dummy));
    if (pc.n > 0) GL_CUDA(ctx, cudaMemcpyAsync(static_cast<char*>(ctx->text_len.p) + 8, pc.block_off + nbc, 8, cudaMemcpyDeviceToDevice, ctx->stream));
    GL_CHECK(format_rows(ctx, pw, 0, &dummy));
    if (pw.n > 0) GL_CUDA(ctx, cudaMemcpyAsync(ctx->text_len.p, pw.block_off + nbw, 8, cudaMemcpyDeviceToDevice, ctx->stream));
    if (pw.n == 0 || pc.n == 0) GL_CUDA(ctx, cudaMemsetAsync(static_cast<char*>(ctx->text_len.p) + (pw.n == 0 ? 0 : 8), 0, 8, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(lens, ctx->text_len.p, 16, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *depth_len = (int64_t)lens[0];
    *callable_len = (int64_t)lens[1];
    if ((int64_t)lens[0] > depth_cap || (int64_t)lens[1] > callable_cap)
        return gl_fail(ctx, GL_ERANGE, "gl_depth_text: text is %lld + %lld bytes, buffers hold %lld + %lld", (long long)lens[0],
                       (long long)lens[1], (long long)depth_cap, (long long)callable_cap);
    if (lens[0] && !depth_bed) return gl_fail(ctx, GL_EINVAL, "gl_depth_text: null depth_bed");
    if (lens[1] && !callable_bed) return gl_fail(ctx, GL_EINVAL, "gl_depth_text: null callable_bed");
    if (lens[0]) GL_CUDA(ctx, cudaMemcpyAsync(depth_bed, ctx->text_out[0].p, (size_t)lens[0], cudaMemcpyDeviceToHost, ctx->stream));
    if (lens[1]) GL_CUDA(ctx, cudaMemcpyAsync(callable_bed, ctx->text_out[1].p, (size_t)lens[1], cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int64_t gl_depth_text_bound(const char* chrom, int64_t n_windows) {
    return n_windows * (int64_t)((chrom ? strlen(chrom) : 0) + 33) + 16;
}

int gl_depth_format_rows(gl_ctx* ctx, const char* chrom, const int32_t* row_s, const int32_t* row_e, const int64_t* row_sum,
                         int64_t n, char* out, int64_t cap, int64_t* len) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || !len || (n > 0 && (!row_s || !row_e || !row_sum))) return gl_fail(ctx, GL_EINVAL, "gl_depth_format_rows: bad argument");
    *len = 0;
    if (n == 0) return GL_OK;
    TextParams p;
    memset(&p, 0, sizeof p);
    GL_CHECK(set_chrom(ctx, p, chrom));
    const size_t sum_off = ((size_t)n * 8 + 15) & ~size_t(15);
    GL_CHECK(gl_buf_reserve(ctx, ctx->misc, sum_off + (size_t)n * 8));
    int* d_s = static_cast<int*>(ctx->misc.p);
    int* d_e = d_s + n;
    long long* d_sum = reinterpret_cast<long long*>(static_cast<char*>(ctx->misc.p) + sum_off);
    GL_CUDA(ctx, cudaMemcpyAsync(d_s, row_s, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(d_e, row_e, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(d_sum, row_sum, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
    p.mode = 0; p.n = n; p.row_s = d_s; p.row_e = d_e; p.row_sum = d_sum;
    int64_t dummy;
    GL_CHECK(format_rows(ctx, p, 0, &dummy));
    const long long nb = (n + kRowsPerBlock - 1) / kRowsPerBlock;
    unsigned long long total = 0;
    GL_CUDA(ctx, cudaMemcpyAsync(&total, p.block_off + nb, 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *len = (int64_t)total;
    if ((int64_t)total > cap) return gl_fail(ctx, GL_ERANGE, "gl_depth_format_rows: text is %lld bytes, buffer holds %lld", (long long)total, (long long)cap);
    if (!out) return gl_fail(ctx, GL_EINVAL, "gl_depth_format_rows: null out");
    GL_CUDA(ctx, cudaMemcpyAsync(out, ctx->text_out[0].p, (size_t)total, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_depthwed_cells(gl_ctx* ctx, const int64_t* sums, const int64_t* lens, int64_t n, const int32_t* grp_of, int64_t n_groups, int64_t* out) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || !out || (n > 0 && (!sums || !lens)) || (grp_of ? n_groups < 0 : n_groups != n))
        return gl_fail(ctx, GL_EINVAL, "gl_depthwed_cells: bad argument");
    for (int64_t i = 0; i < n; i++) {
        if (grp_of && (grp_of[i] < 0 || grp_of[i] >= n_groups)) return gl_fail(ctx, GL_EINVAL, "gl_depthwed_cells: grp_of[%lld] out of range", (long long)i);
        if (sums[i] > 0 && lens[i] > 0 && (sums[i] >= (int64_t(1) << 53) || lens[i] >= (int64_t(1) << 31) || (double)sums[i] / (double)lens[i] >= 1e15))
            return gl_fail(ctx, GL_ERANGE, "gl_depthwed_cells: window %lld: sum %lld over %lld bases is out of range", (long long)i,
                           (long long)sums[i], (long long)lens[i]);
    }
    if (n_groups == 0) return GL_OK;
    gl_scratch tmp(ctx);
    long long *d_sum, *d_len;
    int* d_grp = nullptr;
    unsigned long long* d_out;
    GL_CHECK(tmp.upload(d_sum, reinterpret_cast<const long long*>(sums), (size_t)n));
    GL_CHECK(tmp.upload(d_len, reinterpret_cast<const long long*>(lens), (size_t)n));
    if (grp_of) GL_CHECK(tmp.upload(d_grp, reinterpret_cast<const int*>(grp_of), (size_t)n));
    GL_CHECK(tmp.alloc(d_out, (size_t)n_groups));
    GL_CUDA(ctx, cudaMemsetAsync(d_out, 0, (size_t)n_groups * 8, ctx->stream));
    CellParams p;
    memset(&p, 0, sizeof p);
    p.n = n; p.sum = d_sum; p.len = d_len; p.grp_of = d_grp; p.col = d_out;
    GL_CHECK(launch_cells(ctx, p));
    GL_CUDA(ctx, cudaMemcpyAsync(out, d_out, (size_t)n_groups * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_depthwed_column_begin(gl_ctx* ctx, int64_t* d_col, int64_t n_groups) {
    GL_CHECK(gl_use(ctx));
    if (n_groups < 0 || (n_groups > 0 && !d_col)) return gl_fail(ctx, GL_EINVAL, "gl_depthwed_column_begin: bad argument");
    if (n_groups) GL_CUDA(ctx, cudaMemsetAsync(d_col, 0, (size_t)n_groups * 8, ctx->stream));
    return GL_OK;
}

int gl_depthwed_add_column(gl_ctx* ctx, int64_t w0, const int32_t* d_grp_of, int64_t* d_col) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(depth_resolve(ctx));
    if (!ctx->depth_reduced) return gl_fail(ctx, GL_ESTATE, "gl_depthwed_add_column: call gl_depth_reduce first");
    if (w0 < 0 || !d_grp_of || !d_col) return gl_fail(ctx, GL_EINVAL, "gl_depthwed_add_column: bad argument");
    const int W = ctx->red.W;
    if (ctx->n_windows > 0 && ctx->rs % W != 0)
        return gl_fail(ctx, GL_EINVAL, "gl_depthwed_add_column: region start %lld is not a multiple of the window size", (long long)ctx->rs);
    CellParams p;
    memset(&p, 0, sizeof p);
    p.n = ctx->n_windows;
    p.rs = ctx->rs; p.re = ctx->re; p.wb = ctx->rs / W; p.W = W;
    p.win_sum = static_cast<const unsigned long long*>(ctx->win_sum_p);
    p.grp_of = reinterpret_cast<const int*>(d_grp_of); p.g0 = w0;
    p.col = reinterpret_cast<unsigned long long*>(d_col);
    return launch_cells(ctx, p);
}

}  // extern "C"
