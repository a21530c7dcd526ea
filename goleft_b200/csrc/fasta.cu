// fasta.cu — `goleft depth --stats`: GC / CpG / masked fraction of every emitted window
// (depth/depth.go:191-200 getStats, called for each window row at :299,:334,:355).
//
// The arithmetic lives in github.com/brentp/faidx (go.mod:11, v0.0.0-20200301150453-c39eb85760d8,
// NOT vendored under the reference tree): Faidx.Stats(chrom, start, end) scans the *raw file bytes*
// mmap[position(start) : position(end)+1) — newlines included, the extra byte only when it exists — and for every
// byte but the last of that slice counts G/C, g/c, A/T, a/t; a C/c whose NEXT BYTE is G/g is a CpG (so a CpG split
// by a line break is not one).  GC = (gc)/tot, CpG = 2*cpg/tot, Masked = (lower)/tot with tot = A+C+G+T of either
// case, all zero when tot == 0.  Restated from that package's published source; PARITY UNPINNED (no Go toolchain,
// no vendored copy, and the reference's tests assert no --stats value).
//
// Device layout: the record's bytes are uploaded once per contig (gl_fasta_load); one warp scans one
// piece (a row, or <= 64 KB of a long row) with coalesced byte loads and adds its four counts to the row.
#include "gl_common.cuh"

namespace {

constexpr unsigned kFull = 0xffffffffu;
constexpr int64_t kPiece = 1 << 16;

__device__ __forceinline__ bool is_g(unsigned char c) { return c == 'G' || c == 'g'; }

// piece q examines bytes [pa[q], pb[q]) and may look one byte ahead (index < n_bytes); counts go to row prow[q]
__global__ void __launch_bounds__(256) fasta_stats_kernel(const unsigned char* __restrict__ seq, long long n_bytes,
                                                         const long long* __restrict__ pa, const long long* __restrict__ pb,
                                                         const int* __restrict__ prow, long long n_pieces,
                                                         unsigned long long* __restrict__ counts /* [rows][4] gc, lower, tot, cpg */) {
    const long long q = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= n_pieces) return;
    const long long a = pa[q], b = pb[q];
    unsigned gc = 0, lower = 0, tot = 0, cpg = 0;
    for (long long i = a + lane; i < b; i += 32) {
        const unsigned char v = seq[i];
        const unsigned char up = v & 0xdf;                       // letters: clear the case bit
        const bool letter = (v >= 'A' && v <= 'Z') || (v >= 'a' && v <= 'z');
        const bool isgc = letter && (up == 'G' || up == 'C');
        const bool isat = letter && (up == 'A' || up == 'T');
        if (isgc | isat) {
            tot++;
            gc += isgc;
            lower += (v & 0x20) != 0;
            if (isgc && up == 'C' && i + 1 < n_bytes && is_g(seq[i + 1])) cpg++;
        }
    }
    gc = __reduce_add_sync(kFull, gc);
    lower = __reduce_add_sync(kFull, lower);
    tot = __reduce_add_sync(kFull, tot);
    cpg = __reduce_add_sync(kFull, cpg);
    if (lane == 0 && tot) {
        unsigned long long* c = counts + (size_t)prow[q] * 4;
        atomicAdd(c + 0, (unsigned long long)gc);
        atomicAdd(c + 1, (unsigned long long)lower);
        atomicAdd(c + 2, (unsigned long long)tot);
        atomicAdd(c + 3, (unsigned long long)cpg);
    }
}

}  // namespace

extern "C" {

int gl_fasta_load(gl_ctx* ctx, const uint8_t* bytes, int64_t n) {
    GL_CHECK(gl_use(ctx));
    if (n < 0 || (n > 0 && !bytes)) return gl_fail(ctx, GL_EINVAL, "gl_fasta_load: bad argument");
    GL_CHECK(gl_buf_reserve(ctx, ctx->fasta, (size_t)std::max<int64_t>(n, 16)));
    ctx->fasta_n = 0;
    if (n) GL_CUDA(ctx, cudaMemcpyAsync(ctx->fasta.p, bytes, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));            // the caller may unmap `bytes` right away
    ctx->fasta_n = n;
    return GL_OK;
}

int gl_fasta_stats(gl_ctx* ctx, const int64_t* byte_start, const int64_t* byte_end, int64_t n_rows, int64_t* counts4, double* stats3) {
    GL_CHECK(gl_use(ctx));
    if (n_rows < 0 || (n_rows > 0 && (!byte_start || !byte_end)) || (!counts4 && !stats3))
        return gl_fail(ctx, GL_EINVAL, "gl_fasta_stats: bad argument");
    if (n_rows == 0) return GL_OK;
    if (n_rows > INT32_MAX) return gl_fail(ctx, GL_ERANGE, "gl_fasta_stats: too many rows");
    // pieces: the examined bytes of row r are [byte_start, byte_end - 1) (the slice's last byte is only looked at)
    std::vector<long long> pa, pb;
    std::vector<int> prow;
    pa.reserve((size_t)n_rows); pb.reserve((size_t)n_rows); prow.reserve((size_t)n_rows);
    for (int64_t r = 0; r < n_rows; r++) {
        const int64_t a = byte_start[r], b = byte_end[r];
        if (a < 0 || b < a || b > ctx->fasta_n) return gl_fail(ctx, GL_ERANGE, "gl_fasta_stats: row %lld outside the loaded record", (long long)r);
        for (int64_t x = a; x < b - 1; x += kPiece) { pa.push_back(x); pb.push_back(std::min<int64_t>(x + kPiece, b - 1)); prow.push_back((int)r); }
    }
    const size_t np = pa.size();
    std::vector<unsigned long long> host((size_t)n_rows * 4, 0ull);
    if (np) {
        gl_scratch tmp(ctx);
        long long *d_pa, *d_pb; int* d_row; unsigned long long* d_counts;
        GL_CHECK(tmp.upload(d_pa, pa.data(), np));
        GL_CHECK(tmp.upload(d_pb, pb.data(), np));
        GL_CHECK(tmp.upload(d_row, prow.data(), np));
        GL_CHECK(tmp.alloc(d_counts, (size_t)n_rows * 4));
        GL_CUDA(ctx, cudaMemsetAsync(d_counts, 0, (size_t)n_rows * 32, ctx->stream));
        {
            gl_prof_scope prof(ctx, "fasta_stats_kernel");
            fasta_stats_kernel<<<(unsigned)((np + 7) / 8), 256, 0, ctx->stream>>>(static_cast<const unsigned char*>(ctx->fasta.p), ctx->fasta_n, d_pa, d_pb,
                                                                              d_row, (long long)np, d_counts);
        }
        GL_LAUNCHED(ctx, 1);
        GL_CUDA(ctx, cudaMemcpyAsync(host.data(), d_counts, (size_t)n_rows * 32, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    for (int64_t r = 0; r < n_rows; r++) {
        const unsigned long long gc = host[r * 4], lower = host[r * 4 + 1], tot = host[r * 4 + 2], cpg = host[r * 4 + 3];
        if (counts4) { counts4[r * 4] = (int64_t)gc; counts4[r * 4 + 1] = (int64_t)lower; counts4[r * 4 + 2] = (int64_t)tot; counts4[r * 4 + 3] = (int64_t)cpg; }
        if (stats3) {                                              // faidx Stats{GC, CpG, Masked}: the order depth.go:199 prints
            const double t = (double)tot;
            stats3[r * 3] = tot ? (double)gc / t : 0.0;
            stats3[r * 3 + 1] = tot ? (double)(2 * cpg) / t : 0.0;
            stats3[r * 3 + 2] = tot ? (double)lower / t : 0.0;
        }
    }
    return GL_OK;
}

}  // extern "C"
