// covstats.cu — covstats.BamStats's sampling loop (covstats/covstats.go:122-173) on the GPU.  The reference reads records in
// file order and stops on a count; restated without the loop it is a classification per record, two running counts and a
// cut (DESIGN §2 V1).  Only COMPRESSED bytes cross PCIe; the samples stay in HBM and only histograms and counters come back.
//
//   host        the record-aligned unit starts of the whole file from the BAI (every reference's linear-index offsets, in
//               file order), cut into batches by compressed bytes; batch k+1 is pread into pinned memory by a helper thread
//               while batch k is on the device
//   K_inflate   one warp per BGZF member (inflate.cu)
//   K_units     one thread per unit follows block_size: pass 1 counts its records, a scan places the units, pass 2 writes
//               every record's offset
//   K_fields    one thread per record: class bits, read length, insert, template length; per-CTA counts of the records that
//               give a length (g) and of the eligible pairs (e)
//   K_cut       scan of g and e with the counts carried in from earlier batches: the record the sample ends at
//   K_compact   lengths, inserts and templates before the cut to their place in file order; the five counters
//   K_minmax + bincount_kernel (indexcov.cu)   the three histograms the tail reads (host/covstats.h)
// Anything unexpected makes the call return GL_ESTATE before any result is reported, and the caller takes the host route for
// the whole file.
#include "gl_common.cuh"
#include "ll_scan.cuh"
#include "host/bam_cigar.h"
#include "host/bam_feed.h"
#include "host/covstats.h"
#include <limits.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>
#include <chrono>
#include <future>

extern "C" int gl_bgzf_inflate_device(gl_ctx* ctx, const uint8_t* d_comp, const int64_t* d_comp_off, const int64_t* d_out_off, int64_t n_blocks,
                                      uint8_t* d_out, int32_t* d_status);

namespace {

constexpr int kCta = 256;
enum : unsigned char {
    kUnmapped = 1, kMapped = 2, kBad = 4, kDup = 8, kProper = 16,
    kLen = 32,        // good and its CIGAR lies inside the record: gives a read length, counts in g
    kElig = 64,       // ... and a proper pair's left mate with one M op: gives an insert and a template, counts in e
};
constexpr unsigned long long kNoCut = ~0ull;

// one thread per unit: the records in [unit_pos[u], unit_pos[u+1]) of the inflated stream.  kEmit = false: count them;
// kEmit = true: write the offset of each record's block_size field from rec_off[off[u]] on.  The units tile the stream at
// record starts, so a record that crosses a unit's end means the index lied.
template <bool kEmit>
__global__ void __launch_bounds__(128) cs_units_kernel(const unsigned char* __restrict__ data, const long long* __restrict__ unit_pos, int n_units,
                                                      long long* __restrict__ cnt, const long long* __restrict__ off,
                                                      long long* __restrict__ rec_off, unsigned long long* __restrict__ err) {
    const int u = blockIdx.x * blockDim.x + threadIdx.x;
    if (u >= n_units) return;
    long long p = unit_pos[u];
    const long long pe = unit_pos[u + 1];
    long long n = 0, out = kEmit ? off[u] : 0;
    bool bad = false;
    while (p < pe) {
        if (p + 36 > pe) { bad = true; break; }
        const unsigned bs = glbam::ld_u32(data + p);
        if (bs < 32 || p + 4 + (long long)bs > pe) { bad = true; break; }
        if (kEmit) rec_off[out++] = p;
        n++;
        p += 4 + (long long)bs;
    }
    if (!kEmit) {
        cnt[u] = n;
        if (bad) atomicAdd(err, 1ull);
    }
}

// one thread per record (covstats.go:144-172).  first = the file index of the batch's first record.
__global__ void __launch_bounds__(kCta) cs_fields_kernel(const unsigned char* __restrict__ data, const long long* __restrict__ rec_off, long long n_rec,
                                                        long long first, long long skip, unsigned char* __restrict__ cls, int* __restrict__ f_len,
                                                        int* __restrict__ f_ins, int* __restrict__ f_tmpl, long long* __restrict__ cta_ge) {
    const long long i = (long long)blockIdx.x * kCta + threadIdx.x;
    unsigned char c = 0;
    int read_len = 0, ins = 0, tl = 0;
    if (i < n_rec && first + i >= skip) {
        const long long p = rec_off[i];
        const unsigned bs = glbam::ld_u32(data + p);
        const unsigned char* r = data + p + 4;
        const unsigned l_name = r[8], n_cig = (unsigned)r[12] | ((unsigned)r[13] << 8), flag = (unsigned)r[14] | ((unsigned)r[15] << 8);
        if (flag & 0x4u) c = kUnmapped;
        else if (flag & 0x600u) c = kMapped | kBad | ((flag & 0x400u) ? kDup : 0);
        else {
            c = kMapped | ((flag & 0x2u) ? kProper : 0);
            if (32u + l_name + 4u * n_cig <= bs) {
                c |= kLen;
                const unsigned char* cg = r + 32 + l_name;
                int ref_len = 0;
                for (unsigned k = 0; k < n_cig; k++) {
                    const unsigned v = glbam::ld_u32(cg + 4 * k), op = v & 15u;
                    const int len = (int)(v >> 4);
                    if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) ref_len += len;
                    if (op == 0 || op == 1 || op == 4 || op == 7 || op == 8) read_len += len;
                }
                const int pos = (int)glbam::ld_u32(r + 4), mate_pos = (int)glbam::ld_u32(r + 24);
                if (pos < mate_pos && (flag & 0x2u) && n_cig == 1 && (glbam::ld_u32(cg) & 15u) == 0) {
                    c |= kElig;
                    ins = mate_pos - (pos + ref_len);
                    tl = (int)glbam::ld_u32(r + 28);
                }
            }
        }
    }
    if (i < n_rec) { cls[i] = c; f_len[i] = read_len; f_ins[i] = ins; f_tmpl[i] = tl; }
    const int g = __syncthreads_count(c & kLen), e = __syncthreads_count(c & kElig);
    if (threadIdx.x == 0) cta_ge[blockIdx.x] = ((long long)g << 32) | (long long)e;
}

// inclusive counts of the kLen and kElig records up to this thread's, from the start of the sample: cta_base = the scanned
// cta_ge of this CTA, (g0, e0) = the counts of the earlier batches.  Every thread of the CTA calls it.
__device__ __forceinline__ void cs_rank(unsigned char c, long long cta_base, long long g0, long long e0, long long& g, long long& e) {
    __shared__ int s_g[kCta / 32], s_e[kCta / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned bg = __ballot_sync(0xffffffffu, c & kLen), be = __ballot_sync(0xffffffffu, c & kElig);
    const unsigned upto = 0xffffffffu >> (31 - lane);
    int ig = __popc(bg & upto), ie = __popc(be & upto);
    if (lane == 0) { s_g[warp] = __popc(bg); s_e[warp] = __popc(be); }
    __syncthreads();
    for (int k = 0; k < warp; k++) { ig += s_g[k]; ie += s_e[k]; }
    g = g0 + (cta_base >> 32) + ig;
    e = e0 + (cta_base & 0xffffffffll) + ie;
}

// cut A: the eligible record with e == n.  cut B: the kLen record with g == 2n + 1, if no insert came before it.  Each exists
// at most once; the smaller key wins, and B's key is the smaller one on the same record (covstats.go:159-167 comes first).
__global__ void __launch_bounds__(kCta) cs_cut_kernel(const unsigned char* __restrict__ cls, long long n_rec, const long long* __restrict__ cta_scan,
                                                     long long g0, long long e0, long long n, unsigned long long* __restrict__ cut_key) {
    const long long i = (long long)blockIdx.x * kCta + threadIdx.x;
    const unsigned char c = i < n_rec ? cls[i] : 0;
    long long g, e;
    cs_rank(c, cta_scan[blockIdx.x], g0, e0, g, e);
    if ((c & kLen) && g == 2 * n + 1 && e - ((c & kElig) ? 1 : 0) == 0) atomicMin(cut_key, (unsigned long long)i * 2);
    if ((c & kElig) && e == n) atomicMin(cut_key, (unsigned long long)i * 2 + 1);
}

// ctr: n_unmapped, k, n_bad, n_dup, n_proper, g, e, over the records up to the cut
__global__ void __launch_bounds__(kCta) cs_compact_kernel(const unsigned char* __restrict__ cls, const int* __restrict__ f_len, const int* __restrict__ f_ins,
                                                         const int* __restrict__ f_tmpl, long long n_rec, const long long* __restrict__ cta_scan,
                                                         long long g0, long long e0, long long n, const unsigned long long* __restrict__ cut_key,
                                                         int* __restrict__ out_len, int* __restrict__ out_ins, int* __restrict__ out_tmpl,
                                                         unsigned long long* __restrict__ ctr) {
    const long long i = (long long)blockIdx.x * kCta + threadIdx.x;
    const unsigned long long key = *cut_key;
    const long long last = key == kNoCut ? n_rec - 1 : (long long)(key >> 1);
    unsigned char c = (i < n_rec && i <= last) ? cls[i] : 0;
    if (key != kNoCut && !(key & 1) && i == last) c &= ~(kLen | kElig);      // cut B's record: counted, no length, no insert
    long long g, e;
    cs_rank(c, cta_scan[blockIdx.x], g0, e0, g, e);
    if ((c & kLen) && g <= 2 * n) out_len[g - 1] = f_len[i];
    if (c & kElig) { out_ins[e - 1] = f_ins[i]; out_tmpl[e - 1] = f_tmpl[i]; }
    const unsigned char bits[7] = {kUnmapped, kMapped, kBad, kDup, kProper, kLen, kElig};
#pragma unroll
    for (int k = 0; k < 7; k++) {
        const int s = __syncthreads_count(c & bits[k]);
        if (threadIdx.x == 0 && s) atomicAdd(ctr + k, (unsigned long long)s);
    }
}

// mm[0] = min, mm[1] = max of v[0..n) (mm starts at INT_MAX, INT_MIN)
__global__ void __launch_bounds__(kCta) cs_minmax_kernel(const int* __restrict__ v, long long n, int* __restrict__ mm) {
    int lo = INT_MAX, hi = INT_MIN;
    for (long long i = (long long)blockIdx.x * kCta + threadIdx.x; i < n; i += (long long)gridDim.x * kCta) { const int x = v[i]; lo = min(lo, x); hi = max(hi, x); }
#pragma unroll
    for (int o = 16; o; o >>= 1) { lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
    if ((threadIdx.x & 31) == 0 && lo <= hi) { atomicMin(mm, lo); atomicMax(mm + 1, hi); }
}

double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }
inline uint16_t rd16(const uint8_t* p) { return (uint16_t)(p[0] | (p[1] << 8)); }
inline uint32_t rd32(const uint8_t* p) { return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24); }
inline size_t al(size_t x) { return (x + 255) & ~size_t(255); }

constexpr int64_t kLaterBatch = int64_t(64) << 20;     // compressed bytes per batch after the first
constexpr int64_t kMaxTail = int64_t(64) << 20;        // the unplaced tail is one unit: one thread walks it
constexpr int kEvents = 7;

// what the helper thread makes of one batch: the compressed bytes of units [i0, i1) in pinned memory, the member table and
// the units' positions in the batch's inflated stream
struct Batch {
    size_t i0 = 0, i1 = 0;
    int64_t c0 = 0;
    size_t nbytes = 0;
    uint8_t* h = nullptr;
    std::vector<int64_t> comp_off, out_off;
    std::vector<long long> unit_pos;
    const char* err = nullptr;
};

// gl_bam_covstats_prefetch: the first batch of `b` for a later gl_bam_covstats(ctx, b, n, skip), read by `f` into pin[2]
struct Prefetch {
    gl_bam* b = nullptr;
    int32_t n = 0, skip = 0;
    std::vector<uint64_t> bound;
    Batch B;
    std::future<void> f;
};

struct CsState {
    gl_buf comp, infl, rec, hist;                      // compressed + tables, inflated stream, per-record arrays, histogram
    gl_buf s_len, s_ins, s_tmpl;                       // the samples, file order
    void* pin[3] = {nullptr, nullptr, nullptr};        // [0], [1]: a call's batches; [2]: the prefetched first batch
    size_t pin_cap[3] = {0, 0, 0};
    cudaEvent_t ev[kEvents] = {};
    Prefetch pf;
};

void load_batch(int fd, const std::vector<uint64_t>& bound, Batch& B) {
    for (size_t got = 0; got < B.nbytes;) {
        const ssize_t k = pread(fd, B.h + got, B.nbytes - got, B.c0 + (int64_t)got);
        if (k <= 0) { B.err = "read failed"; return; }
        got += (size_t)k;
    }
    const uint64_t v1 = bound[B.i1];
    const int64_t last_c = (int64_t)(v1 >> 16) - B.c0;
    B.comp_off.assign(1, 0); B.out_off.assign(1, 0);
    const uint8_t* h = B.h;
    size_t q = 0;
    while (q + 18 <= B.nbytes) {
        if ((int64_t)q > last_c || ((int64_t)q == last_c && (v1 & 0xffff) == 0)) break;
        if (h[q] != 0x1f || h[q + 1] != 0x8b || h[q + 2] != 8 || !(h[q + 3] & 4) || h[q + 10] != 6 || h[q + 11] != 0 || h[q + 12] != 'B' || h[q + 13] != 'C') {
            B.err = "unexpected BGZF header layout"; return;
        }
        const size_t bs = (size_t)rd16(h + q + 16) + 1;
        if (bs < 26 || q + bs > B.nbytes) break;
        const uint32_t isize = rd32(h + q + bs - 4);
        if (isize > 65536) { B.err = "bad ISIZE"; return; }
        q += bs;
        B.comp_off.push_back((int64_t)q);
        B.out_off.push_back(B.out_off.back() + isize);
    }
    const size_t n_blocks = B.comp_off.size() - 1;
    B.unit_pos.clear();
    for (size_t i = B.i0; i <= B.i1; i++) {
        const int64_t c = (int64_t)(bound[i] >> 16) - B.c0;
        const int64_t o = (int64_t)(bound[i] & 0xffff);
        const auto it = std::lower_bound(B.comp_off.begin(), B.comp_off.end(), c);
        if (it == B.comp_off.end() || *it != c) { B.err = "index offsets do not land on members"; return; }
        const size_t blk = (size_t)(it - B.comp_off.begin());
        if (blk >= n_blocks ? o != 0 : o > B.out_off[blk + 1] - B.out_off[blk]) { B.err = "index offsets do not land on members"; return; }
        const long long p = B.out_off[blk] + o;
        if (!B.unit_pos.empty() && p < B.unit_pos.back()) { B.err = "index offsets are not in file order"; return; }
        B.unit_pos.push_back(p);
    }
}

// unit boundaries of the whole file, as virtual offsets in file order: the first record, every reference's chunk range and
// linear-index offsets, end of file.  The last unit is the unplaced tail.  Returns why the device cannot take the file, or
// an empty string.
std::string cs_bounds(glhts::BamFile& F, std::vector<uint64_t>& bound) {
    bound.clear();
    if (!F.has_index || F.fd() < 0) return "no index";
    if (F.rec_skip() > 65535) return "the header ends a 64 KB member";
    const uint64_t v_first = ((uint64_t)F.rec_member() << 16) | F.rec_skip(), v_eof = (uint64_t)F.file_size() << 16;
    for (size_t t = 0; t < F.bai.ioffsets.size(); t++) {
        const uint64_t vbeg = t < F.bai.ref_beg.size() ? F.bai.ref_beg[t] : 0, vend = t < F.bai.ref_end.size() ? F.bai.ref_end[t] : 0;
        if (vbeg == 0 || vend <= vbeg) {
            for (uint64_t v : F.bai.ioffsets[t]) if (v) return "the index has no chunk range for reference " + std::to_string(t);
            continue;
        }
        bound.push_back(vbeg); bound.push_back(vend);
        for (uint64_t v : F.bai.ioffsets[t]) if (v > vbeg && v < vend) bound.push_back(v);
    }
    bound.push_back(v_first); bound.push_back(v_eof);
    std::sort(bound.begin(), bound.end());
    bound.erase(std::unique(bound.begin(), bound.end()), bound.end());
    if (bound.front() != v_first || bound.back() != v_eof) return "index offsets outside the file's records";
    return "";
}

// compressed bytes of the first batch (sized to the sample) and of the later ones; GL_COVSTATS_BATCH_BYTES sets both
void cs_batch_bytes(int32_t n, int32_t skip, int64_t& first, int64_t& later) {
    first = std::min<int64_t>(std::max<int64_t>(((int64_t)skip + 3 * (int64_t)n) * 40, int64_t(8) << 20), int64_t(192) << 20);
    later = kLaterBatch;
    if (const char* v = getenv("GL_COVSTATS_BATCH_BYTES")) { const long long x = atoll(v); if (x > 0) first = later = x; }
}

// units [i0, i1) of the batch that starts at i0: as many as fit the byte bound, at least one.  Returns why the device cannot
// take the batch, or nullptr.
const char* cs_plan(const glhts::BamFile& F, const std::vector<uint64_t>& bound, size_t i0, int64_t bytes, Batch& B) {
    const size_t n_bound = bound.size();
    size_t i1 = i0 + 1;
    while (i1 + 1 < n_bound && (int64_t)(bound[i1 + 1] >> 16) - (int64_t)(bound[i0] >> 16) <= bytes) i1++;
    B.i0 = i0; B.i1 = i1;
    B.c0 = (int64_t)(bound[i0] >> 16);
    const int64_t c1 = std::min<int64_t>(F.file_size(), (int64_t)(bound[i1] >> 16) + 65536 + 64);
    if (i1 == n_bound - 1 && c1 - (int64_t)(bound[i1 - 1] >> 16) > kMaxTail) return "the sample reaches a large unplaced tail";
    if (c1 - B.c0 > (int64_t(1) << 31)) return "a unit of more than 2 GB";
    B.nbytes = (size_t)(c1 - B.c0);
    return nullptr;
}

int cs_state(gl_ctx* ctx, CsState*& S) {
    if (!ctx->cs) {
        CsState* N = new CsState();
        ctx->cs = N;
        for (auto& e : N->ev) GL_CUDA(ctx, cudaEventCreate(&e));
    }
    S = static_cast<CsState*>(ctx->cs);
    return GL_OK;
}

int pin_reserve(gl_ctx* ctx, CsState* S, int k, size_t bytes) {
    if (S->pin_cap[k] >= bytes) return GL_OK;
    if (S->pin[k]) cudaFreeHost(S->pin[k]);
    S->pin[k] = nullptr; S->pin_cap[k] = 0;
    const size_t want = bytes + bytes / 4;
    if (cudaHostAlloc(&S->pin[k], want, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); S->pin[k] = nullptr; return gl_fail(ctx, GL_ENOMEM, "cudaHostAlloc(%zu)", want); }
    S->pin_cap[k] = want;
    return GL_OK;
}

// grows a sample array, keeping its first `keep` ints
int grow_keep(gl_ctx* ctx, gl_buf& b, size_t ints, size_t keep) {
    if (ints * 4 <= b.cap) return GL_OK;
    gl_buf nb;
    GL_CHECK(gl_buf_reserve(ctx, nb, std::max(ints * 4, b.cap * 2)));
    if (keep) GL_CUDA(ctx, cudaMemcpyAsync(nb.p, b.p, keep * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (b.p) cudaFree(b.p);
    b = nb;
    return GL_OK;
}

// the multiset of n device ints: min and max on the device, then bincount_kernel into a device histogram and only the
// histogram comes back; a range wider than kMaxHistRange brings the samples back to be sorted
int device_counts(gl_ctx* ctx, CsState* S, const int32_t* d_v, int64_t n, glcs::SortedCounts& out) {
    out = glcs::SortedCounts();
    if (n == 0) return GL_OK;
    GL_CHECK(gl_buf_reserve(ctx, S->hist, 256));
    int* d_mm = static_cast<int*>(S->hist.p);
    int mm[2] = {INT_MAX, INT_MIN};
    GL_CUDA(ctx, cudaMemcpyAsync(d_mm, mm, 8, cudaMemcpyHostToDevice, ctx->stream));
    cs_minmax_kernel<<<(unsigned)std::min<int64_t>((n + kCta - 1) / kCta, (int64_t)ctx->sm_count * 8), kCta, 0, ctx->stream>>>(d_v, n, d_mm);
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaMemcpyAsync(mm, d_mm, 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const long long range = (long long)mm[1] - mm[0] + 1;
    if (range > glcs::kMaxHistRange || mm[1] == INT32_MAX) {
        std::vector<int32_t> v((size_t)n);
        GL_CUDA(ctx, cudaMemcpyAsync(v.data(), d_v, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        out.from_values(v.data(), v.size());
        return GL_OK;
    }
    GL_CHECK(gl_buf_reserve(ctx, S->hist, (size_t)range * 8));
    std::vector<uint64_t> h((size_t)range);
    GL_CHECK(gl_bincount_device(ctx, d_v, n, mm[0], mm[1] + 1, static_cast<unsigned long long*>(S->hist.p)));
    GL_CUDA(ctx, cudaMemcpyAsync(h.data(), S->hist.p, (size_t)range * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    out.from_hist(mm[0], std::move(h));
    return GL_OK;
}

}  // namespace

void cs_prefetch_drop(gl_ctx* ctx) {
    CsState* S = static_cast<CsState*>(ctx->cs);
    if (!S || !S->pf.b) return;
    if (S->pf.f.valid()) S->pf.f.wait();
    S->pf.b->cs_pf = nullptr;
    S->pf = Prefetch();
}

void cs_free(gl_ctx* ctx) {
    CsState* S = static_cast<CsState*>(ctx->cs);
    if (!S) return;
    cs_prefetch_drop(ctx);
    for (gl_buf* b : {&S->comp, &S->infl, &S->rec, &S->hist, &S->s_len, &S->s_ins, &S->s_tmpl}) if (b->p) cudaFree(b->p);
    for (void* p : S->pin) if (p) cudaFreeHost(p);
    for (cudaEvent_t e : S->ev) if (e) cudaEventDestroy(e);
    delete S;
    ctx->cs = nullptr;
}

extern "C" {

int gl_bam_covstats(gl_ctx* ctx, gl_bam* b, int32_t n, int32_t skip, gl_covstats* out, double* H, int64_t h_cap) {
    GL_CHECK(gl_use(ctx));
    if (!b || !out) return gl_fail(ctx, GL_EINVAL, "gl_bam_covstats: null argument");
    memset(out, 0, sizeof *out);
    out->path = 1;
    const double t_wall = now_s();
    CsState* S = nullptr;
    GL_CHECK(cs_state(ctx, S));
    glhts::BamFile& F = b->f;
    std::vector<uint64_t> bound;
    Batch bat[2];
    // a prefetch of this handle: consumed when it was made for this n and skip, discarded otherwise
    const bool pre = S->pf.b == b && S->pf.n == n && S->pf.skip == skip;
    if (pre) {
        const double t0 = now_s();
        S->pf.f.wait();
        out->read_s += now_s() - t0;
        bound = std::move(S->pf.bound);
        bat[0] = std::move(S->pf.B);
        out->prefetched = 1;
    }
    if (S->pf.b == b) cs_prefetch_drop(ctx);
    if (!pre) {
        const std::string e = cs_bounds(F, bound);
        if (!e.empty()) return gl_fail(ctx, GL_ESTATE, "gl_bam_covstats: %s", e.c_str());
    }
    const size_t n_bound = bound.size();

    long long g0 = 0, e0 = 0, first = 0;                 // lengths and inserts so far; file index of the next batch's first record
    unsigned long long ctr[7] = {0, 0, 0, 0, 0, 0, 0};
    bool cut = false;
    if (n > 0 && n_bound >= 2) {
        int64_t batch_first, batch_later;
        cs_batch_bytes(n, skip, batch_first, batch_later);
        auto plan = [&](size_t i0, int64_t bytes, Batch& B) -> int {
            const char* e = cs_plan(F, bound, i0, bytes, B);
            return e ? gl_fail(ctx, GL_ESTATE, "gl_bam_covstats: %s", e) : GL_OK;
        };
        std::future<void> pending;
        // the helper thread must be joined on every return path: it writes into this frame and into pinned memory
        struct Join { std::future<void>& f; ~Join() { if (f.valid()) f.wait(); } } join{pending};
        int cur = 0;
        if (!pre) {
            GL_CHECK(plan(0, batch_first, bat[0]));
            GL_CHECK(pin_reserve(ctx, S, 0, bat[0].nbytes + 256));
            bat[0].h = static_cast<uint8_t*>(S->pin[0]);
            const double t0 = now_s();
            load_batch(F.fd(), bound, bat[0]);
            out->read_s += now_s() - t0;
        }
        for (;;) {
            Batch& B = bat[cur];
            if (B.err) return gl_fail(ctx, GL_ESTATE, "gl_bam_covstats: %s", B.err);
            // the next batch is read while this one is on the device
            Batch& Nx = bat[cur ^ 1];
            const bool more = B.i1 < n_bound - 1;
            if (more) {
                GL_CHECK(plan(B.i1, batch_later, Nx));
                GL_CHECK(pin_reserve(ctx, S, cur ^ 1, Nx.nbytes + 256));
                Nx.h = static_cast<uint8_t*>(S->pin[cur ^ 1]);
                Nx.err = nullptr;
                const int fd = F.fd();
                pending = std::async(std::launch::async, [fd, &bound, &Nx] { load_batch(fd, bound, Nx); });
            }
            out->n_batches++;
            const int64_t n_blocks = (int64_t)B.comp_off.size() - 1;
            const int n_units = (int)(B.i1 - B.i0);
            const int64_t inflated = B.out_off.back();
            const size_t used = (size_t)B.comp_off.back();
            if (B.unit_pos.back() > inflated) return gl_fail(ctx, GL_ESTATE, "gl_bam_covstats: index offsets do not land on members");
            // ---- device buffers: compressed | member tables | status | unit tables | counters, cut key, error
            const size_t tab = al((size_t)(n_blocks + 1) * 8) * 2 + al((size_t)n_blocks * 4 + 4) + al((size_t)(n_units + 2) * 8) * 3 + al(128);
            GL_CHECK(gl_buf_reserve(ctx, S->comp, al(used) + tab));
            GL_CHECK(gl_buf_reserve(ctx, S->infl, (size_t)inflated + 256));
            char* q = static_cast<char*>(S->comp.p);
            uint8_t* d_comp = reinterpret_cast<uint8_t*>(q); q += al(used);
            int64_t* d_coff = reinterpret_cast<int64_t*>(q); q += al((size_t)(n_blocks + 1) * 8);
            int64_t* d_ooff = reinterpret_cast<int64_t*>(q); q += al((size_t)(n_blocks + 1) * 8);
            int32_t* d_stat = reinterpret_cast<int32_t*>(q); q += al((size_t)n_blocks * 4 + 4);
            long long* d_upos = reinterpret_cast<long long*>(q); q += al((size_t)(n_units + 2) * 8);
            long long* d_ucnt = reinterpret_cast<long long*>(q); q += al((size_t)(n_units + 2) * 8);
            long long* d_uoff = reinterpret_cast<long long*>(q); q += al((size_t)(n_units + 2) * 8);
            unsigned long long* d_small = reinterpret_cast<unsigned long long*>(q);      // [0..6] ctr, [8] cut key, [9] malformed units
            const unsigned char* d_data = static_cast<const unsigned char*>(S->infl.p);
            unsigned long long small0[10] = {ctr[0], ctr[1], ctr[2], ctr[3], ctr[4], ctr[5], ctr[6], 0, kNoCut, 0};
            GL_CUDA(ctx, cudaEventRecord(S->ev[0], ctx->stream));
            GL_CUDA(ctx, cudaMemcpyAsync(d_comp, B.h, used, cudaMemcpyHostToDevice, ctx->stream));
            GL_CUDA(ctx, cudaMemcpyAsync(d_coff, B.comp_off.data(), (size_t)(n_blocks + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
            GL_CUDA(ctx, cudaMemcpyAsync(d_ooff, B.out_off.data(), (size_t)(n_blocks + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
            GL_CUDA(ctx, cudaMemcpyAsync(d_upos, B.unit_pos.data(), (size_t)(n_units + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
            GL_CUDA(ctx, cudaMemcpyAsync(d_small, small0, sizeof small0, cudaMemcpyHostToDevice, ctx->stream));
            GL_CHECK(gl_bgzf_inflate_device(ctx, d_comp, d_coff, d_ooff, n_blocks, static_cast<uint8_t*>(S->infl.p), d_stat));
            GL_CUDA(ctx, cudaEventRecord(S->ev[1], ctx->stream));
            {
                gl_prof_scope prof(ctx, "cs_units_count_kernel");
                cs_units_kernel<false><<<(unsigned)((n_units + 127) / 128), 128, 0, ctx->stream>>>(d_data, d_upos, n_units, d_ucnt, nullptr, nullptr, d_small + 9);
                GL_LAUNCHED(ctx, 1);
            }
            ll_scan_kernel<<<1, 1024, 0, ctx->stream>>>(d_ucnt, d_uoff, n_units);
            GL_LAUNCHED(ctx, 1);
            GL_CUDA(ctx, cudaEventRecord(S->ev[2], ctx->stream));
            unsigned long long n_bad_units = 0;
            long long n_rec = 0;
            std::vector<int32_t> st_host((size_t)n_blocks);
            GL_CUDA(ctx, cudaMemcpyAsync(&n_bad_units, d_small + 9, 8, cudaMemcpyDeviceToHost, ctx->stream));
            GL_CUDA(ctx, cudaMemcpyAsync(&n_rec, d_uoff + n_units, 8, cudaMemcpyDeviceToHost, ctx->stream));
            if (n_blocks) GL_CUDA(ctx, cudaMemcpyAsync(st_host.data(), d_stat, (size_t)n_blocks * 4, cudaMemcpyDeviceToHost, ctx->stream));
            GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
            for (int32_t sb : st_host) if (sb != 0) return gl_fail(ctx, GL_ESTATE, "gl_bam_covstats: a BGZF member was rejected by the device inflater (status %d)", sb);
            if (n_bad_units) return gl_fail(ctx, GL_ESTATE, "gl_bam_covstats: malformed BAM record, or index offsets that are not record starts");
            out->bytes_in += (int64_t)used; out->bytes_out += inflated;
            float ms = 0;
            cudaEventElapsedTime(&ms, S->ev[0], S->ev[1]); out->inflate_s += ms * 1e-3;      // the upload and K_inflate
            cudaEventElapsedTime(&ms, S->ev[1], S->ev[2]); out->index_s += ms * 1e-3;
            long long last = -1;
            if (n_rec > 0) {
                const long long n_cta = (n_rec + kCta - 1) / kCta;
                // ---- per-record arrays: offsets | length, insert, template | class | CTA counts and their scan
                const size_t rec_bytes = al((size_t)n_rec * 8) + al((size_t)n_rec * 4) * 3 + al((size_t)n_rec) + al((size_t)(n_cta + 2) * 8) * 2;
                GL_CHECK(gl_buf_reserve(ctx, S->rec, rec_bytes));
                char* r = static_cast<char*>(S->rec.p);
                long long* d_roff = reinterpret_cast<long long*>(r); r += al((size_t)n_rec * 8);
                int* d_flen = reinterpret_cast<int*>(r); r += al((size_t)n_rec * 4);
                int* d_fins = reinterpret_cast<int*>(r); r += al((size_t)n_rec * 4);
                int* d_ftl = reinterpret_cast<int*>(r); r += al((size_t)n_rec * 4);
                unsigned char* d_cls = reinterpret_cast<unsigned char*>(r); r += al((size_t)n_rec);
                long long* d_ge = reinterpret_cast<long long*>(r); r += al((size_t)(n_cta + 2) * 8);
                long long* d_ge_scan = reinterpret_cast<long long*>(r);
                GL_CHECK(grow_keep(ctx, S->s_len, (size_t)std::min<long long>(2ll * n, g0 + n_rec), (size_t)std::min<long long>(2ll * n, g0)));
                GL_CHECK(grow_keep(ctx, S->s_ins, (size_t)std::min<long long>(n, e0 + n_rec), (size_t)e0));
                GL_CHECK(grow_keep(ctx, S->s_tmpl, (size_t)std::min<long long>(n, e0 + n_rec), (size_t)e0));
                GL_CUDA(ctx, cudaEventRecord(S->ev[3], ctx->stream));       // the host has looked at the record count in between
                {
                    gl_prof_scope prof(ctx, "cs_units_emit_kernel");
                    cs_units_kernel<true><<<(unsigned)((n_units + 127) / 128), 128, 0, ctx->stream>>>(d_data, d_upos, n_units, nullptr, d_uoff, d_roff, nullptr);
                    GL_LAUNCHED(ctx, 1);
                }
                GL_CUDA(ctx, cudaEventRecord(S->ev[4], ctx->stream));
                {
                    gl_prof_scope prof(ctx, "cs_fields_kernel");
                    cs_fields_kernel<<<(unsigned)n_cta, kCta, 0, ctx->stream>>>(d_data, d_roff, n_rec, first, (long long)skip, d_cls, d_flen, d_fins, d_ftl, d_ge);
                    GL_LAUNCHED(ctx, 1);
                }
                GL_CUDA(ctx, cudaEventRecord(S->ev[5], ctx->stream));
                ll_scan_kernel<<<1, 1024, 0, ctx->stream>>>(d_ge, d_ge_scan, (int)n_cta);
                GL_LAUNCHED(ctx, 1);
                {
                    gl_prof_scope prof(ctx, "cs_cut_kernel");
                    cs_cut_kernel<<<(unsigned)n_cta, kCta, 0, ctx->stream>>>(d_cls, n_rec, d_ge_scan, g0, e0, (long long)n, d_small + 8);
                    GL_LAUNCHED(ctx, 1);
                }
                {
                    gl_prof_scope prof(ctx, "cs_compact_kernel");
                    cs_compact_kernel<<<(unsigned)n_cta, kCta, 0, ctx->stream>>>(d_cls, d_flen, d_fins, d_ftl, n_rec, d_ge_scan, g0, e0, (long long)n, d_small + 8,
                                                                              static_cast<int*>(S->s_len.p), static_cast<int*>(S->s_ins.p),
                                                                              static_cast<int*>(S->s_tmpl.p), d_small);
                    GL_LAUNCHED(ctx, 1);
                }
                GL_CUDA(ctx, cudaEventRecord(S->ev[6], ctx->stream));
                unsigned long long back[9];
                GL_CUDA(ctx, cudaMemcpyAsync(back, d_small, sizeof back, cudaMemcpyDeviceToHost, ctx->stream));
                GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
                memcpy(ctr, back, sizeof ctr);
                cudaEventElapsedTime(&ms, S->ev[3], S->ev[4]); out->index_s += ms * 1e-3;
                cudaEventElapsedTime(&ms, S->ev[4], S->ev[5]); out->fields_s += ms * 1e-3;
                cudaEventElapsedTime(&ms, S->ev[5], S->ev[6]); out->cut_s += ms * 1e-3;
                g0 = (long long)ctr[5]; e0 = (long long)ctr[6];
                if (back[8] != kNoCut) { cut = true; last = (long long)(back[8] >> 1); }
            }
            out->n_records_read = first + (cut ? last + 1 : n_rec);
            first += n_rec;
            const double t_wait = now_s();
            if (pending.valid()) pending.wait();
            out->read_s += now_s() - t_wait;
            if (cut || !more) break;
            cur ^= 1;
        }
    }
    out->n_unmapped = (int64_t)ctr[0]; out->k = (int64_t)ctr[1]; out->n_bad = (int64_t)ctr[2]; out->n_dup = (int64_t)ctr[3]; out->n_proper = (int64_t)ctr[4];
    const long long n_len = std::min<long long>(g0, 2ll * std::max(n, 0)), n_ins = e0;
    // ---- the tail: three histograms made on the device, then host/covstats.h
    const double t_tail = now_s();
    glcs::SortedCounts rl, ins, tm;
    GL_CHECK(device_counts(ctx, S, static_cast<const int32_t*>(S->s_len.p), n_len, rl));
    GL_CHECK(device_counts(ctx, S, static_cast<const int32_t*>(S->s_ins.p), n_ins, ins));
    GL_CHECK(device_counts(ctx, S, static_cast<const int32_t*>(S->s_tmpl.p), n_ins, tm));
    std::vector<double> h;
    const int rc = glcs::tail(ctx, rl, ins, tm, out, h);
    out->tail_s = now_s() - t_tail;
    out->wall_s = now_s() - t_wall;
    if (rc != GL_OK) return rc;
    return glcs::put_hist(ctx, h, H, h_cap);
}

int gl_bam_covstats_samples(gl_ctx* ctx, const int32_t** d_read_len, const int32_t** d_insert, const int32_t** d_tmpl) {
    if (!ctx || !d_read_len || !d_insert || !d_tmpl) return gl_fail(ctx, GL_EINVAL, "gl_bam_covstats_samples: null argument");
    CsState* S = static_cast<CsState*>(ctx->cs);
    if (!S) return gl_fail(ctx, GL_ESTATE, "gl_bam_covstats_samples: no gl_bam_covstats call on this ctx");
    *d_read_len = static_cast<const int32_t*>(S->s_len.p); *d_insert = static_cast<const int32_t*>(S->s_ins.p); *d_tmpl = static_cast<const int32_t*>(S->s_tmpl.p);
    return GL_OK;
}

int gl_bam_covstats_prefetch(gl_ctx* ctx, gl_bam* next, int32_t n, int32_t skip) {
    GL_CHECK(gl_use(ctx));
    if (!next) return gl_fail(ctx, GL_EINVAL, "gl_bam_covstats_prefetch: null argument");
    CsState* S = nullptr;
    GL_CHECK(cs_state(ctx, S));
    cs_prefetch_drop(ctx);
    if (next->cs_pf) cs_prefetch_drop(next->cs_pf);       // made on another ctx
    if (n <= 0) return GL_OK;
    // a file the device would refuse gets no prefetch: gl_bam_covstats reports it
    Prefetch& P = S->pf;
    if (!cs_bounds(next->f, P.bound).empty() || P.bound.size() < 2) { P.bound.clear(); return GL_OK; }
    int64_t batch_first, batch_later;
    cs_batch_bytes(n, skip, batch_first, batch_later);
    if (cs_plan(next->f, P.bound, 0, batch_first, P.B)) { P = Prefetch(); return GL_OK; }
    const int rc = pin_reserve(ctx, S, 2, P.B.nbytes + 256);
    if (rc != GL_OK) { P = Prefetch(); return rc; }
    P.B.h = static_cast<uint8_t*>(S->pin[2]);
    P.b = next; P.n = n; P.skip = skip;
    next->cs_pf = ctx;
    const int fd = next->f.fd();
    P.f = std::async(std::launch::async, [fd, &P] { load_batch(fd, P.bound, P.B); });
    return GL_OK;
}

}  // extern "C"
