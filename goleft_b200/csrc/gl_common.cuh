// gl_common.cuh — context object and error plumbing shared by every translation unit of
// libgoleft_b200.so.  sm_90a only; there is no CPU fallback anywhere in this library.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>
#include <algorithm>
#include "../../include/goleft_b200.h"

struct gl_buf {            // grow-only device buffer
    void* p = nullptr;
    size_t cap = 0;
};

struct gl_seg_batch {      // one gl_depth_add_segments* call
    const int32_t* s = nullptr;   // device pointers (caller-owned), or null when the batch lives in the ctx store
    const int32_t* e = nullptr;
    int64_t off = 0;              // offset into the ctx store when s == nullptr
    int64_t n = 0;
};

// multidepth.cu: a second epilogue of the depth tile core (depth.cu).  It only ever OVERWRITES what it writes, so a pass the
// device rejects part way (fused paths) and depth_resolve reruns leaves no trace; multidepth.cu folds the outputs in after the
// result has been settled.
struct gl_md_ep {
    int mode = 0;                       // 0 = off (gl_depth_reduce), 1 = count, 2 = block sums
    int mincov = 0;                     // mode 1: bit (d >= mincov) -> ge16, bit (d > 0) -> pos16 (16 bases per halfword)
    unsigned short* ge16 = nullptr;
    unsigned short* pos16 = nullptr;
    const unsigned* suf = nullptr;      // mode 2: sufficient-site bitmask (32 bases per word)
    const int* pair_ptr = nullptr;      // [tiles+1] CSR: the (tile, block) pairs of each 4096-base tile
    const int* pair_blk = nullptr;      // block of each pair
    const int* blk_start = nullptr;     // region-relative [start, end) of every block
    const int* blk_end = nullptr;
    unsigned long long* slots = nullptr;   // [pairs * 8]: slot (pair, c) = Σ d over the block's sufficient sites in the tile's c-th 512 bases
};

// depth.cu: the reduce's paths, numbered as gl_depth_last_path reports them (DESIGN §1.0-1.2)
enum DepthPath : int {
    kPathNone = 0,          // last_path: nothing reduced yet; force_path: choose automatically
    kPathFused = 1,         // fused int32 (segments in BAM order)
    kPathHbmDiff = 2,       // HBM difference array (on request only)
    kPathPacked8 = 3,       // the region's only batch is packed8, read as it is
    kPathEvents = 4,        // bucketed events (the general path)
};

// depth.cu: what one reduce computes.  The defaults ask for nothing: no windows (one window per 2^30 bases), no runs.
struct ReduceArgs {
    int32_t W = 1 << 30;
    int32_t mincov = 0, maxmean = 0;
    int64_t run_break = 0;
    bool do_windows = false, do_runs = false, want_min = false;
    int32_t* d_depth_out = nullptr;     // device per-base depth (may be null)
};

struct gl_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;       // compute stream
    cudaStream_t copy_stream = nullptr;  // H2D staging stream
    cudaStream_t d2h_stream = nullptr;   // streamed packed8 reduce: finished window sums leave while later chunks arrive
    std::string err;
    int64_t launches = 0;
    int sm_count = 132;

    cudaEvent_t ev0 = nullptr, ev1 = nullptr;         // gl_timer_*
    cudaEvent_t ev_copy[2] = {nullptr, nullptr};      // staging ring
    cudaEvent_t ev_used[2] = {nullptr, nullptr};
    std::vector<cudaEvent_t> ev_chunk;                // streamed packed8 upload: one per chunk

    // ---- depth state
    bool depth_active = false, depth_reduced = false;
    int64_t rs = 0, re = 0;
    ReduceArgs red;                         // what the settled result was asked for
    int64_t n_windows = 0, n_runs = 0; int32_t max_depth = 0;
    std::vector<gl_seg_batch> batches;      // segments added since gl_depth_begin
    gl_buf store_s, store_e;                // host-uploaded segments, contiguous
    gl_buf packed;                          // staging for packed16 uploads
    int64_t store_n = 0;
    bool copies_pending = false;            // H2D into the store still in flight on copy_stream
    // what `diff` holds, built from every batch: kPathNone (nothing valid), kPathHbmDiff (the difference array) or
    // kPathEvents (the per-tile event buckets); the two general paths share the buffer
    int diff_holds = kPathNone;
    int last_path = kPathNone;              // the path the settled result took (gl_depth_last_path)
    // index tables of the last fused reduce (valid until the next reduce): used by gl_depth_interval_sums
    const int* idx_flags = nullptr; const unsigned* idx_cells = nullptr; int idx_origin = 0, idx_ncells = 0;
    // gl_depth_set_path: kPathNone = automatic (packed8, else fused, else bucketed events); kPathFused = never the packed8
    // kernel; kPathHbmDiff / kPathEvents = always that general path
    int force_path = kPathNone;
    gl_md_ep md_ep;                         // the tile core's multidepth epilogue for the next reduce (mode 0: none)
    void* md = nullptr;                     // multidepth.cu state (gl_multidepth_begin)
    void* cs = nullptr;                     // covstats.cu state (gl_bam_covstats): batch buffers and the last call's samples
    // a packed8 batch that is the region's only batch stays packed: K_fused8 reads it as it is (kPathPacked8); it is
    // unpacked into the store (its batch descriptor already points there) only when something needs int32 arrays
    struct { const int* anchors = nullptr; const void* ds = nullptr; const void* len = nullptr; int64_t n_blocks = 0, store_off = 0;
             bool pending = false;
             // upload deferred to the reduce (one-call entry with pinned host words): streamed in chunks, each chunk's
             // tiles reduced while the next chunk is on the wire
             const int* h_anchors = nullptr; const void* h_ds = nullptr; const void* h_len = nullptr; bool upload_pending = false; } p8;
    gl_buf diff;          // int32[len+1 (+pad)] + tile sums (general path only)
    void* win_sum_p = nullptr;   // u64[n_windows], inside `scratch`
    int64_t* prefetch_sums = nullptr; int64_t prefetch_cap = 0; bool prefetched = false;   // one-call entries: window sums go home while the header is read
    int32_t* prefetch_run_start = nullptr; uint8_t* prefetch_run_class = nullptr; int64_t prefetch_run_cap = 0, prefetched_runs = 0;   // and the first runs
    // gl_depth_reduce only queues its work: the header (runs claimed, max depth, fast path rejected) travels into the pinned
    // hdr_host (a copy, or on the packed8 path K_gather's store through hdr_dev), and depth_resolve reads it behind ev_hdr
    // at the first result query, with what accepting or rerunning needs
    uint64_t* hdr_host = nullptr;         // 4 words, pinned and mapped
    uint64_t* hdr_dev = nullptr;          // hdr_host's device address
    cudaEvent_t ev_hdr = nullptr;
    uint64_t p8_tag = 2;                  // the next packed8 reduce's rejection tag (never 0 or 1, never reused)
    struct { bool active = false;
             ReduceArgs args;
             int path = kPathNone; long long run_cap = 0; int64_t n_windows = 0;   // the path tried and its run capacity
             bool d2h = false;                                             // window sums also on their way home on d2h_stream
             uint64_t tag = 0;                                             // packed8: header[3] == tag means rejected
             const int* flags = nullptr; const unsigned* cells = nullptr; int origin = 0, ncells = 0; } pend;
    gl_buf win_min;       // i32[n_windows]
    gl_buf run_start;     // i32[run_cap]
    gl_buf run_class;     // u8[run_cap]
    gl_buf run_tmp_start; // claim-order staging of the runs
    gl_buf run_tmp_class;
    gl_buf scratch;       // header | window sums | index flags + cell tables | per-tile run table
    void* pinned[2] = {nullptr, nullptr};
    // pinned host staging (gl_pinned_reserve): the packed words gl_depth_bed_region makes, the compressed bytes gl_bam_decode_device reads
    void* pack_pinned = nullptr; size_t pack_pinned_bytes = 0;
    bool cohort_attr_set = false;                                // ic_cohort2_kernel's dynamic shared-memory limit raised on this ctx's device
    double tr_phase[3] = {0, 0, 0};
    int tr_kind = 0; double tr_pack_s = 0; int64_t tr_bytes = 0, tr_esc = 0;   // gl_depth_transport_stats
    int32_t* esc_buf = nullptr; size_t esc_cap = 0;              // ... and of the raw segments of blocks that do not fit packed16 (2 x esc_cap ints, malloc)
    gl_buf flush;         // L2 flush scratch
    gl_buf misc;          // small outputs of other subsystems
    gl_buf bam_comp, bam_out, bam_seg;   // bamgpu.cu: compressed bytes + tables, inflated stream, decoded segments
    gl_buf text_slots, text_blk, text_len, text_out[2];   // depth_text.cu: row slots, block offsets, lengths, compact BED text (depth, callable)
    gl_buf fasta;         // raw FASTA bytes of one record (gl_fasta_load), newlines included
    int64_t fasta_n = 0;

    // per-kernel CUDA-event profiling (gl_profile_*): (name, start, stop) per launch while enabled
    bool prof_on = false;
    struct prof_rec { const char* name; cudaEvent_t a, b; };
    std::vector<prof_rec> prof;
    std::vector<cudaEvent_t> prof_pool;

    unsigned cohort_fallbacks = 0;   // ic_cohort2_kernel: samples that took the exact fallback select in the last call
    int64_t em_rows = 0, em_uncertified = 0, em_sequential = 0;   // emdepth.cu: the last gl_emdepth* call (gl_emdepth_stats)
    double pca_phase[3] = {0, 0, 0};   // pca.cu: upload, Gram + centring, eigen of the last gl_indexcov_pca* call (seconds)
    double svd_phase[4] = {0, 0, 0, 0};   // dcnv_svd.cu: stats + Gram, eigen, projection, copies of the last gl_dcnv_svd* call
    cudaStream_t comm_stream = nullptr; cudaEvent_t ev_comm = nullptr;   // gl_allgather_device_async
    void* nccl = nullptr; // ncclComm_t when gl_comm_init was called
    int rank = 0, world = 1;
};

extern thread_local std::string g_gl_err;

int gl_fail(gl_ctx* ctx, int code, const char* fmt, ...);
// Grows b.  Freeing the old buffer first synchronises ctx->stream, so no queued work can still be using it.
int gl_buf_reserve(gl_ctx* ctx, gl_buf& b, size_t bytes);
// Grows ctx->pack_pinned to `want` bytes when it holds fewer than `bytes`.  Synchronises copy_stream first: the uploads
// queued out of the old buffer must have left it.  Library-internal: not exported from the .so.
__attribute__((visibility("hidden"))) int gl_pinned_reserve(gl_ctx* ctx, size_t bytes, size_t want);
// depth.cu: settle the last gl_depth_reduce (wait for its header; accept it, or rerun it on the next path or with room for
// every run).  Every reader of the reduce's results calls this first; a no-op when nothing is pending.
int depth_resolve(gl_ctx* ctx);
// depth.cu: one pass of the tile core over the open region with ctx->md_ep as its epilogue (no windows, no runs), settled
// before it returns; d_depth_out (may be null) also receives the per-base depth.
int depth_reduce_epilogue(gl_ctx* ctx, int32_t* d_depth_out);
// multidepth.cu: release ctx->md (gl_ctx_destroy)
void md_free(gl_ctx* ctx);
// covstats.cu: release ctx->cs (gl_ctx_destroy)
void cs_free(gl_ctx* ctx);
// indexcov.cu: bincount_kernel over device values into a device histogram of hi - lo bins (zeroed first), queued on ctx->stream
__attribute__((visibility("hidden"))) int gl_bincount_device(gl_ctx* ctx, const int32_t* d_v, int64_t n, int32_t lo, int32_t hi, unsigned long long* d_hist);

#define GL_CUDA(ctx, expr)                                                             \
    do {                                                                               \
        cudaError_t _e = (expr);                                                       \
        if (_e != cudaSuccess)                                                         \
            return gl_fail((ctx), GL_ECUDA, "%s failed: %s (%s:%d)", #expr,            \
                           cudaGetErrorString(_e), __FILE__, __LINE__);                \
    } while (0)

#define GL_CHECK(expr)                 \
    do {                               \
        int _rc = (expr);              \
        if (_rc != GL_OK) return _rc;  \
    } while (0)

#define GL_LAUNCHED(ctx, n)                                                            \
    do {                                                                               \
        (ctx)->launches += (n);                                                        \
        GL_CUDA((ctx), cudaGetLastError());                                            \
    } while (0)

// Bracket one kernel launch with events on the ctx stream when profiling is on.
struct gl_prof_scope {
    gl_ctx* ctx; cudaEvent_t b = nullptr;
    gl_prof_scope(gl_ctx* c, const char* name) : ctx(c) {
        if (!c->prof_on) return;
        cudaEvent_t ev[2];
        for (int i = 0; i < 2; i++) {
            if (!c->prof_pool.empty()) { ev[i] = c->prof_pool.back(); c->prof_pool.pop_back(); }
            else cudaEventCreate(&ev[i]);
        }
        cudaEventRecord(ev[0], c->stream);
        b = ev[1];
        c->prof.push_back({name, ev[0], ev[1]});
    }
    ~gl_prof_scope() { if (b) cudaEventRecord(b, ctx->stream); }
};

// The device temporaries of one call that takes host arrays: each holds at least 16 bytes, and all are freed when the
// scratch goes out of scope, so every return path frees them.  alloc fails with GL_ENOMEM, upload's copy with GL_ECUDA.
// Library-internal: not exported from the .so.
struct __attribute__((visibility("hidden"))) gl_scratch {
    static constexpr int kMax = 8;
    gl_ctx* ctx;
    void* bufs[kMax] = {};
    int n_bufs = 0;
    explicit gl_scratch(gl_ctx* c) : ctx(c) {}
    gl_scratch(const gl_scratch&) = delete;
    gl_scratch& operator=(const gl_scratch&) = delete;
    ~gl_scratch() { for (int i = 0; i < n_bufs; i++) cudaFree(bufs[i]); }
    // d = room for n elements (null on failure)
    template <class T> int alloc(T*& d, size_t n) {
        d = nullptr;
        if (n_bufs == kMax) return gl_fail(ctx, GL_EINVAL, "gl_scratch: more than %d buffers", kMax);
        gl_buf b;
        GL_CHECK(gl_buf_reserve(ctx, b, std::max<size_t>(n * sizeof(T), 16)));
        bufs[n_bufs++] = b.p;
        d = static_cast<T*>(b.p);
        return GL_OK;
    }
    // d = a device copy of h[0..n), queued on ctx->stream
    template <class T> int upload(T*& d, const T* h, size_t n) {
        GL_CHECK(alloc(d, n));
        if (n) GL_CUDA(ctx, cudaMemcpyAsync(d, h, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
        return GL_OK;
    }
};

static inline int gl_use(gl_ctx* ctx) {
    if (!ctx) return gl_fail(nullptr, GL_EINVAL, "null ctx");
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e != cudaSuccess) return gl_fail(ctx, GL_ECUDA, "cudaSetDevice(%d): %s", ctx->device, cudaGetErrorString(e));
    return GL_OK;
}
