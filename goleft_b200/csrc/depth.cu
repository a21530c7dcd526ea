// depth.cu — the `goleft depth` hot path on sm_90a.
//
// Work per region [rs,re) of one contig, replacing the `samtools depth` child + per-line Go callback
// (depth/depth.go:45,238-364):   segments (start,end) -> per-base depth -> per-window sums (+min)
//                                                                      -> coverage-class run starts
// Per-base depth never exists in HBM: it is produced and consumed inside one 4096-base tile per CTA.
//
// A reduce takes the fastest of four paths the region's segments allow (DESIGN §1.0-1.2; the numbers are those of
// gl_depth_last_path):
//   3 packed8          the region's only batch is packed8, read as it is   K_tileidx8 -> K_fused8 -> K_gather
//   1 fused int32      segments in BAM order, at most 16384 bases          K_index -> K_fused -> K_gather
//   4 bucketed events  the general path: any order, any length             K_evcount -> K_evscan -> K_evscatter -> K_evtile -> K_gather
//   2 HBM diff. array  on request only (gl_depth_set_path)                 memset -> K_scatter -> K_super -> K_scan -> K_gather
// The device checks a fast path's eligibility itself and says so in the reduce's header; depth_resolve then reruns the
// region on the next path down.
//
// Tile core (every path, DESIGN §1.3): 16 or 64 consecutive bases per thread (swizzled smem transpose), one thread-local
// + one warp scan, REDUX-based window sums (one LDS per lane and window edge), class runs detected on warp min/max with a
// per-base slow path, runs claimed per tile with one atomic and put in position order by K_gather.
// All arithmetic is integer; results are bit-exact against oracle/oracle_depth.c.
#include "gl_common.cuh"
#include <string.h>
#include <chrono>
#include <type_traits>

extern "C" int glhost_pool_size(void);          // host/thread_pool.cpp: threads of the library's host pool

namespace {

constexpr int kScanThreads = 256;
constexpr int kWarps = kScanThreads / 32;
constexpr int kWarpElems = 512;                   // bases per warp (16 per lane)
constexpr int kTile = kWarps * kWarpElems;        // 4096 bases per tile
constexpr int kTileShift = 12;
static_assert((1 << kTileShift) == kTile, "tile shift");
constexpr int kSuperShift = 6;                    // 64 tiles per super-tile
constexpr int kHeaderWords = 8;                   // u64 words in front of the per-tile tables
constexpr unsigned kFull = 0xffffffffu;
constexpr int kCellShift = 8;                     // fused path: segment-offset table granularity (256 bases)
constexpr int kMaxLookback = 16384;               // fused path handles segments up to this long
constexpr int kMaxBatches = 8;
constexpr int kLenSlots = 1024;
constexpr int kFlagWords = 16 + kLenSlots;

// Programmatic dependent launch (sm_90): the packed8 reduce's kernels are launched with programmatic stream serialization
// (launch_chained), so each may start while the kernel before it drains.  A chained kernel lets its successor launch at
// its top and waits for its predecessor (complete, memory visible) before it touches anything an earlier kernel writes or
// reads.  Every CTA waits before it exits: a grid that finished without waiting could complete before its predecessor,
// and its successor's wait would then no longer cover the predecessor.  Outside a chained launch both are no-ops.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

__device__ __forceinline__ int4 ld_stream_int4(const int4* p) {
    int4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// 16-byte-chunk swizzle inside a tile (1024 chunks): conflict-free both for a warp touching 32
// consecutive chunks and for a warp whose lane l touches chunks 4l..4l+3 (the blocked layout).
__device__ __forceinline__ int swz_chunk(int c) { return c ^ ((c >> 2) & 7); }
__device__ __forceinline__ int swz_elem(int e) { return e ^ (((e >> 4) & 7) << 2); }   // == (swz_chunk(e>>2)<<2) | (e&3)
// the same for a core whose threads own BPT consecutive bases (BPT/4 chunks): lane l touches chunks (BPT/4)l .. +BPT/4-1.
// BPT 64: thread t's chunk j is 16t ^ (t & 7) ^ j, so the 8 lanes of each quarter-warp phase of an LDS/STS.128 hit chunks
// (t & 7) ^ j mod 8, eight distinct bank groups; and the 64 bases of one thread are XORed with the constant (t & 7) << 2,
// a permutation within each aligned group of 32, so 32 lanes reading 32 of them hit 32 banks.
template <int BPT> __device__ __forceinline__ int swz_chunk_t(int c) { return BPT == 64 ? (c ^ ((c >> 4) & 7)) : (c ^ ((c >> 2) & 7)); }
template <int BPT> __device__ __forceinline__ int swz_elem_t(int e) { return BPT == 64 ? (e ^ (((e >> 6) & 7) << 2)) : (e ^ (((e >> 4) & 7) << 2)); }

// ================================================================================================
// GENERAL path, K_scatter.  One thread = 4 segments (two 128-bit loads), 8 fire-and-forget reds.
// Coordinates are clipped to the region exactly as `samtools depth -r` clips its output
// (depth/depth.go:150-152): a read spanning a chunk edge counts on both sides.
// The same events are summed per 4096-base tile; a warp of sorted segments sits in one or two tiles,
// so it reduces with REDUX and issues one red per distinct tile.
// ================================================================================================
__device__ __forceinline__ void warp_tile_add(int* __restrict__ tile_sum, int t, int c, int sign, int lane) {
    unsigned rem = __ballot_sync(kFull, c != 0);
#pragma unroll 1
    for (int it = 0; rem != 0 && it < 3; it++) {
        const int leader = __ffs(rem) - 1;
        const int key = __shfl_sync(kFull, t, leader);
        const bool m = (c != 0) && (t == key);
        const int tot = __reduce_add_sync(kFull, m ? c : 0);
        if (lane == leader) atomicAdd(tile_sum + key, sign * tot);
        if (m) c = 0;
        rem = __ballot_sync(kFull, c != 0);
    }
    if (c != 0) atomicAdd(tile_sum + t, sign * c);     // unsorted input: fall back to one red per lane
}

template <bool kVec>
__global__ void __launch_bounds__(256) depth_scatter_kernel(const int* __restrict__ start, const int* __restrict__ end,
                                                            long long n, int rs, int re, int* __restrict__ diff,
                                                            int* __restrict__ tile_sum) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int lane = threadIdx.x & 31;
    int s[4], e[4];
    int cnt = 0;
    if (kVec) {
        const long long n4 = n >> 2;
        if (i < n4) {
            int4 a = ld_stream_int4(reinterpret_cast<const int4*>(start) + i);
            int4 b = ld_stream_int4(reinterpret_cast<const int4*>(end) + i);
            s[0] = a.x; s[1] = a.y; s[2] = a.z; s[3] = a.w;
            e[0] = b.x; e[1] = b.y; e[2] = b.z; e[3] = b.w;
            cnt = 4;
        } else {
            const long long k = (n4 << 2) + (i - n4);
            if (k < n) { s[0] = start[k]; e[0] = end[k]; cnt = 1; }
        }
    } else if (i < n) {
        s[0] = start[i]; e[0] = end[i]; cnt = 1;
    }
    int tS = 0, cS = 0, tE = 0, cE = 0;
    bool uni = true;
#pragma unroll
    for (int j = 0; j < 4; j++) {
        if (j < cnt) {
            const int a = max(s[j], rs) - rs, b = min(e[j], re) - rs;
            if (a < b) {
                atomicAdd(diff + a, 1);          // result unused -> RED.E.ADD
                atomicAdd(diff + b, -1);
                const int ta = a >> kTileShift, tb = b >> kTileShift;
                if (cS == 0) { tS = ta; tE = tb; }
                else if (ta != tS || tb != tE) uni = false;
                s[j] = ta; e[j] = tb;            // keep the tile ids for the slow path
                cS++; cE++;
            } else {
                s[j] = -1;
            }
        } else {
            s[j] = -1;
        }
    }
    if (!uni) {                                  // this thread straddles a tile edge: per-event reds
#pragma unroll
        for (int j = 0; j < 4; j++)
            if (s[j] >= 0) { atomicAdd(tile_sum + s[j], 1); atomicAdd(tile_sum + e[j], -1); }
        cS = 0; cE = 0;
    }
    warp_tile_add(tile_sum, tS, cS, 1, lane);
    warp_tile_add(tile_sum, tE, cE, -1, lane);
}

// packed16 -> (start,end): one CTA per 256-slot block (host/seg_pack.cpp); empty slots become empty segments
__global__ void __launch_bounds__(256) depth_unpack16_kernel(const int* __restrict__ anchors, const unsigned short* __restrict__ off,
                                                            const unsigned short* __restrict__ len, int* __restrict__ start,
                                                            int* __restrict__ end) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    const int s = anchors[blockIdx.x] + (int)off[i];
    start[i] = s;
    end[i] = s + (int)len[i];
}

// packed8 -> (start,end): 64-slot blocks, 8 consecutive slots per lane, so 8 lanes per block and 4 blocks per warp;
// starts are the anchor plus the running sum of the uint8 deltas (thread-local sum + an 8-lane segmented scan).
// A warp writes 1 KB of contiguous starts.
__global__ void __launch_bounds__(256) depth_unpack8_kernel(const int* __restrict__ anchors, const uint2* __restrict__ dstart,
                                                           const uint2* __restrict__ len, long long n_blocks,
                                                           int* __restrict__ start, int* __restrict__ end) {
    const long long t = (long long)blockIdx.x * 256 + threadIdx.x;      // one thread per 8 slots
    const long long b = t >> 3;
    const int sub = threadIdx.x & 7;
    const bool live = b < n_blocks;
    uint2 d = make_uint2(0, 0), l = make_uint2(0, 0);
    if (live) { d = dstart[t]; l = len[t]; }
    int ds[8], ln[8];
#pragma unroll
    for (int k = 0; k < 4; k++) {
        ds[k] = (d.x >> (8 * k)) & 0xff; ds[4 + k] = (d.y >> (8 * k)) & 0xff;
        ln[k] = (l.x >> (8 * k)) & 0xff; ln[4 + k] = (l.y >> (8 * k)) & 0xff;
    }
#pragma unroll
    for (int k = 1; k < 8; k++) ds[k] += ds[k - 1];
    int inc = ds[7];
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, inc, o, 8);
        if (sub >= o) inc += v;
    }
    if (!live) return;
    const int base = anchors[b] + inc - ds[7];
    int4* so = reinterpret_cast<int4*>(start + t * 8);
    int4* eo = reinterpret_cast<int4*>(end + t * 8);
    const int s0 = base + ds[0], s1 = base + ds[1], s2 = base + ds[2], s3 = base + ds[3];
    const int s4 = base + ds[4], s5 = base + ds[5], s6 = base + ds[6], s7 = base + ds[7];
    so[0] = make_int4(s0, s1, s2, s3);
    so[1] = make_int4(s4, s5, s6, s7);
    eo[0] = make_int4(s0 + ln[0], s1 + ln[1], s2 + ln[2], s3 + ln[3]);
    eo[1] = make_int4(s4 + ln[4], s5 + ln[5], s6 + ln[6], s7 + ln[7]);
}

// K_super: super_sum[st] = sum of the 64 tile sums of super-tile st (one warp each).  Doing this in the
// scatter itself would put every warp's red on the same handful of addresses — measured 7x slower.
__global__ void __launch_bounds__(256) depth_super_sum_kernel(const int* __restrict__ tile_sum, int* __restrict__ super_sum,
                                                             int tiles) {
    const int st = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    const int t0 = st << kSuperShift;
    if (t0 >= tiles) return;
    int v = 0;
    if (t0 + lane < tiles) v += tile_sum[t0 + lane];
    if (t0 + 32 + lane < tiles) v += tile_sum[t0 + 32 + lane];
    v = __reduce_add_sync(kFull, v);
    if (lane == 0) super_sum[st] = v;
}

// ================================================================================================
// FUSED path, K_index.  For every 256-base cell from `origin`: cell_lo = ~(lowest index of a segment that
// starts in the cell), cell_hi = highest such index + 1, cell_cnt = how many.  Consecutive segments
// mostly share a cell, so each run of equal cells inside a warp issues one atomicMin (its first lane),
// one atomicMax (its last lane) and one atomicAdd (run length).  No ordering assumption is made here;
// the fused kernel compares span and count.  Also: the longest segment, in 1024 slots (a single word
// would serialise one atomic per warp on one address).
// ================================================================================================
__device__ __forceinline__ int index_cell(int s, int len, int origin, int re, int ncells) {
    // segments that start below a non-zero origin cannot reach the region (length <= look-back, else the
    // fused path is rejected anyway); negative starts belong to cell 0 when origin is 0
    return (len > 0 && s < re && (s >= origin || origin == 0)) ? min(max(s - origin, 0) >> kCellShift, ncells - 1) : -1;
}

// 4 segments per thread (128-bit loads keep enough bytes in flight); runs of equal cells are found over
// the warp's 128 consecutive segments.
__global__ void __launch_bounds__(256) depth_index_kernel(const int* __restrict__ start, const int* __restrict__ end,
                                                         long long n, int origin, int re, int ncells,
                                                         unsigned* __restrict__ cell_lo, unsigned* __restrict__ cell_hi,
                                                         unsigned* __restrict__ cell_cnt, int* __restrict__ flags) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long base = t * 4;
    const int lane = threadIdx.x & 31;
    int c[4] = {-1, -1, -1, -1};
    int len = 0;
    const bool vec = ((reinterpret_cast<uintptr_t>(start) | reinterpret_cast<uintptr_t>(end)) & 15) == 0;
    if (base + 3 < n && vec) {
        const int4 s4 = ld_stream_int4(reinterpret_cast<const int4*>(start) + t);
        const int4 e4 = ld_stream_int4(reinterpret_cast<const int4*>(end) + t);
        const int l0 = e4.x - s4.x, l1 = e4.y - s4.y, l2 = e4.z - s4.z, l3 = e4.w - s4.w;
        c[0] = index_cell(s4.x, l0, origin, re, ncells);
        c[1] = index_cell(s4.y, l1, origin, re, ncells);
        c[2] = index_cell(s4.z, l2, origin, re, ncells);
        c[3] = index_cell(s4.w, l3, origin, re, ncells);
        len = max(max(l0, l1), max(l2, l3));
    } else {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (base + j < n) {
                const int sv = start[base + j], l = end[base + j] - sv;
                c[j] = index_cell(sv, l, origin, re, ncells);
                len = max(len, l);
            }
        }
    }
    const int wl = __reduce_max_sync(kFull, len);
    if (lane == 0 && wl > 0) {
        const int slot = (int)((t >> 5) & (kLenSlots - 1));
        if (wl > flags[16 + slot]) atomicMax(flags + 16 + slot, wl);
    }
    const int pc = __shfl_up_sync(kFull, c[3], 1), nc = __shfl_down_sync(kFull, c[0], 1);
    bool first[4], last[4];
    first[0] = lane == 0 || pc != c[0];
    first[1] = c[1] != c[0];
    first[2] = c[2] != c[1];
    first[3] = c[3] != c[2];
    last[0] = first[1];
    last[1] = first[2];
    last[2] = first[3];
    last[3] = lane == 31 || nc != c[3];
    unsigned F[4];
#pragma unroll
    for (int j = 0; j < 4; j++) F[j] = __ballot_sync(kFull, first[j]);
    if (first[0] | first[1] | first[2] | first[3] | last[3]) {
        const unsigned later = (F[0] | F[1] | F[2] | F[3]) & ~((2u << lane) - 1u);     // lanes after mine that start a run
        int q_next = 128;                                                              // position of the first run start after my lane
        if (later) {
            const int l2 = __ffs(later) - 1;
            const int j2 = ((F[0] >> l2) & 1u) ? 0 : ((F[1] >> l2) & 1u) ? 1 : ((F[2] >> l2) & 1u) ? 2 : 3;
            q_next = 4 * l2 + j2;
        }
#pragma unroll
        for (int j = 0; j < 4; j++) {
            if (c[j] >= 0) {
                if (first[j]) {
                    int q = q_next;
#pragma unroll
                    for (int jj = 3; jj > j; jj--)
                        if (first[jj]) q = 4 * lane + jj;
                    atomicMax(cell_lo + c[j], ~(unsigned)(base + j));        // table holds ~min so it can be zero-initialised
                    atomicAdd(cell_cnt + c[j], (unsigned)(q - (4 * lane + j)));
                }
                if (last[j]) atomicMax(cell_hi + c[j], (unsigned)(base + j) + 1u);
            }
        }
    }
}

// ================================================================================================
// Tile core
// ================================================================================================
struct BatchDesc {
    const int* start;
    const int* end;
    const unsigned* cell_lo;   // [ncells] bitwise NOT of the lowest segment index starting in the cell (0: none)
    const unsigned* cell_hi;   // [ncells] highest such index + 1
    const unsigned* cell_cnt;  // [ncells] number of segments starting in the cell
    int n;
};

struct ScanParams {
    // general path inputs
    const int* diff;              // padded to a whole number of tiles, zero beyond len
    const int* tile_sum;          // [num_tiles+1] net (+starts -ends) inside each tile
    const int* super_sum;         // [num_tiles/64+1] the same per 64 tiles
    // fused path inputs
    const int* flags;             // K_index output: [16..16+1024) max segment length slots
    int origin, ncells, n_batches;
    BatchDesc batch[kMaxBatches];
    // region and outputs
    int len;                      // bases in the region
    int rs, re;                   // absolute region
    int W;                        // window size
    long long w0;                 // rs / W  (index of the first window)
    int mincov, maxmean;
    unsigned run_break;           // 0 = never (host clamps values >= 2^32 to 0: no multiple in range)
    unsigned long long* win_sum;  // [n_windows], zero-initialised
    int* win_min;                 // [n_windows], initialised to 0x7f7f7f7f, or null (then not computed)
    int* tmp_start;               // [run_cap] run starts in claim order
    unsigned char* tmp_class;     // [run_cap]
    long long run_cap;
    uint64_t* header;             // [0]=runs claimed (= n_runs) [2]=max_depth [3]=fused path rejected (1) / packed8 rejected (p8_tag)
    uint64_t* chunk_runs;         // [num_tiles*warps] per warp chunk of the core: (claim offset << 32) | count
    unsigned* super_cnt;          // [num_tiles*8/64+1] run starts per 64 chunks
    int* depth_out;               // optional per-base output (debug/parity), else null
    int num_tiles;
    int do_windows, do_runs;
    // packed8 path (K_tileidx8 + K_fused8)
    const int* p8_anchors;        // [p8_nblocks] non-decreasing
    const unsigned* p8_ds;        // [p8_nblocks*16] 4 uint8 start deltas per word
    const unsigned* p8_len;       // [p8_nblocks*16] 4 uint8 lengths per word
    int p8_nblocks;
    int* tile_lo;                 // [num_tiles+1] number of anchors < x_k - 255, x_k = rs + k*4096
    int* tile_hi;                 // [num_tiles+1] number of anchors < x_k
    unsigned W_inv;               // floor(2^32 / W): window index by multiplication (fast window path, W >= 16)
    int tile_begin, tile_end;     // K_fused8 processes these tiles (a streamed upload launches it once per arrived chunk)
    int idx_begin, idx_end;       // K_tileidx8 handles the anchor gaps i in [idx_begin, idx_end), i = -1 .. nb-1
    long long zero_words;         // K_tileidx8: u64 words of scratch to zero first, all but header[3] (the reduce's first launch only)
    uint64_t p8_tag;              // packed8: header[3] == p8_tag marks this reduce rejected (header[3] is never zeroed there)
    gl_md_ep md;                  // multidepth epilogue (mode 0: none)
};

__device__ __forceinline__ int cov_class(int d, int mincov, int maxmean) {
    // depth/depth.go:223-234
    return d == 0 ? GL_NO_COVERAGE
                  : (d < mincov ? GL_LOW_COVERAGE : ((maxmean > 0 && d >= maxmean) ? GL_EXCESSIVE_COVERAGE : GL_CALLABLE));
}

// deepest base seen by this warp -> header[2]; the plain read first keeps most warps off the atomic
__device__ __forceinline__ void flush_max(const ScanParams& p, int acc_max) {
    if ((threadIdx.x & 31) == 0 && acc_max > 0 &&
        (unsigned long long)acc_max > *reinterpret_cast<volatile unsigned long long*>(p.header + 2))
        atomicMax(reinterpret_cast<unsigned long long*>(p.header + 2), (unsigned long long)acc_max);
}

// Clears one warp's kElems-element region of a tile with 32 consecutive chunks per store.  The warp owns the region, so
// the order does not matter, and the addresses are one base plus constants (no per-chunk swizzle kept in registers).
template <int kElems>
__device__ __forceinline__ void clear_warp_region(int* region, int lane) {
#pragma unroll
    for (int j = 0; j < kElems / 128; j++) reinterpret_cast<int4*>(region)[lane + 32 * j] = make_int4(0, 0, 0, 0);
}

// Inclusive scan over the warp's 32 lanes.  shfl.up's predicate says whether the source lane exists, so a step is a SHFL
// and a predicated add; `if (lane >= o) v += t` compiles to a SHFL, a SEL and an add.
__device__ __forceinline__ int warp_incl_scan(int v) {
#pragma unroll
    for (int o = 1; o < 32; o <<= 1)
        asm("{\n\t.reg .s32 t;\n\t.reg .pred p;\n\tshfl.sync.up.b32 t|p, %0, %1, 0, -1;\n\t@p add.s32 %0, %0, t;\n\t}" : "+r"(v) : "r"(o));
    return v;
}

// The window of a thread's first base a = rs + idx0 (iw = a / W, rem = a % W), and cu = the number of the thread's bpt
// bases left of the next window edge when that edge falls inside them (0: none)
__device__ __forceinline__ void window_edge(const ScanParams& p, int idx0, int bpt, unsigned& iw, unsigned& rem, int& cu) {
    const unsigned a = (unsigned)p.rs + (unsigned)idx0;              // absolute, < 2^32
    const unsigned uW = (unsigned)p.W;
    // iw = a / W without a division: q = hi32(a * floor(2^32/W)) is the quotient or one less, because
    // a * floor(2^32/W) > a * 2^32 / W - a and a < 2^32
    iw = __umulhi(a, p.W_inv);
    rem = a - iw * uW;
    if (rem >= uW) { iw++; rem -= uW; }
    cu = uW - rem < (unsigned)bpt ? (int)(uW - rem) : 0;
}

// Per-base run-start bits of one thread's bases
__device__ __forceinline__ int mask_popc(unsigned m) { return __popc(m); }
__device__ __forceinline__ int mask_popc(unsigned long long m) { return __popcll(m); }
__device__ __forceinline__ int mask_ffs(unsigned m) { return __ffs(m); }
__device__ __forceinline__ int mask_ffs(unsigned long long m) { return __ffsll((long long)m); }

// BPT bases per thread (16 or 64), WARPS warps per CTA, BPT * 32 * WARPS == kTile.  64 bases per thread spreads the work
// that is paid per thread and tile (warp scans, class check, window sums, run claim, barrier) over four times the bases
// of the 16-base core — K_fused8 uses <64, 2>.
// kSliceInTile (K_fused8): the depth slice goes over the warp's own region of s_tile instead of s_depth (unused, may be
// null), and the region is cleared when the core is done with it.  The caller must then hold every warp at a barrier
// between the core and the next tile's atomics.
template <int BPT, int WARPS, bool kZeroAfterRead, bool kMD = false, bool kSliceInTile = false>
__device__ __forceinline__ void tile_core(const ScanParams& p, int* __restrict__ s_tile, int* __restrict__ s_depth,
                                          const int* s_carry, int tile, int& acc_max) {
    static_assert(BPT * 32 * WARPS == kTile && (BPT == 16 || BPT == 64), "tile shape");
    constexpr int kWElems = BPT * 32;                         // bases per warp
    using Mask = std::conditional_t<BPT == 64, unsigned long long, unsigned>;   // one bit per base of a thread
    __shared__ int s_warp_tot[WARPS];
    __shared__ int s_has_break;
    __shared__ int s_tbase[WARPS * 32];                       // depth before each thread's first base (slow paths)

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tile_base = tile * kTile;                       // relative position of the tile
    const int warp_base = tile_base + warp * kWElems;
    const int idx0 = tile_base + tid * BPT;                   // relative position of this thread's first base

    // ---- BPT consecutive differences per thread; thread-local inclusive scan; one warp scan
    // a thread's chunks: swz_chunk_t<BPT>(t * (BPT / 4) + j) == c0 ^ j for j < BPT / 4 (the XOR only reads bits of t)
    const int c0 = swz_chunk_t<BPT>(tid * (BPT / 4));
    // depth[k] = tbase + x[k], tbase known only after the barrier: take min / max / sum of the x[k] now, while other
    // warps are still arriving, and add tbase afterwards (the per-base depths are formed only where a slow path needs them)
    int x[BPT];
    int g8[BPT / 8];                                          // sums of groups of 8 (the window path reuses them)
    int xmn, xmx, xsum, xlast;
    // the fast window path's terms (below); kSliceInTile finds them before the barrier
    unsigned iw = 0, rem = 0;
    int cu = 0, lx = 0;
    if constexpr (kSliceInTile) {
        // x[64] held across the barrier would cost ~40 registers (118 in all, 8 CTAs per SM), so the thread reads its
        // differences in two halves of 32 and keeps only what the fast window path needs.  The differences stay in the
        // warp's region of s_tile until the warp clears it, so a warp that needs x after the barrier scans them again.
        // cu depends only on positions: lx is summed half by half, from the half's group sums and one partial group.
        window_edge(p, idx0, BPT, iw, rem, cu);
        xmn = INT_MAX; xmx = INT_MIN; xsum = 0;
        int run = 0;
#pragma unroll
        for (int h = 0; h < BPT / 32; h++) {
#pragma unroll
            for (int j = 0; j < 8; j++) {
                const int4 q = reinterpret_cast<const int4*>(s_tile)[c0 ^ (8 * h + j)];
                x[4 * j] = q.x; x[4 * j + 1] = q.y; x[4 * j + 2] = q.z; x[4 * j + 3] = q.w;
            }
            x[0] += run;
#pragma unroll
            for (int k = 1; k < 32; k++) x[k] += x[k - 1];
            run = x[31];
#pragma unroll
            for (int k = 0; k < 32; k += 2) {                 // three-input min / max (VIMNMX3)
                xmn = __vimin3_s32(xmn, x[k], x[k + 1]);
                xmx = __vimax3_s32(xmx, x[k], x[k + 1]);
            }
#pragma unroll
            for (int g = 0; g < 4; g++) {
                g8[g] = (x[8 * g] + x[8 * g + 1] + x[8 * g + 2]) + (x[8 * g + 3] + x[8 * g + 4] + x[8 * g + 5]) + (x[8 * g + 6] + x[8 * g + 7]);
                xsum += g8[g];
            }
            const int ch = min(max(cu - 32 * h, 0), 32);      // bases of this half left of the edge
            const int gi = ch >> 3, r = ch & 7;
#pragma unroll
            for (int g = 0; g < 4; g++) lx += g < gi ? g8[g] : 0;
#pragma unroll
            for (int j = 0; j < 7; j++) {
                int v = x[j];
#pragma unroll
                for (int g = 1; g < 4; g++) v = gi == g ? x[8 * g + j] : v;
                lx += j < r ? v : 0;
            }
        }
        xlast = run;
    } else {
#pragma unroll
        for (int j = 0; j < BPT / 4; j++) {
            const int4 q = reinterpret_cast<const int4*>(s_tile)[c0 ^ j];
            x[4 * j] = q.x; x[4 * j + 1] = q.y; x[4 * j + 2] = q.z; x[4 * j + 3] = q.w;
            if (kZeroAfterRead) reinterpret_cast<int4*>(s_tile)[c0 ^ j] = make_int4(0, 0, 0, 0);
        }
#pragma unroll
        for (int k = 1; k < BPT; k++) x[k] += x[k - 1];
        xmn = x[0], xmx = x[0];
#pragma unroll
        for (int k = 1; k + 1 < BPT; k += 2) {                // three-input min / max (VIMNMX3)
            xmn = __vimin3_s32(xmn, x[k], x[k + 1]);
            xmx = __vimax3_s32(xmx, x[k], x[k + 1]);
        }
        xmn = min(xmn, x[BPT - 1]);
        xmx = max(xmx, x[BPT - 1]);
#pragma unroll
        for (int g = 0; g < BPT / 8; g++)
            g8[g] = (x[8 * g] + x[8 * g + 1] + x[8 * g + 2]) + (x[8 * g + 3] + x[8 * g + 4] + x[8 * g + 5]) + (x[8 * g + 6] + x[8 * g + 7]);
        xsum = g8[0];
#pragma unroll
        for (int g = 1; g < BPT / 8; g++) xsum += g8[g];
        xlast = x[BPT - 1];
    }
    const int inc = warp_incl_scan(xlast);
    const int lane_excl = inc - xlast;
    if (lane == 31) s_warp_tot[warp] = inc;
    if (tid == 0) {
        // does a forced run break (multiple of run_break) fall inside this tile?  (absolute positions are < 2^32)
        int hb = 0;
        if (p.do_runs && p.run_break > 0) {
            const unsigned a = (unsigned)p.rs + (unsigned)tile_base;
            const unsigned rem = a % p.run_break;
            hb = (rem ? p.run_break - rem : 0u) < (unsigned)kTile;
        }
        s_has_break = hb;
    }
    __syncthreads();

    // depth at the base before this warp's first: everything carried into the tile + the warps before this one
    const int wbase = __reduce_add_sync(kFull, lane < WARPS ? s_carry[lane] + (lane < warp ? s_warp_tot[lane] : 0) : 0);
    const int tbase = wbase + lane_excl;                      // depth at the base before this thread's first

    const int mn = tbase + xmn, mx = tbase + xmx;
    const bool full_warp = warp_base + kWElems <= p.len;   // false only at the region's ragged end
    const int wmin = __reduce_min_sync(kFull, mn), wmax = __reduce_max_sync(kFull, mx);

    const bool tile_has_break = s_has_break != 0;

    // class(d) is monotone in d: the warp's bases plus the base before them are one class iff
    // class(min) == class(max) — then no run starts here and all per-base class work is skipped.
    bool slow_runs = false;
    if (p.do_runs)
        slow_runs = !full_warp || tile_has_break || warp_base == 0 ||
                    cov_class(min(wmin, wbase), p.mincov, p.maxmean) != cov_class(max(wmax, wbase), p.mincov, p.maxmean);
    constexpr int kFastDepth = kWElems > 1024 ? (1 << 21) : (1 << 22);   // kWElems * kFastDepth <= 2^32
    const bool fast_win = p.do_windows && full_warp && p.W >= BPT && p.win_min == nullptr && wmax < kFastDepth;
    const bool slow_win = p.do_windows && !fast_win;

    // Depth by position: this warp's private slice of s_depth holds x[k] (depth relative to the thread's tbase), swizzled
    // like s_tile (base e of the slice at sw[swz_elem_t<BPT>(e)]) so that both a lane storing its BPT/4 chunks and 32 lanes
    // reading 32 consecutive bases of one thread are conflict-free; the threads' tbase go to s_tbase.  Storing x instead of
    // depth saves BPT adds per thread; a reader adds the owner's tbase.  The slice uses the same chunks as the warp's region
    // of s_tile, so a warp only ever touches its own kWElems elements of either buffer.  With kSliceInTile it overwrites
    // that region, which is safe because no warp starts the next tile's atomics before the caller's barrier; otherwise a
    // warp that leaves the core early may already be adding into s_tile, and the slice goes to s_depth.  With kSliceInTile
    // x is not in registers: each thread scans its differences into the slice in place, and the per-base depths below
    // are read from it (depth_out and the multidepth epilogues then need the slice too).
    int* const s_slice = kSliceInTile ? s_tile : s_depth;
    int* sw = s_slice + warp * kWElems;
    int* stb = s_tbase + warp * 32;
    const bool need_slice = slow_runs || slow_win || (kSliceInTile && (p.depth_out != nullptr || (kMD && p.md.mode != 0)));
    if (need_slice) {
        __syncwarp();
        int run = 0;
#pragma unroll
        for (int j = 0; j < BPT / 4; j++) {
            int4 q;
            if constexpr (kSliceInTile) {
                q = reinterpret_cast<const int4*>(s_slice)[c0 ^ j];
                q.x += run; q.y += q.x; q.z += q.y; q.w += q.z;
                run = q.w;
            } else {
                q = make_int4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
            }
            reinterpret_cast<int4*>(s_slice)[c0 ^ j] = q;
        }
        stb[lane] = tbase;
        __syncwarp();
    } else if (kSliceInTile) {
        clear_warp_region<kWElems>(sw, lane);                 // every lane has read its differences (block barrier above)
    }
    // x[4j .. 4j+3]: from registers, or with kSliceInTile from the slice (a thread reads its own chunks: no bank conflict)
    auto xq = [&](int j) -> int4 {
        if constexpr (kSliceInTile) return reinterpret_cast<const int4*>(s_slice)[c0 ^ j];
        else return make_int4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
    };
#define GL_D(q, i) (tbase + ((i) == 0 ? (q).x : (i) == 1 ? (q).y : (i) == 2 ? (q).z : (q).w))   /* depth of base 4j+i, q = xq(j) */

    if (p.depth_out) {
#pragma unroll
        for (int j = 0; j < BPT / 4; j++) {
            const int idx = idx0 + 4 * j;
            const int4 q = xq(j);
            if (idx + 3 < p.len) reinterpret_cast<int4*>(p.depth_out + idx)[0] = make_int4(GL_D(q, 0), GL_D(q, 1), GL_D(q, 2), GL_D(q, 3));
            else {
                if (idx < p.len) p.depth_out[idx] = GL_D(q, 0);
                if (idx + 1 < p.len) p.depth_out[idx + 1] = GL_D(q, 1);
                if (idx + 2 < p.len) p.depth_out[idx + 2] = GL_D(q, 2);
            }
        }
    }
    // ---- multidepth epilogues (multidepth.cu).  Both only overwrite, so a rerun after a rejected fused pass is harmless.
    if (kMD && p.md.mode == 1) {
        // pass 1: this sample's (d >= mincov) and (d > 0) bits, 16 bases per halfword
        const int nv = max(0, min(BPT, p.len - idx0));
        Mask ge = 0, pos = 0;
#pragma unroll
        for (int j = 0; j < BPT / 4; j++) {
            const int4 q = xq(j);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int k = 4 * j + i, d = GL_D(q, i);
                if (k < nv) {
                    ge |= (Mask)(d >= p.md.mincov ? 1u : 0u) << k;
                    pos |= (Mask)(d > 0 ? 1u : 0u) << k;
                }
            }
        }
#pragma unroll
        for (int j = 0; j < BPT / 16; j++) {
            p.md.ge16[idx0 / 16 + j] = (unsigned short)(ge >> (16 * j));
            p.md.pos16[idx0 / 16 + j] = (unsigned short)(pos >> (16 * j));
        }
    } else if (kMD && p.md.mode == 2) {
        // pass 2: Σ d over the sufficient sites of every block that meets this warp's bases, one slot per (pair, 512-base chunk)
        const unsigned sw32 = p.md.suf[idx0 >> 5];
        Mask sm;
        if constexpr (BPT == 64) sm = sw32 | ((Mask)p.md.suf[(idx0 >> 5) + 1] << 32);
        else sm = (sw32 >> (idx0 & 31)) & 0xffffu;
        const int q0 = p.md.pair_ptr[tile], q1 = p.md.pair_ptr[tile + 1];
        for (int q = q0; q < q1; q++) {
            const int b = p.md.pair_blk[q];
            const int bs = p.md.blk_start[b], be = p.md.blk_end[b];
            unsigned long long part = 0;
            if (bs < warp_base + kWElems && be > warp_base) {          // warp-uniform
                const int lo = min(max(bs - idx0, 0), BPT), hi = min(max(be - idx0, 0), BPT);
                const Mask rng = (hi >= BPT ? ~(Mask)0 : (((Mask)1 << hi) - 1u)) & ~(lo >= BPT ? ~(Mask)0 : (((Mask)1 << lo) - 1u));
                const Mask m = sm & rng;
#pragma unroll
                for (int j = 0; j < BPT / 4; j++) {
                    const int4 xj = xq(j);
#pragma unroll
                    for (int i = 0; i < 4; i++)
                        if ((m >> (4 * j + i)) & 1u) part += (unsigned long long)(unsigned)GL_D(xj, i);
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(kFull, part, o);
            }
            // slots are per 512-base chunk, so every path (8 warps x 16 bases/thread or 2 x 64) rewrites all eight of them
            if (lane == 0) {
#pragma unroll
                for (int h = 0; h < BPT / 16; h++) p.md.slots[(size_t)q * 8 + warp * (BPT / 16) + h] = h ? 0ull : part;
            }
        }
    }

    // ---- run starts (slow path): one mask bit per base, rank inside the warp in position order
    Mask mask = 0;
    int lane_rank = 0, warp_cnt = 0;
    int maxd = full_warp ? wmax : 0;
    if (slow_runs || !full_warp) {
        const int nv = max(0, min(BPT, p.len - idx0));
        int cp = cov_class(tbase, p.mincov, p.maxmean);
#pragma unroll
        for (int j = 0; j < BPT / 4; j++) {
            const int4 q = xq(j);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                const int k = 4 * j + i;
                if (k < nv) {
                    if (!full_warp) maxd = max(maxd, GL_D(q, i));
                    if (slow_runs) {
                        const int c = cov_class(GL_D(q, i), p.mincov, p.maxmean);
                        if (c != cp) mask |= (Mask)1 << k;
                        cp = c;
                    }
                }
            }
        }
        if (slow_runs) {
            if (idx0 == 0) mask |= 1u;                        // the region's first base always starts a run
            if (tile_has_break) {
                const unsigned a = (unsigned)p.rs + (unsigned)idx0;
                // rare (one tile in 2441 at 10 Mb): unrolled, its BPT divisions were the register peak of every kernel here
#pragma unroll 1
                for (int k = 0; k < BPT; k++)
                    if ((a + k) % p.run_break == 0) mask |= (Mask)1 << k;
            }
            mask &= (nv >= BPT) ? ~(Mask)0 : (((Mask)1 << nv) - 1u);
            const int c = mask_popc(mask);
            const int ci = warp_incl_scan(c);
            lane_rank = ci - c;
            warp_cnt = __shfl_sync(kFull, ci, 31);
        }
        if (!full_warp) maxd = __reduce_max_sync(kFull, maxd);
    }
    acc_max = max(acc_max, maxd);                             // warp-uniform; the kernel publishes it once (flush_max)

    // ---- window partial sums of this warp's bases
    if (fast_win) {
        // With W >= BPT a thread's BPT bases hold at most one window edge that is not on its first base, and cu of them
        // lie left of it (cu = 0: none).  lx = sum of x[k] for k < cu, from the g8 group sums plus one partial group.
        if constexpr (!kSliceInTile) {
            window_edge(p, idx0, BPT, iw, rem, cu);
            const int gi = cu >> 3, r = cu & 7;
#pragma unroll
            for (int g = 0; g + 1 < BPT / 8; g++) lx += g < gi ? g8[g] : 0;
#pragma unroll
            for (int j = 0; j < 7; j++) {
                int v = x[j];
#pragma unroll
                for (int g = 1; g < BPT / 8; g++) v = gi == g ? x[8 * g + j] : v;
                lx += j < r ? v : 0;
            }
        }
        // An edge lane holds one window edge: inside its bases (cu > 0, it ends window iw) or on its first base (it ends
        // window iw - 1; on lane 0 that is the warp's start, not an edge).  c = the warp's depth sum left of the edge, so a
        // window's part in this warp is c minus the c of the edge lane before it (0 for the first), and the window that
        // runs past the warp's end (or ends exactly at it) gets the warp's total minus the last c.  Every partial sum is
        // < 2^32 because depth < kFastDepth on this path, so unsigned 32-bit arithmetic is exact.
        const unsigned s16 = (unsigned)(BPT * tbase + xsum);
        const unsigned si = (unsigned)warp_incl_scan((int)s16);          // the lanes' depth sums, inclusive (mod 2^32)
        const unsigned total = __shfl_sync(kFull, si, 31);
        const bool at_start = rem == 0 && lane > 0;
        const bool edge = cu > 0 || at_start;
        const unsigned c = si - s16 + (unsigned)(cu * tbase + lx);
        const unsigned M = __ballot_sync(kFull, edge);
        const unsigned before = M & ((1u << lane) - 1u);
        const unsigned cprev = __shfl_sync(kFull, c, before ? 31 - __clz(before) : 0);
        unsigned long long* const ws = p.win_sum + ((long long)iw - p.w0);
        if (edge) atomicAdd(ws - (at_start ? 1 : 0), (unsigned long long)(c - (before ? cprev : 0u)));
        if (lane == (M ? 31 - __clz(M) : 0))                              // lane 0 without edges: c = 0, cu = 0
            atomicAdd(ws + (cu > 0 ? 1 : 0), (unsigned long long)(total - c));
    } else if (slow_win) {
        // General path from this warp's smem slice: any W, min, ragged end, depth up to 2^31.
        const unsigned a0 = (unsigned)p.rs + (unsigned)warp_base;
        const unsigned a1 = (unsigned)p.rs + (unsigned)min(warp_base + kWElems, p.len);
        const unsigned uW = (unsigned)p.W;
        if (a0 < a1) {
            const unsigned iw0 = a0 / uW, iw1 = (a1 - 1) / uW;
            if (p.W > 16) {
                for (unsigned iw = iw0; iw <= iw1; iw++) {
                    const long long ws = (long long)iw * uW, we = ws + uW;
                    const int s = (int)(max((long long)a0, ws) - a0), e = (int)(min((long long)a1, we) - a0);
                    unsigned long long sum = 0;
                    int m = 0x7fffffff;
                    for (int xx = s + lane; xx < e; xx += 32) {
                        const int dd = sw[swz_elem_t<BPT>(xx)] + stb[xx / BPT];
                        sum += (unsigned long long)(unsigned)dd;
                        m = min(m, dd);
                    }
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(kFull, sum, o);
                    m = __reduce_min_sync(kFull, m);
                    if (lane == 0) {
                        atomicAdd(p.win_sum + ((long long)iw - p.w0), sum);
                        if (p.win_min) atomicMin(p.win_min + ((long long)iw - p.w0), m);
                    }
                }
            } else {
                for (unsigned iw = iw0 + lane; iw <= iw1; iw += 32) {
                    const long long ws = (long long)iw * uW, we = ws + uW;
                    const int s = (int)(max((long long)a0, ws) - a0), e = (int)(min((long long)a1, we) - a0);
                    unsigned long long sum = 0;
                    int m = 0x7fffffff;
                    for (int xx = s; xx < e; xx++) {
                        const int dd = sw[swz_elem_t<BPT>(xx)] + stb[xx / BPT];
                        sum += (unsigned long long)(unsigned)dd;
                        m = min(m, dd);
                    }
                    atomicAdd(p.win_sum + ((long long)iw - p.w0), sum);
                    if (p.win_min) atomicMin(p.win_min + ((long long)iw - p.w0), m);
                }
            }
        }
    }

    // ---- claim output slots for this warp chunk's run starts (claim order; K_gather puts them in position order)
    if (p.do_runs) {
        const int chunk = tile * WARPS + warp;
        unsigned long long off = 0;
        if (lane == 0) {
            if (warp_cnt) {
                off = atomicAdd(reinterpret_cast<unsigned long long*>(p.header), (unsigned long long)warp_cnt);
                atomicAdd(p.super_cnt + (chunk >> kSuperShift), (unsigned)warp_cnt);
            }
            p.chunk_runs[chunk] = ((uint64_t)off << 32) | (unsigned)warp_cnt;
        }
        if (warp_cnt) {                                       // warp-uniform
            off = __shfl_sync(kFull, off, 0);
            long long rank = (long long)off + lane_rank;
            Mask m = mask;
            while (m) {
                const int k = mask_ffs(m) - 1;
                m &= m - 1;
                if (rank < p.run_cap) {
                    p.tmp_start[rank] = p.rs + idx0 + k;
                    p.tmp_class[rank] = (unsigned char)cov_class(tbase + sw[swz_elem_t<BPT>(lane * BPT + k)], p.mincov, p.maxmean);
                }
                rank++;
            }
        }
    }
    if (kSliceInTile && need_slice) {                         // the run claim was the slice's last reader: clear for the next tile
        __syncwarp();
        clear_warp_region<kWElems>(sw, lane);
    }
}

#undef GL_D

// GENERAL path, K_scan: coalesced load of the tile's differences -> swizzled smem -> tile core.
template <bool kMD>
__global__ void __launch_bounds__(kScanThreads, 4) depth_scan_kernel(const ScanParams p) {
    __shared__ __align__(16) int s_tile[kTile];
    __shared__ __align__(16) int s_depth[kTile];
    __shared__ int s_carry[kWarps];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int tile = blockIdx.x;
    const int4* src = reinterpret_cast<const int4*>(p.diff + (size_t)tile * kTile);
    int4 v[4];
#pragma unroll
    for (int r = 0; r < 4; r++) v[r] = ld_stream_int4(src + warp * 128 + r * 32 + lane);   // 512 B per warp-instruction
    {   // depth carried into the tile = sum of everything before it (two-level, overlaps the loads above)
        const int st = tile >> kSuperShift;
        int part = 0;
        for (int k = tid; k < st; k += kScanThreads) part += p.super_sum[k];
        const int k2 = (st << kSuperShift) + tid;
        if (tid < (1 << kSuperShift) && k2 < tile) part += p.tile_sum[k2];
        part = __reduce_add_sync(kFull, part);
        if (lane == 0) s_carry[warp] = part;
    }
#pragma unroll
    for (int r = 0; r < 4; r++) reinterpret_cast<int4*>(s_tile)[swz_chunk(warp * 128 + r * 32 + lane)] = v[r];
    __syncwarp();                                                       // a warp only re-reads its own 128 chunks
    int acc_max = 0;
    tile_core<16, kWarps, false, kMD>(p, s_tile, s_depth, s_carry, tile, acc_max);
    flush_max(p, acc_max);
}

// ================================================================================================
// GENERAL path, version 2 ("bucketed events"): any order, any segment length, no difference array in HBM.
// A segment is two events, +1 at its (clipped) start and -1 at its (clipped) end; an event belongs to the 4096-base
// tile it falls in.  K_evcount counts starts and ends per tile (warp-aggregated reds), K_evscan turns the counts into
// bucket offsets and into the depth carried into every tile (running starts - ends), K_evscatter writes each event as
// 16 bits (position in the tile | sign) into its tile's bucket, K_evtile builds the tile's difference array in shared
// memory from its bucket (coalesced 2-byte reads, shared-memory atomics) and runs the tile core.
// Bytes: 8 B/segment read twice, 4 B/segment written and read once — against 8 B/base for the HBM difference array.
// ================================================================================================
__device__ __forceinline__ void ev_clip(int s, int e, int rs, int re, int& a, int& b, bool& live) {
    a = max(s, rs) - rs;
    b = min(e, re) - rs;
    live = a < b;
}

template <bool kScatter>
__global__ void __launch_bounds__(256) depth_events_kernel(const int* __restrict__ start, const int* __restrict__ end, long long n, int rs, int re,
                                                          int num_tiles, int* __restrict__ tile_starts, int* __restrict__ tile_ends,
                                                          const unsigned* __restrict__ bucket_off, unsigned* __restrict__ cursor,
                                                          unsigned short* __restrict__ events) {
    const long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4;
    const int lane = threadIdx.x & 31;
    int s[4], e[4];
    int cnt = 0;
    const bool vec = ((reinterpret_cast<uintptr_t>(start) | reinterpret_cast<uintptr_t>(end)) & 15) == 0;
    if (i0 + 3 < n && vec) {
        const int4 a4 = ld_stream_int4(reinterpret_cast<const int4*>(start + i0));
        const int4 b4 = ld_stream_int4(reinterpret_cast<const int4*>(end + i0));
        s[0] = a4.x; s[1] = a4.y; s[2] = a4.z; s[3] = a4.w;
        e[0] = b4.x; e[1] = b4.y; e[2] = b4.z; e[3] = b4.w;
        cnt = 4;
    } else {
#pragma unroll
        for (int j = 0; j < 4; j++) if (i0 + j < n) { s[j] = start[i0 + j]; e[j] = end[i0 + j]; cnt = j + 1; }
    }
    if (!kScatter) {
        // per-tile start / end counts; sorted input puts a thread's (and most of a warp's) events in one or two tiles
        int tS = 0, cS = 0, tE = 0, cE = 0;
        bool uni = true;
        int ta_[4], tb_[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            ta_[j] = tb_[j] = -1;
            if (j < cnt) {
                int a, b; bool live;
                ev_clip(s[j], e[j], rs, re, a, b, live);
                if (live) {
                    const int ta = a >> kTileShift, tb = b >> kTileShift;          // tb == num_tiles: an end on the region end, no event
                    ta_[j] = ta; tb_[j] = tb < num_tiles ? tb : -1;
                    if (cS == 0) { tS = ta; cS = 1; } else if (ta == tS) cS++; else uni = false;
                    if (tb_[j] >= 0) { if (cE == 0) { tE = tb; cE = 1; } else if (tb == tE) cE++; else uni = false; }
                }
            }
        }
        if (!uni) {
#pragma unroll
            for (int j = 0; j < 4; j++) { if (ta_[j] >= 0) atomicAdd(tile_starts + ta_[j], 1); if (tb_[j] >= 0) atomicAdd(tile_ends + tb_[j], 1); }
            cS = 0; cE = 0;
        }
        warp_tile_add(tile_starts, tS, cS, 1, lane);
        warp_tile_add(tile_ends, tE, cE, 1, lane);
    } else {
#pragma unroll
        for (int j = 0; j < 4; j++) {
            int a = 0, b = 0; bool live = false;
            if (j < cnt) ev_clip(s[j], e[j], rs, re, a, b, live);
            // two events per live segment; lanes whose event falls in the same tile share one cursor atomic.  (Issuing the eight
            // atomics of a thread before the first shuffle was tried: 48 registers instead of 24, 76 us instead of 62.)
#pragma unroll
            for (int which = 0; which < 2; which++) {
                const int pos = which ? b : a;
                const int t = pos >> kTileShift;
                const bool on = live && t < num_tiles;
                const unsigned grp = __match_any_sync(kFull, on ? t : -1 - lane);   // lanes without an event are alone in their group
                if (on) {
                    const int leader = __ffs(grp) - 1;
                    unsigned base = 0;
                    if (lane == leader) base = atomicAdd(cursor + t, (unsigned)__popc(grp));
                    base = __shfl_sync(grp, base, leader);
                    const unsigned slot = bucket_off[t] + base + (unsigned)__popc(grp & ((1u << lane) - 1u));
                    events[slot] = (unsigned short)((pos & (kTile - 1)) | (which << 15));
                }
            }
        }
    }
}

// bucket_off[t] = events in tiles < t; carry[t] = (starts - ends) in tiles < t = the depth carried into tile t.  One CTA; every
// thread owns a contiguous run of tiles (a multiple of 4: 128-bit loads and stores): thread-local totals, ONE block scan (two
// barriers in all), then the thread walks its run again (L1 hits) and writes.  Both scans ride in one 64-bit word: events in
// the high half, net depth (signed) in the low half.  The count arrays are zero-padded to a multiple of 4 entries past
// num_tiles (ev_layout), and so are the outputs.
__global__ void __launch_bounds__(1024) depth_evscan_kernel(const int* __restrict__ tile_starts, const int* __restrict__ tile_ends, int num_tiles,
                                                           unsigned* __restrict__ bucket_off, int* __restrict__ carry) {
    __shared__ long long s_w[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int T4 = (num_tiles + 2 + 3) & ~3;                        // allocated entries (ev_layout)
    const int per = ((num_tiles + 1 + 1023) / 1024 + 3) & ~3;       // entries per thread
    const int i0 = tid * per;
    long long tot = 0;
#pragma unroll 4
    for (int j = 0; j < per; j += 4) {
        const int i = i0 + j;
        if (i < T4) {
            const int4 st = *reinterpret_cast<const int4*>(tile_starts + i), en = *reinterpret_cast<const int4*>(tile_ends + i);
            tot += ((long long)(st.x + en.x) << 32) + (long long)(st.x - en.x);
            tot += ((long long)(st.y + en.y) << 32) + (long long)(st.y - en.y);
            tot += ((long long)(st.z + en.z) << 32) + (long long)(st.z - en.z);
            tot += ((long long)(st.w + en.w) << 32) + (long long)(st.w - en.w);
        }
    }
    long long inc = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long y = __shfl_up_sync(kFull, inc, o); if (lane >= o) inc += y; }
    if (lane == 31) s_w[warp] = inc;
    __syncthreads();
    const long long wv = s_w[lane];                                 // every warp scans the 32 warp totals
    long long winc = wv;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const long long y = __shfl_up_sync(kFull, winc, o); if (lane >= o) winc += y; }
    long long run = __shfl_sync(kFull, winc, warp) - __shfl_sync(kFull, wv, warp) + inc - tot;     // exclusive prefix of this thread's run
#pragma unroll 2
    for (int j = 0; j < per; j += 4) {
        const int i = i0 + j;
        if (i < T4) {
            const int4 st = *reinterpret_cast<const int4*>(tile_starts + i), en = *reinterpret_cast<const int4*>(tile_ends + i);
            const int sv[4] = {st.x, st.y, st.z, st.w}, ev[4] = {en.x, en.y, en.z, en.w};
            unsigned bo[4];
            int ca[4];
#pragma unroll
            for (int k = 0; k < 4; k++) {
                const long long lo = (long long)(int)(run & 0xffffffffll);       // low word, sign-extended
                bo[k] = (unsigned)((run - lo) >> 32);
                ca[k] = (int)lo;
                run += ((long long)(sv[k] + ev[k]) << 32) + (long long)(sv[k] - ev[k]);
            }
            *reinterpret_cast<uint4*>(bucket_off + i) = make_uint4(bo[0], bo[1], bo[2], bo[3]);
            *reinterpret_cast<int4*>(carry + i) = make_int4(ca[0], ca[1], ca[2], ca[3]);
        }
    }
}

// K_evtile: persistent CTAs (tile += gridDim.x), software-pipelined like K_fused8: while tile n runs its core, the first
// kEvPre * 256 events of tile n+1 are already in flight into registers and so is the bucket range of tile n+2 (round 2's
// one-CTA-per-tile version stalled 6 issue slots per instruction on those dependent loads).  The core clears the tile as it
// reads it.  256 threads x 16 bases (the 128 x 32 shape of K_fused8 measured slower here).
constexpr int kEvThreads = kScanThreads;
constexpr int kEvWarps = kWarps;
constexpr int kEvPre = 6;                              // prefetched events per thread: 1536 per tile (a 30x / 150 bp tile holds ~1400)

struct EvRegs { unsigned short e[kEvPre]; };

__device__ __forceinline__ EvRegs evtile_load(const unsigned short* __restrict__ events, unsigned lo, unsigned hi) {
    EvRegs r;
#pragma unroll
    for (int k = 0; k < kEvPre; k++) {
        const unsigned i = lo + threadIdx.x + (unsigned)k * kEvThreads;
        r.e[k] = i < hi ? events[i] : (unsigned short)0;                // slots beyond the bucket are skipped by index, not by value
    }
    return r;
}

template <bool kMD>
__global__ void __launch_bounds__(kEvThreads, 4) depth_evtile_kernel(const ScanParams p, const unsigned short* __restrict__ events,
                                                                     const unsigned* __restrict__ bucket_off, const int* __restrict__ carry) {
    __shared__ __align__(16) int s_tile[kTile];
    __shared__ __align__(16) int s_depth[kTile];
    __shared__ int s_carry2[2][kEvWarps];
    const int tid = threadIdx.x;
    const int G = gridDim.x, T = p.num_tiles;
#pragma unroll
    for (int j = 0; j < 4; j++) reinterpret_cast<int4*>(s_tile)[tid * 4 + j] = make_int4(0, 0, 0, 0);   // later tiles: cleared by the core
    if (tid < 2 * kEvWarps) (&s_carry2[0][0])[tid] = 0;
    int tile = blockIdx.x;
    unsigned lo = 0, hi = 0, lo2 = 0, hi2 = 0;
    int cin = 0, cin2 = 0;
    if (tile < T) { lo = bucket_off[tile]; hi = bucket_off[tile + 1]; cin = carry[tile]; }
    if (tile + G < T) { lo2 = bucket_off[tile + G]; hi2 = bucket_off[tile + G + 1]; cin2 = carry[tile + G]; }
    EvRegs regs = evtile_load(events, lo, hi);
    __syncthreads();
    int acc_max = 0;
    for (int it = 0; tile < T; tile += G, it ^= 1) {
        int* s_carry = s_carry2[it];
        // an event is (position in the tile | sign << 15)
#pragma unroll
        for (int k = 0; k < kEvPre; k++) {
            const unsigned ev = regs.e[k];
            if (lo + tid + (unsigned)k * kEvThreads < hi) atomicAdd(s_tile + swz_elem((int)(ev & (kTile - 1))), (ev >> 15) ? -1 : 1);
        }
        for (unsigned i = lo + tid + (unsigned)kEvPre * kEvThreads; i < hi; i += kEvThreads) {        // deep tiles only
            const unsigned ev = events[i];
            atomicAdd(s_tile + swz_elem((int)(ev & (kTile - 1))), (ev >> 15) ? -1 : 1);
        }
        if (tid == 0) s_carry[0] = cin;                     // slots 1.. stay 0 (only slot 0 of either buffer is ever written)
        __syncthreads();
        lo = lo2; hi = hi2; cin = cin2;
        regs = evtile_load(events, lo, hi);                 // next tile's events: in flight during the core
        lo2 = hi2 = 0; cin2 = 0;
        if (tile + 2 * G < T) { lo2 = bucket_off[tile + 2 * G]; hi2 = bucket_off[tile + 2 * G + 1]; cin2 = carry[tile + 2 * G]; }
        tile_core<16, kEvWarps, true, kMD>(p, s_tile, s_depth, s_carry, tile, acc_max);
    }
    flush_max(p, acc_max);
}

// FUSED path, K_fused: build each tile's difference array in shared memory straight from the segments.
// Persistent CTAs (tile += gridDim.x), software-pipelined two tiles deep so that no CTA ever waits on
// a dependent global load chain: while tile n runs its core, the segments of tile n+1 are already in
// flight into registers (4 per thread) and so are the cell-table entries of tile n+2.
constexpr int kSegRegs = 4;

struct CellRegs { unsigned lo, hi, cnt; };
struct SegRange { unsigned lo, hi, cnt; };

__device__ __forceinline__ void fused_cells_of(const ScanParams& p, int tile, int maxlen, int& lo_cell, int& hi_cell) {
    // cells whose segments can cover base t0-1 or touch the tile: starts in [t0 - maxlen, t1)
    // (t1 = t0 + min(kTile, re - t0): t0 + kTile itself overflows int when the last tile starts at 2^31 - kTile or later)
    const int t0 = p.rs + tile * kTile;
    const int t1 = t0 + min(kTile, p.re - t0);
    lo_cell = (max(t0 - maxlen, p.origin) - p.origin) >> kCellShift;
    hi_cell = min(((t1 - 1 - p.origin) >> kCellShift) + 1, p.ncells);   // exclusive; at most 82 cells
}

__device__ __forceinline__ CellRegs fused_load_cells(const ScanParams& p, const BatchDesc& bd, int tile, int maxlen) {
    CellRegs r = {0xffffffffu, 0u, 0u};
    if (tile < p.num_tiles) {
        int lo_cell, hi_cell;
        fused_cells_of(p, tile, maxlen, lo_cell, hi_cell);
        const int c = lo_cell + (int)threadIdx.x;
        if (c < hi_cell) { r.lo = ~bd.cell_lo[c]; r.hi = bd.cell_hi[c]; r.cnt = bd.cell_cnt[c]; }
    }
    return r;
}

__device__ __forceinline__ void fused_reduce_cells(const CellRegs& r, unsigned (*s_rng)[kWarps]) {
    const unsigned l = __reduce_min_sync(kFull, r.lo), h = __reduce_max_sync(kFull, r.hi), k = __reduce_add_sync(kFull, r.cnt);
    if ((threadIdx.x & 31) == 0) { const int w = threadIdx.x >> 5; s_rng[0][w] = l; s_rng[1][w] = h; s_rng[2][w] = k; }
}

__device__ __forceinline__ SegRange fused_combine(unsigned (*s_rng)[kWarps]) {
    SegRange g = {0xffffffffu, 0u, 0u};
#pragma unroll
    for (int w = 0; w < kWarps; w++) { g.lo = min(g.lo, s_rng[0][w]); g.hi = max(g.hi, s_rng[1][w]); g.cnt += s_rng[2][w]; }
    return g;
}

__device__ __forceinline__ bool fused_out_of_order(const SegRange& g) {
    return g.hi > g.lo && (unsigned long long)(g.hi - g.lo) > 8ull * g.cnt + 4096ull;
}

// one segment into the tile [t0,t1): +1/-1 in shared memory, or +1 carried in when it covers base t0-1
// Region clipping: rs <= t0 and t1 <= re, so only tile 0 can see starts below rs (they count from its first base)
// and an end beyond re only lands in the masked tail of the last tile: neither needs an explicit clip.
__device__ __forceinline__ void fused_apply(int* s_tile, int t0, int t1, bool first_tile, int s, int e, int& carry) {
    const int sc = first_tile ? max(s, t0) : s;                         // t0 == rs on the first tile
    if (sc < e && sc < t1 && e >= t0) {
        if (sc < t0) carry++;                                           // covers base t0-1: carried in
        else atomicAdd(s_tile + swz_elem(sc - t0), 1);
        if (e - t0 < kTile) atomicAdd(s_tile + swz_elem(e - t0), -1);
    }
}

template <bool kMD>
__global__ void __launch_bounds__(kScanThreads, 4) depth_fused_kernel(const ScanParams p) {
    __shared__ __align__(16) int s_tile[kTile];
    __shared__ __align__(16) int s_depth[kTile];
    __shared__ int s_carry2[2][kWarps];      // double-buffered: a fast warp writes tile n+1's carry while a slow one still reads tile n's
    __shared__ unsigned s_rng[3][kWarps];
    __shared__ unsigned s_rng2[3][kWarps];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = gridDim.x;

    // longest segment (1024 slots written by K_index); segments longer than the look-back go the general way
    int maxlen = 0;
#pragma unroll
    for (int k = 0; k < kLenSlots / kScanThreads; k++) maxlen = max(maxlen, p.flags[16 + tid + k * kScanThreads]);
    maxlen = __reduce_max_sync(kFull, maxlen);
    if (lane == 0) s_carry2[0][warp] = maxlen;
#pragma unroll
    for (int j = 0; j < 4; j++) reinterpret_cast<int4*>(s_tile)[tid * 4 + j] = make_int4(0, 0, 0, 0);   // later tiles: cleared by the core
    __syncthreads();
    maxlen = 0;
#pragma unroll
    for (int w = 0; w < kWarps; w++) maxlen = max(maxlen, s_carry2[0][w]);
    __syncthreads();
    if (maxlen > kMaxLookback) {
        if (blockIdx.x == 0 && tid == 0) p.header[3] = 1;
        return;
    }

    const BatchDesc& b0 = p.batch[0];
    const int* __restrict__ bs = b0.start;
    const int* __restrict__ be = b0.end;
    int tile = blockIdx.x;

    // ---- pipeline prologue: range and segments of the first tile, cell entries of the second
    CellRegs cells = fused_load_cells(p, b0, tile, maxlen);
    fused_reduce_cells(cells, s_rng);
    __syncthreads();
    SegRange cur = fused_combine(s_rng);
    int ss[kSegRegs], se[kSegRegs];
#pragma unroll
    for (int j = 0; j < kSegRegs; j++) {
        const unsigned i = cur.lo + tid + j * kScanThreads;
        const bool ok = i < cur.hi;
        ss[j] = ok ? bs[i] : 0;
        se[j] = ok ? be[i] : 0;
    }
    cells = fused_load_cells(p, b0, tile + G, maxlen);
    __syncthreads();          // every warp has read s_rng before iteration 0 rewrites it (found by compute-sanitizer racecheck)

    int acc_max = 0;
    for (int it = 0; tile < p.num_tiles; tile += G, it ^= 1) {
        int* s_carry = s_carry2[it];
        const int t0 = p.rs + tile * kTile, t1 = t0 + min(kTile, p.re - t0);   // no overflow at the top of int32 (fused_cells_of)
        const bool first_tile = tile == 0;
        // (the previous core's barrier guarantees every warp has read + cleared its slice of the tile)
        if (fused_out_of_order(cur)) {                                  // uniform: every thread holds the same range
            if (tid == 0) p.header[3] = 1;
            return;
        }
        int carry = 0;
#pragma unroll
        for (int j = 0; j < kSegRegs; j++) fused_apply(s_tile, t0, t1, first_tile, ss[j], se[j], carry);
        for (unsigned i = cur.lo + tid + kSegRegs * kScanThreads; i < cur.hi; i += kScanThreads)   // deep tiles only
            fused_apply(s_tile, t0, t1, first_tile, bs[i], be[i], carry);
        for (int b = 1; b < p.n_batches; b++) {                         // further batches: not pipelined
            const BatchDesc& bd = p.batch[b];
            fused_reduce_cells(fused_load_cells(p, bd, tile, maxlen), s_rng2);
            __syncthreads();
            const SegRange g = fused_combine(s_rng2);
            __syncthreads();
            if (fused_out_of_order(g)) {
                if (tid == 0) p.header[3] = 1;
                return;
            }
            for (unsigned i = g.lo + tid; i < g.hi; i += kScanThreads) fused_apply(s_tile, t0, t1, first_tile, bd.start[i], bd.end[i], carry);
        }
        carry = __reduce_add_sync(kFull, carry);
        if (lane == 0) s_carry[warp] = carry;
        fused_reduce_cells(cells, s_rng);                               // range of the next tile
        __syncthreads();
        cur = fused_combine(s_rng);
#pragma unroll
        for (int j = 0; j < kSegRegs; j++) {                            // next tile's segments: in flight during the core
            const unsigned i = cur.lo + tid + j * kScanThreads;
            const bool ok = i < cur.hi;
            ss[j] = ok ? bs[i] : 0;
            se[j] = ok ? be[i] : 0;
        }
        cells = fused_load_cells(p, b0, tile + 2 * G, maxlen);          // and the tile after that one's cell entries
        tile_core<16, kWarps, true, kMD>(p, s_tile, s_depth, s_carry, tile, acc_max);
    }
    flush_max(p, acc_max);
}

// ================================================================================================
// packed8 path.  The segments arrive sorted by start in 64-slot blocks with sorted anchors and lengths <= 255,
// so the blocks a tile needs follow from the anchors alone: no per-segment index pass, no int32 copy of the
// segments in HBM, a quarter of the segment bytes read.
// K_tileidx8: for every tile boundary x_k = rs + k*4096 (k = 0..T) the number of anchors < x_k (cnt_hi[k]) and the number
// of anchors < x_k - 255 (cnt_lo[k]).  Block b's starts lie in [anchor[b], anchor[b+1]] and lengths are <= 255, so tile k
// needs the blocks [max(0, cnt_lo[k] - 1), cnt_hi[k+1]).  No search: thread i owns the gap (anchor[i], anchor[i+1]]
// (i = -1 and nb-1 own the open ends) and writes i+1 for every boundary inside it — usually none, one in ~13 threads
// writes one.  Also verifies that the anchors are sorted.
// ================================================================================================
__device__ __forceinline__ long long floordiv_tile(long long x) { return x >> kTileShift; }   // arithmetic shift = floor

// One-wave grid: each CTA strides over the gaps 256 at a time (the stride is uniform, so whole warps iterate together).
// The reduce's first launch also zeroes the scratch the reduce accumulates into (header, super_cnt, window sums), after
// its wait, because the previous reduce's kernels use the same words.  header[3] is left alone: this kernel's CTAs may
// set it, so a rejection is told apart from a stale value by its tag (p8_tag).
__global__ void __launch_bounds__(256) depth_tileidx8_kernel(const ScanParams p) {
    pdl_launch_dependents();
    pdl_wait();
    const long long stride = (long long)gridDim.x * 256;
    for (long long w = (long long)blockIdx.x * 256 + threadIdx.x; w < p.zero_words; w += stride)
        if (w != 3) p.header[w] = 0;
    const int lane = threadIdx.x & 31;
    const int nb = p.p8_nblocks;
    const int T = p.num_tiles;
    for (long long i0 = (long long)blockIdx.x * 256 + p.idx_begin; i0 < p.idx_end; i0 += stride) {
        const long long i = i0 + threadIdx.x;
        long long h0 = 1, h1 = 0, l0 = 1, l1 = 0;                           // empty ranges
        if (i < p.idx_end) {
            const long long lo_x = i >= 0 ? (long long)p.p8_anchors[i] : LLONG_MIN / 2;
            const long long hi_x = i + 1 < nb ? (long long)p.p8_anchors[i + 1] : LLONG_MAX / 2;
            if (lo_x > hi_x) p.header[3] = p.p8_tag;                        // unsorted anchors: the host falls back
            else {
                // boundaries x_k with lo_x < x_k <= hi_x, and the same for x_k - 255
                h0 = max(0ll, floordiv_tile(lo_x - p.rs) + 1); h1 = min((long long)T, floordiv_tile(hi_x - p.rs));
                l0 = max(0ll, floordiv_tile(lo_x - p.rs + 255) + 1); l1 = min((long long)T, floordiv_tile(hi_x - p.rs + 255));
            }
        }
        const int v = (int)(i + 1);
        // a gap without coverage (centromere, contig ends) spans many boundaries: the warp writes those together
        const bool longr = (h1 - h0 > 2) || (l1 - l0 > 2);
        unsigned m = __ballot_sync(kFull, longr);
        if (!longr) {
            for (long long k = h0; k <= h1; k++) p.tile_hi[k] = v;
            for (long long k = l0; k <= l1; k++) p.tile_lo[k] = v;
        }
        while (m) {
            const int src = __ffs(m) - 1;
            m &= m - 1;
            const long long a0 = __shfl_sync(kFull, h0, src), a1 = __shfl_sync(kFull, h1, src);
            const long long b0 = __shfl_sync(kFull, l0, src), b1 = __shfl_sync(kFull, l1, src);
            const int vv = __shfl_sync(kFull, v, src);
            for (long long k = a0 + lane; k <= a1; k += 32) p.tile_hi[k] = vv;
            for (long long k = b0 + lane; k <= b1; k += 32) p.tile_lo[k] = vv;
        }
    }
}

struct P8Regs { uint2 d, l; int anchor; };

// K_fused8 runs 64-thread CTAs whose threads own 64 consecutive bases each (tile_core<64, 2>): the work that is paid per
// thread and tile — warp scans, class check, window sums, run claim, barrier — is spread over four times the bases of the
// 16-per-thread core (ncu, round 1: 568 warp instructions per thread and tile = 35.5 per base, issue-bound), and each
// barrier waits for two warps.
constexpr int kF8Threads = 64;
constexpr int kF8Warps = kF8Threads / 32;
constexpr int kF8BPT = kTile / kF8Threads;          // 64
constexpr int kF8BlocksPerPass = kF8Threads / 8;    // a block is 8 lanes x 8 slots

// K_fused8's tile buffer has a guard band of kF8Guard entries on either side of the tile: s_tile[-32, 0) is the lead
// guard, s_tile[4096, 4128) the trailing one.  swz_elem_t<64> maps each guard onto itself (it XORs bits 2-4 with bits 6-8,
// which are 7 for [-32, 0) and 0 for [4096, 4128)), so one address expression covers the whole buffer.
constexpr int kF8Guard = 32;

// One segment [s, s+len) into the tile that starts at t0, in tile-relative coordinates a = s - t0, b = a + len: +1 at
// clamp(a) and -1 at clamp(b), where clamp() moves a position before the tile to this lane's slot of the lead guard
// (lane - 32) and one at or past the tile's end to its slot of the trailing guard (4096 + lane):
//   - a segment that ends before the tile puts both events in the lead guard, which adds 0 to the guard's sum;
//   - a segment with a < 0 <= b puts +1 in the lead guard and -1 at b (on base 0 when it ends exactly at t0, as the
//     carry then cancels there), so the lead guard sums to the depth carried into the tile;
//   - starts and ends at or past the tile's end land in the trailing guard, which is never read;
//   - a filler slot (len 0) and a thread past the tile's block range (all zero) add +1 and -1 at the same address.
// A start before the region (first tile) is a carry like any other: the region's first base starts a run regardless, so
// the depth "before" it is never looked at.  Starts / ends beyond the region end fall in the masked tail of the last tile.
// `if (p) atomicAdd(smem, v)` compiles to a divergent region per atomic (BSSY / BRA / address math / ATOMS / BSYNC, ~15
// instructions; ptxas does the same to a predicated `red.shared`), so every event is one unconditional atomic at an
// always-valid address: no predicate, no value select, no carry count, and the eight atomics of a thread interleave
// freely.  Per-lane guard slots keep a warp's clamped events conflict-free.  (Adding zeros at masked positions instead of
// branching made K_fused slower — a quarter of its 1024 register slots per tile are idle — so it keeps the branches.)
__device__ __forceinline__ void fused_apply32(int* s_tile, int a, int len, int lane) {
    const int lo = lane - kF8Guard, hi = kTile + lane;
    atomicAdd(s_tile + swz_elem_t<kF8BPT>(min(max(a, lo), hi)), 1);
    atomicAdd(s_tile + swz_elem_t<kF8BPT>(min(max(a + len, lo), hi)), -1);
}

// thread (tid) takes slots 8*(tid&7)..+7 of block lo + (tid>>3) + 8*pass: one uint2 of start deltas, one of lengths
__device__ __forceinline__ P8Regs fused8_load(const ScanParams& p, int lo, int hi, int pass) {
    P8Regs r = {make_uint2(0u, 0u), make_uint2(0u, 0u), 0};
    const int b = lo + (int)(threadIdx.x >> 3) + kF8BlocksPerPass * pass;
    if (b < hi) {
        r.d = reinterpret_cast<const uint2*>(p.p8_ds)[(size_t)b * 8 + (threadIdx.x & 7)];
        r.l = reinterpret_cast<const uint2*>(p.p8_len)[(size_t)b * 8 + (threadIdx.x & 7)];
        r.anchor = p.p8_anchors[b];
    }
    return r;
}

// Inclusive scan over each 8-lane quarter of the warp (one block's words), as warp_incl_scan: shfl.up within 8-lane
// segments (c = 0x1800) says whether the source lane is in this lane's segment, so a step is a SHFL and a predicated add.
__device__ __forceinline__ int quarter_warp_incl_scan(int v) {
#pragma unroll
    for (int o = 1; o < 8; o <<= 1)
        asm("{\n\t.reg .s32 t;\n\t.reg .pred p;\n\tshfl.sync.up.b32 t|p, %0, %1, 0x1800, -1;\n\t@p add.s32 %0, %0, t;\n\t}" : "+r"(v) : "r"(o));
    return v;
}

__device__ __forceinline__ void fused8_apply(const P8Regs& r, int* s_tile, int t0) {
    if (__ballot_sync(kFull, (r.l.x | r.l.y) != 0) == 0) return;   // no live slot in the whole warp (warp-uniform: no divergence)
    const int lane = threadIdx.x & 31;
    // running sum of the thread's 8 start deltas; byte k of a word, zero-extended: one PRMT (__byte_perm selector 0x444k)
    // where a shift and a mask take two
    int d[8];
    d[0] = r.d.x & 0xff;
    d[1] = d[0] + __byte_perm(r.d.x, 0, 0x4441);
    d[2] = d[1] + __byte_perm(r.d.x, 0, 0x4442);
    d[3] = d[2] + (r.d.x >> 24);
    d[4] = d[3] + (r.d.y & 0xff);
    d[5] = d[4] + __byte_perm(r.d.y, 0, 0x4441);
    d[6] = d[5] + __byte_perm(r.d.y, 0, 0x4442);
    d[7] = d[6] + (r.d.y >> 24);
    const int inc = quarter_warp_incl_scan(d[7]);
    const int base = r.anchor + inc - d[7] - t0;            // tile-relative start of the slot before this thread's first
    fused_apply32(s_tile, base + d[0], (int)(r.l.x & 0xff), lane);
    fused_apply32(s_tile, base + d[1], (int)__byte_perm(r.l.x, 0, 0x4441), lane);
    fused_apply32(s_tile, base + d[2], (int)__byte_perm(r.l.x, 0, 0x4442), lane);
    fused_apply32(s_tile, base + d[3], (int)(r.l.x >> 24), lane);
    fused_apply32(s_tile, base + d[4], (int)(r.l.y & 0xff), lane);
    fused_apply32(s_tile, base + d[5], (int)__byte_perm(r.l.y, 0, 0x4441), lane);
    fused_apply32(s_tile, base + d[6], (int)__byte_perm(r.l.y, 0, 0x4442), lane);
    fused_apply32(s_tile, base + d[7], (int)(r.l.y >> 24), lane);
}

// K_fused8: persistent, software-pipelined like K_fused: while tile n runs its core, the packed words of tile n+1 (two
// passes = 16 blocks, what a 30x tile needs) and the block range of tile n+2 are in flight.  The core keeps its depth
// slice in s_tile (16 KB less shared memory than a separate slice buffer), so a barrier at the top of each tile holds
// every warp until all have cleared their regions.  Segments are added into a guard-banded tile (fused_apply32); after the
// second barrier warp 0 turns the lead guard into the carry (s_carry[0]; the other warps' entries stay 0) and clears it.
template <bool kMD>
__global__ void __launch_bounds__(kF8Threads) depth_fused8_kernel(const ScanParams p) {
    __shared__ __align__(16) int s_buf[kF8Guard + kTile + kF8Guard];
    __shared__ int s_carry[kF8Warps];
    int* const s_tile = s_buf + kF8Guard;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int G = gridDim.x;
    pdl_launch_dependents();
#pragma unroll
    for (int j = 0; j < kF8BPT / 4; j++) reinterpret_cast<int4*>(s_tile)[tid * (kF8BPT / 4) + j] = make_int4(0, 0, 0, 0);   // later tiles: cleared by the core
    if (tid < 2 * kF8Guard) s_buf[tid < kF8Guard ? tid : kTile + tid] = 0;   // the lead guard is cleared again after each tile's read
    if (tid < kF8Warps) s_carry[tid] = 0;
    pdl_wait();
    if (p.header[3] == p.p8_tag) return;                    // K_tileidx8 found unsorted anchors: the host falls back
    int tile = p.tile_begin + blockIdx.x;
    const int nb = p.p8_nblocks;                            // (clamps: garbage ranges of a rejected input stay in bounds)
    int lo = 0, hi = 0, lo2 = 0, hi2 = 0;
    if (tile < p.tile_end) { lo = max(0, p.tile_lo[tile] - 1); hi = min(nb, p.tile_hi[tile + 1]); }
    if (tile + G < p.tile_end) { lo2 = max(0, p.tile_lo[tile + G] - 1); hi2 = min(nb, p.tile_hi[tile + G + 1]); }
    P8Regs regs0 = fused8_load(p, lo, hi, 0), regs1 = fused8_load(p, lo, hi, 1);

    int acc_max = 0;
    for (; tile < p.tile_end; tile += G) {
        __syncthreads();                                    // every warp has cleared its region of s_tile
        const int t0 = p.rs + tile * kTile;
        fused8_apply(regs0, s_tile, t0);
        fused8_apply(regs1, s_tile, t0);
        for (int pass = 2; lo + kF8BlocksPerPass * pass < hi; pass++)     // deep tiles only (uniform trip count)
            fused8_apply(fused8_load(p, lo, hi, pass), s_tile, t0);
        __syncthreads();
        if (warp == 0) {                                    // the core reads s_carry after its own barrier
            const int carry = __reduce_add_sync(kFull, s_tile[lane - kF8Guard]);
            s_tile[lane - kF8Guard] = 0;                    // the next tile's atomics wait at the barrier at the loop's top
            if (lane == 0) s_carry[0] = carry;
        }
        lo = lo2; hi = hi2;
        regs0 = fused8_load(p, lo, hi, 0);                  // next tile's packed words: in flight during the core
        regs1 = fused8_load(p, lo, hi, 1);
        lo2 = hi2 = 0;
        if (tile + 2 * G < p.tile_end) { lo2 = max(0, p.tile_lo[tile + 2 * G] - 1); hi2 = min(nb, p.tile_hi[tile + 2 * G + 1]); }
        tile_core<kF8BPT, kF8Warps, true, kMD, true>(p, s_tile, nullptr, s_carry, tile, acc_max);
    }
    flush_max(p, acc_max);
}

// K_gather: one warp per warp chunk of the core (512 bases; 2048 in K_fused8) moves its runs from claim order to position
// order.  The ordered offset of a chunk is the number of runs that start before it: counts per 64 chunks + the chunk
// counts of its own group (only chunks that have runs pay for the sum).  Warps stride over the chunks, so any grid covers them.
// header[3] == reject: the fast path was rejected (fused int32: 1; packed8: the reduce's tag).  hdr_out (packed8: the
// ctx's mapped host header) receives the header's first four words, rejected or not.
__global__ void __launch_bounds__(256) depth_gather_runs_kernel(const uint64_t* __restrict__ header, uint64_t reject,
                                                               uint64_t* __restrict__ hdr_out,
                                                               const uint64_t* __restrict__ chunk_runs,
                                                               const unsigned* __restrict__ super_cnt, int chunks,
                                                               const int* __restrict__ tmp_start,
                                                               const unsigned char* __restrict__ tmp_class,
                                                               int* __restrict__ run_start, unsigned char* __restrict__ run_class,
                                                               long long cap) {
    pdl_launch_dependents();
    pdl_wait();
    if (hdr_out && blockIdx.x == 0 && threadIdx.x < 4) hdr_out[threadIdx.x] = header[threadIdx.x];
    if (header[3] == reject) return;
    const int lane = threadIdx.x & 31;
    for (int base = (blockIdx.x * 8 + (threadIdx.x >> 5)) * 32; base < chunks; base += gridDim.x * 256) {   // 32 chunks per warp (one coalesced load)
        const uint64_t mine = (base + lane < chunks) ? chunk_runs[base + lane] : 0;
        unsigned nz = __ballot_sync(kFull, (unsigned)mine != 0);
        while (nz) {                                                    // warp-uniform: chunks that have runs
            const int l = __ffs(nz) - 1;
            nz &= nz - 1;
            const int t = base + l;
            const uint64_t w = __shfl_sync(kFull, mine, l);
            const unsigned cnt = (unsigned)w;
            const int st = t >> kSuperShift;
            unsigned part = 0;
            for (int k = lane; k < st; k += 32) part += super_cnt[k];
            for (int k = (st << kSuperShift) + lane; k < t; k += 32) part += (unsigned)chunk_runs[k];
            const long long dst = (long long)__reduce_add_sync(kFull, part);
            const long long src = (long long)(w >> 32);
            for (unsigned i = lane; i < cnt; i += 32) {
                if (src + i < cap && dst + i < cap) {
                    run_start[dst + i] = tmp_start[src + i];
                    run_class[dst + i] = tmp_class[src + i];
                }
            }
        }
    }
}

// Sum of per-base depth over arbitrary intervals [a,b) of the open region, straight from the segments:
// sum_x depth(x) = sum over segments of |segment ∩ [a,b)|.  One warp per interval.  With the cell index of the last
// fused reduce only the segments that can reach the interval are visited; without it (general path) every segment is.
// Used for the clipped edge windows of BED regions (depth/depth.go:293-305 with regionStart/regionEnd inside a window).
__global__ void __launch_bounds__(256) depth_interval_sum_kernel(const ScanParams p, const int* __restrict__ ia, const int* __restrict__ ib,
                                                                long long n_iv, int use_index, long long* __restrict__ out) {
    const long long iv = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (iv >= n_iv) return;
    const int a = max(ia[iv], p.rs), b = min(ib[iv], p.re);
    unsigned long long sum = 0;
    if (a < b) {
        int maxlen = 0;
        if (use_index) {
            for (int k = lane; k < kLenSlots; k += 32) maxlen = max(maxlen, p.flags[16 + k]);
            maxlen = __reduce_max_sync(kFull, maxlen);
        }
        for (int bi = 0; bi < p.n_batches; bi++) {
            const BatchDesc& bd = p.batch[bi];
            unsigned lo = 0, hi = (unsigned)bd.n;
            if (use_index) {
                const int lo_cell = (max(a - maxlen, p.origin) - p.origin) >> kCellShift;
                const int hi_cell = min(((b - 1 - p.origin) >> kCellShift) + 1, p.ncells);
                unsigned l = 0xffffffffu, h = 0;
                for (int c = lo_cell + lane; c < hi_cell; c += 32) { l = min(l, ~bd.cell_lo[c]); h = max(h, bd.cell_hi[c]); }
                lo = __reduce_min_sync(kFull, l);
                hi = __reduce_max_sync(kFull, h);
            }
            for (unsigned i = lo + lane; i < hi; i += 32) {
                const int s = max(bd.start[i], a), e = min(bd.end[i], b);
                if (s < e) sum += (unsigned)(e - s);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(kFull, sum, o);
    if (lane == 0) out[iv] = (long long)sum;
}

__global__ void run_ends_kernel(const int* run_start, int* run_end, long long n, int re) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) run_end[i] = (i + 1 < n) ? run_start[i + 1] : re;
}

// ================================================================================================
// host side
// ================================================================================================
inline int64_t num_tiles_for(int64_t len) { return (len + kTile - 1) / kTile; }
inline size_t diff_entries_for(int64_t len) { return (size_t)num_tiles_for(len) * kTile + 4; }
inline size_t tile_entries_for(int64_t len) { return ((size_t)num_tiles_for(len) + 1 + 3) & ~size_t(3); }
inline size_t super_entries_for(int64_t len) { return (((size_t)num_tiles_for(len) >> kSuperShift) + 2 + 3) & ~size_t(3); }
inline int* tile_sum_ptr(gl_ctx* ctx) { return static_cast<int*>(ctx->diff.p) + diff_entries_for(ctx->re - ctx->rs); }
inline int* super_sum_ptr(gl_ctx* ctx) { return tile_sum_ptr(ctx) + tile_entries_for(ctx->re - ctx->rs); }
inline size_t al256(size_t x) { return (x + 255) & ~size_t(255); }

inline const int32_t* batch_start(gl_ctx* ctx, const gl_seg_batch& b) {
    return b.s ? b.s : static_cast<const int32_t*>(ctx->store_s.p) + b.off;
}
inline const int32_t* batch_end(gl_ctx* ctx, const gl_seg_batch& b) {
    return b.e ? b.e : static_cast<const int32_t*>(ctx->store_e.p) + b.off;
}

// a new reduce is queued: the last one's results, settled or not, are not asked for any more (nothing waits for its work)
void drop_result(gl_ctx* ctx) {
    ctx->depth_reduced = false;
    ctx->pend.active = false;
}

// the segments changed: neither the last reduce's results nor what ctx->diff holds describe them any more
void segments_changed(gl_ctx* ctx) {
    ctx->diff_holds = kPathNone;
    drop_result(ctx);
}

// n segments were written at the end of the store: consecutive host adds extend one contiguous batch
void store_append(gl_ctx* ctx, int64_t n) {
    if (!ctx->batches.empty() && ctx->batches.back().s == nullptr &&
        ctx->batches.back().off + ctx->batches.back().n == ctx->store_n) {
        ctx->batches.back().n += n;
    } else {
        gl_seg_batch b;
        b.off = ctx->store_n; b.n = n;
        ctx->batches.push_back(b);
    }
    ctx->store_n += n;
    segments_changed(ctx);
}

// Queues the upload of packed blocks [b0, b1) on copy_stream: the anchors (4 B per block), then the start deltas or
// offsets and the lengths (block_bytes per block each: 64 for packed8, 512 for packed16).  Records `done` behind them and
// makes the compute stream wait for it.
int upload_blocks(gl_ctx* ctx, void* d_anchor, void* d_ds, void* d_len, const void* h_anchor, const void* h_ds, const void* h_len,
                  int64_t b0, int64_t b1, size_t block_bytes, cudaEvent_t done) {
    const size_t nb = (size_t)(b1 - b0), a0 = (size_t)b0 * 4, o0 = (size_t)b0 * block_bytes;
    GL_CUDA(ctx, cudaMemcpyAsync(static_cast<char*>(d_anchor) + a0, static_cast<const char*>(h_anchor) + a0, nb * 4, cudaMemcpyHostToDevice, ctx->copy_stream));
    GL_CUDA(ctx, cudaMemcpyAsync(static_cast<char*>(d_ds) + o0, static_cast<const char*>(h_ds) + o0, nb * block_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
    GL_CUDA(ctx, cudaMemcpyAsync(static_cast<char*>(d_len) + o0, static_cast<const char*>(h_len) + o0, nb * block_bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
    GL_CUDA(ctx, cudaEventRecord(done, ctx->copy_stream));
    GL_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, done, 0));
    return GL_OK;
}

// host segments may still be streaming into the store on the copy stream: the compute stream waits for them
int join_copies(gl_ctx* ctx) {
    if (!ctx->copies_pending) return GL_OK;
    GL_CUDA(ctx, cudaEventRecord(ctx->ev_copy[0], ctx->copy_stream));
    GL_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->ev_copy[0], 0));
    ctx->copies_pending = false;
    return GL_OK;
}

int launch_scatter(gl_ctx* ctx, const int32_t* d_start, const int32_t* d_end, int64_t n) {
    if (n <= 0) return GL_OK;
    bool vec = ((reinterpret_cast<uintptr_t>(d_start) | reinterpret_cast<uintptr_t>(d_end)) & 15) == 0;
    int* diff = static_cast<int*>(ctx->diff.p);
    int* tsum = tile_sum_ptr(ctx);
    gl_prof_scope prof(ctx, "depth_scatter_kernel");
    if (vec) {
        long long threads = (n >> 2) + (n & 3);
        unsigned grid = (unsigned)((threads + 255) / 256);
        depth_scatter_kernel<true><<<grid, 256, 0, ctx->stream>>>(d_start, d_end, n, (int)ctx->rs, (int)ctx->re, diff, tsum);
    } else {
        unsigned grid = (unsigned)((n + 255) / 256);
        depth_scatter_kernel<false><<<grid, 256, 0, ctx->stream>>>(d_start, d_end, n, (int)ctx->rs, (int)ctx->re, diff, tsum);
    }
    GL_LAUNCHED(ctx, 1);
    return GL_OK;
}

// HBM difference-array path: (re)build the difference array from every batch
int accumulate_general(gl_ctx* ctx) {
    if (ctx->diff_holds == kPathHbmDiff) return GL_OK;
    ctx->diff_holds = kPathNone;                 // the two general paths share ctx->diff
    const int64_t len = ctx->re - ctx->rs;
    const size_t entries = diff_entries_for(len) + tile_entries_for(len) + super_entries_for(len);
    GL_CHECK(gl_buf_reserve(ctx, ctx->diff, entries * 4));
    {
        gl_prof_scope prof(ctx, "memset_diff");
        GL_CUDA(ctx, cudaMemsetAsync(ctx->diff.p, 0, entries * 4, ctx->stream));
    }
    for (const gl_seg_batch& b : ctx->batches) GL_CHECK(launch_scatter(ctx, batch_start(ctx, b), batch_end(ctx, b), b.n));
    const int64_t tiles = num_tiles_for(len);
    const int n_super = (int)((tiles + (1 << kSuperShift) - 1) >> kSuperShift);
    {
        gl_prof_scope prof(ctx, "depth_super_sum_kernel");
        depth_super_sum_kernel<<<(unsigned)((n_super + 7) / 8), 256, 0, ctx->stream>>>(tile_sum_ptr(ctx), super_sum_ptr(ctx), (int)tiles);
    }
    GL_LAUNCHED(ctx, 1);
    ctx->diff_holds = kPathHbmDiff;
    return GL_OK;
}

// bucketed-events general path: (re)build the per-tile event buckets from every batch
//   ctx->diff layout: tile_starts[T+1] | tile_ends[T+1] | cursor[T+1] | bucket_off[T+2] | carry[T+2] | events u16[2 * n_total]
struct EvLayout { int* tile_starts; int* tile_ends; unsigned* cursor; unsigned* bucket_off; int* carry; unsigned short* events; size_t zero_bytes; };
EvLayout ev_layout(gl_ctx* ctx, int64_t tiles) {
    const size_t T = ((size_t)tiles + 2 + 3) & ~size_t(3);
    char* b = static_cast<char*>(ctx->diff.p);
    EvLayout L;
    L.tile_starts = reinterpret_cast<int*>(b);
    L.tile_ends = L.tile_starts + T;
    L.cursor = reinterpret_cast<unsigned*>(L.tile_ends + T);
    L.bucket_off = L.cursor + T;
    L.carry = reinterpret_cast<int*>(L.bucket_off + T);
    L.events = reinterpret_cast<unsigned short*>(L.carry + T);
    L.zero_bytes = 3 * T * 4;
    return L;
}

int accumulate_events(gl_ctx* ctx) {
    if (ctx->diff_holds == kPathEvents) return GL_OK;
    ctx->diff_holds = kPathNone;                 // the two general paths share ctx->diff
    const int64_t len = ctx->re - ctx->rs;
    const int64_t tiles = num_tiles_for(len);
    int64_t n_total = 0;
    for (const gl_seg_batch& b : ctx->batches) n_total += b.n;
    if (2 * n_total >= (int64_t(1) << 32)) return gl_fail(ctx, GL_ERANGE, "more than 2^31 segments in one region");
    const size_t T = ((size_t)tiles + 2 + 3) & ~size_t(3);
    GL_CHECK(gl_buf_reserve(ctx, ctx->diff, 5 * T * 4 + (size_t)n_total * 4 + 64));
    const EvLayout L = ev_layout(ctx, tiles);
    GL_CUDA(ctx, cudaMemsetAsync(ctx->diff.p, 0, L.zero_bytes, ctx->stream));
    for (int pass = 0; pass < 2; pass++) {
        for (const gl_seg_batch& b : ctx->batches) {
            if (b.n <= 0) continue;
            const unsigned grid = (unsigned)(((b.n + 3) / 4 + 255) / 256);
            gl_prof_scope prof(ctx, pass == 0 ? "depth_evcount_kernel" : "depth_evscatter_kernel");
            if (pass == 0)
                depth_events_kernel<false><<<grid, 256, 0, ctx->stream>>>(batch_start(ctx, b), batch_end(ctx, b), b.n, (int)ctx->rs, (int)ctx->re, (int)tiles,
                                                                        L.tile_starts, L.tile_ends, nullptr, nullptr, nullptr);
            else
                depth_events_kernel<true><<<grid, 256, 0, ctx->stream>>>(batch_start(ctx, b), batch_end(ctx, b), b.n, (int)ctx->rs, (int)ctx->re, (int)tiles,
                                                                       nullptr, nullptr, L.bucket_off, L.cursor, L.events);
            GL_LAUNCHED(ctx, 1);
        }
        if (pass == 0) {
            gl_prof_scope prof(ctx, "depth_evscan_kernel");
            depth_evscan_kernel<<<1, 1024, 0, ctx->stream>>>(L.tile_starts, L.tile_ends, (int)tiles, L.bucket_off, L.carry);
            GL_LAUNCHED(ctx, 1);
        }
    }
    ctx->diff_holds = kPathEvents;
    return GL_OK;
}

// The reduce's work is queued: send its header home behind it and leave the rest to depth_resolve (ctx->pend is filled in).
// No wait here, so the next region's work queues up behind this one while the device is still busy.  The slot is
// overwritten in stream order by the next reduce's header; depth_resolve reads it behind an event it records itself.
// (The packed8 path needs no copy: its K_gather stores the header through the slot's device alias.)
int defer_header(gl_ctx* ctx) {
    GL_CUDA(ctx, cudaMemcpyAsync(ctx->hdr_host, ctx->scratch.p, 4 * sizeof(uint64_t), cudaMemcpyDeviceToHost, ctx->stream));
    ctx->pend.active = true;
    return GL_OK;
}

// One launch of the packed8 chain (K_tileidx8 -> K_fused8 -> K_gather, and on into the next reduce): programmatic stream
// serialization lets the kernel launch and ramp up while the one before it drains; it waits at pdl_wait().
template <class... Params, class... Args>
int launch_chained(gl_ctx* ctx, void (*kernel)(Params...), unsigned grid, unsigned block, Args... args) {
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(block);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = ctx->stream;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    GL_CUDA(ctx, cudaLaunchKernelEx(&cfg, kernel, args...));
    GL_LAUNCHED(ctx, 1);
    return GL_OK;
}

// CTAs of a 256-thread kernel the device holds at once (a one-wave grid: every CTA is resident when the wait releases)
int one_wave_256(gl_ctx* ctx, const void* kernel) {
    int nblk = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nblk, kernel, 256, 0) != cudaSuccess || nblk < 1) { cudaGetLastError(); nblk = 1; }
    return ctx->sm_count * nblk;
}

constexpr int kP8ChunksMax = 32;
static int p8_chunks() {                                       // streamed upload: chunks per region (GL_P8_CHUNKS=1 turns streaming off)
    static int k = [] { const char* e = getenv("GL_P8_CHUNKS"); int v = e ? atoi(e) : 3; return v < 1 ? 1 : (v > kP8ChunksMax ? kP8ChunksMax : v); }();
    return k;
}
// Chunk c of K ends at this block.  Every copy costs ~10 us of DMA set-up, and only the LAST chunk's reduce is exposed
// (the others hide behind the next copy), so the chunks halve in size: 8/15, 4/15, 2/15, 1/15 for K = 4.
static int64_t p8_chunk_end(int64_t nb, int c, int K) {
    if (c >= K - 1) return nb;
    const double total = (double)((1ll << K) - 1);
    double acc = 0;
    for (int j = 0; j <= c; j++) acc += (double)(1ll << (K - 1 - j));
    return std::min<int64_t>(nb, (int64_t)((double)nb * acc / total));
}

// a packed8 batch whose upload was deferred (gl_depth_region_packed8): copy all of it now, in one piece
int p8_finish_upload(gl_ctx* ctx) {
    if (!ctx->p8.upload_pending) return GL_OK;
    GL_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_used[0], 0));
    GL_CHECK(upload_blocks(ctx, const_cast<int*>(ctx->p8.anchors), const_cast<void*>(ctx->p8.ds), const_cast<void*>(ctx->p8.len),
                           ctx->p8.h_anchors, ctx->p8.h_ds, ctx->p8.h_len, 0, ctx->p8.n_blocks, 64, ctx->ev_copy[1]));
    ctx->p8.upload_pending = false;
    return GL_OK;
}

// packed8 batch -> int32 arrays in the store (only when something needs them: another batch, a forced path, ...)
int p8_materialize(gl_ctx* ctx) {
    if (!ctx->p8.pending) return GL_OK;
    GL_CHECK(p8_finish_upload(ctx));
    {
        gl_prof_scope prof(ctx, "depth_unpack8_kernel");
        depth_unpack8_kernel<<<(unsigned)((ctx->p8.n_blocks + 31) / 32), 256, 0, ctx->stream>>>(
            ctx->p8.anchors, static_cast<const uint2*>(ctx->p8.ds), static_cast<const uint2*>(ctx->p8.len), ctx->p8.n_blocks,
            static_cast<int*>(ctx->store_s.p) + ctx->p8.store_off, static_cast<int*>(ctx->store_e.p) + ctx->p8.store_off);
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaEventRecord(ctx->ev_used[0], ctx->stream));
    ctx->p8.pending = false;
    return GL_OK;
}

int reserve_runs(gl_ctx* ctx, size_t cap) {
    GL_CHECK(gl_buf_reserve(ctx, ctx->run_start, cap * 4));
    GL_CHECK(gl_buf_reserve(ctx, ctx->run_class, cap));
    GL_CHECK(gl_buf_reserve(ctx, ctx->run_tmp_start, cap * 4));
    GL_CHECK(gl_buf_reserve(ctx, ctx->run_tmp_class, cap));
    return GL_OK;
}

// One reduce as every path lays it out.  `scratch` holds, with everything that must start at zero in front so one memset
// clears it:
//   [header u64[8] | super_cnt u32[supers]] [win_sum u64[n_windows]] [zeroed: the path's own] | chunk_runs u64[chunks] | [tail: the path's own]
// The run table has one entry per warp chunk of the kernel that runs: chunks = tiles x its warps per tile.
struct Reduce {
    ScanParams p;                 // the fields every path shares are filled in
    int64_t tiles = 0, n_windows = 0, chunks = 0;
    char* zeroed = nullptr;
    char* tail = nullptr;
};

// zero_on_device: the path's first kernel zeroes the scratch itself (p.zero_words), with no memset in front of it
int reduce_begin(gl_ctx* ctx, const ReduceArgs& a, int warps, size_t zeroed_bytes, size_t tail_bytes, Reduce& r, bool zero_on_device = false) {
    const int64_t len = ctx->re - ctx->rs;
    const int64_t w0 = ctx->rs / a.W;
    const bool want_min = a.do_windows && a.want_min;
    r.tiles = num_tiles_for(len);
    r.n_windows = (ctx->re - 1) / a.W - w0 + 1;
    r.chunks = r.tiles * warps;
    if (want_min) GL_CHECK(gl_buf_reserve(ctx, ctx->win_min, (size_t)r.n_windows * 4));
    const size_t supers = (size_t)(r.chunks >> kSuperShift) + 2;
    const size_t head_bytes = al256(kHeaderWords * 8 + supers * 4);
    const size_t win_bytes = al256(a.do_windows ? (size_t)r.n_windows * 8 : 0);
    const size_t zero_bytes = head_bytes + win_bytes + zeroed_bytes;
    const size_t run_bytes = al256((size_t)r.chunks * 8);
    GL_CHECK(gl_buf_reserve(ctx, ctx->scratch, zero_bytes + run_bytes + tail_bytes));
    if (a.do_runs && ctx->run_start.cap == 0) GL_CHECK(reserve_runs(ctx, (size_t)(len / 16 + 4096)));
    char* sbase = static_cast<char*>(ctx->scratch.p);
    ctx->win_sum_p = sbase + head_bytes;
    r.zeroed = sbase + head_bytes + win_bytes;
    r.tail = sbase + zero_bytes + run_bytes;
    if (!zero_on_device) GL_CUDA(ctx, cudaMemsetAsync(sbase, 0, zero_bytes, ctx->stream));
    if (want_min) GL_CUDA(ctx, cudaMemsetAsync(ctx->win_min.p, 0x7f, (size_t)r.n_windows * 4, ctx->stream));

    ScanParams& p = r.p;
    memset(&p, 0, sizeof p);
    p.zero_words = zero_on_device ? (long long)(zero_bytes / 8) : 0;
    p.len = (int)len;
    p.rs = (int)ctx->rs;
    p.re = (int)ctx->re;
    p.W = a.W;
    p.W_inv = a.W >= 2 ? (unsigned)((uint64_t(1) << 32) / (uint64_t)a.W) : 0u;
    p.w0 = w0;
    p.mincov = a.mincov;
    p.maxmean = a.maxmean;
    p.run_break = (a.run_break >= (int64_t(1) << 32)) ? 0u : (unsigned)a.run_break;
    p.header = reinterpret_cast<uint64_t*>(sbase);
    p.chunk_runs = reinterpret_cast<uint64_t*>(sbase + zero_bytes);
    p.super_cnt = reinterpret_cast<unsigned*>(p.header + kHeaderWords);
    p.depth_out = a.d_depth_out;
    p.num_tiles = (int)r.tiles;
    p.do_windows = a.do_windows ? 1 : 0;
    p.do_runs = a.do_runs ? 1 : 0;
    p.md = ctx->md_ep;
    p.win_sum = static_cast<unsigned long long*>(ctx->win_sum_p);
    p.win_min = want_min ? static_cast<int*>(ctx->win_min.p) : nullptr;
    p.tmp_start = static_cast<int*>(ctx->run_tmp_start.p);
    p.tmp_class = static_cast<unsigned char*>(ctx->run_tmp_class.p);
    if (a.do_runs) {
        p.run_cap = (long long)ctx->run_class.cap;
        p.run_cap = std::min<long long>(p.run_cap, (long long)(ctx->run_start.cap / 4));
        p.run_cap = std::min<long long>(p.run_cap, (long long)ctx->run_tmp_class.cap);
        p.run_cap = std::min<long long>(p.run_cap, (long long)(ctx->run_tmp_start.cap / 4));
    }
    return GL_OK;
}

// The path's kernels are queued: put the claimed runs in position order, send the sums (from window w_sent on: a streamed
// packed8 reduce has sent the ones before already) and the first runs to a one-call entry's host buffers while the header
// is read, and leave the rest to depth_resolve.
int reduce_end(gl_ctx* ctx, const Reduce& r, int path, int64_t w_sent) {
    const ScanParams& p = r.p;
    int* const run_start = static_cast<int*>(ctx->run_start.p);
    unsigned char* const run_class = static_cast<unsigned char*>(ctx->run_class.p);
    if (path == kPathPacked8) {
        // always launched, as the last link of the chain: it also stores the header into the mapped host slot
        static int gather_wave = 0;
        if (gather_wave == 0) gather_wave = one_wave_256(ctx, reinterpret_cast<const void*>(depth_gather_runs_kernel));
        const int chunks = p.do_runs ? (int)r.chunks : 0;
        gl_prof_scope prof(ctx, "depth_gather_runs_kernel");
        GL_CHECK(launch_chained(ctx, depth_gather_runs_kernel, (unsigned)std::max<int64_t>(1, std::min<int64_t>((chunks + 255) / 256, gather_wave)), 256,
                                (const uint64_t*)p.header, (uint64_t)p.p8_tag, ctx->hdr_dev, (const uint64_t*)p.chunk_runs,
                                (const unsigned*)p.super_cnt, chunks, (const int*)p.tmp_start, (const unsigned char*)p.tmp_class,
                                run_start, run_class, p.run_cap));
    } else if (p.do_runs) {
        gl_prof_scope prof(ctx, "depth_gather_runs_kernel");
        depth_gather_runs_kernel<<<(unsigned)((r.chunks + 255) / 256), 256, 0, ctx->stream>>>(
            p.header, 1, nullptr, p.chunk_runs, p.super_cnt, (int)r.chunks, p.tmp_start, p.tmp_class, run_start, run_class, p.run_cap);
        GL_LAUNCHED(ctx, 1);
    }
    ctx->prefetched = false;
    if (ctx->prefetch_sums && p.do_windows && r.n_windows <= ctx->prefetch_cap) {
        if (r.n_windows > w_sent)
            GL_CUDA(ctx, cudaMemcpyAsync(ctx->prefetch_sums + w_sent, static_cast<const char*>(ctx->win_sum_p) + w_sent * 8,
                                         (size_t)(r.n_windows - w_sent) * 8, cudaMemcpyDeviceToHost, ctx->stream));
        ctx->prefetched = true;
    }
    ctx->prefetched_runs = 0;
    if (ctx->prefetch_run_start && ctx->prefetch_run_class && p.do_runs) {     // usually all of them
        const int64_t k = std::min<int64_t>(std::min<int64_t>(ctx->prefetch_run_cap, 16384), (int64_t)p.run_cap);
        if (k > 0) {
            GL_CUDA(ctx, cudaMemcpyAsync(ctx->prefetch_run_start, ctx->run_start.p, (size_t)k * 4, cudaMemcpyDeviceToHost, ctx->stream));
            GL_CUDA(ctx, cudaMemcpyAsync(ctx->prefetch_run_class, ctx->run_class.p, (size_t)k, cudaMemcpyDeviceToHost, ctx->stream));
            ctx->prefetched_runs = k;
        }
    }
    ctx->pend.path = path;
    ctx->pend.run_cap = p.run_cap;
    ctx->pend.n_windows = r.n_windows;
    ctx->pend.d2h = w_sent > 0;
    ctx->pend.flags = p.flags;                 // the fused path's index tables (null on the other paths) start with
    ctx->pend.cells = p.batch[0].cell_hi;      // batch 0's cell_hi
    ctx->pend.origin = p.origin;
    ctx->pend.ncells = p.ncells;
    ctx->pend.tag = p.p8_tag;
    if (path == kPathPacked8) {
        ctx->pend.active = true;
        return GL_OK;
    }
    return defer_header(ctx);
}

// The region's only batch is packed8: K_tileidx8 + K_fused8 straight from the packed words.
// When the anchors turn out unsorted (hand-made input) the header says so and depth_resolve unpacks and takes the other paths.
int reduce_packed8(gl_ctx* ctx, const ReduceArgs& a) {
    const size_t tile_tab = al256((size_t)(num_tiles_for(ctx->re - ctx->rs) + 1) * 4);
    Reduce r;
    GL_CHECK(reduce_begin(ctx, a, kF8Warps, 0, 2 * tile_tab, r, true));   // tail: tile_lo | tile_hi; the first K_tileidx8 zeroes
    static int f8_ctas_per_sm = 0;                            // persistent grid: what fits on an SM (registers decide)
    if (f8_ctas_per_sm == 0) {
        int nblk = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nblk, depth_fused8_kernel<false>, kF8Threads, 0) != cudaSuccess || nblk < 1) { cudaGetLastError(); nblk = 4; }
        f8_ctas_per_sm = nblk;
    }
    static int tileidx_wave = 0;
    if (tileidx_wave == 0) tileidx_wave = one_wave_256(ctx, reinterpret_cast<const void*>(depth_tileidx8_kernel));
    ScanParams& p = r.p;
    p.p8_tag = ctx->p8_tag++;
    p.p8_anchors = ctx->p8.anchors;
    p.p8_ds = static_cast<const unsigned*>(ctx->p8.ds);
    p.p8_len = static_cast<const unsigned*>(ctx->p8.len);
    p.p8_nblocks = (int)ctx->p8.n_blocks;
    p.tile_lo = reinterpret_cast<int*>(r.tail);
    p.tile_hi = reinterpret_cast<int*>(r.tail + tile_tab);
    // One pass over everything that is on the device — or, when the upload was deferred, chunk by chunk: the words
    // are sorted by position, so once a chunk has landed every tile that ends before its last anchor can be reduced
    // while the next chunk is still on the wire.
    const int64_t nb = ctx->p8.n_blocks, tiles = r.tiles, n_windows = r.n_windows;
    const bool streamed = ctx->p8.upload_pending;
    const int n_chunks = streamed ? p8_chunks() : 1;
    if (streamed) {
        while ((int)ctx->ev_chunk.size() < 2 * n_chunks) {
            cudaEvent_t ev;
            GL_CUDA(ctx, cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
            ctx->ev_chunk.push_back(ev);
        }
        GL_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_used[0], 0));   // previous consumer done with the staging buffer
    }
    int64_t b0 = 0, t_prev = 0, w_sent = 0;             // w_sent: window sums already on their way home
    const bool early_sums = streamed && ctx->prefetch_sums && a.do_windows && n_windows <= ctx->prefetch_cap;
    for (int c = 0; c < n_chunks; c++) {
        const bool last = c == n_chunks - 1;
        const int64_t b1 = p8_chunk_end(nb, c, n_chunks);
        if (b1 <= b0 && !last) continue;
        if (streamed && b1 > b0)
            GL_CHECK(upload_blocks(ctx, const_cast<int*>(ctx->p8.anchors), const_cast<void*>(ctx->p8.ds), const_cast<void*>(ctx->p8.len),
                                   ctx->p8.h_anchors, ctx->p8.h_ds, ctx->p8.h_len, b0, b1, 64, ctx->ev_chunk[c]));
        // anchor gaps this chunk completes: (a[i], a[i+1]] for i in [b0-1, b1-1), plus the open end after the last anchor
        p.idx_begin = (int)(b0 - 1);
        p.idx_end = (int)(last ? nb : b1 - 1);
        if (p.idx_end > p.idx_begin) {
            gl_prof_scope prof(ctx, "depth_tileidx8_kernel");
            GL_CHECK(launch_chained(ctx, depth_tileidx8_kernel, (unsigned)std::min<int64_t>(((int64_t)p.idx_end - p.idx_begin + 255) / 256, tileidx_wave),
                                    256, (const ScanParams)p));
            p.zero_words = 0;                                 // later chunks' launches must not zero again
        }
        // tiles whose end boundary is not beyond the last anchor on the device are complete
        int64_t t_ready = tiles;
        if (!last) {
            const int64_t a_last = streamed ? (int64_t)ctx->p8.h_anchors[b1 - 1] : 0;
            t_ready = std::min<int64_t>(tiles, std::max<int64_t>(t_prev, (a_last - ctx->rs) >> kTileShift));
        }
        if (t_ready > t_prev) {
            p.tile_begin = (int)t_prev;
            p.tile_end = (int)t_ready;
            gl_prof_scope prof(ctx, "depth_fused8_kernel");
            auto k8 = p.md.mode ? depth_fused8_kernel<true> : depth_fused8_kernel<false>;   // the multidepth epilogue, or none
            GL_CHECK(launch_chained(ctx, k8, (unsigned)std::min<int64_t>(t_ready - t_prev, (int64_t)ctx->sm_count * f8_ctas_per_sm), kF8Threads,
                                    (const ScanParams)p));
        }
        if (early_sums && !last && t_ready > t_prev) {
            // windows that end at or before the last reduced tile's end are final: send them home on their own stream
            const int64_t w_done = std::min<int64_t>(n_windows, std::max<int64_t>(w_sent, (ctx->rs + t_ready * kTile) / a.W - p.w0));
            if (w_done > w_sent) {
                cudaEvent_t ev = ctx->ev_chunk[(size_t)n_chunks + c];
                GL_CUDA(ctx, cudaEventRecord(ev, ctx->stream));
                GL_CUDA(ctx, cudaStreamWaitEvent(ctx->d2h_stream, ev, 0));
                GL_CUDA(ctx, cudaMemcpyAsync(ctx->prefetch_sums + w_sent, static_cast<const char*>(ctx->win_sum_p) + w_sent * 8,
                                             (size_t)(w_done - w_sent) * 8, cudaMemcpyDeviceToHost, ctx->d2h_stream));
                w_sent = w_done;
            }
        }
        t_prev = t_ready;
        b0 = b1;
    }
    ctx->p8.upload_pending = false;
    GL_CHECK(reduce_end(ctx, r, kPathPacked8, w_sent));
    // words from the packed staging buffer (host adds): it may be overwritten after this.  Device words (the caller's own
    // buffers) need no event, so consecutive resident reduces hold nothing but the chain's kernels.
    if (ctx->p8.anchors == ctx->packed.p) GL_CUDA(ctx, cudaEventRecord(ctx->ev_used[0], ctx->stream));
    return GL_OK;
}

inline bool general_path(int path) { return path == kPathHbmDiff || path == kPathEvents; }

// int32 batches: the fused path (K_index per batch + K_fused; the device decides eligibility), else a general path
// (bucketed events, or the HBM difference array on request).
int reduce_int32(gl_ctx* ctx, const ReduceArgs& a, int from) {
    bool try_fused = !general_path(from) && !general_path(ctx->force_path) && !ctx->batches.empty() && (int)ctx->batches.size() <= kMaxBatches;
    for (const gl_seg_batch& b : ctx->batches) if (b.n >= INT32_MAX) try_fused = false;
    const int path = try_fused ? kPathFused : (ctx->force_path == kPathHbmDiff ? kPathHbmDiff : kPathEvents);
    const int origin = (int)(std::max<int64_t>(0, ctx->rs - kMaxLookback) & ~int64_t((1 << kCellShift) - 1));
    const int ncells = (int)(((ctx->re - 1 - origin) >> kCellShift) + 1);
    const size_t nb = ctx->batches.size();
    const size_t flag_bytes = al256(kFlagWords * 4);
    Reduce r;     // zeroed for the fused path: flags | cell_hi | cell_cnt | cell_lo, each cell table [batch][cell]
    GL_CHECK(reduce_begin(ctx, a, path == kPathEvents ? kEvWarps : kWarps, try_fused ? flag_bytes + al256((size_t)ncells * 4 * 3 * nb) : 0, 0, r));
    ScanParams& p = r.p;
    if (path == kPathFused) {
        int* flags = reinterpret_cast<int*>(r.zeroed);
        unsigned* hi_all = reinterpret_cast<unsigned*>(r.zeroed + flag_bytes);
        unsigned* cnt_all = hi_all + (size_t)ncells * nb;
        unsigned* lo_all = cnt_all + (size_t)ncells * nb;
        p.flags = flags;
        p.origin = origin;
        p.ncells = ncells;
        p.n_batches = (int)nb;
        for (size_t bi = 0; bi < nb; bi++) {
            const gl_seg_batch& b = ctx->batches[bi];
            p.batch[bi].start = batch_start(ctx, b);
            p.batch[bi].end = batch_end(ctx, b);
            p.batch[bi].cell_lo = lo_all + bi * (size_t)ncells;
            p.batch[bi].cell_hi = hi_all + bi * (size_t)ncells;
            p.batch[bi].cell_cnt = cnt_all + bi * (size_t)ncells;
            p.batch[bi].n = (int)b.n;
            gl_prof_scope prof(ctx, "depth_index_kernel");
            depth_index_kernel<<<(unsigned)(((b.n + 3) / 4 + 255) / 256), 256, 0, ctx->stream>>>(
                p.batch[bi].start, p.batch[bi].end, b.n, origin, (int)ctx->re, ncells, lo_all + bi * (size_t)ncells,
                hi_all + bi * (size_t)ncells, cnt_all + bi * (size_t)ncells, flags);
            GL_LAUNCHED(ctx, 1);
        }
    }
    EvLayout evl = {};
    if (path == kPathHbmDiff) {
        GL_CHECK(accumulate_general(ctx));
        p.diff = static_cast<const int*>(ctx->diff.p);
        p.tile_sum = tile_sum_ptr(ctx);
        p.super_sum = super_sum_ptr(ctx);
    } else if (path == kPathEvents) {
        GL_CHECK(accumulate_events(ctx));
        evl = ev_layout(ctx, r.tiles);
    }
    {
        gl_prof_scope prof(ctx, path == kPathFused ? "depth_fused_kernel" : (path == kPathHbmDiff ? "depth_scan_kernel" : "depth_evtile_kernel"));
        const unsigned persistent_grid = (unsigned)std::min<int64_t>(r.tiles, (int64_t)ctx->sm_count * 4);
        const bool md = p.md.mode != 0;                       // the multidepth epilogue, or none
        if (path == kPathFused) (md ? depth_fused_kernel<true> : depth_fused_kernel<false>)<<<persistent_grid, kScanThreads, 0, ctx->stream>>>(p);
        else if (path == kPathHbmDiff) (md ? depth_scan_kernel<true> : depth_scan_kernel<false>)<<<(unsigned)r.tiles, kScanThreads, 0, ctx->stream>>>(p);
        else (md ? depth_evtile_kernel<true> : depth_evtile_kernel<false>)<<<persistent_grid, kEvThreads, 0, ctx->stream>>>(p, evl.events, evl.bucket_off, evl.carry);
    }
    GL_LAUNCHED(ctx, 1);
    return reduce_end(ctx, r, path, 0);
}

// Queues one pass of the tile core over the region on the fastest path the input may take, starting no faster than
// `from` (a rerun: depth_resolve) or ctx->force_path: packed8, else fused int32, else a general path.  The device decides
// a fast path's eligibility; depth_resolve learns it from the header and reruns on the next path when needed.
int run_reduce(gl_ctx* ctx, const ReduceArgs& a, int from = kPathPacked8) {
    drop_result(ctx);
    ctx->pend.args = a;
    GL_CHECK(join_copies(ctx));
    if (ctx->p8.pending) {
        if (from == kPathPacked8 && ctx->force_path == kPathNone && ctx->batches.size() == 1 &&
            num_tiles_for(ctx->re - ctx->rs) < (int64_t(1) << 30) && ctx->p8.n_blocks < INT32_MAX)
            return reduce_packed8(ctx, a);
        GL_CHECK(p8_materialize(ctx));
    }
    return reduce_int32(ctx, a, from);
}

constexpr int64_t kStageSegs = int64_t(1) << 22;      // segments per pinned staging slot (2 x 16 MiB)

bool is_pinned_host(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}

// grow the ctx segment store to hold `need` segments, keeping its contents
int store_reserve(gl_ctx* ctx, int64_t need) {
    const size_t bytes = (size_t)need * 4;
    if (bytes <= ctx->store_s.cap && bytes <= ctx->store_e.cap) return GL_OK;
    const size_t want = std::max(bytes, ctx->store_s.cap * 2);
    gl_buf ns, ne;
    GL_CHECK(gl_buf_reserve(ctx, ns, want));
    GL_CHECK(gl_buf_reserve(ctx, ne, want));
    if (ctx->store_n > 0) {
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
        GL_CUDA(ctx, cudaMemcpyAsync(ns.p, ctx->store_s.p, (size_t)ctx->store_n * 4, cudaMemcpyDeviceToDevice, ctx->stream));
        GL_CUDA(ctx, cudaMemcpyAsync(ne.p, ctx->store_e.p, (size_t)ctx->store_n * 4, cudaMemcpyDeviceToDevice, ctx->stream));
    }
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (ctx->store_s.p) cudaFree(ctx->store_s.p);
    if (ctx->store_e.p) cudaFree(ctx->store_e.p);
    ctx->store_s = ns;
    ctx->store_e = ne;
    return GL_OK;
}

int region_fetch(gl_ctx* ctx, int64_t* sum_out, int64_t win_cap, int64_t* n_windows, int32_t* run_start, uint8_t* run_class,
                 int64_t run_cap, int64_t* n_runs) {
    GL_CHECK(depth_resolve(ctx));
    const int64_t nw = ctx->n_windows, nr = ctx->n_runs;
    if (n_windows) *n_windows = nw;
    if (n_runs) *n_runs = nr;
    if (nw > win_cap) return gl_fail(ctx, GL_ERANGE, "gl_depth_region: %lld windows > cap %lld", (long long)nw, (long long)win_cap);
    if (nr > run_cap) return gl_fail(ctx, GL_ERANGE, "gl_depth_region: %lld runs > cap %lld", (long long)nr, (long long)run_cap);
    const bool have_sums = ctx->prefetched, have_runs = ctx->prefetched_runs >= nr;
    ctx->prefetched = false;
    ctx->prefetched_runs = 0;
    if (have_sums && have_runs) return GL_OK;                  // everything came home with the header (depth_resolve waited for it)
    if (!have_sums) GL_CUDA(ctx, cudaMemcpyAsync(sum_out, ctx->win_sum_p, (size_t)nw * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (nr > 0 && !have_runs) {
        GL_CUDA(ctx, cudaMemcpyAsync(run_start, ctx->run_start.p, (size_t)nr * 4, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaMemcpyAsync(run_class, ctx->run_class.p, (size_t)nr, cudaMemcpyDeviceToHost, ctx->stream));
    }
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

// The one-call entries: begin, add (the entry's own form), reduce with the sums and the first runs sent straight to the
// caller's buffers behind the header, fetch the rest.
template <class Add>
int region_one_call(gl_ctx* ctx, int64_t rs, int64_t re, Add add, int32_t W, int32_t mincov, int32_t maxmean, int64_t run_break,
                    int64_t* sum_out, int64_t win_cap, int64_t* n_windows, int32_t* run_start, uint8_t* run_class, int64_t run_cap,
                    int64_t* n_runs) {
    GL_CHECK(gl_depth_begin(ctx, rs, re));
    GL_CHECK(add());
    ctx->prefetch_sums = sum_out; ctx->prefetch_cap = sum_out ? win_cap : 0;
    ctx->prefetch_run_start = run_start; ctx->prefetch_run_class = run_class; ctx->prefetch_run_cap = (run_start && run_class) ? run_cap : 0;
    const int rc_reduce = gl_depth_reduce(ctx, W, mincov, maxmean, run_break);
    ctx->prefetch_sums = nullptr; ctx->prefetch_cap = 0;
    ctx->prefetch_run_start = nullptr; ctx->prefetch_run_class = nullptr; ctx->prefetch_run_cap = 0;
    GL_CHECK(rc_reduce);
    return region_fetch(ctx, sum_out, win_cap, n_windows, run_start, run_class, run_cap, n_runs);
}

}  // namespace

int depth_resolve(gl_ctx* ctx) {
    while (ctx->pend.active) {
        const auto q = ctx->pend;
        ctx->pend.active = false;
        GL_CUDA(ctx, cudaEventRecord(ctx->ev_hdr, ctx->stream));            // behind the pending reduce and its header
        GL_CUDA(ctx, cudaEventSynchronize(ctx->ev_hdr));
        if (q.d2h) GL_CUDA(ctx, cudaStreamSynchronize(ctx->d2h_stream));
        const volatile uint64_t* hdr = ctx->hdr_host;                       // packed8: written by the device through the mapping
        // packed8 anchors not sorted (this reduce's tag) / int32 input not in BAM order
        if (q.path == kPathPacked8 ? hdr[3] == q.tag : (q.path == kPathFused && hdr[3] != 0)) {
            ctx->prefetched = false;
            ctx->prefetched_runs = 0;
            GL_CHECK(run_reduce(ctx, q.args, q.path == kPathPacked8 ? kPathFused : kPathEvents));   // the next path down
            continue;
        }
        if (q.args.do_runs && (long long)hdr[0] > q.run_cap) {                  // the runs did not fit: grow and take the same path again
            GL_CHECK(reserve_runs(ctx, (size_t)hdr[0] + 1024));
            GL_CHECK(run_reduce(ctx, q.args, q.path));
            continue;
        }
        ctx->last_path = q.path;
        ctx->idx_flags = q.flags;
        ctx->idx_cells = q.cells;
        ctx->idx_origin = q.origin;
        ctx->idx_ncells = q.ncells;
        ctx->n_runs = q.args.do_runs ? (int64_t)hdr[0] : 0;
        ctx->max_depth = (int32_t)hdr[2];
        ctx->red = q.args;
        ctx->n_windows = q.args.do_windows ? q.n_windows : 0;
        ctx->depth_reduced = true;
    }
    return GL_OK;
}

int depth_reduce_epilogue(gl_ctx* ctx, int32_t* d_depth_out) {
    if (!ctx->depth_active) return gl_fail(ctx, GL_ESTATE, "multidepth: no region open (call gl_depth_begin)");
    ReduceArgs a;
    a.W = (int32_t)std::min<int64_t>(ctx->re, INT32_MAX);      // one window; windows are not computed
    a.mincov = 1;
    a.d_depth_out = d_depth_out;
    GL_CHECK(run_reduce(ctx, a));
    return depth_resolve(ctx);
}

extern "C" {

int gl_depth_begin(gl_ctx* ctx, int64_t region_start, int64_t region_end) {
    GL_CHECK(gl_use(ctx));
    if (region_start < 0 || region_end <= region_start || region_end > INT32_MAX)
        return gl_fail(ctx, GL_EINVAL, "gl_depth_begin: bad region [%lld,%lld)", (long long)region_start, (long long)region_end);
    const int64_t len = region_end - region_start;
    if (len >= (int64_t(1) << 30)) return gl_fail(ctx, GL_ERANGE, "gl_depth_begin: region longer than 2^30-1 bases");
    if (ctx->copies_pending) { GL_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream)); ctx->copies_pending = false; }
    ctx->rs = region_start;
    ctx->re = region_end;
    ctx->batches.clear();
    ctx->store_n = 0;
    ctx->p8.pending = false;
    ctx->p8.upload_pending = false;
    ctx->depth_active = true;
    segments_changed(ctx);     // nobody can ask for a pending result any more; its scratch is reused in stream order
    ctx->n_windows = 0;
    ctx->n_runs = 0;
    ctx->max_depth = 0;
    return GL_OK;
}

int gl_depth_add_segments_device(gl_ctx* ctx, const int32_t* d_start, const int32_t* d_end, int64_t n) {
    GL_CHECK(gl_use(ctx));
    if (!ctx->depth_active) return gl_fail(ctx, GL_ESTATE, "gl_depth_add_segments: no region open (call gl_depth_begin)");
    if (n < 0 || (n > 0 && (!d_start || !d_end))) return gl_fail(ctx, GL_EINVAL, "gl_depth_add_segments: bad argument");
    if (n == 0) return GL_OK;
    GL_CHECK(p8_materialize(ctx));
    gl_seg_batch b;
    b.s = d_start; b.e = d_end; b.n = n;
    ctx->batches.push_back(b);
    segments_changed(ctx);
    return GL_OK;
}

int gl_depth_add_segments(gl_ctx* ctx, const int32_t* start, const int32_t* end, int64_t n) {
    GL_CHECK(gl_use(ctx));
    if (!ctx->depth_active) return gl_fail(ctx, GL_ESTATE, "gl_depth_add_segments: no region open (call gl_depth_begin)");
    if (n < 0 || (n > 0 && (!start || !end))) return gl_fail(ctx, GL_EINVAL, "gl_depth_add_segments: bad argument");
    if (n == 0) return GL_OK;
    GL_CHECK(p8_materialize(ctx));
    GL_CHECK(store_reserve(ctx, ctx->store_n + n));
    int32_t* d_s = static_cast<int32_t*>(ctx->store_s.p) + ctx->store_n;
    int32_t* d_e = static_cast<int32_t*>(ctx->store_e.p) + ctx->store_n;
    // a reduce of the previous region may still be queued and reading the store: the copies go after it
    GL_CUDA(ctx, cudaEventRecord(ctx->ev_hdr, ctx->stream));
    GL_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_hdr, 0));
    if (is_pinned_host(start) && is_pinned_host(end)) {
        GL_CUDA(ctx, cudaMemcpyAsync(d_s, start, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->copy_stream));
        GL_CUDA(ctx, cudaMemcpyAsync(d_e, end, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->copy_stream));
    } else {
        // pageable source: stage through two pinned slots so the CPU memcpy overlaps the DMA
        const size_t slot_bytes = (size_t)kStageSegs * 8;
        for (int i = 0; i < 2; i++) {
            if (!ctx->pinned[i]) {
                cudaError_t e = cudaHostAlloc(&ctx->pinned[i], slot_bytes, cudaHostAllocDefault);
                if (e != cudaSuccess) { ctx->pinned[i] = nullptr; cudaGetLastError(); return gl_fail(ctx, GL_ENOMEM, "cudaHostAlloc staging: %s", cudaGetErrorString(e)); }
            }
        }
        int64_t done = 0;
        int slot = 0;
        while (done < n) {
            const int64_t m = (n - done < kStageSegs) ? n - done : kStageSegs;
            GL_CUDA(ctx, cudaEventSynchronize(ctx->ev_used[slot]));       // previous DMA out of this slot has drained
            int32_t* h_s = static_cast<int32_t*>(ctx->pinned[slot]);
            int32_t* h_e = h_s + kStageSegs;
            memcpy(h_s, start + done, (size_t)m * 4);
            memcpy(h_e, end + done, (size_t)m * 4);
            GL_CUDA(ctx, cudaMemcpyAsync(d_s + done, h_s, (size_t)m * 4, cudaMemcpyHostToDevice, ctx->copy_stream));
            GL_CUDA(ctx, cudaMemcpyAsync(d_e + done, h_e, (size_t)m * 4, cudaMemcpyHostToDevice, ctx->copy_stream));
            GL_CUDA(ctx, cudaEventRecord(ctx->ev_used[slot], ctx->copy_stream));
            done += m;
            slot ^= 1;
        }
    }
    ctx->copies_pending = true;
    store_append(ctx, n);
    return GL_OK;
}

int gl_depth_add_segments_packed16(gl_ctx* ctx, const int32_t* anchors, const uint16_t* off, const uint16_t* len, int64_t n_blocks) {
    GL_CHECK(gl_use(ctx));
    if (!ctx->depth_active) return gl_fail(ctx, GL_ESTATE, "gl_depth_add_segments_packed16: no region open (call gl_depth_begin)");
    if (n_blocks < 0 || (n_blocks > 0 && (!anchors || !off || !len))) return gl_fail(ctx, GL_EINVAL, "gl_depth_add_segments_packed16: bad argument");
    if (n_blocks == 0) return GL_OK;
    GL_CHECK(p8_materialize(ctx));
    const int64_t n = n_blocks * 256;
    GL_CHECK(store_reserve(ctx, ctx->store_n + n));
    // staging for the packed bytes: anchors | off | len
    const size_t b_anchor = (size_t)n_blocks * 4, b_u16 = (size_t)n * 2;
    GL_CHECK(gl_buf_reserve(ctx, ctx->packed, al256(b_anchor) + 2 * al256(b_u16)));
    char* d_anchor = static_cast<char*>(ctx->packed.p);
    char* d_off = d_anchor + al256(b_anchor);
    char* d_len = d_off + al256(b_u16);
    const bool pinned = is_pinned_host(anchors) && is_pinned_host(off) && is_pinned_host(len);
    if (!pinned) {       // pageable: let the runtime stage it (the fast path is pinned feeder buffers)
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
    }
    // the previous unpack must be done with the staging buffer before it is overwritten
    GL_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_used[0], 0));
    GL_CHECK(upload_blocks(ctx, d_anchor, d_off, d_len, anchors, off, len, 0, n_blocks, 512, ctx->ev_copy[1]));
    {
        gl_prof_scope prof(ctx, "depth_unpack16_kernel");
        depth_unpack16_kernel<<<(unsigned)n_blocks, 256, 0, ctx->stream>>>(
            reinterpret_cast<const int*>(d_anchor), reinterpret_cast<const unsigned short*>(d_off),
            reinterpret_cast<const unsigned short*>(d_len), static_cast<int*>(ctx->store_s.p) + ctx->store_n,
            static_cast<int*>(ctx->store_e.p) + ctx->store_n);
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaEventRecord(ctx->ev_used[0], ctx->stream));
    if (!pinned) GL_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
    store_append(ctx, n);
    return GL_OK;
}

// registers a packed8 batch whose words are already on the device (stream-ordered after ctx->stream's wait)
static int p8_register(gl_ctx* ctx, const int* d_anchor, const void* d_ds, const void* d_len, int64_t n_blocks) {
    const int64_t n = n_blocks * 64;
    const int64_t base = (ctx->store_n + 3) & ~int64_t(3);        // the unpack kernel stores int4
    GL_CHECK(store_reserve(ctx, base + n));
    gl_seg_batch b;
    b.off = base; b.n = n;
    ctx->batches.push_back(b);
    ctx->store_n = base + n;
    ctx->p8.anchors = d_anchor; ctx->p8.ds = d_ds; ctx->p8.len = d_len; ctx->p8.n_blocks = n_blocks; ctx->p8.store_off = base;
    ctx->p8.pending = true;
    if (ctx->batches.size() > 1) GL_CHECK(p8_materialize(ctx));   // not the only batch: the int32 paths take it
    segments_changed(ctx);
    return GL_OK;
}

int gl_depth_add_segments_packed8_device(gl_ctx* ctx, const int32_t* d_anchors, const uint8_t* d_dstart, const uint8_t* d_len, int64_t n_blocks) {
    GL_CHECK(gl_use(ctx));
    if (!ctx->depth_active) return gl_fail(ctx, GL_ESTATE, "gl_depth_add_segments_packed8_device: no region open (call gl_depth_begin)");
    if (n_blocks < 0 || (n_blocks > 0 && (!d_anchors || !d_dstart || !d_len))) return gl_fail(ctx, GL_EINVAL, "gl_depth_add_segments_packed8_device: bad argument");
    if (((uintptr_t)d_dstart | (uintptr_t)d_len) & 7) return gl_fail(ctx, GL_EINVAL, "gl_depth_add_segments_packed8_device: dstart/len must be 8-byte aligned");
    if (n_blocks == 0) return GL_OK;
    GL_CHECK(p8_materialize(ctx));
    return p8_register(ctx, d_anchors, d_dstart, d_len, n_blocks);
}

static int add_packed8_host(gl_ctx* ctx, const int32_t* anchors, const uint8_t* dstart, const uint8_t* len, int64_t n_blocks, bool may_defer) {
    GL_CHECK(gl_use(ctx));
    if (!ctx->depth_active) return gl_fail(ctx, GL_ESTATE, "gl_depth_add_segments_packed8: no region open (call gl_depth_begin)");
    if (n_blocks < 0 || (n_blocks > 0 && (!anchors || !dstart || !len))) return gl_fail(ctx, GL_EINVAL, "gl_depth_add_segments_packed8: bad argument");
    if (n_blocks == 0) return GL_OK;
    GL_CHECK(p8_materialize(ctx));                                  // an earlier packed8 batch still lives in the staging buffer
    const size_t b_anchor = (size_t)n_blocks * 4, b_u8 = (size_t)n_blocks * 64;
    GL_CHECK(gl_buf_reserve(ctx, ctx->packed, al256(b_anchor) + 2 * al256(b_u8)));
    char* d_anchor = static_cast<char*>(ctx->packed.p);
    char* d_ds = d_anchor + al256(b_anchor);
    char* d_len = d_ds + al256(b_u8);
    const bool pinned = is_pinned_host(anchors) && is_pinned_host(dstart) && is_pinned_host(len);
    if (may_defer && pinned && ctx->batches.empty() && ctx->force_path == kPathNone && n_blocks >= 4096) {
        // one-call entry: the reduce follows at once, so let it stream the words in (chunk k+1 on the wire while chunk k's
        // tiles are reduced)
        GL_CHECK(p8_register(ctx, reinterpret_cast<const int*>(d_anchor), d_ds, d_len, n_blocks));
        ctx->p8.h_anchors = anchors; ctx->p8.h_ds = dstart; ctx->p8.h_len = len;
        ctx->p8.upload_pending = true;
        return GL_OK;
    }
    if (!pinned) GL_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
    GL_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_used[0], 0));   // previous consumer done with the staging buffer
    GL_CHECK(upload_blocks(ctx, d_anchor, d_ds, d_len, anchors, dstart, len, 0, n_blocks, 64, ctx->ev_copy[1]));
    if (!pinned) GL_CUDA(ctx, cudaStreamSynchronize(ctx->copy_stream));
    return p8_register(ctx, reinterpret_cast<const int*>(d_anchor), d_ds, d_len, n_blocks);
}

int gl_depth_add_segments_packed8(gl_ctx* ctx, const int32_t* anchors, const uint8_t* dstart, const uint8_t* len, int64_t n_blocks) {
    return add_packed8_host(ctx, anchors, dstart, len, n_blocks, false);
}

int gl_depth_reduce(gl_ctx* ctx, int32_t W, int32_t mincov, int32_t maxmean, int64_t run_break) {
    GL_CHECK(gl_use(ctx));
    if (!ctx->depth_active) return gl_fail(ctx, GL_ESTATE, "gl_depth_reduce: no region open");
    if (W <= 0 || run_break < 0) return gl_fail(ctx, GL_EINVAL, "gl_depth_reduce: W must be > 0 and run_break >= 0");
    ReduceArgs a;
    a.W = W;
    a.mincov = mincov;
    a.maxmean = maxmean;
    a.run_break = run_break;
    a.do_windows = a.do_runs = true;
    return run_reduce(ctx, a);
}

int gl_depth_result_sizes(gl_ctx* ctx, int64_t* n_windows, int64_t* n_runs, int32_t* max_depth) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(depth_resolve(ctx));
    if (!ctx->depth_reduced) return gl_fail(ctx, GL_ESTATE, "gl_depth_result_sizes: call gl_depth_reduce first");
    if (n_windows) *n_windows = ctx->n_windows;
    if (n_runs) *n_runs = ctx->n_runs;
    if (max_depth) *max_depth = ctx->max_depth;
    return GL_OK;
}

int gl_depth_transport_stats(gl_ctx* ctx, int32_t* transport, double* pack_s, int64_t* h2d_bytes, int64_t* n_escaped) {
    if (!ctx) return GL_EINVAL;
    if (transport) *transport = ctx->tr_kind;
    if (pack_s) *pack_s = ctx->tr_pack_s;
    if (h2d_bytes) *h2d_bytes = ctx->tr_bytes;
    if (n_escaped) *n_escaped = ctx->tr_esc;
    return GL_OK;
}

int gl_depth_transport_phases(gl_ctx* ctx, double phases_s[3]) {
    if (!ctx || !phases_s) return GL_EINVAL;
    for (int i = 0; i < 3; i++) phases_s[i] = ctx->tr_phase[i];
    return GL_OK;
}

int gl_depth_last_path(gl_ctx* ctx, int32_t* path) {
    if (!ctx || !path) return gl_fail(ctx, GL_EINVAL, "null argument");
    GL_CHECK(gl_use(ctx));
    GL_CHECK(depth_resolve(ctx));
    *path = ctx->last_path;
    return GL_OK;
}

int gl_depth_set_path(gl_ctx* ctx, int32_t path) {
    if (!ctx || (path != kPathNone && path != kPathFused && path != kPathHbmDiff && path != kPathEvents)) return gl_fail(ctx, GL_EINVAL, "gl_depth_set_path: path must be 0 (auto), 1 (no packed8 kernel), 2 (HBM difference array only) or 4 (bucketed events only)");
    ctx->force_path = path;
    return GL_OK;
}

int gl_depth_get_windows(gl_ctx* ctx, int64_t* sum_out, int64_t cap) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(depth_resolve(ctx));
    if (!ctx->depth_reduced || ctx->n_windows == 0) return gl_fail(ctx, GL_ESTATE, "gl_depth_get_windows: no window results");
    if (!sum_out) return gl_fail(ctx, GL_EINVAL, "gl_depth_get_windows: null sum_out");
    if (cap < ctx->n_windows) return gl_fail(ctx, GL_ERANGE, "gl_depth_get_windows: cap %lld < %lld windows", (long long)cap, (long long)ctx->n_windows);
    GL_CUDA(ctx, cudaMemcpyAsync(sum_out, ctx->win_sum_p, (size_t)ctx->n_windows * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_depth_get_runs(gl_ctx* ctx, int32_t* run_start, int32_t* run_end, uint8_t* run_class, int64_t cap) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(depth_resolve(ctx));
    if (!ctx->depth_reduced) return gl_fail(ctx, GL_ESTATE, "gl_depth_get_runs: call gl_depth_reduce first");
    const int64_t n = ctx->n_runs;
    if (cap < n) return gl_fail(ctx, GL_ERANGE, "gl_depth_get_runs: cap %lld < %lld runs", (long long)cap, (long long)n);
    if (n == 0) return GL_OK;
    if (run_start) GL_CUDA(ctx, cudaMemcpyAsync(run_start, ctx->run_start.p, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (run_class) GL_CUDA(ctx, cudaMemcpyAsync(run_class, ctx->run_class.p, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
    if (run_end) {
        GL_CHECK(gl_buf_reserve(ctx, ctx->misc, (size_t)n * 4));
        run_ends_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(static_cast<const int*>(ctx->run_start.p),
                                                                          static_cast<int*>(ctx->misc.p), n, (int)ctx->re);
        GL_LAUNCHED(ctx, 1);
        GL_CUDA(ctx, cudaMemcpyAsync(run_end, ctx->misc.p, (size_t)n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    }
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_depth_windows(gl_ctx* ctx, int32_t W, int64_t* sum_out, int32_t* min_out, int64_t n_windows) {
    GL_CHECK(gl_use(ctx));
    if (!ctx->depth_active) return gl_fail(ctx, GL_ESTATE, "gl_depth_windows: no region open");
    if (W <= 0) return gl_fail(ctx, GL_EINVAL, "gl_depth_windows: W must be > 0");
    ReduceArgs ra;
    ra.W = W;
    ra.do_windows = true;
    ra.want_min = min_out != nullptr;
    GL_CHECK(run_reduce(ctx, ra));
    GL_CHECK(depth_resolve(ctx));
    GL_CHECK(gl_depth_get_windows(ctx, sum_out, n_windows));
    if (min_out) {
        GL_CUDA(ctx, cudaMemcpyAsync(min_out, ctx->win_min.p, (size_t)ctx->n_windows * 4, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
    return GL_OK;
}

int gl_depth_classes(gl_ctx* ctx, int32_t mincov, int32_t maxmean, int32_t* run_start, int32_t* run_end,
                     uint8_t* run_class, int64_t cap, int64_t* n_runs) {
    GL_CHECK(gl_use(ctx));
    if (!ctx->depth_active) return gl_fail(ctx, GL_ESTATE, "gl_depth_classes: no region open");
    ReduceArgs ra;
    ra.mincov = mincov;
    ra.maxmean = maxmean;
    ra.do_runs = true;
    GL_CHECK(run_reduce(ctx, ra));
    GL_CHECK(depth_resolve(ctx));
    if (n_runs) *n_runs = ctx->n_runs;
    return gl_depth_get_runs(ctx, run_start, run_end, run_class, cap);
}

int gl_depth_interval_sums(gl_ctx* ctx, const int32_t* a, const int32_t* b, int64_t n, int64_t* sums) {
    GL_CHECK(gl_use(ctx));
    if (!ctx->depth_active) return gl_fail(ctx, GL_ESTATE, "gl_depth_interval_sums: no region open");
    if (n < 0 || (n > 0 && (!a || !b || !sums))) return gl_fail(ctx, GL_EINVAL, "gl_depth_interval_sums: bad argument");
    if (n == 0) return GL_OK;
    GL_CHECK(depth_resolve(ctx));                                  // the last reduce's path decides whether its cell index is used
    GL_CHECK(join_copies(ctx));
    if ((int)ctx->batches.size() > kMaxBatches) return gl_fail(ctx, GL_ERANGE, "gl_depth_interval_sums: more than %d segment batches", kMaxBatches);
    GL_CHECK(p8_materialize(ctx));
    ScanParams p;
    memset(&p, 0, sizeof p);
    p.rs = (int)ctx->rs;
    p.re = (int)ctx->re;
    const bool use_index = ctx->depth_reduced && ctx->last_path == kPathFused && ctx->idx_cells != nullptr;
    p.n_batches = (int)ctx->batches.size();
    p.flags = ctx->idx_flags;
    p.origin = ctx->idx_origin;
    p.ncells = ctx->idx_ncells;
    const size_t nb = ctx->batches.size();
    for (size_t bi = 0; bi < nb; bi++) {
        const gl_seg_batch& bt = ctx->batches[bi];
        p.batch[bi].start = batch_start(ctx, bt);
        p.batch[bi].end = batch_end(ctx, bt);
        p.batch[bi].n = (int)std::min<int64_t>(bt.n, INT32_MAX - 1);
        if (use_index) {                                           // same layout as reduce_int32: hi | cnt | lo
            const unsigned* hi_all = ctx->idx_cells;
            const unsigned* cnt_all = hi_all + (size_t)ctx->idx_ncells * nb;
            const unsigned* lo_all = cnt_all + (size_t)ctx->idx_ncells * nb;
            p.batch[bi].cell_hi = hi_all + bi * (size_t)ctx->idx_ncells;
            p.batch[bi].cell_cnt = cnt_all + bi * (size_t)ctx->idx_ncells;
            p.batch[bi].cell_lo = lo_all + bi * (size_t)ctx->idx_ncells;
        }
    }
    GL_CHECK(gl_buf_reserve(ctx, ctx->misc, (size_t)n * 16));
    long long* d_out = static_cast<long long*>(ctx->misc.p);
    int* d_a = reinterpret_cast<int*>(d_out + n);
    int* d_b = d_a + n;
    GL_CUDA(ctx, cudaMemcpyAsync(d_a, a, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaMemcpyAsync(d_b, b, (size_t)n * 4, cudaMemcpyHostToDevice, ctx->stream));
    {
        gl_prof_scope prof(ctx, "depth_interval_sum_kernel");
        depth_interval_sum_kernel<<<(unsigned)((n + 7) / 8), 256, 0, ctx->stream>>>(p, d_a, d_b, n, use_index ? 1 : 0, d_out);
    }
    GL_LAUNCHED(ctx, 1);
    GL_CUDA(ctx, cudaMemcpyAsync(sums, d_out, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return GL_OK;
}

int gl_depth_perbase(gl_ctx* ctx, int32_t* depth_out) {
    GL_CHECK(gl_use(ctx));
    if (!ctx->depth_active) return gl_fail(ctx, GL_ESTATE, "gl_depth_perbase: no region open");
    if (!depth_out) return gl_fail(ctx, GL_EINVAL, "gl_depth_perbase: null output");
    const int64_t len = ctx->re - ctx->rs;
    GL_CHECK(gl_buf_reserve(ctx, ctx->misc, (size_t)(len + 4) * 4));
    ReduceArgs ra;
    ra.d_depth_out = static_cast<int32_t*>(ctx->misc.p);
    GL_CHECK(run_reduce(ctx, ra));
    GL_CHECK(depth_resolve(ctx));
    GL_CUDA(ctx, cudaMemcpyAsync(depth_out, ctx->misc.p, (size_t)len * 4, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    ctx->depth_reduced = false;
    return GL_OK;
}

int gl_depth_region_packed16(gl_ctx* ctx, int64_t region_start, int64_t region_end, const int32_t* anchors, const uint16_t* off,
                             const uint16_t* len, int64_t n_blocks, int32_t W, int32_t mincov, int32_t maxmean, int64_t run_break,
                             int64_t* sum_out, int64_t win_cap, int64_t* n_windows, int32_t* run_start, uint8_t* run_class,
                             int64_t run_cap, int64_t* n_runs) {
    return region_one_call(ctx, region_start, region_end, [&] { return gl_depth_add_segments_packed16(ctx, anchors, off, len, n_blocks); },
                           W, mincov, maxmean, run_break, sum_out, win_cap, n_windows, run_start, run_class, run_cap, n_runs);
}

int gl_depth_region_packed8(gl_ctx* ctx, int64_t region_start, int64_t region_end, const int32_t* anchors, const uint8_t* dstart,
                            const uint8_t* len, int64_t n_blocks, int32_t W, int32_t mincov, int32_t maxmean, int64_t run_break,
                            int64_t* sum_out, int64_t win_cap, int64_t* n_windows, int32_t* run_start, uint8_t* run_class,
                            int64_t run_cap, int64_t* n_runs) {
    return region_one_call(ctx, region_start, region_end, [&] { return add_packed8_host(ctx, anchors, dstart, len, n_blocks, true); },
                           W, mincov, maxmean, run_break, sum_out, win_cap, n_windows, run_start, run_class, run_cap, n_runs);
}

int gl_depth_region(gl_ctx* ctx, int64_t region_start, int64_t region_end, const int32_t* start, const int32_t* end,
                    int64_t n, int32_t W, int32_t mincov, int32_t maxmean, int64_t run_break, int64_t* sum_out,
                    int64_t win_cap, int64_t* n_windows, int32_t* run_start, uint8_t* run_class, int64_t run_cap,
                    int64_t* n_runs) {
    return region_one_call(ctx, region_start, region_end, [&] { return gl_depth_add_segments(ctx, start, end, n); },
                           W, mincov, maxmean, run_break, sum_out, win_cap, n_windows, run_start, run_class, run_cap, n_runs);
}

// ---- one region of a contig (whole chunks), segments in, BED text out: depth/depth.go:238-364 for every chunk, in order
static int bed_args_ok(gl_ctx* ctx, int64_t rs, int64_t re, int32_t W, int64_t step) {
    if (W <= 0 || step <= 0 || step % W != 0) return gl_fail(ctx, GL_EINVAL, "gl_depth_bed_region: step must be a positive multiple of W (depth.go:132)");
    if (rs < 0 || re <= rs || rs % step != 0) return gl_fail(ctx, GL_EINVAL, "gl_depth_bed_region: the region must start on a chunk boundary (a multiple of step)");
    return GL_OK;
}

int gl_depth_bed_region_packed8(gl_ctx* ctx, const char* chrom, int64_t rs, int64_t re, const int32_t* anchors, const uint8_t* dstart,
                                const uint8_t* len, int64_t n_blocks, int32_t W, int32_t mincov, int32_t maxmean, int64_t step,
                                char* depth_bed, int64_t depth_cap, int64_t* depth_len, char* callable_bed, int64_t callable_cap,
                                int64_t* callable_len) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(bed_args_ok(ctx, rs, re, W, step));
    GL_CHECK(gl_depth_begin(ctx, rs, re));
    GL_CHECK(add_packed8_host(ctx, anchors, dstart, len, n_blocks, true));
    GL_CHECK(gl_depth_reduce(ctx, W, mincov, maxmean, step));
    return gl_depth_text(ctx, chrom, depth_bed, depth_cap, depth_len, callable_bed, callable_cap, callable_len);
}

int gl_depth_bed_region(gl_ctx* ctx, const char* chrom, int64_t rs, int64_t re, const int32_t* start, const int32_t* end, int64_t n,
                        int32_t W, int32_t mincov, int32_t maxmean, int64_t step, int32_t threads,
                        char* depth_bed, int64_t depth_cap, int64_t* depth_len, char* callable_bed, int64_t callable_cap,
                        int64_t* callable_len) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(bed_args_ok(ctx, rs, re, W, step));
    if (n < 0 || (n > 0 && (!start || !end))) return gl_fail(ctx, GL_EINVAL, "gl_depth_bed_region: bad segments");
    // How the int32 arrays travel (GL_BED_PACK; default: auto).  The call is PCIe-bound at 8 B/segment (chr20: 88 MB, 1.9 ms).
    // 16 / auto: the host pool rewrites them as fixed-block packed16 (gl_pack_segments16_fixed_range_mt: 4 B/segment, the
    // caller's order, one vectorised streaming pass, no sort, no count pass) in a few block chunks; chunk c+1 is packed while
    // chunk c is on the wire and unpacked into the segment store by depth_unpack16_kernel.  Auto takes it for >= 2^20
    // segments when the pool has >= 24 threads (with fewer the pack is slower than the bytes it saves: 8 ranks on one
    // host share its memory bandwidth).  0: plain int32.  1: packed8 (2 B/segment, needs a sort: 2-3 ms per chr20).
    // A feeder that emits packed8 itself (gl_bam_decode) calls gl_depth_bed_region_packed8.  tools/e2e_text_probe.py measures all.
    const char* force_env = getenv("GL_BED_PACK");                      // read per call (tests switch it)
    const int force = force_env ? atoi(force_env) : -1;
    if ((force == 16 && n >= 4096) || (force < 0 && n >= (int64_t(1) << 20) && glhost_pool_size() >= 48)) {
        // The pack is DRAM-bound: 16 threads reach most of what 64 do.  More is worse on a 2 x 32-core host: when a
        // burst of 24+ threads starts streaming out of an idle pool, every memory access of the process (and the GPU's DMA)
        // can stall for tens of ms every few calls (tools/e2e_transport_probe.py; none at 16 threads, none when the pool never idles).
        static const int pack_threads_env = [] { const char* e = getenv("GL_BED_PACK_THREADS"); return e ? atoi(e) : 0; }();
        const int pack_threads = threads > 0 ? threads : (pack_threads_env > 0 ? pack_threads_env : std::min(glhost_pool_size(), 16));
        const auto ph0 = std::chrono::steady_clock::now();
        const int64_t nbk = (n + 255) / 256;
        const size_t o_off = ((size_t)nbk * 4 + 255) & ~size_t(255), o_len = o_off + (size_t)nbk * 512, bytes = o_len + (size_t)nbk * 512;
        GL_CHECK(gl_pinned_reserve(ctx, bytes, bytes + bytes / 8));
        char* hp = static_cast<char*>(ctx->pack_pinned);
        int32_t* A = reinterpret_cast<int32_t*>(hp);
        uint16_t* O = reinterpret_cast<uint16_t*>(hp + o_off);
        uint16_t* Ln = reinterpret_cast<uint16_t*>(hp + o_len);
        GL_CHECK(gl_depth_begin(ctx, rs, re));
        GL_CHECK(store_reserve(ctx, nbk * 256 + n / 32 + 65536 + 64));    // blocks + room for the escapes: no regrowth between chunks
        GL_CHECK(gl_buf_reserve(ctx, ctx->packed, bytes));                // device staging, the host buffer's layout
        char* dp = static_cast<char*>(ctx->packed.p);
        // escape list: ctx-owned and grow-only (a fresh zero-filled vector per call cost more page faults than the pack itself)
        const size_t esc_want = (size_t)(n / 32 + 65536);
        if (ctx->esc_cap < esc_want) {
            free(ctx->esc_buf);
            ctx->esc_buf = static_cast<int32_t*>(malloc(2 * esc_want * sizeof(int32_t)));
            ctx->esc_cap = ctx->esc_buf ? esc_want : 0;
            if (!ctx->esc_buf) return gl_fail(ctx, GL_ENOMEM, "malloc(%zu)", 2 * esc_want * sizeof(int32_t));
        }
        int32_t* es = ctx->esc_buf;
        int32_t* ee = ctx->esc_buf + ctx->esc_cap;
        const int64_t esc_cap = (int64_t)ctx->esc_cap;
        int64_t n_esc = 0;
        static const int k_max = [] { const char* e = getenv("GL_BED_PACK_CHUNKS"); const int v = e ? atoi(e) : 8; return v < 1 ? 1 : (v > 64 ? 64 : v); }();
        const int K = (int)std::max<int64_t>(1, std::min<int64_t>(k_max, nbk / 4096));   // >= 1 M segments per chunk
        // (an earlier call's uploads out of the pinned buffer have finished: every entry point synchronises before it returns;
        //  the previous call's unpack kernels out of ctx->packed are ordered before ours on ctx->stream via ev_used[0])
        GL_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_used[0], 0));
        int64_t done_blocks = 0;
        bool fell_back = false;
        const auto ph1 = std::chrono::steady_clock::now();
        ctx->tr_kind = 16; ctx->tr_pack_s = 0; ctx->tr_bytes = 0; ctx->tr_esc = 0;
        for (int c = 0; c < K; c++) {
            const int64_t b0 = nbk * c / K, b1 = nbk * (c + 1) / K;
            if (b1 <= b0) continue;
            const int64_t esc_before = n_esc;
            const auto tp0 = std::chrono::steady_clock::now();
            const int rc = gl_pack_segments16_fixed_range_mt(start, end, n, b0, b1, pack_threads, A, O, Ln, es, ee, esc_cap, &n_esc);
            ctx->tr_pack_s += std::chrono::duration<double>(std::chrono::steady_clock::now() - tp0).count();
            if (rc == GL_ERANGE) { n_esc = esc_before; fell_back = true; break; }   // (almost) every block escapes: long reads / unsorted input
            if (rc != GL_OK) return gl_fail(ctx, rc, "gl_pack_segments16_fixed_range_mt failed");
            GL_CHECK(upload_blocks(ctx, dp, dp + o_off, dp + o_len, A, O, Ln, b0, b1, 512, ctx->ev_copy[1]));
            {
                gl_prof_scope prof(ctx, "depth_unpack16_kernel");
                depth_unpack16_kernel<<<(unsigned)(b1 - b0), 256, 0, ctx->stream>>>(
                    reinterpret_cast<const int*>(dp) + b0, reinterpret_cast<const unsigned short*>(dp + o_off) + b0 * 256,
                    reinterpret_cast<const unsigned short*>(dp + o_len) + b0 * 256, static_cast<int*>(ctx->store_s.p) + b0 * 256,
                    static_cast<int*>(ctx->store_e.p) + b0 * 256);
            }
            GL_LAUNCHED(ctx, 1);
            done_blocks = b1;
            ctx->tr_bytes += (b1 - b0) * (4 + 1024);
        }
        GL_CUDA(ctx, cudaEventRecord(ctx->ev_used[0], ctx->stream));
        ctx->copies_pending = true;
        if (done_blocks > 0) store_append(ctx, done_blocks * 256);         // the region's first batch: store [0, done_blocks * 256)
        const auto ph2 = std::chrono::steady_clock::now();
        ctx->tr_esc = n_esc;
        ctx->tr_bytes += 8 * n_esc + (fell_back ? 8 * (n - done_blocks * 256) : 0);
        if (fell_back)                                                    // the blocks not packed yet go up as plain int32 (another batch)
            GL_CHECK(gl_depth_add_segments(ctx, start + done_blocks * 256, end + done_blocks * 256, n - done_blocks * 256));
        if (n_esc > 0) {
            // the segments of the blocks written as empty: a batch of their OWN (each batch has its own cell index; appended to the
            // packed batch they would sit out of order at its end and the fused path would reject the tiles around every gap)
            ctx->store_n += 4;                                            // a gap in the store keeps gl_depth_add_segments from extending the previous batch
            GL_CHECK(gl_depth_add_segments(ctx, es, ee, n_esc));
        }
        GL_CHECK(gl_depth_reduce(ctx, W, mincov, maxmean, step));
        const int rc_text = gl_depth_text(ctx, chrom, depth_bed, depth_cap, depth_len, callable_bed, callable_cap, callable_len);
        const auto ph3 = std::chrono::steady_clock::now();
        ctx->tr_phase[0] = std::chrono::duration<double>(ph1 - ph0).count();
        ctx->tr_phase[1] = std::chrono::duration<double>(ph2 - ph1).count();
        ctx->tr_phase[2] = std::chrono::duration<double>(ph3 - ph2).count();
        return rc_text;
    }
    bool pack = force == 1 && n >= 4096;
    if (pack) {                                       // long segments would be cut into many 255-base pieces: judged on a sample
        int64_t tot = 0, cnt = 0;
        for (int part = 0; part < 4; part++)
            for (int64_t i = (n - 1024) * part / 3, j = 0; j < 1024; j++, i++) { tot += std::max<int64_t>(0, (int64_t)end[i] - start[i]); cnt++; }
        pack = tot <= 400 * cnt;
    }
    if (!pack) {
        ctx->tr_kind = 0; ctx->tr_pack_s = 0; ctx->tr_bytes = 8 * n; ctx->tr_esc = 0;
        GL_CHECK(gl_depth_begin(ctx, rs, re));
        GL_CHECK(gl_depth_add_segments(ctx, start, end, n));
        GL_CHECK(gl_depth_reduce(ctx, W, mincov, maxmean, step));
        return gl_depth_text(ctx, chrom, depth_bed, depth_cap, depth_len, callable_bed, callable_cap, callable_len);
    }
    int64_t cap = n / 40 + 1024, nb = 0;
    for (int attempt = 0; attempt < 2; attempt++) {
        const size_t bytes = (size_t)cap * 132 + 256;
        GL_CHECK(gl_pinned_reserve(ctx, bytes, bytes));
        const int64_t cap_now = (int64_t)((ctx->pack_pinned_bytes - 256) / 132);
        int32_t* a = static_cast<int32_t*>(ctx->pack_pinned);
        uint8_t* d = reinterpret_cast<uint8_t*>(a + ((cap_now + 3) & ~int64_t(3)));
        uint8_t* l = d + (size_t)cap_now * 64;
        // (an earlier call's upload out of this buffer has finished: every entry point synchronises before it returns)
        const int rc = gl_pack_segments8_mt(start, end, n, threads, a, d, l, cap_now, &nb);
        if (rc == GL_ERANGE) { cap = nb + 16; continue; }
        if (rc != GL_OK) return gl_fail(ctx, rc, "gl_pack_segments8_mt failed");
        return gl_depth_bed_region_packed8(ctx, chrom, rs, re, a, d, l, nb, W, mincov, maxmean, step, depth_bed, depth_cap, depth_len,
                                           callable_bed, callable_cap, callable_len);
    }
    return gl_fail(ctx, GL_ERANGE, "gl_depth_bed_region: packing did not converge");
}

int gl_depth_bed_contig_packed8(gl_ctx* ctx, const char* chrom, int64_t contig_len, const int32_t* anchors, const uint8_t* dstart,
                                const uint8_t* len, int64_t n_blocks, int32_t W, int32_t mincov, int32_t maxmean, int64_t step,
                                char* depth_bed, int64_t depth_cap, int64_t* depth_len, char* callable_bed, int64_t callable_cap,
                                int64_t* callable_len) {
    return gl_depth_bed_region_packed8(ctx, chrom, 0, contig_len, anchors, dstart, len, n_blocks, W, mincov, maxmean, step, depth_bed, depth_cap,
                                       depth_len, callable_bed, callable_cap, callable_len);
}

int gl_depth_bed_contig(gl_ctx* ctx, const char* chrom, int64_t contig_len, const int32_t* start, const int32_t* end, int64_t n,
                        int32_t W, int32_t mincov, int32_t maxmean, int64_t step, int32_t threads,
                        char* depth_bed, int64_t depth_cap, int64_t* depth_len, char* callable_bed, int64_t callable_cap,
                        int64_t* callable_len) {
    return gl_depth_bed_region(ctx, chrom, 0, contig_len, start, end, n, W, mincov, maxmean, step, threads, depth_bed, depth_cap, depth_len,
                               callable_bed, callable_cap, callable_len);
}

}  // extern "C"
