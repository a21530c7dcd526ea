/*
 * goleft_b200.h — C ABI of libgoleft_b200.so, the H100 (sm_90a) engine behind
 * goleft's windowed-depth hot path (`depth`, `indexcov`, `covstats`, `depthwed`).
 *
 * The reference (brentp/goleft, pure Go) has no FFI for this path; each entry point
 * below cites the reference code whose work it replaces (paths relative to the
 * reference checkout).  INTEGRATION.md shows the cgo binding a maintainer would add.
 *
 * Conventions
 *  - extern "C", plain pointers and sizes only.  No torch / C++ types.
 *  - every call returns int: 0 = ok, <0 = error (GL_E*); text via gl_last_error().
 *  - the caller owns every host buffer; the library owns device memory inside an
 *    opaque gl_ctx (one ctx per GPU, one host thread at a time per ctx).
 *  - coordinates are 0-based half-open, like the reference's internal ints.
 *  - pointers named d_* are DEVICE pointers (from gl_dev_alloc); all others are
 *    host pointers (pageable is fine, the library stages through pinned memory).
 *  - calls are synchronous on the ctx's stream unless stated otherwise.
 *  - there is NO CPU fallback: without a CUDA device every call fails with GL_ECUDA.
 */
#ifndef GOLEFT_B200_H
#define GOLEFT_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GL_OK        0
#define GL_EINVAL   -1   /* bad argument */
#define GL_ECUDA    -2   /* CUDA runtime error (message has the cudaError string) */
#define GL_ENOMEM   -3   /* device or pinned-host allocation failed */
#define GL_ESTATE   -4   /* call out of order (e.g. add_segments before begin) */
#define GL_ERANGE   -5   /* output capacity too small / value out of supported range */
#define GL_ENCCL    -6   /* NCCL error */

/* coverage classes of depth/depth.go:223-234 (getCovClass) */
#define GL_NO_COVERAGE        0
#define GL_LOW_COVERAGE       1
#define GL_CALLABLE           2
#define GL_EXCESSIVE_COVERAGE 3

/* indexcov constants: indexcov/indexcov.go:153 (slots), indexcov/types.go:15 (TileWidth) */
#define GL_INDEXCOV_SLOTS 70
#define GL_TILE_WIDTH     16384

typedef struct gl_ctx gl_ctx;
typedef struct gl_bam gl_bam;            /* an open BAM + its index (gl_bam_open) */

/* ---------------------------------------------------------------- context */
const char* gl_version(void);                       /* "goleft_b200 <semver> sm_90a" */
int  gl_device_count(int* n);
int  gl_ctx_create(int device, gl_ctx** out);
int  gl_ctx_destroy(gl_ctx* ctx);
const char* gl_last_error(gl_ctx* ctx);             /* ctx may be NULL: last global error */
int  gl_sync(gl_ctx* ctx);
/* number of kernels this ctx has launched so far (bench.py's gpu_launches claim) */
int  gl_launch_count(gl_ctx* ctx, int64_t* n);
/* raw cudaStream_t of the ctx, as an integer, so a caller can record events on it */
int  gl_stream_handle(gl_ctx* ctx, uint64_t* stream);

/* Pins the calling thread, and the threads created after it (the library's host pool, feeders), to the CPUs of the NUMA
 * node of `device`; with share_count > 1 to the share_index-th slice of that node's cores (ranks sharing a socket).
 * Call it before the first pinned allocation / pool use.  *node = -1 when the topology is unreadable (nothing changed). */
int  gl_device_numa_node(int device, int* node);     /* -1: unknown */
int  gl_bind_numa_for_device(int device, int share_index, int share_count, int* node, int* n_cpus);
/* Longest-processing-time-first placement of n work items (contigs, weight = length) on `bins` GPUs: the unit of
 * independence of depth/depth.go:129-159.  bin_of[i] = GPU of item i, bin_load[b] = total weight (may be NULL). */
int  gl_lpt_assign(const int64_t* weight, int32_t n, int32_t bins, int32_t* bin_of, int64_t* bin_load);

/* device memory owned by the ctx's device (plumbing for callers that keep inputs resident) */
int  gl_dev_alloc(gl_ctx* ctx, int64_t bytes, void** d_ptr);
int  gl_dev_free(gl_ctx* ctx, void* d_ptr);
int  gl_host_alloc_pinned(gl_ctx* ctx, int64_t bytes, void** h_ptr);
int  gl_host_free_pinned(gl_ctx* ctx, void* h_ptr);
int  gl_memcpy_h2d(gl_ctx* ctx, void* d_dst, const void* h_src, int64_t bytes);
int  gl_memcpy_d2h(gl_ctx* ctx, void* h_dst, const void* d_src, int64_t bytes);
/* device-timed interval helpers (CUDA events on the ctx stream) */
int  gl_timer_start(gl_ctx* ctx);
int  gl_timer_stop_ms(gl_ctx* ctx, float* ms);      /* records, synchronizes, returns elapsed */
/* per-kernel CUDA-event timing on the ctx stream: enable, run, then read "name ms\n" lines
 * (one per kernel launched since the last read; synchronizes).  Off by default. */
int  gl_profile_enable(gl_ctx* ctx, int on);
int  gl_profile_read(gl_ctx* ctx, char* buf, int64_t cap, int64_t* needed);
/* write `bytes` of junk to a scratch buffer (> L2) so the next launch starts cold */
int  gl_flush_l2(gl_ctx* ctx);

/* ------------------------------------------------------------------ depth
 * Replaces, per region [region_start, region_end) of one contig:
 *   - the `samtools depth -Q q -d D -r chr:b-e` child of depth/depth.go:45,116,152
 *     (per-base counting of the M/=/X blocks of records that pass the flag/MAPQ filter;
 *      the filter itself is applied by the segment feeder, see gl_bam_* below),
 *   - the per-line window accumulation of depth/depth.go:282-306,329-341 (Σ depth per
 *     genome-aligned window, clipped to the region),
 *   - the per-line class run-length encoding of depth/depth.go:307-327,343-350.
 * Text formatting (%.4g of sum/len, BED rows, the Q2/Q3 chunk-edge quirks) stays on the
 * host: gl_depth_format_chunk().
 */

/* Start a region [region_start, region_end) of one contig.  0 <= start < end, end-start < 2^30. */
int  gl_depth_begin(gl_ctx* ctx, int64_t region_start, int64_t region_end);

/* Add n segments [start[i], end[i]) (absolute contig coordinates, end>start; clipped to the region
 * by the kernels; segments outside are ignored).  May be called repeatedly between begin and reduce.
 * Host-pointer variant copies into a ctx-owned device store on a copy stream (pinned sources DMA
 * directly after the call returns: leave a pinned source unchanged until the region's results have
 * been read; pageable ones are staged); _device variant references HBM-resident arrays, which must
 * stay valid until the region's results have been read or the next gl_depth_begin (a reduce whose fast
 * path the device rejects is rerun from them at the first result query).
 * Any order is accepted.  Coordinate-sorted segments (non-decreasing start, what a BAM yields) of at
 * most 16384 bases take the fused path: each 4096-base tile's difference array is built in shared
 * memory straight from the segments.  Anything else takes the general path (bucketed events, see
 * gl_depth_last_path).  The device checks eligibility itself; results are identical. */
int  gl_depth_add_segments(gl_ctx* ctx, const int32_t* start, const int32_t* end, int64_t n);
int  gl_depth_add_segments_device(gl_ctx* ctx, const int32_t* d_start, const int32_t* d_end, int64_t n);

/* The feeder's compact format ("packed16", half the PCIe bytes): blocks of 256 slots, one int32 anchor per
 * block, slot k = [anchor+off[k], anchor+off[k]+len[k]) with uint16 off/len (len 0 = empty slot).
 * gl_pack_segments16 builds it on the host from plain arrays (splitting segments longer than 65535, opening
 * a new block when a start does not fit 16 bits); returns GL_ERANGE with the needed *n_blocks when
 * cap_blocks is too small (pass NULL outputs to only count).  The GPU unpacks into its segment store. */
int64_t gl_pack_segments16_bound(int64_t n);
int  gl_pack_segments16(const int32_t* start, const int32_t* end, int64_t n, int32_t* anchors, uint16_t* off,
                        uint16_t* len, int64_t cap_blocks, int64_t* n_blocks);
/* the same from `threads` host threads (0 = the whole pool): order-preserving, no sort; index chunks are packed independently */
int  gl_pack_segments16_mt(const int32_t* start, const int32_t* end, int64_t n, int32_t threads, int32_t* anchors, uint16_t* off,
                           uint16_t* len, int64_t cap_blocks, int64_t* n_blocks);
int  gl_depth_add_segments_packed16(gl_ctx* ctx, const int32_t* anchors, const uint16_t* off, const uint16_t* len,
                                    int64_t n_blocks);
/* The same device format with FIXED block boundaries: block b = input segments [256 b, 256 b + 256) in the caller's order,
 * anchor = their lowest start; n_blocks = ceil(n / 256) (caller-sized outputs: anchors[n_blocks], off/len[256 n_blocks]).
 * One streaming pass on the host pool, no sort, no count pass.  A block that cannot be expressed (starts more than 65535
 * bases apart, or a segment longer than 65535) is written as 256 empty slots and its segments are appended raw to
 * esc_start/esc_end (*n_esc in/out for the _range form); GL_ERANGE when they exceed esc_cap (*n_esc = needed).  Adding the
 * blocks (gl_depth_add_segments_packed16) and the escapes (gl_depth_add_segments) gives exactly the input's segments.
 * This is how gl_depth_bed_region moves decoder-native int32 arrays at 4 B/segment (DESIGN.md 1.7). */
int  gl_pack_segments16_fixed_mt(const int32_t* start, const int32_t* end, int64_t n, int32_t threads, int32_t* anchors, uint16_t* off,
                                 uint16_t* len, int32_t* esc_start, int32_t* esc_end, int64_t esc_cap, int64_t* n_esc);
int  gl_pack_segments16_fixed_range_mt(const int32_t* start, const int32_t* end, int64_t n, int64_t block_begin, int64_t block_end,
                                       int32_t threads, int32_t* anchors, uint16_t* off, uint16_t* len, int32_t* esc_start,
                                       int32_t* esc_end, int64_t esc_cap, int64_t* n_esc);
/* "packed8": a quarter of the bytes, for short-read data.  Blocks of 64 slots: int32 anchor (start of slot 0) +
 * per slot uint8 dstart (start - previous slot's start) and uint8 len (0 = empty/filler).  gl_pack_segments8 puts the
 * segments in start order (depth is order-independent), cuts segments longer than 255 into pieces and bridges gaps
 * > 255 bases with filler slots or a new block, whichever is smaller; same return convention as gl_pack_segments16.
 * Use it when 132 * n_blocks < 8 * n (always for 100-250 bp reads at >= 1x). */
int64_t gl_pack_segments8_bound(int64_t n);
int  gl_pack_segments8(const int32_t* start, const int32_t* end, int64_t n, int32_t* anchors, uint8_t* dstart, uint8_t* len,
                       int64_t cap_blocks, int64_t* n_blocks);
/* The same format from `threads` host threads (0 = all of the library's pool; GL_THREADS sets its size): the input is cut
 * into position ranges that are packed independently and concatenated, so the blocks differ from gl_pack_segments8's at the
 * range edges (a block may end early) but decode to the same multiset of pieces.  Host-only. */
int  gl_pack_segments8_mt(const int32_t* start, const int32_t* end, int64_t n, int32_t threads, int32_t* anchors, uint8_t* dstart,
                          uint8_t* len, int64_t cap_blocks, int64_t* n_blocks);
int  gl_depth_add_segments_packed8(gl_ctx* ctx, const int32_t* anchors, const uint8_t* dstart, const uint8_t* len, int64_t n_blocks);
/* same with the three arrays already in device memory (caller-owned, 8-byte aligned, must stay valid until the region's
 * results have been read or the next gl_depth_begin): nothing is copied; a region whose only batch is packed8 is reduced
 * straight from these words. */
int  gl_depth_add_segments_packed8_device(gl_ctx* ctx, const int32_t* d_anchors, const uint8_t* d_dstart, const uint8_t* d_len,
                                          int64_t n_blocks);

/* One fused pass: prefix scan -> per-base depth (never written to HBM) ->
 *   (a) per-window int64 sums for genome-aligned windows of size W clipped to the region:
 *       window k covers [max(rs,(rs/W+k)*W), min(re,(rs/W+k+1)*W)),
 *   (b) class run starts: position x starts a run when x==rs, class(x)!=class(x-1), or
 *       run_break>0 and x%run_break==0 (the reference never merges runs across its 10 Mb
 *       chunks, depth/depth.go:132,150: pass run_break=step to reproduce that).
 * mincov/maxmean as depth/depth.go:223-234.  Asynchronous: the arguments are checked at once, the work is queued on the
 * ctx stream and the call returns without waiting for it, so regions reduced back to back keep the device busy.  Errors
 * in the device work and fallbacks (input the fast path rejects, a run table that has to grow) are settled at the first
 * result query (gl_depth_result_sizes, gl_depth_last_path, gl_depth_get_*, gl_depth_text, gl_depth_interval_sums); a
 * result nobody queried is dropped by the next gl_depth_begin or add.  Results stay on the device until fetched. */
int  gl_depth_reduce(gl_ctx* ctx, int32_t W, int32_t mincov, int32_t maxmean, int64_t run_break);

/* Sizes of the results of the last gl_depth_reduce (waits for it). */
int  gl_depth_result_sizes(gl_ctx* ctx, int64_t* n_windows, int64_t* n_runs, int32_t* max_depth);
/* Which path the last reduce took: 1 = fused (nearly sorted int32 segments), 2 = HBM difference array (the north-star
 * pipeline: red.global scatter + scan; on request only), 3 = packed8 (the region's only batch is packed8: read as it is, no
 * int32 copy, no per-segment index), 4 = bucketed events (the general path: any order, any length; two 16-bit events per
 * segment bucketed by 4096-base tile, difference arrays built in shared memory). */
int  gl_depth_last_path(gl_ctx* ctx, int32_t* path);
/* How the last gl_depth_bed_region / gl_depth_bed_contig call moved its int32 arrays: transport 0 = as they are (8 B/segment),
 * 16 = fixed-block packed16 made by the host pool chunk by chunk (4 B/segment); host seconds spent packing (the calling
 * thread's wall time inside the pool runs), bytes sent host->device, segments that went up raw as escapes. */
int  gl_depth_transport_stats(gl_ctx* ctx, int32_t* transport, double* pack_s, int64_t* h2d_bytes, int64_t* n_escaped);
/* host wall-clock phases of the same call: [0] setup (buffers, gl_depth_begin), [1] the pack + enqueue loop, [2] reduce + text + D2H */
int  gl_depth_transport_phases(gl_ctx* ctx, double phases_s[3]);
/* 0 = choose automatically (default: packed8 -> fused -> bucketed events), 1 = never the packed8 kernel, 2 = always the HBM
 * difference array, 4 = always bucketed events (tests, comparison runs). */
int  gl_depth_set_path(gl_ctx* ctx, int32_t path);

/* Fetch results (host buffers).  run_end may be NULL (run i ends where run i+1 starts; the last
 * ends at region_end). */
int  gl_depth_get_windows(gl_ctx* ctx, int64_t* sum_out, int64_t cap);
int  gl_depth_get_runs(gl_ctx* ctx, int32_t* run_start, int32_t* run_end, uint8_t* run_class, int64_t cap);

/* Forms named in SURVEY.md §8(b): run the pass for one output only.  gl_depth_windows also gives the
 * per-window minimum depth when min_out != NULL (an extra: the reference prints means only). */
int  gl_depth_windows(gl_ctx* ctx, int32_t W, int64_t* sum_out, int32_t* min_out, int64_t n_windows);
int  gl_depth_classes(gl_ctx* ctx, int32_t mincov, int32_t maxmean, int32_t* run_start, int32_t* run_end,
                      uint8_t* run_class, int64_t cap, int64_t* n_runs);
/* Sum of per-base depth over n arbitrary intervals [a[i], b[i]) of the open region (clipped to it), computed straight
 * from the segments (sum of overlaps); uses the cell index of the last gl_depth_reduce when that took the fused path.
 * This is what BED mode needs for the clipped first/last window of every region (depth/depth.go:293-305,329-341). */
int  gl_depth_interval_sums(gl_ctx* ctx, const int32_t* a, const int32_t* b, int64_t n, int64_t* sums);
/* Per-base depth of the region (debug / parity): depth_out has region_end-region_start entries. */
int  gl_depth_perbase(gl_ctx* ctx, int32_t* depth_out);

/* One-call form used by the CLI and the end-to-end benchmark: host segments in, host
 * results out, for one region; uploads are chunked and overlapped with the scatter. */
int  gl_depth_region(gl_ctx* ctx, int64_t region_start, int64_t region_end,
                     const int32_t* start, const int32_t* end, int64_t n,
                     int32_t W, int32_t mincov, int32_t maxmean, int64_t run_break,
                     int64_t* sum_out, int64_t win_cap, int64_t* n_windows,
                     int32_t* run_start, uint8_t* run_class, int64_t run_cap, int64_t* n_runs);

int  gl_depth_region_packed16(gl_ctx* ctx, int64_t region_start, int64_t region_end, const int32_t* anchors,
                              const uint16_t* off, const uint16_t* len, int64_t n_blocks,
                              int32_t W, int32_t mincov, int32_t maxmean, int64_t run_break,
                              int64_t* sum_out, int64_t win_cap, int64_t* n_windows,
                              int32_t* run_start, uint8_t* run_class, int64_t run_cap, int64_t* n_runs);
int  gl_depth_region_packed8(gl_ctx* ctx, int64_t region_start, int64_t region_end, const int32_t* anchors,
                             const uint8_t* dstart, const uint8_t* len, int64_t n_blocks, int32_t W, int32_t mincov, int32_t maxmean,
                             int64_t run_break, int64_t* sum_out, int64_t win_cap, int64_t* n_windows, int32_t* run_start,
                             uint8_t* run_class, int64_t run_cap, int64_t* n_runs);

/* BED text of the last gl_depth_reduce, formatted ON THE DEVICE (depth_text.cu): only finished bytes cross PCIe.
 *   depth_bed    : "chrom\tstart\tend\t%.4g\n" per window (depth/depth.go:301,337,357; mean = float64(sum)/float64(e-s),
 *                  depth.go:181-189; the four digits are rounded half-even on the exact binary value, like strconv),
 *   callable_bed : "chrom\tstart\tend\tCLASS\n" per class run (depth.go:312-349).
 * Needs region_start % W == 0 and run_break % W == 0: then the reference's per-chunk rows (incl. its tail rows,
 * depth.go:329-358) are exactly the genome-aligned windows of the region, each once.  BED-mode regions with unaligned
 * starts go through gl_depth_chunk_rows + gl_depth_format_rows (explicit rows) or gl_depth_format_chunk (host).
 * GL_ERANGE with both lengths set when a buffer is too small; gl_depth_text_bound() is always enough for depth_bed. */
int  gl_depth_text(gl_ctx* ctx, const char* chrom, char* depth_bed, int64_t depth_cap, int64_t* depth_len,
                   char* callable_bed, int64_t callable_cap, int64_t* callable_len);
int64_t gl_depth_text_bound(const char* chrom, int64_t n_windows);
/* n explicit window rows (s, e, sum) -> the same row text (the misaligned / re-emitted rows of depth.go:329-358) */
int  gl_depth_format_rows(gl_ctx* ctx, const char* chrom, const int32_t* row_s, const int32_t* row_e, const int64_t* row_sum,
                          int64_t n, char* out, int64_t cap, int64_t* len);
/* One contig end to end, the call `goleft depth` makes per reference sequence in .fai mode (depth.go:129-159 + the
 * callback 238-364 for each of its chunks, concatenated in order): host segments in -> BED bytes out.  step = the chunk
 * length (depth.go:132: a multiple of W).  The int32 arrays go over PCIe as fixed-block packed16 (4 B/segment), rewritten
 * chunk by chunk by the library's host pool (`threads` of it, 0 = the default 16) while the previous chunk is on the wire,
 * when there are >= 2^20 segments and the pool has >= 48 threads; otherwise, and for long reads, as they are (GL_BED_PACK,
 * gl_depth_transport_stats; DESIGN.md 1.7).  Everything is inside the call; it is synchronous. */
/* The same for [region_start, region_end) of a contig: region_start must be a multiple of step (whole chunks), so that
 * contigs longer than 2^30-1 bases, or one GPU's share of a contig, can be done in pieces whose texts concatenate. */
int  gl_depth_bed_region(gl_ctx* ctx, const char* chrom, int64_t region_start, int64_t region_end, const int32_t* start, const int32_t* end,
                         int64_t n, int32_t W, int32_t mincov, int32_t maxmean, int64_t step, int32_t threads,
                         char* depth_bed, int64_t depth_cap, int64_t* depth_len, char* callable_bed, int64_t callable_cap,
                         int64_t* callable_len);
int  gl_depth_bed_region_packed8(gl_ctx* ctx, const char* chrom, int64_t region_start, int64_t region_end, const int32_t* anchors,
                                 const uint8_t* dstart, const uint8_t* len, int64_t n_blocks, int32_t W, int32_t mincov, int32_t maxmean,
                                 int64_t step, char* depth_bed, int64_t depth_cap, int64_t* depth_len, char* callable_bed,
                                 int64_t callable_cap, int64_t* callable_len);
int  gl_depth_bed_contig(gl_ctx* ctx, const char* chrom, int64_t contig_len, const int32_t* start, const int32_t* end, int64_t n,
                         int32_t W, int32_t mincov, int32_t maxmean, int64_t step, int32_t threads,
                         char* depth_bed, int64_t depth_cap, int64_t* depth_len, char* callable_bed, int64_t callable_cap,
                         int64_t* callable_len);
int  gl_depth_bed_contig_packed8(gl_ctx* ctx, const char* chrom, int64_t contig_len, const int32_t* anchors, const uint8_t* dstart,
                                 const uint8_t* len, int64_t n_blocks, int32_t W, int32_t mincov, int32_t maxmean, int64_t step,
                                 char* depth_bed, int64_t depth_cap, int64_t* depth_len, char* callable_bed, int64_t callable_cap,
                                 int64_t* callable_len);

/* Host-side text: reproduces the rows the reference callback writes for ONE chunk
 * [rs,re) (depth/depth.go:293-305,326-358 incl. the chunk-edge quirks) from window sums
 * and runs restricted to that chunk.  Appends to malloc'd buffers; free with gl_free_text. */
int  gl_depth_format_chunk(const char* chrom, int64_t rs, int64_t re, int32_t W,
                           const int64_t* win_sum /* windows of [rs,re) */, int64_t n_windows,
                           const int32_t* run_start, const uint8_t* run_class, int64_t n_runs,
                           char** depth_bed, int64_t* depth_len, char** callable_bed, int64_t* callable_len);
void gl_free_text(char* p);

/* ---- `goleft depth --stats` (depth/depth.go:191-200 getStats, :246-252): GC / CpG / masked fraction per window row.
 * The arithmetic is github.com/brentp/faidx Faidx.Stats (go.mod:11, not vendored; parity unpinned), which scans the raw
 * bytes of the FASTA record, newlines included.
 * gl_depth_chunk_rows lists the (s,e) of the window rows gl_depth_format_chunk writes for a chunk, in order (including
 *   the misaligned / re-emitted rows of depth.go:329-358); returns GL_ERANGE with *n_rows set when cap is too small.
 * gl_fasta_load uploads the bytes of one FASTA record (from the .fai offset to the end of its last line, plus the one
 *   byte after it when the file has one), gl_fasta_stats counts, for row r, the slice [byte_start[r], byte_end[r]) of it
 *   the way Faidx.Stats does (every byte but the slice's last is classified, the next byte decides CpG):
 *   counts4[r] = {G+C, lower-case, A+C+G+T, CpG} and/or stats3[r] = {GC, CpG, Masked} as float64 (0 when no ACGT).
 *   byte_start = position(s), byte_end = min(position(e)+1, file length) relative to the loaded record.
 * gl_depth_format_chunk_stats = gl_depth_format_chunk with the three "%.3g" columns appended to every window row. */
int  gl_depth_chunk_rows(int64_t rs, int64_t re, int32_t W, const int32_t* run_start, const uint8_t* run_class, int64_t n_runs,
                         int64_t* row_s, int64_t* row_e, int64_t cap, int64_t* n_rows);
int  gl_fasta_load(gl_ctx* ctx, const uint8_t* bytes, int64_t n);
int  gl_fasta_stats(gl_ctx* ctx, const int64_t* byte_start, const int64_t* byte_end, int64_t n_rows, int64_t* counts4, double* stats3);
int  gl_depth_format_chunk_stats(const char* chrom, int64_t rs, int64_t re, int32_t W, const int64_t* win_sum, int64_t n_windows,
                                 const int32_t* run_start, const uint8_t* run_class, int64_t n_runs,
                                 const double* stats3, int64_t n_stat_rows,
                                 char** depth_bed, int64_t* depth_len, char** callable_bed, int64_t* callable_len);

/* ---------------------------------------------------------------- feeder (host-only, no GPU needed)
 * BGZF (multi-threaded inflate) + BAM decode + the `samtools depth` record filter: records with
 * (flag & 0x704) == 0 and MAPQ >= min_mapq contribute their M/=/X blocks (D and N advance without
 * counting; blocks separated only by I/S/H/P are merged), per reference, in record order.
 * Replaces the decode half of the `samtools depth` child (depth/depth.go:45).  only_tid < 0: all refs. */
typedef struct gl_segset gl_segset;
int  gl_bam_decode_segments(const char* path, int32_t min_mapq, int32_t threads, int32_t only_tid, gl_segset** out,
                            char* err, int64_t err_cap);
int  gl_segset_n_refs(const gl_segset* s, int32_t* n_refs, int64_t* n_records, int64_t* n_pass);
int  gl_segset_ref(const gl_segset* s, int32_t tid, const char** name, int64_t* length, const int32_t** start,
                   const int32_t** end, int64_t* n);
void gl_segset_free(gl_segset* s);
/* Index-guided parallel feeder: what `samtools depth -r chr:b-e` gives the reference (depth/depth.go:116,152) — only
 * the BGZF blocks of the requested reference range are read (BAI linear index -> record-aligned virtual offsets); the
 * range is cut into units at those offsets and every host-pool thread inflates and parses its own units.
 * gl_bam_open also loads path + ".bai" (or .bam -> .bai); decoding needs that index.
 * gl_bam_decode: the M/=/X blocks of the records of `tid` that pass the filter and can overlap [beg,end), as
 *   format 8  : packed8 words  (a0 = int32 anchors[n], a1 = uint8 dstart[64 n], a2 = uint8 len[64 n]; n blocks), or
 *   format 32 : (a0 = int32 start[n], a1 = int32 end[n]) sorted by start,
 * want_format 0 chooses (packed8 unless the blocks average more than 400 bases: long reads).  The arrays belong to the
 * handle and stay valid until its next gl_bam_decode / gl_bam_close; one handle per decoding thread. */
typedef struct {
    int32_t format, units, max_len, _pad;
    int64_t n;
    const int32_t* a0; const void* a1; const void* a2;
    int64_t n_records, n_pass, bytes_in, bytes_out;      /* records seen / passing; compressed bytes read / bytes inflated */
    double inflate_s, parse_s, wall_s;                   /* summed over the workers; wall clock of the call */
} gl_bam_segments;
int  gl_bam_open(const char* path, gl_bam** out, char* err, int64_t err_cap);
void gl_bam_close(gl_bam* b);
int  gl_bam_info(const gl_bam* b, int32_t* n_refs, int32_t* has_index);
int  gl_bam_ref(const gl_bam* b, int32_t tid, const char** name, int64_t* length, int64_t* n_mapped /* -1: no stats bin */);
int  gl_bam_decode(gl_bam* b, int32_t tid, int64_t beg, int64_t end, int32_t min_mapq, int32_t threads, int32_t want_format,
                   gl_bam_segments* out, char* err, int64_t err_cap);
/* The whole feeder on the GPU for one reference of an indexed BAM: its compressed BGZF range is read into pinned memory and
 * uploaded, every member is inflated by a warp (gl_bgzf_inflate_device), the records between consecutive linear-index
 * offsets are walked by one thread each (filter + CIGAR, as gl_bam_decode), and the M/=/X blocks land in ctx-owned device
 * arrays *d_start / *d_end (*n of them, BAM order; valid until the next call on this ctx) — feed them to
 * gl_depth_add_segments_device.  Only compressed bytes cross PCIe.  GL_ESTATE: not possible for this reference on the device
 * (no usable index, a member or record the device code rejects): use gl_bam_decode. */
int  gl_bam_decode_device(gl_ctx* ctx, gl_bam* b, int32_t tid, int32_t min_mapq, const int32_t** d_start, const int32_t** d_end, int64_t* n,
                          gl_bam_segments* stats);
/* BGZF inflate ON THE GPU (inflate.cu): one warp per BGZF member, thousands in flight — the stage the reference's samtools
 * children (and this library's host feeder) spend their time in.  Block b = d_comp[comp_off[b], comp_off[b+1]) (the whole
 * member) -> d_out[out_off[b], out_off[b+1]), out_off from the members' ISIZE fields; d_status[b] != 0: malformed or
 * unsupported member (fall back to zlib).  Device pointers; asynchronous on the ctx stream. */
int  gl_bgzf_inflate_device(gl_ctx* ctx, const uint8_t* d_comp, const int64_t* d_comp_off, const int64_t* d_out_off, int64_t n_blocks,
                            uint8_t* d_out, int32_t* d_status);
/* BAI: per-reference linear index (16 KB tiles) + the 0x924a stats bin (indexcov/types.go:19,45-58),
 * what indexcov takes from biogo's bam.ReadIndex (indexcov/indexcov.go:514). */
typedef struct gl_bai gl_bai;
int  gl_bai_read(const char* path, gl_bai** out, char* err, int64_t err_cap);
int  gl_bai_n_refs(const gl_bai* b, int32_t* n_refs, uint64_t* n_no_coor);
int  gl_bai_ref(const gl_bai* b, int32_t tid, const uint64_t** ioffsets, int64_t* n_intv, uint64_t* mapped,
                uint64_t* unmapped, int32_t* has_stats);
void gl_bai_free(gl_bai* b);

/* CRAM index: one reference's slices (alignment start, span, slice bytes) -> 16 KB pseudo-tile sizes
 * (indexcov/crai/crai.go:56-127).  GL_ERANGE where the reference panics, or when cap is too small
 * (*n_sizes then holds the needed count). */
int  gl_crai_make_sizes(const int64_t* aln_start, const int64_t* aln_span, const int32_t* slice_len, int64_t n,
                        int64_t* sizes, int64_t cap, int64_t* n_sizes);

/* ---------------------------------------------------------------- indexcov
 * Replaces indexcov/types.go:45-82 (getSizes), indexcov/indexcov.go:83-125 (Index.init),
 * :129-151 (NormalizedDepth), :170-177 (CountsAtDepth), :1050-1078 (counter.count),
 * :549-597 (normalizeAcrossSamples).  float32/float64 results are bit-exact (no FMA contraction,
 * same rounding points as Go on amd64). */

/* I1: tile sizes from BAI linear-index virtual offsets.  voff: concatenated per-ref linear
 * index entries of one sample; ref_ptr: CSR offsets (n_refs+1).  sizes gets, per ref with
 * >=2 intervals, n_intv-1 deltas; size_ptr (n_refs+1) their CSR offsets.  Returns GL_ERANGE
 * if any delta is negative (the reference panics, types.go:75-77). */
int  gl_indexcov_sizes(gl_ctx* ctx, const uint64_t* voff, const int64_t* ref_ptr, int32_t n_refs,
                       int64_t* sizes, int64_t* size_ptr);
/* I2: the capped weighted median of Index.init: sorted[first i with cumsum(min(s,n98))[i] > total/2]. */
int  gl_indexcov_scale(gl_ctx* ctx, const int64_t* sizes, int64_t n, int64_t* median_out);
/* I3: depth[i] = min(float32(float64(sizes[i])/median), 50000). */
int  gl_indexcov_normalize(gl_ctx* ctx, const int64_t* sizes, int64_t n, double median, float* depth_out);
/* I2+I3 for a cohort in one kernel (a CTA per sample): the two order statistics are bracketed by a sorted strided
 * sample of the tiles and read off the few tiles inside the brackets after one pass (samples of <= 8192 tiles are sorted
 * whole; when a bracket fails, an exact histogram select takes over), then a second pass writes the depths.
 * S samples, tile sizes in CSR layout (sample_ptr, S+1); medians[S]; depths in the same layout
 * (depth_out may be NULL).  A sample with median 0 gets zero depths (the reference returns none). */
int  gl_indexcov_cohort(gl_ctx* ctx, const int64_t* sizes, const int64_t* sample_ptr, int32_t S,
                        double* medians, float* depth_out);
int  gl_indexcov_cohort_device(gl_ctx* ctx, const int64_t* d_sizes, const int64_t* d_sample_ptr, int32_t S,
                               double* d_medians, float* d_depth_out);
/* how many samples of the last gl_indexcov_cohort* call needed the exact fallback select (heavy ties / overlapping
 * brackets) instead of the two-pass bracketed path; the results are identical either way */
int  gl_indexcov_cohort_fallbacks(gl_ctx* ctx, int32_t* n);
/* I1 for a whole cohort in ONE launch, on device-resident data: d_voff = every sample's linear-index virtual offsets
 * concatenated; descriptor d (one per sample x reference with >= 2 entries) = its n_intv[d] entries start at voff_off[d] and
 * its n_intv[d]-1 sizes go to size_off[d].  GL_ERANGE on a negative delta (types.go:75-77). */
int  gl_indexcov_sizes_batch_device(gl_ctx* ctx, const uint64_t* d_voff, const int64_t* d_voff_off, const int32_t* d_n_intv,
                                    const int64_t* d_size_off, int64_t n_desc, int64_t* d_sizes);
/* I4: 70-slot histogram of one depth array (counts += ..., like the reference's counts[...]++). */
int  gl_indexcov_counts(gl_ctx* ctx, const float* depth, int64_t n, int32_t counts[GL_INDEXCOV_SLOTS]);
/* I5: counter.count over depth[0..n) with `longest` tiles expected; out4 += {out, low, hi, in}. */
int  gl_indexcov_bins(gl_ctx* ctx, const float* depth, int64_t n, int64_t longest, int64_t out4[4]);
/* I4+I5 for many (sample, chromosome) segments at once: seg_ptr CSR (n_seg+1) into depth,
 * longest[n_seg] (may be NULL); counts70[n_seg*70] and bins4[n_seg*4] are overwritten. */
int  gl_indexcov_counts_batch(gl_ctx* ctx, const float* depth, const int64_t* seg_ptr, const int64_t* longest,
                              int32_t n_seg, int32_t* counts70, int64_t* bins4);
int  gl_indexcov_counts_batch_device(gl_ctx* ctx, const float* d_depth, const int64_t* d_seg_ptr,
                                     const int64_t* d_longest, int32_t n_seg, int32_t* d_counts70, int64_t* d_bins4);
/* the same for arbitrary slices [seg_start[k], seg_start[k] + seg_len[k]) of a device-resident depth array: every
 * (chromosome, sample) pair of a cohort in one launch, straight from gl_indexcov_cohort_device's output */
int  gl_indexcov_counts_segs_device(gl_ctx* ctx, const float* d_depth, const int64_t* d_seg_start, const int64_t* d_seg_len,
                                    const int64_t* d_longest, int32_t n_seg, int32_t* d_counts70, int64_t* d_bins4);
/* I6: the "%.3g" of every value (the bed.gz row writer, indexcov.go:678-680,1038-1048): 10-byte tokens,
 * bytes [0..len) = text, byte 9 = len; len 0 means the magnitude is outside [1e-15,1e15) and the host formats it. */
int  gl_format_g3(gl_ctx* ctx, const float* vals, int64_t n, uint8_t* tokens);
int  gl_format_g3_device(gl_ctx* ctx, const float* d_vals, int64_t n, uint8_t* d_tokens);
/* I7: in-place cross-sample normalisation of one chromosome; depths is S rows of stride T,
 * lens[i] valid entries in row i.  No-op for S < 5 (indexcov.go:551). */
int  gl_indexcov_xnorm(gl_ctx* ctx, float* depths, const int32_t* lens, int32_t S, int32_t T);
/* PCA (the .ped's PC1..PC5, indexcov.go:686-705,773-807; DESIGN §1.11).
 *   gl_indexcov_pca8       : host-only: the byte of each depth: clip at 8, uint8(8191.875f * d + 0.5f) as Go converts it
 *                            (truncation to int32, low byte).
 *   gl_indexcov_pca        : x is S rows of D bytes (row stride ld >= D).  k_out = min(k, S, D); proj (S x k, row-major) gets
 *                            X V[:, :k_out] (gonum stat.PC: V from the SVD of the column-centred X; X uncentred), each
 *                            column's sign chosen so the left singular vector's largest-magnitude entry is positive (lowest
 *                            sample on a tie); sv[0..k) the singular values.  A column whose squared singular value is at most
 *                            1e-12 times the first one (or all of them when the first is 0) is 0 with sv 0.  Columns from
 *                            k_out on are 0.  gram (nullable, S x S) receives the exact X X^T.  1 <= S <= 65535.
 *                            GL_ENOMEM when X and the S x S buffers do not fit in free device memory.
 *   gl_indexcov_pca_device : the same on a device-resident X; d_x and ld must be multiples of 16 bytes.  The outputs are host.
 *   gl_indexcov_pca_phases : seconds of the last call: upload, Gram + centring, eigenvectors + projections.
 *   gl_pca_tridiag_top     : host-only: the k largest eigenvalues w (descending) of the symmetric tridiagonal (d[n], e[n-1])
 *                            and, when z is not NULL, unit eigenvectors (column j at z[j*n]), as gl_indexcov_pca finds them. */
int  gl_indexcov_pca8(const float* d, int64_t n, uint8_t* out);
int  gl_indexcov_pca(gl_ctx* ctx, const uint8_t* x, int64_t ld, int32_t S, int64_t D, int32_t k, double* proj, double* sv,
                     int32_t* k_out, int64_t* gram);
int  gl_indexcov_pca_device(gl_ctx* ctx, const uint8_t* d_x, int64_t ld, int32_t S, int64_t D, int32_t k, double* proj, double* sv,
                            int32_t* k_out, int64_t* gram);
int  gl_indexcov_pca_phases(gl_ctx* ctx, double* t3);
/* host-only: ||X_c||_F^2, the squared Frobenius norm of the column-centred byte matrix (S rows of D bytes, stride ld), exactly:
 * sum over columns of (S * sum x^2 - (sum x)^2), in 128-bit integers, divided by S once.  sv[k]^2 / total is gonum's
 * normalised `vars` (indexcov.go:787-789), the "variance explained" of component k. */
int  gl_indexcov_pca_total(const uint8_t* x, int64_t ld, int32_t S, int64_t D, double* total);
int  gl_pca_tridiag_top(const double* d, const double* e, int32_t n, int32_t k, double* w, double* z);

/* ---------------------------------------------------------------- indexcov charts (plot.cu; DESIGN §1.14)
 * A chart's lines are drawn into an INDEX IMAGE: W x H uint32 over its data area (row 0 at the top), 0 where no line passes,
 * else the largest draw index whose line covers the pixel (opaque lines: the last one drawn shows).  Images of several
 * charts are stacked: chart c at img + c*W*H.  A dataset d is one line: chart[d] is its chart, draw[d] (>= 1) its index.
 * The depth and ROC charts are GL_PLOT_CW x GL_PLOT_CH pixels (4 x 3 in at 96 px/in) with a GL_PLOT_W x GL_PLOT_H data area
 * whose top-left pixel is (GL_PLOT_AX, GL_PLOT_AY).
 *   gl_plot_select_device / _host : per dataset (values at off[d], len[d] of them): sel3 = {first, m, stride}: the first
 *       value != 0 (NaN counts), the number of plotted vertices (0 when none or when one of them is NaN: not drawn) and the
 *       thinning stride (10 above 2000 values after the skip, 5 above 1000, else 1); yext2 = min, max of min(v, 2.5) over
 *       them (0, 0 when not drawn).  Vertex j is x = (first + j*stride) * mult, y = min(v[first + j*stride], 2.5).
 *   gl_plot_transform : ext4 = {xmin, xmax, ymin, ymax} of the plotted vertices (an empty extent widened to +-1) ->
 *       xf4 = {xmin, W / (xmax - xmin), ymin, H / (ymax - ymin)}: X = (x - xmin) * sx, Y = H - (y - ymin) * sy.
 *   gl_plot_line_radius : r = max(0.5, w * 96 / 72 / 2) for w = 0.8 pt, or 0.65 pt above 30 datasets.
 *   gl_plot_raster_series_device / _host : the image of selected value series (xf4: 4 doubles per chart).  A segment AB
 *       covers pixel (i, j) when the squared float64 distance from (i + 0.5, j + 0.5) to AB is <= r*r (see plot.cu for the
 *       exact order of operations).  The image is cleared first.
 *   gl_plot_raster_xy / _host : the same for explicit float64 vertices: dataset d is x[ptr[d] .. ptr[d+1]), y likewise;
 *       host arrays in, host image out (the device entry rasterises on the GPU).
 *   gl_plot_color   : host-only: the colour of sample k: grey (180,180,180) below n_background, else a hash of k.
 *   gl_plot_ticks   : host-only: multiples of the smallest step 1, 2 or 5 x 10^k that gives at most 8 ticks in [lo, hi].
 *   gl_plot_millions: host-only: an x label of a depth chart (indexcov/plot.go makeMillions).
 *   gl_plot_text    : host-only: s in the built-in 5x7 font, black, top-left at (x, y); vertical: bottom to top from (x, y).
 *   gl_plot_compose : host-only: the GL_PLOT_CW x GL_PLOT_CH RGB8 chart: palette[3*v] for pixel value v (palette[0..2] for
 *       v >= n_pal), white where 0, axes, ticks, tick labels and titles.  kind GL_PLOT_DEPTH: y ticks 0.0..2.0, x labels
 *       in KB/MB; GL_PLOT_PLAIN: nice ticks on both axes; GL_PLOT_SQUARE: the same on the square canvas (rgb and img then
 *       have its sizes).  ext4 as gl_plot_transform takes it.
 *   gl_plot_png     : host-only: the PNG of W x H RGB8 pixels: filter 0 on every row, one IDAT.  out == NULL: *len = the
 *       room needed. */
#define GL_PLOT_CW 384
#define GL_PLOT_CH 288
#define GL_PLOT_AX 56
#define GL_PLOT_AY 8
#define GL_PLOT_W  316
#define GL_PLOT_H  244
#define GL_PLOT_DEPTH 0
#define GL_PLOT_PLAIN 1
#define GL_PLOT_SQUARE 2   /* the sex chart: GL_PLOT_SQ_CW x GL_PLOT_SQ_CH (6 x 6 in), data area GL_PLOT_SQ_W x GL_PLOT_SQ_H, plain ticks */
#define GL_PLOT_SQ_CW 576
#define GL_PLOT_SQ_CH 576
#define GL_PLOT_SQ_W  508
#define GL_PLOT_SQ_H  532
int  gl_plot_select_device(gl_ctx* ctx, const float* d_vals, const int64_t* d_off, const int64_t* d_len, int32_t n, int64_t* d_sel3,
                           float* d_yext2);
int  gl_plot_select_host(const float* vals, const int64_t* off, const int64_t* len, int32_t n, int64_t* sel3, float* yext2);
int  gl_plot_transform(const double* ext4, int32_t W, int32_t H, double* xf4);
double gl_plot_line_radius(int32_t n_datasets);
int  gl_plot_raster_series_device(gl_ctx* ctx, const float* d_vals, const int64_t* d_off, const int64_t* d_sel3, double mult,
                                  const int32_t* d_chart, const uint32_t* d_draw, int32_t n, const double* d_xf4, int32_t n_charts,
                                  int32_t W, int32_t H, double r, uint32_t* d_img);
int  gl_plot_raster_series_host(const float* vals, const int64_t* off, const int64_t* sel3, double mult, const int32_t* chart,
                                const uint32_t* draw, int32_t n, const double* xf4, int32_t n_charts, int32_t W, int32_t H, double r,
                                uint32_t* img);
int  gl_plot_raster_xy(gl_ctx* ctx, const double* x, const double* y, const int64_t* ptr, const int32_t* chart, const uint32_t* draw,
                       int32_t n, const double* xf4, int32_t n_charts, int32_t W, int32_t H, double r, uint32_t* img);
int  gl_plot_raster_xy_host(const double* x, const double* y, const int64_t* ptr, const int32_t* chart, const uint32_t* draw, int32_t n,
                            const double* xf4, int32_t n_charts, int32_t W, int32_t H, double r, uint32_t* img);
void gl_plot_color(int32_t k, int32_t n_background, uint8_t* rgb3);
int  gl_plot_ticks(double lo, double hi, double* out, int32_t cap, int32_t* n);
int  gl_plot_millions(double v, char* buf, int32_t cap);
int  gl_plot_text(uint8_t* rgb, int32_t CW, int32_t CH, int32_t x, int32_t y, const char* s, int32_t vertical);
int  gl_plot_compose(const uint32_t* img, const uint8_t* palette, int32_t n_pal, int32_t kind, const double* ext4, const char* xtitle,
                     const char* ytitle, uint8_t* rgb);
int  gl_plot_png(const uint8_t* rgb, int32_t W, int32_t H, uint8_t* out, int64_t cap, int64_t* len);

/* indexsplit (indexsplit/indexsplit.go:92-115): amount of cohort data per 16 KB tile = sum over the S samples, in path
 * order, of float64(size)/1e9 — bit-identical to the reference's sequential adds.  sizes: every sample's tile sizes
 * (gl_indexcov_sizes / gl_crai_make_sizes) concatenated; ptr[s*(R+1)+r] = offset of sample s's tiles of reference r
 * (a sample whose index has fewer references repeats its end offset); out_ptr[r] = prefix sum of max_s(len) per
 * reference; out[out_ptr[r] + j] = the tile's sum. */
int  gl_indexsplit_accumulate(gl_ctx* ctx, const int64_t* sizes, const int64_t* ptr, int32_t S, int32_t R, const int64_t* out_ptr,
                              double* out);
/* Host-only: the rest of indexsplit.Split (indexsplit.go:37-65,119-188): chop outliers, share N regions over the
 * references by their data, walk the tiles and cut.  tile_sum/out_ptr as filled by gl_indexsplit_accumulate (R index
 * references); the n_refs listed references (name, length, id into the index references or -1) are reported in order;
 * problematic intervals (-p) are (listed-reference number, start, end).  Returns the lines "chrom\tstart\tend\t%.2f\t%d\n"
 * in *text (release with gl_free_text). */
int  gl_indexsplit_chunks(const double* tile_sum, const int64_t* out_ptr, int32_t R, const char* const* ref_names, const int64_t* ref_lens,
                          const int32_t* ref_ids, int32_t n_refs, int32_t N, const int32_t* prob_ref, const int64_t* prob_start,
                          const int64_t* prob_end, int64_t n_prob, char** text, int64_t* text_len);

/* ---------------------------------------------------------------- multidepth
 * Replaces multidepth/multidepth.go: the `samtools depth -Q q -r chrom:k*C+1` child over all BAMs of one chunk (:208-221),
 * sufficientDepth (:158-166), the chunk state machine of aggregate (:222-266), splitBlocks (:183-200) and means (:268-283).
 * One contig [0, L), S samples, L < 2^30, 1 <= S <= 65535.  Device memory is O(L) plus the blocks x S outputs.
 *   gl_multidepth_begin   : minSamples = int(0.5 + min_samples * S) (:64) as Go converts on amd64 (NaN, +-Inf and values
 *                           outside [-2^63, 2^63) give INT64_MIN); zeroes the per-base counters.
 *   pass 1, per sample    : gl_depth_begin(ctx, 0, L), gl_depth_add_segments* (any form), gl_multidepth_count.  The depth tile
 *                           core (any path, same eligibility checks and fallbacks as gl_depth_reduce) counts, per base, the
 *                           samples with d >= mincov and whether any sample has d > 0 (a `samtools depth` line).
 *   gl_multidepth_sites   : class runs of the contig, in position order: class 0 = no sample covers the base (no line),
 *                           1 = insufficient site, 2 = sufficient site (more than minSamples samples with d >= mincov).
 *                           Pass NULL arrays to get *n_runs only; GL_ERANGE when cap is too small.
 *   gl_multidepth_blocks  : host-only, no GPU needed: the chunk state machine over the runs (chunk = 0: 5e6 bases, / 5 when
 *                           S > 50, :60-62,121).  Blocks (start, end, sufficient sites) in chunk order: the reference's
 *                           output with -p 1, duplicate blocks of overlapping chunks included.  NULL outputs: count only.
 *   gl_multidepth_set_blocks : uploads the blocks.
 *   pass 2, per sample    : gl_depth_begin(ctx, 0, L), the same segments again, gl_multidepth_sums(ctx, sample): exact Σd over
 *                           each block's sufficient sites.  A cell whose "%.2f" follows from the integers (gl_multidepth_certify)
 *                           gets q = round(100 Σd / l); the others take the reference's float64 chain on the device (val).
 *   gl_multidepth_result  : blocks x S arrays, row-major by block (any may be NULL).
 *   gl_multidepth_stats   : blocks, cells that took the float64 chain, cells certified, minSamples.
 *   gl_multidepth_text    : host-only: the rows after the header ("chrom\tstart\tend" + "\t%.2f" per sample), certified cells
 *                           printed from q, the others from val; made on `threads` of the host pool (0 = all).  gl_free_text. */
int  gl_multidepth_begin(gl_ctx* ctx, int64_t contig_len, int32_t n_samples, int32_t mincov, double min_samples);
int  gl_multidepth_count(gl_ctx* ctx);
int  gl_multidepth_sites(gl_ctx* ctx, int32_t* run_start, uint8_t* run_class, int64_t cap, int64_t* n_runs);
int  gl_multidepth_blocks(const int32_t* run_start, const uint8_t* run_class, int64_t n_runs, int64_t contig_len, int32_t n_samples,
                          int64_t chunk, int64_t max_skip, int64_t min_size, int64_t window, int64_t* blk_start, int64_t* blk_end,
                          int64_t* blk_sites, int64_t cap, int64_t* n_blocks);
int  gl_multidepth_set_blocks(gl_ctx* ctx, const int64_t* blk_start, const int64_t* blk_end, const int64_t* blk_sites, int64_t n_blocks);
int  gl_multidepth_sums(gl_ctx* ctx, int32_t sample);
int  gl_multidepth_result(gl_ctx* ctx, uint64_t* sums, int64_t* q, double* val, uint8_t* certified);
int  gl_multidepth_stats(gl_ctx* ctx, int64_t* n_blocks, int64_t* n_walked, int64_t* n_certified, int64_t* min_samples);
/* host-only: certified[i] = 1 and q[i] = round(100 sum / span) when the reference's "%.2f" of its float64 chain over n_sites
 * terms is provably those digits (host/md_cert.h) */
int  gl_multidepth_certify(const int64_t* sum, const int64_t* n_sites, const int64_t* span, int64_t n, int64_t* q, uint8_t* certified);
int  gl_multidepth_text(const char* chrom, const int64_t* blk_start, const int64_t* blk_end, int64_t n_blocks, int32_t S, const int64_t* q,
                        const double* val, const uint8_t* certified, int32_t threads, char** text, int64_t* text_len);

/* ---------------------------------------------------------------- dcnv
 * Replaces dcnv/dcnv.go:323-354 (a separate binary of the reference), the step after depthwed: GC-debias and median-normalise
 * an n-sites x S-samples matrix (DESIGN §1.9).
 *   gl_go_argsort_f64  : host-only: inds = the permutation gonum's floats.Argsort(v) leaves, i.e. Go's unstable sort.Sort
 *                        (pdqsort, go 1.21) over (value, index) pairs.  The order inside ties is Go's own.
 *   gl_dcnv_normalize_device : columns [c0, c1) of the row-major n x ld float64 matrix d_x, rows in position order; d_inds =
 *                        the GC argsort (a permutation of [0, n), not checked here).  Per column: divide every row by
 *                        max(1, the moving median of 9 along the GC order, with the reference's window quirks), then by the
 *                        sample median (sorted[k + int(0.65 (n - k))], k = leading exact zeros, 0 when a value is
 *                        negative).  Writes the result to columns [0, c1 - c0) of d_out (row stride ld_out; must not overlap
 *                        d_x) and the sample medians to d_medians[0, c1 - c0).  n >= 5.  An all-zero column (the
 *                        reference panics) returns GL_ERANGE naming it.
 *   gl_dcnv_normalize  : the same from host arrays; checks inds, streams blocks of block_cols columns (0: as many as fit in free
 *                        device memory, 24 bytes per cell).  out may be x itself (out = x + c0, ld_out = ld).
 *   gl_format_f2[_device] : the exact "%.2f" of every value as a 16-byte token, the text NUL-padded; an empty token means the
 *                        text does not fit (|v| near or above 1e12) and the caller formats it.  NaN / ±Inf are spelled as Go
 *                        does.  d_tokens is 16-byte aligned.
 *   gl_format_f2_host  : host-only mirror of the same tokens. */
int  gl_go_argsort_f64(const double* v, int64_t n, int64_t* inds);
int  gl_dcnv_normalize_device(gl_ctx* ctx, const double* d_x, int64_t n, int64_t ld, const int64_t* d_inds, int32_t c0, int32_t c1,
                              double* d_out, int64_t ld_out, double* d_medians);
int  gl_dcnv_normalize(gl_ctx* ctx, const double* x, int64_t n, int64_t ld, const int64_t* inds, int32_t c0, int32_t c1, int32_t block_cols,
                       double* out, int64_t ld_out, double* medians);
int  gl_format_f2(gl_ctx* ctx, const double* vals, int64_t n, uint8_t* tokens);
int  gl_format_f2_device(gl_ctx* ctx, const double* d_vals, int64_t n, uint8_t* d_tokens);
int  gl_format_f2_host(const double* vals, int64_t n, uint8_t* tokens);
/* dcnv --svd (DESIGN §1.13): remove a cohort's leading components from the n x S row-major float64 matrix (row stride ld >= S),
 * in place: the reference's ZScore.Scale, SVD.Debias{MinVariancePct} and ZScore.UnScale.  Each row is z-scored (m = mean,
 * sd with S - 1, z = (x - m) * (1 / sd)); a row whose values are all equal, and every row when S < 2, is excluded and never
 * written.  s = the singular values of Z (the kept rows), from the eigenvalues of the S x S Gram Z^T Z, descending; an
 * eigenvalue <= 1e-12 times the largest counts as 0.  n_removed = the first index n with n >= min(15, rank) or
 * 100 s[n] / sum(s) <= min_pct; each kept row becomes max(0, (z - V_n V_n^T z) sd + m).  n_removed = 0 leaves x untouched.
 *   gl_dcnv_svd        : host x, streamed through the device in row blocks of block_rows (0: as many as fit; rounded down to a
 *                        multiple of 4), twice when the matrix does not fit.  The result does not depend on block_rows.
 *   gl_dcnv_svd_device : the same on a device-resident d_x (8-byte aligned).
 *   sv (nullable) receives S values (0 past the rank); gram (nullable) the S x S Z^T Z; n_kept (nullable) the rows that took part.  min_pct must be finite and
 *   >= 0; a non-finite value in a row that is not excluded is GL_EINVAL naming the row; GL_ENOMEM when the S x S Gram and its
 *   workspace do not fit.  1 <= S <= 65535.
 *   gl_dcnv_svd_phases : seconds of the last call: stats + Gram, eigen, projection, host <-> device copies.
 *   gl_pca_tridiag_above : host-only: every eigenvalue above rel times the largest of the symmetric tridiagonal (d[n], e[n-1]),
 *                        descending, into w (room for n), *count of them; each bisected on the host pool, bit for bit as
 *                        gl_pca_tridiag_top finds it.  0 <= rel < 1. */
int  gl_dcnv_svd(gl_ctx* ctx, double* x, int64_t n, int64_t ld, int32_t S, double min_pct, int64_t block_rows, double* sv,
                 double* gram, int32_t* n_removed, int64_t* n_kept);
int  gl_dcnv_svd_device(gl_ctx* ctx, double* d_x, int64_t n, int64_t ld, int32_t S, double min_pct, double* sv, double* gram,
                        int32_t* n_removed, int64_t* n_kept);
int  gl_dcnv_svd_phases(gl_ctx* ctx, double* t4);
int  gl_pca_tridiag_above(const double* d, const double* e, int32_t n, double rel, double* w, int32_t* count);

/* ---------------------------------------------------------------- dcnv's depth chart (dcnv_chart.cu; DESIGN §1.9)
 * x is the n x S row-major float64 matrix depth.bed holds (after the normalisation, and --svd when given).  Sample k's line
 * (dcnv.go asValues, no thinning): rows i >= first[k], the first row whose value is not == 0 (NaN is not; n when none), are
 * vertices x = i * 16384, y = min(v, 2.5).  The line is stepped: step i runs (x_i, y_i) -> (x_{i+1}, y_i) -> (x_{i+1}, y_{i+1})
 * and is not drawn when either y is NaN or -Inf.  The image is an index image as the gl_plot_* entries describe it, sample k
 * drawn with index S - k (sample 0 on top, as Chart.js 2 stacks the page's datasets), under the same float64 pixel rule.
 *   gl_dcnv_chart_select_host : first[S] and yext2[2S] = min, max of the drawn y of each sample (-0.0 as 0.0; +Inf, -Inf when
 *       it has none).
 *   gl_dcnv_chart_extent : host-only: ext4 = {xmin, xmax, ymin, ymax} over every sample's vertices (x) and drawn y, 0 where
 *       there are none; gl_plot_transform's input.
 *   gl_dcnv_chart_raster_host : the W x H image of every sample's steps under transform xf4 and line radius r; cleared first.
 *       W * H <= 393216.
 *   gl_dcnv_chart : the select, the extent and the image on the GPU, the matrix streamed through the device in row blocks of
 *       block_rows (0: as many as fit in free device memory), once when it fits and twice when it does not.  xf4 is
 *       gl_plot_transform(ext4, W, H).  Nothing depends on block_rows. */
int  gl_dcnv_chart_select_host(const double* x, int64_t n, int64_t S, int64_t* first, double* yext2);
int  gl_dcnv_chart_extent(const int64_t* first, const double* yext2, int64_t n, int64_t S, double* ext4);
int  gl_dcnv_chart_raster_host(const double* x, int64_t n, int64_t S, const int64_t* first, const double* xf4, int32_t W, int32_t H,
                               double r, uint32_t* img);
int  gl_dcnv_chart(gl_ctx* ctx, const double* x, int64_t n, int64_t S, int64_t block_rows, int32_t W, int32_t H, double r, int64_t* first,
                   double* yext2, double* ext4, uint32_t* img);

/* ---------------------------------------------------------------- emdepth
 * Restates emdepth/emdepth.go (a library of the reference with no command): a cn.mops-style EM per row of an n x S depth
 * matrix, the copy number (CN) of every cell, and the Cache that merges non-CN2 rows into per-sample CNVs (DESIGN §1.10).
 * Values are used as given (float32, no normalisation); each must be finite, non-negative (sign bit clear) and below 2^62,
 * else GL_EINVAL naming the row (a policy: the reference panics only for some of these values).  S = 2 is GL_EINVAL (the reference's even median indexes out of range); 1 <= S <= 65535.
 * One byte per cell, row-major n x S: bits 0-3 the CN (0..9; 9 = above the top centre), bits 4-5 the Same class of
 * Log2FC = log2(d / lambda[2]) (0: -0.8 < fc < 0.4, 1: fc <= -0.8, 2: fc >= 0.4, 3: NaN), bit 6 set when fc is outside
 * (-0.5, 0.3).
 *   gl_emdepth_device : rows of the row-major float32 matrix d_x (row stride ld >= S); d_cells n x S; d_lambda (nullable)
 *                       n x 9 final centres.
 *   gl_emdepth        : the same from host arrays, streamed in blocks of block_rows rows (0: as many as fit in free device
 *                       memory, 5 bytes per cell).
 *   gl_emdepth_stats  : of the last call: rows, cells whose Poisson test or Log2FC thresholds fell inside the error band of
 *                       the reference's CPU-dependent Exp / Log (decided by the device's functions: UNPINNED), and bin
 *                       means that were summed in sample order because a tree sum could round differently.
 *   gl_emdepth_factors : host-only: the centres' factors math.Pow(i / 2, 1.1), i = 0..8, as the kernel uses them.
 *   gl_emdepth_cnvs   : host-only: the reference's Cache over the rows in order, Clear(nil) before every row in breaks[]
 *                       (sorted row indices where a chromosome starts) and after the last row; starts / ends are the rows'
 *                       uint32 positions.  CNV i is sample cnv_sample[i] with PSize cnv_psize[i]; its rows are
 *                       rows[cnv_ptr[i], cnv_ptr[i+1]).  Within one Clear, CNVs come in sample order.  NULL outputs count
 *                       only; GL_ERANGE (with the counts set) when cap or rows_cap is too small.
 *   gl_emdepth_sum_host : host-only mirror of the kernel's bin sum: the float64 sum of v in a warp's order (32 strided
 *                       partial sums, then a butterfly) and whether the exactness certificate holds for it. */
int  gl_emdepth_device(gl_ctx* ctx, const float* d_x, int64_t n, int64_t ld, int32_t S, uint8_t* d_cells, double* d_lambda);
int  gl_emdepth(gl_ctx* ctx, const float* x, int64_t n, int64_t ld, int32_t S, int64_t block_rows, uint8_t* cells, double* lambda);
int  gl_emdepth_stats(gl_ctx* ctx, int64_t* n_rows, int64_t* n_uncertified, int64_t* n_sequential);
int  gl_emdepth_factors(double* f9);
int  gl_emdepth_cnvs(const uint8_t* cells, int64_t n, int32_t S, const int64_t* starts, const int64_t* ends, const int64_t* breaks,
                     int64_t n_breaks, int32_t* cnv_sample, int32_t* cnv_psize, int64_t* cnv_ptr, int64_t cap, int64_t* n_cnvs,
                     int64_t* rows, int64_t rows_cap, int64_t* n_rows);
int  gl_emdepth_sum_host(const float* v, int64_t n, double* sum, uint8_t* certified);

/* ---------------------------------------------------------------- cnveval
 * Restates cnveval/cnveval.go Evaluate (a separate binary of the reference): TP, FP, FN and TN of CNV calls against a truth
 * set, per sample and size class (DESIGN §1.12).  stats is uint64 [S][3][4]: class 0 (end - start < 20000), 1 (< 100000),
 * 2 (the rest); counts TP, FP, FN, TN.  A sample without calls counts nothing (the reference's updatePositive and updateFP
 * return early for it, so its missed truths are not FNs).  Chromosomes are ranks (int32 >= 0) that must follow the bytewise
 * order of their names: the reference compares names, the library compares ranks.  Coordinates are int64; a call or truth
 * with end < start or a coordinate outside [0, 2^62) is GL_EINVAL naming it (a policy: the reference takes them, but its
 * walk then has no order-free form, and lengths must fit int64).  po is the minimum overlap, in (0, 1] or NaN (NaN: nothing
 * qualifies, as in the reference), else GL_EINVAL.
 *   gl_cnveval_order  : host-only: perm = the permutation Go 1.21's sort.Slice leaves when it sorts n calls given in file order
 *                       by (chrom, start) (pdqsort, unstable: the order inside a tie is Go's own and changes the counts).
 *   gl_cnveval        : from host arrays.  Calls (sample, chrom, start, end, CN) in file order; truths (chrom, start, end, CN)
 *                       and their samples as a CSR: truth t carries t_mem_sample[t_mem_ptr[t], t_mem_ptr[t+1]) (a sample listed
 *                       twice counts twice).  Orders on the host, uploads, runs the device pass, downloads stats.
 *   gl_cnveval_device : the same on resident arrays laid out as gl_cnveval lays them out: calls grouped by sample (sample s has
 *                       calls [c_ptr[s], c_ptr[s+1]), n_calls in all) in gl_cnveval_order's order; truths sorted by (chrom,
 *                       start); memberships sample-major (sample s carries truths m_truth[m_ptr[s], m_ptr[s+1]), ascending,
 *                       n_mem in all).  The layout is checked on the device (GL_EINVAL naming the first bad position). */
int  gl_cnveval_order(const int32_t* chrom, const int64_t* start, int64_t n, int64_t* perm);
int  gl_cnveval(gl_ctx* ctx, int32_t S, const int32_t* c_sample, const int32_t* c_chrom, const int64_t* c_start, const int64_t* c_end,
                const int64_t* c_cn, int64_t n_calls, const int32_t* t_chrom, const int64_t* t_start, const int64_t* t_end,
                const int64_t* t_cn, int64_t n_truths, const int64_t* t_mem_ptr, const int32_t* t_mem_sample, double po,
                uint64_t* stats);
int  gl_cnveval_device(gl_ctx* ctx, int32_t S, const int64_t* d_c_ptr, int64_t n_calls, const int32_t* d_c_chrom, const int64_t* d_c_start,
                       const int64_t* d_c_end, const int64_t* d_c_cn, int64_t n_truths, const int32_t* d_t_chrom, const int64_t* d_t_start,
                       const int64_t* d_t_end, const int64_t* d_t_cn, const int64_t* d_m_ptr, int64_t n_mem, const int64_t* d_m_truth,
                       double po, uint64_t* d_stats);

/* ---------------------------------------------------------------- covstats
 * V2: histogram of int32 values in [lo,hi) -> hist[v-lo].  `goleft covstats` builds it over the sampled insert sizes,
 * template lengths and read lengths and reads every order statistic of covstats/covstats.go:57-76,175-199 off its running
 * count (k-th smallest = a search, madFilter's cut = a count) and feeds meanStd (:78-89) the values in ascending order
 * with multiplicity — no host sort (cli/goleft.cpp SortedCounts).  Any lo < hi: up to 2^32 - 1 bins. */
int  gl_bincount_i32(gl_ctx* ctx, const int32_t* v, int64_t n, int32_t lo, int32_t hi, uint64_t* hist);

/* ---------------------------------------------------------------- depthwed
 * W1: depthwed/depthwed.go:93-157.  means: S samples x R rows (sample-major) of the float64 4th BED
 * column; starts/ends/chrom_id[R] of the rows.  Computes int(0.5+mean) and sums consecutive rows of
 * one chrom until end-start >= size.  out: n_out rows x S (row-major by OUTPUT ROW, like the
 * reference's TSV lines).  The conversion is Go's on amd64: NaN, +-Inf and 0.5+mean outside
 * [-2^63, 2^63) give INT64_MIN, and the sums wrap modulo 2^64. */
int  gl_depthwed_aggregate(gl_ctx* ctx, const double* means, int32_t S, int64_t R,
                           const int32_t* starts, const int32_t* ends, const int32_t* chrom_id, int64_t size,
                           int32_t* out_start, int32_t* out_end, int32_t* out_chrom, int64_t* out, int64_t out_cap,
                           int64_t* n_out);
/* device form: d_grp[n_out+1] row groups (NULL: one row per output line); d_out n_out x S */
int  gl_depthwed_aggregate_device(gl_ctx* ctx, const double* d_means, int32_t S, int64_t R, const int64_t* d_grp,
                                  int64_t n_out, int64_t* d_out);

/* int32 forms — what BASELINE budgets (4 B in + 4 B out per cell): the reference rounds when it parses a line
 * (depthwed.go:103 d.depth = int(0.5 + dep)), so the caller hands over int32 depths and the matrix that travels over NVLink is
 * int32.  Group sums are taken in 64 bits; one that does not fit int32 makes the host form return GL_ERANGE with *n_out = -1
 * (rerun with gl_depthwed_aggregate).  The device form does the groups [g_begin, g_end) only (so the all-gather of one row
 * chunk can overlap the aggregation of the next), is ASYNCHRONOUS on the ctx stream, and sets *d_overflow (a device int the
 * caller zeroed) instead. */
int  gl_depthwed_aggregate_i32(gl_ctx* ctx, const int32_t* depth, int32_t S, int64_t R, const int32_t* starts, const int32_t* ends,
                               const int32_t* chrom_id, int64_t size, int32_t* out_start, int32_t* out_end, int32_t* out_chrom,
                               int32_t* out, int64_t out_cap, int64_t* n_out);
int  gl_depthwed_aggregate_i32_device(gl_ctx* ctx, const int32_t* d_depth, int32_t S, int64_t R, const int64_t* d_grp, int64_t g_begin,
                                      int64_t g_end, int32_t* d_out, int32_t* d_overflow);

/* W1 fused with its collective: the aggregation kernel stores every output row straight into the row-major n-sites x
 * n-samples matrix of EVERY GPU of the box (its own + NVLink peer mappings of the others): d_dst[d] = base of rank d's matrix
 * as a pointer valid on this ctx's device (gl_ipc_open between processes; plain peer pointers inside one process), row stride
 * `row_stride` ints, this rank's samples at columns [col_off, col_off + S).  No separate all-gather, no re-assembly.
 * 16-byte stores when row_stride and col_off are multiples of 4 and every d_dst[d] is 16-byte aligned; 4-byte stores
 * otherwise (any 4-byte aligned destination is accepted).  ASYNCHRONOUS on the ctx stream; after gl_sync on every rank and a host barrier the matrix is complete everywhere. */
int  gl_depthwed_aggregate_i32_p2p(gl_ctx* ctx, const int32_t* d_depth, int32_t S, int64_t R, const int64_t* d_grp, int64_t g_begin,
                                   int64_t g_end, int32_t* const* d_dst, int32_t world, int64_t row_stride, int32_t col_off,
                                   int32_t* d_overflow);
/* peer memory between the per-GPU processes of one box: export a gl_dev_alloc allocation as a 64-byte handle, open another
 * rank's handle as a device pointer usable by kernels of this ctx (cudaIpc*; the link is NVLink / NVSwitch) */
int  gl_ipc_export(gl_ctx* ctx, void* d_ptr, uint8_t handle64[64]);
int  gl_ipc_open(gl_ctx* ctx, const uint8_t handle64[64], void** d_peer_ptr);
int  gl_ipc_close(gl_ctx* ctx, void* d_peer_ptr);

/* ------------------------------------------------------------- multi-GPU
 * One process per GPU.  The caller distributes a 128-byte NCCL unique id (rank 0 creates it).
 * The one collective on this path: an all-gather over NVLink that assembles the depthwed
 * n-sites x n-samples matrix (or the indexcov cohort) from per-GPU sample shards. */
int  gl_comm_unique_id(uint8_t id128[128]);
int  gl_comm_init(gl_ctx* ctx, const uint8_t id128[128], int rank, int world);
int  gl_comm_destroy(gl_ctx* ctx);
/* all-gather equal-sized blocks that live on the device: d_recv holds world*bytes */
int  gl_allgather_device(gl_ctx* ctx, const void* d_send, void* d_recv, int64_t bytes);
/* asynchronous on the ctx's communication stream: starts when the work queued on the compute stream so far is done, runs
 * beside later kernels; gl_comm_wait() joins both streams */
int  gl_allgather_device_async(gl_ctx* ctx, const void* d_send, void* d_recv, int64_t bytes);
int  gl_comm_wait(gl_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* GOLEFT_B200_H */
