// bam_cigar.h — what `samtools depth` counts from a BAM record, for the three record walkers: bam_parse_kernel
// (bamgpu.cu), Emitter::record and bam_decode_segments (bam_feed.cpp).  depth_counts is the filter, depth_blocks the
// CIGAR walk; record_cigar picks the CIGAR that walk reads.
//
// BAM keeps n_cigar_op in 16 bits.  A record with more operations stores the placeholder `kSmN` (k = l_seq, m = the
// reference span) and the real CIGAR in the CG:B,I tag (SAMv1 §4.2.2).  htslib's bam_read1 swaps it back in
// (bam_tag2cigar), so `samtools depth` counts the real M/=/X blocks; record_cigar makes the same decision:
//   tid >= 0 and pos >= 0, the first stored op is S of length l_seq, the first CG tag has type B with subtype I or i,
//   and its count is at least n_cigar_op (and below 2^29, as htslib).  Otherwise the stored CIGAR is the CIGAR.
// Every aux field is walked with bounds checks against block_size: malformed aux data means "the stored CIGAR".
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define GL_BAM_HD __host__ __device__ __forceinline__
#define GL_BAM_COLD __host__ __device__ inline __noinline__
#else
#define GL_BAM_HD inline
#define GL_BAM_COLD inline
#endif

namespace glbam {

GL_BAM_HD uint32_t ld_u32(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// r: the record after its block_size field (refID at r[0]); bs: block_size.  The caller has checked
// 32 + l_read_name + 4 * n_cigar_op <= bs.  Out: the CIGAR to walk (4-byte ops, not necessarily aligned) and its length.
// Out of line on the device: only records that may hold the placeholder reach it (depth_blocks), and the aux walk inlined
// into the parse kernel would cost every record registers.
GL_BAM_COLD void record_cigar(const uint8_t* r, uint32_t bs, const uint8_t** cig, uint32_t* n_cig) {
    const uint32_t l_name = r[8], n_stored = (uint32_t)r[12] | ((uint32_t)r[13] << 8);
    const uint8_t* stored = r + 32 + l_name;
    *cig = stored;
    *n_cig = n_stored;
    if (n_stored == 0 || (stored[0] & 15u) != 4u) return;                  // the one compare every ordinary record pays
    const uint32_t l_seq = ld_u32(r + 16);
    if ((ld_u32(stored) >> 4) != l_seq) return;
    if ((int32_t)ld_u32(r) < 0 || (int32_t)ld_u32(r + 4) < 0) return;
    const uint64_t end = bs;
    uint64_t o = 32ull + l_name + 4ull * n_stored + (((uint64_t)l_seq + 1) >> 1) + l_seq;
    while (o + 3 <= end) {
        const uint8_t t0 = r[o], t1 = r[o + 1], type = r[o + 2];
        o += 3;
        uint64_t sz;
        switch (type) {
            case 'A': case 'c': case 'C': sz = 1; break;
            case 's': case 'S': sz = 2; break;
            case 'i': case 'I': case 'f': sz = 4; break;
            case 'Z': case 'H': {
                while (o < end && r[o] != 0) o++;
                if (o >= end) return;                                          // unterminated string
                sz = 1;
                break;
            }
            case 'B': {
                if (o + 5 > end) return;
                const uint8_t sub = r[o];
                const uint32_t cnt = ld_u32(r + o + 1);
                uint64_t el;
                switch (sub) {
                    case 'c': case 'C': el = 1; break;
                    case 's': case 'S': el = 2; break;
                    case 'i': case 'I': case 'f': el = 4; break;
                    default: return;                                           // malformed
                }
                if (o + 5 + el * cnt > end) return;
                if (t0 == 'C' && t1 == 'G') {
                    if ((sub == 'I' || sub == 'i') && cnt >= n_stored && cnt < (1u << 29)) { *cig = r + o + 5; *n_cig = cnt; }
                    return;                                                    // the first CG tag decides
                }
                sz = 5 + el * cnt;
                break;
            }
            default: return;                                                   // malformed
        }
        if (t0 == 'C' && t1 == 'G') return;                                    // a CG tag that is not an array
        o += sz;
    }
}

// The `samtools depth` filter (depth.go:45: its defaults + -Q): (flag & 0x704) == 0, MAPQ >= min_mapq, and the stored
// CIGAR lies inside the record (32 + l_read_name + 4 * n_cigar_op <= bs).  r, bs as for record_cigar.
GL_BAM_HD bool depth_counts(const uint8_t* r, uint32_t bs, int min_mapq) {
    const uint32_t l_name = r[8], mapq = r[9], n_cig = (uint32_t)r[12] | ((uint32_t)r[13] << 8), flag = (uint32_t)r[14] | ((uint32_t)r[15] << 8);
    if ((flag & 0x704u) != 0 || (int)mapq < min_mapq) return false;            // two tests, not one chain: the device
    return 32u + l_name + 4u * n_cig <= bs;                                    // parse is 2.5 % slower with the chain
}

// emit(b, e) for each M/=/X block [b, e) of a record that depth_counts, in CIGAR order: blocks separated only by I/S/H/P
// merge, D and N advance without counting, empty blocks are dropped.  The CIGAR is record_cigar's, asked only when the
// first stored op is S of length l_seq (the placeholder's shape), so every other record walks its stored CIGAR directly.
template <class Emit>
GL_BAM_HD void depth_blocks(const uint8_t* r, uint32_t bs, Emit&& emit) {
    const uint8_t* cg = r + 32 + r[8];
    uint32_t n_op = (uint32_t)r[12] | ((uint32_t)r[13] << 8);
    int32_t ref = (int32_t)ld_u32(r + 4), b0 = 0, b1 = 0;
    bool open = false, checked = false;
    for (uint32_t k = 0; k < n_op; k++) {
        const uint32_t v = ld_u32(cg + 4 * k), op = v & 15u;
        const int32_t len = (int32_t)(v >> 4);
        if (op == 0 || op == 7 || op == 8) {                                   // M = X count
            if (len == 0) continue;
            if (open && b1 == ref) b1 = ref + len;
            else {
                if (open && b1 > b0) emit(b0, b1);
                b0 = ref; b1 = ref + len; open = true;
            }
            ref += len;
        } else if (op == 2 || op == 3) {                                       // D N advance without counting
            ref += len;
        } else if (op == 4 && k == 0 && !checked && v == ((ld_u32(r + 16) << 4) | 4u)) {
            checked = true;                                                    // maybe the CG placeholder: walk what
            record_cigar(r, bs, &cg, &n_op);                                   // record_cigar picks from its first op
            k = ~0u;
        }                                                                      // I S H P: no reference movement
    }
    if (open && b1 > b0) emit(b0, b1);
}

}  // namespace glbam
