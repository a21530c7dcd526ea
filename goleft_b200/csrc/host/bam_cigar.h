// bam_cigar.h — which CIGAR a BAM record has.  Shared by the three CIGAR walkers: bam_parse_kernel (bamgpu.cu),
// Emitter::record (bam_feed.cpp) and seg_record (hts_io.cpp).
//
// BAM keeps n_cigar_op in 16 bits.  A record with more operations stores the placeholder `kSmN` (k = l_seq, m = the
// reference span) and the real CIGAR in the CG:B,I tag (SAMv1 §4.2.2).  htslib's bam_read1 swaps it back in
// (bam_tag2cigar), so `samtools depth` counts the real M/=/X blocks; this function makes the same decision:
//   tid >= 0 and pos >= 0, the first stored op is S of length l_seq, the first CG tag has type B with subtype I or i,
//   and its count is at least n_cigar_op (and below 2^29, as htslib).  Otherwise the stored CIGAR is the CIGAR.
// Every aux field is walked with bounds checks against block_size: malformed aux data means "the stored CIGAR".
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define GL_BAM_HD __host__ __device__ __forceinline__
#else
#define GL_BAM_HD inline
#endif

namespace glbam {

GL_BAM_HD uint32_t ld_u32(const uint8_t* p) {
    return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// r: the record after its block_size field (refID at r[0]); bs: block_size.  The caller has checked
// 32 + l_read_name + 4 * n_cigar_op <= bs.  Out: the CIGAR to walk (4-byte ops, not necessarily aligned) and its length.
GL_BAM_HD void record_cigar(const uint8_t* r, uint32_t bs, const uint8_t** cig, uint32_t* n_cig) {
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

}  // namespace glbam
