// emdepth.cpp — the host-only parts of `goleft emdepth` (emdepth/emdepth.go):
//
//   gl_emdepth_cnvs     : the reference's Cache (Add, Clear, makecnvs; emdepth.go:330-398) over the cells the kernel made.  It
//                         is sequential along the rows and needs only each cell's byte: Same compares Log2FC classes, makecnvs
//                         keeps the rows whose Log2FC is outside (-0.5, 0.3) and takes their CN.  Every quirk is kept:
//                           - the first Add compares the row with itself;
//                           - Clear's gap p.Start - End < 30000 is uint32 arithmetic, so it wraps;
//                           - Clear's keys slice starts as len(map) zeros, so while the map is non-empty every Clear deletes
//                             sample 0's pending rows, emitted or not;
//                           - a sample whose makecnvs is nil stays in the map;
//                           - PSize = len(map) at the Clear.
//                         The driver (the reference has none) calls Clear(nil) at every chromosome change and at the end: a
//                         Position has no chromosome.  The reference walks a Go map inside Clear; here CNVs come in sample order.
//   gl_emdepth_sum_host : the kernel's bin sum on the host, to test the exactness certificate (em_core.h).
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../../include/goleft_b200.h"
#include "em_core.h"

extern "C" {

int gl_emdepth_cnvs(const uint8_t* cells, int64_t n, int32_t S, const int64_t* starts, const int64_t* ends, const int64_t* breaks,
                    int64_t n_breaks, int32_t* cnv_sample, int32_t* cnv_psize, int64_t* cnv_ptr, int64_t cap, int64_t* n_cnvs,
                    int64_t* rows, int64_t rows_cap, int64_t* n_rows) {
    if (n < 0 || S < 1 || n_breaks < 0 || !n_cnvs || !n_rows || (n > 0 && (!cells || !starts || !ends)) || (n_breaks > 0 && !breaks))
        return GL_EINVAL;
    for (int64_t r = 0; r < n; r++)
        if (starts[r] < 0 || starts[r] > UINT32_MAX || ends[r] < 0 || ends[r] > UINT32_MAX) return GL_EINVAL;
    for (int64_t b = 1; b < n_breaks; b++)
        if (breaks[b] < breaks[b - 1]) return GL_EINVAL;
    std::vector<std::vector<int64_t>> pend((size_t)S);          // c.cnvs: the rows pending for each sample in the map
    std::vector<uint8_t> in_map((size_t)S, 0);
    int64_t map_size = 0, last = -1, nc = 0, nr = 0;
    std::vector<int64_t> kept;
    auto cls = [&](int64_t r, int s) { return glem::cell_class(cells[r * S + s]); };
    auto clear = [&](uint32_t p_start) {                       // Clear(&Position{Start: p_start})
        if (map_size == 0) return;                             // keys is empty
        std::vector<int> del(1, 0);                            // keys := make([]int, len(c.cnvs)): zeros
        for (int s = 0; s < S; s++) {
            if (!in_map[(size_t)s]) continue;
            const std::vector<int64_t>& emd = pend[(size_t)s];
            if ((uint32_t)(p_start - (uint32_t)ends[emd.back()]) < 30000u) continue;
            kept.clear();
            for (int64_t r : emd)                              // makecnvs: rows with fc outside (-0.5, 0.3)
                if (cells[r * S + s] & glem::kOutside) kept.push_back(r);
            if (kept.empty()) continue;                        // nil: the sample stays in the map
            if (cnv_sample && nc < cap) {
                cnv_sample[nc] = s;
                cnv_psize[nc] = (int32_t)map_size;
                cnv_ptr[nc] = nr;
            }
            for (int64_t r : kept) {
                if (rows && nr < rows_cap) rows[nr] = r;
                nr++;
            }
            nc++;
            if (cnv_ptr && nc <= cap) cnv_ptr[nc] = nr;
            del.push_back(s);
        }
        for (int s : del)
            if (in_map[(size_t)s]) { in_map[(size_t)s] = 0; pend[(size_t)s].clear(); map_size--; }
    };
    auto clear_nil = [&]() {                                   // Clear(nil): the last position + 100000, in uint32
        if (last >= 0) clear((uint32_t)starts[last] + 100000u);
    };
    int64_t b = 0;
    if (cnv_ptr && cap > 0) cnv_ptr[0] = 0;
    for (int64_t r = 0; r < n; r++) {
        bool brk = false;
        while (b < n_breaks && breaks[b] <= r) brk |= breaks[b++] == r;
        if (brk) clear_nil();
        if (last < 0) last = r;                                // Add: the first row is compared with itself
        clear((uint32_t)starts[r]);
        for (int s = 0; s < S; s++) {                          // Same(last, r): non2 = both hi or both lo
            const int a = cls(last, s), c = cls(r, s);
            if (a == c && (a == glem::kLo || a == glem::kHi)) {
                if (!in_map[(size_t)s]) { in_map[(size_t)s] = 1; map_size++; }
                pend[(size_t)s].push_back(r);
            }
        }
        last = r;
    }
    clear_nil();
    *n_cnvs = nc;
    *n_rows = nr;
    if ((cnv_sample && nc > cap) || (rows && nr > rows_cap)) return GL_ERANGE;
    return GL_OK;
}

int gl_emdepth_sum_host(const float* v, int64_t n, double* sum, uint8_t* certified) {
    if (n < 0 || (n > 0 && !v) || !sum || !certified) return GL_EINVAL;
    double part[32] = {};
    int lo = INT32_MAX, hi = INT32_MIN;
    for (int64_t i = 0; i < n; i++) {
        part[i & 31] += (double)v[i];
        uint32_t bits;
        memcpy(&bits, &v[i], 4);
        int a, z;
        if (glem::f32_span(bits, a, z)) { lo = a < lo ? a : lo; hi = z > hi ? z : hi; }
    }
    for (int o = 16; o; o >>= 1) {                             // __shfl_xor_sync butterfly: lane i adds lane i ^ o
        double nxt[32];
        for (int i = 0; i < 32; i++) nxt[i] = part[i] + part[i ^ o];
        memcpy(part, nxt, sizeof part);
    }
    *sum = part[0];
    *certified = glem::sum_exact(lo, hi, n) ? 1 : 0;
    return GL_OK;
}

}  // extern "C"
