// em_core.h — constants and exact-arithmetic rules of `goleft emdepth` (emdepth/emdepth.go), shared by the kernel
// (emdepth.cu) and the host side (host/emdepth.cpp).  DESIGN §1.10.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define GL_EM_HD __host__ __device__ __forceinline__
#else
#define GL_EM_HD inline
#endif

namespace glem {

constexpr int kCN = 9;                 // lambda[0..8] (maxCN + 1)
constexpr int kMaxIter = 10;
constexpr int kMaxSamples = 65535;

// math.Pow(i/2, 1.1) for i = 0..8 as Go's pow.go computes it: Modf(1.1) gives yf = 1.1 - 1 = 0.10000000000000009, then
// Exp(yf * Log(x)) times Frexp(x)'s mantissa, scaled by Ldexp.  Evaluated with glibc's exp / log (a host test redoes it);
// Go's amd64 Exp / Log are assembly and may differ in the last bit (UNPINNED until the goldens print Go's own bits).
// [0] and [2] are never used (lambda[0] = 0.01 m, lambda[2] = m).
GL_EM_HD double pow_factor(int i) {
    switch (i) {
    case 1: return 0x1.ddb680117ab12p-2;
    case 2: return 1.0;
    case 3: return 0x1.8fe3cb5abf130p+0;
    case 4: return 0x1.125fbee250664p+1;
    case 5: return 0x1.5eb4e5dd2222bp+1;
    case 6: return 0x1.ac975f5c2ccd2p+1;
    case 7: return 0x1.fbca711ef58a2p+1;
    case 8: return 0x1.2611186bae675p+2;
    default: return 0.0;
    }
}

// One cell byte: bits 0-3 the CN (0..9), bits 4-5 the Same class of Log2FC (kMid: -0.8 < fc < 0.4, kLo: fc <= -0.8,
// kHi: fc >= 0.4, kNaN: fc is NaN, which every comparison rejects), bit 6 set when fc is outside (-0.5, 0.3) (makecnvs
// keeps the row for that sample).
enum : uint8_t { kMid = 0, kLo = 1, kHi = 2, kNaN = 3 };
constexpr uint8_t kOutside = 0x40;
GL_EM_HD uint8_t cell(int cn, int cls, bool outside) { return (uint8_t)(cn | (cls << 4) | (outside ? kOutside : 0)); }
GL_EM_HD int cell_cn(uint8_t c) { return c & 15; }
GL_EM_HD int cell_class(uint8_t c) { return (c >> 4) & 3; }

// The bits a positive float32 occupies: v = m 2^lo with m odd, v < 2^hi.  Zero occupies none (lo = hi = 0, returns false).
GL_EM_HD bool f32_span(uint32_t bits, int& lo, int& hi) {
    const uint32_t e = (bits >> 23) & 0xffu, m = bits & 0x7fffffu;
    if (e == 0 && m == 0) { lo = hi = 0; return false; }
    const uint32_t sig = e ? (m | 0x800000u) : m;
    const int base = e ? (int)e - 150 : -149;
#ifdef __CUDA_ARCH__
    const int tz = __ffs((int)sig) - 1, top = 32 - __clz((int)sig);
#else
    const int tz = __builtin_ctz(sig), top = 32 - __builtin_clz(sig);
#endif
    lo = base + tz;
    hi = base + top;
    return true;
}

// A float64 sum of cnt non-negative float32 values whose non-zero bits lie in [lo, hi) is exact in any order (every
// partial sum is a multiple of 2^lo below 2^(hi + ceil(log2 cnt))) when that range is at most 53 bits wide.  Then the
// reference's sequential mean64 and any tree sum agree bit for bit.
GL_EM_HD bool sum_exact(int lo, int hi, int64_t cnt) {
    if (cnt <= 1 || hi <= lo) return true;             // no non-zero value, or one term
    int lg = 0;
    while ((int64_t(1) << lg) < cnt) lg++;
    return hi - lo + lg <= 53;
}

}  // namespace glem
