// f2_token.h — the bytes of printf("%.2f", v) for one float64, exactly: 100 v is rounded to an integer in integer arithmetic
// on the binary value, ties to even, which is what glibc's printf and Go's strconv both do.  Shared by fmt_f2_kernel
// (dcnv.cu) and the host mirror gl_format_f2_host (dcnv.cpp).
//
// A token is 16 bytes: the text, NUL-padded.  An empty token (byte 0 is NUL) means the text would not fit in 16 bytes
// (|v| near or above 1e12) and the caller formats that value itself.  Non-finite values are spelled as Go's fmt spells
// them ("NaN", "+Inf", "-Inf"): the reference is a Go program.
#pragma once
#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define GL_F2_HD __host__ __device__ __forceinline__
#else
#define GL_F2_HD inline
#endif

namespace glf2 {

constexpr int kTok = 16;

// t[0..16) = the token of v; returns the text length (0: formatted by the caller)
GL_F2_HD int token(double v, unsigned char* t) {
    for (int k = 0; k < kTok; k++) t[k] = 0;
    uint64_t bits;
    memcpy(&bits, &v, 8);
    const bool neg = bits >> 63;
    const int ex = (int)((bits >> 52) & 0x7ff);
    const uint64_t frac = bits & ((uint64_t(1) << 52) - 1);
    int len = 0;
    if (ex == 0x7ff) {
        if (frac) { t[0] = 'N'; t[1] = 'a'; t[2] = 'N'; return 3; }
        t[0] = neg ? '-' : '+'; t[1] = 'I'; t[2] = 'n'; t[3] = 'f';
        return 4;
    }
    if (ex >= 1023 + 47) return 0;                              // |v| >= 2^47 > 1e14: more than 16 bytes of text
    const uint64_t m = ex ? (frac | (uint64_t(1) << 52)) : frac;
    const int e2 = ex ? ex - 1075 : -1074;                      // |v| = m 2^e2
    uint64_t N;                                                 // round(100 |v|), ties to even
    if (e2 >= 0) {
        N = (m << e2) * 100;                                    // < 2^47 * 100
    } else {
        const int sh = -e2;
        const uint64_t num = m * 100;                           // < 2^60
        if (sh >= 61) {
            N = 0;                                              // num < 2^60 <= 2^(sh-1): below one half
        } else {
            const uint64_t q = num >> sh, r = num & ((uint64_t(1) << sh) - 1), half = uint64_t(1) << (sh - 1);
            N = q + ((r > half || (r == half && (q & 1))) ? 1 : 0);
        }
    }
    const uint64_t ip = N / 100;
    const unsigned fp = (unsigned)(N % 100);
    char dig[20];
    int nd = 0;
    uint64_t x = ip;
    do { dig[nd++] = (char)('0' + x % 10); x /= 10; } while (x);
    if ((neg ? 1 : 0) + nd + 3 > kTok) return 0;
    if (neg) t[len++] = '-';
    while (nd) t[len++] = (unsigned char)dig[--nd];
    t[len++] = '.';
    t[len++] = (unsigned char)('0' + fp / 10);
    t[len++] = (unsigned char)('0' + fp % 10);
    return len;
}

}  // namespace glf2
