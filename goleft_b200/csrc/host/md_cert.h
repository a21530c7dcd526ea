// md_cert.h — when the "%.2f" of a multidepth mean follows from exact integers.  Shared by the pass-2 certify kernel
// (multidepth.cu) and the host export gl_multidepth_certify (multidepth.cpp).
//
// The reference prints fmt.Sprintf("%.2f", v) with v = acc / float64(l) * 1000 and acc += float64(d) / 1000. over the n
// sufficient sites of the block in position order (multidepth/multidepth.go:268-283).  Every term is >= 0, so with
// u = 2^-53 the computed v = V (1 + θ), |θ| <= γ_{n+2} = (n+2) u / (1 - (n+2) u), V = Σd / l: n divisions and n-1 additions
// (the first adds to 0 exactly), one division by l and one product.  "%.2f" rounds 100 v to an integer (ties to even on the
// exact binary value).  When the exact E = 100 Σd / l is farther than γ_{n+2} E from every k + 1/2, 100 v lies on the same
// side of it, and the digits are round(E), computed here in integers.  Otherwise (exact ties included) the caller runs the
// literal chain.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define GL_MD_HD __host__ __device__ __forceinline__
#else
#define GL_MD_HD inline
#endif

namespace glmd {

// sum = Σd over the block's n sufficient sites (n >= 1), l = span of the block (1 <= l < 2^31).  Returns true and
// *q = round(100 Σd / l) (the printed value times 100) when certified.
GL_MD_HD bool certify(uint64_t sum, int64_t n, int64_t l, int64_t* q) {
    if (n < 1 || l < 1 || l >= (int64_t(1) << 31) || n > (int64_t(1) << 40) || sum >= (uint64_t(1) << 56)) return false;
    const uint64_t ul = (uint64_t)l;
    const uint64_t a = sum / ul, b = sum % ul;              // 100 sum = (100 a) l + 100 b
    const uint64_t qf = 100 * a + (100 * b) / ul;           // floor(E)
    const uint64_t r = (100 * b) % ul;                      // E = qf + r / l
    const uint64_t dist = r * 2 > ul ? r * 2 - ul : ul - r * 2;   // |2r - l| = 2 l * distance to qf + 1/2
    // certified iff |2r - l| > 2 l γ E = 2 γ (100 sum); γ_{K} <= K u (1 + 2^-10) for K = n + 2 <= 2^41 + 2.
    // In integers: |2r - l| * 2^53 * 1024 > 2 * 100 sum * K * 1025.
    const unsigned __int128 lhs = (unsigned __int128)dist << 63;
    const unsigned __int128 rhs = (unsigned __int128)(2 * 100) * sum * (uint64_t)(n + 2) * 1025u;
    if (!(lhs > rhs)) return false;
    *q = (int64_t)(qf + (r * 2 > ul ? 1 : 0));
    return true;
}

}  // namespace glmd
