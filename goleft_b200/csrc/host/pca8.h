// pca8.h — the byte indexcov's PCA reads for one depth value (indexcov.go:688-699): clip at MaxCN = 8, then
// uint8(65535/MaxCN*dp + 0.5) in float32.  Go converts float -> uint8 by a truncating conversion to int32 and keeps the low
// byte, so depth 8 maps to 65535.5 -> 0xFF and depth 1.0 to 8192.375 -> 0x00.  Out-of-range or NaN products take amd64's
// 0x80000000 "integer indefinite", whose low byte is 0.  Shared by the CLI's matrix fill and gl_indexcov_pca8.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define GL_PCA8_HD __host__ __device__ __forceinline__
#else
#define GL_PCA8_HD inline
#endif

namespace glpca {

GL_PCA8_HD uint8_t pca8_byte(float dp) {
    if (dp > 8.0f) dp = 8.0f;                                   // MaxCN
#ifdef __CUDA_ARCH__
    const float v = __fadd_rn(__fmul_rn(8191.875f, dp), 0.5f); // 65535 / MaxCN is exactly 8191.875 in float32
#else
    volatile float p = 8191.875f * dp;                          // two float32 roundings, never one fused one
    const float v = p + 0.5f;
#endif
    if (!(v > -2147483648.0f && v < 2147483648.0f)) return 0;
    return (uint8_t)((int32_t)v & 0xFF);
}

}  // namespace glpca
