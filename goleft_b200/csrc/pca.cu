// pca.cu — the PC1..PC5 columns of `goleft indexcov`'s .ped (indexcov.go:773-807): gonum's stat.PC of the S x D byte
// matrix (one row per sample, host/pca8.h), projected as proj = X V[:, :k] with the uncentred X.  DESIGN §1.11.
//
// Everything the projections need is in the exact integer Gram G = X X^T (S x S).  With r = G 1, q = 1^T r, n = S:
//   n^2 Gc = n^2 G - n (r_i + r_j) + q            (Gc = Xc Xc^T, exactly, in __int128; one rounding to double, one division)
//   proj(i, k) = sigma_k u(i, k) + (c . u_k) / sigma_k,   c = r / n - q / n^2,   (sigma_k^2, u_k) = eigenpairs of Gc
// so the only D-sized pass is the Gram, and everything after it is S x S:
//   gram_kernel     u8 x u8 -> s32 tensor-core MMA (mma.sync m16n8k32), 128 x 128 tiles I <= J only, split-K: each CTA sums
//                   at most 32768 columns (32768 * 255^2 < 2^31, so s32 cannot overflow) and adds its tile into the int64
//                   Gram with integer atomics, which are exact, so the result does not depend on order or on the SM count.
//   centre_kernel   mirrors the upper triangle, forms Gc in place over the Gram (int64 -> double).
//   house/symv/rank2_kernel  Householder tridiagonalisation of Gc (Golub & Van Loan 8.3.1; sym_tridiag, shared with dcnv_svd.cu), one reflector per step; every
//                   reduction has a fixed order (lane-strided partial sums, then a fixed shuffle tree).
// The top k eigenvalues (Sturm bisection), their vectors (inverse iteration) and the back-transformation through the
// reflectors run on the host (host/pca_eig.cpp), on O(S k) and O(S^2 k) data.
#include <float.h>
#include <chrono>
#include "gl_common.cuh"
#include "host/pca8.h"
#include "host/pca_eig.h"
#include "sym_eig.cuh"

namespace {

constexpr int kBM = 128;                       // Gram tile (rows and columns)
constexpr int kBK = 64;                        // bytes of K per pipeline stage
constexpr int kStages = 4;
constexpr int kThreads = 256;                  // 8 warps: 2 (rows) x 4 (columns), 64 x 32 outputs each
constexpr int kTileBytes = kBM * kBK;
constexpr int kSmem = kStages * 2 * kTileBytes;   // 64 KB
constexpr int64_t kKMax = 32768;               // columns per CTA: 32768 * 65025 < 2^31
constexpr unsigned kFull = 0xffffffffu;

// 16-byte chunk c (0..3) of tile row r: XOR-swizzled so that ldmatrix's 8 rows of one chunk hit 8 distinct bank groups
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)(r * kBK + ((c ^ ((r >> 1) & 3)) << 4)); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, int bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(bytes));
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}

__device__ __forceinline__ void mma_u8(int (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// one CTA: the 128 x 128 tile (I, J), I <= J (blockIdx.x enumerates the upper triangle row by row), columns
// [blockIdx.y * kc, min(D, (blockIdx.y + 1) * kc)) of X (row stride ld, 16-byte aligned); adds into G (S x S, zeroed)
__global__ void __launch_bounds__(kThreads, 1) gram_kernel(const uint8_t* __restrict__ x, long long ld, int S, long long D,
                                                           int T, long long kc, unsigned long long* __restrict__ G) {
    extern __shared__ __align__(128) uint8_t smem[];
    int t = blockIdx.x, I = 0;
    while (t >= T - I) { t -= T - I; I++; }
    const int J = I + t;
    const long long k0 = (long long)blockIdx.y * kc, k1 = min(D, k0 + kc);
    const int nk = (int)((k1 - k0 + kBK - 1) / kBK);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wm = warp >> 2, wn = warp & 3;
    const uint32_t s0 = (uint32_t)__cvta_generic_to_shared(smem);

    auto load = [&](int stage, int kb) {
        const uint32_t sa = s0 + stage * 2 * kTileBytes, sb = sa + kTileBytes;
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int ci = tid + h * kThreads, r = ci >> 2, c = ci & 3;
            const long long col = k0 + (long long)kb * kBK + c * 16;
            const int cb = (int)max(0LL, min(16LL, k1 - col));
            const int ra = I * kBM + r, rb = J * kBM + r;
            const int na = ra < S ? cb : 0, nb = rb < S ? cb : 0;
            cp_async16(sa + swz(r, c), na ? x + (long long)ra * ld + col : x, na);
            cp_async16(sb + swz(r, c), nb ? x + (long long)rb * ld + col : x, nb);
        }
    };

    int acc[4][4][4];
#pragma unroll
    for (int a = 0; a < 4; a++)
#pragma unroll
        for (int b = 0; b < 4; b++)
#pragma unroll
            for (int c = 0; c < 4; c++) acc[a][b][c] = 0;

#pragma unroll
    for (int s = 0; s < kStages - 1; s++) {
        if (s < nk) load(s, s);
        asm volatile("cp.async.commit_group;\n" ::);
    }
    for (int kb = 0; kb < nk; kb++) {
        asm volatile("cp.async.wait_group %0;\n" ::"n"(kStages - 2));
        __syncthreads();
        const int nxt = kb + kStages - 1;
        if (nxt < nk) load(nxt % kStages, nxt);
        asm volatile("cp.async.commit_group;\n" ::);
        const uint32_t sa = s0 + (kb % kStages) * 2 * kTileBytes, sb = sa + kTileBytes;
#pragma unroll
        for (int ks = 0; ks < 2; ks++) {
            uint32_t af[4][4], bf[4][2];
#pragma unroll
            for (int mi = 0; mi < 4; mi++) {
                const int r = wm * 64 + mi * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, c = ks * 2 + (lane >> 4);
                ldsm_x4(sa + swz(r, c), af[mi][0], af[mi][1], af[mi][2], af[mi][3]);
            }
#pragma unroll
            for (int p = 0; p < 2; p++) {
                const int r = wn * 32 + p * 16 + (lane & 7) + ((lane >> 4) & 1) * 8, c = ks * 2 + ((lane >> 3) & 1);
                ldsm_x4(sb + swz(r, c), bf[2 * p][0], bf[2 * p][1], bf[2 * p + 1][0], bf[2 * p + 1][1]);
            }
#pragma unroll
            for (int mi = 0; mi < 4; mi++)
#pragma unroll
                for (int nj = 0; nj < 4; nj++) mma_u8(acc[mi][nj], af[mi], bf[nj][0], bf[nj][1]);
        }
    }
    asm volatile("cp.async.wait_group 0;\n" ::);
    const int g = lane >> 2, tq = lane & 3;
#pragma unroll
    for (int mi = 0; mi < 4; mi++)
#pragma unroll
        for (int nj = 0; nj < 4; nj++)
#pragma unroll
            for (int h = 0; h < 4; h++) {
                const int row = I * kBM + wm * 64 + mi * 16 + g + (h >> 1) * 8, col = J * kBM + wn * 32 + nj * 8 + tq * 2 + (h & 1);
                if (row < S && col < S && acc[mi][nj][h])
                    atomicAdd(&G[(long long)row * S + col], (unsigned long long)(unsigned)acc[mi][nj][h]);
            }
}

// r_i = sum_j G(i, j) over the upper triangle's mirror: G(i, j) = G(min, max); one warp per row
__global__ void rowsum_kernel(const long long* __restrict__ G, int S, long long* __restrict__ r) {
    const int lane = threadIdx.x & 31;
    const int i = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (i >= S) return;
    long long s = 0;
    for (int j = lane; j < S; j += 32) s += j >= i ? G[(long long)i * S + j] : G[(long long)j * S + i];
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(kFull, s, o);
    if (lane == 0) r[i] = s;
}

// the double nearest v (one rounding)
__host__ __device__ __forceinline__ double i128_to_double(__int128 v) {
    const bool neg = v < 0;
    const unsigned __int128 m = neg ? (unsigned __int128)0 - (unsigned __int128)v : (unsigned __int128)v;
    const uint64_t hi = (uint64_t)(m >> 64), lo = (uint64_t)m;
    double d;
    if (hi == 0) {
        d = (double)lo;
    } else {
#ifdef __CUDA_ARCH__
        const int lz = __clzll((long long)hi);
#else
        const int lz = __builtin_clzll(hi);
#endif
        const int sh = 64 - lz;                                          // 1..64
        const uint64_t mask = sh == 64 ? ~0ull : (1ull << sh) - 1;
        const uint64_t top = (uint64_t)(m >> sh) | ((lo & mask) != 0);   // 64 bits + sticky: rounds as the full value does
        d = ldexp((double)top, sh);
    }
    return neg ? -d : d;
}

// Gc(i, j) = (n^2 G(i, j) - n (r_i + r_j) + q) / n^2 over the whole matrix, in place over the Gram, whose upper triangle
// holds the sums: pass 0 writes the strict lower triangle from the mirrored upper entries, pass 1 then converts the upper
// triangle and the diagonal where they stand.
__global__ void centre_kernel(long long* __restrict__ G, int S, const long long* __restrict__ r, long long q_hi,
                              unsigned long long q_lo, int pass) {
    const long long n2 = (long long)S * S;
    const __int128 q = ((__int128)q_hi << 64) | (__int128)q_lo;
    const double dn2 = (double)n2;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < n2; t += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(t / S), j = (int)(t % S);
        if ((pass == 0) != (i > j)) continue;
        const long long g = pass == 0 ? G[(long long)j * S + i] : G[t];
        const __int128 num = (__int128)n2 * g - (__int128)S * ((__int128)r[i] + r[j]) + q;
        reinterpret_cast<double*>(G)[t] = i128_to_double(num) / dn2;
    }
}

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    return v;
}

// fixed-order sum over a 256-thread block; every thread gets the result
__device__ __forceinline__ double block_sum(double v, double* sh) {
    v = warp_sum(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double s = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) s += sh[w];
    return s;
}

// step j: the reflector H = I - tau v v^T that zeroes A(j, j+2..) (rows are columns: A stays exactly symmetric).  v (v_0 = 1)
// replaces x = A(j, j+1..); d[j] = A(j, j), e[j] = beta, tau[j]
__global__ void __launch_bounds__(256) house_kernel(double* __restrict__ A, int n, int j, double* __restrict__ dg,
                                                    double* __restrict__ ed, double* __restrict__ tau) {
    __shared__ double sh[8];
    __shared__ double scale;
    double* x = A + (long long)j * n + j + 1;
    const int m = n - j - 1;
    double s = 0;
    for (int i = 1 + threadIdx.x; i < m; i += 256) s += x[i] * x[i];
    const double xn2 = block_sum(s, sh);
    const double alpha = x[0];
    if (threadIdx.x == 0) {
        double beta = alpha, t = 0, sc = 0;
        if (xn2 != 0) {
            beta = -copysign(sqrt(alpha * alpha + xn2), alpha);
            t = (beta - alpha) / beta;
            sc = alpha - beta;
        }
        dg[j] = A[(long long)j * n + j];
        ed[j] = beta;
        tau[j] = t;
        scale = sc;
    }
    __syncthreads();
    const double sc = scale;
    for (int i = threadIdx.x; i < m; i += 256) x[i] = i == 0 ? 1.0 : (sc != 0 ? x[i] / sc : 0.0);
}

// p = tau A22 v, one warp per row of the trailing matrix A22 = A(j+1.., j+1..)
__global__ void __launch_bounds__(256) symv_kernel(const double* __restrict__ A, int n, int j, const double* __restrict__ tau,
                                                   double* __restrict__ p) {
    const int m = n - j - 1, lane = threadIdx.x & 31;
    const int i = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (i >= m) return;
    const double t = tau[j];
    const double* v = A + (long long)j * n + j + 1;
    const double* row = A + (long long)(j + 1 + i) * n + j + 1;
    double s = 0;
    if (t != 0)
        for (int l = lane; l < m; l += 32) s += row[l] * v[l];
    s = warp_sum(s);
    if (lane == 0) p[i] = t * s;
}

constexpr int kRank2Rows = 8;

// A22 -= v w^T + w v^T, w = p - (tau/2)(p . v) v; every CTA forms p . v itself, in the same order
__global__ void __launch_bounds__(256) rank2_kernel(double* __restrict__ A, int n, int j, const double* __restrict__ tau,
                                                    const double* __restrict__ p) {
    __shared__ double sh[8];
    const int m = n - j - 1;
    const double t = tau[j];
    if (t == 0) return;
    const double* v = A + (long long)j * n + j + 1;
    double s = 0;
    for (int l = threadIdx.x; l < m; l += 256) s += p[l] * v[l];
    const double K = 0.5 * t * block_sum(s, sh);
    const int i0 = blockIdx.x * kRank2Rows, i1 = min(m, i0 + kRank2Rows);
    for (int i = i0; i < i1; i++) {
        const double vi = v[i], wi = p[i] - K * vi;
        double* row = A + (long long)(j + 1 + i) * n + j + 1;
        for (int l = threadIdx.x; l < m; l += 256) {
            const double vl = v[l], wl = p[l] - K * vl;
            row[l] -= vi * wl + wi * vl;
        }
    }
}

int check_shape(gl_ctx* ctx, const char* fn, int64_t ld, int32_t S, int64_t D, int32_t k, const void* x, const void* proj,
                const void* sv, const void* k_out) {
    if (S < 1 || D < 1 || ld < D || k < 1 || !x || !proj || !sv || !k_out)
        return gl_fail(ctx, GL_EINVAL, "%s: bad argument (S = %d, D = %lld, ld = %lld, k = %d)", fn, S, (long long)D, (long long)ld, k);
    if (S > 65535) return gl_fail(ctx, GL_EINVAL, "%s: %d samples; at most 65535", fn, S);
    if (D > 65535 * kKMax) return gl_fail(ctx, GL_EINVAL, "%s: %lld columns; at most %lld", fn, (long long)D, (long long)(65535 * kKMax));
    return GL_OK;
}

}  // namespace

int sym_tridiag(gl_ctx* ctx, double* A, int S, SymTridiag& t) {
    gl_scratch tmp(ctx);
    double *d_d, *d_e, *d_tau, *d_p;
    GL_CHECK(tmp.alloc(d_d, (size_t)S));
    GL_CHECK(tmp.alloc(d_e, (size_t)S));
    GL_CHECK(tmp.alloc(d_tau, (size_t)S));
    GL_CHECK(tmp.alloc(d_p, (size_t)S));
    for (int j = 0; j + 2 < S; j++) {                              // Householder tridiagonalisation
        const int m = S - j - 1;
        house_kernel<<<1, 256, 0, ctx->stream>>>(A, S, j, d_d, d_e, d_tau);
        symv_kernel<<<(m + 7) / 8, 256, 0, ctx->stream>>>(A, S, j, d_tau, d_p);
        rank2_kernel<<<(m + kRank2Rows - 1) / kRank2Rows, 256, 0, ctx->stream>>>(A, S, j, d_tau, d_p);
        GL_LAUNCHED(ctx, 3);
    }
    const size_t n2 = (size_t)S * S;
    t.n = S;
    t.hA.assign(n2, 0.0);
    t.d.assign((size_t)S, 0.0);
    t.e.assign((size_t)S, 0.0);
    t.tau.assign((size_t)S, 0.0);
    GL_CUDA(ctx, cudaMemcpyAsync(t.hA.data(), A, n2 * 8, cudaMemcpyDeviceToHost, ctx->stream));
    if (S > 2) {
        GL_CUDA(ctx, cudaMemcpyAsync(t.d.data(), d_d, (size_t)(S - 2) * 8, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaMemcpyAsync(t.e.data(), d_e, (size_t)(S - 2) * 8, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaMemcpyAsync(t.tau.data(), d_tau, (size_t)(S - 2) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    }
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int i = std::max(0, S - 2); i < S; i++) t.d[(size_t)i] = t.hA[(size_t)i * S + i];
    if (S >= 2) t.e[(size_t)S - 2] = t.hA[(size_t)(S - 1) * S + (S - 2)];
    return GL_OK;
}

void SymTridiag::back_transform(double* u, int k) const {
    const int S = n;
    for (int jv = 0; jv < k; jv++) {                               // u = H_0 H_1 ... H_{S-3} z
        double* y = &u[(size_t)jv * S];
        for (int j = S - 3; j >= 0; j--) {
            const double t = tau[(size_t)j];
            if (t == 0) continue;
            const double* v = &hA[(size_t)j * S + j + 1];
            double s = 0;
            for (int i = 0; i < S - j - 1; i++) s += v[i] * y[j + 1 + i];
            s *= t;
            for (int i = 0; i < S - j - 1; i++) y[j + 1 + i] -= s * v[i];
        }
    }
}

namespace {

// the whole computation on the byte matrix d_x (row stride ld, 16-byte aligned) already on the device
int pca_run(gl_ctx* ctx, const uint8_t* d_x, int64_t ld, int32_t S, int64_t D, int32_t k, double* proj, double* sv,
            int32_t* k_out, int64_t* gram, double t_upload) {
    const int kk = (int)std::min<int64_t>({(int64_t)k, (int64_t)S, D});
    const size_t n2 = (size_t)S * S;
    size_t free_b = 0, total_b = 0;
    GL_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
    if (n2 * 8 + (size_t)S * 40 + (1 << 20) > free_b)
        return gl_fail(ctx, GL_ENOMEM, "gl_indexcov_pca: the %d x %d Gram does not fit in free device memory", S, S);
    const auto now = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    double t0 = now();
    gl_scratch tmp(ctx);
    unsigned long long* d_G;
    long long* d_r;
    GL_CHECK(tmp.alloc(d_G, n2));
    GL_CHECK(tmp.alloc(d_r, (size_t)S));
    GL_CUDA(ctx, cudaMemsetAsync(d_G, 0, n2 * 8, ctx->stream));
    const int T = (S + kBM - 1) / kBM, tiles = T * (T + 1) / 2;
    const int64_t want = std::max<int64_t>(1, (2 * (int64_t)ctx->sm_count + tiles - 1) / tiles);
    int64_t kc = ((D + want - 1) / want + kBK - 1) / kBK * kBK;
    kc = std::min<int64_t>(kKMax, std::max<int64_t>(kc, 1024));
    const int64_t splits = (D + kc - 1) / kc;
    GL_CUDA(ctx, cudaFuncSetAttribute(gram_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    {
        gl_prof_scope prof(ctx, "gram_kernel");
        gram_kernel<<<dim3((unsigned)tiles, (unsigned)splits), kThreads, kSmem, ctx->stream>>>(d_x, (long long)ld, S, (long long)D, T,
                                                                                            (long long)kc, d_G);
    }
    GL_LAUNCHED(ctx, 1);
    if (gram) {
        GL_CUDA(ctx, cudaMemcpyAsync(gram, d_G, n2 * 8, cudaMemcpyDeviceToHost, ctx->stream));
        GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        for (int i = 0; i < S; i++)
            for (int j = 0; j < i; j++) gram[(size_t)i * S + j] = gram[(size_t)j * S + i];
    }
    rowsum_kernel<<<(S + 7) / 8, 256, 0, ctx->stream>>>((const long long*)d_G, S, d_r);
    GL_LAUNCHED(ctx, 1);
    std::vector<long long> r((size_t)S);
    GL_CUDA(ctx, cudaMemcpyAsync(r.data(), d_r, (size_t)S * 8, cudaMemcpyDeviceToHost, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    __int128 q = 0;
    for (int i = 0; i < S; i++) q += r[(size_t)i];
    std::vector<double> c((size_t)S);                               // c_i = (n r_i - q) / n^2
    for (int i = 0; i < S; i++) c[(size_t)i] = i128_to_double((__int128)S * r[(size_t)i] - q) / ((double)S * S);
    const unsigned cb = (unsigned)std::min<size_t>((n2 + 255) / 256, (size_t)ctx->sm_count * 16);
    for (int pass = 0; pass < 2; pass++) {
        centre_kernel<<<cb, 256, 0, ctx->stream>>>((long long*)d_G, S, d_r, (long long)(q >> 64), (unsigned long long)q, pass);
        GL_LAUNCHED(ctx, 1);
    }
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const double t_gram = now() - t0;
    t0 = now();
    SymTridiag tri;
    GL_CHECK(sym_tridiag(ctx, reinterpret_cast<double*>(d_G), S, tri));
    std::vector<double> lam((size_t)kk), u((size_t)kk * S);
    glpca::tridiag_top_values(tri.d.data(), tri.e.data(), S, kk, lam.data());
    glpca::tridiag_vectors(tri.d.data(), tri.e.data(), S, lam.data(), kk, u.data());
    tri.back_transform(u.data(), kk);
    std::vector<double> pj((size_t)S * kk);
    glpca::project(lam.data(), u.data(), c.data(), S, kk, pj.data(), sv);
    for (int i = 0; i < S; i++)
        for (int j = 0; j < k; j++) proj[(size_t)i * k + j] = j < kk ? pj[(size_t)i * kk + j] : 0.0;
    for (int j = kk; j < k; j++) sv[j] = 0.0;
    *k_out = kk;
    ctx->pca_phase[0] = t_upload;
    ctx->pca_phase[1] = t_gram;
    ctx->pca_phase[2] = now() - t0;
    return GL_OK;
}

}  // namespace

extern "C" {

int gl_indexcov_pca8(const float* d, int64_t n, uint8_t* out) {
    if (n < 0 || (n > 0 && (!d || !out))) return GL_EINVAL;
    for (int64_t i = 0; i < n; i++) out[i] = glpca::pca8_byte(d[i]);
    return GL_OK;
}

int gl_indexcov_pca_device(gl_ctx* ctx, const uint8_t* d_x, int64_t ld, int32_t S, int64_t D, int32_t k, double* proj, double* sv,
                           int32_t* k_out, int64_t* gram) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(check_shape(ctx, "gl_indexcov_pca_device", ld, S, D, k, d_x, proj, sv, k_out));
    if ((ld & 15) || ((uintptr_t)d_x & 15))
        return gl_fail(ctx, GL_EINVAL, "gl_indexcov_pca_device: the matrix and its row stride (%lld) must be 16-byte aligned", (long long)ld);
    return pca_run(ctx, d_x, ld, S, D, k, proj, sv, k_out, gram, 0.0);
}

int gl_indexcov_pca(gl_ctx* ctx, const uint8_t* x, int64_t ld, int32_t S, int64_t D, int32_t k, double* proj, double* sv,
                    int32_t* k_out, int64_t* gram) {
    GL_CHECK(gl_use(ctx));
    GL_CHECK(check_shape(ctx, "gl_indexcov_pca", ld, S, D, k, x, proj, sv, k_out));
    const int64_t ldp = (D + 63) / 64 * 64;
    size_t free_b = 0, total_b = 0;
    GL_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
    if ((double)S * ldp + 8.0 * S * S + 40.0 * S + (1 << 20) > (double)free_b)
        return gl_fail(ctx, GL_ENOMEM, "gl_indexcov_pca: %d x %lld bytes and the %d x %d Gram do not fit in free device memory", S,
                       (long long)D, S, S);
    const double t0 = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
    gl_scratch tmp(ctx);
    uint8_t* d_x;
    GL_CHECK(tmp.alloc(d_x, (size_t)S * ldp));
    GL_CUDA(ctx, cudaMemcpy2DAsync(d_x, (size_t)ldp, x, (size_t)ld, (size_t)D, (size_t)S, cudaMemcpyHostToDevice, ctx->stream));
    GL_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const double t_up = std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count() - t0;
    return pca_run(ctx, d_x, ldp, S, D, k, proj, sv, k_out, gram, t_up);
}

int gl_indexcov_pca_phases(gl_ctx* ctx, double* t3) {
    if (!ctx || !t3) return gl_fail(ctx, GL_EINVAL, "gl_indexcov_pca_phases: bad argument");
    for (int i = 0; i < 3; i++) t3[i] = ctx->pca_phase[i];
    return GL_OK;
}

int gl_sym_tridiag(gl_ctx* ctx, const double* a, int32_t n, double* d, double* e, double* tau, double* refl, int32_t k, double* u) {
    GL_CHECK(gl_use(ctx));
    if (n < 1 || k < 0 || !a || !d || (n > 1 && !e) || (n > 2 && !tau) || !refl || (k > 0 && !u))
        return gl_fail(ctx, GL_EINVAL, "gl_sym_tridiag: bad argument (n = %d, k = %d)", n, k);
    if (n > 65535) return gl_fail(ctx, GL_EINVAL, "gl_sym_tridiag: n = %d; at most 65535", n);
    gl_scratch tmp(ctx);
    double* d_A;
    GL_CHECK(tmp.upload(d_A, a, (size_t)n * n));
    SymTridiag tri;
    GL_CHECK(sym_tridiag(ctx, d_A, n, tri));
    std::copy(tri.d.begin(), tri.d.end(), d);
    std::copy(tri.e.begin(), tri.e.begin() + (n - 1), e);
    std::copy(tri.tau.begin(), tri.tau.begin() + std::max(0, n - 2), tau);
    std::copy(tri.hA.begin(), tri.hA.end(), refl);
    if (k > 0) tri.back_transform(u, k);
    return GL_OK;
}

}  // extern "C"
