// sym_eig.cuh — the symmetric eigenproblem that indexcov's PCA (pca.cu, DESIGN §1.11) and `dcnv --svd` (dcnv_svd.cu,
// DESIGN §1.13) share: the device tridiagonalises, the host finds eigenvalues and vectors of the tridiagonal
// (host/pca_eig.h) and takes the vectors back through the reflectors.  Library-internal: not exported from the .so.
#pragma once
#include <vector>
#include "gl_common.cuh"

struct __attribute__((visibility("hidden"))) SymTridiag {
    int n = 0;
    std::vector<double> hA;              // n x n: row j holds the reflector v_j (v_j[0] = 1) from column j + 1
    std::vector<double> d, e, tau;       // T = tridiag(e, d, e); H_j = I - tau[j] v_j v_j^T
    // k vectors of T (vector j at u[j * n]) -> the same vectors of A, in place: u = H_0 H_1 ... H_{n-3} u
    void back_transform(double* u, int k) const;
};

// Householder tridiagonalisation (Golub & Van Loan 8.3.1) of the symmetric n x n row-major d_A on the device, which it
// overwrites with the reflectors; every reduction has a fixed order, so the same A gives the same bits.
__attribute__((visibility("hidden"))) int sym_tridiag(gl_ctx* ctx, double* d_A, int n, SymTridiag& t);
