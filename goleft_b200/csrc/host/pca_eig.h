// pca_eig.h — the host half of indexcov's PCA (pca.cu, DESIGN §1.11): the top eigenpairs of a symmetric tridiagonal matrix,
// and the projections the reference prints from them.  Textbook algorithms (Golub & Van Loan, Matrix Computations, 8.4-8.5;
// Demmel, Applied Numerical Linear Algebra, 5.3): Sturm-count bisection to the last representable double, then inverse
// iteration with partial pivoting, re-orthogonalised inside clusters.  Nothing here has a tolerance or an iteration cap a
// caller can set; every loop has a fixed bound.
#pragma once
#include <stdint.h>

namespace glpca {

// w[0..k) = the k largest eigenvalues of T = tridiag(e, d, e) (d[0..n), e[0..n-1)), in descending order; k <= n
void tridiag_top_values(const double* d, const double* e, int n, int k, double* w);
// w[0..k) = every eigenvalue of T above rel * (the largest), descending, as tridiag_top_values finds each (bit for bit);
// returns k (0 when the largest is not positive).  One Sturm count finds how many lie at or above the threshold, so only those
// are bisected, each on its own task of the host pool.  w has room for n values.
int tridiag_values_above(const double* d, const double* e, int n, double rel, double* w);
// z[j*n .. j*n+n) = a unit eigenvector of T for w[j], j < k (w descending, as tridiag_top_values made them)
void tridiag_vectors(const double* d, const double* e, int n, const double* w, int k, double* z);
// The reference's projections from the eigenpairs (lambda descending, u column j at u[j*S..]) of the centred Gram Gc and
// c = X mean: proj(i, j) = sigma_j u(i, j) + (c . u_j) / sigma_j, sigma_j = sqrt(lambda_j), after the sign rule (the entry
// of u_j with the largest magnitude is made positive; the lowest sample on a tie).  Rank rule: when lambda_0 <= 0 or
// lambda_j <= kRankTol * lambda_0 the column is 0 and sv[j] = 0.  proj is S x k, row-major.
constexpr double kRankTol = 1e-12;
void project(const double* lambda, double* u, const double* c, int S, int k, double* proj, double* sv);

}  // namespace glpca
