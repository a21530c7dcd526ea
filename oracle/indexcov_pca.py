"""Test oracle for the PC columns of `goleft indexcov`'s .ped (indexcov.go:686-705,773-807, gonum stat.PC v0.14.0).

Independent of the product's route (an exact Gram, then Householder + bisection + inverse iteration): the byte matrix is
a literal restatement of the reference's append loop in numpy float32, and the PCA is gonum's own route: float64 column
means, the thin SVD of the centred matrix, then X V[:, :k] with the uncentred X.  On top of it the two rules the product
documents (DESIGN §1.11): each column's sign makes the largest-magnitude entry of its left singular vector positive (the
lowest sample on a tie), and a column whose squared singular value is at most 1e-12 of the first one is 0.
"""
import numpy as np

MAX_CN = np.float32(8)
RANK_TOL = 1e-12


def pca8_bytes(d) -> np.ndarray:
    """uint8(65535/MaxCN*dp+0.5) after the clip at MaxCN, as Go on amd64 converts it: float32 arithmetic, truncation to
    int32, the low byte (0x80000000, low byte 0, for NaN or out of int32 range)"""
    d = np.array(d, np.float32).ravel()
    d = np.where(d > MAX_CN, MAX_CN, d).astype(np.float32)
    v = (np.float32(65535) / MAX_CN) * d                     # float32 * float32 -> float32
    v = (v + np.float32(0.5)).astype(np.float32)
    ok = (v > np.float32(-2147483648.0)) & (v < np.float32(2147483648.0))
    t = np.zeros(v.size, np.int64)
    t[ok] = np.trunc(v[ok].astype(np.float64)).astype(np.int64)
    return (t & 0xFF).astype(np.uint8)


def pca8_matrix(refs) -> np.ndarray:
    """refs: for every kept reference that is not a sex chromosome, in order, the list of each sample's values (after -n).
    The append loop of indexcov.go:688-704, literally: each sample's bytes, then zeros for i from the last index (or -1)
    up to longest."""
    S = len(refs[0]) if refs else 0
    rows = [[] for _ in range(S)]
    for per_sample in refs:
        longest = max(len(v) for v in per_sample)
        for k, dps in enumerate(per_sample):
            i = -1
            b = pca8_bytes(dps) if len(dps) else []
            for i in range(len(dps)):
                rows[k].append(int(b[i]))
            while i < longest:
                rows[k].append(0)
                i += 1
    return np.array(rows, np.uint8).reshape(S, -1)


def pca(X, k: int = 5):
    """(proj S x k_out, sv[k_out], k_out): gonum's PrincipalComponents + VectorsTo + proj.Mul(imat, V[:, :k]), with the sign
    and rank rules above.  k_out = min(k, S, D)."""
    Xf = np.asarray(X, np.float64)
    S, D = Xf.shape
    kk = min(k, S, D)
    Xc = Xf - Xf.mean(axis=0)
    U, s, Vt = np.linalg.svd(Xc, full_matrices=False)
    proj = Xf @ Vt[:kk].T
    sv = s[:kk].copy()
    for j in range(kk):
        if not s[0] > 0 or not s[j] * s[j] > RANK_TOL * s[0] * s[0]:
            proj[:, j] = 0.0
            sv[j] = 0.0
            continue
        u = U[:, j]
        i = int(np.argmax(np.abs(u)))                         # first maximum: the lowest sample
        if u[i] < 0:
            proj[:, j] = -proj[:, j]
    return proj, sv, kk


def half_cent_near(v, tol) -> np.ndarray:
    """cells whose value lies within tol of a "%.2f" rounding boundary (an odd multiple of 0.005)"""
    v = np.asarray(v, np.float64)
    f = v * 100.0 - 0.5
    return np.abs(f - np.round(f)) * 0.01 <= tol
