"""The host parts of indexcov's PCA (DESIGN §1.11), no GPU needed: the byte rule against the float32 restatement, the
integer Gram identity and the projection formula against gonum's SVD route, the tridiagonal eigensolver, and the byte
matrix's layout quirks in the oracle."""
import numpy as np
import pytest
import scipy.linalg

from goleft_b200 import capi
from oracle import indexcov_pca as op


# ---- the byte rule
def test_pca8_strided_float32_range():
    """every float32 in [0, 8] with a stride of 61 in the bit pattern, plus 8 itself"""
    hi = int(np.float32(8).view(np.uint32))
    bits = np.arange(0, hi + 1, 61, dtype=np.uint32)
    d = np.concatenate([bits.view(np.float32), [np.float32(8)]])
    assert np.array_equal(capi.indexcov_pca8(d), op.pca8_bytes(d))


def test_pca8_byte_boundaries():
    """every value within 2 ulp of each point where 8191.875 d + 0.5 crosses an integer, and the special values"""
    b = np.arange(1, 65536, dtype=np.float64)
    c = ((b - 0.5) / 8191.875).astype(np.float32)
    near = [c]
    for _ in range(2):
        near.append(np.nextafter(near[-1], np.float32(np.inf)))
    lo = c
    for _ in range(2):
        lo = np.nextafter(lo, np.float32(-np.inf))
        near.append(lo)
    special = np.array([0.0, -0.0, 8.0, 8.0000005, 9.5, 1e30, np.inf, 1.0, 0.5, 2.0, 1.4e-45, 1e-40, 1.17549435e-38, 7.9999995],
                       np.float32)
    d = np.concatenate(near + [special])
    got = capi.indexcov_pca8(d)
    assert np.array_equal(got, op.pca8_bytes(d))
    # the quirks, spelled out: depth 1.0 -> 8192.375 -> byte 0; 8 and above -> 65535.5 -> 0xFF; 0 -> 0.5 -> 0
    assert capi.indexcov_pca8(np.array([1.0, 8.0, 100.0, 0.0], np.float32)).tolist() == [0, 255, 255, 0]


# ---- the Gram identity and the projection formula
def _matrices(rng):
    yield rng.integers(0, 256, (7, 300)).astype(np.uint8)
    x = rng.integers(0, 256, (40, 2000)).astype(np.uint8)
    x[:15, :400] = 0                                                   # a planted group: zero stretches shared by 15 samples
    yield x
    x = rng.integers(100, 140, (25, 500)).astype(np.uint8)
    x[5:12, 100:300] = 255
    yield x
    yield rng.integers(0, 256, (4, 3)).astype(np.uint8)                 # D < S


@pytest.mark.parametrize("seed", [0, 1])
def test_gram_identity_and_projection(seed):
    """n^2 Gc = n^2 G - n (r_i + r_j) + q holds exactly (Python integers); proj = sigma u + (c . u) / sigma from the
    eigenpairs of Gc equals X V[:, :k] from the SVD of Xc"""
    rng = np.random.default_rng(seed)
    for x in _matrices(rng):
        S, D = x.shape
        X = x.astype(object)
        G = X.dot(X.T)
        r = G.sum(axis=1)
        q = int(r.sum())
        n2Gc = S * S * G - S * (r[:, None] + r[None, :]) + q
        Xc_n = X * S - X.sum(axis=0)[None, :]                           # n Xc, exact
        assert (n2Gc == Xc_n.dot(Xc_n.T)).all()
        Gc = np.array([[float(v) for v in row] for row in n2Gc]) / float(S * S)
        lam, V = np.linalg.eigh(Gc)
        lam, V = lam[::-1], V[:, ::-1]
        c = np.array([float(S * int(ri) - q) for ri in r]) / float(S * S)
        proj, sv, kk = op.pca(x)
        for j in range(kk):
            if sv[j] == 0:
                continue
            u = V[:, j] * (1 if V[np.argmax(np.abs(V[:, j])), j] > 0 else -1)
            sig = np.sqrt(lam[j])
            got = sig * u + (c @ u) / sig
            assert abs(sig - sv[j]) <= 1e-9 * sv[0]
            assert np.abs(got - proj[:, j]).max() <= 1e-9 * np.abs(proj[:, j]).max()


# ---- the tridiagonal eigensolver
def _tridiagonals(rng):
    yield rng.normal(size=50), rng.normal(size=49)
    n = 21                                                             # Wilkinson's W21+: pairs agreeing to ~1e-14
    yield np.abs(np.arange(n) - 10).astype(np.float64), np.ones(n - 1)
    d = np.repeat([5.0, 5.0, 3.0, 1.0], 10)                            # exact multiplicity across split blocks
    e = rng.normal(size=39) * 1e-3
    e[9::10] = 0
    yield d, e
    yield np.zeros(6), np.zeros(5)
    yield np.array([3.5]), np.zeros(0)
    a = rng.integers(0, 256, (300, 60)).astype(np.float64)             # the clustered top of a pure-noise Gram
    a -= a.mean(axis=0)
    T = scipy.linalg.hessenberg(a.T @ a)
    yield np.diag(T).copy(), np.diag(T, -1).copy()
    yield 1e10 * rng.random(200), 1e3 * rng.normal(size=199)


def test_tridiag_top():
    rng = np.random.default_rng(5)
    for d, e in _tridiagonals(rng):
        n = d.size
        k = min(5, n)
        w, z = capi.pca_tridiag_top(d, e, k)
        ref = scipy.linalg.eigh_tridiagonal(d, e, eigvals_only=True)[::-1][:k]
        T = np.diag(d) + np.diag(e, 1) + np.diag(e, -1)
        nrm = max(np.abs(T).sum(axis=1).max(), 1e-300)
        assert np.all(np.diff(w) <= 0)
        assert np.abs(w - ref).max() <= 8 * n * np.finfo(float).eps * nrm + 1e-300
        for j in range(k):
            assert abs(np.linalg.norm(z[j]) - 1) < 1e-12
            assert np.linalg.norm(T @ z[j] - w[j] * z[j]) <= 64 * n * np.finfo(float).eps * nrm
        assert np.abs(z @ z.T - np.eye(k)).max() < 1e-10
        w2, z2 = capi.pca_tridiag_top(d, e, k)
        assert np.array_equal(w, w2) and np.array_equal(z, z2)


def test_tridiag_top_bad_args():
    with pytest.raises(capi.GlError):
        capi.pca_tridiag_top(np.ones(3), np.ones(2), 4)
    with pytest.raises(capi.GlError):
        capi.pca_tridiag_top(np.ones(3), np.ones(2), 0)


# ---- the layout of the byte matrix (indexcov.go:688-704), on hand cases
def test_pca8_layout_quirks():
    one = np.float32(1.0)      # byte 0
    two = np.float32(2.0)      # 16383.75 + 0.5 -> 16384 -> 0x00
    half = np.float32(0.5)     # 4095.9375 + 0.5 -> 4096 -> 0x00
    v = np.float32(0.1)        # 819.1875 + 0.5 -> 819 -> 0x33
    refs = [
        [[v, v, v], [v], []],                                           # sample 3 has no values: longest + 1 zeros
        [[], [], []],                                                   # longest == 0: one zero column
        [[v], [np.float32(9.0)], [v, one]],                             # a GL contig: clipped at 8 -> 0xFF
    ]
    x = op.pca8_matrix(refs)
    assert x.shape == (3, 4 + 1 + 3)
    assert x[0].tolist() == [0x33, 0x33, 0x33, 0, 0, 0x33, 0, 0]
    assert x[1].tolist() == [0x33, 0, 0, 0, 0, 0xFF, 0, 0]
    assert x[2].tolist() == [0, 0, 0, 0, 0, 0x33, 0, 0]
    assert op.pca8_bytes([two, half, v]).tolist() == [0, 0, 0x33]
