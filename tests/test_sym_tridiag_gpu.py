"""The device Householder tridiagonalisation that indexcov's PCA and `dcnv --svd` share (pca.cu: house_kernel, symv_kernel,
rank2_kernel; sym_eig.cuh), through gl_sym_tridiag, against plain references of the same operation: a literal Householder
reduction in np.longdouble with the kernels' conventions, and LAPACK in float64 (numpy's eigvalsh, scipy's
eigvalsh_tridiagonal).  No product code computes an expected value here; capi.pca_tridiag_top only supplies vectors of T.

Every c·n·ε bound below uses the one constant C:
  forward   d and e within 1e-9 max|A|, tau within 1e-9 of the longdouble reduction (n <= 400, the full-rank kinds)
  backward  Q = H_0 H_1 ... H_{n-3} built from the returned reflectors and tau: ||Q^T Q - I|| <= C n eps and
            ||(Q^T A Q - T) p|| <= C n eps ||A|| ||p||; in longdouble with the whole Q for n <= 400, in float64 on 8 random
            probes above
  values    the eigenvalues of T = eigvalsh(A) within C n eps ||A||; the wide cohort's null values below the 1e-12 lambda_1
            rank rule both callers apply
  vectors   the top 5 vectors of T taken back through the reflectors by the entry: ||A u - lambda u|| <= C n eps ||A|| and
            ||U^T U - I|| < 1e-10
  exact     bit for bit where the reduction has nothing to round, and the same A twice gives the same bits
A float64 restatement of the kernels' formulas, run through these checks on the same matrices, reaches at most 0.7 n eps
(relative to ||A|| where the bound has it) for n <= 5, where the references' own rounding is as large as the reduction's,
0.06 n eps at n = 300 and 0.04 n eps at n = 1000; C = 4 leaves room for a different summation order.  A wrong reflector or
rank-2 term is O(1)."""
import ctypes as C

import numpy as np
import pytest
import scipy.linalg

from goleft_b200 import capi

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
C_BOUND = 4.0                    # the c of every c·n·ε bound
LD = np.longdouble
SIZES = [1, 2, 3, 4, 5, 300, 1000, 2504, 4097]
KINDS = ["gauss", "noise", "planted", "wide", "cluster"]
FULL_RANK = ("gauss", "noise", "planted")
FULL_Q_MAX = 400                 # the whole Q in longdouble up to here, probes above
D_BYTES = 3000


# ---- matrices
def _sym(b):
    """the exactly symmetric matrix of b's upper triangle"""
    return np.triu(b) + np.triu(b, 1).T


def _centred_gram(x):
    """Gc = Xc Xc^T of the byte rows x as pca_run forms it: (n^2 G - n (r_i + r_j) + q) / n^2 from the exact integer Gram,
    the numerator rounded once"""
    S = x.shape[0]
    xf = x.astype(np.float64)
    g = (xf @ xf.T).astype(np.int64)                               # every partial sum is an integer below 2^53
    r = g.sum(axis=1)
    num = S * S * g - S * (r[:, None] + r[None, :]) + r.sum()       # below 2^63 for S <= 4097, D = 3000
    return _sym(num.astype(np.float64) / float(S * S))


def _planted_bytes(rng, S, D):
    """depth-like bytes with groups: zero stretches shared by subsets of the samples (test_indexcov_pca_gpu.py's kind)"""
    x = rng.integers(20, 90, (S, D), dtype=np.uint8)
    for a, b, frac in [(0, S // 3, 0.10), (S // 3, S // 2, 0.25), (S // 2, S, 0.05)]:
        c0 = int(rng.integers(0, D // 2))
        x[a:b, c0:c0 + int(frac * D)] = 0
    x[:, ::97] = 0
    return x


def _matrix(kind, n, seed=0):
    rng = np.random.default_rng([n, KINDS.index(kind), seed])
    if kind == "gauss":                                               # symmetric Gaussian
        return _sym(rng.normal(size=(n, n)))
    if kind == "noise":                                               # centred uint8 Gram: one dominant eigenvalue, wide spread
        return _centred_gram(rng.integers(0, 256, (n, D_BYTES), dtype=np.uint8))
    if kind == "planted":
        return _centred_gram(_planted_bytes(rng, n, D_BYTES))
    if kind == "wide":                                                # z-score Gram Z^T Z of n // 2 rows: rank min(rows, n - 1)
        if n < 2:
            return np.zeros((n, n))
        x = rng.gamma(30.0, 1.0 / 30.0, (max(1, n // 2), n)) * rng.uniform(0.5, 2.0, (max(1, n // 2), 1))
        z = (x - x.mean(axis=1, keepdims=True)) / x.std(axis=1, ddof=1, keepdims=True)
        return _sym(z.T @ z)
    # cluster: three equal groups, each the same planted cohort, on columns of their own: the Gram is three copies of one
    # block (every eigenvalue threefold, the top one included), plus a remainder of 1 or 2 small diagonal entries, with the
    # samples shuffled
    k = n // 3
    xf = _planted_bytes(rng, k, D_BYTES).astype(np.float64)
    m = xf @ xf.T                                                     # exact integers
    b = scipy.linalg.block_diag(m, m, m, np.diag(np.arange(1.0, n - 3 * k + 1))) if n - 3 * k else scipy.linalg.block_diag(m, m, m)
    p = rng.permutation(n)
    return np.ascontiguousarray(b[p][:, p])


def _rank(kind, n):
    """the exact rank of the wide cohort's Gram"""
    return 0 if n < 2 else min(max(1, n // 2), n - 1)


# ---- references
def householder_ld(a):
    """(d, e, tau, reflector rows) of a literal Householder reduction of a in np.longdouble with the kernels' conventions:
    beta = -copysign(sqrt(alpha^2 + |x2|^2), alpha), tau = (beta - alpha) / beta, v = x / (alpha - beta) with v_0 = 1, and no
    reflector when |x2|^2 = 0"""
    A = np.array(a, LD)
    n = A.shape[0]
    d, e, tau = np.zeros(n, LD), np.zeros(max(n - 1, 0), LD), np.zeros(max(n - 2, 0), LD)
    V = np.zeros((n, n), LD)
    for j in range(n - 2):
        x = A[j, j + 1:].copy()
        alpha, xn2 = x[0], x[1:] @ x[1:]
        beta, t, v = alpha, LD(0), np.zeros_like(x)
        if xn2 != 0:
            beta = -np.copysign(np.sqrt(alpha * alpha + xn2), alpha)
            t = (beta - alpha) / beta
            v = x / (alpha - beta)
        v[0] = 1
        d[j], e[j], tau[j], V[j, j + 1:] = A[j, j], beta, t, v
        if t != 0:
            A22 = A[j + 1:, j + 1:]
            p = t * (A22 @ v)
            w = p - (t / 2) * (p @ v) * v
            A22 -= np.outer(v, w) + np.outer(w, v)
    if n >= 2:
        d[n - 2], e[n - 2] = A[n - 2, n - 2], A[n - 1, n - 2]
    if n >= 1:
        d[n - 1] = A[n - 1, n - 1]
    return d, e, tau, V


def _apply_q(refl, tau, y, transpose=False):
    """Q y (or Q^T y) in y's precision for Q = H_0 H_1 ... H_{n-3}, H_j = I - tau_j v_j v_j^T, v_j = refl[j, j+1:]"""
    y = y.copy()
    n, dt = refl.shape[0], y.dtype.type
    order = range(n - 2) if transpose else range(n - 3, -1, -1)
    for j in order:
        if tau[j] == 0:
            continue
        v = refl[j, j + 1:].astype(dt)
        y[j + 1:] -= dt(tau[j]) * np.outer(v, v @ y[j + 1:])
    return y


def _tri_mul(d, e, y):
    """T y in y's precision, T = tridiag(e, d, e)"""
    d, e = d.astype(y.dtype), e.astype(y.dtype)
    out = d[:, None] * y
    out[:-1] += e[:, None] * y[1:]
    out[1:] += e[:, None] * y[:-1]
    return out


def _norm2(m):
    m = np.asarray(m, np.float64)
    return float(np.linalg.norm(m, 2)) if m.size else 0.0


# ---- checks (each takes the entry's outputs)
def check_forward(a, d, e, tau):
    dl, el, tl, _ = householder_ld(a)
    scale = np.abs(a).max()
    for name, got, want, tol in (("d", d, dl, 1e-9 * scale), ("e", e, el, 1e-9 * scale), ("tau", tau, tl, 1e-9)):
        err = float(np.abs(got.astype(LD) - want).max()) if got.size else 0.0
        assert err <= tol, ("forward", name, err, tol)


def check_backward(a, d, e, tau, refl, a_norm, probes=8, seed=0):
    n = a.shape[0]
    if n <= FULL_Q_MAX:
        y = np.eye(n, dtype=LD)
    else:                               # float64: applying the reflectors rounds by about sqrt(n) eps, far inside the bound
        y = np.random.default_rng(seed).normal(size=(n, probes))
    qy = _apply_q(refl, tau, y)
    orth = _apply_q(refl, tau, qy, transpose=True) - y
    resid = _apply_q(refl, tau, a.astype(y.dtype) @ qy, transpose=True) - _tri_mul(d, e, y)
    if n <= FULL_Q_MAX:                                               # y = I: the spectral norms of Q^T Q - I and Q^T A Q - T
        o, r = _norm2(orth), _norm2(resid)
    else:                                                             # the worst probe, relative to its length
        pn = np.linalg.norm(y.astype(np.float64), axis=0)
        o = float((np.linalg.norm(orth.astype(np.float64), axis=0) / pn).max())
        r = float((np.linalg.norm(resid.astype(np.float64), axis=0) / pn).max())
    assert o <= C_BOUND * n * EPS, ("Q^T Q - I", o / (n * EPS))
    assert r <= C_BOUND * n * EPS * a_norm, ("Q^T A Q - T", r / (n * EPS * max(a_norm, 1e-300)))


def check_values(d, e, w_a, a_norm):
    w_t = scipy.linalg.eigvalsh_tridiagonal(d, e) if d.size > 1 else d.copy()
    err = float(np.abs(np.sort(w_t) - np.sort(w_a)).max())
    assert err <= C_BOUND * d.size * EPS * a_norm, ("eigenvalues", err / (d.size * EPS * max(a_norm, 1e-300)))
    return w_t


def check_vectors(a, lam, u, a_norm):
    n = a.shape[0]
    res = np.linalg.norm(u @ a - lam[:, None] * u, axis=1)            # a is symmetric: row j of U A is (A u_j)^T
    assert res.max() <= C_BOUND * n * EPS * a_norm, ("A u - lambda u", res.max() / (n * EPS * max(a_norm, 1e-300)))
    orth = np.abs(u @ u.T - np.eye(u.shape[0])).max()
    assert orth < 1e-10, ("U^T U - I", orth)


# ---- the reduction on every kind and size
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("kind", KINDS)
def test_reduction(ctx, kind, n):
    a = _matrix(kind, n)
    d, e, tau, refl, _ = ctx.sym_tridiag(a)
    assert d.shape == (n,) and e.shape == (max(n - 1, 0),) and tau.shape == (max(n - 2, 0),) and refl.shape == (n, n)
    assert np.all(np.isfinite(d)) and np.all(np.isfinite(e)) and np.all(np.isfinite(tau))
    if kind in FULL_RANK and n <= FULL_Q_MAX:
        check_forward(a, d, e, tau)
    w_a = np.linalg.eigvalsh(a)
    a_norm = float(np.abs(w_a).max()) if n else 0.0
    check_backward(a, d, e, tau, refl, a_norm)
    w_t = check_values(d, e, w_a, a_norm)
    if kind == "wide":                                                # the null space stays below the rank rule
        rank = _rank(kind, n)
        top = max(w_t.max(), 0.0)
        assert int((w_t > 1e-12 * top).sum()) == rank
        assert capi.pca_tridiag_above(d, e, 1e-12).size == rank
        assert np.abs(np.sort(w_t)[:n - rank]).max() <= 1e-12 * top
    k = min(5, n)
    lam, z = capi.pca_tridiag_top(d, e, k)
    _, _, _, _, u = ctx.sym_tridiag(a, u=z)
    check_vectors(a, lam, u, a_norm)


# ---- exact cases
def test_no_reflector_sizes_are_copies(ctx):
    """n = 1 and n = 2 run no step: d and e are a's bits, and the reflector matrix is a itself"""
    rng = np.random.default_rng(1)
    for n in (1, 2):
        a = _sym(rng.normal(size=(n, n)))
        d, e, tau, refl, u = ctx.sym_tridiag(a, u=np.eye(n))
        assert np.array_equal(d.view(np.uint64), np.diag(a).copy().view(np.uint64))
        assert np.array_equal(e.view(np.uint64), np.diag(a, -1).copy().view(np.uint64)) and tau.size == 0
        assert np.array_equal(refl.view(np.uint64), a.view(np.uint64)) and np.array_equal(u, np.eye(n))


@pytest.mark.parametrize("n", [3, 4, 33, 300])
def test_tridiagonal_input_takes_no_reflector(ctx, n):
    """every x2 is 0: tau = 0 at every step (symv_kernel's and rank2_kernel's tau == 0 exits), d and e are a's bits, each
    reflector row is (1, 0, ...), and the back-transformation is the identity"""
    rng = np.random.default_rng(n)
    dg, off = rng.normal(size=n), rng.normal(size=n - 1)
    off[::7] = -off[::7]
    a = np.diag(dg) + np.diag(off, 1) + np.diag(off, -1)
    u0 = rng.normal(size=(3, n))
    d, e, tau, refl, u = ctx.sym_tridiag(a, u=u0)
    assert np.array_equal(d.view(np.uint64), dg.view(np.uint64)) and np.array_equal(e.view(np.uint64), off.view(np.uint64))
    assert np.array_equal(tau.view(np.uint64), np.zeros(n - 2).view(np.uint64))
    for j in range(n - 2):
        assert refl[j, j + 1] == 1.0 and not refl[j, j + 2:].any()
    assert np.array_equal(u.view(np.uint64), u0.view(np.uint64))


@pytest.mark.parametrize("n", [3, 300])
def test_diagonal_input(ctx, n):
    dg = np.random.default_rng(n).normal(size=n)
    d, e, tau, _, _ = ctx.sym_tridiag(np.diag(dg))
    assert np.array_equal(d.view(np.uint64), dg.view(np.uint64))
    assert np.array_equal(e.view(np.uint64), np.zeros(n - 1).view(np.uint64)) and not tau.any()


@pytest.mark.parametrize("n", [4, 5, 300, 1000])
def test_zero_row_stays_decoupled(ctx, n):
    """a zero first (last) row and column: T's first (last) row is 0, and the rest is the reduction of the other n - 1 rows,
    bit for bit: every sum meets the same terms in the same order, plus exact zeros"""
    a = _matrix("gauss", n, seed=5)
    first = a.copy()
    first[0], first[:, 0] = 0.0, 0.0
    d, e, tau, _, _ = ctx.sym_tridiag(first)
    d1, e1, t1, _, _ = ctx.sym_tridiag(first[1:, 1:])
    assert d[0] == 0 and e[0] == 0 and tau[0] == 0
    assert np.array_equal(d[1:], d1) and np.array_equal(e[1:], e1) and np.array_equal(tau[1:], t1)
    last = a.copy()
    last[-1], last[:, -1] = 0.0, 0.0
    d, e, tau, _, _ = ctx.sym_tridiag(last)
    d1, e1, t1, _, _ = ctx.sym_tridiag(last[:-1, :-1])
    assert d[-1] == 0 and e[-1] == 0 and tau[-1] == 0
    assert np.array_equal(d[:-1], d1) and np.array_equal(e[:-1], e1) and np.array_equal(tau[:-1], t1)


@pytest.mark.parametrize("n,x", [(n, x) for n in (3, 5, 300) for x in ((3.0, 4.0), (0.0, 3.0, 4.0), (-0.0, 3.0, 4.0))
                                 if len(x) < n], ids=lambda v: str(v) if isinstance(v, int) else "x=" + ",".join("%g" % t for t in v))
def test_first_reflector_exact(ctx, n, x):
    """x = (3, 4, 0, ...): beta = -5 exactly, tau = 8/5, v = (1, 1/2, 0, ...); alpha = +0 (-0) with |x2| = 5: beta = -5 (+5),
    tau = 1, v = (1, 3/(alpha - beta), 4/(alpha - beta), 0, ...).  The rest of the reduction is checked backward."""
    a = _matrix("gauss", n, seed=9)
    row = np.zeros(n - 1)
    row[:len(x)] = x
    a[0, 1:], a[1:, 0] = row, row
    d, e, tau, refl, _ = ctx.sym_tridiag(a)
    alpha = np.float64(x[0])
    beta = -np.copysign(np.sqrt(alpha * alpha + np.float64(sum(v * v for v in x[1:]))), alpha)
    assert abs(beta) == 5.0 and e[0] == beta
    assert tau[0] == (beta - alpha) / beta
    v = row / (alpha - beta)                                          # the zeros past x keep the quotient's sign
    v[0] = 1.0
    assert np.array_equal(refl[0, 1:].view(np.uint64), v.view(np.uint64))
    a_norm = float(np.abs(np.linalg.eigvalsh(a)).max())
    check_backward(a, d, e, tau, refl, a_norm)


def test_same_matrix_same_bits(ctx):
    a = _matrix("noise", 2504)
    u0 = np.random.default_rng(3).normal(size=(5, 2504))
    r1 = ctx.sym_tridiag(a, u=u0)
    r2 = ctx.sym_tridiag(a, u=u0)
    for x, y in zip(r1, r2):
        assert np.array_equal(x.view(np.uint64), y.view(np.uint64))


def test_bad_arguments(ctx):
    with pytest.raises(capi.GlError) as ei:
        ctx.sym_tridiag(np.zeros((0, 0)))
    assert ei.value.code == capi.GL_EINVAL
    with pytest.raises(ValueError):
        ctx.sym_tridiag(np.zeros((3, 4)))
    with pytest.raises(ValueError):
        ctx.sym_tridiag(np.eye(3), u=np.zeros((2, 4)))
    buf = np.zeros(16)
    p = buf.ctypes.data_as(C.c_void_p)
    for args in ((None, 4, p, p, p, p, 0, None), (p, 2, p, p, p, None, 0, None), (p, 2, p, p, p, p, -1, None),
                 (p, 2, p, p, p, p, 1, None), (p, 65536, p, p, p, p, 0, None), (p, 3, p, None, p, p, 0, None)):
        assert capi.lib.gl_sym_tridiag(ctx.h, *args) == capi.GL_EINVAL, args
