"""The host side of `dcnv --svd` (DESIGN §1.13), no GPU needed: the oracle's count rule and log text on hand cases, the
exclusion of constant rows, and the pool-parallel bisection of every eigenvalue above the rank threshold against the serial
one and scipy."""
import numpy as np
import pytest
import scipy.linalg

from goleft_b200 import capi
from oracle import dcnv_svd as osv


# ---- the count rule (debiaser.go:185, capped at min(15, rank)) and the log line
def test_count_pct_zero_caps_at_15():
    s = np.linspace(20, 1, 40)
    assert osv.count(s, 0.0) == 15
    assert osv.variance_text(s, 2) == b"variance: %.2f %.2f" % (100 * 20 / s.sum(), 100 * s[1] / s.sum())


def test_count_caps_at_rank():
    s = np.array([5.0, 3.0, 1.0, 0.0, 0.0, 0.0])                        # S < 15 and a rank of 3
    assert osv.count(s, 0.0) == 3
    assert osv.count(np.zeros(4), 0.0) == 0
    assert osv.variance_text(np.zeros(4), 0) == b"variance:"


def test_count_tie_at_pct_stops():
    s = np.array([2.0, 1.0, 1.0])                                       # shares 50, 25, 25: exactly representable
    assert osv.count(s, 25.0) == 1
    assert osv.count(s, 24.999) == 3
    assert osv.count(s, 50.0) == 0
    assert osv.variance_text(s, 1) == b"variance: 50.00"


def test_one_and_two_samples():
    rng = np.random.default_rng(0)
    x1 = rng.normal(10, 1, (50, 1))
    out, s, n, kept = osv.svd_debias(x1, 0.0)
    assert n == 0 and not kept.any() and np.array_equal(out, x1) and s.tolist() == [0.0]
    x2 = rng.normal(10, 1, (50, 2))
    out, s, n, kept = osv.svd_debias(x2, 0.0)
    # two samples: every z row is (-1/sqrt 2, 1/sqrt 2) up to sign, so Z has rank 1 and removing it leaves the row means
    assert n == 1 and kept.all() and s[1] == 0
    assert np.allclose(out, np.repeat(x2.mean(axis=1, keepdims=True), 2, axis=1))


def test_constant_rows_excluded():
    rng = np.random.default_rng(1)
    S = 10
    x = rng.normal(5, 1, (30, S))
    x[3] = 0.1                                                           # sd of 0.1 x S by the two-pass formula is not 0
    x[4] = 0.0
    x[5] = 7.0
    z, kept, m, sd = osv.zscore(x)
    assert kept.sum() == 27 and not kept[3:6].any() and np.isfinite(z).all()
    out, s, n, _ = osv.svd_debias(x, 0.0)
    assert n >= 1
    assert np.array_equal(out[3:6], x[3:6])


# ---- the bisection of every eigenvalue above the threshold, one pool task per index
def _tridiagonals(rng):
    yield rng.normal(size=300), rng.normal(size=299)
    a = rng.normal(size=(2000, 80))
    a -= a.mean(axis=1, keepdims=True)                                  # rows sum to 0, as z-scored rows do: one zero eigenvalue
    T = scipy.linalg.hessenberg(a.T @ a)
    yield np.diag(T).copy(), np.diag(T, -1).copy()
    d = np.repeat([9.0, 4.0, 1e-20, 0.0], 8)
    e = np.zeros(31)
    yield d, e
    yield np.array([3.0]), np.zeros(0)
    yield np.zeros(5), np.zeros(4)


@pytest.mark.parametrize("rel", [1e-12, 0.0, 0.5])
def test_tridiag_above_equals_serial_and_scipy(rel):
    rng = np.random.default_rng(9)
    for d, e in _tridiagonals(rng):
        w = capi.pca_tridiag_above(d, e, rel)
        ref = scipy.linalg.eigvalsh_tridiagonal(d, e)[::-1] if d.size > 1 else d.copy()
        top = ref[0]
        want = ref[ref > rel * top] if top > 0 else ref[:0]
        assert w.size == want.size, (w.size, want.size)
        if w.size:
            ser, _ = capi.pca_tridiag_top(d, e, w.size, vectors=False)
            assert np.array_equal(w, ser)                               # bit for bit with the serial bisection
            nrm = max(np.abs(d).max() + 2 * (np.abs(e).max() if e.size else 0), 1e-300)
            assert np.abs(w - want).max() <= 8 * d.size * np.finfo(float).eps * nrm
        assert np.array_equal(w, capi.pca_tridiag_above(d, e, rel))


def test_tridiag_above_bad_args():
    for rel in (-1.0, 1.0, float("nan")):
        with pytest.raises(capi.GlError):
            capi.pca_tridiag_above(np.ones(3), np.ones(2), rel)
