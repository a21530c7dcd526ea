"""`goleft emdepth` without a GPU: the oracle against the reference's own tests and hand cases, the Cache walk
(gl_emdepth_cnvs) against the oracle's literal Cache, the bin-sum certificate and the Pow table."""
import math

import numpy as np
import pytest

from goleft_b200 import capi
from oracle import emdepth as oe
from oracle.dcnv import Panic


def test_reference_test_depth():
    assert oe.cns([1, 8, 33, 34, 35, 37, 31, 22, 66]) == [0, 1, 2, 2, 2, 2, 2, 2, 4]
    assert oe.cns([30, 28, 33, 34, 35, 37, 31, 22, 38]) == [2] * 9


def test_reference_test_big():
    """TestBig expects 8 for the two samples above the top centre, but Type returns len(Lambda) = 9 there (emdepth.go:278):
    the reference's own test fails, and the code, not the test, is what is restated"""
    v = [296.6, 16.7, 17.0, 3019.2, 14.4, 16.5, 14.2, 26, 7]
    cells, lam, fc = oe.emdepth(v)
    got = [int(c) & 15 for c in cells[0]]
    assert got == [9, 2, 2, 9, 2, 2, 2, 3, 1]
    assert got != [8, 2, 2, 8, 2, 2, 2, 3, 1]
    assert v[0] > lam[0, 8] and v[3] > lam[0, 8]
    c2, _, fc2 = oe.emdepth([96.6, 16.7, 17.0, 319.2, 14.4, 16.5, 14.2, 7, 16])
    e, o = oe.EMD(fc2[0], None, (123, 456)), oe.EMD(fc[0], None, (123, 456))
    non2, changed, pct = oe.same(e, o)                                   # em2.Same(cns)
    assert non2 == [0, 3] and changed == [7, 8] and pct == 7 / 9


def test_even_median_and_two_samples():
    # S = 4: median32 takes (b[2] + b[3]) / 2, not (b[1] + b[2]) / 2
    _, lam, _ = oe.emdepth([10, 20, 30, 1000])
    _, lam_odd, _ = oe.emdepth([10, 20, 30, 1000, 5000])
    assert lam[0, 0] == 0.01 * (30 + 1000) / 2 and lam_odd[0, 0] == 0.01 * 30
    for S in (0, 2):
        with pytest.raises(Panic):
            oe.emdepth(np.ones((1, S), np.float32))


def test_lambda2_zero_branch():
    """mostly zeros: bin 2 is empty or all zero, and lambda[2] comes from bins 1..7 with the eps writes"""
    x = np.array([[0, 0, 0, 0, 0, 3, 0, 0, 9], [0, 0, 0, 0, 0, 0, 0, 0, 0], [0, 0, 0, 1, 0, 0, 0, 0, 0]], np.float32)
    cells, lam, fc = oe.emdepth(x)
    assert (lam[:, 2] > 0).all()                                         # the fallback starts lambda[2] at eps
    assert lam[1, 2] == 0.01 and lam[1, 0] == 0                          # all zero: lambda[2] = eps exactly
    assert np.isneginf(fc[1]).all() and ((cells[1] >> 4) & 3 == 1).all()


def test_maxiter_and_large_k():
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.integers(1000, 5000, 40), rng.integers(1, 20, 40), [3019.2, 1e7]]).astype(np.float32)[None, :]
    cells, lam, _ = oe.emdepth(x)                                        # k >= 1000 uses Lgamma beyond the table
    assert np.isfinite(lam).all() and (cells & 15).max() == 9


def _pmf_exponent(k, mu):
    return k * math.log(mu) - math.lgamma(k + 1) - mu


@pytest.mark.parametrize("M", [1e6, 1e7])
def test_pmf_underflow_keeps_cn(M):
    """centres around M, d = 1.9 M between lambda[3] and lambda[4]: both pmfs underflow to 0, o * 0.9 < o2 is false and
    the CN stays 3"""
    x = np.array([[M] * 8 + [1.9 * M]], np.float32)
    cells, lam, _ = oe.emdepth(x)
    k = int(0.5 + float(x[0, 8]))
    assert _pmf_exponent(k, lam[0, 3]) < -750 and _pmf_exponent(k, lam[0, 2]) < -750
    assert cells[0, 8] & 15 == 3


def test_near_tie_rows_are_in_the_band():
    rows = oe.near_tie_rows(4)
    cells, lam, fc = oe.emdepth(rows)
    for r in range(len(rows)):
        q = float(rows[r, 500]) / lam[r, 2]
        assert abs(q / oe.Q_M08 - 1) < 5e-13                             # inside the library's 1e-12 band
        assert (cells[r, :500] == 2).all() and (cells[r, 501:] == 2).all()


def test_pow_table_is_go_route():
    def route(x):
        yf = 1.1 - 1                                                    # Modf(1.1)
        a1 = math.exp(yf * math.log(x))
        x1, xe = math.frexp(x)
        return math.ldexp(a1 * x1, xe)
    want = np.array([0.0, route(0.5), 1.0] + [route(i / 2) for i in range(3, 9)])
    assert (1.1 - 1) == 0.10000000000000009
    assert np.array_equal(capi.emdepth_factors().view(np.uint64), want.view(np.uint64))
    assert np.array_equal(oe.factors().view(np.uint64), want.view(np.uint64))


def _seq(v):
    s = 0.0
    for x in np.asarray(v, np.float32):
        s += float(x)
    return s


def test_certified_sums_are_sequential():
    rng = np.random.default_rng(3)
    n_cert = 0
    for t in range(3000):
        n = int(rng.integers(1, 400))
        kind = t % 4
        if kind == 0:
            v = rng.integers(0, 5000, n).astype(np.float32)
        elif kind == 1:
            v = np.round(rng.gamma(2, 30, n), 2).astype(np.float32)
        elif kind == 2:
            v = (rng.random(n) * 2.0 ** rng.integers(-20, 20)).astype(np.float32)
        else:
            v = rng.random(n).astype(np.float32) * np.float32(2.0) ** rng.integers(-30, 30, n).astype(np.float32)
        s, ok = capi.emdepth_sum_host(v)
        if ok:
            n_cert += 1
            assert s == _seq(v), (t, n)
    assert n_cert > 1500


def test_wide_spread_takes_the_fallback():
    v = np.array([2.0 ** 53, 1, 0, 1], np.float32)                      # sequential: both 1s round away; a tree keeps 2
    s, ok = capi.emdepth_sum_host(v)
    assert not ok and s != _seq(v)                                       # the order matters, and the certificate knows it
    s, ok = capi.emdepth_sum_host(np.array([2.0 ** 20, 1.0 + 2.0 ** -23, 3.0], np.float32))
    assert ok
    assert capi.emdepth_sum_host(np.zeros(50, np.float32)) == (0.0, True)


# ---- the Cache
_FC = np.array([-np.inf, -1.0, -0.6, 0.0, 0.35, 1.0, np.nan, np.inf])


def _cell(cn, f):
    if -0.8 < f < 0.4:
        cls = 0
    elif f <= -0.8:
        cls = 1
    elif f >= 0.4:
        cls = 2
    else:
        cls = 3
    return cn | cls << 4 | (0 if -0.5 < f < 0.3 else 0x40)


def _oracle_cnvs(chroms, starts, ends, fc, cn):
    return [(v["sample"], v["psize"], v["rows"]) for v in oe.drive(chroms, starts, ends, fc, cn)]


def _lib_cnvs(chroms, starts, ends, cells):
    breaks = [r for r in range(1, len(chroms)) if chroms[r] != chroms[r - 1]]
    return [(s, p, list(map(int, rows))) for s, p, rows in capi.emdepth_cnvs(cells, starts, ends, breaks)]


def test_cache_random_patterns():
    rng = np.random.default_rng(11)
    for t in range(3000):
        n, S = int(rng.integers(1, 40)), int(rng.integers(1, 6))
        p_non2 = rng.random()
        idx = np.where(rng.random((n, S)) < p_non2, rng.choice([0, 1, 5, 6, 7], (n, S)), rng.choice([2, 3, 4], (n, S)))
        fc = _FC[idx]
        cn = rng.integers(0, 10, (n, S))
        with np.errstate(invalid="ignore"):
            cells = np.vectorize(_cell)(cn, fc).astype(np.uint8)
        step = int(rng.choice([1000, 20000, 40000, 2 ** 31]))
        starts = (np.cumsum(rng.integers(0, step, n)) % (1 << 32)).astype(np.int64)
        ends = ((starts + rng.integers(0, 3 * step, n)) % (1 << 32)).astype(np.int64)
        chroms = np.sort(rng.integers(0, 3, n)) if t % 2 else np.zeros(n, int)
        want = _oracle_cnvs(list(chroms), starts, ends, fc, cn)
        assert _lib_cnvs(list(chroms), starts, ends, cells) == want, t


def _pattern(rows, starts=None, ends=None, chroms=None):
    fc = np.array(rows, np.float64)
    n, S = fc.shape
    starts = np.arange(n, dtype=np.int64) * 1000 if starts is None else np.asarray(starts, np.int64)
    ends = starts + 1000 if ends is None else np.asarray(ends, np.int64)
    chroms = [0] * n if chroms is None else chroms
    cn = np.full((n, S), 3)
    cells = np.vectorize(_cell)(cn, fc).astype(np.uint8)
    want = _oracle_cnvs(chroms, starts, ends, fc, cn)
    assert _lib_cnvs(chroms, starts, ends, cells) == want
    return want


def test_cache_quirks():
    # the first Add compares the row with itself: a lone high row is pending and emitted at the end
    assert _pattern([[1.0, 0.0]]) == [(0, 1, [0])]
    # keys starts as zeros: sample 0's pending run is dropped at the next Clear while sample 1's (gap too small) waits
    got = _pattern([[1.0, 1.0], [1.0, 1.0], [0.0, 0.0]], starts=[0, 1000, 2000], ends=[1000, 2000, 3000])
    assert [g[0] for g in got] == [1] and got[0][2] == [0, 1]
    # the gap is uint32: a start before the pending end wraps to a huge gap and emits at once
    got = _pattern([[0.0, 1.0], [0.0, 1.0], [0.0, 0.0]], starts=[50000, 60000, 10000], ends=[60000, 70000, 20000])
    assert got[0] == (1, 1, [0, 1])
    # PSize = len(map) at the Clear
    got = _pattern([[1.0, 1.0, 1.0], [1.0, 1.0, 1.0]], starts=[0, 1000], ends=[1000, 2000])
    assert [g[1] for g in got] == [3, 3, 3]


def test_chromosome_breaks():
    rows = [[1.0, 0.0]] * 3 + [[0.0, 1.0]] * 3
    got = _pattern(rows, starts=[0, 1000, 2000, 0, 1000, 2000], ends=[1000, 2000, 3000, 1000, 2000, 3000], chroms=[0, 0, 0, 1, 1, 1])
    # Clear(nil) at the break emits sample 0, whose earlier rows every Add's Clear dropped (keys starts as zeros); on the
    # second chromosome sample 1 turns non-CN2 from row 4 (row 3 is compared with row 2) and is emitted at the end
    assert got == [(0, 1, [2]), (1, 1, [4, 5])]
