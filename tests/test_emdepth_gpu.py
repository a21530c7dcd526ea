"""`goleft emdepth` on the GPU (gl_emdepth, gl_emdepth_device) against the C oracle: cells and centres bit for bit."""
import numpy as np
import pytest

from goleft_b200 import capi
from oracle import emdepth as oe

pytestmark = pytest.mark.gpu


def _matrix(rng, n, S):
    """integer columns (what depthwed writes), "%.2f" columns (what dcnv writes), zeros, planted CN1 / CN3 cells, huge
    outliers and an all-zero row"""
    base = rng.gamma(6.0, 6.0, (n, 1)) + 1
    x = base * rng.gamma(30.0, 1 / 30.0, (n, S))
    x[:, ::2] = np.floor(x[:, ::2])
    x[:, 1::2] = np.round(x[:, 1::2] / base.mean(), 2)
    hit = rng.random((n, S))
    x[hit < 0.03] *= 0.5
    x[(hit >= 0.03) & (hit < 0.06)] *= 1.5
    x[hit > 0.995] = 0
    x[(hit > 0.99) & (hit <= 0.991)] = rng.choice([1e6, 3e9, 7.5e12], int(((hit > 0.99) & (hit <= 0.991)).sum()))
    if n > 3:
        x[3] = 0
    return x.astype(np.float32)


def _check(ctx, x, **kw):
    cells, lam, _ = oe.emdepth(x)
    got, glam = ctx.emdepth(x, **kw)
    assert ctx.emdepth_stats()["uncertified"] == 0
    assert np.array_equal(glam.view(np.uint64), lam.view(np.uint64))
    assert np.array_equal(got, cells)
    return got


SAMPLES = [1, 3, 4, 9, 33, 128, 1000, 2504]


@pytest.mark.parametrize("n", [1, 1000])
@pytest.mark.parametrize("S", SAMPLES)
def test_matches_oracle(ctx, n, S):
    rng = np.random.default_rng(n * 7 + S)
    _check(ctx, _matrix(rng, n, S))


@pytest.mark.parametrize("S", SAMPLES)
def test_matches_oracle_2p20_rows(ctx, S):
    """2^20 + 7 rows in one call: a block of 4099 distinct rows, repeated (rows are independent, so every repeat must equal
    the block's oracle).  For S <= 9 the oracle also runs on the whole matrix."""
    n, B = (1 << 20) + 7, 4099
    rng = np.random.default_rng(S)
    block = _matrix(rng, B, S)
    x = np.tile(block, ((n + B - 1) // B, 1))[:n]
    got, lam = ctx.emdepth(x)
    assert ctx.emdepth_stats() == dict(rows=n, uncertified=0, sequential=0)
    if S <= 9:
        cells, olam, _ = oe.emdepth(x)
        assert np.array_equal(got, cells) and np.array_equal(lam.view(np.uint64), olam.view(np.uint64))
        return
    cells, olam, _ = oe.emdepth(block)                                 # every row: the repeats against the block's oracle
    for i in range(0, n, B):
        m = min(B, n - i)
        assert np.array_equal(got[i:i + m], cells[:m]), i
        assert np.array_equal(lam[i:i + m].view(np.uint64), olam[:m].view(np.uint64)), i


def test_near_ties_are_counted(ctx):
    """rows whose Log2FC for one cell lies within 4e-13 of -0.8: exactly those cells are counted as uncertified, and every
    other cell and every centre still equals the oracle"""
    rng = np.random.default_rng(21)
    ties = oe.near_tie_rows(6)
    S = ties.shape[1]
    x = _matrix(rng, 200, S)
    at = np.array([3, 17, 50, 51, 120, 199])
    x[at] = ties
    cells, lam, _ = oe.emdepth(x)
    got, glam = ctx.emdepth(x)
    assert ctx.emdepth_stats()["uncertified"] == len(at)
    assert np.array_equal(glam.view(np.uint64), lam.view(np.uint64))
    mask = np.ones(x.shape, bool)
    mask[at, S // 2] = False
    assert np.array_equal(got[mask], cells[mask])
    assert ((got[at, S // 2] >> 4) & 3 <= 2).all()                      # decided one way or the other, never NaN
    got2, _ = ctx.emdepth(np.delete(x, at, axis=0))
    assert ctx.emdepth_stats()["uncertified"] == 0 and np.array_equal(got2, np.delete(cells, at, axis=0))


@pytest.mark.parametrize("M", [1e6, 1e7])
def test_pmf_underflow_keeps_cn(ctx, M):
    x = np.array([[M] * 8 + [1.9 * M]], np.float32)
    cells, lam, _ = oe.emdepth(x)
    got, glam = ctx.emdepth(x)
    assert got[0, 8] & 15 == 3 and np.array_equal(got, cells) and np.array_equal(glam, lam)
    assert ctx.emdepth_stats()["uncertified"] == 0


def test_row_blocks_ld_and_device_entry(ctx):
    rng = np.random.default_rng(5)
    n, S = 5000, 37
    x = _matrix(rng, n, S)
    whole = _check(ctx, x)
    for br in (1, 7, 4999, n):
        got, _ = ctx.emdepth(x, block_rows=br)
        assert np.array_equal(got, whole)
    wide = np.zeros((n, S + 11), np.float32)                          # ld > S: the extra columns are never read
    wide[:, :S] = x
    wide[:, S:] = -1
    got, _ = ctx.emdepth(wide, ld=S + 11, S=S, block_rows=333)
    assert np.array_equal(got, whole)
    d_x = ctx.dev_array(wide)
    d_cells, d_lam = ctx.dev_empty(n * S), ctx.dev_empty(n * 9 * 8)
    ctx.emdepth_device(d_x, n, S + 11, S, d_cells, d_lam)
    assert np.array_equal(d_cells.download(np.uint8, n * S).reshape(n, S), whole)
    assert np.array_equal(d_lam.download(np.float64, n * 9).reshape(n, 9), oe.emdepth(x)[1])
    for b in (d_x, d_cells, d_lam):
        b.free()


def test_reference_vectors(ctx):
    for v, want in (([1, 8, 33, 34, 35, 37, 31, 22, 66], [0, 1, 2, 2, 2, 2, 2, 2, 4]),
                    ([30, 28, 33, 34, 35, 37, 31, 22, 38], [2] * 9),
                    ([296.6, 16.7, 17.0, 3019.2, 14.4, 16.5, 14.2, 26, 7], [9, 2, 2, 9, 2, 2, 2, 3, 1])):
        got, _ = ctx.emdepth(np.array([v], np.float32))
        assert list(got[0] & 15) == want


def test_mostly_zero_rows(ctx):
    """exome-like rows: the median is 0, bin 2 starts empty and lambda[2] comes from the fallback over bins 1..7"""
    rng = np.random.default_rng(8)
    n, S = 3000, 65
    x = rng.integers(0, 60, (n, S)).astype(np.float32)
    x[rng.random((n, S)) < 0.8] = 0
    x[::7] = 0
    x[1::7, :40] = 0
    x[2::7] = np.round(rng.random((n // 7 + 1, S)), 2)[: x[2::7].shape[0]]
    _check(ctx, x)
    assert ctx.emdepth_stats()["rows"] == n


def test_errors(ctx):
    with pytest.raises(capi.GlError):
        ctx.emdepth(np.ones((4, 2), np.float32))                       # S = 2
    for bad in (-1.0, np.inf, np.nan, -0.0, 2.0 ** 62):
        x = np.ones((10, 5), np.float32)
        x[6, 3] = bad
        with pytest.raises(capi.GlError) as ei:
            ctx.emdepth(x)
        assert ei.value.code == capi.GL_EINVAL and "row 6" in str(ei.value)
