"""`goleft dcnv` on the GPU (gl_dcnv_normalize, gl_format_f2) against the C oracle, bit for bit."""
import numpy as np
import pytest

from goleft_b200 import capi
from oracle import dcnv as od

pytestmark = pytest.mark.gpu


def _matrix(rng, n, S):
    """tie-heavy GC; even columns integer (what depthwed writes), odd columns fractional; a few rows below 1"""
    gc = rng.integers(0, 300, n) / 300.0
    x = np.empty((n, S), np.float64)
    for c in range(S):
        base = rng.gamma(4.0, 8.0, n)
        x[:, c] = np.floor(base) if c % 2 == 0 else np.round(base, 3)
        x[rng.integers(0, n, max(1, n // 50)), c] = 0.5
    if (x == 0).all(axis=0).any():
        x[0, :] = 3
    return x, gc


def _check(ctx, x, gc, **kw):
    want, inds, med = od.matrix(x, gc)
    got_inds = capi.go_argsort(gc)
    assert np.array_equal(got_inds, inds)
    got, got_med = ctx.dcnv_normalize(x, got_inds, **kw)
    assert np.array_equal(got_med.view(np.uint64), med.view(np.uint64))
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    return got


@pytest.mark.parametrize("n", [5, 6, 9, 10, 11, 12, 13, 14, 20, 1000, (1 << 20) + 7])
@pytest.mark.parametrize("S", [1, 3, 33, 128])
def test_matches_oracle(ctx, n, S):
    rng = np.random.default_rng(n * 1000 + S)
    x, gc = _matrix(rng, n, S)
    if S == 1 and n % 2:
        x[:, 0] = np.round(rng.gamma(4.0, 8.0, n), 2)                  # a lone fractional column
    _check(ctx, x, gc)


def test_exome_zeros_and_negatives(ctx):
    rng = np.random.default_rng(5)
    n, S = 20_000, 6
    x, gc = _matrix(rng, n, S)
    for c in (0, 1, 2):                                                # exome-like: most rows are zero
        x[rng.random(n) < 0.7 + 0.1 * c, c] = 0
    x[::97, 3] = -rng.integers(1, 20, x[::97, 3].size)                 # negatives: k = 0, the median may be among the zeros
    x[rng.random(n) < 0.5, 3] = 0
    x[:, 4] = rng.integers(0, 3, n)                                    # medians and windows of tiny integers
    _check(ctx, x, gc)
    x[:, 5] = 0                                                        # all zero: the reference's median index is out of range
    with pytest.raises(capi.GlError) as ei:
        ctx.dcnv_normalize(x, capi.go_argsort(gc))
    assert ei.value.code == capi.GL_ERANGE and "column 5 is all zero" in str(ei.value)
    with pytest.raises(od.Panic):
        od.matrix(x, gc)


def test_column_blocks_equal_whole(ctx):
    rng = np.random.default_rng(9)
    x, gc = _matrix(rng, 50_000, 37)
    inds = capi.go_argsort(gc)
    whole, med = ctx.dcnv_normalize(x, inds)
    for bc in (1, 5, 16):
        got, gm = ctx.dcnv_normalize(x, inds, block_cols=bc)
        assert np.array_equal(got, whole) and np.array_equal(gm, med)
    got, gm = ctx.dcnv_normalize(x, inds, c0=7, c1=30, block_cols=4)
    assert np.array_equal(got, whole[:, 7:30]) and np.array_equal(gm, med[7:30])
    # the device entry on a column range of a resident matrix, into a wider output
    n, S = x.shape
    d_x = ctx.dev_array(x)
    d_inds = ctx.dev_array(inds)
    d_out = ctx.dev_empty(n * 40 * 8)
    d_med = ctx.dev_empty(40 * 8)
    ctx.dcnv_normalize_device(d_x, n, S, d_inds, 3, 35, d_out, 40, d_med)
    out = d_out.download(np.float64, n * 40).reshape(n, 40)
    assert np.array_equal(out[:, :32], whole[:, 3:35]) and np.array_equal(d_med.download(np.float64, 32), med[3:35])
    for b in (d_x, d_inds, d_out, d_med):
        b.free()


def test_bad_arguments(ctx):
    x = np.ones((4, 2))
    with pytest.raises(capi.GlError):
        ctx.dcnv_normalize(x, np.arange(4))                            # fewer than 5 rows
    x = np.ones((6, 2))
    with pytest.raises(capi.GlError):
        ctx.dcnv_normalize(x, np.array([0, 1, 2, 3, 4, 4]))            # not a permutation


def test_device_tokens_equal_host_mirror(ctx):
    rng = np.random.default_rng(4)
    x5 = (np.arange(0, 100_000) + 0.5) / 100.0
    v = np.concatenate([x5, np.nextafter(x5, 0), np.nextafter(x5, 10), -x5, 2.5 * 2.0 ** -np.arange(60),
                        rng.standard_normal(500_000) * 10.0 ** rng.integers(-6, 16, 500_000),
                        [0.0, -0.0, 5e-324, np.nan, np.inf, -np.inf, 1e15, 999999999999.995]])
    dev = ctx.format_f2(v)
    assert np.array_equal(dev, capi.format_f2_host(v))
    assert od.f2_mismatches(v, dev)[0] == 0


def test_normalised_text(ctx):
    """library path end to end (argsort, device normalisation, device tokens) equals the oracle's "%.2f" rows"""
    rng = np.random.default_rng(8)
    n, S = 3000, 5
    x, gc = _matrix(rng, n, S)
    starts = np.arange(n, dtype=np.int64) * 1000 + 250
    ends = starts + 750
    want, _, _ = od.matrix(x, gc)
    got, _ = ctx.dcnv_normalize(x, capi.go_argsort(gc))
    toks = capi.f2_text(ctx.format_f2(got), got)
    text = b"".join(b"chr1\t%d\t%d\t" % (s, e) + b"\t".join(toks[i * S:(i + 1) * S]) + b"\n" for i, (s, e) in enumerate(zip(starts, ends)))
    assert text == od.rows(b"chr1", starts, ends, want)
