"""`goleft dcnv --chunk W` on the GPU (gl_dcnv_normalize_chunked[_device]) against the C oracle's literal ChunkDebiaser,
bit for bit: one chunk, chunks of one row, lengths either side of each bucket's limit (16 rows a thread, 1024 a warp, 65536
a 256-thread CTA, longer a 1024-thread CTA), zero-heavy, all-zero, negative and -0.0 chunks, ties, S = 1 and S > 1024,
column blocks, the device entry and a matrix of a few million rows."""
import numpy as np
import pytest

from goleft_b200 import capi
from oracle import dcnv_chunk as oc

pytestmark = pytest.mark.gpu

LIMITS = (16, 1024, 65536)


def _check(ctx, x, gc, w, **kw):
    want, inds, slices, med = oc.matrix(x, gc, w)
    got_inds = capi.go_argsort(gc)
    assert np.array_equal(got_inds, inds)
    ptr = capi.dcnv_chunk_slices(gc[got_inds], w)
    assert np.array_equal(ptr, slices)
    got, got_med = ctx.dcnv_normalize_chunked(x, got_inds, ptr, **kw)
    assert np.array_equal(got_med.view(np.uint64), med.view(np.uint64))
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    return got, ptr


def _depths(rng, n, S):
    x = np.empty((n, S), np.float64)
    for c in range(S):
        base = rng.gamma(4.0, 8.0, n)
        x[:, c] = np.floor(base) if c % 2 == 0 else np.round(base, 3)
    x[0, :] = 3                                                          # no all-zero sample
    return x


def _gc_of_lengths(rng, lengths):
    """GC values whose chunks under W = 0.5 have the given lengths (chunk j holds the value j), rows shuffled"""
    gc = np.repeat(np.arange(len(lengths), dtype=np.float64), lengths)
    return gc[rng.permutation(gc.size)]


def test_one_chunk(ctx):
    rng = np.random.default_rng(1)
    n, S = 5000, 7
    gc = rng.integers(0, 300, n) / 300.0
    _, ptr = _check(ctx, _depths(rng, n, S), gc, 2.0)
    assert ptr.size == 2


@pytest.mark.parametrize("n", [1, 2, 5, 100_003])
def test_every_chunk_one_row(ctx, n):
    rng = np.random.default_rng(n)
    gc = rng.permutation(n) / max(n, 1)                                  # distinct, as BED-mode rows often are
    x = _depths(rng, n, 3)
    x[rng.random(n) < 0.1, 1] = 0
    x[0, 1] = 2
    _, ptr = _check(ctx, x, gc, 1e-12)
    assert ptr.size == n + 1


def test_lengths_either_side_of_each_limit(ctx):
    rng = np.random.default_rng(2)
    lengths = [1, 2, 3]
    for L in LIMITS:
        lengths += [L - 1, L, L + 1]
    lengths += [4, 700, 200_001, 9, 31, 33]
    gc = _gc_of_lengths(rng, rng.permutation(lengths))
    n = gc.size
    x = _depths(rng, n, 5)
    x[rng.random(n) < 0.3, 2] = 0
    x[rng.random(n) < 0.6, 3] = 0
    _, ptr = _check(ctx, x, gc, 0.5)
    assert sorted(np.diff(ptr).tolist()) == sorted(lengths)


def test_zeros_negatives_and_ties(ctx):
    """per chunk: zero-heavy (the median among the zeros, left alone), all zero, negatives (k = 0), -0.0, and few values"""
    rng = np.random.default_rng(3)
    lengths = [5, 17, 40, 1500, 3000, 70_000, 12, 2048]
    gc = _gc_of_lengths(rng, lengths)
    n, S = gc.size, 8
    x = _depths(rng, n, S)
    x[rng.random(n) < 0.55, 0] = 0                                       # about half zero: some medians are zeros
    x[rng.random(n) < 0.8, 1] = 0
    x[:, 2] = 0
    x[::7, 2] = 5                                                        # sparse: most chunks left alone
    x[::13, 3] = -rng.integers(1, 20, x[::13, 3].size)                   # negatives: k = 0
    x[rng.random(n) < 0.4, 3] = 0
    x[rng.random(n) < 0.5, 4] = -0.0                                     # -0.0 counts as a zero and keeps its sign
    x[:, 5] = rng.integers(0, 3, n)                                      # heavy ties of tiny integers
    x[:, 6] = 7.0                                                        # one value
    x[rng.random(n) < 0.3, 7] = -0.0
    x[rng.random(n) < 0.3, 7] = 0.0
    x[0, :] = 3
    got, _ = _check(ctx, x, gc, 0.5)
    assert np.signbit(got[x[:, 4] == 0, 4]).any()
    inds = capi.go_argsort(gc)
    ptr = capi.dcnv_chunk_slices(gc[inds], 0.5)
    z = x.copy()
    z[:, 3] = 0                                                          # an all-zero sample: GL_ERANGE naming it
    with pytest.raises(capi.GlError) as ei:
        ctx.dcnv_normalize_chunked(z, inds, ptr)
    assert ei.value.code == capi.GL_ERANGE and "column 3 is all zero" in str(ei.value)
    with pytest.raises(oc.Panic):
        oc.matrix(z, gc, 0.5)


@pytest.mark.parametrize("S", [1, 1100])
def test_sample_counts(ctx, S):
    rng = np.random.default_rng(S)
    lengths = [1, 16, 17, 300, 1025, 4000, 3, 9]
    gc = _gc_of_lengths(rng, lengths)
    x = _depths(rng, gc.size, S)
    x[rng.random(x.shape) < 0.2] = 0
    x[0, :] = 3
    _check(ctx, x, gc, 0.5)


def test_column_blocks_and_device_entry(ctx):
    rng = np.random.default_rng(9)
    n, S = 60_000, 37
    gc = rng.integers(0, 400, n) / 400.0
    x = _depths(rng, n, S)
    x[rng.random(x.shape) < 0.3] = 0
    x[0, :] = 3
    whole, ptr = _check(ctx, x, gc, 0.01)
    inds = capi.go_argsort(gc)
    med = ctx.dcnv_normalize_chunked(x, inds, ptr)[1]
    for bc in (1, 5, 16):
        got, gm = ctx.dcnv_normalize_chunked(x, inds, ptr, block_cols=bc)
        assert np.array_equal(got.view(np.uint64), whole.view(np.uint64)) and np.array_equal(gm, med)
    got, gm = ctx.dcnv_normalize_chunked(x, inds, ptr, c0=7, c1=30, block_cols=4)
    assert np.array_equal(got, whole[:, 7:30]) and np.array_equal(gm, med[7:30])
    d_x, d_inds = ctx.dev_array(x), ctx.dev_array(inds)
    d_out, d_med = ctx.dev_empty(n * 40 * 8), ctx.dev_empty(40 * 8)
    ctx.dcnv_normalize_chunked_device(d_x, n, S, d_inds, ptr, 3, 35, d_out, 40, d_med)
    out = d_out.download(np.float64, n * 40).reshape(n, 40)
    assert np.array_equal(out[:, :32], whole[:, 3:35]) and np.array_equal(d_med.download(np.float64, 32), med[3:35])
    for b in (d_x, d_inds, d_out, d_med):
        b.free()


def test_bad_arguments(ctx):
    x = np.ones((6, 2))
    inds = np.arange(6)
    for ptr in ([0, 6, 6], [1, 6], [0, 5], [0, 3, 2, 6], [0], [0, 7]):
        with pytest.raises(capi.GlError):
            ctx.dcnv_normalize_chunked(x, inds, np.array(ptr))
    with pytest.raises(capi.GlError):
        ctx.dcnv_normalize_chunked(x, np.array([0, 1, 2, 3, 4, 4]), np.array([0, 6]))      # not a permutation


def test_a_few_million_rows(ctx):
    """the benchmark's row count, GC fractions of 1000-base windows (heavy ties), four samples, two window sizes"""
    rng = np.random.default_rng(10)
    n, S = 3_088_281, 4
    gc = rng.binomial(1000, 0.41, n) / 1000.0
    x = np.floor(rng.gamma(4.0, 8.0, (n, S)))
    x[rng.random((n, S)) < 0.05] = 0
    for w in (0.01, 1e-9):
        _check(ctx, x, gc, w)
