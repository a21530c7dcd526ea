"""The depthwed cells on the device (depth_text.cu): gl_depthwed_cells against a Python restatement of `goleft depth` then
`goleft depthwed` (int(0.5 + float('%.4g' % (sum / len))) per window, grouped by the oracle's depthwed), and
gl_depthwed_add_column after a reduce against gl_depthwed_cells of the same windows, on every depth path and across two
passes whose boundary falls inside a group."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from goleft_b200 import capi, synth  # noqa: E402
from oracle import loader as orc  # noqa: E402

pytestmark = pytest.mark.gpu


def cell_ref(s, l):
    """what depthwed.go:103 makes of the row depth.go prints: Python's %.4g rounds half-even on the exact double, as Go does"""
    if s <= 0 or l <= 0:
        return 0
    return int(0.5 + float("%.4g" % (s / l)))


def grouped_ref(sums, lens, size):
    """rows of 10 bases on one contig holding these windows: the oracle's depthwed over the parsed means, and the row -> group
    map gl_depthwed_plan gives"""
    R = len(sums)
    starts = np.arange(R, dtype=np.int32) * 10
    ends = starts + 10
    means = np.array([[float("%.4g" % (s / l)) if s > 0 and l > 0 else 0.0 for s, l in zip(sums, lens)]])
    o_s, o_e, o_c, out = orc.depthwed(means, starts, ends, np.zeros(R, np.int32), size)
    first, *_ = capi.depthwed_plan(starts, ends, np.zeros(R, np.int32), size)
    grp = np.repeat(np.arange(first.size - 1, dtype=np.int32), np.diff(first))
    return out[:, 0], grp


@pytest.fixture(scope="module")
def ctx():
    if capi.device_count() < 1:
        pytest.skip("no CUDA device")
    with capi.Ctx(0) as c:
        yield c


def check(ctx, sums, lens, size=1):
    sums, lens = np.asarray(sums, np.int64), np.asarray(lens, np.int64)
    one = ctx.depthwed_cells(sums, lens)
    assert one.tolist() == [cell_ref(int(s), int(l)) for s, l in zip(sums, lens)]
    exp, grp = grouped_ref(sums, lens, size)
    got = ctx.depthwed_cells(sums, lens, grp, int(grp.max()) + 1 if grp.size else 0)
    assert np.array_equal(got, exp)
    return got


def test_seeded_random(ctx):
    rng = np.random.default_rng(11)
    lens = rng.integers(1, 2000, 20000)
    sums = (lens * rng.gamma(2.0, 20.0, lens.size)).astype(np.int64)
    sums[rng.random(lens.size) < 0.05] = 0
    for size in (1, 70, 500, 10**7):
        check(ctx, sums, lens, size)


def test_ties_and_decade_edges(ctx):
    pairs = [(1, 2), (3, 2), (5, 2), (247, 2), (1999, 2), (19999, 2), (199999, 2), (1999999, 2),   # .5 ties and 9999.5 / 99999.5
             (4999, 10000), (5000, 10000), (5001, 10000), (49999, 100000), (1, 8), (97, 8), (12125, 1000),
             (9999, 1), (10000, 1), (10001, 1), (10005, 1), (10015, 1), (99985, 1), (99995, 1), (123456, 10), (999950, 1),
             (99999, 1), (100000, 1), (123456789, 1), (987654321987, 1000)]
    sums, lens = zip(*pairs)
    got = check(ctx, sums, lens)
    assert got.tolist()[:8] == [1, 2, 3, 124, 1000, 10000, 100000, 1000000]
    assert dict(zip(pairs, got.tolist()))[(123456, 10)] == 12350              # 12345.6 prints 1.235e+04


def test_small_means_and_zero(ctx):
    sums = [0, 0, 1, 1, 3, 7, 1, -5]
    lens = [1, 0, 2**31 - 1, 100000, 100000, 20000, 3, 10]
    got = check(ctx, sums, lens)
    assert got.tolist() == [0, 0, 0, 0, 0, 0, 0, 0]


def test_group_sums_past_int32(ctx):
    lens = np.full(40, 1000, np.int64)
    sums = lens * 900_000_000
    got = check(ctx, sums, lens, size=200)
    assert got.tolist() == [18 * 10**9, 18 * 10**9]


def test_range_errors(ctx):
    with pytest.raises(capi.GlError):
        ctx.depthwed_cells([2**53], [1])
    with pytest.raises(capi.GlError):
        ctx.depthwed_cells([10**16], [2])
    with pytest.raises(capi.GlError):
        ctx.depthwed_cells([1, 2], [1, 1], [0, 3], 2)


def _segments(L, seed):
    s, e = synth.segments(synth.reads(L, coverage=25.0, contig_index=seed))
    return np.asarray(s, np.int32), np.asarray(e, np.int32)


def _column(ctx, passes, segs, W, grp, G, packed8=False):
    """the device column after one reduce per pass [ps, pe)"""
    d_map = capi.DevBuf(ctx, max(16, grp.nbytes)).upload(grp)
    d_col = capi.DevBuf(ctx, max(16, G * 8))
    d_32 = capi.DevBuf(ctx, max(16, G * 4))
    d_ovf = capi.DevBuf(ctx, 16)
    try:
        ctx.depthwed_column_begin(d_col, G)
        s, e = segs
        for ps, pe in passes:
            ctx.depth_begin(ps, pe)
            if packed8:
                ctx.depth_add_segments_packed8(*capi.pack_segments8(s, e))
            else:
                ctx.depth_add_segments(s, e)
            ctx.depth_reduce(W, 4, 0, 0)
            ctx.depthwed_add_column(ps // W, d_map, d_col)
        ctx.depthwed_column_i32(d_col, G, d_32, d_ovf)
        col = d_col.download(np.int64, G)
        assert d_ovf.download(np.int32, 1)[0] == int(col.max(initial=0) > 2**31 - 1)
        if col.max(initial=0) <= 2**31 - 1:
            assert np.array_equal(d_32.download(np.int32, G), col)
        return col
    finally:
        for b in (d_map, d_col, d_32, d_ovf):
            b.free()


def _explicit(ctx, L, segs, W, size):
    """window sums of one whole reduce, their lengths and groups, and gl_depthwed_cells of them"""
    ctx.depth_set_path(0)
    ctx.depth_begin(0, L)
    ctx.depth_add_segments(*segs)
    ctx.depth_reduce(W, 4, 0, 0)
    sums = ctx.depth_get_windows()
    n = sums.size
    starts = np.arange(n, dtype=np.int64) * W
    ends = np.minimum(starts + W, L)
    first, *_ = capi.depthwed_plan(starts, ends, np.zeros(n, np.int32), size)
    grp = np.repeat(np.arange(first.size - 1, dtype=np.int32), np.diff(first))
    G = first.size - 1
    exp = ctx.depthwed_cells(sums, ends - starts, grp, G)
    depth = orc.pileup_diff(segs[0], segs[1], 0, L)
    ws, _ = orc.window_sums(depth, 0, L, W)
    assert np.array_equal(sums, ws)
    assert np.array_equal(exp, np.bincount(grp, [cell_ref(int(a), int(b)) for a, b in zip(ws, ends - starts)], G).astype(np.int64))
    return grp, G, exp


@pytest.mark.parametrize("path", [0, 1, 2, 4, "packed8"])
@pytest.mark.parametrize("W, size", [(250, 250), (100, 1000), (37, 500), (2001, 10**6)])
def test_device_column_every_path(ctx, path, W, size):
    L = 200_003
    segs = _segments(L, 3)
    grp, G, exp = _explicit(ctx, L, segs, W, size)
    try:
        ctx.depth_set_path(0 if path == "packed8" else path)
        got = _column(ctx, [(0, L)], segs, W, grp, G, packed8=path == "packed8")
        if path == "packed8":
            assert ctx.depth_last_path() == 3
        elif path:
            assert ctx.depth_last_path() == path
    finally:
        ctx.depth_set_path(0)
    assert np.array_equal(got, exp)


@pytest.mark.parametrize("path", [0, 4])
def test_two_passes_group_straddles(ctx, path):
    """[0, P) and [P, L) reduced apart, P a multiple of W inside a group of 10 windows: the group gets both parts"""
    L, W, size, P = 120_000, 100, 1000, 53_300
    segs = _segments(L, 4)
    grp, G, exp = _explicit(ctx, L, segs, W, size)
    assert grp[P // W - 1] == grp[P // W]
    try:
        ctx.depth_set_path(path)
        got = _column(ctx, [(0, P), (P, L)], segs, W, grp, G)
    finally:
        ctx.depth_set_path(0)
    assert np.array_equal(got, exp)


def test_device_column_past_int32(ctx):
    """a deep pile-up in one group of a huge SIZE: the int64 column holds it and the narrowing reports the overflow"""
    L, W = 40_000, 1
    s = np.zeros(70_000, np.int32)
    e = np.full(70_000, L, np.int32)
    grp = np.zeros(L // W, np.int32)
    got = _column(ctx, [(0, L)], (s, e), W, grp, 1)
    assert got.tolist() == [70_000 * 40_000]


def test_add_column_errors(ctx):
    d = capi.DevBuf(ctx, 64)
    try:
        ctx.depth_begin(50, 1000)
        ctx.depth_add_segments(np.array([60], np.int32), np.array([90], np.int32))
        ctx.depth_reduce(100, 4, 0, 0)
        with pytest.raises(capi.GlError):
            ctx.depthwed_add_column(0, d, d)                                  # region start not a multiple of W
    finally:
        d.free()
