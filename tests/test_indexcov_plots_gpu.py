"""indexcov's charts on the GPU (plot.cu): the device selection against the host mirror, the device index image against the
numpy restatement of the raster rule (tests/plot_rule.py) and, at cohort scale, against the host mirror; sample shards
drawn apart and max-combined against the whole."""
import numpy as np
import pytest

from goleft_b200 import capi
import plot_rule as pr

pytestmark = pytest.mark.gpu
W, H = capi.PLOT_W, capi.PLOT_H


def _series(rng, S, T, ties=False, empty=None):
    base = rng.normal(1.0, 0.15, T).astype(np.float32)
    vals = []
    for k in range(S):
        v = base.copy() if ties else rng.normal(1.0, 0.2, T).astype(np.float32)
        if not ties:
            v[rng.random(T) < 0.01] = rng.uniform(2.6, 4.0)           # clipped at 2.5: jumps across the data area
            v[:int(rng.integers(0, 4))] = 0
        if empty is not None and k == empty:
            v[:] = 0
        vals.append(np.maximum(v, 0))
    return vals


def _flat(vals):
    off = np.concatenate([[0], np.cumsum([len(v) for v in vals])[:-1]]).astype(np.int64)
    return np.concatenate(vals), off, np.array([len(v) for v in vals], np.int64)


def _device_chart(ctx, vals):
    flat, off, ln = _flat(vals)
    sel, yext = ctx.plot_select(flat, off, ln)
    hs, hy = capi.plot_select_host(flat, off, ln)
    assert np.array_equal(sel, hs) and np.array_equal(yext, hy)
    _, ext = pr.series_lines(vals)
    xf = pr.transform(*ext, W, H)
    r = pr.line_radius(len(vals))
    img = ctx.plot_raster_series(flat, off, sel, 16384.0, np.zeros(len(vals)), np.arange(1, len(vals) + 1), xf, 1, W, H, r)[0]
    return img, xf, r, (flat, off, sel)


@pytest.mark.parametrize("S,ties", [(1, False), (2, False), (31, False), (101, False), (101, True)])
def test_device_image_equals_numpy(S, ties):
    rng = np.random.default_rng(S + 7 * ties)
    vals = _series(rng, S, 40, ties=ties, empty=1 if S > 1 else None)
    with capi.Ctx(0) as ctx:
        img, xf, r, _ = _device_chart(ctx, vals)
    lines, _ = pr.series_lines(vals)
    assert np.array_equal(img, pr.raster(lines, xf, W, H, r))
    if ties:
        assert set(np.unique(img)) <= {0, S}                      # identical lines: the last sample shows everywhere


def test_device_xy_equals_numpy_with_exact_r_and_zero_length():
    # a segment at Y = 2.0 with r = 1.5 puts pixel centres at distance exactly r; a repeated vertex is a zero-length segment
    xs, ys = [2.5, 7.5, 7.5, 9.0], [4.0, 4.0, 4.0, 0.0]
    xf = np.array([0.0, 1.0, 0.0, 1.0])
    with capi.Ctx(0) as ctx:
        got = ctx.plot_raster_xy(xs, ys, [0, 4], [0], [3], xf, 1, 12, 6, 1.5)[0]
    assert np.array_equal(got, pr.raster([(3, xs, ys)], xf, 12, 6, 1.5))
    assert got[0, 4] == 3 and got[3, 4] == 3


@pytest.mark.parametrize("T,charts", [(15_000, 1), (191_000, 24)])
def test_cohort_scale_device_equals_host_mirror(T, charts):
    """2504 samples; the 191 k-tile shape is split over 24 references as a genome is"""
    S = 2504
    rng = np.random.default_rng(T)
    per = T // charts
    flat = rng.normal(1.0, 0.15, S * per * charts).astype(np.float32)
    flat[rng.random(flat.size) < 1e-4] = 3.0
    flat = np.maximum(flat, 0)
    n = S * charts
    off = (np.arange(n, dtype=np.int64) * per)
    ln = np.full(n, per, np.int64)
    ln[5] = 0
    flat[off[7]:off[7] + 30] = 0
    with capi.Ctx(0) as ctx:
        sel, yext = ctx.plot_select(flat, off, ln)
        hs, hy = capi.plot_select_host(flat, off, ln)
        assert np.array_equal(sel, hs) and np.array_equal(yext, hy)
        chart = np.repeat(np.arange(charts), S).astype(np.int32)           # dataset j = chart * S + sample
        draw = (np.arange(n) % S + 1).astype(np.uint32)
        xf = []
        for c in range(charts):
            s = sel[c * S:(c + 1) * S]
            d = s[:, 1] > 0
            x0 = (s[d, 0] * 16384.0).min()
            x1 = ((s[d, 0] + (s[d, 1] - 1) * s[d, 2]) * 16384.0).max()
            y = yext[c * S:(c + 1) * S][d]
            xf.append(pr.transform(x0, x1, float(y[:, 0].min()), float(y[:, 1].max()), W, H))
        xf = np.concatenate(xf)
        r = pr.line_radius(S)
        got = ctx.plot_raster_series(flat, off, sel, 16384.0, chart, draw, xf, charts, W, H, r)
        want = capi.plot_raster_series_host(flat, off, sel, 16384.0, chart, draw, xf, charts, W, H, r)
        assert np.array_equal(got, want)
        # sample shards drawn apart combine by max into the whole
        cut = 1000
        a = (np.arange(n) % S) < cut
        parts = [ctx.plot_raster_series(flat, off[m], sel[m], 16384.0, chart[m], draw[m], xf, charts, W, H, r) for m in (a, ~a)]
        assert np.array_equal(np.maximum(*parts), got)
    assert (got > 0).any()
