"""`goleft dcnv`'s depth chart on the host: the selection (dcnv.go asValues, float64) and the stepped-line index image of the
host mirrors (gl_dcnv_chart_select_host, gl_dcnv_chart_raster_host) against a literal restatement here and the numpy raster
rule of tests/plot_rule.py, bit for bit, and row-block splits of both against the whole."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from goleft_b200 import capi  # noqa: E402
import plot_rule as pr  # noqa: E402

W, H = capi.PLOT_W, capi.PLOT_H
MULT = 16384.0


def as_values(col):
    """dcnv.go asValues: skip leading values == 0 (-0.0 too, not NaN); x = float64(i) * 16384, y = min(v, 2.5)"""
    xs, ys, seen = [], [], False
    for i, r in enumerate(col):
        if r == 0 and not seen:
            continue
        seen = True
        xs.append(float(i) * MULT)
        ys.append(2.5 if r > 2.5 else float(r))
    return xs, ys


def drawn(y):
    return not (y != y or y == -np.inf)


def expect_select(x):
    n, S = x.shape
    first, yext = np.full(S, n, np.int64), np.empty((S, 2))
    for k in range(S):
        xs, ys = as_values(x[:, k])
        if xs:
            first[k] = int(xs[0] / MULT)
        ok = [y + 0.0 if y == 0 else y for y in ys if drawn(y)]
        yext[k] = (min(ok), max(ok)) if ok else (np.inf, -np.inf)
    return first, yext


def step_lines(x):
    """[(S - k, xs, ys)]: every drawn step of every sample as its own three-vertex polyline"""
    n, S = x.shape
    lines = []
    for k in range(S):
        xs, ys = as_values(x[:, k])
        for j in range(len(xs) - 1):
            if drawn(ys[j]) and drawn(ys[j + 1]):
                lines.append((S - k, [xs[j], xs[j + 1], xs[j + 1]], [ys[j], ys[j], ys[j + 1]]))
    return lines


def expect_image(x, xf, r):
    return pr.raster(step_lines(x), xf, W, H, r)


def chart_host(x, r=None):
    first, yext = capi.dcnv_chart_select_host(x)
    ext = capi.dcnv_chart_extent(first, yext, x.shape[0])
    xf = capi.plot_transform(ext, W, H)
    return first, yext, ext, xf, capi.dcnv_chart_raster_host(x, first, xf, r=r)


def test_select_edges():
    nan, inf = np.nan, np.inf
    cols = [
        [0, 0, 0.5, 1.0, 2.0],                 # leading zeros
        [-0.0, 0.0, -0.0, 1.25, -0.0],         # -0.0 is skipped while leading, then a plotted 0
        [nan, 0, 1, 2, 3],                     # NaN is not zero: it is the first vertex, and not in the extent
        [0, 2.5, np.nextafter(2.5, 3), 3.0, inf],   # at 2.5 and just above: capped
        [0, -1.5, -1e300, 0.75, 1],            # negatives
        [0, 0, 0, 0, 4.0],                     # zero until the last row
        [0, 0, 0, 0, 0],                       # empty
        [0, -inf, nan, -inf, nan],             # vertices, but no drawn y
        [1e-300, 0, 0, 0, 0],
    ]
    x = np.array(cols, np.float64).T.copy()
    first, yext = capi.dcnv_chart_select_host(x)
    ef, ey = expect_select(x)
    assert first.tolist() == ef.tolist() == [2, 3, 0, 1, 1, 4, 5, 1, 0]
    assert np.array_equal(yext, ey)
    assert yext[1].tolist() == [0.0, 1.25] and not np.signbit(yext[1, 0])
    assert yext[3].tolist() == [2.5, 2.5] and yext[4].tolist() == [-1e300, 1.0]
    assert yext[6].tolist() == [np.inf, -np.inf] and yext[7].tolist() == [np.inf, -np.inf]
    ext = capi.dcnv_chart_extent(first, yext, x.shape[0])
    assert ext.tolist() == [0.0, 4 * MULT, -1e300, 2.5]
    # nothing to draw at all: a zero extent, which the transform widens
    z = np.zeros((6, 3))
    f, y = capi.dcnv_chart_select_host(z)
    assert f.tolist() == [6, 6, 6] and capi.dcnv_chart_extent(f, y, 6).tolist() == [0, 0, 0, 0]
    assert not capi.dcnv_chart_raster_host(z, f, capi.plot_transform([0, 0, 0, 0], W, H)).any()


@pytest.mark.parametrize("S", [1, 2, 31, 51])
def test_raster_against_numpy(S):
    rng = np.random.default_rng(S)
    n = 40
    x = rng.gamma(6.0, 1 / 6.0, (n, S))
    x[rng.random((n, S)) < 0.05] = 3.0
    for k in range(0, S, 3):
        x[: k % 9, k] = 0.0                               # leading zeros of several lengths
    if S > 1:
        x[:, S - 1] = 0.0
        x[n - 1, S - 1] = 1.0                             # a single vertex: nothing drawn
    if S > 2:
        x[5, 1] = np.nan                                   # the steps on both sides of it are not drawn
    first, yext, ext, xf, img = chart_host(x)
    assert np.array_equal(img, expect_image(x, xf, pr.line_radius(S)))
    assert img.any()
    assert set(np.unique(img)) <= set(range(S + 1))


@pytest.mark.parametrize("S", [1, 2, 31, 51])
def test_raster_pixel_centres_at_r(S):
    """y on sixteenths under sy = 16: horizontal runs on pixel edges, so the centres next to them are exactly r away"""
    rng = np.random.default_rng(100 + S)
    n = 30
    x = rng.integers(0, 40, (n, S)) / 16.0
    x[0] = 1.0
    first, _ = capi.dcnv_chart_select_host(x)
    xf = np.array([0.0, 8.0 / MULT, 0.0, 16.0])          # X = 8 i, Y = 244 - 16 y: both exact
    for r in (0.5, pr.line_radius(S)):
        got = capi.dcnv_chart_raster_host(x, first, xf, r=r)
        assert np.array_equal(got, expect_image(x, xf, r)), r
    # the radius decides: r = 0.5 covers both rows next to a run along a pixel edge, a hair less covers neither
    one = np.array([[1.0], [1.0], [1.0]])
    f1, _ = capi.dcnv_chart_select_host(one)
    a = capi.dcnv_chart_raster_host(one, f1, xf, r=0.5)
    b = capi.dcnv_chart_raster_host(one, f1, xf, r=np.nextafter(0.5, 0))
    row = H - 16
    assert a[row - 1, 2:14].all() and a[row, 2:14].all() and not b[row - 1:row + 1, 2:14].any()
    assert np.array_equal(a, expect_image(one, xf, 0.5)) and np.array_equal(b, expect_image(one, xf, np.nextafter(0.5, 0)))


def test_single_row_datasets():
    x = np.array([[0.0, 1.0, 0.0], [0.0, 2.0, 0.0], [3.0, 0.5, 0.0]])
    first, yext, ext, xf, img = chart_host(x)
    assert first.tolist() == [2, 0, 3]
    assert np.array_equal(img, expect_image(x, xf, pr.line_radius(3)))
    assert set(np.unique(img)) == {0, 2}                 # sample 0 has one vertex, sample 2 none


def split_select(x, bounds):
    """the select restated over row blocks [bounds[b], bounds[b+1]) in order, with the carried state"""
    n, S = x.shape
    first, lo, hi = np.full(S, n, np.int64), np.full(S, np.inf), np.full(S, -np.inf)
    for a, b in zip(bounds[:-1], bounds[1:]):
        for k in range(S):
            for i in range(a, b):
                if first[k] == n and x[i, k] != 0:
                    first[k] = i
                if i >= first[k]:
                    y = 2.5 if x[i, k] > 2.5 else x[i, k]
                    if drawn(y):
                        lo[k], hi[k] = min(lo[k], y + 0.0), max(hi[k], y + 0.0)
    return first, np.stack([lo, hi], 1)


def split_raster(x, first, xf, r, bounds):
    """the image as the sum (max) of row blocks that each hold their rows and the row before"""
    img = np.zeros((H, W), np.uint32)
    for a, b in zip(bounds[:-1], bounds[1:]):
        lo = max(a - 1, 0)
        sub = np.ascontiguousarray(x[lo:b])
        f = np.clip(first - lo, 0, None)
        sxf = xf.copy()
        sxf[0] -= lo * MULT                               # exact: every x and xmin are multiples of 16384
        img = np.maximum(img, capi.dcnv_chart_raster_host(sub, f, sxf, r=r))
    return img


@pytest.mark.parametrize("split", ["1", "7", "uneven"])
def test_row_blocks_equal_whole(split):
    rng = np.random.default_rng(7)
    n, S = 97, 5
    x = rng.gamma(5.0, 0.25, (n, S))
    x[:60, 0] = 0.0                                      # first row in a later block
    x[:, 1] = 0.0                                        # never drawn
    x[40, 2] = np.nan
    x[70, 3] = -np.inf
    bounds = {"1": list(range(n + 1)), "7": list(range(0, n, 7)) + [n], "uneven": [0, 1, 2, 13, 14, 60, 61, 96, 97]}[split]
    first, yext, ext, xf, img = chart_host(x)
    f2, y2 = split_select(x, bounds)
    assert np.array_equal(first, f2) and np.array_equal(yext, y2)
    r = pr.line_radius(S)
    assert np.array_equal(split_raster(x, first, xf, r, bounds), img)
    assert np.array_equal(img, expect_image(x, xf, r))
