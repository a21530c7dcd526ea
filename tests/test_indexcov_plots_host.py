"""indexcov's charts, host side: the point selection, the raster rule's host mirror, the frame's ticks, labels and font,
and the PNG writer (plot.cu), each against a restatement in Python (tests/plot_rule.py)."""
import struct
import zlib

import numpy as np
import pytest

from goleft_b200 import capi
import plot_rule as pr


def _cohort(rng, lens, lead=None, nan_at=None):
    vals, off, ln = [], [], []
    pos = 0
    for k, n in enumerate(lens):
        v = rng.uniform(0, 3, n).astype(np.float32)
        v[rng.random(n) < 0.05] = 0
        if lead is not None:
            v[:min(n, lead[k])] = 0
            if lead[k] < n:
                v[lead[k]] = 1.5                                    # the skip ends exactly there
        if nan_at is not None and nan_at[k] is not None and nan_at[k] < n:
            v[nan_at[k]] = np.nan
        vals.append(v); off.append(pos); ln.append(n); pos += n
    return vals, np.concatenate(vals) if vals else np.zeros(0, np.float32), np.array(off), np.array(ln)


def test_select_matches_asvalues_and_sample():
    rng = np.random.default_rng(1)
    # n after the skip straddles every thinning boundary; leading zeros, an all-zero and an empty dataset
    lens = [999 + 7, 1000 + 3, 1001 + 3, 2000 + 5, 2001 + 5, 40, 50, 0, 3000, 1200, 700]
    lead = [7, 3, 3, 5, 5, 0, 50, 0, 0, 0, 0]
    nan_at = [None, None, None, None, None, None, None, None, 21, 15, 300]   # thinned-out / kept / stride-1 NaN
    vals, flat, off, ln = _cohort(rng, lens, lead, nan_at)
    sel, yext = capi.plot_select_host(flat, off, ln)
    for k, v in enumerate(vals):
        first, m, stride, lo, hi = pr.select(v)
        assert tuple(sel[k]) == (first, m, stride), k
        assert (float(yext[k, 0]), float(yext[k, 1])) == (lo, hi), k
    assert [tuple(sel[k][1:]) for k in range(5)] == [(999, 1), (1000, 1), (201, 5), (400, 5), (201, 10)]
    assert sel[6][1] == 0 and sel[7][1] == 0                    # all zero, empty
    assert sel[8][1] == 300                                      # NaN at post-skip position 21: thinned away (p % 10 == 0 kept)
    assert sel[9][1] == 0 and sel[10][1] == 0                    # NaN kept by stride 5, NaN at stride 1: not drawn


def test_leading_nan_ends_the_skip():
    v = np.array([0, 0, np.nan, 0, 1], np.float32)
    sel, _ = capi.plot_select_host(v, [0], [5])
    assert tuple(sel[0]) == (2, 0, 1)                            # first = the NaN; a NaN left in: not drawn


@pytest.mark.parametrize("v,want", [(0, "0.0"), (9999, "9999.0"), (10000, "10000.0"), (10001, "10.0KB"), (2000000, "2000.0KB"),
                                    (2000001, "2MB"), (2500000, "2.5MB"), (150000000, "150MB"), (123456789, "123.5MB")])
def test_make_millions(v, want):
    assert capi.plot_millions(v) == want


@pytest.mark.parametrize("lo,hi", [(0, 1), (0, 2.5), (0.3, 1.7), (0, 248_000_000), (16384, 3_000_000), (-3, 7), (0, 0.04), (5, 5.5)])
def test_ticks(lo, hi):
    t = capi.plot_ticks(lo, hi)
    assert 3 <= len(t) <= 8
    assert t[0] >= lo and t[-1] <= hi
    step = t[1] - t[0]
    e = np.floor(np.log10(step))
    m = step / 10 ** e
    assert min(abs(m - c) for c in (1, 2, 5, 10)) < 1e-9
    assert np.allclose(np.diff(t), step)
    smaller = {1: 0.5, 2: 1, 5: 2, 10: 5}[min((1, 2, 5, 10), key=lambda c: abs(m - c))] * 10 ** e
    assert np.floor(hi / smaller) - np.ceil(lo / smaller) + 1 > 8     # the smallest step that fits


def test_font_covers_printable_ascii():
    for c in range(0x21, 0x7F):
        rgb = np.full((9, 7, 3), 255, np.uint8)
        capi.plot_text(rgb, 1, 1, chr(c))
        ink = rgb[..., 0] == 0
        assert ink.any(), hex(c)
        assert not ink[0].any() and not ink[8].any() and not ink[:, 0].any() and not ink[:, 6].any()
    rgb = np.full((9, 7, 3), 255, np.uint8)
    capi.plot_text(rgb, 1, 1, " ")
    assert (rgb == 255).all()
    glyphs = set()
    for c in range(0x20, 0x7F):
        rgb = np.full((7, 5, 3), 255, np.uint8)
        glyphs.add(capi.plot_text(rgb, 0, 0, chr(c)).tobytes())
    assert len(glyphs) == 95


def _chunks(png):
    assert png[:8] == b"\x89PNG\r\n\x1a\n"
    p, out = 8, []
    while p < len(png):
        n, = struct.unpack(">I", png[p:p + 4])
        t, data = png[p + 4:p + 8], png[p + 8:p + 8 + n]
        crc, = struct.unpack(">I", png[p + 8 + n:p + 12 + n])
        assert crc == zlib.crc32(t + data), t
        out.append((t, data))
        p += 12 + n
    return out


def test_png_round_trip():
    rng = np.random.default_rng(2)
    rgb = rng.integers(0, 256, (37, 53, 3), dtype=np.uint8)
    png = capi.plot_png(rgb)
    ch = _chunks(png)
    assert [t for t, _ in ch] == [b"IHDR", b"IDAT", b"IEND"]
    assert ch[0][1] == struct.pack(">IIBBBBB", 53, 37, 8, 2, 0, 0, 0)
    raw = zlib.decompress(ch[1][1])
    rows = np.frombuffer(raw, np.uint8).reshape(37, 53 * 3 + 1)
    assert (rows[:, 0] == 0).all()
    assert np.array_equal(rows[:, 1:].reshape(37, 53, 3), rgb)
    assert capi.plot_png(rgb) == png


def test_colors():
    assert capi.plot_color(0, 3) == (180, 180, 180) and capi.plot_color(2, 3) == (180, 180, 180)
    assert capi.plot_color(3, 3) == capi.plot_color(3, 0)
    cs = {capi.plot_color(k) for k in range(200)}
    assert len(cs) > 190 and all(max(c) <= 220 for c in cs)


def test_transform_and_radius():
    assert np.array_equal(capi.plot_transform([0, 10, 2, 2], 100, 50), pr.transform(0, 10, 2, 2, 100, 50))
    assert np.array_equal(capi.plot_transform([3, 3, 0, 2.5], 316, 244), pr.transform(3, 3, 0, 2.5, 316, 244))
    assert capi.plot_line_radius(30) == pr.line_radius(30) and capi.plot_line_radius(31) == pr.line_radius(31)


def _xy_case(rng, S, W, H, special=False):
    lines = []
    for k in range(S):
        m = int(rng.integers(0, 12))
        xs = np.sort(rng.uniform(0, 100, m)).tolist()
        ys = rng.uniform(0, 2.5, m).tolist()
        if special and m > 3:
            xs[1] = xs[2]; ys[1] = ys[2]                            # zero-length segment
            ys[3] = 2.5 if ys[2] < 1.25 else 0.0                     # a jump across the data area
        lines.append((k + 1, xs, ys))
    xs_all = [x for _, xs, _ in lines for x in xs]
    ys_all = [y for _, _, ys in lines for y in ys]
    ext = [min(xs_all), max(xs_all), min(ys_all), max(ys_all)] if xs_all else [0, 0, 0, 0]
    return lines, pr.transform(*ext, W, H)


@pytest.mark.parametrize("seed", range(6))
def test_host_raster_equals_numpy(seed):
    rng = np.random.default_rng(10 + seed)
    W, H = int(rng.integers(20, 90)), int(rng.integers(15, 70))
    charts = [_xy_case(rng, int(rng.integers(1, 40)), W, H, special=seed % 2 == 0) for _ in range(3)]
    x, y, ptr, chart, draw, xf = [], [], [0], [], [], []
    for c, (lines, f) in enumerate(charts):
        for idx, xs, ys in lines:
            x += xs; y += ys; ptr.append(ptr[-1] + len(xs)); chart.append(c); draw.append(idx)
        xf += f.tolist()
    r = pr.line_radius(len(draw)) if seed < 3 else 1.5
    got = capi.plot_raster_xy_host(x, y, ptr, chart, draw, xf, len(charts), W, H, r)
    for c, (lines, f) in enumerate(charts):
        assert np.array_equal(got[c], pr.raster(lines, f, W, H, r)), c


def test_pixel_centre_at_exactly_r():
    # a horizontal segment at Y = 2.0 and r = 1.5: centres at distance 1.5 (j = 0 and j = 3) are covered, 1.5 + tiny is not
    W, H = 10, 6
    xf = np.array([0.0, 1.0, 0.0, 1.0])
    img = capi.plot_raster_xy_host([2.5, 7.5], [4.0, 4.0], [0, 2], [0], [1], xf, 1, W, H, 1.5)[0]
    assert np.array_equal(img, pr.raster([(1, [2.5, 7.5], [4.0, 4.0])], xf, W, H, 1.5))
    assert img[0, 4] == 1 and img[3, 4] == 1 and img[4, 4] == 0
    assert img[1, 1] == 1 and img[1, 8] == 1 and img[1, 0] == 0 and img[1, 9] == 0   # round end caps of radius r


def test_series_host_raster_equals_numpy():
    rng = np.random.default_rng(5)
    lens = [1500, 2500, 800, 60, 0, 1200]
    vals, flat, off, ln = _cohort(rng, lens, [0, 100, 5, 60, 0, 0])
    sel, yext = capi.plot_select_host(flat, off, ln)
    lines, ext = pr.series_lines(vals)
    W, H = capi.PLOT_W, capi.PLOT_H
    xf = pr.transform(*ext, W, H)
    r = pr.line_radius(len(vals))
    got = capi.plot_raster_series_host(flat, off, sel, 16384.0, np.zeros(len(vals)), np.arange(1, len(vals) + 1), xf, 1, W, H, r)
    assert np.array_equal(got[0], pr.raster(lines, xf, W, H, r))


def test_compose_places_the_data_area():
    rng = np.random.default_rng(7)
    img = rng.integers(0, 4, (capi.PLOT_H, capi.PLOT_W)).astype(np.uint32)
    pal = np.array([[255, 255, 255], [10, 20, 30], [40, 50, 60], [70, 80, 90]], np.uint8)
    rgb = capi.plot_compose(img, pal, capi.PLOT_DEPTH, [0, 3e6, 0, 2.5], "position on 1", "scaled coverage")
    area = rgb[capi.PLOT_AY:capi.PLOT_AY + capi.PLOT_H, capi.PLOT_AX:capi.PLOT_AX + capi.PLOT_W]
    assert np.array_equal(area, pal[img])
    assert (rgb[capi.PLOT_AY:capi.PLOT_AY + capi.PLOT_H + 1, capi.PLOT_AX - 1] == 0).all()   # the y axis
    assert (rgb[:, :capi.PLOT_AX - 1] == 0).any()                                               # tick labels and title


@pytest.mark.parametrize("S,D", [(3, 5), (40, 700), (101, 64)])
def test_pca_total_gives_numpy_vars(S, D):
    """gonum's normalised vars = s_k^2 / sum s^2 of the centred byte matrix; the total comes exactly from the bytes"""
    rng = np.random.default_rng(S * D)
    ld = (D + 63) // 64 * 64
    x = np.zeros((S, ld), np.uint8)
    x[:, :D] = rng.integers(0, 256, (S, D))
    total = C_total(x, ld, S, D)
    xc = x[:, :D].astype(np.float64)
    xc -= xc.mean(axis=0)
    s = np.linalg.svd(xc, compute_uv=False)
    assert np.allclose(s ** 2 / total, s ** 2 / (s ** 2).sum(), rtol=1e-10, atol=0)
    colsum = x[:, :D].astype(object).sum(axis=0)
    exact = sum(S * int((x[:, j].astype(np.int64) ** 2).sum()) - int(colsum[j]) ** 2 for j in range(D))
    assert total == exact / S


def C_total(x, ld, S, D):
    import ctypes as C
    t = C.c_double()
    assert capi.lib.gl_indexcov_pca_total(x.ctypes.data_as(C.c_void_p), ld, S, D, C.byref(t)) == 0
    return t.value
