"""indexcov's vector charts, host side: the path text's host mirror against a Python restatement of the point transform and
"%.2f" (tests/vector_rule.py), exact ties, the SVG and EPS documents, label escaping and the capacity checks (plot.cu)."""
import re
import xml.etree.ElementTree as ET

import numpy as np
import pytest

from goleft_b200 import capi
import plot_rule as pr
import vector_rule as vr


def _cohort(rng, lens, lead, nan_at):
    vals, off, pos = [], [], 0
    for k, n in enumerate(lens):
        v = rng.uniform(0, 3, n).astype(np.float32)
        v[rng.random(n) < 0.05] = 0
        v[:min(n, lead[k])] = 0
        if nan_at[k] is not None:
            v[nan_at[k]] = np.nan
        vals.append(v); off.append(pos); pos += n
    return vals, np.concatenate(vals), np.array(off, np.int64), np.array(lens, np.int64)


def _series_case(seed=3):
    rng = np.random.default_rng(seed)
    # after the skip: either side of 1000 and 2000; leading zeros; a kept NaN; one vertex; all zero
    lens = [999 + 4, 1001 + 9, 2000 + 2, 2001 + 30, 500, 1, 40, 3000]
    lead = [4, 9, 2, 30, 0, 0, 40, 11]
    nan_at = [None, None, None, None, 250, None, None, None]
    return _cohort(rng, lens, lead, nan_at)


def _expected(vals, xf, kind, fmt, mult=16384.0):
    out = []
    for v in vals:
        s = pr.sample(*pr.as_values(v, mult))
        out.append(b"" if s is None else vr.path_text(s[0], s[1], xf, kind, fmt))
    return out


@pytest.mark.parametrize("fmt", [vr.SVG, vr.EPS])
def test_series_paths_match_restatement(fmt):
    vals, flat, off, ln = _series_case()
    sel, yext = capi.plot_select_host(flat, off, ln)
    lines, ext = pr.series_lines(vals)
    xf = capi.plot_transform(ext, capi.PLOT_W, capi.PLOT_H)
    lens, text = capi.plot_path_series_host(flat, off, sel, 16384.0, np.zeros(len(vals), np.int32), xf, 1, capi.PLOT_DEPTH, fmt)
    want = _expected(vals, xf, 0, fmt)
    assert list(lens) == [len(w) for w in want]
    assert text == b"".join(want)
    assert lens[4] == 0 and lens[5] == 0 and lens[6] == 0             # a NaN kept, one vertex, all zero: not written
    assert all(lens[k] > 0 for k in (0, 1, 2, 3, 7))
    pos = np.concatenate([[0], np.cumsum(lens)])
    for k in (0, 3, 7):
        pts = vr.parse_path(text[pos[k]:pos[k + 1]], fmt)
        assert len(pts) == sel[k][1]


def test_two_charts_use_their_own_transform():
    vals, flat, off, ln = _series_case(5)
    sel, _ = capi.plot_select_host(flat, off, ln)
    chart = np.array([0, 1, 0, 1, 0, 1, 0, 1], np.int32)
    xf = np.concatenate([pr.transform(0, 5e7, 0, 2.5, capi.PLOT_W, capi.PLOT_H), pr.transform(1e6, 3e7, 0.5, 2.0, capi.PLOT_W, capi.PLOT_H)])
    lens, text = capi.plot_path_series_host(flat, off, sel, 16384.0, chart, xf, 2, capi.PLOT_PLAIN, vr.SVG)
    want = []
    for k, v in enumerate(vals):
        s = pr.sample(*pr.as_values(v, 16384.0))
        want.append(b"" if s is None else vr.path_text(s[0], s[1], xf[4 * chart[k]:4 * chart[k] + 4], 1, vr.SVG))
    assert text == b"".join(want)


def test_f2_ties_round_to_even_on_the_binary_value():
    # identity transform on the square canvas: Xpt = 0.75 * (56 + x).  With v = k / 8 for odd k divisible by 3, x = k / 6 - 56
    # and every step is exact, so Xpt is v, a float64 whose decimal expansion ends in an exact 5 at the third place
    ks = [3, 9, 15, 21, 27, 33, 45, 75, 801, 1605]
    ties = [k / 8 for k in ks]
    xf = np.array([0.0, 1.0, 0.0, 1.0])
    xs = [(k // 3) / 2 - 56 for k in ks]
    assert all(0.75 * (56 + x) == v for x, v in zip(xs, ties))
    ys = [float(j) for j in range(len(ks))]
    lens, text = capi.plot_path_xy_host(xs, ys, [0, len(xs)], [0], xf, 1, capi.PLOT_SQUARE, vr.SVG)
    assert text == vr.path_text(xs, ys, xf, 2, vr.SVG)
    got = [p[0] for p in vr.parse_path(text, vr.SVG)]
    assert got == ["%.2f" % v for v in ties]
    assert got[:4] == ["0.38", "1.12", "1.88", "2.62"]                  # ties to even, as printf does


@pytest.mark.parametrize("fmt", [vr.SVG, vr.EPS])
@pytest.mark.parametrize("kind", [0, 1, 2])
def test_xy_paths_match_restatement(kind, fmt):
    rng = np.random.default_rng(11 + kind)
    sizes = [0, 1, 2, 17, 999, 1001, 2003]
    xs = [rng.uniform(-3, 5, n) for n in sizes]
    ys = [rng.uniform(-1, 4, n) for n in sizes]
    ys[3][5] = np.nan                                                    # a NaN vertex: not written
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    W, H = vr.CANVAS[kind][:2]
    xf = pr.transform(-3, 5, -1, 4, W, H)
    lens, text = capi.plot_path_xy_host(np.concatenate(xs), np.concatenate(ys), ptr, np.zeros(len(sizes), np.int32), xf, 1, kind, fmt)
    want = [vr.path_text(list(x), list(y), xf, kind, fmt) for x, y in zip(xs, ys)]
    assert list(lens) == [len(w) for w in want]
    assert text == b"".join(want)
    assert lens[0] == lens[1] == lens[3] == 0


def test_undersized_buffers_are_rejected():
    vals, flat, off, ln = _series_case()
    sel, _ = capi.plot_select_host(flat, off, ln)
    xf = pr.transform(0, 5e7, 0, 2.5, capi.PLOT_W, capi.PLOT_H)
    lens, _ = capi.plot_path_series_host(flat, off, sel, 16384.0, np.zeros(len(vals), np.int32), xf, 1, 0, vr.SVG)
    with pytest.raises(capi.GlError) as e:
        capi.plot_path_series_host(flat, off, sel, 16384.0, np.zeros(len(vals), np.int32), xf, 1, 0, vr.SVG, cap=int(lens.sum()) - 1)
    assert e.value.code == capi.GL_ERANGE
    with pytest.raises(capi.GlError) as e:
        capi.plot_path_xy_host([0, 1, 2], [0, 1, 0], [0, 3], [0], xf, 1, 0, vr.EPS, cap=5)
    assert e.value.code == capi.GL_ERANGE
    with pytest.raises(capi.GlError) as e:                               # chart index out of range
        capi.plot_path_xy_host([0, 1], [0, 1], [0, 2], [1], xf, 1, 0, vr.EPS)
    assert e.value.code == capi.GL_EINVAL
    with pytest.raises(capi.GlError) as e:                               # unknown format
        capi.plot_path_xy_host([0, 1], [0, 1], [0, 2], [0], xf, 1, 0, 2)
    assert e.value.code == capi.GL_EINVAL


NASTY = 'chr<1> & "x" (y) \\z'


def _doc(tmp_path, fmt, kind=1):
    xs = [[0.0, 0.5, 1.0], [0.0, 1.0], [0.2, 0.8, 0.4, 0.9]]
    ys = [[0.0, 1.0, 0.5], [1.0, 0.0], [0.3, 0.3, 0.7, 0.1]]
    ext = [0.0, 1.0, 0.0, 1.0]
    W, H = vr.CANVAS[kind][:2]
    xf = capi.plot_transform(ext, W, H)
    texts = [vr.path_text(x, y, xf, kind, fmt) for x, y in zip(xs, ys)] + [b""]
    rgb = np.array([capi.plot_color(k, 1) for k in range(4)], np.uint8)
    path = str(tmp_path / ("c.svg" if fmt == vr.SVG else "c.eps"))
    capi.plot_vector_write(path, kind, fmt, ext, "scaled coverage for " + NASTY, "proportion of " + NASTY, rgb, 0.65, texts)
    return open(path, "rb").read(), texts, rgb


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_svg_document_parses(tmp_path, kind):
    data, texts, rgb = _doc(tmp_path, vr.SVG, kind)
    root = ET.fromstring(data)
    ns = "{http://www.w3.org/2000/svg}"
    W, H, CW, CH = vr.CANVAS[kind]
    assert root.get("width") == "%dpt" % (CW * 3 // 4) and root.get("height") == "%dpt" % (CH * 3 // 4)
    assert root.get("viewBox") == "0 0 %d %d" % (CW * 3 // 4, CH * 3 // 4)
    paths = [p for p in root.iter(ns + "path") if p.get("stroke") != "#000000"]
    assert [p.get("d").encode() for p in paths] == texts[:3]
    assert [p.get("stroke") for p in paths] == ["#%02x%02x%02x" % tuple(c) for c in rgb[:3]]
    assert all(p.get("stroke-width") == "0.65" and p.get("fill") == "none" for p in paths)
    labels = [t.text for t in root.iter(ns + "text")]
    assert "scaled coverage for " + NASTY in labels and "proportion of " + NASTY in labels
    assert len(labels) >= 4                                              # tick labels too
    # every data path is a line of its own
    lines = data.decode().split("\n")
    assert sum(1 for ln in lines if ln.startswith('<path d="M ') and 'stroke="#000000"' not in ln) == 3


def _ps_tokens(data):
    """PostScript tokens: strings (unescaped), numbers, names and comments dropped"""
    s, i, toks = data.decode("latin-1"), 0, []
    while i < len(s):
        c = s[i]
        if c.isspace():
            i += 1
        elif c == "%":
            i = s.index("\n", i) + 1
        elif c == "(":
            i += 1
            out, depth = [], 0
            while True:
                c = s[i]
                if c == "\\":
                    nxt = s[i + 1]
                    if nxt in "()\\":
                        out.append(nxt); i += 2
                    else:
                        out.append(chr(int(s[i + 1:i + 4], 8))); i += 4
                    continue
                assert c not in "()", "unescaped parenthesis in a string"
                out.append(c); i += 1
                if s[i] == ")" and depth == 0:
                    i += 1
                    break
            toks.append(("str", "".join(out)))
        else:
            m = re.match(r"[^\s()%]+", s[i:])
            toks.append(("tok", m.group(0)))
            i += len(m.group(0))
    return toks


@pytest.mark.parametrize("kind", [0, 1, 2])
def test_eps_document_tokenises(tmp_path, kind):
    data, texts, rgb = _doc(tmp_path, vr.EPS, kind)
    W, H, CW, CH = vr.CANVAS[kind]
    head = data.decode().split("\n")
    assert head[0] == "%!PS-Adobe-3.0 EPSF-3.0"
    assert head[1] == "%%%%BoundingBox: 0 0 %d %d" % (CW * 3 // 4, CH * 3 // 4)
    assert data.endswith(b"showpage\n%%EOF\n")
    assert max(len(ln) for ln in head) < 256
    toks = _ps_tokens(data)
    strs = [v for t, v in toks if t == "str"]
    assert "scaled coverage for " + NASTY in strs and "proportion of " + NASTY in strs
    for t, v in toks:
        if t == "tok":
            assert re.fullmatch(r"-?\d+(\.\d+)?|/?[A-Za-z]+|\[|\]|\{|\}", v), v
    # the datasets: colour, width, the path text, stroke
    body = data.decode()
    for k in range(3):
        c = rgb[k] / 255.0
        pre = "%.4f %.4f %.4f setrgbcolor 0.65 setlinewidth newpath\n" % tuple(c)
        assert pre + texts[k].decode() + "stroke\n" in body
    assert [round(float(x) * 255) for x in re.findall(r"([\d.]+) [\d.]+ [\d.]+ setrgbcolor", body)] == [int(c[0]) for c in rgb[:3]]


def test_line_width():
    assert capi.plot_line_width(30) == 0.8 and capi.plot_line_width(31) == 0.65
