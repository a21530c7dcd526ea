"""`goleft indexcov` with INDEXCOV_FMT end to end: one .svg or .eps beside every chart PNG, every path's vertices against the
oracle's depths through the chart transform in "%.2f" (tests/vector_rule.py), stroke colours from the palette (with
INDEXCOV_N_BACKGROUNDS), --gpus invariance, and every other output file unchanged by the variable."""
import os
import re
import subprocess
import sys
import xml.etree.ElementTree as ET

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from goleft_b200 import capi  # noqa: E402
from indexcov_cli_oracle import cohort_bais, oracle_depths  # noqa: E402
import plot_rule as pr  # noqa: E402
import vector_rule as vr  # noqa: E402
from oracle import loader as orc  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
NS = "{http://www.w3.org/2000/svg}"
ROC_MULT = (1.0 / 70) / (2.0 / 3.0)


def go(tmp_path, tag, fai, paths, *extra, env=None):
    d = tmp_path / tag / "o"
    d.parent.mkdir()
    e = dict(os.environ)
    e.pop("INDEXCOV_FMT", None)
    e.update(env or {})
    p = subprocess.run([GOLEFT, "indexcov", "-d", str(d), "--fai", fai, *extra, *paths], capture_output=True, text=True, env=e)
    assert p.returncode == 0, p.stderr
    return str(d)


def files(d):
    return {f: open(os.path.join(d, f), "rb").read() for f in os.listdir(d)}


def svg_paths(data):
    """[(d, stroke, width)] of the data paths (the frame is stroked black)"""
    root = ET.fromstring(data)
    return [(p.get("d"), p.get("stroke"), p.get("stroke-width")) for p in root.iter(NS + "path") if p.get("stroke") != "#000000"]


def eps_paths(data):
    body = data.decode()
    out = []
    for m in re.finditer(r"([\d.]+) ([\d.]+) ([\d.]+) setrgbcolor ([\d.]+) setlinewidth newpath\n(.*?)stroke\n", body, re.S):
        rgb = "#%02x%02x%02x" % tuple(round(float(m.group(i)) * 255) for i in (1, 2, 3))
        out.append((m.group(5), rgb, m.group(4)))
    return out


def expected_paths(lines, xf, kind, fmt, pal, width):
    out = []
    for idx, xs, ys in lines:
        t = vr.path_text(xs, ys, xf, kind, fmt)
        if t:
            out.append((t.decode(), "#%02x%02x%02x" % tuple(pal[idx]), width))
    return out


def test_file_set_and_other_outputs(tmp_path):
    refs, fai, paths, lin = cohort_bais(tmp_path, S=7)
    base = files(go(tmp_path, "none", fai, paths))
    pngs = sorted(f for f in base if f.endswith(".png"))
    assert len(pngs) > 3 and "o-indexcov-sex.png" in pngs
    for tag, v, ext in (("svg", "svg", ".svg"), ("eps", "eps", ".eps"), ("x", "x", ".eps"), ("SVG", "SVG", ".eps"), ("pdf", "pdf", ".eps")):
        got = files(go(tmp_path, tag, fai, paths, env={"INDEXCOV_FMT": v}))
        new = sorted(set(got) - set(base))
        assert new == sorted(p[:-3] + ext[1:] for p in pngs), tag
        for f in base:
            assert got[f] == base[f], (tag, f)                         # every other output: byte-identical
    for tag, extra, env in (("empty", (), {"INDEXCOV_FMT": ""}), ("noplots", ("--noplots",), {"INDEXCOV_FMT": "svg"})):
        got = files(go(tmp_path, tag, fai, paths, *extra, env=env))
        assert not any(f.endswith((".svg", ".eps")) for f in got), tag
    assert set(files(go(tmp_path, "empty2", fai, paths, env={"INDEXCOV_FMT": ""}))) == set(base)


@pytest.mark.parametrize("S,fmt,n_bg", [(7, vr.SVG, 0), (7, vr.EPS, 3), (101, vr.SVG, 0), (101, vr.EPS, 0)])
def test_vertices_against_oracle(tmp_path, S, fmt, n_bg):
    refs, fai, paths, lin = cohort_bais(tmp_path, S=S)
    env = {"INDEXCOV_FMT": "svg" if fmt == vr.SVG else "eps"}
    if n_bg:
        env["INDEXCOV_N_BACKGROUNDS"] = str(n_bg)
    od = go(tmp_path, "v", fai, paths, env=env)
    ext = ".svg" if fmt == vr.SVG else ".eps"
    parse = svg_paths if fmt == vr.SVG else eps_paths
    pal = np.array([(255, 255, 255)] + [capi.plot_color(k, n_bg) for k in range(S)], np.uint8)
    width = "0.65" if S > 30 else "0.80"
    names = [n for n, _ in refs]
    depths = oracle_depths(lin)
    plotted = [n for r, n in enumerate(names) if not n.startswith("NC") and not n.startswith("GL") and max(len(depths[k][r]) for k in range(S)) > 2]
    assert plotted
    for n in plotted:
        r = names.index(n)
        ds = [depths[k][r] for k in range(S)]
        lines, e = pr.series_lines(ds)
        want = expected_paths(lines, pr.transform(*e, capi.PLOT_W, capi.PLOT_H), 0, fmt, pal, width)
        got = parse(open(os.path.join(od, "o-indexcov-depth-%s%s" % (n, ext)), "rb").read())
        assert got == want, n
        if n_bg:
            assert got[0][1] == "#b4b4b4"                              # sample 0 is a background: grey
        rocs = [np.asarray(orc.ic_roc(orc.ic_counts(d)), np.float32) for d in ds]
        lines, e = pr.series_lines(rocs, ROC_MULT)
        want = expected_paths(lines, pr.transform(*e, capi.PLOT_W, capi.PLOT_H), 1, fmt, pal, width)
        assert parse(open(os.path.join(od, "o-indexcov-roc-%s%s" % (n, ext)), "rb").read()) == want, n
    x, y = names.index("X"), names.index("Y")
    cx = [float(orc.ic_getcn(depths[k][x])) for k in range(S)]
    cy = [float(orc.ic_getcn(depths[k][y])) for k in range(S)]
    inferred = [int(0.5 + v) for v in cx]
    cns = sorted(set(inferred))
    lines, ks_all = [], []
    for g, c in enumerate(cns):
        ks = [k for k in range(max(n_bg, 0), S) if inferred[k] == c]
        ks_all += ks
        lines.append((g + 1, [cx[k] for k in ks], [cy[k] for k in ks]))
    spal = np.array([(255, 255, 255)] + [capi.plot_color(c, 0) for c in cns], np.uint8)
    xf = pr.transform(min(cx[k] for k in ks_all), max(cx[k] for k in ks_all), min(cy[k] for k in ks_all), max(cy[k] for k in ks_all), 508, 532)
    want = expected_paths(lines, xf, 2, fmt, spal, "0.65" if len(cns) > 30 else "0.80")
    assert parse(open(os.path.join(od, "o-indexcov-sex" + ext), "rb").read()) == want


def test_gpus_give_identical_vector_files(tmp_path):
    refs, fai, paths, lin = cohort_bais(tmp_path, S=7)
    one = files(go(tmp_path, "g1", fai, paths, env={"INDEXCOV_FMT": "svg"}))
    assert any(f.endswith(".svg") for f in one)
    for g in (2, 3, 7):
        other = files(go(tmp_path, "g%d" % g, fai, paths, "--gpus", str(g), env={"INDEXCOV_FMT": "svg", "GL_OVERSUBSCRIBE": "1"}))
        assert sorted(other) == sorted(one)
        for f in one:
            assert other[f] == one[f], (g, f)
