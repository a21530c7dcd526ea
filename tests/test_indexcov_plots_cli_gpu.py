"""`goleft indexcov`'s charts end to end: the PNG file set, the data-area pixels of every chart against the numpy index image
(tests/plot_rule.py) of the oracle's depths and the run's .roc through the product's colour table, INDEXCOV_N_BACKGROUNDS,
--gpus invariance, and --noplots leaving every other output as it was."""
import json
import math
import os
import re
import struct
import subprocess
import sys
import zlib

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from goleft_b200 import capi  # noqa: E402
from indexcov_cli_oracle import _xnorm, cohort_bais, oracle_depths, read_ped  # noqa: E402
from oracle import indexcov_pca as op  # noqa: E402
import plot_rule as pr  # noqa: E402
from oracle import loader as orc  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")


def run(*args, env=None):
    p = subprocess.run([GOLEFT, *args], capture_output=True, text=True, env=dict(os.environ, **env) if env else None)
    assert p.returncode == 0, p.stderr
    return p


def read_png(path):
    b = open(path, "rb").read()
    assert b[:8] == b"\x89PNG\r\n\x1a\n"
    p, chunks = 8, {}
    while p < len(b):
        n, = struct.unpack(">I", b[p:p + 4])
        t = b[p + 4:p + 8]
        assert struct.unpack(">I", b[p + 8 + n:p + 12 + n])[0] == zlib.crc32(b[p + 4:p + 8 + n])
        chunks[t] = b[p + 8:p + 8 + n]
        p += 12 + n
    w, h = struct.unpack(">II", chunks[b"IHDR"][:8])
    rows = np.frombuffer(zlib.decompress(chunks[b"IDAT"]), np.uint8).reshape(h, w * 3 + 1)
    return rows[:, 1:].reshape(h, w, 3)


def data_area(rgb):
    return rgb[capi.PLOT_AY:capi.PLOT_AY + capi.PLOT_H, capi.PLOT_AX:capi.PLOT_AX + capi.PLOT_W]


def palette(S, n_bg=0):
    return np.array([(255, 255, 255)] + [capi.plot_color(k, n_bg) for k in range(S)], np.uint8)


def expected_depth_area(ds, S, n_bg=0):
    lines, ext = pr.series_lines(ds)
    xf = pr.transform(*ext, capi.PLOT_W, capi.PLOT_H)
    return palette(S, n_bg)[pr.raster(lines, xf, capi.PLOT_W, capi.PLOT_H, pr.line_radius(S))]


def page_charts(path):
    """{name: config} of every chart config on a page"""
    html = open(path).read()
    return {m.group(1): json.loads(m.group(2)) for m in re.finditer(r"/\*chart (\w+) begin\*/var cfg_\1 = (.*?);/\*chart \1 end\*/", html, re.S)}


def same_tokens(pts, xs, ys, xf, yf):
    assert len(pts) == len(xs)
    for p, x, y in zip(pts, xs, ys):
        for got, v, f in ((p["x"], x, xf), (p["y"], y, yf)):
            assert (math.isnan(got) and math.isnan(v)) or got == float(f % v), (got, v, f)


ROC_MULT = (1.0 / 70) / (2.0 / 3.0)


@pytest.mark.parametrize("S,extranorm,includegl", [(7, False, False), (7, True, True), (101, False, False), (101, True, True)])
def test_charts_against_numpy(tmp_path, S, extranorm, includegl):
    refs, fai, paths, lin = cohort_bais(tmp_path, S=S)
    out = tmp_path / "out"
    p = run("indexcov", "-d", str(out), "--fai", fai, *(["-n"] if extranorm else []), *(["-e"] if includegl else []), *paths)
    assert ("creating only static (no interactive) plots for depth" in p.stderr) == (S > 100)
    stem = "out-indexcov"
    od = str(out)
    names = [n for n, _ in refs]
    depths = oracle_depths(lin)
    plotted = [n for r, n in enumerate(names) if not n.startswith("NC") and (includegl or not n.startswith("GL"))
               and max(len(depths[k][r]) for k in range(S)) > 2]   # indexcov.go:709-711
    assert "GL000207.1" not in plotted                               # one tile: never charted, -e or not
    files = set(os.listdir(od))
    for n in names:
        for kind in ("depth", "roc"):
            assert (stem + "-%s-%s.png" % (kind, n) in files) == (n in plotted), (kind, n)
        assert (stem + "-depth-%s.html" % n in files) == (n in plotted and S <= 100), n
        assert (stem + "-roc-%s.html" % n in files) == (n in plotted), n
    assert stem + "-sex.png" in files
    html = open(os.path.join(od, "index.html")).read()
    assert all(stem + "-roc-%s.html" % n in html for n in plotted)
    samples = [row[1] for row in read_ped(out)[1:]]
    for n in plotted:
        r = names.index(n)
        ds = [depths[k][r] for k in range(S)]
        if extranorm and n not in ("X", "Y"):
            ds = _xnorm(ds)
        got = data_area(read_png(os.path.join(od, stem + "-depth-%s.png" % n)))
        assert np.array_equal(got, expected_depth_area(ds, S)), n
        rocs = [np.asarray(orc.ic_roc(orc.ic_counts(d)), np.float32) for d in ds]
        lines, ext = pr.series_lines(rocs, ROC_MULT)
        xf = pr.transform(*ext, capi.PLOT_W, capi.PLOT_H)
        want = palette(S)[pr.raster(lines, xf, capi.PLOT_W, capi.PLOT_H, pr.line_radius(S))]
        got = data_area(read_png(os.path.join(od, stem + "-roc-%s.png" % n)))
        assert np.array_equal(got, want), n
        # the pages: every asValues vertex, datasets last sample first (plot.go:142-144,347-349)
        roc = page_charts(os.path.join(od, stem + "-roc-%s.html" % n))["roc"]["data"]["datasets"]
        assert [d["label"] for d in roc] == samples[::-1]
        for d, k in zip(roc, range(S - 1, -1, -1)):
            xs, ys = pr.as_values(rocs[k], ROC_MULT)
            same_tokens(d["data"], xs, ys, "%.2f", "%.2f")
        if S <= 100:
            dep = page_charts(os.path.join(od, stem + "-depth-%s.html" % n))["depth"]["data"]["datasets"]
            assert [d["label"] for d in dep] == samples[::-1]
            for d, k in zip(dep, range(S - 1, -1, -1)):
                xs, ys = pr.as_values(ds[k], 16384.0)
                same_tokens(d["data"], xs, ys, "%.0f", "%.2f")
    # the sex chart: one dataset per inferred CN of X, ascending; asPng joins each dataset's points in sample order
    x, y = names.index("X"), names.index("Y")
    cx = [float(orc.ic_getcn(depths[k][x])) for k in range(S)]
    cy = [float(orc.ic_getcn(depths[k][y])) for k in range(S)]
    inferred = [int(0.5 + v) for v in cx]
    cns = sorted(set(inferred))
    sex = page_charts(os.path.join(od, "index.html"))["sex"]["data"]["datasets"]
    assert [d["label"] for d in sex] == ["Inferred CN for X: %d" % c for c in cns]
    lines = []
    for g, c in enumerate(cns):
        ks = [k for k in range(S) if inferred[k] == c]
        same_tokens(sex[g]["data"], [cx[k] for k in ks], [cy[k] for k in ks], "%.2f", "%.2f")
        lines.append((g + 1, [cx[k] for k in ks], [cy[k] for k in ks]))
    W, H = 508, 532
    xf = pr.transform(min(cx), max(cx), min(cy), max(cy), W, H)
    pal = np.array([(255, 255, 255)] + [capi.plot_color(c, 0) for c in cns], np.uint8)
    got = read_png(os.path.join(od, stem + "-sex.png"))
    assert got.shape == (576, 576, 3)
    assert np.array_equal(got[capi.PLOT_AY:capi.PLOT_AY + H, capi.PLOT_AX:capi.PLOT_AX + W], pal[pr.raster(lines, xf, W, H, pr.line_radius(len(cns)))])
    # the PCA labels: gonum's vars from numpy's SVD of the centred byte matrix
    autos = [n for n in names if n not in ("X", "Y") and not n.startswith("NC")]
    refs_b = []
    for r, n in enumerate(names):
        if n in autos:
            ds = [depths[k][r] for k in range(S)]
            refs_b.append(_xnorm(ds) if extranorm else ds)
    xm = op.pca8_matrix(refs_b).astype(np.float64)
    xm -= xm.mean(axis=0)
    s = np.linalg.svd(xm, compute_uv=False)
    v = s ** 2 / (s ** 2).sum()
    charts = page_charts(os.path.join(od, "index.html"))
    for pc in (2, 3):
        sc = charts["pca%d" % pc]["options"]["scales"]
        assert sc["xAxes"][0]["scaleLabel"]["labelString"] == "PC1 (variance explained: %.2f%%)" % (100 * v[0])
        assert sc["yAxes"][0]["scaleLabel"]["labelString"] == "PC%d (variance explained: %.2f%%)" % (pc, 100 * v[pc - 1])
    bins = charts["bins"]["data"]["datasets"]
    assert len(bins) == 1 and len(bins[0]["data"]) == S
    assert len(charts["mapped"]["data"]["datasets"][0]["data"]) == S


def test_backgrounds_and_gpus_and_noplots(tmp_path):
    S = 7
    refs, fai, paths, lin = cohort_bais(tmp_path, S=S)
    stem = "o-indexcov"

    def go(tag, *extra, env=None):
        d = tmp_path / tag / "o"
        d.parent.mkdir()
        run("indexcov", "-d", str(d), "--fai", fai, *extra, *paths, env=env)
        return str(d)

    one = go("g1")
    for g in (2, 3, 7):
        other = go("g%d" % g, "--gpus", str(g), env={"GL_OVERSUBSCRIBE": "1"})
        assert sorted(os.listdir(one)) == sorted(os.listdir(other))
        for f in os.listdir(one):
            assert open(os.path.join(one, f), "rb").read() == open(os.path.join(other, f), "rb").read(), (g, f)
    plain = go("np", "--noplots")
    assert sorted(os.listdir(plain)) == sorted(["index.html", stem + ".bed.gz", stem + ".roc", stem + ".ped"])
    assert "plots are not built" in open(os.path.join(plain, "index.html")).read()
    for f in (".bed.gz", ".roc", ".ped"):
        assert open(os.path.join(one, stem + f), "rb").read() == open(os.path.join(plain, stem + f), "rb").read(), f
    bg = go("bg", env={"INDEXCOV_N_BACKGROUNDS": "3"})
    depths = oracle_depths(lin)
    got = data_area(read_png(os.path.join(bg, stem + "-depth-1.png")))
    assert np.array_equal(got, expected_depth_area([depths[k][0] for k in range(S)], S, n_bg=3))
    assert not np.array_equal(got, data_area(read_png(os.path.join(one, stem + "-depth-1.png"))))
