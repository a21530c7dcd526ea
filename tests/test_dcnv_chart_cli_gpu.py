"""`goleft dcnv`'s depth chart end to end (bin/goleft): dd-depth-<label>.html's data against the oracle's normalised values
(oracle/dcnv.py), dd-depth-<label>.png's data area against the numpy raster rule (tests/plot_rule.py) through the colour
table, --svd, the input forms, the block knobs, --noplots and the flag order."""
import gzip
import json
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
from bamutil import make_bam_indexed  # noqa: E402
from fautil import make_fasta  # noqa: E402
from goleft_b200 import capi  # noqa: E402
from oracle import dcnv as od  # noqa: E402
import plot_rule as pr  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
REFS = [("chrM", 16571), ("chr22", 60001)]
W, H = capi.PLOT_W, capi.PLOT_H


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    d = tmp_path_factory.mktemp("dcnv_chart")
    fa, fai, _ = make_fasta(REFS, seed=3, line=60)
    path = str(d / "ref.fa")
    open(path, "wb").write(fa)
    open(path + ".fai", "w").write(fai)
    return path, fa, fai


@pytest.fixture(scope="module")
def ctx():
    with capi.Ctx(0) as c:
        yield c


def run(ref, d, text, *flags, name="m.tsv", stdin=False, env=None):
    """goleft dcnv in directory d -> (process, {file name: bytes} of what it wrote there)"""
    for f in os.listdir(d):
        if f.startswith("dd-depth-") or f == "depth.bed":
            os.remove(os.path.join(d, f))
    p = d / name
    p.write_bytes(gzip.compress(text) if name.endswith(".gz") else text)
    src = "-" if stdin else str(p)
    r = subprocess.run([GOLEFT, "dcnv", *flags, src, ref[0]], capture_output=True, cwd=str(d), input=text if stdin else None,
                       env=dict(os.environ, **env) if env else None)
    out = {f: (d / f).read_bytes() for f in os.listdir(d) if f.startswith("dd-depth-") or f == "depth.bed"}
    return r, out


def matrix_text(rng, rows, S, names=None):
    names = names or ["s%d" % i for i in range(S)]
    lines = ["#chrom\tstart\tend\t" + "\t".join(names)]
    for c, s, e in rows:
        lines.append("%s\t%d\t%d\t" % (c, s, e) + "\t".join("%d" % int(v) for v in rng.gamma(4.0, 8.0, S)))
    return ("\n".join(lines) + "\n").encode()


def tiled(chrom, L, size, start=0):
    return [(chrom, a, min(a + size, L)) for a in range(start, L - size, size)]


def oracle(ref, text, ctx=None, svd=None):
    """(sample names, label, the n x S values depth.bed holds)"""
    samples, label, _, _, gc, x = od.read_regions(text, ref[1], od.parse_fai(ref[2]))
    out, _, _ = od.matrix(x, gc)
    if svd is not None:
        out = ctx.dcnv_svd(out, svd)[0]
    return [s.decode() for s in samples], label.decode(), out


def read_png(b):
    assert b[:8] == b"\x89PNG\r\n\x1a\n"
    p, chunks = 8, {}
    while p < len(b):
        n, = struct.unpack(">I", b[p:p + 4])
        chunks[b[p + 4:p + 8]] = b[p + 8:p + 8 + n]
        p += 12 + n
    w, h = struct.unpack(">II", chunks[b"IHDR"][:8])
    rows = np.frombuffer(zlib.decompress(chunks[b"IDAT"]), np.uint8).reshape(h, w * 3 + 1)
    return rows[:, 1:].reshape(h, w, 3)


def data_area(png):
    return read_png(png)[capi.PLOT_AY:capi.PLOT_AY + H, capi.PLOT_AX:capi.PLOT_AX + W]


def palette(S):
    """colour of draw index v: sample S - v"""
    return np.array([(255, 255, 255)] + [capi.plot_color(S - v) for v in range(1, S + 1)], np.uint8)


def numpy_image(x):
    """the stepped lines of x (sample k drawn with index S - k) through plot_rule, with the extent of the plotted vertices"""
    n, S = x.shape
    lines, ext = [], [np.inf, -np.inf, np.inf, -np.inf]
    for k in range(S):
        nz = np.nonzero(x[:, k] != 0)[0]
        if not nz.size:
            continue
        i = np.arange(nz[0], n)
        xs, ys = i * 16384.0, np.minimum(x[i, k], 2.5)
        ext = [min(ext[0], xs[0]), (n - 1) * 16384.0, min(ext[2], ys.min()), max(ext[3], ys.max())]
        for j in range(len(xs) - 1):
            lines.append((S - k, [xs[j], xs[j + 1], xs[j + 1]], [ys[j], ys[j], ys[j + 1]]))
    ext = ext if lines or np.isfinite(ext[0]) else [0.0] * 4
    return pr.raster(lines, pr.transform(*ext, W, H), W, H, pr.line_radius(S))


def page_chart(html):
    m = re.search(r"/\*chart depth begin\*/var cfg_depth = (.*?);/\*chart depth end\*/", html.decode(), re.S)
    return json.loads(m.group(1))


def check_page(html, names, label, x):
    cfg = page_chart(html)
    n, S = x.shape
    ds = cfg["data"]["datasets"]
    assert [d["label"] for d in ds] == names
    w = 0.2 if S > 50 else (0.3 if S > 30 else 0.4)
    for k, d in enumerate(ds):
        assert d["borderWidth"] == w and d["steppedLine"] is True and d["pointRadius"] == 0 and d["pointHitRadius"] == 6
        assert d["fill"] is False and d["borderColor"] == "rgba(%d,%d,%d,0.94)" % capi.plot_color(k)
        nz = np.nonzero(x[:, k] != 0)[0]
        i = np.arange(nz[0] if nz.size else n, n)
        y = np.minimum(x[i, k], 2.5)
        tok = capi.format_f2_host(y)
        want = [float(bytes(t).rstrip(b"\0")) for t in tok]
        assert [p["x"] for p in d["data"]] == [int(v) * 16384 for v in i]
        assert [p["y"] for p in d["data"]] == want
    sc = cfg["options"]["scales"]
    assert sc["yAxes"][0]["ticks"] == {"min": 0, "max": 2.5} and sc["yAxes"][0]["scaleLabel"]["labelString"] == "scaled coverage"
    assert sc["xAxes"][0]["scaleLabel"]["labelString"] == "position on " + label
    assert cfg["options"]["tooltips"]["mode"] == "nearest" and cfg["options"]["responsive"] is False
    assert b'width="850" height="550"' in html and b'<a href="index.html">back to index</a>' in html


def test_pipeline(ref, tmp_path):
    """depth -> depthwed -> dcnv: both files under the label's name, against the oracle and numpy"""
    beds = []
    for k in range(3):
        rng = np.random.default_rng(40 + k)
        recs = []
        for tid, (_, L) in enumerate(REFS):
            for p in np.sort(rng.integers(0, L - 100, int((20 + 5 * k) * L / 100))):
                recs.append((tid, int(p), 60, 0, [(100, "M")]))
        bam, bai = make_bam_indexed(REFS, recs, sample="S%d" % k)
        (tmp_path / ("s%d.bam" % k)).write_bytes(bam)
        (tmp_path / ("s%d.bam.bai" % k)).write_bytes(bai)
        prefix = str(tmp_path / ("s%d" % k))
        p = subprocess.run([GOLEFT, "depth", "-Q", "1", "--ordered", "-w", "250", "--prefix", prefix, "-r", ref[0], str(tmp_path / ("s%d.bam" % k))],
                           capture_output=True)
        assert p.returncode == 0, p.stderr
        beds.append(prefix + ".depth.bed")
    p = subprocess.run([GOLEFT, "depthwed", "-s", "1000", *beds], capture_output=True)
    assert p.returncode == 0, p.stderr
    text = p.stdout
    d = tmp_path / "run"
    d.mkdir()
    r, out = run(ref, d, text)
    assert r.returncode == 0, r.stderr
    names, label, x = oracle(ref, text)
    assert sorted(out) == ["dd-depth-%s.html" % label, "dd-depth-%s.png" % label, "depth.bed"]
    assert out["depth.bed"] == od.dcnv(text, ref[1], ref[2])
    check_page(out["dd-depth-%s.html" % label], names, label, x)
    area = data_area(out["dd-depth-%s.png" % label])
    img = numpy_image(x)
    assert img.any() and np.array_equal(area, palette(x.shape[1])[img])


@pytest.mark.parametrize("S", [30, 31, 50, 51])
def test_hand_made(ref, tmp_path, ctx, S):
    """border widths either side of 30 and 50 samples, a label from the second data line, names that need quoting"""
    rng = np.random.default_rng(S)
    rows = [("chrM", 0, 500)] + tiled("chr22", 60001, 500, 500)[:60]
    text = matrix_text(rng, rows, S, names=["smp-%d\"q" % i for i in range(S)])
    lines = text.split(b"\n")
    for j in range(1, 5):                                   # sample 3's first rows are zero
        f = lines[j].split(b"\t")
        f[3 + 3] = b"0"
        lines[j] = b"\t".join(f)
    text = b"\n".join(lines)
    r, out = run(ref, tmp_path, text)
    assert r.returncode == 0, r.stderr
    names, label, x = oracle(ref, text)
    assert label == "chr22"
    check_page(out["dd-depth-chr22.html"], names, label, x)
    area = data_area(out["dd-depth-chr22.png"])
    first, yext, ext, img = ctx.dcnv_chart(x)
    assert np.array_equal(img, capi.dcnv_chart_raster_host(x, first, capi.plot_transform(ext, W, H)))
    assert np.array_equal(area, palette(S)[img])
    if S == 31:
        assert np.array_equal(img, numpy_image(x))


def test_svd_inputs_knobs_noplots_flags(ref, tmp_path, ctx):
    rng = np.random.default_rng(9)
    rows = tiled("chrM", 16571, 250) + tiled("chr22", 60001, 250)
    text = matrix_text(rng, rows, 12)
    names, label, x = oracle(ref, text, ctx, svd=5.0)
    base, out = run(ref, tmp_path, text, "--svd", "5")
    assert base.returncode == 0, base.stderr
    html, png = out["dd-depth-%s.html" % label], out["dd-depth-%s.png" % label]
    check_page(html, names, label, x)                       # drawn from the SVD output
    first, yext, ext, img = ctx.dcnv_chart(x)
    assert np.array_equal(data_area(png), palette(12)[img])
    plain = oracle(ref, text)[2]
    assert not np.array_equal(plain, x)
    # gzip, stdin and the block knobs: every file byte for byte
    for kw in (dict(name="m.tsv.gz"), dict(stdin=True), dict(env={"GL_DCNV_BLOCK_COLS": "2"}), dict(env={"GL_DCNV_CHART_BLOCK_ROWS": "7"}),
               dict(env={"GL_DCNV_CHART_BLOCK_ROWS": "1", "GL_DCNV_BLOCK_COLS": "5"})):
        r, again = run(ref, tmp_path, text, "--svd", "5", **kw)
        assert r.returncode == 0 and again == out, kw
    # --noplots: depth.bed, stdout and stderr as with charts (the log's timestamp aside), no chart file; any flag order
    for flags in (("--noplots", "--svd", "5"), ("--svd", "5", "--noplots"), ("--svd=5", "--noplots"), ("--noplots", "--svd=5")):
        r, none = run(ref, tmp_path, text, *flags)
        assert r.returncode == 0, (flags, r.stderr)
        assert sorted(none) == ["depth.bed"] and none["depth.bed"] == out["depth.bed"], flags
        assert r.stdout == base.stdout and r.stderr[20:] == base.stderr[20:] and len(r.stderr) == len(base.stderr), flags
    r, none = run(ref, tmp_path, text, "--noplots")
    r2, withp = run(ref, tmp_path, text)
    assert r.returncode == 0 and r2.returncode == 0
    assert sorted(none) == ["depth.bed"] and none["depth.bed"] == withp["depth.bed"] == od.dcnv(text, ref[1], ref[2])
    assert r.stdout == r2.stdout == b"" and r.stderr == r2.stderr
    assert len(withp) == 3
