"""End-to-end `goleft dcnv --chunk W` (bin/goleft, DESIGN §1.9): depth.bed byte for byte against the oracle's ChunkDebiaser
text, alone, with --svd (the library's SVD on the oracle's values) and with --noplots, with the flags in several orders;
the chart's data against the chunk-normalised values; and fewer than five rows, which the moving median needs and the
chunks do not."""
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from fautil import make_fasta  # noqa: E402
from goleft_b200 import capi  # noqa: E402
from oracle import dcnv as od  # noqa: E402
from oracle import dcnv_chunk as oc  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
REFS = [("chr1", 900_000)]


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    d = tmp_path_factory.mktemp("dcnv_chunk")
    fa, fai, _ = make_fasta(REFS, seed=21, line=60)
    path = str(d / "ref.fa")
    open(path, "wb").write(fa)
    open(path + ".fai", "w").write(fai)
    return path, fa, fai


def run(ref, d, text, *flags):
    for f in os.listdir(d):
        if f.startswith("dd-depth-") or f == "depth.bed":
            os.remove(os.path.join(d, f))
    (d / "m.tsv").write_bytes(text)
    r = subprocess.run([GOLEFT, "dcnv", *flags, str(d / "m.tsv"), ref[0]], capture_output=True, cwd=str(d))
    return r, {f: (d / f).read_bytes() for f in os.listdir(d) if f.startswith("dd-depth-") or f == "depth.bed"}


def matrix_text(rng, n, S, size=1000, zero_frac=0.1):
    lines = ["#chrom\tstart\tend\t" + "\t".join("s%d" % i for i in range(S))]
    for a in range(0, n * size, size):
        v = np.floor(rng.gamma(4.0, 8.0, S)) * (rng.random(S) > zero_frac)
        lines.append("chr1\t%d\t%d\t" % (a, a + size) + "\t".join("%d" % int(t) for t in v))
    return ("\n".join(lines) + "\n").encode()


@pytest.mark.parametrize("w", ["0.01", "0.001", "1e-9", "1"])
def test_text_against_oracle(ref, tmp_path, w):
    rng = np.random.default_rng(31)
    text = matrix_text(rng, 850, 9)
    want = oc.dcnv(text, ref[1], ref[2], float(w))
    r, out = run(ref, tmp_path, text, "--noplots", "--chunk", w)
    assert r.returncode == 0, r.stderr
    assert out["depth.bed"] == want and r.stdout == b""
    assert out["depth.bed"] != od.dcnv(text, ref[1], ref[2])              # not the moving median's text


def test_flag_orders_and_noplots(ref, tmp_path):
    rng = np.random.default_rng(32)
    text = matrix_text(rng, 600, 6, zero_frac=0.3)
    want = oc.dcnv(text, ref[1], ref[2], 0.02)
    for flags in (("--chunk", "0.02"), ("--chunk=0.02",), ("--noplots", "--chunk", "0.02"), ("--chunk", "0.02", "--noplots"),
                  ("--chunk=2e-2", "--noplots")):
        r, out = run(ref, tmp_path, text, *flags)
        assert r.returncode == 0, (flags, r.stderr)
        assert out["depth.bed"] == want, flags
        assert ("--noplots" in flags) == (len(out) == 1), (flags, sorted(out))


def test_with_svd(ref, tmp_path):
    """--chunk then --svd: the library's SVD of the oracle's chunk-normalised values (its bits do not depend on row blocks)"""
    rng = np.random.default_rng(33)
    n, S = 700, 16
    text = matrix_text(rng, n, S)
    samples, label, starts, ends, vals = oc.values(text, ref[1], ref[2], 0.01)
    with capi.Ctx(0) as ctx:
        after, _, n_removed, _ = ctx.dcnv_svd(vals, 5.0)[:4]
    assert n_removed > 0
    want = b"#chrom\tstart\tend\t" + b"\t".join(samples) + b"\n" + od.rows(label, starts, ends, after)
    for flags in (("--chunk", "0.01", "--svd", "5"), ("--svd=5", "--chunk=0.01"), ("--noplots", "--svd", "5", "--chunk", "0.01"),
                  ("--chunk", "0.01", "--noplots", "--svd=5")):
        r, out = run(ref, tmp_path, text, *flags)
        assert r.returncode == 0, (flags, r.stderr)
        assert out["depth.bed"] == want, flags
        assert re.search(rb" variance:( \d+\.\d\d)+\n", r.stderr)


def test_chart_data_is_chunk_normalised(ref, tmp_path):
    rng = np.random.default_rng(34)
    n, S = 400, 4
    text = matrix_text(rng, n, S, zero_frac=0.2)
    samples, label, _, _, vals = oc.values(text, ref[1], ref[2], 0.01)
    r, out = run(ref, tmp_path, text, "--chunk", "0.01")
    assert r.returncode == 0, r.stderr
    html = out["dd-depth-%s.html" % label.decode()].decode()
    m = re.search(r"/\*chart depth begin\*/var cfg_depth = (.*?);/\*chart depth end\*/", html, re.S)
    ds = json.loads(m.group(1))["data"]["datasets"]
    assert [d["label"] for d in ds] == [s.decode() for s in samples]
    for k, d in enumerate(ds):
        nz = np.nonzero(vals[:, k] != 0)[0]
        i = np.arange(nz[0] if nz.size else n, n)
        y = np.minimum(vals[i, k], 2.5)
        want = [float(bytes(t).rstrip(b"\0")) for t in capi.format_f2_host(y)]
        assert [p["x"] for p in d["data"]] == [int(v) * 16384 for v in i]
        assert [p["y"] for p in d["data"]] == want


def test_fewer_than_five_rows(ref, tmp_path):
    """ChunkDebiaser needs no window: three rows are normalised where the default panics"""
    rng = np.random.default_rng(35)
    text = matrix_text(rng, 3, 2, zero_frac=0.0)
    r, _ = run(ref, tmp_path, text, "--noplots")
    assert r.returncode == 2
    r, out = run(ref, tmp_path, text, "--noplots", "--chunk", "0.05")
    assert r.returncode == 0, r.stderr
    samples, label, starts, ends, gc, x = [], None, [], [], [], []
    for ln in text.split(b"\n")[1:-1]:
        f = ln.split(b"\t")
        label = f[0]
        s, e = max(int(f[1]), 250), int(f[2])
        starts.append(s); ends.append(e)
        gc.append(od.faidx_stats(ref[1], od.parse_fai(ref[2])["chr1"], s - 250, e)[0])
        x.append([float(v) for v in f[3:]])
    vals = oc.matrix(np.array(x), np.array(gc), 0.05)[0]
    assert out["depth.bed"] == b"#chrom\tstart\tend\ts0\ts1\n" + od.rows(label, np.array(starts), np.array(ends), vals)
