"""End-to-end `goleft emdepth` (bin/goleft): P.cn.bed and P.cnv.bed must equal the oracle's bytes, after `depth` ->
`depthwed` and after `dcnv`; input forms; every error is exit 2."""
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bamutil import make_bam_indexed  # noqa: E402
from fautil import make_fasta  # noqa: E402
from oracle import emdepth as oe  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
REFS = [("chrM", 16571), ("chr22", 60001)]


def run(*args, cwd=None, input=None, env=None):
    return subprocess.run([GOLEFT, *args], capture_output=True, cwd=cwd, input=input, env=dict(os.environ, **env) if env else None)


def emdepth(text, tmp_path, name="m.tsv", stdin=False, env=None):
    p = tmp_path / name
    p.write_bytes(gzip.compress(text) if name.endswith(".gz") else text)
    prefix = str(tmp_path / "out")
    r = run("emdepth", "--prefix", prefix, "-" if stdin else str(p), input=text if stdin else None, env=env)
    if r.returncode != 0:
        return r, None
    return r, (open(prefix + ".cn.bed", "rb").read(), open(prefix + ".cnv.bed", "rb").read())


def _matrix_text(rng, rows, S, plant=None):
    lines = [b"#chrom\tstart\tend\t" + b"\t".join(b"s%d" % i for i in range(S))]
    for k, (c, s, e) in enumerate(rows):
        v = rng.gamma(40.0, 1.0, S)
        if plant and plant[0] <= k < plant[1]:
            v[plant[2]] *= plant[3]
        lines.append(b"%s\t%d\t%d\t" % (c.encode(), s, e) + b"\t".join(b"%d" % int(x) for x in v))
    return b"\n".join(lines) + b"\n"


@pytest.fixture(scope="module")
def tools():
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")


def test_pipeline_depth_depthwed_emdepth_and_dcnv(tools, tmp_path):
    fa, fai, _ = make_fasta(REFS, seed=3, line=60)
    fa_path = str(tmp_path / "ref.fa")
    open(fa_path, "wb").write(fa)
    open(fa_path + ".fai", "w").write(fai)
    beds = []
    for k in range(5):
        rng = np.random.default_rng(70 + k)
        recs = []
        for tid, (_, L) in enumerate(REFS):
            cov = (20 + 3 * k) * (0.5 if (k == 3 and tid == 1) else 1.0)          # sample 3: one copy of chr22
            for p in np.sort(rng.integers(0, L - 100, int(cov * L / 100))):
                recs.append((tid, int(p), 60, 0, [(100, "M")]))
        bam, bai = make_bam_indexed(REFS, recs, sample="S%d" % k)
        bp = tmp_path / ("s%d.bam" % k)
        bp.write_bytes(bam)
        (tmp_path / ("s%d.bam.bai" % k)).write_bytes(bai)
        prefix = str(tmp_path / ("s%d" % k))
        p = run("depth", "-Q", "1", "--ordered", "-w", "250", "--prefix", prefix, "-r", fa_path, str(bp))
        assert p.returncode == 0, p.stderr
        beds.append(prefix + ".depth.bed")
    p = run("depthwed", "-s", "1000", *beds)
    assert p.returncode == 0, p.stderr
    mat = p.stdout
    r, got = emdepth(mat, tmp_path)
    assert r.returncode == 0, r.stderr
    assert got == oe.files(mat)
    p = run("dcnv", str(tmp_path / "m.tsv"), fa_path, cwd=str(tmp_path))
    assert p.returncode == 0, p.stderr
    norm = (tmp_path / "depth.bed").read_bytes()
    r, got = emdepth(norm, tmp_path, name="n.tsv")
    assert r.returncode == 0, r.stderr
    assert got == oe.files(norm)


def test_planted_cnv_and_input_forms(tools, tmp_path):
    rng = np.random.default_rng(4)
    rows = [("chr1", a, a + 1000) for a in range(0, 400_000, 1000)] + [("chr2", a, a + 1000) for a in range(0, 200_000, 1000)]
    text = _matrix_text(rng, rows, 24, plant=(100, 140, 5, 0.5))
    text2 = _matrix_text(rng, rows, 24, plant=(450, 480, 9, 1.5))
    for t, sample, lo, hi, cn in ((text, b"s5", 100, 140, b"1"), (text2, b"s9", 450, 480, b"3")):
        r, (cn_bed, cnv_bed) = emdepth(t, tmp_path)
        assert r.returncode == 0, r.stderr
        assert (cn_bed, cnv_bed) == oe.files(t)
        hits = [ln.split(b"\t") for ln in cnv_bed.split(b"\n")[1:-1] if ln.split(b"\t")[3] == sample]
        assert any(int(h[4]) >= 10 and h[5].count(cn) >= 10 for h in hits), cnv_bed
        assert cn_bed.split(b"\n")[0] == b"#chrom\tstart\tend\t" + b"\t".join(b"s%d" % i for i in range(24))
    want = oe.files(text)
    for kw in (dict(name="m.tsv.gz"), dict(stdin=True), dict(env={"GL_EMDEPTH_BLOCK_ROWS": "77"})):
        r, got = emdepth(text, tmp_path, **kw)
        assert r.returncode == 0, (kw, r.stderr)
        assert got == want, kw


def test_errors(tools, tmp_path):
    rng = np.random.default_rng(1)
    rows = [("chrM", a, a + 1000) for a in range(0, 16000, 1000)]
    good = _matrix_text(rng, rows, 3)
    hdr, body = good.split(b"\n", 1)
    cases = {
        "two samples": _matrix_text(rng, rows, 2),
        "no header": body,
        "bad number": good + b"chrM\t1000\t2000\t1\tabc\t3\n",
        "negative": good + b"chrM\t1000\t2000\t1\t-4\t3\n",
        "column count": good + b"chrM\t1000\t2000\t1\t2\n",
    }
    for what, text in cases.items():
        r, _ = emdepth(text, tmp_path)
        assert r.returncode == 2 and b"panic" in r.stderr, (what, r.returncode, r.stderr)
    r = run("emdepth")
    assert r.returncode == 2
    r = run("emdepth", str(tmp_path / "absent.tsv"))
    assert r.returncode == 2
