"""End-to-end `goleft depth` -> `goleft depthwed` -> `goleft dcnv` (bin/goleft) on BAMs and a FASTA written here; depth.bed
must equal the oracle's bytes.  Also the input forms, the reference's quirks and its panics (exit 2 here)."""
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
from oracle import dcnv as od  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
REFS = [("chrM", 16571), ("chr22", 60001)]


def run(*args, cwd=None, input=None, env=None):
    return subprocess.run([GOLEFT, *args], capture_output=True, cwd=cwd, input=input, env=dict(os.environ, **env) if env else None)


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    d = tmp_path_factory.mktemp("dcnv")
    fa, fai, _ = make_fasta(REFS, seed=3, line=60)
    path = str(d / "ref.fa")
    open(path, "wb").write(fa)
    open(path + ".fai", "w").write(fai)
    return d, path, fa, fai


def dcnv(ref, text, tmp_path, *extra, name="m.tsv", env=None):
    _, fa_path, fa, fai = ref
    if text is not None:
        p = tmp_path / name
        p.write_bytes(gzip.compress(text) if name.endswith(".gz") else text)
    p = run("dcnv", *(extra or (str(tmp_path / name),)), fa_path, cwd=str(tmp_path), input=text if extra == ("-",) else None, env=env)
    out = (tmp_path / "depth.bed").read_bytes() if p.returncode == 0 else None
    return p, out


def _matrix_text(rng, rows, S, header=True, frac=False):
    lines = [b"#chrom\tstart\tend\t" + b"\t".join(b"s%d" % i for i in range(S))] if header else []
    for c, s, e in rows:
        v = rng.gamma(4.0, 8.0, S)
        toks = [b"%.3f" % x for x in v] if frac else [b"%d" % int(x) for x in v]
        lines.append(b"%s\t%d\t%d\t" % (c.encode(), s, e) + b"\t".join(toks))
    return b"\n".join(lines) + b"\n"


def _tiled(chrom, L, size, start=0):
    return [(chrom, a, min(a + size, L)) for a in range(start, L - size, size)]


def test_pipeline_depth_depthwed_dcnv(ref, tmp_path):
    d, fa_path, fa, fai = ref
    beds = []
    for k in range(3):
        rng = np.random.default_rng(40 + k)
        recs = []
        for tid, (_, L) in enumerate(REFS):
            for p in np.sort(rng.integers(0, L - 100, int((20 + 5 * k) * L / 100))):
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
    assert mat.count(b"\n") > 60
    p, got = dcnv(ref, mat, tmp_path)
    assert p.returncode == 0, p.stderr
    assert got == od.dcnv(mat, fa, fai)


@pytest.mark.parametrize("frac", [False, True])
def test_tie_heavy_matrix(ref, tmp_path, frac):
    """a few thousand rows of one window size: a few hundred distinct GC values, pdqsort's partition paths"""
    _, _, fa, fai = ref
    rng = np.random.default_rng(2 + frac)
    rows = _tiled("chrM", 16571, 40) + _tiled("chr22", 60001, 40)
    text = _matrix_text(rng, rows, 7, frac=frac)
    p, got = dcnv(ref, text, tmp_path)
    assert p.returncode == 0, p.stderr
    assert got == od.dcnv(text, fa, fai)
    assert got.count(b"\n") == len(rows) + 1
    # the same through gzip, stdin and several column blocks
    for extra, name, env in (((), "m.tsv.gz", None), (("-",), "m.tsv", None), ((), "m.tsv", {"GL_DCNV_BLOCK_COLS": "2"})):
        p, again = dcnv(ref, text, tmp_path, *extra, name=name, env=env)
        assert p.returncode == 0, p.stderr
        assert again == got, (extra, name, env)


def test_quirks(ref, tmp_path):
    _, _, fa, fai = ref
    rng = np.random.default_rng(6)
    # label: every row is labelled with the SECOND data line's chromosome; GC still uses each row's own
    rows = [("chrM", 0, 100)] + [("chr22", a, a + 500) for a in range(100, 5100, 500)] + _tiled("chrM", 16571, 500, 1000)
    text = _matrix_text(rng, rows, 3)
    # two header lines before the first data line: the second names the samples; an unterminated last line is dropped
    text = b"#chrom\tstart\tend\tx\ty\tz\n" + text + b"chrM\t9\t99\t1\t2\t3"
    p, got = dcnv(ref, text, tmp_path)
    assert p.returncode == 0, p.stderr
    assert got == od.dcnv(text, fa, fai)
    lines = got.split(b"\n")
    assert lines[0] == b"#chrom\tstart\tend\ts0\ts1\ts2"
    assert all(ln.startswith(b"chr22\t") for ln in lines[1:-1]) and len(lines) == len(rows) + 2
    assert lines[1].startswith(b"chr22\t250\t100\t")                  # start < 250 is printed as 250
    assert b"WARNING: no change after sorting" not in p.stderr
    # every GC equal (a sequence the FASTA does not have): the permutation is the identity, and the reference says so
    same = _matrix_text(rng, [("chrUn", a, a + 1000) for a in range(0, 20000, 1000)], 2)
    p, got = dcnv(ref, same, tmp_path)
    assert p.returncode == 0, p.stderr
    assert b"WARNING: no change after sorting" in p.stderr and b"unknown sequence chrUn" in p.stderr
    assert got == od.dcnv(same, fa, fai)


def test_errors(ref, tmp_path):
    _, fa_path, fa, fai = ref
    rng = np.random.default_rng(1)
    rows = _tiled("chrM", 16571, 1000)
    good = _matrix_text(rng, rows, 3)
    hdr, body = good.split(b"\n", 1)
    cases = {
        "no header": body,
        "zero samples": b"#chrom\tstart\tend\n" + b"".join(b"chrM\t%d\t%d\n" % (s, e) for _, s, e in rows),
        "column count": good.replace(b"\n", b"\t7\n", 3).replace(hdr + b"\t7", hdr, 1),
        "few rows": b"\n".join(good.split(b"\n")[:5]) + b"\n",
        "past the end": good + b"chrM\t16000\t17000\t1\t2\t3\n",
        "bad token": good + b"chrM\t1000\t2000\t1\tabc\t3\n",
        "nan token": good + b"chrM\t1000\t2000\t1\tNaN\t3\n",
        "overflow": good + b"chrM\t1000\t2000\t1\t1e999\t3\n",
        "bad start": good + b"chrM\tx\t2000\t1\t2\t3\n",
        "all zero": b"\n".join([hdr] + [ln.rsplit(b"\t", 1)[0] + b"\t0" for ln in body.split(b"\n")[:-1]]) + b"\n",
    }
    for what, text in cases.items():
        with pytest.raises(od.Panic):
            od.dcnv(text, fa, fai)
        p, _ = dcnv(ref, text, tmp_path)
        assert p.returncode == 2 and b"panic" in p.stderr, (what, p.returncode, p.stderr)
    p = run("dcnv", str(tmp_path / "m.tsv"))
    assert p.returncode == 2 and b"panic" in p.stderr
    p = run("dcnv", str(tmp_path / "absent.tsv"), fa_path, cwd=str(tmp_path))
    assert p.returncode == 2
