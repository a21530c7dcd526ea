"""End-to-end `goleft dcnv --svd PCT` (bin/goleft, DESIGN §1.13): depth.bed against the numpy SVD oracle's "%.2f" text, the
input forms, the log line, the flag's errors, the unchanged default, and the point of the feature: batch-driven false CNVs
gone from `dcnv` -> `emdepth` -> `cnveval` while the planted CNVs are all still found."""
import gzip
import os
import re
import subprocess
from collections import Counter

import numpy as np
import pytest

from fautil import make_fasta
from oracle import cnveval as oc
from oracle import dcnv as od
from oracle import dcnv_svd as osv

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLEFT = os.path.join(ROOT, "bin", "goleft")
REFS = [("chr1", 1_200_000)]


@pytest.fixture(scope="module")
def ref(tmp_path_factory):
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    d = tmp_path_factory.mktemp("dcnv_svd")
    fa, fai, _ = make_fasta(REFS, seed=11, line=60)
    path = str(d / "ref.fa")
    open(path, "wb").write(fa)
    open(path + ".fai", "w").write(fai)
    return path, fa, fai


def dcnv(ref, tmp_path, text, *flags, stdin=False, gz=False):
    p = tmp_path / ("m.tsv.gz" if gz else "m.tsv")
    p.write_bytes(gzip.compress(text) if gz else text)
    r = subprocess.run([GOLEFT, "dcnv", *flags, "-" if stdin else str(p), ref[0]], capture_output=True, cwd=str(tmp_path),
                       input=text if stdin else None)
    return r, (tmp_path / "depth.bed").read_bytes() if r.returncode == 0 else None


def _matrix(rows, x):
    S = x.shape[1]
    lines = [b"#chrom\tstart\tend\t" + b"\t".join(b"s%d" % i for i in range(S))]
    lines += [b"%s\t%d\t%d\t" % r + b"\t".join(b"%d" % v for v in x[k]) for k, r in enumerate(rows)]
    return b"\n".join(lines) + b"\n"


def _batch_cohort(rng, S=32, n_rows=1100, plants=()):
    """Poisson(100) depths on 1 kb rows; samples 0..S/2-1 carry a batch term, up or down on stretches of rows"""
    rows = [(b"chr1", a, a + 1000) for a in range(0, n_rows * 1000, 1000)]
    f = np.ones(n_rows)
    for k, a in enumerate(range(30, n_rows - 40, 60)):
        f[a:a + 25] = 1.8 if k % 2 == 0 else 0.45
    lam = 100.0 * np.ones((n_rows, S))
    lam[:, :S // 2] *= f[:, None]
    for a, b, s, fac, _ in plants:
        lam[a:b, s] *= fac
    return rows, rng.poisson(lam)


def _f2_boundary(v):
    """distance of v from the nearest "%.2f" rounding boundary (x.xx5)"""
    t = np.abs(np.asarray(v)) * 100 - 0.5
    return np.abs(t - np.round(t)) / 100


def test_text_against_oracle(ref, tmp_path):
    rng = np.random.default_rng(1301)
    rows, x = _batch_cohort(rng, S=24, n_rows=700)
    text = _matrix(rows, x)
    pct = 5.0
    want, vals, logline = osv.dcnv(text, ref[1], ref[2], pct)
    r, got = dcnv(ref, tmp_path, text, "--svd", "5")
    assert r.returncode == 0, r.stderr
    assert logline.startswith(b"variance: ") and re.search(rb"\d{4}/\d\d/\d\d \d\d:\d\d:\d\d " + re.escape(logline) + b"\n", r.stderr)
    gl, wl = got.split(b"\n"), want.split(b"\n")
    assert len(gl) == len(wl) and gl[0] == wl[0]
    near = 0
    for i, (a, b) in enumerate(zip(gl[1:-1], wl[1:-1])):
        if a == b:
            continue
        fa, fb = a.split(b"\t"), b.split(b"\t")
        assert fa[:3] == fb[:3]
        for j, (p, q) in enumerate(zip(fa[3:], fb[3:])):
            if p != q:                                                    # only where the oracle sits on a rounding edge
                assert _f2_boundary(vals[i, j]) <= 1e-6 and abs(float(p) - float(q)) <= 0.0100001, (i, j, p, q, vals[i, j])
                near += 1
    assert near <= 5, near
    # the same through gzip, stdin and --svd=PCT
    for kw, flags in (({"gz": True}, ("--svd", "5")), ({"stdin": True}, ("--svd", "5")), ({}, ("--svd=5.0",))):
        r, again = dcnv(ref, tmp_path, text, *flags, **kw)
        assert r.returncode == 0 and again == got, (kw, flags)


def test_default_and_nothing_removed_unchanged(ref, tmp_path):
    rng = np.random.default_rng(1302)
    rows, x = _batch_cohort(rng, S=12, n_rows=300)
    text = _matrix(rows, x)
    want = od.dcnv(text, ref[1], ref[2])
    r, plain = dcnv(ref, tmp_path, text)
    assert r.returncode == 0 and plain == want and b"variance" not in r.stderr
    r, none = dcnv(ref, tmp_path, text, "--svd", "100")                   # no component above 100 %: the same bytes
    assert r.returncode == 0 and none == plain
    assert re.search(rb" variance:\n", r.stderr), r.stderr
    r, _ = dcnv(ref, tmp_path, text, "--svd", "0")
    assert r.returncode == 0 and re.search(rb" variance:( \d+\.\d\d)+\n", r.stderr)


def test_bad_pct_exit_255(ref, tmp_path):
    text = _matrix(*_batch_cohort(np.random.default_rng(3), S=4, n_rows=50))
    for flags in (("--svd", "-1"), ("--svd", "nan"), ("--svd", "inf"), ("--svd", "abc"), ("--svd=",), ("--svd=-0.5",)):
        r, _ = dcnv(ref, tmp_path, text, *flags)
        assert r.returncode == 255 and b"error" in r.stderr, (flags, r.returncode, r.stderr)
    r = subprocess.run([GOLEFT, "dcnv", "--svd"], capture_output=True, cwd=str(tmp_path))
    assert r.returncode == 255


def _calls(prefix):
    test = []
    for ln in open(prefix + ".cnv.bed", "rb").read().split(b"\n")[1:-1]:
        chrom, start, end, sample, _, cns, _ = ln.split(b"\t")
        cn = (Counter(c for c in cns.split(b",") if c != b"2").most_common(1) or [(b"2", 0)])[0][0]
        test.append(b"\t".join([chrom, start, end, cn, sample]))
    return test


def test_pipeline_batch_false_calls_removed(ref, tmp_path):
    """A cohort with rare planted CN1 / CN3 runs and a strong batch term on half the samples.  depth.bed holds relative
    depths (1 = the sample's median); emdepth's Poisson test wants counts, so its input is depth.bed times 100, the
    cohort's depth.  Without --svd the batch stretches come out as dozens of false CNVs; with it they are gone, and every
    planted CNV is still found."""
    rng = np.random.default_rng(1303)
    plants = [(100, 130, 20, 0.5, 1), (400, 430, 5, 1.5, 3), (700, 740, 27, 0.5, 1), (950, 990, 9, 1.5, 3)]
    rows, x = _batch_cohort(rng, S=32, plants=plants)
    text = _matrix(rows, x)
    truth = b"\n".join(b"chr1\t%d\t%d\t%d\ts%d" % (rows[a][1], rows[b - 1][2], cn, s) for a, b, s, _, cn in plants) + b"\n"
    (tmp_path / "truth.bed").write_bytes(truth)
    stats = {}
    for mode, flags in (("plain", ()), ("svd", ("--svd", "10"))):
        r, got = dcnv(ref, tmp_path, text, *flags)
        assert r.returncode == 0, r.stderr
        lines = got.split(b"\n")
        scaled = [lines[0]] + [b"\t".join(f[:3] + [b"%.0f" % (100 * float(v)) for v in f[3:]])
                               for f in (ln.split(b"\t") for ln in lines[1:-1])]
        (tmp_path / "em.tsv").write_bytes(b"\n".join(scaled) + b"\n")
        prefix = str(tmp_path / ("em_" + mode))
        p = subprocess.run([GOLEFT, "emdepth", "--prefix", prefix, str(tmp_path / "em.tsv")], capture_output=True)
        assert p.returncode == 0, p.stderr
        test = b"\n".join(_calls(prefix)) + b"\n"
        (tmp_path / "test.bed").write_bytes(test)
        p = subprocess.run([GOLEFT, "cnveval", str(tmp_path / "truth.bed"), str(tmp_path / "test.bed")], capture_output=True)
        assert p.returncode == 0, p.stderr
        assert p.stdout == oc.cnveval(truth, test)
        m = re.findall(rb"\((\d+) +/ \((\d+) +\+ (\d+) *\)\)", p.stdout.splitlines()[3])      # precision, recall
        assert len(m) == 2, p.stdout
        (tp, _, fp), (rtp, _, fn) = [[int(v) for v in g] for g in m]
        stats[mode] = (tp, fp, rtp, fn)
    assert stats["plain"][1] >= 24, stats                                # dozens of batch-driven false CNVs without the flag
    assert stats["svd"][1] <= 2, stats                                   # gone with it
    assert stats["svd"][2] == 4 and stats["svd"][3] == 0, stats          # recall 1
