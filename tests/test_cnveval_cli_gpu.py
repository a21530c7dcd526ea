"""End-to-end `goleft cnveval` (bin/goleft): stdout must equal the oracle's text for every input form; exit codes; and a
pipeline from planted copy-number runs through `goleft emdepth` to a recall of 1."""
import gzip
import os
import subprocess
from collections import Counter

import numpy as np
import pytest

from cnveval_sets import cohort
from oracle import cnveval as oc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLEFT = os.path.join(ROOT, "bin", "goleft")
CHROMS = [b"chr1", b"chr10", b"chr2"]                              # bytewise order is not numeric order


@pytest.fixture(scope="module")
def tools():
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")


def run(*args, input=None, env=None):
    return subprocess.run([GOLEFT, "cnveval", *args], capture_output=True, input=input,
                          env=dict(os.environ, **env) if env else None)


def _texts(rng, S=40, T=400):
    cs, cc, cb, ce, ccn, tc, tb, te, tcn, mp, ms = cohort(rng, S, T)
    test = [b"%s\t%d\t%d\t%d\ts%d" % (CHROMS[c], b, e, n, s) + (b",s%d" % ((s + 1) % S) if k % 5 == 0 else b"")
            for k, (s, c, b, e, n) in enumerate(zip(cs, cc, cb, ce, ccn))]
    truth = [b"%s\t%d\t%d\t%d\t%s" % (CHROMS[tc[t]], tb[t], te[t], tcn[t], b",".join(b"s%d" % x for x in ms[mp[t]:mp[t + 1]]))
             for t in range(T)]
    return truth, test


def _join(lines, crlf_every=0, header=True):
    out = [b"#chrom\tstart\tend\tcn\tsamples"] if header else []
    for k, ln in enumerate(lines):
        out.append(ln + (b"\r" if crlf_every and k % crlf_every == 0 else b""))
    return b"\n".join(out) + b"\n"


def test_text_equals_oracle(tools, tmp_path):
    rng = np.random.default_rng(1401)
    truth, test = _texts(rng)
    tr, te = _join(truth, crlf_every=7), _join(test, crlf_every=3)
    te_unterminated = te + b"chr1\t0\t5000\t1\ts0"                    # dropped, as ReadString drops it
    (tmp_path / "truth.bed").write_bytes(tr)
    (tmp_path / "test.bed").write_bytes(te_unterminated)
    (tmp_path / "truth.bed.gz").write_bytes(gzip.compress(tr))
    (tmp_path / "test.bed.gz").write_bytes(gzip.compress(te_unterminated))
    t, x = str(tmp_path / "truth.bed"), str(tmp_path / "test.bed")
    for args, po, limit in ((([t, x]), 0.4, False), (["-s", t, x], 0.4, True), (["-m", "0.5", t, x], 0.5, False),
                            (["--minoverlap=1", "--limitsamples", t, x], 1.0, True), (["-m", "NaN", t, x], float("nan"), False)):
        r = run(*args)
        assert r.returncode == 0, (args, r.stderr)
        assert r.stdout == oc.cnveval(tr, te, po, limit), args
        assert b"cnvs in test-set (%d)" % len(test) in r.stderr
    want = oc.cnveval(tr, te)
    r = run(str(tmp_path / "truth.bed.gz"), str(tmp_path / "test.bed.gz"))
    assert r.returncode == 0 and r.stdout == want
    r = run(t, "-", input=te_unterminated, env={"GL_TIMING": "1"})
    assert r.returncode == 0 and r.stdout == want and b"[cnveval timing]" in r.stderr
    n_mem = sum(ln.split(b"\t")[4].count(b",") + 1 for ln in truth)
    assert b"%d total cnvs in truth-set (%d)" % (n_mem, len(truth)) in r.stderr
    assert not os.path.exists("x.cpu.pprof")


def test_exit_codes(tools, tmp_path):
    good = tmp_path / "good.bed"
    good.write_bytes(b"chr1\t100\t200\t1\tA\n")
    cases = {"fields": b"chr1\t100\t200\t1\n", "int": b"chr1\t100\tx\t1\tA\n", "end_before_start": b"chr1\t300\t200\t1\tA\n"}
    for name, text in cases.items():
        p = tmp_path / (name + ".bed")
        p.write_bytes(text)
        for args in ((str(good), str(p)), (str(p), str(good))):
            r = run(*args)
            assert r.returncode == 2 and b"panic: " in r.stderr, (name, r.returncode, r.stderr)
    assert run(str(good), str(tmp_path / "absent.bed")).returncode == 2
    for m in ("0", "1.5"):
        assert run("-m", m, str(good), str(good)).returncode == 255
    r = run(str(good), str(good))
    assert r.returncode == 0 and r.stdout.splitlines()[3].startswith(b"size-class: all          | precision: 1.0000 (1    /")


def test_pipeline_emdepth_recall(tools, tmp_path):
    """planted CN1 / CN3 runs -> `goleft emdepth` -> P.cnv.bed rows as test lines (CN = the majority of
    the run's non-2 CNs) -> recall 1"""
    rng = np.random.default_rng(1402)
    S = 24
    rows = [(b"chr1", a, a + 1000) for a in range(0, 400_000, 1000)] + [(b"chr2", a, a + 1000) for a in range(0, 200_000, 1000)]
    plants = [(100, 140, 5, 0.5, 1), (450, 480, 9, 1.5, 3), (250, 290, 2, 0.5, 1), (520, 560, 17, 1.5, 3)]
    x = rng.gamma(40.0, 1.0, (len(rows), S))
    for a, b, s, f, _ in plants:
        x[a:b, s] *= f
    mat = [b"#chrom\tstart\tend\t" + b"\t".join(b"s%d" % i for i in range(S))]
    mat += [b"%s\t%d\t%d\t" % r + b"\t".join(b"%d" % int(v) for v in x[k]) for k, r in enumerate(rows)]
    (tmp_path / "m.tsv").write_bytes(b"\n".join(mat) + b"\n")
    prefix = str(tmp_path / "em")
    p = subprocess.run([GOLEFT, "emdepth", "--prefix", prefix, str(tmp_path / "m.tsv")], capture_output=True)
    assert p.returncode == 0, p.stderr
    test = []
    for ln in open(prefix + ".cnv.bed", "rb").read().split(b"\n")[1:-1]:
        chrom, start, end, sample, _, cns, _ = ln.split(b"\t")
        # the run's majority CN among its non-2 rows: emdepth's Poisson test puts noisy rows of a run back at CN 2
        cn = (Counter(c for c in cns.split(b",") if c != b"2").most_common(1) or [(b"2", 0)])[0][0]
        test.append(b"\t".join([chrom, start, end, cn, sample]))
    truth = [b"%s\t%d\t%d\t%d\ts%d" % (rows[a][0], rows[a][1], rows[b - 1][2], cn, s) for a, b, s, _, cn in plants]
    (tmp_path / "truth.bed").write_bytes(b"\n".join(truth) + b"\n")
    (tmp_path / "test.bed").write_bytes(b"\n".join(test) + b"\n")
    r = run(str(tmp_path / "truth.bed"), str(tmp_path / "test.bed"))
    assert r.returncode == 0, r.stderr
    assert r.stdout == oc.cnveval((tmp_path / "truth.bed").read_bytes(), (tmp_path / "test.bed").read_bytes())
    assert b"recall: 1.0000 (4    / (4    + 0   ))" in r.stdout.splitlines()[3], r.stdout
