"""`goleft covstats --gpus N` over a cohort: every N prints the bytes `--gpus 1` prints (stdout, stderr, exit code and the
--hist files), the rows are the single-BAM runs' rows, and a BAM that fails mid-cohort ends the run at the same row with
the same message whichever worker sampled it."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench_covstats  # noqa: E402
import covstats_ref as cr  # noqa: E402
from covstats_bams import odd_member  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
N_ARGS = ("-n", "50000")
GPUS = (2, 3, 7, 12)


def run(bams, gpus, hist=None, env=None):
    args = [GOLEFT, "covstats", *N_ARGS, "--gpus", str(gpus)] + (["--hist", hist] if hist else []) + list(bams)
    return subprocess.run(args, capture_output=True, env=dict(os.environ, GL_OVERSUBSCRIBE="1", **(env or {})))


def hist_files(d):
    return {f: open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))}


@pytest.fixture(scope="module")
def cohort(tmp_path_factory):
    """11 BAMs: paired BAMs of 120 k to 500 k records with distinct samples, one the device refuses (an odd BGZF member),
    one without a read group, one whose index has no stats bin for an empty 3 Mb reference, and two sharing sample D"""
    d = tmp_path_factory.mktemp("cohort")

    def paired(name, n, seed, sample):
        p = str(d / name)
        bench_covstats.write_paired_bam(p, n_records=n, seed=seed, sample=sample)
        return p
    refs, recs, mates = cr.records(np.random.default_rng(70), [104_000, 0], ref_len=3_000_000)
    empty_ref = cr.write(d, "emptyref.bam", refs, recs, mates)
    bams = [paired("a.bam", 150_000, 1, "A"), paired("b.bam", 400_000, 2, "B"), odd_member(paired("c.bam", 200_000, 3, "C")),
            paired("norg.bam", 120_000, 4, ""), empty_ref, paired("d1.bam", 300_000, 5, "D"), paired("d2.bam", 180_000, 6, "D"),
            paired("e.bam", 250_000, 7, "E"), paired("f.bam", 130_000, 8, "F"), paired("g.bam", 500_000, 9, "G"),
            paired("h.bam", 160_000, 10, "H")]
    return d, bams


def test_every_gpu_count_prints_the_same_bytes(cohort, tmp_path):
    _, bams = cohort
    outs = {}
    for g in (1,) + GPUS:
        hd = tmp_path / ("g%d" % g)
        hd.mkdir()
        r = run(bams, g, str(hd / "x"))
        outs[g] = (r, hist_files(str(hd)))
    ref, ref_hist = outs[1]
    assert ref.returncode == 0, ref.stderr
    assert ref.stdout.count(b"\n") == 1 + len(bams)
    assert b"<no-read-groups>" in ref.stdout and b"chromosomes: c1 not found in " in ref.stderr
    assert sorted(ref_hist) == sorted("x.%s.template_hist.tsv" % s for s in ("A", "B", "C", "<no-read-groups>", "S1", "D", "E", "F", "G", "H"))
    for g, (r, h) in outs.items():
        assert (r.returncode, r.stdout, r.stderr) == (ref.returncode, ref.stdout, ref.stderr), g
        assert h == ref_hist, g
    # the last BAM of sample D wins, as in the sequential loop
    hd = tmp_path / "d2"
    hd.mkdir()
    assert run([bams[6]], 1, str(hd / "x")).returncode == 0
    assert hist_files(str(hd))["x.D.template_hist.tsv"] == ref_hist["x.D.template_hist.tsv"]
    # the rows are the single-BAM runs' rows
    singles = [run([b], 1) for b in bams]
    assert ref.stdout == singles[0].stdout.split(b"\n")[0] + b"\n" + b"".join(s.stdout.split(b"\n", 1)[1] for s in singles)
    assert ref.stderr == b"".join(s.stderr for s in singles)
    # the host sampler on every worker
    hd = tmp_path / "host"
    hd.mkdir()
    r = run(bams, 3, str(hd / "x"), env={"GL_GPU_FEED": "0"})
    assert (r.returncode, r.stdout, r.stderr) == (ref.returncode, ref.stdout, ref.stderr) and hist_files(str(hd)) == ref_hist


@pytest.fixture(scope="module")
def failing(cohort):
    """three BAMs that end a run: no .bai, and one whose sample has two insert sizes (madFilter's panic)"""
    d, bams = cohort
    noidx = str(d / "noidx.bam")
    shutil.copy(bams[0], noidx)
    rng = np.random.default_rng(71)
    refs, recs, mates = cr.records(rng, [102_000, 3000], flags=[0, 16, 0x400])
    for i in (100_100, 100_105):
        recs[i] = (recs[i][0], recs[i][1], 60, 99, [(100, "M")])
        mates[i] = (recs[i][1] + 300, 400)
    two = cr.write(d, "two_inserts.bam", refs, recs, mates)
    return {"missing": str(d / "missing.bam"), "no_bai": noidx, "two_inserts": two}


@pytest.mark.parametrize("kind", ["missing", "no_bai", "two_inserts"])
def test_failure_mid_cohort(cohort, failing, tmp_path, kind):
    _, bams = cohort
    good = [bams[i] for i in (0, 1, 3, 5, 7, 8, 9, 10)]              # samples A, B, <no-read-groups>, D, E, F, G, H
    row = good[:4] + [failing[kind]] + good[4:]
    head = run(good[:4], 1)
    assert head.returncode == 0
    ref = None
    for g in (1,) + GPUS:
        hd = tmp_path / ("g%d" % g)
        hd.mkdir()
        r = run(row, g, str(hd / "x"))
        ref = ref or r
        assert r.returncode == (2 if kind == "two_inserts" else 1), r.stderr
        assert r.stdout == head.stdout, g
        assert (r.returncode, r.stderr) == (ref.returncode, ref.stderr), g
        assert sorted(os.listdir(str(hd))) == sorted("x.%s.template_hist.tsv" % s for s in ("A", "B", "<no-read-groups>", "D")), g
    if kind == "two_inserts":
        assert ref.stderr.startswith(b"panic: runtime error: index out of range")
