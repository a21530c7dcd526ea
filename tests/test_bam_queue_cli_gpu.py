"""What the BAM subcommands share, end to end (bin/goleft): the in-order BAM queue of covstats and depthwed (a run ends with
the first failure in argument order, and prints the same bytes for every --gpus split; GL_OVERSUBSCRIBE=1 keeps N workers
on fewer devices), the unindexed-BAM rule (a stub .bai is no index, in multidepth as in depth and depthwed), and the pass
length of depth and depthwed."""
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
from bamutil import make_bai, make_bam, make_bam_indexed  # noqa: E402
from test_multidepth_cli_gpu import _expect, _sample_bam  # noqa: E402

GOLEFT = os.path.join(ROOT, "bin", "goleft")
REFS = [("chr1", 40000), ("chr2", 9000)]
GPUS = ("1", "2", "3", "7")
NOTE = "goleft depthwed: no usable index (.bai or .csi) next to %s: decoding the whole file\n"


def run(*args, **env):
    return subprocess.run([GOLEFT, *args], capture_output=True, env=dict(os.environ, GL_OVERSUBSCRIBE="1", **env))


def _records(seed):
    rng = np.random.default_rng(seed)
    return [(tid, int(p), 60, 0, [(100, "M")]) for tid, (_, L) in enumerate(REFS) for p in np.sort(rng.integers(0, L - 100, L // 4))]


@pytest.fixture(scope="module")
def wed(tmp_path_factory):
    """BAMs without an index (u*) and with one (i*), cut.bam (no index, truncated half way: its whole-file decode fails),
    and ref.fa.fai"""
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    d = tmp_path_factory.mktemp("queue")
    paths = {}
    for k, name in enumerate(("u0", "i1", "u2", "u3", "i4", "u5")):
        p = str(d / (name + ".bam"))
        if name[0] == "i":
            bam, bai = make_bam_indexed(REFS, _records(k), sample=name)
            open(p + ".bai", "wb").write(bai)
        else:
            bam = make_bam(REFS, _records(k), sample=name)
        open(p, "wb").write(bam)
        paths[name] = p
    bam = make_bam(REFS, _records(9), sample="cut")
    paths["cut"] = str(d / "cut.bam")
    open(paths["cut"], "wb").write(bam[:len(bam) // 2 + 7])
    open(d / "ref.fa.fai", "w").write("".join("%s\t%d\t6\t60\t61\n" % r for r in REFS))
    return str(d / "ref.fa"), paths


@pytest.mark.gpu
@pytest.mark.parametrize("feed", ["1", "0"])
def test_depthwed_failure_mid_cohort(wed, feed):
    """the notes of the BAMs committed up to the failure, in argument order, then the failure; nothing on stdout"""
    ref, p = wed
    bams = [p[k] for k in ("u0", "i1", "u2", "cut", "u3", "i4", "u5")]
    want = "".join(NOTE % p[k] for k in ("u0", "u2", "cut")) + "truncated BGZF block in %s\n" % p["cut"]
    for g in GPUS:
        r = run("depthwed", "-s", "500", "-r", ref, "--gpus", g, *bams, GL_GPU_FEED=feed)
        assert (r.returncode, r.stdout, r.stderr.decode()) == (1, b"", want), g


@pytest.mark.gpu
def test_depthwed_unopenable_first_or_last(wed, tmp_path):
    ref, p = wed
    good = [p[k] for k in ("u0", "i1", "u2")]
    missing = str(tmp_path / "missing.bam")
    for bams, notes in (([missing] + good, ""), (good + [missing], NOTE % p["u0"] + NOTE % p["u2"])):
        one = run("depthwed", "-s", "500", "-r", ref, "--gpus", "1", *bams)
        assert one.returncode == 1 and not one.stdout
        assert one.stderr.decode().startswith(notes) and missing in one.stderr.decode()[len(notes):]
        for g in GPUS[1:]:
            r = run("depthwed", "-s", "500", "-r", ref, "--gpus", g, *bams)
            assert (r.returncode, r.stdout, r.stderr) == (one.returncode, one.stdout, one.stderr), g


@pytest.mark.gpu
def test_covstats_unopenable_first_or_last(tmp_path):
    """the rows of the BAMs before the one that cannot be opened, then its error; a second such BAM later is not reported"""
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    good = []
    for k in range(3):
        good.append(str(tmp_path / ("g%d.bam" % k)))
        bench_covstats.write_paired_bam(good[-1], n_records=120_000, seed=30 + k, sample="G%d" % k)
    missing, missing2 = str(tmp_path / "missing.bam"), str(tmp_path / "missing2.bam")
    head = run("covstats", "-n", "50000", "--gpus", "1", *good)
    assert head.returncode == 0 and head.stdout.count(b"\n") == 4
    header = head.stdout.split(b"\n", 1)[0] + b"\n"
    for bams, rows in (([missing] + good, header), (good + [missing], head.stdout), ([missing] + good + [missing2], header)):
        one = run("covstats", "-n", "50000", "--gpus", "1", *bams)
        assert (one.returncode, one.stdout) == (1, rows)
        err = one.stderr[len(head.stderr):] if rows == head.stdout else one.stderr
        assert missing.encode() in err and missing2.encode() not in one.stderr and err.count(b"\n") == 1
        for g in GPUS[1:]:
            r = run("covstats", "-n", "50000", "--gpus", g, *bams)
            assert (r.returncode, r.stdout, r.stderr) == (one.returncode, one.stdout, one.stderr), g


@pytest.mark.gpu
@pytest.mark.parametrize("feed", ["1", "0"])
def test_multidepth_stub_index_is_no_index(tmp_path, feed):
    """a sample whose .bai has a stats bin but an all-zero linear index is decoded whole, as without an index"""
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    covs = [30, 3, 28, 25]
    paths, depths = [], []
    for i, c in enumerate(covs):
        paths.append(str(tmp_path / ("s%d.bam" % i)))
        depths.append(_sample_bam(paths[-1], "SM%d" % i, c, 80 + i, indexed=i != 2))
    (tmp_path / "stub").mkdir()
    stub = str(tmp_path / "stub" / "s2.bam")
    shutil.copy(paths[2], stub)
    open(stub + ".bai", "wb").write(make_bai([[0], [0]], [(1000, 0), (300, 0)]))
    exp = _expect(np.stack(depths), ["SM%d" % i for i in range(len(covs))])
    for g in ("1", "3"):
        plain = run("multidepth", "-c", "chr1", "--gpus", g, *paths, GL_GPU_FEED=feed)
        assert (plain.returncode, plain.stdout) == (0, exp), plain.stderr
        r = run("multidepth", "-c", "chr1", "--gpus", g, *paths[:2], stub, paths[3], GL_GPU_FEED=feed)
        assert (r.returncode, r.stdout, r.stderr) == (0, exp, plain.stderr), g


def test_window_above_one_pass(wed):
    """a window wider than the 2^30 - 1 bases of one pass leaves no pass: depth and depthwed refuse it before any GPU work"""
    ref, p = wed
    for prog, args in (("depth", ["--prefix", ref + ".x"]), ("depthwed", ["-s", "500"])):
        r = run(prog, *args, "-r", ref, "-w", "2000000000", p["i1"])
        assert (r.returncode, r.stderr) == (1, b"goleft %s: windowsize 2000000000 is above the 2^30 - 1 bases of one pass\n" % prog.encode())
