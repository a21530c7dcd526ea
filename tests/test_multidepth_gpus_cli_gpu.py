"""`goleft multidepth --gpus N` end to end (bin/goleft): the samples sharded over N workers print the oracle's bytes and
those of --gpus 1, with the same stderr and exit codes.  GL_OVERSUBSCRIBE=1 keeps N workers on fewer devices, so every N
runs on a one-GPU box; with several devices the workers spread over them (worker g on device g % n)."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_multidepth_cli_gpu import _expect, _sample_bam  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
GPUS = ["1", "2", "3", "7"]
FLAGS = [([], {}), (["-w", "15", "-m", "3", "-k", "4", "--mincov", "5", "--minsamples", "0.3"],
                    dict(window=15, min_size=3, max_skip=4, mincov=5, min_samples=0.3))]


def run(*args, **env):
    return subprocess.run([GOLEFT, *args], capture_output=True, env=dict(os.environ, GL_OVERSUBSCRIBE="1", **env))


@pytest.fixture(scope="module")
def cohort(tmp_path_factory):
    """seven indexed BAMs of uneven size, one with no reads passing the filters (coverage 0), and the same cohort with
    samples 0, 3 and 5 unindexed"""
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    d = tmp_path_factory.mktemp("mdg")
    covs = [30, 3, 28, 0, 35, 32, 30]
    paths, plain, depths = [], [], []
    for i, c in enumerate(covs):
        p = str(d / f"s{i}.bam")
        depths.append(_sample_bam(p, f"SM{i}", c, 70 + i))
        paths.append(p)
        if i in (0, 3, 5):
            q = str(d / f"plain{i}.bam")
            assert np.array_equal(_sample_bam(q, f"SM{i}", c, 70 + i, indexed=False), depths[-1])
            plain.append(q)
        else:
            plain.append(p)
    return paths, plain, np.stack(depths), [f"SM{i}" for i in range(len(covs))]


@pytest.mark.parametrize("feed", ["1", "0"])
def test_every_split_prints_the_same_bytes(cohort, feed):
    paths, _, depths, names = cohort
    for args, kw in FLAGS:
        exp = _expect(depths, names, **kw)
        assert exp.count(b"\n") > 2
        one = run("multidepth", "-c", "chr1", "--gpus", "1", *args, *paths, GL_GPU_FEED=feed)
        assert one.returncode == 0, one.stderr
        assert one.stdout == exp
        for g in GPUS[1:] + ["9", "0"]:                      # 9 > S: one worker per sample; 0: every visible device
            p = run("multidepth", "-c", "chr1", "--gpus", g, *args, *paths, GL_GPU_FEED=feed)
            assert (p.returncode, p.stdout, p.stderr) == (0, exp, one.stderr), (g, args)


@pytest.mark.parametrize("gpus", GPUS)
def test_unindexed_bams(cohort, gpus):
    _, plain, depths, names = cohort
    exp = _expect(depths, names, window=1000)
    p = run("multidepth", "-c", "chr1", "-w", "1000", "--gpus", gpus, *plain)
    assert p.returncode == 0, p.stderr
    assert p.stdout == exp


def test_gpus_without_oversubscribe(cohort):
    """without GL_OVERSUBSCRIBE, --gpus above the device count means one worker per device"""
    paths, _, depths, names = cohort
    env = {k: v for k, v in os.environ.items() if k != "GL_OVERSUBSCRIBE"}
    p = subprocess.run([GOLEFT, "multidepth", "-c", "chr1", "--gpus", "7", *paths], capture_output=True, env=env)
    assert p.returncode == 0, p.stderr
    assert p.stdout == _expect(depths, names)


def test_errors_same_for_every_split(cohort, tmp_path):
    paths, _, _, _ = cohort
    from bamutil import make_bam_indexed
    other = str(tmp_path / "other.bam")
    bam, bai = make_bam_indexed([("chr2", 1000)], [(0, 10, 60, 0, [(100, "M")])], sample="Z")
    open(other, "wb").write(bam)
    open(other + ".bai", "wb").write(bai)
    cases = [("-c", "chrX", *paths),                         # missing from every BAM: the first one is named
             ("-c", "chr1", *paths[:4], other, *paths[4:]),  # missing from the fifth
             ("-c", "chr1", paths[0], str(tmp_path / "missing.bam"), *paths[1:])]
    for args in cases:
        ref = run("multidepth", "--gpus", "1", *args)
        assert ref.returncode != 0 and ref.stderr and not ref.stdout
        for g in GPUS[1:]:
            p = run("multidepth", "--gpus", g, *args)
            assert (p.returncode, p.stdout, p.stderr) == (ref.returncode, ref.stdout, ref.stderr), (g, args)
