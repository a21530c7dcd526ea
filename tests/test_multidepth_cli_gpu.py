"""End-to-end `goleft multidepth` and `goleft samplename` (bin/goleft) on BAMs written here, against the oracle's bytes."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bamutil import make_bam, make_bam_indexed  # noqa: E402
from oracle import loader as orc  # noqa: E402
from oracle import multidepth as omd  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
REFS = [("chr1", 30000), ("chr7", 12000)]


def run(*args, env=None):
    return subprocess.run([GOLEFT, *args], capture_output=True, env=dict(os.environ, **env) if env else None)


def _sample_bam(path, sm, cov, seed, indexed=True):
    """reads of 100M on both references; MAPQ 5 and duplicate reads (filtered by -Q 10 / flag 0x704) mixed in.
    Returns the per-base depth of chr1 that `samtools depth -Q 10` would give."""
    rng = np.random.default_rng(seed)
    recs, keep = [], []
    for tid, (_, L) in enumerate(REFS):
        n = int(cov * L / 100)
        for p in np.sort(rng.integers(0, L - 100, n)):
            mapq = int(rng.choice([60, 60, 60, 5]))
            flag = int(rng.choice([0, 16, 0, 0x400]))
            recs.append((tid, int(p), mapq, flag, [(100, "M")]))
            if tid == 0 and mapq >= 10 and not flag & 0x704:
                keep.append(int(p))
    if indexed:
        bam, bai = make_bam_indexed(REFS, recs, sample=sm)
        open(path + ".bai", "wb").write(bai)
    else:
        bam = make_bam(REFS, recs, sample=sm)
    open(path, "wb").write(bam)
    s = np.asarray(keep, np.int32)
    return orc.pileup_diff(s, s + 100, 0, REFS[0][1])


@pytest.fixture(scope="module")
def cohort(tmp_path_factory):
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    d = tmp_path_factory.mktemp("md")
    covs = [30, 3, 28, 0, 35, 32, 30]                 # about half the reads are filtered: 15-18x pass -Q 10 / 0x704
    paths, depths = [], []
    for i, c in enumerate(covs):
        p = str(d / f"s{i}.bam")
        depths.append(_sample_bam(p, f"SM{i}", c, 50 + i))
        paths.append(p)
    return d, paths, np.stack(depths)


def _expect(depths, names, **kw):
    rows, _ = omd.text("chr1", depths, **kw)
    return ("#chrom\tstart\tend\t" + "\t".join(names) + "\n").encode() + rows


@pytest.mark.parametrize("feed", ["1", "0"])
def test_matches_oracle(cohort, feed):
    _, paths, depths = cohort
    names = [f"SM{i}" for i in range(len(paths))]
    for args, kw in (([], {}), (["-w", "15", "-m", "3", "-k", "4", "--mincov", "5", "--minsamples", "0.3"],
                                dict(window=15, min_size=3, max_skip=4, mincov=5, min_samples=0.3))):
        p = run("multidepth", "-c", "chr1", *args, *paths, env={"GL_GPU_FEED": feed})
        assert p.returncode == 0, p.stderr
        assert p.stdout == _expect(depths, names, **kw)
        assert p.stdout.count(b"\n") > 1


def test_unindexed_bam(cohort, tmp_path):
    _, paths, depths = cohort
    p0 = str(tmp_path / "plain.bam")
    d0 = _sample_bam(p0, "SM0", 30, 50, indexed=False)
    assert np.array_equal(d0, depths[0])
    p = run("multidepth", "-c", "chr1", "-w", "1000", p0, *paths[1:])
    assert p.returncode == 0, p.stderr
    assert p.stdout == _expect(depths, [f"SM{i}" for i in range(len(paths))], window=1000)


def test_errors(cohort, tmp_path):
    _, paths, _ = cohort
    p = run("multidepth", *paths)
    assert p.returncode == 255 and b"chrom is required" in p.stderr
    p = run("multidepth", "-c", "chrX", *paths)
    assert p.returncode != 0 and b"chrX not found" in p.stderr
    other = str(tmp_path / "other.bam")
    bam, bai = make_bam_indexed([("chr2", 1000)], [(0, 10, 60, 0, [(100, "M")])], sample="Z")
    open(other, "wb").write(bam)
    open(other + ".bai", "wb").write(bai)
    p = run("multidepth", "-c", "chr1", paths[0], other)                 # the contig is missing from the second BAM
    assert p.returncode != 0 and b"not found in" in p.stderr
    multi = str(tmp_path / "multi.bam")
    bam, bai = make_bam_indexed(REFS, [(0, 10, 60, 0, [(100, "M")])], sample="A\n@RG\tID:b\tSM:B")
    open(multi, "wb").write(bam)
    open(multi + ".bai", "wb").write(bai)
    p = run("multidepth", "-c", "chr1", paths[0], multi)                 # two SM values (indexcov.go:231-233)
    assert p.returncode != 0 and b"more than one RG" in p.stderr


def test_samplename(tmp_path):
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")

    def bam(name, sample):
        p = str(tmp_path / name)
        open(p, "wb").write(make_bam(REFS, [(0, 10, 60, 0, [(100, "M")])], sample=sample))
        return p

    one = bam("one.bam", "NA12878")
    several = bam("several.bam", "B\n@RG\tID:b\tSM:A\n@RG\tID:c\tSM:B\n@RG\tID:d\tSM:")
    empty = bam("empty.bam", "")
    p = run("samplename", one)
    assert p.returncode == 0 and p.stdout == b"NA12878\n"
    p = run("samplename", several)
    assert p.returncode == 0 and p.stdout == b"B\nA\n"
    p = run("samplename", empty)
    assert p.returncode == 0 and p.stdout == b"\n"
    assert run("samplename", "-e", one).stdout == b"NA12878\n"
    for b in (several, empty):
        p = run("samplename", "-e", b)
        assert p.returncode != 0 and b"found multiple samples" in p.stderr
