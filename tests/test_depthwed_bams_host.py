"""`goleft depthwed` with BAM inputs, the parts that need no GPU: argument errors and exit codes, the header names (a run
whose .fai gives no windows prints the header alone), and gl_depthwed_plan against a restatement of depthwed.go:117-157."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bamutil import make_bam_indexed  # noqa: E402

GOLEFT = os.path.join(ROOT, "bin", "goleft")


def plan_ref(starts, ends, chrom, size):
    """depthwed.go:117-157: a group takes rows while its span is below size and the next row is on the same chrom"""
    first, o_s, o_e, o_c = [], [], [], []
    r, R = 0, len(starts)
    while r < R:
        first.append(r)
        st, en, c = int(starts[r]), int(ends[r]), int(chrom[r])
        r += 1
        while r < R and en - st < size and int(chrom[r]) == c:
            en = int(ends[r])
            r += 1
        o_s.append(st); o_e.append(en); o_c.append(c)
    first.append(R)
    return first, o_s, o_e, o_c


def fai_rows(lens, W):
    s, e, c = [], [], []
    for k, L in enumerate(lens):
        n = (L + W - 1) // W
        s += [i * W for i in range(n)]
        e += [min((i + 1) * W, L) for i in range(n)]
        c += [k] * n
    return np.array(s, np.int64), np.array(e, np.int64), np.array(c, np.int32)


@pytest.mark.parametrize("W", [1, 13, 100, 250, 2001, 10**9])
def test_plan_fai_rows(W):
    from goleft_b200 import capi
    lens = [1, 12, 999, 1000, 4321, 25000, 3 * 2**30 + 7] if W >= 2001 else [1, 12, 999, 1000, 4321, 25000]
    starts, ends, chrom = fai_rows(lens, W)
    for size in sorted({1, W - 1 if W > 1 else 1, W, W + 1, 3 * W + 7, 10 * W, 10**6, 2**62}):
        got = capi.depthwed_plan(starts, ends, chrom, size)
        exp = plan_ref(starts, ends, chrom, size)
        for g, x in zip(got, exp):
            assert g.tolist() == x, (W, size)


def test_plan_irregular_rows():
    """rows of any width, repeated chrom ids and runs that come back to an earlier chrom"""
    from goleft_b200 import capi
    rng = np.random.default_rng(5)
    R = 5000
    chrom = np.repeat(rng.integers(0, 4, 60), rng.integers(1, 160, 60))[:R].astype(np.int32)
    w = rng.integers(0, 700, chrom.size)
    starts = np.cumsum(rng.integers(0, 50, chrom.size)).astype(np.int64)
    ends = starts + w
    for size in (1, 100, 555, 3000, 10**9):
        got = capi.depthwed_plan(starts, ends, chrom, size)
        exp = plan_ref(starts, ends, chrom, size)
        for g, x in zip(got, exp):
            assert g.tolist() == x, size


def test_plan_errors():
    from goleft_b200 import capi
    with pytest.raises(capi.GlError):
        capi.depthwed_plan([0], [10], [0], 0)
    assert [a.tolist() for a in capi.depthwed_plan([], [], [], 10)] == [[0], [], [], []]


@pytest.fixture(scope="module")
def files(tmp_path_factory):
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    d = tmp_path_factory.mktemp("wedh")
    bam, bai = make_bam_indexed([("chr1", 1000)], [(0, 10, 60, 0, [(100, "M")])], sample="Z")
    for nm in ("s1.bam", "x.depth.bam", "a.b.gz.bam"):
        open(d / nm, "wb").write(bam)
        open(d / (nm + ".bai"), "wb").write(bai)
    open(d / "ref.fa", "w").write(">chr1\n" + "A" * 1000 + "\n")
    open(d / "ref.fa.fai", "w").write("chr1\t1000\t6\t1000\t1001\n")
    open(d / "empty.fa.fai", "w").write("")
    open(d / "a.depth.bed", "w").write("chr1\t0\t10\t1.5\n")
    return d


def run(d, *args):
    return subprocess.run([GOLEFT, "depthwed", *args], capture_output=True, cwd=str(d))


@pytest.mark.parametrize("args, msg", [
    (["-s", "100", "-r", "ref.fa", "s1.bam", "a.depth.bed"], b"all BAMs or all depth.bed"),
    (["-s", "100", "a.depth.bed", "s1.bam"], b"all BAMs or all depth.bed"),
    (["-s", "100", "s1.bam"], b"--reference is required"),
    (["-s", "100", "-r", "ref.fa", "-b", "t.bed", "s1.bam"], b"--bed is not supported"),
    (["-s", "100", "-b", "t.bed", "a.depth.bed"], b"--bed is not supported"),
    (["-s", "100", "-w", "10", "a.depth.bed"], b"--windowsize needs BAM inputs"),
    (["-s", "100", "-Q", "0", "a.depth.bed"], b"--q needs BAM inputs"),
    (["-s", "100", "-r", "ref.fa", "a.depth.bed"], b"--reference needs BAM inputs"),
    (["-s", "100", "-c", "chr1", "a.depth.bed"], b"--chrom needs BAM inputs"),
    (["-s", "100", "-p", "2", "a.depth.bed"], b"--processes needs BAM inputs"),
    (["-s", "100", "--gpus", "2", "a.depth.bed"], b"--gpus needs BAM inputs"),
    (["-s", "100", "--timing", "a.depth.bed"], b"--timing needs BAM inputs"),
    (["-s", "100", "-r", "ref.fa", "-w", "0", "s1.bam"], b"windowsize must be > 0"),
    (["-r", "ref.fa", "s1.bam"], b"size is required"),
])
def test_argument_errors(files, args, msg):
    p = run(files, *args)
    assert p.returncode == 255, p.stderr
    assert msg in p.stderr and not p.stdout


def test_header_names(files):
    """the names getNameFromFile gives <base>[.chrom].depth.bed: the BAM's base name without .bam, and .chrom under -c"""
    p = run(files, "-s", "100", "-r", "empty.fa", "s1.bam", str(files / "x.depth.bam"), "a.b.gz.bam")
    assert (p.returncode, p.stdout, p.stderr) == (0, b"#chrom\tstart\tend\ts1\tx.depth\ta.b.gz\n", b"")
    p = run(files, "-s", "100", "-r", "ref.fa", "-c", "chrX", "s1.bam", "x.depth.bam", "a.b.gz.bam")
    assert (p.returncode, p.stdout, p.stderr) == (0, b"#chrom\tstart\tend\ts1.chrX\tx.depth.chrX\ta.b.gz.chrX\n", b"")


def test_missing_bam(files):
    p = run(files, "-s", "100", "-r", "empty.fa", "s1.bam", "missing.bam")
    assert p.returncode == 1 and b"missing.bam" in p.stderr and not p.stdout
