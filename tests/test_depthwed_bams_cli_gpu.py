"""`goleft depthwed -s SIZE -r ref.fa *.bam` end to end (bin/goleft): stdout is byte-identical to `goleft depth --prefix <base>`
on every BAM followed by `goleft depthwed` on the depth.bed files, and to a pure oracle (bamref pile-up -> walk_chunk ->
parse -> depthwed).  Every --gpus split (GL_OVERSUBSCRIBE=1 keeps N workers on fewer devices) and both feeders print the
same bytes and the same stderr."""
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bamref  # noqa: E402
from bamutil import make_bam, make_bam_indexed  # noqa: E402
from oracle import loader as orc  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
BAM_REFS = [("chr1", 30011), ("chr2", 12000), ("chrM", 517)]
FAI = [("chr1", 30011), ("chrU", 7003), ("chr2", 12000), ("chrM", 517)]      # chrU: in the .fai, in no BAM
SAMPLES = [("s0", 20, 0, True), ("s1.x", 3, 1, True), ("empty", 0, 2, True), ("plain", 15, 3, False), ("deep", 0, 4, True)]


def run(*args, cwd, **env):
    return subprocess.run([GOLEFT, *args], capture_output=True, cwd=cwd, env=dict(os.environ, GL_OVERSUBSCRIBE="1", **env))


def _records(cov, seed, deep):
    rng = np.random.default_rng(seed)
    recs = []
    for tid, (_, L) in enumerate(BAM_REFS):
        n = int(cov * L / 100)
        pos = list(np.sort(rng.integers(0, L - 100, n)))
        if deep and tid == 1:                                  # a pile-up whose window means pass 10^4
            pos = sorted(pos + [1000 + int(x) for x in rng.integers(0, 40, 30000)])
        for p in pos:
            mapq = int(rng.choice([60, 60, 25, 10, 0])) if not deep else 60
            flag = int(rng.choice([0, 16, 0, 0x400])) if not deep else 0
            recs.append((tid, int(p), mapq, flag, [(100, "M")]))
    if cov == 0 and not deep:                                  # reads, none of which pass the filters
        recs = [(0, 100 * i, 60, 0x400, [(100, "M")]) for i in range(50)]
    return recs


@pytest.fixture(scope="module")
def cohort(tmp_path_factory):
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    d = str(tmp_path_factory.mktemp("wedb"))
    paths, recs = [], []
    for name, cov, seed, indexed in SAMPLES:
        r = _records(cov, 90 + seed, name == "deep")
        p = os.path.join(d, name + ".bam")
        if indexed:
            bam, bai = make_bam_indexed(BAM_REFS, r, sample=name)
            open(p + ".bai", "wb").write(bai)
        else:
            bam = make_bam(BAM_REFS, r, sample=name)
        open(p, "wb").write(bam)
        paths.append(p)
        recs.append(r)
    with open(os.path.join(d, "ref.fa"), "w") as f:
        for n, L in FAI:
            f.write(">%s\n%s\n" % (n, "A" * L))
    with open(os.path.join(d, "ref.fa.fai"), "w") as f:
        off = 0
        for n, L in FAI:
            off += len(n) + 2
            f.write("%s\t%d\t%d\t%d\t%d\n" % (n, L, off, L, L + 1))
            off += L + 1
    return d, paths, recs


def two_step(d, paths, W, Q, size, chrom=None):
    """goleft depth once per BAM into its own directory, then goleft depthwed on the depth.bed files"""
    wd = os.path.join(d, "two_%d_%d_%s" % (W, Q, chrom))
    sfx = "." + chrom if chrom else ""
    beds = []
    if not os.path.isdir(wd):
        os.makedirs(wd)
        for p in paths:
            base = os.path.basename(p)[:-4]
            a = ["depth", "--prefix", base, "-w", str(W), "-Q", str(Q), "-r", os.path.join(d, "ref.fa"), p] + (["-c", chrom] if chrom else [])
            r = run(*a, cwd=wd)
            assert r.returncode == 0, r.stderr
    for p in paths:
        beds.append(os.path.basename(p)[:-4] + sfx + ".depth.bed")
    r = run("depthwed", "-s", str(size), *beds, cwd=wd)
    assert r.returncode == 0, r.stderr
    return r.stdout


_SEGS = {}


def oracle(paths, recs, W, Q, size, chrom=None):
    """bamref pile-up -> walk_chunk -> parse -> the oracle's depthwed"""
    step = max(1, 10_000_000 // W) * W
    names = [os.path.basename(p)[:-4] + ("." + chrom if chrom else "") for p in paths]
    fai = [(n, L) for n, L in FAI if chrom is None or n == chrom]
    means, starts, ends, cid = [], None, None, None
    for r in recs:
        key = (id(r), Q)
        if key not in _SEGS:
            _SEGS[key] = bamref.segments(r, len(BAM_REFS), Q)
        segs = _SEGS[key]
        rows = []
        for ci, (n, L) in enumerate(fai):
            tid = [b for b, _ in BAM_REFS].index(n) if n in [b for b, _ in BAM_REFS] else None
            depth = bamref.pileup(*segs[tid], 0, L) if tid is not None else np.zeros(L, np.int32)
            for cs in range(0, L, step):
                ce = min(L, cs + step)
                hd, _ = orc.walk_chunk(n, cs, ce, W, 4, 0, depth[cs:ce])
                rows += [(ci,) + tuple(ln.split(b"\t")[1:]) for ln in hd.splitlines()]
        means.append([float(x[3]) for x in rows])
        if starts is None:
            starts = np.array([int(x[1]) for x in rows], np.int32)
            ends = np.array([int(x[2]) for x in rows], np.int32)
            cid = np.array([x[0] for x in rows], np.int32)
    o_s, o_e, o_c, out = orc.depthwed(np.array(means), starts, ends, cid, size)
    text = "#chrom\tstart\tend\t" + "\t".join(names) + "\n"
    for g in range(o_s.size):
        text += "%s\t%d\t%d\t%s\n" % (fai[o_c[g]][0], o_s[g], o_e[g], "\t".join(str(v) for v in out[g]))
    return text.encode()


def sizes(W):
    return sorted({max(1, W // 3), W, W * 5 // 2 + 1, 10**6})


@pytest.mark.parametrize("W", [13, 100, 250, 2001, 10**9])
def test_matches_two_step_and_oracle(cohort, W):
    d, paths, recs = cohort
    for size in sizes(W):
        p = run("depthwed", "-s", str(size), "-w", str(W), "-r", "ref.fa", *paths, cwd=d)
        assert p.returncode == 0, p.stderr
        assert p.stdout == two_step(d, paths, W, 1, size), size
        assert p.stdout == oracle(paths, recs, W, 1, size), size
        assert p.stderr.count(b"no usable index") == 1


@pytest.mark.parametrize("Q", [0, 20])
def test_mapq(cohort, Q):
    d, paths, recs = cohort
    p = run("depthwed", "-s", "500", "-Q", str(Q), "-r", "ref.fa", *paths, cwd=d)
    assert p.returncode == 0, p.stderr
    assert p.stdout == two_step(d, paths, 250, Q, 500)
    assert p.stdout == oracle(paths, recs, 250, Q, 500)


@pytest.mark.parametrize("chrom", ["chr2", "chrU"])
def test_chrom(cohort, chrom):
    d, paths, recs = cohort
    p = run("depthwed", "-s", "1000", "-w", "100", "-c", chrom, "-r", "ref.fa", *paths, cwd=d)
    assert p.returncode == 0, p.stderr
    assert p.stdout.split(b"\n")[0].endswith(b"\tdeep." + chrom.encode())
    assert p.stdout == two_step(d, paths, 100, 1, 1000, chrom)
    assert p.stdout == oracle(paths, recs, 100, 1, 1000, chrom)


def test_deep_pileup(cohort):
    """window means of 10^4 and more (printed as 1.234e+04 by goleft depth) give the same cells"""
    d, paths, recs = cohort
    p = run("depthwed", "-s", "13", "-w", "13", "-c", "chr2", "-r", "ref.fa", paths[-1], cwd=d)
    assert p.returncode == 0, p.stderr
    cells = [int(ln.split(b"\t")[3]) for ln in p.stdout.splitlines()[1:]]
    assert max(cells) >= 10**4
    assert p.stdout == two_step(d, [paths[-1]], 13, 1, 13, "chr2") == oracle([paths[-1]], [recs[-1]], 13, 1, 13, "chr2")


@pytest.mark.parametrize("feed", ["1", "0"])
def test_every_split_prints_the_same(cohort, feed):
    d, paths, recs = cohort
    args = ["depthwed", "-s", "700", "-w", "100", "-r", "ref.fa", *paths, *paths[:2]]
    one = run(*args, "--gpus", "1", cwd=d, GL_GPU_FEED=feed)
    assert one.returncode == 0, one.stderr
    assert one.stdout == oracle(paths + paths[:2], recs + recs[:2], 100, 1, 700)
    for g in ("2", "3", "7", "0"):
        p = run(*args, "--gpus", g, cwd=d, GL_GPU_FEED=feed)
        assert (p.returncode, p.stdout, p.stderr) == (0, one.stdout, one.stderr), g


def test_timing_and_errors(cohort, tmp_path):
    d, paths, _ = cohort
    p = run("depthwed", "-s", "500", "-r", "ref.fa", "--timing", *paths, cwd=d)
    assert p.returncode == 0 and b'"goleft_depthwed_timing"' in p.stderr
    shutil.copy(paths[0], tmp_path / "bad.bam")
    open(tmp_path / "bad.bam", "r+b").truncate(200)
    for g in ("1", "3"):
        q = run("depthwed", "-s", "500", "-r", os.path.join(d, "ref.fa"), "--gpus", g, *paths[:2], str(tmp_path / "bad.bam"), *paths[2:],
                cwd=d)
        assert q.returncode != 0 and not q.stdout, g
