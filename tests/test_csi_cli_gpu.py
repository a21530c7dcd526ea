"""The goleft CLI on CSI-indexed inputs.  `depth` (.fai mode, -c, --bed, --stats, --gpus), `multidepth`, `covstats`,
`indexcov` and `indexsplit` give the bytes they give with BAIs of the same BAMs; `goleft depth` decodes every pass of a
2^31 - 1 base contig on the GPU once it has a CSI, with the oracle's bytes; indexcov refuses a CSI whose tiles are wider
than 16 KB.  Needs an H100 (`-m gpu`)."""
import gzip
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bamref  # noqa: E402
import csi_bams as cb  # noqa: E402
from bamutil import make_bai  # noqa: E402
from region_bams import read_bai  # noqa: E402
from fautil import make_fasta  # noqa: E402
from goleft_b200 import capi  # noqa: E402
from oracle import loader as orc  # noqa: E402

GOLEFT = os.path.join(ROOT, "bin", "goleft")
REFS = [("chr1", 3_000_000), ("chr2", 1_200_000), ("chrM", 16_569)]


def run(*args, cwd=None, env=None, check=True):
    p = subprocess.run([GOLEFT, *args], capture_output=True, cwd=cwd, env=dict(os.environ, **env) if env else None)
    if check:
        assert p.returncode == 0, p.stderr.decode()
    return p


def sample_records(rng, refs, cov=2.0):
    """(records, mates) of one sample: 100 bp reads of mixed CIGARs, flags and MAPQs, mates for covstats' insert sizes,
    and a few unplaced reads"""
    recs, mates = [], []
    cig = [[(100, "M")], [(100, "M")], [(45, "M"), (7, "D"), (55, "M")], [(30, "M"), (2, "I"), (68, "M")], [(12, "S"), (88, "M")],
           [(50, "M"), (400, "N"), (50, "M")]]
    for tid, (name, L) in enumerate(refs):
        for p0 in np.sort(rng.integers(0, L - 600, int(L * cov / 100))).tolist():
            flag = int(rng.choice([99, 147, 0, 16, 0x400 | 99, 0x100, 0x200, 99, 147]))
            recs.append((tid, p0, int(rng.choice([0, 1, 20, 60, 60])), flag, cig[int(rng.integers(0, len(cig)))]))
            ins = int(rng.normal(350, 40))
            mates.append((p0 + ins - 100, ins) if flag & 1 and not flag & 16 else (max(0, p0 - 250), -ins))
    for _ in range(20):
        recs.append((-1, -1, 0, 4, [(100, "M")])); mates.append((-1, 0))
    return recs, mates


@pytest.fixture(scope="module")
def cohort(tmp_path_factory):
    """three samples, each BAM written twice: bai/sK.bam with its BAI, csi/sK.bam with a depth-6 CSI; a FASTA for --stats"""
    d = tmp_path_factory.mktemp("csicli")
    for sub in ("bai", "csi"):
        (d / sub).mkdir()
    fa, fai, _ = make_fasta(REFS, seed=3)
    rng = np.random.default_rng(11)
    all_recs = []
    for k in range(3):
        recs, mates = sample_records(rng, REFS)
        bam, csi, bai = cb.make_bam_csi(REFS, recs, 14, 6, sample="s%d" % k, mates=mates)
        for sub, name, idx in (("bai", "s%d.bam.bai" % k, bai), ("csi", "s%d.bam.csi" % k, csi)):
            (d / sub / ("s%d.bam" % k)).write_bytes(bam)
            (d / sub / name).write_bytes(idx)
        all_recs.append(recs)
    for sub in ("bai", "csi"):
        (d / sub / "g.fa").write_bytes(fa)
        (d / sub / "g.fa.fai").write_text(fai)
        (d / sub / "lines.bed").write_text("chr1\t1000\t250000\nchr1\t900000\t905000\nchr2\t5\t1199000\nchrM\t0\t16569\nchr1\t2999000\t3000000\n")
    return d, all_recs


def _files(dirpath, prefix):
    return {n: open(os.path.join(dirpath, n), "rb").read() for n in sorted(os.listdir(dirpath)) if n.startswith(prefix)}


@pytest.mark.parametrize("args", [["-w", "250"], ["-w", "1000", "-c", "chr2"], ["-w", "100", "--bed", "lines.bed"],
                                  ["-w", "500", "--stats"], ["-w", "250", "--gpus", "2"], ["-w", "250", "-Q", "20"]],
                         ids=["fai", "chrom", "bed", "stats", "gpus2", "q20"])
def test_depth_csi_equals_bai(cohort, args):
    d, _ = cohort
    out = {}
    prefix = "o" + "".join(args).replace("-", "_").replace(".", "_")             # one set of files per parameter set
    for sub in ("bai", "csi"):
        p = run("depth", *args, "--prefix", prefix, "--reference", "g.fa", "--timing", "s0.bam", cwd=str(d / sub), env={"GL_OVERSUBSCRIBE": "1"})
        assert b"decoding the whole file" not in p.stderr
        out[sub] = _files(str(d / sub), prefix + ".")
    assert out["bai"] == out["csi"] and len(out["csi"]) == 2 and all(len(v) > 0 for v in out["csi"].values())


@pytest.mark.parametrize("feed", ["1", "0"])
def test_multidepth_csi_equals_bai(cohort, feed):
    d, _ = cohort
    got = {}
    for sub in ("bai", "csi"):
        got[sub] = [run("multidepth", *a, "s0.bam", "s1.bam", "s2.bam", cwd=str(d / sub), env={"GL_GPU_FEED": feed}).stdout
                    for a in (["-c", "chr1"], ["-c", "chr2", "--gpus", "2"])]
    assert got["bai"] == got["csi"] and all(len(x) > 0 for x in got["csi"])


def test_covstats_csi_equals_bai(cohort):
    d, _ = cohort
    got = {sub: run("covstats", "-n", "5000", "s0.bam", "s1.bam", "s2.bam", cwd=str(d / sub)).stdout for sub in ("bai", "csi")}
    assert got["bai"] == got["csi"] and got["csi"].count(b"\n") == 4


def test_covstats_without_any_index_keeps_its_error(cohort, tmp_path):
    d, _ = cohort
    shutil.copy(str(d / "csi" / "s0.bam"), str(tmp_path / "u.bam"))
    ref = run("covstats", "-n", "5000", "u.bam", cwd=str(tmp_path), check=False)
    assert ref.returncode != 0
    shutil.copy(str(d / "csi" / "s0.bam.csi"), str(tmp_path / "u.csi"))
    assert run("covstats", "-n", "5000", "u.bam", cwd=str(tmp_path)).stdout.count(b"\n") == 2


# ---- the contig of 2^31 - 1 bases (tests/test_depth_int32_top_gpu.py's CLI fixture), now with a CSI of depth 6
TOP = 2 ** 31 - 1


def _big_contig(tmp_path):
    L, W = TOP, 100_000
    rng = np.random.default_rng(31)
    edges = [0, 1_070_000_000, 2_140_000_000]
    pos = [rng.integers(max(0, x - 3000), x + 3000, 400) for x in edges]
    pos.append(rng.integers(L - 300, L - 150, 60))
    pos = np.sort(np.concatenate(pos))
    cigars = [[(150, "M")], [(45, "M"), (7, "D"), (55, "M")], [(12, "S"), (88, "M")], [(60, "M"), (300, "N"), (40, "M")]]
    recs = []
    for p0 in pos.tolist():
        cig = cigars[int(rng.integers(0, len(cigars)))]
        if p0 + 400 > L:
            cig = [(int(min(150, L - p0)), "M")]
        recs.append((0, p0, 60, int(rng.choice([0, 16])), cig))
    recs.append((0, L - 100, 60, 0, [(100, "M")]))
    recs.sort(key=lambda r: r[1])
    refs = [("chrBig", L)]
    bam, csi, _ = cb.make_bam_csi(refs, recs, 14, 6, with_bai=False)
    (tmp_path / "big.bam").write_bytes(bam)
    (tmp_path / "big.bam.csi").write_bytes(csi)
    (tmp_path / "ref.fa.fai").write_text("chrBig\t%d\t8\t60\t61\n" % L)
    s, e = bamref.segments(recs, 1, 1)[0]
    exp_hd, exp_ca = [], []
    for cs, ce in orc.gen_chunks(L, W):
        h, c = orc.walk_chunk("chrBig", cs, ce, W, 4, 0, orc.pileup_diff(s, e, cs, ce))
        exp_hd.append(h); exp_ca.append(c)
    return W, b"".join(exp_hd), b"".join(exp_ca)


def test_cli_depth_contig_of_int32_max_bases_with_csi(tmp_path):
    """three passes ([0, 1.07e9), [1.07e9, 2.14e9), [2.14e9, 2^31-1)), each decoded on the GPU from the CSI's bin query;
    == the oracle's walker chunk by chunk, == GL_GPU_FEED=0, == --gpus 2"""
    W, exp_hd, exp_ca = _big_contig(tmp_path)
    got = []
    for name, extra, env in (("gpu", ["--timing"], None), ("host", [], {"GL_GPU_FEED": "0"}),
                             ("gpus2", ["--gpus", "2"], {"GL_OVERSUBSCRIBE": "1"})):
        prefix = str(tmp_path / name)
        p = run("depth", "-w", str(W), *extra, "--prefix", prefix, "--reference", str(tmp_path / "ref.fa"), str(tmp_path / "big.bam"), env=env)
        assert b"decoding the whole file" not in p.stderr
        if name == "gpu":
            t = json.loads(p.stderr.decode().strip().splitlines()[-1])["goleft_depth_timing"]
            assert t["gpu_fed_passes"] == 3, t
        got.append((open(prefix + ".depth.bed", "rb").read(), open(prefix + ".callable.bed", "rb").read()))
    assert got[0][0].count(b"\n") == (TOP - 1) // W + 1
    assert got[0] == (exp_hd, exp_ca)
    assert got[1] == got[0] and got[2] == got[0]


# ---- indexcov / indexsplit
def tiled_records(rng, refs, n_per_tile, ms):
    """reads that never cross a 16 KB tile edge, one inside the first 2^ms bases of every tile and up to n_per_tile[tid] - 1
    more, so the CSI's rebuilt linear index equals the BAI's"""
    recs = []
    for tid, (name, L) in enumerate(refs):
        for t in range((L - 200) // 16384):
            base = t * 16384
            extra = int(rng.integers(0, n_per_tile[tid])) if n_per_tile[tid] > 0 else 0
            offs = [int(rng.integers(0, (1 << ms) - 100))] + rng.integers(0, 16384 - 100, extra).tolist()
            for o in sorted(offs):
                recs.append((tid, base + o, 60, int(rng.choice([0, 16, 4])), [(100, "M")]))
    recs.append((-1, -1, 0, 4, [(100, "M")]))
    return recs


IC_REFS = [("1", 2_000_000), ("2", 1_500_000), ("X", 1_000_000), ("Y", 300_000)]


def _indexcov_outputs(outdir):
    return (gzip.decompress(open(os.path.join(outdir, "tt-indexcov.bed.gz"), "rb").read()),
            open(os.path.join(outdir, "tt-indexcov.roc"), "rb").read(), open(os.path.join(outdir, "tt-indexcov.ped"), "rb").read())


@pytest.mark.parametrize("ms,depth", [(14, 6), (12, 6), (14, 5)])
def test_indexcov_and_indexsplit_on_csi(tmp_path, ms, depth):
    """.csi inputs (with --fai) and CSI-only .bam inputs give the BAI cohort's indexcov outputs and indexsplit text"""
    rng = np.random.default_rng(ms * 10 + depth)
    (tmp_path / "g.fa.fai").write_text("".join("%s\t%d\t6\t60\t61\n" % r for r in IC_REFS))
    for sub in ("bai", "csi"):
        (tmp_path / sub).mkdir()
    for k in range(6):
        n = 6 + 4 * (k % 3)
        recs = tiled_records(rng, IC_REFS, [n, n, n // 2 if k % 2 else n, n // 2 if k % 2 else 0], ms)    # odd k: male
        bam, csi, bai = cb.make_bam_csi(IC_REFS, recs, ms, depth, sample="smp%d" % k)
        for sub, idx in (("bai", bai), ("csi", csi)):
            (tmp_path / sub / ("smp%d.bam" % k)).write_bytes(bam)
            (tmp_path / sub / ("smp%d.bam.%s" % (k, sub))).write_bytes(idx)
        lin_c = capi.bai_read(str(tmp_path / "csi" / ("smp%d.bam.csi" % k)))["ioffsets"]
        lin_b = capi.bai_read(str(tmp_path / "bai" / ("smp%d.bam.bai" % k)))["ioffsets"]
        assert [x.tolist() for x in lin_c] == [x.tolist() for x in lin_b]             # the fixture makes them agree
    fai = str(tmp_path / "g.fa.fai")
    res = {}
    for sub in ("bai", "csi"):
        idx = [str(tmp_path / sub / ("smp%d.bam.%s" % (k, sub))) for k in range(6)]
        bams = [str(tmp_path / sub / ("smp%d.bam" % k)) for k in range(6)]
        o1, o2 = tmp_path / sub / "a" / "tt", tmp_path / sub / "b" / "tt"
        o1.parent.mkdir(); o2.parent.mkdir()                                      # indexcov makes only the last level
        run("indexcov", "-d", str(o1), "--fai", fai, *idx)
        run("indexcov", "-d", str(o2), *bams)
        split = [run("indexsplit", "-n", "7", "--fai", fai, *x).stdout for x in (idx, bams)]
        res[sub] = (_indexcov_outputs(str(o1)), _indexcov_outputs(str(o2)), split)
    assert res["bai"] == res["csi"]
    assert b"smp0-bam" in res["csi"][0][2] and b"smp0\t" in res["csi"][1][2]
    assert len(res["csi"][0][0].splitlines()) > 200 and res["csi"][2][0].count(b"\n") >= 5


def test_indexcov_on_csi_whose_index_differs(tmp_path):
    """reads across tile edges, so the CSI's rebuilt linear index is not the BAI's: the outputs equal those of BAIs that hold
    the rebuilt index (the restatement)"""
    rng = np.random.default_rng(5)
    refs = IC_REFS[:3]
    (tmp_path / "g.fa.fai").write_text("".join("%s\t%d\t6\t60\t61\n" % r for r in refs))
    csis, bais = [], []
    for k in range(5):
        recs = []
        for tid, (name, L) in enumerate(refs):
            for p0 in np.sort(rng.integers(0, L - 3000, int(L * (0.01 + 0.004 * k) / 100))).tolist():
                recs.append((tid, p0, 60, 0, [(int(rng.integers(80, 2500)), "M")]))
        recs.append((-1, -1, 0, 4, [(100, "M")]))
        _, csi, bai = cb.make_bam_csi(refs, recs, 12, 6)
        c = tmp_path / ("s%d.bam.csi" % k)
        c.write_bytes(csi)
        parsed = cb.read_csi(csi)
        lin = [cb.rebuild_linear(R["loff"], 12, 6) for R in parsed["refs"]]
        stats = [(s[1][0], s[1][1]) if s is not None else None for _, s, _ in read_bai(bai)[0]]
        b = tmp_path / ("s%d.bam.bai" % k)
        b.write_bytes(make_bai(lin, stats))
        csis.append(str(c)); bais.append(str(b))
    (tmp_path / "c").mkdir(); (tmp_path / "b").mkdir()
    run("indexcov", "-d", str(tmp_path / "c" / "tt"), "--fai", str(tmp_path / "g.fa.fai"), *csis)
    run("indexcov", "-d", str(tmp_path / "b" / "tt"), "--fai", str(tmp_path / "g.fa.fai"), *bais)
    assert _indexcov_outputs(str(tmp_path / "c" / "tt")) == _indexcov_outputs(str(tmp_path / "b" / "tt"))


def test_indexcov_refuses_wide_tiles(tmp_path):
    """a CSI with min_shift 16: exit 1, naming the file and its min_shift; indexsplit likewise"""
    refs = IC_REFS[:2]
    rng = np.random.default_rng(2)
    recs = tiled_records(rng, refs, [4, 4], 14)
    _, csi, _ = cb.make_bam_csi(refs, recs, 16, 5, with_bai=False)
    p = tmp_path / "w.bam.csi"
    p.write_bytes(csi)
    (tmp_path / "g.fa.fai").write_text("".join("%s\t%d\t6\t60\t61\n" % r for r in refs))
    for args in (["indexcov", "-d", str(tmp_path / "o" / "tt")], ["indexsplit", "-n", "3"]):
        r = run(*args, "--fai", str(tmp_path / "g.fa.fai"), str(p), check=False)
        assert r.returncode == 1, r.stderr
        assert str(p).encode() in r.stderr and b"min_shift 16" in r.stderr
