"""End-to-end: the C++ `goleft` CLI (bin/goleft over libgoleft_b200.so) on files written here, compared with the
oracle.  Mirrors the reference's functional tests (depth/functional-test.sh, indexcov/functional-tests.sh) in
shape: exit codes, file names, exact tiling, and — beyond the reference — exact text."""
import gzip
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bamref  # noqa: E402
from bamutil import cg_mix_records, cigar_lens, make_bai, make_bam, make_bam_indexed  # noqa: E402
from goleft_b200 import capi  # noqa: E402
from indexcov_cli_oracle import check_ped_columns, cohort_bais, expected_outputs, oracle_depths, read_ped  # noqa: E402
from oracle import loader as orc  # noqa: E402

GOLEFT = os.path.join(ROOT, "bin", "goleft")


def run(*args, check=True, env=None):
    p = subprocess.run([GOLEFT, *args], capture_output=True, text=True, env=dict(os.environ, **env) if env else None)
    if check:
        assert p.returncode == 0, p.stderr
    return p


def test_dispatcher_and_arg_errors():
    """no GPU needed for these: cmd/goleft/goleft.go:55-69 and go-arg's exit code 255"""
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    assert run().returncode == 0
    p = run("nosuchprog", check=False)
    assert p.returncode == 1 and "goleft Version: 0.2.6" in p.stderr
    p = run("indexcov", "-d", "/tmp/tt", check=False)                       # functional-tests.sh:39-42
    assert p.returncode == 255 and "error: bam is required" in p.stderr
    p = run("depth", "x.bam", check=False)
    assert p.returncode == 255 and "prefix is required" in p.stderr
    p = run("depthwed", "a.bed", check=False)
    assert p.returncode == 255 and "size is required" in p.stderr


def _make_bam(tmp_path, seed=0, n=40000, indexed=True, long_reads=False):
    """long_reads: a fourth reference holds ultra-long reads stored through CG, 150 bp reads and the CG edge cases
    (bamutil.cg_mix_records)"""
    rng = np.random.default_rng(seed)
    refs = [("chrM", 16571), ("chr22", 20001), ("HLA-A*01:01:01:01", 3000)]
    recs, mates = [], []
    for tid, (name, L) in enumerate(refs):
        m = n if tid == 0 else n // 20
        pos = np.sort(rng.integers(0, max(1, L - 160), m))
        for p0 in pos:
            flag = int(rng.choice([99, 147, 0, 16, 0x400 | 99, 0x100, 0x200, 0x800]))
            mapq = int(rng.choice([0, 1, 20, 60, 60, 60]))
            kind = int(rng.integers(0, 5))
            cigar = [[(100, "M")], [(100, "M")], [(45, "M"), (7, "D"), (55, "M")], [(30, "M"), (2, "I"), (68, "M")], [(12, "S"), (88, "M")]][kind]
            recs.append((tid, int(p0), mapq, flag, cigar))
            ins = int(rng.normal(350, 40))
            mates.append((int(p0) + ins - 100, ins) if flag & 1 and not flag & 16 else (max(0, int(p0) - 250), -ins))
    if long_reads:
        long_recs, end = cg_mix_records(np.random.default_rng(seed + 100), len(refs), n_long=30, n_short=3000)
        refs.append(("chrL", end + 2000))
        recs += long_recs
        mates += [(-1, 0)] * len(long_recs)
    for _ in range(50):
        recs.append((-1, -1, 0, 4, [(100, "M")])); mates.append((-1, 0))
    bam = tmp_path / "s.bam"
    fai = tmp_path / "ref.fa.fai"
    fai.write_text("".join("%s\t%d\t6\t60\t61\n" % r for r in refs))
    if indexed:                                       # a real .bai: the CLI seeks with it (samtools depth -r needs one too)
        bam_b, bai_b = make_bam_indexed(refs, recs, sample="S1", mates=mates)
        bam.write_bytes(bam_b)
        (tmp_path / "s.bam.bai").write_bytes(bai_b)
    else:                                             # linear index absent: stats bin only -> the CLI decodes the whole file
        bam.write_bytes(make_bam(refs, recs, sample="S1", mates=mates))
        n_mapped = [sum(1 for r in recs if r[0] == t) for t in range(len(refs))]
        (tmp_path / "s.bam.bai").write_bytes(make_bai([[0] for _ in refs], [(n_mapped[t], 0) for t in range(len(refs))]))
    return str(bam), str(tmp_path / "ref.fa"), refs, recs, mates


@pytest.mark.gpu
@pytest.mark.parametrize("W", [100, 250, 13, 2001, 1000000000])
def test_depth_fai_mode(tmp_path, W):
    bam, ref, refs, recs, _ = _make_bam(tmp_path)
    prefix = str(tmp_path / "x")
    run("depth", "-Q", "1", "--ordered", "--windowsize", str(W), "--prefix", prefix, "--reference", ref, bam)
    seg = bamref.segments(recs, len(refs), 1)
    exp_hd, exp_ca = b"", b""
    for tid, (name, L) in enumerate(refs):
        s, e = seg[tid]
        d = bamref.pileup(s, e, 0, L)
        for cs, ce in orc.gen_chunks(L, W):
            h, c = orc.walk_chunk(name, cs, ce, W, 4, 0, d[cs:ce])
            exp_hd += h; exp_ca += c
    assert open(prefix + ".depth.bed", "rb").read() == exp_hd
    assert open(prefix + ".callable.bed", "rb").read() == exp_ca


@pytest.mark.gpu
def test_depth_unindexed_bam_falls_back_to_whole_file_decode(tmp_path):
    bam, ref, refs, recs, _ = _make_bam(tmp_path, seed=4, indexed=False)
    prefix = str(tmp_path / "u")
    p = run("depth", "-Q", "1", "-w", "100", "--prefix", prefix, "--reference", ref, bam)
    assert "decoding the whole file" in p.stderr
    seg = bamref.segments(recs, len(refs), 1)
    exp_hd, exp_ca = b"", b""
    for tid, (name, L) in enumerate(refs):
        s, e = seg[tid]
        h, c = orc.walk_chunk(name, 0, L, 100, 4, 0, bamref.pileup(s, e, 0, L))
        exp_hd += h; exp_ca += c
    assert open(prefix + ".depth.bed", "rb").read() == exp_hd
    assert open(prefix + ".callable.bed", "rb").read() == exp_ca


@pytest.mark.gpu
def test_depth_cg_long_reads(tmp_path):
    """ultra-long reads whose CIGAR is in the CG tag, among short reads: whole references through the GPU feeder and the
    host feeder, and BED lines that start and end inside long reads, byte-equal to the oracle's text over bamref depth"""
    import json
    bam, ref, refs, recs, _ = _make_bam(tmp_path, seed=6, long_reads=True)
    seg = bamref.segments(recs, len(refs), 1)
    depth = {name: bamref.pileup(*seg[tid], 0, L) for tid, (name, L) in enumerate(refs)}
    assert depth["chrL"].sum() > 1_000_000
    W = 250
    exp_hd, exp_ca = b"", b""
    for name, L in refs:
        for cs, ce in orc.gen_chunks(L, W):
            h, c = orc.walk_chunk(name, cs, ce, W, 4, 0, depth[name][cs:ce])
            exp_hd += h; exp_ca += c
    for env, fed in (({}, len(refs)), ({"GL_GPU_FEED": "0"}, 0)):
        prefix = str(tmp_path / ("w%d" % fed))
        p = run("depth", "--timing", "-Q", "1", "--ordered", "-w", str(W), "--prefix", prefix, "-r", ref, bam, env=env)
        assert json.loads(p.stderr.strip().splitlines()[-1])["goleft_depth_timing"]["gpu_fed_passes"] == fed
        assert open(prefix + ".depth.bed", "rb").read() == exp_hd, env
        assert open(prefix + ".callable.bed", "rb").read() == exp_ca, env
    longs = [r for r in recs if r[0] == 3 and len(r[4]) > 65535]
    regions = []
    for r in longs[::3]:
        span = cigar_lens(r[4])[1]
        regions += [("chrL", r[1] + span // 4, r[1] + span // 4 + 3333), ("chrL", r[1] + 17, r[1] + span - 17), ("chrL", max(0, r[1] - 500), r[1] + 900)]
    regions += [("chrM", 100, 1000), ("chrL", 0, refs[3][1])]
    bed = tmp_path / "cg.bed"
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in regions))
    prefix = str(tmp_path / "b")
    run("depth", "--bed", str(bed), "-Q", "1", "-w", "100", "--prefix", prefix, "-r", ref, bam)
    exp_hd, exp_ca = b"", b""
    for name, rs, re in regions:
        h, c = orc.walk_chunk(name, rs, re, 100, 4, 0, depth[name][rs:re])
        exp_hd += h; exp_ca += c
    assert open(prefix + ".depth.bed", "rb").read() == exp_hd
    assert open(prefix + ".callable.bed", "rb").read() == exp_ca
    # the same records without a linear index: the whole-file decode
    os.makedirs(str(tmp_path / "u"))
    bam_u, ref_u, _, _, _ = _make_bam(tmp_path / "u", seed=6, indexed=False, long_reads=True)
    prefix = str(tmp_path / "u" / "x")
    p = run("depth", "-Q", "1", "-w", str(W), "--prefix", prefix, "-r", ref_u, bam_u)
    assert "decoding the whole file" in p.stderr
    exp_hd, exp_ca = b"", b""
    for name, L in refs:
        h, c = orc.walk_chunk(name, 0, L, W, 4, 0, depth[name])
        exp_hd += h; exp_ca += c
    assert open(prefix + ".depth.bed", "rb").read() == exp_hd
    assert open(prefix + ".callable.bed", "rb").read() == exp_ca


@pytest.mark.gpu
def test_depth_synthetic_bam_index_seek_and_gpus(tmp_path):
    """a BGZF-realistic BAM (records straddle blocks, every flag/MAPQ class, deletions) + its BAI from the workload generator:
    the index-guided parallel feeder -> packed8 -> device BED text; -c reads only that contig's blocks; --gpus N output is
    byte-identical to --gpus 1"""
    import json
    sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
    import glsynth
    contigs = [("chr1", 23_000_000, 1), ("chr2", 4_100_000, 2), ("chrM", 16_569, 24)]
    bam = str(tmp_path / "synth.bam")
    glsynth.write_bam(bam, contigs, coverage=6.0)
    (tmp_path / "g.fa.fai").write_text("".join("%s\t%d\t6\t60\t61\n" % (c[0], c[1]) for c in contigs))
    ref = str(tmp_path / "g.fa")
    prefix = str(tmp_path / "s1")
    p = run("depth", "--gpus", "1", "--timing", "-w", "500", "--prefix", prefix, "-r", ref, bam)
    t_all = json.loads(p.stderr.strip().splitlines()[-1])["goleft_depth_timing"]
    exp_hd, exp_ca = b"", b""
    for name, L, idx in contigs:
        s, e = glsynth.segments(L, idx, coverage=6.0)
        o = np.argsort(s, kind="stable")
        s, e = s[o], e[o]
        for cs, ce in orc.gen_chunks(L, 500):
            lo = max(0, int(np.searchsorted(s, cs - 1000)) - 64)
            hi = int(np.searchsorted(s, ce))
            h, c = orc.walk_chunk(name, cs, ce, 500, 4, 0, orc.pileup_diff(s[lo:hi], e[lo:hi], cs, ce))
            exp_hd += h; exp_ca += c
    assert open(prefix + ".depth.bed", "rb").read() == exp_hd
    assert open(prefix + ".callable.bed", "rb").read() == exp_ca
    assert t_all["gpu_fed_passes"] == 3                      # every reference went through the GPU feeder (inflate + parse on the device)
    # the host feeder (zlib on the pool threads -> packed8 words) gives the same bytes
    prefix_h = str(tmp_path / "s1h")
    p = run("depth", "--gpus", "1", "--timing", "-w", "500", "--prefix", prefix_h, "-r", ref, bam, env={"GL_GPU_FEED": "0"})
    assert json.loads(p.stderr.strip().splitlines()[-1])["goleft_depth_timing"]["gpu_fed_passes"] == 0
    assert open(prefix_h + ".depth.bed", "rb").read() == exp_hd
    assert open(prefix_h + ".callable.bed", "rb").read() == exp_ca
    # -c chrM: only chrM's BGZF blocks are read (samtools depth -r gives the reference that, depth.go:116,152)
    prefix2 = str(tmp_path / "s2")
    p = run("depth", "-c", "chrM", "--timing", "-w", "500", "--prefix", prefix2, "-r", ref, bam)
    t_m = json.loads(p.stderr.strip().splitlines()[-1])["goleft_depth_timing"]
    assert t_m["bgzf_bytes_in"] < t_all["bgzf_bytes_in"] / 50 and t_m["records"] < 5000
    sM, eM = glsynth.segments(16_569, 24, coverage=6.0)
    assert open(prefix2 + ".chrM.depth.bed", "rb").read() == orc.walk_chunk("chrM", 0, 16_569, 500, 4, 0, orc.pileup_diff(sM, eM, 0, 16_569))[0]
    # every visible GPU: same bytes
    if capi.device_count() > 1:
        prefix3 = str(tmp_path / "s3")
        run("depth", "-w", "500", "--prefix", prefix3, "-r", ref, bam)
        assert open(prefix3 + ".depth.bed", "rb").read() == exp_hd
        assert open(prefix3 + ".callable.bed", "rb").read() == exp_ca
    # BED mode on the indexed BAM: region queries through the linear index
    bed = tmp_path / "r.bed"
    regions = [("chr1", 10_000_123, 10_050_456), ("chr2", 5, 900), ("chr1", 22_990_000, 23_000_000), ("chr1", 9_999_000, 10_001_000)]
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in regions))
    prefix4 = str(tmp_path / "s4")
    run("depth", "--bed", str(bed), "-w", "250", "--prefix", prefix4, "-r", ref, bam)
    segs = {c[0]: glsynth.segments(c[1], c[2], coverage=6.0) for c in contigs}
    exp_hd, exp_ca = b"", b""
    for name, rs, re in regions:
        s, e = segs[name]
        h, c = orc.walk_chunk(name, rs, re, 250, 4, 0, orc.pileup_diff(s, e, rs, re))
        exp_hd += h; exp_ca += c
    assert open(prefix4 + ".depth.bed", "rb").read() == exp_hd
    assert open(prefix4 + ".callable.bed", "rb").read() == exp_ca


@pytest.mark.gpu
def test_depth_chrom_and_flags(tmp_path):
    bam, ref, refs, recs, _ = _make_bam(tmp_path, seed=1)
    prefix = str(tmp_path / "y")
    run("depth", "-c", "chr22", "-w", "71", "--mincov", "2", "-m", "9", "--q", "20", "--prefix", prefix, "-r", ref, bam)
    s, e = bamref.segments(recs, len(refs), 20)[1]
    d = orc.pileup_brute(s, e, 0, 20001)
    exp = orc.walk_chunk("chr22", 0, 20001, 71, 2, 9, d)
    assert open(prefix + ".chr22.depth.bed", "rb").read() == exp[0]            # depth.go:378-389 file naming
    assert open(prefix + ".chr22.callable.bed", "rb").read() == exp[1]
    assert b"EXCESSIVE_COVERAGE" in exp[1]


@pytest.mark.gpu
@pytest.mark.parametrize("W", [10, 50, 1000000])
def test_depth_bed_mode(tmp_path, W):
    bam, ref, refs, recs, _ = _make_bam(tmp_path, seed=2)
    bed = tmp_path / "w.bed"
    regions = [("chr22", 14250, 15500), ("chr22", 1575, 15800), ("chrM", 100, 1000), ("chrM", 2000, 5000), ("chrM", 1, 3),
               ("chrM", 9, 13), ("chrM", 16, 17), ("chrM", 24, 29), ("chrM", 39, 43)]
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in regions) + "chrM\t50\t60")     # last line unterminated: dropped like Go's ReadBytes loop
    prefix = str(tmp_path / "z")
    run("depth", "--bed", str(bed), "-Q", "1", "--windowsize", str(W), "--prefix", prefix, "--reference", ref, bam)
    seg = bamref.segments(recs, len(refs), 1)
    tid_of = {n: i for i, (n, _) in enumerate(refs)}
    exp_hd, exp_ca = b"", b""
    for name, rs, re in regions:
        s, e = seg[tid_of[name]]
        h, c = orc.walk_chunk(name, rs, re, W, 4, 0, orc.pileup_brute(s, e, rs, re))
        exp_hd += h; exp_ca += c
    assert open(prefix + ".depth.bed", "rb").read() == exp_hd
    assert open(prefix + ".callable.bed", "rb").read() == exp_ca


@pytest.mark.gpu
@pytest.mark.parametrize("W", [7, 100, 250])
def test_depth_bed_mode_many_regions(tmp_path, W):
    """Batched BED mode (one pass per contig + gl_depth_interval_sums for the clipped edge windows) against the
    per-line walk of the oracle: random, overlapping, unsorted, window-aligned and out-of-contig regions."""
    bam, ref, refs, recs, _ = _make_bam(tmp_path, seed=3)
    rng = np.random.default_rng(W)
    regions = []
    for _ in range(300):
        name, L = refs[int(rng.integers(0, 3))]
        a = int(rng.integers(0, L))
        ln = int(rng.choice([1, 2, W - 1, W, W + 1, 3 * W, int(rng.integers(1, 2000))]))
        if rng.random() < 0.3:
            a = a // W * W                                                        # aligned start
        regions.append((name, a, max(a + 1, a + ln)))
    regions += [("chr22", 19990, 20500), ("chrUn_absent", 10, 700), ("chr22", 0, 20001), ("chrM", 3 * W, 5 * W)]
    bed = tmp_path / "many.bed"
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in regions))
    prefix = str(tmp_path / "m")
    run("depth", "--bed", str(bed), "-Q", "1", "--windowsize", str(W), "--prefix", prefix, "--reference", ref, bam)
    seg = bamref.segments(recs, len(refs), 1)
    tid_of = {n: i for i, (n, _) in enumerate(refs)}
    exp_hd, exp_ca = b"", b""
    for line in regions:
        name, rs, re = orc.chrom_start_end("%s\t%d\t%d" % line)      # HLA names: the lazy regex mis-splits them (depth.go:34-43,143)
        if re <= rs:
            continue
        if name in tid_of:
            s, e = seg[tid_of[name]]
        else:
            s = e = np.zeros(0, np.int32)
        h, c = orc.walk_chunk(name, rs, re, W, 4, 0, orc.pileup_brute(s, e, rs, re))
        exp_hd += h; exp_ca += c
    assert open(prefix + ".depth.bed", "rb").read() == exp_hd
    assert open(prefix + ".callable.bed", "rb").read() == exp_ca


def _with_stats(hd: bytes, fa: bytes, recs) -> bytes:
    """append getStats(chrom, s, e) to every window row (depth.go:299,334,355 call it with the printed s and e)"""
    out = []
    for ln in hd.decode().splitlines():
        c, s, e, _ = ln.split("\t")
        st = orc.faidx_stats(fa, recs[c], int(s), int(e)) if c in recs else np.zeros(3)
        out.append(ln.encode() + orc.stats_text(st) + b"\n")
    return b"".join(out)


@pytest.mark.gpu
@pytest.mark.parametrize("W", [100, 333])
def test_depth_stats_columns(tmp_path, W):
    """--stats: GC / CpG / masked columns in fai mode and BED mode (every functional test of the reference passes
    --stats, depth/functional-test.sh; values follow the Faidx.Stats restatement — parity unpinned)."""
    from fautil import make_fasta
    bam, ref, refs, bam_recs, _ = _make_bam(tmp_path, seed=5)
    fa, fai, recs = make_fasta(refs, seed=W, line=60)
    open(ref, "wb").write(fa)
    open(ref + ".fai", "w").write(fai)
    seg = bamref.segments(bam_recs, len(refs), 1)
    prefix = str(tmp_path / "st")
    run("depth", "--stats", "-Q", "1", "--ordered", "--windowsize", str(W), "--prefix", prefix, "--reference", ref, bam)
    exp_hd, exp_ca = b"", b""
    for tid, (name, L) in enumerate(refs):
        s, e = seg[tid]
        d = bamref.pileup(s, e, 0, L)
        for cs, ce in orc.gen_chunks(L, W):
            h, c = orc.walk_chunk(name, cs, ce, W, 4, 0, d[cs:ce])
            exp_hd += _with_stats(h, fa, recs); exp_ca += c
    assert open(prefix + ".depth.bed", "rb").read() == exp_hd
    assert open(prefix + ".callable.bed", "rb").read() == exp_ca
    assert len({ln.split(b"\t")[4] for ln in exp_hd.splitlines()}) > 10          # the columns are not constant
    # BED mode, incl. misaligned regions and a contig the FASTA index does not know (zeros, like faidx's error path)
    regions = [("chr22", 14250, 15500), ("chrM", 101, 1000), ("chr22", 1575, 15800), ("chrM", 16000, 16571), ("chrQ", 5, 700), ("chrM", 24, 29)]
    bed = tmp_path / "st.bed"
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in regions))
    prefix = str(tmp_path / "stb")
    run("depth", "-s", "--bed", str(bed), "-Q", "1", "--windowsize", str(W), "--prefix", prefix, "--reference", ref, bam)
    tid_of = {n: i for i, (n, _) in enumerate(refs)}
    exp_hd, exp_ca = b"", b""
    for name, rs, re in regions:
        s, e = seg[tid_of[name]] if name in tid_of else (np.zeros(0, np.int32),) * 2
        h, c = orc.walk_chunk(name, rs, re, W, 4, 0, orc.pileup_brute(s, e, rs, re))
        exp_hd += _with_stats(h, fa, recs); exp_ca += c
    assert open(prefix + ".depth.bed", "rb").read() == exp_hd
    assert open(prefix + ".callable.bed", "rb").read() == exp_ca


@pytest.mark.gpu
def test_depth_empty_bam(tmp_path):
    """check_empty (functional-test.sh:102-109)"""
    refs = [("chrM", 16571), ("chr22", 20001)]
    (tmp_path / "e.bam").write_bytes(make_bam(refs, []))
    (tmp_path / "r.fa.fai").write_text("".join("%s\t%d\t6\t60\t61\n" % r for r in refs))
    prefix = str(tmp_path / "e")
    run("depth", "--windowsize", "10", "--q", "1", "--mincov", "4", "--reference", str(tmp_path / "r.fa"), "--processes", "1",
        "--prefix", prefix, str(tmp_path / "e.bam"))
    ca = open(prefix + ".callable.bed").read().splitlines()
    assert ca == ["chrM\t0\t16571\tNO_COVERAGE", "chr22\t0\t20001\tNO_COVERAGE"]
    hd = [ln.split("\t") for ln in open(prefix + ".depth.bed").read().splitlines()]
    assert len(hd) == 1658 + 2001 and all(r[3] == "0" for r in hd)


@pytest.mark.gpu
@pytest.mark.parametrize("N", [10, 200])
def test_indexsplit(tmp_path, N):
    """goleft indexsplit (indexsplit/indexsplit.go): regions of about equal cohort data.  Text equals the oracle's
    restatement of Split; the regions tile every chromosome exactly once (indexsplit/functional-tests.sh:33-36)."""
    refs, fai, paths, lin = cohort_bais(tmp_path, S=9, seed=N)
    bed = tmp_path / "prob.bed"
    bed.write_text("1\t1000000\t1100000\nX\t5\t10\n2\t7\t3\n")
    p = run("indexsplit", "-n", str(N), "--fai", fai, "-p", str(bed), *paths)
    per_sample = []
    for k in range(len(paths)):
        voff = np.array([v for r in lin[k] for v in r], np.uint64)
        ptr = np.concatenate([[0], np.cumsum([len(r) for r in lin[k]])]).astype(np.int64)
        sizes, sptr = orc.ic_sizes(voff, ptr)
        per_sample.append([sizes[sptr[r]:sptr[r + 1]] for r in range(len(refs))])
    exp = orc.indexsplit(per_sample, [n for n, _ in refs], [L for _, L in refs], N, problems=[(0, 1000000, 1100000), (3, 5, 10)])
    assert p.stdout.encode() == exp
    rows = [ln.split("\t") for ln in p.stdout.splitlines()]
    if N == 10:                                     # regions of many tiles: exact tiling (with regions near one tile the
        for name, L in refs:                        # reference's own heavy-tile rows overlap at chromosome ends)
            iv = [(int(r[1]), int(r[2])) for r in rows if r[0] == name]
            assert iv[0][0] == 0 and iv[-1][1] == L
            assert all(a[1] == b[0] for a, b in zip(iv, iv[1:]))
    assert len(rows) >= min(N, 5)
    assert run("indexsplit", "--fai", fai, *paths, check=False).returncode == 255           # -n is required


@pytest.mark.gpu
@pytest.mark.parametrize("extranorm,form", [(False, "bai"), (True, "bai"), (False, "bam"), (True, "bam")],
                         ids=["False", "True", "bam-False", "bam-True"])
def test_indexcov_cohort(tmp_path, extranorm, form):
    """form "bam": header-only BAMs next to the same indexes, with `-c 2`.  RefsFromBam appends the named reference to the
    header's (indexcov.go:333-335), so "2" is reported twice: its rows and ROC block twice, its bins counted twice, and with
    -n both copies normalised from the original values (NormalizedDepth returns a fresh slice, indexcov.go:129-151)."""
    refs, fai, paths, lin = cohort_bais(tmp_path)
    out = tmp_path / "tt"
    order = list(range(len(refs)))
    names = ["smp%d-rest" % k for k in range(len(paths))]          # GetShortName for .bai (indexcov.go:238-245)
    args = ["indexcov", "-d", str(out)] + (["-n"] if extranorm else [])
    if form == "bam":
        bams = []
        for k, bai in enumerate(paths):
            b = tmp_path / ("smp%d.bam" % k)
            b.write_bytes(make_bam(refs, [], sample="smp%d" % k))
            (tmp_path / ("smp%d.bam.bai" % k)).write_bytes(open(bai, "rb").read())
            bams.append(str(b))
        paths, names = bams, ["smp%d" % k for k in range(len(bams))]              # names from SM
        args += ["-c", "2"]
        order.append(1)
    else:
        args += ["--fai", fai]
    p = run(*args, *paths)
    assert "indexcov finished" in p.stderr
    depths = oracle_depths(lin)
    rows, roc_txt, bins = expected_outputs(refs, depths, names, order, extranorm)
    assert gzip.open(str(out / "tt-indexcov.bed.gz"), "rt").read().splitlines() == rows
    assert open(str(out / "tt-indexcov.roc")).read() == roc_txt
    check_ped_columns(read_ped(out), refs, depths, bins)


@pytest.mark.gpu
@pytest.mark.parametrize("gpus,extranorm", [(2, False), (3, False), (7, False), (3, True)], ids=["2", "3", "7", "n-3"])
def test_indexcov_cohort_sample_sharded(tmp_path, gpus, extranorm):
    """SURVEY 8(e): samples shard across the GPUs through I5, the rows gather on the host.  `--gpus N` must give the bytes of
    `--gpus 1` (GL_OVERSUBSCRIBE lets a one-GPU box run N shards: shard g -> device g % n_dev), with -n too."""
    refs, fai, paths, lin = cohort_bais(tmp_path)
    outs = []
    for g in (1, gpus):
        out = tmp_path / ("g%d" % g) / "tt"
        os.makedirs(str(out.parent))
        run("indexcov", "-d", str(out), "--gpus", str(g), "--fai", fai, *(["-n"] if extranorm else []), *paths, env={"GL_OVERSUBSCRIBE": "1"})
        outs.append([open(str(out / ("tt-indexcov." + ext)), "rb").read() for ext in ("bed.gz", "roc", "ped")])
    assert gzip.decompress(outs[0][0]) == gzip.decompress(outs[1][0]) and outs[0][1] == outs[1][1] and outs[0][2] == outs[1][2]
    assert len(gzip.decompress(outs[1][0]).splitlines()) > 400


@pytest.mark.gpu
def test_depth_gpus_oversubscribed_same_bytes(tmp_path):
    """`goleft depth --gpus 3` (LPT over three workers, here on however many devices the box has) == `--gpus 1`"""
    sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
    import glsynth
    contigs = [("chr1", 3_000_000, 1), ("chr2", 2_100_000, 2), ("chr3", 1_000_000, 3), ("chr4", 500_000, 4), ("chrM", 16_569, 24)]
    bam = str(tmp_path / "synth.bam")
    glsynth.write_bam(bam, contigs, coverage=8.0)
    (tmp_path / "g.fa.fai").write_text("".join("%s\t%d\t6\t60\t61\n" % (c[0], c[1]) for c in contigs))
    got = []
    for g in (1, 3):
        prefix = str(tmp_path / ("o%d" % g))
        run("depth", "--gpus", str(g), "-w", "250", "--prefix", prefix, "-r", str(tmp_path / "g.fa"), bam, env={"GL_OVERSUBSCRIBE": "1"})
        got.append((open(prefix + ".depth.bed", "rb").read(), open(prefix + ".callable.bed", "rb").read()))
    assert got[0] == got[1] and got[0][0].count(b"\n") == sum((c[1] - 1) // 250 + 1 for c in contigs)


@pytest.mark.gpu
def test_indexcov_no_usable_chromosomes(tmp_path):
    refs = [("1", 100000)]
    (tmp_path / "g.fa.fai").write_text("1\t100000\t6\t60\t61\n")
    p = tmp_path / "a.bai"
    p.write_bytes(make_bai([[5]], [None]))                          # one interval -> no tiles
    r = run("indexcov", "-d", str(tmp_path / "o"), "--fai", str(tmp_path / "g.fa.fai"), str(p), check=False)
    assert r.returncode == 1 and "no usable chromsomes in bam" in r.stderr     # functional-tests.sh:58-62


@pytest.mark.gpu
def test_covstats(tmp_path):
    bam, ref, refs, recs, mates = _make_bam(tmp_path, seed=4, n=150000)
    p = run("covstats", "-n", "20000", bam)
    lines = p.stdout.splitlines()
    assert lines[0].startswith("coverage\tinsert_mean\tinsert_sd\tinsert_5th")
    t = lines[1].split("\t")
    # restate BamStats (covstats.go:122-220) on the records written above
    sizes, ins, tm = [], [], []
    k = nbad = ndup = nproper = nun = 0
    for i, (tid, pos, mapq, flag, cigar) in enumerate(recs):
        if i < 100000:
            continue
        if len(ins) >= 20000:
            break
        if flag & 4:
            nun += 1; continue
        k += 1
        if flag & (0x400 | 0x200):
            ndup += 1 if flag & 0x400 else 0
            nbad += 1; continue
        if flag & 2:
            nproper += 1
        if len(sizes) < 40000:
            sizes.append(sum(l for l, op in cigar if op in "MIS=X"))
        elif not ins:
            break
        mp, tl = mates[i]
        if pos < mp and flag & 2 and len(cigar) == 1 and cigar[0][1] == "M":
            ins.append(mp - (pos + cigar[0][0])); tm.append(tl)
    out6, H = orc.cs_tail(np.array(ins, np.int32), np.array(tm, np.int32), max(sizes))
    rl = np.sort(np.array(sizes))
    rl_mean = 0.0
    for a in rl:
        rl_mean += float(a) / len(rl)
    mapped = sum(1 for r in recs if r[0] >= 0)
    cov = (1 - nbad / (k + nun)) * mapped * rl_mean / sum(L for _, L in refs)
    exp = ["%.2f" % cov, "%.2f" % out6[2], "%.2f" % out6[3], "%d" % out6[0], "%d" % out6[1], "%.2f" % out6[4], "%.2f" % out6[5],
           "%.2f" % (100 * nun / (k + nun)), "%.1f" % (100 * nbad / (k + nun)), "%.1f" % (100 * ndup / (k + nun)),
           "%.1f" % (100 * nproper / (k + nun)), "%d" % max(sizes), bam, "S1"]
    assert t == exp


@pytest.mark.gpu
def test_depthwed(tmp_path):
    rng = np.random.default_rng(5)
    rows = [("chr1", a, min(a + 250, 10100)) for a in range(0, 10100, 250)] + [("chrX", a, min(a + 250, 1300)) for a in range(0, 1300, 250)]
    files, means = [], []
    for k in range(4):
        vals = [float("%.4g" % x) for x in rng.gamma(8, 4, len(rows))]
        p = tmp_path / ("s%d.depth.bed" % k)
        p.write_text("".join("%s\t%d\t%d\t%.4g\n" % (c, s, e, v) for (c, s, e), v in zip(rows, vals)))
        files.append(str(p)); means.append(vals)
    out = run("depthwed", "-s", "1000", *files).stdout.splitlines()
    cid = {"chr1": 0, "chrX": 1}
    s_, e_, c_, m_ = orc.depthwed(np.array(means), [r[1] for r in rows], [r[2] for r in rows], [cid[r[0]] for r in rows], 1000)
    assert out[0] == "#chrom\tstart\tend\ts0\ts1\ts2\ts3"
    exp = ["%s\t%d\t%d\t" % (["chr1", "chrX"][c], s, e) + "\t".join(str(int(v)) for v in row) for s, e, c, row in zip(s_, e_, c_, m_)]
    assert out[1:] == exp


@pytest.mark.gpu
def test_indexcov_crai_cohort(tmp_path):
    """CRAM indexes (.crai): interpolated 16 KB pseudo-tiles (indexcov/crai/crai.go:56-127) through the same cohort path"""
    rng = np.random.default_rng(9)
    refs = [("1", 4_000_000), ("2", 2_500_000)]
    fai = tmp_path / "g.fa.fai"
    fai.write_text("".join("%s\t%d\t6\t60\t61\n" % r for r in refs))
    paths, slices = [], []
    for k in range(5):
        per = []
        lines = []
        for si, (name, L) in enumerate(refs):
            st = np.cumsum(rng.integers(150_000, 400_000, 9)).astype(np.int64) + 1
            st = st[st < L - 10]
            sp = rng.integers(200_000, 420_000, st.size).astype(np.int64)
            by = rng.integers(2_000_000, 4_000_000, st.size).astype(np.int32)
            per.append((st, sp, by))
            lines += ["%d\t%d\t%d\t%d\t%d\t%d\n" % (si, a, b, 1000 + i, 10, c) for i, (a, b, c) in enumerate(zip(st, sp, by))]
        lines.append("-1\t0\t0\t99\t10\t500\n")
        p = tmp_path / ("cram%d.crai" % k)
        p.write_bytes(gzip.compress("".join(lines).encode()))
        paths.append(str(p)); slices.append(per)
    out = tmp_path / "cc"
    run("indexcov", "-d", str(out), "--fai", str(fai), *paths)
    exp_rows = ["#chrom\tstart\tend\t" + "\t".join("cram%d" % k for k in range(5))]
    depths = []
    for k in range(5):
        sz = [orc.crai_sizes(*slices[k][r]) for r in range(2)]
        m = orc.ic_median(np.concatenate(sz))
        depths.append([orc.ic_normalize(x, float(m)) for x in sz])
    for r, (name, L) in enumerate(refs):
        longest = max(len(depths[k][r]) for k in range(5))
        for i in range(longest):
            exp_rows.append("%s\t%d\t%d\t" % (name, i * 16384, (i + 1) * 16384) +
                            "\t".join("0" if i >= len(depths[k][r]) else "%.3g" % depths[k][r][i] for k in range(5)))
    assert gzip.open(str(out / "cc-indexcov.bed.gz"), "rt").read().splitlines() == exp_rows
