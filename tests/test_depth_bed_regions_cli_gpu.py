"""`goleft depth --bed` through the GPU feeder's region query: the BED lines of a contig are decoded on the device from only
the BGZF members their bin queries name.  The text is byte-identical to the oracle's per-line walk and to GL_GPU_FEED=0
(the host feeder), every contig with lines counts one GPU-fed pass, and a clustered panel reads a small share of the BAM."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
from oracle import loader as orc  # noqa: E402

GOLEFT = os.path.join(ROOT, "bin", "goleft")
CONTIGS = [("chr1", 23_000_000, 1), ("chr2", 4_100_000, 2), ("chrM", 16_569, 24)]
COV = 4.0


def run(*args, env=None):
    p = subprocess.run([GOLEFT, *args], capture_output=True, text=True, env=dict(os.environ, **env) if env else None)
    assert p.returncode == 0, p.stderr
    return p


def timing(p):
    return json.loads(p.stderr.strip().splitlines()[-1])["goleft_depth_timing"]


@pytest.fixture(scope="module")
def synth_bam(tmp_path_factory):
    import glsynth
    d = tmp_path_factory.mktemp("bedgpu")
    bam = str(d / "s.bam")
    glsynth.write_bam(bam, CONTIGS, coverage=COV)
    (d / "g.fa.fai").write_text("".join("%s\t%d\t6\t60\t61\n" % (c[0], c[1]) for c in CONTIGS))
    segs = {}
    for name, L, idx in CONTIGS:
        s, e = glsynth.segments(L, idx, coverage=COV)
        o = np.argsort(s, kind="stable")
        segs[name] = (s[o], e[o])
    return d, bam, str(d / "g.fa"), segs


def oracle_text(regions, W, segs):
    hd, ca = b"", b""
    for line in regions:
        name, rs, re = orc.chrom_start_end("%s\t%d\t%d" % line)
        if re <= rs:
            continue
        s, e = segs.get(name, (np.zeros(0, np.int32), np.zeros(0, np.int32)))
        lo = max(0, int(np.searchsorted(s, rs - 2000)) - 64)
        hi = int(np.searchsorted(s, re))
        h, c = orc.walk_chunk(name, rs, re, W, 4, 0, orc.pileup_diff(s[lo:hi], e[lo:hi], rs, re))
        hd += h; ca += c
    return hd, ca


def mixed_lines(W, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(250):
        name, L, _ = CONTIGS[int(rng.choice(3, p=[0.6, 0.3, 0.1]))]
        a = int(rng.integers(0, L))
        if rng.random() < 0.3:
            a = a // W * W                                                        # window-aligned
        ln = int(rng.choice([1, W - 1 if W > 1 else 1, W, W + 1, int(rng.integers(1, 20_000))]))
        out.append((name, a, a + max(ln, 1)))
    out += [("chr1", 5_000_000, 5_400_000), ("chr1", 5_100_000, 5_100_500), ("chr1", 5_300_000, 5_900_000),   # overlapping
            ("chr2", 4_099_000, 4_200_000), ("chr2", 4_200_000, 4_300_000), ("chrM", 16_000, 20_000),       # past the end
            ("chrUn_absent", 10, 700), ("chr2", 0, 1)]
    rng.shuffle(out)                                                              # unsorted
    return out


@pytest.mark.parametrize("W", [7, 250, 1_000_000])
def test_bed_gpu_feed_equals_oracle_and_host(synth_bam, W):
    d, bam, ref, segs = synth_bam
    regions = mixed_lines(W, W)
    bed = d / ("mixed%d.bed" % W)
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in regions))
    exp = oracle_text(regions, W, segs)
    got = {}
    for feed in ("1", "0"):
        prefix = str(d / ("m%d_%s" % (W, feed)))
        t = timing(run("depth", "--timing", "--bed", str(bed), "-w", str(W), "--prefix", prefix, "-r", ref, bam, env={"GL_GPU_FEED": feed}))
        got[feed] = (open(prefix + ".depth.bed", "rb").read(), open(prefix + ".callable.bed", "rb").read())
        assert t["gpu_fed_passes"] == (3 if feed == "1" else 0), t
    assert got["1"] == exp
    assert got["0"] == exp


def test_single_line_contigs(synth_bam):
    """a contig with one line reduces the device blocks directly"""
    d, bam, ref, segs = synth_bam
    regions = [("chr2", 1_000_003, 1_020_011), ("chrM", 0, 16_569), ("chr1", 22_999_000, 23_100_000)]
    bed = d / "single.bed"
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in regions))
    prefix = str(d / "single")
    t = timing(run("depth", "--timing", "--bed", str(bed), "-w", "100", "--prefix", prefix, "-r", ref, bam))
    assert t["gpu_fed_passes"] == 3
    assert (open(prefix + ".depth.bed", "rb").read(), open(prefix + ".callable.bed", "rb").read()) == oracle_text(regions, 100, segs)


def test_panel_reads_a_small_share(synth_bam):
    """8 genes of 10 exons on the 23 Mb contig read under 1/50 of what the .fai-mode run reads"""
    d, bam, ref, segs = synth_bam
    rng = np.random.default_rng(50)
    regions = []
    for g in np.sort(rng.integers(0, 22_900_000, 8)):
        for x in np.sort(rng.integers(0, 3000, 10)):
            regions.append(("chr1", int(g + x), int(g + x + rng.integers(80, 300))))
    bed = d / "panel.bed"
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in regions))
    t_fai = timing(run("depth", "--timing", "-w", "500", "--prefix", str(d / "fai"), "-r", ref, bam))
    prefix = str(d / "panel")
    t = timing(run("depth", "--timing", "--bed", str(bed), "-w", "250", "--prefix", prefix, "-r", ref, bam))
    assert t["gpu_fed_passes"] == 1
    assert t["bgzf_bytes_in"] < t_fai["bgzf_bytes_in"] / 50, (t["bgzf_bytes_in"], t_fai["bgzf_bytes_in"])
    assert (open(prefix + ".depth.bed", "rb").read(), open(prefix + ".callable.bed", "rb").read()) == oracle_text(regions, 250, segs)


def test_stats_and_gpus_unchanged(synth_bam):
    """--stats --bed and --gpus 3 (GL_OVERSUBSCRIBE=1) print the bytes of the host feeder's run"""
    d, bam, ref, segs = synth_bam
    rng = np.random.default_rng(9)
    fa = d / "st.fa"
    with open(fa, "w") as fh:
        for name, L, _ in CONTIGS:
            seq = "".join(rng.choice(list("ACGTNacgt"), L))
            fh.write(">%s\n" % name + "".join(seq[i:i + 60] + "\n" for i in range(0, L, 60)))
    off, lines = 0, []
    for name, L, _ in CONTIGS:
        off += len(">%s\n" % name)
        lines.append("%s\t%d\t%d\t60\t61\n" % (name, L, off))
        off += L + (L + 59) // 60
    (d / "st.fa.fai").write_text("".join(lines))
    regions = mixed_lines(250, 77)
    bed = d / "st.bed"
    bed.write_text("".join("%s\t%d\t%d\n" % r for r in regions))
    outs = {}
    for key, args, env in (("host", ["-s"], {"GL_GPU_FEED": "0"}), ("dev", ["-s"], {}),
                           ("gpus1", ["--gpus", "1"], {}), ("gpus3", ["--gpus", "3"], {"GL_OVERSUBSCRIBE": "1"})):
        prefix = str(d / ("st_" + key))
        run("depth", *args, "--bed", str(bed), "-w", "250", "--prefix", prefix, "-r", str(fa), bam, env=env)
        outs[key] = (open(prefix + ".depth.bed", "rb").read(), open(prefix + ".callable.bed", "rb").read())
    assert outs["dev"] == outs["host"]
    assert outs["gpus3"] == outs["gpus1"] == oracle_text(regions, 250, segs)
