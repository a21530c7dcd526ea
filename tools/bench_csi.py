#!/usr/bin/env python3
"""`goleft depth` on CSI-indexed BAMs.

    python tools/bench_csi.py [--runs 5] [--out DIR]

Two comparisons, each with one warm-up run of both arms and then `runs` runs of each arm alternated, in one process:
  chr20     the 30x synthetic chr20 BAM (tools/synth, the BAM bench.py's CLI leg uses) with its BAI against the same BAM
            with its CSI (tools/synth's CSI output: min_shift 14, depth 5): `goleft depth -w 250`.  The two should take
            the same time; their outputs are compared byte for byte.
  long      one contig of 1.2e9 bases at 0.1x coverage (150 bp reads, tests/csi_bams.py's writer, CSI of depth 6), longer
            than one depth pass, so its two passes are region queries: GL_GPU_FEED=1 (decoded on the device) against
            GL_GPU_FEED=0 (host feeder), outputs compared byte for byte.
The time is the process wall clock.  Prints one JSON line with the medians and ranges, and the card's name and power limit
as nvidia-smi reports them in this run.  Needs a GPU."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
sys.path.insert(0, os.path.join(ROOT, "tests"))


def long_contig(d, L=1_200_000_000, cov=0.1, seed=9):
    import csi_bams as cb
    rng = np.random.default_rng(seed)
    pos = np.sort(rng.integers(0, L - 200, int(L * cov / 150))).tolist()
    cig = [[(150, "M")], [(70, "M"), (5, "D"), (80, "M")], [(10, "S"), (140, "M")]]
    recs = [(0, p0, 60, 0 if k % 5 else 16, cig[k % 3]) for k, p0 in enumerate(pos)]
    bam, csi, _ = cb.make_bam_csi([("chrLong", L)], recs, 14, 6, with_bai=False)
    open(os.path.join(d, "long.bam"), "wb").write(bam)
    open(os.path.join(d, "long.bam.csi"), "wb").write(csi)
    open(os.path.join(d, "long.fa.fai"), "w").write("chrLong\t%d\t9\t60\t61\n" % L)
    return len(recs)


def summary(v):
    return {"median_s": round(float(np.median(v)), 4), "min_s": round(min(v), 4), "max_s": round(max(v), 4)}


def alternate(exe, arms, runs):
    """arms: {name: (argv, env, output prefix)} -> ({name: [wall]}, {name: timing json}, outputs equal)"""
    walls, tim, outs = {k: [] for k in arms}, {}, {}
    for rep in range(runs + 1):
        for name, (argv, env, prefix) in arms.items():
            t0 = time.perf_counter()
            p = subprocess.run([exe, *argv], capture_output=True, text=True, env=dict(os.environ, **env))
            w = time.perf_counter() - t0
            if p.returncode != 0:
                raise RuntimeError(p.stderr[-300:])
            if rep > 0:
                walls[name].append(w)
            t = json.loads(p.stderr.strip().splitlines()[-1])["goleft_depth_timing"]
            tim[name] = {k: t[k] for k in ("wall_s", "records", "bgzf_bytes_in", "gpu_fed_passes")}
            outs[name] = open(prefix + ".depth.bed", "rb").read() + open(prefix + ".callable.bed", "rb").read()
    same = len({outs[k] for k in outs}) == 1
    return {k: dict(summary(walls[k]), **tim[k]) for k in arms}, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for bench_csi.json (besides stdout)")
    a = ap.parse_args()
    import glsynth
    exe = os.path.join(ROOT, "bin", "goleft")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    tmp = tempfile.mkdtemp(prefix="glcsibench_")
    res = {"gpu": gpu[0] if gpu else "unknown", "runs": a.runs}
    try:
        for sub in ("bai", "csi"):
            os.makedirs(os.path.join(tmp, sub))
        L = glsynth.CHR20_LEN
        bam = os.path.join(tmp, "bai", "chr20.bam")
        glsynth.write_bam(bam, [("chr20", L, 19)])
        glsynth.write_bam(os.path.join(tmp, "csi", "chr20.bam"), [("chr20", L, 19)], index="csi")      # the same BAM
        open(os.path.join(tmp, "ref.fa.fai"), "w").write("chr20\t%d\t6\t60\t61\n" % L)
        arms = {sub: (["depth", "--timing", "-w", "250", "--prefix", os.path.join(tmp, "o_" + sub), "-r", os.path.join(tmp, "ref.fa"),
                       os.path.join(tmp, sub, "chr20.bam")], {}, os.path.join(tmp, "o_" + sub)) for sub in ("bai", "csi")}
        r, same = alternate(exe, arms, a.runs)
        res["chr20"] = {"bam_bytes": os.path.getsize(bam), "bai": r["bai"], "csi": r["csi"], "outputs_equal": same}
        t0 = time.perf_counter()
        n = long_contig(tmp)
        res["long"] = {"contig_bases": 1_200_000_000, "records": n, "write_s": round(time.perf_counter() - t0, 1)}
        arms = {"gpu_feed_%s" % f: (["depth", "--timing", "-w", "1000", "--prefix", os.path.join(tmp, "l" + f), "-r", os.path.join(tmp, "long.fa"),
                                     os.path.join(tmp, "long.bam")], {"GL_GPU_FEED": f}, os.path.join(tmp, "l" + f)) for f in ("1", "0")}
        r, same = alternate(exe, arms, a.runs)
        res["long"].update(r)
        res["long"]["outputs_equal"] = same
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_csi.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
