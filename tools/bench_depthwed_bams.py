#!/usr/bin/env python3
"""depthwed from BAMs: `goleft depthwed -s SIZE -r ref.fa *.bam` against the two-step route it replaces.

    python tools/bench_depthwed_bams.py [--samples 8] [--length 64444167] [--coverage 30] [-w 250] [-s 1000] [--repeats 3]
                                        [--gpus 1] [--out DIR]

Writes `samples` seeded BAMs of one chr20-sized contig with tools/synth/bamsynth.c (a distinct seed per sample) and their .bai
into a temporary directory, with a .fai naming the contig; they are read from the page cache in every timed run.  Then times
  direct    goleft depthwed -s SIZE -w W -r ref.fa --gpus G *.bam
  two_step  goleft depth --prefix <base> -w W -r ref.fa --gpus G x.bam for every BAM, one after the other, then
            goleft depthwed -s SIZE *.depth.bed
one warm-up run of each, then `repeats` runs of each, alternated.  The two stdouts are compared byte for byte on every run.
Prints one JSON line with the medians and ranges, the depth.bed bytes the two-step route wrote, the direct route's
--timing line, and the card's name and power limit as nvidia-smi reports them in this run.  Needs a GPU."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
import glsynth  # noqa: E402

GOLEFT = os.path.join(ROOT, "bin", "goleft")


def summary(v):
    return {"median_s": round(float(np.median(v)), 3), "min_s": round(min(v), 3), "max_s": round(max(v), 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=8)
    ap.add_argument("--length", type=int, default=glsynth.CHR20_LEN)
    ap.add_argument("--coverage", type=float, default=30.0)
    ap.add_argument("-w", type=int, default=250)
    ap.add_argument("-s", type=int, default=1000)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--gpus", default="1")
    ap.add_argument("--out", default=None, help="directory for bench_depthwed_bams.json (besides stdout)")
    args = ap.parse_args()
    from goleft_b200 import capi
    if capi.device_count() < 1:
        raise SystemExit("bench_depthwed_bams needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    res = {"samples": args.samples, "length": args.length, "coverage": args.coverage, "W": args.w, "SIZE": args.s, "repeats": args.repeats,
           "gpus": args.gpus, "gpu": gpu[0] if gpu else "unknown", "bams_from": "page cache"}
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.time()
        paths = []
        for k in range(args.samples):
            p = os.path.join(tmp, "s%02d.bam" % k)
            glsynth.write_bam(p, [("chr20", args.length, 100 + k)], coverage=args.coverage)
            paths.append(p)
        ref = os.path.join(tmp, "ref.fa")
        open(ref, "w").close()
        open(ref + ".fai", "w").write("chr20\t%d\t7\t60\t61\n" % args.length)
        res["write_s"] = round(time.time() - t0, 1)
        res["bam_bytes"] = sum(os.path.getsize(p) for p in paths)
        wd = os.path.join(tmp, "two_step")
        os.makedirs(wd)

        def direct():
            cmd = [GOLEFT, "depthwed", "-s", str(args.s), "-w", str(args.w), "-r", ref, "--gpus", args.gpus, "--timing"] + paths
            t = time.perf_counter()
            r = subprocess.run(cmd, capture_output=True, check=True)
            return time.perf_counter() - t, r.stdout, r.stderr.decode().strip().splitlines()[-1]

        def two_step():
            t = time.perf_counter()
            for p in paths:
                subprocess.run([GOLEFT, "depth", "--prefix", os.path.basename(p)[:-4], "-w", str(args.w), "-r", ref, "--gpus", args.gpus, p],
                               capture_output=True, check=True, cwd=wd)
            beds = [os.path.basename(p)[:-4] + ".depth.bed" for p in paths]
            r = subprocess.run([GOLEFT, "depthwed", "-s", str(args.s)] + beds, capture_output=True, check=True, cwd=wd)
            dt = time.perf_counter() - t
            return dt, r.stdout, sum(os.path.getsize(os.path.join(wd, b)) for b in beds)

        walls = {"direct": [], "two_step": []}
        identical = True
        for it in range(args.repeats + 1):                                  # the first run of each route warms up
            dt_d, out_d, timing = direct()
            dt_t, out_t, bed_bytes = two_step()
            identical = identical and out_d == out_t
            if it:
                walls["direct"].append(dt_d)
                walls["two_step"].append(dt_t)
        res["direct"] = summary(walls["direct"])
        res["two_step"] = summary(walls["two_step"])
        res["identical"] = identical
        res["matrix_bytes"] = len(out_d)
        res["matrix_rows"] = out_d.count(b"\n") - 1
        res["depth_bed_bytes"] = bed_bytes
        res["direct_timing"] = json.loads(timing)
        res["runs_direct_s"] = [round(x, 3) for x in walls["direct"]]
        res["runs_two_step_s"] = [round(x, 3) for x in walls["two_step"]]
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "bench_depthwed_bams.json"), "w").write(line + "\n")
    if not identical:
        raise SystemExit("bench_depthwed_bams: the two routes printed different bytes")


if __name__ == "__main__":
    main()
