#!/usr/bin/env python3
"""`goleft depth --bed` on the GPU feeder's region query against the host feeder, and the region decode against the whole
reference decode.

    python tools/bench_depth_bed.py [--runs 5] [--out DIR]

Writes the 30x synthetic chr20 BAM + BAI (tools/synth, the BAM bench.py's CLI leg uses) into a temporary directory, and two
BEDs on it: bench.py's exome shape (4,200 lines of 120-400 bp) and a clustered panel (50 genes of 10 exons each, about
500 lines).  Then, for each BED:
  cli      `goleft depth --timing --bed` with GL_GPU_FEED=1 (region query on the device) and GL_GPU_FEED=0 (host feeder),
           one warm-up run of each, then `runs` runs of each alternated; the wall clock of the process, the compressed bytes
           read and the records parsed, and the outputs of both routes compared byte for byte.
  library  gl_bam_decode_device_regions with the BED's intervals and gl_bam_decode_device on the whole chromosome, on one
           context, alternated, after one warm-up call each: the wall clock of the call (it returns after a device
           synchronise), bytes read, records parsed.
Prints one JSON line with the medians and ranges and the card's name and power limit as nvidia-smi reports them in this
run.  Needs a GPU."""
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


def beds(L):
    rng = np.random.default_rng(20)                                   # bench.py's exome leg
    starts = np.sort(rng.integers(100_000, L - 1000, 4200))
    lens = rng.integers(120, 400, starts.size)
    exome = [(int(a), int(a + n)) for a, n in zip(starts, lens)]
    rng = np.random.default_rng(21)
    panel = []
    for g in np.sort(rng.integers(100_000, L - 100_000, 50)):
        for x in np.sort(rng.integers(0, 30_000, 10)):
            panel.append((int(g + x), int(g + x + rng.integers(100, 300))))
    return {"exome": exome, "panel": panel}


def summary(v):
    return {"median_s": round(float(np.median(v)), 4), "min_s": round(min(v), 4), "max_s": round(max(v), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for bench_depth_bed.json (besides stdout)")
    a = ap.parse_args()
    import glsynth
    from goleft_b200 import capi
    exe = os.path.join(ROOT, "bin", "goleft")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    tmp = tempfile.mkdtemp(prefix="glbedbench_")
    res = {"gpu": gpu[0] if gpu else "unknown", "runs": a.runs}
    try:
        bam = os.path.join(tmp, "chr20.bam")
        L = glsynth.CHR20_LEN
        glsynth.write_bam(bam, [("chr20", L, 19)])
        open(os.path.join(tmp, "ref.fa.fai"), "w").write("chr20\t%d\t6\t60\t61\n" % L)
        res["bam_bytes"] = os.path.getsize(bam)
        ctx = capi.Ctx(0)
        b = capi.Bam(bam)
        for name, iv in beds(L).items():
            bed = os.path.join(tmp, name + ".bed")
            with open(bed, "w") as fh:
                fh.write("".join("chr20\t%d\t%d\n" % x for x in iv))
            walls = {"1": [], "0": []}
            tim, outs = {}, {}
            for rep in range(a.runs + 1):
                for feed in ("1", "0"):
                    prefix = os.path.join(tmp, "%s_%s" % (name, feed))
                    t0 = time.perf_counter()
                    p = subprocess.run([exe, "depth", "--timing", "-w", "250", "--bed", bed, "--prefix", prefix, "-r", os.path.join(tmp, "ref.fa"), bam],
                                       capture_output=True, text=True, env=dict(os.environ, GL_GPU_FEED=feed))
                    w = time.perf_counter() - t0
                    if p.returncode != 0:
                        raise RuntimeError(p.stderr[-300:])
                    if rep > 0:
                        walls[feed].append(w)
                    t = json.loads(p.stderr.strip().splitlines()[-1])["goleft_depth_timing"]
                    tim[feed] = {k: t[k] for k in ("wall_s", "records", "bgzf_bytes_in", "bgzf_bytes_out", "gpu_fed_passes")}
                    outs[feed] = open(prefix + ".depth.bed", "rb").read() + open(prefix + ".callable.bed", "rb").read()
            beg = np.array([x[0] for x in iv], np.int64)
            end = np.array([x[1] for x in iv], np.int64)
            lib = {"regions": [], "whole": []}
            last = {}
            for rep in range(a.runs + 1):
                for arm in ("regions", "whole"):
                    t0 = time.perf_counter()
                    d = capi.bam_decode_device_regions(ctx, b, 0, beg, end) if arm == "regions" else capi.bam_decode_device(ctx, b, 0)
                    w = time.perf_counter() - t0
                    if rep > 0:
                        lib[arm].append(w)
                    last[arm] = {k: d[k] for k in ("n", "n_records", "bytes_in", "bytes_out", "units", "inflate_s", "parse_s", "wall_s")}
            res[name] = {"lines": len(iv),
                         "cli": {"gpu_feed": dict(summary(walls["1"]), **tim["1"]), "host_feed": dict(summary(walls["0"]), **tim["0"]),
                                 "outputs_equal": outs["1"] == outs["0"]},
                         "library": {"regions": dict(summary(lib["regions"]), **last["regions"]), "whole_reference": dict(summary(lib["whole"]), **last["whole"])}}
        b.close()
        ctx.close()
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_depth_bed.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
