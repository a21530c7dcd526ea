#!/usr/bin/env python3
"""covstats over a cohort: the library's BAM-to-BAM prefetch on one GPU, and `goleft covstats --gpus N` end to end.

    python tools/bench_covstats_cohort.py [--bams 8] [--records 6000000] [--n 1000000] [--repeats 5] [--out DIR]

Writes `bams` paired BAMs (tools/bench_covstats.write_paired_bam, distinct seeds) with their .bai into a temporary
directory; they are read from the page cache in every timed run.  Then:
  library  on one context, the cohort back to back without and with gl_bam_covstats_prefetch (BAM i+1's first batch read
           from the end of BAM i's call on), alternated: one warm-up round of each, then `repeats` timed rounds of each.  Every call
           returns after a device synchronise, so the wall clock around a round is the round.  The results of both arms are
           compared bit for bit.
  cli      `goleft covstats -n N` over the cohort for --gpus 1 .. every visible GPU, once each after one warm-up run, with
           stdout compared across them.
Prints one JSON line with the medians and ranges, the card's name and power limit as nvidia-smi reports them in this run,
and the host pool's thread count.  Needs a GPU."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench_covstats  # noqa: E402


def cohort_round(capi, ctx, paths, n, skip, prefetch):
    """-> (seconds, per-BAM (stats bytes, H bytes), prefetched flags)"""
    t = time.perf_counter()
    hs = [capi.Bam(p) for p in paths]
    out, flags = [], []
    for i, h in enumerate(hs):
        st, H = capi.bam_covstats(ctx, h, n, skip)
        if prefetch and i + 1 < len(hs):
            capi.bam_covstats_prefetch(ctx, hs[i + 1], n, skip)
        out.append((b"".join(np.float64(getattr(st, k)).tobytes() for k in capi.CovStats.STATS + capi.CovStats.COUNTERS), H.tobytes()))
        flags.append(st.prefetched)
    for h in hs:
        h.close()
    return time.perf_counter() - t, out, flags


def summary(v):
    return {"median_s": round(float(np.median(v)), 4), "min_s": round(min(v), 4), "max_s": round(max(v), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bams", type=int, default=8)
    ap.add_argument("--records", type=int, default=6_000_000)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--skip", type=int, default=100_000)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for bench_covstats_cohort.json (besides stdout)")
    args = ap.parse_args()
    from goleft_b200 import capi
    if capi.device_count() < 1:
        raise SystemExit("bench_covstats_cohort needs a CUDA device")
    capi.lib.glhost_pool_size.restype = C.c_int
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    res = {"bams": args.bams, "records": args.records, "n": args.n, "skip": args.skip, "repeats": args.repeats, "gpu": gpu[0] if gpu else "unknown",
           "gpus_visible": capi.device_count(), "host_threads": int(capi.lib.glhost_pool_size()), "bams_from": "page cache"}
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        t0 = time.time()
        for k in range(args.bams):
            p = os.path.join(tmp, "s%d.bam" % k)
            bench_covstats.write_paired_bam(p, args.records, seed=100 + k, sample="S%d" % k)
            paths.append(p)
        res["write_s"] = round(time.time() - t0, 1)
        res["bam_bytes"] = sum(os.path.getsize(p) for p in paths)
        walls = {False: [], True: []}
        last = {}
        with capi.Ctx(0) as ctx:
            for it in range(args.repeats + 1):                              # the first round of each arm warms up
                for pre in (False, True):
                    dt, out, flags = cohort_round(capi, ctx, paths, args.n, args.skip, pre)
                    if it:
                        walls[pre].append(dt)
                    last[pre] = (out, flags)
        res["library_one_gpu"] = {"no_prefetch": summary(walls[False]), "prefetch": summary(walls[True]),
                                  "identical": last[False][0] == last[True][0], "prefetched": sum(last[True][1])}
        goleft = os.path.join(ROOT, "bin", "goleft")
        cli, ref = {}, None
        for g in range(1, capi.device_count() + 1):
            cmd = [goleft, "covstats", "-n", str(args.n), "--gpus", str(g)] + paths
            subprocess.run(cmd, capture_output=True, check=True)               # warm-up
            t = time.perf_counter()
            r = subprocess.run(cmd, capture_output=True, check=True)
            cli[str(g)] = round(time.perf_counter() - t, 3)
            ref = ref if ref is not None else r.stdout
            cli.setdefault("identical", True)
            cli["identical"] = cli["identical"] and r.stdout == ref
        res["cli_s_by_gpus"] = cli
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        open(os.path.join(args.out, "bench_covstats_cohort.json"), "w").write(line + "\n")


if __name__ == "__main__":
    main()
