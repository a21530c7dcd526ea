#!/usr/bin/env python
"""`goleft multidepth` throughput: S synthetic chr20-sized samples resident on the devices as packed8 words.

    python tools/bench_multidepth.py [--samples 32] [--reps 2] [--gpus 1]

--gpus N splits the samples into N contiguous ranges, one context per range on device g % (visible devices), each keeping
its own samples resident (more contexts than devices only with GL_OVERSUBSCRIBE=1: that shows correctness, not scaling).
Prints one JSON object: sample-Gbases/s = S x contig length / (pass 1 + merge + sites + host blocks + pass 2), the phase
times, the bytes the merge moved, the number of blocks and of cells that took the float64 chain, and the result of the
oracle check that runs before timing.  Writes nothing to the tree."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
import glsynth  # noqa: E402
from goleft_b200 import capi  # noqa: E402
from oracle import loader as orc  # noqa: E402   (the checker, never the thing measured)
from oracle import multidepth as omd  # noqa: E402


def multidepth_leg(ctxs, n_cpus, S=32, check_len=5_200_000, reps=2):
    """`goleft multidepth` on S synthetic samples of a chr20-sized contig (glsynth seeds differ per sample), split over the
    contexts in contiguous ranges and resident on each context's device as packed8.  9 of every 16 samples at 5x, the
    rest at 30x (18 and 14 at S = 32): a site is sufficient when more than 16 samples reach 7, so about half the sites are,
    chains break and blocks stay short, as in a cohort of mixed depth.  Checked first against the oracle on the contig's
    first check_len bases (chunk 0 and the start of chunk 1); then pass 1 (counts), the merge of the contexts' counters,
    the site classes, the host block machine and pass 2 (adopted sites, sums + certification + float64 chains, results)
    are timed with a host clock around synchronising calls (Ctx.multidepth_sharded)."""
    L = glsynth.CHR20_LEN
    G = len(ctxs)
    covs = [5.0 if i % 16 >= 7 else 30.0 for i in range(S)]
    cuts = [S * g // G for g in range(G + 1)]
    dev, host = [[] for _ in range(G)], []
    for g in range(G):
        for i in range(cuts[g], cuts[g + 1]):
            s, e = glsynth.segments(L, 200 + i, coverage=covs[i], min_mapq=10, threads=n_cpus)
            a, d, ln = capi.pack_segments8(s, e, threads=0)
            dev[g].append((ctxs[g].dev_array(a), ctxs[g].dev_array(d), ctxs[g].dev_array(ln), a.size))
            host.append((s, e))

    def adders():
        return [[lambda c, w=w: capi.lib.gl_depth_add_segments_packed8_device(c.h, w[0].ptr, w[1].ptr, w[2].ptr, w[3]) for w in ws]
                for ws in dev]

    # oracle check: the same cohort on the first check_len bases of the contig
    got = capi.Ctx.multidepth_sharded(ctxs, "chr20", check_len, adders())
    depth = np.stack([orc.pileup_diff(s, e, 0, check_len) for s, e in host])
    exp, _ = omd.text("chr20", depth)
    del depth, host
    ok = got == exp
    runs = []
    for _ in range(reps):
        _, parts = capi.Ctx.multidepth_sharded(ctxs, "chr20", L, adders(), parts=True)
        ms = parts["ms"]
        runs.append((sum(ms.values()), ms, parts["merge_bytes"]))
    total, ms, merge_bytes = min(runs, key=lambda r: r[0])
    st = [c.multidepth_stats() for c in ctxs]
    for ws in dev:
        for w in ws:
            for b in w[:3]:
                b.free()
    return {"value": S * L / total * 1e3 / 1e9, "unit": "sample-Gbases/s", "samples": S, "bases": L, "coverage": covs,
            "contexts": G, "devices": sorted({c.device for c in ctxs}), "samples_per_context": [b - a for a, b in zip(cuts, cuts[1:])],
            "ms": dict(total=total, **ms), "merge_bytes": merge_bytes,
            "merge_GB_per_s": merge_bytes / ms["merge"] / 1e6 if G > 1 and ms["merge"] > 0 else None,
            "blocks": int(st[0]["blocks"]), "walked_cells": int(sum(x["walked"] for x in st)),
            "certified_cells": int(sum(x["certified"] for x in st)),
            "oracle_check": {"bases": check_len, "rows": exp.count(b"\n"), "identical": bool(ok)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=32)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--gpus", type=int, default=1, help="contexts, one per device (0: every visible device)")
    args = ap.parse_args()
    n_dev = capi.device_count()
    if n_dev < 1:
        raise SystemExit("bench_multidepth.py: no CUDA device; goleft_b200 has no CPU fallback")
    G = args.gpus if args.gpus > 0 else n_dev
    if G > n_dev and not os.environ.get("GL_OVERSUBSCRIBE"):
        G = n_dev
    G = min(G, args.samples)
    ctxs = [capi.Ctx(g % n_dev) for g in range(G)]
    try:
        out = multidepth_leg(ctxs, os.cpu_count() or 1, S=args.samples, reps=args.reps)
    finally:
        for c in ctxs:
            c.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
