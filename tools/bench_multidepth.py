#!/usr/bin/env python
"""`goleft multidepth` throughput on one H100: S synthetic chr20-sized samples resident on the device as packed8 words.

    python tools/bench_multidepth.py [--samples 32] [--reps 2]

Prints one JSON object: sample-Gbases/s = S x contig length / (pass 1 + host blocks + pass 2), the phase times, the number
of blocks and of cells that took the float64 chain, and the result of the oracle check that runs before timing.
Writes nothing to the tree."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
import glsynth  # noqa: E402
from goleft_b200 import capi  # noqa: E402
from oracle import loader as orc  # noqa: E402   (the checker, never the thing measured)
from oracle import multidepth as omd  # noqa: E402


def multidepth_leg(ctx, n_cpus, S=32, check_len=5_200_000, reps=2):
    """`goleft multidepth` on S synthetic samples of a chr20-sized contig (glsynth seeds differ per sample), resident on the
    device as packed8.  9 of every 16 samples at 5x, the rest at 30x (18 and 14 at S = 32): a site is sufficient when more
    than 16 samples reach 7, so about half the sites are, chains break and blocks stay short, as in a cohort of mixed depth.
    Checked first against the oracle on the contig's first check_len bases (chunk 0 and the start of chunk 1); then pass 1
    (counts + site classes), the host block machine and pass 2 (sums + certification + float64 chains) are timed with a
    host clock around synchronising calls."""
    L = glsynth.CHR20_LEN
    covs = [5.0 if i % 16 >= 7 else 30.0 for i in range(S)]
    dev, host = [], []
    for i in range(S):
        s, e = glsynth.segments(L, 200 + i, coverage=covs[i], min_mapq=10, threads=n_cpus)
        a, d, ln = capi.pack_segments8(s, e, threads=0)
        dev.append((ctx.dev_array(a), ctx.dev_array(d), ctx.dev_array(ln), a.size))
        host.append((s, e))

    def adders():
        return [lambda c, w=w: capi.lib.gl_depth_add_segments_packed8_device(c.h, w[0].ptr, w[1].ptr, w[2].ptr, w[3]) for w in dev]

    # oracle check: the same cohort on the first check_len bases of the contig
    got = ctx.multidepth("chr20", check_len, adders())
    depth = np.stack([orc.pileup_diff(s, e, 0, check_len) for s, e in host])
    exp, _ = omd.text("chr20", depth)
    del depth, host
    ok = got == exp
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        ctx.multidepth_begin(L, S)
        for add in adders():
            ctx.depth_begin(0, L)
            add(ctx)
            ctx.multidepth_count()
        rs, rc = ctx.multidepth_sites()
        t1 = time.perf_counter()
        bs, be, bn = capi.multidepth_blocks(rs, rc, L, S)
        t2 = time.perf_counter()
        ctx.multidepth_set_blocks(bs, be, bn)
        for i, add in enumerate(adders()):
            ctx.depth_begin(0, L)
            add(ctx)
            ctx.multidepth_sums(i)
        _, q, val, cert = ctx.multidepth_result(bs.size, S)
        t3 = time.perf_counter()
        times.append((t3 - t0, t1 - t0, t2 - t1, t3 - t2))
    best = min(times)
    st = ctx.multidepth_stats()
    for w in dev:
        for b in w[:3]:
            b.free()
    return {"value": S * L / best[0] / 1e9, "unit": "sample-Gbases/s", "samples": S, "bases": L, "coverage": covs,
            "ms": {"total": best[0] * 1e3, "pass1": best[1] * 1e3, "blocks_host": best[2] * 1e3, "pass2": best[3] * 1e3},
            "blocks": int(st["blocks"]), "walked_cells": int(st["walked"]), "certified_cells": int(st["certified"]),
            "oracle_check": {"bases": check_len, "rows": exp.count(b"\n"), "identical": bool(ok)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=32)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_multidepth.py: no CUDA device; goleft_b200 has no CPU fallback")
    with capi.Ctx(0) as ctx:
        out = multidepth_leg(ctx, os.cpu_count() or 1, S=args.samples, reps=args.reps)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
