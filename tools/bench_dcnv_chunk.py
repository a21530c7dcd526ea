#!/usr/bin/env python
"""`goleft dcnv --chunk W` against the default moving median on one H100, at tools/bench_dcnv.py's shape: a GRCh38-shaped
cohort matrix at `depthwed -s 1000` (3.09 M rows x 128 samples by default), seeded, GC from the same synthetic FASTA.

    python tools/bench_dcnv_chunk.py [--samples 128] [--runs 3] [--widths 0.05,0.01,0.001,1e-9] [--check-cols 2]

For each W: the chunk boundaries (gl_dcnv_chunk_slices, host), their count and length distribution (with how many fall in
each select bucket: <= 16 rows a thread, <= 1024 a warp, <= 65536 a 256-thread CTA, longer a 1024-thread CTA), then
gl_dcnv_normalize and gl_dcnv_normalize_chunked alternated --runs times, each timed with a host clock around the
synchronising call: from host arrays (pageable copies included) and on a device-resident matrix (the _device entries).
Medians over the runs are reported.  --check-cols sample columns are compared with the oracle at full n, bit for bit.
Prints one JSON object with the card name and power limit.  Writes nothing to the tree."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_dcnv import card, gc_library, genome, rows_of  # noqa: E402
from goleft_b200 import capi  # noqa: E402
from oracle import dcnv_chunk as oc  # noqa: E402   (the checker, never the thing measured)

BUCKETS = (16, 1024, 65536)


def timed(f):
    t0 = time.perf_counter()
    r = f()
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=128)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--widths", default="0.05,0.01,0.001,1e-9")
    ap.add_argument("--check-cols", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    a = ap.parse_args()
    rng = np.random.default_rng(a.seed)
    S = a.samples
    contigs = genome(rng)
    cid, starts, ends = rows_of(contigs)
    n = starts.size
    x = rng.poisson(30.0, (n, S)).astype(np.float64)
    x[rng.random((n, S)) < 0.002] = 0
    res = {"card": card(), "rows": int(n), "samples": S, "runs": a.runs, "widths": {}}
    with capi.Ctx(0) as ctx:
        gc = gc_library(ctx, contigs, cid, starts, ends)
        inds = capi.go_argsort(gc)
        v = gc[inds]
        res["distinct_gc"] = int(np.unique(gc).size)
        out = np.empty((n, S))
        d_x, d_inds = ctx.dev_array(x), ctx.dev_array(inds)
        d_out, d_med = ctx.dev_empty(n * S * 8), ctx.dev_empty(S * 8)
        cols = np.linspace(0, S - 1, a.check_cols).astype(int)
        for w in [float(t) for t in a.widths.split(",")]:
            t_sl, ptr = timed(lambda: capi.dcnv_chunk_slices(v, w))
            ln = np.diff(ptr)
            edges = (0,) + BUCKETS + (n,)
            r = {"chunks": int(ln.size), "slices_host_s": round(t_sl, 4),
                 "length": {"min": int(ln.min()), "median": float(np.median(ln)), "max": int(ln.max()), "mean": float(ln.mean())},
                 "chunks_per_bucket": [int(((ln > lo) & (ln <= hi)).sum()) for lo, hi in zip(edges[:-1], edges[1:])]}
            t = {"median9_host": [], "chunk_host": [], "median9_device": [], "chunk_device": []}
            for _ in range(a.runs):
                t["median9_host"].append(timed(lambda: ctx.dcnv_normalize(x, inds))[0])
                dt, (out, med) = timed(lambda: ctx.dcnv_normalize_chunked(x, inds, ptr))
                t["chunk_host"].append(dt)
                t["median9_device"].append(timed(lambda: ctx.dcnv_normalize_device(d_x, n, S, d_inds, 0, S, d_out, S, d_med))[0])
                t["chunk_device"].append(timed(lambda: ctx.dcnv_normalize_chunked_device(d_x, n, S, d_inds, ptr, 0, S, d_out, S, d_med))[0])
            r["s"] = {k: round(float(np.median(vs)), 4) for k, vs in t.items()}
            r["s_all"] = {k: [round(u, 4) for u in vs] for k, vs in t.items()}
            dev = d_out.download(np.float64, n * S).reshape(n, S)
            want, _, want_ptr, want_med = oc.matrix(x[:, cols], gc, w)
            r["oracle_check"] = {"columns": cols.tolist(),
                                 "identical": bool(np.array_equal(out[:, cols].view(np.uint64), want.view(np.uint64))
                                                   and np.array_equal(dev[:, cols].view(np.uint64), want.view(np.uint64))
                                                   and np.array_equal(med[cols], want_med) and np.array_equal(ptr, want_ptr))}
            res["widths"]["%g" % w] = r
            print(json.dumps({"%g" % w: r}), file=sys.stderr, flush=True)
        for b in (d_x, d_inds, d_out, d_med):
            b.free()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
