"""Fixed cost of a resident packed8 reduce, and the gap between the kernels of a 25-contig step (GPU only).

    python tools/bench_p8_chain.py [--regions 200] [--reps 7] [--steps 10] [--no-genome]

(a) fixed: R back-to-back resident packed8 reduces (gl_depth_begin / add_segments_packed8_device / gl_depth_reduce) of one
    64 kb region (16 tiles, 30x, glsynth) with nothing queried in the timed window; step time / R.  The ctx stream is
    held by a sleep kernel while the host queues the R reduces, so the window times the device, not the host's enqueue.
(b) step:  bench.py's `value` step, the 25 GRCh38 contigs resident as packed8, L2 flushed before every step.
(c) gap:   (b) minus the sum of the per-kernel event times of the same step in profile mode (gl_profile_*).
Prints the card, its power limit and SM clock, then one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))

W, MINCOV, MAXMEAN, STEP = 500, 4, 0, 10_000_000      # bench.py's value step


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except Exception as ex:
        out = "nvidia-smi failed: %s" % ex
    return dict(zip(q.split(","), [t.strip() for t in out.split(",")])) if out.count(",") == 3 else {"raw": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--regions", type=int, default=200)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--no-genome", action="store_true", help="only (a)")
    args = ap.parse_args()

    import torch
    from goleft_b200 import capi
    import glsynth
    if capi.device_count() < 1:
        raise SystemExit("bench_p8_chain.py: no CUDA device")
    import ctypes as C
    ctx = capi.Ctx(0)
    handle = C.c_uint64(0)
    ctx._ck(capi.lib.gl_stream_handle(ctx.h, C.byref(handle)))
    stream = torch.cuda.ExternalStream(handle.value, device=torch.device("cuda", 0))
    info = {"card_before": card()}

    def put(L, idx):
        s, e = glsynth.segments(L, idx)
        qa, qd, ql = capi.pack_segments8(s, e, threads=0)
        return {"L": L, "nb": int(qa.size), "d": (ctx.dev_array(qa), ctx.dev_array(qd), ctx.dev_array(ql))}

    def resident(w):
        ctx.depth_begin(0, w["L"])
        ctx.depth_add_segments_packed8_device(*w["d"], w["nb"])
        ctx.depth_reduce(W, MINCOV, MAXMEAN, STEP)

    # ---- (a) fixed cost per reduce
    small = put(1 << 16, 1)
    for _ in range(20):
        resident(small)
    ref = (ctx.depth_get_windows().copy(),) + tuple(a.copy() for a in ctx.depth_get_runs())
    per_region, enqueue = [], []
    for _ in range(args.reps):
        ctx.sync()
        with torch.cuda.stream(stream):
            torch.cuda._sleep(100_000_000)                   # ~50 ms: the host queues every reduce before the first runs
        ctx.timer_start()
        t0 = time.perf_counter()
        for _ in range(args.regions):
            resident(small)
        enqueue.append((time.perf_counter() - t0) * 1e6 / args.regions)
        per_region.append(ctx.timer_stop_ms() * 1e3 / args.regions)
    got = (ctx.depth_get_windows(),) + ctx.depth_get_runs()
    same = all(np.array_equal(x, y) for x, y in zip(ref, got))
    out = {"a_us_per_region": {"median": float(np.median(per_region)), "min": float(min(per_region)), "max": float(max(per_region))},
           "a_host_enqueue_us_per_region": float(np.median(enqueue)), "a_regions": args.regions, "a_tiles": 16, "a_results_equal": same}

    # ---- (b) the 25-contig resident step, (c) its gap
    if not args.no_genome:
        work = [put(L, i) for i, (_, L) in enumerate(glsynth.GRCH38)]
        for _ in range(3):
            for w in work:
                resident(w)
        steps = []
        for _ in range(args.steps):
            ctx.flush_l2()
            ctx.timer_start()
            for w in work:
                resident(w)
            steps.append(ctx.timer_stop_ms())
        ctx.profile_enable(True)
        ctx.profile_read()
        ksum, per_kernel = [], {}
        for _ in range(args.steps):
            ctx.flush_l2()
            for w in work:
                resident(w)
            recs = ctx.profile_read()
            ksum.append(sum(t for _, t in recs))
            for nm, t in recs:
                per_kernel.setdefault(nm, [0.0, 0])
                per_kernel[nm][0] += t / args.steps
                per_kernel[nm][1] += 1
        ctx.profile_enable(False)
        b, k = float(np.median(steps)), float(np.median(ksum))
        out.update({"b_step_ms": {"median": b, "min": float(min(steps)), "max": float(max(steps))},
                    "b_gbases_per_s": sum(w["L"] for w in work) / b / 1e6,
                    "c_kernel_sum_ms": k, "c_gap_ms": b - k,
                    "c_per_kernel_ms": {nm: round(v[0], 4) for nm, v in per_kernel.items()},
                    "c_launches_per_step": {nm: v[1] // args.steps for nm, v in per_kernel.items()}})
    info["card_after"] = card()
    out.update(info)
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
