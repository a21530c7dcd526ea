#!/usr/bin/env python
"""indexcov's vector charts (INDEXCOV_FMT; plot.cu's path text) at cohort scale: 2504 samples x 191 k tiles split over 24
references, resident on the GPU, as tools/bench_indexcov_plots.py lays them out.  Prints one JSON object with
  - the device path: gl_plot_path_series_size (pl_path_kernel pass 1 + the scan) and gl_plot_path_series_emit (pass 2)
    times (CUDA events, after a warm-up, L2 flushed before every timed call), and the copy of the text home,
  - the host mirror (gl_plot_path_series_size_host + _emit_host on every pool thread) as the CPU baseline,
  - the bytes of path text and the vertices, for SVG and EPS,
and the card, power limit and SM clock it ran on.  The device text is checked against the host mirror's.

    python tools/bench_indexcov_vector.py [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from goleft_b200 import capi  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    S, T, charts = 2504, 191_000, 24
    rng = np.random.default_rng(1)
    per = T // charts
    flat = np.maximum(rng.normal(1.0, 0.15, S * per * charts).astype(np.float32), 0)
    flat[rng.random(flat.size) < 1e-4] = 3.0
    n = S * charts
    off = np.arange(n, dtype=np.int64) * per                             # dataset (c, k) at c * S + k, chart c
    ln = np.full(n, per, np.int64)
    sel, yext = capi.plot_select_host(flat, off, ln)
    chart = np.repeat(np.arange(charts, dtype=np.int32), S)
    xf = np.concatenate([capi.plot_transform([0, (per - 1) * 16384.0, 0, 2.5], capi.PLOT_W, capi.PLOT_H)] * charts)
    res = {"samples": S, "tiles": per * charts, "charts": charts, "vertices": int(sel[:, 1].sum()), "card": card()}
    lib = capi.lib
    with capi.Ctx(0) as ctx:
        d = {k: capi.DevBuf(ctx, max(16, x.nbytes)).upload(x) for k, x in (("v", flat), ("o", off), ("s", sel), ("c", chart), ("x", xf))}
        d_len, d_pos = capi.DevBuf(ctx, n * 8), capi.DevBuf(ctx, (n + 1) * 8)

        def size(fmt):
            ctx._ck(lib.gl_plot_path_series_size(ctx.h, d["v"].ptr, d["o"].ptr, d["s"].ptr, 16384.0, d["c"].ptr, n, d["x"].ptr, charts,
                                                 capi.PLOT_DEPTH, fmt, d_len.ptr, d_pos.ptr))

        def timed(fn):
            fn(); ctx.sync()                                                 # warm-up
            ts = []
            for _ in range(a.reps):
                ctx.flush_l2(); ctx.sync()
                ctx.timer_start(); fn(); ts.append(ctx.timer_stop_ms())
            return ts

        for name, fmt in (("svg", capi.PLOT_SVG), ("eps", capi.PLOT_EPS)):
            r = {}
            r["size_ms"] = timed(lambda: size(fmt))
            total = int(d_pos.download(np.int64, n + 1)[n])
            d_out = capi.DevBuf(ctx, max(16, total))

            def emit():
                ctx._ck(lib.gl_plot_path_series_emit(ctx.h, d["v"].ptr, d["o"].ptr, d["s"].ptr, 16384.0, d["c"].ptr, n, d["x"].ptr, charts,
                                                     capi.PLOT_DEPTH, fmt, d_pos.ptr, total, d_out.ptr, total))
            r["emit_ms"] = timed(emit)
            t0 = time.perf_counter()
            dev = d_out.download(np.uint8, total)
            r["d2h_ms"] = (time.perf_counter() - t0) * 1e3
            d_out.free()
            t0 = time.perf_counter()
            hl, ht = capi.plot_path_series_host(flat, off, sel, 16384.0, chart, xf, charts, capi.PLOT_DEPTH, fmt)
            r["host_mirror_ms"] = (time.perf_counter() - t0) * 1e3
            r["bytes"] = total
            r["bytes_per_vertex"] = total / res["vertices"]
            r["device_equals_host"] = bool(dev.tobytes() == ht)
            res[name] = r
        for b in list(d.values()) + [d_len, d_pos]:
            b.free()
    res["host_threads"] = os.cpu_count()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
