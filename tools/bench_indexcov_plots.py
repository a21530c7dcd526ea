#!/usr/bin/env python
"""indexcov's charts (plot.cu) at cohort scale: 2504 samples x 191 k tiles split over 24 references, resident on the GPU.
Prints one JSON object with
  - pl_select_kernel and pl_raster_kernel times (CUDA events, after a warm-up, L2 flushed before every timed launch),
  - the host mirror of the raster (gl_plot_raster_series_host, every pool thread) as the CPU baseline,
  - the host frame + PNG time per image (gl_plot_compose + gl_plot_png),
  - `bin/goleft indexcov` wall time with and without --noplots at S = 313 and 2504 (tools/bench_indexcov_cli.py's .bai writer),
and the card, power limit and SM clock it ran on.

    python tools/bench_indexcov_plots.py [--reps 5] [--cli-samples 313,2504]
"""
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
from goleft_b200 import capi  # noqa: E402
from bench_indexcov_cli import HS37D5, write_bai  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip().splitlines()[0]
    except OSError:
        return "unknown"


def kernels(reps, S=2504, T=191_000, charts=24):
    rng = np.random.default_rng(1)
    per = T // charts
    flat = np.maximum(rng.normal(1.0, 0.15, S * per * charts).astype(np.float32), 0)
    flat[rng.random(flat.size) < 1e-4] = 3.0
    n = S * charts
    off = np.arange(n, dtype=np.int64) * per
    ln = np.full(n, per, np.int64)
    W, H = capi.PLOT_W, capi.PLOT_H
    res = {"samples": S, "tiles": per * charts, "charts": charts}
    with capi.Ctx(0) as ctx:
        bufs = {k: capi.DevBuf(ctx, max(16, a.nbytes)).upload(a) for k, a in (("v", flat), ("o", off), ("l", ln))}
        d_sel, d_y = capi.DevBuf(ctx, n * 24), capi.DevBuf(ctx, n * 8)

        def timed(fn):
            fn()                                                          # warm-up
            ts = []
            for _ in range(reps):
                ctx.flush_l2(); ctx.sync()
                ctx.timer_start(); fn(); ts.append(ctx.timer_stop_ms())
            return ts

        ts = timed(lambda: ctx.plot_select_device(bufs["v"], bufs["o"], bufs["l"], n, d_sel, d_y))
        res["select_ms"] = {"median": float(np.median(ts)), "all": ts, "bytes_read": int(flat.nbytes)}
        sel = d_sel.download(np.int64, n * 3).reshape(n, 3)
        yext = d_y.download(np.float32, n * 2).reshape(n, 2)
        chart = np.repeat(np.arange(charts), S).astype(np.int32)
        draw = (np.arange(n) % S + 1).astype(np.uint32)
        xf = []
        for c in range(charts):
            s, y = sel[c * S:(c + 1) * S], yext[c * S:(c + 1) * S]
            x0, x1 = float((s[:, 0] * 16384.0).min()), float(((s[:, 0] + (s[:, 1] - 1) * s[:, 2]) * 16384.0).max())
            xf.append(capi.plot_transform([x0, x1, float(y[:, 0].min()), float(y[:, 1].max())], W, H))
        xf = np.concatenate(xf)
        r = capi.plot_line_radius(S)
        extra = {k: capi.DevBuf(ctx, max(16, a.nbytes)).upload(a) for k, a in (("s", sel), ("c", chart), ("d", draw), ("x", xf))}
        d_img = capi.DevBuf(ctx, charts * W * H * 4)
        ts = timed(lambda: ctx.plot_raster_series_device(bufs["v"], bufs["o"], extra["s"], 16384.0, extra["c"], extra["d"], n, extra["x"],
                                                         charts, W, H, r, d_img))
        res["raster_ms"] = {"median": float(np.median(ts)), "all": ts, "segments": int(np.maximum(sel[:, 1] - 1, 0).sum())}
        dev = d_img.download(np.uint32, charts * W * H).reshape(charts, H, W)
        t0 = time.perf_counter()
        host = capi.plot_raster_series_host(flat, off, sel, 16384.0, chart, draw, xf, charts, W, H, r)
        res["host_mirror_raster_s"] = time.perf_counter() - t0
        res["host_threads"] = os.cpu_count()
        res["device_equals_host_mirror"] = bool(np.array_equal(dev, host))
        pal = np.array([(255, 255, 255)] + [capi.plot_color(k) for k in range(S)], np.uint8)
        t0 = time.perf_counter()
        for c in range(charts):
            capi.plot_png(capi.plot_compose(dev[c], pal, capi.PLOT_DEPTH, [0, 1e8, 0, 2.5], "position on %d" % c, "scaled coverage"))
        res["host_frame_png_ms_per_image"] = (time.perf_counter() - t0) * 1e3 / charts
    return res


def cli(samples):
    exe = os.path.join(ROOT, "bin", "goleft")
    tmp = tempfile.mkdtemp(prefix="glplots_")
    try:
        rng = np.random.default_rng(7)
        paths = []
        for k in range(samples):
            p = os.path.join(tmp, "s%04d.bai" % k)
            write_bai(p, rng, 0.6 + 0.8 * rng.random())
            paths.append(p)
        fai = os.path.join(tmp, "ref.fai")
        open(fai, "w").write("".join("%s\t%d\t0\t60\t61\n" % (str(i + 1) if i < 22 else ("X", "Y", "MT")[i - 22] if i < 25 else "GL%06d" % i, L)
                                     for i, L in enumerate(HS37D5)))
        out = {}
        for tag, extra in (("plots", []), ("noplots", ["--noplots"]), ("plots_again", []), ("noplots_again", ["--noplots"])):
            d = os.path.join(tmp, tag)
            t0 = time.perf_counter()
            p = subprocess.run([exe, "indexcov", "-d", d, "--fai", fai] + extra + paths, capture_output=True, text=True,
                               env=dict(os.environ, GL_TIMING="1"))
            out[tag + "_s"] = time.perf_counter() - t0
            if p.returncode != 0:
                out["error"] = p.stderr[-500:]
                break
            out[tag + "_charts_phase"] = [ln.strip() for ln in p.stderr.splitlines() if "charts" in ln and "timing" in ln]
        return out
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cli-samples", default="313,2504")
    args = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_indexcov_plots needs a CUDA device")
    res = {"card": card(), "reps": args.reps, "kernels": kernels(args.reps)}
    res["cli"] = {s: cli(int(s)) for s in args.cli_samples.split(",") if s}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
