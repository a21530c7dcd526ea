#!/usr/bin/env python
"""Device-resident throughput of the cohort-scale kernels on one H100 (BASELINE configs 3 and 4 at 1-GPU shard size):
  indexcov: S samples x T tiles -> per-sample capped weighted median + normalised depth (ic_cohort2_kernel)
  depthwed: S samples x R windows of float64 means -> int matrix, row-major (depthwed_kernel)
Prints one JSON object; CUDA-event timing on the ctx stream, L2 flushed before every repetition."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from goleft_b200 import capi  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=313)          # 2504 / 8 GPUs
    ap.add_argument("--tiles", type=int, default=191_000)
    ap.add_argument("--wed-samples", type=int, default=63)       # 500 / 8 GPUs
    ap.add_argument("--wed-rows", type=int, default=6_176_584)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0
    out = {"peak_gbs": peak}
    ctx = capi.Ctx(0)

    # ---- indexcov cohort
    S, T = args.samples, args.tiles
    rng = np.random.default_rng(0)
    one = np.round(rng.lognormal(np.log(1.6e9), 0.25, T)).astype(np.int64)
    sizes = np.empty((S, T), np.int64)
    for k in range(S):
        sizes[k] = np.roll(one, k * 97) + k                       # distinct per sample, cheap to make
    ptr = (np.arange(S + 1, dtype=np.int64) * T)
    d_sizes, d_ptr = ctx.dev_array(sizes.reshape(-1)), ctx.dev_array(ptr)
    d_med, d_dep = ctx.dev_empty(S * 8), ctx.dev_empty(S * T * 4)
    ctx.indexcov_cohort_device(d_sizes, d_ptr, S, d_med, d_dep)
    ms = []
    for _ in range(args.reps):
        ctx.flush_l2(); ctx.timer_start()
        ctx.indexcov_cohort_device(d_sizes, d_ptr, S, d_med, d_dep)
        ms.append(ctx.timer_stop_ms())
    fallbacks = ctx.indexcov_cohort_fallbacks()
    med = d_med.download(np.float64, S)
    from oracle import loader as orc                               # spot check against the oracle (the checker only)
    for k in (0, S // 2, S - 1):
        assert med[k] == float(orc.ic_median(sizes[k]))
    t0 = time.perf_counter()
    for k in range(4):
        orc.ic_median(sizes[k])
    cpu_per_sample = (time.perf_counter() - t0) / 4
    alg = S * T * 12
    out["indexcov_cohort"] = {"samples": S, "tiles": T, "ms": float(np.mean(ms)), "tile_samples_per_s": S * T / (np.mean(ms) * 1e-3),
                              "alg_bytes": alg, "achieved_gbs": alg / (np.mean(ms) * 1e-3) / 1e9,
                              "frac_of_measured_peak": alg / (np.mean(ms) * 1e-3) / 1e9 / peak,
                              "kernel": "ic_cohort2_kernel (sorted-sample brackets: one counting/collecting pass + one normalise pass)",
                              "fallback_samples": fallbacks,
                              "cpu_port_ms_per_sample_1thread": cpu_per_sample * 1e3}
    for b in (d_sizes, d_ptr, d_med, d_dep):
        b.free()

    # ---- depthwed
    S2, R = args.wed_samples, args.wed_rows
    means = rng.gamma(9, 3.3, R)
    d_means = ctx.dev_empty(S2 * R * 8)
    for k in range(S2):
        capi.lib.gl_memcpy_h2d(ctx.h, d_means.ptr + k * R * 8, means.ctypes.data, R * 8)
    d_out = ctx.dev_empty(S2 * R * 8)
    ctx.depthwed_aggregate_device(d_means, S2, R, None, R, d_out)
    ms = []
    for _ in range(args.reps):
        ctx.flush_l2(); ctx.timer_start()
        ctx.depthwed_aggregate_device(d_means, S2, R, None, R, d_out)
        ms.append(ctx.timer_stop_ms())
    got = d_out.download(np.int64, S2 * 1000).reshape(1000, S2)
    assert np.array_equal(got[:, 0], (0.5 + means[:1000]).astype(np.int64))
    alg = S2 * R * 16
    out["depthwed"] = {"samples": S2, "rows": R, "ms": float(np.mean(ms)), "cells_per_s": S2 * R / (np.mean(ms) * 1e-3),
                       "alg_bytes": alg, "achieved_gbs": alg / (np.mean(ms) * 1e-3) / 1e9,
                       "frac_of_measured_peak": alg / (np.mean(ms) * 1e-3) / 1e9 / peak}
    # ---- depthwed, int32 in / int32 out (the form that travels over NVLink)
    d_i32 = ctx.dev_empty(S2 * R * 4)
    dep32 = (0.5 + means).astype(np.int32)
    for k in range(S2):
        capi.lib.gl_memcpy_h2d(ctx.h, d_i32.ptr + k * R * 4, dep32.ctypes.data, R * 4)
    d_o32, d_ovf = ctx.dev_empty(S2 * R * 4), ctx.dev_array(np.zeros(4, np.int32))
    ctx.depthwed_aggregate_i32_device(d_i32, S2, R, None, 0, R, d_o32.ptr, d_ovf); ctx.sync()
    ms = []
    for _ in range(args.reps):
        ctx.flush_l2(); ctx.timer_start()
        ctx.depthwed_aggregate_i32_device(d_i32, S2, R, None, 0, R, d_o32.ptr, d_ovf)
        ms.append(ctx.timer_stop_ms())
    got = d_o32.download(np.int32, S2 * 1000).reshape(1000, S2)
    assert np.array_equal(got[:, 0], dep32[:1000]) and int(d_ovf.download(np.int32, 1)[0]) == 0
    alg = S2 * R * 8
    out["depthwed_i32"] = {"samples": S2, "rows": R, "ms": float(np.mean(ms)), "cells_per_s": S2 * R / (np.mean(ms) * 1e-3),
                           "alg_bytes": alg, "achieved_gbs": alg / (np.mean(ms) * 1e-3) / 1e9,
                           "frac_of_measured_peak": alg / (np.mean(ms) * 1e-3) / 1e9 / peak}
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
