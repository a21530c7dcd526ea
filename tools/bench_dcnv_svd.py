#!/usr/bin/env python
"""`goleft dcnv --svd` (gl_dcnv_svd, DESIGN §1.13) on one H100, at two seeded shapes with a planted rank-5 batch term:
3,088,281 x 128 (the `tools/bench_dcnv.py` shape) and an exome-shaped 200,000 x 2,504.

    python tools/bench_dcnv_svd.py [--shapes 3088281x128,200000x2504] [--reps 5] [--numpy-rows 200000]

Per shape:
  gram      svd_gram_kernel (+ stats, reduce) from CUDA events over --reps calls of gl_dcnv_svd_device with PCT 100 (nothing
            removed, so the matrix is unchanged between calls); FP64 rate n S (S + 1) / t against the data sheet's 67 TFLOP/s
            FP64 tensor-core figure (a reference point, not a measured peak).
  project   svd_project_kernel from CUDA events (the matrix re-uploaded before each call), at the PCT halfway between the
            fifth and sixth shares, so the planted five are removed; 16 n S bytes / t against 3.35 TB/s.
  eigen     the eigen phase (gl_dcnv_svd_phases), host clock.
  host      the whole gl_dcnv_svd from host arrays (copies included), host clock, with its phases.
  numpy     np.linalg.svd(Z, full_matrices=False) of the first --numpy-rows rows on the host, timed, rows stated.
The GPU result is checked against the first rows of the host result: the device and host entries must agree bit for bit.
Prints one JSON object with the card name and power limit read in the same run.  Writes nothing to the tree."""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_dcnv import card  # noqa: E402
from goleft_b200 import capi  # noqa: E402
from oracle import dcnv_svd as osv  # noqa: E402   (the comparison, never the thing measured)

PEAK_FP64_TC = 67e12
PEAK_BW = 3.35e12


def matrix(rng, n, S, k=5):
    """normalised depths around 1 with a rank-k batch term, rows in blocks to bound the temporaries"""
    x = np.empty((n, S), np.float64)
    v = rng.normal(0, 1, (k, S))
    for a in range(0, n, 1 << 18):
        b = min(n, a + (1 << 18))
        u = rng.normal(0, 1, (b - a, k)) * (0.3 * 0.7 ** np.arange(k))
        x[a:b] = np.maximum(0.0, rng.gamma(40.0, 1 / 40.0, (b - a, S)) + u @ v)
    return x


def kernel_ms(prof, name):
    return sum(ms for nm, ms in prof if nm == name)


def one_shape(ctx, n, S, reps, numpy_rows, rng):
    out = {"rows": n, "samples": S}
    x = matrix(rng, n, S)
    d = ctx.dev_array(x)
    sv, _, _, _ = ctx.dcnv_svd_device(d, n, S, S, 100.0)                 # warm-up
    share = 100 * sv / sv.sum()
    pct = 0.5 * (share[4] + share[5])                                    # the planted five, as a user would set it
    ctx.profile_enable(True)
    ctx.profile_read()
    g = st = rd = 0.0
    for _ in range(reps):
        ctx.dcnv_svd_device(d, n, S, S, 100.0)
        prof = ctx.profile_read()
        g += kernel_ms(prof, "svd_gram_kernel")
        st += kernel_ms(prof, "svd_stats_kernel")
        rd += kernel_ms(prof, "svd_reduce_kernel")
    g, st, rd = g / reps, st / reps, rd / reps
    flops = float(n) * S * (S + 1)
    out["gram_ms"] = g
    out["stats_ms"] = st
    out["reduce_ms"] = rd
    out["gram_tflops"] = flops / (g * 1e-3) / 1e12
    out["gram_share_of_67tf"] = flops / (g * 1e-3) / PEAK_FP64_TC
    pj, eig = [], []
    for _ in range(reps):
        d.upload(x)
        sv, nr, nk, _ = ctx.dcnv_svd_device(d, n, S, S, pct)
        prof = ctx.profile_read()
        pj.append(kernel_ms(prof, "svd_project_kernel"))
        eig.append(ctx.dcnv_svd_phases()["eigen"])
    ctx.profile_enable(False)
    dev_first = d.download(np.float64, min(n, 4096) * S).reshape(-1, S)
    d.free()
    out["pct"] = pct
    out["n_removed"] = nr
    out["project_ms"] = float(np.median(pj))
    out["project_tbps"] = 16.0 * n * S / (out["project_ms"] * 1e-3) / 1e12
    out["project_share_of_3.35tbs"] = 16.0 * n * S / (out["project_ms"] * 1e-3) / PEAK_BW
    out["eigen_s"] = float(np.median(eig))
    host = np.array(x)
    sv_b, nr_b, nk_b = np.empty(S), C.c_int32(0), C.c_int64(0)
    t0 = time.perf_counter()
    rc = capi.lib.gl_dcnv_svd(ctx.h, host.ctypes.data_as(C.c_void_p), n, S, S, pct, 0, sv_b.ctypes.data_as(C.c_void_p), None,
                              C.byref(nr_b), C.byref(nk_b))
    out["host_call_s"] = time.perf_counter() - t0
    ctx._ck(rc)
    out["host_phases_s"] = ctx.dcnv_svd_phases()
    out["device_equals_host"] = bool(np.array_equal(dev_first, host[:dev_first.shape[0]]) and np.array_equal(sv, sv_b))
    del host
    m = min(n, numpy_rows)
    z, _, _, _ = osv.zscore(x[:m])
    t0 = time.perf_counter()
    np.linalg.svd(z, full_matrices=False)
    out["numpy_svd_rows"] = m
    out["numpy_svd_s"] = time.perf_counter() - t0
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="3088281x128,200000x2504")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--numpy-rows", type=int, default=200_000)
    a = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_dcnv_svd needs a CUDA device")
    res = {"card": card(), "shapes": []}
    rng = np.random.default_rng(20261016)
    with capi.Ctx(0) as ctx:
        for sh in a.shapes.split(","):
            n, S = (int(v) for v in sh.split("x"))
            res["shapes"].append(one_shape(ctx, n, S, a.reps, a.numpy_rows, rng))
            print(json.dumps(res["shapes"][-1]), file=sys.stderr, flush=True)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
