#!/usr/bin/env python
"""`goleft dcnv`'s depth chart on one H100.

    python tools/bench_dcnv_chart.py [--rows 3088281] [--samples 128] [--reps 5] [--cli-samples 128]

Library leg, at the dcnv benchmark's shape (3,088,281 rows x 128 samples, seeded normalised-looking depths): gl_dcnv_chart's
kernels (dc_first_kernel + dc_ext_kernel = select, dc_raster_kernel = raster) timed with CUDA events, the median of --reps
calls after a warm-up, L2 flushed before each; the entry's wall time (host -> device copies included); the host mirror
(gl_dcnv_chart_select_host + gl_dcnv_chart_raster_host on every host thread) as the CPU baseline, and that both images are
equal; the page's "%.2f" tokens (gl_format_f2 on capped values, 16 M cells per call).  CLI leg: `goleft dcnv` with and
without --noplots on a chr1 + chr2 matrix (491,151 rows, DESIGN §1.9's CLI shape), GL_TIMING phases, the page's size and
its assembly rate (page bytes / "chart" phase).  Prints one JSON object with the card name and power limit.  Writes
nothing to the tree (temporary files go to a temporary directory)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from goleft_b200 import capi  # noqa: E402

CONTIGS = [("chr1", 248956422), ("chr2", 242193529)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:                                              # the numbers are still reported; say why the card is not
        return {"name": "unknown (%s)" % e, "power_limit": "unknown"}


def cohort(n, S, rng):
    x = rng.normal(1.0, 0.15, (n, S))
    x[rng.random((n, S)) < 0.01] = 0.0
    x[rng.random((n, S)) < 0.002] = 3.5
    return x


def library_leg(ctx, n, S, reps, rng):
    x = cohort(n, S, rng)
    out = {"rows": n, "samples": S, "vertices": int(n * S)}
    ctx.dcnv_chart(x)                                                   # warm-up
    sel, ras, wall = [], [], []
    ctx.profile_enable(True)
    for _ in range(reps):
        ctx.flush_l2()
        ctx.profile_read()
        t0 = time.perf_counter()
        first, yext, ext, img = ctx.dcnv_chart(x)
        wall.append(time.perf_counter() - t0)
        prof = ctx.profile_read()
        sel.append(sum(ms for nm, ms in prof if nm in ("dc_first_kernel", "dc_ext_kernel")))
        ras.append(sum(ms for nm, ms in prof if nm == "dc_raster_kernel"))
    ctx.profile_enable(False)
    out["select_ms"] = round(statistics.median(sel), 3)
    out["raster_ms"] = round(statistics.median(ras), 3)
    out["entry_wall_s"] = round(statistics.median(wall), 3)
    t0 = time.perf_counter()
    hf, hy = capi.dcnv_chart_select_host(x)
    he = capi.dcnv_chart_extent(hf, hy, n)
    himg = capi.dcnv_chart_raster_host(x, hf, capi.plot_transform(he, capi.PLOT_W, capi.PLOT_H))
    out["host_mirror_s"] = round(time.perf_counter() - t0, 3)
    out["host_threads"] = os.cpu_count()
    out["identical_to_host"] = bool(np.array_equal(hf, first) and np.array_equal(hy, yext) and np.array_equal(himg, img))
    # the page's tokens: capped values through the device formatter, 16 M cells per call
    flat = np.minimum(x.reshape(-1)[: min(x.size, 8 << 24)], 2.5)
    t0 = time.perf_counter()
    for a in range(0, flat.size, 1 << 24):
        ctx.format_f2(flat[a:a + (1 << 24)])
    t = time.perf_counter() - t0
    out["tokens"] = {"cells": int(flat.size), "s": round(t, 3), "cells_per_s": round(flat.size / t)}
    return out


def write_inputs(tmp, S, rng):
    """a FASTA of chr1 + chr2 (one-line records, isochores of GC) and their depthwed -s 1000 matrix"""
    fa_path, fai, off = os.path.join(tmp, "ref.fa"), "", 0
    lut = np.frombuffer(b"ACGTGCAT", np.uint8)
    with open(fa_path, "wb") as f:
        for name, L in CONTIGS:
            base = rng.integers(0, 4, L, dtype=np.uint8)
            bias = np.repeat(rng.integers(0, 3, L // 100_000 + 1, dtype=np.uint8), 100_000)[:L]
            seq = lut[np.where((bias == 1) & (base >= 2), base + 2, np.where((bias == 2) & (base < 2), base + 6, base)) & 7]
            head = b">" + name.encode() + b"\n"
            f.write(head)
            f.write(seq.tobytes() + b"\n")
            off += len(head)
            fai += "%s\t%d\t%d\t%d\t%d\n" % (name, L, off, L, L + 1)
            off += L + 1
    open(fa_path + ".fai", "w").write(fai)
    digits = np.frombuffer(b"".join(b"\t%d" % v for v in range(10, 100)), np.uint8).reshape(90, 3)
    mpath, n = os.path.join(tmp, "m.tsv"), 0
    with open(mpath, "wb") as f:
        f.write(b"#chrom\tstart\tend\t" + b"\t".join(b"s%d" % i for i in range(S)) + b"\n")
        for name, L in CONTIGS:
            a = np.arange(0, L, 1000, dtype=np.int64)
            body = digits[rng.integers(10, 100, (a.size, S)) - 10].reshape(a.size, 3 * S)
            f.write(b"".join(b"%s\t%d\t%d" % (name.encode(), s, min(s + 1000, L)) + body[i].tobytes() + b"\n" for i, s in enumerate(a)))
            n += a.size
    return fa_path, mpath, n


def cli_run(tmp, fa_path, mpath, *flags):
    run_dir = tempfile.mkdtemp(dir=tmp)
    t0 = time.perf_counter()
    p = subprocess.run([os.path.join(ROOT, "bin", "goleft"), "dcnv", *flags, mpath, fa_path], capture_output=True, cwd=run_dir,
                       env=dict(os.environ, GL_TIMING="1"))
    wall = time.perf_counter() - t0
    if p.returncode != 0:
        raise SystemExit("goleft dcnv failed: %s" % p.stderr.decode())
    phases = {}
    for ln in p.stderr.decode().splitlines():
        if ln.startswith("[dcnv timing]"):
            phases[ln[len("[dcnv timing]"):].rsplit(None, 2)[0].strip()] = float(ln.split()[-2])
    files = {f: os.path.getsize(os.path.join(run_dir, f)) for f in os.listdir(run_dir)}
    bed = open(os.path.join(run_dir, "depth.bed"), "rb").read()
    for f in os.listdir(run_dir):
        os.remove(os.path.join(run_dir, f))
    return {"wall_s": round(wall, 3), "phases_s": phases, "files": files}, bed


def cli_leg(S, rng, tmp):
    fa_path, mpath, n = write_inputs(tmp, S, rng)
    plain, bed0 = cli_run(tmp, fa_path, mpath, "--noplots")
    charts, bed1 = cli_run(tmp, fa_path, mpath)
    page = sum(v for k, v in charts["files"].items() if k.endswith(".html"))
    chart_s = charts["phases_s"].get("chart", float("nan"))
    return {"rows": n, "samples": S, "noplots": plain, "charts": charts, "depth_bed_identical": bed0 == bed1, "page_bytes": page,
            "page_bytes_per_s_of_chart_phase": round(page / chart_s) if chart_s > 0 else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=3_088_281)
    ap.add_argument("--samples", type=int, default=128)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cli-samples", type=int, default=128)
    args = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_dcnv_chart.py: no CUDA device; goleft_b200 has no CPU fallback")
    rng = np.random.default_rng(2026)
    out = {"card": card()}
    with capi.Ctx(0) as ctx:
        out["library"] = library_leg(ctx, args.rows, args.samples, args.reps, rng)
    print(json.dumps(out["library"]), file=sys.stderr, flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        out["cli"] = cli_leg(args.cli_samples, rng, tmp)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
