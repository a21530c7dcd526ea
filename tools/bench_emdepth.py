#!/usr/bin/env python
"""`goleft emdepth` on one H100: the `tools/bench_dcnv.py` shape (GRCh38 at `depthwed -s 1000`, 3.09 M rows x 128 samples by
default), seeded, normalised depths around 1 with planted CN1 / CN3 runs.

    python tools/bench_emdepth.py [--samples 128] [--rows 0] [--check-rows 20000] [--cli-rows 100000]

Kernel: gl_emdepth_device on a resident matrix, timed with CUDA events (gl_timer_*).  Library: gl_emdepth from host arrays,
copies included, host clock.  Oracle: the single-threaded C restatement on the first --check-rows rows, timed, and its cells
and centres compared with the library's bit for bit.  CLI: `goleft emdepth` on --cli-rows rows written as text, GL_TIMING
phases and wall time, its two files compared with the oracle's on the first rows.  Prints one JSON object with the card name
and power limit read in the same run.  Writes nothing to the tree (temporary files go to a temporary directory)."""
import argparse
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
from bench_dcnv import GRCH38, SIZE, card  # noqa: E402
from goleft_b200 import capi  # noqa: E402
from oracle import emdepth as oe  # noqa: E402   (the checker, never the thing measured)


def matrix(rng, n, S):
    x = rng.gamma(40.0, 1 / 40.0, (n, S)) * rng.gamma(20.0, 1 / 20.0, (n, 1))
    for _ in range(max(1, n // 2000)):                                 # planted runs of 5..60 rows in one sample
        r0, ln, s = int(rng.integers(0, n - 60)), int(rng.integers(5, 60)), int(rng.integers(0, S))
        x[r0:r0 + ln, s] *= rng.choice([0.5, 1.5])
    return np.round(x, 2).astype(np.float32)                            # what dcnv writes, read back as float32


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=128)
    ap.add_argument("--rows", type=int, default=0, help="0: the GRCh38 row count at -s 1000")
    ap.add_argument("--check-rows", type=int, default=20000)
    ap.add_argument("--cli-rows", type=int, default=100000)
    a = ap.parse_args()
    S = a.samples
    n = a.rows or sum((L + SIZE - 1) // SIZE for _, L in GRCH38)
    rng = np.random.default_rng(12)
    x = matrix(rng, n, S)
    out = {"rows": n, "samples": S, "card": card()}
    with capi.Ctx(0) as ctx:
        d_x, d_c = ctx.dev_array(x), ctx.dev_empty(n * S)
        ctx.emdepth_device(d_x, n, S, S, d_c)                           # warm-up
        ms = []
        for _ in range(3):
            ctx.timer_start()
            ctx.emdepth_device(d_x, n, S, S, d_c)
            ms.append(ctx.timer_stop_ms())
        out["kernel_ms"] = ms
        out["kernel_stats"] = ctx.emdepth_stats()
        d_x.free(); d_c.free()
        t = time.perf_counter()
        cells, lam = ctx.emdepth(x)
        out["library_s"] = time.perf_counter() - t
        out["library_stats"] = ctx.emdepth_stats()
    k = min(a.check_rows, n)
    t = time.perf_counter()
    oc, ol, _ = oe.emdepth(x[:k])
    out["oracle_rows"], out["oracle_s"] = k, time.perf_counter() - t
    out["oracle_match"] = bool(np.array_equal(oc, cells[:k]) and np.array_equal(ol.view(np.uint64), lam[:k].view(np.uint64)))
    m = min(a.cli_rows, n)
    rows = []
    for c, L in GRCH38:
        for s in range(0, L, SIZE):
            rows.append((c, s, min(s + SIZE, L)))
            if len(rows) == m:
                break
        if len(rows) == m:
            break
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "m.tsv")
        with open(path, "wb") as f:
            f.write(b"#chrom\tstart\tend\t" + b"\t".join(b"s%d" % i for i in range(S)) + b"\n")
            for (c, s, e), v in zip(rows, x[:m]):
                f.write(b"%s\t%d\t%d\t" % (c.encode(), s, e) + b"\t".join(b"%.2f" % float(t) for t in v) + b"\n")
        t = time.perf_counter()
        p = subprocess.run([os.path.join(ROOT, "bin", "goleft"), "emdepth", "--prefix", os.path.join(tmp, "o"), path],
                           capture_output=True, env=dict(os.environ, GL_TIMING="1"))
        out["cli_rows"], out["cli_wall_s"] = m, time.perf_counter() - t
        out["cli_rc"] = p.returncode
        out["cli_timing"] = [ln for ln in p.stderr.decode().splitlines() if "timing" in ln]
        cn_bed = open(os.path.join(tmp, "o.cn.bed"), "rb").read() if p.returncode == 0 else b""
        out["cli_cnvs"] = open(os.path.join(tmp, "o.cnv.bed"), "rb").read().count(b"\n") - 1 if p.returncode == 0 else -1
        head = b"".join(open(path, "rb").readlines()[:2001])
        want_cn, _ = oe.files(head)
        out["cli_cn_bed_head_match"] = cn_bed.startswith(want_cn)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
