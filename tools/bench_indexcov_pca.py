#!/usr/bin/env python
"""indexcov's PCA (the .ped's PC1..PC5) on one H100: the 2504-sample cohort over a GRCh38-shaped autosomal byte matrix
(every chr1..chr22 16 KB tile, plus the zero column each reference ends with: ~176 k columns), planted bytes (uniform noise
with zero stretches shared by three sample groups).

    python tools/bench_indexcov_pca.py [--samples 2504] [--cli-samples 313]

Library: gl_indexcov_pca from host bytes to projections, split into upload, Gram + centring and eigen (host clock, with the
syncs the call has anyway), and the Gram kernel alone (CUDA events): its int8 rate S(S+1)D / t against the data sheet's
1,979 dense int8 TOPS.  Checks: one 64-row block of the Gram against numpy, and the projections against numpy's eigh of the
exact centred Gram.  CLI: tools/bench_indexcov_cli.py's cohort with GL_TIMING, whose phases include `pca`.  Prints one JSON
object with the card name and power limit read in the same run.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_dcnv import GRCH38, card  # noqa: E402
from goleft_b200 import capi  # noqa: E402

TILE = 16384


def planted(rng, S, D):
    x = rng.integers(0, 256, (S, D), dtype=np.uint8)
    for g, (a, b) in enumerate([(0, S // 4), (S // 4, S // 2), (S // 2, S // 2 + S // 8)]):
        c0 = int(rng.integers(0, D // 2))
        x[a:b, c0:c0 + D // (8 + 4 * g)] = 0
    return x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=2504)
    ap.add_argument("--cli-samples", type=int, default=313)
    a = ap.parse_args()
    S = a.samples
    D = sum(L // TILE + 1 + 1 for c, L in GRCH38 if c not in ("chrX", "chrY"))
    rng = np.random.default_rng(3)
    x = planted(rng, S, D)
    out = {"samples": S, "columns": D, "card": card()}
    with capi.Ctx(0) as ctx:
        ctx.indexcov_pca(x[:64, :4096])                                  # warm-up: module load, first allocations
        ctx.profile_enable(True)
        t = time.perf_counter()
        proj, sv, k, gram = ctx.indexcov_pca(x, want_gram=True)
        out["library_s_with_gram_copy"] = time.perf_counter() - t
        ctx.profile_read()
        t = time.perf_counter()
        proj2, sv2, _, _ = ctx.indexcov_pca(x)
        out["library_s"] = time.perf_counter() - t
        out["phases_s"] = ctx.indexcov_pca_phases()
        gk = [ms for nm, ms in ctx.profile_read() if nm == "gram_kernel"]
        ctx.profile_enable(False)
    out["gram_kernel_ms"] = gk
    out["gram_int8_tops"] = S * (S + 1) * D / (gk[0] * 1e-3) / 1e12 if gk else None
    out["gram_int8_tops_of_1979"] = out["gram_int8_tops"] / 1979 if gk else None
    out["repeat_identical"] = bool(np.array_equal(proj, proj2) and np.array_equal(sv, sv2))
    blk = np.zeros((64, S))                                              # block check: 64 rows x all samples, in float64
    for c0 in range(0, D, 8192):                                         # chunks: every partial sum is an integer < 2^53
        blk += x[:64, c0:c0 + 8192].astype(np.float64) @ x[:, c0:c0 + 8192].astype(np.float64).T
    out["gram_block_exact"] = bool(np.array_equal(gram[:64], blk.astype(np.int64)))
    r = gram.sum(axis=1)                                                 # exact centred Gram: every term fits in int64 here
    q = int(r.sum())
    n2gc = S * S * gram - S * (r[:, None] + r[None, :]) + q
    gc = n2gc.astype(np.float64) / float(S * S)
    t = time.perf_counter()
    lam, V = np.linalg.eigh(gc)
    out["numpy_eigh_s"] = time.perf_counter() - t
    lam, V = lam[::-1][:k], V[:, ::-1][:, :k]
    c = (S * r - q).astype(np.float64) / float(S * S)
    worst = 0.0
    for j in range(k):
        u = V[:, j] * (1 if V[np.argmax(np.abs(V[:, j])), j] > 0 else -1)
        sig = np.sqrt(lam[j])
        ref = sig * u + (c @ u) / sig
        worst = max(worst, float(np.abs(ref - proj[:, j]).max() / np.abs(ref).max()))
    out["proj_vs_eigh_max_rel"] = worst
    out["sv"] = sv.tolist()
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_indexcov_cli.py"), "--samples", str(a.cli_samples)],
                       capture_output=True, text=True)
    try:
        cli = json.loads(p.stdout.strip().splitlines()[-1])
        out["cli"] = {k2: cli.get(k2) for k2 in ("samples", "cli_wall_s", "phases", "error")}
    except Exception:
        out["cli"] = {"error": p.stderr[-500:]}
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
