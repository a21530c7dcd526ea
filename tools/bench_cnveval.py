#!/usr/bin/env python
"""`goleft cnveval` on one H100: a seeded 1000-Genomes-shaped cohort (2504 samples, 50,000 truth sites on 22 chromosomes,
carrier counts from a skewed allele-frequency distribution, 100-500 calls per sample: 80 % from carried sites with
jittered ends, one in ten with a wrong CN, the rest false calls).

    python tools/bench_cnveval.py [--samples 2504] [--truths 50000] [--oracle-samples 32] [--reps 10]

Library: gl_cnveval from host arrays to stats (host ordering, upload, kernels, download; it ends in a synchronise), host
clock.  Kernels: gl_cnveval_device on the resident layout, CUDA events (gl_timer_*) over --reps calls after two warm-up
calls, plus the per-phase event times of one call.  Oracle: the single-threaded C restatement of the reference's walk on the
first --oracle-samples samples (each sample's counts depend only on its calls and memberships), timed, its stats compared
with the library's rows.  Prints one JSON object with the card name and power limit read in the same run."""
import argparse
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
from oracle import cnveval as oc  # noqa: E402   (the checker, never the thing measured)


def cohort(rng, S, T):
    t_chrom = rng.integers(0, 22, T).astype(np.int32)
    t_start = rng.integers(0, 150_000_000, T) // 100 * 100
    t_end = t_start + np.exp(rng.uniform(np.log(1000), np.log(1_000_000), T)).astype(np.int64)
    t_cn = rng.choice([0, 1, 3, 4], T, p=[0.2, 0.5, 0.2, 0.1]).astype(np.int64)
    k = np.maximum(1, (rng.random(T) ** 8 * S).astype(np.int64))       # most sites rare, a few common
    mem_ptr = np.concatenate([[0], np.cumsum(k)]).astype(np.int64)
    mem_sample = np.concatenate([rng.choice(S, int(x), replace=False) for x in k]).astype(np.int32)
    owner = np.repeat(np.arange(T), k)
    by = np.argsort(mem_sample, kind="stable")
    ptr = np.searchsorted(mem_sample[by], np.arange(S + 1))
    cs, ci = [], []
    n_false = 0
    for s in range(S):
        n = int(rng.integers(100, 501))
        mine = owner[by[ptr[s]:ptr[s + 1]]]
        take = rng.choice(mine, min(mine.size, int(0.8 * n)), replace=False)
        cs.append(np.full(take.size, s, np.int32)); ci.append(take)
        n_false += n - take.size
    cs, ci = np.concatenate(cs), np.concatenate(ci)
    L = t_end[ci] - t_start[ci]
    c_start = np.maximum(0, t_start[ci] + (rng.normal(0, 0.1, ci.size) * L).astype(np.int64) // 100 * 100)
    c_end = np.maximum(c_start, t_end[ci] + (rng.normal(0, 0.1, ci.size) * L).astype(np.int64))
    c_cn = np.where(rng.random(ci.size) < 0.1, rng.choice([1, 3], ci.size), t_cn[ci])
    f_start = rng.integers(0, 150_000_000, n_false) // 100 * 100
    c_sample = np.concatenate([cs, rng.integers(0, S, n_false).astype(np.int32)])
    c_chrom = np.concatenate([t_chrom[ci], rng.integers(0, 22, n_false).astype(np.int32)])
    c_start = np.concatenate([c_start, f_start])
    c_end = np.concatenate([c_end, f_start + np.exp(rng.uniform(np.log(1000), np.log(500_000), n_false)).astype(np.int64)])
    c_cn = np.concatenate([c_cn, rng.choice([1, 3], n_false)]).astype(np.int64)
    o = rng.permutation(c_sample.size)                                  # file order is not sample order
    return (c_sample[o], c_chrom[o], c_start[o], c_end[o], c_cn[o], t_chrom, t_start, t_end, t_cn, mem_ptr, mem_sample)


def layout(S, cs, cc, cb, ce, ccn, tc, tb, te, tcn, mp, ms):
    """the resident layout gl_cnveval_device takes (include/goleft_b200.h)"""
    by = np.argsort(cs, kind="stable")
    c_ptr = np.searchsorted(cs[by], np.arange(S + 1)).astype(np.int64)
    order = np.concatenate([by[c_ptr[s]:c_ptr[s + 1]][capi.cnveval_order(cc[by[c_ptr[s]:c_ptr[s + 1]]], cb[by[c_ptr[s]:c_ptr[s + 1]]])]
                            for s in range(S)])
    to = np.lexsort((tb, tc))
    rank = np.empty(tc.size, np.int64)
    rank[to] = np.arange(tc.size)
    mt = rank[np.repeat(np.arange(tc.size), np.diff(mp))]
    mo = np.lexsort((mt, ms))
    m_ptr = np.searchsorted(ms[mo], np.arange(S + 1)).astype(np.int64)
    return (c_ptr, cc[order], cb[order], ce[order], ccn[order], tc[to], tb[to], te[to], tcn[to], m_ptr, mt[mo])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=2504)
    ap.add_argument("--truths", type=int, default=50000)
    ap.add_argument("--oracle-samples", type=int, default=32)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    S, T = a.samples, a.truths
    rng = np.random.default_rng(2504)
    arrays = cohort(rng, S, T)
    out = {"samples": S, "truths": T, "calls": int(arrays[0].size), "memberships": int(arrays[10].size), "card": card()}
    with capi.Ctx(0) as ctx:
        st = ctx.cnveval(S, *arrays, po=0.4)                           # warm-up
        wall = []
        for _ in range(3):
            t0 = time.perf_counter()
            st = ctx.cnveval(S, *arrays, po=0.4)
            wall.append(time.perf_counter() - t0)
        out["library_wall_s"] = wall
        lay = layout(S, *arrays)
        d = [ctx.dev_array(x) for x in lay]
        d_st = ctx.dev_empty(S * 12 * 8)
        n_calls, n_mem = int(lay[1].size), int(lay[10].size)

        def dev():
            ctx.cnveval_device(S, d[0], n_calls, d[1], d[2], d[3], d[4], T, d[5], d[6], d[7], d[8], d[9], n_mem, d[10], 0.4, d_st)
        dev(); dev()
        ctx.timer_start()
        for _ in range(a.reps):
            dev()
        out["kernels_ms_per_call"] = ctx.timer_stop_ms() / a.reps
        ctx.profile_enable(True)
        dev()
        ctx.sync()
        out["phases_ms"] = ctx.profile_read()
        ctx.profile_enable(False)
        out["device_equals_host"] = bool(np.array_equal(d_st.download(np.uint64, S * 12).reshape(S, 3, 4), st))
        for x in d + [d_st]:
            x.free()
    k = min(a.oracle_samples, S)
    cs, cc, cb, ce, ccn, tc, tb, te, tcn, mp, ms = arrays
    keep = cs < k
    own = np.repeat(np.arange(T), np.diff(mp))
    mk = ms < k
    mp_k = np.concatenate([[0], np.cumsum(np.bincount(own[mk], minlength=T))])
    t0 = time.perf_counter()
    want = oc.evaluate_arrays(k, cs[keep], cc[keep], cb[keep], ce[keep], ccn[keep], tc, tb, te, tcn, mp_k, ms[mk], 0.4)
    o_s = time.perf_counter() - t0
    out["oracle_samples"] = k
    out["oracle_s"] = o_s
    out["oracle_s_per_sample"] = o_s / k
    out["oracle_equals_library"] = bool(np.array_equal(want, st[:k]))
    tab = oc.tabulate(st)
    out["all"] = {"TP": int(tab[3, 0]), "FP": int(tab[3, 1]), "FN": int(tab[3, 2]), "TN": int(tab[3, 3])}
    print(json.dumps(out))
    return 0 if out["oracle_equals_library"] and out["device_equals_host"] else 1


if __name__ == "__main__":
    sys.exit(main())
