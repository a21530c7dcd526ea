#!/usr/bin/env python
"""`goleft dcnv` on one H100: a GRCh38-shaped cohort matrix at `depthwed -s 1000` (3.09 M rows x 128 samples by default),
seeded, with GC taken from a synthetic FASTA of the same shape.

    python tools/bench_dcnv.py [--samples 128] [--check-cols 4] [--cli-contigs 2]

Library leg, from host arrays to "%.2f" tokens, each phase timed with a host clock around synchronising calls: the host
argsort (gl_go_argsort_f64), GC (gl_fasta_load + gl_fasta_stats per contig), the device debias + normalisation
(gl_dcnv_normalize, copies included) and the device tokens (gl_format_f2, 16 M cells per call).  The normalised values and
tokens of --check-cols sample columns are compared with the oracle at full n (columns are independent, so the subset check
is exact).  CLI leg: `goleft dcnv` end to end (GL_TIMING phases) on the rows of the first --cli-contigs contigs written as
text, its depth.bed compared byte for byte with the oracle.  Prints one JSON object with the card name and power limit.
Writes nothing to the tree (temporary files go to a temporary directory)."""
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
from goleft_b200 import capi  # noqa: E402
from oracle import dcnv as od  # noqa: E402   (the checker, never the thing measured)
from oracle import loader as orc  # noqa: E402

GRCH38 = [("chr1", 248956422), ("chr2", 242193529), ("chr3", 198295559), ("chr4", 190214555), ("chr5", 181538259),
          ("chr6", 170805979), ("chr7", 159345973), ("chr8", 145138636), ("chr9", 138394717), ("chr10", 133797422),
          ("chr11", 135086622), ("chr12", 133275309), ("chr13", 114364328), ("chr14", 107043718), ("chr15", 101991189),
          ("chr16", 90338345), ("chr17", 83257441), ("chr18", 80373285), ("chr19", 58617616), ("chr20", 64444167),
          ("chr21", 46709983), ("chr22", 50818468), ("chrX", 156040895), ("chrY", 57227415)]
SIZE = 1000


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
        name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
        return {"name": name, "power_limit": power}
    except Exception as e:                                              # the numbers are still reported; say why the card is not
        return {"name": "unknown (%s)" % e, "power_limit": "unknown"}


def genome(rng):
    """per contig: one-line record bytes (A/C/G/T with GC-rich and AT-rich stretches) + "\n" """
    out = []
    lut = np.frombuffer(b"ACGTGCAT", np.uint8)
    for name, L in GRCH38:
        base = rng.integers(0, 4, L, dtype=np.uint8)
        bias = np.repeat(rng.integers(0, 3, L // 100_000 + 1, dtype=np.uint8), 100_000)[:L]   # 100 kb isochores
        seq = lut[np.where((bias == 1) & (base >= 2), base + 2, np.where((bias == 2) & (base < 2), base + 6, base)) & 7]
        out.append((name, L, np.concatenate([seq, np.frombuffer(b"\n", np.uint8)])))
    return out


def rows_of(contigs):
    """depthwed -s 1000 rows: [a, a + 1000) up to the contig end"""
    c, s, e = [], [], []
    for k, (name, L, _) in enumerate(contigs):
        a = np.arange(0, L, SIZE, dtype=np.int64)
        c.append(np.full(a.size, k, np.int32)); s.append(a); e.append(np.minimum(a + SIZE, L))
    return np.concatenate(c), np.concatenate(s), np.concatenate(e)


def gc_library(ctx, contigs, cid, starts, ends):
    """Faidx.Stats(chrom, max(s, 250) - 250, e).GC of every row: one load + one stats call per contig"""
    gc = np.zeros(starts.size)
    for k, (_, L, rec) in enumerate(contigs):
        m = cid == k
        a = np.maximum(starts[m], 250) - 250
        ctx.fasta_load(rec)
        _, st = ctx.fasta_stats(a, ends[m] + 1)            # one-line records: position(p) = p; the slice runs one byte past the end
        gc[m] = st[:, 0]
    return gc


def library_leg(ctx, contigs, S, check_cols, rng):
    cid, starts, ends = rows_of(contigs)
    n = starts.size
    x = rng.poisson(30.0, (n, S)).astype(np.float64)
    x[rng.random((n, S)) < 0.002] = 0
    t = {}
    t0 = time.perf_counter()
    gc = gc_library(ctx, contigs, cid, starts, ends)
    t["gc"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    inds = capi.go_argsort(gc)
    t["argsort"] = time.perf_counter() - t0
    t0 = time.perf_counter()
    out, med = ctx.dcnv_normalize(x, inds)
    t["normalize"] = time.perf_counter() - t0
    cols = np.linspace(0, S - 1, check_cols).astype(int)
    t0 = time.perf_counter()
    flat = out.reshape(-1)
    chunk = 1 << 24
    keep = []
    for a in range(0, flat.size, chunk):
        tok = ctx.format_f2(flat[a:a + chunk])
        r0, r1 = a // S, (a + tok.shape[0]) // S
        keep.append(tok.reshape(r1 - r0, S, 16)[:, cols])
    t["tokens"] = time.perf_counter() - t0
    toks = np.concatenate(keep)
    # oracle: the checked columns at full n
    want, want_inds, want_med = od.matrix(x[:, cols], gc)
    same_vals = bool(np.array_equal(out[:, cols].view(np.uint64), want.view(np.uint64)) and np.array_equal(inds, want_inds)
                     and np.array_equal(med[cols], want_med))
    bad, _ = od.f2_mismatches(want.reshape(-1), toks.reshape(-1, 16))
    cells = n * S
    return {"rows": int(n), "samples": S, "cells": int(cells), "distinct_gc": int(np.unique(gc).size),
            "s": {k: round(v, 4) for k, v in t.items()}, "total_s": round(sum(t.values()), 4),
            "cells_per_s_device_normalize": cells / t["normalize"],
            "oracle_check": {"columns": cols.tolist(), "values_identical": same_vals, "token_mismatches": bad}}


def cli_leg(contigs, S, rng, tmp):
    sub = contigs
    fa_path = os.path.join(tmp, "ref.fa")
    fai = ""
    with open(fa_path, "wb") as f:
        off = 0
        for name, L, rec in sub:
            head = b">" + name.encode() + b"\n"
            f.write(head); f.write(rec.tobytes())
            off += len(head)
            fai += "%s\t%d\t%d\t%d\t%d\n" % (name, L, off, L, L + 1)
            off += rec.size
    open(fa_path + ".fai", "w").write(fai)
    cid, starts, ends = rows_of(sub)
    n = starts.size
    x = rng.integers(10, 100, (n, S))
    digits = np.frombuffer(b"".join(b"\t%d" % v for v in range(10, 100)), np.uint8).reshape(90, 3)
    body = digits[x - 10].reshape(n, 3 * S)
    names = [c[0].encode() for c in sub]
    lines = [b"#chrom\tstart\tend\t" + b"\t".join(b"s%d" % i for i in range(S)) + b"\n"]
    for i in range(n):
        lines.append(b"%s\t%d\t%d" % (names[cid[i]], starts[i], ends[i]) + body[i].tobytes() + b"\n")
    text = b"".join(lines)
    del lines
    mpath = os.path.join(tmp, "m.tsv")
    open(mpath, "wb").write(text)
    t0 = time.perf_counter()
    p = subprocess.run([os.path.join(ROOT, "bin", "goleft"), "dcnv", mpath, fa_path], capture_output=True, cwd=tmp,
                       env=dict(os.environ, GL_TIMING="1"))
    wall = time.perf_counter() - t0
    if p.returncode != 0:
        raise SystemExit("goleft dcnv failed: %s" % p.stderr.decode())
    phases = {}
    for ln in p.stderr.decode().splitlines():
        if ln.startswith("[dcnv timing]"):
            k, v = ln[len("[dcnv timing]"):].rsplit(None, 2)[0].strip(), float(ln.split()[-2])
            phases[k] = v
    got = open(os.path.join(tmp, "depth.bed"), "rb").read()
    # oracle: GC through orc.faidx_stats row by row, then the C restatement of main
    fa = open(fa_path, "rb").read()
    recs = od.parse_fai(fai)
    gc = np.empty(n)
    for i in range(n):
        s = max(int(starts[i]), 250)
        gc[i] = orc.faidx_stats(fa, recs[sub[cid[i]][0]], s - 250, int(ends[i]))[0]
    want, _, _ = od.matrix(x.astype(np.float64), gc)
    label = names[cid[1]]
    exp = text[:text.index(b"\n") + 1] + od.rows(label, np.maximum(starts, 250), ends, want)
    return {"rows": int(n), "samples": S, "text_bytes": len(text), "wall_s": round(wall, 3), "phases_s": phases,
            "oracle_check": {"identical": got == exp, "bytes": len(got)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=128)
    ap.add_argument("--check-cols", type=int, default=4)
    ap.add_argument("--cli-contigs", type=int, default=2)
    ap.add_argument("--cli-samples", type=int, default=128)
    args = ap.parse_args()
    if capi.device_count() < 1:
        raise SystemExit("bench_dcnv.py: no CUDA device; goleft_b200 has no CPU fallback")
    rng = np.random.default_rng(2026)
    contigs = genome(rng)
    out = {"card": card()}
    with capi.Ctx(0) as ctx:
        out["library"] = library_leg(ctx, contigs, args.samples, args.check_cols, rng)
    print(json.dumps(out["library"]), file=sys.stderr, flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        out["cli"] = cli_leg(contigs[:args.cli_contigs], args.cli_samples, rng, tmp)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
