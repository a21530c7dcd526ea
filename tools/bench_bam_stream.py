#!/usr/bin/env python
"""The host BAM reader's whole-file and header-only paths, end to end on the synthetic 30x chr20 BAM + BAI that bench.py
writes (tools/synth/bamsynth.c).  bench.py times none of them:
  decode      gl_bam_decode_segments on every pool thread (BamFile::stream)
  depth       `goleft depth` on a copy without its .bai: the whole file is decoded, then the GPU makes the BED files
  multidepth  `goleft multidepth -c chr20` over 4 copies without a .bai: each is decoded on a helper thread beside the GPU
              work of the previous one
  covstats    `goleft covstats -n 1000000`
  indexcov    the `read indexes` phase of `GL_TIMING=1 goleft indexcov` over 64 symlinked BAM + BAI copies
Every leg records its wall clock and a digest of what it wrote.  With several --root trees (builds of this repository,
e.g. two commits) the legs run tree after tree, --reps times over, on the same BAM; the JSON line gives each tree's median
per leg and whether every run of every tree wrote the same outputs.

    python tools/bench_bam_stream.py                                  # this tree, once
    python tools/bench_bam_stream.py --root /path/a --root /path/b --reps 3
"""
import argparse
import glob
import hashlib
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))

# the decode leg runs in a child process so that each tree's library is the one loaded
DECODE = r"""
import ctypes as C, hashlib, json, sys, time
import numpy as np
from goleft_b200 import capi
bam = sys.argv[1]
threads = capi.lib.glhost_pool_size()
t0 = time.perf_counter()
r = capi.bam_segments(bam, 1, threads)
wall = time.perf_counter() - t0
h = hashlib.sha256(json.dumps([r["refs"], r["n_records"], r["n_pass"]]).encode())
for tid in sorted(r["segments"]):
    s, e = r["segments"][tid]
    h.update(np.int64(tid).tobytes()); h.update(s.tobytes()); h.update(e.tobytes())
print(json.dumps({"wall_s": wall, "threads": threads, "records": r["n_records"], "digest": h.hexdigest()}))
"""


def digest_files(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(os.path.basename(p).encode())
        h.update(open(p, "rb").read())
    return h.hexdigest()


def run(cmd, env=None):
    t0 = time.perf_counter()
    p = subprocess.run(cmd, capture_output=True, env=dict(os.environ, **(env or {})))
    wall = time.perf_counter() - t0
    if p.returncode != 0:
        raise RuntimeError("%s: exit %d: %s" % (" ".join(cmd[:2]), p.returncode, p.stderr.decode()[-400:]))
    return wall, p


def one_pass(root, work, out):
    """every leg once with the tree at `root`; outputs under `out` -> {leg: {"wall_s", "digest", ...}}"""
    exe = os.path.join(root, "bin", "goleft")
    bam = os.path.join(work, "chr20.bam")
    res = {}
    os.makedirs(out, exist_ok=True)

    env = {"GOLEFT_B200_LIB": os.path.join(root, "goleft_b200", "libgoleft_b200.so"), "PYTHONPATH": ROOT}
    _, p = run([sys.executable, "-c", DECODE, bam], env)
    res["decode"] = json.loads(p.stdout.decode().strip().splitlines()[-1])

    wall, _ = run([exe, "depth", "--prefix", os.path.join(out, "d"), "-r", os.path.join(work, "ref.fa"), os.path.join(work, "nobai", "a.bam")])
    res["depth"] = {"wall_s": wall, "digest": digest_files(glob.glob(os.path.join(out, "d.*.bed")))}

    wall, p = run([exe, "multidepth", "-c", "chr20"] + [os.path.join(work, "nobai", x + ".bam") for x in "abcd"])
    res["multidepth"] = {"wall_s": wall, "digest": hashlib.sha256(p.stdout).hexdigest()}

    wall, p = run([exe, "covstats", "-n", "1000000", bam])
    res["covstats"] = {"wall_s": wall, "digest": hashlib.sha256(p.stdout).hexdigest(), "row": p.stdout.decode().splitlines()[-1]}

    ic = os.path.join(out, "ic")
    wall, p = run([exe, "indexcov", "-d", ic] + sorted(glob.glob(os.path.join(work, "ic", "*.bam"))), {"GL_TIMING": "1"})
    phase = [ln for ln in p.stderr.decode().splitlines() if ln.startswith("[indexcov timing]") and "read indexes" in ln]
    res["indexcov"] = {"wall_s": wall, "read_indexes_s": float(phase[0].split()[-2]),
                       "digest": digest_files(f for f in glob.glob(os.path.join(ic, "*")) if os.path.isfile(f))}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", action="append", help="a built tree of this repository (repeatable; default: this one)")
    ap.add_argument("--reps", type=int, default=1)
    ap.add_argument("--keep", action="store_true")
    args = ap.parse_args()
    roots = [os.path.abspath(r) for r in (args.root or [ROOT])]
    import glsynth
    work = tempfile.mkdtemp(prefix="glbamstream_")
    try:
        bam = os.path.join(work, "chr20.bam")
        t0 = time.perf_counter()
        glsynth.write_bam(bam, [("chr20", glsynth.CHR20_LEN, 19)])
        t_write = time.perf_counter() - t0
        open(os.path.join(work, "ref.fa.fai"), "w").write("chr20\t%d\t6\t60\t61\n" % glsynth.CHR20_LEN)
        for d in ("nobai", "ic"):
            os.makedirs(os.path.join(work, d))
        for x in "abcd":
            os.symlink(bam, os.path.join(work, "nobai", x + ".bam"))
        for k in range(64):
            os.symlink(bam, os.path.join(work, "ic", "s%02d.bam" % k))
            os.symlink(bam + ".bai", os.path.join(work, "ic", "s%02d.bam.bai" % k))
        runs = {r: [] for r in roots}
        for rep in range(args.reps):
            for i, r in enumerate(roots):
                runs[r].append(one_pass(r, work, os.path.join(work, "out%d_%d" % (i, rep))))
        legs = list(runs[roots[0]][0])
        digests = {leg: {x[leg]["digest"] for r in roots for x in runs[r]} for leg in legs}
        res = {"bam_bytes": os.path.getsize(bam), "bam_write_s": t_write, "reps": args.reps, "host_threads": os.cpu_count(),
               "outputs_identical": {leg: len(d) == 1 for leg, d in digests.items()},
               "median_s": {r: {leg: statistics.median(x[leg]["wall_s"] for x in runs[r]) for leg in legs} for r in roots},
               "median_read_indexes_s": {r: statistics.median(x["indexcov"]["read_indexes_s"] for x in runs[r]) for r in roots},
               "runs": runs}
        try:
            res["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                                        text=True).stdout.strip().splitlines()[0]
        except (OSError, IndexError):
            res["gpu"] = None
        print(json.dumps(res))
    finally:
        if not args.keep:
            shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
