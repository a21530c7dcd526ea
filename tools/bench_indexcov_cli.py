#!/usr/bin/env python
"""`bin/goleft indexcov` end to end on a synthetic 1000G-shaped cohort of .bai files (BASELINE configs[3]): S indexes of an
hs37d5-shaped reference (86 sequences, ~189k 16 KB tiles), written here with numpy, then the product CLI:
read S indexes -> I1..I5 on the GPU -> %.3g tokens on the GPU -> rows on all host threads -> BGZF.  Prints one JSON object.

    python tools/bench_indexcov_cli.py --samples 313          # one GPU's share of the 2504-sample cohort
    python tools/bench_indexcov_cli.py --samples 313 --extranorm   # the same with -n (I7)
"""
import argparse
import json
import os
import shutil
import struct
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

HS37D5 = [249250621, 243199373, 198022430, 191154276, 180915260, 171115067, 159138663, 146364022, 141213431, 135534747, 135006516,
          133851895, 115169878, 107349540, 102531392, 90354753, 81195210, 78077248, 59128983, 63025520, 48129895, 51304566,
          155270560, 59373566, 16569] + [int(x) for x in np.linspace(4262, 547496, 59)] + [171823, 35477943]


def write_bai(path, rng, scale):
    parts = [b"BAI\x01", struct.pack("<i", len(HS37D5))]
    at = 1 << 16
    for L in HS37D5:
        n = L // 16384 + 1
        step = np.maximum(1, np.round(rng.lognormal(np.log(2.1e5 * scale), 0.25, n))).astype(np.uint64)
        v = (np.cumsum(step) + np.uint64(at)) << np.uint64(16)
        at = int(v[-1] >> np.uint64(16)) + 1
        parts.append(struct.pack("<i", 1) + struct.pack("<Ii", 37450, 2) + struct.pack("<4Q", int(v[0]), int(v[-1]), n * 100, 3))
        parts.append(struct.pack("<i", n) + v.astype("<u8").tobytes())
    parts.append(struct.pack("<Q", 0))
    open(path, "wb").write(b"".join(parts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=313)
    ap.add_argument("--keep", action="store_true")
    ap.add_argument("--extranorm", action="store_true", help="run indexcov with -n")
    args = ap.parse_args()
    exe = os.path.join(ROOT, "bin", "goleft")
    tmp = tempfile.mkdtemp(prefix="glcohort_")
    try:
        rng = np.random.default_rng(7)
        t0 = time.perf_counter()
        paths = []
        for k in range(args.samples):
            p = os.path.join(tmp, "s%04d.bai" % k)
            write_bai(p, rng, 0.6 + 0.8 * rng.random())
            paths.append(p)
        t_write = time.perf_counter() - t0
        open(os.path.join(tmp, "ref.fai"), "w").write("".join("%s\t%d\t0\t60\t61\n" % (str(i + 1) if i < 22 else ("X", "Y", "MT")[i - 22] if i < 25 else "GL%06d" % i, L)
                                                              for i, L in enumerate(HS37D5)))
        out = os.path.join(tmp, "out")
        t0 = time.perf_counter()
        os.environ["GL_TIMING"] = "1"
        p = subprocess.run([exe, "indexcov", "-d", out, "--fai", os.path.join(tmp, "ref.fai"), "--includegl", "--excludepatt", "^$"] + (["-n"] if args.extranorm else []) + paths, capture_output=True, text=True)
        wall = time.perf_counter() - t0
        if p.returncode != 0:
            print(json.dumps({"error": p.stderr[-500:]})); return
        tiles = sum(L // 16384 for L in HS37D5)
        bed = os.path.join(out, "out-indexcov.bed.gz")
        res = {"samples": args.samples, "extranorm": args.extranorm, "tiles_per_sample": tiles, "tile_samples": args.samples * tiles, "index_bytes": sum(os.path.getsize(x) for x in paths),
               "write_indexes_s": t_write, "cli_wall_s": wall, "tile_samples_per_s": args.samples * tiles / wall,
               "bed_gz_bytes": os.path.getsize(bed), "host_threads": os.cpu_count(),
               "phases": [ln.replace("[indexcov timing]", "").strip() for ln in p.stderr.splitlines() if ln.startswith("[indexcov timing]")],
               "stderr_tail": p.stderr.strip().splitlines()[-2:]}
        print(json.dumps(res))
    finally:
        if not args.keep:
            shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
