#!/usr/bin/env python3
"""Write the two .bai cohorts the PC-column goldens are made from (tools/make_reference_goldens.sh runs the reference's
`indexcov --fai` on them; tests/test_reference_goldens_indexcov_pca.py runs ours on the same files).  Standard library
only, so it runs wherever the reference toolchain does; the same seed gives the same bytes everywhere.

    python3 tests/golden/make_pca_cohort.py OUTDIR

OUTDIR/g.fa.fai, OUTDIR/pca8/s0..s7.bai (8 samples) and OUTDIR/pca4/s0..s3.bai (4 samples).  Each sample loses coverage
over a stretch of chromosome 1 that depends on its group (k % 3), so the components have structure to find; chromosome 2
is short in one sample; X and Y give the sex columns."""
import os
import random
import struct
import sys

REFS = [("1", 3_000_000), ("2", 2_000_000), ("GL000207.1", 4262), ("X", 1_500_000), ("Y", 600_000)]
TILE = 16384


def bai(per_ref, stats):
    parts = [b"BAI\x01", struct.pack("<i", len(per_ref))]
    for iv, (mapped, unmapped) in zip(per_ref, stats):
        parts.append(struct.pack("<i", 1) + struct.pack("<Ii", 37450, 2) + struct.pack("<4Q", iv[0], iv[-1], mapped, unmapped))
        parts.append(struct.pack("<i", len(iv)) + b"".join(struct.pack("<Q", v) for v in iv))
    parts.append(struct.pack("<Q", 0))
    return b"".join(parts)


def cohort(path, S, seed):
    rng = random.Random(seed)
    os.makedirs(path, exist_ok=True)
    for k in range(S):
        grp = k % 3
        per_ref, v = [], 1 << 16
        for name, L in REFS:
            nt = L // TILE + 1 - (7 if (k == 1 and name == "2") else 0)
            scale = {"X": 0.5 if k % 2 == 0 else 1.0, "Y": 0.5 if k % 2 == 0 else 0.01}.get(name, 1.0)
            iv = [v << 16]
            for i in range(nt):
                m = 25_000 * scale
                if name == "1" and 30 + 40 * grp <= i < 60 + 40 * grp:
                    m *= 0.35 + 0.1 * grp
                v += max(1, int(rng.gauss(m, 1_800)))
                iv.append(v << 16)
            per_ref.append(iv)
        with open(os.path.join(path, "s%d.bai" % k), "wb") as f:
            f.write(bai(per_ref, [(1000 * (k + 1), 10 + k)] * len(REFS)))


def main():
    out = sys.argv[1]
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "g.fa.fai"), "w") as f:
        f.write("".join("%s\t%d\t6\t60\t61\n" % r for r in REFS))
    cohort(os.path.join(out, "pca8"), 8, 8)
    cohort(os.path.join(out, "pca4"), 4, 4)


if __name__ == "__main__":
    main()
