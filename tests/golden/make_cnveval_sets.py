#!/usr/bin/env python3
"""Write the truth / test sets the cnveval goldens are made from (tools/make_reference_goldens.sh runs the reference's
`cnveval` on them; tests/test_reference_goldens_cnveval.py runs ours on the same files).  Standard library only, so it runs
wherever the reference toolchain does; the same seed gives the same bytes everywhere.

    python3 tests/golden/make_cnveval_sets.py OUTDIR

OUTDIR/<case>.truth.bed and OUTDIR/<case>.test.bed for each case in CASES:
  cohort  40 samples, 3 chromosomes named so that bytewise order is not numeric order, starts on a 500-base grid (many
          equal starts in one sample, so the sort.Slice order inside ties matters), jittered calls with some wrong CNs,
          false calls, test lines with a second sample, `#` lines and CRLF endings
  quirks  the hand cases: an uncalled carrier, two qualifying calls, an FP run through a non-overlapping call, a large call
          over a medium truth, duplicate members, CN clamping, zero-length intervals, and a final line without a newline"""
import os
import random
import sys

CASES = ["cohort", "quirks"]
# the reference's argument lists per mode (the CLI takes the same ones)
MODES = {"default": [], "limit": ["-s"], "m05": ["-m", "0.5"]}
CHROMS = ["chr1", "chr10", "chr2"]


def cohort(seed=2718):
    rng = random.Random(seed)
    S, T = 40, 300
    truth, test = ["#chrom\tstart\tend\tcn\tsamples"], ["#chrom\tstart\tend\tcn\tsample"]
    for t in range(T):
        c = rng.choice(CHROMS)
        s = rng.randrange(0, 2_000_000) // 500 * 500
        e = s + int(rng.choice([300, 800, 5000, 19999, 20000, 45000, 99999, 100000, 250000]) * rng.uniform(0.5, 1.5))
        cn = rng.choice([0, 1, 3, 4, 5])
        carriers = [rng.randrange(S) for _ in range(min(S, int(rng.expovariate(0.3))))]
        truth.append("%s\t%d\t%d\t%d\t%s%s" % (c, s, e, cn, ",".join("s%d" % x for x in carriers), "\r" if t % 11 == 0 else ""))
        for x in carriers:
            if rng.random() < 0.8:
                L = e - s
                b = max(0, s + rng.randint(-L // 4, L // 4) // 500 * 500)
                test.append("%s\t%d\t%d\t%d\ts%d%s" % (c, b, max(b, e + rng.randint(-L // 4, L // 4)),
                                                      cn if rng.random() < 0.9 else rng.choice([1, 3]), x,
                                                      ",s%d" % ((x + 1) % S) if rng.random() < 0.1 else ""))
    for _ in range(120):
        c, b = rng.choice(CHROMS), rng.randrange(0, 2_000_000) // 500 * 500
        test.append("%s\t%d\t%d\t%d\ts%d" % (c, b, b + rng.randrange(100, 150000), rng.choice([1, 3]), rng.randrange(S)))
    body = test[1:]
    rng.shuffle(body)
    return "\n".join(truth) + "\n", "\n".join(test[:1] + body) + "\n"


def quirks():
    truth = ["chr1\t100\t200\t1\tB", "chr1\t100\t200\t1\tA,A", "chr1\t1000\t1200\t1\tC", "chr1\t1180\t1200\t1\tA",
             "chr1\t0\t50000\t1\tC", "chr1\t5000\t5100\t3\tA", "chr1\t7000\t7000\t1\tA", "chr2\t100\t200\t2\tZ"]
    test = ["chr1\t110\t190\t1\tA", "chr1\t100\t200\t1\tA", "chr1\t950\t1150\t1\tA", "chr1\t960\t970\t1\tA",
            "chr1\t1180\t1200\t1\tA", "chr1\t0\t150000\t1\tD", "chr1\t5000\t5100\t7\tA,B", "chr1\t7000\t7000\t1\tA",
            "chr2\t100\t200\t4\tE"]
    return "\n".join(truth) + "\n", "\n".join(test) + "\nchr1\t1\t2\t1\tA"      # the last line has no newline: dropped


def write(out):
    os.makedirs(out, exist_ok=True)
    for name, (truth, test) in (("cohort", cohort()), ("quirks", quirks())):
        with open(os.path.join(out, name + ".truth.bed"), "wb") as f:
            f.write(truth.encode())
        with open(os.path.join(out, name + ".test.bed"), "wb") as f:
            f.write(test.encode())


if __name__ == "__main__":
    write(sys.argv[1])
