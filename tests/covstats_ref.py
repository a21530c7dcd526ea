"""Helpers for the covstats tests: BAMs with paired records written through bamutil, and covstats.BamStats's loop
(covstats/covstats.go:122-173) restated in Python on the records as they are stored."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bamutil import _stored_cigar, cigar_u32, make_bam, make_bam_indexed  # noqa: E402

CIGARS = [[(100, "M")], [(100, "M")], [(100, "M")], [(45, "M"), (7, "D"), (55, "M")], [(30, "M"), (2, "I"), (68, "M")], [(12, "S"), (88, "M")],
          [(151, "M")], [(75, "="), (1, "X"), (74, "=")]]
# proper pairs (left and right mates), unpaired, dup, QC-fail, secondary, unmapped with coordinates, supplementary
FLAGS = [99, 163, 147, 83, 99, 163, 0, 16, 0x400 | 99, 0x200 | 163, 0x100, 0x4 | 0x1 | 0x40, 0x800 | 99]


def records(rng, per_ref, flags=FLAGS, unplaced=0, ref_len=400_000, cg_every=0):
    """(refs, records, mates) sorted by (tid, pos): per_ref[t] records on reference t (0: a reference without reads), then
    `unplaced` records with tid -1.  cg_every: every so many records a proper pair's CIGAR is stored as the CG placeholder."""
    refs = [("c%d" % t, ref_len) for t in range(len(per_ref))]
    recs, mates = [], []
    for tid, m in enumerate(per_ref):
        for p0 in np.sort(rng.integers(0, ref_len - 400, m)):
            flag = int(flags[int(rng.integers(0, len(flags)))])
            cigar = CIGARS[int(rng.integers(0, len(CIGARS)))]
            ins = int(rng.normal(350, 40)) if rng.random() > 0.01 else int(rng.integers(2000, 90000))
            left = flag & 0x20 or not flag & 0x1
            mp = int(p0) + ins if left else max(0, int(p0) - ins)
            if rng.random() < 0.02:
                mp = int(p0)                                                   # pos == mate_pos: not an insert
            opts = {}
            if cg_every and len(recs) % cg_every == 0:
                flag, cigar, opts = 99, [(60, "M"), (3, "D"), (40, "M")], dict(cg=True)
            recs.append((tid, int(p0), 60, flag, cigar, opts) if opts else (tid, int(p0), 60, flag, cigar))
            mates.append((mp, (ins + 100) if left else -(ins + 100)))
    for _ in range(unplaced):
        recs.append((-1, -1, 0, 0x4 | 0x1 | 0x40, []))
        mates.append((-1, 0))
    return refs, recs, mates


def write(tmp_path, name, refs, recs, mates, indexed=True, block=60000):
    p = str(tmp_path / name)
    if indexed:
        bam, bai = make_bam_indexed(refs, recs, "S1", mates, block=block)
        open(p + ".bai", "wb").write(bai)
    else:
        bam = make_bam(refs, recs, "S1", mates, block=block)
    open(p, "wb").write(bam)
    return p


def stored(rec):
    """the CIGAR as the record stores it (uint32 ops)"""
    return _stored_cigar(rec[4], rec[5])[0] if len(rec) > 5 and rec[5] else cigar_u32(rec[4])


def restate(recs, mates, n, skip):
    """-> dict of the counters, the three sample arrays in file order, and the index of the last record looked at"""
    sizes, ins, tm = [], [], []
    c = dict(n_unmapped=0, k=0, n_bad=0, n_dup=0, n_proper=0)
    read = 0
    if n > 0:
        for i, rec in enumerate(recs):
            if i < skip:
                read = i + 1
                continue
            if len(ins) >= n:
                break
            read = i + 1
            pos, flag = rec[1], rec[3]
            if flag & 4:
                c["n_unmapped"] += 1
                continue
            c["k"] += 1
            if flag & 0x600:
                c["n_dup"] += 1 if flag & 0x400 else 0
                c["n_bad"] += 1
                continue
            if flag & 2:
                c["n_proper"] += 1
            cig = stored(rec)
            ln, op = (cig >> 4).astype(np.int64), cig & 15
            if len(sizes) < 2 * n:
                sizes.append(int(ln[np.isin(op, (0, 1, 4, 7, 8))].sum()))
            elif not ins:
                break
            mp, tl = mates[i]
            if pos < mp and flag & 2 and cig.size == 1 and op[0] == 0:
                ins.append(mp - (pos + int(ln[0])))
                tm.append(tl)
    c.update(n_read_len=len(sizes), n_insert=len(ins), n_records_read=read)
    return c, (np.array(sizes, np.int32), np.array(ins, np.int32), np.array(tm, np.int32))


def stats_numpy(c, sizes, ins, tm):
    """covstats.go:175-218 on sorted arrays -> (dict of Stats fields, H)"""
    s = dict(insert_mean=0.0, insert_sd=0.0, insert_pct5=0, insert_pct95=0, template_mean=0.0, template_sd=0.0, read_length_mean=0.0,
             read_length_median=0.0, proportion_bad=0.0, proportion_unmapped=0.0, proportion_properly_paired=0.0, proportion_duplicate=0.0,
             max_read_length=0)

    def mean_std(a):
        l, m, sd = float(len(a)), 0.0, 0.0
        for x in a:
            m += float(x) / l
        for x in a:
            sd += (float(x) - m) ** 2 / l
        return m, float(np.sqrt(sd))

    def mad(a):
        a = np.sort(a)
        med = int(a[len(a) // 2])
        um = np.sort(a[len(a) // 2 + 1:] - med)
        upper = med + 10 * int(um[len(um) // 2])
        i = int(np.searchsorted(a, upper, "right"))
        return a[:min(i, len(a) - 1)]
    if len(sizes):
        den = float(c["k"] + c["n_unmapped"])
        s.update(proportion_bad=c["n_bad"] / den, proportion_duplicate=c["n_dup"] / den, proportion_properly_paired=c["n_proper"] / den,
                 proportion_unmapped=c["n_unmapped"] / den)
        a = np.sort(sizes)
        s.update(read_length_median=float(a[(len(a) - 1) // 2]) - 1, read_length_mean=mean_std(a)[0], max_read_length=int(a[-1]))
    H = np.zeros(0)
    if len(ins):
        a = np.sort(ins)
        l = float(len(a) - 1)
        s.update(insert_pct5=int(a[int(0.05 * l + 0.5)]), insert_pct95=int(a[int(0.95 * l + 0.5)]))
        s["insert_mean"], s["insert_sd"] = mean_std(mad(ins))
        t = mad(tm)
        s["template_mean"], s["template_sd"] = mean_std(t)
        start, stop = float(s["max_read_length"]), s["template_mean"] + s["template_sd"] * 4
        H = np.zeros(int(stop - start + 1))
        keep = t[(t >= start) & (t <= stop)]
        for x in keep:
            H[int(x - start)] += 1
        with np.errstate(invalid="ignore", divide="ignore"):
            H = H / float(len(keep))
    return s, H
