"""Region queries of indexed BAMs, restated for the tests: the fixtures (BAMs whose reads cross 16 KB tile edges, long reads
in low-level bins and in bin 0, CG reads, D/N CIGARs, unmapped placed reads), every record's virtual offset, the BAI's
binning section read and rewritten, htslib's chunk merging (hts.c compress_binning), and the planner and block filter the
library must match.  Written from the SAM spec (5.2 the BAI, 5.3 reg2bins) and htslib's documented query rule."""
import struct

import numpy as np

from bamutil import BLOCK, _bgzf, cg_mix_records, cigar_lens, make_bam

MIN_MARKER_DIST = 0x10000          # htslib HTS_MIN_MARKER_DIST: a bin spanning fewer compressed bytes moves into its parent


def record_voffsets(refs, records, block=BLOCK):
    """[(v0, v1)]: the virtual offsets of every record's start and end, as make_bam_indexed lays the file out"""
    rec_off, blocks = [], []
    payload = make_bam(refs, records, _raw=True, _rec_off=rec_off)
    _bgzf(payload, blocks, block)

    def voff(o):
        return (blocks[o // block] << 16) | (o % block)
    return [(voff(a), voff(b)) for a, b in rec_off]


def record_span(rec):
    """[pos, end) the index files a record under (an unmapped placed read covers one base)"""
    tid, pos, mapq, flag, cigar = rec[:5]
    return pos, pos + 1 if flag & 4 else pos + max(cigar_lens(cigar)[1], 1)


def read_bai(bai: bytes):
    """[(bins {bin: [[cb, ce], ...]} without the stats bin, stats chunks or None, linear index list)] per reference, n_no_coor"""
    off = 4
    n_ref = struct.unpack_from("<i", bai, off)[0]; off += 4
    out = []
    for _ in range(n_ref):
        n_bin = struct.unpack_from("<i", bai, off)[0]; off += 4
        bins, stats = {}, None
        for _ in range(n_bin):
            b, nc = struct.unpack_from("<Ii", bai, off); off += 8
            ch = [list(struct.unpack_from("<QQ", bai, off + 16 * c)) for c in range(nc)]
            off += 16 * nc
            if b == 37450:
                stats = ch
            else:
                bins[b] = ch
        n_lin = struct.unpack_from("<i", bai, off)[0]; off += 4
        lin = list(struct.unpack_from("<%dQ" % n_lin, bai, off)); off += 8 * n_lin
        out.append((bins, stats, lin))
    return out, struct.unpack_from("<Q", bai, off)[0]


def write_bai(refs_idx, n_no_coor) -> bytes:
    b = b"BAI\x01" + struct.pack("<i", len(refs_idx))
    for bins, stats, lin in refs_idx:
        b += struct.pack("<i", len(bins) + (stats is not None))
        for k in sorted(bins):
            b += struct.pack("<Ii", k, len(bins[k])) + b"".join(struct.pack("<QQ", *c) for c in bins[k])
        if stats is not None:
            b += struct.pack("<Ii", 37450, len(stats)) + b"".join(struct.pack("<QQ", *c) for c in stats)
        b += struct.pack("<i", len(lin)) + struct.pack("<%dQ" % len(lin), *lin)
    return b + struct.pack("<Q", n_no_coor)


def parent(b):
    return (b - 1) >> 3


def first_of_level(level):
    return ((1 << (3 * level)) - 1) // 7


def htslib_merged(bai: bytes, min_dist=MIN_MARKER_DIST) -> bytes:
    """the BAI as samtools index writes it (compress_binning): from the leaves up, a bin whose chunks span fewer than
    min_dist compressed bytes moves its chunks into its parent when the parent exists; then every bin's chunks are sorted and
    a chunk is merged into the one before it when that one ends in the BGZF block it starts in.  So one chunk can cover
    records of other bins, and chunks of different bins overlap."""
    refs_idx, n_nc = read_bai(bai)
    out = []
    for bins, stats, lin in refs_idx:
        bins = {k: [list(c) for c in v] for k, v in bins.items()}
        for level in range(5, 0, -1):
            for k in sorted(b for b in bins if first_of_level(level) <= b < first_of_level(level + 1)):
                p = bins[k]
                p.sort()
                if (p[-1][1] >> 16) - (p[0][0] >> 16) < min_dist and parent(k) in bins:
                    bins[parent(k)] += p
                    del bins[k]
        for k in bins:
            p = sorted(bins[k])
            m = [p[0]]
            for c in p[1:]:
                if m[-1][1] >> 16 >= c[0] >> 16:
                    m[-1][1] = max(m[-1][1], c[1])
                else:
                    m.append(c)
            bins[k] = m
        out.append((bins, stats, lin))
    return write_bai(out, n_nc)


def reg2bins(beg, end):
    """SAM spec 5.3: the bins that may hold records overlapping [beg, end)"""
    end -= 1
    out = [0]
    for first, shift in ((1, 26), (9, 23), (73, 20), (585, 17), (4681, 14)):
        out += range(first + (beg >> shift), first + (end >> shift) + 1)
    return out


def max_off(bins, end):
    """htslib's max_off for an interval ending at end: the first chunk of the nearest bin with chunks to its right, moving
    right along the leaves and up to the parent at a first child; None when there is none"""
    k = 4681 + ((end - 1) >> 14) + 1
    while True:
        if k >= 37450:
            k = 0
        while k % 8 == 1:
            k = (k - 1) >> 3
        if k == 0:
            return None
        if bins.get(k):
            return min(cb for cb, _ in bins[k])
        k += 1


def plan(bins, lin, intervals):
    """the ranges a query reads: chunks of the bins reg2bins names for an interval that end after the linear-index offset
    of its first tile (the last entry past the index) and begin before max_off; a bin several intervals name keeps what
    lies between the smallest of their min_offs and the largest of their max_offs; sorted, merged where they overlap or
    touch"""
    lo, hi = {}, {}
    for b, e in intervals:
        b, e = max(b, 0), min(e, 1 << 29)
        if e <= b:
            continue
        min_off = lin[min(b >> 14, len(lin) - 1)] if lin else 0
        mx = max_off(bins, e)
        mx = (1 << 64) - 1 if mx is None else mx
        for k in reg2bins(b, e):
            lo[k] = min(lo.get(k, min_off), min_off)
            hi[k] = max(hi.get(k, mx), mx)
    got = sorted((cb, ce) for k in lo for cb, ce in bins.get(k, ()) if ce > lo[k] and cb < hi[k] and ce > cb)
    out = []
    for cb, ce in got:
        if out and cb <= out[-1][1]:
            out[-1][1] = max(out[-1][1], ce)
        else:
            out.append([cb, ce])
    return [tuple(x) for x in out]


def meets(s, e, intervals):
    """bool mask: the blocks [s, e) that meet at least one interval"""
    s, e = np.asarray(s, np.int64), np.asarray(e, np.int64)
    m = np.zeros(s.size, bool)
    for b, x in intervals:
        if x > b:
            m |= (s < x) & (e > b)
    return m


def expected_blocks(segs, tid, intervals):
    """of bamref.segments' blocks (segs), those of tid that meet the intervals, in BAM order"""
    s, e = segs[tid]
    m = meets(s, e, intervals)
    return s[m], e[m]


def fixture(seed=5, n_short=6000):
    """(refs, records) sorted by (tid, pos), unplaced last.  chrA (2.2 Mb): short reads with D/N/I/S CIGARs, crossing
    tile edges, in clusters with read-free gaps, unmapped placed reads, MAPQ 0..60 and every flag class, and long reads
    (20-600 kb spans) that land in bins of levels 1-4.  chrB (70 Mb): a few reads on either side of 2^26 and two that
    cross it, so they sit in bin 0.  chrL: ultra-long CG reads and the CG edge cases (bamutil.cg_mix_records).  chrE: no
    reads."""
    rng = np.random.default_rng(seed)
    refs = [("chrA", 2_200_000), ("chrB", 70_000_000)]
    recs = []
    cig = [[(150, "M")], [(70, "M"), (5, "D"), (80, "M")], [(60, "M"), (2, "I"), (88, "M")], [(10, "S"), (140, "M")],
           [(40, "M"), (900, "N"), (60, "M")], [(75, "="), (1, "X"), (74, "=")]]
    centres = np.sort(rng.integers(0, 2_150_000, 40))
    pos = np.concatenate([c + rng.integers(0, 30_000, n_short // 40) for c in centres])
    pos = np.concatenate([pos, 16384 * np.arange(1, 130) - rng.integers(1, 140, 129)])      # across tile edges
    for p0 in np.sort(np.clip(pos, 0, 2_190_000)):
        recs.append((0, int(p0), int(rng.choice([0, 1, 5, 20, 60, 60])), int(rng.choice([0, 16, 0x400, 0x100, 0x200, 0x800, 4, 0])),
                     cig[int(rng.integers(0, len(cig)))]))
    for p0, span in zip(np.sort(rng.integers(0, 1_500_000, 12)), rng.integers(20_000, 600_000, 12)):
        recs.append((0, int(p0), 60, int(rng.choice([0, 16])), [(100, "M"), (int(span), "N"), (100, "M")]))
    two26 = 1 << 26
    for p0 in (two26 - 5_000_000, two26 - 30_000, two26 - 400, two26 - 100, two26 + 50, two26 + 2_000_000):
        recs.append((1, p0, 60, 0, [(150, "M")]))
    recs.append((1, two26 - 200, 60, 0, [(150, "M"), (300, "D"), (150, "M")]))              # crosses 2^26: bin 0
    recs.append((1, two26 - 3_000_000, 60, 16, [(100, "M"), (5_000_000, "N"), (100, "M")]))
    long_recs, end = cg_mix_records(np.random.default_rng(seed + 1), 2, n_long=12, n_short=1500)
    refs.append(("chrL", end + 1000))
    recs += long_recs
    refs.append(("chrE", 50_000))
    recs.sort(key=lambda r: (r[0], r[1]))
    recs.append((-1, -1, 0, 4, [(100, "M")]))
    return refs, recs


def interval_sets(rng, L):
    """named lists of query intervals on a contig of length L"""
    one = int(rng.integers(0, L - 1000))
    many = [(int(a), int(a + n)) for a, n in zip(rng.integers(0, L, 300), rng.integers(1, 5000, 300))]
    return {
        "single": [(one, one + 500)],
        "hundreds_unsorted": many,
        "overlapping": [(a, a + 20_000) for a in range(0, min(L, 400_000), 7_000)][::-1],
        "with_empty": [(5, 5), (100, 50), (1000, 1001)] + many[:20],
        "past_end": [(L - 300, L + 100_000), (L + 10, L + 2_000_000), (1 << 30, (1 << 30) + 5)],
        "whole": [(0, L)],
        "none": [],
        "only_empty": [(7, 7), (10, 3)],
    }


def gap_intervals(records, tid, L, min_gap=20_000):
    """intervals inside the read-free gaps of reference tid (no record's indexed span reaches them), and in tiles past
    its last read (so past its linear index)"""
    spans = sorted(record_span(r) for r in records if r[0] == tid)
    out, reach = [], 0
    for b, e in spans:
        if b - reach > min_gap:
            out.append((reach + min_gap // 4, b - min_gap // 4))
        reach = max(reach, e)
    last_tile = (reach >> 14) + 3
    if (last_tile << 14) + 1000 < L:
        out.append((last_tile << 14, (last_tile << 14) + 1000))
    return out
