"""An independent reference for BAM decoding: the (start, end) blocks `samtools depth` counts for a list of records as
tests/bamutil.py writes them, restated from the SAM spec and htslib's rules rather than from this project's walkers.

  filter     flag & 0x704 == 0 and MAPQ >= Q (samtools depth's defaults plus -Q)
  CIGAR      M, = and X count; D and N advance without counting; I, S, H and P neither count nor advance.  A record's
             blocks are the maximal runs of reference bases its counting ops cover.
  CG         the CIGAR written to the CG tag replaces the stored one exactly when htslib's bam_read1 would swap it in
             (bam_tag2cigar): tid >= 0 and pos >= 0, the first stored op is S of length l_seq, a CG tag of type B with
             subtype I or i is present, and it holds at least as many ops as the stored CIGAR.  Otherwise the stored
             CIGAR (for a long read: the kSmN placeholder, which counts nothing) is walked as written.

The stored CIGAR and the CG tag are recomputed here from the record's options (bamutil's documented encodings), not read
back from the file."""
import numpy as np

from bamutil import cigar_lens, cigar_u32


def effective_cigar(rec):
    """the CIGAR htslib hands to samtools for this record: the written one (as given), or the stored placeholder (uint32 ops)"""
    tid, pos, mapq, flag, cigar = rec[:5]
    opts = rec[5] if len(rec) > 5 else {}
    mode = opts.get("cg")
    if mode is None:
        mode = len(cigar) > 65535
    if mode is False:
        return cigar
    real = cigar_u32(cigar)
    lseq, span = cigar_lens(real)
    if mode == "bad_s":
        stored = [((lseq - 1) << 4) | 4, (1 << 4) | 1, (span << 4) | 3]
    else:
        stored = [(lseq << 4) | 4, (span << 4) | 3]
    cg_type = {True: "I", "B:i": "i", "B:S": "S", "B:f": "f", "short": "I", "bad_s": "I", "absent": None}[mode]
    cg_count = 1 if mode == "short" else real.size
    first_is_lseq_s = (stored[0] & 15) == 4 and (stored[0] >> 4) == lseq
    if tid >= 0 and pos >= 0 and first_is_lseq_s and cg_type in ("I", "i") and cg_count >= len(stored):
        return cigar
    return np.array(stored, np.uint32)


def record_blocks(pos, cig):
    """(start, end) int64 arrays: the maximal runs of reference bases covered by M/=/X.  cig: a list of (length, op) or
    uint32 ops"""
    if not isinstance(cig, np.ndarray):                         # short CIGARs: the same rule, op by op
        s, e = [], []
        ref = pos
        for ln, op in cig:
            if op in "M=X" and ln > 0:
                if e and e[-1] == ref:
                    e[-1] = ref + ln
                else:
                    s.append(ref); e.append(ref + ln)
            if op in "MDN=X":
                ref += ln
        return np.array(s, np.int64), np.array(e, np.int64)
    ln, op = (cig >> 4).astype(np.int64), cig & 15
    adv = np.isin(op, (0, 2, 3, 7, 8))
    cnt = np.isin(op, (0, 7, 8)) & (ln > 0)
    ref0 = pos + np.concatenate([[0], np.cumsum(np.where(adv, ln, 0))[:-1]])
    s, e = ref0[cnt], ref0[cnt] + ln[cnt]
    if s.size == 0:
        return s, e
    brk = np.concatenate([[True], s[1:] != e[:-1]])            # a new block unless it starts where the last one ended
    first = np.flatnonzero(brk)
    last = np.concatenate([first[1:], [s.size]]) - 1
    return s[first], e[last]


def passes(rec, min_mapq) -> bool:
    tid, pos, mapq, flag = rec[:4]
    return tid >= 0 and (flag & 0x704) == 0 and mapq >= min_mapq


def segments(records, n_refs, min_mapq=1):
    """{tid: (start, end)} int32 arrays for every reference, in record order"""
    acc = {t: ([], []) for t in range(n_refs)}
    for rec in records:
        if not passes(rec, min_mapq):
            continue
        s, e = record_blocks(rec[1], effective_cigar(rec))
        acc[rec[0]][0].append(s); acc[rec[0]][1].append(e)
    out = {}
    for t, (ss, ee) in acc.items():
        out[t] = (np.concatenate(ss).astype(np.int32) if ss else np.zeros(0, np.int32),
                  np.concatenate(ee).astype(np.int32) if ee else np.zeros(0, np.int32))
    return out


def pileup(s, e, rs, re) -> np.ndarray:
    """per-base depth on [rs, re), brute force: every block adds one to each base it covers"""
    s = np.clip(np.asarray(s, np.int64), rs, re)
    e = np.clip(np.asarray(e, np.int64), rs, re)
    n = e - s
    base = np.repeat(s, n) + (np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n))
    return np.bincount(base - rs, minlength=re - rs).astype(np.int32)


def split255(s, e):
    """blocks cut into pieces of at most 255 bases from their start, as the packed8 format stores them"""
    s, e = np.asarray(s, np.int64), np.asarray(e, np.int64)
    k = (e - s + 254) // 255
    rep = np.repeat(np.arange(s.size), k)
    off = np.arange(rep.size) - np.repeat(np.cumsum(k) - k, k)
    ps = s[rep] + 255 * off
    return ps, np.minimum(ps + 255, e[rep])


def same_multiset(s1, e1, s2, e2) -> bool:
    """equal as multisets of (start, end) (the walkers may emit blocks in another order)"""
    s1, e1, s2, e2 = (np.asarray(x, np.int64) for x in (s1, e1, s2, e2))
    if s1.size != s2.size:
        return False
    o1, o2 = np.lexsort((e1, s1)), np.lexsort((e2, s2))
    return bool(np.array_equal(s1[o1], s2[o2]) and np.array_equal(e1[o1], e2[o2]))
