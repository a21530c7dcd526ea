"""Test helpers: write small BAM / BAI files from Python (BAM spec, SURVEY.md Appendix D).

A record is (tid, pos, mapq, flag, cigar) or (tid, pos, mapq, flag, cigar, opts).  `cigar` is a list of (length, op) or a
uint32 array of BAM-encoded ops (length << 4 | code).  `opts` (a dict) may hold:
  name  the read name (at most 254 characters; default "r")
  aux   a list of (tag, type, value) in file order: type one of A c C s S i I f Z H, or "B:<sub>" with a list value;
        the string "CG" in the list marks where the CG tag goes (default: after the other tags); a bytes item is written
        as it is (malformed aux data: the reader must keep the stored CIGAR and stay inside the record)
  cg    how the CIGAR is stored.  None: through CG exactly when it has more than 65535 ops (SAMv1 4.2.2); True: through CG
        anyway.  Forms htslib must NOT convert (the placeholder stays, so the read counts nothing):
          "absent"  placeholder, no CG tag          "B:S" / "B:f"  CG of another array type
          "short"   CG holding fewer ops than the placeholder (its first op only)
          "bad_s"   placeholder whose first op is S of length l_seq - 1 (then 1I keeps the query length right)
        and "B:i": a CG of signed ints, which htslib does convert.
The placeholder is `kSmN` with k = l_seq and m = the real CIGAR's reference span."""
import struct
import zlib

import numpy as np

BLOCK = 60000
OPS = "MIDNSHP=X"
_B_SUB = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}
_SCALAR = {"A": "c", "c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}


def cigar_u32(cigar) -> np.ndarray:
    """a CIGAR as BAM-encoded uint32 ops"""
    if isinstance(cigar, np.ndarray):
        return cigar.astype(np.uint32, copy=False)
    return np.array([(ln << 4) | OPS.index(op) for ln, op in cigar], np.uint32)


def cigar_lens(cigar):
    """(query length: M I S = X, reference span: M D N = X)"""
    c = cigar_u32(cigar)
    ln, op = (c >> 4).astype(np.int64), c & 15
    return int(ln[np.isin(op, (0, 1, 4, 7, 8))].sum()), int(ln[np.isin(op, (0, 2, 3, 7, 8))].sum())


def _aux_bytes(tag, typ, val) -> bytes:
    if typ.startswith("B:"):
        sub = typ[2]
        return tag.encode() + b"B" + sub.encode() + struct.pack("<I", len(val)) + np.asarray(val, "<" + _B_SUB[sub]).tobytes()
    if typ in ("Z", "H"):
        return tag.encode() + typ.encode() + val.encode() + b"\0"
    return tag.encode() + typ.encode() + struct.pack("<" + _SCALAR[typ], val.encode() if typ == "A" else val)


def _stored_cigar(cigar, opts):
    """(cigar stored in the record as uint32 ops, CG tag bytes or b"") for `cigar` under opts["cg"]"""
    real = cigar_u32(cigar)
    mode = opts.get("cg")
    if mode is None:
        mode = True if real.size > 65535 else False
    if mode is False:
        return real, b""
    lseq, span = cigar_lens(real)
    place = np.array([(lseq << 4) | 4, (span << 4) | 3], np.uint32)
    if mode == "bad_s":
        assert lseq >= 1
        place = np.array([((lseq - 1) << 4) | 4, (1 << 4) | 1, (span << 4) | 3], np.uint32)
    if mode == "absent":
        return place, b""
    typ = {True: "I", "B:i": "i", "B:S": "S", "B:f": "f", "short": "I", "bad_s": "I"}[mode]
    val = real[:1] if mode == "short" else real
    body = np.asarray(val, np.uint32)
    if typ == "f":
        body = body.astype(np.float32)
    elif typ == "S":
        body = (body & 0xffff).astype(np.uint16)
    return place, b"CGB" + typ.encode() + struct.pack("<I", body.size) + body.astype("<" + _B_SUB[typ]).tobytes()


def _record(tid, pos, mapq, flag, cigar, opts, mates_row, with_mates) -> bytes:
    name = opts.get("name", "r").encode() + b"\0"
    assert len(name) <= 255
    mate_pos, tlen = mates_row if mates_row is not None else (-1, 0)
    if not opts:                                      # the original layout, op by op
        cig = b"".join(struct.pack("<I", (ln << 4) | OPS.index(op)) for ln, op in cigar)
        lseq = sum(ln for ln, op in cigar if op in "MIS=X")
        n_cig, aux = len(cigar), b""
    else:
        stored, cg = _stored_cigar(cigar, opts)
        cig, n_cig = stored.astype("<u4").tobytes(), int(stored.size)
        lseq = cigar_lens(cigar)[0]
        tags = list(opts.get("aux", []))
        if "CG" not in tags:
            tags.append("CG")
        aux = b"".join(cg if t == "CG" else t if isinstance(t, bytes) else _aux_bytes(*t) for t in tags)
    body = struct.pack("<iiBBHHHiiii", tid, pos, len(name), mapq, 0, n_cig, flag, lseq, tid if with_mates else -1, mate_pos, tlen)
    body += name + cig + b"\0" * ((lseq + 1) // 2) + b"\xff" * lseq + aux
    return struct.pack("<i", len(body)) + body


def _bgzf(payload: bytes, offsets=None, block=BLOCK, level=6, flush=None) -> bytes:
    """offsets (a list) receives the compressed offset of every block.  block: payload bytes per member (<= 65536);
    level: deflate level (0: stored blocks, as `samtools view -u`); flush: (zlib flush mode, bytes between flush points)."""
    assert 0 < block <= 65536
    parts = []
    at = 0
    for i in range(0, len(payload), block):
        if offsets is not None:
            offsets.append(at)
        chunk = payload[i:i + block]
        c = zlib.compressobj(level, zlib.DEFLATED, -15)
        if flush is None:
            comp = c.compress(chunk) + c.flush()
        else:
            mode, every = flush
            comp = b"".join(c.compress(chunk[k:k + every]) + c.flush(mode) for k in range(0, len(chunk), every)) + c.flush()
        bsize = 18 + len(comp) + 8
        assert bsize <= 65536, "member does not fit a BGZF block"
        parts.append(b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", bsize - 1) + comp)
        parts.append(struct.pack("<II", zlib.crc32(chunk) & 0xffffffff, len(chunk)))
        at += bsize
    if offsets is not None:
        offsets.append(at)
    parts.append(bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000"))
    return b"".join(parts)


def _reg2bin(beg, end):
    end -= 1
    if beg >> 14 == end >> 14: return ((1 << 15) - 1) // 7 + (beg >> 14)
    if beg >> 17 == end >> 17: return ((1 << 12) - 1) // 7 + (beg >> 17)
    if beg >> 20 == end >> 20: return ((1 << 9) - 1) // 7 + (beg >> 20)
    if beg >> 23 == end >> 23: return ((1 << 6) - 1) // 7 + (beg >> 23)
    if beg >> 26 == end >> 26: return ((1 << 3) - 1) // 7 + (beg >> 26)
    return 0


def make_bam_indexed(refs, records, sample="sampleA", mates=None, block=BLOCK, level=6, flush=None):
    """(bam bytes, bai bytes): a real index — bins with merged chunks, back-filled 16 KB linear index, the 37450 stats bin
    (SAM spec 5.2) — for records sorted by (tid, pos); unplaced records (tid -1) last.  block / level / flush: see _bgzf."""
    rec_off = []
    bam_payload = make_bam(refs, records, sample, mates, _raw=True, _rec_off=rec_off)
    blocks = []
    bam = _bgzf(bam_payload, blocks, block, level, flush)

    def voff(o):
        return (blocks[o // block] << 16) | (o % block)
    bai = b"BAI\x01" + struct.pack("<i", len(refs))
    n_no_coor = 0
    per_ref = [dict(bins={}, lin={}, beg=None, end=0, mapped=0, unmapped=0, last_bin=None) for _ in refs]
    for rec, (o0, o1) in zip(records, rec_off):
        tid, pos, mapq, flag, cigar = rec[:5]
        if tid < 0:
            n_no_coor += 1
            continue
        span = cigar_lens(cigar)[1]                   # a CG read: its real span (= the placeholder's N)
        end = pos + 1 if flag & 4 else pos + max(span, 1)
        R = per_ref[tid]
        b = _reg2bin(pos, end)
        v0, v1 = voff(o0), voff(o1)
        if R["beg"] is None:
            R["beg"] = v0
        R["end"] = v1
        R["unmapped" if flag & 4 else "mapped"] += 1
        ch = R["bins"].setdefault(b, [])
        if R["last_bin"] == b and ch:
            ch[-1][1] = v1
        else:
            ch.append([v0, v1])
        R["last_bin"] = b
        for k in range(pos >> 14, ((end - 1) >> 14) + 1):
            R["lin"].setdefault(k, v0)
    for R in per_ref:
        n_bins = len(R["bins"]) + (1 if R["beg"] is not None else 0)
        bai += struct.pack("<i", n_bins)
        for b in sorted(R["bins"]):
            bai += struct.pack("<Ii", b, len(R["bins"][b]))
            for c0, c1 in R["bins"][b]:
                bai += struct.pack("<QQ", c0, c1)
        if R["beg"] is not None:
            bai += struct.pack("<Ii", 37450, 2) + struct.pack("<4Q", R["beg"], R["end"], R["mapped"], R["unmapped"])
        n_lin = max(R["lin"]) + 1 if R["lin"] else 0
        lin = [R["lin"].get(k, 0) for k in range(n_lin)]
        for k in range(n_lin - 2, -1, -1):
            if lin[k] == 0:
                lin[k] = lin[k + 1]
        bai += struct.pack("<i", n_lin) + struct.pack("<%dQ" % n_lin, *lin)
    return bam, bai + struct.pack("<Q", n_no_coor)


def make_bam(refs, records, sample="sampleA", mates=None, _raw=False, _rec_off=None, block=BLOCK, level=6, flush=None) -> bytes:
    text = b"@HD\tVN:1.6\tSO:coordinate\n@RG\tID:a\tSM:" + sample.encode() + b"\n"
    parts = [b"BAM\x01" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))]
    for n, l in refs:
        parts.append(struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", l))
    at = sum(len(x) for x in parts)
    for ri, rec in enumerate(records):
        tid, pos, mapq, flag, cigar = rec[:5]
        rb = _record(tid, pos, mapq, flag, cigar, rec[5] if len(rec) > 5 else {}, mates[ri] if mates is not None else None, mates is not None)
        if _rec_off is not None:
            _rec_off.append((at, at + len(rb)))
        at += len(rb)
        parts.append(rb)
    return b"".join(parts) if _raw else _bgzf(b"".join(parts), None, block, level, flush)


def make_bai(linear, stats=None) -> bytes:
    """linear: per reference list of u64 virtual offsets; stats: per reference (mapped, unmapped) or None"""
    b = b"BAI\x01" + struct.pack("<i", len(linear))
    for r, iv in enumerate(linear):
        if stats is not None and stats[r] is not None:
            b += struct.pack("<i", 1) + struct.pack("<Ii", 37450, 2) + struct.pack("<4Q", 0, 0, stats[r][0], stats[r][1])
        else:
            b += struct.pack("<i", 0)
        b += struct.pack("<i", len(iv)) + struct.pack("<%dQ" % len(iv), *iv)
    return b + struct.pack("<Q", 0)


def long_read_cigar(rng, span_min=80_000, span_max=300_000, n_min=70_000, n_max=200_000) -> np.ndarray:
    """an ultra-long-read CIGAR (BAM-encoded uint32): 1-3 base M/=/X blocks between I and D, some N, soft / hard clips at
    the ends; more than 65535 ops, so it can only be stored through CG.  The span is near the target where the op count
    allows (at least the M/=/X bases)."""
    n = int(rng.integers(n_min, n_max)) // 2
    target = int(rng.integers(span_min, span_max))
    mlen = rng.integers(1, 4, n)
    mop = rng.choice(np.array([0, 7, 8], np.uint32), n, p=[0.6, 0.3, 0.1])
    gap_op = np.full(n, 1, np.uint32)                  # I by default
    gap_len = rng.integers(1, 3, n)
    k_n = max(1, n // 5000)
    at = rng.choice(n - 1, k_n, replace=False)
    gap_op[at] = 3
    gap_len[at] = rng.integers(20, 200, k_n)
    budget = target - int(mlen.sum()) - int(gap_len[at].sum())
    free = np.flatnonzero(gap_op == 1)
    k_d = int(np.clip(budget // 1.5, 0, free.size))
    gap_op[rng.choice(free, k_d, replace=False)] = 2
    body = np.empty(2 * n, np.uint32)
    body[0::2] = (mlen.astype(np.uint32) << 4) | mop
    body[1::2] = (gap_len.astype(np.uint32) << 4) | gap_op
    body = body[:-1]                                    # end on an M/=/X block
    head = np.array([(int(rng.integers(1, 50)) << 4) | 5, (int(rng.integers(1, 500)) << 4) | 4], np.uint32)      # H then S
    tail = np.array([(int(rng.integers(1, 500)) << 4) | 4], np.uint32)
    return np.concatenate([head, body, tail])


def cg_mix_records(rng, tid, start=0, n_long=40, n_short=4000, long_kw=None):
    """(records sorted by pos, end of the last one) for reference `tid` from `start`: ultra-long reads (long_read_cigar, so
    written through CG) mixed with 150 bp reads, plus the CG edge cases on short CIGARs — forced CG (htslib converts it),
    B:i, and the forms it must not convert (see the module doc) — and placeholder records the flag filter or MAPQ removes.
    Long reads follow each other with gaps or overlaps of up to 20 kb; the CG tag sits at varied places among the other tags."""
    recs = []
    at = start
    others = [("NM", "i", 12345), ("MD", "Z", "10A5^AC6"), ("XB", "B:c", [1, -2, 3]), ("XH", "H", "1AE301"), ("XF", "f", 0.25)]
    for k in range(n_long):
        cig = long_read_cigar(rng, **(long_kw or {}))
        span = cigar_lens(cig)[1]
        tags = [others[j] for j in rng.permutation(len(others))[:int(rng.integers(0, len(others) + 1))]]
        tags.insert(int(rng.integers(0, len(tags) + 1)), "CG")
        flag, mapq = [(0, 60), (16, 60), (0, 7), (0x400, 60), (0x100, 60), (0, 0)][k % 6] if k < 12 else (int(rng.choice([0, 16])), 60)
        name = "L%d_" % k + "x" * int(rng.integers(0, 250 - len("L%d_" % k)))
        recs.append((tid, at, mapq, flag, cig, dict(name=name, aux=tags)))
        at = max(start, at + span + int(rng.integers(-20_000, 5_000)))
    end = max(r[1] + cigar_lens(r[4])[1] for r in recs) if recs else start + 1000
    shorts = [[(150, "M")], [(70, "M"), (5, "D"), (80, "M")], [(60, "M"), (2, "I"), (88, "M")], [(10, "S"), (140, "M")],
              [(75, "="), (1, "X"), (74, "=")], [(3, "H"), (50, "M"), (400, "N"), (100, "M")]]
    for p0 in np.sort(rng.integers(start, end - 200, n_short)):
        recs.append((tid, int(p0), int(rng.choice([0, 30, 60, 60])), int(rng.choice([0, 16, 0x400, 0])), shorts[int(rng.integers(0, len(shorts)))]))
    edge = [dict(cg=True), dict(cg=True, aux=["CG", ("NM", "i", 3)]), dict(cg="B:i"), dict(cg="absent"), dict(cg="B:S"),
            dict(cg="B:f"), dict(cg="short"), dict(cg="bad_s"), dict(cg=True, aux=[("MD", "Z", "150"), "CG", ("XF", "f", 1.5)]),
            dict(cg="absent", aux=[b"CGBI" + struct.pack("<I", 1 << 20) + b"\x00" * 12]),            # CG count overruns the record
            dict(cg="absent", aux=[("NM", "i", 1), b"XQq\x01CGBI" + struct.pack("<3I", 2, 80 << 4, 70 << 4)]),  # unknown type, then a CG
            dict(cg="absent", aux=[b"XZZunterminated"])]
    for p0 in np.sort(rng.integers(start, end - 500, 6 * len(edge))):
        o = edge[int(rng.integers(0, len(edge)))]
        recs.append((tid, int(p0), 60, int(rng.choice([0, 16])), shorts[int(rng.integers(0, len(shorts)))], o))
    for p0 in np.sort(rng.integers(start, end - 500, 12)):                       # placeholders the filters remove
        recs.append((tid, int(p0), int(rng.choice([0, 60])), int(rng.choice([0x4, 0x100, 0x200, 0x400, 0])), [(40, "M"), (3, "D"), (60, "M")], dict(cg=True)))
    recs.sort(key=lambda r: r[1])
    return recs, end
