"""CSI indexes for the tests, written from the CSIv1 spec (independently of the library's reader): bins at any
(min_shift, depth), each bin's loffset from a linear index at the bin's first tile, the stats pseudo-bin, the optional
n_no_coor, BGZF-compressed; a variant whose chunks are merged across bins as samtools merges a BAI's
(region_bams.htslib_merged); the file read back; and restatements of what the library derives from it: the 16 KB linear
index rebuilt from the loffsets and the region planner at the index's geometry.

CSIv1:  "CSI\\1" min_shift:i32 depth:i32 l_aux:i32 aux[l_aux] n_ref:i32
        per ref: n_bin:i32, per bin: bin:u32 loffset:u64 n_chunk:i32 (beg:u64 end:u64)[n_chunk]
        [n_no_coor:u64]
Level l (0..depth) starts at bin ((1 << 3l) - 1) / 7 and its bins cover 2^(min_shift + 3 (depth - l)) bases; the stats
pseudo-bin is ((1 << (3 depth + 3)) - 1) / 7 + 1 with chunks (ref_beg, ref_end), (mapped, unmapped)."""
import struct
import zlib

from bamutil import BLOCK, _bgzf, cigar_lens, make_bam, make_bam_indexed
from region_bams import MIN_MARKER_DIST, htslib_merged, record_voffsets

GEOMETRIES = [(14, 5), (14, 6), (12, 6), (16, 5)]


def first_of_level(level):
    return ((1 << (3 * level)) - 1) // 7


def stats_bin(depth):
    return ((1 << (3 * depth + 3)) - 1) // 7 + 1


def level_of(b, depth):
    level = 0
    while level < depth and b >= first_of_level(level + 1):
        level += 1
    return level


def bin_first_tile(b, depth):
    """the first 2^min_shift tile a bin covers"""
    level = level_of(b, depth)
    return (b - first_of_level(level)) << (3 * (depth - level))


def reg2bin(beg, end, min_shift, depth):
    """the smallest bin that holds [beg, end): the lowest level whose one bin covers both ends"""
    end -= 1
    for level in range(depth, 0, -1):
        shift = min_shift + 3 * (depth - level)
        if beg >> shift == end >> shift:
            return first_of_level(level) + (beg >> shift)
    return 0


def reg2bins(beg, end, min_shift, depth):
    """every bin that may hold records overlapping [beg, end)"""
    end -= 1
    out = []
    for level in range(depth + 1):
        shift = min_shift + 3 * (depth - level)
        out += range(first_of_level(level) + (beg >> shift), first_of_level(level) + (end >> shift) + 1)
    return out


def _span(rec):
    tid, pos, mapq, flag, cigar = rec[:5]
    return pos, pos + 1 if flag & 4 else pos + max(cigar_lens(cigar)[1], 1)


def index_records(refs, records, min_shift, depth, block=BLOCK, voffs=None):
    """per reference dict(bins {bin: [[cb, ce]]}, loff {bin: loffset}, beg, end, mapped, unmapped), n_no_coor: the bins as
    make_bam_indexed fills a BAI's (consecutive records of one bin extend its last chunk), and each bin's loffset the linear
    index at 2^min_shift tiles, built as make_bam_indexed builds its 16 KB one, at the bin's first tile.  voffs: the records'
    virtual offsets when the BAM is not make_bam's (default: record_voffsets)"""
    if voffs is None:
        voffs = record_voffsets(refs, records, block)
    per_ref = [dict(bins={}, lin={}, beg=None, end=0, mapped=0, unmapped=0, last_bin=None) for _ in refs]
    n_no_coor = 0
    for rec, (v0, v1) in zip(records, voffs):
        tid, pos, mapq, flag = rec[:4]
        if tid < 0:
            n_no_coor += 1
            continue
        s, e = _span(rec)
        R = per_ref[tid]
        b = reg2bin(s, e, min_shift, depth)
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
        for k in range(s >> min_shift, ((e - 1) >> min_shift) + 1):
            R["lin"].setdefault(k, v0)
    out = []
    for R in per_ref:
        n_lin = max(R["lin"]) + 1 if R["lin"] else 0
        lin = [R["lin"].get(k, 0) for k in range(n_lin)]
        for k in range(n_lin - 2, -1, -1):
            if lin[k] == 0:
                lin[k] = lin[k + 1]
        loff = {}
        for b in R["bins"]:
            t = bin_first_tile(b, depth)
            loff[b] = lin[t] if t < n_lin else 0
        out.append(dict(bins=R["bins"], loff=loff, beg=R["beg"], end=R["end"], mapped=R["mapped"], unmapped=R["unmapped"]))
    return out, n_no_coor


def merge_bins(bins, depth, min_dist=MIN_MARKER_DIST):
    """samtools' chunk merging (as region_bams.htslib_merged does it for a BAI): from the leaves up, a bin whose chunks span
    fewer than min_dist compressed bytes moves them into its parent when the parent exists; then each bin's chunks are sorted
    and one that starts in the BGZF block the one before it ends in joins it"""
    bins = {k: [list(c) for c in v] for k, v in bins.items()}
    for level in range(depth, 0, -1):
        for k in sorted(b for b in bins if first_of_level(level) <= b < first_of_level(level + 1)):
            p = sorted(bins[k])
            if (p[-1][1] >> 16) - (p[0][0] >> 16) < min_dist and (k - 1) >> 3 in bins:
                bins[(k - 1) >> 3] += p
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
    return bins


def write_csi(idx, n_no_coor, min_shift, depth, trailer=True, aux=b"") -> bytes:
    """the uncompressed CSI of index_records' output"""
    out = [b"CSI\x01", struct.pack("<iii", min_shift, depth, len(aux)), aux, struct.pack("<i", len(idx))]
    for R in idx:
        has_stats = R["beg"] is not None
        out.append(struct.pack("<i", len(R["bins"]) + has_stats))
        for b in sorted(R["bins"]):
            out.append(struct.pack("<IQi", b, R["loff"].get(b, 0), len(R["bins"][b])))
            out += [struct.pack("<QQ", *c) for c in R["bins"][b]]
        if has_stats:
            out.append(struct.pack("<IQi", stats_bin(depth), 0, 2) + struct.pack("<4Q", R["beg"], R["end"], R["mapped"], R["unmapped"]))
    if trailer:
        out.append(struct.pack("<Q", n_no_coor))
    return b"".join(out)


def bgzf_with_voffsets(payload: bytes, rec_off):
    """(BGZF of an uncompressed BAM payload, the virtual offsets of its records [(start, end)] given as payload offsets)"""
    blocks = []
    bam = _bgzf(payload, blocks)
    return bam, [((blocks[a // BLOCK] << 16) | (a % BLOCK), (blocks[z // BLOCK] << 16) | (z % BLOCK)) for a, z in rec_off]


def make_bam_csi(refs, records, min_shift=14, depth=5, trailer=True, merged=False, min_dist=MIN_MARKER_DIST, aux=b"",
                 with_bai=True, raw=False, sample="sampleA", mates=None):
    """(bam, csi, bai or None) for records sorted by (tid, pos), unplaced last; the BAI is make_bam_indexed's (merged the
    same way when merged), so both describe one file.  raw: the CSI uncompressed.  sample, mates: as make_bam."""
    rec_off = []
    bam, voffs = bgzf_with_voffsets(make_bam(refs, records, sample, mates, _raw=True, _rec_off=rec_off), rec_off)
    idx, n_nc = index_records(refs, records, min_shift, depth, voffs=voffs)
    if merged:
        for R in idx:
            if R["bins"]:
                R["bins"] = merge_bins(R["bins"], depth, min_dist)
    csi = write_csi(idx, n_nc, min_shift, depth, trailer, aux)
    if not raw:
        csi = _bgzf(csi)
    bai = None
    if with_bai:
        bam2, bai = make_bam_indexed(refs, records, sample, mates)
        assert bam2 == bam
    if merged and bai is not None:
        bai = htslib_merged(bai, min_dist)
    return bam, csi, bai


def gunzip(data: bytes) -> bytes:
    out, rest = [], data
    while rest:
        d = zlib.decompressobj(31)
        out.append(d.decompress(rest))
        rest = d.unused_data
    return b"".join(out)


def read_csi(data: bytes):
    """a (compressed) CSI -> dict(min_shift, depth, refs [dict(bins, loff, stats)], n_no_coor or None)"""
    b = gunzip(data)
    assert b[:4] == b"CSI\x01"
    min_shift, depth, l_aux = struct.unpack_from("<iii", b, 4)
    off = 16 + l_aux
    n_ref = struct.unpack_from("<i", b, off)[0]; off += 4
    refs = []
    for _ in range(n_ref):
        n_bin = struct.unpack_from("<i", b, off)[0]; off += 4
        bins, loff, stats = {}, {}, None
        for _ in range(n_bin):
            k, lo, nc = struct.unpack_from("<IQi", b, off); off += 16
            ch = [list(struct.unpack_from("<QQ", b, off + 16 * c)) for c in range(nc)]
            off += 16 * nc
            if k == stats_bin(depth):
                stats = ch
            else:
                bins[k], loff[k] = ch, lo
        refs.append(dict(bins=bins, loff=loff, stats=stats))
    n_nc = struct.unpack_from("<Q", b, off)[0] if off + 8 <= len(b) else None
    return dict(min_shift=min_shift, depth=depth, refs=refs, n_no_coor=n_nc)


def rebuild_linear(loff, min_shift, depth):
    """the 16 KB linear index the library rebuilds from one reference's loffsets: F[x] = the smallest nonzero loffset of
    the bins whose first tile is x, a tile no bin starts in the nearest known value to its left (leading ones the first
    known), |F| = max x + 1; then lin[t] = F[t << (14 - min_shift)] (ceil(|F| / 2^(14 - min_shift)) entries) or
    F[t >> (min_shift - 14)] (|F| << (min_shift - 14) entries)"""
    known = {}
    for b, v in loff.items():
        if v:
            x = bin_first_tile(b, depth)
            if (x << min_shift) < 1 << 31:
                known[x] = min(known.get(x, v), v)
    if not known:
        return []
    xs = sorted(known)
    F, cur = [], known[xs[0]]
    for x in range(xs[-1] + 1):
        cur = known.get(x, cur)
        F.append(cur)
    if min_shift <= 14:
        s = 14 - min_shift
        return [F[t << s] for t in range((len(F) + (1 << s) - 1) >> s)]
    d = min_shift - 14
    return [F[t >> d] for t in range(min(len(F) << d, 1 << 17))]


def max_off(bins, end, min_shift, depth):
    """htslib's max_off at any geometry: the first chunk of the nearest bin with chunks right of the interval, moving right
    along the leaves and up to the parent at a first child; None when there is none"""
    n_bins = stats_bin(depth)
    k = first_of_level(depth) + ((end - 1) >> min_shift) + 1
    while True:
        if k >= n_bins:
            k = 0
        while k % 8 == 1:
            k = (k - 1) >> 3
        if k == 0:
            return None
        if bins.get(k):
            return min(cb for cb, _ in bins[k])
        k += 1


def plan(bins, lin, intervals, min_shift, depth):
    """region_bams.plan at the index's geometry: intervals clamped to [0, min(2^(min_shift + 3 depth), 2^31))"""
    lo, hi = {}, {}
    k_max = min(1 << (min_shift + 3 * depth), 1 << 31)
    for b, e in intervals:
        b, e = max(b, 0), min(e, k_max)
        if e <= b:
            continue
        min_off = lin[min(b >> 14, len(lin) - 1)] if lin else 0
        mx = max_off(bins, e, min_shift, depth)
        mx = (1 << 64) - 1 if mx is None else mx
        for k in reg2bins(b, e, min_shift, depth):
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
