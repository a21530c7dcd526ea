"""GPU BGZF inflate (inflate.cu) against zlib: every DEFLATE block type, long / overlapping matches, code lengths beyond the
primary table, empty members, records straddling members, malformed input."""
import os
import struct
import sys
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bamref  # noqa: E402
from bamutil import cg_mix_records, make_bam_indexed  # noqa: E402


def bgzf(payload: bytes, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, block=0xff00, memlevel=8) -> bytes:
    parts = []
    for i in range(0, max(len(payload), 1), block):
        chunk = payload[i:i + block]
        c = zlib.compressobj(level, zlib.DEFLATED, -15, memlevel, strategy)
        comp = c.compress(chunk) + c.flush()
        bsize = 18 + len(comp) + 8
        assert bsize <= 65536
        parts.append(b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", bsize - 1) + comp)
        parts.append(struct.pack("<II", zlib.crc32(chunk) & 0xffffffff, len(chunk)))
    parts.append(bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000"))      # EOF marker: an empty member
    return b"".join(parts)


def payloads():
    rng = np.random.default_rng(42)
    text = (b"chr20\t1234567\t1234817\t29.87\n" * 4000)
    rand = rng.integers(0, 256, 200_000, dtype=np.uint8).tobytes()
    runs = b"".join(bytes([int(v)]) * int(n) for v, n in zip(rng.integers(0, 256, 3000), rng.integers(1, 600, 3000)))
    skew = rng.choice(np.arange(256, dtype=np.uint8), 300_000, p=np.array([2.0 ** -(i // 8 + 1) for i in range(256)]) / sum(2.0 ** -(i // 8 + 1) for i in range(256))).tobytes()
    period = (bytes(range(7)) * 20000) + (b"ab" * 30000) + (b"x" * 70000)
    return {"text": text, "random": rand, "runs": runs, "skewed": skew, "periodic": period, "tiny": b"A", "empty": b""}


@pytest.mark.parametrize("name", ["text", "random", "runs", "skewed", "periodic", "tiny", "empty"])
@pytest.mark.parametrize("mode", ["default6", "fast1", "best9", "stored", "fixed", "huffman_only", "rle", "small_blocks"])
def test_inflate_equals_zlib(ctx, name, mode):
    data = payloads()[name]
    kw = {"default6": dict(level=6), "fast1": dict(level=1), "best9": dict(level=9), "stored": dict(level=0, block=0xf000),
          "fixed": dict(level=6, strategy=zlib.Z_FIXED), "huffman_only": dict(level=6, strategy=zlib.Z_HUFFMAN_ONLY),
          "rle": dict(level=6, strategy=zlib.Z_RLE), "small_blocks": dict(level=6, block=1000, memlevel=1)}[mode]
    if mode == "stored" and name == "random":
        kw["block"] = 0xf000
    z = bgzf(data, **kw)
    out, status = ctx.bgzf_inflate(z)
    assert (status == 0).all(), status[status != 0][:10]
    assert out == data


def test_inflate_synthetic_bam(ctx, tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
    import glsynth
    bam = str(tmp_path / "s.bam")
    glsynth.write_bam(bam, [("chrA", 1_500_000, 1), ("chrM", 16_569, 24)], coverage=12.0)
    z = open(bam, "rb").read()
    exp = b"".join(zlib.decompress(z[p + 18:p + bs - 8], -15) for p, bs in _members(z))
    out, status = ctx.bgzf_inflate(z)
    assert (status == 0).all() and out == exp and out[:4] == b"BAM\x01"


def _members(z):
    p = 0
    while p + 18 <= len(z):
        bs = struct.unpack_from("<H", z, p + 16)[0] + 1
        yield p, bs
        p += bs


def test_malformed_members_are_flagged(ctx):
    data = payloads()["text"]
    z = bytearray(bgzf(data))
    good, status = ctx.bgzf_inflate(bytes(z))
    assert (status == 0).all()
    # corrupt the deflate payload of the second member: either it decodes to the wrong bytes count / an invalid code (flagged)
    mem = list(_members(bytes(z)))
    p, bs = mem[1]
    z[p + 30:p + 60] = bytes(30)
    out, status = ctx.bgzf_inflate(bytes(z))
    assert status[0] == 0 and status[1] != 0 and (status[2:] == 0).all()
    # a member whose magic is wrong
    z2 = bytearray(bgzf(data))
    z2[0] = 0
    _, status = ctx.bgzf_inflate(bytes(z2))
    assert status[0] == 1


def test_gpu_feeder_equals_generator_and_host_feeder(ctx, tmp_path):
    """gl_bam_decode_device: inflate + parse + filter + CIGAR walk on the device give exactly the generator's segments in BAM
    order, for every reference; the depth text from them equals the host-feeder route"""
    from goleft_b200 import capi
    sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
    import glsynth
    contigs = [("chrA", 2_500_000, 1), ("chrB", 300_000, 2), ("chrM", 16_569, 24)]
    bam = str(tmp_path / "g.bam")
    glsynth.write_bam(bam, contigs, coverage=15.0)
    b = capi.Bam(bam)
    for tid, (nm, L, idx) in enumerate(contigs):
        s, e = glsynth.segments(L, idx, coverage=15.0)
        d = capi.bam_decode_device(ctx, b, tid)
        assert d["n"] == s.size and np.array_equal(d["start"], s) and np.array_equal(d["end"], e), nm
        host = b.decode(tid, want=32)
        assert d["n_records"] == host["n_records"] and d["n_pass"] == host["n_pass"]
    # MAPQ threshold and a BAM made by the Python writer (other record layouts: mates, unplaced reads at the end), against bamref
    p, refs, recs = _handmade_bam(tmp_path)
    b2 = capi.Bam(p)
    for q in (1, 20):
        exp = bamref.segments(recs, len(refs), q)
        for t in range(2):
            d = capi.bam_decode_device(ctx, b2, t, min_mapq=q)
            assert np.array_equal(d["start"], exp[t][0]) and np.array_equal(d["end"], exp[t][1]), (q, t)
    b.close(); b2.close()


def _handmade_bam(tmp_path, cg=False, **layout):
    """(path, refs, records) of an indexed BAM from the Python writer.  cg: a third reference with ultra-long reads stored
    through CG, short reads and the CG edge cases (bamutil.cg_mix_records); layout: BGZF knobs of make_bam_indexed."""
    rng = np.random.default_rng(2)
    refs = [("chrM", 16571), ("chr22", 300001)]
    recs = []
    for t, (nm, L) in enumerate(refs):
        for p0 in np.sort(rng.integers(0, L - 200, 40000)):
            cig = [[(100, "M")], [(45, "M"), (7, "D"), (55, "M")], [(30, "M"), (2, "I"), (68, "M")], [(12, "S"), (88, "M")], [(20, "M"), (300, "N"), (80, "M")],
                   [(50, "="), (1, "X"), (49, "=")]][int(rng.integers(0, 6))]
            recs.append((t, int(p0), int(rng.choice([0, 5, 30, 60])), int(rng.choice([0, 16, 0x400, 0x100, 0x200, 0x800, 4])), cig))
    if cg:
        long_recs, end = cg_mix_records(np.random.default_rng(8), 2)
        refs.append(("chrL", end + 1000))
        recs += long_recs
    recs.append((-1, -1, 0, 4, [(100, "M")]))
    bam_b, bai_b = make_bam_indexed(refs, recs, **layout)
    p = tmp_path / "p.bam"
    p.write_bytes(bam_b); (tmp_path / "p.bam.bai").write_bytes(bai_b)
    return str(p), refs, recs


LAYOUTS = {"default": {}, "members_1000": dict(block=1000), "members_65536": dict(block=65536), "stored": dict(level=0, block=0xff00),
           "sync_flush": dict(flush=(zlib.Z_SYNC_FLUSH, 3001)), "full_flush": dict(flush=(zlib.Z_FULL_FLUSH, 7919))}


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_gpu_decode_cg_reads(ctx, tmp_path, layout):
    """gl_bam_decode_device on ultra-long reads whose CIGAR is in the CG tag (and the CG edge cases) equals bamref, for every
    BGZF layout; the device path is taken (a GL_ESTATE would mean the caller fell back to the host feeder)"""
    from goleft_b200 import capi
    p, refs, recs = _handmade_bam(tmp_path, cg=True, **LAYOUTS[layout])
    b = capi.Bam(p)
    for q in (1, 30):
        exp = bamref.segments(recs, len(refs), q)
        for t, (nm, L) in enumerate(refs):
            d = capi.bam_decode_device(ctx, b, t, min_mapq=q)                # raises GlError(GL_ESTATE) on the fallback
            assert d["n_records"] == sum(1 for r in recs if r[0] == t)
            assert d["n_pass"] == sum(1 for r in recs if r[0] == t and bamref.passes(r, q))
            assert bamref.same_multiset(d["start"], d["end"], *exp[t]), (layout, q, nm)
            assert np.array_equal(bamref.pileup(d["start"], d["end"], 0, L), bamref.pileup(*exp[t], 0, L))
    assert exp[2][0].size > 100_000
    b.close()


# ------------------------------------------------------------------ flush points, window sizes, full-size members
def member(comp: bytes, data: bytes, isize=None) -> bytes:
    """one BGZF member around raw deflate bytes (isize: the ISIZE field to write, default the true size)"""
    bsize = 18 + len(comp) + 8
    assert bsize <= 65536
    return (b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", bsize - 1) + comp +
            struct.pack("<II", zlib.crc32(data) & 0xffffffff, len(data) if isize is None else isize))


def _flushed(data: bytes, mode, points, wbits=15, level=6) -> bytes:
    c = zlib.compressobj(level, zlib.DEFLATED, -wbits)
    out, at = [], 0
    for p in sorted(set(points)):
        out += [c.compress(data[at:p]), c.flush(mode)]
        at = p
    return b"".join(out) + c.compress(data[at:]) + c.flush()


@pytest.mark.parametrize("mode", ["Z_SYNC_FLUSH", "Z_FULL_FLUSH", "Z_PARTIAL_FLUSH", "Z_BLOCK"])
@pytest.mark.parametrize("name", ["text", "random", "runs", "skewed"])
def test_inflate_flush_points(ctx, mode, name):
    """zlib streams cut by flush points at random places, at the first bytes and inside the last few bytes of a member"""
    rng = np.random.default_rng(zlib.crc32((mode + name).encode()))
    data = payloads()[name]
    z, exp = [], []
    for i in range(0, min(len(data), 40 * 0xff00), 0xff00):
        chunk = data[i:i + 0xff00]
        n = len(chunk)
        pts = [int(x) for x in rng.integers(1, n, 12)] + [1, 2, n - 1, n - 2, n - 3, n]
        comp = _flushed(chunk, getattr(zlib, mode), [p for p in pts if 0 < p <= n])
        assert zlib.decompress(comp, -15) == chunk
        z.append(member(comp, chunk)); exp.append(chunk)
    out, status = ctx.bgzf_inflate(b"".join(z))
    assert (status == 0).all(), status
    assert out == b"".join(exp)


@pytest.mark.parametrize("wbits", [9, 10, 11, 12, 13, 14, 15])
def test_inflate_window_bits(ctx, wbits):
    data = payloads()["periodic"][:0xff00] + payloads()["text"][:0xff00]
    z = b"".join(member(_flushed(data[i:i + 0xff00], zlib.Z_NO_FLUSH, [], wbits, 9), data[i:i + 0xff00]) for i in range(0, len(data), 0xff00))
    out, status = ctx.bgzf_inflate(z)
    assert (status == 0).all() and out == data


def test_inflate_isize_65536(ctx):
    """members holding 65536 bytes: the largest ISIZE a BGZF member can have"""
    data = (payloads()["text"] * 2)[:65536 * 3] + payloads()["runs"][:65536]
    z = bgzf(data, block=65536)
    assert all(struct.unpack_from("<I", z, p + bs - 4)[0] == 65536 for p, bs in list(_members(z))[:4])
    out, status = ctx.bgzf_inflate(z)
    assert (status == 0).all() and out == data


# ------------------------------------------------------------------ a hand-written deflate writer: blocks zlib never emits
class BitWriter:
    def __init__(self):
        self.acc, self.n, self.out = 0, 0, bytearray()

    def bits(self, v, n):                                          # LSB first (RFC 1951 3.1.1)
        self.acc |= (v & ((1 << n) - 1)) << self.n
        self.n += n
        while self.n >= 8:
            self.out.append(self.acc & 255); self.acc >>= 8; self.n -= 8

    def code(self, c, n):                                          # Huffman codes go most significant bit first
        self.bits(int("{:0{}b}".format(c, n)[::-1], 2) if n else 0, n)

    def done(self) -> bytes:
        if self.n:
            self.out.append(self.acc & 255)
        return bytes(self.out)


def canonical(lens):
    """RFC 1951 3.2.2: canonical codes from code lengths"""
    count = [0] * 16
    for ln in lens:
        count[ln] += 1
    count[0] = 0
    nxt, code = [0] * 16, 0
    for b in range(1, 16):
        code = (code + count[b - 1]) << 1
        nxt[b] = code
    out = []
    for ln in lens:
        out.append(nxt[ln] if ln else 0)
        if ln:
            nxt[ln] += 1
    return out


def huffman_lengths(freq, limit):
    """code lengths from symbol frequencies (plain Huffman; asserts the limit holds)"""
    import heapq
    items = [(f, i, [s]) for i, (s, f) in enumerate(sorted(freq.items()))]
    if len(items) == 1:
        return {items[0][2][0]: 1}
    heapq.heapify(items)
    depth = {s: 0 for s in freq}
    k = len(items)
    while len(items) > 1:
        f1, _, a = heapq.heappop(items)
        f2, _, b = heapq.heappop(items)
        for s in a + b:
            depth[s] += 1
        heapq.heappush(items, (f1 + f2, k, a + b)); k += 1
    assert max(depth.values()) <= limit
    return depth


LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
             8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


def _len_sym(n):
    i = max(k for k in range(29) if LEN_BASE[k] <= n) if n < 258 else 28
    return 257 + i, n - LEN_BASE[i], LEN_EXTRA[i]


def _dist_sym(d):
    i = max(k for k in range(30) if DIST_BASE[k] <= d)
    return i, d - DIST_BASE[i], DIST_EXTRA[i]


def rle_lengths(lens):
    """the code-length symbols for lens (lit and dist concatenated): 16 repeats a nonzero length, 17 / 18 runs of zeros.
    Runs are not cut at the literal / distance boundary (zlib always cuts them there)."""
    out, i = [], 0
    while i < len(lens):
        v, j = lens[i], i
        while j < len(lens) and lens[j] == v:
            j += 1
        run = j - i
        if v == 0:
            while run >= 11:
                k = min(run, 138); out.append((18, k - 11, 7)); run -= k
            if run >= 3:
                out.append((17, run - 3, 3)); run = 0
            out += [(0, 0, 0)] * run
        else:
            out.append((v, 0, 0)); run -= 1
            while run >= 3:
                k = min(run, 6); out.append((16, k - 3, 2)); run -= k
            out += [(v, 0, 0)] * run
        i = j
    return out


def dynamic_block(bw, items, lit_lens, dist_lens, final=True, cl_seq=None, hclen=None):
    """items: ints (literal bytes) and (length, distance) pairs; lit_lens / dist_lens: the code lengths (HLIT / HDIST are
    their sizes); cl_seq: the code-length symbols to send (default rle_lengths); hclen: code-length code entries to send"""
    cl_seq = rle_lengths(list(lit_lens) + list(dist_lens)) if cl_seq is None else cl_seq
    freq = {}
    for s, _, _ in cl_seq:
        freq[s] = freq.get(s, 0) + 1
    if len(freq) == 1:
        freq[next(s for s in (0, 1, 2) if s not in freq)] = 1     # a complete code-length code needs two symbols
    cll = huffman_lengths({sym: 1 for sym in freq}, 7)                  # equal weights: lengths <= 5
    cl_lens = [cll.get(s, 0) for s in range(19)]
    n_cl = hclen if hclen is not None else max(4, max(i + 1 for i, s in enumerate(CL_ORDER) if cl_lens[s]))
    assert all(cl_lens[CL_ORDER[i]] == 0 for i in range(n_cl, 19))
    bw.bits(1 if final else 0, 1); bw.bits(2, 2)
    bw.bits(len(lit_lens) - 257, 5); bw.bits(len(dist_lens) - 1, 5); bw.bits(n_cl - 4, 4)
    for i in range(n_cl):
        bw.bits(cl_lens[CL_ORDER[i]], 3)
    clc = canonical(cl_lens)
    for s, extra, nb in cl_seq:
        bw.code(clc[s], cl_lens[s]); bw.bits(extra, nb)
    lc, dc = canonical(lit_lens), canonical(dist_lens)
    for it in items:
        if isinstance(it, int):
            bw.code(lc[it], lit_lens[it])
        else:
            s, e, n = _len_sym(it[0]); bw.code(lc[s], lit_lens[s]); bw.bits(e, n)
            s, e, n = _dist_sym(it[1]); bw.code(dc[s], dist_lens[s]); bw.bits(e, n)
    bw.code(lc[256], lit_lens[256])


def expand(items) -> bytes:
    out = bytearray()
    for it in items:
        if isinstance(it, int):
            out.append(it)
        else:
            for _ in range(it[0]):
                out.append(out[-it[1]])
    return bytes(out)


def lens_for(items, n_lit, n_dist, limit=15):
    """Huffman code lengths for the symbols items use (plus end of block), as lists of n_lit / n_dist entries"""
    lf, df = {256: 1}, {}
    for it in items:
        if isinstance(it, int):
            lf[it] = lf.get(it, 0) + 1
        else:
            s = _len_sym(it[0])[0]; lf[s] = lf.get(s, 0) + 1
            s = _dist_sym(it[1])[0]; df[s] = df.get(s, 0) + 1
    ll, dl = huffman_lengths(lf, limit), huffman_lengths(df, limit) if df else {}
    return [ll.get(i, 0) for i in range(n_lit)], [dl.get(i, 0) for i in range(n_dist)]


def handmade_streams():
    rng = np.random.default_rng(11)
    text = [int(x) for x in rng.integers(97, 123, 400)]
    cases = {}
    # a single distance code (length 1, an incomplete code RFC 1951 allows): every match at distance 4
    items = text[:50] + [(int(n), 4) for n in rng.integers(3, 40, 60)] + text[50:80]
    lit, _ = lens_for(items, 286, 4)
    cases["single_distance_code"] = [(items, lit, [0, 0, 0, 1])]
    # literals only: one distance code of length zero
    items = text
    lit, _ = lens_for(items, 257, 1)
    cases["no_distance_codes"] = [(items, lit, [0])]
    # a repeat-16 run from the last literal/length lengths into the distance lengths: lit[258] = 2, dist[0..3] = 2
    lit = [0] * 259
    lit[65], lit[66], lit[256], lit[257], lit[258] = 2, 2, 3, 3, 2
    items = [65, 66, 65, 66, (3, 1), (4, 2), (3, 3), (4, 4), 66, (4, 1)] * 20
    assert (16, 1, 2) in rle_lengths(lit + [2, 2, 2, 2])             # "2" for lit[258], then 16 x4 for dist[0..3]
    cases["repeat16_across_boundary"] = [(items, lit, [2, 2, 2, 2])]
    # 15-bit literal codes: a chain of lengths 1..14 and two codes of length 15
    syms = [97 + k for k in range(14)] + [256, 122]
    lit = [0] * 257
    for k, s in enumerate(syms):
        lit[s] = min(k + 1, 15)
    items = [int(x) for x in rng.choice(syms[:14] + [122], 300)] + [122, 122, 110, 122]
    cases["literal_codes_15_bits"] = [(items, lit, [0])]
    # HLIT = 257 with a five-entry code-length code (16, 17, 18, 0, 8): 256 codes of length 8, byte 255 absent
    lit = [8] * 255 + [0, 8]
    items = [int(x) for x in rng.integers(0, 255, 700)]
    seq = rle_lengths(lit + [0])
    assert {s for s, _, _ in seq} <= {16, 17, 18, 0, 8}
    cases["hlit_257_hclen_5"] = [(items, lit, [0], seq, 5)]
    # length 258 at distance 1 up to 32 KB of output, then matches reaching back 32768 bytes
    head = [int(x) for x in rng.integers(0, 256, 1000)]
    items = head + [(258, 1)] * 124 + [(258, 32768), (3, 32768), (200, 32768), (258, 1)]
    lit, dist = lens_for(items, 286, 30)
    cases["len258_dist1_dist32768"] = [(items, lit, dist)]
    return cases


def _encode(blocks) -> tuple:
    """(deflate bytes, inflated bytes) of a list of dynamic blocks (items, lit_lens, dist_lens[, cl_seq, hclen])"""
    bw = BitWriter()
    items_all = []
    for k, b in enumerate(blocks):
        items, lit, dist = b[:3]
        dynamic_block(bw, items, lit, dist, final=k == len(blocks) - 1, cl_seq=b[3] if len(b) > 3 else None, hclen=b[4] if len(b) > 4 else None)
        items_all += items
    return bw.done(), expand(items_all)


@pytest.mark.parametrize("case", ["single_distance_code", "no_distance_codes", "repeat16_across_boundary", "literal_codes_15_bits",
                                  "hlit_257_hclen_5", "len258_dist1_dist32768"])
def test_inflate_handmade_dynamic_blocks(ctx, case):
    blocks = handmade_streams()[case]
    comp, data = _encode(blocks)
    assert zlib.decompress(comp, -15) == data                        # a valid stream, by zlib
    z = member(comp, data) + bgzf(b"tail" * 100)                      # and one zlib member after it
    out, status = ctx.bgzf_inflate(z)
    assert (status == 0).all(), status
    assert out == data + b"tail" * 100


def test_inflate_handmade_malformed(ctx):
    """inputs whose reads stay inside the member and whose writes the ISIZE checks bound: each must be flagged"""
    bad = []
    # over-subscribed code-length code: three symbols of length 1
    bw = BitWriter(); bw.bits(1, 1); bw.bits(2, 2); bw.bits(0, 5); bw.bits(0, 5); bw.bits(0, 4)
    for ln in (1, 1, 1, 0):
        bw.bits(ln, 3)
    bw.bits(0, 16)
    bad.append((bw.done(), b"x"))
    # HLIT 287 (field 30)
    bw = BitWriter(); bw.bits(1, 1); bw.bits(2, 2); bw.bits(30, 5); bw.bits(0, 5); bw.bits(0, 4); bw.bits(0, 32)
    bad.append((bw.done(), b"x"))
    # distance codes 30 and 31 in a fixed block (after one literal and a length-3 symbol)
    for dcode in (30, 31):
        bw = BitWriter(); bw.bits(1, 1); bw.bits(1, 2)
        bw.code(0x30 + 65, 8)                                          # literal 'A' (fixed code 00110000 + 65)
        bw.code(1, 7)                                                  # symbol 257: length 3
        bw.code(dcode, 5)
        bw.code(0, 7)                                                  # end of block
        bad.append((bw.done(), b"AAAA"))
    # a distance reaching before the start of the output
    bw = BitWriter(); bw.bits(1, 1); bw.bits(1, 2)
    bw.code(0x30 + 65, 8); bw.code(1, 7); bw.code(1, 5); bw.code(0, 7)   # 'A', then length 3 at distance 2
    bad.append((bw.done(), b"AAAA"))
    # ISIZE too small and too large
    good = zlib.compressobj(6, zlib.DEFLATED, -15)
    comp = good.compress(b"hello hello hello") + good.flush()
    z_small = member(comp, b"hello hello hello", isize=5)
    z_large = member(comp, b"hello hello hello", isize=40)
    ok = bgzf(b"fine" * 50)
    z = b"".join(member(c, d) for c, d in bad) + z_small + z_large + ok
    out, status = ctx.bgzf_inflate(z)
    n_bad = len(bad) + 2
    assert (status[:n_bad] != 0).all(), status
    assert (status[n_bad:] == 0).all() and out[-200:] == b"fine" * 50
