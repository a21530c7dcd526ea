"""CPU tests: the depth oracle against the reference's own invariants, and the product's host-side
formatter (gl_depth_format_chunk, no GPU needed) against the oracle's line-by-line walker.

The reference ships no expected outputs for `goleft depth`; what its functional tests pin is
  * depth.bed and callable.bed exactly tile the genome / the BED (depth/functional-test.sh:10-20,48-49),
  * no duplicate rows or regions (functional-test.sh:22-39),
  * window means within 0.5 of an independent per-base count (depth/test/cmp.py:7-16).
Those are the checks below (with tolerance 0: the independent count here is exact).
"""
import numpy as np
import pytest

from goleft_b200 import capi, synth
from oracle import loader as orc

FAI_WINDOWS = [100, 1000000000, 55, 60, 71, 13, 2001]          # functional-test.sh:45-70
BED_WINDOWS = [10, 1000000, 50, 55, 60, 71, 13, 2002]          # functional-test.sh:73-97


def parse_bed(b: bytes):
    rows = []
    for ln in b.decode().splitlines():
        t = ln.split("\t")
        rows.append((t[0], int(t[1]), int(t[2]), t[3]))
    return rows


def assert_tiles(rows, rs, re):
    """bedtools-subtract-both-ways == '' for a single region: rows abut exactly from rs to re."""
    assert rows, "no rows"
    assert rows[0][1] == rs
    for a, b in zip(rows, rows[1:]):
        assert a[2] == b[1], (a, b)
    assert rows[-1][2] == re
    assert len(set(rows)) == len(rows)
    assert len({r[:3] for r in rows}) == len(rows)


def random_depth(rng, n, p_zero=0.3, hi=12):
    """piecewise-constant-ish per-base depth with gaps"""
    d = np.zeros(n, np.int32)
    x = 0
    while x < n:
        ln = int(rng.integers(1, 40))
        v = 0 if rng.random() < p_zero else int(rng.integers(1, hi))
        d[x:x + ln] = v
        x += ln
    return d


# ------------------------------------------------------------------ region parsing (depth.go:73-100)
@pytest.mark.parametrize("line,exp", [
    ("chr1:1-10000000", ("chr1", 0, 10000000)),
    ("chr22\t14250\t15500\n", ("chr22", 14250, 15500)),
    ("HLA-A*01:01:01:01:1-3000", ("HLA-A*01:01:01:01", 0, 3000)),      # functional-test.sh:118
    # reference quirk: in a BED line the lazy group stops at the FIRST ":digits<TAB>digits" it can use
    ("HLA-A*01:01:01:01\t5\t38\textra", ("HLA-A*01:01:01", 1, 5)),
    ("chr1\t5\t38\textra", ("chr1", 5, 38)),
    ("chrM:0-5", ("chrM", 0, 5)),                                      # max(istart,0), depth.go:93
    ("GL000207.1:17-4262", ("GL000207.1", 16, 4262)),
])
def test_region_regex(line, exp):
    assert orc.chrom_start_end(line) == exp


def test_region_regex_rejects():
    with pytest.raises(ValueError):
        orc.chrom_start_end("no_region_here")


# ------------------------------------------------------------------ chunking (depth.go:122-159)
def test_chunks():
    assert orc.gen_chunks(16571, 100) == [(0, 16571)]
    ch = orc.gen_chunks(64_444_167, 500)
    assert len(ch) == 7 and ch[0] == (0, 10_000_000) and ch[-1] == (60_000_000, 64_444_167)
    # step is rounded down to a multiple of W (depth.go:132)
    ch = orc.gen_chunks(25_000_000, 2001)
    step = 10_000_000 // 2001 * 2001
    assert ch[0] == (0, step) and ch[1] == (step, 2 * step) and ch[-1][1] == 25_000_000
    # W larger than the step: one chunk per W
    assert orc.gen_chunks(20001, 1_000_000_000) == [(0, 20001)]


# ------------------------------------------------------------------ per-base counting
def test_pileup_diff_equals_bruteforce():
    rng = np.random.default_rng(1)
    for rs, re in [(0, 5000), (1234, 9000), (77, 78)]:
        n = 3000
        s = rng.integers(-200, 9500, n).astype(np.int32)
        e = (s + rng.integers(1, 400, n)).astype(np.int32)
        a = orc.pileup_brute(s, e, rs, re)
        b = orc.pileup_diff(s, e, rs, re)
        assert np.array_equal(a, b)
        # numpy third opinion
        x = np.arange(rs, re)
        c = ((s[None, :] <= x[:, None]) & (x[:, None] < e[None, :])).sum(1) if (re - rs) * n < 5e7 else a
        assert np.array_equal(a, c)


@pytest.mark.parametrize("W", [1, 3, 16, 500, 4096, 10 ** 7, 2 ** 30])
def test_oracle_at_top_of_int32(W):
    """the GPU tests at the top of the int32 range (test_depth_int32_top_gpu.py) rest on the oracle there: its per-base
    counts, window sums / minima and class runs against a numpy int64 restatement, for regions ending at INT32_MAX whose
    genome-aligned last window ends past it, reads that end on INT32_MAX and forced run breaks inside the region"""
    top = 2 ** 31 - 1
    rng = np.random.default_rng(W)
    for rs, re in [(top - 3 * 4096 - 4095, top), (top - 13_000, top - 1), (2 ** 31 - 4096 - 3 * 4096, 2 ** 31 - 4095)]:
        s = rng.integers(rs - 300, re, 2500)
        e = np.minimum(s + rng.integers(-5, 300, s.size), top)
        s[:4] = [top - 1, top - 255, top - 4096, rs - 10]
        e[:4] = top
        s32, e32 = s.astype(np.int32), e.astype(np.int32)
        x = np.arange(rs, re, dtype=np.int64)
        lo, hi = np.clip(s, rs, re), np.clip(e, rs, re)
        live = lo < hi
        diff = np.zeros(re - rs + 1, np.int64)
        np.add.at(diff, lo[live] - rs, 1)
        np.add.at(diff, hi[live] - rs, -1)
        depth = np.cumsum(diff)[:-1]
        assert np.array_equal(orc.pileup_diff(s32, e32, rs, re), depth)
        assert np.array_equal(orc.pileup_brute(s32, e32, rs, re), depth)
        # windows k = rs//W .. (re-1)//W over [max(rs, kW), min(re, (k+1)W)); with re = INT32_MAX the last one's genome end
        # is past it for every W here except 1
        k = np.arange(rs // W, (re - 1) // W + 1, dtype=np.int64)
        assert re != top or W == 1 or (k[-1] + 1) * W > top
        edge = np.maximum(k * W, rs) - rs
        ws, wm = orc.window_sums(depth, rs, re, W)
        assert np.array_equal(ws, np.add.reduceat(depth, edge))
        assert np.array_equal(wm, np.minimum.reduceat(depth, edge))
        for mincov, maxmean, brk in [(4, 0, 0), (1, 6, 4096), (3, 8, 999), (2, 0, W)]:
            cls = np.where(depth == 0, 0, np.where(depth < mincov, 1, np.where((maxmean > 0) & (depth >= maxmean), 3, 2)))
            new = np.ones(x.size, bool)
            new[1:] = cls[1:] != cls[:-1]
            if brk:
                new |= x % brk == 0
            ra, rc = orc.class_runs(depth, rs, re, mincov, maxmean, brk)
            assert np.array_equal(ra, x[new]) and np.array_equal(rc, cls[new])
        # the walker's rows end on the region end
        hd, ca = orc.walk_chunk("big", rs, re, W, 4, 0, depth)
        assert parse_bed(hd)[-1][2] == re and parse_bed(ca)[-1][2] == re


def test_synth_segments_shape():
    r = synth.reads(2_000_000)
    s, e = synth.segments(r)
    assert s.size == e.size and (e > s).all()
    ok = ((r.flag & 0x704) == 0) & (r.mapq >= 1)
    n_del = int((r.kind[ok] == 1).sum())
    assert s.size == int(ok.sum()) + n_del
    # roughly 30x less the filtered ~18%
    d = orc.pileup_diff(s, e, 0, 2_000_000)
    assert 20 < d.mean() < 30
    assert d[int(0.41 * 2_000_000)] == 0              # the gap
    assert d[int(0.70 * 2_000_000) + 50] > 100        # the pile-up


# ------------------------------------------------------------------ walker invariants, fai mode
@pytest.mark.parametrize("W", FAI_WINDOWS)
def test_walker_tiles_fai_mode(W):
    rng = np.random.default_rng(W)
    L = 20001
    depth = random_depth(rng, L)
    hd, ca = orc.walk_chunk("chr22", 0, L, W, 4, 0, depth)
    hrows, crows = parse_bed(hd), parse_bed(ca)
    assert_tiles(hrows, 0, L)
    assert_tiles(crows, 0, L)
    for _, s, e, v in hrows:
        assert float(v) == float("%.4g" % (depth[s:e].sum() / (e - s)))       # cmp.py with tolerance 0
    for _, s, e, c in crows:
        d = depth[s:e]
        if c == "NO_COVERAGE":
            assert (d == 0).all()
        elif c == "LOW_COVERAGE":
            assert ((d > 0) & (d < 4)).all()
        else:
            assert c == "CALLABLE" and (d >= 4).all()
    # adjacent callable rows differ in class (pure run-length encoding)
    for a, b in zip(crows, crows[1:]):
        assert a[3] != b[3]


def test_walker_empty_chunk():
    """check_empty (functional-test.sh:102-115): an empty BAM still tiles."""
    for rs, re, W in [(0, 16571, 10), (100, 1000, 10), (1, 3, 10), (16, 17, 50)]:
        hd, ca = orc.walk_chunk("chrM", rs, re, W, 4, 0, np.zeros(re - rs, np.int32))
        assert_tiles(parse_bed(hd), rs, re)
        assert parse_bed(ca) == [("chrM", rs, re, "NO_COVERAGE")]
        assert all(r[3] == "0" for r in parse_bed(hd))


def test_walker_excessive_class_and_mincov():
    depth = np.array([0, 1, 3, 4, 9, 10, 50, 0, 0, 7], np.int32)
    _, ca = orc.walk_chunk("c", 0, 10, 5, 4, 10, depth)
    assert parse_bed(ca) == [("c", 0, 1, "NO_COVERAGE"), ("c", 1, 3, "LOW_COVERAGE"), ("c", 3, 5, "CALLABLE"),
                             ("c", 5, 7, "EXCESSIVE_COVERAGE"), ("c", 7, 9, "NO_COVERAGE"), ("c", 9, 10, "CALLABLE")]


def test_walker_text_source_equals_array_source():
    rng = np.random.default_rng(7)
    for rs, re, W in [(0, 5000, 100), (1575, 15800, 10), (14250, 15500, 71), (24, 29, 13)]:
        depth = random_depth(rng, re - rs)
        a = orc.walk_chunk("chr22", rs, re, W, 4, 0, depth)
        txt = orc.samtools_text("chr22", rs, re, depth)
        assert txt.split(b"\n", 1)[0] == b"chr22:%d-%d" % (rs + 1, re)
        b = orc.walk_text(txt, W, 4, 0)
        assert a == b


# ------------------------------------------------------------------ bed mode: rows cover the region; quirks Q2/Q3 are reproduced
@pytest.mark.parametrize("W", BED_WINDOWS)
def test_walker_bed_mode_covers_region(W):
    rng = np.random.default_rng(100 + W)
    regions = [(14250, 15500), (1575, 15800), (100, 1000), (2000, 5000), (1, 3), (9, 13), (16, 17), (24, 29), (39, 43)]
    for rs, re in regions:                                                    # depth/test/windows.bed
        depth = random_depth(rng, re - rs)
        hd, ca = orc.walk_chunk("chrM", rs, re, W, 4, 0, depth)
        assert_tiles(parse_bed(ca), rs, re)
        rows = parse_bed(hd)
        # bedtools subtract both ways == "" : union of rows == region (rows may overlap after quirk Q3)
        cov = np.zeros(re - rs, bool)
        for _, s, e, _v in rows:
            assert rs <= s < e <= re
            cov[s - rs:e - rs] = True
        assert cov.all()
        # adjacent duplicates are what check_uniq tests in bed mode (functional-test.sh:29-32)
        assert all(a != b for a, b in zip(rows, rows[1:]))


def test_walker_quirk_q2_q3_pinned():
    """Last covered base inside the chunk's leading partial window: misaligned end, then a re-emitted
    overlapping window (depth.go:330-339,351).  Restated by hand from the cited lines."""
    rs, re, W = 1575, 15800, 1000
    depth = np.zeros(re - rs, np.int32)
    depth[1600 - rs] = 5          # pos 1600 lies in window [1000,2000) whose start precedes rs
    hd, _ = orc.walk_chunk("chr22", rs, re, W, 4, 0, depth)
    rows = parse_bed(hd)
    # :332-333  s=max(1000,1575)=1575 ; e=min(re, 1575+1000)=2575  -> mean 5/1000
    assert rows[0] == ("chr22", 1575, 2575, "0.005")
    # :351 ds = max(rs,pos=2575)/W*W = 2000 -> window (2000,3000) overlaps the previous row
    assert rows[1] == ("chr22", 2000, 3000, "0")
    assert rows[-1] == ("chr22", 15000, 15800, "0")


# ------------------------------------------------------------------ product host formatter == oracle walker
def _summaries(depth, rs, re, W, mincov, maxmean):
    s, _ = orc.window_sums(depth, rs, re, W)
    a, c = orc.class_runs(depth, rs, re, mincov, maxmean, 0)
    return s, a, c


@pytest.mark.parametrize("seed", range(6))
def test_format_chunk_equals_walker_random(seed):
    rng = np.random.default_rng(seed)
    for _ in range(60):
        rs = int(rng.integers(0, 3000))
        re = rs + int(rng.integers(1, 4000))
        W = int(rng.choice([1, 2, 7, 10, 13, 50, 55, 71, 100, 250, 1000, 2002, 10 ** 6, 10 ** 9]))
        mincov = int(rng.integers(1, 6))
        maxmean = int(rng.choice([0, 0, 8]))
        pz = float(rng.choice([0.0, 0.3, 0.9, 1.0]))
        depth = random_depth(rng, re - rs, p_zero=pz)
        # make the tail behaviour vary: sometimes only the first few bases are covered
        if rng.random() < 0.3:
            depth[int(rng.integers(1, 30)):] = 0
        exp = orc.walk_chunk("chr1", rs, re, W, mincov, maxmean, depth)
        s, a, c = _summaries(depth, rs, re, W, mincov, maxmean)
        got = capi.format_chunk("chr1", rs, re, W, s, a, c)
        assert got[0] == exp[0], (rs, re, W)
        assert got[1] == exp[1], (rs, re, W)


def test_format_chunk_large_values_and_names():
    depth = np.full(1000, 123456, np.int32)
    depth[500:] = 7
    for chrom in ["HLA-A*01:01:01:01", "chrUn_KI270742v1"]:
        exp = orc.walk_chunk(chrom, 0, 1000, 250, 4, 0, depth)
        s, a, c = _summaries(depth, 0, 1000, 250, 4, 0)
        assert capi.format_chunk(chrom, 0, 1000, 250, s, a, c) == exp
    assert b"1.235e+05" in exp[0]          # %.4g switches to exponent form at >= 1e4 with 4 digits


def test_go_g_format_table():
    """Go's %.4g == C's %.4g on the values this path prints (SURVEY.md §8c): spot table restated from
    strconv's rules (shortest of %e/%f, exponent < -4 or >= precision uses %e, >= 2 exponent digits)."""
    table = {0.0: "0", 30.0: "30", 29.96: "29.96", 1234.5: "1234", 1234.6: "1235", 12345.0: "1.234e+04",
             0.005: "0.005", 0.00001234: "1.234e-05", 608.2: "608.2", 1101.0: "1101", 100000.0: "1e+05",
             0.5: "0.5", 2.0 / 3.0: "0.6667", 99995.0: "9.999e+04" if "%.4g" % 99995.0 == "9.999e+04" else "1e+05"}
    for v, exp in table.items():
        assert "%.4g" % v == exp, v


# ------------------------------------------------------------------ the feeder's packed16 format (host-only)
def _unpack16(a, o, ln):
    st = np.repeat(a.astype(np.int64), 256) + o
    en = st + ln
    keep = ln > 0
    return st[keep], en[keep]


def test_pack_segments16_roundtrip():
    rng = np.random.default_rng(9)
    # BAM-like: nearly sorted, a sparse stretch, long segments that must be split, empties that are dropped
    s = np.sort(rng.integers(0, 3_000_000, 50_000)).astype(np.int32)
    s[20_000:] += 50_000_000
    e = (s + rng.integers(1, 300, s.size)).astype(np.int32)
    s[1000], e[1000] = s[1000], s[1000] + 200_000            # split into 65535-base pieces
    e[2000] = s[2000]                                        # empty
    s[3000] = s[2999] - 9000                                 # starts earlier than its predecessor (fits below the anchor)
    e[3000] = s[3000] + 100
    a, o, ln = capi.pack_segments16(s, e)
    assert o.size == a.size * 256 and ln.dtype == np.uint16
    st, en = _unpack16(a, o, ln)
    # same multiset of covered bases: compare per-base depth over a window that contains everything interesting
    for lo, hi in [(0, 3_100_000), (50_000_000, 53_100_000)]:
        assert np.array_equal(orc.pileup_diff(st.astype(np.int32), en.astype(np.int32), lo, hi), orc.pileup_diff(s, e, lo, hi))
    assert a.size <= s.size // 256 + 8                       # nearly every block is full
    assert capi.pack_segments16(np.zeros(0, np.int32), np.zeros(0, np.int32))[0].size == 0


def test_faidx_stats_restatement_hand_cases():
    """Faidx.Stats as restated (un-vendored brentp/faidx, parity unpinned): hand-computed cases incl. its edge
    behaviours — newline between C and G is not a CpG, the byte after the window decides the last CpG, the very last base
    of a file with no trailing byte is dropped."""
    fa = b">c\nACGT\nCGcg\nNNNN\nccgC\nG"
    rec = (3, 17, 4, 5)                                       # offset, length, bases/line, bytes/line
    st = orc.faidx_stats(fa, rec, 0, 4)                       # ACGT, next byte '\n': A,C(G follows ->cpg),G,T
    assert np.allclose(st, [0.5, 2 * 1 / 4, 0.0])
    st = orc.faidx_stats(fa, rec, 2, 6)                       # G T \n C G: T|C line break; CG inside line 2
    assert np.allclose(st, [3 / 4, 2 * 1 / 4, 0.0])
    st = orc.faidx_stats(fa, rec, 3, 5)                       # T \n C + lookahead G -> cpg
    assert np.allclose(st, [1 / 2, 2 * 1 / 2, 0.0])
    st = orc.faidx_stats(fa, rec, 4, 8)                       # CGcg: C-G, c-g; masked 2/4; last g followed by \n
    assert np.allclose(st, [1.0, 2 * 2 / 4, 0.5])
    st = orc.faidx_stats(fa, rec, 8, 12)                      # NNNN: nothing counted
    assert np.allclose(st, [0, 0, 0])
    st = orc.faidx_stats(fa, rec, 12, 16)                     # ccgC then '\n': C at line end, G on next line: not a CpG
    assert np.allclose(st, [1.0, 2 * 1 / 4, 3 / 4])
    st = orc.faidx_stats(fa, rec, 16, 17)                     # last base, no byte after it in the file: dropped
    assert np.allclose(st, [0, 0, 0])
    st = orc.faidx_stats(fa, rec, 12, 17)                     # ... but it still is the look-ahead of the byte before
    assert np.allclose(st, [1.0, 2 * 1 / 4, 3 / 4])
    assert orc.faidx_stats(fa, rec, 0, 18) is None            # faidx panics past the contig
    assert orc.stats_text(np.array([0.5, 0.04166, 1.0])) == b"\t0.5\t0.0417\t1"


def test_pack_segments8_roundtrip():
    """packed8 (uint8 start delta + uint8 length per slot): the decoded pieces are in start order and give the
    oracle's per-base depth — short reads in BAM order (a quarter of the int32 bytes), and the awkward inputs: long
    segments (cut in 255-base pieces), gaps (filler slots / new blocks), negative starts, shuffled order, empties."""
    L = 1_000_000
    s, e = synth.segments(synth.reads(L, contig_index=4))
    a, d, ln = capi.pack_segments8(s, e)
    assert a.size * 132 < 0.27 * s.size * 8
    s2, e2 = capi.unpack_segments8(a, d, ln)
    assert (np.diff(s2) >= 0).all() and s2.size == s.size
    assert np.array_equal(orc.pileup_diff(s, e, 0, L), orc.pileup_diff(s2.astype(np.int32), e2.astype(np.int32), 0, L))
    rng = np.random.default_rng(0)
    s = np.concatenate([rng.integers(-300, 5000, 300), rng.integers(10_000_000, 10_001_000, 50), [2_000_000_000]]).astype(np.int32)
    e = (s + rng.choice([0, 1, 5, 150, 255, 256, 1000, 70000], s.size)).astype(np.int32)
    e[-1] = s[-1] + 100
    a, d, ln = capi.pack_segments8(s, e)
    s2, e2 = capi.unpack_segments8(a, d, ln)
    assert (e2 - s2).max() <= 255 and (np.diff(s2) >= 0).all()
    for rs, re in [(0, 100000), (9_990_000, 10_100_000), (1_999_999_000, 2_000_001_000)]:
        assert np.array_equal(orc.pileup_brute(s, e, rs, re), orc.pileup_brute(s2.astype(np.int32), e2.astype(np.int32), rs, re))
    p = rng.permutation(s.size)                                   # order does not matter
    a3, d3, l3 = capi.pack_segments8(s[p], e[p])
    s3, e3 = capi.unpack_segments8(a3, d3, l3)
    assert np.array_equal(np.sort(s3), np.sort(s2)) and (e3 - s3).sum() == (e2 - s2).sum()
    assert capi.pack_segments8(np.zeros(0, np.int32), np.zeros(0, np.int32))[0].size == 0


def test_chunk_rows_match_the_formatted_text():
    """gl_depth_chunk_rows (what --stats computes GC/CpG/masked for) lists exactly the (s, e) of the rows
    gl_depth_format_chunk prints, quirk rows included (misaligned last window, re-emitted window: depth.go:329-358)."""
    rng = np.random.default_rng(21)
    for _ in range(400):
        W = int(rng.choice([1, 7, 10, 50, 100, 1000]))
        rs = int(rng.integers(0, 3000))
        re = rs + int(rng.integers(1, 2500))
        depth = np.zeros(re - rs, np.int32)
        for _ in range(int(rng.integers(0, 4))):                    # a few covered stretches, often ending early
            a = int(rng.integers(0, re - rs)); b = min(re - rs, a + int(rng.integers(1, 600)))
            depth[a:b] += int(rng.integers(1, 9))
        es, _ = orc.window_sums(depth, rs, re, W)
        ea, ec = orc.class_runs(depth, rs, re, 4, 0, 0)
        hd, _ = capi.format_chunk("c", rs, re, W, es, ea, ec)
        s, e = capi.chunk_rows(rs, re, W, ea, ec)
        rows = [ln.split(b"\t") for ln in hd.splitlines()]
        assert [int(r[1]) for r in rows] == s.tolist() and [int(r[2]) for r in rows] == e.tolist()
        assert hd == orc.walk_chunk("c", rs, re, W, 4, 0, depth)[0]


def test_pack_segments8_mt_same_pieces():
    """the parallel packer yields sorted anchors and the same multiset of pieces as the single-threaded one"""
    from goleft_b200 import capi, synth
    for L, cov, idx in ((3_000_000, 30.0, 1), (500_000, 200.0, 2), (2_000_000, 2.0, 3)):
        s, e = synth.segments(synth.reads(L, coverage=cov, contig_index=idx))
        a1, d1, l1 = capi.pack_segments8(s, e)
        u1s, u1e = capi.unpack_segments8(a1, d1, l1)
        o1 = np.lexsort((u1e, u1s))
        for T in (0, 2, 3, 8):
            a2, d2, l2 = capi.pack_segments8(s, e, threads=T)
            assert (np.diff(a2) >= 0).all()
            u2s, u2e = capi.unpack_segments8(a2, d2, l2)
            o2 = np.lexsort((u2e, u2s))
            assert np.array_equal(u1s[o1], u2s[o2]) and np.array_equal(u1e[o1], u2e[o2])
            # every block's starts stay within [anchor, next anchor]
            st = a2.astype(np.int64)[:, None] + np.cumsum(d2.reshape(-1, 64).astype(np.int64), axis=1)
            assert (st[:-1].max(axis=1) <= a2[1:]).all()
    # long segments and wild disorder still decode to the same coverage
    rng = np.random.default_rng(0)
    s = rng.integers(0, 1_000_000, 50_000).astype(np.int32)
    e = (s + rng.integers(1, 5000, s.size)).astype(np.int32)
    a2, d2, l2 = capi.pack_segments8(s, e, threads=4)
    assert (np.diff(a2) >= 0).all()
    u2s, u2e = capi.unpack_segments8(a2, d2, l2)
    assert int((u2e - u2s).sum()) == int((e.astype(np.int64) - s).sum())
    assert np.array_equal(orc.pileup_diff(u2s.astype(np.int32), u2e.astype(np.int32), 0, 1_010_000), orc.pileup_diff(s, e, 0, 1_010_000))


def test_pack16_fixed_roundtrip():
    """host-only: fixed-block packed16 (gl_pack_segments16_fixed_mt) decodes to the input's segments, in order; blocks that do not
    fit 16 bits come back raw in the escape list"""
    from goleft_b200 import capi
    rng = np.random.default_rng(2)
    for n in (0, 1, 255, 256, 257, 100_000):
        s = np.sort(rng.integers(0, 3_000_000, n)).astype(np.int32)
        e = (s + rng.integers(-3, 200, n)).astype(np.int32)
        if n > 1000:
            s[5000:5300] += 2_000_000                            # a gap inside a block
            e[5000:5300] += 2_000_000
            e[777] = s[777] + 70_000                             # one long segment
        for thr in (1, 3):
            a, o, ln, es, ee = capi.pack_segments16_fixed(s, e, threads=thr)
            nb = (n + 255) // 256
            assert a.size == nb and o.size == nb * 256
            S = (np.repeat(a.astype(np.int64), 256) + o)[:n]
            E = S + ln[:n]
            escaped = np.repeat(ln.reshape(-1, 256).max(1) == 0, 256)[:n] if n else np.zeros(0, bool)
            live = e > s
            keep = ~escaped & live
            assert np.array_equal(S[keep], s[keep]) and np.array_equal(E[keep], e[keep])
            assert np.all(ln[:n][~escaped & ~live] == 0)
            assert np.all(ln[n:] == 0)
            # a block is escaped only when it has to be ... or holds no live segment at all (then it is empty either way)
            m = escaped & live
            assert np.array_equal(es, s[m]) and np.array_equal(ee, e[m])
            if n > 1000:
                assert 0 < es.size < 2000
    with pytest.raises(capi.GlError):
        s = np.arange(0, 100_000 * 1000, 100_000, dtype=np.int32)
        capi.pack_segments16_fixed(s, s + 10, esc_cap=10)


def test_host_pool_small_jobs_and_thread_limits():
    """host-only: the library's thread pool (a job is complete when its TASKS are done; workers that sat out a job sleep; a
    small job wakes only the first 16 workers) under back-to-back small jobs with changing thread limits, over-subscribed on
    purpose (GL_THREADS=40): every range call of the fixed-block packer must give the single-threaded bytes."""
    import os
    import subprocess
    import sys
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = r'''
import ctypes as C, sys, time
import numpy as np
sys.path.insert(0, %r)
from goleft_b200 import capi
rng = np.random.default_rng(5)
n = 3_000_001
s = np.sort(rng.integers(0, 40_000_000, n)).astype(np.int32)
e = (s + rng.integers(1, 200, n)).astype(np.int32)
ref = capi.pack_segments16_fixed(s, e, threads=1)
nb = (n + 255) // 256
a = np.zeros(nb, np.int32); o = np.zeros(nb * 256, np.uint16); l = np.zeros(nb * 256, np.uint16)
es = np.zeros(n, np.int32); ee = np.zeros(n, np.int32)
m = C.c_int64(0)
L = capi.lib
L.gl_pack_segments16_fixed_range_mt.argtypes = [C.c_void_p, C.c_void_p, C.c_int64, C.c_int64, C.c_int64, C.c_int32] + [C.c_void_p] * 5 + [C.c_int64, C.POINTER(C.c_int64)]
assert L.glhost_pool_size() == 40
for rep in range(120):
    K = 1 + rep %% 23
    thr = [0, 16, 3, 40, 8, 17, 1][rep %% 7]
    a[:] = 0; o[:] = 0; l[:] = 0; m.value = 0
    for c in range(K):
        rc = L.gl_pack_segments16_fixed_range_mt(s.ctypes.data, e.ctypes.data, n, nb * c // K, nb * (c + 1) // K, thr, a.ctypes.data, o.ctypes.data,
                                                 l.ctypes.data, es.ctypes.data, ee.ctypes.data, n, C.byref(m))
        assert rc == 0
    if rep %% 10 == 0:
        time.sleep(0.005)                       # let the workers fall asleep: the next job has to wake them
    assert np.array_equal(a, ref[0]) and np.array_equal(o, ref[1]) and np.array_equal(l, ref[2]) and np.array_equal(es[:m.value], ref[3]), rep
print("ok")
''' % ROOT
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, GL_THREADS="40"), timeout=300)
    assert p.returncode == 0 and p.stdout.strip().endswith("ok"), p.stderr[-2000:]
