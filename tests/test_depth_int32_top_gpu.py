"""The depth paths at the top of the int32 coordinate range, against oracle/oracle_depth.c (int64 position arithmetic
throughout; test_oracle_depth.py pins it there against a numpy restatement).  A BAM reference may be 2^31-1 bases long
and gl_depth_begin takes any region end up to INT32_MAX: the region's last tile then starts at or above 2^31 - 4096,
so tile start + 4096 no longer fits an int; genome-aligned windows end past INT32_MAX; and `goleft depth` splits such a
contig into passes of at most 2^30-1 bases.  Needs an H100 (`-m gpu`)."""
import os
import subprocess
import sys

import numpy as np
import pytest

from goleft_b200 import capi
from oracle import loader as orc
from test_depth_gpu import check_region, rand_segments

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bamref  # noqa: E402
from bamutil import make_bam  # noqa: E402

pytestmark = pytest.mark.gpu

TOP = 2 ** 31 - 1                         # INT32_MAX: the largest region end, the end of a 2^31-1 base contig
TILE = 4096
LAST_TILE = 2 ** 31 - TILE                # a tile that starts here or later would end past INT32_MAX
RE_TOP = [TOP, TOP - 1, 2 ** 31 - 4095, 2 ** 31 - 4096, 2 ** 31 - 4097]
WINDOWS = [1, 3, 16, 500, 1000, 4096, 10 ** 7, 2 ** 30]


def step_for(W):
    return max(1, 10_000_000 // W) * W    # the CLI's chunk (depth/depth.go:132)


def last_tile_starts(re):
    """starts of a region's last tile that end at re: exactly 2^31 - 4096, inside the top 4096 bases (incl. a one-base
    last tile), and just below them"""
    c = [LAST_TILE, LAST_TILE + 777, re - 1, LAST_TILE - 1, LAST_TILE - 300]
    return sorted({t for t in c if 1 <= re - t <= TILE})


def region_for(t_last):
    """three full tiles and a ragged (or full) last one that starts at t_last"""
    return t_last - 3 * TILE


def top_segments(rng, rs, re, n=2500, maxlen=300):
    """sorted int32 (start, end) around [rs, re): random reads; reads that end exactly at INT32_MAX; reads that start in the
    last 255 bases (one packed8 piece each); reads across rs; reads that clip to nothing (before rs, empty, reversed)"""
    parts = [tuple(x.astype(np.int64) for x in rand_segments(rng, n, rs - 400, re - maxlen, maxlen=maxlen))]
    k = np.array([1, 2, 100, 254, 255, 256, 300, 4095, 4096, 4097, 9000], np.int64)
    parts.append((TOP - k, np.full(k.size, TOP, np.int64)))
    s = TOP - rng.integers(1, 256, 60)
    parts.append((s, s + rng.integers(1, TOP - s + 1)))
    s = rs - rng.integers(1, 300, 40)
    parts.append((s, rs + rng.integers(-5, 300, 40)))
    s = rs - rng.integers(300, 2000, 20)
    parts.append((s, s + rng.integers(-10, 200, 20)))
    s = np.concatenate([p[0] for p in parts])
    e = np.concatenate([p[1] for p in parts])
    o = np.argsort(s, kind="stable")
    s, e = s[o], e[o]
    assert s.min() >= 0 and e.max() == TOP
    return s.astype(np.int32), e.astype(np.int32)


@pytest.mark.parametrize("re", RE_TOP)
def test_region_end_at_top(ctx, re):
    """every path, with the region's last tile at, inside and just below the top 4096 bases of int32"""
    rng = np.random.default_rng(re & 0xffff)
    for t_last in last_tile_starts(re):
        rs = region_for(t_last)
        s, e = top_segments(rng, rs, re)
        for W in (500, 16):
            check_region(ctx, s, e, rs, re, W, mincov=4, maxmean=30, run_break=TILE)


@pytest.mark.parametrize("W", WINDOWS)
def test_windows_past_int32_max(ctx, W):
    """genome-aligned windows whose end exceeds INT32_MAX (W = 2^30 and re = 2^31-1: the last window is [2^30, 2^31)),
    with class thresholds that change inside the top tiles and forced run breaks that fall in them"""
    rng = np.random.default_rng(W)
    for re, t_last in ((TOP, LAST_TILE), (TOP, TOP - 1), (2 ** 31 - 4095, LAST_TILE), (TOP - 1, LAST_TILE - 1)):
        rs = region_for(t_last)
        s, e = top_segments(rng, rs, re, n=700)
        for (mincov, maxmean), run_break in zip(((4, 0), (1, 6), (3, 8)), (step_for(W), TILE, 999)):
            check_region(ctx, s, e, rs, re, W, mincov=mincov, maxmean=maxmean, run_break=run_break)


def test_interval_sums_at_top(ctx):
    """gl_depth_interval_sums over intervals that reach INT32_MAX: with the fused path's cell index, and from the segments
    alone after the general paths"""
    rng = np.random.default_rng(17)
    re = TOP
    rs = region_for(LAST_TILE)
    s, e = top_segments(rng, rs, re)
    depth = orc.pileup_diff(s, e, rs, re).astype(np.int64)
    cs = np.concatenate([[0], np.cumsum(depth)])
    a = rng.integers(rs - 500, re, 3000)
    b = np.minimum(a + rng.choice([0, 1, 2, 99, 255, 4096, 4097, 70_000], a.size), TOP)
    special = [(rs, re), (re - 1, TOP), (LAST_TILE, TOP), (LAST_TILE - 1, LAST_TILE + 1), (TOP - 255, TOP), (rs - 50, rs + 1),
               (TOP, TOP), (TOP - 1, TOP - 1)]
    a[:len(special)] = [x for x, _ in special]
    b[:len(special)] = [y for _, y in special]
    ac, bc = np.clip(a, rs, re), np.clip(b, rs, re)
    exp = np.where(bc > ac, cs[np.maximum(bc, ac) - rs] - cs[ac - rs], 0)
    a, b = a.astype(np.int32), b.astype(np.int32)
    half = s.size // 2
    for path in (0, 2, 4):
        ctx.depth_set_path(path)
        try:
            ctx.depth_begin(rs, re)
            ctx.depth_add_segments(s[:half], e[:half])
            ds, de = ctx.dev_array(s[half:]), ctx.dev_array(e[half:])
            ctx.depth_add_segments_device(ds, de, s.size - half)
            ctx.depth_reduce(500, 4, 0, 0)
            assert ctx.depth_last_path() == (1 if path == 0 else path)
            assert np.array_equal(ctx.depth_interval_sums(a, b), exp)
            ds.free(); de.free()
        finally:
            ctx.depth_set_path(0)


def test_batches_and_device_segments_at_top(ctx):
    """several host batches and a device batch in one region at the top: sums, minima, runs and per-base depth"""
    rng = np.random.default_rng(23)
    re = TOP
    rs = region_for(TOP - 100)
    s, e = top_segments(rng, rs, re, n=4000)
    exp = orc.pileup_diff(s, e, rs, re)
    W = 1000
    es, em = orc.window_sums(exp, rs, re, W)
    ea, ec = orc.class_runs(exp, rs, re, 4, 40, TILE)
    cut = [0, 7, s.size // 3, 2 * s.size // 3, s.size]
    for forced in (0, 4, 2):
        ctx.depth_set_path(forced)
        try:
            ctx.depth_begin(rs, re)
            ctx.depth_add_segments(s[cut[0]:cut[1]], e[cut[0]:cut[1]])
            ctx.depth_add_segments(s[cut[1]:cut[2]], e[cut[1]:cut[2]])
            ds, de = ctx.dev_array(s[cut[2]:cut[3]]), ctx.dev_array(e[cut[2]:cut[3]])
            ctx.depth_add_segments_device(ds, de, cut[3] - cut[2])
            ctx.depth_add_segments(s[cut[3]:], e[cut[3]:])
            ctx.depth_reduce(W, 4, 40, TILE)
            assert ctx.depth_last_path() == (1 if forced == 0 else forced)
            assert np.array_equal(ctx.depth_get_windows(), es)
            r0, r1, rc = ctx.depth_get_runs(want_end=True)
            assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
            assert r1[-1] == TOP
            ws, wm = ctx.depth_windows(W, es.size)
            assert np.array_equal(ws, es) and np.array_equal(wm, em)
            assert np.array_equal(ctx.depth_perbase(re - rs), exp)
            ds.free(); de.free()
        finally:
            ctx.depth_set_path(0)


def test_packed_formats_round_trip_at_top(ctx):
    """packed16, fixed-block packed16 and packed8 of segments up to INT32_MAX: the host words decode to the same depth
    (numpy), and the device's unpack kernels (start + length in int) give the oracle's integers"""
    rng = np.random.default_rng(29)
    re = TOP
    rs = region_for(LAST_TILE)
    s, e = top_segments(rng, rs, re, n=6000)
    exp = orc.pileup_diff(s, e, rs, re)
    assert np.array_equal(orc.pileup_brute(s, e, rs, re), exp)
    es, _ = orc.window_sums(exp, rs, re, 500)
    ea, ec = orc.class_runs(exp, rs, re, 4, 0, 0)

    # packed16: host decode, then two batches through depth_unpack16_kernel, then the one-call entry
    a, o, ln = capi.pack_segments16(s, e)
    st = a.astype(np.int64).repeat(256) + o
    keep = ln > 0
    assert st[keep].max() < TOP and (st + ln)[keep].max() == TOP
    assert np.array_equal(orc.pileup_brute(st[keep], (st + ln)[keep], rs, re), exp)
    h = a.size // 2
    ctx.depth_begin(rs, re)
    ctx.depth_add_segments_packed16(a[:h], o[:h * 256], ln[:h * 256])
    ctx.depth_add_segments_packed16(a[h:], o[h * 256:], ln[h * 256:])
    ctx.depth_reduce(500, 4, 0, 0)
    assert ctx.depth_last_path() == 1
    assert np.array_equal(ctx.depth_get_windows(), es)
    r0, rc = ctx.depth_get_runs()
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
    assert np.array_equal(ctx.depth_perbase(re - rs), exp)
    ws, r0, rc = ctx.depth_region_packed16(rs, re, a, o, ln, 500, 4, 0)
    assert np.array_equal(ws, es) and np.array_equal(r0, ea) and np.array_equal(rc, ec)

    # fixed-block packed16 (what GL_BED_PACK=16 sends): blocks plus the escaped segments
    a, o, ln, xs, xe = capi.pack_segments16_fixed(s, e)
    st = a.astype(np.int64).repeat(256) + o
    keep = ln > 0
    ds = np.concatenate([st[keep], xs.astype(np.int64)])
    de = np.concatenate([(st + ln)[keep], xe.astype(np.int64)])
    assert de.max() == TOP
    assert np.array_equal(orc.pileup_brute(ds, de, rs, re), exp)

    # packed8: host decode, then the packed8 kernel and the unpacked words through the int32 fused path
    a, d, ln = capi.pack_segments8(s, e)
    us, ue = capi.unpack_segments8(a, d, ln)
    assert ue.max() == TOP and us.max() < TOP
    assert np.array_equal(orc.pileup_brute(us, ue, rs, re), exp)
    for forced, paths in ((0, (3,)), (1, (1, 4))):
        ctx.depth_set_path(forced)
        try:
            ctx.depth_begin(rs, re)
            ctx.depth_add_segments_packed8(a, d, ln)
            ctx.depth_reduce(500, 4, 0, 0)
            assert ctx.depth_last_path() in paths
            assert np.array_equal(ctx.depth_get_windows(), es)
            r0, rc = ctx.depth_get_runs()
            assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
            assert np.array_equal(ctx.depth_perbase(re - rs), exp)
        finally:
            ctx.depth_set_path(0)


def _pass_segments(rng, rs, n=12_000):
    """sorted reads for the CLI's last pass over a 2^31-1 base contig: a pile at its start (a chunk edge), sparse reads
    through it, and a pile over the contig's last bases, incl. reads that end at INT32_MAX"""
    s1 = rng.integers(rs - 300, rs + 60_000, n // 2)
    s2 = rng.integers(rs, TOP - 300, n // 10)
    s3 = rng.integers(TOP - 40_000, TOP - 300, n // 2)
    s = np.concatenate([s1, s2, s3])
    e = s + rng.integers(1, 300, s.size)
    s4 = TOP - rng.integers(1, 300, 200)
    s = np.concatenate([s, s4])
    e = np.concatenate([e, np.minimum(TOP, s4 + rng.integers(1, 300, s4.size))])
    o = np.argsort(s, kind="stable")
    return s[o].astype(np.int32), e[o].astype(np.int32)


@pytest.mark.parametrize("pack", ["0", "16", "1"])
@pytest.mark.parametrize("W,mincov,maxmean", [(500, 4, 0), (100_000, 1, 5), (4096, 2, 8)])
def test_bed_region_text_last_pass(ctx, monkeypatch, pack, W, mincov, maxmean):
    """gl_depth_bed_region over the last whole chunks of a 2^31-1 base contig, ending at INT32_MAX, in each transport
    (GL_BED_PACK: 0 plain int32, 16 fixed-block packed16, 1 packed8), == the oracle's walker run chunk by chunk"""
    monkeypatch.setenv("GL_BED_PACK", pack)
    step = step_for(W)
    rs = 2_140_000_000 // step * step
    rng = np.random.default_rng(W)
    s, e = _pass_segments(rng, rs)
    exp_hd, exp_ca = [], []
    for cs in range(rs, TOP, step):
        ce = min(cs + step, TOP)
        h, c = orc.walk_chunk("chrBig", cs, ce, W, mincov, maxmean, orc.pileup_diff(s, e, cs, ce))
        exp_hd.append(h); exp_ca.append(c)
    hd, ca = ctx.depth_bed_region("chrBig", rs, TOP, s, e, W, mincov, maxmean, step)
    assert ctx.depth_last_path() == (3 if pack == "1" else 1)
    assert hd == b"".join(exp_hd)
    assert ca == b"".join(exp_ca)
    assert hd.splitlines()[-1].split(b"\t")[2] == b"%d" % TOP and ca.splitlines()[-1].split(b"\t")[2] == b"%d" % TOP


def test_format_rows_ending_at_int32_max(ctx):
    """the device formatter's explicit rows (the --stats-free BED text) for rows that end at INT32_MAX"""
    starts = [TOP - 1, TOP - 2, TOP - 255, LAST_TILE, LAST_TILE - 1, 2 ** 30, 2_140_000_000, 0, 1]
    sums = [0, 1, 7, 123_456_789, 2 ** 40 + 3, 5, 99_999, 2 ** 31 - 1, 3]
    row_s = np.array(starts, np.int64)
    row_e = np.full(row_s.size, TOP, np.int64)
    row_sum = np.array(sums, np.int64)
    got = ctx.depth_format_rows("chrBig", row_s, row_e, row_sum).decode().splitlines()
    assert len(got) == row_s.size
    for i in range(row_s.size):
        mean = 0.0 if sums[i] == 0 else float(sums[i]) / float(TOP - starts[i])
        assert got[i] == "chrBig\t%d\t%d\t%s" % (starts[i], TOP, "%.4g" % mean), i


GOLEFT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "bin", "goleft")


def test_cli_depth_contig_of_int32_max_bases(tmp_path):
    """`goleft depth` on a 2^31-1 base contig: three GPU passes of whole 10 Mb chunks ([0, 1.07e9), [1.07e9, 2.14e9),
    [2.14e9, 2^31-1)), reads at the contig's start, across both pass edges and over its last bases; unindexed BAM (a BAI
    cannot address past 2^29), so the whole file is decoded.  == the oracle's walker chunk by chunk."""
    L, W = TOP, 100_000
    rng = np.random.default_rng(31)
    edges = [0, 1_070_000_000, 2_140_000_000]
    pos = [rng.integers(max(0, x - 3000), x + 3000, 400) for x in edges]
    pos.append(rng.integers(L - 300, L - 150, 60))
    pos = np.sort(np.concatenate(pos))
    cigars = [[(150, "M")], [(45, "M"), (7, "D"), (55, "M")], [(12, "S"), (88, "M")], [(60, "M"), (300, "N"), (40, "M")]]
    recs = []
    for p0 in pos.tolist():
        cig = cigars[int(rng.integers(0, len(cigars)))]
        if p0 + 400 > L:                                   # the contig's last bases: reads that end on it, one at INT32_MAX
            cig = [(int(min(150, L - p0)), "M")]
        recs.append((0, p0, 60, int(rng.choice([0, 16])), cig))
    recs.append((0, L - 100, 60, 0, [(100, "M")]))
    recs.sort(key=lambda r: r[1])
    refs = [("chrBig", L)]
    bam = tmp_path / "big.bam"
    bam.write_bytes(make_bam(refs, recs))                  # no .bai; make_bam writes bin 0, the readers take pos (checked below)
    (tmp_path / "ref.fa.fai").write_text("chrBig\t%d\t8\t60\t61\n" % L)
    s, e = bamref.segments(recs, 1, 1)[0]
    assert int(np.max(e)) == TOP and int(np.max(s)) > 2 ** 29
    got = capi.bam_segments(str(bam))                      # the host reader gives these records' blocks, positions past 2^29 included
    assert bamref.same_multiset(got["segments"][0][0], got["segments"][0][1], s, e)
    prefix = str(tmp_path / "o")
    p = subprocess.run([GOLEFT, "depth", "-w", str(W), "--prefix", prefix, "--reference", str(tmp_path / "ref.fa"), str(bam)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    assert "decoding the whole file" in p.stderr
    exp_hd, exp_ca = [], []
    for cs, ce in orc.gen_chunks(L, W):
        h, c = orc.walk_chunk("chrBig", cs, ce, W, 4, 0, orc.pileup_diff(s, e, cs, ce))
        exp_hd.append(h); exp_ca.append(c)
    hd = open(prefix + ".depth.bed", "rb").read()
    ca = open(prefix + ".callable.bed", "rb").read()
    assert hd.count(b"\n") == (L - 1) // W + 1
    assert hd == b"".join(exp_hd)
    assert ca == b"".join(exp_ca)
