"""GPU parity: the CUDA depth path, called through the C ABI, against oracle/oracle_depth.c.
Integer work -> bit-exact.  Every test here needs an H100 (`-m gpu`)."""
import numpy as np
import pytest

from goleft_b200 import capi, synth
from oracle import loader as orc

pytestmark = pytest.mark.gpu

FAI_WINDOWS = [100, 1000000000, 55, 60, 71, 13, 2001]          # depth/functional-test.sh:45-70
BED_WINDOWS = [10, 1000000, 50, 55, 60, 71, 13, 2002]          # depth/functional-test.sh:73-97


def rand_segments(rng, n, lo, hi, maxlen=300):
    s = rng.integers(lo, hi, n).astype(np.int32)
    e = (s + rng.integers(1, maxlen, n)).astype(np.int32)
    return s, e


def _run_once(ctx, s, e, rs, re, W, mincov, maxmean, run_break, device, expect_path, exp, packed8=False):
    exp_depth, es, em, ea, ec = exp
    ctx.depth_begin(rs, re)
    bufs = []
    if packed8:
        a, d, ln = capi.pack_segments8(s, e)
        if device and a.size:
            bufs = [ctx.dev_array(a), ctx.dev_array(d), ctx.dev_array(ln)]
            ctx.depth_add_segments_packed8_device(bufs[0], bufs[1], bufs[2], a.size)
        else:
            ctx.depth_add_segments_packed8(a, d, ln)
        if a.size == 0:
            expect_path = None
    elif device:
        ds, de = ctx.dev_array(s), ctx.dev_array(e)
        bufs = [ds, de]
        ctx.depth_add_segments_device(ds, de, s.size)
    else:
        ctx.depth_add_segments(s, e)
    ctx.depth_reduce(W, mincov, maxmean, run_break)
    if expect_path is not None and s.size:
        assert ctx.depth_last_path() == expect_path
    nw, nr, md = ctx.depth_result_sizes()
    ws = ctx.depth_get_windows()
    r0, r1, rc = ctx.depth_get_runs(want_end=True)
    assert nw == es.size
    assert np.array_equal(ws, es)
    assert nr == ea.size
    assert np.array_equal(r0, ea)
    assert np.array_equal(rc, ec)
    assert np.array_equal(r1, np.append(ea[1:], re).astype(np.int32))
    assert md == int(exp_depth.max(initial=0))
    ws2, wm2 = ctx.depth_windows(W, nw)                      # sums + per-window minimum (general window path)
    assert np.array_equal(ws2, es) and np.array_equal(wm2, em)
    got_depth = ctx.depth_perbase(re - rs)
    assert np.array_equal(got_depth, exp_depth)
    for b in bufs:
        b.free()
    return ws, r0, rc


def check_region(ctx, s, e, rs, re, W, mincov=4, maxmean=0, run_break=0, device=False):
    """Both ways of building the difference array must give the oracle's integers:
    as given (general scatter path unless already sorted), sorted (fused smem path), sorted + forced general."""
    exp_depth = orc.pileup_brute(s, e, rs, re) if s.size * 300 < 5e8 else orc.pileup_diff(s, e, rs, re)
    es, em = orc.window_sums(exp_depth, rs, re, W)
    ea, ec = orc.class_runs(exp_depth, rs, re, mincov, maxmean, run_break)
    exp = (exp_depth, es, em, ea, ec)
    is_sorted = bool((np.diff(s) >= 0).all()) if s.size else True
    short = bool(((e - s) <= 16384).all()) if s.size else True
    # unsorted input is correct on either path (the fused kernel only bails out when its index span explodes)
    out = _run_once(ctx, s, e, rs, re, W, mincov, maxmean, run_break, device,
                    (1 if short else 4) if is_sorted else (None if short else 4), exp)
    if not is_sorted:
        o = np.argsort(s, kind="stable")
        _run_once(ctx, s[o], e[o], rs, re, W, mincov, maxmean, run_break, device, 1 if short else 4, exp)
    # both general paths, forced: 4 = bucketed events (the default fallback), 2 = the HBM difference array
    for forced in (4, 2):
        ctx.depth_set_path(forced)
        try:
            _run_once(ctx, s, e, rs, re, W, mincov, maxmean, run_break, device, forced, exp)
        finally:
            ctx.depth_set_path(0)
    # the packed8 kernel (any input packs: long segments are cut, order does not matter), then the same packed batch
    # unpacked and taken through the int32 paths
    _run_once(ctx, s, e, rs, re, W, mincov, maxmean, run_break, device, 3, exp, packed8=True)
    ctx.depth_set_path(1)
    try:
        _run_once(ctx, s, e, rs, re, W, mincov, maxmean, run_break, device, None, exp, packed8=True)
    finally:
        ctx.depth_set_path(0)
    ws, r0, rc = out
    return exp_depth, ws, r0, rc


@pytest.mark.parametrize("W", FAI_WINDOWS)
def test_small_region_all_fai_windows(ctx, W):
    rng = np.random.default_rng(W)
    s, e = rand_segments(rng, 20000, -100, 20100)
    check_region(ctx, s, e, 0, 20001, W)


@pytest.mark.parametrize("W", BED_WINDOWS)
def test_bed_regions(ctx, W):
    """the nine regions of depth/test/windows.bed, incl. 1- and 2-base regions"""
    rng = np.random.default_rng(W + 1000)
    s, e = rand_segments(rng, 5000, 0, 16000, maxlen=120)
    for rs, re in [(14250, 15500), (1575, 15800), (100, 1000), (2000, 5000), (1, 3), (9, 13), (16, 17), (24, 29), (39, 43)]:
        depth, ws, r0, rc = check_region(ctx, s, e, rs, re, W)
        exp = orc.walk_chunk("chrM", rs, re, W, 4, 0, depth)
        assert capi.format_chunk("chrM", rs, re, W, ws, r0, rc) == exp


def test_empty_and_out_of_region_segments(ctx):
    z = np.zeros(0, np.int32)
    check_region(ctx, z, z, 0, 16571, 10)                      # t-empty.bam (functional-test.sh:102)
    s = np.array([0, 50, 5000, 99, 100, 10], np.int32)
    e = np.array([10, 101, 6000, 100, 101, 5000], np.int32)
    check_region(ctx, s, e, 100, 1000, 10)                     # only clipped pieces count


def test_tile_edges_and_run_break(ctx):
    rng = np.random.default_rng(5)
    for L in [4095, 4096, 4097, 8192, 12289]:
        s, e = rand_segments(rng, 3000, -50, L + 50, maxlen=200)
        check_region(ctx, s, e, 0, L, 500, run_break=4096)
        check_region(ctx, s, e, 7, L + 7, 512, run_break=1000, device=True)


def test_window_sizes_extreme(ctx):
    rng = np.random.default_rng(6)
    s, e = rand_segments(rng, 40000, 0, 100000, maxlen=151)
    for W in [1, 2, 16, 17, 4096, 5000, 2 ** 30]:
        check_region(ctx, s, e, 0, 100000, W, mincov=3, maxmean=25)


def test_bam_order_segments_take_fused_path(ctx):
    """BAM order = reads sorted by position; the second block of a deletion read starts after the next reads
    do, so segment starts are only nearly sorted.  That must still take the fused path."""
    L = 3_000_000
    s, e = synth.segments(synth.reads(L, contig_index=7))
    assert not (np.diff(s) >= 0).all()
    ctx.depth_begin(0, L)
    ctx.depth_add_segments(s, e)
    ctx.depth_reduce(500, 4, 0, 0)
    assert ctx.depth_last_path() == 1
    exp = orc.pileup_diff(s, e, 0, L)
    es, _ = orc.window_sums(exp, 0, L, 500)
    ea, ec = orc.class_runs(exp, 0, L, 4, 0, 0)
    assert np.array_equal(ctx.depth_get_windows(), es)
    r0, rc = ctx.depth_get_runs()
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
    # shuffled: the fused kernel notices the index span explosion and the general path takes over
    rng = np.random.default_rng(3)
    p = rng.permutation(s.size)
    ctx.depth_begin(0, L)
    ctx.depth_add_segments(s[p], e[p])
    ctx.depth_reduce(500, 4, 0, 0)
    assert ctx.depth_last_path() == 4
    assert np.array_equal(ctx.depth_get_windows(), es)
    r0, rc = ctx.depth_get_runs()
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)


def test_long_segments_fall_back(ctx):
    """segments longer than the fused path's look-back (16384) -> general path, same integers"""
    rng = np.random.default_rng(11)
    s = np.sort(rng.integers(0, 200000, 3000)).astype(np.int32)
    e = (s + rng.integers(1, 60000, 3000)).astype(np.int32)
    check_region(ctx, s, e, 1000, 180000, 500)


def test_fused_lookback_edges(ctx):
    """sorted segments whose length is exactly at / around tile and cell edges"""
    s = np.array([0, 0, 255, 256, 4095, 4096, 4096, 8191, 12000, 16383, 20000], np.int32)
    e = np.array([4096, 16384, 4097, 257, 4096, 4097, 20480, 8192, 28384, 16385, 20001], np.int32)
    for rs, re in [(0, 30000), (100, 20000), (4096, 8192), (4095, 8193)]:
        check_region(ctx, s, e, rs, re, 100, mincov=2)


def test_deep_pileup_int64_sums(ctx):
    """500k identical reads: window sums exceed 2^32"""
    s = np.full(500_000, 1000, np.int32)
    e = np.full(500_000, 21000, np.int32)
    depth, ws, _, _ = check_region(ctx, s, e, 0, 30000, 10000, maxmean=1000)
    assert ws.max() > 2 ** 32


def test_multiple_add_calls_and_unsorted(ctx):
    rng = np.random.default_rng(8)
    s, e = rand_segments(rng, 30001, 0, 50000)
    p = rng.permutation(s.size)
    s, e = s[p], e[p]
    exp = orc.pileup_diff(s, e, 0, 50000)
    ctx.depth_begin(0, 50000)
    ctx.depth_add_segments(s[:7], e[:7])                       # unaligned tail path
    ds, de = ctx.dev_array(s), ctx.dev_array(e)
    ctx.depth_add_segments_device(ds, de, 10000 - 7, offset=7)  # misaligned device pointers -> scalar kernel
    ctx.depth_add_segments(s[10000:], e[10000:])
    assert np.array_equal(ctx.depth_perbase(50000), exp)
    ws, wm = ctx.depth_windows(250, 200)
    es, em = orc.window_sums(exp, 0, 50000, 250)
    assert np.array_equal(ws, es) and np.array_equal(wm, em)
    r0, r1, rc = ctx.depth_classes(4, 0, 50000)
    ea, ec = orc.class_runs(exp, 0, 50000, 4, 0)
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
    ds.free(); de.free()


def test_state_errors(ctx):
    c2 = capi.Ctx(0)
    with pytest.raises(capi.GlError) as ei:
        c2.depth_add_segments(np.zeros(1, np.int32), np.ones(1, np.int32))
    assert ei.value.code == capi.GL_ESTATE
    with pytest.raises(capi.GlError) as ei:
        c2.depth_begin(10, 10)
    assert ei.value.code == capi.GL_EINVAL
    c2.depth_begin(0, 100)
    with pytest.raises(capi.GlError) as ei:
        c2.depth_reduce(0)
    assert ei.value.code == capi.GL_EINVAL
    c2.close()


def test_sparse_region_far_from_origin(ctx):
    """bed-style region deep inside a contig with a handful of reads (index table starts at rs-16384)"""
    s = np.array([99_990_000, 100_000_100, 100_000_100, 100_004_000, 100_100_000], np.int32)
    e = s + np.array([20000, 150, 151, 9000, 10], np.int32)
    check_region(ctx, s, e, 100_000_000, 100_050_000, 250, mincov=1)
    s2 = s[1:4]; e2 = (s2 + 150).astype(np.int32)
    check_region(ctx, s2, e2, 100_000_000, 100_050_000, 250, mincov=1)


def test_run_capacity_regrow(ctx):
    """alternating covered/uncovered bases: one run per base, far above the initial capacity"""
    L = 300_000
    s = np.arange(0, L, 2, dtype=np.int32)
    e = s + 1
    check_region(ctx, s, e, 0, L, 1000, mincov=1)


def test_fai_mode_whole_contig_text(ctx):
    """25 Mb synthetic 30x contig, whole contig in one launch with run_break = step, then per-chunk text
    == the oracle's per-chunk walker (what `goleft depth -w 500 --ordered` writes)."""
    L, W = 25_000_000, 500
    s, e = synth.segments(synth.reads(L, contig_index=3))
    exp_depth = orc.pileup_diff(s, e, 0, L)
    chunks = orc.gen_chunks(L, W)
    step = chunks[0][1] - chunks[0][0]
    ws, r0, rc = ctx.depth_region(0, L, s, e, W, 4, 0, run_break=step)
    got_hd, got_ca, exp_hd, exp_ca = [], [], [], []
    for cs, ce in chunks:
        h, c = orc.walk_chunk("chr4", cs, ce, W, 4, 0, exp_depth[cs:ce])
        exp_hd.append(h); exp_ca.append(c)
        lo, hi = np.searchsorted(r0, cs), np.searchsorted(r0, ce)
        h, c = capi.format_chunk("chr4", cs, ce, W, ws[cs // W:(ce - 1) // W + 1], r0[lo:hi], rc[lo:hi])
        got_hd.append(h); got_ca.append(c)
    assert b"".join(got_hd) == b"".join(exp_hd)
    assert b"".join(got_ca) == b"".join(exp_ca)


def test_full_size_chr20(ctx):
    """BASELINE config 1 (chr20, 30x, W=500) at full size: bit-exact vs the oracle, plus the size-independent
    properties: sum of window sums == total clipped segment length; runs tile the contig."""
    L, W = synth.CHR20_LEN, 500
    s, e = synth.chr20_like()
    ds, de = ctx.dev_array(s), ctx.dev_array(e)
    ctx.depth_begin(0, L)
    ctx.depth_add_segments_device(ds, de, s.size)
    ctx.depth_reduce(W, 4, 0, 10_000_000)
    assert ctx.depth_last_path() == 1
    ws = ctx.depth_get_windows()
    r0, rc = ctx.depth_get_runs()
    assert int(ws.sum()) == int((np.minimum(e, L).astype(np.int64) - np.maximum(s, 0)).clip(0).sum())
    assert r0[0] == 0 and (np.diff(r0) > 0).all() and r0[-1] < L
    exp = orc.pileup_diff(s, e, 0, L)
    es, em = orc.window_sums(exp, 0, L, W)
    ea, ec = orc.class_runs(exp, 0, L, 4, 0, 10_000_000)
    assert np.array_equal(ws, es)
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
    # both general paths at full size give the same integers (4: bucketed events, 2: HBM difference array)
    for forced in (4, 2):
        ctx.depth_set_path(forced)
        ctx.depth_begin(0, L)
        ctx.depth_add_segments_device(ds, de, s.size)
        ctx.depth_reduce(W, 4, 0, 10_000_000)
        assert ctx.depth_last_path() == forced
        assert np.array_equal(ctx.depth_get_windows(), es)
        r0, rc = ctx.depth_get_runs()
        assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
        ws2, wm2 = ctx.depth_windows(W, es.size)
        assert np.array_equal(ws2, es) and np.array_equal(wm2, em)
    ctx.depth_set_path(0)
    ds.free(); de.free()
    # the packed8 kernel at full size, packed words resident on the device
    a, d, ln = capi.pack_segments8(s, e)
    bufs = [ctx.dev_array(a), ctx.dev_array(d), ctx.dev_array(ln)]
    ctx.depth_begin(0, L)
    ctx.depth_add_segments_packed8_device(bufs[0], bufs[1], bufs[2], a.size)
    ctx.depth_reduce(W, 4, 0, 10_000_000)
    assert ctx.depth_last_path() == 3
    assert np.array_equal(ctx.depth_get_windows(), es)
    r0, rc = ctx.depth_get_runs()
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
    for b in bufs:
        b.free()


def test_packed16_path(ctx):
    """the feeder's compact format (half the PCIe bytes) gives the same integers as plain int32 arrays"""
    L = 5_000_000
    s, e = synth.segments(synth.reads(L, contig_index=9))
    a, o, ln = capi.pack_segments16(s, e)
    exp = orc.pileup_diff(s, e, 0, L)
    es, _ = orc.window_sums(exp, 0, L, 500)
    ea, ec = orc.class_runs(exp, 0, L, 4, 0, 1_000_000)
    ws, r0, rc = ctx.depth_region_packed16(0, L, a, o, ln, 500, 4, 0, run_break=1_000_000)
    assert ctx.depth_last_path() == 1
    assert np.array_equal(ws, es) and np.array_equal(r0, ea) and np.array_equal(rc, ec)
    # two packed batches + one plain batch in one region, sub-region with clipping
    h = s.size // 3
    a1, o1, l1 = capi.pack_segments16(s[:h], e[:h])
    a2, o2, l2 = capi.pack_segments16(s[h:2 * h], e[h:2 * h])
    ctx.depth_begin(1234, 4_000_000)
    ctx.depth_add_segments_packed16(a1, o1, l1)
    ctx.depth_add_segments_packed16(a2, o2, l2)
    ctx.depth_add_segments(s[2 * h:], e[2 * h:])
    ctx.depth_reduce(250, 4, 0, 0)
    exp = orc.pileup_diff(s, e, 1234, 4_000_000)
    assert np.array_equal(ctx.depth_get_windows(), orc.window_sums(exp, 1234, 4_000_000, 250)[0])
    r0, rc = ctx.depth_get_runs()
    ea, ec = orc.class_runs(exp, 1234, 4_000_000, 4, 0, 0)
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)


def test_packed8_path(ctx):
    """the feeder's densest format (a quarter of the PCIe bytes; short reads) gives the same integers"""
    L = 5_000_000
    s, e = synth.segments(synth.reads(L, contig_index=9))
    a, d, ln = capi.pack_segments8(s, e)
    exp = orc.pileup_diff(s, e, 0, L)
    es, em = orc.window_sums(exp, 0, L, 500)
    ea, ec = orc.class_runs(exp, 0, L, 4, 0, 1_000_000)
    ws, r0, rc = ctx.depth_region_packed8(0, L, a, d, ln, 500, 4, 0, run_break=1_000_000)
    assert ctx.depth_last_path() == 3
    assert np.array_equal(ws, es) and np.array_equal(r0, ea) and np.array_equal(rc, ec)
    # window sums and minima straight from the packed words (the only batch, queried through gl_depth_windows)
    ctx.depth_begin(0, L)
    ctx.depth_add_segments_packed8(a, d, ln)
    ws, wm = ctx.depth_windows(500, es.size)
    assert ctx.depth_last_path() == 3
    assert np.array_equal(ws, es) and np.array_equal(wm, em)
    # an int32 batch of odd length first (the packed8 unpack realigns the store), then packed8 + packed16 batches; clipping
    h = s.size // 3 | 1
    a1, d1, l1 = capi.pack_segments8(s[h:2 * h], e[h:2 * h])
    a2, o2, l2 = capi.pack_segments16(s[2 * h:], e[2 * h:])
    ctx.depth_begin(1234, 4_000_000)
    ctx.depth_add_segments(s[:h], e[:h])
    ctx.depth_add_segments_packed8(a1, d1, l1)
    ctx.depth_add_segments_packed16(a2, o2, l2)
    ctx.depth_reduce(250, 4, 0, 0)
    exp = orc.pileup_diff(s, e, 1234, 4_000_000)
    assert np.array_equal(ctx.depth_get_windows(), orc.window_sums(exp, 1234, 4_000_000, 250)[0])
    r0, rc = ctx.depth_get_runs()
    ea, ec = orc.class_runs(exp, 1234, 4_000_000, 4, 0, 0)
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
    # long segments and gaps: pieces + fillers, general path
    rng = np.random.default_rng(5)
    s = np.sort(rng.integers(0, 3_000_000, 20000)).astype(np.int32)
    e = (s + rng.choice([1, 100, 255, 256, 3000, 40000], s.size)).astype(np.int32)
    a, d, ln = capi.pack_segments8(s, e)
    exp = orc.pileup_diff(s, e, 500, 2_900_000)
    ws, r0, rc = ctx.depth_region_packed8(500, 2_900_000, a, d, ln, 333, 4, 0)
    assert ctx.depth_last_path() == 3
    ea, ec = orc.class_runs(exp, 500, 2_900_000, 4, 0, 0)
    assert np.array_equal(ws, orc.window_sums(exp, 500, 2_900_000, 333)[0]) and np.array_equal(r0, ea) and np.array_equal(rc, ec)


def _pinned(ctx, *arrays):
    out = []
    for a in arrays:
        h = ctx.pinned_empty(a.size, a.dtype)
        h[:] = a
        out.append(h)
    return out


def test_packed8_streamed_upload(ctx):
    """one-call entry with pinned host words: the upload is streamed in chunks and every chunk's tiles are reduced while
    the next chunk is on the wire — same integers; also a sparse region (few anchors per chunk), a region that starts
    after the first chunks' data, and hand-shuffled blocks (rejected after streaming, unpacked, int32 paths)"""
    L = 6_000_000
    s, e = synth.segments(synth.reads(L, contig_index=11))
    a, d, ln = capi.pack_segments8(s, e)
    assert a.size >= 4096
    ha, hd, hl = _pinned(ctx, a, d, ln)
    for rs, re, W, brk in [(0, L, 500, 1_000_000), (4_500_000, L - 3, 333, 0), (0, 70_000, 100, 0)]:
        exp = orc.pileup_diff(s, e, rs, re)
        ws, r0, rc = ctx.depth_region_packed8(rs, re, ha, hd, hl, W, 4, 0, run_break=brk)
        assert ctx.depth_last_path() == 3
        ea, ec = orc.class_runs(exp, rs, re, 4, 0, brk)
        assert np.array_equal(ws, orc.window_sums(exp, rs, re, W)[0]) and np.array_equal(r0, ea) and np.array_equal(rc, ec)
        got = ctx.depth_perbase(re - rs)                      # a second reduce of the same (now resident) batch
        assert np.array_equal(got, exp)
    # sparse: 1x coverage with long empty stretches
    rng = np.random.default_rng(8)
    s2 = np.sort(np.concatenate([rng.integers(0, 2_000_000, 300_000), rng.integers(40_000_000, 41_000_000, 100_000)])).astype(np.int32)
    e2 = (s2 + rng.integers(30, 151, s2.size)).astype(np.int32)
    a2, d2, l2 = capi.pack_segments8(s2, e2)
    h2 = _pinned(ctx, a2, d2, l2)
    exp = orc.pileup_diff(s2, e2, 0, 45_000_000)
    ws, r0, rc = ctx.depth_region_packed8(0, 45_000_000, h2[0], h2[1], h2[2], 1000, 4, 0)
    assert ctx.depth_last_path() == 3
    ea, ec = orc.class_runs(exp, 0, 45_000_000, 4, 0, 0)
    assert np.array_equal(ws, orc.window_sums(exp, 0, 45_000_000, 1000)[0]) and np.array_equal(r0, ea) and np.array_equal(rc, ec)
    # shuffled blocks through the streamed entry
    nb = a.size
    perm = rng.permutation(nb)
    hs = _pinned(ctx, np.ascontiguousarray(a[perm]), np.ascontiguousarray(d.reshape(nb, 64)[perm]).reshape(-1),
                 np.ascontiguousarray(ln.reshape(nb, 64)[perm]).reshape(-1))
    exp = orc.pileup_diff(s, e, 0, L)
    ws, r0, rc = ctx.depth_region_packed8(0, L, hs[0], hs[1], hs[2], 500, 4, 0)
    assert ctx.depth_last_path() in (1, 4)                     # unsorted anchors are rejected: the batch is unpacked, the general path takes it
    ea, ec = orc.class_runs(exp, 0, L, 4, 0, 0)
    assert np.array_equal(ws, orc.window_sums(exp, 0, L, 500)[0]) and np.array_equal(r0, ea) and np.array_equal(rc, ec)
    # more runs than a fresh context's first run table holds (len/16 + 4096): every other base covered, one run per base.
    # The region is rerun with a larger table from the words the streamed upload left on the device.
    L3, W3 = 600_000, 500
    s3 = np.arange(0, L3, 2, dtype=np.int32)
    e3 = s3 + 1
    a3, d3, l3 = capi.pack_segments8(s3, e3)
    assert a3.size >= 4096
    exp = orc.pileup_diff(s3, e3, 0, L3)
    ea, ec = orc.class_runs(exp, 0, L3, 4, 0, 0)
    assert ea.size > L3 // 16 + 4096
    out = (np.empty((L3 - 1) // W3 + 1, np.int64), np.empty(L3, np.int32), np.empty(L3, np.uint8))
    with capi.Ctx(0) as c3:
        h3 = _pinned(c3, a3, d3, l3)
        ws, r0, rc = c3.depth_region_packed8(0, L3, h3[0], h3[1], h3[2], W3, 4, 0, out=out)
        assert c3.depth_last_path() == 3
    assert np.array_equal(ws, orc.window_sums(exp, 0, L3, W3)[0]) and np.array_equal(r0, ea) and np.array_equal(rc, ec)


def test_packed8_unsorted_anchors_fall_back(ctx):
    """hand-made packed8 blocks whose anchors are not sorted: K_tileidx8 notices, the batch is unpacked and the int32
    paths give the right integers"""
    L = 400_000
    s, e = synth.segments(synth.reads(L, contig_index=2))
    a, d, ln = capi.pack_segments8(s, e)
    nb = a.size
    perm = np.random.default_rng(0).permutation(nb)
    a2 = np.ascontiguousarray(a[perm])
    d2 = np.ascontiguousarray(d.reshape(nb, 64)[perm]).reshape(-1)
    l2 = np.ascontiguousarray(ln.reshape(nb, 64)[perm]).reshape(-1)
    exp = orc.pileup_diff(s, e, 0, L)
    ws, r0, rc = ctx.depth_region_packed8(0, L, a2, d2, l2, 500, 4, 0)
    assert ctx.depth_last_path() in (1, 4)                     # unsorted anchors are rejected: the batch is unpacked, the general path takes it
    ea, ec = orc.class_runs(exp, 0, L, 4, 0, 0)
    assert np.array_equal(ws, orc.window_sums(exp, 0, L, 500)[0]) and np.array_equal(r0, ea) and np.array_equal(rc, ec)


def test_chr1_sized_contig(ctx):
    """BASELINE config[2]'s largest shard unit: a 248,956,422 bp contig at 30x (41 M reads), one launch per kernel.
    Checks the size-independent properties (sum of window sums == total clipped segment length; runs strictly
    increasing from 0; packed16 path == int32 path) and then the full oracle comparison."""
    L, W = 248_956_422, 500
    s, e = synth.segments(synth.reads(L, contig_index=0))
    step = 10_000_000
    ws, r0, rc = ctx.depth_region(0, L, s, e, W, 4, 0, run_break=step,
                                  out=(np.empty((L - 1) // W + 1, np.int64), np.empty(1 << 22, np.int32), np.empty(1 << 22, np.uint8)))
    assert ctx.depth_last_path() == 1
    assert int(ws.sum()) == int((np.minimum(e, L).astype(np.int64) - np.maximum(s, 0)).clip(0).sum())
    assert r0[0] == 0 and (np.diff(r0) > 0).all() and r0[-1] < L
    a, o, ln = capi.pack_segments16(s, e)
    ws2, r02, rc2 = ctx.depth_region_packed16(0, L, a, o, ln, W, 4, 0, run_break=step,
                                              out=(np.empty(ws.size, np.int64), np.empty(1 << 22, np.int32), np.empty(1 << 22, np.uint8)))
    assert np.array_equal(ws, ws2) and np.array_equal(r0, r02) and np.array_equal(rc, rc2)
    exp = orc.pileup_diff(s, e, 0, L)
    es, _ = orc.window_sums(exp, 0, L, W)
    ea, ec = orc.class_runs(exp, 0, L, 4, 0, step)
    assert np.array_equal(ws, es) and np.array_equal(r0, ea) and np.array_equal(rc, ec)


def test_interval_sums(ctx):
    """gl_depth_interval_sums = sum of per-base depth over arbitrary [a,b): with the fused path's cell index,
    after the general path (no index: every segment visited), before any reduce, with several batches, and clipped
    to the open region."""
    L = 600_000
    s, e = synth.segments(synth.reads(L, contig_index=5))
    rs, re = 1234, L - 777
    depth = orc.pileup_diff(s, e, rs, re).astype(np.int64)
    cs = np.concatenate([[0], np.cumsum(depth)])
    rng = np.random.default_rng(9)
    a = rng.integers(rs - 500, re + 500, 5000).astype(np.int32)
    b = (a + rng.choice([0, 1, 2, 99, 100, 250, 4096, 4097, 70000], 5000)).astype(np.int32)
    a[:3] = [rs, rs - 50, re - 1]
    b[:3] = [re, rs + 1, re + 100]
    ac, bc = np.clip(a, rs, re), np.clip(b, rs, re)
    exp = np.where(bc > ac, cs[np.maximum(bc, ac) - rs] - cs[ac - rs], 0)
    half = s.size // 2
    for path in (0, 2, 4):
        ctx.depth_set_path(path)
        ctx.depth_begin(rs, re)
        ctx.depth_add_segments(s[:half], e[:half])
        ctx.depth_add_segments(s[half:], e[half:])
        if path == 2:
            assert np.array_equal(ctx.depth_interval_sums(a[:200], b[:200]), exp[:200])      # before any reduce
        ctx.depth_reduce(500, 4, 0, 0)
        assert ctx.depth_last_path() == (1 if path == 0 else path)
        n = a.size if path == 0 else 300                     # no index -> brute force over all segments: keep it small
        assert np.array_equal(ctx.depth_interval_sums(a[:n], b[:n]), exp[:n])
        assert ctx.depth_interval_sums(a[:0], b[:0]).size == 0
    ctx.depth_set_path(0)


@pytest.mark.parametrize("line,crlf", [(60, False), (7, False), (50, True)])
def test_fasta_stats_kernel(ctx, line, crlf):
    """gl_fasta_stats (--stats columns, depth.go:191-200) against the Faidx.Stats restatement: windows of every size
    incl. empty, single-base, line-straddling, > 64 KB (several pieces) and the contig's very end, for the last record
    of the file (no byte after it) and an inner one."""
    import os, sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from fautil import make_fasta, position
    refs = [("a", 5000), ("big", 300_001), ("last", 1234)]
    fa, _, recs = make_fasta(refs, seed=line, line=line, crlf=crlf)
    if line == 7:
        fa = fa.rstrip(b"\n")                                  # file ends with the last base itself
    rng = np.random.default_rng(1)
    for name, L in refs:
        rec = recs[name]
        off = rec[0]
        nbytes = min(len(fa) - off, position(rec, L) + 1)
        ctx.fasta_load(fa[off:off + nbytes])
        s = rng.integers(0, L + 1, 400)
        e = np.minimum(L, s + rng.choice([0, 1, 2, line - 1, line, line + 1, 500, 70_000, 200_000], 400))
        s[:4] = [0, L - 1, L, 0]
        e[:4] = [L, L, L, 1]
        ba = np.array([position(rec, int(x)) for x in s], np.int64)
        bb = np.array([min(position(rec, int(x)) + (1 if off + position(rec, int(x)) < len(fa) else 0), nbytes) for x in e], np.int64)
        counts, stats = ctx.fasta_stats(ba, bb)
        exp = np.array([orc.faidx_stats(fa, rec, int(a), int(b)) for a, b in zip(s, e)])
        assert np.array_equal(stats, exp), name
        assert (counts[:, 2] >= counts[:, 0]).all() and counts[0, 2] > 0
