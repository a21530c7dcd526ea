"""K_fused8's staged tile words and in-place depth slice, against oracle/oracle_depth.c through the packed8 entry.

The kernel loads the first 16 blocks of the next tile's block range while the current tile runs its core (deeper tiles
read the rest from global memory), and keeps each warp's depth slice in its own region of the tile buffer, cleared
before the next tile's segments are added.  These cases push on both: deep pile-ups, block ranges at every residue of 4
and at the end of the arrays,
contigs of a few blocks, streamed uploads, the per-base run and slow window paths, and one context reused across
contigs.  Integer work -> bit-exact."""
import os

import numpy as np
import pytest

from goleft_b200 import capi, synth
from oracle import loader as orc

pytestmark = pytest.mark.gpu

TILE = 4096


def _tile_ranges(a, rs, re):
    """Each tile's block range [lo, hi) as K_tileidx8 defines it: blocks whose segments can touch the tile."""
    T = (re - rs + TILE - 1) // TILE
    x = rs + TILE * np.arange(T + 1, dtype=np.int64)
    cnt_hi = np.searchsorted(a, x, side="left")
    cnt_lo = np.searchsorted(a, x - 255, side="left")
    return np.maximum(0, cnt_lo[:-1] - 1), np.minimum(a.size, cnt_hi[1:])


def _unpack8(a, d, ln):
    """The segments a packed8 batch holds: slot j of a block starts at anchor + the first j+1 deltas; length 0 = empty."""
    nb = a.size
    st = a.astype(np.int64)[:, None] + np.cumsum(d.reshape(nb, 64).astype(np.int64), axis=1)
    ll = ln.reshape(nb, 64).astype(np.int64)
    live = ll != 0
    return st[live].astype(np.int32), (st + ll)[live].astype(np.int32)


def _pinned(ctx, *arrays):
    out = []
    for x in arrays:
        h = ctx.pinned_empty(x.size, x.dtype)
        h[:] = x
        out.append(h)
    return out


def _check(ctx, s, e, packed, rs, re, W, mincov=4, maxmean=0, run_break=0, minima=True):
    """window sums, runs and per-base depth from K_fused8; window minima too (gl_depth_windows)"""
    a, d, ln = packed
    exp = orc.pileup_diff(s, e, rs, re)
    es, em = orc.window_sums(exp, rs, re, W)
    ea, ec = orc.class_runs(exp, rs, re, mincov, maxmean, run_break)
    ws, r0, rc = ctx.depth_region_packed8(rs, re, a, d, ln, W, mincov, maxmean, run_break=run_break)
    assert ctx.depth_last_path() == 3
    assert np.array_equal(ws, es)
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
    assert np.array_equal(ctx.depth_perbase(re - rs), exp)
    if minima:
        ctx.depth_begin(rs, re)
        ctx.depth_add_segments_packed8(a, d, ln)
        ws, wm = ctx.depth_windows(W, es.size)
        assert ctx.depth_last_path() == 3
        assert np.array_equal(ws, es) and np.array_equal(wm, em)
    return exp


def _piled(L, contig_index, piles):
    """30x synthetic reads plus pile-ups: (first start, last start, reads, read length)"""
    s, e = synth.segments(synth.reads(L, contig_index=contig_index))
    rng = np.random.default_rng(contig_index)
    ss, ee = [s], [e]
    for lo, hi, n, rl in piles:
        p = np.sort(rng.integers(lo, hi + 1, n)).astype(np.int32)
        ss.append(p)
        ee.append((p + rl).astype(np.int32))
    s, e = np.concatenate(ss), np.concatenate(ee)
    o = np.argsort(s, kind="stable")
    return s[o], e[o]


# ~150x over one tile, ~1000x over half of another, and 3000 reads that all start at one base 50 bases before a tile edge
PILES = [(300_000, 306_000, 9_000, 100), (700_100, 702_000, 11_500, 175), (268 * TILE - 50, 268 * TILE - 50, 3_000, 200)]


def test_deep_tiles(ctx):
    """tiles of more than 16 and more than 64 blocks: the prefetched first 16, the rest from global memory"""
    L = 1_500_000
    s, e = _piled(L, 21, PILES)
    packed = capi.pack_segments8(s, e)
    lo, hi = _tile_ranges(packed[0], 0, L)
    assert (hi - lo).max() > 64 and ((hi - lo) > 16).sum() >= 3
    for W, maxmean in [(500, 0), (500, 200), (13, 200)]:           # maxmean: the pile-ups are their own class
        exp = _check(ctx, s, e, packed, 0, L, W, maxmean=maxmean)
    assert exp.max() >= 1000


def test_block_range_residues_and_array_end(ctx):
    """tile block ranges that start and end at every residue of 4, and batches of nb, nb-1, nb-2, nb-3 blocks, so the last
    tile's range ends at the array's last block at every residue"""
    L = 400_000
    s, e = synth.segments(synth.reads(L, contig_index=23))
    a, d, ln = capi.pack_segments8(s, e)
    us, ue = _unpack8(a, d, ln)
    o, uo = np.lexsort((e, s)), np.lexsort((ue, us))
    assert np.array_equal(us[uo], s[o]) and np.array_equal(ue[uo], e[o])   # the decoder below reads the format right
    for rs, re in [(0, L), (777, L - 1234)]:
        lo, hi = _tile_ranges(a, rs, re)
        assert set((lo % 4).tolist()) == {0, 1, 2, 3} and set((hi % 4).tolist()) == {0, 1, 2, 3}
    for k in range(4):
        nb = a.size - k
        part = (a[:nb].copy(), d[:nb * 64].copy(), ln[:nb * 64].copy())
        ps, pe = _unpack8(*part)
        assert _tile_ranges(part[0], 0, L)[1].max() == nb
        _check(ctx, ps, pe, part, 0, L, 500, minima=(k == 0))
        _check(ctx, ps, pe, part, 1 + 13 * k, L - 7 * k, 333 + k, minima=False)


def test_contigs_of_a_few_blocks(ctx):
    """1, 2 and 3 blocks: fewer blocks than the 16 prefetched per tile"""
    rng = np.random.default_rng(25)
    for n, L in [(1, 9_000), (40, 9_000), (100, 20_000), (150, 70_000)]:
        s = np.sort(rng.integers(1000, 1000 + 4 * n + 1, n)).astype(np.int32)
        e = (s + rng.integers(1, 200, n)).astype(np.int32)
        packed = capi.pack_segments8(s, e)
        assert 1 <= packed[0].size < 4
        for rs, re, W in [(0, L, 500), (1100, L, 13), (0, 1 + int(s.max()), 71)]:
            _check(ctx, s, e, packed, rs, re, W, mincov=1)


def test_streamed_upload_chunks_inside_tiles(ctx):
    """pinned host words: the upload is streamed in chunks and K_fused8 runs once per chunk on the tiles it completes, so
    a launch starts and ends inside the tiles' block ranges"""
    L = 3_000_000
    s, e = _piled(L, 27, [(1_712_000, 1_716_000, 30_000, 150), (2_571_000, 2_572_000, 5_000, 120)])
    a, d, ln = capi.pack_segments8(s, e)
    lo, hi = _tile_ranges(a, 0, L)
    if "GL_P8_CHUNKS" not in os.environ:                           # the default three chunks end at 4/7 and 6/7 of the blocks
        for b1 in (a.size * 4 // 7, a.size * 6 // 7):
            assert ((lo < b1) & (b1 < hi)).any()
    host = tuple(_pinned(ctx, a, d, ln))
    for rs, re, W, brk in [(0, L, 500, 1_000_000), (1_234_567, L - 5, 31, 0)]:
        _check(ctx, s, e, host, rs, re, W, run_break=brk, minima=False)


def test_low_coverage_per_base_runs(ctx):
    """~2x coverage: most warps see a class change and take the per-base run path, which reads the slice in the tile
    buffer; runs only (no windows: the core clears the region without writing a slice), then windows only"""
    L = 800_000
    s, e = synth.segments(synth.reads(L, coverage=2.0, contig_index=29))
    packed = capi.pack_segments8(s, e)
    for W, mincov, brk in [(500, 1, 0), (13, 2, 1000), (31, 3, 0)]:
        exp = _check(ctx, s, e, packed, 0, L, W, mincov=mincov, run_break=brk)
    ctx.depth_begin(0, L)
    ctx.depth_add_segments_packed8(*packed)
    r0, _, rc = ctx.depth_classes(2, 5, 1 << 20)
    assert ctx.depth_last_path() == 3
    ea, ec = orc.class_runs(exp, 0, L, 2, 5, 0)
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
    ws, wm = ctx.depth_windows(97, (L - 1) // 97 + 1)
    assert ctx.depth_last_path() == 3
    es, em = orc.window_sums(exp, 0, L, 97)
    assert np.array_equal(ws, es) and np.array_equal(wm, em)


def test_one_context_across_contigs():
    """a fresh context, reused: long and short contigs, deep and shallow, so that persistent CTAs carry the prefetch, the
    cleared tile buffer and the barriers across many tiles and launches of different sizes"""
    big = _piled(2_000_000, 31, PILES)
    tiny_s = np.array([5, 9, 4000, 4100, 8191], np.int32)
    tiny = (tiny_s, (tiny_s + np.array([100, 255, 96, 1, 3], np.int32)).astype(np.int32))
    mid = synth.segments(synth.reads(700_000, coverage=5.0, contig_index=33))
    seq = [(big, 0, 2_000_000, 500, 0), (tiny, 0, 9_000, 13, 0), (mid, 0, 700_000, 1000, 40),
           (big, 99_999, 1_400_000, 60, 150), (tiny, 0, 12_289, 500, 0), (big, 0, 2_000_000, 500, 0)]
    with capi.Ctx(0) as c:
        for (s, e), rs, re, W, maxmean in seq:
            _check(c, s, e, capi.pack_segments8(s, e), rs, re, W, maxmean=maxmean)
