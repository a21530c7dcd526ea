"""K_fused8's guard-banded tile, against oracle/oracle_depth.c through the packed8 entry.

Every segment of a tile's block range adds +1 at its start and -1 at its end, each clamped into the tile buffer: a
position before the tile goes to the lane's slot of a 32-entry lead guard, one at or past its end to the trailing guard.
The lead guard's sum is the depth carried into the tile.  These hand-built batches put segments where each rule acts:
ends exactly at a tile start, starts 1 and 255 bases before it, leading blocks far before the tile, a warp whose 32
lanes all clamp, starts at base 4095, ends at 4096, 4097 and 4096 + 254, starts past the tile, filler slots, deep
pile-ups that need four and more passes, region starts off the tile grid, a ragged last tile, the top of the int32
range, and one context reused across contigs.  Integer work -> bit-exact."""
import numpy as np
import pytest

from goleft_b200 import capi
from oracle import loader as orc
from oracle import multidepth as omd

pytestmark = pytest.mark.gpu

TILE = 4096
INT32_MAX = 2**31 - 1


def _pack(segs):
    """packed8 words for (start, len) pairs in start order, len <= 255 (0 = filler slot): a block is 64 slots, a new one
    starts when the block is full or the next start is more than 255 bases on; a block's unused slots are fillers at its
    last start.  Returns the words and the live segments as (start, end)."""
    segs = sorted(segs, key=lambda x: x[0])
    blocks, cur = [], []
    for s, ln in segs:
        if cur and (len(cur) == 64 or s - cur[-1][0] > 255):
            blocks.append(cur)
            cur = []
        cur.append((s, ln))
    blocks.append(cur)
    nb = len(blocks)
    a = np.empty(nb, np.int32)
    d = np.zeros(nb * 64, np.uint8)
    ln = np.zeros(nb * 64, np.uint8)
    for b, blk in enumerate(blocks):
        st = np.array([x for x, _ in blk], np.int64)
        a[b] = st[0]
        d[b * 64: b * 64 + len(blk)] = np.diff(st, prepend=st[0])
        ln[b * 64: b * 64 + len(blk)] = [x for _, x in blk]
    live = [(s, s + x) for s, x in segs if x]
    s = np.array([x for x, _ in live], np.int32)
    e = np.array([x for _, x in live], np.int32)
    return (a, d, ln), s, e


def _check(ctx, packed, s, e, rs, re, W=500, mincov=4, maxmean=0):
    a, d, ln = packed
    exp = orc.pileup_diff(s, e, rs, re)
    es, em = orc.window_sums(exp, rs, re, W)
    ea, ec = orc.class_runs(exp, rs, re, mincov, maxmean, 0)
    ws, r0, rc = ctx.depth_region_packed8(rs, re, a, d, ln, W, mincov, maxmean)
    assert ctx.depth_last_path() == 3
    assert np.array_equal(ctx.depth_perbase(re - rs), exp)
    assert np.array_equal(ws, es)
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
    ctx.depth_begin(rs, re)
    ctx.depth_add_segments_packed8(a, d, ln)
    ws, wm = ctx.depth_windows(W, es.size)
    assert ctx.depth_last_path() == 3
    assert np.array_equal(ws, es) and np.array_equal(wm, em)
    return exp


def _background(rng, lo, hi, n, holes, top=INT32_MAX):
    """n random segments starting in [lo, hi), none of them covering a base of a hole [h0, h1); ~5 % filler slots"""
    st = rng.integers(lo, hi, n)
    ln = rng.integers(1, 256, n)
    ln = np.minimum(ln, top - st)
    ok = np.ones(n, bool)
    for h0, h1 in holes:
        ok &= (st + ln <= h0) | (st >= h1)
    ln = np.where(rng.random(n) < 0.05, 0, ln)
    return [(int(x), int(y)) for x, y in zip(st[ok], ln[ok])]


def _edges(rs, tiles, seed):
    """segments at the positions each clamp rule handles, in tiles 1..tiles-2 of a region starting at rs"""
    t = [rs + TILE * k for k in range(tiles + 1)]
    rng = np.random.default_rng(seed)
    segs = []
    # tile 1: ends exactly at the tile start (b == 0), starts at -1 and at -255 (length 255 ends at 0), ends before it
    segs += [(t[1] - 100, 100), (t[1] - 1, 1), (t[1] - 1, 50), (t[1] - 255, 255), (t[1] - 255, 254), (t[1] - 255, 1),
             (t[1] - 2, 2), (t[1] - 1, 255)]
    # tile 2: starts at 4095, ends at 4096, 4097 and 4096 + 254 (trailing guard), one starting exactly at the next tile
    segs += [(t[2] + 4095, 1), (t[2] + 4095, 255), (t[2] + 4096 - 100, 100), (t[2] + 4096 - 3, 4), (t[2] + 4096 - 1, 2),
             (t[2] + 4096, 7), (t[2] + 4000, 0)]
    # tile 4: after a long coverage gap, its leading block lies wholly more than 255 bases before it (every event clamps),
    # with fillers among its slots
    segs += [(t[4] - 3000 + i, 0 if i % 9 == 4 else 100) for i in range(60)]
    segs += [(t[4] + 50 + 3 * i, 120) for i in range(40)]
    # tile 6: warp 0 of the first pass is the leading block plus a block of segments in [-250, -37): all 32 lanes clamp
    # both events; the next block starts 1 base before the tile
    segs += [(t[6] - 2000 + i, 100) for i in range(64)]
    segs += [(t[6] - 250 + i, 150 - (i & 31)) for i in range(64)]
    segs += [(t[6] - 1, 30 + i) for i in range(64)]
    segs += [(t[6] + 10 * i, 200) for i in range(64)]
    # tile 8: a pile-up across the tile start and a deep one inside it: more than 32 blocks, five passes
    segs += [(int(x), 255) for x in np.sort(rng.integers(t[8] - 255, t[8], 500))]
    segs += [(int(x), int(y)) for x, y in zip(np.sort(rng.integers(t[8] + 100, t[8] + 1000, 2200)),
                                              np.where(rng.random(2200) < 0.1, 0, rng.integers(1, 256, 2200)))]
    # tile 10: a trailing block whose later slots start past the tile's end
    segs += [(t[10] + 3990 + 5 * i, 0 if i == 63 else 60) for i in range(64)]
    holes = [(t[4] - 7000, t[4] + 40), (t[6] - 3000, t[6] + 700), (t[10] + 3000, t[11] + 400)]
    return segs, holes


@pytest.mark.parametrize("rs", [0, 1000, 4096 * 3 + 17])
def test_guard_edges(ctx, rs):
    """every clamp rule, with region starts on and off the tile grid and a ragged last tile"""
    tiles = 13
    re = rs + TILE * (tiles - 1) + 777
    segs, holes = _edges(rs, tiles, rs)
    segs += _background(np.random.default_rng(rs + 1), max(0, rs - 300), re, 2500, holes)
    packed, s, e = _pack(segs)
    lo = np.searchsorted(packed[0], rs + TILE * 8 - 255) - 1
    hi = np.searchsorted(packed[0], rs + TILE * 9)
    assert hi - lo > 32                                              # tile 8 needs five passes
    exp = _check(ctx, packed, s, e, rs, re)
    assert exp.max() >= 400
    _check(ctx, packed, s, e, rs, re, W=13, mincov=2, maxmean=300)


def test_region_ending_at_int32_max(ctx):
    """the last tiles of the int32 range: ends at INT32_MAX, starts in the trailing guard of the last tile"""
    rs = INT32_MAX - (TILE * 5 + 123)
    re = INT32_MAX
    t = [rs + TILE * k for k in range(6)]
    segs = [(t[1] - 1, 1), (t[1] - 255, 255), (t[2] + 4095, 255), (re - 255, 255), (re - 1, 1), (re - 2, 0),
            (rs - 200, 255), (rs - 1, 1)]
    segs += _background(np.random.default_rng(5), rs - 255, re, 2000, [])
    packed, s, e = _pack(segs)
    _check(ctx, packed, s, e, rs, re)
    _check(ctx, packed, s, e, rs + 4096, re - 1, W=97, mincov=1)


def test_one_context_across_contigs():
    """a fresh context, reused: contigs whose lead guards take many events, then ones where stale guard sums would show
    as a wrong depth"""
    runs = []
    for rs in (0, 1000):
        re = rs + TILE * 12 + 777
        segs, holes = _edges(rs, 13, 40 + rs)
        runs.append((segs + _background(np.random.default_rng(41 + rs), rs, re, 2500, holes), rs, re))
    runs.append(([(5, 100), (4000, 96), (4095, 255), (8191, 1)], 0, 9000))
    runs.append(([(5000 + 3 * i, 200) for i in range(300)], 4096, 4096 * 4))
    with capi.Ctx(0) as c:
        for segs, rs, re in runs + runs[::-1]:
            packed, s, e = _pack(segs)
            _check(c, packed, s, e, rs, re)


def test_multidepth_through_fused8(ctx):
    """`goleft multidepth` counts each sample through the same kernel"""
    L = TILE * 12 + 777
    samples = []
    for k in range(3):
        segs, holes = _edges(0, 13, 60 + k)
        samples.append(_pack(segs + _background(np.random.default_rng(61 + k), 0, L, 2500, holes)))
    depth = np.stack([orc.pileup_diff(s, e, 0, L) for _, s, e in samples])
    exp, _ = omd.text("chrG", depth, mincov=5, window=1000)
    adders = [lambda c, p=p: c.depth_add_segments_packed8(*p) for p, _, _ in samples]
    assert ctx.multidepth("chrG", L, adders, mincov=5, window=1000) == exp
