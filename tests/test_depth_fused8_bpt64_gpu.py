"""K_fused8's core gives each thread 64 consecutive bases in 64-thread CTAs (tile_core<64, 2>): a warp covers 2048 bases,
run-start masks are 64 bits wide, the fast window path holds for W >= 64 with depth below 2^21, and a thread reads its
differences in two halves of 32, so what happens in bases 32-63 of a thread is where this shape differs from the
others.  These regions put window edges, class changes, forced run breaks, the ragged end and multidepth block edges
there, and check every depth path against oracle/oracle_depth.c through the C ABI (check_region), and multidepth
against oracle/multidepth.py.  Needs an H100 (`-m gpu`)."""
import numpy as np
import pytest

from oracle import multidepth as omd
from test_depth_gpu import check_region, rand_segments
from test_depth_window_edges_gpu import _deep_stack
from test_multidepth_gpu import CHROM, _depths, _run

pytestmark = pytest.mark.gpu

TILE = 4096
BPT = 64
WARP = 32 * BPT                                              # 2048 bases
WINDOWS = [32, 33, 63, 64, 65, 500, 10000]
CU = [0, 1, 31, 32, 33, 63]                                  # bases of a thread left of its window edge
LANES = [0, 31, 32, 33]                                      # lane 0 and the last lane of warp 0, warp 1's first two
LEN = 3 * TILE + 1555                                        # three full tiles and a ragged last one


def _coverage(rng, rs, re, cov, read_len=150):
    n = max(1, int(cov * (re - rs) / read_len))
    s, e = rand_segments(rng, n, rs - read_len, re, maxlen=2 * read_len)
    o = np.argsort(s, kind="stable")
    return s[o], e[o]


def _cut(s, e, h0, h1):
    """the reads with [h0, h1) taken out: depth drops to 0 exactly at h0 and comes back exactly at h1"""
    s0, e0 = s[s < h0], np.minimum(e[s < h0], h0)
    s1, e1 = np.maximum(s[e > h1], h1), e[e > h1]
    s, e = np.concatenate([s0, s1]), np.concatenate([e0, e1])
    keep = s < e
    o = np.argsort(s[keep], kind="stable")
    return s[keep][o], e[keep][o]


def _first_edge_at(W, t):
    """a region start off the tile grid whose first window edge at or after it lies t bases in (t < W) or t mod W bases in"""
    return W * (7 * TILE // W + 1) - t % W


@pytest.mark.parametrize("W", WINDOWS)
def test_window_edges_in_64_base_threads(ctx, W):
    """30x everywhere: window edges at cu = 0, 1, 31, 32, 33, 63 of lane 0, lane 31 and warp 1's first lanes"""
    rng = np.random.default_rng(W)
    seen = set()
    for lane in LANES:
        for cu in CU:
            rs = _first_edge_at(W, BPT * lane + cu)
            if rs in seen:
                continue
            seen.add(rs)
            s, e = _coverage(rng, rs, rs + LEN, 30)
            check_region(ctx, s, e, rs, rs + LEN, W)


@pytest.mark.parametrize("depth", [(1 << 21) - 200, (1 << 21) + 1])
def test_depth_around_2_21_in_one_warp(ctx, depth):
    """a stack of `depth` reads over one 2048-base warp: just under 2^21 its window sums come close to 2^32 on the fast
    path; just over, that warp takes the slice loop while its neighbour in the tile stays on the fast path"""
    rng = np.random.default_rng(depth & 0xff)
    rs, L = 5000 - 37, 3 * TILE + 501
    ds, de = _deep_stack(depth, rs + WARP, rs + 2 * WARP)
    s, e = rand_segments(rng, 3000, rs - 100, rs + L + 100, maxlen=250)
    s = np.concatenate([s, ds]); e = np.concatenate([e, de])
    o = np.argsort(s, kind="stable")
    for W in (500, 4096):
        check_region(ctx, s[o], e[o], rs, rs + L, W, maxmean=1000)


@pytest.mark.parametrize("W", [64, 500])
@pytest.mark.parametrize("off", [32, 45, 63])
def test_class_changes_and_breaks_in_upper_half(ctx, W, off):
    """a zero-coverage hole that starts and ends in bases 32-63 of a thread, and a forced 10 Mb run break there: the
    warp with the hole needs the 64-bit run mask and the depth slice, the tile's other warp stays on the fast path"""
    rng = np.random.default_rng(100 * W + off)
    rs = 10_000_000 - 2 * TILE - (BPT * 5 + off)             # the 10 Mb break: tile 2, lane 5, base `off`
    L = 4 * TILE + WARP + BPT * 3 + off                      # the ragged end: warp 1, lane 3, base `off`
    s, e = _coverage(rng, rs, rs + L, 30)
    h0 = rs + TILE + WARP + BPT * 7 + off                    # tile 1, warp 1
    h1 = rs + TILE + WARP + BPT * 20 + (off + 9) % BPT
    s, e = _cut(s, e, h0, h1)
    check_region(ctx, s, e, rs, rs + L, W, mincov=4, maxmean=0, run_break=10_000_000)
    check_region(ctx, s, e, rs, rs + L, W, mincov=25, maxmean=35, run_break=10_000_000)


def test_region_ending_at_int32_max(ctx):
    """the ragged last tile at the top of the coordinate range, ending in the upper half of a warp-1 thread"""
    rng = np.random.default_rng(31)
    re = 2 ** 31 - 1
    rs = re - (3 * TILE + WARP + BPT * 9 + 40)
    s, e = rand_segments(rng, 600, rs - 150, re - 300, maxlen=300)
    o = np.argsort(s, kind="stable")
    for W in (64, 500):
        check_region(ctx, s[o], e[o], rs, re, W)


def _tiled(L, cov, seed, read_len=150):
    rng = np.random.default_rng(seed)
    n = int(cov * L / read_len)
    s = np.sort(rng.integers(-read_len, L, n)).astype(np.int32)
    e = (s + read_len).astype(np.int32)
    return np.maximum(s, 0), np.minimum(e, L)


def test_multidepth_block_edges_in_upper_half(ctx):
    """multidepth pass 1 (site classes) and pass 2 (block sums): holes in one sample start and end in bases 32-63 of a
    thread, so sufficient-site blocks begin and end there, in both warps of a tile"""
    L = 9 * TILE + 1000
    samples = [_tiled(L, c, 40 + i) for i, c in enumerate([14, 20, 12])]
    s, e = samples[1]
    for h0, h1 in [(TILE + BPT * 3 + 40, TILE + BPT * 8 + 50),                     # warp 0
                   (3 * TILE + WARP + BPT * 2 + 33, 4 * TILE + BPT * 30 + 63),      # warp 1 into the next tile's warp 0
                   (6 * TILE + WARP - 20, 6 * TILE + WARP + BPT + 32)]:             # across the warp boundary
        s, e = _cut(s, e, h0, h1)
    samples[1] = (s, e)
    exp, _ = omd.text(CHROM, _depths(L, samples), window=500)
    for form in ("packed8", "host32"):
        got, _ = _run(ctx, L, samples, form, window=500)
        assert got == exp, form
