"""The tile core's fast window path works from registers: each thread finds the one window edge inside its bases (cu of
them left of it, cu = 0: none), a warp scan of the threads' depth sums gives each edge its window's part, and the edge
lanes add those parts together, plus one add for the window that runs past the warp's end.  These regions put edges at
every position that distinguishes: on a thread's first base (cu = 0), at cu = 1 and cu = BPT - 1 for both core shapes
(16 and 32 bases per thread), on lane 0, at warp and tile boundaries, and warps with no edge at all.  Other regions mix
warps that need the depth slice (class runs at 5x, a forced run break, a zero-coverage gap, the ragged last tile, W < BPT,
depth around 2^22) with warps that do not.  Every depth path (packed8, fused int32, both general paths) and the
per-window minima against oracle/oracle_depth.c, through the C ABI (check_region).  Needs an H100 (`-m gpu`)."""
import numpy as np
import pytest

from oracle import multidepth as omd
from test_depth_gpu import check_region, rand_segments
from test_depth_window_edges_gpu import _deep_stack
from test_multidepth_gpu import CHROM, _cohort, _depths, _run

pytestmark = pytest.mark.gpu

TILE = 4096
WINDOWS = [16, 17, 32, 33, 250, 500, 511, 4096, 10000]
# offset of the first window edge from the region start: cu = 1 on lane 0, cu = 15 / 16 / 17, a thread boundary of both
# shapes (32), cu = 31, the last base of and exactly at a 512- and a 1024-base warp's end, a tile boundary and just past it
EDGE_OFFSETS = [1, 15, 16, 17, 31, 32, 33, 511, 512, 1023, 1024, 1025, 4095, 4096, 4097]
LEN = 4 * TILE + 777                                         # four full tiles and a ragged last one


def _coverage(rng, rs, re, cov, read_len=150):
    n = max(1, int(cov * (re - rs) / read_len))
    return rand_segments(rng, n, rs - read_len, re, maxlen=2 * read_len)


@pytest.mark.parametrize("W", WINDOWS)
def test_edge_positions(ctx, W):
    """30x everywhere: apart from the region's first warp, the warps of full tiles take the fast window path and store
    no depth slice"""
    rng = np.random.default_rng(W)
    seen = set()
    for t in EDGE_OFFSETS:
        rs = 7 * max(W, TILE) - t % W                        # window edges at rs + t + k*W; rs is off the 4096 grid
        if rs in seen:
            continue
        seen.add(rs)
        s, e = _coverage(rng, rs, rs + LEN, 30)
        check_region(ctx, s, e, rs, rs + LEN, W)


@pytest.mark.parametrize("W", [17, 250, 500, 4096, 10000])
def test_slow_and_fast_warps_in_one_tile(ctx, W):
    """30x tiles whose warps have no class change beside 5x stretches (class runs at mincov 4), a zero-coverage gap
    inside a tile and a forced run break inside a tile: warps that store the depth slice and warps that do not"""
    rng = np.random.default_rng(1000 + W)
    rs = 3 * TILE + 1234
    re = rs + 6 * TILE + 501
    parts = [_coverage(rng, rs, rs + 2 * TILE + 300, 30),
             _coverage(rng, rs + 2 * TILE + 300, rs + 2 * TILE + 1800, 5),
             _coverage(rng, rs + 2 * TILE + 3000, re, 30)]   # no read starts in [2*TILE + 1800, 2*TILE + 3000)
    s = np.concatenate([p[0] for p in parts]); e = np.concatenate([p[1] for p in parts])
    o = np.argsort(s, kind="stable")
    s, e = s[o], e[o]
    check_region(ctx, s, e, rs, re, W, mincov=4, maxmean=0)
    check_region(ctx, s, e, rs, re, W, mincov=4, maxmean=0, run_break=rs + 5 * TILE + 77)
    check_region(ctx, s, e, rs, re, W, mincov=25, maxmean=45)


@pytest.mark.parametrize("W", [5, 31])
def test_window_below_bases_per_thread(ctx, W):
    """W < 32 takes the general window loop in the packed8 core; W = 31 still takes the fast path in the 16-base cores"""
    rng = np.random.default_rng(W)
    rs = 2 * TILE + 99
    s, e = _coverage(rng, rs, rs + 2 * TILE + 300, 30)
    check_region(ctx, s, e, rs, rs + 2 * TILE + 300, W)


@pytest.mark.parametrize("depth", [(1 << 22) - 200, (1 << 22) + 1])
def test_depth_around_fast_window_limit(ctx, depth):
    """a stack of `depth` reads over one 1024-base warp, under ~30x of other reads: just under 2^22 that warp's partial
    sums come close to 2^32 on the fast path; just over, it takes the general loop while the others stay on the fast path"""
    rng = np.random.default_rng(depth & 0xff)
    rs, L = 5000 - 37, 3 * TILE + 501
    ds, de = _deep_stack(depth, rs + 1024, rs + 1024 + 1024)
    s, e = rand_segments(rng, 3000, rs - 100, rs + L + 100, maxlen=250)
    s = np.concatenate([s, ds]); e = np.concatenate([e, de])
    for W in (250, 10000):
        check_region(ctx, s, e, rs, rs + L, W, maxmean=1000)


def test_multidepth_with_slow_warps(ctx):
    """multidepth pass 1 (site classes) and pass 2 (block sums) share the tile core: a cohort where a 3x sample and an
    empty stretch put class changes inside warps of 14x tiles, packed8 and int32"""
    L = 90_000
    samples = _cohort(L, [14, 3, 20], 17)
    s, e = samples[2]
    keep = (s < 30_000) | (s > 31_500)                       # a zero-coverage gap in sample 3
    samples[2] = (s[keep], e[keep])
    exp, _ = omd.text(CHROM, _depths(L, samples), window=500)
    for form in ("packed8", "host32"):
        got, _ = _run(ctx, L, samples, form, window=500)
        assert got == exp, form
