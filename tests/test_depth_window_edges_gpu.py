"""Window edges at every position the tile core's fast window path distinguishes, on every depth path (the packed8 core owns
32 bases per thread, 1024 per warp; the others 16 and 512), against oracle/oracle_depth.c.  An edge falls at offset
el * BPT + cu of a warp: on a thread boundary (cu = 0), inside lane 0, on the warp's last base, exactly at the warp's end,
or beyond it.  Needs an H100 (`-m gpu`)."""
import numpy as np
import pytest

from goleft_b200 import synth
from test_depth_gpu import check_region, rand_segments

pytestmark = pytest.mark.gpu

EDGE_WINDOWS = [16, 31, 32, 33, 63, 64, 511, 512, 513, 1023, 1024, 1025, 4095, 4097]
# offset of the first window edge from the region start (= from every warp start modulo W): lane 0, a thread boundary,
# the last base of a 512- and of a 1024-base warp, exactly at their ends, and just past them
EDGE_OFFSETS = [1, 5, 16, 31, 32, 33, 511, 512, 513, 1023, 1024, 1025]
TAIL = 3 * 4096 + 777                                        # three full tiles and a ragged last one


@pytest.mark.parametrize("W", EDGE_WINDOWS)
def test_window_edge_positions(ctx, W):
    rng = np.random.default_rng(W)
    seen = set()
    for t in EDGE_OFFSETS:
        rs = 3 * W + (-t) % W                                # window edges at rs + t + k*W
        if rs in seen:
            continue
        seen.add(rs)
        s, e = rand_segments(rng, 2500, rs - 200, rs + TAIL + 100, maxlen=300)
        check_region(ctx, s, e, rs, rs + TAIL, W)


def _deep_stack(depth, a, b):
    return np.full(depth, a, np.int32), np.full(depth, b, np.int32)


@pytest.mark.parametrize("depth", [(1 << 22) - 1, (1 << 22) + 1])
def test_depth_around_fast_window_limit(ctx, depth):
    """A stack of `depth` reads over whole warps: just under 2^22 a full 1024-base window of it sums to just under 2^32
    inside one warp (the fast path's unsigned REDUX); just over, those warps take the general loop and the rest do not."""
    rng = np.random.default_rng(depth & 0xff)
    rs, L = 3000, 3 * 4096 + 501
    ds, de = _deep_stack(depth, rs + 1024, rs + 1024 + 200)
    ds2, de2 = _deep_stack(depth // 64, rs + 4096 + 100, rs + 4096 + 355)
    s, e = rand_segments(rng, 3000, rs - 100, rs + L + 100, maxlen=250)
    s = np.concatenate([s, ds, ds2]); e = np.concatenate([e, de, de2])
    for W in (1024, 500):
        check_region(ctx, s, e, rs, rs + L, W, maxmean=1000)


@pytest.mark.parametrize("W", [500, 1024, 33])
def test_30x_region_classes(ctx, W):
    """30x / 150 bp reads: mincov and maxmean classes change inside warps while the windows take the fast path"""
    L = 200_000
    s, e = synth.segments(synth.reads(L, contig_index=3))
    check_region(ctx, s, e, 0, L, W, mincov=20, maxmean=40)
    check_region(ctx, s, e, 777, L - 301, W, mincov=4, maxmean=35)
