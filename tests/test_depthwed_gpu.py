"""depthwed (W1) kernels and the covstats histogram (V2) at the shapes, widths and values where they can go wrong.

Expectations come from the C oracle (oracle/oracle_indexcov.c: `orc.depthwed`, `orc.bincount`) where it is defined, from
closed forms at the benchmark's 500 x 6,176,584 shape, and — for Go's `int(0.5 + dep)` (depthwed.go:103) on NaN, +-Inf and
values outside [-2^63, 2^63), where the oracle's C conversion is undefined — from `go_int` below, a numpy restatement of
what Go compiles that line to on amd64 (CVTTSD2SQ): truncation toward zero, INT64_MIN for every input it cannot convert,
and group sums that wrap modulo 2^64.  Tests without the gpu marker check those references themselves."""
import os
import subprocess

import numpy as np
import pytest

from goleft_b200 import capi, multigpu
from oracle import loader as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLEFT = os.path.join(ROOT, "bin", "goleft")
I32_MIN, I32_MAX = -2 ** 31, 2 ** 31 - 1
I64_MIN = -2 ** 63
SENTINEL = -123456789


# ---------------------------------------------------------------------------------------------------- references
def go_int(x) -> np.ndarray:
    """int(0.5 + x) as Go compiles it for amd64: trunc(0.5 + x) when that is finite and in [-2^63, 2^63), else INT64_MIN"""
    y = np.float64(0.5) + np.asarray(x, np.float64)
    with np.errstate(invalid="ignore"):
        ok = np.isfinite(y) & (y >= -2.0 ** 63) & (y < 2.0 ** 63)
    out = np.full(y.shape, I64_MIN, np.int64)
    out[ok] = np.trunc(y[ok]).astype(np.int64)
    return out


def go_sums(cells: np.ndarray, grp: np.ndarray) -> np.ndarray:
    """cells: S x R int64; rows [grp[g], grp[g+1]) summed with int64 wrap-around -> n_out x S"""
    return np.add.reduceat(cells, grp[:-1], axis=1).T.copy()


def layout(rng, R: int, n_chrom: int = 3):
    """R rows over n_chrom chromosomes, mostly 250 bases wide with some of 1000 and 3000: at -s 1000 that gives one-row
    groups, groups of 2-4 rows, and a short last group on every chromosome (a 250-base row after a 3000-base one)"""
    chrom = np.repeat(np.arange(n_chrom), np.diff(np.linspace(0, R, n_chrom + 1).astype(np.int64))).astype(np.int32)
    widths = rng.choice([250, 250, 250, 250, 250, 1000, 3000], R)
    starts = np.zeros(R, np.int64)
    for c in range(n_chrom):
        idx = np.flatnonzero(chrom == c)
        widths[idx[-2]], widths[idx[-1]] = 3000, 250
        starts[idx] = np.concatenate([[0], np.cumsum(widths[idx])[:-1]])
    return starts.astype(np.int32), (starts + widths).astype(np.int32), chrom


def oracle_groups(starts, ends, chrom, size):
    """the oracle's row groups as a table grp[0..n_out]: its sums of all-ones means are the group lengths"""
    o_s, o_e, o_c, n = orc.depthwed(np.ones((1, starts.size)), starts, ends, chrom, size)
    return np.concatenate([[0], np.cumsum(n[:, 0])]).astype(np.int64), o_s, o_e, o_c


def oracle_i32(depth: np.ndarray, starts, ends, chrom, size) -> np.ndarray:
    """int64 group sums of int32 depths from the oracle: int(0.5 + (d - 0.5)) == d exactly for |d| < 2^51"""
    return orc.depthwed(depth.astype(np.float64) - 0.5, starts, ends, chrom, size)[3]


def chunk_list(n: int, scheme, rng):
    if scheme == "whole":
        return [(0, n)]
    if scheme == "uneven":
        cuts = np.unique(np.concatenate([[0, n], rng.integers(0, n, max(1, n // 40))]))
        return list(zip(cuts[:-1].tolist(), cuts[1:].tolist()))
    return [(a, min(a + scheme, n)) for a in range(0, n, scheme)]


# ---------------------------------------------------------------------------------------------------- CPU: the references
def test_go_int_rule_hand_values():
    """the numpy rule on the values where int(0.5 + x) is easy to get wrong"""
    cases = [(0.5, 1), (-0.5, 0), (1.5, 2), (-1.5, -1), (2.5, 3), (0.49999999999999994, 1), (-0.0, 0), (-0.7, 0),
             (-1.2, 0), (-1.7, -1), (2.0 ** 52 + 1, 2 ** 52 + 2), (2.0 ** 52 + 2, 2 ** 52 + 2), (2.0 ** 53 - 1, 2 ** 53),
             (2.0 ** 31 - 1, 2 ** 31 - 1), (2.0 ** 31, 2 ** 31), (2.0 ** 31 + 1, 2 ** 31 + 1),
             (2.0 ** 63 - 1024, 2 ** 63 - 1024), (-2.0 ** 63, I64_MIN), (2.0 ** 63, I64_MIN), (-2.0 ** 63 - 2048, I64_MIN),
             (1e19, I64_MIN), (-1e19, I64_MIN), (np.inf, I64_MIN), (-np.inf, I64_MIN), (np.nan, I64_MIN)]
    got = go_int(np.array([c[0] for c in cases]))
    assert got.tolist() == [c[1] for c in cases]
    # sums wrap as Go's int does
    cells = np.array([[2 ** 62, 2 ** 62, I64_MIN, I64_MIN, -1, I64_MIN]], np.int64)
    assert go_sums(cells, np.array([0, 2, 4, 6])).ravel().tolist() == [I64_MIN, 0, 2 ** 63 - 1]


def test_go_int_rule_equals_oracle_on_finite_cells():
    """on every finite, in-range cell the numpy rule is the oracle's (int64_t)(0.5 + x), cell by cell and summed"""
    rng = np.random.default_rng(21)
    starts, ends, chrom = layout(rng, 900)
    S = 9
    means = np.concatenate([rng.gamma(9, 3.3, (3, 900)), rng.normal(0, 40, (2, 900)),
                            rng.uniform(-2.0 ** 58, 2.0 ** 58, (2, 900)), np.round(rng.normal(0, 5, (2, 900))) * 0.5])
    edges = np.array([0.5, -0.5, 1.5, -1.5, 2.5, 0.49999999999999994, -0.0, -0.7, 2.0 ** 52 + 1, 2.0 ** 52 + 3,
                      2.0 ** 53 - 1, 2.0 ** 31 - 1, 2.0 ** 31, 2.0 ** 31 + 1, -2.0 ** 31 - 1])
    means[rng.integers(0, S, 400), rng.integers(0, 900, 400)] = rng.choice(edges, 400)
    cells = go_int(means)
    assert np.array_equal(orc.depthwed(means, starts, ends, chrom, 1)[3], cells.T)
    for size in (1000, 5000):
        grp = oracle_groups(starts, ends, chrom, size)[0]
        assert np.array_equal(orc.depthwed(means, starts, ends, chrom, size)[3], go_sums(cells, grp))
    # the extremes the oracle can still convert: the largest double below 2^63 and -2^63 itself
    top = np.array([[2.0 ** 63 - 1024, -2.0 ** 63, 2.0 ** 62]])
    o = orc.depthwed(top, np.array([0, 1, 2], np.int32), np.array([1, 2, 3], np.int32), np.zeros(3, np.int32), 1)[3]
    assert np.array_equal(o.ravel(), go_int(top).ravel())


def test_layout_has_every_group_shape():
    rng = np.random.default_rng(1)
    starts, ends, chrom = layout(rng, 3000)
    grp, o_s, o_e, o_c = oracle_groups(starts, ends, chrom, 1000)
    n = np.diff(grp)
    assert n.min() == 1 and n.max() == 4 and {1, 2, 3, 4} <= set(n.tolist())
    for c in range(3):
        last = np.flatnonzero(o_c == c)[-1]
        assert o_e[last] - o_s[last] < 1000                       # a short last group on every chromosome


def test_bincount_oracle_at_int32_edges():
    """the oracle histogram equals numpy's at the ranges the GPU test uses"""
    rng = np.random.default_rng(2)
    for lo, hi in bincount_ranges():
        v = bincount_values(rng, lo, hi, 257)
        m = (v.astype(np.int64) >= lo) & (v.astype(np.int64) < hi)
        exp = np.bincount(v[m].astype(np.int64) - lo, minlength=hi - lo).astype(np.uint64)
        assert np.array_equal(orc.bincount(v, lo, hi), exp), (lo, hi)


# ---------------------------------------------------------------------------------------------------- 1. depthwed_i32_kernel
def run_i32_chunks(ctx, d_depth, S, R, d_grp, n_out, chunks, extra=64):
    """every chunk [g0, g1) written at row g0 of one sentinel-filled buffer; returns (n_out x S, tail, overflow flag)"""
    d_out = ctx.dev_array(np.full(n_out * S + extra, SENTINEL, np.int32))
    d_ovf = ctx.dev_array(np.zeros(4, np.int32))
    for g0, g1 in chunks:
        ctx.depthwed_aggregate_i32_device(d_depth, S, R, d_grp, g0, g1, d_out.ptr + g0 * S * 4, d_ovf)
    ctx.sync()
    flat = d_out.download(np.int32, n_out * S + extra)
    ovf = int(d_ovf.download(np.int32, 1)[0])
    d_out.free(); d_ovf.free()
    return flat[:n_out * S].reshape(n_out, S), flat[n_out * S:], ovf


@pytest.mark.gpu
@pytest.mark.parametrize("S", [1, 4, 31, 32, 33, 127, 128, 129, 500, 2504])
def test_i32_device_row_ranges_groups_and_widths(ctx, S):
    rng = np.random.default_rng(100 + S)
    R, size = 3000, 1000
    starts, ends, chrom = layout(rng, R)
    depth = rng.integers(-50, 1000, (S, R)).astype(np.int32)
    big = rng.random((S, R)) < 0.01
    depth[big] = rng.integers(-10 ** 6, 10 ** 6, int(big.sum()))
    grp = oracle_groups(starts, ends, chrom, size)[0]
    d_depth, d_grp = ctx.dev_array(depth), ctx.dev_array(grp)
    for grouped in (True, False):
        exp = oracle_i32(depth, starts, ends, chrom, size if grouped else 1)
        n_out = exp.shape[0]
        assert n_out == (grp.size - 1 if grouped else R)
        for scheme in ("whole", 1, 31, 32, 33, "uneven"):
            got, tail, ovf = run_i32_chunks(ctx, d_depth, S, R, d_grp if grouped else None, n_out,
                                            chunk_list(n_out, scheme, rng))
            assert np.array_equal(got.astype(np.int64), exp), (S, grouped, scheme)
            assert (tail == SENTINEL).all() and ovf == 0, (S, grouped, scheme)
    d_depth.free(); d_grp.free()


def planted_overflow_problem():
    """5 samples; group sums of exactly INT32_MAX, INT32_MAX + 1, INT32_MIN, INT32_MIN - 1, a 3-row group whose running
    sum leaves int32 but whose total does not, and one-row groups holding INT32_MAX / INT32_MIN"""
    rng = np.random.default_rng(33)
    R, S = 400, 5
    starts, ends, chrom = layout(rng, R)
    grp = oracle_groups(starts, ends, chrom, 1000)[0]
    n = np.diff(grp)
    depth = rng.integers(-30, 300, (S, R)).astype(np.int64)
    multi = np.flatnonzero(n >= 3)
    one = np.flatnonzero(n == 1)
    for s, target in enumerate([I32_MAX, I32_MAX + 1, I32_MIN, I32_MIN - 1]):
        g = multi[5 + 7 * s]
        r = grp[g]
        depth[s, r:grp[g + 1]] = 0
        depth[s, r], depth[s, r + 1] = target // 2, target - target // 2
    g = multi[40]
    depth[4, grp[g]:grp[g + 1]] = 0
    depth[4, grp[g]:grp[g] + 3] = [I32_MAX, I32_MAX, I32_MIN]
    depth[0, grp[one[3]]] = I32_MAX
    depth[1, grp[one[4]]] = I32_MIN
    depth = depth.astype(np.int32)
    sums = oracle_i32(depth, starts, ends, chrom, 1000)
    ovf = ((sums > I32_MAX) | (sums < I32_MIN)).any(axis=1)
    assert ovf.sum() == 2
    return depth, grp, sums, ovf


@pytest.mark.gpu
def test_i32_overflow_flag_exactly_when_a_sum_leaves_int32(ctx):
    depth, grp, sums, ovf = planted_overflow_problem()
    S, R = depth.shape
    n_out = grp.size - 1
    assert ((sums == I32_MAX).any() and (sums == I32_MIN).any() and (sums == I32_MAX + 1).any() and (sums == I32_MIN - 1).any())
    d_depth, d_grp = ctx.dev_array(depth), ctx.dev_array(grp)
    rng = np.random.default_rng(3)
    fits = ~ovf
    for scheme in (1, 31, 32, 33, "uneven", "whole"):
        for g0, g1 in chunk_list(n_out, scheme, rng):
            got, tail, flag = run_i32_chunks(ctx, d_depth, S, R, d_grp, n_out, [(g0, g1)])
            assert flag == int(ovf[g0:g1].any()), (scheme, g0, g1)
            rows = np.arange(g0, g1)[fits[g0:g1]]
            assert np.array_equal(got[rows].astype(np.int64), sums[rows]), (scheme, g0, g1)
            assert (tail == SENTINEL).all()
    # the fused kernel raises the same flag
    for g in range(n_out):
        d_dst = ctx.dev_array(np.full(n_out * S, SENTINEL, np.int32))
        d_ovf = ctx.dev_array(np.zeros(4, np.int32))
        ctx.depthwed_aggregate_i32_p2p(d_depth, S, R, d_grp, g, g + 1, [d_dst.ptr], S, 0, d_ovf)
        ctx.sync()
        assert int(d_ovf.download(np.int32, 1)[0]) == int(ovf[g]), g
        if not ovf[g]:
            assert np.array_equal(d_dst.download(np.int32, n_out * S).reshape(n_out, S)[g].astype(np.int64), sums[g])
        d_dst.free(); d_ovf.free()
    d_depth.free(); d_grp.free()


# ---------------------------------------------------------------------------------------------------- 2. depthwed_i32_p2p_kernel
# (world, S, row_stride, col_off, destination offsets in bytes, grouped, chunking)
P2P_CASES = [
    (1, 128, 128, 0, [0], True, "whole"),                            # 16-byte stores
    (1, 129, 132, 0, [0], False, "whole"),                           # S % 4 == 1: a scalar tail
    (2, 130, 264, 132, [0, 0], True, 33),                            # S % 4 == 2, second rank's columns
    (3, 131, 140, 8, [0, 0, 0], False, "uneven"),                    # S % 4 == 3
    (2, 127, 130, 2, [0, 0], True, "whole"),                         # row_stride and col_off not multiples of 4: scalar
    (3, 256, 261, 4, [0, 0, 0], True, 32),                           # odd row_stride
    (2, 255, 260, 3, [0, 0], False, 1),                              # col_off not a multiple of 4
    (16, 257, 260, 0, [0] * 16, True, 32),                           # 16 destinations
    (16, 129, 133, 1, [0] * 16, False, "uneven"),
    (4, 253, 256, 0, [0] * 4, True, 31),
    (5, 254, 512, 256, [0] * 5, False, "whole"),
    (1, 258, 264, 4, [0], True, "uneven"),
    (2, 259, 259, 0, [0, 0], True, "whole"),                         # row_stride == S
    (1, 4, 4, 0, [0], False, "whole"),
    (2, 1, 5, 3, [0, 0], True, 1),
    (1, 128, 128, 0, [4], True, "whole"),                            # destinations 4-byte but not 16-byte aligned
    (2, 256, 256, 0, [0, 8], False, 33),
    (3, 132, 136, 4, [12, 0, 4], True, "uneven"),
    (16, 64, 64, 0, [0, 4, 8, 12] * 4, True, "whole"),
    (1, 131, 132, 0, [16], False, "whole"),                          # offset by a whole int4: still 16-byte stores
]


@pytest.mark.gpu
@pytest.mark.parametrize("world,S,row_stride,col_off,offs,grouped,scheme", P2P_CASES)
def test_p2p_kernel_on_one_device(ctx, world, S, row_stride, col_off, offs, grouped, scheme):
    rng = np.random.default_rng(world * 1000 + S)
    R, size = 1500, 1000
    starts, ends, chrom = layout(rng, R)
    depth = rng.integers(-100, 5000, (S, R)).astype(np.int32)
    grp = oracle_groups(starts, ends, chrom, size)[0]
    exp = oracle_i32(depth, starts, ends, chrom, size if grouped else 1)
    n_out = exp.shape[0]
    d_depth, d_grp = ctx.dev_array(depth), ctx.dev_array(grp)
    n_cells = n_out * row_stride + 64
    bufs = [ctx.dev_array(np.full(n_cells + 8, SENTINEL, np.int32)) for _ in range(world)]
    ptrs = [b.ptr + o for b, o in zip(bufs, offs)]
    d_ovf = ctx.dev_array(np.zeros(4, np.int32))
    for g0, g1 in chunk_list(n_out, scheme, rng):
        ctx.depthwed_aggregate_i32_p2p(d_depth, S, R, d_grp if grouped else None, g0, g1, ptrs, row_stride, col_off, d_ovf)
    ctx.sync()
    assert int(d_ovf.download(np.int32, 1)[0]) == 0
    for d, (b, o) in enumerate(zip(bufs, offs)):
        flat = b.download(np.int32, n_cells + 8)
        head, m, tail = flat[:o // 4], flat[o // 4:o // 4 + n_out * row_stride].reshape(n_out, row_stride), flat[o // 4 + n_out * row_stride:]
        assert np.array_equal(m[:, col_off:col_off + S].astype(np.int64), exp), d
        assert (m[:, :col_off] == SENTINEL).all() and (m[:, col_off + S:] == SENTINEL).all(), d
        assert (head == SENTINEL).all() and (tail == SENTINEL).all(), d
    for b in bufs + [d_depth, d_grp, d_ovf]:
        b.free()


@pytest.mark.gpu
def test_p2p_rejections(ctx):
    S, R = 8, 16
    d_depth = ctx.dev_array(np.ones((S, R), np.int32))
    d_dst = ctx.dev_array(np.zeros(R * 16, np.int32))
    d_ovf = ctx.dev_array(np.zeros(4, np.int32))
    bad = [dict(ptrs=[]), dict(ptrs=[d_dst.ptr] * 17), dict(ptrs=[d_dst.ptr, None]), dict(ptrs=[None]),
           dict(row_stride=S - 1), dict(row_stride=S + 3, col_off=4), dict(g0=5, g1=4), dict(g0=-1)]
    for b in bad:
        with pytest.raises(capi.GlError) as ei:
            ctx.depthwed_aggregate_i32_p2p(d_depth, S, R, None, b.get("g0", 0), b.get("g1", R), b.get("ptrs", [d_dst.ptr]),
                                           b.get("row_stride", 16), b.get("col_off", 0), d_ovf)
        assert ei.value.code == capi.GL_EINVAL, b
    ctx.depthwed_aggregate_i32_p2p(d_depth, S, R, None, 3, 3, [d_dst.ptr], 16, 0, d_ovf)     # an empty range is accepted
    ctx.depthwed_aggregate_i32_p2p(d_depth, S, R, None, 0, R, [d_dst.ptr] * 16, S, 0, d_ovf)
    ctx.sync()
    assert np.array_equal(d_dst.download(np.int32, R * S).reshape(R, S), np.ones((R, S), np.int32))
    for b in (d_depth, d_dst, d_ovf):
        b.free()


# ---------------------------------------------------------------------------------------------------- 3. the benchmark's shape
BENCH_S, BENCH_R = 500, 6_176_584            # 3.09e9 cells: sample-major and row-major offsets both pass 2^31


def bench_closed_form():
    """depth(s, r) = base[r] + col[s], uploaded column by column as bench.py does"""
    base = ((np.arange(BENCH_R, dtype=np.int64) * 2654435761) % 97).astype(np.int32)
    col = ((np.arange(BENCH_S, dtype=np.int64) * 104729) % 1000).astype(np.int32)
    return base, col


def fill(ctx, d, n_ints: int, value: int):
    piece = np.full(1 << 24, value, np.int32)
    for a in range(0, n_ints, piece.size):
        k = min(piece.size, n_ints - a)
        ctx._ck(capi.lib.gl_memcpy_h2d(ctx.h, d.ptr + a * 4, piece.ctypes.data, k * 4))


def check_rows(ctx, ptr: int, n_rows: int, S: int, rowval: np.ndarray, colval: np.ndarray, step: int = 1 << 17):
    """the row-major n_rows x S int32 matrix at ptr equals rowval[r] + colval[s] everywhere, read back in pieces"""
    got = np.empty((step, S), np.int32)
    exp = np.empty((step, S), np.int32)
    for g0 in range(0, n_rows, step):
        k = min(step, n_rows - g0)
        ctx._ck(capi.lib.gl_memcpy_d2h(ctx.h, got.ctypes.data, ptr + g0 * S * 4, k * S * 4))
        np.add(rowval[g0:g0 + k, None], colval[None, :], out=exp[:k])
        if not np.array_equal(got[:k], exp[:k]):
            bad = np.argwhere(got[:k] != exp[:k])[:5]
            raise AssertionError("rows %d..: first differences at %s: got %s want %s" % (
                g0, (bad + [g0, 0]).tolist(), got[:k][tuple(bad.T)].tolist(), exp[:k][tuple(bad.T)].tolist()))


@pytest.fixture(scope="module")
def bench_matrix():
    if capi.device_count() < 1:
        pytest.skip("no CUDA device")
    import torch  # noqa: F401  (loads the NCCL build that gl_comm_init finds with dlopen)
    base, col = bench_closed_form()
    c = capi.Ctx(0)
    d_depth = c.dev_empty(BENCH_S * BENCH_R * 4)
    for s in range(BENCH_S):
        h = base + col[s]
        c._ck(capi.lib.gl_memcpy_h2d(c.h, d_depth.ptr + s * BENCH_R * 4, h.ctypes.data, BENCH_R * 4))
    yield c, d_depth, base, col
    d_depth.free()
    c.close()


@pytest.mark.gpu
def test_benchmark_shape_kernels(bench_matrix):
    c, d_depth, base, col = bench_matrix
    S, R = BENCH_S, BENCH_R
    d_out = c.dev_empty(S * R * 4)
    d_ovf = c.dev_array(np.zeros(4, np.int32))
    try:
        # one-row groups (the benchmark's call), 8 row chunks
        fill(c, d_out, S * R, SENTINEL)
        for g0, g1 in multigpu.chunk_bounds(R, 8):
            c.depthwed_aggregate_i32_device(d_depth, S, R, None, g0, g1, d_out.ptr + g0 * S * 4, d_ovf)
        c.sync()
        check_rows(c, d_out.ptr, R, S, base, col)
        # 4-row groups from a table, 8 chunks of groups; the rows past the last group keep the sentinel
        grp = np.arange(0, R + 1, 4, dtype=np.int64)
        assert grp[-1] == R
        n_g = grp.size - 1
        d_grp = c.dev_array(grp)
        fill(c, d_out, S * R, SENTINEL)
        for g0, g1 in multigpu.chunk_bounds(n_g, 8):
            c.depthwed_aggregate_i32_device(d_depth, S, R, d_grp, g0, g1, d_out.ptr + g0 * S * 4, d_ovf)
        c.sync()
        check_rows(c, d_out.ptr, n_g, S, base.astype(np.int64).reshape(-1, 4).sum(1).astype(np.int32), 4 * col)
        check_rows(c, d_out.ptr + n_g * S * 4, 1 << 14, S, np.full(1 << 14, SENTINEL, np.int32), np.zeros(S, np.int32))
        d_grp.free()
        # the fused kernel with one destination: the whole row-major matrix
        fill(c, d_out, S * R, SENTINEL)
        c.depthwed_aggregate_i32_p2p(d_depth, S, R, None, 0, R, [d_out.ptr], S, 0, d_ovf)
        c.sync()
        check_rows(c, d_out.ptr, R, S, base, col)
        assert int(d_ovf.download(np.int32, 1)[0]) == 0
    finally:
        d_out.free(); d_ovf.free()


@pytest.mark.gpu
def test_benchmark_shape_overlapped_gather_world1(bench_matrix):
    """the benchmark's chunked aggregation + NCCL all-gather, on one rank"""
    c, d_depth, base, col = bench_matrix
    S, R = BENCH_S, BENCH_R
    try:
        c.comm_init(capi.comm_unique_id(), 0, 1)
    except capi.GlError as ex:
        if ex.code in (capi.GL_ENCCL, capi.GL_ENOMEM):
            pytest.skip("gl_comm_init(world=1) failed with %s: %s" % ("GL_ENCCL" if ex.code == capi.GL_ENCCL else "GL_ENOMEM", ex))
        raise
    d_local, d_all = c.dev_empty(S * R * 4), c.dev_empty(S * R * 4)
    d_ovf = c.dev_array(np.zeros(4, np.int32))
    try:
        fill(c, d_all, S * R, SENTINEL)
        multigpu.depthwed_gather_overlapped(c, d_depth, S, R, 1, d_local, d_all, d_ovf, 8)
        c.sync()
        check_rows(c, d_all.ptr, R, S, base, col)                   # one rank: [chunk][rank][rows][width] is row-major R x S
        assert int(d_ovf.download(np.int32, 1)[0]) == 0
    finally:
        d_local.free(); d_all.free(); d_ovf.free()


# ---------------------------------------------------------------------------------------------------- 4. float64 path at Go's edges
EDGES = [0.5, -0.5, 1.5, -1.5, 2.5, 0.49999999999999994, -0.0, -0.7, 2.0 ** 52 + 1, 2.0 ** 52 + 2, 2.0 ** 53 - 1,
         2.0 ** 31 - 1, 2.0 ** 31, 2.0 ** 31 + 1, -2.0 ** 31 - 1, 2.0 ** 63, -2.0 ** 63, 2.0 ** 63 - 1024, -2.0 ** 63 - 2048,
         1e19, -1e19, np.inf, -np.inf, np.nan]


def float64_edge_problem(S=70, R=700):
    rng = np.random.default_rng(44)
    starts, ends, chrom = layout(rng, R)
    grp = oracle_groups(starts, ends, chrom, 1000)[0]
    means = rng.gamma(9, 3.3, (S, R))
    means[1] = rng.normal(0, 3, R)
    means[rng.integers(0, S, 600), rng.integers(0, R, 600)] = rng.choice(np.array(EDGES), 600)
    means[2, :len(EDGES)] = EDGES                                   # every edge at least once
    two = np.flatnonzero(np.diff(grp) == 2)
    wraps = [[2.0 ** 62, 2.0 ** 62], [np.nan, np.inf], [2.0 ** 63 - 1024, 2.0 ** 63 - 1024], [-2.0 ** 62, -2.0 ** 62 - 2048],
             [-1e19, -1.0], [1e19, 3.0]]
    for k, pair in enumerate(wraps):                                # group sums that wrap modulo 2^64
        means[3 + k, grp[two[k]]:grp[two[k]] + 2] = pair
    return means, starts, ends, chrom, grp


def first_differences(means, got, want, n=12):
    """got / want: S x (rows or groups); one line per distinct mean (per cell when means is None)"""
    bad = np.argwhere(got != want)
    seen, rows = set(), []
    for s, r in bad:
        key = "mean %r" % float(means[s, r]) if means is not None else "sample %d group %d" % (s, r)
        if key in seen:
            continue
        seen.add(key)
        rows.append("%s: got %d want %d" % (key, got[s, r], want[s, r]))
        if len(rows) == n:
            break
    return "%d cells differ; %s" % (bad.shape[0], "; ".join(rows))


@pytest.mark.gpu
def test_float64_device_and_host_entries_at_go_edges(ctx):
    means, starts, ends, chrom, grp = float64_edge_problem()
    S, R = means.shape
    cells = go_int(means)
    sums = go_sums(cells, grp)
    assert (sums == I64_MIN).any() and (sums == 0).any()
    d_means = ctx.dev_array(means)
    # device entry, simple rows: one cell per conversion
    d_out = ctx.dev_empty(R * S * 8)
    ctx.depthwed_aggregate_device(d_means, S, R, None, R, d_out)
    got = d_out.download(np.int64, R * S).reshape(R, S).T
    assert np.array_equal(got, cells), first_differences(means, got, cells)
    # device entry, the group table
    d_grp = ctx.dev_array(grp)
    n_out = grp.size - 1
    ctx.depthwed_aggregate_device(d_means, S, R, d_grp, n_out, d_out)
    got = d_out.download(np.int64, n_out * S).reshape(n_out, S)
    assert np.array_equal(got, sums), first_differences(None, got.T, sums.T)
    # host entry: the groups it forms and their sums
    o_s, o_e, o_c, out = ctx.depthwed_aggregate(means, starts, ends, chrom, 1000)
    e_s, e_e, e_c = oracle_groups(starts, ends, chrom, 1000)[1:]
    assert np.array_equal(o_s, e_s) and np.array_equal(o_e, e_e) and np.array_equal(o_c, e_c)
    assert np.array_equal(out, sums), first_differences(None, out.T, sums.T)
    for b in (d_means, d_out, d_grp):
        b.free()


# ---------------------------------------------------------------------------------------------------- 5. the CLI at cohort width
def go_matrix_text(names, chrom_names, starts, ends, chrom, vals, size):
    """what the reference prints: the header and one line per group of int(0.5 + dep) sums; also the sums"""
    grp, o_s, o_e, o_c = oracle_groups(starts, ends, chrom, size)
    sums = go_sums(go_int(vals), grp)
    lines = ["\t".join(["#chrom", "start", "end"] + names)]
    for g in range(grp.size - 1):
        lines.append("%s\t%d\t%d\t" % (chrom_names[o_c[g]], o_s[g], o_e[g]) + "\t".join("%d" % v for v in sums[g]))
    return lines, sums


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["ordinary", "int32_overflow", "nonfinite"])
def test_cli_depthwed_300_samples(tmp_path, case):
    rng = np.random.default_rng({"ordinary": 1, "int32_overflow": 2, "nonfinite": 3}[case])
    S, R = 300, 240
    starts, ends, chrom = layout(rng, R)
    chrom_names = ["chr1", "chr2", "chrX"]
    tokens = np.array([["%.4g" % x for x in row] for row in rng.gamma(8, 4, (S, R))], dtype=object)
    if case == "int32_overflow":
        grp = oracle_groups(starts, ends, chrom, 1000)[0]
        g = np.flatnonzero(np.diff(grp) == 4)[2]
        tokens[123, grp[g]:grp[g + 1]] = "600000000"                 # 4 x 6e8 > INT32_MAX: the int32 attempt gives way
    if case == "nonfinite":
        specials = ["NaN", "+Inf", "-Inf", "1e19"]
        for k in range(40):
            tokens[rng.integers(0, S), rng.integers(0, R)] = specials[k % 4]
        tokens[7, :4] = specials
    vals = np.array([[float(t) for t in row] for row in tokens])
    names = ["smp%03d" % k for k in range(S)]
    files = []
    for k in range(S):
        p = tmp_path / (names[k] + ".depth.bed")
        p.write_text("".join("%s\t%d\t%d\t%s\n" % (chrom_names[c], a, b, t) for c, a, b, t in zip(chrom, starts, ends, tokens[k])))
        files.append(str(p))
    proc = subprocess.run([GOLEFT, "depthwed", "-s", "1000", *files], capture_output=True, text=True)
    assert proc.returncode == 0, proc.stderr
    exp, sums = go_matrix_text(names, chrom_names, starts, ends, chrom, vals, 1000)
    assert (sums.max() > I32_MAX) == (case == "int32_overflow")
    assert (sums == I64_MIN).any() == (case == "nonfinite")
    assert proc.stdout.splitlines() == exp


# ---------------------------------------------------------------------------------------------------- 6. gl_bincount_i32
def bincount_ranges():
    out = []
    for w in (8191, 8192, 8193):                                    # shared-memory histogram up to 8192 bins, global above
        out += [(I32_MIN, I32_MIN + w), (I32_MAX - w, I32_MAX), (-w // 2, w - w // 2)]
    return out


def bincount_values(rng, lo, hi, n):
    special = [lo, hi - 1, hi, I32_MIN, I32_MAX, lo + 1, hi - 2]
    special += [lo - 1] if lo > I32_MIN else []
    special += [hi + 1] if hi < I32_MAX else []
    inside = rng.integers(lo, hi, n).astype(np.int64)
    outside = rng.integers(I32_MIN, I32_MAX, n, endpoint=True).astype(np.int64)
    v = np.where(rng.random(n) < 0.7, inside, outside)
    v[:min(n, len(special))] = special[:n]
    return rng.permutation(v).astype(np.int32)


@pytest.mark.gpu
def test_bincount_edges(ctx):
    rng = np.random.default_rng(66)
    for lo, hi in bincount_ranges():
        for n in (1, 255, 256, 257):
            v = bincount_values(rng, lo, hi, n)
            assert np.array_equal(ctx.bincount(v, lo, hi), orc.bincount(v, lo, hi)), (lo, hi, n)
        for x in (lo, hi - 1, hi, I32_MIN, I32_MAX):
            v = np.array([x], np.int32)
            assert np.array_equal(ctx.bincount(v, lo, hi), orc.bincount(v, lo, hi)), (lo, hi, x)
        # the grid-stride loop wraps many times; one bin takes 10^7 counts
        v = np.concatenate([np.full(10 ** 7, hi - 1, np.int32), bincount_values(rng, lo, hi, 300_001)])
        v = rng.permutation(v)
        h = ctx.bincount(v, lo, hi)
        assert h[-1] >= 10 ** 7 and np.array_equal(h, orc.bincount(v, lo, hi)), (lo, hi)


@pytest.mark.gpu
def test_bincount_width_above_int32(ctx):
    """hi - lo = 2^31 + 1 bins (16 GB of counters): the width and x - lo do not fit int32.  The oracle computes both in
    int32 too, so the expectation is numpy's exact count of each in-range value"""
    lo, hi = I32_MIN, 1
    rng = np.random.default_rng(77)
    v = np.concatenate([np.array([lo, lo, -1, 0, 0, 0, 1, 2, I32_MAX, 12345, -12345], np.int64),
                        rng.integers(I32_MIN, I32_MAX, 100_000, endpoint=True)]).astype(np.int32)
    h = ctx.bincount(v, lo, hi)
    assert h.size == 2 ** 31 + 1
    inr = v[v < hi].astype(np.int64) - lo
    keys, counts = np.unique(inr, return_counts=True)
    assert np.array_equal(h[keys], counts.astype(np.uint64))
    assert int(h.sum()) == inr.size                                 # and nothing anywhere else
    assert h[0] >= 2 and h[2 ** 31] >= 3 and h[2 ** 31 - 1] >= 1      # lo, 0 (the last bin) and -1 were counted
