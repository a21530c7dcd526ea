"""gl_depth_reduce only queues its work: its header is read, and a rejected fast path or an overflowing run table settled,
at the first result query.  These drive that through the sequence API (begin / add / reduce / queries) against
oracle/oracle_depth.c.  Integer work -> bit-exact.  Every test here needs an H100 (`-m gpu`)."""
import numpy as np
import pytest

from goleft_b200 import capi, synth
from oracle import loader as orc

pytestmark = pytest.mark.gpu


def _shuffled_blocks(a, d, ln, seed):
    """packed8 blocks in a random order: the anchors are no longer sorted, which the packed8 kernel rejects"""
    nb = a.size
    perm = np.random.default_rng(seed).permutation(nb)
    return (np.ascontiguousarray(a[perm]), np.ascontiguousarray(d.reshape(nb, 64)[perm]).reshape(-1),
            np.ascontiguousarray(ln.reshape(nb, 64)[perm]).reshape(-1))


def _check_results(ctx, s, e, rs, re, W, mincov=4, run_break=0):
    depth = orc.pileup_diff(s, e, rs, re)
    es, _ = orc.window_sums(depth, rs, re, W)
    ea, ec = orc.class_runs(depth, rs, re, mincov, 0, run_break)
    nw, nr, md = ctx.depth_result_sizes()
    assert (nw, nr, md) == (es.size, ea.size, int(depth.max(initial=0)))
    assert np.array_equal(ctx.depth_get_windows(), es)
    r0, rc = ctx.depth_get_runs()
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)


def test_back_to_back_regions_only_last_queried(ctx):
    """several regions reduced one after another with no query in between (packed8 device words, some of them rejected
    if anyone asked, int32 host arrays, shuffled int32 device arrays); only the last is queried.  A result dropped by
    gl_depth_begin is gone: nothing of it shows in the next region."""
    L = 1_500_000
    s1, e1 = synth.segments(synth.reads(L, contig_index=12))
    s2, e2 = synth.segments(synth.reads(L - 4321, contig_index=13))
    a1, d1, l1 = capi.pack_segments8(s1, e1)
    p8 = [ctx.dev_array(x) for x in (a1, d1, l1)]
    a2, d2, l2 = _shuffled_blocks(*capi.pack_segments8(s2, e2), seed=1)
    p8_shuffled = [ctx.dev_array(x) for x in (a2, d2, l2)]
    perm = np.random.default_rng(2).permutation(s2.size)
    i32 = [ctx.dev_array(s2[perm]), ctx.dev_array(e2[perm])]
    for last in ("packed8", "packed8_shuffled", "int32"):
        ctx.depth_begin(0, L)
        ctx.depth_add_segments_packed8_device(p8[0], p8[1], p8[2], a1.size)
        ctx.depth_reduce(500, 4, 0, 10_000_000)
        ctx.depth_reduce(250, 3, 0, 0)                             # the same region again: the first result is dropped
        ctx.depth_begin(1000, L - 4321)
        ctx.depth_add_segments_packed8_device(p8_shuffled[0], p8_shuffled[1], p8_shuffled[2], a2.size)
        ctx.depth_reduce(500, 4, 0, 0)
        ctx.depth_begin(0, L)
        ctx.depth_add_segments(s1, e1)                             # host arrays: copied into the ctx store
        ctx.depth_reduce(500, 4, 0, 0)
        ctx.depth_begin(0, L - 4321)
        ctx.depth_add_segments(s2[perm], e2[perm])                 # the store again, while the reduce above may still run
        ctx.depth_reduce(333, 4, 0, 0)
        ctx.depth_begin(0, L - 4321)
        ctx.depth_add_segments_device(i32[0], i32[1], s2.size)
        ctx.depth_reduce(333, 4, 0, 0)
        if last == "packed8":
            ctx.depth_begin(0, L)
            ctx.depth_add_segments_packed8_device(p8[0], p8[1], p8[2], a1.size)
            ctx.depth_reduce(500, 4, 0, 1_000_000)
            assert ctx.depth_last_path() == 3
            _check_results(ctx, s1, e1, 0, L, 500, run_break=1_000_000)
        elif last == "packed8_shuffled":
            ctx.depth_begin(1000, L - 4321)
            ctx.depth_add_segments_packed8_device(p8_shuffled[0], p8_shuffled[1], p8_shuffled[2], a2.size)
            ctx.depth_reduce(500, 4, 0, 0)
            assert ctx.depth_last_path() in (1, 4)
            _check_results(ctx, s2, e2, 1000, L - 4321, 500)
        else:
            assert ctx.depth_last_path() == 4
            _check_results(ctx, s2, e2, 0, L - 4321, 333)
    # a pending result dropped by gl_depth_begin: the new region has no results until it is reduced
    ctx.depth_begin(0, L)
    ctx.depth_add_segments_packed8_device(p8[0], p8[1], p8[2], a1.size)
    ctx.depth_reduce(500, 4, 0, 0)
    ctx.depth_begin(5000, 900_000)
    with pytest.raises(capi.GlError) as ei:
        ctx.depth_result_sizes()
    assert ei.value.code == capi.GL_ESTATE
    ctx.depth_add_segments_packed8_device(p8[0], p8[1], p8[2], a1.size)
    ctx.depth_reduce(100, 4, 0, 0)
    _check_results(ctx, s1, e1, 5000, 900_000, 100)
    for b in p8 + p8_shuffled + i32:
        b.free()


def test_unsorted_packed8_sequence_api(ctx):
    """unsorted packed8 anchors through begin / add_packed8_device / reduce / get_*: the rejection and the fallback happen
    at the first query, which gives the oracle's integers"""
    L = 400_000
    s, e = synth.segments(synth.reads(L, contig_index=2))
    a2, d2, l2 = _shuffled_blocks(*capi.pack_segments8(s, e), seed=0)
    bufs = [ctx.dev_array(x) for x in (a2, d2, l2)]
    ctx.depth_begin(0, L)
    ctx.depth_add_segments_packed8_device(bufs[0], bufs[1], bufs[2], a2.size)
    ctx.depth_reduce(500, 4, 0, 0)
    assert ctx.depth_last_path() in (1, 4)
    _check_results(ctx, s, e, 0, L, 500)
    for b in bufs:
        b.free()


@pytest.mark.parametrize("packed8", [False, True])
def test_run_overflow_sequence_api(packed8):
    """alternating covered/uncovered bases on a fresh ctx: far more runs than the first run table holds.  The table grows
    and the reduce reruns at the first query; queried as result_sizes, get_runs, then the device text."""
    L, W = 300_000, 1000
    s = np.arange(0, L, 2, dtype=np.int32)
    e = s + 1
    depth = orc.pileup_diff(s, e, 0, L)
    ea, ec = orc.class_runs(depth, 0, L, 1, 0, 0)
    with capi.Ctx(0) as c:
        bufs = []
        c.depth_begin(0, L)
        if packed8:
            a, d, ln = capi.pack_segments8(s, e)
            bufs = [c.dev_array(x) for x in (a, d, ln)]
            c.depth_add_segments_packed8_device(bufs[0], bufs[1], bufs[2], a.size)
        else:
            bufs = [c.dev_array(s), c.dev_array(e)]
            c.depth_add_segments_device(bufs[0], bufs[1], s.size)
        c.depth_reduce(W, 1, 0, 0)
        nw, nr, md = c.depth_result_sizes()
        assert (nw, nr, md) == ((L - 1) // W + 1, ea.size, 1)
        assert c.depth_last_path() == (3 if packed8 else 1)
        r0, rc = c.depth_get_runs()
        assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
        assert c.depth_text("chrT") == orc.walk_chunk("chrT", 0, L, W, 1, 0, depth)
        for b in bufs:
            b.free()


def test_shuffled_int32_first_query_interval_sums_or_classes(ctx):
    """int32 segments in random order (the fused pass is rejected): the first query after the reduce is
    gl_depth_interval_sums, or gl_depth_classes, and both give the oracle's integers"""
    L = 600_000
    s, e = synth.segments(synth.reads(L, contig_index=5))
    perm = np.random.default_rng(3).permutation(s.size)
    s, e = s[perm], e[perm]
    depth = orc.pileup_diff(s, e, 0, L)
    cs = np.concatenate([[0], np.cumsum(depth.astype(np.int64))])
    rng = np.random.default_rng(4)
    a = rng.integers(0, L, 300).astype(np.int32)
    b = np.minimum(a + rng.choice([1, 99, 4097, 70000], a.size), L).astype(np.int32)
    ctx.depth_begin(0, L)
    ctx.depth_add_segments(s, e)
    ctx.depth_reduce(500, 4, 0, 0)
    assert np.array_equal(ctx.depth_interval_sums(a, b), cs[b] - cs[a])
    assert ctx.depth_last_path() == 4
    assert np.array_equal(ctx.depth_get_windows(), orc.window_sums(depth, 0, L, 500)[0])
    ea, ec = orc.class_runs(depth, 0, L, 4, 0, 0)
    ctx.depth_begin(0, L)
    ctx.depth_add_segments(s, e)
    ctx.depth_reduce(500, 4, 0, 0)
    r0, r1, rc = ctx.depth_classes(4, 0, L)
    assert ctx.depth_last_path() == 4
    assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
    assert np.array_equal(r1, np.append(ea[1:], L).astype(np.int32))
