"""The packed8 reduce as one chain of kernels: K_tileidx8 -> K_fused8 -> K_gather, and on into the next reduce, with no
memset, copy or event between them.  The first K_tileidx8 of a reduce zeroes the scratch, a rejection is a per-reduce tag
in header[3], and K_gather stores the header into the mapped host slot.  One context reduces regions back to back; every
result is compared with a fresh context and with oracle/oracle_depth.c.  Integer work -> bit-exact.  Needs an H100."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

from goleft_b200 import capi, synth
from oracle import loader as orc

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _expect(s, e, rs, re, W, mincov=4, run_break=0):
    depth = orc.pileup_diff(s, e, rs, re)
    es, _ = orc.window_sums(depth, rs, re, W)
    ea, ec = orc.class_runs(depth, rs, re, mincov, 0, run_break)
    return (es.size, ea.size, int(depth.max(initial=0))), es, ea, ec


def _results(c):
    sizes = c.depth_result_sizes()
    r0, rc = c.depth_get_runs()
    return sizes, c.depth_get_windows().copy(), r0.copy(), rc.copy()


def _same(got, exp):
    return got[0] == exp[0] and all(np.array_equal(x, y) for x, y in zip(got[1:], exp[1:]))


class _Region:
    def __init__(self, c, L, idx, coverage=30.0, shuffle=None):
        self.L = L
        self.s, self.e = synth.segments(synth.reads(L, coverage=coverage, contig_index=idx))
        a, d, ln = capi.pack_segments8(self.s, self.e)
        if shuffle is not None:                                 # blocks in a random order: unsorted anchors
            perm = np.random.default_rng(shuffle).permutation(a.size)
            a = np.ascontiguousarray(a[perm])
            d = np.ascontiguousarray(d.reshape(-1, 64)[perm]).reshape(-1)
            ln = np.ascontiguousarray(ln.reshape(-1, 64)[perm]).reshape(-1)
        self.nb = a.size
        self.bufs = [c.dev_array(x) for x in (a, d, ln)]

    def reduce(self, c, rs=0, re=None, W=500, mincov=4, run_break=0):
        c.depth_begin(rs, self.L if re is None else re)
        c.depth_add_segments_packed8_device(*self.bufs, self.nb)
        c.depth_reduce(W, mincov, 0, run_break)

    def expect(self, rs=0, re=None, W=500, mincov=4, run_break=0):
        return _expect(self.s, self.e, rs, self.L if re is None else re, W, mincov, run_break)

    def free(self):
        for b in self.bufs:
            b.free()


# (region, rs, re, W, mincov, run_break): long -> short -> long, a one-tile region among them
def _sequence(regions):
    big, small, tiny = regions
    return [(big, 0, None, 500, 4, 10_000_000), (small, 0, None, 500, 4, 0), (tiny, 0, None, 100, 2, 0),
            (big, 12_345, 1_900_000, 333, 4, 0), (small, 0, 4096, 64, 3, 0), (big, 0, None, 500, 4, 10_000_000)]


@pytest.fixture(scope="module")
def regions(ctx):
    rs = [_Region(ctx, 2_000_000, 41), _Region(ctx, 150_000, 42), _Region(ctx, 4000, 43)]
    yield rs
    for r in rs:
        r.free()


@pytest.mark.parametrize("query_each", [False, True])
def test_long_short_long(ctx, regions, query_each):
    """back-to-back reduces of different lengths on one context, queried after each or only after the last"""
    seq = _sequence(regions)
    for i, (r, rs, re, W, mc, brk) in enumerate(seq):
        r.reduce(ctx, rs, re, W, mc, brk)
        if query_each or i == len(seq) - 1:
            assert ctx.depth_last_path() == 3
            exp = r.expect(rs, re, W, mc, brk)
            assert _same(_results(ctx), exp), i


def test_against_fresh_context(ctx, regions):
    """the last reduce of a long sequence gives what a fresh context gives for that region alone"""
    for r, rs, re, W, mc, brk in _sequence(regions):
        r.reduce(ctx, rs, re, W, mc, brk)
    got = _results(ctx)
    big = regions[0]
    with capi.Ctx(0) as c:
        bufs = [c.dev_array(x) for x in capi.pack_segments8(big.s, big.e)]
        c.depth_begin(0, big.L)
        c.depth_add_segments_packed8_device(*bufs, big.nb)
        c.depth_reduce(500, 4, 0, 10_000_000)
        fresh = _results(c)
        for b in bufs:
            b.free()
    assert _same(got, fresh)


def test_unsorted_sorted_unsorted(ctx, regions):
    """a rejected packed8 reduce leaves its tag in header[3]; the sorted reduce after it must not read it as its own"""
    bad = _Region(ctx, 300_000, 44, shuffle=3)
    good = regions[1]
    for query_each in (True, False):
        for k, r in enumerate((bad, good, bad, good)):
            r.reduce(ctx)
            if query_each or k == 3:
                assert ctx.depth_last_path() in ((3,) if r is good else (1, 4)), k
                assert _same(_results(ctx), r.expect()), k
    bad.free()


def test_rejected_fused_then_packed8(ctx, regions):
    """a fused int32 reduce rejected by the device (header[3] = 1), then a packed8 reduce: it stays on path 3"""
    L = 200_000
    s, e = synth.segments(synth.reads(L, contig_index=45))
    perm = np.random.default_rng(4).permutation(s.size)
    d_s, d_e = ctx.dev_array(s[perm]), ctx.dev_array(e[perm])
    ctx.depth_begin(0, L)
    ctx.depth_add_segments_device(d_s, d_e, s.size)
    ctx.depth_reduce(500, 4, 0, 0)
    assert ctx.depth_last_path() == 4                           # the fused pass was rejected and rerun
    r = regions[1]
    r.reduce(ctx)
    assert ctx.depth_last_path() == 3
    assert _same(_results(ctx), r.expect())
    d_s.free(); d_e.free()


def test_windows_only_header_comes_home(ctx, regions):
    """a reduce without runs (do_runs = 0) still sends its header: max depth and zero runs, after a deeper region"""
    deep = _Region(ctx, 60_000, 46, coverage=90.0)
    shallow = regions[1]
    for first in (deep, shallow, deep):
        first.reduce(ctx)
        L = shallow.L
        W = 250
        ctx.depth_begin(0, L)
        ctx.depth_add_segments_packed8_device(*shallow.bufs, shallow.nb)
        ws, wm = ctx.depth_windows(W, (L - 1) // W + 1)
        assert ctx.depth_last_path() == 3
        depth = orc.pileup_diff(shallow.s, shallow.e, 0, L)
        es, em = orc.window_sums(depth, 0, L, W)
        assert np.array_equal(ws, es) and np.array_equal(wm, em)
        assert ctx.depth_result_sizes() == (es.size, 0, int(depth.max()))
    deep.free()


def test_run_overflow_mid_sequence():
    """a fresh context's run table is sized by its first region; a later region with far more runs overflows it and reruns,
    between reduces that fit"""
    L = 300_000
    s = np.arange(0, L, 2, dtype=np.int32)
    e = s + 1
    depth = orc.pileup_diff(s, e, 0, L)
    ea, ec = orc.class_runs(depth, 0, L, 1, 0, 0)
    with capi.Ctx(0) as c:
        small = _Region(c, 20_000, 47)
        a, d, ln = capi.pack_segments8(s, e)
        many = [c.dev_array(x) for x in (a, d, ln)]
        for query_each in (True, False):
            small.reduce(c)
            if query_each:
                assert _same(_results(c), small.expect())
            c.depth_begin(0, L)
            c.depth_add_segments_packed8_device(*many, a.size)
            c.depth_reduce(1000, 1, 0, 0)
            if query_each:
                assert c.depth_result_sizes()[1] == ea.size and c.depth_last_path() == 3
                r0, rc = c.depth_get_runs()
                assert np.array_equal(r0, ea) and np.array_equal(rc, ec)
            small.reduce(c)
            assert c.depth_last_path() == 3
            assert _same(_results(c), small.expect())
        small.free()
        for b in many:
            b.free()


def test_profiling_gives_the_same_outputs(ctx, regions):
    """profile mode puts events between the kernels; the outputs do not change"""
    outs = []
    for on in (False, True, False):
        ctx.profile_enable(on)
        got = []
        for r, rs, re, W, mc, brk in _sequence(regions):
            r.reduce(ctx, rs, re, W, mc, brk)
            got.append(_results(ctx))
        ctx.profile_enable(False)
        names = {nm for nm, _ in ctx.profile_read()}
        if on:
            assert {"depth_tileidx8_kernel", "depth_fused8_kernel", "depth_gather_runs_kernel"} <= names
        outs.append(got)
    for a, b in zip(outs[0], outs[1]):
        assert _same(a, b)
    for a, b in zip(outs[0], outs[2]):
        assert _same(a, b)


_STREAMED = textwrap.dedent("""
    import sys
    import numpy as np
    sys.path.insert(0, sys.argv[1])
    from goleft_b200 import capi, synth
    from oracle import loader as orc
    L, W = 3_000_000, 500
    s, e = synth.segments(synth.reads(L, contig_index=48))
    packed = capi.pack_segments8(s, e)
    assert packed[0].size >= 4096                               # a one-call entry streams only from 4096 blocks on
    with capi.Ctx(0) as c:
        host = []
        for x in packed:
            h = c.pinned_empty(x.size, x.dtype)
            h[:] = x
            host.append(h)
        dev = [c.dev_array(x) for x in packed]
        small_s, small_e = synth.segments(synth.reads(100_000, contig_index=49))
        small_p = capi.pack_segments8(small_s, small_e)
        small = [c.dev_array(x) for x in small_p]
        for rs, re, brk in [(0, L, 1_000_000), (1_234_567, L - 5, 0)]:
            depth = orc.pileup_diff(s, e, rs, re)
            es, _ = orc.window_sums(depth, rs, re, W)
            ea, ec = orc.class_runs(depth, rs, re, 4, 0, brk)
            c.depth_begin(0, 100_000)                            # a resident reduce queued in front, not queried
            c.depth_add_segments_packed8_device(*small, small_p[0].size)
            c.depth_reduce(W, 4, 0, 0)
            ws, r0, rc = c.depth_region_packed8(rs, re, *host, W, 4, 0, run_break=brk)
            assert c.depth_last_path() == 3
            assert np.array_equal(ws, es) and np.array_equal(r0, ea) and np.array_equal(rc, ec), (rs, re)
            c.depth_begin(rs, re)                                # the same words resident, after the streamed reduce
            c.depth_add_segments_packed8_device(*dev, packed[0].size)
            c.depth_reduce(W, 4, 0, brk)
            r0, rc = c.depth_get_runs()
            assert np.array_equal(c.depth_get_windows(), es) and np.array_equal(r0, ea) and np.array_equal(rc, ec)
    print("ok")
""")


@pytest.mark.parametrize("chunks", [1, 3, 4])
def test_streamed_region(chunks):
    """pinned host words through gl_depth_region_packed8: K_tileidx8 runs once per upload chunk and only the first zeroes
    (GL_P8_CHUNKS is read once per process, so each count runs in its own)"""
    env = dict(os.environ, GL_P8_CHUNKS=str(chunks))
    r = subprocess.run([sys.executable, "-c", _STREAMED, ROOT], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stdout + r.stderr
