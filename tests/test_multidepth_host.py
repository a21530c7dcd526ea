"""CPU tests of `goleft multidepth`'s host side: the chunk state machine (gl_multidepth_blocks) against the literal
site-by-site oracle on hand cases for every quirk of multidepth.go and on random site-class patterns, and the
certification of a mean's "%.2f" digits (gl_multidepth_certify) against the reference's float64 chain."""
import numpy as np
import pytest

from goleft_b200 import capi
from oracle import multidepth as omd

ABSENT, INSUF, SUF = 0, 1, 2


def runs_of(cls):
    cls = np.asarray(cls, np.uint8)
    if cls.size == 0:
        return np.zeros(0, np.int32), np.zeros(0, np.uint8)
    st = np.flatnonzero(np.concatenate([[True], cls[1:] != cls[:-1]])).astype(np.int32)
    return st, cls[st]


def lib_blocks(cls, chunk, n_samples=1, **kw):
    rs, rc = runs_of(cls)
    s, e, n = capi.multidepth_blocks(rs, rc, len(cls), n_samples, chunk=chunk, **kw)
    return [tuple(x) for x in np.stack([s, e, n], 1).tolist()]


def both(cls, chunk, expect, **kw):
    """gl_multidepth_blocks and the oracle agree with each other and with the hand-derived blocks"""
    cls = np.asarray(cls, np.uint8)
    o = [tuple(r) for r in omd.blocks(cls, chunk, **kw).tolist()]
    got = lib_blocks(cls, chunk, **kw)
    assert o == expect, ("oracle", o)
    assert got == expect, ("library", got)


def test_seen0_in_chunk_0():
    """sufficient sites before the first insufficient one are never cached, in chunk 0 too"""
    cls = [SUF] * 20 + [INSUF] + [SUF] * 20
    both(cls, 1000, [(21, 41, 20)], max_skip=10, min_size=1)


def _kill_case(gap):
    # chunk 0 (C = 10, kill sites lie beyond 11): an insufficient site at 0, sufficient 1..13, an insufficient site at
    # 13 + gap, two sufficient sites after it
    cls = [INSUF] + [SUF] * 13 + [ABSENT] * (gap - 1) + [INSUF, SUF, SUF]
    return cls


def test_kill_at_max_skip():
    """pos0 - last == MaxSkip kills (>=): the cache (13 sites < MinSize) is flushed as it is"""
    cls = _kill_case(3)              # insufficient at 16, last = 13
    both(cls, 10, [(1, 14, 13), (17, 19, 2)], max_skip=3, min_size=15)


def test_kill_at_max_skip_plus_one():
    cls = _kill_case(4)              # insufficient at 17
    both(cls, 10, [(1, 14, 13), (18, 20, 2)], max_skip=3, min_size=15)


def test_no_kill_below_max_skip_and_overlap_duplicates():
    """pos0 - last == MaxSkip - 1 does not kill; the chain goes on past the chunk, and chunk 1 reports the tail again"""
    cls = _kill_case(2)              # insufficient at 15
    both(cls, 10, [(1, 18, 15), (16, 18, 2)], max_skip=3, min_size=15)


def test_min_size_only_on_a_broken_chain():
    """a chain broken by a gap is kept only with >= MinSize sites; the one left at the contig end is kept regardless"""
    cls = [INSUF] + [SUF] * 3 + [ABSENT] * 12 + [SUF] * 3
    both(cls, 1000, [(16, 19, 3)], max_skip=10, min_size=4)
    both(cls, 1000, [(1, 4, 3), (16, 19, 3)], max_skip=10, min_size=3)


def test_duplicate_block_in_chunk_overlap():
    """chunk 0 runs past its end until its kill; chunk 1 starts at its own first insufficient site: the same block twice"""
    cls = [ABSENT] * 40
    cls[0] = INSUF
    cls[11] = INSUF
    cls[12:15] = [SUF] * 3
    cls[30] = INSUF
    both(cls, 10, [(12, 15, 3), (12, 15, 3)], max_skip=10, min_size=1)


def test_window_split():
    both([INSUF] + [SUF] * 10, 1000, [(1, 5, 4), (5, 9, 4), (9, 11, 2)], max_skip=10, min_size=1, window=4)
    both([INSUF, SUF, ABSENT, ABSENT, ABSENT, SUF, SUF], 1000, [(1, 2, 1), (5, 7, 2)], max_skip=10, min_size=1, window=3)
    # Window 1 (and below): every site is its own block
    both([INSUF, SUF, SUF, ABSENT, SUF], 1000, [(1, 2, 1), (2, 3, 1), (4, 5, 1)], max_skip=10, min_size=1, window=1)


def test_min_samples_rounding_and_strict_greater():
    """minSamples = int(0.5 + f*S); a site is sufficient only when MORE than minSamples samples reach MinCov"""
    assert omd.min_samples(0.5, 3) == 2 and omd.min_samples(0.5, 4) == 2 and omd.min_samples(0.5, 5) == 3
    assert omd.min_samples(0.0, 7) == 0 and omd.min_samples(1.0, 7) == 7 and omd.min_samples(0.25, 2) == 1
    d = np.zeros((4, 6), np.int32)
    d[:, 0] = [1, 0, 0, 0]          # insufficient: starts the cache
    d[:, 1] = [7, 7, 0, 0]          # 2 samples >= 7, minSamples 2: insufficient
    d[:, 2] = [7, 7, 7, 0]          # 3 > 2: sufficient
    d[:, 3] = [7, 7, 6, 1]          # 2: insufficient
    _, cls = omd.text("c", d, mincov=7, min_samples=0.5, min_size=1)
    assert cls.tolist() == [INSUF, INSUF, SUF, INSUF, ABSENT, ABSENT]


def test_chunk_size_fifth_above_50_samples():
    """S > 50: chunks of 1e6 bases instead of 5e6 — here that adds the block chunk 1 sees"""
    L = 3_000_000
    cls = np.zeros(L, np.uint8)
    cls[0] = INSUF
    cls[1:1_500_000] = SUF
    cls[1_500_000] = INSUF
    cls[1_500_001:2_500_000] = SUF
    cls[2_600_000] = INSUF
    assert omd.chunk_size(50) == 5_000_000 and omd.chunk_size(51) == 1_000_000
    for S, exp in ((50, [(1, 2_500_000, 2_499_998)]), (51, [(1, 2_500_000, 2_499_998), (1_500_001, 2_500_000, 999_999)])):
        o = [tuple(r) for r in omd.blocks(cls, omd.chunk_size(S), min_size=15).tolist()]
        assert o == exp
        assert lib_blocks(cls, 0, n_samples=S, min_size=15) == exp


def _random_classes(rng, L):
    out = np.empty(L, np.uint8)
    i = 0
    p = rng.dirichlet([1, 1, 2])
    while i < L:
        k = int(rng.geometric(rng.choice([0.5, 0.1, 0.02])))
        out[i:i + k] = rng.choice(3, p=p)
        i += k
    return out


def test_blocks_random_patterns():
    rng = np.random.default_rng(20261015)
    for it in range(4000):
        L = int(rng.integers(1, 600))
        cls = _random_classes(rng, L)
        chunk = int(rng.integers(1, 200))
        kw = dict(max_skip=int(rng.integers(0, 8)), min_size=int(rng.integers(0, 8)), window=int(rng.integers(0, 60)))
        o = [tuple(r) for r in omd.blocks(cls, chunk, **kw).tolist()]
        assert lib_blocks(cls, chunk, **kw) == o, (it, L, chunk, kw)


def _digits(q):
    return b"%d.%02d" % (q // 100, q % 100)


def _check_cells(d, off, n, l):
    """every certified cell prints the oracle's digits; returns the number certified"""
    sums = np.add.reduceat(d.astype(np.int64), off) if d.size else np.zeros(0, np.int64)
    sums = np.where(n > 0, sums, 0)
    q, ok = capi.multidepth_certify(sums, n, l)
    exp = omd.chain_batch(d, off, n, l)
    bad = [i for i in np.flatnonzero(ok) if _digits(int(q[i])) != exp[i]]
    assert not bad, [(int(i), int(sums[i]), int(n[i]), int(l[i]), exp[i], _digits(int(q[i]))) for i in bad[:5]]
    return int(ok.sum())


def test_certify_random_cells():
    rng = np.random.default_rng(7)
    ncell = 1_000_000
    n = rng.integers(1, 12, ncell)
    l = n + rng.integers(0, 30, ncell)
    d = rng.integers(0, rng.choice([10, 60, 2000], ncell).repeat(n)).astype(np.int32)
    off = np.concatenate([[0], np.cumsum(n)[:-1]])
    k = _check_cells(d, off, n, l)
    assert k > 0.9 * ncell


def test_certify_near_ties():
    """cells whose exact mean is k + 1/2 (must not certify) or within a few 1/l of it (may, when provably safe)"""
    rng = np.random.default_rng(11)
    ncell = 1_000_000
    l = rng.integers(1, 400, ncell)
    k = rng.integers(0, 5000, ncell)
    # Σd ≈ (k + 1/2) l / 100, nudged by -2..2
    target = ((2 * k + 1) * l) // 200 + rng.integers(-2, 3, ncell)
    target = np.maximum(target, 0)
    n = np.minimum(l, rng.integers(1, 40, ncell))
    # spread target over n sites: n-1 random cut points
    d_parts, offs, pos = [], np.empty(ncell, np.int64), 0
    base = target // n
    rem = target - base * n
    d = np.repeat(base, n).astype(np.int64)
    offs = np.concatenate([[0], np.cumsum(n)[:-1]])
    # add the remainder one unit at a time to the first rem sites of each cell
    idx = np.arange(d.size) - np.repeat(offs, n)
    d += (idx < np.repeat(rem, n))
    d = d.astype(np.int32)
    cert = _check_cells(d, offs, n, l)
    exact_tie = (200 * target) == (2 * k + 1) * l
    sums = target
    q, ok = capi.multidepth_certify(sums, n, l)
    assert not ok[(200 * sums) % (2 * l) == l].any(), "an exact tie was certified"
    assert exact_tie.any() and cert > 0


def test_certify_long_cells():
    """n up to 1e7 terms: the error bound grows with n, and certified digits still match the chain"""
    rng = np.random.default_rng(3)
    for n in (10 ** 5, 10 ** 6, 10 ** 7):
        d = rng.integers(0, 60, n).astype(np.int32)
        for l in (n, n + 12345):
            got = _check_cells(d, np.array([0]), np.array([n]), np.array([l]))
            assert got in (0, 1)
        c = np.full(n, 30, np.int32)                       # mean exactly 30: far from every tie
        assert _check_cells(c, np.array([0]), np.array([n]), np.array([n])) == 1
