"""`goleft cnveval` on the GPU (gl_cnveval, gl_cnveval_device): stats equal the C oracle's literal walk exactly."""
import math

import numpy as np
import pytest

from cnveval_sets import HAND, cohort, flat, random_set
from goleft_b200 import capi
from oracle import cnveval as oc

pytestmark = pytest.mark.gpu


def _check(ctx, S, arrays, po):
    want = oc.evaluate_arrays(S, *arrays, po)
    got = ctx.cnveval(S, *arrays, po=po)
    assert np.array_equal(got, want)
    return got


def test_random_sets(ctx):
    rng = np.random.default_rng(1301)
    for _ in range(400):
        S, calls, truths, po = random_set(rng)
        _check(ctx, S, flat(calls, truths), po)


@pytest.mark.parametrize("case", HAND, ids=[h[0] for h in HAND])
def test_hand_case(ctx, case):
    _, S, calls, truths, po, want = case
    assert np.array_equal(ctx.cnveval(S, *flat(calls, truths), po=po), want)


@pytest.mark.parametrize("T", [0, 1, 100, 5000])
@pytest.mark.parametrize("S", [1, 3, 33, 257, 2504])
def test_cohort(ctx, S, T):
    rng = np.random.default_rng(S * 7919 + T)
    arrays = cohort(rng, S, T)
    got = _check(ctx, S, arrays, 0.4)
    if T >= 100 and S >= 33:
        assert got[..., oc.TP].sum() > 0 and got[..., oc.FP].sum() > 0 and got[..., oc.TN].sum() > 0


@pytest.mark.parametrize("po", [1e-9, 0.4, 1.0])
def test_structured(ctx, po):
    """nested calls, more than 12 equal starts in one sample, a truth spanning hundreds of calls and a call spanning many
    truths, every CN class, duplicate members, samples with truths but no calls and with calls but no truths"""
    calls, truths = [], []
    for i in range(40):                                          # sample 0: 40 calls at one start, nested ends
        calls.append((0, 1, 10_000, 10_000 + 500 * (40 - i) + (i % 7), [0, 1, 2, 3, 4, 7, -1][i % 7]))
    for i in range(300):                                         # sample 1: 300 small calls under one big truth
        calls.append((1, 0, 1000 * i, 1000 * i + 400 + i % 3 * 300, 1 + (i % 2) * 2))
    truths.append((0, 0, 300_000, 1, [1, 2]))
    truths.append((0, 0, 300_000, 3, [3]))
    calls.append((2, 0, 0, 2_000_000, 1))                        # sample 2: one call over 200 truths
    for i in range(200):
        truths.append((0, 10_000 * i, 10_000 * i + 3000 + (i % 5) * 4000, [1, 3, 0, 2][i % 4], [2, 2] if i % 9 == 0 else [i % 6]))
    for i in range(30):
        truths.append((1, 10_000, 10_000 + 500 * (i + 1), [0, 1, 2, 3, 4, 7, -1][i % 7], [0] if i % 3 else [4, 0]))
    calls += [(5, 2, 100, 200, 1), (5, 2, 100, 150, 1)]          # sample 5: calls but no truths; sample 4: truths, no calls
    S = 6
    rng = np.random.default_rng(5)
    calls = [calls[i] for i in rng.permutation(len(calls))]
    _check(ctx, S, flat(calls, truths), po)


def test_global_memory_path(ctx):
    """a sample with more calls than one CTA stages in shared memory"""
    rng = np.random.default_rng(1302)
    calls = [(0, int(rng.integers(0, 2)), int(s), int(s) + int(rng.integers(0, 5000)), int(rng.choice([1, 3])))
             for s in rng.integers(0, 2000, 3000) * 100]
    calls += [(1, 0, 100, 9000, 1), (2, 1, 50_000, 60_000, 3)]
    truths = [(int(rng.integers(0, 2)), int(s), int(s) + int(rng.integers(100, 20000)), int(rng.choice([1, 3])),
               [int(x) for x in rng.integers(0, 3, int(rng.integers(0, 3)))]) for s in rng.integers(0, 2000, 2500) * 100]
    _check(ctx, 3, flat(calls, truths), 0.4)


def _layout(S, cs, cc, cb, ce, ccn, tc, tb, te, tcn, mp, ms):
    """the resident layout gl_cnveval_device takes"""
    order, c_ptr = [], [0]
    for s in range(S):
        idx = np.nonzero(cs == s)[0]
        order += idx[capi.cnveval_order(cc[idx], cb[idx])].tolist()
        c_ptr.append(len(order))
    order = np.asarray(order, np.int64)
    to = np.lexsort((tb, tc))
    rank = np.empty(tc.size, np.int64)
    rank[to] = np.arange(tc.size)
    owner = np.repeat(np.arange(tc.size), np.diff(mp))
    mem = sorted(zip(ms.tolist(), rank[owner].tolist()))
    m_ptr = np.searchsorted(np.asarray([m[0] for m in mem], np.int64), np.arange(S + 1))
    return (np.asarray(c_ptr, np.int64), cc[order], cb[order], ce[order], ccn[order], tc[to], tb[to], te[to], tcn[to],
            m_ptr.astype(np.int64), np.asarray([m[1] for m in mem], np.int64))


def test_device_entry_equals_host_entry(ctx):
    rng = np.random.default_rng(1303)
    S, T = 257, 5000
    arrays = cohort(rng, S, T)
    want = ctx.cnveval(S, *arrays, po=0.4)
    c_ptr, cc, cb, ce, ccn, tc, tb, te, tcn, m_ptr, m_truth = _layout(S, *arrays)
    d = [ctx.dev_array(a) for a in (c_ptr, cc, cb, ce, ccn, tc, tb, te, tcn, m_ptr, m_truth)]
    st = ctx.dev_empty(S * 12 * 8)
    ctx.cnveval_device(S, d[0], cc.size, d[1], d[2], d[3], d[4], T, d[5], d[6], d[7], d[8], d[9], m_truth.size, d[10], 0.4, st)
    assert np.array_equal(st.download(np.uint64, S * 12).reshape(S, 3, 4), want)
    i = int(np.nonzero((tc[1:] == tc[:-1]) & (tb[1:] > tb[:-1]))[0][0])
    bad = tb.copy()
    bad[[i, i + 1]] = bad[[i + 1, i]]                            # truths out of (chrom, start) order
    d[6].upload(bad)
    with pytest.raises(capi.GlError) as e:
        ctx.cnveval_device(S, d[0], cc.size, d[1], d[2], d[3], d[4], T, d[5], d[6], d[7], d[8], d[9], m_truth.size, d[10], 0.4, st)
    assert e.value.code == capi.GL_EINVAL
    for b in d + [st]:
        b.free()


def test_einval_policy(ctx):
    ok_calls, ok_truths = [(0, 0, 100, 200, 1)], [(0, 100, 200, 1, [0])]
    assert ctx.cnveval(1, *flat(ok_calls, ok_truths), po=0.4)[0, 0, oc.TP] == 1
    bad = [
        ([(0, 0, 200, 100, 1)], ok_truths, 0.4),                 # call end < start
        (ok_calls, [(0, 200, 100, 1, [0])], 0.4),                # truth end < start
        ([(0, 0, -1, 100, 1)], ok_truths, 0.4),                  # negative coordinate
        (ok_calls, [(0, 0, 1 << 62, 1, [0])], 0.4),              # outside [0, 2^62)
        ([(1, 0, 100, 200, 1)], ok_truths, 0.4),                 # sample out of range
        (ok_calls, [(0, 100, 200, 1, [3])], 0.4),
        ([(0, -1, 100, 200, 1)], ok_truths, 0.4),                # negative chrom rank
        (ok_calls, ok_truths, 0.0), (ok_calls, ok_truths, 1.5), (ok_calls, ok_truths, -0.4), (ok_calls, ok_truths, math.inf),
    ]
    for calls, truths, po in bad:
        with pytest.raises(capi.GlError) as e:
            ctx.cnveval(1, *flat(calls, truths), po=po)
        assert e.value.code == capi.GL_EINVAL, (calls, truths, po)
    assert ctx.cnveval(1, *flat(ok_calls, ok_truths), po=0.4)[0, 0, oc.TP] == 1
    assert ctx.cnveval(0, *flat([], []), po=0.4).shape == (0, 3, 4)
