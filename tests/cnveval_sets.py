"""Inputs for the `cnveval` tests: random tie-heavy call / truth sets, one hand case per quirk of the reference's walk, and
the order-free form of its counts (DESIGN §1.12) restated in Python.

A set is (S, calls, truths, po): calls [(sample, chrom, start, end, cn)] in file order, truths [(chrom, start, end, cn,
[samples])], chromosomes as ranks."""
import math

import numpy as np

from oracle import cnveval as oc

LENS = [0, 1, 7, 10, 50, 100, 300, 1000, 19999, 20000, 25000, 99999, 100000, 150000]
CNS = [-3, -1, 0, 1, 2, 3, 4, 5, 9]
POS = [1e-9, 0.1, 0.4, 0.5, 0.9, 1.0]


def random_set(rng, max_calls=40, max_truths=25):
    """a few starts on a coarse grid (ties are common), nested, zero-length and spanning intervals, duplicate memberships"""
    S = int(rng.integers(1, 6))
    n_chrom = int(rng.integers(1, 3))
    grid = rng.integers(0, 5000, int(rng.integers(2, 12))) * 10
    if rng.random() < 0.1:
        max_calls, max_truths = 200, 60

    def iv():
        c = int(rng.integers(0, n_chrom))
        s = int(rng.choice(grid))
        return c, s, s + int(rng.choice(LENS))

    calls = [(int(rng.integers(0, S)), *iv(), int(rng.choice(CNS))) for _ in range(int(rng.integers(0, max_calls + 1)))]
    truths = []
    for _ in range(int(rng.integers(0, max_truths + 1))):
        k = int(rng.integers(0, 4))
        truths.append((*iv(), int(rng.choice(CNS)), [int(x) for x in rng.integers(0, S, k)]))
    return S, calls, truths, float(rng.choice(POS))


def order_free(S, calls, truths, po):
    """the counts from min Q, k_tp and b in each sample's sort.Slice order, as the kernels compute them"""
    st = np.zeros((S, 3, 4), np.uint64)

    def q(c, t):
        if c[0] != t[0]:
            return False
        total = min(float(c[2] - c[1]), float(t[2] - t[1]))
        ovl = min(c[2], t[2]) - max(c[1], t[1])
        r = 0.0 if ovl < 0 else (float(ovl) / total if total else math.nan)
        return r >= po and min(c[3], 3) == min(t[3], 3)

    def cls(s, e):
        return 0 if e - s < 20000 else (1 if e - s < 100000 else 2)

    for s in range(S):
        cs = [c[1:] for c in calls if c[0] == s]
        cs = [cs[i] for i in oc.go_order([c[0] for c in cs], [c[1] for c in cs])]
        if not cs:
            continue
        own = [t for t in truths for x in t[4] if x == s]
        counted = [False] * len(cs)
        for t in own:
            Q = [k for k, c in enumerate(cs) if q(c, t)]
            st[s, cls(t[1], t[2]), oc.TP if Q else oc.FN] += 1
            if Q:
                counted[Q[0]] = True
        for k, c in enumerate(cs):
            if not counted[k]:
                st[s, cls(c[1], c[2]), oc.FP] += 1
        tp_any = [any(q(c, t) for t in own) for c in cs]
        for o in truths:
            if s in o[4]:
                continue
            Q = [k for k, c in enumerate(cs) if q(c, o)]
            if not Q:
                st[s, cls(o[1], o[2]), oc.TN] += 1
                continue
            b = next((k for k, c in enumerate(cs) if c[0] > o[0] or (c[0] == o[0] and c[1] > o[2])), len(cs))
            k_tp = next((k for k in Q if tp_any[k]), math.inf)
            st[s, cls(o[1], o[2]), oc.FP] += int(min(k_tp, b) - Q[0])
    return st


def flat(calls, truths):
    """(c_sample, c_chrom, c_start, c_end, c_cn, t_chrom, t_start, t_end, t_cn, mem_ptr, mem_sample)"""
    return oc._arrays(calls, truths)


def cohort(rng, S, T, n_chrom=3, span=3_000_000, p_call=0.8, false_calls=3, tie=500):
    """flat arrays of a cohort: truths with skewed lengths and carrier counts (duplicates possible), calls from carried
    truths with jittered ends and some wrong CNs, plus false calls; starts rounded to `tie` so equal starts are common"""
    t_chrom = rng.integers(0, n_chrom, T)
    t_start = rng.integers(0, span, T) // tie * tie
    t_end = t_start + np.exp(rng.uniform(np.log(200), np.log(400_000), T)).astype(np.int64)
    t_cn = rng.choice([0, 1, 3, 4, 5, -1], T)
    k = np.minimum(rng.geometric(0.25, T) - 1, S)
    mem_ptr = np.concatenate([[0], np.cumsum(k)])
    mem_sample = rng.integers(0, S, int(mem_ptr[-1])) if S else np.zeros(0, np.int64)
    cs, cc, cb, ce, ccn = [], [], [], [], []
    for t in range(T):
        for s in mem_sample[mem_ptr[t]:mem_ptr[t + 1]]:
            if rng.random() < p_call:
                L = int(t_end[t] - t_start[t])
                b = max(0, int(t_start[t]) + int(rng.integers(-L // 4 - 1, L // 4 + 1)) // tie * tie)
                e = max(b, int(t_end[t]) + int(rng.integers(-L // 4 - 1, L // 4 + 1)))
                cn = int(t_cn[t]) if rng.random() < 0.9 else int(rng.choice([1, 3]))
                cs.append(int(s)); cc.append(int(t_chrom[t])); cb.append(b); ce.append(e); ccn.append(cn)
    for _ in range(int(false_calls * S)):
        b = int(rng.integers(0, span)) // tie * tie
        cs.append(int(rng.integers(0, S))); cc.append(int(rng.integers(0, n_chrom))); cb.append(b)
        ce.append(b + int(np.exp(rng.uniform(np.log(100), np.log(200_000))))); ccn.append(int(rng.choice([1, 3])))
    order = rng.permutation(len(cs))                                   # file order is not sample order
    a = lambda v, dt: np.asarray(v, dt)[order] if len(v) else np.zeros(0, dt)  # noqa: E731
    return (a(cs, np.int32), a(cc, np.int32), a(cb, np.int64), a(ce, np.int64), a(ccn, np.int64), t_chrom.astype(np.int32),
            t_start.astype(np.int64), t_end.astype(np.int64), t_cn.astype(np.int64), mem_ptr.astype(np.int64),
            mem_sample.astype(np.int32))


def _st(S, entries):
    """expected stats from {(sample, class): (TP, FP, FN, TN)}"""
    st = np.zeros((S, 3, 4), np.uint64)
    for (s, c), v in entries.items():
        st[s, c] = v
    return st


# (name, S, calls, truths, po, expected stats)
HAND = [
    # sample 1 carries a truth but has no call: no FN for it; sample 0's call is an FP and the truth a TN for it
    ("uncalled_sample_no_fn", 2, [(0, 0, 5000, 5100, 1)], [(0, 100, 200, 1, [1])], 0.4,
     _st(2, {(0, 0): (0, 1, 0, 1)})),
    # two calls qualify against one carried truth: the first in sort order is the TP, the second stays an FP
    ("first_qualifying_call_counted", 1, [(0, 0, 110, 190, 1), (0, 0, 100, 200, 1)], [(0, 100, 200, 1, [0])], 0.4,
     _st(1, {(0, 0): (1, 1, 0, 0)})),
    # o = [100, 200) is not sample 0's: c0 qualifies without a matching own truth, so c0 and the non-overlapping c1 are FPs
    # until c2, which qualifies against o and against sample 0's own truth
    ("fp_run_to_matching_call", 2, [(0, 0, 50, 150, 1), (0, 0, 60, 70, 1), (0, 0, 180, 200, 1)],
     [(0, 100, 200, 1, [1]), (0, 180, 200, 1, [0])], 0.4, _st(2, {(0, 0): (1, 4, 0, 0)})),
    # the same without the matching call: the run goes on to b, the first call past o's end
    ("fp_run_to_window_end", 2, [(0, 0, 50, 150, 1), (0, 0, 60, 70, 1), (0, 0, 90, 95, 3), (0, 0, 201, 300, 1)],
     [(0, 100, 200, 1, [1])], 0.4, _st(2, {(0, 0): (0, 7, 0, 0)})),
    # an FP against another sample's truth counts in that truth's class; the uncounted call in its own
    ("fp_class_other_vs_own", 2, [(0, 0, 0, 150000, 1)], [(0, 0, 50000, 1, [1])], 0.4,
     _st(2, {(0, 1): (0, 1, 0, 0), (0, 2): (0, 1, 0, 0)})),
    # a sample listed twice in a truth counts twice
    ("duplicate_membership_tp", 1, [(0, 0, 100, 200, 1)], [(0, 100, 200, 1, [0, 0])], 0.4, _st(1, {(0, 0): (2, 0, 0, 0)})),
    ("duplicate_membership_fn", 1, [(0, 0, 5000, 5100, 1)], [(0, 100, 200, 1, [0, 0])], 0.4, _st(1, {(0, 0): (0, 1, 2, 0)})),
    # sameCN clamps CN > 2 to 3: 5 matches 3, 4 does not match 2, -1 matches -1
    ("same_cn_clamp", 1, [(0, 0, 100, 200, 5), (0, 0, 1000, 1100, 4), (0, 0, 3000, 3100, -1)],
     [(0, 100, 200, 3, [0]), (0, 1000, 1100, 2, [0]), (0, 3000, 3100, -1, [0])], 0.4, _st(1, {(0, 0): (2, 1, 1, 0)})),
    # zero-length intervals: 0 / 0 is NaN, which never reaches po
    ("zero_length_nan", 1, [(0, 0, 100, 100, 1)], [(0, 100, 100, 1, [0])], 0.4, _st(1, {(0, 0): (0, 1, 1, 0)})),
    # -m NaN: nothing qualifies
    ("nan_minoverlap", 2, [(0, 0, 100, 200, 1)], [(0, 100, 200, 1, [0]), (0, 100, 200, 1, [1])], math.nan,
     _st(2, {(0, 0): (0, 1, 1, 1)})),
]
