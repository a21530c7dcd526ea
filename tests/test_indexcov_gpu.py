"""GPU parity for the indexcov / covstats / depthwed kernels against oracle/oracle_indexcov.c.
Integers bit-exact; float32/float64 results bit-exact too (same rounding points, no FMA)."""
import json
import os

import numpy as np
import pytest

from goleft_b200 import capi
from oracle import loader as orc

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def fixture():
    j = json.load(open(os.path.join(ROOT, "tests", "golden", "sample_issue_27_bai_linear_index.json")))
    refs = j["ioffsets"]
    voff = np.array([v for r in refs for v in r], np.uint64)
    ptr = np.concatenate([[0], np.cumsum([len(r) for r in refs])]).astype(np.int64)
    return voff, ptr


def synth_cohort(rng, S, T):
    """per-sample tile sizes shaped like SURVEY.md §8d C4: lognormal * copy-number blocks, some zeros"""
    base = rng.lognormal(np.log(1.6e9), 0.25, (S, T))
    cn = rng.choice([1.0, 0.5, 1.5, 0.0], p=[0.94, 0.02, 0.02, 0.02], size=(S, T // 64 + 1)).repeat(64, 1)[:, :T]
    return np.round(base * cn).astype(np.int64)


def test_fixture_through_gpu(ctx):
    voff, ptr = fixture()
    sizes, sptr = ctx.indexcov_sizes(voff, ptr)
    es, eptr = orc.ic_sizes(voff, ptr)
    assert np.array_equal(sizes, es) and np.array_equal(sptr, eptr)
    med = ctx.indexcov_scale(sizes)
    assert med == orc.ic_median(es) == 1484454039397
    d = ctx.indexcov_normalize(sizes, float(med))
    assert np.array_equal(d.view(np.uint32), orc.ic_normalize(es, float(med)).view(np.uint32))
    assert np.array_equal(ctx.indexcov_counts(d), orc.ic_counts(d))
    assert np.array_equal(ctx.indexcov_bins(d, d.size + 5), orc.ic_bins(d, d.size + 5))
    assert ctx.indexcov_bins(d, d.size).tolist() == [312, 304, 6, 1]


def test_negative_delta_is_an_error(ctx):
    from goleft_b200 import capi
    voff = np.array([100, 50, 70], np.uint64)
    with pytest.raises(capi.GlError) as ei:
        ctx.indexcov_sizes(voff, np.array([0, 3], np.int64))
    assert ei.value.code == capi.GL_ERANGE                      # the reference panics (types.go:75-77)
    with pytest.raises(ValueError):
        orc.ic_sizes(voff, np.array([0, 3], np.int64))


def test_cohort_medians_and_depths(ctx):
    rng = np.random.default_rng(4)
    S = 37
    lens = rng.integers(1, 5000, S)
    lens[0], lens[1], lens[2] = 1, 2, 50
    rows = [synth_cohort(rng, 1, int(n))[0] for n in lens]
    rows[3][:] = 0                                              # all-zero sample: median 0
    rows[4][:] = 7                                              # all ties
    sizes = np.concatenate(rows)
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    med, dep = ctx.indexcov_cohort(sizes, ptr)
    for i in range(S):
        m = orc.ic_median(rows[i])
        assert med[i] == float(m), i
        if m != 0:
            exp = orc.ic_normalize(rows[i], float(m))
            assert np.array_equal(dep[ptr[i]:ptr[i + 1]].view(np.uint32), exp.view(np.uint32)), i
        else:
            assert (dep[ptr[i]:ptr[i + 1]] == 0).all()


def test_cohort_large_samples_bracketed_path_and_fallbacks(ctx):
    """n > 8192 takes the sorted-sample bracketing (two passes); heavy ties / odd shapes must fall back and still be exact"""
    rng = np.random.default_rng(14)
    rows = [synth_cohort(rng, 1, n)[0] for n in (8193, 20_000, 191_000, 191_000, 250_000)]
    rows.append(np.sort(synth_cohort(rng, 1, 60_000)[0]))                       # ascending input (strided sample = quantiles)
    rows.append(np.sort(synth_cohort(rng, 1, 60_000)[0])[::-1].copy())          # descending
    rows.append(rng.choice(np.array([0, 5, 7, 1_000_000_007], np.int64), 100_000))    # four distinct values: ties everywhere
    rows.append(np.full(30_000, 123_456_789, np.int64))                         # all ties
    rows.append(np.zeros(50_000, np.int64))                                     # all zero: median 0
    heavy = synth_cohort(rng, 1, 120_000)[0]
    heavy[::3] *= 40                                                            # a third of the tiles 40x larger: the weighted median sits near the cap
    rows.append(heavy)
    cram = np.repeat(rng.integers(10_000, 90_000, 400), 300).astype(np.int64)   # CRAM pseudo-tiles: long constant runs (crai.go:56-127)
    rows.append(cram)
    lens = [r.size for r in rows]
    sizes = np.concatenate(rows)
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    med, dep = ctx.indexcov_cohort(sizes, ptr)
    for i, r in enumerate(rows):
        m = orc.ic_median(r)
        assert med[i] == float(m), (i, med[i], m)
        if m != 0:
            assert np.array_equal(dep[ptr[i]:ptr[i + 1]].view(np.uint32), orc.ic_normalize(r, float(m)).view(np.uint32)), i
        else:
            assert (dep[ptr[i]:ptr[i + 1]] == 0).all()
    fb = ctx.indexcov_cohort_fallbacks()
    assert 1 <= fb <= 6, fb                                                     # the tie-heavy samples fall back, the realistic ones do not
    # realistic samples only: the bracketed path must carry all of them
    real = [synth_cohort(rng, 1, 189_000)[0] for _ in range(24)]
    ptr2 = np.concatenate([[0], np.cumsum([r.size for r in real])]).astype(np.int64)
    med2, _ = ctx.indexcov_cohort(np.concatenate(real), ptr2, want_depth=False)
    assert [float(orc.ic_median(r)) for r in real] == med2.tolist()
    assert ctx.indexcov_cohort_fallbacks() == 0


def test_sizes_batch_equals_per_sample(ctx):
    rng = np.random.default_rng(15)
    voffs, voff_off, n_intv, size_off, exp = [], [], [], [], []
    samples = []                                                # (voff, ref_ptr, sizes, size_ptr) of each sample alone
    at = so = 0
    for s in range(7):
        first = len(voffs)
        for r in range(int(rng.integers(1, 30))):
            k = int(rng.choice([0, 1, 2, 3, 50, 4000]))
            v = np.cumsum(rng.integers(0, 1 << 30, k)).astype(np.uint64)
            voffs.append(v)
            if k >= 2:
                voff_off.append(at); n_intv.append(k); size_off.append(so)
                exp.append(np.diff(v.astype(np.int64)))
                so += k - 1
            at += k
        refs = voffs[first:]
        ref_ptr = np.concatenate([[0], np.cumsum([v.size for v in refs])]).astype(np.int64)
        size_ptr = np.concatenate([[0], np.cumsum([max(v.size - 1, 0) for v in refs])]).astype(np.int64)
        samples.append((np.concatenate(refs), ref_ptr, np.concatenate([np.diff(v.astype(np.int64)) for v in refs]), size_ptr))
    got = ctx.indexcov_sizes_batch(np.concatenate(voffs), voff_off, n_intv, size_off, so)
    assert np.array_equal(got, np.concatenate(exp))
    # the per-sample entry gives the same sizes and offsets
    for voff, ref_ptr, sizes, size_ptr in samples:
        got_s, got_p = ctx.indexcov_sizes(voff, ref_ptr)
        assert np.array_equal(got_s, sizes) and np.array_equal(got_p, size_ptr)
    # one negative delta inside a middle reference of a many-reference sample: the reference panics (types.go:75-77)
    voff, ref_ptr, _, _ = max(samples, key=lambda t: t[1].size)
    mid = [r for r in range(1, ref_ptr.size - 2) if ref_ptr[r + 1] - ref_ptr[r] >= 2]
    r = mid[len(mid) // 2]
    k = int(ref_ptr[r] + (ref_ptr[r + 1] - ref_ptr[r]) // 2)    # ref_ptr[r] < k < ref_ptr[r + 1]
    bad = voff.copy()
    bad[k - 1] = bad[k] + np.uint64(1)
    with pytest.raises(capi.GlError) as ei:
        ctx.indexcov_sizes(bad, ref_ptr)
    assert ei.value.code == capi.GL_ERANGE


def test_counts_batch(ctx):
    rng = np.random.default_rng(5)
    n_seg = 40
    lens = rng.integers(0, 3000, n_seg)
    d = np.abs(rng.normal(1.0, 0.4, int(lens.sum()))).astype(np.float32)
    d[rng.random(d.size) < 0.02] = 0
    d[rng.random(d.size) < 0.01] = 60000.0
    d[:4] = [0.85, 1.15, 0.15, 8.0]                             # threshold values themselves
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    longest = lens + rng.integers(0, 50, n_seg)
    counts, bins = ctx.indexcov_counts_batch(d, ptr, longest)
    for s in range(n_seg):
        seg = d[ptr[s]:ptr[s + 1]]
        assert np.array_equal(counts[s], orc.ic_counts(seg)), s
        assert np.array_equal(bins[s], orc.ic_bins(seg, int(longest[s]))), s


def test_xnorm(ctx):
    rng = np.random.default_rng(6)
    for S, T in [(5, 40), (23, 300), (64, 1000)]:
        d = np.abs(rng.normal(1.0, 0.3, (S, T))).astype(np.float32)
        d[rng.random((S, T)) < 0.03] = 0
        d[0, 5] = 1e-7                                          # forces the ordered (non order-free) summation path
        d[1, 7] = 3e4
        lens = rng.integers(T - 20, T + 1, S).astype(np.int32)
        lens[0] = T
        got = ctx.indexcov_xnorm(d, lens)
        exp = orc.ic_xnorm(d, lens)
        for i in range(S):
            n = lens[i]
            assert np.array_equal(got[i, :n].view(np.uint32), exp[i, :n].view(np.uint32)), (S, T, i)


def test_bincount(ctx):
    rng = np.random.default_rng(7)
    v = rng.normal(450, 80, 1_000_000).astype(np.int32)
    for lo, hi in [(150, 900), (0, 20000), (-100, 5)]:
        assert np.array_equal(ctx.bincount(v, lo, hi), orc.bincount(v, lo, hi))
    assert ctx.bincount(np.zeros(0, np.int32), 0, 10).sum() == 0


def test_depthwed(ctx):
    rng = np.random.default_rng(8)
    S = 45
    rows = []
    for chrom, L in enumerate([10_050, 3_000, 777]):
        st = np.arange(0, L, 100)
        rows += [(chrom, int(a), int(min(a + 100, L))) for a in st]
    chrom_id = np.array([r[0] for r in rows], np.int32)
    starts = np.array([r[1] for r in rows], np.int32)
    ends = np.array([r[2] for r in rows], np.int32)
    R = len(rows)
    # values as the reference would parse them back from "%.4g" text
    means = np.array([[float("%.4g" % x) for x in rng.gamma(9, 3.3, R)] for _ in range(S)])
    means[0, :5] = [0.5, 1.5, 2.4999, 0.49, 1e5]
    for size in [100, 500, 1000, 100000]:
        g = ctx.depthwed_aggregate(means, starts, ends, chrom_id, size)
        e = orc.depthwed(means, starts, ends, chrom_id, size)
        for a, b in zip(g, e):
            assert np.array_equal(a, b), size


def test_depthwed_i32(ctx):
    """int32 form: the reference rounds at parse time (depthwed.go:103); same groups, int32 sums, overflow detected"""
    from goleft_b200 import capi
    rng = np.random.default_rng(8)
    for S, R, size in [(3, 40, 1000), (17, 1000, 750), (64, 5000, 250), (5, 333, 10_000)]:
        starts = (np.arange(R) * 250).astype(np.int32)
        chrom = np.sort(rng.integers(0, 3, R)).astype(np.int32)
        for c in range(3):
            m = chrom == c
            starts[m] -= starts[m][0] if m.any() else 0
        ends = starts + 250
        means = np.array([[float("%.4g" % x) for x in rng.gamma(9, 3.3, R)] for _ in range(S)])
        depth = (0.5 + means).astype(np.int64).astype(np.int32)              # int(0.5 + dep)
        es, ee, ec, eo = orc.depthwed(means, starts, ends, chrom, size)
        gs, ge, gc, go = ctx.depthwed_aggregate_i32(depth, starts, ends, chrom, size)
        assert np.array_equal(gs, es) and np.array_equal(ge, ee) and np.array_equal(gc, ec)
        assert np.array_equal(go.astype(np.int64), eo)
    big = np.full((2, 8), 2_000_000_000, np.int32)
    st = (np.arange(8) * 250).astype(np.int32)
    with pytest.raises(capi.GlError) as ei:
        ctx.depthwed_aggregate_i32(big, st, st + 250, np.zeros(8, np.int32), 1000)
    assert ei.value.code == capi.GL_ERANGE


def test_format_g3_exact(ctx):
    """I6: the GPU "%.3g" tokens equal printf's for every value tried: random magnitudes, the half-way cases of
    3-digit rounding, powers of ten, denormals/huge values (host fallback), zero, inf, nan"""
    rng = np.random.default_rng(10)
    vals = [np.float32(x) for x in (0.0, -0.0, 1.0, 0.5, 999.5, 999.4999, 99.95, 9.995, 0.9995, 0.09995, 1000.0, 1000.5, 1005.0,
                                      9995.0, 99950.0, 1e-4, 9.9949e-5, 9.995e-5, 1e-5, 1.2345e-7, 50000.0, 0.125, 0.375, 2.5,
                                      1.005, 1.015, 1.025, 100.5, 101.5, 1e15, 9.99e14, 1e-15, 9.9e-16, 1e-30, 3e38, 1e-45,
                                      np.inf, -np.inf, np.nan, -3.14159, 123456.0, 12.25, 12.35, 12.45)]
    a = np.concatenate([np.array(vals, np.float32),
                        np.exp(rng.uniform(np.log(1e-16), np.log(1e16), 400_000)).astype(np.float32),
                        np.abs(rng.normal(1.0, 0.4, 400_000)).astype(np.float32),
                        (rng.integers(1, 10000, 200_000) / np.float32(8.0)).astype(np.float32),       # many exact ties
                        (rng.integers(100, 100000, 200_000).astype(np.float32) * np.float32(0.005)),
                        -np.abs(rng.normal(3, 5, 1000)).astype(np.float32)])
    tok = ctx.format_g3(a)
    n_host = 0
    for v, t in zip(a, tok):
        ln = int(t[9])
        if ln == 0:
            n_host += 1
            assert not (1e-15 <= abs(float(v)) < 1e15)
            continue
        got = bytes(t[:ln]).decode()
        if np.isnan(v):
            exp = "NaN"
        elif np.isinf(v):
            exp = "+Inf" if v > 0 else "-Inf"
        else:
            exp = "%.3g" % float(v)
        assert got == exp, (float(v), got, exp)
    assert n_host < 60_000


def test_indexsplit_accumulate_bit_exact(ctx):
    """gl_indexsplit_accumulate: per-tile float64 sums over the samples in path order — bit-identical to the sequential
    adds of indexsplit.go:92-115 (ragged samples, a sample with fewer references, an empty reference)."""
    rng = np.random.default_rng(4)
    R = 6
    lens = [900, 1, 0, 4000, 37, 12000]
    samples = []
    for k in range(23):
        nref = R if k % 5 else R - 2
        per = []
        for r in range(nref):
            n = max(0, lens[r] - int(rng.integers(0, 3)) * (k % 3 == 0))
            per.append(rng.integers(0, 4_000_000_000, n).astype(np.int64))
        samples.append(per)
    sizes, ptr, out_ptr = capi.indexsplit_layout(samples, R)
    got = ctx.indexsplit_accumulate(sizes, ptr, len(samples), R, out_ptr)
    exp = np.zeros(int(out_ptr[-1]))
    for s in range(len(samples)):
        for r in range(R):
            a, b = ptr[s * (R + 1) + r], ptr[s * (R + 1) + r + 1]
            exp[out_ptr[r]:out_ptr[r] + (b - a)] += sizes[a:b].astype(np.float64) / 1e9
    assert np.array_equal(got.view(np.uint64), exp.view(np.uint64))
    names = ["r%d" % r for r in range(R)]
    ref_lens = [max(1, n) * 16384 + 5 for n in lens]
    assert capi.indexsplit_chunks(got, out_ptr, names, ref_lens, list(range(R)), 50) == orc.indexsplit(samples, names, ref_lens, 50)
