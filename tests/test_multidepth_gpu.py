"""GPU tests of `goleft multidepth` at the library level: pass 1 (counts + site classes), the host block machine, pass 2
(exact sums, certified digits or the float64 chain) against the literal oracle (oracle/oracle_multidepth.c), byte for byte."""
import numpy as np
import pytest

from goleft_b200 import capi, synth
from oracle import loader as orc
from oracle import multidepth as omd

pytestmark = pytest.mark.gpu

CHROM = "chrT"


def _sample(L, cov, idx, read_len=150):
    if cov == 0:
        return np.zeros(0, np.int32), np.zeros(0, np.int32)
    return synth.segments(synth.reads(L, coverage=cov, read_len=read_len, contig_index=idx, gap=False, pileup=False))


def _long_reads(L, n, seed, span=20_000):
    rng = np.random.default_rng(seed)
    s = np.sort(rng.integers(0, L - span, n)).astype(np.int32)
    return s, (s + rng.integers(span // 2, span + 1, n)).astype(np.int32)


def _cohort(L, covs, seed):
    return [_sample(L, c, seed + i) for i, c in enumerate(covs)]


def _depths(L, samples):
    return np.stack([orc.pileup_diff(s, e, 0, L) for s, e in samples])


def _adders(ctx, samples, form):
    out, keep = [], []
    for s, e in samples:
        if form == "host32":
            out.append(lambda c, s=s, e=e: c.depth_add_segments(s, e))
        elif form == "unsorted32":
            p = np.random.default_rng(s.size).permutation(s.size)
            ss, ee = s[p].copy(), e[p].copy()
            keep.append((ss, ee))
            out.append(lambda c, s=ss, e=ee: c.depth_add_segments(s, e))
        elif form == "device32":
            if s.size == 0:
                out.append(lambda c: None)
                continue
            ds, de = ctx.dev_array(s), ctx.dev_array(e)
            keep.append((ds, de))
            out.append(lambda c, ds=ds, de=de, n=s.size: c.depth_add_segments_device(ds, de, n))
        elif form == "packed8":
            a, d, ln = capi.pack_segments8(s, e)
            keep.append((a, d, ln))
            out.append(lambda c, a=a, d=d, ln=ln: c.depth_add_segments_packed8(a, d, ln))
    return out, keep


def _run(ctx, L, samples, form, **kw):
    adders, keep = _adders(ctx, samples, form)
    txt = ctx.multidepth(CHROM, L, adders, **kw)
    del keep
    return txt, ctx.multidepth_stats()


@pytest.mark.parametrize("S", [1, 3, 51])
@pytest.mark.parametrize("window", [1, 15, 1000, 10_000_000])
def test_matches_oracle(ctx, S, window):
    L = 120_000 if S < 51 else 40_000
    covs = [(0 if i % 7 == 3 else (3 if i % 3 == 1 else 14)) for i in range(S)]
    if S == 1:
        covs = [12]
    samples = _cohort(L, covs, 100 * S)
    exp, _ = omd.text(CHROM, _depths(L, samples), window=window)
    got, st = _run(ctx, L, samples, "packed8", window=window)
    assert got == exp
    assert st["min_samples"] == omd.min_samples(0.5, S)
    assert st["blocks"] == exp.count(b"\n")


def test_three_segment_forms_identical(ctx):
    L = 200_000
    samples = _cohort(L, [14, 3, 9, 0, 20], 7)
    exp, _ = omd.text(CHROM, _depths(L, samples), window=1000)
    for form in ("packed8", "device32", "host32", "unsorted32"):
        got, _ = _run(ctx, L, samples, form, window=1000)
        assert got == exp, form


def test_paths_taken(ctx):
    """packed8 -> path 3, sorted device int32 -> fused (1), shuffled int32 / 20 kb reads -> bucketed events (4)"""
    L = 100_000
    s, e = _sample(L, 10, 5)
    lr = _long_reads(L, 60, 1)
    p = np.random.default_rng(0).permutation(s.size)
    cases = [("packed8", (s, e), 3), ("device32", (s, e), 1), ("host32", (s[p].copy(), e[p].copy()), 4), ("host32", lr, 4)]
    for form, seg, path in cases:
        adders, keep = _adders(ctx, [seg], form)
        ctx.multidepth_begin(L, 1)
        ctx.depth_begin(0, L)
        adders[0](ctx)
        ctx.multidepth_count()
        assert ctx.depth_last_path() == path, form


def test_long_reads_general_path(ctx):
    L = 150_000
    samples = [_long_reads(L, 120, 2), _sample(L, 12, 3), _long_reads(L, 200, 4)]
    exp, _ = omd.text(CHROM, _depths(L, samples), window=15, min_size=5)
    for form in ("host32", "device32"):
        got, _ = _run(ctx, L, samples, form, window=15, min_size=5)
        assert got == exp


def test_small_chunks_duplicate_blocks(ctx):
    """chunk size as a parameter: overlapping chunks print blocks twice, as the reference does"""
    L = 60_000
    samples = _cohort(L, [12, 2, 12], 40)
    exp, _ = omd.text(CHROM, _depths(L, samples), window=500, chunk=5000)
    got, _ = _run(ctx, L, samples, "packed8", window=500, chunk=5000)
    assert got == exp and len(exp) > 0


def test_ties_take_the_walk(ctx):
    """blocks of span 8 (Window 8 over fully covered bases) with an odd depth sum are exact ties: the float64 chain decides"""
    L = 50_000
    samples = _cohort(L, [25, 25, 25], 60)
    exp, _ = omd.text(CHROM, _depths(L, samples), window=8)
    got, st = _run(ctx, L, samples, "packed8", window=8)
    assert got == exp
    assert st["walked"] > 0 and st["certified"] > 0


def test_30x_large_blocks_all_certified(ctx):
    L = 2_000_000
    samples = _cohort(L, [30, 30, 30, 30], 80)
    exp, _ = omd.text(CHROM, _depths(L, samples))
    got, st = _run(ctx, L, samples, "packed8")
    assert got == exp
    assert st["walked"] == 0 and st["certified"] == st["blocks"] * 4


def test_errors(ctx):
    with pytest.raises(capi.GlError) as e:
        ctx.multidepth_begin(1 << 30, 2)
    assert e.value.code == capi.GL_ERANGE and "2^30" in str(e.value)
    with pytest.raises(capi.GlError) as e:
        ctx.multidepth_begin(1000, 65536)
    assert e.value.code == capi.GL_ERANGE
    ctx.multidepth_begin(1000, 2)
    with pytest.raises(capi.GlError) as e:
        ctx.multidepth_sites()
    assert e.value.code == capi.GL_ESTATE


def test_mixed_forms_in_one_cohort(ctx):
    """samples of one run on different paths (8-warp int32 kernels and the 4-warp packed8 kernel) share the block tables"""
    L = 150_000
    samples = _cohort(L, [14, 12, 9, 16], 90)
    exp, _ = omd.text(CHROM, _depths(L, samples), window=1000)
    forms = ["host32", "packed8", "unsorted32", "packed8"]
    adders, keep = [], []
    for seg, form in zip(samples, forms):
        a, k = _adders(ctx, [seg], form)
        adders += a
        keep.append(k)
    assert ctx.multidepth(CHROM, L, adders, window=1000) == exp
