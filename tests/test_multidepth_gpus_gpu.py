"""`goleft multidepth` with the cohort split over several contexts (gl_multidepth_merge / gl_multidepth_adopt_sites): every
split gives the runs, blocks, sums, q, val and certified flags of a one-context run, and the oracle's rows, byte for byte.

Contexts live on device 0 ("same") and, when two or more devices are visible, on distinct devices ("distinct": context k
on device k % n), so the merge's cudaMemcpyPeerAsync runs within one device and between devices."""
import numpy as np
import pytest

from goleft_b200 import capi
from oracle import multidepth as omd
from test_multidepth_gpu import CHROM, _adders, _cohort, _depths
from test_multidepth_scale_gpu import MULT, _cat, _mult_text, _tiles, runs_of

pytestmark = pytest.mark.gpu

N_CTX = 4
PLACES = ["same", "distinct"]


@pytest.fixture(scope="module")
def pools():
    n_dev = capi.device_count()
    out = {"same": [capi.Ctx(0) for _ in range(N_CTX)]}
    if n_dev >= 2:
        out["distinct"] = [capi.Ctx(k % n_dev) for k in range(N_CTX)]
    yield out
    for cs in out.values():
        for c in cs:
            c.close()


def _ctxs(pools, place, n):
    if place not in pools:
        pytest.skip("fewer than two CUDA devices visible")
    return pools[place][:n]


FORMS = ["packed8", "host32", "device32", "unsorted32"]


def _shard(ctxs, samples, split):
    """adders per context for the contiguous split (sample counts per context); sample j takes FORMS[j % 4], made on its
    own context's device"""
    adders, keep, j = [], [], 0
    for c, n in zip(ctxs, split):
        a = []
        for seg in samples[j:j + n]:
            ad, k = _adders(c, [seg], FORMS[j % len(FORMS)])
            a += ad
            keep.append(k)
            j += 1
        adders.append(a)
    assert j == len(samples)
    return adders, keep


def _same_parts(got, ref):
    for k in ("sums", "q", "val", "certified"):
        assert np.array_equal(got[k], ref[k]), k
    for a, b in zip(got["runs"] + got["blocks"], ref["runs"] + ref["blocks"]):
        assert np.array_equal(a, b)


SPLITS4 = [(1, 1, 1, 1), (3, 1), (1, 3), (2, 2), (1, 2, 1)]
SPLITS7 = [(6, 1), (1, 6), (2, 3, 2), (3, 4), (1, 1, 4, 1)]


@pytest.mark.parametrize("place", PLACES)
@pytest.mark.parametrize("frac", [0.5, 0.3])
@pytest.mark.parametrize("S,splits", [(4, SPLITS4), (7, SPLITS7)])
def test_splits_match_one_context_and_oracle(pools, place, frac, S, splits):
    L = 150_000
    covs = [14, 3, 0, 16, 9, 12, 20][:S]                       # a zero-coverage sample in both cohorts
    samples = _cohort(L, covs, 300 + S)
    exp, cls = omd.text(CHROM, _depths(L, samples), window=1000, min_samples=frac)
    assert exp.count(b"\n") > 3
    one = _ctxs(pools, "same", 1)
    adders, keep = _shard(one, samples, (S,))
    rows1, ref = capi.Ctx.multidepth_sharded(one, CHROM, L, adders, window=1000, min_samples=frac, parts=True)
    assert rows1 == exp
    es, ec = runs_of(cls)
    assert np.array_equal(ref["runs"][0], es) and np.array_equal(ref["runs"][1], ec)
    for split in splits:
        ctxs = _ctxs(pools, place, len(split))
        adders, keep = _shard(ctxs, samples, split)
        rows, got = capi.Ctx.multidepth_sharded(ctxs, CHROM, L, adders, window=1000, min_samples=frac, parts=True)
        assert rows == exp, split
        _same_parts(got, ref)
        assert got["merge_bytes"] == (len(split) - 1) * ((L + 4095) // 4096) * 4096 * 17 // 8
        for c in ctxs[1:]:                                     # adopted sites: the same runs from every context
            rs, rc = c.multidepth_sites()
            assert np.array_equal(rs, es) and np.array_equal(rc, ec)
    del keep


@pytest.mark.parametrize("place", PLACES)
def test_merge_in_many_chunks(pools, place, monkeypatch):
    """GL_MD_MERGE_CHUNK_BASES small and not a whole tile: ~70 chunks per source through the two staging buffers, a ragged
    last chunk, and a contig that ends inside a 32-base word"""
    L = 1_000_003
    samples = _cohort(L, [14, 3, 9, 16, 12], 77)
    exp, _ = omd.text(CHROM, _depths(L, samples), window=1000)
    monkeypatch.setenv("GL_MD_MERGE_CHUNK_BASES", "14399")     # 450 words
    ctxs = _ctxs(pools, place, 3)
    adders, keep = _shard(ctxs, samples, (2, 2, 1))
    launches = ctxs[0].launch_count()
    rows, got = capi.Ctx.multidepth_sharded(ctxs, CHROM, L, adders, window=1000, parts=True)
    assert rows == exp
    words = (L + 4095) // 4096 * 128
    merges = 2 * -(-words // 450)
    assert ctxs[0].launch_count() - launches >= merges
    one = _ctxs(pools, "same", 1)
    adders1, keep1 = _shard(one, samples, (5,))
    _, ref = capi.Ctx.multidepth_sharded(one, CHROM, L, adders1, window=1000, parts=True)
    _same_parts(got, ref)
    del keep, keep1


def _edge_cohort(L):
    """five distinct samples (repeated MULT times: 65535 samples).  Every one covers [1000, 3001) and [4001, 6000) at depth
    >= 10 and nothing in [3001, 4001): bases 3000 (low half of its 32-bit lane) and 4001 (high half) are counted by all
    65535 samples, their lane partners 3001 and 4000 by none.  Samples 0 and 2 add depth 3 over [7000, 9000) and sample
    4 depth 8 there, so those sites count 1 and stay insufficient.  Sample 4 also has one base at depth 1 first (an
    insufficient site: the block machine starts caching after one)."""
    out = []
    for k in range(5):
        parts = [_tiles(1000, 3001, 10 + k), _tiles(4001, 6000, 10 + (k % 2)), _tiles(1000 + 37 * k, 1100 + 37 * k, 1)]
        if k in (0, 2):
            parts.append(_tiles(7000, 9000, 3))
        if k == 4:
            parts += [_tiles(7000, 9000, 8), _tiles(200, 201, 1)]
        out.append(_cat(*parts))
    return out


def test_counter_edge_65535(pools):
    L = 12_000
    samples = _edge_cohort(L)
    d = _depths(L, samples)
    cnt = sum(m * (dk >= 7) for dk, m in zip(d, MULT))
    assert cnt[3000] == cnt[4001] == 65535 and cnt[3001] == cnt[4000] == 0
    assert 3000 % 2 == 0 and 3001 // 2 == 3000 // 2 and 4000 // 2 == 4001 // 2
    frac = 65534 / 65535                                        # minSamples 65534: sufficient only at a count of 65535
    exp, cls, blk = _mult_text(d, MULT, frac=frac)
    assert cls[3000] == cls[4001] == 2 and cls[3001] == cls[4000] == 0 and cls[8000] == cls[200] == 1
    assert [1000, 3001, 2001] in blk.tolist()
    ctxs = _ctxs(pools, "same", 3)
    distinct = [[_adders(c, [seg], "packed8")[0][0] for seg in samples] for c in ctxs]
    cohort = [k for k, m in enumerate(MULT) for _ in range(m)]
    cuts = [0, 21_845, 43_690, 65_535]                          # the 32767 copies of sample 0 straddle the first cut
    adders = [[distinct[g][k] for k in cohort[cuts[g]:cuts[g + 1]]] for g in range(3)]
    rows, got = capi.Ctx.multidepth_sharded(ctxs, CHROM, L, adders, min_samples=frac, parts=True)
    es, ec = runs_of(cls)
    assert np.array_equal(got["runs"][0], es) and np.array_equal(got["runs"][1], ec)
    assert rows == exp
    assert np.array_equal(np.stack(got["blocks"], 1), blk)


# ---------------------------------------------------------------------------------------------------- error states
def _begin_count(c, L, S, n, seg=None, **kw):
    c.multidepth_begin(L, S, **kw)
    for _ in range(n):
        c.depth_begin(0, L)
        if seg is not None:
            c.depth_add_segments(*seg)
        c.multidepth_count()


def _code(fn, *a):
    with pytest.raises(capi.GlError) as e:
        fn(*a)
    return e.value.code


def test_errors(pools):
    a, b, c, d = _ctxs(pools, "same", 4)
    L = 20_000
    seg = _cohort(L, [12], 5)[0]
    _begin_count(a, L, 3, 1, seg)
    _begin_count(b, L, 3, 1, seg)
    with capi.Ctx(0) as fresh:                                                       # a context never begun
        assert _code(a.multidepth_merge, [fresh]) == capi.GL_ESTATE
        assert _code(fresh.multidepth_merge, [b]) == capi.GL_ESTATE
        assert _code(fresh.multidepth_adopt_sites, a) == capi.GL_ESTATE
        assert _code(a.multidepth_adopt_sites, fresh) == capi.GL_ESTATE
    assert _code(a.multidepth_merge, [b, a]) == capi.GL_EINVAL                       # the destination among the sources
    assert _code(a.multidepth_merge, [b, b]) == capi.GL_EINVAL                       # a repeated source
    assert _code(a.multidepth_merge, [None]) == capi.GL_EINVAL
    for L2, S2, mc, f in ((L + 1, 3, 7, 0.5), (L, 4, 7, 0.5), (L, 3, 8, 0.5), (L, 3, 7, 0.9)):   # another run
        c.multidepth_begin(L2, S2, mc, f)
        assert _code(a.multidepth_merge, [c]) == capi.GL_EINVAL, (L2, S2, mc, f)
        assert _code(a.multidepth_adopt_sites, c) == capi.GL_EINVAL, (L2, S2, mc, f)
    _begin_count(c, L, 3, 2, seg, min_samples=0.6)                                   # int(0.5 + 0.6 * 3) = 2: the same run
    assert _code(a.multidepth_merge, [b, c]) == capi.GL_ESTATE                       # 1 + 1 + 2 samples > S = 3
    a.multidepth_merge([b])                                                          # the refused merge changed nothing
    assert _code(b.multidepth_count) == capi.GL_ESTATE                               # a merged source refuses counts,
    assert _code(b.multidepth_sites) == capi.GL_ESTATE                               # sites,
    assert _code(a.multidepth_merge, [b]) == capi.GL_ESTATE                          # a second merge
    assert _code(b.multidepth_merge, []) == capi.GL_ESTATE                           # and a merge into it
    assert _code(b.multidepth_adopt_sites, a) == capi.GL_ESTATE                      # a has not run its sites
    assert _code(a.multidepth_sites) == capi.GL_ESTATE                               # 2 of 3 samples counted
    _begin_count(d, L, 3, 1, seg)
    assert _code(d.multidepth_adopt_sites, d) == capi.GL_EINVAL
    assert _code(d.multidepth_adopt_sites, None) == capi.GL_EINVAL
    a.multidepth_merge([d])
    rs, rc = a.multidepth_sites()
    assert _code(a.multidepth_merge, []) == capi.GL_ESTATE                           # the destination has run its sites
    _begin_count(c, L, 3, 1, seg)
    assert _code(c.multidepth_merge, [a]) == capi.GL_ESTATE                          # so has the source
    for x in (b, d):                                                                 # adopting makes them usable again
        x.multidepth_adopt_sites(a)
        s2, c2 = x.multidepth_sites()
        assert np.array_equal(s2, rs) and np.array_equal(c2, rc)
    a.multidepth_begin(L, 1)                                                         # and a one-context run is as before
    a.depth_begin(0, L)
    a.depth_add_segments(*seg)
    a.multidepth_count()
    s1, c1 = a.multidepth_sites()
    exp, cls = omd.text(CHROM, _depths(L, [seg]))
    es, ec = runs_of(cls)
    assert np.array_equal(s1, es) and np.array_equal(c1, ec)
