"""gl_bam_covstats_prefetch: the next BAM's first batch read while the current one is sampled.  A call that starts from a
prefetch gives the same bits as one that does not (every Stats field, counter, H and sample array, and the restatement),
a file the device refuses is still refused and answered by the host route, and the prefetch lives exactly as long as its
contract says."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench_covstats  # noqa: E402
import covstats_ref as cr  # noqa: E402
from covstats_bams import odd_member  # noqa: E402
from goleft_b200 import capi  # noqa: E402

pytestmark = pytest.mark.gpu
KNOB = "GL_COVSTATS_BATCH_BYTES"


@pytest.fixture(scope="module")
def ctx():
    with capi.Ctx(0) as c:
        yield c


@pytest.fixture(autouse=True)
def _no_knob():
    os.environ.pop(KNOB, None)
    yield
    os.environ.pop(KNOB, None)


def small(tmp_path, name, seed, **kw):
    """(path, records, mates) of a small indexed BAM"""
    block = kw.pop("block", 60000)
    refs, recs, mates = cr.records(np.random.default_rng(seed), kw.pop("per_ref", [6000, 0, 2500]), **kw)
    return cr.write(tmp_path, name, refs, recs, mates, block=block), recs, mates


def baseline(ctx, path, n, skip, host=False):
    """(st, H, samples) of a call without a prefetch, on a handle of its own"""
    bam = capi.Bam(path)
    try:
        return (capi.bam_covstats_host if host else capi.bam_covstats)(ctx, bam, n, skip, samples=True)
    finally:
        bam.close()


def same(a, b):
    (sa, Ha, ga), (sb, Hb, gb) = a, b
    for k in capi.CovStats.STATS + capi.CovStats.COUNTERS + ("h_len",):
        assert np.float64(getattr(sa, k)).tobytes() == np.float64(getattr(sb, k)).tobytes(), k
    assert Ha.tobytes() == Hb.tobytes()
    assert all(np.array_equal(x, y) for x, y in zip(ga, gb))


def restated(res, recs, mates, n, skip):
    c, arrs = cr.restate(recs, mates, n, skip)
    st, _, got = res
    assert all(getattr(st, k) == v for k, v in c.items())
    assert all(np.array_equal(a, b) for a, b in zip(got, arrs))


def test_sequence_of_bams(ctx, tmp_path):
    """A -> B -> C, each prefetched once the call on the one before it has returned (one prefetch slot per ctx: a prefetch
    made before that call would replace the one that call is about to use)"""
    n, skip = 400, 300
    bams = [small(tmp_path, "%s.bam" % k, 30 + i, per_ref=[5000 + 2000 * i, 0, 3000]) for i, k in enumerate("abc")]
    base = [baseline(ctx, p, n, skip) for p, _, _ in bams]
    hs = [capi.Bam(p) for p, _, _ in bams]
    res = []
    for i, h in enumerate(hs):
        res.append(capi.bam_covstats(ctx, h, n, skip, samples=True))
        if i + 1 < len(hs):
            capi.bam_covstats_prefetch(ctx, hs[i + 1], n, skip)
    for h in hs:
        h.close()
    assert [r[0].prefetched for r in res] == [0, 1, 1] and [b[0].prefetched for b in base] == [0, 0, 0]
    for r, b, (_, recs, mates) in zip(res, base, bams):
        same(r, b)
        restated(r, recs, mates, n, skip)


@pytest.fixture(scope="module")
def paired(tmp_path_factory):
    d = tmp_path_factory.mktemp("paired")
    out = []
    for seed in (3, 4):
        p = str(d / ("p%d.bam" % seed))
        bench_covstats.write_paired_bam(p, n_records=3_200_000, seed=seed)
        out.append(p)
    return out


def test_real_size_first_batch(ctx, paired):
    """the command's n and skip on two 3.2 M-record paired BAMs: the second one's first batch (the real size) is prefetched
    while the first is sampled, and its later batches follow"""
    n, skip = 1_000_000, 100_000
    base = [baseline(ctx, p, n, skip) for p in paired]
    x, y = capi.Bam(paired[0]), capi.Bam(paired[1])
    capi.bam_covstats_prefetch(ctx, y, n, skip)
    rx = capi.bam_covstats(ctx, x, n, skip, samples=True)
    ry = capi.bam_covstats(ctx, y, n, skip, samples=True)
    x.close(); y.close()
    assert rx[0].prefetched == 0 and ry[0].prefetched == 1 and ry[0].n_batches >= 2 and ry[0].n_insert == n
    same(rx, base[0]); same(ry, base[1])


def test_next_bam_refused_by_the_device(ctx, tmp_path):
    """no index, or an odd BGZF member: the prefetch returns GL_OK, the call GL_ESTATE, the host route the same answer"""
    n, skip = 200, 100
    cur, _, _ = small(tmp_path, "cur.bam", 40)
    good, recs, mates = small(tmp_path, "good.bam", 41, per_ref=[5000, 2000], block=20000)
    noidx = str(tmp_path / "noidx.bam")
    open(noidx, "wb").write(open(good, "rb").read())
    for path in (noidx, odd_member(good)):
        want = baseline(ctx, path, n, skip, host=True)
        restated(want, recs, mates, n, skip)
        c, nx = capi.Bam(cur), capi.Bam(path)
        capi.bam_covstats_prefetch(ctx, nx, n, skip)
        capi.bam_covstats(ctx, c, n, skip)
        with pytest.raises(capi.GlError) as e:
            capi.bam_covstats(ctx, nx, n, skip)
        assert e.value.code == capi.GL_ESTATE
        same(capi.bam_covstats_host(ctx, nx, n, skip, samples=True), want)
        c.close(); nx.close()


SHAPES = {
    "n0": dict(n=0, skip=10, prefetched=0),
    "ends_inside_skip": dict(n=10, skip=10 ** 6, prefetched=1),
    "whole_file_first_batch": dict(n=300, skip=200, prefetched=1),
    "one_unit_first_batch": dict(n=300, skip=200, prefetched=1, knob="1"),
}


@pytest.mark.parametrize("shape", sorted(SHAPES))
def test_shapes_of_the_next_bam(ctx, tmp_path, shape):
    kw = SHAPES[shape]
    n, skip = kw["n"], kw["skip"]
    if "knob" in kw:
        os.environ[KNOB] = kw["knob"]
    cur, _, _ = small(tmp_path, "cur.bam", 50)
    path, recs, mates = small(tmp_path, "next.bam", 51, per_ref=[5000, 0, 3000], ref_len=200_000, block=4000)
    want = baseline(ctx, path, n, skip)
    c, nx = capi.Bam(cur), capi.Bam(path)
    capi.bam_covstats_prefetch(ctx, nx, n, skip)
    capi.bam_covstats(ctx, c, n, skip)
    got = capi.bam_covstats(ctx, nx, n, skip, samples=True)
    c.close(); nx.close()
    assert got[0].prefetched == kw["prefetched"]
    if shape == "whole_file_first_batch":
        assert got[0].n_batches == 1
    if shape == "one_unit_first_batch":
        assert got[0].n_batches >= 3
    same(got, want)
    restated(got, recs, mates, n, skip)


@pytest.mark.parametrize("other", ["n", "skip"])
def test_another_n_or_skip_discards(ctx, tmp_path, other):
    n, skip = 300, 200
    path, recs, mates = small(tmp_path, "b.bam", 60)
    want = baseline(ctx, path, n, skip)
    b = capi.Bam(path)
    capi.bam_covstats_prefetch(ctx, b, n + 1 if other == "n" else n, skip + 1 if other == "skip" else skip)
    got = capi.bam_covstats(ctx, b, n, skip, samples=True)
    again = capi.bam_covstats(ctx, b, n, skip, samples=True)
    b.close()
    assert got[0].prefetched == 0 and again[0].prefetched == 0
    same(got, want); same(again, want)
    restated(got, recs, mates, n, skip)


def test_close_without_sampling(ctx, tmp_path):
    """the prefetch's handle is closed unsampled: the prefetch goes with it and the ctx keeps working"""
    n, skip = 300, 200
    a, _, _ = small(tmp_path, "a.bam", 61)
    path, recs, mates = small(tmp_path, "b.bam", 62)
    want = baseline(ctx, path, n, skip)
    h = capi.Bam(a)
    capi.bam_covstats_prefetch(ctx, h, n, skip)
    h.close()
    b = capi.Bam(path)
    got = capi.bam_covstats(ctx, b, n, skip, samples=True)
    capi.bam_covstats_prefetch(ctx, b, n, skip)
    prefetched = capi.bam_covstats(ctx, b, n, skip, samples=True)
    b.close()
    assert got[0].prefetched == 0 and prefetched[0].prefetched == 1
    same(got, want); same(prefetched, want)


def test_ctx_destroyed_with_a_prefetch(tmp_path):
    """gl_ctx_destroy joins the prefetch and forgets it; the handle stays usable on another ctx"""
    n, skip = 300, 200
    path, recs, mates = small(tmp_path, "b.bam", 63)
    b = capi.Bam(path)
    with capi.Ctx(0) as c1:
        capi.bam_covstats_prefetch(c1, b, n, skip)
    with capi.Ctx(0) as c2:
        got = capi.bam_covstats(c2, b, n, skip, samples=True)
    b.close()
    assert got[0].prefetched == 0
    restated(got, recs, mates, n, skip)


def test_second_prefetch_replaces_the_first(ctx, tmp_path):
    n, skip = 300, 200
    (pb, rb, mb), (pc, rc, mc) = small(tmp_path, "b.bam", 64), small(tmp_path, "c.bam", 65)
    wb, wc = baseline(ctx, pb, n, skip), baseline(ctx, pc, n, skip)
    b, c = capi.Bam(pb), capi.Bam(pc)
    capi.bam_covstats_prefetch(ctx, b, n, skip)
    capi.bam_covstats_prefetch(ctx, c, n, skip)
    gb = capi.bam_covstats(ctx, b, n, skip, samples=True)
    gc = capi.bam_covstats(ctx, c, n, skip, samples=True)
    b.close(); c.close()
    assert gb[0].prefetched == 0 and gc[0].prefetched == 1
    same(gb, wb); same(gc, wc)


def test_calls_on_the_current_bam_leave_it(ctx, tmp_path):
    """the --hist pattern: two calls on the current BAM, and its host route, between the prefetch and its use"""
    n, skip = 300, 200
    (pa, _, _), (pb, rb, mb) = small(tmp_path, "a.bam", 66), small(tmp_path, "b.bam", 67)
    wa, wb = baseline(ctx, pa, n, skip), baseline(ctx, pb, n, skip)
    a, b = capi.Bam(pa), capi.Bam(pb)
    capi.bam_covstats_prefetch(ctx, b, n, skip)
    r1 = capi.bam_covstats(ctx, a, n, skip, samples=True)
    r2 = capi.bam_covstats(ctx, a, n, skip, samples=True)
    rh = capi.bam_covstats_host(ctx, a, n, skip, samples=True)
    gb = capi.bam_covstats(ctx, b, n, skip, samples=True)
    a.close(); b.close()
    assert r1[0].prefetched == r2[0].prefetched == 0 and gb[0].prefetched == 1
    same(r1, wa); same(r2, wa); same(rh, wa); same(gb, wb)
    restated(gb, rb, mb, n, skip)
