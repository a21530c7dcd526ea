"""gl_bam_region_chunks, the host half of a BAM region query: the virtual-offset ranges equal a restatement of reg2bins +
the linear-index cut + merging, on plain BAIs and on BAIs whose chunks are merged as samtools writes them; every record
overlapping a query lies inside one range.  No GPU needed."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import region_bams as rb  # noqa: E402
from bamutil import make_bam  # noqa: E402

VARIANTS = {"plain": {}, "htslib": dict(merged=True), "block_merge": dict(merged=True, min_dist=0)}


@pytest.fixture(scope="module")
def fx():
    return rb.fixture()


def _write(tmp_path, fx, variant):
    refs, recs = fx
    kw = VARIANTS[variant]
    from bamutil import make_bam_indexed
    bam_b, bai_b = make_bam_indexed(refs, recs)
    if kw.get("merged"):
        bai_b = rb.htslib_merged(bai_b, kw.get("min_dist", rb.MIN_MARKER_DIST))
    p = tmp_path / "q.bam"
    p.write_bytes(bam_b)
    (tmp_path / "q.bam.bai").write_bytes(bai_b)
    return str(p), bai_b


def _queries(fx, seed):
    refs, recs = fx
    rng = np.random.default_rng(seed)
    for tid, (nm, L) in enumerate(refs):
        sets = rb.interval_sets(rng, L)
        sets["gaps"] = rb.gap_intervals(recs, tid, L)
        sets["gaps_and_reads"] = sets["gaps"] + sets["single"]
        for name, iv in sets.items():
            yield tid, name, iv


def _chunks(b, tid, iv):
    from goleft_b200 import capi
    vb, ve = capi.bam_region_chunks(b, tid, [x[0] for x in iv], [x[1] for x in iv])
    return list(zip(vb.tolist(), ve.tolist()))


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_planner_equals_restatement(tmp_path, fx, variant):
    from goleft_b200 import capi
    p, bai = _write(tmp_path, fx, variant)
    idx, _ = rb.read_bai(bai)
    b = capi.Bam(p)
    n_nonempty = 0
    for tid, name, iv in _queries(fx, 3):
        got = _chunks(b, tid, iv)
        assert got == rb.plan(idx[tid][0], idx[tid][2], iv), (variant, tid, name)
        n_nonempty += bool(got)
    assert n_nonempty > 10
    b.close()


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_ranges_hold_every_overlapping_record(tmp_path, fx, variant):
    """sorted, disjoint, not touching; every record of tid overlapping an interval lies inside one range, for intervals in
    read-free gaps, past the contig and past the linear index too; empty intervals read nothing"""
    from goleft_b200 import capi
    refs, recs = fx
    p, _ = _write(tmp_path, fx, variant)
    voffs = rb.record_voffsets(refs, recs)
    b = capi.Bam(p)
    for tid, name, iv in _queries(fx, 4):
        got = _chunks(b, tid, iv)
        assert all(got[i][1] < got[i + 1][0] for i in range(len(got) - 1)) and all(x < y for x, y in got), (tid, name)
        starts = np.array([x for x, _ in got], np.uint64)
        for rec, (v0, v1) in zip(recs, voffs):
            if rec[0] != tid:
                continue
            s, e = rb.record_span(rec)
            if not any(s < y and e > x for x, y in iv if y > x):
                continue
            k = int(np.searchsorted(starts, np.uint64(v0), "right")) - 1
            assert k >= 0 and got[k][0] <= v0 and v1 <= got[k][1], (variant, tid, name, rec[:4])
        if name in ("none", "only_empty"):
            assert got == [], (variant, tid, name)
    b.close()


def test_whole_reference_query_covers_the_index_range(tmp_path, fx):
    """[0, len) reads exactly the reference's records: one range from its first chunk to its last"""
    from goleft_b200 import capi
    refs, recs = fx
    p, bai = _write(tmp_path, fx, "htslib")
    voffs = rb.record_voffsets(refs, recs)
    b = capi.Bam(p)
    for tid, (nm, L) in enumerate(refs):
        got = _chunks(b, tid, [(0, L)])
        mine = [v for r, v in zip(recs, voffs) if r[0] == tid]
        if not mine:
            assert got == []
            continue
        assert got[0][0] == mine[0][0] and got[-1][1] == mine[-1][1]
    b.close()


def test_region_chunks_arguments(tmp_path, fx):
    from goleft_b200 import capi
    p, _ = _write(tmp_path, fx, "plain")
    b = capi.Bam(p)
    for tid in (-1, len(fx[0])):
        with pytest.raises(capi.GlError) as e:
            capi.bam_region_chunks(b, tid, [0], [100])
        assert e.value.code == capi.GL_EINVAL
    n = capi.C.c_int64(0)
    assert capi.lib.gl_bam_region_chunks(b.h, 0, None, None, -1, None, None, 0, capi.C.byref(n)) == capi.GL_EINVAL
    assert capi.lib.gl_bam_region_chunks(b.h, 0, None, None, 3, None, None, 0, capi.C.byref(n)) == capi.GL_EINVAL
    assert capi.lib.gl_bam_region_chunks(None, 0, None, None, 0, None, None, 0, capi.C.byref(n)) == capi.GL_EINVAL
    vb, ve = capi.bam_region_chunks(b, 0, [], [])
    assert vb.size == 0 and ve.size == 0
    b.close()
    u = tmp_path / "u.bam"                                               # no index next to it
    u.write_bytes(make_bam(fx[0], fx[1]))
    bu = capi.Bam(str(u))
    with pytest.raises(capi.GlError) as e:
        capi.bam_region_chunks(bu, 0, [0], [100])
    assert e.value.code == capi.GL_ESTATE
    bu.close()
