"""gl_bam_decode_device_regions: a BAM region query decoded on the device from only the BGZF members the index's bins name.
Its blocks equal bamref's blocks that meet the intervals, as an exact sequence in BAM order, on plain and htslib-style
merged BAIs, for MAPQ 0, 1 and 20; [0, len) equals gl_bam_decode_device; a one-tile query reads a small share of the file;
edge cases return the documented status."""
import os
import struct
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bamref  # noqa: E402
import region_bams as rb  # noqa: E402
from bamutil import make_bam, make_bam_indexed  # noqa: E402


@pytest.fixture(scope="module")
def fx():
    return rb.fixture()


def _write(tmp_path, fx, merged):
    refs, recs = fx
    bam_b, bai_b = make_bam_indexed(refs, recs)
    if merged:
        bai_b = rb.htslib_merged(bai_b)
    p = tmp_path / "q.bam"
    p.write_bytes(bam_b)
    (tmp_path / "q.bam.bai").write_bytes(bai_b)
    return str(p)


def _regions(ctx, b, tid, iv, q):
    from goleft_b200 import capi
    return capi.bam_decode_device_regions(ctx, b, tid, [x[0] for x in iv], [x[1] for x in iv], min_mapq=q)


@pytest.mark.parametrize("merged", [False, True], ids=["plain_bai", "htslib_bai"])
@pytest.mark.parametrize("q", [0, 1, 20])
def test_regions_equal_bamref(ctx, tmp_path, fx, merged, q):
    from goleft_b200 import capi
    refs, recs = fx
    b = capi.Bam(_write(tmp_path, fx, merged))
    segs = bamref.segments(recs, len(refs), q)
    rng = np.random.default_rng(q + 10 * merged)
    n_checked = 0
    for tid, (nm, L) in enumerate(refs):
        sets = rb.interval_sets(rng, L)
        sets["gaps"] = rb.gap_intervals(recs, tid, L)
        for name, iv in sets.items():
            d = _regions(ctx, b, tid, iv, q)
            es, ee = rb.expected_blocks(segs, tid, iv)
            assert np.array_equal(d["start"], es) and np.array_equal(d["end"], ee), (nm, name, d["n"], es.size)
            assert d["n"] == es.size and (es.size == 0 or d["max_len"] == int((ee - es).max()))
            n_checked += es.size
    assert n_checked > 20_000
    b.close()


@pytest.mark.parametrize("merged", [False, True], ids=["plain_bai", "htslib_bai"])
def test_whole_interval_equals_whole_reference(ctx, tmp_path, fx, merged):
    from goleft_b200 import capi
    refs, recs = fx
    b = capi.Bam(_write(tmp_path, fx, merged))
    for q in (0, 1):
        for tid, (nm, L) in enumerate(refs):
            w = capi.bam_decode_device(ctx, b, tid, min_mapq=q)
            r = _regions(ctx, b, tid, [(0, L)], q)
            assert np.array_equal(r["start"], w["start"]) and np.array_equal(r["end"], w["end"]), nm
            assert r["n_records"] == w["n_records"] and r["n_pass"] == w["n_pass"]
    b.close()


def test_one_tile_reads_a_small_share(ctx, tmp_path):
    """a 16 KB tile of a multi-MB BAM: under 1/20 of the file is read, and the blocks equal the whole decode's blocks that
    meet the tile"""
    from goleft_b200 import capi
    sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
    import glsynth
    bam = str(tmp_path / "g.bam")
    glsynth.write_bam(bam, [("chrA", 3_000_000, 1), ("chrB", 400_000, 2)], coverage=15.0)
    size = os.path.getsize(bam)
    assert size > 4 << 20
    b = capi.Bam(bam)
    w = capi.bam_decode_device(ctx, b, 0)
    for k in (w["n"] // 10, w["n"] // 2, w["n"] * 9 // 10):              # tiles with reads
        a = int(w["start"][k]) // 16384 * 16384
        r = _regions(ctx, b, 0, [(a, a + 16384)], 1)
        m = rb.meets(w["start"], w["end"], [(a, a + 16384)])
        assert np.array_equal(r["start"], w["start"][m]) and np.array_equal(r["end"], w["end"][m])
        assert 0 < r["bytes_in"] < size / 20 and r["n_records"] < w["n_records"] / 20, (a, r["bytes_in"], size)
    b.close()


def test_edge_cases(ctx, tmp_path, fx):
    from goleft_b200 import capi
    refs, recs = fx
    b = capi.Bam(_write(tmp_path, fx, True))
    assert _regions(ctx, b, 3, [(0, 50_000)], 1)["n"] == 0                     # chrE: no reads
    assert _regions(ctx, b, 0, [], 1)["n"] == 0
    for tid in (-1, len(refs)):
        with pytest.raises(capi.GlError) as e:
            _regions(ctx, b, tid, [(0, 100)], 1)
        assert e.value.code == capi.GL_EINVAL
    ps, pe, n = capi._vp(), capi._vp(), capi.C.c_int64(0)
    assert capi.lib.gl_bam_decode_device_regions(ctx.h, b.h, 0, None, None, -1, 1, capi.C.byref(ps), capi.C.byref(pe), capi.C.byref(n), None) == capi.GL_EINVAL
    assert capi.lib.gl_bam_decode_device_regions(ctx.h, b.h, 0, None, None, 2, 1, capi.C.byref(ps), capi.C.byref(pe), capi.C.byref(n), None) == capi.GL_EINVAL
    b.close()
    u = tmp_path / "u.bam"
    u.write_bytes(make_bam(refs, recs))
    bu = capi.Bam(str(u))
    with pytest.raises(capi.GlError) as e:
        _regions(ctx, bu, 0, [(0, 100)], 1)
    assert e.value.code == capi.GL_ESTATE
    bu.close()


def test_flagged_member_in_range_is_estate(ctx, tmp_path, fx):
    """a member whose ISIZE is wrong (the inflater flags it) inside the queried range gives GL_ESTATE; a query that does not
    reach that member still decodes"""
    from goleft_b200 import capi
    refs, recs = fx
    p = _write(tmp_path, fx, False)
    voffs = rb.record_voffsets(refs, recs)
    k = next(i for i, r in enumerate(recs) if r[0] == 0 and r[1] > 1_000_000)
    c = voffs[k][0] >> 16
    z = bytearray(open(p, "rb").read())
    bs = struct.unpack_from("<H", z, c + 16)[0] + 1
    isize = struct.unpack_from("<I", z, c + bs - 4)[0]
    struct.pack_into("<I", z, c + bs - 4, isize + 7)
    open(p, "wb").write(bytes(z))
    b = capi.Bam(p)
    with pytest.raises(capi.GlError) as e:
        _regions(ctx, b, 0, [(recs[k][1], recs[k][1] + 10)], 1)
    assert e.value.code == capi.GL_ESTATE
    segs = bamref.segments(recs, len(refs), 1)
    d = _regions(ctx, b, 0, [(1000, 1200)], 1)
    es, ee = rb.expected_blocks(segs, 0, [(1000, 1200)])
    assert np.array_equal(d["start"], es) and np.array_equal(d["end"], ee)
    b.close()


def test_alternating_calls_on_one_ctx(ctx, tmp_path, fx):
    """region and whole-reference calls on one ctx, sizes growing and shrinking: every call gives its own result"""
    from goleft_b200 import capi
    refs, recs = fx
    b = capi.Bam(_write(tmp_path, fx, True))
    segs = bamref.segments(recs, len(refs), 1)
    L = refs[0][1]
    plan = [("r", [(100_000, 100_500)]), ("w", 0), ("r", [(0, L)]), ("r", [(5, 6)]), ("w", 2), ("r", [(a, a + 3000) for a in range(0, L, 40_000)]),
            ("w", 0), ("r", [(1_000_000, 1_000_001)]), ("w", 1)]
    for kind, arg in plan * 2:
        if kind == "w":
            d = capi.bam_decode_device(ctx, b, arg)
            es, ee = segs[arg]
        else:
            d = _regions(ctx, b, 0, arg, 1)
            es, ee = rb.expected_blocks(segs, 0, arg)
        assert np.array_equal(d["start"], es) and np.array_equal(d["end"], ee), (kind, str(arg)[:40])
    b.close()
