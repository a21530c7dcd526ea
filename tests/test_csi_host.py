"""CSI indexes on the host: the reader (stats, n_no_coor, the 16 KB linear index rebuilt from the bins' loffsets), its
errors, the region planner at a CSI's geometry, and the index lookup order.  The CSIs come from tests/csi_bams.py, written
from the CSIv1 spec; each is compared with the BAI of the same records.  No GPU needed."""
import os
import struct
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import csi_bams as cb  # noqa: E402
import region_bams as rb  # noqa: E402
from bamutil import _bgzf, make_bam  # noqa: E402

GEOMS = cb.GEOMETRIES


@pytest.fixture(scope="module")
def fx():
    return rb.fixture()


def _capi():
    from goleft_b200 import capi
    return capi


def _write(tmp_path, fx, geom, merged=False, trailer=True, name="q.bam"):
    refs, recs = fx
    bam, csi, bai = cb.make_bam_csi(refs, recs, *geom, trailer=trailer, merged=merged)
    p = tmp_path / name
    p.write_bytes(bam)
    (tmp_path / (name + ".csi")).write_bytes(csi)
    (tmp_path / "ref.bai").write_bytes(bai)
    return str(p), csi, bai


@pytest.mark.parametrize("trailer", [True, False])
@pytest.mark.parametrize("geom", GEOMS)
def test_reader_stats_against_bai(tmp_path, fx, geom, trailer):
    """mapped, unmapped, has_stats per reference and n_no_coor equal the BAI's; the geometry is the file's"""
    capi = _capi()
    p, _, _ = _write(tmp_path, fx, geom, trailer=trailer)
    c = capi.bai_read(p + ".csi")
    b = capi.bai_read(str(tmp_path / "ref.bai"))
    assert (c["min_shift"], c["depth"], c["is_csi"]) == (geom[0], geom[1], True)
    assert (b["min_shift"], b["depth"], b["is_csi"]) == (14, 5, False)
    assert c["mapped"] == b["mapped"] and c["unmapped"] == b["unmapped"] and c["has_stats"] == b["has_stats"]
    assert sum(b["mapped"]) > 0 and not b["has_stats"][3]                 # chrE has no reads and no stats bin
    assert b["n_no_coor"] == 1
    assert c["n_no_coor"] == (1 if trailer else 0)


@pytest.mark.parametrize("merged", [False, True])
@pytest.mark.parametrize("geom", GEOMS)
def test_linear_index_rebuild(tmp_path, fx, geom, merged):
    """ioffsets == the restatement; equal to the BAI's linear index at every 16 KB tile some bin starts in, never above it
    elsewhere"""
    capi = _capi()
    ms, depth = geom
    p, csi, bai = _write(tmp_path, fx, geom, merged=merged)
    got = capi.bai_read(p + ".csi")["ioffsets"]
    parsed = cb.read_csi(csi)
    bai_lin = [x[2] for x in rb.read_bai(bai)[0]]
    n_equal = 0
    for tid, R in enumerate(parsed["refs"]):
        exp = cb.rebuild_linear(R["loff"], ms, depth)
        assert got[tid].tolist() == exp, (geom, tid)
        starts = {cb.bin_first_tile(k, depth) for k, v in R["loff"].items() if v}
        if ms <= 14:
            s = 14 - ms
            at_starts = {x >> s for x in starts if x % (1 << s) == 0}
        else:
            at_starts = {x << (ms - 14) for x in starts}
        lin = bai_lin[tid]
        for t, v in enumerate(exp[:len(lin)]):
            assert v <= lin[t], (geom, tid, t)
            if t in at_starts:
                assert v == lin[t], (geom, tid, t)
                n_equal += 1
        assert all(v != 0 for v in exp)
    assert n_equal > 10


def test_rebuild_prefers_the_smallest_loffset_and_fills_gaps(tmp_path):
    """hand-made loffsets: two bins starting in one tile (the smaller wins), gaps on the left of the first known tile and
    between known tiles, a zero loffset that is ignored, and a bin whose first base lies past 2^31"""
    capi = _capi()
    ms, depth = 14, 6
    leaf = cb.first_of_level(depth)
    lvl5 = cb.first_of_level(5)
    loff = {leaf + 8: 900 << 16, lvl5 + 1: 700 << 16, leaf + 12: 1000 << 16, leaf + 3: 0, leaf + 20: 1500 << 16,
            leaf + (1 << 17) + 5: 99 << 16}
    idx = [dict(bins={k: [[v or 5, (v or 5) + 1]] for k, v in loff.items()}, loff=loff, beg=None, end=0, mapped=0, unmapped=0)]
    path = tmp_path / "h.csi"
    path.write_bytes(_bgzf(cb.write_csi(idx, 0, ms, depth)))
    got = capi.bai_read(str(path))["ioffsets"][0].tolist()
    exp = cb.rebuild_linear(loff, ms, depth)
    assert got == exp
    assert exp[:8] == [700 << 16] * 8 and exp[8] == 700 << 16 and exp[12] == 1000 << 16 and exp[13] == 1000 << 16
    assert exp[20] == 1500 << 16 and len(exp) == 21


def _corrupt_cases(fx):
    refs, recs = fx
    _, raw, _ = cb.make_bam_csi(refs[:2], [r for r in recs if 0 <= r[0] < 2] + [recs[-1]], 14, 6, raw=True)
    _, comp, _ = cb.make_bam_csi(refs[:2], [r for r in recs if 0 <= r[0] < 2] + [recs[-1]], 14, 6)
    n_ref_at = 16
    cases = {
        "cut_member": comp[:len(comp) // 2],
        "cut_header": comp[:10],
        "gzip_garbage": comp[:18] + b"\x00" * 40,
        "bad_magic": _bgzf(b"CSJ\x01" + raw[4:]),
        "short": _bgzf(raw[:12]),
        "neg_n_ref": _bgzf(raw[:n_ref_at] + struct.pack("<i", -1) + raw[n_ref_at + 4:]),
        "neg_l_aux": _bgzf(raw[:12] + struct.pack("<i", -5) + raw[16:]),
        "huge_l_aux": _bgzf(raw[:12] + struct.pack("<i", 1 << 30) + raw[16:]),
        "depth_11": _bgzf(raw[:8] + struct.pack("<i", 11) + raw[12:]),
        "neg_depth": _bgzf(raw[:8] + struct.pack("<i", -1) + raw[12:]),
        "neg_min_shift": _bgzf(raw[:4] + struct.pack("<i", -3) + raw[8:]),
        "positions_past_2^62": _bgzf(raw[:4] + struct.pack("<i", 40) + struct.pack("<i", 8) + raw[12:]),
        "not_an_index": b"hello world, not an index at all",
        "empty": b"",
    }
    n_bin = struct.unpack_from("<i", raw, n_ref_at + 4)[0]
    assert n_bin > 2
    first_bin = n_ref_at + 8                                              # bin, loffset, n_chunk of the first bin
    cases["neg_n_chunk"] = _bgzf(raw[:first_bin + 12] + struct.pack("<i", -2) + raw[first_bin + 16:])
    cases["n_chunk_overruns"] = _bgzf(raw[:first_bin + 12] + struct.pack("<i", 1 << 28) + raw[first_bin + 16:])
    cases["neg_n_bin"] = _bgzf(raw[:n_ref_at + 4] + struct.pack("<i", -7) + raw[n_ref_at + 8:])
    for cut in (n_ref_at + 2, first_bin + 5, first_bin + 15, first_bin + 30, len(raw) // 2, len(raw) - 40):
        cases["truncated_%d" % cut] = _bgzf(raw[:cut])
    return cases


def test_truncated_and_corrupt_csis_are_errors(tmp_path, fx):
    capi = _capi()
    for name, data in _corrupt_cases(fx).items():
        p = tmp_path / (name + ".csi")
        p.write_bytes(data)
        with pytest.raises(capi.GlError) as e:
            capi.bai_read(str(p))
        assert e.value.code == capi.GL_EINVAL, name
        assert str(p) in str(e.value), name


def test_tabix_aux_is_skipped(tmp_path, fx):
    """l_aux > 0 (a tabix header): read past; the result equals the same index without it"""
    capi = _capi()
    refs, recs = fx
    _, a, _ = cb.make_bam_csi(refs, recs, 14, 6)
    _, b, _ = cb.make_bam_csi(refs, recs, 14, 6, aux=struct.pack("<6i", 0, 1, 2, 3, 35, 0) + b"\x00" * 9)
    (tmp_path / "a.csi").write_bytes(a)
    (tmp_path / "b.csi").write_bytes(b)
    x, y = capi.bai_read(str(tmp_path / "a.csi")), capi.bai_read(str(tmp_path / "b.csi"))
    assert all(np.array_equal(u, v) for u, v in zip(x["ioffsets"], y["ioffsets"]))
    assert x["mapped"] == y["mapped"] and x["n_no_coor"] == y["n_no_coor"]


def _queries(fx, seed):
    refs, recs = fx
    rng = np.random.default_rng(seed)
    for tid, (nm, L) in enumerate(refs):
        sets = rb.interval_sets(rng, L)
        sets["gaps"] = rb.gap_intervals(recs, tid, L)
        sets["gaps_and_reads"] = sets["gaps"] + sets["single"]
        for name, iv in sets.items():
            yield tid, name, iv


def _chunks(capi, b, tid, iv):
    vb, ve = capi.bam_region_chunks(b, tid, [x[0] for x in iv], [x[1] for x in iv])
    return list(zip(vb.tolist(), ve.tolist()))


@pytest.mark.parametrize("merged", [False, True])
@pytest.mark.parametrize("geom", GEOMS)
def test_planner_on_csi(tmp_path, fx, geom, merged):
    """the ranges equal the restatement at the CSI's geometry; every record overlapping a query lies inside one range"""
    capi = _capi()
    ms, depth = geom
    refs, recs = fx
    p, csi, _ = _write(tmp_path, fx, geom, merged=merged)
    parsed = cb.read_csi(csi)
    voffs = rb.record_voffsets(refs, recs)
    b = capi.Bam(p)
    assert b.index_path == p + ".csi" and b.index_geometry == (ms, depth, True)
    lins = capi.bai_read(p + ".csi")["ioffsets"]
    n_nonempty = 0
    for tid, name, iv in _queries(fx, 3):
        got = _chunks(capi, b, tid, iv)
        assert got == cb.plan(parsed["refs"][tid]["bins"], lins[tid].tolist(), iv, ms, depth), (geom, merged, tid, name)
        n_nonempty += bool(got)
        starts = np.array([x for x, _ in got], np.uint64)
        for rec, (v0, v1) in zip(recs, voffs):
            if rec[0] != tid:
                continue
            s, e = rb.record_span(rec)
            if not any(s < y and e > x for x, y in iv if y > x):
                continue
            k = int(np.searchsorted(starts, np.uint64(v0), "right")) - 1
            assert k >= 0 and got[k][0] <= v0 and v1 <= got[k][1], (geom, merged, tid, name, rec[:4])
    assert n_nonempty > 10
    b.close()


def test_host_feeder_on_csi_equals_bai(tmp_path, fx):
    """the host feeder's blocks that meet the range, for whole references and for sub-ranges, are the same with either index
    (past the last tile a CSI bin starts in, its feeder starts at the last entry and may also give blocks that end before
    the range, which the depth reduce clamps away)"""
    capi = _capi()
    refs, recs = fx
    bam, csi, bai = cb.make_bam_csi(refs, recs, 12, 6)
    for d, idx in (("b", ("x.bam.bai", bai)), ("c", ("x.bam.csi", csi))):
        (tmp_path / d).mkdir()
        (tmp_path / d / "x.bam").write_bytes(bam)
        (tmp_path / d / idx[0]).write_bytes(idx[1])
    hb, hc = capi.Bam(str(tmp_path / "b" / "x.bam")), capi.Bam(str(tmp_path / "c" / "x.bam"))
    assert hc.index_geometry == (12, 6, True) and hb.index_geometry == (14, 5, False)
    n_blocks = 0
    for tid, (nm, L) in enumerate(refs):
        for beg, end in ((0, L), (L // 3, L // 2), (L - 20_000, L)):
            x, y = hb.decode(tid, beg, end, want=32), hc.decode(tid, beg, end, want=32)
            keep = [(u.get("start", np.zeros(0, np.int32)), u.get("end", np.zeros(0, np.int32))) for u in (x, y)]
            keep = [(s[(e > beg) & (s < end)], e[(e > beg) & (s < end)]) for s, e in keep]
            assert np.array_equal(keep[0][0], keep[1][0]) and np.array_equal(keep[0][1], keep[1][1]), (tid, beg, end)
            n_blocks += keep[0][0].size
    assert n_blocks > 1000
    hb.close(); hc.close()


def test_record_bin_field_is_not_read(tmp_path):
    """records past 2^29 keep a meaningless 16-bit bin field (make_bam writes 0); the host readers take pos, so any value
    there decodes to the same blocks"""
    capi = _capi()
    rng = np.random.default_rng(7)
    L = 2 ** 31 - 1
    pos = np.sort(np.concatenate([rng.integers(2 ** 29 - 5000, 2 ** 29 + 5000, 300), rng.integers(L - 10_000, L - 200, 100)]))
    recs = [(0, int(p), 60, 0, [(150, "M")]) for p in pos]
    refs = [("chrBig", L)]
    offs = []
    payload = bytearray(make_bam(refs, recs, _raw=True, _rec_off=offs))
    assert all(payload[a + 14:a + 16] == b"\x00\x00" for a, _ in offs)
    patched = bytearray(payload)
    for i, (a, _) in enumerate(offs):
        patched[a + 14:a + 16] = struct.pack("<H", [4681, 37449, 0xffff, 12345][i % 4])
    out = []
    for d, pl in (("zero", payload), ("patched", patched)):
        bam, voffs = cb.bgzf_with_voffsets(bytes(pl), offs)             # the two compress to different sizes
        idx, n_nc = cb.index_records(refs, recs, 14, 6, voffs=voffs)
        (tmp_path / d).mkdir()
        (tmp_path / d / "x.bam").write_bytes(bam)
        (tmp_path / d / "x.bam.csi").write_bytes(_bgzf(cb.write_csi(idx, n_nc, 14, 6)))
        h = capi.Bam(str(tmp_path / d / "x.bam"))
        out.append(h.decode(0, 0, L, want=32))
        out.append(capi.bam_segments(str(tmp_path / d / "x.bam"))["segments"][0])
        h.close()
    assert out[0]["n"] == len(recs)
    assert np.array_equal(out[0]["start"], out[2]["start"]) and np.array_equal(out[0]["end"], out[2]["end"])
    assert np.array_equal(out[1][0], out[3][0]) and np.array_equal(out[1][1], out[3][1])


def test_lookup_order(tmp_path, fx):
    """x.bam.bai, x.bai, x.bam.csi, x.csi: a BAI wins over a CSI, x.bam.csi over x.csi; an index that does not read is
    passed over"""
    capi = _capi()
    refs, recs = fx
    bam, csi, bai = cb.make_bam_csi(refs[:2], [r for r in recs if 0 <= r[0] < 2], 14, 6)
    _, csi16, _ = cb.make_bam_csi(refs[:2], [r for r in recs if 0 <= r[0] < 2], 16, 5, with_bai=False)
    cases = [
        ({"x.bam.bai": bai, "x.bam.csi": csi}, "x.bam.bai", False),
        ({"x.bai": bai, "x.csi": csi}, "x.bai", False),
        ({"x.bai": bai, "x.bam.csi": csi}, "x.bai", False),
        ({"x.bam.csi": csi, "x.csi": csi16}, "x.bam.csi", True),
        ({"x.csi": csi16}, "x.csi", True),
        ({"x.bam.bai": b"not an index", "x.csi": csi}, "x.csi", True),
        ({"x.bam.csi": csi[:30], "x.csi": csi16}, "x.csi", True),
        ({}, None, None),
    ]
    for i, (files, want, is_csi) in enumerate(cases):
        d = tmp_path / ("c%d" % i)
        d.mkdir()
        (d / "x.bam").write_bytes(bam)
        for n, data in files.items():
            (d / n).write_bytes(data)
        h = capi.Bam(str(d / "x.bam"))
        if want is None:
            assert not h.has_index and h.index_path is None
        else:
            assert h.has_index and h.index_path == str(d / want), (i, h.index_path)
            assert h.index_geometry[2] == is_csi
            assert h.refs[0][2] == sum(1 for r in recs if r[0] == 0 and not r[3] & 4)      # mapped, from the stats bin
        h.close()
