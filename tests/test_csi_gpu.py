"""The device decode on CSI-indexed BAMs: gl_bam_decode_device equals the same call with the BAI and bamref's blocks, and
gl_bam_decode_device_regions reads a contig of 2^31 - 1 bases, which no BAI can index: read clusters just below and above
2^29, around both of `goleft depth`'s pass edges at W = 100000 (1.07e9 and 2.14e9) and within a read length of the end.
Its blocks equal bamref's blocks that meet the query, as an exact sequence in BAM order, at MAPQ 0, 1 and 20.  Needs an
H100 (`-m gpu`)."""
import os
import struct
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bamref  # noqa: E402
import csi_bams as cb  # noqa: E402
import region_bams as rb  # noqa: E402
from bamutil import _bgzf, make_bam  # noqa: E402

TOP = 2 ** 31 - 1
PASS_EDGES = [1_070_000_000, 2_140_000_000]


@pytest.fixture(scope="module")
def fx():
    return rb.fixture()


def _pair(tmp_path, refs, recs, geom, merged=False):
    """(Bam with only the BAI, Bam with only the CSI) of one file"""
    from goleft_b200 import capi
    bam, csi, bai = cb.make_bam_csi(refs, recs, *geom, merged=merged)
    out = []
    for d, name, idx in (("b", "x.bam.bai", bai), ("c", "x.bam.csi", csi)):
        (tmp_path / d).mkdir()
        (tmp_path / d / "x.bam").write_bytes(bam)
        (tmp_path / d / name).write_bytes(idx)
        out.append(capi.Bam(str(tmp_path / d / "x.bam")))
    assert out[1].index_geometry == (geom[0], geom[1], True)
    return out


@pytest.mark.parametrize("geom", cb.GEOMETRIES)
def test_decode_device_csi_equals_bai_and_bamref(ctx, tmp_path, fx, geom):
    from goleft_b200 import capi
    refs, recs = fx
    hb, hc = _pair(tmp_path, refs, recs, geom, merged=geom == (14, 6))
    n = 0
    for q in (0, 1):
        segs = bamref.segments(recs, len(refs), q)
        for tid, (nm, L) in enumerate(refs):
            wb = capi.bam_decode_device(ctx, hb, tid, min_mapq=q)
            wc = capi.bam_decode_device(ctx, hc, tid, min_mapq=q)
            es, ee = rb.expected_blocks(segs, tid, [(0, L)])
            assert np.array_equal(wc["start"], wb["start"]) and np.array_equal(wc["end"], wb["end"]), (geom, nm)
            assert np.array_equal(wc["start"], es) and np.array_equal(wc["end"], ee), (geom, nm)
            assert wc["n_records"] == wb["n_records"] and wc["n_pass"] == wb["n_pass"]
            n += es.size
    assert n > 20_000
    hb.close(); hc.close()


def big_records(seed=41):
    """records of one 2^31-1 base contig: clusters around 2^29, both pass edges and the end (reads ending at INT32_MAX),
    sparse reads between them, D/N/S/I CIGARs, every MAPQ class and the flags the filter removes"""
    rng = np.random.default_rng(seed)
    L = TOP
    centres = [2 ** 29] + PASS_EDGES
    pos = [rng.integers(c - 4000, c + 4000, 500) for c in centres]
    pos.append(rng.integers(0, L - 1000, 400))
    pos.append(rng.integers(L - 2000, L - 300, 150))
    pos = np.sort(np.concatenate(pos))
    cigars = [[(150, "M")], [(45, "M"), (7, "D"), (55, "M")], [(12, "S"), (88, "M")], [(60, "M"), (300, "N"), (40, "M")],
              [(30, "M"), (2, "I"), (68, "M")], [(40, "M"), (20_000, "N"), (60, "M")]]
    recs = []
    for p0 in pos.tolist():
        cig = cigars[int(rng.integers(0, len(cigars)))]
        if p0 + 25_000 > L:
            cig = [(int(min(150, L - p0)), "M")]
        recs.append((0, p0, int(rng.choice([0, 1, 5, 20, 60, 60])), int(rng.choice([0, 16, 0, 0x400, 0x100, 4])), cig))
    for k in (150, 100, 1):                                    # reads that end exactly at INT32_MAX
        recs.append((0, L - k, 60, 0, [(k, "M")]))
    recs.sort(key=lambda r: r[1])
    return [("chrBig", L)], recs


def _queries():
    e0, e1 = PASS_EDGES
    return {
        "passes": [(0, e0), (e0, e1), (e1, TOP)],
        "pass_0": [(0, e0)],
        "pass_1": [(e0, e1)],
        "pass_2": [(e1, TOP)],
        "around_2^29": [(2 ** 29 - 2500, 2 ** 29 + 2500)],
        "below_2^29": [(2 ** 29 - 6000, 2 ** 29)],
        "above_2^29": [(2 ** 29, 2 ** 29 + 6000)],
        "pass_edges": [(e0 - 300, e0 + 300), (e1 - 1, e1 + 1)],
        "end": [(TOP - 150, TOP)],
        "last_base": [(TOP - 1, TOP)],
        "whole": [(0, TOP)],
        "past_end": [(TOP - 10, 2 ** 40)],
    }


@pytest.mark.parametrize("geom,merged", [((14, 6), False), ((14, 6), True), ((16, 5), False), ((12, 7), False)],
                         ids=["14-6", "14-6-merged", "16-5", "12-7"])
def test_regions_on_a_contig_of_int32_max_bases(ctx, tmp_path, geom, merged):
    from goleft_b200 import capi
    refs, recs = big_records()
    bam, csi, _ = cb.make_bam_csi(refs, recs, *geom, merged=merged, with_bai=False)
    (tmp_path / "x.bam").write_bytes(bam)
    (tmp_path / "x.bam.csi").write_bytes(csi)
    b = capi.Bam(str(tmp_path / "x.bam"))
    assert b.index_geometry == (geom[0], geom[1], True)
    n = 0
    for q in (0, 1, 20):
        segs = bamref.segments(recs, 1, q)
        assert int(segs[0][1].max()) == TOP and int(segs[0][0].max()) > 2 ** 31 - 200
        for name, iv in _queries().items():
            d = capi.bam_decode_device_regions(ctx, b, 0, [x[0] for x in iv], [x[1] for x in iv], min_mapq=q)
            es, ee = rb.expected_blocks(segs, 0, iv)
            assert np.array_equal(d["start"], es) and np.array_equal(d["end"], ee), (geom, q, name, d["n"], es.size)
            n += es.size
        w = capi.bam_decode_device(ctx, b, 0, min_mapq=q)
        assert np.array_equal(w["start"], segs[0][0]) and np.array_equal(w["end"], segs[0][1])
    assert n > 10_000
    b.close()


def test_record_bin_field_is_not_read_on_the_device(ctx, tmp_path):
    """the device parser takes pos: a BAM whose records hold arbitrary 16-bit bin fields decodes to the same blocks"""
    from goleft_b200 import capi
    refs, recs = big_records(seed=43)
    offs = []
    payload = bytearray(make_bam(refs, recs, _raw=True, _rec_off=offs))
    patched = bytearray(payload)
    for i, (a, _) in enumerate(offs):
        patched[a + 14:a + 16] = struct.pack("<H", [4681, 37449, 0xffff, 12345][i % 4])
    got = []
    for d, pl in (("zero", payload), ("patched", patched)):
        bam, voffs = cb.bgzf_with_voffsets(bytes(pl), offs)
        idx, n_nc = cb.index_records(refs, recs, 14, 6, voffs=voffs)
        (tmp_path / d).mkdir()
        (tmp_path / d / "x.bam").write_bytes(bam)
        (tmp_path / d / "x.bam.csi").write_bytes(_bgzf(cb.write_csi(idx, n_nc, 14, 6)))
        b = capi.Bam(str(tmp_path / d / "x.bam"))
        got.append(capi.bam_decode_device_regions(ctx, b, 0, [0, PASS_EDGES[1]], [PASS_EDGES[0], TOP], min_mapq=0))
        b.close()
    segs = bamref.segments(recs, 1, 0)
    es, ee = rb.expected_blocks(segs, 0, [(0, PASS_EDGES[0]), (PASS_EDGES[1], TOP)])
    for g in got:
        assert np.array_equal(g["start"], es) and np.array_equal(g["end"], ee)
