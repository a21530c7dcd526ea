"""The reference's own fixture depth/test/t.bam (as tests/golden/t_bam_segments.npz, see make_tbam_fixture.py)
through the oracle (CPU) and through the CUDA path (GPU), in the configurations of depth/functional-test.sh."""
import os
import sys

import numpy as np
import pytest

from goleft_b200 import capi
from oracle import loader as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
FAI_WINDOWS = [100, 1000000000, 55, 60, 71, 13, 2001]          # functional-test.sh:45-70
BED_WINDOWS = [10, 1000000, 50, 55, 60, 71, 13, 2002]          # functional-test.sh:73-97
WINDOWS_BED = [("chr22", 14250, 15500), ("chr22", 1575, 15800), ("chrM", 100, 1000), ("chrM", 2000, 5000), ("chrM", 1, 3),
               ("chrM", 9, 13), ("chrM", 16, 17), ("chrM", 24, 29), ("chrM", 39, 43)]   # depth/test/windows.bed


def load():
    z = np.load(os.path.join(ROOT, "tests", "golden", "t_bam_segments.npz"))
    refs = list(zip([str(x) for x in z["ref_names"]], [int(x) for x in z["ref_lens"]]))
    segs = {i: (z["start_%d" % i], z["end_%d" % i]) for i in range(len(refs))}
    return refs, segs, int(z["n_records"]), int(z["n_pass"])


def rows(b):
    return [ln.split("\t") for ln in b.decode().splitlines()]


def oracle_fai(refs, segs, W):
    hd, ca = b"", b""
    for tid, (name, L) in enumerate(refs):
        s, e = segs[tid]
        depth = orc.pileup_brute(s, e, 0, L)
        for cs, ce in orc.gen_chunks(L, W):
            h, c = orc.walk_chunk(name, cs, ce, W, 4, 0, depth[cs:ce])
            hd += h; ca += c
    return hd, ca


def test_fixture_facts():
    """SURVEY.md §4 (derived there with an independent throw-away reader): record / pass counts, covered bases,
    total and maximum depth per contig at -Q 1."""
    refs, segs, nrec, npass = load()
    assert refs == [("chrM", 16571), ("chr22", 20001)] and nrec == 80330 and npass == 75808 + 246
    d = orc.pileup_brute(*segs[0], 0, 16571)
    assert (int((d > 0).sum()), int(d.sum()), int(d.max())) == (5076, 5743876, 2012)
    d = orc.pileup_brute(*segs[1], 0, 20001)
    assert (int((d > 0).sum()), int(d.sum()), int(d.max())) == (9811, 23813, 39)


@pytest.mark.parametrize("W", FAI_WINDOWS)
def test_oracle_fai_mode_invariants(W):
    refs, segs, _, _ = load()
    hd, ca = oracle_fai(refs, segs, W)
    for text in (hd, ca):                                   # check_with_fai_bt + check_uniq (functional-test.sh:10-39)
        r = rows(text)
        assert len({tuple(x) for x in r}) == len(r) and len({tuple(x[:3]) for x in r}) == len(r)
        for name, L in refs:
            rr = [x for x in r if x[0] == name]
            assert int(rr[0][1]) == 0 and int(rr[-1][2]) == L
            assert all(a[2] == b[1] for a, b in zip(rr, rr[1:]))
    if W == 100:
        assert len(rows(hd)) == 367 and len(rows(ca)) == 148
        assert [x[3] for x in rows(hd)[:8]] == ["608.2", "1101", "625.5", "457.4", "789.3", "897.3", "1583", "1801"]


def test_oracle_w250_row_counts():
    refs, segs, _, _ = load()
    hd, ca = oracle_fai(refs, segs, 250)                    # the depth default window (depth.go:164)
    assert len(rows(hd)) == 148 and len(rows(ca)) == 148


# ------------------------------------------------------------------ the feeder on a BAM written here
import bamref  # noqa: E402
from bamutil import cg_mix_records, cigar_lens, make_bam as _bam, make_bam_indexed  # noqa: E402


def _feeder_records(cg=False):
    """(refs, records).  cg: the unplaced reads move to the end (so the BAM can be indexed) and a third reference holds
    ultra-long reads stored through CG, short reads, and the CG edge cases (bamutil.cg_mix_records)."""
    rng = np.random.default_rng(0)
    refs = [("chrA", 100000), ("HLA-A*01:01:01:01", 5000)]
    recs = []
    pos = 0
    for i in range(30000):
        tid = 0 if i < 25000 else 1
        if i == 25000:
            pos = 0
        pos += int(rng.integers(0, 4)) if tid == 0 else int(rng.integers(0, 2)) % 2
        flag = int(rng.choice([0, 16, 0x400, 0x100, 0x200, 0x4, 0x800, 99]))
        mapq = int(rng.choice([0, 1, 30, 60]))
        kind = int(rng.integers(0, 6))
        cigar = [[(100, "M")], [(40, "M"), (5, "D"), (60, "M")], [(30, "M"), (3, "I"), (67, "M")], [(10, "S"), (90, "M")],
                 [(50, "="), (1, "X"), (20, "N"), (49, "M")], [(5, "H"), (20, "M"), (2, "P"), (30, "M"), (1000, "N"), (50, "M")]][kind]
        recs.append((tid if not (flag & 4) else -1, pos, mapq, flag, cigar))
    if cg:
        long_recs, end = cg_mix_records(np.random.default_rng(7), 2)
        refs.append(("chrL", end + 1000))
        recs = [r for r in recs if r[0] >= 0] + long_recs + [r for r in recs if r[0] < 0]
    return refs, recs


def _check_segments(got_s, got_e, exp_s, exp_e, L, what):
    """the same blocks as bamref (as a multiset) and the same per-base depth"""
    assert bamref.same_multiset(got_s, got_e, exp_s, exp_e), what
    assert np.array_equal(bamref.pileup(got_s, got_e, 0, L), bamref.pileup(exp_s, exp_e, 0, L)), what


def test_feeder_on_synthetic_bam(tmp_path):
    refs, recs = _feeder_records()
    exp = bamref.segments(recs, len(refs), 1)
    p = tmp_path / "x.bam"
    p.write_bytes(_bam(refs, recs))
    for threads in (1, 4):
        r = capi.bam_segments(str(p), 1, threads)
        assert r["refs"] == refs and r["n_records"] == len(recs)
        for tid in (0, 1):
            assert r["segments"][tid][0].tolist() == exp[tid][0].tolist() and r["segments"][tid][1].tolist() == exp[tid][1].tolist()
    only = capi.bam_segments(str(p), 1, 2, only_tid=1)
    assert 0 not in only["segments"] and only["segments"][1][0].tolist() == exp[1][0].tolist()
    with pytest.raises(capi.GlError):
        capi.bam_segments(str(tmp_path / "missing.bam"))


def _cg_bam(tmp_path):
    refs, recs = _feeder_records(cg=True)
    bam_b, bai_b = make_bam_indexed(refs, recs)
    p = tmp_path / "cg.bam"
    p.write_bytes(bam_b)
    (tmp_path / "cg.bam.bai").write_bytes(bai_b)
    return str(p), refs, recs


def test_stream_decoder_cg_reads(tmp_path):
    """bam_decode_segments (the whole-file decoder) on ultra-long reads whose CIGAR is in the CG tag, the CG edge cases and filtered
    placeholders, against bamref: the real CIGAR's blocks where htslib swaps it in, nothing where the placeholder stays"""
    p, refs, recs = _cg_bam(tmp_path)
    for q in (1, 30):
        exp = bamref.segments(recs, len(refs), q)
        assert exp[2][0].size > 100_000                               # the long reads do count
        for threads in (1, 4):
            r = capi.bam_segments(p, q, threads)
            assert r["n_records"] == len(recs)
            assert r["n_pass"] == sum(1 for rec in recs if bamref.passes(rec, q))
            for tid, (nm, L) in enumerate(refs):
                s, e = r["segments"].get(tid, (np.zeros(0, np.int32),) * 2)
                _check_segments(s, e, *exp[tid], L, (q, threads, nm))


def test_indexed_feeder_cg_reads(tmp_path):
    """Emitter::record (the index-guided host feeder) on the same BAM: whole references as packed8 and int32 words on 1, 3
    and all threads, and region queries whose ends cut through long CG reads"""
    p, refs, recs = _cg_bam(tmp_path)
    b = capi.Bam(p)
    exp = bamref.segments(recs, len(refs), 1)
    for tid, (nm, L) in enumerate(refs):
        n_rec = sum(1 for r in recs if r[0] == tid)
        n_pass = sum(1 for r in recs if r[0] == tid and bamref.passes(r, 1))
        es, ee = exp[tid]
        for threads in (1, 3, 0):
            d = b.decode(tid, threads=threads, want=8)
            assert d["format"] == 8 and d["n_records"] == n_rec and d["n_pass"] == n_pass
            us, ue = capi.unpack_segments8(d["anchors"], d["dstart"], d["len"])
            _check_segments(us, ue, *bamref.split255(es, ee), L, (nm, threads, 8))
            d = b.decode(tid, threads=threads, want=32)
            assert d["format"] == 32 and d["n_records"] == n_rec and d["n_pass"] == n_pass
            _check_segments(d.get("start", es[:0]), d.get("end", ee[:0]), es, ee, L, (nm, threads, 32))
    L = refs[2][1]
    longs = [r for r in recs if r[0] == 2 and len(r[4]) > 65535]
    regions = [(0, 1), (L - 500, L)]
    for r in longs[::5]:
        span = cigar_lens(r[4])[1]
        regions += [(r[1] + span // 3, r[1] + span // 3 + 777), (r[1] - 100, r[1] + span // 2), (r[1] + span - 1000, r[1] + span + 5000)]
    es, ee = exp[2]
    for rs, re in regions:
        rs, re = max(rs, 0), min(re, L)
        for want in (8, 32):
            d = b.decode(2, rs, re, want=want)
            if d["n"] == 0:
                s = e = np.zeros(0, np.int32)
            elif want == 8:
                s, e = capi.unpack_segments8(d["anchors"], d["dstart"], d["len"])
            else:
                s, e = d["start"], d["end"]
            assert np.array_equal(bamref.pileup(s, e, rs, re), bamref.pileup(es, ee, rs, re)), (rs, re, want)
    b.close()


# ------------------------------------------------------------------ GPU: the fixture through the CUDA path
@pytest.mark.gpu
@pytest.mark.parametrize("W", FAI_WINDOWS)
def test_gpu_fai_mode_text(ctx, W):
    refs, segs, _, _ = load()
    exp_hd, exp_ca = oracle_fai(refs, segs, W)
    hd, ca = b"", b""
    for tid, (name, L) in enumerate(refs):
        s, e = segs[tid]
        chunks = orc.gen_chunks(L, W)
        step = chunks[0][1] - chunks[0][0] if len(chunks) > 1 else 0
        ws, r0, rc = ctx.depth_region(0, L, s, e, W, 4, 0, run_break=step)
        for cs, ce in chunks:
            lo, hi = np.searchsorted(r0, cs), np.searchsorted(r0, ce)
            h, c = capi.format_chunk(name, cs, ce, W, ws[cs // W:(ce - 1) // W + 1], r0[lo:hi], rc[lo:hi])
            hd += h; ca += c
    assert hd == exp_hd and ca == exp_ca


@pytest.mark.gpu
@pytest.mark.parametrize("W", BED_WINDOWS)
def test_gpu_bed_mode_text(ctx, W):
    refs, segs, _, _ = load()
    tid_of = {n: i for i, (n, _) in enumerate(refs)}
    for name, rs, re in WINDOWS_BED:
        s, e = segs[tid_of[name]]
        depth = orc.pileup_brute(s, e, rs, re)
        exp = orc.walk_chunk(name, rs, re, W, 4, 0, depth)
        ws, r0, rc = ctx.depth_region(rs, re, s, e, W, 4, 0)
        assert capi.format_chunk(name, rs, re, W, ws, r0, rc) == exp


def test_indexed_feeder_equals_stream_decoder(tmp_path):
    """bam_feed (index-guided, parallel units, sorted emission) yields the same M/=/X blocks as the streaming decoder, as
    packed8 and as sorted int32, on a BGZF-realistic synthetic BAM; region queries return every block that can overlap"""
    import os, sys
    ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
    import glsynth
    from goleft_b200 import capi
    from oracle import loader as orc
    contigs = [("chrA", 3_000_000, 1), ("chrB", 700_000, 2), ("chrM", 16_569, 24)]
    bam = str(tmp_path / "t.bam")
    glsynth.write_bam(bam, contigs, coverage=20.0)
    old = capi.bam_segments(bam, 1, 4)
    b = capi.Bam(bam)
    assert b.has_index and [r[0] for r in b.refs] == [c[0] for c in contigs]
    for tid, (nm, L, idx) in enumerate(contigs):
        s, e = glsynth.segments(L, idx, coverage=20.0)
        gs, ge = old["segments"][tid]
        assert np.array_equal(gs, s) and np.array_equal(ge, e)                  # the stream decoder's filter == the generator's
        o = np.lexsort((e, s))
        for threads in (1, 3, 0):
            d = b.decode(tid, threads=threads)
            assert d["format"] == 8 and (np.diff(d["anchors"]) >= 0).all()
            us, ue = capi.unpack_segments8(d["anchors"], d["dstart"], d["len"])
            o2 = np.lexsort((ue, us))
            assert np.array_equal(us[o2], s[o]) and np.array_equal(ue[o2], e[o])
            d = b.decode(tid, threads=threads, want=32)
            assert (np.diff(d["start"]) >= 0).all()
            o3 = np.lexsort((d["end"], d["start"]))
            assert np.array_equal(d["start"][o3], s[o]) and np.array_equal(d["end"][o3], e[o])
    s, e = glsynth.segments(3_000_000, 1, coverage=20.0)
    for rs, re in ((0, 1), (1_000_000, 1_000_001), (1_234_567, 1_300_000), (2_990_000, 3_000_000), (16_383, 16_385)):
        d = b.decode(0, rs, re, want=32)
        got = orc.pileup_diff(d["start"], d["end"], rs, re) if d["n"] else np.zeros(re - rs, np.int32)
        assert np.array_equal(got, orc.pileup_diff(s, e, rs, re))
        assert d["n_records"] < 400_000 * (re - rs + 40_000) / 3_000_000 + 20_000     # only the region's blocks were parsed
    b.close()


def test_stream_decoder_across_read_chunks(tmp_path):
    """the whole-file decoder on an unindexed BAM larger than one 32 MiB read: members cut by a chunk's end are read again
    and records cut by it are carried over, so every reference's blocks equal the generator's, in record order"""
    sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
    import glsynth
    contigs = [("chrA", 4_000_000, 1), ("chrB", 700_000, 2), ("chrM", 16_569, 24)]
    bam = str(tmp_path / "t.bam")
    glsynth.write_bam(bam, contigs, coverage=20.0)
    os.remove(bam + ".bai")
    assert os.path.getsize(bam) > 36 << 20
    exp = [glsynth.segments(L, idx, coverage=20.0) for _, L, idx in contigs]
    for threads in (1, 4):
        r = capi.bam_segments(bam, 1, threads)
        assert [n for n, _ in r["refs"]] == [c[0] for c in contigs]
        for tid, (s, e) in enumerate(exp):
            gs, ge = r["segments"][tid]
            assert np.array_equal(gs, s) and np.array_equal(ge, e), (threads, tid)
    only = capi.bam_segments(bam, 1, 4, only_tid=1)
    assert list(only["segments"]) == [1] and only["n_records"] == r["n_records"] and only["n_pass"] < r["n_pass"]
    assert np.array_equal(only["segments"][1][0], exp[1][0]) and np.array_equal(only["segments"][1][1], exp[1][1])
