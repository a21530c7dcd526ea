"""CPU tests: the indexcov / covstats / depthwed oracle against the reference's in-tree fixture and
against independent numpy restatements; and that libgoleft_b200.so exports every symbol the header declares."""
import json
import os
import re

import numpy as np
import pytest

from oracle import loader as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def fixture():
    j = json.load(open(os.path.join(ROOT, "tests", "golden", "sample_issue_27_bai_linear_index.json")))
    refs = j["ioffsets"]
    voff = np.array([v for r in refs for v in r], np.uint64)
    ptr = np.concatenate([[0], np.cumsum([len(r) for r in refs])]).astype(np.int64)
    return voff, ptr, j


def test_fixture_sizes_and_median():
    """indexcov/test-data/sample_issue_27_0001.bam.bai: 180 refs, 493 linear-index entries -> 313 tiles over 18
    refs with >= 2 intervals, all deltas > 0, mapped 6,517,502 (SURVEY.md §4; restatement-derived pins)."""
    voff, ptr, j = fixture()
    assert len(j["ioffsets"]) == 180 and voff.size == 493 and j["mapped"] == 6517502 and j["unmapped"] == 0
    sizes, sptr = orc.ic_sizes(voff, ptr)
    assert sizes.size == 313
    assert int((np.diff(sptr) > 0).sum()) == 18
    assert (sizes > 0).all()
    med = orc.ic_median(sizes)
    assert med == 1484454039397
    # numpy restatement of Index.init (indexcov.go:96-124)
    s = np.sort(sizes)
    n98 = s[int(0.98 * s.size)]
    cum = np.cumsum(np.minimum(s, n98))
    idx = int(np.searchsorted(cum, cum[-1] // 2, side="right"))
    assert s[min(idx, s.size - 1)] == med


def test_fixture_depths_slots_counter():
    voff, ptr, _ = fixture()
    sizes, sptr = orc.ic_sizes(voff, ptr)
    med = orc.ic_median(sizes)
    d0 = orc.ic_normalize(sizes[sptr[0]:sptr[1]], float(med))
    assert ["%.3g" % x for x in d0] == ["1.27", "1.22", "1.3", "1.27", "1.33", "1", "1.34"]
    K = np.float32(46.66666793823242)
    slots = np.minimum((d0 * K + np.float32(0.5)).astype(np.int32), 69)
    assert slots.tolist() == [59, 57, 61, 59, 62, 47, 63]
    c = orc.ic_counts(d0)
    assert c.sum() == 7 and all(c[s] >= 1 for s in slots)
    dall = orc.ic_normalize(sizes, float(med))
    b = orc.ic_bins(dall, dall.size)
    assert b.tolist() == [312, 304, 6, 1]                 # out, low, hi, in  (SURVEY.md §4)
    roc = orc.ic_roc(orc.ic_counts(dall))
    assert roc[0] == 1.0 and (np.diff(roc) <= 0).all()


def test_normalize_double_rounding():
    """float32(float64(o)/median): one float64 division, then one rounding to float32"""
    rng = np.random.default_rng(0)
    s = rng.integers(0, 2 ** 42, 10000)
    med = 1484454039397.0
    exp = (s.astype(np.float64) / med).astype(np.float32)
    exp = np.minimum(exp, np.float32(50000))
    assert np.array_equal(orc.ic_normalize(s, med), exp)
    assert orc.ic_normalize(np.array([2 ** 62]), 3.0)[0] == np.float32(50000)


def test_median_edge_cases():
    assert orc.ic_median(np.array([5])) == 5
    assert orc.ic_median(np.zeros(10, np.int64)) == 0          # cumsum never exceeds 0: clamp to the last element
    assert orc.ic_median(np.array([1, 1, 1, 1000])) == 1000    # n=4: index int(0.98*4)=3, no cap
    assert orc.ic_median(np.array([1] * 100 + [10 ** 6])) == 1  # the 98th-percentile cap tames the outlier
    rng = np.random.default_rng(1)
    for n in [2, 3, 49, 50, 51, 1000]:
        s = rng.integers(0, 10 ** 12, n)
        ss = np.sort(s)
        n98 = ss[int(0.98 * n)]
        cum = np.cumsum(np.minimum(ss, n98))
        idx = min(int(np.searchsorted(cum, cum[-1] // 2, side="right")), n - 1)
        assert orc.ic_median(s) == ss[idx]


def test_xnorm_small_pinned():
    """normalizeAcrossSamples on a flat cohort: means of 1 leave interior values at 7/7 within float rounding"""
    S, T = 6, 12
    d = np.ones((S, T), np.float32)
    out = orc.ic_xnorm(d, np.full(S, T, np.int32))
    assert np.allclose(out, 1.0, atol=1e-6)
    d2 = np.ones((4, T), np.float32) * 3                        # fewer than 5 samples: untouched (indexcov.go:551)
    assert np.array_equal(orc.ic_xnorm(d2, np.full(4, T, np.int32)), d2)


def test_getcn():
    d = np.array([0, 0, 1.0, 1.1, 0.9, 1.0, 1.05, 0.95, 1.0, 1.0], np.float32)
    assert orc.ic_getcn(d) == pytest.approx(2.0, abs=0.21)
    assert orc.ic_getcn(np.zeros(5, np.float32)) == -0.1        # indexcov.go:986-988


def test_mad_filter_and_tail():
    rng = np.random.default_rng(2)
    ins = rng.normal(300, 30, 5000).astype(np.int32)
    ins[:5] = 100000                                            # outliers dropped by the 10-MAD filter
    tm = (ins + 150).astype(np.int32)
    out6, H = orc.cs_tail(ins, tm, 150)
    s = np.sort(ins)
    assert out6[0] == s[int(0.05 * (s.size - 1) + 0.5)] and out6[1] == s[int(0.95 * (s.size - 1) + 0.5)]
    assert 290 < out6[2] < 310 and 20 < out6[3] < 40
    assert abs(H.sum() - 1.0) < 1e-9


def test_depthwed_groups():
    # two chroms; 3 rows of width 100 then a short last row; aggregate to 200
    starts = np.array([0, 100, 200, 300, 0, 100], np.int32)
    ends = np.array([100, 200, 300, 350, 100, 150], np.int32)
    chrom = np.array([0, 0, 0, 0, 1, 1], np.int32)
    means = np.array([[1.4, 2.5, 3.49, 0.5, 10.0, 0.2], [0.0, 0.49, 0.5, 9.99, 1.0, 1.0]])
    s, e, c, out = orc.depthwed(means, starts, ends, chrom, 200)
    assert s.tolist() == [0, 200, 0] and e.tolist() == [200, 350, 150] and c.tolist() == [0, 0, 1]
    assert out.tolist() == [[1 + 3, 0 + 0], [3 + 1, 1 + 10], [10 + 0, 1 + 1]]
    s, e, c, out = orc.depthwed(means, starts, ends, chrom, 100)      # no aggregation
    assert out.shape == (6, 2) and out[:, 0].tolist() == [1, 3, 3, 1, 10, 0]


def test_crai_sizes_reference_test_vector():
    """the index embedded in indexcov/crai/crai_test.go:1030-1036 (TestSizes only prints it; these pins are
    restatement-derived): gaps are back-filled with the previous value then zeros, spans become whole tiles"""
    from goleft_b200 import capi
    rows = [(10000, 98379, 376975), (108293, 223811, 340259), (332008, 216930, 339687), (149775203, 134825, 357798),
            (149909940, 135166, 313541)]
    st, sp, by = zip(*rows)
    a = orc.crai_sizes(st, sp, by)
    assert a.size == 9157 and a[:6].tolist() == [383186] * 6 and a[6] == 152029
    assert a[-8:].tolist() == [231967] * 8 and int((a == 0).sum()) > 9000
    assert np.array_equal(capi.crai_make_sizes(st, sp, by), a)             # the product's host code agrees
    assert orc.crai_sizes([], [], []).size == 0


def test_crai_sizes_viral_fixture_and_random():
    from goleft_b200 import capi
    z = np.load(os.path.join(ROOT, "tests", "golden", "viral_crai_slices.npz"))
    total = 0
    for si in np.unique(z["seq"]):
        m = z["seq"] == si
        a = orc.crai_sizes(z["start"][m], z["span"][m], z["nbytes"][m])
        assert np.array_equal(capi.crai_make_sizes(z["start"][m], z["span"][m], z["nbytes"][m]), a)
        total += a.size
    assert total == 191442
    rng = np.random.default_rng(12)
    for _ in range(200):                                                    # long-read style overlapping slices
        n = int(rng.integers(1, 40))
        st = np.cumsum(rng.integers(1, 400000, n)).astype(np.int64)
        sp = rng.integers(1, 600000, n).astype(np.int64)
        by = rng.integers(1, 4_000_000, n).astype(np.int32)
        try:
            a = orc.crai_sizes(st, sp, by)
        except ValueError:
            with pytest.raises(capi.GlError):
                capi.crai_make_sizes(st, sp, by)
            continue
        assert np.array_equal(capi.crai_make_sizes(st, sp, by), a)


def test_library_exports_every_declared_symbol():
    """-m 'not gpu': the C-ABI library loads and exports every entry point include/goleft_b200.h declares."""
    from goleft_b200 import capi
    hdr = open(os.path.join(ROOT, "include", "goleft_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    names = set(re.findall(r"\b(gl_[a-z0-9_]+)\s*\(", hdr))
    assert len(names) > 40
    missing = [n for n in sorted(names) if not hasattr(capi.lib, n)]
    assert not missing, missing
    assert "sm_90a" in capi.version()


def test_no_cuda_device_fails_loudly():
    from goleft_b200 import capi
    if capi.device_count() > 0:
        pytest.skip("a GPU is present")
    with pytest.raises(capi.GlError) as ei:
        capi.Ctx(0)
    assert ei.value.code == capi.GL_ECUDA


def test_indexsplit_restatement_tiles_every_chromosome():
    """indexsplit/functional-tests.sh:33-36: the regions cover every chromosome exactly once (no gap, no overlap), also
    with heavy tiles (cut in up to 8 pieces), problematic regions (cut in 3) and an empty chromosome; the host chunker
    of the library (no GPU needed) prints the same lines as the oracle."""
    from goleft_b200 import capi
    rng = np.random.default_rng(1)
    names = ["1", "2", "X", "MT", "empty"]
    lens = [3_000_000, 2_000_000, 1_500_000, 16571, 5000]
    samples = []
    for k in range(6):
        per = []
        for r, L in enumerate(lens[:4]):
            n = max(0, L // 16384 - (k % 2 if r == 1 else 0))
            v = rng.lognormal(np.log(1.6e9), 0.25, n)
            if r == 0:
                v[50] *= 30
            per.append(v.astype(np.int64))
        samples.append(per)
    problems = [(0, 1_000_000, 1_100_000), (1, 5, 10)]
    for N in (5, 40, 1000):
        txt = orc.indexsplit(samples, names, lens, N, problems)
        rows = [ln.split("\t") for ln in txt.decode().splitlines()]
        for name, L in zip(names, lens):
            if N == 1000:
                break           # regions smaller than a tile: every tile is cut in pieces and indexsplit.go:159-165 emits
                                # overlapping rows near a chromosome's end — restated as is, only compared with the host code
            iv = [(int(r[1]), int(r[2])) for r in rows if r[0] == name]
            assert iv[0][0] == 0 and iv[-1][1] == L, (name, iv[:2], iv[-2:])
            assert all(a[1] == b[0] and a[0] < a[1] for a, b in zip(iv, iv[1:]))
        assert [r for r in rows if r[0] == "empty"] == [["empty", "0", "5000", "0.00", "0"]]
        if N >= 40:                                     # small enough regions: problematic tiles are cut in 3, the heavy tile in more
            assert any(r[4] == "3" for r in rows)
        if N == 1000:
            assert any(int(r[4]) > 3 for r in rows)
        sizes, ptr, out_ptr = capi.indexsplit_layout(samples, len(names))
        acc = np.zeros(int(out_ptr[-1]))
        R = len(names)
        for s in range(len(samples)):
            for r in range(R):
                a, b = ptr[s * (R + 1) + r], ptr[s * (R + 1) + r + 1]
                acc[out_ptr[r]:out_ptr[r] + (b - a)] += sizes[a:b].astype(np.float64) / 1e9
        assert capi.indexsplit_chunks(acc, out_ptr, names, lens, list(range(R)), N, problems) == txt
