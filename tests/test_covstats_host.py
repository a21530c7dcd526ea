"""CPU tests of covstats in the library: gl_covstats_tail (covstats.go:175-218) against the C oracle and a numpy restatement,
and gl_bam_covstats_host's counters and samples against the loop restated in Python.  Both entries take a NULL context here,
so no device is touched: the order statistics then come from sorted arrays instead of device histograms."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import covstats_ref as cr  # noqa: E402
from goleft_b200 import capi  # noqa: E402
from oracle import loader as orc  # noqa: E402


def bits(x):
    return np.float64(x).tobytes()


def check_tail(sizes, ins, tm, counters=None):
    c = dict(n_unmapped=3, k=1000, n_bad=17, n_dup=5, n_proper=800)
    c.update(counters or {})
    st, H = capi.covstats_tail(None, sizes, ins, tm, c["n_unmapped"], c["k"], c["n_bad"], c["n_dup"], c["n_proper"])
    exp, eH = cr.stats_numpy(c, np.asarray(sizes), np.asarray(ins), np.asarray(tm))
    for k, v in exp.items():
        assert bits(getattr(st, k)) == bits(v), (k, getattr(st, k), v)
    assert st.h_len == len(eH) == len(H) and H.tobytes() == eH.tobytes()
    if len(ins) and len(H) < (1 << 16):
        out6, oH = orc.cs_tail(ins, tm, st.max_read_length)
        got6 = [st.insert_pct5, st.insert_pct95, st.insert_mean, st.insert_sd, st.template_mean, st.template_sd]
        assert [bits(a) for a in got6] == [bits(b) for b in out6]
        assert oH.tobytes() == H.tobytes()
    return st, H


def test_tail_random():
    rng = np.random.default_rng(1)
    for n in (3, 4, 5, 100, 5001):
        ins = rng.normal(350, 40, n).astype(np.int32)
        ins[rng.random(n) < 0.02] = 50000
        check_tail(rng.choice([100, 101, 151], 2 * n), ins, ins + 200)


def test_tail_adversarial():
    rng = np.random.default_rng(2)
    check_tail([100, 100, 150, 150], [300, 300, 300, 400, 400, 400], [500, 500, 500, 600, 600, 600])      # ties at the median
    check_tail([100] * 9, [321] * 50, [521] * 50)                                                         # every insert equal
    st, H = check_tail([1000] * 5, [300] * 20, [0] * 10 + [900] * 10)                                      # H exists, nothing in range
    assert st.h_len > 0 and np.isnan(H).all()
    wide = rng.integers(-(1 << 30), 1 << 30, 4000).astype(np.int32)                                        # wider than 2^22
    check_tail(rng.integers(50, 250, 100), wide, np.abs(wide) // 4096 + 300)
    check_tail([151] * 7, [10, 20, 30], [210, 220, 230])                                                   # 3 inserts
    check_tail([], [], [])
    check_tail([100, 200], [], [])


def test_tail_panics():
    with pytest.raises(capi.GlError) as e:                                                                 # 2 inserts: madFilter's index
        capi.covstats_tail(None, [100] * 4, [300, 310], [500, 510])
    assert e.value.code == capi.GL_EINVAL and e.value.stats.n_insert == 2
    with pytest.raises(capi.GlError) as e:                                                                 # negative H length: makeslice
        capi.covstats_tail(None, [5000] * 4, [300] * 10, [500] * 10)
    assert e.value.code == capi.GL_ERANGE and "negative length" in str(e.value)


def test_tail_h_cap_two_call():
    import ctypes as C
    st = capi.CovStats()
    a = np.full(10, 100, np.int32)
    b = np.arange(300, 340, dtype=np.int32)
    rc = capi.lib.gl_covstats_tail(None, capi._ptr(a), a.size, capi._ptr(b), b.size, capi._ptr(b), b.size, C.byref(st), None, 0)
    assert rc == capi.GL_ERANGE and st.h_len > 0


CASES = {"cut_a": (40, 2000), "cut_b_none": (30, 500), "eof_sampling": (10 ** 6, 1000), "eof_skip": (10, 10 ** 6), "n0": (0, 10), "skip0": (25, 0)}


@pytest.mark.parametrize("case", sorted(CASES))
def test_host_sampler_equals_restatement(tmp_path, case):
    n, skip = CASES[case]
    rng = np.random.default_rng(7)
    flags = [0, 16, 0x400, 0x4 | 0x1] if case == "cut_b_none" else cr.FLAGS
    refs, recs, mates = cr.records(rng, [6000, 0, 3000], flags=flags, unplaced=50, cg_every=97)
    bam = capi.Bam(cr.write(tmp_path, "a.bam", refs, recs, mates, block=3000))
    try:
        c, arrs = cr.restate(recs, mates, n, skip)
        try:
            st, H, got = capi.bam_covstats_host(None, bam, n, skip, samples=True)
        except capi.GlError as e:                                          # 1 or 2 inserts: the counters still stand
            assert e.code == capi.GL_EINVAL and 0 < c["n_insert"] < 3
            st = e.stats
        else:
            for a, b in zip(got, arrs):
                assert np.array_equal(a, b)
            exp, eH = cr.stats_numpy(c, *arrs)
            for k, v in exp.items():
                assert bits(getattr(st, k)) == bits(v), k
            assert H.tobytes() == eH.tobytes()
        for k, v in c.items():
            assert getattr(st, k) == v, (k, getattr(st, k), v)
        assert st.path == 0
    finally:
        bam.close()
