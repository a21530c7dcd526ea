"""`goleft emdepth` against the REAL reference package (emdepth/emdepth.go driven by a small Go program) when its outputs
exist.

Expected under tests/golden/, written on a box with `go`:
  ref_emdepth_pow.txt        the seven math.Pow(i/2, 1.1) factors as Go prints their bits (%x of math.Float64bits)
  emdepth_cohort.tsv         a generated 9-sample matrix with planted CN1 / CN3 runs (ref_depthwed.tsv has 2 samples, where
                             the reference's median32 panics)
  ref_emdepth.cn.bed         the driver's P.cn.bed on emdepth_cohort.tsv
  ref_emdepth.cnv.bed        the driver's P.cnv.bed on emdepth_cohort.tsv
  ref_emdepth_gotest.txt     `go test ./emdepth`, whose TestBig fails (it expects CN 8 where the code gives 9)
Without them these tests SKIP LOUDLY: the Pow factors' last bits and the CPU-dependent Exp / Log decisions stay 'unpinned'
until then (DESIGN §1.10)."""
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
GOLEFT = os.path.join(os.path.dirname(HERE), "bin", "goleft")
POW = os.path.join(GOLD, "ref_emdepth_pow.txt")
FILES = [os.path.join(GOLD, f) for f in ("emdepth_cohort.tsv", "ref_emdepth.cn.bed", "ref_emdepth.cnv.bed")]
SKIP = ("emdepth reference goldens absent: run tools/make_reference_goldens.sh on a box with go "
        "(the Pow bits and the CPU-dependent Exp / Log decisions stay 'unpinned' until then)")


@pytest.mark.skipif(not os.path.exists(POW), reason=SKIP)
def test_pow_factors_are_go_bits():
    from goleft_b200 import capi
    want = [int(t, 16) for t in open(POW).read().split()]
    got = capi.emdepth_factors().view(np.uint64)
    assert [int(got[i]) for i in (1, 3, 4, 5, 6, 7, 8)] == want


GOTEST = os.path.join(GOLD, "ref_emdepth_gotest.txt")


@pytest.mark.skipif(not os.path.exists(GOTEST), reason=SKIP)
def test_reference_test_big_fails_as_restated():
    text = open(GOTEST).read()
    assert "TestBig" in text and "FAIL" in text and "[9 2 2 9 2 2 2 3 1]" in text


@pytest.mark.gpu
@pytest.mark.skipif(not all(os.path.exists(f) for f in FILES), reason=SKIP)
def test_cli_matches_reference(tmp_path):
    prefix = str(tmp_path / "o")
    p = subprocess.run([GOLEFT, "emdepth", "--prefix", prefix, FILES[0]], capture_output=True)
    assert p.returncode == 0, p.stderr
    assert open(prefix + ".cn.bed", "rb").read() == open(FILES[1], "rb").read()
    assert open(prefix + ".cnv.bed", "rb").read() == open(FILES[2], "rb").read()
