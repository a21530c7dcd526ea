"""`goleft indexcov`'s PC columns against the REAL reference when its outputs exist.

tools/make_reference_goldens.sh writes, on a box with `go` and `samtools`:
  tests/golden/ref_indexcov_pca8.ped    the reference's indexcov --fai on the 8-sample cohort of make_pca_cohort.py
  tests/golden/ref_indexcov_pca4.ped    ... and on its 4-sample cohort (rank 3 after centring)
Without them these tests SKIP LOUDLY: the byte rule (Go's float -> uint8 conversion), gonum's sign choice and the constant
it prints for a rank-deficient column stay 'unpinned' until then (DESIGN §1.11)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
ROOT = os.path.dirname(HERE)
GOLEFT = os.path.join(ROOT, "bin", "goleft")
CASES = ["pca8", "pca4"]
PRESENT = [c for c in CASES if os.path.exists(os.path.join(GOLD, "ref_indexcov_%s.ped" % c))]
SKIP = ("indexcov PCA reference goldens absent: run tools/make_reference_goldens.sh on a box with go + samtools "
        "(the PC columns' byte rule, sign and rank-deficient constant stay 'unpinned' until then)")


def _rows(path):
    return [ln.split("\t") for ln in open(path).read().splitlines()]


@pytest.mark.gpu
@pytest.mark.skipif(not PRESENT, reason=SKIP)
@pytest.mark.parametrize("case", PRESENT or ["absent"])
def test_cli_pcs_equal_reference(case, tmp_path):
    subprocess.check_call([sys.executable, os.path.join(GOLD, "make_pca_cohort.py"), str(tmp_path / "c")])
    bais = sorted(str(tmp_path / "c" / case / f) for f in os.listdir(str(tmp_path / "c" / case)))
    p = subprocess.run([GOLEFT, "indexcov", "-d", str(tmp_path / case), "--fai", str(tmp_path / "c" / "g.fa.fai"), *bais],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    ref = _rows(os.path.join(GOLD, "ref_indexcov_%s.ped" % case))
    got = _rows(str(tmp_path / case / ("%s-indexcov.ped" % case)))
    assert got[0] == ref[0]                                              # the column layout, PC columns included
    pcs = [j for j, h in enumerate(ref[0]) if h.startswith("PC")]
    for a, b in zip(got[1:], ref[1:]):                                   # every non-PC column byte for byte
        assert [x for j, x in enumerate(a) if j not in pcs] == [x for j, x in enumerate(b) if j not in pcs]
    signs = []
    for j in pcs:
        g = [float(r[j]) for r in got[1:]]
        r = [float(x[j]) for x in ref[1:]]
        if case == "pca4" and j == pcs[-1]:
            assert len(set(r)) == 1                                      # rank-deficient: the reference prints a constant
            assert set(g) == {0.0}                                       # ... and this engine 0.00 (the rank rule)
            continue
        s = 1 if max(abs(x - y) for x, y in zip(g, r)) <= max(abs(x + y) for x, y in zip(g, r)) else -1
        assert max(abs(x - s * y) for x, y in zip(g, r)) <= 0.01 + 1e-9
        signs.append(s)
    print("%s: gonum's sign relative to the product's rule, per PC column: %s" % (case, signs))
