"""`goleft cnveval` against the REAL reference when its outputs exist.

tools/make_reference_goldens.sh writes, on a box with `go`:
  tests/golden/ref_cnveval_<case>_<mode>.txt   the reference's cnveval stdout on the sets of make_cnveval_sets.py
Without them these tests SKIP LOUDLY: Go's sort.Slice order inside ties stays 'unpinned' until then (DESIGN §1.12)."""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
ROOT = os.path.dirname(HERE)
GOLEFT = os.path.join(ROOT, "bin", "goleft")
sys.path.insert(0, GOLD)
from make_cnveval_sets import CASES, MODES, write  # noqa: E402

ALL = [(c, m) for c in CASES for m in MODES]
PRESENT = [cm for cm in ALL if os.path.exists(os.path.join(GOLD, "ref_cnveval_%s_%s.txt" % cm))]
SKIP = ("cnveval reference goldens absent: run tools/make_reference_goldens.sh on a box with go "
        "(Go's sort.Slice order inside ties stays 'unpinned' until then)")


def test_sets_are_deterministic(tmp_path):
    write(str(tmp_path / "a"))
    write(str(tmp_path / "b"))
    for c in CASES:
        for k in ("truth", "test"):
            assert (tmp_path / "a" / ("%s.%s.bed" % (c, k))).read_bytes() == (tmp_path / "b" / ("%s.%s.bed" % (c, k))).read_bytes()


@pytest.mark.gpu
@pytest.mark.skipif(not PRESENT, reason=SKIP)
@pytest.mark.parametrize("case,mode", PRESENT or [("absent", "absent")])
def test_cli_equals_reference(case, mode, tmp_path):
    write(str(tmp_path))
    p = subprocess.run([GOLEFT, "cnveval", *MODES[mode], str(tmp_path / (case + ".truth.bed")), str(tmp_path / (case + ".test.bed"))],
                       capture_output=True)
    assert p.returncode == 0, p.stderr
    assert p.stdout == open(os.path.join(GOLD, "ref_cnveval_%s_%s.txt" % (case, mode)), "rb").read()
