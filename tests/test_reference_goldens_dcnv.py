"""`goleft dcnv` against the REAL reference (dcnv/dcnv.go built from the reference checkout) when its outputs exist.

tools/make_reference_goldens.sh writes, on a box with `go` and `samtools`:
  tests/golden/ref_dcnv_depthwed.bed     dcnv ref_depthwed.tsv hg19.fa   (the reference's depth/test/hg19.fa, copied as
                                         tests/golden/hg19.fa(.fai))
  tests/golden/ref_dcnv_ties.bed         dcnv on tests/golden/dcnv_ties.tsv: a generated, tie-heavy matrix of a few thousand
                                         rows on chrM / chr22, so that pdqsort's partition paths run
Without them these tests SKIP LOUDLY: pdqsort's tie order, the even-count median and faidx's error behaviour stay
'unpinned' until then."""
import os
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
ROOT = os.path.dirname(HERE)
GOLEFT = os.path.join(ROOT, "bin", "goleft")
FASTA = os.path.join(GOLD, "hg19.fa")
CASES = [("ref_depthwed.tsv", "ref_dcnv_depthwed.bed"), ("dcnv_ties.tsv", "ref_dcnv_ties.bed")]
PRESENT = [c for c in CASES if all(os.path.exists(os.path.join(GOLD, f)) for f in c)] if os.path.exists(FASTA + ".fai") else []
SKIP = ("dcnv reference goldens absent: run tools/make_reference_goldens.sh on a box with go + samtools "
        "(dcnv parity stays 'unpinned' until then)")


def _read(name):
    return open(os.path.join(GOLD, name), "rb").read()


@pytest.mark.skipif(not PRESENT, reason=SKIP)
@pytest.mark.parametrize("case", PRESENT or [("absent", "absent")])
def test_oracle_equals_reference_dcnv(case):
    from oracle import dcnv as od
    assert od.dcnv(_read(case[0]), _read("hg19.fa"), _read("hg19.fa.fai").decode()) == _read(case[1])


@pytest.mark.gpu
@pytest.mark.skipif(not PRESENT, reason=SKIP)
@pytest.mark.parametrize("case", PRESENT or [("absent", "absent")])
def test_cli_equals_reference_dcnv(case, tmp_path):
    p = subprocess.run([GOLEFT, "dcnv", os.path.join(GOLD, case[0]), FASTA], capture_output=True, cwd=str(tmp_path))
    assert p.returncode == 0, p.stderr
    assert (tmp_path / "depth.bed").read_bytes() == _read(case[1])
