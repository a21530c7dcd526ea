"""samtools-written CSIs against the BAI of the same BAM (tests/golden/ref_csi_*, made by tools/make_reference_goldens.sh on
a box with samtools): the stats, n_no_coor and the rebuilt linear index agree with the BAI's, which never lies below it.
Every other CSI the tests read comes from tests/csi_bams.py; without these files parity with real CSIs is unverified, and
the tests say so as they skip.  No GPU needed."""
import glob
import os

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
CSIS = sorted(glob.glob(os.path.join(GOLD, "ref_csi_*.csi")))
SKIP = ("samtools-written CSI goldens absent: run tools/make_reference_goldens.sh on a box with samtools; the CSI reader is "
        "checked only against tests/csi_bams.py's writer until then")


def _bai_of(csi):
    base = os.path.basename(csi)
    stem = base.split(".")[0]
    return os.path.join(GOLD, stem + ".bam.bai")


@pytest.mark.skipif(not CSIS, reason=SKIP)
@pytest.mark.parametrize("csi", CSIS, ids=[os.path.basename(c) for c in CSIS])
def test_samtools_csi_agrees_with_its_bai(csi):
    from goleft_b200 import capi
    c, b = capi.bai_read(csi), capi.bai_read(_bai_of(csi))
    assert c["is_csi"] and not b["is_csi"]
    assert c["mapped"] == b["mapped"] and c["unmapped"] == b["unmapped"] and c["has_stats"] == b["has_stats"]
    assert c["n_no_coor"] == b["n_no_coor"]
    for x, y in zip(c["ioffsets"], b["ioffsets"]):
        n = min(x.size, y.size)
        assert (x[:n] <= y[:n]).all() and (x[:n] != 0).all()


def test_csi_goldens_present_or_skipped_loudly():
    if not CSIS:
        pytest.skip(SKIP)
    assert all(os.path.exists(_bai_of(c)) for c in CSIS)
