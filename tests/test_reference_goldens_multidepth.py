"""`goleft multidepth` against the REAL reference (multidepth/multidepth.go + samtools >= 1.13) when its outputs exist.

tools/make_reference_goldens.sh writes tests/golden/ref_multidepth_t_<chrom>.txt (multidepth -Q 1 -p 1 --minsamples 0 on depth/test/t.bam: one sample, so any sufficient site needs minSamples = 0)
on a box with `go` and `samtools`; without them these tests SKIP LOUDLY.  Input: the committed decoded fixture
tests/golden/t_bam_segments.npz.  The rows after the header line are compared (the header holds the sample name)."""
import glob
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")
REF_FILES = sorted(glob.glob(os.path.join(GOLD, "ref_multidepth_t_*.txt")))
SKIP = ("multidepth reference goldens absent: run tools/make_reference_goldens.sh on a box with go + samtools >= 1.13 "
        "(multidepth parity stays 'unpinned' until then)")


def _segments(chrom):
    z = np.load(os.path.join(GOLD, "t_bam_segments.npz"), allow_pickle=True)
    names = [str(n) for n in z["ref_names"]]
    tid = names.index(chrom)
    s = z["start_%d" % tid] if "start_%d" % tid in z else np.zeros(0, np.int32)
    e = z["end_%d" % tid] if "end_%d" % tid in z else np.zeros(0, np.int32)
    return int(z["ref_lens"][tid]), np.asarray(s, np.int32), np.asarray(e, np.int32)


def _rows(path):
    return open(path, "rb").read().split(b"\n", 1)[1]


def _chrom(path):
    return os.path.basename(path)[len("ref_multidepth_t_"):-len(".txt")]


@pytest.mark.skipif(not REF_FILES, reason=SKIP)
@pytest.mark.parametrize("path", REF_FILES or ["absent"])
def test_oracle_equals_reference_multidepth(path):
    from oracle import loader as orc
    from oracle import multidepth as omd
    c = _chrom(path)
    L, s, e = _segments(c)
    rows, _ = omd.text(c, orc.pileup_diff(s, e, 0, L)[None, :], min_samples=0)
    assert rows == _rows(path)


@pytest.mark.gpu
@pytest.mark.skipif(not REF_FILES, reason=SKIP)
@pytest.mark.parametrize("path", REF_FILES or ["absent"])
def test_gpu_equals_reference_multidepth(ctx, path):
    c = _chrom(path)
    L, s, e = _segments(c)
    got = ctx.multidepth(c, L, [lambda x: x.depth_add_segments(s, e)], min_samples=0)
    assert got == _rows(path)
