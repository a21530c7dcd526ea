"""`goleft dcnv --chunk W`, the parts that need no GPU: ChunkDebiaser's chunk boundaries (gl_dcnv_chunk_slices against a
Python restatement of debiaser.go:133-141), the C oracle's ChunkDebiaser against a numpy restatement, and the flag's
argument errors."""
import os
import subprocess

import numpy as np
import pytest

from goleft_b200 import capi
from oracle import dcnv_chunk as oc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLEFT = os.path.join(ROOT, "bin", "goleft")


def _slices(v, w):
    """debiaser.go:133-141, restated"""
    out, v0 = [0], v[0]
    for i in range(len(v)):
        if v[i] - v0 > w:
            v0 = v[i]
            out.append(i)
    return np.array(out + [len(v)], np.int64)


def _gc_cases(rng):
    yield np.sort(rng.random(1000)), 0.01                                  # distinct
    yield np.sort(rng.integers(0, 300, 5000) / 300.0), 0.01                # tie-heavy, like GC fractions of one window size
    yield np.full(77, 0.42), 1e-9                                          # all equal: one chunk
    yield np.arange(40) * 0.25, 0.25                                       # steps of exactly W (exact in binary): not a cut
    yield np.arange(40) * 0.1, 0.1                                         # steps of W in decimal: cuts by float64 rounding
    yield np.sort(rng.random(500)), 1.0                                    # W at the range
    yield np.sort(rng.random(500)), 5.0                                    # W above it
    yield np.sort(rng.random(300)), 1e-12                                  # every chunk one row
    yield np.array([0.5]), 0.1                                             # one row
    yield np.sort(rng.integers(0, 1000, 20000) / 1000.0), 0.001


def test_slices_match_restatement():
    rng = np.random.default_rng(1)
    for v, w in _gc_cases(rng):
        want = _slices(v, w)
        got = capi.dcnv_chunk_slices(v, w)
        assert np.array_equal(got, want), (v.size, w)
        assert np.array_equal(got, oc.chunk_slices(v, w))
    assert capi.dcnv_chunk_slices(np.full(9, 0.3), 1e-9).tolist() == [0, 9]
    assert capi.dcnv_chunk_slices(np.arange(4) * 0.25, 0.25).tolist() == [0, 2, 4]        # 0.25 - 0 is not > 0.25
    assert capi.dcnv_chunk_slices(np.array([0.0, 0.1, 0.2, 0.3]), 1.0).tolist() == [0, 4]


def test_slices_sizing_and_errors():
    v = np.arange(10) * 0.5
    n = capi.C.c_int64(-1)
    assert capi.lib.gl_dcnv_chunk_slices(capi._ptr(v), v.size, 0.4, None, 0, capi.C.byref(n)) == capi.GL_OK and n.value == 10
    small = np.zeros(10, np.int64)                                         # room for 10 offsets, 11 needed
    assert capi.lib.gl_dcnv_chunk_slices(capi._ptr(v), v.size, 0.4, capi._ptr(small), small.size, capi.C.byref(n)) == capi.GL_ERANGE
    assert n.value == 10
    for w in (0.0, -0.1, np.nan, np.inf, -np.inf):
        with pytest.raises(capi.GlError):
            capi.dcnv_chunk_slices(v, w)
    with pytest.raises(capi.GlError):
        capi.dcnv_chunk_slices(np.zeros(0), 0.1)


def _numpy_chunk(x, slices):
    """ChunkDebiaser.Debias on one GC-sorted column, restated in numpy"""
    x = np.array(x, np.float64)
    for a, b in zip(slices[:-1], slices[1:]):
        s = np.sort(x[a:b])
        k = 0
        while k < s.size and s[k] == 0:
            k += 1
        med = s[(b - a - k) // 2]
        if med > 0:
            x[a:b] = x[a:b] / med
    return x


def test_oracle_hand_cases():
    one = lambda c: oc.chunk_debias(np.array(c, np.float64), [0, len(c)]).ravel()
    assert np.array_equal(one([0, 0, 5, 7, 9]), [0, 0, 5, 7, 9])           # index (5 - 2) / 2 = 1: a zero, left alone
    assert np.array_equal(one([0, 4, 6, 8]), np.array([0, 4, 6, 8]) / 4)   # index (4 - 1) / 2 = 1 into the whole chunk: 4, not 6
    assert np.array_equal(one([0, 5, 7, 9, 11]), np.array([0, 5, 7, 9, 11]) / 7)
    assert np.array_equal(one([0, 0, 0]), [0, 0, 0])                      # all zero: index 0
    assert np.array_equal(one([-2, 0, 0, 3, 8]), [-2, 0, 0, 3, 8])         # a negative: k = 0, index 2 is a zero
    assert np.array_equal(one([-2, 3, 8]), np.array([-2, 3, 8]) / 3)
    assert np.array_equal(one([-0.0, 4, 6]), np.array([-0.0, 4, 6]) / 4)   # -0 counts as a zero: index (3 - 1) / 2 = 1
    got = one([7, -0.0, 0, 0])
    assert np.array_equal(got, [7, 0, 0, 0]) and np.signbit(got[1])        # unchanged, -0 kept
    assert np.array_equal(one([9]), [1.0])
    # two chunks, each its own median
    got = oc.chunk_debias(np.array([2.0, 4, 6, 10, 30, 50]), [0, 3, 6]).ravel()
    assert np.array_equal(got, [0.5, 1, 1.5, 1 / 3, 1, 50 / 30])


def test_oracle_matches_numpy():
    rng = np.random.default_rng(7)
    for t in range(300):
        n = int(rng.integers(1, 60))
        S = int(rng.integers(1, 4))
        x = rng.integers(-2, 6, (n, S)).astype(np.float64) if t % 3 == 0 else np.round(rng.gamma(2.0, 3.0, (n, S)) * (rng.random((n, S)) > 0.4), 2)
        cuts = np.sort(rng.choice(np.arange(1, n), size=min(n - 1, int(rng.integers(0, 6))), replace=False)) if n > 1 else []
        slices = np.array([0, *cuts, n], np.int64)
        got = oc.chunk_debias(x, slices)
        for c in range(S):
            assert np.array_equal(got[:, c].view(np.uint64), _numpy_chunk(x[:, c], slices).view(np.uint64)), (t, c)


def test_oracle_matrix_sorts_and_unsorts():
    """the chunks follow the GC order, and the result goes back to position order"""
    rng = np.random.default_rng(8)
    n, S = 400, 3
    gc = rng.integers(0, 50, n) / 50.0
    x = np.floor(rng.gamma(4.0, 8.0, (n, S)))
    out, inds, slices, med = oc.matrix(x, gc, 0.05)
    assert np.array_equal(slices, _slices(gc[inds], 0.05))
    deb = np.empty_like(x)
    for c in range(S):
        deb[inds, c] = _numpy_chunk(x[inds, c], slices)
    assert np.array_equal(out * 0 + deb / med, out)


BAD = [("--chunk",), ("--chunk", "abc"), ("--chunk", "nan"), ("--chunk", "NaN"), ("--chunk", "inf"), ("--chunk", "-Inf"),
       ("--chunk", "0"), ("--chunk", "-0"), ("--chunk", "-0.01"), ("--chunk", ""), ("--chunk=",), ("--chunk=0",), ("--chunk=x1",),
       ("--chunk=-5",), ("--noplots", "--chunk", "0"), ("--svd", "5", "--chunk", "nan")]


@pytest.mark.parametrize("flags", BAD, ids=["_".join(f) or "empty" for f in BAD])
def test_bad_chunk_exit_255(tmp_path, flags):
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    args = [GOLEFT, "dcnv", *flags] + ([] if flags == ("--chunk",) else ["m.tsv", "ref.fa"])
    r = subprocess.run(args, capture_output=True, cwd=str(tmp_path))
    assert r.returncode == 255, (flags, r.returncode, r.stderr)
    assert r.stdout == b"" and b"chunk" in r.stderr and b"Usage: goleft dcnv" in r.stderr, (flags, r.stderr)
    assert not os.path.exists(tmp_path / "depth.bed")
