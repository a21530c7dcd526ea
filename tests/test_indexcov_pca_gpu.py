"""indexcov's PCA on the GPU (gl_indexcov_pca, gl_indexcov_pca_device): the tensor-core Gram bit for bit, and the
projections against the oracle's SVD route (oracle/indexcov_pca.py)."""
import numpy as np
import pytest

from goleft_b200 import capi
from oracle import indexcov_pca as op

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("S,D,fill", [(1, 1, None), (3, 7, None), (7, 300, None), (33, 32768, None), (33, 32769, None),
                                      (33, 65537, 255), (127, 20011, None), (128, 100003, None), (129, 30011, None),
                                      (257, 50021, None), (1000, 2 ** 17 + 5, None),
                                      # 36 tiles: pca_run's split gives kc = 32768, the kKMax limit, at 132 SMs and at 114,
                                      # so eight of each tile's nine CTAs sum 32768 columns of 255^2: 2,130,739,200 < 2^31
                                      (1000, 2 ** 18 + 5, 255)])
def test_gram_exact(ctx, S, D, fill):
    rng = np.random.default_rng(S * 7 + D)
    x = np.full((S, D), fill, np.uint8) if fill is not None else rng.integers(0, 256, (S, D), dtype=np.uint8)
    _, _, _, g = ctx.indexcov_pca(x, want_gram=True)
    if fill is not None:
        assert np.array_equal(g, np.full((S, S), fill * fill * D, np.int64))
        return
    xf = x.astype(np.float64)
    assert np.array_equal(g, (xf @ xf.T).astype(np.int64))            # every partial sum is an integer below 2^53


def test_gram_row_stride(ctx):
    """ld > D: the bytes past D in each row are not part of the matrix"""
    rng = np.random.default_rng(2)
    S, D, ld = 45, 1000, 1037
    x = rng.integers(0, 256, (S, ld), dtype=np.uint8)
    _, _, _, g = ctx.indexcov_pca(x, D=D, want_gram=True)
    xf = x[:, :D].astype(np.float64)
    assert np.array_equal(g, (xf @ xf.T).astype(np.int64))
    d_x = ctx.dev_array(np.ascontiguousarray(np.pad(x, ((0, 0), (0, 1040 - ld)), constant_values=7)))
    p1, s1, k1, g1 = ctx.indexcov_pca_device(d_x, 1040, S, D, want_gram=True)
    p2, s2, k2, _ = ctx.indexcov_pca(x, D=D)
    assert np.array_equal(g1, g) and k1 == k2 == 5
    assert np.array_equal(p1, p2) and np.array_equal(s1, s2)


def _noise(rng, S, D):
    return rng.integers(0, 256, (S, D), dtype=np.uint8)


def _planted(rng, S, D):
    """depth-like bytes with groups: zero stretches shared by subsets of the samples"""
    x = rng.integers(20, 90, (S, D), dtype=np.uint8)
    groups = [(0, S // 3, 0.10), (S // 3, S // 2, 0.25), (S // 2, S, 0.05)]
    for a, b, frac in groups:
        c0 = int(rng.integers(0, D // 2))
        x[a:b, c0:c0 + int(frac * D)] = 0
    x[:, ::97] = 0                                                      # the zero column at every reference's end
    return x


def _check(ctx, x):
    """|proj - oracle| <= 1e-7 max|column|; the "%.2f" text is identical except in cells within that tolerance of a
    half-cent boundary, and there are no more of those than twice what a uniform spread of values predicts (plus 3)"""
    proj, sv, k, _ = ctx.indexcov_pca(x)
    ep, es, ek = op.pca(x)
    assert k == ek
    proj = proj[:, :k]
    near_total, near_expected = 0, 0.0
    for j in range(k):
        tol = 1e-7 * max(np.abs(ep[:, j]).max(), 1e-300)
        assert np.abs(sv[j] - es[j]) <= 1e-7 * es[0], (j, sv[j], es[j])
        assert np.abs(proj[:, j] - ep[:, j]).max() <= tol, (j, np.abs(proj[:, j] - ep[:, j]).max(), tol)
        near = op.half_cent_near(ep[:, j], tol)
        got_t = ["%.2f" % v for v in proj[:, j]]
        exp_t = ["%.2f" % v for v in ep[:, j]]
        assert all(a == b for a, b, nr in zip(got_t, exp_t, near) if not nr)
        near_total += int(near.sum())
        near_expected += x.shape[0] * min(1.0, 200 * tol) if es[j] > 0 else 0.0
    assert near_total <= 2 * near_expected + 3
    return proj, sv, k


@pytest.mark.parametrize("S", [3, 4, 5, 6, 7, 100, 1000, 2504])
@pytest.mark.parametrize("kind", ["noise", "planted"])
def test_pca_against_oracle(ctx, S, kind):
    rng = np.random.default_rng(S + (0 if kind == "noise" else 1000))
    D = 3000 if S < 1000 else 4000
    x = (_noise if kind == "noise" else _planted)(rng, S, D)
    proj, sv, k = _check(ctx, x)
    if S <= 5:                                                          # rank S - 1: the last column is the rank rule's
        assert sv[S - 1] == 0 and np.all(proj[:, S - 1] == 0)


def test_pca_rank_deficient(ctx):
    rng = np.random.default_rng(11)
    base = rng.integers(0, 256, (3, 500), dtype=np.uint8)
    x = np.concatenate([base, base, base[:1]])                          # duplicated samples: rank 2 after centring
    proj, sv, k, _ = ctx.indexcov_pca(x)
    assert k == 5 and np.all(sv[2:] == 0) and np.all(proj[:, 2:] == 0) and sv[1] > 0
    _check(ctx, x)
    same = np.tile(base[:1], (6, 1))                                    # all samples identical: sigma_1 = 0
    proj, sv, k, _ = ctx.indexcov_pca(same)
    assert k == 5 and np.all(sv == 0) and np.all(proj == 0)
    assert ["%.2f" % v for v in proj.ravel()] == ["0.00"] * proj.size


def test_pca_deterministic(ctx):
    rng = np.random.default_rng(4)
    x = _planted(rng, 300, 20011)
    a = ctx.indexcov_pca(x, want_gram=True)
    b = ctx.indexcov_pca(x, want_gram=True)
    assert all(np.array_equal(u, v) for u, v in zip((a[0], a[1], a[3]), (b[0], b[1], b[3])))


def test_pca_bad_shapes(ctx):
    x = np.zeros((4, 10), np.uint8)
    with pytest.raises(capi.GlError):
        ctx.indexcov_pca(x, D=0)
    with pytest.raises(capi.GlError):
        ctx.indexcov_pca(x, D=11)                                       # ld < D
    with pytest.raises(capi.GlError):
        ctx.indexcov_pca(x, k=0)
    with pytest.raises(capi.GlError):
        ctx.indexcov_pca(np.zeros((0, 10), np.uint8))
    d_x = ctx.dev_array(np.zeros(4 * 24, np.uint8))
    with pytest.raises(capi.GlError):
        ctx.indexcov_pca_device(d_x, 24, 4, 10)                         # device row stride not a multiple of 16
    p, s, k, _ = ctx.indexcov_pca(np.zeros((2, 10), np.uint8))
    assert k == 2 and np.all(p == 0)
