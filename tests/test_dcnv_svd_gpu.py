"""gl_dcnv_svd (DESIGN §1.13) on the GPU: the FP64 tensor-core Gram against numpy's Z^T Z, its bits across row blocks and
runs, the device entry against the host entry, the count and the singular values against the numpy SVD oracle on planted
batch effects, the output within a bound derived from the eigengap, the rows that must stay untouched, and bad arguments."""
import numpy as np
import pytest

from goleft_b200 import capi
from oracle import dcnv_svd as osv

pytestmark = pytest.mark.gpu
EPS = np.finfo(float).eps


def _cohort(rng, n, S, const_every=0):
    x = rng.gamma(30.0, 1.0 / 30.0, (n, S)) * rng.uniform(0.5, 2.0, (n, 1))
    if const_every:
        x[::const_every] = 0.0
        x[1::const_every] = 0.1
        x[2::const_every] = 1.25
    return x


def _zt_z(x):
    z, kept, _, _ = osv.zscore(x)
    return z.T @ z, kept


@pytest.mark.parametrize("S,n", [(1, 1000), (2, 5000), (3, 2 ** 20 + 7), (8, 100_003), (33, 50_001), (63, 30_011), (65, 30_013),
                                 (128, 70_000), (257, 20_011), (2504, 3_001)])
def test_gram_against_numpy(ctx, S, n):
    rng = np.random.default_rng(S)
    x = _cohort(rng, n, S, const_every=97)
    _, _, _, kept, gram = ctx.dcnv_svd(x, 100.0, want_gram=True)
    want, mask = _zt_z(x)
    assert kept == int(mask.sum())
    assert np.array_equal(gram, gram.T)
    scale = max(np.abs(want).max(), 1e-300)
    assert np.abs(gram - want).max() <= 1e-11 * scale


def test_bits_across_blocks_runs_and_entries(ctx):
    rng = np.random.default_rng(7)
    n, S = 20_011, 33
    x = _cohort(rng, n, S, const_every=50)
    x[:, :S // 2] += rng.normal(0, 0.3, n)[:, None]                       # a batch term: something to remove
    ref = ctx.dcnv_svd(x, 1.0, want_gram=True)
    assert ref[2] >= 1
    for br in (4, 1000, 2017, 4099, n - 1, n):
        got = ctx.dcnv_svd(x, 1.0, block_rows=br, want_gram=True)
        for a, b in zip(ref, got):
            assert np.array_equal(a, b), br
    again = ctx.dcnv_svd(x, 1.0, want_gram=True)
    for a, b in zip(ref, again):
        assert np.array_equal(a, b)
    ld = S + 3                                                            # the device entry, on a padded resident matrix
    xp = np.zeros((n, ld))
    xp[:, :S] = x
    d = ctx.dev_array(xp)
    sv, nr, nk, gram = ctx.dcnv_svd_device(d, n, ld, S, 1.0, want_gram=True)
    dev = d.download(np.float64, n * ld).reshape(n, ld)
    d.free()
    assert np.array_equal(dev[:, :S], ref[0]) and np.array_equal(dev[:, S:], 0 * dev[:, S:])
    assert np.array_equal(sv, ref[1]) and nr == ref[2] and nk == ref[3] and np.array_equal(gram, ref[4])


def _planted(rng, n, S, k):
    """noise plus k batch components of geometrically falling strength: clear eigengaps at every index up to k"""
    x = 40.0 + rng.normal(0, 1.0, (n, S))
    for c in range(k):
        u = rng.normal(0, 1.0, n)
        v = rng.normal(0, 1.0, S)
        x += (12.0 * 0.8 ** c) * np.outer(u, v)
    return np.maximum(x, 0.0)


@pytest.mark.parametrize("S,n,k", [pytest.param(64, 30_000, k, id=str(k)) for k in (0, 1, 5, 20)] +
                         [pytest.param(1000, 6_000, k, id="1000-%d" % k) for k in (0, 1, 5, 20)] +
                         [pytest.param(2504, 1_200, 5, id="wide-2504-5")])  # S > n: rank 1200, a null space of 1304
def test_planted_batch_effects_against_oracle(ctx, S, n, k):
    rng = np.random.default_rng(100 + k if S == 64 else [S, k])
    x = _planted(rng, n, S, k)
    z, kept, m, sd = osv.zscore(x)
    s = osv.singular_values(z, S)
    share = 100 * s / s[s > 0].sum()
    want_n = min(k, osv.MAX_REMOVE)
    pct = share[0] * 1.5 if want_n == 0 else 0.5 * (share[want_n - 1] + share[want_n]) if k <= osv.MAX_REMOVE else share[k] / 2
    assert osv.count(s, pct) == want_n
    if want_n:                                                            # the cases are built with room at the cut
        assert share[want_n - 1] - pct > 0.05 * pct and (k > osv.MAX_REMOVE or pct - share[want_n] > 0.05 * pct)
        assert (s[want_n - 1] ** 2 - s[want_n] ** 2) / s[want_n - 1] ** 2 >= 1e-2
    out, sv, nr, nk, _ = ctx.dcnv_svd(x, pct)
    want, s2, n2, _ = osv.svd_debias(x, pct)
    assert nr == n2 == want_n and nk == int(kept.sum())
    pos = s > 0
    assert np.array_equal(sv > 0, pos)
    assert np.abs(sv - s).max() <= 1e-9 * s[0]
    if nr == 0:
        assert np.array_equal(out, x)
        return
    # |x' - x'_oracle| / sd: the Gram's rounding (a few ulp of lambda_1 per entry) moves V_n by about
    # S eps lambda_1 / (lambda_n - lambda_{n+1}), and |z| <= sqrt(S - 1) carries that into z'
    lam = s ** 2
    gap = lam[nr - 1] - lam[nr]
    bound = max(1e-8, 1e3 * S * EPS * lam[0] / gap * np.sqrt(S))
    err = np.abs(out[kept] - want[kept]) / sd[:, None]
    assert err.max() <= bound, (err.max(), bound)
    assert np.array_equal(out[~kept], x[~kept])


def test_constant_rows_untouched(ctx):
    rng = np.random.default_rng(3)
    n, S = 4000, 16
    x = _planted(rng, n, S, 2)
    x[::10] = 0.1                                                          # sd of 0.1 x S is ~1e-17 from rounding, not 0
    x[5::10] = 0.0
    x[7::10] = 1e300
    out, sv, nr, nk, _ = ctx.dcnv_svd(x, 0.0)
    assert nr >= 1 and nk == n - 3 * (n // 10)
    for off in (0, 5, 7):
        assert np.array_equal(out[off::10].view(np.uint64), x[off::10].view(np.uint64))
    # S < 2: every row is excluded, nothing is removed
    one = rng.normal(5, 1, (100, 1))
    out, sv, nr, nk, _ = ctx.dcnv_svd(one, 0.0)
    assert nr == 0 and nk == 0 and np.array_equal(out, one) and sv.tolist() == [0.0]


def test_nothing_removed_is_identity(ctx):
    rng = np.random.default_rng(4)
    x = _planted(rng, 5000, 24, 3)
    out, sv, nr, _, _ = ctx.dcnv_svd(x, 100.0)
    assert nr == 0 and np.array_equal(out.view(np.uint64), x.view(np.uint64))
    assert sv[0] > 0
    # all rows constant: no rank at all
    out, sv, nr, nk, _ = ctx.dcnv_svd(np.full((50, 6), 2.5), 0.0)
    assert nr == 0 and nk == 0 and not sv.any()


def test_bad_arguments(ctx):
    x = _cohort(np.random.default_rng(5), 100, 8)
    for pct in (float("nan"), float("inf"), -1.0):
        with pytest.raises(capi.GlError) as e:
            ctx.dcnv_svd(x, pct)
        assert e.value.code == capi.GL_EINVAL
    bad = x.copy()
    bad[37, 3] = np.inf
    with pytest.raises(capi.GlError) as e:
        ctx.dcnv_svd(bad, 1.0)
    assert e.value.code == capi.GL_EINVAL and "row 37" in str(e.value)
    bad[37, 3] = np.nan
    with pytest.raises(capi.GlError):
        ctx.dcnv_svd(bad, 1.0)
    inf_row = x.copy()
    inf_row[11] = np.inf                                                  # constant: excluded, so not an error
    out, _, _, nk, _ = ctx.dcnv_svd(inf_row, 1.0)
    assert nk == 99 and np.isinf(out[11]).all()
    with pytest.raises(capi.GlError):
        ctx.dcnv_svd(x, 1.0, block_rows=-1)
    with pytest.raises(capi.GlError):
        ctx.dcnv_svd(np.zeros((0, 4)), 1.0)
    d = ctx.dev_array(x)
    with pytest.raises(capi.GlError):
        ctx.dcnv_svd_device(d, 100, 7, 8, 1.0)                             # ld < S
    d.free()
