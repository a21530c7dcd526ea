"""`goleft dcnv`, the parts that need no GPU: Go's sort.Sort permutation (gl_go_argsort_f64 against the oracle's own
pdqsort restatement), the debias window model (the oracle's literal moving median against a brute-force closed form), and
the "%.2f" token (gl_format_f2_host against printf)."""
import numpy as np
import pytest

from goleft_b200 import capi
from oracle import dcnv as od


def _arrays(rng, count):
    for t in range(count):
        n = int(rng.choice([1, 2, 3, 5, 8, 11, 12, 13, 49, 50, 51, 200, 1000, 4097, 100_000])) if t % 3 else int(rng.integers(1, 3000))
        kind = t % 5
        if kind == 0:
            v = rng.random(n)                                            # distinct
        elif kind == 1:
            v = rng.integers(0, max(1, n // 20 + 1), n) / 7.0             # tie-heavy, like GC fractions of one window size
        elif kind == 2:
            v = np.sort(rng.integers(0, 300, n) / 300.0)                  # sorted, with ties
        elif kind == 3:
            v = np.sort(rng.integers(0, 300, n) / 300.0)[::-1].copy()     # reversed: the decreasing hint
        else:
            v = np.sort(rng.random(n))
            k = max(1, n // 50)
            idx = rng.integers(0, n, k)
            v[idx] = rng.random(k)                                        # nearly sorted: partialInsertionSort
        yield v


def test_argsort_matches_go_restatement():
    rng = np.random.default_rng(11)
    for v in _arrays(rng, 2000):
        got = capi.go_argsort(v)
        n = v.size
        assert np.array_equal(np.sort(got), np.arange(n))
        assert np.all(np.diff(v[got]) >= 0)
        assert np.array_equal(got, od.argsort(v)), n
        if n <= 12:                                                       # insertion sort: stable
            assert np.array_equal(got, np.argsort(v, kind="stable"))


def test_argsort_is_not_stable():
    """the order inside ties is pdqsort's, not a stable sort's: what the window of each depth is depends on it"""
    rng = np.random.default_rng(3)
    v = rng.integers(0, 40, 5000) / 40.0
    got = capi.go_argsort(v)
    assert not np.array_equal(got, np.argsort(v, kind="stable"))
    assert np.array_equal(got, od.argsort(v))
    assert np.array_equal(capi.go_argsort(np.full(1000, 0.5)), np.arange(1000))   # all equal: the identity


def _closed_form(c):
    """row i divides by max(1, median of p[max(0, j-8) .. j]), p = c[0..4] ++ c[10..], j = clamp(i, 4, max(4, n-6))"""
    n = c.size
    p = np.concatenate([c[:5], c[10:]])
    out = np.empty(n)
    for i in range(n):
        j = min(max(i, 4), max(4, n - 6))
        w = np.sort(p[max(0, j - 8):j + 1])
        m = w.size
        med = w[m // 2] if m % 2 else (w[m // 2 - 1] + w[m // 2]) / 2
        out[i] = c[i] / max(med, 1.0)
    return out


@pytest.mark.parametrize("n", list(range(5, 26)) + [1000])
def test_window_model(n):
    rng = np.random.default_rng(n)
    for trial in range(20):
        c = rng.integers(0, 6, n).astype(np.float64) if trial % 2 else rng.random(n) * 4
        assert np.array_equal(od.debias(c), _closed_form(c)), (n, trial)


def test_pushes_skip_rows_5_to_9():
    """c[5..9] are never pushed: changing them changes no divisor"""
    rng = np.random.default_rng(2)
    c = rng.integers(1, 50, 40).astype(np.float64)
    c2 = c.copy()
    c2[5:10] = [1000, 2000, 3000, 4000, 5000]
    a, b = od.debias(c), od.debias(c2)
    assert np.array_equal(a[:5], b[:5]) and np.array_equal(a[10:], b[10:])
    assert np.allclose(c[5:10] / a[5:10], c2[5:10] / b[5:10], rtol=1e-12, atol=0)
    with pytest.raises(od.Panic):
        od.debias(np.ones(4))


def test_sample_median_rule():
    """sorted[k + int(0.65 (n - k))], k = leading exact zeros; with a negative value k = 0"""
    col = np.array([0, 0, 0, 5, 1, 2, 3, 4, 0, 6], np.float64)
    s = np.sort(col)
    assert od.sample_median(col) == s[4 + int(0.65 * 6)]
    neg = col.copy()
    neg[0] = -1
    assert od.sample_median(neg) == np.sort(neg)[int(0.65 * 10)]
    with pytest.raises(od.Panic):
        od.sample_median(np.zeros(8))


def _token_cases(rng):
    parts = []
    j = np.arange(0, 60)
    parts.append(np.concatenate([2.5 * 2.0 ** -j, 0.125 * np.arange(-4000, 4000)]))                  # exact binary values, ties
    x5 = (np.arange(0, 200_000) + 0.5) / 100.0                                                        # x.xx5 and its neighbours
    parts.append(np.concatenate([x5, np.nextafter(x5, 0), np.nextafter(x5, 10), -x5, -np.nextafter(x5, 0)]))
    big = rng.integers(0, 10 ** 12, 400_000) + rng.integers(0, 1000, 400_000) / 1000.0 + 0.005
    parts.append(np.concatenate([big, np.nextafter(big, 0), np.nextafter(big, np.inf)]))
    parts.append(np.arange(-100_000, 100_000) * 0.005)                                              # 0.005 steps
    parts.append(np.array([0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308, 1e-300, 0.004999, 0.005, 0.015, 0.025]))
    parts.append(rng.random(500_000) * 1e-305)                                                      # subnormal and tiny
    parts.append(10.0 ** rng.uniform(11, 300, 300_000) * rng.choice([-1, 1], 300_000))             # 1e11 .. 1e300: too long for a token
    parts.append(np.array([1e15, -1e15, 1e12, 999999999999.995, 9999999999999.99, 99999999999999.99, -9999999999999.99, 2.0 ** 47, 2.0 ** 53]))
    n_rest = 10_000_000 - sum(p.size for p in parts)
    mags = 10.0 ** rng.integers(-4, 15, n_rest)
    parts.append(rng.standard_normal(n_rest) * mags)
    return np.concatenate(parts)


def test_f2_tokens_equal_printf():
    v = _token_cases(np.random.default_rng(7))
    assert v.size >= 10_000_000
    tok = capi.format_f2_host(v)
    bad, first = od.f2_mismatches(v, tok)
    assert bad == 0, (first, repr(v[first]), tok[first].tobytes())
    assert capi.f2_text(capi.format_f2_host([np.nan, np.inf, -np.inf, -0.0, 0.125, 0.375]), [0] * 6) == \
        [b"NaN", b"+Inf", b"-Inf", b"-0.00", b"0.12", b"0.38"]
