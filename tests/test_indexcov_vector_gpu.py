"""indexcov's vector charts on the GPU (plot.cu): the device path text and per-dataset lengths against the host mirror, for
both vertex sources up to the 2504-sample cohort at 191 k tiles; sample shards made apart and concatenated in draw order
against the whole; a too-small buffer rejected."""
import numpy as np
import pytest

from goleft_b200 import capi
import plot_rule as pr
import vector_rule as vr

pytestmark = pytest.mark.gpu
W, H = capi.PLOT_W, capi.PLOT_H


def _cohort(S, T, seed):
    rng = np.random.default_rng(seed)
    vals = rng.standard_normal((S, T), dtype=np.float32)
    vals *= 0.2
    vals += 1.0
    np.maximum(vals, 0, out=vals)
    vals[:, :3] = 0                                                     # leading zeros: the skip
    vals[::7, 5] = 3.5                                                  # clipped at 2.5
    if S > 2:
        vals[1, 43] = np.nan                                            # a kept NaN (stride 10: position 40 after the skip)
        vals[2, :] = 0                                                  # nothing to draw
    return vals.reshape(-1), np.arange(S, dtype=np.int64) * T, np.full(S, T, np.int64)


def _series_args(S, T, seed):
    flat, off, ln = _cohort(S, T, seed)
    sel, yext = capi.plot_select_host(flat, off, ln)
    drawn = sel[:, 1] > 0
    xmax = ((sel[:, 0] + (sel[:, 1] - 1) * sel[:, 2]) * 16384.0)[drawn]
    ext = [float((sel[drawn, 0] * 16384.0).min()), float(xmax.max()), float(yext[drawn, 0].min()), float(yext[drawn, 1].max())]
    return flat, off, sel, capi.plot_transform(ext, W, H)


@pytest.mark.parametrize("T", [15_000, 191_000])
@pytest.mark.parametrize("S", [1, 2, 31, 101, 2504])
def test_series_device_matches_host(ctx, S, T):
    flat, off, sel, xf = _series_args(S, T, S * 7 + T)
    chart = np.zeros(S, np.int32)
    fmt = vr.SVG if (S + T) % 2 else vr.EPS
    dl, dt = ctx.plot_path_series(flat, off, sel, 16384.0, chart, xf, 1, capi.PLOT_DEPTH, fmt)
    hl, ht = capi.plot_path_series_host(flat, off, sel, 16384.0, chart, xf, 1, capi.PLOT_DEPTH, fmt)
    assert np.array_equal(dl, hl)
    assert dt == ht
    if S > 2:
        assert dl[1] == 0 and dl[2] == 0 and dl[0] > 0
    # spot-check the first dataset against the Python restatement
    v = flat[:T]
    s = pr.sample(*pr.as_values(v, 16384.0))
    assert dt[:dl[0]] == vr.path_text(s[0], s[1], xf, 0, fmt)


def _xy(S, m, seed):
    rng = np.random.default_rng(seed)
    sizes = np.full(S, m, np.int64)
    sizes[::5] = np.minimum(sizes[::5], 1 + np.arange(len(sizes[::5])) % 3)   # 1, 2 and 3 vertices too
    ptr = np.concatenate([[0], np.cumsum(sizes)])
    x = rng.uniform(0, 1.5, int(ptr[-1]))
    y = rng.uniform(0, 1.0, int(ptr[-1]))
    if S > 3:
        y[ptr[3] + sizes[3] // 2] = np.nan
    return x, y, ptr


@pytest.mark.parametrize("m", [70, 19_100])
@pytest.mark.parametrize("S", [1, 2, 31, 101, 2504])
def test_xy_device_matches_host(ctx, S, m):
    x, y, ptr = _xy(S, m, S + m)
    kind = capi.PLOT_SQUARE if S == 31 else capi.PLOT_PLAIN
    Wk, Hk = vr.CANVAS[kind][:2]
    chart = (np.arange(S) % 2).astype(np.int32) if kind == capi.PLOT_PLAIN else np.zeros(S, np.int32)
    nc = int(chart.max()) + 1
    xf = np.concatenate([pr.transform(0, 1.5, 0, 1.0, Wk, Hk), pr.transform(-0.5, 2.0, -0.25, 1.25, Wk, Hk)])[:4 * nc]
    for fmt in (vr.SVG, vr.EPS):
        dl, dt = ctx.plot_path_xy(x, y, ptr, chart, xf, nc, kind, fmt)
        hl, ht = capi.plot_path_xy_host(x, y, ptr, chart, xf, nc, kind, fmt)
        assert np.array_equal(dl, hl)
        assert dt == ht
        if S > 3:
            assert dl[3] == 0


@pytest.mark.parametrize("G", [2, 3, 7])
def test_shards_concatenate_to_the_whole(ctx, G):
    S, T, nc = 101, 15_000, 2
    flat, off, ln = _cohort(S, T, 5)
    sel, _ = capi.plot_select_host(flat, off, ln)
    xf = np.concatenate([pr.transform(0, 2.5e8, 0, 2.5, W, H), pr.transform(0, 1.2e8, 0.5, 2.0, W, H)])
    # (chart, sample) datasets; chart 1 reads the second half of each sample's tiles
    offs = np.concatenate([off, off + T // 2])
    sels = np.concatenate([sel, capi.plot_select_host(flat, off + T // 2, ln // 2)[0]])
    chart = np.repeat(np.arange(nc, dtype=np.int32), S)
    whole_l, whole_t = ctx.plot_path_series(flat, offs, sels, 16384.0, chart, xf, nc, capi.PLOT_DEPTH, vr.SVG)
    cut = np.linspace(0, S, G + 1).astype(int)
    parts = []
    for g in range(G):
        idx = np.concatenate([c * S + np.arange(cut[g], cut[g + 1]) for c in range(nc)])
        pl, pt = ctx.plot_path_series(flat, offs[idx], sels[idx], 16384.0, chart[idx], xf, nc, capi.PLOT_DEPTH, vr.SVG)
        pos = np.concatenate([[0], np.cumsum(pl)])
        parts.append({int(i): pt[pos[j]:pos[j + 1]] for j, i in enumerate(idx)})
    got = b"".join(parts[int(np.searchsorted(cut, i % S, side="right")) - 1][i] for i in range(nc * S))
    assert got == whole_t


def test_too_small_buffer_is_rejected(ctx):
    flat, off, sel, xf = _series_args(31, 15_000, 9)
    chart = np.zeros(31, np.int32)
    ln, text = ctx.plot_path_series(flat, off, sel, 16384.0, chart, xf, 1, capi.PLOT_DEPTH, vr.EPS)
    for cap in (0, int(ln.sum()) - 1):
        with pytest.raises(capi.GlError) as e:
            ctx.plot_path_series(flat, off, sel, 16384.0, chart, xf, 1, capi.PLOT_DEPTH, vr.EPS, cap=cap)
        assert e.value.code == capi.GL_ERANGE
    with pytest.raises(capi.GlError) as e:
        ctx.plot_path_xy([0.0, 1.0], [0.0, 1.0], [0, 2], [0], xf, 1, capi.PLOT_PLAIN, vr.SVG, cap=3)
    assert e.value.code == capi.GL_ERANGE
    l2, t2 = ctx.plot_path_series(flat, off, sel, 16384.0, chart, xf, 1, capi.PLOT_DEPTH, vr.EPS)
    assert np.array_equal(l2, ln) and t2 == text                       # the ctx is still usable
