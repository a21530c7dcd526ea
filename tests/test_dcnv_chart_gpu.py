"""`goleft dcnv`'s depth chart on the GPU (gl_dcnv_chart): the selection, the extent and the stepped-line index image equal the
host mirrors bit for bit, for any row-block size, and once at the benchmark's shape (3,088,281 rows x 128 samples)."""
import os
import sys
import threading
import time

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from goleft_b200 import capi  # noqa: E402

pytestmark = pytest.mark.gpu
W, H = capi.PLOT_W, capi.PLOT_H


@pytest.fixture(scope="module")
def ctx():
    if capi.device_count() < 1:
        pytest.skip("no CUDA device")
    with capi.Ctx(0) as c:
        yield c


def cohort(n, S, seed):
    """normalised-looking depths: ~1 with noise, a few deletions and duplications, leading zeros of several lengths"""
    rng = np.random.default_rng(seed)
    x = rng.normal(1.0, 0.15, (n, S))
    x[rng.random((n, S)) < 0.01] = 0.0
    x[rng.random((n, S)) < 0.002] = 3.5
    for k in range(S):
        x[: (k * 37) % max(1, n // 3), k] = 0.0
    if S > 2:
        x[:, 2] = 0.0
        x[n - 1, 2] = 1.0                                  # one vertex only
        x[rng.integers(0, n, 3), 1] = np.nan               # breaks in the line
        x[rng.integers(0, n, 2), 1] = -np.inf
        x[0, 1] = -0.0
    return x


def host(x):
    first, yext = capi.dcnv_chart_select_host(x)
    ext = capi.dcnv_chart_extent(first, yext, x.shape[0])
    xf = capi.plot_transform(ext, W, H)
    return first, yext, ext, capi.dcnv_chart_raster_host(x, first, xf)


def same(got, want):
    for g, w in zip(got, want):
        assert g.shape == w.shape and np.array_equal(g, w)


@pytest.mark.parametrize("n", [5, 1000, (1 << 20) + 7])
@pytest.mark.parametrize("S", [1, 2, 31, 33, 128])
def test_chart_equals_host(ctx, S, n):
    x = cohort(n, S, S * 7 + n % 97)
    want = host(x)
    got = ctx.dcnv_chart(x)
    same(got, want)
    assert got[3].any()


@pytest.mark.parametrize("block_rows", [1, 7, 333, 999, 1000, 5000])
def test_row_blocks(ctx, block_rows):
    x = cohort(1000, 33, 5)
    x[:700, 0] = 0.0                                      # first row past several blocks
    want = host(x)
    same(ctx.dcnv_chart(x, block_rows=block_rows), want)


def test_degenerate(ctx):
    for x in (np.zeros((5, 3)), np.full((5, 2), np.nan), np.ones((1, 4)), np.zeros((0, 2))):
        got = ctx.dcnv_chart(x)
        want = host(x)
        same(got, want)
        assert not got[3].any()
    with pytest.raises(capi.GlError):
        ctx.dcnv_chart(np.ones((5, 2)), block_rows=-1)


def test_benchmark_shape(ctx):
    """the dcnv benchmark's matrix, once: device = host mirror; time and peak device memory on stderr"""
    import torch
    n, S = 3_088_281, 128
    x = cohort(n, S, 2026)
    t0 = time.perf_counter()
    free0, total = torch.cuda.mem_get_info(0)
    low, stop = [free0], threading.Event()

    def poll():
        while not stop.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info(0)[0])
            time.sleep(0.001)
    th = threading.Thread(target=poll)
    th.start()
    try:
        t1 = time.perf_counter()
        got = ctx.dcnv_chart(x)
        t_dev = time.perf_counter() - t1
    finally:
        stop.set()
        th.join()
    t1 = time.perf_counter()
    want = host(x)
    t_host = time.perf_counter() - t1
    same(got, want)
    print("dcnv chart %d x %d: device entry %.2f s, host mirror %.2f s, test %.1f s, peak device memory %.0f MiB (%.0f MiB above the start)"
          % (n, S, t_dev, t_host, time.perf_counter() - t0, (total - low[0]) / 2**20, (free0 - low[0]) / 2**20), file=sys.stderr)
