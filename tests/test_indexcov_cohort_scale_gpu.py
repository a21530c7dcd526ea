"""indexcov's cohort path at cohort scale: more samples than ic_xnorm_kernel's one CTA has threads, the 2504-sample shape of
the 1000 Genomes cohort for the medians (ic_cohort2_kernel), the device entries `goleft indexcov` calls, the PCA Gram at
20 x 20 tiles, and the CLI end to end past 1024 samples.  Every comparison is with the C oracle (oracle/oracle_indexcov.c
through oracle/loader.py) or oracle/indexcov_pca.py, bit for bit wherever the smaller tests are."""
import gzip
import math
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
from goleft_b200 import capi  # noqa: E402
from indexcov_cli_oracle import (check_ped_columns, cohort_bais, compare_pcs, expected_outputs, expected_pcs,  # noqa: E402
                                 oracle_depths, read_ped)
from oracle import loader as orc  # noqa: E402
from test_indexcov_gpu import synth_cohort  # noqa: E402
from test_indexcov_pca_gpu import _check, _planted  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
SLOTS = capi.INDEXCOV_SLOTS
XN_THREADS = 1024                     # ic_xnorm_kernel is one CTA: sample i belongs to thread i % 1024


# ------------------------------------------------------------------------------------------------ I7 at S > 1024
def _tile_addends(raw, done, lens, j):
    """(A, n): tile j's addends in the reference's order, one row per sample (d[j], d[j-1], d[j+1]) with 0.0 where a term
    is absent (an exact no-op in a float64 sum), and their count.  Tile j reads the finished column j-1 (from `done`, the
    oracle's output) and the raw columns j and j+1."""
    live = lens > j
    right = live & (j < lens - 1)
    A = np.zeros((raw.shape[0], 3))
    A[live, 0] = raw[live, j]
    if j > 0:
        A[live, 1] = done[live, j - 1]
    if right.any():
        A[right, 2] = raw[right, j + 1]
    return A, int(live.sum()) * (2 if j > 0 else 1) + int(right.sum())


def _seq_sum(A):
    """the reference's float64 sum: samples in order, each sample's terms in order (indexcov.go:566-574)"""
    m = 0.0
    for v in A.ravel().tolist():
        m += v
    return m


def _order_free_sum(A):
    """the kernel's order-free sum: each thread's samples i = tid, tid + 1024, ... in turn, the xor-shuffle tree inside a
    warp, then the 32 warp sums in order"""
    part = np.zeros(XN_THREADS)
    for b in range(0, A.shape[0], XN_THREADS):
        blk = A[b:b + XN_THREADS]
        for k in range(3):
            part[:blk.shape[0]] += blk[:, k]
    lane = np.arange(XN_THREADS)
    for o in (16, 8, 4, 2, 1):
        part = part + part[lane ^ o]
    m = 0.0
    for w in part[::32].tolist():
        m += w
    return m


def _span(A, n):
    """the kernel's exactness measure: (max ulp exponent + 24) + ceil(log2 n) + 1 - (min ulp exponent); <= 52 is order-free"""
    a = A[A != 0].astype(np.float32)
    if a.size == 0:
        return None
    e = np.maximum((a.view(np.uint32) >> 23) & 0xFF, 1).astype(np.int64) - 150
    lg = 0
    while (1 << lg) < n:
        lg += 1
    return int(e.max()) + 24 + lg + 1 - int(e.min())


def _threshold(n):
    """the smallest float64 sum whose mean over n is not below 0.1"""
    s = 0.1 * n
    while s / n >= 0.1:
        s = math.nextafter(s, -math.inf)
    while s / n < 0.1:
        s = math.nextafter(s, math.inf)
    return s


def _plant_threshold(rng, d, lens, j, seq_skips):
    """Column j (whose neighbours add nothing) such that tile j's mean sits on 0.1 with the reference's sequential sum on
    one side (below it when seq_skips) and the kernel's order-free sum on the other.  Samples 3.. hold 0.25..0.5 up to
    about 0.1 n, the rest ~1e-7 values whose low bits sit a quarter below (or above) half of the sum's ulp, so the sequential
    sum rounds every one of them the same way while the threads' small partial sums keep them; samples 0-2 are knobs
    (ulps 2^-25, 2^-37, 2^-43) that put the exact sum where the two orders straddle the threshold."""
    S = d.shape[0]
    n = _tile_addends(d, d, lens, j)[1]
    g = 2.0 ** (math.floor(math.log2(0.1 * n)) - 52)                  # the float64 ulp of the running sum past the big values
    q = int(round(g / 2.0 ** -47))
    assert q >= 8
    target = 0.1 * n
    col = np.zeros(S, np.float32)
    big = rng.uniform(0.25, 0.5, S).astype(np.float32)
    cs = np.cumsum(big[3:].astype(np.float64))
    m = int(np.searchsorted(cs, target - 0.375, side="right"))
    col[3:3 + m] = big[3:3 + m]
    rest = target - 0.375 - (cs[m - 1] if m else 0.0)
    col[3 + m] = np.float32(round(rest * 2 ** 25) / 2 ** 25)            # a filler on the 2^-25 grid: exact in either order
    tiny = slice(4 + m, S)
    r = rng.integers(0, (1 << 23) // q - 1, S - 4 - m) * q + (3 * q // 8 if seq_skips else 5 * q // 8)
    col[tiny] = (2.0 ** -24 + r * 2.0 ** -47).astype(np.float32)
    col[0], col[1], col[2] = 0.375, 1.5 * 2.0 ** -14, 1.5 * 2.0 ** -20
    s_star = _threshold(n)
    for _ in range(6):
        d[:, j] = col
        A = _tile_addends(d, d, lens, j)[0]
        seq, free = _seq_sum(A), _order_free_sum(A)
        if (seq < s_star) == seq_skips and (free < s_star) != seq_skips:
            return
        D = s_star - (seq + free) / 2
        for k, ulp in ((0, 2.0 ** -25), (1, 2.0 ** -37), (2, 2.0 ** -43)):
            step = round(D / ulp)
            v = float(col[k]) + step * ulp
            col[k] = v
            assert float(col[k]) == v
            D -= step * ulp
    raise AssertionError("tile %d: no knob setting puts the two summation orders on both sides of 0.1" % j)


def _plant_span(d, j, rows, span, lg):
    """values at exponents 6 and 6 - (span - 25 - lg) in column j: the tile's span is then exactly `span` as long as every
    other addend lies between (checked afterwards)"""
    d[rows[0], j] = 100.0
    d[rows[1], j] = np.float32(1.25 * 2.0 ** (6 - (span - 25 - lg)))


def _xnorm_compare(ctx, d, lens):
    got = ctx.indexcov_xnorm(d, lens)
    exp = orc.ic_xnorm(d.copy(), lens)
    for i in range(d.shape[0]):
        n = lens[i]
        assert np.array_equal(got[i, :n].view(np.uint32), exp[i, :n].view(np.uint32)), (d.shape, i, n)
    return exp


XN_S = [5, 1023, 1024, 1025, 2047, 2048, 2049, 2504]


@pytest.mark.parametrize("S", XN_S)
def test_xnorm_summation_paths(ctx, S):
    """T = 3000 tiles.  Tiles 1 and 3 sit on the 0.1 threshold with the two summation orders on opposite sides of it
    (S >= 1023; the span there is 55..60, so the kernel must take the ordered sum); interior tiles mix ~3e4 and ~1e-7 values
    over samples that share a thread and samples that do not; two tiles sit at the classifier's limit (span 52 and 53);
    two short samples on one thread's two owners make tile T - 2 count exactly 3S - 4 terms."""
    rng = np.random.default_rng(S)
    T = 3000
    d = rng.uniform(0.25, 2.0, (S, T)).astype(np.float32)
    d[rng.random((S, T)) < 0.03] = 0
    lens = np.full(S, T, np.int32)
    a = 5 if S > 8 else 1
    b = a + XN_THREADS if S > a + XN_THREADS else S - 2
    lens[a], lens[b] = T - 1, T - 2
    engineered = S >= 1023
    if engineered:
        d[:, [0, 2, 4]] = 0                                            # tiles 1 and 3 see only their own column
        _plant_threshold(rng, d, lens, 1, seq_skips=True)
        _plant_threshold(rng, d, lens, 3, seq_skips=False)
    # order-dependent tiles: a few ~3e4 values, many ~1e-7 ones
    mixed = [T // 3, T // 3 + 40, T // 2, 2 * T // 3]

    def plant_mixed(t, j):
        base = (7 + 97 * t) % S if S > 64 else t % 2               # few samples: the small values come after the large one
        owners = [i for i in (base, base + XN_THREADS, base + 2 * XN_THREADS) if i < S]
        d[owners[0], j] = 3e4 + t
        d[owners[1:], j] = (1e-7 * rng.uniform(1, 2, len(owners) - 1)).astype(np.float32)
        others = rng.choice(S, min(S - 1, 300), replace=False)
        others = others[~np.isin(others, owners)]
        k = len(others) // 2 if S > 64 else len(others)
        d[others[:k], j] = (1e-7 * rng.uniform(1, 2, k)).astype(np.float32)
        if t % 2 and S > 64:
            d[others[-3:], j] = 2.9e4

    for t, j in enumerate(mixed):
        plant_mixed(t, j)
    n_full = 3 * S
    lg = math.ceil(math.log2(n_full))
    span_tiles = {T // 4: 52, T // 4 + 50: 53}
    for j, sp in span_tiles.items():
        _plant_span(d, j, [(11 + j) % S, (S - 3 - j) % S], sp, lg)
    for _ in range(8):                       # redraw a mixed tile where the two orders happen to give the same float64
        exp = orc.ic_xnorm(d.copy(), lens)
        tiles = [_tile_addends(d, exp, lens, j)[0] for j in mixed]
        same = [t for t, A in enumerate(tiles) if _seq_sum(A) == _order_free_sum(A)]
        if not same:
            break
        for t in same:
            plant_mixed(t, mixed[t])
    exp = _xnorm_compare(ctx, d, lens)
    # the checks that give the comparison its teeth, on the state the kernel saw at each tile
    for j in mixed:
        A, n = _tile_addends(d, exp, lens, j)
        assert _span(A, n) > 52, j
        assert _seq_sum(A) != _order_free_sum(A), j                   # the order-free path would give another float64
    for j, sp in span_tiles.items():
        A, n = _tile_addends(d, exp, lens, j)
        assert n == n_full and _span(A, n) == sp, (j, _span(A, n), sp)
    if engineered:
        for j, seq_skips in ((1, True), (3, False)):
            A, n = _tile_addends(d, exp, lens, j)
            s_star = _threshold(n)
            assert 52 < _span(A, n) <= 60, (j, _span(A, n))
            assert (_seq_sum(A) < s_star) == seq_skips and (_order_free_sum(A) < s_star) != seq_skips, j
            live = lens > j
            written = not np.array_equal(exp[live, j].view(np.uint32), d[live, j].view(np.uint32))
            assert written != seq_skips, j                             # the reference's decision shows in the output
    counts = [_tile_addends(d, exp, lens, j)[1] for j in (T - 3, T - 2, T - 1)]
    assert counts[1] == 3 * S - 4 and counts[0] > 3 * S - 4 and counts[2] < 3 * S - 4
    if S >= 1023:
        assert not np.array_equal(exp[:, T - 2].view(np.uint32), d[:, T - 2].view(np.uint32))   # n == 3S - 4 is normalised


@pytest.mark.parametrize("S", XN_S)
def test_xnorm_ragged_lengths_and_threshold(ctx, S):
    """Short samples (lengths 0..7: the 7-tap window's j > 2 && j < len - 3 and the neighbour terms' edges), alone on a
    thread that also owns a full-length sample, and in pairs on both owners of one thread.  Then tiles whose mean is the
    last float64 below 0.1 and the first one at or above it, on the order-free path."""
    rng = np.random.default_rng(100 + S)
    T = 40
    owner = 3 + XN_THREADS if S > 3 + XN_THREADS else S // 2
    cases = [{owner: L} for L in (0, 1, 2, 3, 4, 6, 7)]
    cases.append({3: 6, owner: 7} if owner != 3 else {3: 6, S - 1: 7})
    cases.append({3: 7, owner: 4} if owner != 3 else {3: 7, S - 1: 4})
    for short in cases:
        d = rng.uniform(0.25, 2.0, (S, T)).astype(np.float32)
        lens = np.full(S, T, np.int32)
        for i, L in short.items():
            lens[i] = L
            d[i, L:] = np.nan                                          # past a sample's end: never read
        _xnorm_compare(ctx, d, lens)
    # the 0.1 threshold on the order-free path: tiles 1 and 3 see only their own column, every sample holds c
    d = rng.uniform(0.25, 2.0, (S, 8)).astype(np.float32)
    d[:, [0, 2, 4]] = 0
    lens = np.full(S, 8, np.int32)
    n = 3 * S
    s_star = _threshold(n)
    c = np.float32(s_star / S)
    while float(c) * S >= s_star:
        c = np.nextafter(c, np.float32(0))
    while float(np.nextafter(c, np.float32(1))) * S < s_star:
        c = np.nextafter(c, np.float32(1))
    d[:, 1] = c                                                        # mean just below 0.1: skipped
    d[:, 3] = np.nextafter(c, np.float32(1))                           # just at or above: normalised
    exp = _xnorm_compare(ctx, d, lens)
    for j, skipped in ((1, True), (3, False)):
        A, nn = _tile_addends(d, exp, lens, j)
        assert nn == n and _span(A, nn) <= 52 and (_seq_sum(A) < s_star) == skipped
        assert np.array_equal(exp[:, j].view(np.uint32), d[:, j].view(np.uint32)) == skipped


# ------------------------------------------------------------------------------------------------ I2+I3 at 2504 samples
def test_cohort_2504_samples(ctx):
    """2504 samples of ~12 k tiles (chromosome 1 at 16 kb), shaped like synth_cohort, with an all-zero, an all-tie, a
    CRAM-run and a tie-heavy sample first: the host entry and the device entry against the oracle, bit for bit"""
    rng = np.random.default_rng(2504)
    S = 2504
    lens = rng.integers(11_500, 12_500, S)
    rows = [synth_cohort(rng, 1, int(n))[0] for n in lens]
    rows[0][:] = 0
    rows[1][:] = 123_456_789
    rows[2] = np.repeat(rng.integers(10_000, 90_000, lens[2] // 300 + 1), 300)[:lens[2]].astype(np.int64)
    rows[3] = rng.choice(np.array([0, 5, 7, 1_000_000_007], np.int64), lens[3])
    odd = 4                                                            # rows [0, odd) are not realistic samples
    sizes = np.concatenate(rows)
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    med, dep = ctx.indexcov_cohort(sizes, ptr)
    assert ctx.indexcov_cohort_fallbacks() <= odd
    d_sizes, d_ptr = ctx.dev_array(sizes), ctx.dev_array(ptr)
    d_med = ctx.dev_array(np.full(S, np.nan))
    d_dep = ctx.dev_array(np.full(sizes.size, np.nan, np.float32))
    d_ptr2 = ctx.dev_array(ptr[odd:])
    try:
        ctx.indexcov_cohort_device(d_sizes, d_ptr, S, d_med, d_dep)
        assert np.array_equal(d_med.download(np.float64, S), med)
        assert np.array_equal(d_dep.download(np.float32, sizes.size).view(np.uint32), dep.view(np.uint32))
        ctx.indexcov_cohort_device(d_sizes, d_ptr2, S - odd, d_med, None)     # the realistic samples alone
        assert ctx.indexcov_cohort_fallbacks() == 0
        assert np.array_equal(d_med.download(np.float64, S - odd), med[odd:])
    finally:
        for x in (d_sizes, d_ptr, d_med, d_dep, d_ptr2):
            x.free()
    for i, r in enumerate(rows):
        m = orc.ic_median(r)
        assert med[i] == float(m), (i, med[i], m)
        seg = dep[ptr[i]:ptr[i + 1]]
        if m != 0:
            assert np.array_equal(seg.view(np.uint32), orc.ic_normalize(r, float(m)).view(np.uint32)), i
        else:
            assert (seg == 0).all(), i


# ------------------------------------------------------------------------------------------------ I4-I6 device entries
def test_counts_segs_and_tokens_device(ctx):
    """gl_indexcov_counts_segs_device and gl_format_g3_device on the layout `goleft indexcov` hands them: 2504 samples back
    to back, 24 chromosomes each (every fifth one left out of the segments, as an excluded reference is), some samples
    short or empty on a chromosome"""
    rng = np.random.default_rng(24)
    S, R = 2504, 24
    chrom = (np.array([249, 242, 198, 190, 181, 171, 159, 145, 138, 134, 135, 133, 114, 107, 102, 90, 83, 80, 59, 64, 47, 51, 156, 57])
             * 12 // 10).astype(np.int64)                              # tiles per chromosome: 1.2 per Mb of the human one
    L = np.tile(chrom, (S, 1))
    short = rng.random((S, R)) < 0.05
    L[short] -= rng.integers(1, 20, int(short.sum()))
    L[rng.random((S, R)) < 0.01] = 0
    total = int(L.sum())
    dep = np.abs(rng.normal(1.0, 0.4, total)).astype(np.float32)
    dep[rng.random(total) < 0.02] = 0
    dep[rng.random(total) < 0.005] = 60000.0
    dep[rng.choice(total, 4000, replace=False)] = rng.choice(np.array([0.85, 1.15, 0.15, 8.0, 2.0 / 3.0], np.float32), 4000)
    off = np.concatenate([[0], np.cumsum(L.ravel())]).astype(np.int64)
    kept = [q for q in range(R) if q % 5 != 4]
    longest = L[:, kept].max(axis=0)
    seg_start = np.array([off[k * R + q] for k in range(S) for q in kept], np.int64)
    seg_len = np.array([L[k, q] for k in range(S) for q in kept], np.int64)
    seg_longest = np.tile(longest, S).astype(np.int64)
    nseg = seg_start.size
    bufs = [ctx.dev_array(dep), ctx.dev_array(seg_start), ctx.dev_array(seg_len), ctx.dev_array(seg_longest),
            ctx.dev_array(np.full(nseg * SLOTS, -1, np.int32)), ctx.dev_array(np.full(nseg * 4, -1, np.int64)),
            ctx.dev_array(np.full(total * 10, 0xEE, np.uint8))]
    d_dep, d_ss, d_sl, d_lg, d_c, d_b, d_tok = bufs
    try:
        ctx.indexcov_counts_segs_device(d_dep, d_ss, d_sl, d_lg, nseg, d_c, d_b)
        counts = d_c.download(np.int32, nseg * SLOTS).reshape(nseg, SLOTS)
        bins = d_b.download(np.int64, nseg * 4).reshape(nseg, 4)
        ctx.format_g3_device(d_dep, total, d_tok)
        tok = d_tok.download(np.uint8, total * 10).reshape(total, 10)
    finally:
        for x in bufs:
            x.free()
    kept_vals = np.concatenate([dep[s:s + n] for s, n in zip(seg_start, seg_len)])
    c2, b2 = ctx.indexcov_counts_batch(kept_vals, np.concatenate([[0], np.cumsum(seg_len)]), seg_longest)
    assert np.array_equal(counts, c2) and np.array_equal(bins, b2)
    for s in range(nseg):
        v = dep[seg_start[s]:seg_start[s] + seg_len[s]]
        assert np.array_equal(counts[s], orc.ic_counts(v)), s
        assert np.array_equal(bins[s], orc.ic_bins(v, int(seg_longest[s]))), s
    assert np.array_equal(tok, ctx.format_g3(dep))
    for v, t in zip(dep[-20_000:], tok[-20_000:]):                      # the last sample's tiles as printf writes them
        assert bytes(t[:t[9]]).decode() == "%.3g" % float(v), (float(v), bytes(t))


# ------------------------------------------------------------------------------------------------ PCA at the README's shape
def test_pca_2504_samples(ctx):
    """S = 2504: 20 x 20 Gram tiles, 210 CTAs over the upper triangle.  The Gram equals numpy's x @ x.T exactly; the
    projections follow the tolerance and "%.2f" rule of test_indexcov_pca_gpu"""
    rng = np.random.default_rng(2504)
    x = _planted(rng, 2504, 3000)
    _, _, _, g = ctx.indexcov_pca(x, want_gram=True)
    xf = x.astype(np.float64)
    assert np.array_equal(g, (xf @ xf.T).astype(np.int64))
    _check(ctx, x)


# ------------------------------------------------------------------------------------------------ the CLI at S = 1100
def run(*args, env=None):
    p = subprocess.run([GOLEFT, *args], capture_output=True, text=True, env=dict(os.environ, **env) if env else None)
    assert p.returncode == 0, p.stderr
    return p


@pytest.mark.parametrize("extranorm", [False, True])
def test_indexcov_cli_1100_samples(tmp_path, extranorm):
    """`goleft indexcov` on 1100 .bai files: -n normalises across more samples than one CTA has threads, the PCA has more
    than 8 x 128 samples.  .bed.gz, .roc and the .ped columns against the oracle; `--gpus 3` gives the same bytes."""
    refs, fai, paths, lin = cohort_bais(tmp_path, S=1100, seed=11)
    names = ["smp%d-rest" % k for k in range(len(paths))]
    outs = []
    for g in (1, 3):
        out = tmp_path / ("g%d" % g) / "tt"
        os.makedirs(str(out.parent))
        run("indexcov", "-d", str(out), "--gpus", str(g), "--fai", fai, *(["-n"] if extranorm else []), *paths,
            env={"GL_OVERSUBSCRIBE": "1"})
        outs.append([open(str(out / ("tt-indexcov." + ext)), "rb").read() for ext in ("bed.gz", "roc", "ped")])
    assert gzip.decompress(outs[0][0]) == gzip.decompress(outs[1][0]) and outs[0][1:] == outs[1][1:]
    out = tmp_path / "g1" / "tt"
    depths = oracle_depths(lin)
    rows, roc_txt, bins = expected_outputs(refs, depths, names, list(range(len(refs))), extranorm)
    assert gzip.decompress(outs[0][0]).decode().splitlines() == rows
    assert outs[0][1].decode() == roc_txt
    ped = read_ped(out)
    check_ped_columns(ped, refs, depths, bins)
    proj, sv, kk = expected_pcs(depths, [n for n, _ in refs], extranorm, {"1", "2", "GL000207.1"})
    assert kk == 5 and sv[4] > 0
    compare_pcs(ped, proj, kk)
