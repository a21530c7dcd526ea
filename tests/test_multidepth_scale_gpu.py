"""`goleft multidepth` at the limits it advertises (DESIGN §1.8): one contig of up to 2^30 - 1 bases, 1 to 65535 samples.

Each leg targets code the smaller tests never reach: contig ends at 32 / 4096 / 8192-base edges, the one-CTA scan of the
run counts past its first 1024 entries, a chromosome of 13 chunks, the top of the coordinate range, the 1 Mb chunks of
S > 50, the uint16 per-base counters at 32767 / 32768 / 65534 / 65535, coverage holes that do not line up across samples
(the count and sum epilogues only overwrite, nothing is cleared between samples), the float64 walk over a 10^7-site
block, Go's conversion of minSamples, and the CLI at S > 50.

Expectations are the literal site-by-site oracle (oracle/oracle_multidepth.c, `omd.text`) over per-base depths, byte for
byte.  Where a full S x L depth matrix is impractical, two references are made from oracle pieces and checked against the
full oracle on the CPU:
- the tail oracle (`_tail_text`): `omd.text` over [W0, L), W0 = one whole chunk before the chunk of the first read, with
  the run's chunk size, coordinates shifted back by W0.  A chunk that starts at or before W0 - C meets its first
  insufficient site beyond its kill point with an empty cache (sufficient sites before it are never cached), so it prints
  nothing; the chunk starting at W0 is not killed before W0 + C + 1, so it can still cache the first reads' sites, which
  is why the window starts there;
- the multiplicity reference (`_mult_text`): a cohort of a few distinct samples repeated with multiplicities; classes
  from counts weighted by multiplicity, `omd.blocks`, each distinct sample's "%.2f" from the oracle's chain, columns
  repeated.
Every GPU leg runs more than one segment form and asserts the depth path each sample's count pass took (packed8 host or
device -> 3, sorted device int32 -> fused 1, shuffled host int32 -> bucketed events 4).  The fused path takes unsorted
input as long as each tile's segments stay within a compact index range, so a small shuffled sample stays on it:
`events32` is the same shuffled input with the bucketed-events path chosen by gl_depth_set_path(4), and `shuffled32` is
used where the fused path rejects it and the reduce reruns on path 4."""
import os
import subprocess
import sys

import numpy as np
import pytest

from goleft_b200 import capi
from oracle import loader as orc
from oracle import multidepth as omd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLEFT = os.path.join(ROOT, "bin", "goleft")
CHROM = "chrT"
I64_MIN = -2 ** 63
TOP = (1 << 30) - 1                    # the longest contig gl_multidepth_begin accepts
RUN_CTA = 8192                         # bases per md_runs_* CTA
PATH = {"packed8": 3, "packed8_dev": 3, "device32": 1, "shuffled32": 4, "events32": 4}
gpu = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------- segments
def _reads(cov, seed, lo, hi, read_len=150):
    """sorted reads of read_len bases starting in [lo, hi - read_len) at coverage cov"""
    rng = np.random.default_rng(seed)
    n = int(cov * (hi - lo) / read_len)
    s = np.sort(rng.integers(lo, max(lo + 1, hi - read_len), n)).astype(np.int32)
    return s, s + np.int32(read_len)


def _tiles(a, b, d, step=100):
    """depth d over [a, b): d layers of step-base segments"""
    x = np.repeat(np.arange(a, b, step, dtype=np.int64), d)
    return x.astype(np.int32), np.minimum(x + step, b).astype(np.int32)


def _cat(*segs):
    """segments sorted by start"""
    segs = [x for x in segs if x[0].size]
    if not segs:
        return np.zeros(0, np.int32), np.zeros(0, np.int32)
    s, e = np.concatenate([x[0] for x in segs]), np.concatenate([x[1] for x in segs])
    o = np.argsort(s, kind="stable")
    return s[o].astype(np.int32), e[o].astype(np.int32)


def _depths(L, samples, rs=0):
    return np.stack([orc.pileup_diff(s, e, rs, L) for s, e in samples])


# ---------------------------------------------------------------------------------------------------- references
def go_min_samples(frac: float, S: int) -> int:
    """int(0.5 + MinSamples * S) as Go compiles it for amd64: trunc when 0.5 + x is in [-2^63, 2^63), else INT64_MIN"""
    x = np.float64(0.5) + np.float64(frac) * np.float64(S)
    if not (-2.0 ** 63 <= x < 2.0 ** 63):
        return I64_MIN
    return int(np.trunc(x))


def certified(total: int, n: int, l: int) -> bool:
    """host/md_cert.h in Python integers: does "%.2f" of the chain follow from round(100 Σd / l)?"""
    if n < 1 or l < 1 or l >= 1 << 31 or n > 1 << 40 or total >= 1 << 56:
        return False
    r = (100 * total) % l
    return (abs(2 * r - l) << 63) > 200 * total * (n + 2) * 1025


def runs_of(cls):
    st = np.flatnonzero(np.concatenate([[True], cls[1:] != cls[:-1]])).astype(np.int32)
    return st, cls[st]


def _block_sums(depth, cls, blk):
    """Σd over each block's sufficient sites, per sample -> (n_blocks, S) python ints"""
    suf = (cls == 2)
    out = []
    for row in depth:
        c = np.concatenate([[0], np.cumsum(np.where(suf, row, 0).astype(np.int64))])
        out.append(c[blk[:, 1]] - c[blk[:, 0]])
    return np.stack(out, 1) if out else np.zeros((len(blk), 0), np.int64)


def _uncertified(depth, cls, blk):
    sums = _block_sums(depth, cls, blk)
    return sum(not certified(int(sums[b, i]), int(blk[b, 2]), int(blk[b, 1] - blk[b, 0]))
               for b in range(len(blk)) for i in range(sums.shape[1]))


def _shift(text: bytes, off: int) -> bytes:
    rows = []
    for r in text.split(b"\n")[:-1]:
        f = r.split(b"\t", 3)
        rows.append(b"\t".join([f[0], b"%d" % (int(f[1]) + off), b"%d" % (int(f[2]) + off), f[3]]))
    return b"".join(x + b"\n" for x in rows)


def _tail_window(first: int, C: int) -> int:
    return (first // C - 1) * C


def _tail_text(L, samples, first, C, **kw):
    """(rows, site classes of [W0, L), W0, depths of [W0, L)) of a cohort whose reads all start at or after `first`"""
    w0 = _tail_window(first, C)
    assert w0 >= 0
    d = _depths(L, samples, rs=w0)
    t, cls = omd.text(CHROM, d, chunk=C, **kw)
    return _shift(t, w0), cls, w0, d


def _mult_classes(depths, mult, mincov, ms):
    cnt = np.zeros(depths.shape[1], np.int64)
    site = np.zeros(depths.shape[1], bool)
    for d, m in zip(depths, mult):
        if m:
            cnt += m * (d >= mincov)
            site |= d > 0
    return np.where(site, np.where(cnt > ms, 2, 1), 0).astype(np.uint8)


def _mult_text(depths, mult, mincov=7, frac=0.5):
    """rows of a cohort of sum(mult) samples: distinct sample k (depths[k]) repeated mult[k] times, in order"""
    S = int(sum(mult))
    cls = _mult_classes(depths, mult, mincov, omd.min_samples(frac, S))
    blk = omd.blocks(cls, omd.chunk_size(S))
    rows = []
    for s, e, _ in blk.tolist():
        sites = s + np.flatnonzero(cls[s:e] == 2)
        d = np.concatenate([dk[sites] for dk in depths])
        n = np.full(len(depths), sites.size, np.int64)
        tok = omd.chain_batch(d, np.arange(len(depths)) * sites.size, n, np.full(len(depths), e - s, np.int64))
        rows.append(b"%s\t%d\t%d" % (CHROM.encode(), s, e) + b"".join((b"\t" + t) * m for t, m in zip(tok, mult)) + b"\n")
    return b"".join(rows), cls, blk


def _same(got: bytes, exp: bytes, what=""):
    """byte equality, reported as the first differing row (the texts run to megabytes)"""
    if got == exp:
        return
    g, x = got.split(b"\n"), exp.split(b"\n")
    i = next((k for k in range(min(len(g), len(x))) if g[k] != x[k]), min(len(g), len(x)))
    pytest.fail("%s: %d rows, oracle %d; first difference at row %d:\n  got %r\n  exp %r"
                % (what, len(g) - 1, len(x) - 1, i, g[i][:300] if i < len(g) else None, x[i][:300] if i < len(x) else None))


# ---------------------------------------------------------------------------------------------------- the library run
def _adder(ctx, seg, form, keep):
    s, e = seg
    if form in ("packed8", "packed8_dev"):
        a, d, ln = capi.pack_segments8(s, e)
        if form == "packed8":
            keep.append((a, d, ln))
            return lambda c: c.depth_add_segments_packed8(a, d, ln)
        da, dd, dl = ctx.dev_array(a), ctx.dev_array(d), ctx.dev_array(ln)
        keep.append((da, dd, dl))
        return lambda c: c.depth_add_segments_packed8_device(da, dd, dl, a.size)
    if form == "device32":
        if s.size == 0:
            return lambda c: None
        ds, de = ctx.dev_array(s), ctx.dev_array(e)
        keep.append((ds, de))
        return lambda c: c.depth_add_segments_device(ds, de, s.size)
    assert form in ("shuffled32", "events32")
    p = np.random.default_rng(s.size).permutation(s.size)
    ss, ee = s[p].copy(), e[p].copy()
    keep.append((ss, ee))
    return lambda c: c.depth_add_segments(ss, ee)


def _expected_path(seg, form):
    """the path a sample's count pass must take (None for an empty sample).  The fused path rejects a tile only when its
    segments span more than 8 x their count + 4096 index entries, so it takes a shuffled sample of <= 4096 segments."""
    if seg[0].size == 0:
        return None
    return 1 if form == "shuffled32" and seg[0].size <= 4096 else PATH[form]


def _run(ctx, L, adders, mincov=7, min_samples=0.5, max_skip=10, min_size=15, window=10_000_000, chunk=0):
    """ctx.multidepth, step by step, keeping the path of every count pass -> (text, stats, paths, run starts, run classes)"""
    S = len(adders)
    ctx.multidepth_begin(L, S, mincov, min_samples)
    paths = []
    for add in adders:
        ctx.depth_begin(0, L)
        add(ctx)
        ctx.multidepth_count()
        paths.append(ctx.depth_last_path())
    rs, rc = ctx.multidepth_sites()
    bs, be, bn = capi.multidepth_blocks(rs, rc, L, S, max_skip, min_size, window, chunk)
    ctx.multidepth_set_blocks(bs, be, bn)
    for i, add in enumerate(adders):
        ctx.depth_begin(0, L)
        add(ctx)
        ctx.multidepth_sums(i)
    _, q, val, ok = ctx.multidepth_result(bs.size, S)
    return capi.multidepth_text(CHROM, bs, be, S, q, val, ok), ctx.multidepth_stats(), paths, rs, rc


def _check(ctx, L, samples, forms, exp, cls=None, what="", **kw):
    """run the cohort once per form (a str: every sample; a list: per sample) and compare with the oracle's rows and,
    when given, its site classes; returns the last run's stats"""
    for form in forms:
        fs = [form] * len(samples) if isinstance(form, str) else form
        keep = []
        adders = [_adder(ctx, seg, f, keep) for seg, f in zip(samples, fs)]
        ctx.depth_set_path(4 if form == "events32" else 0)
        try:
            got, st, paths, rs, rc = _run(ctx, L, adders, **kw)
        finally:
            ctx.depth_set_path(0)
        tag = "%s %s" % (what, form if isinstance(form, str) else "mixed")
        _same(got, exp, tag)
        for i, (seg, f) in enumerate(zip(samples, fs)):
            want = _expected_path(seg, f)
            assert want is None or paths[i] == want, (tag, i, paths[i], want)
        if cls is not None:
            es, ec = runs_of(cls)
            assert np.array_equal(rs, es) and np.array_equal(rc, ec), (tag, rs.size, es.size)
        del keep
    return st


# ---------------------------------------------------------------------------------------------------- 1. contig-length edges
EDGE_L = [1, 31, 32, 33, 4095, 4096, 4097, 8191, 8192, 8193, 12289]


def _edge_cohort(L, seed):
    """S = 3: a dense sample, a sparse one, and one whose only reads start in the contig's last tile; reads of 1-120
    bases anywhere in [0, L), so many overhang L"""
    rng = np.random.default_rng(seed)

    def rand(n, lo):
        s = np.sort(rng.integers(lo, L, n)).astype(np.int32)
        return s, (s + rng.integers(1, 121, n)).astype(np.int32)
    last_tile = (L - 1) // 4096 * 4096
    return [rand(max(12, L // 4), 0), rand(max(4, L // 14), 0), rand(10, max(last_tile, L - 150))]


@gpu
@pytest.mark.parametrize("L", EDGE_L)
def test_contig_length_edges(ctx, L):
    samples = _edge_cohort(L, L)
    assert samples[2][0].min() >= (L - 1) // 4096 * 4096 and max(int(x[1].max()) for x in samples) > L
    d = _depths(L, samples)
    for frac in (0.5, 0.2):
        exp, cls = omd.text(CHROM, d, min_samples=frac, min_size=3)
        _check(ctx, L, samples, ["packed8", "packed8_dev", "device32", "events32"], exp, cls, "L=%d f=%g" % (L, frac),
               min_samples=frac, min_size=3)
    assert (cls == 2).any() or L < 64


# ---------------------------------------------------------------------------------------------------- 2. the run scan past 1024 CTAs
def _scan_cohort(L):
    """S = 5 at coverages around MinCov (class runs in every 8192-base CTA), and the last base made a run of its own:
    samples 0-3 at depth 10 up to L - 1, sample 4 alone on the last base with a read overhanging L"""
    samples = [_reads(c, 500 + i, 0, L) for i, c in enumerate([6, 8, 7, 5, 9])]
    for i in range(4):
        samples[i] = _cat(samples[i], _tiles(L - 300, L - 1, 10))
    samples[4] = _cat(samples[4], (np.array([L - 1], np.int32), np.array([L + 100], np.int32)))
    return samples


@gpu
@pytest.mark.parametrize("L", [1024 * RUN_CTA, 1024 * RUN_CTA + 1])
def test_run_scan_past_1024_ctas(ctx, L):
    samples = _scan_cohort(L)
    exp, cls = omd.text(CHROM, _depths(L, samples))
    es, _ = runs_of(cls)
    ctas = (L + RUN_CTA - 1) // RUN_CTA
    assert np.unique(es // RUN_CTA).size == ctas                     # runs start in every run CTA
    assert es[-1] == L - 1
    _check(ctx, L, samples, ["packed8", "device32", "shuffled32"], exp, cls, "L=%d" % L)
    rs, rc = ctx.multidepth_sites()
    assert np.all(np.diff(rs) > 0)
    assert np.array_equal(np.repeat(rc, np.diff(np.append(rs, L))), cls)
    assert (rs < 1024 * RUN_CTA).any()
    if L > 1024 * RUN_CTA:                                           # the scan's second slice of 1024 counts
        assert rs[-1] == 1024 * RUN_CTA


# ---------------------------------------------------------------------------------------------------- 3. a chromosome
@gpu
def test_chromosome_chr20_length(ctx):
    sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
    import glsynth
    L = 64_444_167                                                    # chr20
    samples = [glsynth.segments(L, 40 + i, coverage=c) for i, c in enumerate([30, 5, 30, 5])]
    d = _depths(L, samples)
    exp, cls = omd.text(CHROM, d)
    del d
    assert (L + RUN_CTA - 1) // RUN_CTA == 7867 and (L + 4_999_999) // 5_000_000 == 13
    st = _check(ctx, L, samples, ["packed8", "device32"], exp, cls, "chr20")
    assert st["walked"] > 0 and st["certified"] > 0
    assert st["blocks"] == exp.count(b"\n")
    starts = np.array([int(r.split(b"\t")[1]) for r in exp.split(b"\n")[:-1]])
    assert np.unique(starts // 5_000_000).size == 13                  # blocks from every chunk


# ---------------------------------------------------------------------------------------------------- 4. the top of the range
def test_tail_oracle_equals_full_oracle():
    """the tail-oracle technique, on a 12 Mb contig with 1 Mb chunks: byte-identical to the full oracle"""
    L, C, first = 12_000_000, 1_000_000, 8_300_017
    samples = [_reads(c, 900 + i, first, L - 2000) for i, c in enumerate([14, 6, 12])]
    samples[0] = _cat(samples[0], (np.array([L - 40], np.int32), np.array([L + 60], np.int32)))
    exp, _ = omd.text(CHROM, _depths(L, samples), chunk=C)
    got, _, w0, _ = _tail_text(L, samples, first, C)
    assert w0 == 7_000_000 and exp.count(b"\n") > 100
    assert got == exp


def _top_cohort():
    """S = 3 with reads only in the last ~13.7 Mb of a 2^30 - 1 base contig, an exact tie in the last tile (sample 0:
    depth 10 over 200 bases but one at 11 -> 10.005) and reads overhanging L"""
    L = TOP
    first = 1_060_000_000 + 12_345
    samples = [_reads(c, 700 + i, first, L - 10_000) for i, c in enumerate([20, 12, 20])]
    tie = (L - 1) // 4096 * 4096 + 1000
    for i in range(3):
        samples[i] = _cat(samples[i], _tiles(tie, tie + 200, 10))
    samples[0] = _cat(samples[0], _tiles(tie + 7, tie + 8, 1), (np.array([L - 30], np.int32), np.array([L + 100], np.int32)))
    samples[1] = _cat(samples[1], _tiles(L - 5, L + 200, 8, step=205))
    samples[2] = _cat(samples[2], _tiles(L - 5, L + 200, 8, step=205))
    return L, first, tie, samples


@gpu
def test_top_of_range(ctx):
    L, first, tie, samples = _top_cohort()
    C = omd.chunk_size(3)
    exp, cls_w, w0, d = _tail_text(L, samples, first, C)
    blk = omd.blocks(cls_w, C)
    assert [tie - w0, tie + 200 - w0, 200] in blk.tolist()             # the planted tie is a block of its own
    assert exp.count(b"\n") > 100
    n_walk = _uncertified(d, cls_w, blk)
    n_tie = sum(1 for b in blk.tolist() if b[0] == tie - w0)
    assert n_walk >= n_tie >= 1
    ws, wc = runs_of(cls_w)
    assert wc[0] == 0 and ws[-1] + w0 == L - 30                        # [0, W0) holds no site; the overhang is the last run
    for form in ("packed8", "device32"):
        st = _check(ctx, L, samples, [form], exp, None, "2^30-1")
        rs, rc = ctx.multidepth_sites()
        assert rs[0] == 0 and rc[0] == 0
        assert np.array_equal(rs[1:], ws[1:] + w0) and np.array_equal(rc[1:], wc[1:]), form
        assert st["walked"] == n_walk and st["certified"] == 3 * len(blk) - n_walk


# ---------------------------------------------------------------------------------------------------- 5. more than 50 samples
def _big_cohort(S, L, seed):
    covs = [0 if i == 7 else (12 if i % 5 < 3 else 3) for i in range(S)]
    return [_reads(c, seed + i, 0, L) if c else (np.zeros(0, np.int32), np.zeros(0, np.int32)) for i, c in enumerate(covs)]


@gpu
@pytest.mark.parametrize("S", [51, 52, 64])
def test_more_than_50_samples(ctx, S):
    L = 3_456_789
    samples = _big_cohort(S, L, 10 * S)
    exp, cls = omd.text(CHROM, _depths(L, samples))
    rows = exp.split(b"\n")[:-1]
    starts = np.array([int(r.split(b"\t")[1]) for r in rows])
    ends = np.array([int(r.split(b"\t")[2]) for r in rows])
    assert ((starts // 1_000_000) != ((ends - 1) // 1_000_000)).any()  # blocks straddle chunk edges
    assert (starts[1:] < ends[:-1]).any()                              # and the next 1 Mb chunk prints their tail again
    _check(ctx, L, samples, ["packed8", "device32"], exp, cls, "S=%d" % S)


# ---------------------------------------------------------------------------------------------------- 6. the uint16 counters at their limit
MULT = [32767, 1, 32765, 1, 1]           # 65535 samples from 5 distinct ones


def _mult_cohort(L):
    """distinct samples over four regions: R1 only sample 0 (32767 samples reach MinCov), R2 also sample 1 (32768), R3
    also samples 2 and 4 (65534), R4 also sample 3 (65535); sample 4 has one low base first (an insufficient site)"""
    R = [(1000, 3000), (3100, 5300), (5400, 7700), (7800, 10_300)]
    cover = {0: [0, 1, 2, 3], 1: [1, 2, 3], 2: [2, 3], 3: [3], 4: [2, 3]}
    dep = [10, 12, 9, 8, 11]
    samples = []
    for k in range(5):
        parts = [_tiles(R[r][0], R[r][1], dep[k] + (r % 2)) for r in cover[k]]
        parts.append(_tiles(R[cover[k][0]][0] + 37, R[cover[k][0]][0] + 137, 3))       # means off the integers
        if k == 4:
            parts.append(_tiles(200, 201, 1))
        samples.append(_cat(*parts))
    return samples


def test_multiplicity_reference_equals_oracle():
    """the S = 65535 reference, at S = 60, equals the oracle on the expanded depth matrix"""
    L = 12_000
    samples = _mult_cohort(L)
    d = _depths(L, samples)
    mult = [20, 10, 15, 10, 5]
    full = np.repeat(d, mult, axis=0)
    for frac in (0.2, 0.5, 0.75, 49 / 60):
        exp, cls = omd.text(CHROM, full, min_samples=frac)
        got, gcls, _ = _mult_text(d, mult, frac=frac)
        assert np.array_equal(gcls, cls)
        assert got == exp and len(exp) > 0, frac


@gpu
def test_uint16_counters_at_65535_samples(ctx):
    L = 12_000
    samples = _mult_cohort(L)
    d = _depths(L, samples)
    cnt = sum(m * (dk >= 7) for dk, m in zip(d, MULT))
    assert {32767, 32768, 65534, 65535} <= set(np.unique(cnt).tolist())
    forms = ["device32", "packed8_dev", "device32", "packed8_dev", "device32"]
    keep = []
    distinct = [_adder(ctx, seg, f, keep) for seg, f in zip(samples, forms)]
    adders = [a for a, m in zip(distinct, MULT) for _ in range(m)]
    first = np.cumsum([0] + MULT[:-1])
    for frac, ms, lowest in ((32767 / 65535, 32767, 32768), (0.5, 32768, 65534), (65534 / 65535, 65534, 65535), (1.0, 65535, None)):
        exp, cls, blk = _mult_text(d, MULT, frac=frac)
        suf_counts = set(np.unique(cnt[cls == 2]).tolist())
        assert (min(suf_counts) if suf_counts else None) == lowest
        n_walk = sum(m for b in blk.tolist() for t, m in zip(_block_sums(d, cls, np.array([b]))[0], MULT)
                     if not certified(int(t), int(b[2]), int(b[1] - b[0])))
        got, st, paths, rs, rc = _run(ctx, L, adders, min_samples=frac)
        assert st["min_samples"] == ms
        es, ec = runs_of(cls)
        assert np.array_equal(rs, es) and np.array_equal(rc, ec), frac
        _same(got, exp, "S=65535 f=%r" % frac)
        assert [paths[i] for i in first] == [PATH[f] for f in forms]
        assert st["walked"] == n_walk and st["blocks"] == len(blk)
    del keep


# ---------------------------------------------------------------------------------------------------- 7. coverage holes that do not line up
def _holes_cohort(L, seed):
    """A on the first third, B empty, C on the middle third, D only base 0, E only the last base (its reads overhang
    L), F on the last third"""
    t = L // 3
    one = lambda x, d: (np.full(d, x, np.int32), np.full(d, x + 1, np.int32))          # noqa: E731
    return [_reads(10, seed, 0, t), (np.zeros(0, np.int32), np.zeros(0, np.int32)), _reads(12, seed + 1, t, 2 * t),
            one(0, 8), (np.full(8, L - 1, np.int32), np.full(8, L + 50, np.int32)), _reads(10, seed + 2, 2 * t, L)]


@gpu
@pytest.mark.parametrize("L", [5 * 4096 + 123, 9_000_011])
def test_coverage_holes(ctx, L):
    """min_samples 0: a site is sufficient when one sample reaches MinCov, so every sample's cells in the other samples'
    regions must read 0.00 — a pass that kept the previous sample's bits or slots would show there"""
    samples = _holes_cohort(L, L % 1000)
    exp, cls = omd.text(CHROM, _depths(L, samples), min_samples=0.0)
    assert cls[0] == 2 and cls[L - 1] == 2 and exp.count(b"\n") > 3
    forms = ["packed8", "packed8_dev", "device32", "events32"] + (["shuffled32"] if L > 1_000_000 else [])
    _check(ctx, L, samples, forms, exp, cls, "holes L=%d" % L, min_samples=0.0)


@gpu
def test_one_ctx_reused_across_contig_lengths():
    """9 Mb, then 50 kb, then 9 Mb again on one context: grow-only buffers and state left from a run change nothing"""
    cases = []
    for L in (9_000_011, 50_000):
        samples = _holes_cohort(L, 3)
        samples[1] = _reads(14, 77, 0, L)
        exp, cls = omd.text(CHROM, _depths(L, samples), min_samples=0.3)
        cases.append((L, samples, exp, cls))
    with capi.Ctx(0) as c:
        for L, samples, exp, cls in (cases[0], cases[1], cases[0]):
            _check(c, L, samples, ["packed8", "device32"], exp, cls, "reuse L=%d" % L, min_samples=0.3)


# ---------------------------------------------------------------------------------------------------- 8. walking long blocks
def _near_tie_depth(l: int, base: int):
    """extra bases x (at depth base + 1 over a block of l sites at depth base) for the largest distance |2r - l| from a
    tie that certify rejects, and for the next one, which it accepts -> (x_rejected, x_accepted)"""
    inv = pow(100, -1, l)
    prev = None
    for dist in range(1, 100_000, 2):
        x = ((l + dist) // 2 * inv) % l
        ok = certified(base * l + x, l, l)
        if ok:
            assert prev is not None
            return prev, x
        prev = x
    raise AssertionError("no certified distance")


def _walk_cohort():
    """S = 2.  An insufficient site at 100 (seen0).  Block A = [1000, 1000 + 10^7), the full default window: sample 0 at
    depth 15 with 50,000 bases at 16 (mean 15.005, an exact tie), sample 1 at 20.  Block B of l = 9,999,999 sites: each
    sample at 15 plus x bases at 16, x chosen so that sample 0's cell lies one step inside certify's bound (walked) and
    sample 1's one step outside (certified)."""
    a0, a1 = 1000, 1000 + 10 ** 7
    lb = 9_999_999
    b0 = a1 + 1000
    b1 = b0 + lb
    L = b1 + 1000
    x_rej, x_acc = _near_tie_depth(lb, 15)
    s0 = _cat(_tiles(100, 101, 1), _tiles(a0, a1, 15), _tiles(a0, a0 + 50_000, 1), _tiles(b0, b1, 15), _tiles(b0, b0 + x_rej, 1))
    s1 = _cat(_tiles(a0, a1, 20), _tiles(b0, b1, 15), _tiles(b0, b0 + x_acc, 1))
    return L, [s0, s1], (a0, a1), (b0, b1), (x_rej, x_acc)


def test_walk_cohort_plants():
    L, samples, (a0, a1), (b0, b1), (x_rej, x_acc) = _walk_cohort()
    lb = b1 - b0
    assert (200 * (15 * 10 ** 7 + 50_000)) % (2 * 10 ** 7) == 10 ** 7               # 100 mean = k + 1/2 exactly
    assert not certified(15 * 10 ** 7 + 50_000, 10 ** 7, 10 ** 7) and certified(20 * 10 ** 7, 10 ** 7, 10 ** 7)
    assert not certified(15 * lb + x_rej, lb, lb) and certified(15 * lb + x_acc, lb, lb)
    r_rej, r_acc = (100 * x_rej) % lb, (100 * x_acc) % lb
    assert abs(2 * r_acc - lb) == abs(2 * r_rej - lb) + 2


@gpu
def test_walk_long_blocks(ctx):
    L, samples, (a0, a1), (b0, b1), _ = _walk_cohort()
    exp, cls = omd.text(CHROM, _depths(L, samples))
    assert exp.startswith(b"%s\t%d\t%d\t15.0" % (CHROM.encode(), a0, a1)) and exp.count(b"\n") == 2
    assert b"\t%d\t%d\t" % (b0, b1) in exp
    st = _check(ctx, L, samples, ["packed8", "device32"], exp, cls, "walk")
    assert st["walked"] == 2 and st["certified"] == 2


# ---------------------------------------------------------------------------------------------------- 9. minSamples as Go converts it
FRACS3 = [float("nan"), float("inf"), float("-inf"), 1e300, -1e300, -1e9, 0.0, 0.5, 1.0, 1.0 + 2.0 ** -52]
FRACS1 = [-2147483649.5, -2147483648.5, -1.5]          # int(0.5 + f) = INT32_MIN - 1, INT32_MIN, -1


def test_min_samples_conversion_host():
    cases = [(f, 3) for f in FRACS3] + [(f, 1) for f in FRACS1]
    cases += [(f, S) for f in (2.0 ** 62, 2.0 ** 63, -2.0 ** 63, -2.0 ** 63 - 2048, 0.4999999999999999, -0.5, -0.7)
              for S in (1, 2, 65535)]
    for f, S in cases:
        assert omd.min_samples(f, S) == go_min_samples(f, S), (f, S)
    assert go_min_samples(float("nan"), 3) == I64_MIN and go_min_samples(-1e9, 3) == -2_999_999_999
    assert [go_min_samples(f, 1) for f in FRACS1] == [-2 ** 31 - 1, -2 ** 31, -1]
    # every site is sufficient when minSamples is INT64_MIN (count > minSamples always holds)
    d = np.array([[1, 0, 9], [0, 2, 0], [0, 0, 0]], np.int32)
    for f in (float("nan"), float("inf"), -1e300, -1e9):
        assert omd.text("c", d, min_samples=f)[1].tolist() == [2, 2, 2]


@gpu
def test_min_samples_conversion(ctx):
    L = 30_000
    cohort3 = [_reads(c, 60 + i, 0, L) for i, c in enumerate([14, 3, 9])]
    cohort1 = [_reads(5, 63, 0, L)]
    for samples, fracs in ((cohort3, FRACS3), (cohort1, FRACS1)):
        S = len(samples)
        d = _depths(L, samples)
        for f in fracs:
            exp, cls = omd.text(CHROM, d, min_samples=f)
            for form in ("packed8", "device32"):
                keep = []
                got, st, _, rs, rc = _run(ctx, L, [_adder(ctx, x, form, keep) for x in samples], min_samples=f)
                assert st["min_samples"] == go_min_samples(f, S), (f, S)
                es, ec = runs_of(cls)
                assert np.array_equal(rs, es) and np.array_equal(rc, ec), (f, S, form)
                _same(got, exp, "f=%r S=%d %s" % (f, S, form))
            if go_min_samples(f, S) < -1:
                assert (cls[cls > 0] == 2).all()


# ---------------------------------------------------------------------------------------------------- 10. the CLI at S > 50
@pytest.fixture(scope="module")
def bam_cohort(tmp_path_factory):
    if not os.path.exists(GOLEFT):
        pytest.skip("bin/goleft not built")
    sys.path.insert(0, os.path.join(ROOT, "tools", "synth"))
    import glsynth
    d = tmp_path_factory.mktemp("md52")
    L = 2_500_000
    paths, depths = [], []
    for i in range(52):
        p = str(d / ("s%02d.bam" % i))
        glsynth.write_bam(p, [("chrS", L, 300 + i)], coverage=4.0 if i % 3 == 1 else 10.0)
        seg = capi.bam_segments(p, min_mapq=10)["segments"].get(0, (np.zeros(0, np.int32), np.zeros(0, np.int32)))
        depths.append(orc.pileup_diff(seg[0], seg[1], 0, L))
        paths.append(p)
    return paths, np.stack(depths)


def _cli(paths, feed, *args):
    p = subprocess.run([GOLEFT, "multidepth", "-c", "chrS", *args, *paths], capture_output=True,
                       env=dict(os.environ, GL_GPU_FEED=feed))
    assert p.returncode == 0, p.stderr
    hdr, _, rows = p.stdout.partition(b"\n")
    assert hdr.startswith(b"#chrom\tstart\tend\t") and hdr.count(b"\t") == 2 + len(paths)
    return rows


@gpu
@pytest.mark.parametrize("feed", ["1", "0"])
def test_cli_52_bams(bam_cohort, feed):
    paths, depths = bam_cohort
    exp, _ = omd.text("chrS", depths)
    assert exp.count(b"\n") > 1000
    _same(_cli(paths, feed), exp, "cli feed=%s" % feed)


@gpu
def test_cli_minsamples_nan(bam_cohort):
    """`--minsamples nan` parses (as Go's ParseFloat does).  minSamples = INT64_MIN makes every site sufficient, so no
    chunk ever meets the insufficient site it starts caching after: the reference prints the header alone"""
    paths, depths = bam_cohort
    exp, cls = omd.text("chrS", depths[:3], min_samples=float("nan"))
    assert (cls[cls > 0] == 2).all() and exp == b""
    assert omd.text("chrS", depths[:3])[0].count(b"\n") > 0
    _same(_cli(paths[:3], "1", "--minsamples", "nan"), exp, "cli nan")
