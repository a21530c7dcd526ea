"""gl_bam_covstats: the device sampler == the host sampler == the loop restated in Python, on every counter, on the three
sample arrays in file order and on every Stats field and H bit for bit; and `goleft covstats` over both routes."""
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import covstats_ref as cr  # noqa: E402
from goleft_b200 import capi  # noqa: E402

pytestmark = pytest.mark.gpu
GOLEFT = os.path.join(ROOT, "bin", "goleft")
KNOB = "GL_COVSTATS_BATCH_BYTES"


@pytest.fixture(scope="module")
def ctx():
    with capi.Ctx(0) as c:
        yield c


@pytest.fixture(autouse=True)
def _no_knob():
    os.environ.pop(KNOB, None)
    yield
    os.environ.pop(KNOB, None)


def compare(ctx, path, recs, mates, n, skip, expect_batches=None):
    """device == host == restatement; returns the device route's struct"""
    c, arrs = cr.restate(recs, mates, n, skip)
    bam = capi.Bam(path)
    try:
        res = []
        for fn in (capi.bam_covstats, capi.bam_covstats_host):
            try:
                res.append(fn(ctx, bam, n, skip, samples=True))
            except capi.GlError as e:
                assert e.code == capi.GL_EINVAL and 0 < c["n_insert"] < 3, str(e)
                res.append((e.stats, None, None))
        for st, H, got in res:
            for k, v in c.items():
                assert getattr(st, k) == v, (k, getattr(st, k), v, st.path)
            if got is not None:
                for a, b in zip(got, arrs):
                    assert np.array_equal(a, b), st.path
        (sd, Hd, _), (sh, Hh, _) = res
        assert sd.path == 1 and sh.path == 0
        for k in capi.CovStats.STATS:
            assert np.float64(getattr(sd, k)).tobytes() == np.float64(getattr(sh, k)).tobytes(), k
        if Hd is not None:
            exp, eH = cr.stats_numpy(c, *arrs)
            for k, v in exp.items():
                assert np.float64(getattr(sd, k)).tobytes() == np.float64(v).tobytes(), k
            assert Hd.tobytes() == Hh.tobytes() == eH.tobytes()
        if expect_batches is not None:
            assert sd.n_batches >= expect_batches
        return sd
    finally:
        bam.close()


CASES = {
    "cut_a": dict(n=300, skip=2000),
    "cut_b": dict(n=40, skip=500, flags=[0, 16, 0x400, 0x4 | 0x1, 0x100]),
    "eof_sampling": dict(n=10 ** 6, skip=1000),
    "eof_skip": dict(n=10, skip=10 ** 6),
    "n0": dict(n=0, skip=10),
    "skip0": dict(n=25, skip=0),
    "small_blocks": dict(n=500, skip=100, block=700),
    "tail_reached": dict(n=10 ** 6, skip=0, unplaced=400, block=5000),
    "cg_placeholder": dict(n=200, skip=50, cg_every=7),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_device_equals_host_and_restatement(ctx, tmp_path, case):
    kw = dict(CASES[case])
    n, skip, block = kw.pop("n"), kw.pop("skip"), kw.pop("block", 60000)
    refs, recs, mates = cr.records(np.random.default_rng(11), [9000, 0, 0, 4000, 2500, 0], unplaced=kw.pop("unplaced", 30), **kw)
    p = cr.write(tmp_path, "a.bam", refs, recs, mates, block=block)
    compare(ctx, p, recs, mates, n, skip)


def test_cut_b_does_not_apply_after_an_early_insert(ctx, tmp_path):
    refs, recs, mates = cr.records(np.random.default_rng(12), [6000, 3000], flags=[0, 16, 0x400])
    recs[120] = (recs[120][0], recs[120][1], 60, 99, [(100, "M")])
    mates[120] = (recs[120][1] + 300, 400)
    p = cr.write(tmp_path, "a.bam", refs, recs, mates)
    st = compare(ctx, p, recs, mates, 30, 100)                  # one insert among the first 2n lengths: 1 insert -> the panic code
    assert st.n_insert == 1 and st.n_records_read == len(recs)
    for k in (3, 5):                                            # and with three of them the sample runs to end of file with Stats
        recs[120 + k] = (recs[120 + k][0], recs[120 + k][1], 60, 99, [(100, "M")])
        mates[120 + k] = (recs[120 + k][1] + 310 + k, 410 + k)
    p = cr.write(tmp_path, "b.bam", refs, recs, mates)
    st = compare(ctx, p, recs, mates, 30, 100)
    assert st.n_insert == 3 and st.n_read_len == 60


def unit_starts(recs):
    """record indices where an index unit starts: the first record overlapping each 16 KB tile of each reference"""
    out, seen = set(), set()
    for i, r in enumerate(recs):
        if r[0] < 0:
            continue
        span = max(sum(l for l, op in r[4] if op in "MDN=X"), 1)
        end = r[1] + 1 if r[3] & 4 else r[1] + span
        for k in range(r[1] >> 14, ((end - 1) >> 14) + 1):
            if (r[0], k) not in seen:
                seen.add((r[0], k)); out.add(i)
    return out


@pytest.mark.parametrize("where", ["first_of_batch", "last_of_batch", "inside_unit"])
def test_cut_on_batch_and_unit_edges(ctx, tmp_path, where):
    """one unit per batch (the knob at 1 byte): n is chosen so that cut A's record is the first record of a unit, the last
    one, or neither"""
    refs, recs, mates = cr.records(np.random.default_rng(13), [5000, 3000], ref_len=200_000)
    p = cr.write(tmp_path, "a.bam", refs, recs, mates, block=4000)
    starts = unit_starts(recs)
    skip = 1500
    _, (_, ins, _) = cr.restate(recs, mates, 10 ** 6, skip)
    pick = None
    for n in range(20, len(ins)):
        c, _ = cr.restate(recs, mates, n, skip)
        i = c["n_records_read"] - 1
        ok = {"first_of_batch": i in starts, "last_of_batch": i + 1 in starts, "inside_unit": i not in starts and i + 1 not in starts}[where]
        if ok and c["n_insert"] == n:
            pick = n
            break
    assert pick is not None
    os.environ[KNOB] = "1"
    compare(ctx, p, recs, mates, pick, skip, expect_batches=3)
    os.environ[KNOB] = "20000"
    compare(ctx, p, recs, mates, pick, skip, expect_batches=2)


def run_cli(*args, env=None):
    return subprocess.run([GOLEFT, "covstats", *args], capture_output=True, env=dict(os.environ, **(env or {})))


def test_device_refuses_and_host_answers(ctx, tmp_path):
    """no index, and a BGZF member whose extra field has a subfield before BC (legal gzip, read by the host's block reader,
    not by the device route): GL_ESTATE from the device entry, the answer from the host entry, the CLI's row the same"""
    refs, recs, mates = cr.records(np.random.default_rng(14), [5000, 2000])
    good = cr.write(tmp_path, "good.bam", refs, recs, mates, block=20000)
    raw = open(good, "rb").read()
    noidx = str(tmp_path / "noidx.bam")
    open(noidx, "wb").write(raw)
    # rewrite the third member with a 4-byte subfield in front of BC; the members after it move by 4 bytes, so the index is
    # rebuilt by shifting every virtual offset behind it
    offs, q = [], 0
    while q < len(raw):
        offs.append(q)
        q += struct.unpack_from("<H", raw, q + 16)[0] + 1
    m0, m1 = offs[2], offs[3]
    mem = raw[m0:m1]
    new = mem[:10] + struct.pack("<H", 10) + b"XX\x00\x00" + mem[12:16] + struct.pack("<H", len(mem) + 4 - 1) + mem[18:]
    odd = str(tmp_path / "odd.bam")
    open(odd, "wb").write(raw[:m0] + new + raw[m1:])
    bai = bytearray(open(good + ".bai", "rb").read())

    def shift(v):
        return v + (4 << 16) if (v >> 16) >= m1 else v
    o = 8
    for _ in refs:
        nb = struct.unpack_from("<i", bai, o)[0]; o += 4
        for _ in range(nb):
            b, nc = struct.unpack_from("<Ii", bai, o); o += 8
            for k in range(nc * 2):
                if b != 37450 or k < 2:
                    struct.pack_into("<Q", bai, o + 8 * k, shift(struct.unpack_from("<Q", bai, o + 8 * k)[0]))
            o += 16 * nc
        nl = struct.unpack_from("<i", bai, o)[0]; o += 4
        for k in range(nl):
            struct.pack_into("<Q", bai, o + 8 * k, shift(struct.unpack_from("<Q", bai, o + 8 * k)[0]))
        o += 8 * nl
    open(odd + ".bai", "wb").write(bytes(bai))
    c, arrs = cr.restate(recs, mates, 200, 100)
    for path in (noidx, odd):
        bam = capi.Bam(path)
        with pytest.raises(capi.GlError) as e:
            capi.bam_covstats(ctx, bam, 200, 100)
        assert e.value.code == capi.GL_ESTATE
        st, H, got = capi.bam_covstats_host(ctx, bam, 200, 100, samples=True)
        assert all(getattr(st, k) == v for k, v in c.items()) and all(np.array_equal(a, b) for a, b in zip(got, arrs))
        bam.close()
    rows = [run_cli("-n", "200", p).stdout.split(b"\n")[1].split(b"\t")[:12] for p in (good, odd)]
    assert rows[0] == rows[1]


def test_cli_both_routes_and_hist(ctx, tmp_path):
    paths = []
    for k in range(3):
        refs, recs, mates = cr.records(np.random.default_rng(20 + k), [120_000 + 5000 * k, 3000], ref_len=3_000_000)
        paths.append(cr.write(tmp_path, "s%d.bam" % k, refs, recs, mates))
    a = run_cli("-n", "2000", "--hist", str(tmp_path / "d"), *paths)
    b = run_cli("-n", "2000", "--hist", str(tmp_path / "h"), *paths, env={"GL_GPU_FEED": "0"})
    plain = run_cli("-n", "2000", *paths)
    assert a.returncode == 0 and b.returncode == 0, (a.stderr, b.stderr)
    assert a.stdout == b.stdout == plain.stdout and a.stderr == b.stderr and a.stdout.count(b"\n") == 4
    bam = capi.Bam(paths[2])
    st, H = capi.bam_covstats(ctx, bam, 2000)
    bam.close()
    # the three BAMs share a sample name, so each call leaves the last BAM's histogram
    for pre in ("d", "h"):
        lines = open(str(tmp_path / (pre + ".S1.template_hist.tsv"))).read().splitlines()
        assert lines == ["%d\t%s" % (st.max_read_length + j, "NaN" if np.isnan(h) else "%.6g" % h) for j, h in enumerate(H)] and len(lines) > 10
    assert not (tmp_path / "s0.bam.S1.template_hist.tsv").exists()


def test_default_n_on_a_paired_bam(ctx, tmp_path):
    """the command's default -n 1000000 (and its skip of 100000) on a few million paired 150 bp records: several batches,
    the cut far into the file, device == host on everything"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import bench_covstats
    p = str(tmp_path / "big.bam")
    n_rec = bench_covstats.write_paired_bam(p, n_records=3_200_000, seed=3)
    bam = capi.Bam(p)
    sd, Hd, gd = capi.bam_covstats(ctx, bam, 1_000_000, 100_000, samples=True)
    sh, Hh, gh = capi.bam_covstats_host(ctx, bam, 1_000_000, 100_000, samples=True)
    bam.close()
    assert sd.n_insert == 1_000_000 and sd.n_records_read < n_rec and sd.n_batches >= 2
    for k in capi.CovStats.STATS + capi.CovStats.COUNTERS:
        assert np.float64(getattr(sd, k)).tobytes() == np.float64(getattr(sh, k)).tobytes(), k
    assert Hd.tobytes() == Hh.tobytes() and all(np.array_equal(a, b) for a, b in zip(gd, gh))
