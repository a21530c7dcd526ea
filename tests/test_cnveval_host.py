"""`goleft cnveval` without a GPU: the C oracle's walk against a second literal walk in Python and against the order-free form
the kernels compute; one hand case per quirk of the reference; gl_cnveval_order against the oracle's sort.Slice; Stat.String
text; the command's argument and parse errors."""
import math
import os
import subprocess

import numpy as np
import pytest

from cnveval_sets import HAND, order_free, random_set
from goleft_b200 import capi
from oracle import cnveval as oc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLEFT = os.path.join(ROOT, "bin", "goleft")


def test_c_oracle_equals_python_walk_and_order_free_form():
    rng = np.random.default_rng(1201)
    for k in range(2000):
        S, calls, truths, po = random_set(rng)
        c = oc.evaluate(S, calls, truths, po)
        assert np.array_equal(c, oc.evaluate_py(S, calls, truths, po)), k
        assert np.array_equal(c, order_free(S, calls, truths, po)), k


@pytest.mark.parametrize("case", HAND, ids=[h[0] for h in HAND])
def test_hand_case(case):
    _, S, calls, truths, po, want = case
    assert np.array_equal(oc.evaluate_py(S, calls, truths, po), want)
    assert np.array_equal(oc.evaluate(S, calls, truths, po), want)
    assert np.array_equal(order_free(S, calls, truths, po), want)


def test_fp_can_exceed_calls():
    """one FP-qualifying call opens a run over every later call up to b, for each truth the sample does not carry"""
    calls = [(0, 0, 0, 1000, 1)] + [(0, 0, 10 * i, 10 * i + 5, 1) for i in range(1, 20)]
    truths = [(0, 0, 1000, 1, [1]), (0, 0, 900, 1, [1])]
    st = oc.evaluate(2, calls, truths, 0.4)
    assert int(st[0, :, oc.FP].sum()) > len(calls)
    assert np.array_equal(st, oc.evaluate_py(2, calls, truths, 0.4))


def test_order_equals_oracle_sort_slice():
    rng = np.random.default_rng(1202)
    unstable = 0
    for k in range(2000):
        n = int(rng.integers(0, 80)) if k % 4 else int(rng.integers(13, 400))
        chrom = rng.integers(0, 3, n).astype(np.int32)
        start = rng.integers(0, int(rng.integers(1, 8)), n) * 100
        got = capi.cnveval_order(chrom, start)
        assert np.array_equal(got, oc.go_order(chrom, start)), k
        keys = list(zip(chrom.tolist(), start.tolist()))
        assert all(keys[got[i]] <= keys[got[i + 1]] for i in range(n - 1))
        stable = np.lexsort((np.arange(n), start, chrom))
        if n <= 12:
            assert np.array_equal(got, stable), k                # insertion sort
        else:
            unstable += not np.array_equal(got, stable)
    assert unstable > 0


def test_stat_string():
    assert oc.stat_string(0, 0, 0) == b"precision: NaN (0    / (0    + 0   )) recall: NaN (0    / (0    + 0   ))"
    # 1/32 = 0.03125 exactly: "%.4f" rounds the tie to even in Go and C alike
    assert oc.stat_string(1, 31, 0) == b"precision: 0.0312 (1    / (1    + 31  )) recall: 1.0000 (1    / (1    + 0   ))"
    assert oc.stat_string(3, 29, 0).startswith(b"precision: 0.0938 ")     # 3/32 = 0.09375 -> even
    assert oc.stat_string(123456, 7, 99999) == (b"precision: 0.9999 (123456 / (123456 + 7   )) "
                                                 b"recall: 0.5525 (123456 / (123456 + 99999))")
    t = oc.text(np.zeros((0, 3, 4), np.uint64))
    assert t.count(b"\n") == 4 and t.startswith(b"size-class: 0-20000      | precision: NaN")
    assert b"size-class: >=100000     |" in t and b"size-class: all          |" in t


def test_parse_rules():
    text = (b"#header\tx\n"
            b"chr1\t100\t200\t1\tA,B\r\n"
            b"chr1\t+5\t-3\t-1\t\n"
            b"chr2\t1\t2\t3\tC")                                      # no final newline: dropped
    recs = oc.parse(text)
    assert recs == [(b"chr1", 100, 200, 1, [b"A", b"B"]), (b"chr1", 5, -3, -1, [b""])]
    assert oc.parse(text, {b"B"}) == recs[:1]
    for bad in (b"chr1\t1\t2\t3\n", b"chr1\t1x\t2\t3\tA\n", b"chr1\t1\t2\t9223372036854775808\tA\n", b"\n"):
        with pytest.raises(oc.Panic):
            oc.parse(bad)


def test_limitsamples_and_first_sample():
    test = b"chr1\t100\t200\t1\tA,B\n"
    truth = b"chr1\t100\t200\t1\tB\n"
    # B is not the first sample of any test line: without -s the truth is A's other truth (one more FP); with -s it is gone
    assert oc.cnveval(truth, test).splitlines()[3].endswith(b"(0    / (0    + 2   )) recall: NaN (0    / (0    + 0   ))")
    assert oc.cnveval(truth, test, limit=True).splitlines()[3].endswith(b"(0    / (0    + 1   )) recall: NaN (0    / (0    + 0   ))")
    for limit in (False, True):
        for po in (0.4, math.nan, 1.0):
            assert oc.cnveval(truth, test, po, limit) == oc.cnveval(truth, test, po, limit, literal=True)


def _run(*args):
    return subprocess.run([GOLEFT, "cnveval", *args], capture_output=True)


@pytest.mark.skipif(not os.path.exists(GOLEFT), reason="bin/goleft not built")
def test_cli_argument_and_parse_errors(tmp_path):
    good = tmp_path / "good.bed"
    good.write_bytes(b"chr1\t100\t200\t1\tA\n")
    for m in ("0", "1.5", "-0.5", "x"):
        assert _run("-m", m, str(good), str(good)).returncode == 255, m
    assert _run(str(good)).returncode == 255
    bad = {"fields": b"chr1\t100\t200\t1\n", "int": b"chr1\t1e3\t200\t1\tA\n"}
    for name, text in bad.items():
        p = tmp_path / (name + ".bed")
        p.write_bytes(text)
        for args in ((str(good), str(p)), (str(p), str(good))):
            r = _run(*args)
            assert r.returncode == 2 and r.stderr.startswith(b"panic: ") or b"\npanic: " in r.stderr, (name, r.stderr)
    r = _run(str(good), str(tmp_path / "missing.bed"))
    assert r.returncode == 2 and b"panic: open" in r.stderr
