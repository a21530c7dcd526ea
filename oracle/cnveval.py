"""ctypes bindings of oracle/oracle_cnveval.c, a second literal walk of cnveval/cnveval.go Evaluate in Python, and the
`cnveval` command's text side (cnveval/cmd/cnveval/cnveval.go: parseTruth, parseLine, Tabulate, Stat.String) —
TEST INFRASTRUCTURE ONLY (same rules as oracle/loader.py)."""
from __future__ import annotations

import ctypes as C
import math
import re

import numpy as np

from oracle.dcnv import Panic
from oracle.loader import _proto, _ptr, _vp, lib

_proto("orc_go_sort_calls", None, _vp, _vp, C.c_int64, _vp)
_proto("orc_cnveval", None, C.c_int32, _vp, _vp, _vp, _vp, _vp, C.c_int64, _vp, _vp, _vp, _vp, C.c_int64, _vp, _vp, C.c_double, _vp)

CLASSES = (b"0-20000", b"20000-100000", b">=100000", b"all")
TP, FP, FN, TN = range(4)


def go_order(chrom, start) -> np.ndarray:
    """the permutation Go 1.21's sort.Slice leaves for (chrom, start) keys in file order"""
    chrom, start = np.ascontiguousarray(chrom, np.int32), np.ascontiguousarray(start, np.int64)
    perm = np.empty(chrom.size, np.int64)
    lib.orc_go_sort_calls(_ptr(chrom), _ptr(start), chrom.size, _ptr(perm))
    return perm


def _arrays(calls, truths):
    """calls: [(sample, chrom, start, end, cn)]; truths: [(chrom, start, end, cn, [samples])] -> flat arrays"""
    c = np.asarray(calls, np.int64).reshape(-1, 5)
    mem_ptr = np.zeros(len(truths) + 1, np.int64)
    mem = []
    for i, t in enumerate(truths):
        mem += list(t[4])
        mem_ptr[i + 1] = len(mem)
    t = np.asarray([x[:4] for x in truths], np.int64).reshape(-1, 4)
    return (c[:, 0].astype(np.int32), c[:, 1].astype(np.int32), c[:, 2].copy(), c[:, 3].copy(), c[:, 4].copy(),
            t[:, 0].astype(np.int32), t[:, 1].copy(), t[:, 2].copy(), t[:, 3].copy(), mem_ptr, np.asarray(mem, np.int32))


def evaluate(S: int, calls, truths, po: float) -> np.ndarray:
    """the C oracle's CohortStats as uint64 (S, 3, 4): TP, FP, FN, TN per sample and size class"""
    return evaluate_arrays(S, *_arrays(calls, truths), po)


def evaluate_arrays(S: int, c_sample, c_chrom, c_start, c_end, c_cn, t_chrom, t_start, t_end, t_cn, mem_ptr, mem_sample,
                    po: float) -> np.ndarray:
    """evaluate() on flat arrays: calls in file order, truth t carries mem_sample[mem_ptr[t]:mem_ptr[t + 1]]"""
    i32 = [np.ascontiguousarray(a, np.int32) for a in (c_sample, c_chrom, t_chrom, mem_sample)]
    i64 = [np.ascontiguousarray(a, np.int64) for a in (c_start, c_end, c_cn, t_start, t_end, t_cn, mem_ptr)]
    out = np.zeros((S, 3, 4), np.uint64)
    lib.orc_cnveval(S, _ptr(i32[0]), _ptr(i32[1]), _ptr(i64[0]), _ptr(i64[1]), _ptr(i64[2]), i32[0].size, _ptr(i32[2]), _ptr(i64[3]),
                    _ptr(i64[4]), _ptr(i64[5]), i32[2].size, _ptr(i64[6]), _ptr(i32[3]), float(po), _ptr(out))
    return out


# ---------------------------------------------------------------- the walk again, in Python
def _size_class(s, e):
    n = e - s
    return 0 if n < 20000 else (1 if n < 100000 else 2)


def _same_cn(a, b):
    return min(a, 3) == min(b, 3)


def _poverlap(a, b):
    if a["chrom"] != b["chrom"]:
        return 0.0
    total = min(float(a["end"] - a["start"]), float(b["end"] - b["start"]))
    ovl = min(a["end"], b["end"]) - max(a["start"], b["start"])
    if ovl < 0:
        return 0.0
    return float(ovl) / total if total != 0 else (math.nan if ovl == 0 else math.inf)


def _sort_slice(recs):
    p = go_order([r["chrom"] for r in recs], [r["start"] for r in recs])
    return [recs[i] for i in p]


def evaluate_py(S: int, calls, truths, po: float) -> np.ndarray:
    """Evaluate / updatePositive / updateFP (cnveval.go:163-341), literally, with plain Python integers"""
    st = np.zeros((S, 3, 4), np.uint64)
    for s in range(S):
        own = [dict(chrom=t[0], start=t[1], end=t[2], cn=t[3]) for t in truths for x in t[4] if x == s]
        others = [dict(chrom=t[0], start=t[1], end=t[2], cn=t[3]) for t in truths if s not in t[4]]
        cnvs = [dict(chrom=c[1], start=c[2], end=c[3], cn=c[4], counted=False) for c in calls if c[0] == s]
        own, cnvs = _sort_slice(own), _sort_slice(cnvs)
        if not cnvs:
            continue
        i = 0
        for t in own:                                                     # updatePositive
            found, used = False, False
            val = st[s, _size_class(t["start"], t["end"])]
            while i < len(cnvs) and (cnvs[i]["chrom"] < t["chrom"] or (cnvs[i]["chrom"] == t["chrom"] and cnvs[i]["end"] < t["start"])):
                i += 1
            if i > 0:
                i -= 1
            for cnv in cnvs[i:]:
                if cnv["chrom"] > t["chrom"] or (cnv["chrom"] == t["chrom"] and cnv["start"] > t["end"]):
                    break
                if _poverlap(cnv, t) >= po and _same_cn(cnv["cn"], t["cn"]) and not used:
                    val[TP] += 1
                    cnv["counted"] = found = used = True
            if not found:
                val[FN] += 1
        for cnv in cnvs:
            if not cnv["counted"]:
                st[s, _size_class(cnv["start"], cnv["end"]), FP] += 1
        others = _sort_slice(others)
        i = 0
        for o in others:                                                  # updateFP
            val = st[s, _size_class(o["start"], o["end"])]
            while i < len(cnvs) and (cnvs[i]["chrom"] < o["chrom"] or (cnvs[i]["chrom"] == o["chrom"] and cnvs[i]["end"] < o["start"])):
                i += 1
            if i > 0:
                i -= 1
            tpfound = fpfound = found = False
            for cnv in cnvs[i:]:
                if cnv["chrom"] > o["chrom"] or (cnv["chrom"] == o["chrom"] and cnv["start"] > o["end"]):
                    break
                if _poverlap(cnv, o) >= po and _same_cn(cnv["cn"], o["cn"]):
                    fpfound = True
                    for t in own:
                        if t["chrom"] != cnv["chrom"]:
                            continue
                        if _poverlap(cnv, t) >= po and _same_cn(cnv["cn"], t["cn"]):
                            tpfound = True
                            break
                if fpfound and not tpfound:
                    val[FP] += 1
                    found = True
            if not (found or tpfound):
                val[TN] += 1
    return st


# ---------------------------------------------------------------- the command's text side
_INT = re.compile(rb"[+-]?[0-9]+")


def _atoi(tok: bytes) -> int:
    """strconv.Atoi: optional sign, decimal digits, int64 range"""
    if not _INT.fullmatch(tok):
        raise Panic("strconv.Atoi: parsing %r: invalid syntax" % tok)
    v = int(tok)
    if not -(1 << 63) <= v < 1 << 63:
        raise Panic("strconv.Atoi: parsing %r: value out of range" % tok)
    return v


def parse(text: bytes, samples=None):
    """parseTruth: -> [(chrom bytes, start, end, cn, [sample bytes])]"""
    out = []
    for ln in text.split(b"\n")[:-1]:                                     # ReadString: a final line without "\n" is dropped
        line = ln + b"\n"
        if line[:1] == b"#":
            continue
        toks = line.rstrip(b"\r\n").split(b"\t")
        if len(toks) < 5:
            raise Panic("expected five fields for CNVs")
        rec = (toks[0], _atoi(toks[1]), _atoi(toks[2]), _atoi(toks[3]), toks[4].split(b","))
        if samples is not None and not any(s in samples for s in rec[4]):
            continue
        out.append(rec)
    return out


def _go_f4(v: float) -> bytes:
    return b"NaN" if math.isnan(v) else b"%.4f" % v


def stat_string(tp: int, fp: int, fn: int) -> bytes:
    """Stat.String (cnveval.go:93-96)"""
    p = float(tp) / float(tp + fp) if tp + fp else math.nan
    r = float(tp) / float(tp + fn) if tp + fn else math.nan
    return b"precision: %s (%-4d / (%-4d + %-4d)) recall: %s (%-4d / (%-4d + %-4d))" % (_go_f4(p), tp, tp, fp, _go_f4(r), tp, tp, fn)


def tabulate(stats) -> np.ndarray:
    """CohortStats.Tabulate: (4, 4) TP, FP, FN, TN for the three classes and all"""
    t = np.zeros((4, 4), np.uint64)
    t[:3] = np.asarray(stats, np.uint64).reshape(-1, 3, 4).sum(axis=0)
    t[3] = t[:3].sum(axis=0)
    return t


def text(stats) -> bytes:
    t = tabulate(stats)
    return b"".join(b"size-class: %-12s | %s\n" % (CLASSES[i], stat_string(int(t[i, TP]), int(t[i, FP]), int(t[i, FN])))
                    for i in range(4))


def cnveval(truth_text: bytes, test_text: bytes, po: float = 0.4, limit: bool = False, literal: bool = False) -> bytes:
    """stdout of `cnveval [-m po] [-s] truth.bed test.bed` (literal: the Python walk instead of the C one)"""
    tests = parse(test_text)
    samples = {t[4][0] for t in tests} if limit else None
    truths = parse(truth_text, samples)
    chroms = sorted({r[0] for r in tests} | {r[0] for r in truths})      # ranks in bytewise order
    rank = {c: i for i, c in enumerate(chroms)}
    names = {}
    for r in truths:
        for s in r[4]:
            names.setdefault(s, len(names))
    for r in tests:
        names.setdefault(r[4][0], len(names))
    calls = [(names[r[4][0]], rank[r[0]], r[1], r[2], r[3]) for r in tests]
    tr = [(rank[r[0]], r[1], r[2], r[3], [names[s] for s in r[4]]) for r in truths]
    return text((evaluate_py if literal else evaluate)(len(names), calls, tr, po))
