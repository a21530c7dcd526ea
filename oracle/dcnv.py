"""ctypes bindings of oracle/oracle_dcnv.c and the text side of dcnv/dcnv.go (ReadRegions, addFromLine, main's writer) —
TEST INFRASTRUCTURE ONLY (same rules as oracle/loader.py)."""
from __future__ import annotations

import ctypes as C
import re

import numpy as np

from oracle.loader import _proto, _ptr, _take, _vp, _i64p, faidx_stats, lib

_proto("orc_go_argsort", None, _vp, C.c_int64, _vp)
_proto("orc_dcnv_debias", C.c_int, _vp, C.c_int64)
_proto("orc_dcnv_sample_median", C.c_int, _vp, C.c_int64, C.POINTER(C.c_double))
_proto("orc_dcnv_matrix", C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp, _vp)
_proto("orc_dcnv_rows", C.c_int, C.c_char_p, _vp, _vp, _vp, C.c_int64, C.c_int64, C.POINTER(_vp), _i64p)
_proto("orc_f2_mismatches", C.c_int64, _vp, C.c_int64, _vp, _i64p)


class Panic(ValueError):
    """Where the reference panics (the engine exits 2 with a message)."""


def argsort(v) -> np.ndarray:
    """floats.Argsort: Go's sort.Sort permutation"""
    v = np.ascontiguousarray(v, np.float64)
    inds = np.empty(v.size, np.int64)
    lib.orc_go_argsort(_ptr(v), v.size, _ptr(inds))
    return inds


def debias(col) -> np.ndarray:
    """GeneralDebiaser.Debias replayed literally on one GC-sorted column"""
    col = np.array(col, np.float64)
    if lib.orc_dcnv_debias(_ptr(col), col.size) != 0:
        raise Panic("fewer than 5 rows")
    return col


def sample_median(col) -> float:
    col = np.ascontiguousarray(col, np.float64)
    m = C.c_double(0)
    if lib.orc_dcnv_sample_median(_ptr(col), col.size, C.byref(m)) != 0:
        raise Panic("all-zero sample")
    return m.value


def matrix(x, gc):
    """Sort, Debias, Unsort, NormalizeBySampleMedian of the n x S matrix x -> (normalised, inds, medians)"""
    x = np.array(x, np.float64, order="C")
    n, S = x.shape
    gc = np.ascontiguousarray(gc, np.float64)
    inds, med = np.empty(n, np.int64), np.empty(S, np.float64)
    rc = lib.orc_dcnv_matrix(_ptr(x), n, S, _ptr(gc), _ptr(inds), _ptr(med))
    if rc == -1:
        raise Panic("fewer than 5 rows")
    if rc < -1:
        raise Panic("sample column %d is all zero" % (-2 - rc))
    return x, inds, med


def rows(label: bytes, starts, ends, x) -> bytes:
    x = np.ascontiguousarray(x, np.float64)
    starts, ends = np.ascontiguousarray(starts, np.int64), np.ascontiguousarray(ends, np.int64)
    p, n = _vp(), C.c_int64(0)
    lib.orc_dcnv_rows(label, _ptr(starts), _ptr(ends), _ptr(x), x.shape[0], x.shape[1], C.byref(p), C.byref(n))
    return _take(p, n)


def f2_mismatches(v, tokens):
    """(number of 16-byte tokens that differ from snprintf "%.2f", index of the first)"""
    v = np.ascontiguousarray(v, np.float64)
    tokens = np.ascontiguousarray(tokens, np.uint8)
    assert tokens.size == 16 * v.size
    first = C.c_int64(-1)
    bad = lib.orc_f2_mismatches(_ptr(v), v.size, _ptr(tokens), C.byref(first))
    return int(bad), first.value


_INT = re.compile(rb"[+-]?[0-9]+")                                       # strconv.Atoi
_FLOAT = re.compile(rb"[+-]?([0-9]+(\.[0-9]*)?|\.[0-9]+)([eE][+-]?[0-9]+)?")   # ParseFloat, decimal form
_WS = b" \t\n\r\x0b\x0c"


def _atoi(tok: bytes) -> int:
    if not _INT.fullmatch(tok):
        raise Panic("strconv.Atoi: parsing %r: invalid syntax" % tok)
    v = int(tok)
    if not 0 <= v < 1 << 32:
        raise Panic("coordinate %d outside uint32" % v)
    return v


def _atof(tok: bytes) -> float:
    if not _FLOAT.fullmatch(tok):
        raise Panic("strconv.ParseFloat: parsing %r: invalid syntax" % tok)
    v = float(tok)
    if np.isinf(v):
        raise Panic("strconv.ParseFloat: parsing %r: value out of range" % tok)
    return v


def parse_fai(fai: str):
    recs = {}
    for ln in fai.splitlines():
        f = ln.split("\t")
        recs[f[0]] = (int(f[2]), int(f[1]), int(f[3]), int(f[4]))
    return recs


def read_regions(text: bytes, fasta: bytes, recs):
    """ReadRegions: -> (samples, label, starts, ends, gc, x (n x S))"""
    lines = text.split(b"\n")[:-1]                                      # ReadString: a final line without "\n" is dropped
    samples, label, i = None, None, 0
    starts, ends, gcs, vals = [], [], [], []
    for ln in lines:
        line = ln + b"\n"
        if i == 0 and (line[:1] == b"#" or line.startswith(b"chrom")):
            f = line.strip(_WS).split(b"\t")
            if len(f) < 3:
                raise Panic("slice bounds out of range (header)")
            samples = f[3:]
            continue
        if i in (0, 1):
            if b"\t" not in line:
                raise Panic("slice bounds out of range (no tab)")
            label = line[:line.index(b"\t")]
        i += 1
        toks = line.split(b"\t")
        toks[-1] = toks[-1].strip(_WS)
        if len(toks) < 3:
            raise Panic("index out of range (fewer than 3 columns)")
        s, e = _atoi(toks[1]), _atoi(toks[2])
        s = max(s, 250)
        chrom = toks[0].decode()
        if chrom in recs:
            st = faidx_stats(fasta, recs[chrom], s - 250, e)
            if st is None:
                raise Panic("faidx: %s:%d-%d outside the sequence" % (chrom, s - 250, e))
            gc = st[0]
        else:
            gc = 0.0                                                    # the error is printed and zeros are used
        ns = len(samples) if samples is not None else 0
        if len(toks) - 3 != ns:
            raise Panic("row has %d values, header has %d samples" % (len(toks) - 3, ns))
        starts.append(s); ends.append(e); gcs.append(gc)
        vals.append([_atof(t) for t in toks[3:]])
    if not samples:
        raise Panic("no samples (integer divide by zero)")
    if len(vals) < 5:
        raise Panic("fewer than 5 rows")
    return samples, label, np.asarray(starts, np.int64), np.asarray(ends, np.int64), np.asarray(gcs, np.float64), \
        np.asarray(vals, np.float64).reshape(len(vals), len(samples))


def dcnv(text: bytes, fasta: bytes, fai: str) -> bytes:
    """The bytes of depth.bed for a depthwed matrix (text), a FASTA and its .fai text."""
    samples, label, starts, ends, gc, x = read_regions(text, fasta, parse_fai(fai))
    out, _, _ = matrix(x, gc)
    return b"#chrom\tstart\tend\t" + b"\t".join(samples) + b"\n" + rows(label, starts, ends, out)
