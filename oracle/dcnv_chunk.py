"""ctypes bindings of oracle/oracle_dcnv_chunk.c (`goleft dcnv --chunk W`: ChunkDebiaser.Debias over the GC-sorted rows) and
the depth.bed text built from it as oracle/dcnv.py builds the default's — TEST INFRASTRUCTURE ONLY (same rules as
oracle/loader.py)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle.loader import _proto, _ptr, _vp, _i64p, lib
from oracle import dcnv as od

_proto("orc_dcnv_chunk_slices", None, _vp, C.c_int64, C.c_double, _vp, _i64p)
_proto("orc_dcnv_chunk_debias", None, _vp, C.c_int64, C.c_int64, _vp, C.c_int64)
_proto("orc_dcnv_chunk_matrix", C.c_int, _vp, C.c_int64, C.c_int64, _vp, C.c_double, _vp, _vp, _i64p, _vp)

Panic = od.Panic


def chunk_slices(vals, w: float) -> np.ndarray:
    """debiaser.go:133-141's slices over the sorted GC values vals"""
    vals = np.ascontiguousarray(vals, np.float64)
    out, m = np.empty(vals.size + 1, np.int64), C.c_int64(0)
    lib.orc_dcnv_chunk_slices(_ptr(vals), vals.size, float(w), _ptr(out), C.byref(m))
    return out[:m.value].copy()


def chunk_debias(x_sorted, slices) -> np.ndarray:
    """ChunkDebiaser.Debias on a copy of the n x S matrix whose rows are in GC order"""
    x = np.array(x_sorted, np.float64, order="C")
    if x.ndim == 1:
        x = x.reshape(-1, 1)
    slices = np.ascontiguousarray(slices, np.int64)
    lib.orc_dcnv_chunk_debias(_ptr(x), x.shape[0], x.shape[1], _ptr(slices), slices.size)
    return x


def matrix(x, gc, w: float):
    """Sort, ChunkDebiaser.Debias, Unsort, NormalizeBySampleMedian of the n x S matrix x -> (normalised, inds, slices,
    medians)"""
    x = np.array(x, np.float64, order="C")
    n, S = x.shape
    gc = np.ascontiguousarray(gc, np.float64)
    inds, slices, med, m = np.empty(n, np.int64), np.empty(n + 1, np.int64), np.empty(S, np.float64), C.c_int64(0)
    rc = lib.orc_dcnv_chunk_matrix(_ptr(x), n, S, _ptr(gc), float(w), _ptr(inds), _ptr(slices), C.byref(m), _ptr(med))
    if rc == -1:
        raise Panic("no rows")
    if rc < -1:
        raise Panic("sample column %d is all zero" % (-2 - rc))
    return x, inds, slices[:m.value].copy(), med


def dcnv(text: bytes, fasta: bytes, fai: str, w: float) -> bytes:
    """The bytes of depth.bed from `dcnv --chunk w` (no --svd) for a depthwed matrix (text), a FASTA and its .fai text."""
    samples, label, starts, ends, gc, x = od.read_regions(text, fasta, od.parse_fai(fai))
    out, _, _, _ = matrix(x, gc, w)
    return b"#chrom\tstart\tend\t" + b"\t".join(samples) + b"\n" + od.rows(label, starts, ends, out)


def values(text: bytes, fasta: bytes, fai: str, w: float):
    """-> (samples, label, starts, ends, the chunk-normalised n x S matrix)"""
    samples, label, starts, ends, gc, x = od.read_regions(text, fasta, od.parse_fai(fai))
    out, _, _, _ = matrix(x, gc, w)
    return samples, label, starts, ends, out
