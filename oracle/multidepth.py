"""ctypes bindings of oracle/oracle_multidepth.c — TEST INFRASTRUCTURE ONLY (same rules as oracle/loader.py)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from oracle.loader import _proto, _ptr, _take, _vp, _i64p, lib

_proto("orc_md_chunk_size", C.c_int64, C.c_int64)
_proto("orc_md_min_samples", C.c_int64, C.c_double, C.c_int64)
_proto("orc_md_blocks", C.c_int64, _vp, C.c_int64, C.c_int64, C.c_int64, C.c_int64, C.c_int64, _vp, C.c_int64)
_proto("orc_md_mean_masked", C.c_double, _vp, _vp, C.c_int64, C.c_int64)
_proto("orc_md_chain", C.c_double, _vp, C.c_int64, C.c_int64)
_proto("orc_md_fmt2", C.c_int, C.c_double, C.c_char_p, C.c_int)
_proto("orc_md_chain_batch", None, _vp, _vp, _vp, _vp, C.c_int64, C.c_char_p, C.c_int)
_proto("orc_md_text", C.c_int, C.c_char_p, _vp, C.c_int64, C.c_int64, C.c_int64, C.c_double, C.c_int64, C.c_int64, C.c_int64,
       C.c_int64, _vp, C.POINTER(_vp), _i64p)


def chunk_size(S: int) -> int:
    return int(lib.orc_md_chunk_size(S))


def min_samples(frac: float, S: int) -> int:
    return int(lib.orc_md_min_samples(float(frac), S))


def blocks(cls, C_: int, max_skip: int = 10, min_size: int = 15, window: int = 10_000_000):
    """Blocks from a per-base site-class array (0 absent, 1 insufficient, 2 sufficient), chunk size C_ -> int64 (n, 3)."""
    cls = np.ascontiguousarray(cls, np.uint8)
    n = lib.orc_md_blocks(_ptr(cls), cls.size, C_, max_skip, min_size, window, None, 0)
    out = np.empty((n, 3), np.int64)
    lib.orc_md_blocks(_ptr(cls), cls.size, C_, max_skip, min_size, window, _ptr(out), n)
    return out


def chain(d, l: int) -> float:
    """acc += float64(d)/1000. in order, acc/float64(l)*1000."""
    d = np.ascontiguousarray(d, np.int32)
    return float(lib.orc_md_chain(_ptr(d), d.size, l))


def chain_batch(d, off, n, l):
    """"%.2f" of the chain for many cells (cell i = d[off[i]:off[i]+n[i]] over span l[i]) -> list of bytes"""
    d = np.ascontiguousarray(d, np.int32)
    off, n, l = (np.ascontiguousarray(a, np.int64) for a in (off, n, l))
    stride = 32
    buf = C.create_string_buffer(stride * max(off.size, 1))
    lib.orc_md_chain_batch(_ptr(d), _ptr(off), _ptr(n), _ptr(l), off.size, buf, stride)
    raw = buf.raw
    return [raw[i * stride:raw.index(b"\0", i * stride)] for i in range(off.size)]


def fmt2(v: float) -> bytes:
    b = C.create_string_buffer(64)
    n = lib.orc_md_fmt2(float(v), b, 64)
    return b.raw[:n]


def text(chrom: str, depth, mincov: int = 7, min_samples: float = 0.5, max_skip: int = 10, min_size: int = 15,
         window: int = 10_000_000, chunk: int = 0):
    """The reference's rows after the header for depth = S x L int32 per-base depths -> (bytes, site classes)."""
    depth = np.ascontiguousarray(depth, np.int32)
    S, L = depth.shape
    cls = np.empty(L, np.uint8)
    p, n = _vp(), C.c_int64(0)
    lib.orc_md_text(chrom.encode(), _ptr(depth), S, L, mincov, float(min_samples), max_skip, min_size, window, chunk, _ptr(cls),
                    C.byref(p), C.byref(n))
    return _take(p, n), cls
