"""goleft_b200 — H100 (sm_90a) engine for goleft's windowed-depth hot path.

The product is the C ABI in include/goleft_b200.h (libgoleft_b200.so) plus the C++ `goleft`
CLI; this package is the thin ctypes binding the tests and bench.py use.
"""
from . import capi  # noqa: F401  (raises ImportError if the shared library is not built)
from .capi import Ctx, GlError, device_count, version  # noqa: F401
