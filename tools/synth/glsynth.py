"""ctypes wrapper of tools/synth/libglsynth.so (glsynth.c): the bench's WGS-scale workload generator.
Stand-alone on purpose: both bench arms load it, and the reference arm must not import the product package."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libglsynth.so")

CHR20_LEN = 64_444_167
GRCH38 = [
    ("chr1", 248956422), ("chr2", 242193529), ("chr3", 198295559), ("chr4", 190214555), ("chr5", 181538259),
    ("chr6", 170805979), ("chr7", 159345973), ("chr8", 145138636), ("chr9", 138394717), ("chr10", 133797422),
    ("chr11", 135086622), ("chr12", 133275309), ("chr13", 114364328), ("chr14", 107043718), ("chr15", 101991189),
    ("chr16", 90338345), ("chr17", 83257441), ("chr18", 80373285), ("chr19", 58617616), ("chr20", 64444167),
    ("chr21", 46709983), ("chr22", 50818468), ("chrX", 156040895), ("chrY", 57227415), ("chrM", 16569),
]
SEED0 = 0x601EF7


def _lib():
    if not os.path.exists(_SO):
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-o", _SO, os.path.join(_HERE, "glsynth.c"),
                               os.path.join(_HERE, "bamsynth.c"), "-lpthread", "-lz"])
    lib = C.CDLL(_SO)
    lib.gls_segments.restype = C.c_int
    lib.gls_segments.argtypes = [C.c_int64, C.c_double, C.c_int, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                                 C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
    for fn in (lib.gls_write_bam, lib.gls_write_bam_csi):
        fn.restype = C.c_int
        fn.argtypes = [C.c_char_p, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.POINTER(C.c_int), C.c_double, C.c_int, C.c_int]
    return lib


def write_bam(path, contigs, coverage=30.0, read_len=150, threads=0, index="bai"):
    """contigs = [(name, length, contig_index)] -> path + path.bai holding EVERY read of the recipe (the filter is the
    decoder's job); segments(length, contig_index) are exactly what `samtools depth -Q 1` would count from it.
    index="csi": path.csi (min_shift 14, depth 5) instead of path.bai; the BAM is the same."""
    lib = _lib()
    n = len(contigs)
    names = (C.c_char_p * n)(*[c[0].encode() for c in contigs])
    lens = (C.c_int64 * n)(*[c[1] for c in contigs])
    seeds = (C.c_int * n)(*[c[2] for c in contigs])
    fn = {"bai": lib.gls_write_bam, "csi": lib.gls_write_bam_csi}[index]
    rc = fn(path.encode(), n, names, lens, seeds, coverage, read_len, threads or (os.cpu_count() or 1))
    if rc != 0:
        raise RuntimeError("gls_write_bam failed")


def segments(length, contig_index=0, coverage=30.0, read_len=150, min_mapq=1, gap=True, pileup=True, threads=0, alloc=None):
    """(start, end) int32 arrays in BAM record order.  alloc(n, dtype) -> array lets the caller supply pinned memory."""
    lib = _lib()
    threads = threads or (os.cpu_count() or 1)
    n = C.c_int64(0)
    seed = SEED0 + contig_index
    rc = lib.gls_segments(length, coverage, read_len, seed, min_mapq, int(gap), int(pileup), threads, None, None, 0, C.byref(n))
    if rc != 0:
        raise RuntimeError("gls_segments failed: %d" % rc)
    alloc = alloc or (lambda k, dt: np.empty(k, dt))
    s, e = alloc(n.value, np.int32), alloc(n.value, np.int32)
    rc = lib.gls_segments(length, coverage, read_len, seed, min_mapq, int(gap), int(pileup), threads, s.ctypes.data, e.ctypes.data,
                          n.value, C.byref(n))
    if rc != 0:
        raise RuntimeError("gls_segments failed: %d" % rc)
    return s, e
