"""ctypes binding of libgoleft_b200.so (the C ABI in include/goleft_b200.h).

This is what tests/ and bench.py call; it adds nothing but argument marshalling.  There is no
CPU fallback: if the shared library is missing the import fails, and every call on a box
without a CUDA device raises GlError (GL_ECUDA).
"""
from __future__ import annotations

import ctypes as C
import os
import time
from concurrent.futures import ThreadPoolExecutor
from typing import Optional, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# GOLEFT_B200_LIB: another build of the same library (A/B runs); tests and bench use the default
LIB_PATH = os.environ.get("GOLEFT_B200_LIB") or os.path.join(_HERE, "libgoleft_b200.so")

GL_OK, GL_EINVAL, GL_ECUDA, GL_ENOMEM, GL_ESTATE, GL_ERANGE, GL_ENCCL = 0, -1, -2, -3, -4, -5, -6
CLASS_NAMES = ("NO_COVERAGE", "LOW_COVERAGE", "CALLABLE", "EXCESSIVE_COVERAGE")
INDEXCOV_SLOTS = 70


class GlError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"goleft_b200 error {code}: {msg}")
        self.code = code


def _load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: build it with `make lib` (or __graft_entry__.build()); "
            "goleft_b200 has no CPU fallback")
    return C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)


lib = _load()

_i32p = C.POINTER(C.c_int32)
_i64p = C.POINTER(C.c_int64)
_u8p = C.POINTER(C.c_uint8)
_u64p = C.POINTER(C.c_uint64)
_f32p = C.POINTER(C.c_float)
_f64p = C.POINTER(C.c_double)
_vp = C.c_void_p


def _proto(name, restype, *argtypes):
    fn = getattr(lib, name)
    fn.restype = restype
    fn.argtypes = list(argtypes)
    return fn


_proto("gl_version", C.c_char_p)
_proto("gl_device_count", C.c_int, C.POINTER(C.c_int))
_proto("gl_ctx_create", C.c_int, C.c_int, C.POINTER(_vp))
_proto("gl_ctx_destroy", C.c_int, _vp)
_proto("gl_last_error", C.c_char_p, _vp)
_proto("gl_sync", C.c_int, _vp)
_proto("gl_launch_count", C.c_int, _vp, _i64p)
_proto("gl_stream_handle", C.c_int, _vp, _u64p)
_proto("gl_dev_alloc", C.c_int, _vp, C.c_int64, C.POINTER(_vp))
_proto("gl_dev_free", C.c_int, _vp, _vp)
_proto("gl_host_alloc_pinned", C.c_int, _vp, C.c_int64, C.POINTER(_vp))
_proto("gl_host_free_pinned", C.c_int, _vp, _vp)
_proto("gl_memcpy_h2d", C.c_int, _vp, _vp, _vp, C.c_int64)
_proto("gl_memcpy_d2h", C.c_int, _vp, _vp, _vp, C.c_int64)
_proto("gl_timer_start", C.c_int, _vp)
_proto("gl_timer_stop_ms", C.c_int, _vp, C.POINTER(C.c_float))
_proto("gl_flush_l2", C.c_int, _vp)
_proto("gl_profile_enable", C.c_int, _vp, C.c_int)
_proto("gl_profile_read", C.c_int, _vp, _vp, C.c_int64, _i64p)

_proto("gl_bind_numa_for_device", C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int))
_proto("gl_device_numa_node", C.c_int, C.c_int, C.POINTER(C.c_int))
_proto("gl_lpt_assign", C.c_int, _vp, C.c_int32, C.c_int32, _vp, _vp)
_proto("gl_depth_begin", C.c_int, _vp, C.c_int64, C.c_int64)
_proto("gl_depth_add_segments", C.c_int, _vp, _vp, _vp, C.c_int64)
_proto("gl_depth_add_segments_device", C.c_int, _vp, _vp, _vp, C.c_int64)
_proto("gl_depth_reduce", C.c_int, _vp, C.c_int32, C.c_int32, C.c_int32, C.c_int64)
_proto("gl_depth_result_sizes", C.c_int, _vp, _i64p, _i64p, _i32p)
_proto("gl_depth_get_windows", C.c_int, _vp, _vp, C.c_int64)
_proto("gl_depth_last_path", C.c_int, _vp, _i32p)
_proto("gl_depth_set_path", C.c_int, _vp, C.c_int32)
_proto("gl_depth_get_runs", C.c_int, _vp, _vp, _vp, _vp, C.c_int64)
_proto("gl_depth_windows", C.c_int, _vp, C.c_int32, _vp, _vp, C.c_int64)
_proto("gl_depth_classes", C.c_int, _vp, C.c_int32, C.c_int32, _vp, _vp, _vp, C.c_int64, _i64p)
_proto("gl_depth_perbase", C.c_int, _vp, _vp)
_proto("gl_depth_interval_sums", C.c_int, _vp, _vp, _vp, C.c_int64, _vp)
_proto("gl_fasta_load", C.c_int, _vp, _vp, C.c_int64)
_proto("gl_fasta_stats", C.c_int, _vp, _vp, _vp, C.c_int64, _vp, _vp)
_proto("gl_depth_chunk_rows", C.c_int, C.c_int64, C.c_int64, C.c_int32, _vp, _vp, C.c_int64, _vp, _vp, C.c_int64, _i64p)
_proto("gl_depth_region", C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp, C.c_int64, C.c_int32, C.c_int32,
       C.c_int32, C.c_int64, _vp, C.c_int64, _i64p, _vp, _vp, C.c_int64, _i64p)
_proto("gl_indexcov_sizes", C.c_int, _vp, _vp, _vp, C.c_int32, _vp, _vp)
_proto("gl_indexcov_scale", C.c_int, _vp, _vp, C.c_int64, _i64p)
_proto("gl_indexcov_normalize", C.c_int, _vp, _vp, C.c_int64, C.c_double, _vp)
_proto("gl_indexcov_cohort", C.c_int, _vp, _vp, _vp, C.c_int32, _vp, _vp)
_proto("gl_indexcov_cohort_device", C.c_int, _vp, _vp, _vp, C.c_int32, _vp, _vp)
_proto("gl_indexcov_cohort_fallbacks", C.c_int, _vp, _i32p)
_proto("gl_indexcov_sizes_batch_device", C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_int64, _vp)
_proto("gl_indexcov_counts", C.c_int, _vp, _vp, C.c_int64, _vp)
_proto("gl_indexcov_bins", C.c_int, _vp, _vp, C.c_int64, C.c_int64, _vp)
_proto("gl_indexcov_counts_batch", C.c_int, _vp, _vp, _vp, _vp, C.c_int32, _vp, _vp)
_proto("gl_indexcov_counts_batch_device", C.c_int, _vp, _vp, _vp, _vp, C.c_int32, _vp, _vp)
_proto("gl_indexcov_counts_segs_device", C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_int32, _vp, _vp)
_proto("gl_indexcov_xnorm", C.c_int, _vp, _vp, _vp, C.c_int32, C.c_int32)
_proto("gl_indexcov_pca_total", C.c_int, _vp, C.c_int64, C.c_int32, C.c_int64, _f64p)
_proto("gl_plot_select_device", C.c_int, _vp, _vp, _vp, _vp, C.c_int32, _vp, _vp)
_proto("gl_plot_select_host", C.c_int, _vp, _vp, _vp, C.c_int32, _vp, _vp)
_proto("gl_plot_transform", C.c_int, _vp, C.c_int32, C.c_int32, _vp)
_proto("gl_plot_line_radius", C.c_double, C.c_int32)
_proto("gl_plot_raster_series_device", C.c_int, _vp, _vp, _vp, _vp, C.c_double, _vp, _vp, C.c_int32, _vp, C.c_int32, C.c_int32,
       C.c_int32, C.c_double, _vp)
_proto("gl_plot_raster_series_host", C.c_int, _vp, _vp, _vp, C.c_double, _vp, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32,
       C.c_double, _vp)
_proto("gl_plot_raster_xy", C.c_int, _vp, _vp, _vp, _vp, _vp, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, C.c_double, _vp)
_proto("gl_plot_raster_xy_host", C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, C.c_double, _vp)
_proto("gl_plot_color", None, C.c_int32, C.c_int32, _vp)
_proto("gl_plot_ticks", C.c_int, C.c_double, C.c_double, _vp, C.c_int32, _i32p)
_proto("gl_plot_millions", C.c_int, C.c_double, C.c_char_p, C.c_int32)
_proto("gl_plot_text", C.c_int, _vp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_char_p, C.c_int32)
_proto("gl_plot_compose", C.c_int, _vp, _vp, C.c_int32, C.c_int32, _vp, C.c_char_p, C.c_char_p, _vp)
_proto("gl_plot_png", C.c_int, _vp, C.c_int32, C.c_int32, _vp, C.c_int64, _i64p)
_proto("gl_plot_path_series_size", C.c_int, _vp, _vp, _vp, _vp, C.c_double, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, _vp, _vp)
_proto("gl_plot_path_series_emit", C.c_int, _vp, _vp, _vp, _vp, C.c_double, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, _vp,
       C.c_int64, _vp, C.c_int64)
_proto("gl_plot_path_series_size_host", C.c_int, _vp, _vp, _vp, C.c_double, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, _vp, _vp)
_proto("gl_plot_path_series_emit_host", C.c_int, _vp, _vp, _vp, C.c_double, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, _vp, _vp,
       C.c_int64)
_proto("gl_plot_path_xy_size", C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, _vp, _vp)
_proto("gl_plot_path_xy_emit", C.c_int, _vp, _vp, _vp, _vp, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, _vp, C.c_int64, _vp, C.c_int64)
_proto("gl_plot_path_xy_size_host", C.c_int, _vp, _vp, _vp, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, _vp, _vp)
_proto("gl_plot_path_xy_emit_host", C.c_int, _vp, _vp, _vp, _vp, C.c_int32, _vp, C.c_int32, C.c_int32, C.c_int32, _vp, _vp, C.c_int64)
_proto("gl_plot_line_width", C.c_double, C.c_int32)
_proto("gl_plot_vector_write", C.c_int, C.c_char_p, C.c_int32, C.c_int32, _vp, C.c_char_p, C.c_char_p, C.c_int32, _vp, C.c_double,
       C.POINTER(C.c_char_p), _vp)
_proto("gl_format_g3", C.c_int, _vp, _vp, C.c_int64, _vp)
_proto("gl_format_g3_device", C.c_int, _vp, _vp, C.c_int64, _vp)
_proto("gl_bincount_i32", C.c_int, _vp, _vp, C.c_int64, C.c_int32, C.c_int32, _vp)
_proto("gl_bam_covstats", C.c_int, _vp, _vp, C.c_int32, C.c_int32, _vp, _vp, C.c_int64)
_proto("gl_bam_covstats_host", C.c_int, _vp, _vp, C.c_int32, C.c_int32, _vp, _vp, C.c_int64)
_proto("gl_bam_covstats_prefetch", C.c_int, _vp, _vp, C.c_int32, C.c_int32)
_proto("gl_bam_covstats_samples", C.c_int, _vp, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp))
_proto("gl_bam_covstats_host_samples", C.c_int, _vp, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp))
_proto("gl_covstats_tail", C.c_int, _vp, _vp, C.c_int64, _vp, C.c_int64, _vp, C.c_int64, _vp, _vp, C.c_int64)
_proto("gl_depthwed_aggregate", C.c_int, _vp, _vp, C.c_int32, C.c_int64, _vp, _vp, _vp, C.c_int64, _vp, _vp, _vp, _vp,
       C.c_int64, _i64p)
_proto("gl_depthwed_aggregate_device", C.c_int, _vp, _vp, C.c_int32, C.c_int64, _vp, C.c_int64, _vp)
_proto("gl_depthwed_aggregate_i32", C.c_int, _vp, _vp, C.c_int32, C.c_int64, _vp, _vp, _vp, C.c_int64, _vp, _vp, _vp, _vp, C.c_int64, _i64p)
_proto("gl_depthwed_aggregate_i32_device", C.c_int, _vp, _vp, C.c_int32, C.c_int64, _vp, C.c_int64, C.c_int64, _vp, _vp)
_proto("gl_depthwed_aggregate_i32_p2p", C.c_int, _vp, _vp, C.c_int32, C.c_int64, _vp, C.c_int64, C.c_int64, _vp, C.c_int32, C.c_int64, C.c_int32, _vp)
_proto("gl_depthwed_plan", C.c_int, _vp, _vp, _vp, C.c_int64, C.c_int64, _vp, _vp, _vp, _vp, C.c_int64, _i64p)
_proto("gl_depthwed_cells", C.c_int, _vp, _vp, _vp, C.c_int64, _vp, C.c_int64, _vp)
_proto("gl_depthwed_column_begin", C.c_int, _vp, _vp, C.c_int64)
_proto("gl_depthwed_add_column", C.c_int, _vp, C.c_int64, _vp, _vp)
_proto("gl_depthwed_column_i32", C.c_int, _vp, _vp, C.c_int64, _vp, _vp)
_proto("gl_ipc_export", C.c_int, _vp, _vp, _vp)
_proto("gl_ipc_open", C.c_int, _vp, _vp, C.POINTER(_vp))
_proto("gl_ipc_close", C.c_int, _vp, _vp)
_proto("gl_allgather_device_async", C.c_int, _vp, _vp, _vp, C.c_int64)
_proto("gl_comm_wait", C.c_int, _vp)
_proto("gl_comm_unique_id", C.c_int, _vp)
_proto("gl_comm_init", C.c_int, _vp, _vp, C.c_int, C.c_int)
_proto("gl_comm_destroy", C.c_int, _vp)
_proto("gl_allgather_device", C.c_int, _vp, _vp, _vp, C.c_int64)
_proto("gl_bam_decode_segments", C.c_int, C.c_char_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(_vp), _vp, C.c_int64)
_proto("gl_segset_n_refs", C.c_int, _vp, _i32p, _i64p, _i64p)
_proto("gl_segset_ref", C.c_int, _vp, C.c_int32, C.POINTER(C.c_char_p), _i64p, C.POINTER(_vp), C.POINTER(_vp), _i64p)
_proto("gl_segset_free", None, _vp)
_proto("gl_bam_open", C.c_int, C.c_char_p, C.POINTER(_vp), _vp, C.c_int64)
_proto("gl_bam_close", None, _vp)
_proto("gl_bam_info", C.c_int, _vp, _i32p, _i32p)
_proto("gl_bam_ref", C.c_int, _vp, C.c_int32, C.POINTER(C.c_char_p), _i64p, _i64p)
_proto("gl_bam_index", C.c_int, _vp, C.POINTER(C.c_char_p), _i32p, _i32p, _i32p)
_proto("gl_bam_decode", C.c_int, _vp, C.c_int32, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_int32, _vp, _vp, C.c_int64)
_proto("gl_bam_decode_device", C.c_int, _vp, _vp, C.c_int32, C.c_int32, C.POINTER(_vp), C.POINTER(_vp), _i64p, _vp)
_proto("gl_bam_decode_device_regions", C.c_int, _vp, _vp, C.c_int32, _vp, _vp, C.c_int64, C.c_int32, C.POINTER(_vp), C.POINTER(_vp), _i64p, _vp)
_proto("gl_bam_region_chunks", C.c_int, _vp, C.c_int32, _vp, _vp, C.c_int64, _vp, _vp, C.c_int64, _i64p)
_proto("gl_bgzf_inflate_device", C.c_int, _vp, _vp, _vp, _vp, C.c_int64, _vp, _vp)
_proto("gl_bai_read", C.c_int, C.c_char_p, C.POINTER(_vp), _vp, C.c_int64)
_proto("gl_bai_n_refs", C.c_int, _vp, _i32p, _u64p)
_proto("gl_bai_ref", C.c_int, _vp, C.c_int32, C.POINTER(_vp), _i64p, _u64p, _u64p, _i32p)
_proto("gl_bai_geometry", C.c_int, _vp, _i32p, _i32p, _i32p)
_proto("gl_bai_free", None, _vp)
_proto("gl_pack_segments16_bound", C.c_int64, C.c_int64)
_proto("gl_pack_segments16", C.c_int, _vp, _vp, C.c_int64, _vp, _vp, _vp, C.c_int64, _i64p)
_proto("gl_pack_segments16_mt", C.c_int, _vp, _vp, C.c_int64, C.c_int32, _vp, _vp, _vp, C.c_int64, _i64p)
_proto("gl_depth_add_segments_packed16", C.c_int, _vp, _vp, _vp, _vp, C.c_int64)
_proto("gl_depth_region_packed16", C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp, _vp, C.c_int64, C.c_int32, C.c_int32,
       C.c_int32, C.c_int64, _vp, C.c_int64, _i64p, _vp, _vp, C.c_int64, _i64p)
_proto("gl_pack_segments8_bound", C.c_int64, C.c_int64)
_proto("gl_pack_segments8", C.c_int, _vp, _vp, C.c_int64, _vp, _vp, _vp, C.c_int64, _i64p)
_proto("gl_depth_transport_phases", C.c_int, _vp, C.POINTER(C.c_double))
_proto("gl_depth_transport_stats", C.c_int, _vp, _i32p, C.POINTER(C.c_double), _i64p, _i64p)
_proto("gl_pack_segments16_fixed_mt", C.c_int, _vp, _vp, C.c_int64, C.c_int32, _vp, _vp, _vp, _vp, _vp, C.c_int64, _i64p)
_proto("gl_pack_segments8_mt", C.c_int, _vp, _vp, C.c_int64, C.c_int32, _vp, _vp, _vp, C.c_int64, _i64p)
_proto("gl_depth_add_segments_packed8", C.c_int, _vp, _vp, _vp, _vp, C.c_int64)
_proto("gl_depth_add_segments_packed8_device", C.c_int, _vp, _vp, _vp, _vp, C.c_int64)
_proto("gl_depth_region_packed8", C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp, _vp, C.c_int64, C.c_int32, C.c_int32,
       C.c_int32, C.c_int64, _vp, C.c_int64, _i64p, _vp, _vp, C.c_int64, _i64p)
_proto("gl_depth_text", C.c_int, _vp, C.c_char_p, _vp, C.c_int64, _i64p, _vp, C.c_int64, _i64p)
_proto("gl_depth_text_bound", C.c_int64, C.c_char_p, C.c_int64)
_proto("gl_depth_format_rows", C.c_int, _vp, C.c_char_p, _vp, _vp, _vp, C.c_int64, _vp, C.c_int64, _i64p)
_proto("gl_depth_bed_contig", C.c_int, _vp, C.c_char_p, C.c_int64, _vp, _vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int64,
       C.c_int32, _vp, C.c_int64, _i64p, _vp, C.c_int64, _i64p)
_proto("gl_depth_bed_region", C.c_int, _vp, C.c_char_p, C.c_int64, C.c_int64, _vp, _vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
       C.c_int64, C.c_int32, _vp, C.c_int64, _i64p, _vp, C.c_int64, _i64p)
_proto("gl_depth_bed_contig_packed8", C.c_int, _vp, C.c_char_p, C.c_int64, _vp, _vp, _vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32,
       C.c_int64, _vp, C.c_int64, _i64p, _vp, C.c_int64, _i64p)
_proto("gl_indexsplit_accumulate", C.c_int, _vp, _vp, _vp, C.c_int32, C.c_int32, _vp, _vp)
_proto("gl_indexsplit_chunks", C.c_int, _vp, _vp, C.c_int32, C.POINTER(C.c_char_p), _vp, _vp, C.c_int32, C.c_int32, _vp, _vp, _vp, C.c_int64,
       C.POINTER(_vp), _i64p)
_proto("gl_crai_make_sizes", C.c_int, _vp, _vp, _vp, C.c_int64, _vp, C.c_int64, _i64p)
_proto("gl_depth_format_chunk", C.c_int, C.c_char_p, C.c_int64, C.c_int64, C.c_int32, _vp, C.c_int64, _vp, _vp,
       C.c_int64, C.POINTER(_vp), _i64p, C.POINTER(_vp), _i64p)
_proto("gl_free_text", None, _vp)
_proto("gl_multidepth_begin", C.c_int, _vp, C.c_int64, C.c_int32, C.c_int32, C.c_double)
_proto("gl_multidepth_count", C.c_int, _vp)
_proto("gl_multidepth_merge", C.c_int, _vp, C.POINTER(_vp), C.c_int32)
_proto("gl_multidepth_adopt_sites", C.c_int, _vp, _vp)
_proto("gl_multidepth_sites", C.c_int, _vp, _vp, _vp, C.c_int64, _i64p)
_proto("gl_multidepth_blocks", C.c_int, _vp, _vp, C.c_int64, C.c_int64, C.c_int32, C.c_int64, C.c_int64, C.c_int64, C.c_int64,
       _vp, _vp, _vp, C.c_int64, _i64p)
_proto("gl_multidepth_set_blocks", C.c_int, _vp, _vp, _vp, _vp, C.c_int64)
_proto("gl_multidepth_sums", C.c_int, _vp, C.c_int32)
_proto("gl_multidepth_result", C.c_int, _vp, _vp, _vp, _vp, _vp)
_proto("gl_multidepth_stats", C.c_int, _vp, _i64p, _i64p, _i64p, _i64p)
_proto("gl_multidepth_certify", C.c_int, _vp, _vp, _vp, C.c_int64, _vp, _vp)
_proto("gl_multidepth_text", C.c_int, C.c_char_p, _vp, _vp, C.c_int64, C.c_int32, _vp, _vp, _vp, C.c_int32, C.POINTER(_vp), _i64p)
_proto("gl_go_argsort_f64", C.c_int, _vp, C.c_int64, _vp)
_proto("gl_dcnv_normalize_device", C.c_int, _vp, _vp, C.c_int64, C.c_int64, _vp, C.c_int32, C.c_int32, _vp, C.c_int64, _vp)
_proto("gl_dcnv_normalize", C.c_int, _vp, _vp, C.c_int64, C.c_int64, _vp, C.c_int32, C.c_int32, C.c_int32, _vp, C.c_int64, _vp)
_proto("gl_dcnv_chunk_slices", C.c_int, _vp, C.c_int64, C.c_double, _vp, C.c_int64, _i64p)
_proto("gl_dcnv_normalize_chunked_device", C.c_int, _vp, _vp, C.c_int64, C.c_int64, _vp, _vp, C.c_int64, C.c_int32, C.c_int32, _vp,
       C.c_int64, _vp)
_proto("gl_dcnv_normalize_chunked", C.c_int, _vp, _vp, C.c_int64, C.c_int64, _vp, _vp, C.c_int64, C.c_int32, C.c_int32, C.c_int32, _vp,
       C.c_int64, _vp)
_proto("gl_format_f2", C.c_int, _vp, _vp, C.c_int64, _vp)
_proto("gl_format_f2_device", C.c_int, _vp, _vp, C.c_int64, _vp)
_proto("gl_format_f2_host", C.c_int, _vp, C.c_int64, _vp)
_proto("gl_dcnv_chart_select_host", C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp)
_proto("gl_dcnv_chart_extent", C.c_int, _vp, _vp, C.c_int64, C.c_int64, _vp)
_proto("gl_dcnv_chart_raster_host", C.c_int, _vp, C.c_int64, C.c_int64, _vp, _vp, C.c_int32, C.c_int32, C.c_double, _vp)
_proto("gl_dcnv_chart", C.c_int, _vp, _vp, C.c_int64, C.c_int64, C.c_int64, C.c_int32, C.c_int32, C.c_double, _vp, _vp, _vp, _vp)
_proto("gl_emdepth_device", C.c_int, _vp, _vp, C.c_int64, C.c_int64, C.c_int32, _vp, _vp)
_proto("gl_emdepth", C.c_int, _vp, _vp, C.c_int64, C.c_int64, C.c_int32, C.c_int64, _vp, _vp)
_proto("gl_emdepth_stats", C.c_int, _vp, _i64p, _i64p, _i64p)
_proto("gl_emdepth_factors", C.c_int, _vp)
_proto("gl_emdepth_cnvs", C.c_int, _vp, C.c_int64, C.c_int32, _vp, _vp, _vp, C.c_int64, _vp, _vp, _vp, C.c_int64, _i64p,
       _vp, C.c_int64, _i64p)
_proto("gl_emdepth_sum_host", C.c_int, _vp, C.c_int64, C.POINTER(C.c_double), C.POINTER(C.c_uint8))
_proto("gl_cnveval_order", C.c_int, _vp, _vp, C.c_int64, _vp)
_proto("gl_cnveval", C.c_int, _vp, C.c_int32, _vp, _vp, _vp, _vp, _vp, C.c_int64, _vp, _vp, _vp, _vp, C.c_int64, _vp, _vp, C.c_double, _vp)
_proto("gl_cnveval_device", C.c_int, _vp, C.c_int32, _vp, C.c_int64, _vp, _vp, _vp, _vp, C.c_int64, _vp, _vp, _vp, _vp, _vp,
       C.c_int64, _vp, C.c_double, _vp)
_proto("gl_indexcov_pca8", C.c_int, _vp, C.c_int64, _vp)
_proto("gl_indexcov_pca", C.c_int, _vp, _vp, C.c_int64, C.c_int32, C.c_int64, C.c_int32, _vp, _vp, _i32p, _vp)
_proto("gl_indexcov_pca_device", C.c_int, _vp, _vp, C.c_int64, C.c_int32, C.c_int64, C.c_int32, _vp, _vp, _i32p, _vp)
_proto("gl_indexcov_pca_phases", C.c_int, _vp, C.POINTER(C.c_double))
_proto("gl_pca_tridiag_top", C.c_int, _vp, _vp, C.c_int32, C.c_int32, _vp, _vp)
_proto("gl_sym_tridiag", C.c_int, _vp, _vp, C.c_int32, _vp, _vp, _vp, _vp, C.c_int32, _vp)
_proto("gl_dcnv_svd", C.c_int, _vp, _vp, C.c_int64, C.c_int64, C.c_int32, C.c_double, C.c_int64, _vp, _vp, _i32p, _i64p)
_proto("gl_dcnv_svd_device", C.c_int, _vp, _vp, C.c_int64, C.c_int64, C.c_int32, C.c_double, _vp, _vp, _i32p, _i64p)
_proto("gl_dcnv_svd_phases", C.c_int, _vp, C.POINTER(C.c_double))
_proto("gl_pca_tridiag_above", C.c_int, _vp, _vp, C.c_int32, C.c_double, _vp, _i32p)


def version() -> str:
    return lib.gl_version().decode()


def device_count() -> int:
    n = C.c_int(0)
    rc = lib.gl_device_count(C.byref(n))
    if rc != GL_OK:
        return 0
    return n.value


def bind_numa_for_device(device: int, share_index: int = 0, share_count: int = 1) -> Tuple[int, int]:
    """(numa node or -1, cpus bound) — call before the first pinned allocation / pool use"""
    node, n = C.c_int(-1), C.c_int(0)
    lib.gl_bind_numa_for_device(device, share_index, share_count, C.byref(node), C.byref(n))
    return node.value, n.value


def device_numa_node(device: int) -> int:
    node = C.c_int(-1)
    lib.gl_device_numa_node(device, C.byref(node))
    return node.value


def lpt_assign(weights, bins: int):
    """(bin_of int32[n], bin_load int64[bins]) — longest first onto the least loaded bin"""
    w = np.ascontiguousarray(weights, np.int64)
    bin_of, load = np.empty(w.size, np.int32), np.empty(bins, np.int64)
    rc = lib.gl_lpt_assign(w.ctypes.data_as(_vp), w.size, bins, bin_of.ctypes.data_as(_vp), load.ctypes.data_as(_vp))
    if rc != GL_OK:
        raise GlError(rc, "gl_lpt_assign: bad arguments")
    return bin_of, load


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(_vp)


def _as(a, dtype) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=dtype)


def format_chunk(chrom: str, rs: int, re: int, W: int, win_sum: np.ndarray, run_start: np.ndarray,
                 run_class: np.ndarray) -> Tuple[bytes, bytes]:
    """Host-only: the reference's rows for one chunk (no GPU needed)."""
    win_sum = _as(win_sum, np.int64)
    run_start = _as(run_start, np.int32)
    run_class = _as(run_class, np.uint8)
    d, c = _vp(), _vp()
    dl, cl = C.c_int64(0), C.c_int64(0)
    rc = lib.gl_depth_format_chunk(chrom.encode(), rs, re, W, _ptr(win_sum), len(win_sum), _ptr(run_start),
                                   _ptr(run_class), len(run_start), C.byref(d), C.byref(dl), C.byref(c), C.byref(cl))
    if rc != GL_OK:
        raise GlError(rc, "gl_depth_format_chunk: bad arguments")
    try:
        return C.string_at(d, dl.value), C.string_at(c, cl.value)
    finally:
        lib.gl_free_text(d)
        lib.gl_free_text(c)


# ---- multidepth (multidepth/multidepth.go), host-only parts
MD_DEFAULTS = dict(Q=10, mincov=7, maxcov=1000, min_samples=0.5, min_size=15, max_skip=10, window=10_000_000)


def multidepth_blocks(run_start, run_class, contig_len: int, n_samples: int, max_skip: int = 10, min_size: int = 15,
                      window: int = 10_000_000, chunk: int = 0):
    """Host-only: the reference's chunk state machine over site-class runs -> (start, end, sufficient sites) arrays."""
    run_start, run_class = _as(run_start, np.int32), _as(run_class, np.uint8)
    n = C.c_int64(0)
    args = (_ptr(run_start), _ptr(run_class), run_start.size, contig_len, n_samples, chunk, max_skip, min_size, window)
    rc = lib.gl_multidepth_blocks(*args, None, None, None, 0, C.byref(n))
    if rc != GL_OK:
        raise GlError(rc, "gl_multidepth_blocks: bad arguments")
    s, e, k = np.empty(n.value, np.int64), np.empty(n.value, np.int64), np.empty(n.value, np.int64)
    rc = lib.gl_multidepth_blocks(*args, _ptr(s), _ptr(e), _ptr(k), n.value, C.byref(n))
    if rc != GL_OK:
        raise GlError(rc, "gl_multidepth_blocks: bad arguments")
    return s, e, k


def multidepth_certify(sums, n_sites, spans):
    """Host-only: (q, certified): q = round(100 sum / span) where the "%.2f" of the reference's chain is provably that."""
    sums, n_sites, spans = _as(sums, np.int64), _as(n_sites, np.int64), _as(spans, np.int64)
    q, ok = np.empty(sums.size, np.int64), np.empty(sums.size, np.uint8)
    rc = lib.gl_multidepth_certify(_ptr(sums), _ptr(n_sites), _ptr(spans), sums.size, _ptr(q), _ptr(ok))
    if rc != GL_OK:
        raise GlError(rc, "gl_multidepth_certify: bad arguments")
    return q, ok.astype(bool)


def multidepth_text(chrom: str, blk_start, blk_end, S: int, q, val, certified, threads: int = 0) -> bytes:
    """Host-only: the rows after the header line."""
    blk_start, blk_end = _as(blk_start, np.int64), _as(blk_end, np.int64)
    q, val, certified = _as(q, np.int64), _as(val, np.float64), _as(certified, np.uint8)
    p, n = _vp(), C.c_int64(0)
    rc = lib.gl_multidepth_text(chrom.encode(), _ptr(blk_start), _ptr(blk_end), blk_start.size, S, _ptr(q), _ptr(val),
                                _ptr(certified), threads, C.byref(p), C.byref(n))
    if rc != GL_OK:
        raise GlError(rc, "gl_multidepth_text: bad arguments")
    try:
        return C.string_at(p, n.value)
    finally:
        lib.gl_free_text(p)


# ---- dcnv (dcnv/dcnv.go), host-only parts
F2_TOKEN = 16


def go_argsort(v) -> np.ndarray:
    """Host-only: the permutation gonum's floats.Argsort (Go's unstable sort.Sort) gives v."""
    v = _as(v, np.float64)
    inds = np.empty(v.size, np.int64)
    rc = lib.gl_go_argsort_f64(_ptr(v), v.size, _ptr(inds))
    if rc != GL_OK:
        raise GlError(rc, "gl_go_argsort_f64: bad arguments")
    return inds


def dcnv_chunk_slices(gc_sorted, w: float) -> np.ndarray:
    """Host-only: ChunkDebiaser's chunks of the GC values in sorted order, as CSR offsets (ptr[0] = 0, ptr[-1] = n)."""
    v = _as(gc_sorted, np.float64)
    nc = C.c_int64(0)
    rc = lib.gl_dcnv_chunk_slices(_ptr(v), v.size, float(w), None, 0, C.byref(nc))
    if rc != GL_OK:
        raise GlError(rc, "gl_dcnv_chunk_slices: bad arguments (n >= 1, w finite and > 0)")
    ptr = np.empty(nc.value + 1, np.int64)
    rc = lib.gl_dcnv_chunk_slices(_ptr(v), v.size, float(w), _ptr(ptr), ptr.size, C.byref(nc))
    if rc != GL_OK:
        raise GlError(rc, "gl_dcnv_chunk_slices: failed")
    return ptr


def format_f2_host(vals) -> np.ndarray:
    """Host-only: n x 16 "%.2f" tokens (text, NUL-padded; an empty token: the caller formats the value)."""
    vals = _as(vals, np.float64)
    tok = np.empty((vals.size, F2_TOKEN), np.uint8)
    rc = lib.gl_format_f2_host(_ptr(vals), vals.size, _ptr(tok))
    if rc != GL_OK:
        raise GlError(rc, "gl_format_f2_host: bad arguments")
    return tok


def f2_text(tokens, vals) -> list:
    """the "%.2f" strings (bytes) of tokens, with Python formatting where a token is empty"""
    out = []
    for t, v in zip(np.asarray(tokens, np.uint8).reshape(-1, F2_TOKEN), np.asarray(vals, np.float64).ravel()):
        b = t.tobytes().rstrip(b"\0")
        out.append(b if b else b"%.2f" % v)
    return out


# ---- emdepth (emdepth/emdepth.go), host-only parts
EM_CN_MASK, EM_OUTSIDE = 0x0F, 0x40


def emdepth_factors() -> np.ndarray:
    """Host-only: math.Pow(i / 2, 1.1), i = 0..8, as the kernel uses them"""
    f = np.empty(9, np.float64)
    lib.gl_emdepth_factors(_ptr(f))
    return f


def emdepth_cnvs(cells, starts, ends, breaks=()):
    """Host-only: the reference's Cache over the cells (n x S) -> [(sample, psize, row indices)], Clear(nil) before every row
    in breaks and after the last"""
    cells = _as(cells, np.uint8)
    n, S = cells.shape
    starts, ends, breaks = _as(starts, np.int64), _as(ends, np.int64), _as(breaks, np.int64)
    nc, nr = C.c_int64(0), C.c_int64(0)
    args = (_ptr(cells), n, S, _ptr(starts), _ptr(ends), _ptr(breaks), breaks.size)
    rc = lib.gl_emdepth_cnvs(*args, None, None, None, 0, C.byref(nc), None, 0, C.byref(nr))
    if rc != GL_OK:
        raise GlError(rc, "gl_emdepth_cnvs: bad arguments")
    smp, psz, ptr = np.empty(nc.value, np.int32), np.empty(nc.value, np.int32), np.zeros(nc.value + 1, np.int64)
    rows = np.empty(nr.value, np.int64)
    rc = lib.gl_emdepth_cnvs(*args, _ptr(smp), _ptr(psz), _ptr(ptr), nc.value, C.byref(nc), _ptr(rows), nr.value, C.byref(nr))
    if rc != GL_OK:
        raise GlError(rc, "gl_emdepth_cnvs: bad arguments")
    return [(int(smp[i]), int(psz[i]), rows[ptr[i]:ptr[i + 1]]) for i in range(nc.value)]


def emdepth_sum_host(v):
    """Host-only: (the kernel's tree-order float64 sum of v, whether its exactness certificate holds)"""
    v = _as(v, np.float32)
    s, ok = C.c_double(0), C.c_uint8(0)
    rc = lib.gl_emdepth_sum_host(_ptr(v), v.size, C.byref(s), C.byref(ok))
    if rc != GL_OK:
        raise GlError(rc, "gl_emdepth_sum_host: bad arguments")
    return s.value, bool(ok.value)


# ---- cnveval (cnveval/cnveval.go), host-only part
def cnveval_order(chrom, start) -> np.ndarray:
    """Host-only: the permutation Go 1.21's sort.Slice leaves when it sorts calls given in file order by (chrom, start)"""
    chrom, start = _as(chrom, np.int32), _as(start, np.int64)
    if chrom.size != start.size:
        raise ValueError("cnveval_order: chrom and start differ in length")
    perm = np.empty(chrom.size, np.int64)
    rc = lib.gl_cnveval_order(_ptr(chrom), _ptr(start), chrom.size, _ptr(perm))
    if rc != GL_OK:
        raise GlError(rc, "gl_cnveval_order: bad arguments")
    return perm


# ---- indexcov PCA (indexcov.go:686-705,773-807), host-only parts
def indexcov_pca8(d) -> np.ndarray:
    """the PCA byte of each float32 depth (clip at 8, uint8(8191.875 d + 0.5) the way Go converts it)"""
    d = _as(d, np.float32).ravel()
    out = np.empty(d.size, np.uint8)
    if lib.gl_indexcov_pca8(_ptr(d), d.size, _ptr(out)) != GL_OK:
        raise GlError(GL_EINVAL, "gl_indexcov_pca8: bad arguments")
    return out


def pca_tridiag_top(d, e, k: int, vectors: bool = True):
    """(w[k] descending, z (k x n) or None): the k largest eigenpairs of the symmetric tridiagonal (d, e)"""
    d, e = _as(d, np.float64), _as(e, np.float64)
    w = np.empty(k, np.float64)
    z = np.empty((k, d.size), np.float64) if vectors else None
    if lib.gl_pca_tridiag_top(_ptr(d), _ptr(e), d.size, k, _ptr(w), _ptr(z)) != GL_OK:
        raise GlError(GL_EINVAL, "gl_pca_tridiag_top: bad arguments")
    return w, z


def pca_tridiag_above(d, e, rel: float = 1e-12) -> np.ndarray:
    """every eigenvalue above rel times the largest of the symmetric tridiagonal (d, e), descending, bisected on the host pool"""
    d, e = _as(d, np.float64), _as(e, np.float64)
    w, k = np.empty(d.size, np.float64), C.c_int32(0)
    if lib.gl_pca_tridiag_above(_ptr(d), _ptr(e), d.size, rel, _ptr(w), C.byref(k)) != GL_OK:
        raise GlError(GL_EINVAL, "gl_pca_tridiag_above: bad arguments")
    return w[:k.value].copy()


# ---- indexcov charts (plot.cu)
PLOT_CW, PLOT_CH, PLOT_AX, PLOT_AY, PLOT_W, PLOT_H = 384, 288, 56, 8, 316, 244
PLOT_DEPTH, PLOT_PLAIN, PLOT_SQUARE = 0, 1, 2
PLOT_SVG, PLOT_EPS = 0, 1


def _ck0(rc: int):
    if rc != GL_OK:
        raise GlError(rc, lib.gl_last_error(None).decode())


def depthwed_plan(starts, ends, chrom_id, size: int):
    """gl_depthwed_plan (host only): (grp_first [n+1], out_start, out_end, out_chrom) of the groups depthwed.go:117-157 makes"""
    starts, ends, chrom_id = _as(starts, np.int64), _as(ends, np.int64), _as(chrom_id, np.int32)
    R = starts.size
    assert ends.size == R and chrom_id.size == R
    cap = max(R, 1)
    first, o_s, o_e, o_c = np.empty(cap + 1, np.int64), np.empty(cap, np.int64), np.empty(cap, np.int64), np.empty(cap, np.int32)
    n = C.c_int64(0)
    _ck0(lib.gl_depthwed_plan(_ptr(starts), _ptr(ends), _ptr(chrom_id), R, size, _ptr(first), _ptr(o_s), _ptr(o_e), _ptr(o_c), cap,
                              C.byref(n)))
    k = n.value
    return first[:k + 1], o_s[:k], o_e[:k], o_c[:k]


def plot_select_host(vals, off, lens):
    """(sel (n,3) int64 {first, m, stride}, yext (n,2) float32) of every dataset vals[off[d]:off[d]+lens[d]]"""
    vals, off, lens = _as(vals, np.float32), _as(off, np.int64), _as(lens, np.int64)
    n = off.size
    sel, yext = np.empty((n, 3), np.int64), np.empty((n, 2), np.float32)
    _ck0(lib.gl_plot_select_host(_ptr(vals), _ptr(off), _ptr(lens), n, _ptr(sel), _ptr(yext)))
    return sel, yext


def plot_transform(ext4, W: int, H: int) -> np.ndarray:
    e, xf = _as(ext4, np.float64), np.empty(4, np.float64)
    _ck0(lib.gl_plot_transform(_ptr(e), W, H, _ptr(xf)))
    return xf


def plot_line_radius(n_datasets: int) -> float:
    return lib.gl_plot_line_radius(n_datasets)


def plot_raster_series_host(vals, off, sel, mult: float, chart, draw, xf, n_charts: int, W: int, H: int, r: float) -> np.ndarray:
    vals, off, sel = _as(vals, np.float32), _as(off, np.int64), _as(sel, np.int64)
    chart, draw, xf = _as(chart, np.int32), _as(draw, np.uint32), _as(xf, np.float64)
    img = np.empty((n_charts, H, W), np.uint32)
    _ck0(lib.gl_plot_raster_series_host(_ptr(vals), _ptr(off), _ptr(sel), mult, _ptr(chart), _ptr(draw), chart.size, _ptr(xf), n_charts,
                                        W, H, r, _ptr(img)))
    return img


def plot_raster_xy_host(x, y, ptr, chart, draw, xf, n_charts: int, W: int, H: int, r: float) -> np.ndarray:
    x, y, ptr = _as(x, np.float64), _as(y, np.float64), _as(ptr, np.int64)
    chart, draw, xf = _as(chart, np.int32), _as(draw, np.uint32), _as(xf, np.float64)
    img = np.empty((n_charts, H, W), np.uint32)
    _ck0(lib.gl_plot_raster_xy_host(_ptr(x), _ptr(y), _ptr(ptr), _ptr(chart), _ptr(draw), chart.size, _ptr(xf), n_charts, W, H, r,
                                    _ptr(img)))
    return img


def plot_path_series_host(vals, off, sel, mult: float, chart, xf, n_charts: int, kind: int, fmt: int, cap: Optional[int] = None):
    """(len [n] int64, text bytes) of every dataset's path text (gl_plot_path_series_size_host + _emit_host); cap: the room
    given to the emit (default: exactly the total)"""
    vals, off, sel = _as(vals, np.float32), _as(off, np.int64), _as(sel, np.int64)
    chart, xf = _as(chart, np.int32), _as(xf, np.float64)
    n = chart.size
    ln, pos = np.empty(max(n, 1), np.int64), np.empty(n + 1, np.int64)
    _ck0(lib.gl_plot_path_series_size_host(_ptr(vals), _ptr(off), _ptr(sel), mult, _ptr(chart), n, _ptr(xf), n_charts, kind, fmt, _ptr(ln),
                                           _ptr(pos)))
    out = np.empty(max(int(pos[n]) if cap is None else cap, 1), np.uint8)
    _ck0(lib.gl_plot_path_series_emit_host(_ptr(vals), _ptr(off), _ptr(sel), mult, _ptr(chart), n, _ptr(xf), n_charts, kind, fmt, _ptr(pos),
                                           _ptr(out), int(pos[n]) if cap is None else cap))
    return ln[:n].copy(), out[:int(pos[n])].tobytes()


def plot_path_xy_host(x, y, ptr, chart, xf, n_charts: int, kind: int, fmt: int, cap: Optional[int] = None):
    """(len [n] int64, text bytes) of every dataset's path text from explicit vertices (gl_plot_path_xy_size_host + _emit_host)"""
    x, y, ptr = _as(x, np.float64), _as(y, np.float64), _as(ptr, np.int64)
    chart, xf = _as(chart, np.int32), _as(xf, np.float64)
    n = chart.size
    ln, pos = np.empty(max(n, 1), np.int64), np.empty(n + 1, np.int64)
    _ck0(lib.gl_plot_path_xy_size_host(_ptr(x), _ptr(y), _ptr(ptr), _ptr(chart), n, _ptr(xf), n_charts, kind, fmt, _ptr(ln), _ptr(pos)))
    out = np.empty(max(int(pos[n]) if cap is None else cap, 1), np.uint8)
    _ck0(lib.gl_plot_path_xy_emit_host(_ptr(x), _ptr(y), _ptr(ptr), _ptr(chart), n, _ptr(xf), n_charts, kind, fmt, _ptr(pos), _ptr(out),
                                       int(pos[n]) if cap is None else cap))
    return ln[:n].copy(), out[:int(pos[n])].tobytes()


def plot_line_width(n_datasets: int) -> float:
    return lib.gl_plot_line_width(n_datasets)


def plot_vector_write(path: str, kind: int, fmt: int, ext4, xtitle: str, ytitle: str, rgb, width: float, texts):
    """gl_plot_vector_write: texts[d] is dataset d's path text (bytes), rgb (n, 3) uint8 its colour"""
    e, rgb = _as(ext4, np.float64), _as(rgb, np.uint8)
    n = len(texts)
    data = (C.c_char_p * max(n, 1))(*texts)
    lens = np.array([len(t) for t in texts] or [0], np.int64)
    _ck0(lib.gl_plot_vector_write(path.encode(), kind, fmt, _ptr(e), xtitle.encode(), ytitle.encode(), n, _ptr(rgb), width, data,
                                  _ptr(lens)))


def dcnv_chart_select_host(x):
    """dcnv's chart selection of the n x S float64 matrix x: (first[S] int64, yext (S,2) float64)"""
    x = np.ascontiguousarray(x, np.float64)
    n, S = x.shape
    first, yext = np.empty(S, np.int64), np.empty((S, 2), np.float64)
    _ck0(lib.gl_dcnv_chart_select_host(_ptr(x), n, S, _ptr(first), _ptr(yext)))
    return first, yext


def dcnv_chart_extent(first, yext, n: int) -> np.ndarray:
    first, yext = _as(first, np.int64), _as(yext, np.float64)
    ext = np.empty(4, np.float64)
    _ck0(lib.gl_dcnv_chart_extent(_ptr(first), _ptr(yext), n, first.size, _ptr(ext)))
    return ext


def dcnv_chart_raster_host(x, first, xf, W: int = PLOT_W, H: int = PLOT_H, r: Optional[float] = None) -> np.ndarray:
    """the (H, W) index image of dcnv's stepped lines of x (sample k drawn with index S - k)"""
    x = np.ascontiguousarray(x, np.float64)
    n, S = x.shape
    first, xf = _as(first, np.int64), _as(xf, np.float64)
    img = np.empty((H, W), np.uint32)
    _ck0(lib.gl_dcnv_chart_raster_host(_ptr(x), n, S, _ptr(first), _ptr(xf), W, H, plot_line_radius(S) if r is None else r, _ptr(img)))
    return img


def plot_color(k: int, n_background: int = 0):
    c = (C.c_uint8 * 3)()
    lib.gl_plot_color(k, n_background, c)
    return tuple(c)


def plot_ticks(lo: float, hi: float) -> np.ndarray:
    out, n = np.empty(64, np.float64), C.c_int32()
    _ck0(lib.gl_plot_ticks(lo, hi, _ptr(out), 64, C.byref(n)))
    return out[:n.value].copy()


def plot_millions(v: float) -> str:
    b = C.create_string_buffer(64)
    _ck0(lib.gl_plot_millions(v, b, 64))
    return b.value.decode()


def plot_text(rgb: np.ndarray, x: int, y: int, s: str, vertical: bool = False) -> np.ndarray:
    """draws s into rgb (H, W, 3) uint8 in place"""
    assert rgb.dtype == np.uint8 and rgb.flags.c_contiguous and rgb.ndim == 3
    _ck0(lib.gl_plot_text(_ptr(rgb), rgb.shape[1], rgb.shape[0], x, y, s.encode(), int(vertical)))
    return rgb


def plot_compose(img, palette, kind: int, ext4, xtitle: str, ytitle: str) -> np.ndarray:
    img, pal, e = _as(img, np.uint32), _as(palette, np.uint8), _as(ext4, np.float64)
    assert img.size == PLOT_W * PLOT_H
    rgb = np.empty((PLOT_CH, PLOT_CW, 3), np.uint8)
    _ck0(lib.gl_plot_compose(_ptr(img), _ptr(pal), pal.size // 3, kind, _ptr(e), xtitle.encode(), ytitle.encode(), _ptr(rgb)))
    return rgb


def plot_png(rgb) -> bytes:
    rgb = _as(rgb, np.uint8)
    H, W = rgb.shape[:2]
    n = C.c_int64()
    _ck0(lib.gl_plot_png(_ptr(rgb), W, H, None, 0, C.byref(n)))
    out = np.empty(n.value, np.uint8)
    _ck0(lib.gl_plot_png(_ptr(rgb), W, H, _ptr(out), out.size, C.byref(n)))
    return out[:n.value].tobytes()


def chunk_rows(rs: int, re: int, W: int, run_start: np.ndarray, run_class: np.ndarray):
    """Host-only: (s, e) of the window rows gl_depth_format_chunk writes for a chunk, in order."""
    run_start = _as(run_start, np.int32)
    run_class = _as(run_class, np.uint8)
    n = C.c_int64(0)
    lib.gl_depth_chunk_rows(rs, re, W, _ptr(run_start), _ptr(run_class), run_start.size, None, None, 0, C.byref(n))
    s, e = np.empty(n.value, np.int64), np.empty(n.value, np.int64)
    rc = lib.gl_depth_chunk_rows(rs, re, W, _ptr(run_start), _ptr(run_class), run_start.size, _ptr(s), _ptr(e), n.value, C.byref(n))
    if rc != GL_OK:
        raise GlError(rc, "gl_depth_chunk_rows: bad arguments")
    return s, e


def pack_segments16(start: np.ndarray, end: np.ndarray, threads: Optional[int] = None):
    """Host-only: (anchors int32[nb], off uint16[nb*256], len uint16[nb*256]) — the feeder's compact format.
    threads=None: single-threaded; an int: gl_pack_segments16_mt (0 = the whole pool)."""
    start, end = _as(start, np.int32), _as(end, np.int32)
    nb = C.c_int64(0)
    cap = max(1, int(lib.gl_pack_segments16_bound(start.size)) // 8 + start.size // 256 + 2)
    while True:
        a = np.empty(cap, np.int32)
        o = np.empty(cap * 256, np.uint16)
        ln = np.empty(cap * 256, np.uint16)
        if threads is None:
            rc = lib.gl_pack_segments16(_ptr(start), _ptr(end), start.size, _ptr(a), _ptr(o), _ptr(ln), cap, C.byref(nb))
        else:
            rc = lib.gl_pack_segments16_mt(_ptr(start), _ptr(end), start.size, threads, _ptr(a), _ptr(o), _ptr(ln), cap, C.byref(nb))
        if rc == GL_OK:
            k = nb.value
            return a[:k], o[: k * 256], ln[: k * 256]
        if rc != GL_ERANGE:
            raise GlError(rc, "gl_pack_segments16: bad arguments")
        cap = nb.value + 1


def indexsplit_layout(sample_sizes, R: int):
    """CSR layout gl_indexsplit_accumulate wants: (sizes int64, ptr int64[S*(R+1)], out_ptr int64[R+1])"""
    S = len(sample_sizes)
    flat, ptr, maxlen = [], np.zeros(S * (R + 1), np.int64), np.zeros(R, np.int64)
    off = 0
    for s, per_ref in enumerate(sample_sizes):
        for r in range(R):
            ptr[s * (R + 1) + r] = off
            if r < len(per_ref):
                a = np.asarray(per_ref[r], np.int64)
                flat.append(a); off += a.size
                maxlen[r] = max(maxlen[r], a.size)
        ptr[s * (R + 1) + R] = off
    sizes = np.concatenate(flat) if flat else np.zeros(0, np.int64)
    return sizes, ptr, np.concatenate([[0], np.cumsum(maxlen)]).astype(np.int64)


def indexsplit_chunks(tile_sum, out_ptr, names, ref_lens, ref_ids, N: int, problems=()) -> bytes:
    """Host-only: gl_indexsplit_chunks -> the output lines."""
    tile_sum = _as(tile_sum, np.float64)
    out_ptr = _as(out_ptr, np.int64)
    arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
    lens, ids = _as(np.asarray(ref_lens), np.int64), _as(np.asarray(ref_ids), np.int32)
    pr = _as(np.asarray([p[0] for p in problems]), np.int32)
    ps = _as(np.asarray([p[1] for p in problems]), np.int64)
    pe = _as(np.asarray([p[2] for p in problems]), np.int64)
    t, n = _vp(), C.c_int64(0)
    rc = lib.gl_indexsplit_chunks(_ptr(tile_sum), _ptr(out_ptr), out_ptr.size - 1, arr, _ptr(lens), _ptr(ids), len(names), N,
                                  _ptr(pr), _ptr(ps), _ptr(pe), len(problems), C.byref(t), C.byref(n))
    if rc != GL_OK:
        raise GlError(rc, "gl_indexsplit_chunks: bad arguments")
    try:
        return C.string_at(t, n.value)
    finally:
        lib.gl_free_text(t)


def pack_segments16_fixed(start: np.ndarray, end: np.ndarray, threads: int = 0, esc_cap: Optional[int] = None):
    """fixed-block packed16 (gl_pack_segments16_fixed_mt): (anchors, off, len, esc_start, esc_end)"""
    start, end = _as(start, np.int32), _as(end, np.int32)
    n = start.size
    nb = (n + 255) // 256
    anchors, off, ln = np.empty(nb, np.int32), np.empty(nb * 256, np.uint16), np.empty(nb * 256, np.uint16)
    cap = n if esc_cap is None else esc_cap
    es, ee = np.empty(max(cap, 1), np.int32), np.empty(max(cap, 1), np.int32)
    m = C.c_int64(0)
    rc = lib.gl_pack_segments16_fixed_mt(_ptr(start), _ptr(end), n, threads, _ptr(anchors), _ptr(off), _ptr(ln), _ptr(es), _ptr(ee), cap, C.byref(m))
    if rc != 0:
        raise GlError(rc, "gl_pack_segments16_fixed_mt (needs %d escapes)" % m.value)
    return anchors, off, ln, es[: m.value].copy(), ee[: m.value].copy()


def pack_segments8(start: np.ndarray, end: np.ndarray, threads: Optional[int] = None):
    """Host-only: (anchors int32[nb], dstart uint8[nb*64], len uint8[nb*64]) — the feeder's densest format (short reads).
    threads=None: the single-threaded packer; an int: gl_pack_segments8_mt (0 = all pool threads)."""
    start, end = _as(start, np.int32), _as(end, np.int32)
    nb = C.c_int64(0)
    cap = max(1, start.size // 48 + 64)
    while True:
        a = np.empty(cap, np.int32)
        d = np.empty(cap * 64, np.uint8)
        ln = np.empty(cap * 64, np.uint8)
        if threads is None:
            rc = lib.gl_pack_segments8(_ptr(start), _ptr(end), start.size, _ptr(a), _ptr(d), _ptr(ln), cap, C.byref(nb))
        else:
            rc = lib.gl_pack_segments8_mt(_ptr(start), _ptr(end), start.size, threads, _ptr(a), _ptr(d), _ptr(ln), cap, C.byref(nb))
        if rc == GL_OK:
            k = nb.value
            return a[:k], d[: k * 64], ln[: k * 64]
        if rc != GL_ERANGE:
            raise GlError(rc, "gl_pack_segments8: bad arguments")
        cap = nb.value + 1


def unpack_segments8(anchors, dstart, ln):
    """numpy decode of packed8 (what depth_unpack8_kernel computes): -> (start, end) int64, empty slots dropped"""
    nb = anchors.size
    d = dstart.reshape(nb, 64).astype(np.int64)
    s = anchors.astype(np.int64)[:, None] + np.cumsum(d, axis=1)
    l = ln.reshape(nb, 64).astype(np.int64)
    keep = l > 0
    return s[keep], (s + l)[keep]


def bam_segments(path: str, min_mapq: int = 1, threads: int = 4, only_tid: int = -1):
    """Host-only feeder: {"refs": [(name, length)], "segments": {tid: (start, end)}, "n_records", "n_pass"}."""
    h = _vp()
    err = C.create_string_buffer(512)
    rc = lib.gl_bam_decode_segments(path.encode(), min_mapq, threads, only_tid, C.byref(h), C.cast(err, _vp), 512)
    if rc != GL_OK:
        raise GlError(rc, err.value.decode())
    try:
        n, nrec, npass = C.c_int32(0), C.c_int64(0), C.c_int64(0)
        lib.gl_segset_n_refs(h, C.byref(n), C.byref(nrec), C.byref(npass))
        refs, segs = [], {}
        for tid in range(n.value):
            name, ln, ps, pe, k = C.c_char_p(), C.c_int64(0), _vp(), _vp(), C.c_int64(0)
            lib.gl_segset_ref(h, tid, C.byref(name), C.byref(ln), C.byref(ps), C.byref(pe), C.byref(k))
            refs.append((name.value.decode(), ln.value))
            if k.value:
                s_ = np.ctypeslib.as_array(C.cast(ps, _i32p), (k.value,)).copy()
                e_ = np.ctypeslib.as_array(C.cast(pe, _i32p), (k.value,)).copy()
                segs[tid] = (s_, e_)
        return {"refs": refs, "segments": segs, "n_records": nrec.value, "n_pass": npass.value}
    finally:
        lib.gl_segset_free(h)


class _BamSegments(C.Structure):
    _fields_ = [("format", C.c_int32), ("units", C.c_int32), ("max_len", C.c_int32), ("_pad", C.c_int32), ("n", C.c_int64),
                ("a0", _vp), ("a1", _vp), ("a2", _vp), ("n_records", C.c_int64), ("n_pass", C.c_int64), ("bytes_in", C.c_int64),
                ("bytes_out", C.c_int64), ("inflate_s", C.c_double), ("parse_s", C.c_double), ("wall_s", C.c_double)]


class Bam:
    """Index-guided parallel feeder (gl_bam_*): host-only."""

    def __init__(self, path: str):
        h = _vp()
        err = C.create_string_buffer(512)
        rc = lib.gl_bam_open(path.encode(), C.byref(h), C.cast(err, _vp), 512)
        if rc != GL_OK:
            raise GlError(rc, err.value.decode())
        self.h = h
        n, hi = C.c_int32(0), C.c_int32(0)
        lib.gl_bam_info(h, C.byref(n), C.byref(hi))
        self.has_index = bool(hi.value)
        self.index_path, self.index_geometry = None, None      # the .bai / .csi loaded, and its (min_shift, depth, is_csi)
        if self.has_index:
            ip, ms, dp, ic = C.c_char_p(), C.c_int32(0), C.c_int32(0), C.c_int32(0)
            if lib.gl_bam_index(h, C.byref(ip), C.byref(ms), C.byref(dp), C.byref(ic)) == GL_OK:
                self.index_path, self.index_geometry = ip.value.decode(), (ms.value, dp.value, bool(ic.value))
        self.refs = []
        for tid in range(n.value):
            name, ln, nm = C.c_char_p(), C.c_int64(0), C.c_int64(0)
            lib.gl_bam_ref(h, tid, C.byref(name), C.byref(ln), C.byref(nm))
            self.refs.append((name.value.decode(), ln.value, nm.value))

    def close(self):
        if self.h:
            lib.gl_bam_close(self.h)
            self.h = None

    def decode(self, tid: int, beg: int = 0, end: int = 1 << 40, min_mapq: int = 1, threads: int = 0, want: int = 0):
        """-> dict(format, arrays (copies), stats)"""
        o = _BamSegments()
        err = C.create_string_buffer(512)
        rc = lib.gl_bam_decode(self.h, tid, beg, end, min_mapq, threads, want, C.byref(o), C.cast(err, _vp), 512)
        if rc != GL_OK:
            raise GlError(rc, err.value.decode())
        out = {"format": o.format, "n": o.n, "units": o.units, "max_len": o.max_len, "n_records": o.n_records, "n_pass": o.n_pass,
               "bytes_in": o.bytes_in, "bytes_out": o.bytes_out, "inflate_s": o.inflate_s, "parse_s": o.parse_s, "wall_s": o.wall_s}
        if o.format == 8 and o.n:
            out["anchors"] = np.ctypeslib.as_array(C.cast(o.a0, _i32p), (o.n,)).copy()
            out["dstart"] = np.ctypeslib.as_array(C.cast(o.a1, _u8p), (o.n * 64,)).copy()
            out["len"] = np.ctypeslib.as_array(C.cast(o.a2, _u8p), (o.n * 64,)).copy()
        elif o.format == 32 and o.n:
            out["start"] = np.ctypeslib.as_array(C.cast(o.a0, _i32p), (o.n,)).copy()
            out["end"] = np.ctypeslib.as_array(C.cast(o.a1, _i32p), (o.n,)).copy()
        return out


def bam_decode_device(ctx: "Ctx", bam: Bam, tid: int, min_mapq: int = 1):
    """The GPU feeder (BGZF inflate + record parse on the device) -> dict(start, end (copies), stats); GlError(GL_ESTATE) when
    the reference cannot be done on the device."""
    o = _BamSegments()
    ps, pe, n = _vp(), _vp(), C.c_int64(0)
    rc = lib.gl_bam_decode_device(ctx.h, bam.h, tid, min_mapq, C.byref(ps), C.byref(pe), C.byref(n), C.byref(o))
    return _device_segments(ctx, rc, o, ps, pe, n)


def bam_decode_device_regions(ctx: "Ctx", bam: Bam, tid: int, beg, end, min_mapq: int = 1):
    """The GPU feeder over a region query: the blocks of reference tid's passing records that meet one of the intervals
    [beg[i], end[i]), in BAM order, decoded from only the BGZF members the index's bins name -> the dict bam_decode_device
    gives; GlError(GL_ESTATE) when the device cannot do it."""
    b_ = np.ascontiguousarray(beg, np.int64)
    e_ = np.ascontiguousarray(end, np.int64)
    if b_.shape != e_.shape or b_.ndim != 1:
        raise ValueError("beg and end must be 1-D arrays of one length")
    o = _BamSegments()
    ps, pe, n = _vp(), _vp(), C.c_int64(0)
    rc = lib.gl_bam_decode_device_regions(ctx.h, bam.h, tid, _ptr(b_) if b_.size else None, _ptr(e_) if e_.size else None, b_.size, min_mapq,
                                          C.byref(ps), C.byref(pe), C.byref(n), C.byref(o))
    return _device_segments(ctx, rc, o, ps, pe, n)


def bam_region_chunks(bam: Bam, tid: int, beg, end):
    """(vb, ve) uint64 arrays: the virtual-offset ranges a region query of the intervals [beg[i], end[i]) on reference tid
    reads (gl_bam_region_chunks; host only)"""
    b_ = np.ascontiguousarray(beg, np.int64)
    e_ = np.ascontiguousarray(end, np.int64)
    if b_.shape != e_.shape or b_.ndim != 1:
        raise ValueError("beg and end must be 1-D arrays of one length")
    args = (bam.h, tid, _ptr(b_) if b_.size else None, _ptr(e_) if e_.size else None, b_.size)
    n = C.c_int64(0)
    rc = lib.gl_bam_region_chunks(*args, None, None, 0, C.byref(n))
    if rc == GL_ERANGE:
        vb, ve = np.empty(n.value, np.uint64), np.empty(n.value, np.uint64)
        rc = lib.gl_bam_region_chunks(*args, _ptr(vb), _ptr(ve), n.value, C.byref(n))
    else:
        vb, ve = np.zeros(0, np.uint64), np.zeros(0, np.uint64)
    if rc != GL_OK:
        raise GlError(rc, "gl_bam_region_chunks")
    return vb, ve


def _device_segments(ctx, rc, o, ps, pe, n):
    if rc != GL_OK:
        raise GlError(rc, lib.gl_last_error(ctx.h).decode())
    out = {"n": n.value, "units": o.units, "max_len": o.max_len, "n_records": o.n_records, "n_pass": o.n_pass, "bytes_in": o.bytes_in,
           "bytes_out": o.bytes_out, "inflate_s": o.inflate_s, "parse_s": o.parse_s, "wall_s": o.wall_s, "d_start": ps.value, "d_end": pe.value}
    if n.value:
        s_, e_ = np.empty(n.value, np.int32), np.empty(n.value, np.int32)
        ctx._ck(lib.gl_memcpy_d2h(ctx.h, _ptr(s_), ps.value, n.value * 4))
        ctx._ck(lib.gl_memcpy_d2h(ctx.h, _ptr(e_), pe.value, n.value * 4))
        out["start"], out["end"] = s_, e_
    else:
        out["start"], out["end"] = np.zeros(0, np.int32), np.zeros(0, np.int32)
    return out


class CovStats(C.Structure):
    """gl_covstats: the reference's Stats, the counters behind it, which route ran and its phase times"""
    _fields_ = ([(k, C.c_double) for k in ("insert_mean", "insert_sd", "template_mean", "template_sd", "read_length_mean", "read_length_median",
                                           "proportion_bad", "proportion_unmapped", "proportion_properly_paired", "proportion_duplicate")] +
                [(k, C.c_int32) for k in ("insert_pct5", "insert_pct95", "max_read_length", "path")] +
                [(k, C.c_int64) for k in ("n_unmapped", "k", "n_bad", "n_dup", "n_proper", "n_read_len", "n_insert", "n_records_read", "h_len",
                                          "bytes_in", "bytes_out")] +
                [(k, C.c_double) for k in ("read_s", "inflate_s", "index_s", "fields_s", "cut_s", "tail_s", "wall_s")] +
                [("n_batches", C.c_int32), ("prefetched", C.c_int32)])
    STATS = ("insert_mean", "insert_sd", "insert_pct5", "insert_pct95", "template_mean", "template_sd", "read_length_mean", "read_length_median",
             "proportion_bad", "proportion_unmapped", "proportion_properly_paired", "proportion_duplicate", "max_read_length")
    COUNTERS = ("n_unmapped", "k", "n_bad", "n_dup", "n_proper", "n_read_len", "n_insert", "n_records_read")

    def as_dict(self):
        return {k: getattr(self, k) for k, _ in self._fields_}


def _covstats_two_call(ctx, fn, st=None):
    """the two-call convention: once for h_len, once more with room -> (CovStats, H)"""
    st = st if st is not None else CovStats()
    H = np.empty(1 << 14, np.float64)                      # room for most histograms, so one call is the usual case
    rc = fn(C.byref(st), _ptr(H), H.size)
    if rc == GL_ERANGE and st.h_len > H.size:
        H = np.empty(st.h_len, np.float64)
        rc = fn(C.byref(st), _ptr(H), H.size)
    if rc != GL_OK:
        e = GlError(rc, lib.gl_last_error(ctx.h if ctx is not None else None).decode())
        e.stats = st
        raise e
    return st, H[: st.h_len].copy()


def bam_covstats(ctx: "Ctx", bam: Bam, n: int, skip: int = 100000, samples: bool = False):
    """covstats.BamStats sampled on the device -> (CovStats, H[, (read_len, insert, tmpl) in file order]); GlError(GL_ESTATE)
    when the file cannot be sampled there."""
    st, H = _covstats_two_call(ctx, lambda o, h, cap: lib.gl_bam_covstats(ctx.h, bam.h, n, skip, o, h, cap))
    if not samples:
        return st, H
    ps = [_vp(), _vp(), _vp()]
    ctx._ck(lib.gl_bam_covstats_samples(ctx.h, *[C.byref(p) for p in ps]))
    out = []
    for p, k in zip(ps, (st.n_read_len, st.n_insert, st.n_insert)):
        a = np.empty(k, np.int32)
        if k:
            ctx._ck(lib.gl_memcpy_d2h(ctx.h, _ptr(a), p.value, k * 4))
        out.append(a)
    return st, H, tuple(out)


def bam_covstats_prefetch(ctx: "Ctx", bam: Bam, n: int, skip: int = 100000):
    """start reading bam's first batch for a later bam_covstats(ctx, bam, n, skip) and return at once; a file the device would
    refuse gets no prefetch (bam_covstats reports it)"""
    ctx._ck(lib.gl_bam_covstats_prefetch(ctx.h, bam.h, n, skip))


def bam_covstats_host(ctx: Optional["Ctx"], bam: Bam, n: int, skip: int = 100000, samples: bool = False):
    """the same from the host sampler; ctx may be None (no device is touched then)"""
    h = ctx.h if ctx is not None else None
    st, H = _covstats_two_call(ctx, lambda o, hh, cap: lib.gl_bam_covstats_host(h, bam.h, n, skip, o, hh, cap))
    if not samples:
        return st, H
    ps = [_vp(), _vp(), _vp()]
    lib.gl_bam_covstats_host_samples(bam.h, *[C.byref(p) for p in ps])
    out = tuple(np.ctypeslib.as_array(C.cast(p, _i32p), (k,)).copy() if k else np.zeros(0, np.int32)
                for p, k in zip(ps, (st.n_read_len, st.n_insert, st.n_insert)))
    return st, H, out


def covstats_tail(ctx: Optional["Ctx"], read_len, insert, tmpl, n_unmapped=0, k=0, n_bad=0, n_dup=0, n_proper=0):
    """covstats.go:175-218 from host sample arrays and the five counters -> (CovStats, H); ctx may be None"""
    read_len, insert, tmpl = _as(read_len, np.int32), _as(insert, np.int32), _as(tmpl, np.int32)
    h = ctx.h if ctx is not None else None

    st = CovStats()
    st.n_unmapped, st.k, st.n_bad, st.n_dup, st.n_proper = n_unmapped, k, n_bad, n_dup, n_proper
    return _covstats_two_call(ctx, lambda o, hh, cap: lib.gl_covstats_tail(h, _ptr(read_len), read_len.size, _ptr(insert), insert.size,
                                                                         _ptr(tmpl), tmpl.size, o, hh, cap), st)


def crai_make_sizes(start, span, nbytes) -> np.ndarray:
    """Host-only: 16 KB pseudo-tile sizes of one reference from its CRAM slices (crai.go:56-127)."""
    start, span, nbytes = _as(start, np.int64), _as(span, np.int64), _as(nbytes, np.int32)
    cap = int((start[-1] + max(int(span[-1]), 0)) // 16384 + 64) if start.size else 1
    out = np.empty(cap, np.int64)
    n = C.c_int64(0)
    rc = lib.gl_crai_make_sizes(_ptr(start), _ptr(span), _ptr(nbytes), start.size, _ptr(out), cap, C.byref(n))
    if rc != GL_OK:
        raise GlError(rc, "gl_crai_make_sizes: tile-width logic error (the reference panics) or capacity")
    return out[: n.value].copy()


def bai_read(path: str):
    """A BAI or CSI -> dict(ioffsets (16 KB linear index per reference; rebuilt from the bins for a CSI), mapped, unmapped,
    has_stats, n_no_coor, min_shift, depth, is_csi); GlError on a file that is neither, or a malformed one."""
    h = _vp()
    err = C.create_string_buffer(512)
    rc = lib.gl_bai_read(path.encode(), C.byref(h), C.cast(err, _vp), 512)
    if rc != GL_OK:
        raise GlError(rc, err.value.decode())
    try:
        n, nc = C.c_int32(0), C.c_uint64(0)
        lib.gl_bai_n_refs(h, C.byref(n), C.byref(nc))
        ms, dp, ic = C.c_int32(0), C.c_int32(0), C.c_int32(0)
        lib.gl_bai_geometry(h, C.byref(ms), C.byref(dp), C.byref(ic))
        out = {"ioffsets": [], "mapped": [], "unmapped": [], "has_stats": [], "n_no_coor": nc.value, "min_shift": ms.value,
               "depth": dp.value, "is_csi": bool(ic.value)}
        for tid in range(n.value):
            p, k, m, u, hs = _vp(), C.c_int64(0), C.c_uint64(0), C.c_uint64(0), C.c_int32(0)
            lib.gl_bai_ref(h, tid, C.byref(p), C.byref(k), C.byref(m), C.byref(u), C.byref(hs))
            out["ioffsets"].append(np.ctypeslib.as_array(C.cast(p, _u64p), (k.value,)).copy() if k.value else np.zeros(0, np.uint64))
            out["mapped"].append(m.value); out["unmapped"].append(u.value); out["has_stats"].append(bool(hs.value))
        return out
    finally:
        lib.gl_bai_free(h)


class DevBuf:
    """A device allocation owned by a Ctx."""

    def __init__(self, ctx: "Ctx", nbytes: int):
        self.ctx, self.nbytes = ctx, int(nbytes)
        p = _vp()
        ctx._ck(lib.gl_dev_alloc(ctx.h, self.nbytes, C.byref(p)))
        self.ptr = p.value

    def upload(self, a: np.ndarray) -> "DevBuf":
        a = np.ascontiguousarray(a)
        assert a.nbytes <= self.nbytes
        self.ctx._ck(lib.gl_memcpy_h2d(self.ctx.h, self.ptr, _ptr(a), a.nbytes))
        return self

    def download(self, dtype, count: int) -> np.ndarray:
        out = np.empty(count, dtype=dtype)
        assert out.nbytes <= self.nbytes
        self.ctx._ck(lib.gl_memcpy_d2h(self.ctx.h, _ptr(out), self.ptr, out.nbytes))
        return out

    def free(self):
        if self.ptr:
            lib.gl_dev_free(self.ctx.h, self.ptr)
            self.ptr = None


class Ctx:
    """One GPU context (gl_ctx)."""

    def __init__(self, device: int = 0):
        h = _vp()
        rc = lib.gl_ctx_create(device, C.byref(h))
        if rc != GL_OK:
            raise GlError(rc, lib.gl_last_error(None).decode())
        self.h = h
        self.device = device

    def close(self):
        if self.h:
            lib.gl_ctx_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _ck(self, rc: int):
        if rc != GL_OK:
            raise GlError(rc, lib.gl_last_error(self.h).decode())

    # ---- plumbing
    def sync(self):
        self._ck(lib.gl_sync(self.h))

    def launch_count(self) -> int:
        n = C.c_int64(0)
        self._ck(lib.gl_launch_count(self.h, C.byref(n)))
        return n.value

    def dev_array(self, a: np.ndarray) -> DevBuf:
        a = np.ascontiguousarray(a)
        return DevBuf(self, max(a.nbytes, 16)).upload(a)

    def dev_empty(self, nbytes: int) -> DevBuf:
        return DevBuf(self, nbytes)

    def pinned_empty(self, count: int, dtype) -> np.ndarray:
        dt = np.dtype(dtype)
        p = _vp()
        self._ck(lib.gl_host_alloc_pinned(self.h, max(count * dt.itemsize, 16), C.byref(p)))
        buf = (C.c_char * (count * dt.itemsize)).from_address(p.value)
        arr = np.frombuffer(buf, dtype=dt, count=count)
        self._pinned = getattr(self, "_pinned", [])
        self._pinned.append(p.value)
        return arr

    def timer_start(self):
        self._ck(lib.gl_timer_start(self.h))

    def timer_stop_ms(self) -> float:
        ms = C.c_float(0)
        self._ck(lib.gl_timer_stop_ms(self.h, C.byref(ms)))
        return ms.value

    def profile_enable(self, on: bool):
        self._ck(lib.gl_profile_enable(self.h, 1 if on else 0))

    def profile_read(self):
        """[(kernel name, ms), ...] for every kernel launched since the last read"""
        buf = C.create_string_buffer(1 << 20)
        need = C.c_int64(0)
        self._ck(lib.gl_profile_read(self.h, C.cast(buf, _vp), len(buf), C.byref(need)))
        out = []
        for ln in buf.value.decode().splitlines():
            nm, ms = ln.rsplit(" ", 1)
            out.append((nm, float(ms)))
        return out

    def flush_l2(self):
        self._ck(lib.gl_flush_l2(self.h))

    # ---- depth
    def depth_begin(self, rs: int, re: int):
        self._ck(lib.gl_depth_begin(self.h, rs, re))

    def depth_add_segments(self, start: np.ndarray, end: np.ndarray):
        start, end = _as(start, np.int32), _as(end, np.int32)
        assert start.shape == end.shape
        self._ck(lib.gl_depth_add_segments(self.h, _ptr(start), _ptr(end), start.size))

    def depth_add_segments_device(self, d_start: DevBuf, d_end: DevBuf, n: int, offset: int = 0):
        self._ck(lib.gl_depth_add_segments_device(self.h, d_start.ptr + 4 * offset, d_end.ptr + 4 * offset, n))

    def depth_add_segments_packed16(self, anchors: np.ndarray, off: np.ndarray, ln: np.ndarray):
        self._ck(lib.gl_depth_add_segments_packed16(self.h, _ptr(anchors), _ptr(off), _ptr(ln), anchors.size))

    def depth_add_segments_packed8(self, anchors: np.ndarray, dstart: np.ndarray, ln: np.ndarray):
        self._ck(lib.gl_depth_add_segments_packed8(self.h, _ptr(anchors), _ptr(dstart), _ptr(ln), anchors.size))

    def depth_add_segments_packed8_device(self, d_anchors: "DevBuf", d_dstart: "DevBuf", d_len: "DevBuf", n_blocks: int):
        self._ck(lib.gl_depth_add_segments_packed8_device(self.h, d_anchors.ptr, d_dstart.ptr, d_len.ptr, n_blocks))

    def depth_region_packed8(self, rs: int, re: int, anchors, dstart, ln, W: int, mincov: int = 4, maxmean: int = 0,
                             run_break: int = 0, out=None):
        n_win = (re - 1) // W - rs // W + 1
        if out is None:
            out = (np.empty(n_win, np.int64), np.empty(max(1024, (re - rs) // 8), np.int32),
                   np.empty(max(1024, (re - rs) // 8), np.uint8))
        s, r0, rc_ = out
        nw, nr = C.c_int64(0), C.c_int64(0)
        self._ck(lib.gl_depth_region_packed8(self.h, rs, re, _ptr(anchors), _ptr(dstart), _ptr(ln), anchors.size, W, mincov,
                                             maxmean, run_break, _ptr(s), s.size, C.byref(nw), _ptr(r0), _ptr(rc_),
                                             min(r0.size, rc_.size), C.byref(nr)))
        return s[: nw.value], r0[: nr.value], rc_[: nr.value]

    def depth_region_packed16(self, rs: int, re: int, anchors, off, ln, W: int, mincov: int = 4, maxmean: int = 0,
                              run_break: int = 0, out=None):
        n_win = (re - 1) // W - rs // W + 1
        if out is None:
            out = (np.empty(n_win, np.int64), np.empty(max(1024, (re - rs) // 8), np.int32),
                   np.empty(max(1024, (re - rs) // 8), np.uint8))
        s, r0, rc_ = out
        nw, nr = C.c_int64(0), C.c_int64(0)
        self._ck(lib.gl_depth_region_packed16(self.h, rs, re, _ptr(anchors), _ptr(off), _ptr(ln), anchors.size, W, mincov,
                                              maxmean, run_break, _ptr(s), s.size, C.byref(nw), _ptr(r0), _ptr(rc_),
                                              min(r0.size, rc_.size), C.byref(nr)))
        return s[: nw.value], r0[: nr.value], rc_[: nr.value]

    def depth_reduce(self, W: int, mincov: int = 4, maxmean: int = 0, run_break: int = 0):
        self._ck(lib.gl_depth_reduce(self.h, W, mincov, maxmean, run_break))

    def depth_result_sizes(self) -> Tuple[int, int, int]:
        nw, nr, md = C.c_int64(0), C.c_int64(0), C.c_int32(0)
        self._ck(lib.gl_depth_result_sizes(self.h, C.byref(nw), C.byref(nr), C.byref(md)))
        return nw.value, nr.value, md.value

    def depth_get_windows(self) -> np.ndarray:
        nw, _, _ = self.depth_result_sizes()
        s = np.empty(nw, np.int64)
        self._ck(lib.gl_depth_get_windows(self.h, _ptr(s), nw))
        return s

    def depth_last_path(self) -> int:
        p = C.c_int32(0)
        self._ck(lib.gl_depth_last_path(self.h, C.byref(p)))
        return p.value

    def depth_transport_stats(self):
        """(transport, host pack seconds, bytes sent host->device, escaped segments) of the last depth_bed_contig call"""
        t, ps, hb, ne = C.c_int32(0), C.c_double(0), C.c_int64(0), C.c_int64(0)
        self._ck(lib.gl_depth_transport_stats(self.h, C.byref(t), C.byref(ps), C.byref(hb), C.byref(ne)))
        return t.value, ps.value, hb.value, ne.value

    def depth_transport_phases(self):
        ph = (C.c_double * 3)()
        self._ck(lib.gl_depth_transport_phases(self.h, ph))
        return [ph[0], ph[1], ph[2]]

    def depth_set_path(self, path: int):
        self._ck(lib.gl_depth_set_path(self.h, path))

    def depth_get_runs(self, want_end: bool = False):
        _, nr, _ = self.depth_result_sizes()
        rs_ = np.empty(nr, np.int32)
        rc_ = np.empty(nr, np.uint8)
        re_ = np.empty(nr, np.int32) if want_end else None
        self._ck(lib.gl_depth_get_runs(self.h, _ptr(rs_), _ptr(re_), _ptr(rc_), nr))
        return (rs_, re_, rc_) if want_end else (rs_, rc_)

    def depth_windows(self, W: int, n_windows: int, want_min: bool = True):
        s = np.empty(n_windows, np.int64)
        m = np.empty(n_windows, np.int32) if want_min else None
        self._ck(lib.gl_depth_windows(self.h, W, _ptr(s), _ptr(m), n_windows))
        return s, m

    def depth_classes(self, mincov: int, maxmean: int, cap: int):
        rs_ = np.empty(cap, np.int32)
        re_ = np.empty(cap, np.int32)
        rc_ = np.empty(cap, np.uint8)
        n = C.c_int64(0)
        self._ck(lib.gl_depth_classes(self.h, mincov, maxmean, _ptr(rs_), _ptr(re_), _ptr(rc_), cap, C.byref(n)))
        return rs_[: n.value], re_[: n.value], rc_[: n.value]

    def indexsplit_accumulate(self, sizes, ptr, S: int, R: int, out_ptr) -> np.ndarray:
        sizes, ptr, out_ptr = _as(sizes, np.int64), _as(ptr, np.int64), _as(out_ptr, np.int64)
        out = np.zeros(int(out_ptr[-1]), np.float64)
        self._ck(lib.gl_indexsplit_accumulate(self.h, _ptr(sizes), _ptr(ptr), S, R, _ptr(out_ptr), _ptr(out)))
        return out

    def depth_interval_sums(self, a, b) -> np.ndarray:
        a, b = _as(a, np.int32), _as(b, np.int32)
        out = np.empty(a.size, np.int64)
        self._ck(lib.gl_depth_interval_sums(self.h, _ptr(a), _ptr(b), a.size, _ptr(out)))
        return out

    def fasta_load(self, record_bytes):
        a = np.frombuffer(record_bytes, np.uint8) if not isinstance(record_bytes, np.ndarray) else _as(record_bytes, np.uint8)
        self._ck(lib.gl_fasta_load(self.h, _ptr(a), a.size))

    def fasta_stats(self, byte_start, byte_end):
        """-> (counts[n,4] = G+C, lower, ACGT, CpG ; stats[n,3] = GC, CpG, Masked)"""
        a, b = _as(byte_start, np.int64), _as(byte_end, np.int64)
        counts = np.zeros((a.size, 4), np.int64)
        stats = np.zeros((a.size, 3), np.float64)
        self._ck(lib.gl_fasta_stats(self.h, _ptr(a), _ptr(b), a.size, _ptr(counts), _ptr(stats)))
        return counts, stats

    def depth_perbase(self, length: int) -> np.ndarray:
        out = np.empty(length, np.int32)
        self._ck(lib.gl_depth_perbase(self.h, _ptr(out)))
        return out

    def depth_region(self, rs: int, re: int, start: np.ndarray, end: np.ndarray, W: int, mincov: int = 4,
                     maxmean: int = 0, run_break: int = 0, out=None):
        """One call, host in / host out.  `out` = (sum, run_start, run_class) preallocated arrays."""
        n_win = (re - 1) // W - rs // W + 1
        if out is None:
            out = (np.empty(n_win, np.int64), np.empty(max(1024, (re - rs) // 8), np.int32),
                   np.empty(max(1024, (re - rs) // 8), np.uint8))
        s, r0, rc_ = out
        nw, nr = C.c_int64(0), C.c_int64(0)
        self._ck(lib.gl_depth_region(self.h, rs, re, _ptr(start), _ptr(end), start.size, W, mincov, maxmean, run_break,
                                     _ptr(s), s.size, C.byref(nw), _ptr(r0), _ptr(rc_), min(r0.size, rc_.size),
                                     C.byref(nr)))
        return s[: nw.value], r0[: nr.value], rc_[: nr.value]

    # ---- depth text (device formatter)
    def _text_bufs(self, chrom: str, n_win: int, out):
        if out is None:
            out = (np.empty(int(lib.gl_depth_text_bound(chrom.encode(), n_win)), np.uint8), np.empty(1 << 16, np.uint8))
        return out

    def depth_text(self, chrom: str, out=None) -> Tuple[bytes, bytes]:
        """(depth.bed bytes, callable.bed bytes) of the last reduce, formatted on the device."""
        nw, _, _ = self.depth_result_sizes()
        hd, ca = self._text_bufs(chrom, nw, out)
        hl, cl = C.c_int64(0), C.c_int64(0)
        rc = lib.gl_depth_text(self.h, chrom.encode(), _ptr(hd), hd.size, C.byref(hl), _ptr(ca), ca.size, C.byref(cl))
        if rc == GL_ERANGE and out is None:
            hd, ca = np.empty(hl.value + 16, np.uint8), np.empty(cl.value + 16, np.uint8)
            rc = lib.gl_depth_text(self.h, chrom.encode(), _ptr(hd), hd.size, C.byref(hl), _ptr(ca), ca.size, C.byref(cl))
        self._ck(rc)
        return hd[: hl.value].tobytes(), ca[: cl.value].tobytes()

    def depth_format_rows(self, chrom: str, row_s, row_e, row_sum) -> bytes:
        row_s, row_e, row_sum = _as(row_s, np.int32), _as(row_e, np.int32), _as(row_sum, np.int64)
        out = np.empty(row_s.size * (len(chrom) + 33) + 16, np.uint8)
        ln = C.c_int64(0)
        self._ck(lib.gl_depth_format_rows(self.h, chrom.encode(), _ptr(row_s), _ptr(row_e), _ptr(row_sum), row_s.size, _ptr(out),
                                          out.size, C.byref(ln)))
        return out[: ln.value].tobytes()

    def _bed_text(self, fn, args, chrom: str, n_win: int, out, raw: bool):
        """fn(*args, depth_bed, cap, &len, callable_bed, cap, &len): BED text into `out` or buffers of the size it asks for"""
        keep = out is not None
        hd, ca = self._text_bufs(chrom, n_win, out)
        hl, cl = C.c_int64(0), C.c_int64(0)
        rc = fn(*args, _ptr(hd), hd.size, C.byref(hl), _ptr(ca), ca.size, C.byref(cl))
        if rc == GL_ERANGE and not keep:
            hd, ca = np.empty(hl.value + 16, np.uint8), np.empty(cl.value + 16, np.uint8)
            rc = fn(*args, _ptr(hd), hd.size, C.byref(hl), _ptr(ca), ca.size, C.byref(cl))
        self._ck(rc)
        if raw:
            return hl.value, cl.value
        return hd[: hl.value].tobytes(), ca[: cl.value].tobytes()

    def depth_bed_contig(self, chrom: str, length: int, start, end, W: int, mincov: int = 4, maxmean: int = 0,
                         step: int = 10_000_000, threads: int = 0, out=None, raw: bool = False):
        """One call: host int32 segments in -> (depth.bed, callable.bed) bytes out.  raw=True returns the two lengths only
        (the bytes are in `out`)."""
        args = (self.h, chrom.encode(), length, _ptr(start), _ptr(end), start.size, W, mincov, maxmean, step, threads)
        return self._bed_text(lib.gl_depth_bed_contig, args, chrom, (length - 1) // W + 1, out, raw)

    def depth_bed_region(self, chrom: str, rs: int, re: int, start, end, W: int, mincov: int = 4, maxmean: int = 0,
                         step: int = 10_000_000, threads: int = 0, out=None, raw: bool = False):
        """depth_bed_contig for the whole chunks [rs, re) of a contig (rs a multiple of step): what `goleft depth` writes for
        one pass over a contig longer than a pass"""
        args = (self.h, chrom.encode(), rs, re, _ptr(start), _ptr(end), start.size, W, mincov, maxmean, step, threads)
        return self._bed_text(lib.gl_depth_bed_region, args, chrom, (re - 1) // W - rs // W + 1, out, raw)

    def depth_bed_contig_packed8(self, chrom: str, length: int, anchors, dstart, ln, W: int, mincov: int = 4, maxmean: int = 0,
                                 step: int = 10_000_000, out=None, raw: bool = False):
        args = (self.h, chrom.encode(), length, _ptr(anchors), _ptr(dstart), _ptr(ln), anchors.size, W, mincov, maxmean, step)
        return self._bed_text(lib.gl_depth_bed_contig_packed8, args, chrom, (length - 1) // W + 1, out, raw)

    def bgzf_inflate(self, data: bytes):
        """GPU inflate of a whole BGZF byte string -> (inflated bytes, per-block status int32[]); test / tool helper"""
        b = np.frombuffer(data, np.uint8)
        offs, outs, p = [0], [0], 0
        while p + 18 <= b.size:
            bs = int(b[p + 16]) + (int(b[p + 17]) << 8) + 1
            if p + bs > b.size:
                break
            isize = int.from_bytes(bytes(b[p + bs - 4:p + bs]), "little")
            p += bs
            offs.append(p); outs.append(outs[-1] + isize)
        nb = len(offs) - 1
        d_c, d_co, d_oo = self.dev_array(b), self.dev_array(np.array(offs, np.int64)), self.dev_array(np.array(outs, np.int64))
        d_out, d_st = self.dev_empty(max(outs[-1], 16)), self.dev_array(np.full(max(nb, 1), -1, np.int32))
        try:
            self._ck(lib.gl_bgzf_inflate_device(self.h, d_c.ptr, d_co.ptr, d_oo.ptr, nb, d_out.ptr, d_st.ptr))
            self.sync()
            return d_out.download(np.uint8, outs[-1]).tobytes(), d_st.download(np.int32, nb)
        finally:
            for x in (d_c, d_co, d_oo, d_out, d_st):
                x.free()

    # ---- indexcov
    def indexcov_sizes(self, voff: np.ndarray, ref_ptr: np.ndarray):
        voff, ref_ptr = _as(voff, np.uint64), _as(ref_ptr, np.int64)
        n_refs = ref_ptr.size - 1
        size_ptr = np.zeros(n_refs + 1, np.int64)
        sizes = np.empty(max(int(voff.size), 1), np.int64)
        self._ck(lib.gl_indexcov_sizes(self.h, _ptr(voff), _ptr(ref_ptr), n_refs, _ptr(sizes), _ptr(size_ptr)))
        return sizes[: size_ptr[-1]], size_ptr

    def indexcov_scale(self, sizes: np.ndarray) -> int:
        sizes = _as(sizes, np.int64)
        m = C.c_int64(0)
        self._ck(lib.gl_indexcov_scale(self.h, _ptr(sizes), sizes.size, C.byref(m)))
        return m.value

    def indexcov_normalize(self, sizes: np.ndarray, median: float) -> np.ndarray:
        sizes = _as(sizes, np.int64)
        out = np.empty(sizes.size, np.float32)
        self._ck(lib.gl_indexcov_normalize(self.h, _ptr(sizes), sizes.size, float(median), _ptr(out)))
        return out

    def indexcov_cohort(self, sizes: np.ndarray, sample_ptr: np.ndarray, want_depth: bool = True):
        sizes, sample_ptr = _as(sizes, np.int64), _as(sample_ptr, np.int64)
        S = sample_ptr.size - 1
        med = np.empty(S, np.float64)
        dep = np.empty(sizes.size, np.float32) if want_depth else None
        self._ck(lib.gl_indexcov_cohort(self.h, _ptr(sizes), _ptr(sample_ptr), S, _ptr(med), _ptr(dep)))
        return med, dep

    def indexcov_cohort_fallbacks(self) -> int:
        n = C.c_int32(0)
        self._ck(lib.gl_indexcov_cohort_fallbacks(self.h, C.byref(n)))
        return n.value

    def indexcov_sizes_batch(self, voff: np.ndarray, voff_off, n_intv, size_off, total_sizes: int) -> np.ndarray:
        """I1 for many (sample, reference) descriptors in one launch (arrays uploaded here; the device form keeps them resident)"""
        d_v, d_o = self.dev_array(_as(voff, np.uint64)), self.dev_array(_as(voff_off, np.int64))
        d_n, d_s = self.dev_array(_as(n_intv, np.int32)), self.dev_array(_as(size_off, np.int64))
        d_out = self.dev_empty(max(total_sizes, 1) * 8)
        try:
            self._ck(lib.gl_indexcov_sizes_batch_device(self.h, d_v.ptr, d_o.ptr, d_n.ptr, d_s.ptr, len(n_intv), d_out.ptr))
            return d_out.download(np.int64, total_sizes)
        finally:
            for b in (d_v, d_o, d_n, d_s, d_out):
                b.free()

    def indexcov_counts(self, depth: np.ndarray, counts: Optional[np.ndarray] = None) -> np.ndarray:
        depth = _as(depth, np.float32)
        if counts is None:
            counts = np.zeros(INDEXCOV_SLOTS, np.int32)
        self._ck(lib.gl_indexcov_counts(self.h, _ptr(depth), depth.size, _ptr(counts)))
        return counts

    def indexcov_bins(self, depth: np.ndarray, longest: int, out4: Optional[np.ndarray] = None) -> np.ndarray:
        depth = _as(depth, np.float32)
        if out4 is None:
            out4 = np.zeros(4, np.int64)
        self._ck(lib.gl_indexcov_bins(self.h, _ptr(depth), depth.size, longest, _ptr(out4)))
        return out4

    def indexcov_counts_batch(self, depth: np.ndarray, seg_ptr: np.ndarray, longest: Optional[np.ndarray] = None):
        depth, seg_ptr = _as(depth, np.float32), _as(seg_ptr, np.int64)
        n = seg_ptr.size - 1
        lg = None if longest is None else _as(longest, np.int64)
        counts = np.empty((n, INDEXCOV_SLOTS), np.int32)
        bins = np.empty((n, 4), np.int64)
        self._ck(lib.gl_indexcov_counts_batch(self.h, _ptr(depth), _ptr(seg_ptr), _ptr(lg), n, _ptr(counts), _ptr(bins)))
        return counts, bins

    def indexcov_xnorm(self, depths: np.ndarray, lens: np.ndarray) -> np.ndarray:
        d = np.ascontiguousarray(depths, np.float32).copy()
        lens = _as(lens, np.int32)
        S, T = d.shape
        self._ck(lib.gl_indexcov_xnorm(self.h, _ptr(d), _ptr(lens), S, T))
        return d

    def indexcov_cohort_device(self, d_sizes: DevBuf, d_sample_ptr: DevBuf, S: int, d_medians: DevBuf, d_depth: Optional[DevBuf]):
        self._ck(lib.gl_indexcov_cohort_device(self.h, d_sizes.ptr, d_sample_ptr.ptr, S, d_medians.ptr,
                                               d_depth.ptr if d_depth is not None else None))

    def indexcov_counts_segs_device(self, d_depth: DevBuf, d_seg_start: DevBuf, d_seg_len: DevBuf, d_longest: Optional[DevBuf],
                                    n_seg: int, d_counts70: DevBuf, d_bins4: DevBuf):
        self._ck(lib.gl_indexcov_counts_segs_device(self.h, d_depth.ptr, d_seg_start.ptr, d_seg_len.ptr,
                                                    d_longest.ptr if d_longest is not None else None, n_seg, d_counts70.ptr,
                                                    d_bins4.ptr))

    def plot_select_device(self, d_vals: DevBuf, d_off: DevBuf, d_len: DevBuf, n: int, d_sel3: DevBuf, d_yext2: DevBuf):
        self._ck(lib.gl_plot_select_device(self.h, d_vals.ptr, d_off.ptr, d_len.ptr, n, d_sel3.ptr, d_yext2.ptr))

    def plot_raster_series_device(self, d_vals: DevBuf, d_off: DevBuf, d_sel3: DevBuf, mult: float, d_chart: DevBuf, d_draw: DevBuf,
                                  n: int, d_xf: DevBuf, n_charts: int, W: int, H: int, r: float, d_img: DevBuf):
        self._ck(lib.gl_plot_raster_series_device(self.h, d_vals.ptr, d_off.ptr, d_sel3.ptr, mult, d_chart.ptr, d_draw.ptr, n, d_xf.ptr,
                                                  n_charts, W, H, r, d_img.ptr))

    def plot_select(self, vals, off, lens):
        """gl_plot_select_device on host arrays: (sel (n,3), yext (n,2))"""
        vals, off, lens = _as(vals, np.float32), _as(off, np.int64), _as(lens, np.int64)
        n = off.size
        bufs = [DevBuf(self, max(16, a.nbytes)).upload(a) for a in (vals, off, lens)] + [DevBuf(self, max(16, n * 24)), DevBuf(self, max(16, n * 8))]
        try:
            self.plot_select_device(*bufs[:3], n, *bufs[3:])
            return bufs[3].download(np.int64, n * 3).reshape(n, 3), bufs[4].download(np.float32, n * 2).reshape(n, 2)
        finally:
            for b in bufs:
                b.free()

    def plot_raster_series(self, vals, off, sel, mult: float, chart, draw, xf, n_charts: int, W: int, H: int, r: float) -> np.ndarray:
        """gl_plot_raster_series_device on host arrays: the (n_charts, H, W) index image"""
        arrs = [_as(vals, np.float32), _as(off, np.int64), _as(sel, np.int64), _as(chart, np.int32), _as(draw, np.uint32),
                _as(xf, np.float64)]
        bufs = [DevBuf(self, max(16, a.nbytes)).upload(a) for a in arrs] + [DevBuf(self, max(16, n_charts * W * H * 4))]
        try:
            v, o, sl, ch, dr, x, img = bufs
            self.plot_raster_series_device(v, o, sl, mult, ch, dr, arrs[3].size, x, n_charts, W, H, r, img)
            return img.download(np.uint32, n_charts * W * H).reshape(n_charts, H, W)
        finally:
            for b in bufs:
                b.free()

    def _paths(self, size, emit, arrs, n: int, cap: Optional[int]):
        bufs = [DevBuf(self, max(16, a.nbytes)).upload(a) for a in arrs]
        d_len, d_pos = DevBuf(self, max(16, n * 8)), DevBuf(self, (n + 1) * 8)
        d_out = None
        try:
            size(bufs, d_len, d_pos)
            self.sync()
            ln, pos = d_len.download(np.int64, n), d_pos.download(np.int64, n + 1)
            total = int(pos[n])
            room = total if cap is None else cap
            d_out = DevBuf(self, max(16, room))
            emit(bufs, d_pos, total, d_out, room)
            self.sync()
            return ln, d_out.download(np.uint8, total).tobytes()
        finally:
            for b in bufs + [d_len, d_pos] + ([d_out] if d_out is not None else []):
                b.free()

    def plot_path_series(self, vals, off, sel, mult: float, chart, xf, n_charts: int, kind: int, fmt: int, cap: Optional[int] = None):
        """the device path text of selected value series on host arrays: (len [n] int64, text bytes)"""
        arrs = [_as(vals, np.float32), _as(off, np.int64), _as(sel, np.int64), _as(chart, np.int32), _as(xf, np.float64)]
        n = arrs[3].size

        def size(b, d_len, d_pos):
            self._ck(lib.gl_plot_path_series_size(self.h, b[0].ptr, b[1].ptr, b[2].ptr, mult, b[3].ptr, n, b[4].ptr, n_charts, kind, fmt,
                                                  d_len.ptr, d_pos.ptr))

        def emit(b, d_pos, total, d_out, room):
            self._ck(lib.gl_plot_path_series_emit(self.h, b[0].ptr, b[1].ptr, b[2].ptr, mult, b[3].ptr, n, b[4].ptr, n_charts, kind, fmt,
                                                  d_pos.ptr, total, d_out.ptr, room))
        return self._paths(size, emit, arrs, n, cap)

    def plot_path_xy(self, x, y, ptr, chart, xf, n_charts: int, kind: int, fmt: int, cap: Optional[int] = None):
        """the device path text of explicit vertices on host arrays: (len [n] int64, text bytes)"""
        arrs = [_as(x, np.float64), _as(y, np.float64), _as(ptr, np.int64), _as(chart, np.int32), _as(xf, np.float64)]
        n = arrs[3].size

        def size(b, d_len, d_pos):
            self._ck(lib.gl_plot_path_xy_size(self.h, b[0].ptr, b[1].ptr, b[2].ptr, b[3].ptr, n, b[4].ptr, n_charts, kind, fmt, d_len.ptr,
                                              d_pos.ptr))

        def emit(b, d_pos, total, d_out, room):
            self._ck(lib.gl_plot_path_xy_emit(self.h, b[0].ptr, b[1].ptr, b[2].ptr, b[3].ptr, n, b[4].ptr, n_charts, kind, fmt, d_pos.ptr,
                                              total, d_out.ptr, room))
        return self._paths(size, emit, arrs, n, cap)

    def plot_raster_xy(self, x, y, ptr, chart, draw, xf, n_charts: int, W: int, H: int, r: float) -> np.ndarray:
        x, y, ptr = _as(x, np.float64), _as(y, np.float64), _as(ptr, np.int64)
        chart, draw, xf = _as(chart, np.int32), _as(draw, np.uint32), _as(xf, np.float64)
        img = np.empty((n_charts, H, W), np.uint32)
        self._ck(lib.gl_plot_raster_xy(self.h, _ptr(x), _ptr(y), _ptr(ptr), _ptr(chart), _ptr(draw), chart.size, _ptr(xf), n_charts,
                                       W, H, r, _ptr(img)))
        return img

    def format_g3_device(self, d_vals: DevBuf, n: int, d_tokens: DevBuf):
        self._ck(lib.gl_format_g3_device(self.h, d_vals.ptr, n, d_tokens.ptr))

    def depthwed_aggregate_device(self, d_means: DevBuf, S: int, R: int, d_grp: Optional[DevBuf], n_out: int, d_out: DevBuf):
        self._ck(lib.gl_depthwed_aggregate_device(self.h, d_means.ptr, S, R, d_grp.ptr if d_grp is not None else None, n_out,
                                                  d_out.ptr))

    def format_g3(self, vals: np.ndarray) -> np.ndarray:
        """(n,10) uint8 tokens: text in [0:len), len in byte 9"""
        vals = _as(vals, np.float32)
        tok = np.empty((vals.size, 10), np.uint8)
        self._ck(lib.gl_format_g3(self.h, _ptr(vals), vals.size, _ptr(tok)))
        return tok

    # ---- covstats / depthwed
    def bincount(self, v: np.ndarray, lo: int, hi: int) -> np.ndarray:
        v = _as(v, np.int32)
        h = np.empty(hi - lo, np.uint64)
        self._ck(lib.gl_bincount_i32(self.h, _ptr(v), v.size, lo, hi, _ptr(h)))
        return h

    def depthwed_aggregate(self, means: np.ndarray, starts, ends, chrom_id, size: int):
        means = np.ascontiguousarray(means, np.float64)
        S, R = means.shape
        starts, ends, chrom_id = _as(starts, np.int32), _as(ends, np.int32), _as(chrom_id, np.int32)
        cap = max(R, 1)
        o_s, o_e, o_c = np.empty(cap, np.int32), np.empty(cap, np.int32), np.empty(cap, np.int32)
        out = np.empty((cap, S), np.int64)
        n = C.c_int64(0)
        self._ck(lib.gl_depthwed_aggregate(self.h, _ptr(means), S, R, _ptr(starts), _ptr(ends), _ptr(chrom_id), size,
                                           _ptr(o_s), _ptr(o_e), _ptr(o_c), _ptr(out), cap, C.byref(n)))
        k = n.value
        return o_s[:k], o_e[:k], o_c[:k], out[:k]

    def depthwed_aggregate_i32(self, depth: np.ndarray, starts, ends, chrom_id, size: int):
        """int32 form: depth = int(0.5 + mean) per (sample, row), as the reference rounds at parse time (depthwed.go:103)"""
        depth = np.ascontiguousarray(depth, np.int32)
        S, R = depth.shape
        starts, ends, chrom_id = _as(starts, np.int32), _as(ends, np.int32), _as(chrom_id, np.int32)
        cap = max(R, 1)
        o_s, o_e, o_c = np.empty(cap, np.int32), np.empty(cap, np.int32), np.empty(cap, np.int32)
        out = np.empty((cap, S), np.int32)
        n = C.c_int64(0)
        self._ck(lib.gl_depthwed_aggregate_i32(self.h, _ptr(depth), S, R, _ptr(starts), _ptr(ends), _ptr(chrom_id), size,
                                               _ptr(o_s), _ptr(o_e), _ptr(o_c), _ptr(out), cap, C.byref(n)))
        k = n.value
        return o_s[:k], o_e[:k], o_c[:k], out[:k]

    def depthwed_aggregate_i32_device(self, d_depth: DevBuf, S: int, R: int, d_grp: Optional[DevBuf], g_begin: int, g_end: int,
                                      d_out_ptr: int, d_overflow: DevBuf):
        self._ck(lib.gl_depthwed_aggregate_i32_device(self.h, d_depth.ptr, S, R, d_grp.ptr if d_grp is not None else None, g_begin, g_end,
                                                      d_out_ptr, d_overflow.ptr))

    def depthwed_cells(self, sums, lens, grp_of=None, n_groups: Optional[int] = None) -> np.ndarray:
        """int64 cells of explicit windows (sums[i] depth over lens[i] bases) as `goleft depth` then `depthwed` make them,
        summed per group grp_of[i] (None: one cell per window)"""
        sums, lens = _as(sums, np.int64), _as(lens, np.int64)
        assert sums.size == lens.size
        if grp_of is not None:
            grp_of = _as(grp_of, np.int32)
            assert grp_of.size == sums.size
            n_groups = int(grp_of.max()) + 1 if n_groups is None and grp_of.size else int(n_groups or 0)
        else:
            n_groups = sums.size
        out = np.empty(max(n_groups, 1), np.int64)
        self._ck(lib.gl_depthwed_cells(self.h, _ptr(sums), _ptr(lens), sums.size, _ptr(grp_of) if grp_of is not None else None, n_groups,
                                       _ptr(out)))
        return out[:n_groups]

    def depthwed_column_begin(self, d_col: DevBuf, n_groups: int):
        self._ck(lib.gl_depthwed_column_begin(self.h, d_col.ptr, n_groups))

    def depthwed_add_column(self, w0: int, d_grp_of: DevBuf, d_col: DevBuf):
        """asynchronous: the last gl_depth_reduce's window cells added into d_col[d_grp_of[w0 + k]]"""
        self._ck(lib.gl_depthwed_add_column(self.h, w0, d_grp_of.ptr, d_col.ptr))

    def depthwed_column_i32(self, d_col: DevBuf, n_groups: int, d_col32: DevBuf, d_overflow: DevBuf):
        self._ck(lib.gl_depthwed_column_i32(self.h, d_col.ptr, n_groups, d_col32.ptr, d_overflow.ptr))

    def ipc_export(self, buf: DevBuf) -> bytes:
        h = (C.c_uint8 * 64)()
        self._ck(lib.gl_ipc_export(self.h, buf.ptr, C.cast(h, _vp)))
        return bytes(h)

    def ipc_open(self, handle: bytes) -> int:
        h = (C.c_uint8 * 64).from_buffer_copy(handle)
        p = _vp()
        self._ck(lib.gl_ipc_open(self.h, C.cast(h, _vp), C.byref(p)))
        return p.value

    def ipc_close(self, ptr: int):
        self._ck(lib.gl_ipc_close(self.h, ptr))

    def depthwed_aggregate_i32_p2p(self, d_depth: DevBuf, S: int, R: int, d_grp: Optional[DevBuf], g_begin: int, g_end: int, dst_ptrs,
                                   row_stride: int, col_off: int, d_overflow: DevBuf):
        arr = (_vp * len(dst_ptrs))(*dst_ptrs)
        self._ck(lib.gl_depthwed_aggregate_i32_p2p(self.h, d_depth.ptr, S, R, d_grp.ptr if d_grp is not None else None, g_begin, g_end,
                                                   C.cast(arr, _vp), len(dst_ptrs), row_stride, col_off, d_overflow.ptr))

    def allgather_device_async(self, send_ptr: int, recv_ptr: int, nbytes: int):
        self._ck(lib.gl_allgather_device_async(self.h, send_ptr, recv_ptr, nbytes))

    def comm_wait(self):
        self._ck(lib.gl_comm_wait(self.h))

    # ---- multidepth
    def multidepth_begin(self, contig_len: int, n_samples: int, mincov: int = 7, min_samples: float = 0.5):
        self._ck(lib.gl_multidepth_begin(self.h, contig_len, n_samples, mincov, float(min_samples)))

    def multidepth_count(self):
        self._ck(lib.gl_multidepth_count(self.h))

    def multidepth_merge(self, sources):
        """Add the pass-1 counters, site bits and counted samples of every context in `sources` (None stands for a null
        handle) into this one's."""
        arr = (_vp * max(len(sources), 1))(*[None if s is None else s.h for s in sources])
        self._ck(lib.gl_multidepth_merge(self.h, arr, len(sources)))

    def multidepth_adopt_sites(self, src):
        """Copy src's site and sufficient bits and its class runs into this context."""
        self._ck(lib.gl_multidepth_adopt_sites(self.h, None if src is None else src.h))

    def multidepth_sites(self):
        n = C.c_int64(0)
        self._ck(lib.gl_multidepth_sites(self.h, None, None, 0, C.byref(n)))
        s, c = np.empty(n.value, np.int32), np.empty(n.value, np.uint8)
        self._ck(lib.gl_multidepth_sites(self.h, _ptr(s), _ptr(c), n.value, C.byref(n)))
        return s, c

    def multidepth_set_blocks(self, blk_start, blk_end, blk_sites):
        blk_start, blk_end, blk_sites = _as(blk_start, np.int64), _as(blk_end, np.int64), _as(blk_sites, np.int64)
        self._ck(lib.gl_multidepth_set_blocks(self.h, _ptr(blk_start), _ptr(blk_end), _ptr(blk_sites), blk_start.size))

    def multidepth_sums(self, sample: int):
        self._ck(lib.gl_multidepth_sums(self.h, sample))

    def multidepth_result(self, n_blocks: int, S: int):
        """(sums, q, val, certified), each n_blocks x S"""
        sums, q = np.empty((n_blocks, S), np.uint64), np.empty((n_blocks, S), np.int64)
        val, ok = np.empty((n_blocks, S), np.float64), np.empty((n_blocks, S), np.uint8)
        self._ck(lib.gl_multidepth_result(self.h, _ptr(sums), _ptr(q), _ptr(val), _ptr(ok)))
        return sums, q, val, ok.astype(bool)

    def multidepth_stats(self):
        """{blocks, walked, certified, min_samples}"""
        v = [C.c_int64(0) for _ in range(4)]
        self._ck(lib.gl_multidepth_stats(self.h, *[C.byref(x) for x in v]))
        return dict(zip(("blocks", "walked", "certified", "min_samples"), (x.value for x in v)))

    def multidepth(self, chrom: str, contig_len: int, adders, mincov: int = 7, min_samples: float = 0.5, max_skip: int = 10,
                   min_size: int = 15, window: int = 10_000_000, chunk: int = 0) -> bytes:
        """The whole tool for one contig: adders[i](ctx) adds sample i's segments to the open region (it is called twice, once
        per pass).  Returns the rows after the header line."""
        S = len(adders)
        self.multidepth_begin(contig_len, S, mincov, min_samples)
        for add in adders:
            self.depth_begin(0, contig_len)
            add(self)
            self.multidepth_count()
        rs, rc = self.multidepth_sites()
        bs, be, bn = multidepth_blocks(rs, rc, contig_len, S, max_skip, min_size, window, chunk)
        self.multidepth_set_blocks(bs, be, bn)
        for i, add in enumerate(adders):
            self.depth_begin(0, contig_len)
            add(self)
            self.multidepth_sums(i)
        _, q, val, ok = self.multidepth_result(bs.size, S)
        return multidepth_text(chrom, bs, be, S, q, val, ok)

    @staticmethod
    def multidepth_sharded(ctxs, chrom: str, contig_len: int, adders, mincov: int = 7, min_samples: float = 0.5,
                           max_skip: int = 10, min_size: int = 15, window: int = 10_000_000, chunk: int = 0, parts: bool = False):
        """The whole tool for one contig with the cohort split over several contexts: adders[k] are context k's samples
        (adders[k][j](ctx) adds one sample's segments to the open region, once per pass), numbered in context order.  Each
        context runs its passes on a thread of its own; ctxs[0] merges the others' counts and finds the sites, the host makes
        the blocks once, every other context adopts ctxs[0]'s sites, and each sample's columns come from its own context.
        Returns the rows after the header line, or (rows, parts) with parts=True: the runs, blocks, sums / q / val /
        certified (n_blocks x S), the phase times in ms (pass 2 includes each context's gl_multidepth_result; gather is
        the host's column copy) and the bytes the merge moved."""
        if len(ctxs) < 1 or len(ctxs) != len(adders):
            raise ValueError("multidepth_sharded: one list of adders per context")
        n = [len(a) for a in adders]
        S = sum(n)
        first = [sum(n[:k]) for k in range(len(n))]
        t = [time.perf_counter()]

        def each(pool, fn):
            if len(ctxs) == 1:                                  # one context: on the calling thread, as Ctx.multidepth
                fn(0)
            else:
                for f in [pool.submit(fn, k) for k in range(len(ctxs))]:
                    f.result()
            t.append(time.perf_counter())

        def pass1(k):
            c = ctxs[k]
            c.multidepth_begin(contig_len, S, mincov, min_samples)
            for add in adders[k]:
                c.depth_begin(0, contig_len)
                add(c)
                c.multidepth_count()

        def pass2(k):
            c = ctxs[k]
            if k:
                c.multidepth_adopt_sites(ctxs[0])
            c.multidepth_set_blocks(bs, be, bn)
            for j, add in enumerate(adders[k]):
                c.depth_begin(0, contig_len)
                add(c)
                c.multidepth_sums(first[k] + j)
            res[k] = c.multidepth_result(bs.size, S)

        res = [None] * len(ctxs)
        with ThreadPoolExecutor(len(ctxs)) as pool:
            each(pool, pass1)
            if len(ctxs) > 1:
                ctxs[0].multidepth_merge(ctxs[1:])
            t.append(time.perf_counter())
            rs, rc = ctxs[0].multidepth_sites()
            t.append(time.perf_counter())
            bs, be, bn = multidepth_blocks(rs, rc, contig_len, S, max_skip, min_size, window, chunk)
            t.append(time.perf_counter())
            each(pool, pass2)
        sums, q, val, ok = res[0]                           # each sample's columns from the context that summed it
        for k in range(1, len(ctxs)):
            cols = slice(first[k], first[k] + n[k])
            for dst, src in zip((sums, q, val, ok), res[k]):
                dst[:, cols] = src[:, cols]
        t.append(time.perf_counter())
        rows = multidepth_text(chrom, bs, be, S, q, val, ok)
        if not parts:
            return rows
        words = (contig_len + 4095) // 4096 * 128
        ms = {k: (t[i + 1] - t[i]) * 1e3 for i, k in enumerate(("pass1", "merge", "sites", "blocks_host", "pass2"))}
        ms["gather"] = (t[6] - t[5]) * 1e3
        return rows, dict(runs=(rs, rc), blocks=(bs, be, bn), sums=sums, q=q, val=val, certified=ok, ms=ms,
                          merge_bytes=(len(ctxs) - 1) * words * 68)

    # ---- dcnv
    def dcnv_normalize(self, x: np.ndarray, inds, c0: int = 0, c1: Optional[int] = None, block_cols: int = 0):
        """Columns [c0, c1) of the n x S matrix x (rows in position order), inds = the GC argsort -> (normalised n x (c1 - c0),
        sample medians)"""
        x = np.ascontiguousarray(x, np.float64)
        n, S = x.shape
        c1 = S if c1 is None else c1
        inds = _as(inds, np.int64)
        out, med = np.empty((n, c1 - c0), np.float64), np.empty(c1 - c0, np.float64)
        self._ck(lib.gl_dcnv_normalize(self.h, _ptr(x), n, S, _ptr(inds), c0, c1, block_cols, _ptr(out), c1 - c0, _ptr(med)))
        return out, med

    def dcnv_normalize_device(self, d_x: DevBuf, n: int, ld: int, d_inds: DevBuf, c0: int, c1: int, d_out: DevBuf, ld_out: int,
                              d_medians: DevBuf):
        self._ck(lib.gl_dcnv_normalize_device(self.h, d_x.ptr, n, ld, d_inds.ptr, c0, c1, d_out.ptr, ld_out, d_medians.ptr))

    def dcnv_normalize_chunked(self, x: np.ndarray, inds, chunk_ptr, c0: int = 0, c1: Optional[int] = None, block_cols: int = 0):
        """dcnv_normalize with ChunkDebiaser's chunks (chunk_ptr, from dcnv_chunk_slices) in place of the moving median"""
        x = np.ascontiguousarray(x, np.float64)
        n, S = x.shape
        c1 = S if c1 is None else c1
        inds, chunk_ptr = _as(inds, np.int64), _as(chunk_ptr, np.int64)
        out, med = np.empty((n, c1 - c0), np.float64), np.empty(c1 - c0, np.float64)
        self._ck(lib.gl_dcnv_normalize_chunked(self.h, _ptr(x), n, S, _ptr(inds), _ptr(chunk_ptr), chunk_ptr.size - 1, c0, c1, block_cols,
                                               _ptr(out), c1 - c0, _ptr(med)))
        return out, med

    def dcnv_normalize_chunked_device(self, d_x: DevBuf, n: int, ld: int, d_inds: DevBuf, chunk_ptr, c0: int, c1: int, d_out: DevBuf,
                                      ld_out: int, d_medians: DevBuf):
        """chunk_ptr is a host array"""
        chunk_ptr = _as(chunk_ptr, np.int64)
        self._ck(lib.gl_dcnv_normalize_chunked_device(self.h, d_x.ptr, n, ld, d_inds.ptr, _ptr(chunk_ptr), chunk_ptr.size - 1, c0, c1,
                                                      d_out.ptr, ld_out, d_medians.ptr))

    def format_f2(self, vals: np.ndarray) -> np.ndarray:
        vals = _as(vals, np.float64)
        tok = np.empty((vals.size, F2_TOKEN), np.uint8)
        self._ck(lib.gl_format_f2(self.h, _ptr(vals), vals.size, _ptr(tok)))
        return tok

    def format_f2_device(self, d_vals: DevBuf, n: int, d_tokens: DevBuf):
        self._ck(lib.gl_format_f2_device(self.h, d_vals.ptr, n, d_tokens.ptr))

    def dcnv_svd(self, x: np.ndarray, min_pct: float, block_rows: int = 0, want_gram: bool = False):
        """dcnv --svd on a copy of the n x S float64 matrix x -> (result, singular values[S], n_removed, n_kept,
        Z^T Z (S x S) or None)"""
        out = np.array(x, np.float64, order="C", copy=True)
        n, S = out.shape
        sv, nr, nk = np.empty(S, np.float64), C.c_int32(0), C.c_int64(0)
        gram = np.empty((S, S), np.float64) if want_gram else None
        self._ck(lib.gl_dcnv_svd(self.h, _ptr(out), n, S, S, float(min_pct), block_rows, _ptr(sv), _ptr(gram), C.byref(nr),
                                 C.byref(nk)))
        return out, sv, nr.value, nk.value, gram

    def dcnv_svd_device(self, d_x: DevBuf, n: int, ld: int, S: int, min_pct: float, want_gram: bool = False):
        """dcnv --svd in place on the device matrix d_x -> (singular values[S], n_removed, n_kept, Z^T Z or None)"""
        sv, nr, nk = np.empty(S, np.float64), C.c_int32(0), C.c_int64(0)
        gram = np.empty((S, S), np.float64) if want_gram else None
        self._ck(lib.gl_dcnv_svd_device(self.h, d_x.ptr, n, ld, S, float(min_pct), _ptr(sv), _ptr(gram), C.byref(nr), C.byref(nk)))
        return sv, nr.value, nk.value, gram

    def dcnv_svd_phases(self):
        """seconds of the last dcnv_svd call: {gram, eigen, project, copies}"""
        t = (C.c_double * 4)()
        self._ck(lib.gl_dcnv_svd_phases(self.h, t))
        return dict(zip(("gram", "eigen", "project", "copies"), list(t)))

    def dcnv_chart(self, x: np.ndarray, block_rows: int = 0, W: int = PLOT_W, H: int = PLOT_H, r: Optional[float] = None):
        """dcnv's chart of the n x S float64 matrix x on the GPU: (first[S], yext (S,2), ext4, the (H, W) index image)"""
        x = np.ascontiguousarray(x, np.float64)
        n, S = x.shape
        first, yext, ext = np.empty(S, np.int64), np.empty((S, 2), np.float64), np.empty(4, np.float64)
        img = np.empty((H, W), np.uint32)
        self._ck(lib.gl_dcnv_chart(self.h, _ptr(x), n, S, block_rows, W, H, plot_line_radius(S) if r is None else r, _ptr(first),
                                   _ptr(yext), _ptr(ext), _ptr(img)))
        return first, yext, ext, img

    # ---- emdepth
    def emdepth(self, x: np.ndarray, block_rows: int = 0, ld: Optional[int] = None, S: Optional[int] = None, want_lambda: bool = True):
        """cells (n x S uint8) and the final centres (n x 9, or None) of the float32 rows of x (columns [0, S) of each row)"""
        x = np.ascontiguousarray(x, np.float32)
        n, ld = x.shape[0], x.shape[1] if ld is None else ld
        S = x.shape[1] if S is None else S
        cells = np.empty((n, S), np.uint8)
        lam = np.empty((n, 9), np.float64) if want_lambda else None
        self._ck(lib.gl_emdepth(self.h, _ptr(x), n, ld, S, block_rows, _ptr(cells), _ptr(lam)))
        return cells, lam

    def emdepth_device(self, d_x: DevBuf, n: int, ld: int, S: int, d_cells: DevBuf, d_lambda: Optional[DevBuf] = None):
        self._ck(lib.gl_emdepth_device(self.h, d_x.ptr, n, ld, S, d_cells.ptr, d_lambda.ptr if d_lambda else None))

    def emdepth_stats(self):
        """{rows, uncertified, sequential} of the last emdepth call"""
        v = [C.c_int64(0) for _ in range(3)]
        self._ck(lib.gl_emdepth_stats(self.h, *[C.byref(x) for x in v]))
        return dict(zip(("rows", "uncertified", "sequential"), (x.value for x in v)))

    # ---- cnveval
    def cnveval(self, S: int, c_sample, c_chrom, c_start, c_end, c_cn, t_chrom, t_start, t_end, t_cn, t_mem_ptr, t_mem_sample,
                po: float = 0.4) -> np.ndarray:
        """(S, 3, 4) uint64 TP, FP, FN, TN per sample and size class.  Calls in file order; truth t carries the samples
        t_mem_sample[t_mem_ptr[t]:t_mem_ptr[t + 1]]; chrom ranks follow the names' bytewise order."""
        c = [_as(c_sample, np.int32), _as(c_chrom, np.int32), _as(c_start, np.int64), _as(c_end, np.int64), _as(c_cn, np.int64)]
        t = [_as(t_chrom, np.int32), _as(t_start, np.int64), _as(t_end, np.int64), _as(t_cn, np.int64)]
        mp, ms = _as(t_mem_ptr, np.int64), _as(t_mem_sample, np.int32)
        if any(a.size != c[0].size for a in c) or any(a.size != t[0].size for a in t) or mp.size != t[0].size + 1 or ms.size != mp[-1]:
            raise ValueError("cnveval: array lengths disagree")
        out = np.empty((S, 3, 4), np.uint64)
        self._ck(lib.gl_cnveval(self.h, S, *[_ptr(a) for a in c], c[0].size, *[_ptr(a) for a in t], t[0].size, _ptr(mp), _ptr(ms),
                                float(po), _ptr(out)))
        return out

    def cnveval_device(self, S: int, d_c_ptr: DevBuf, n_calls: int, d_c_chrom: DevBuf, d_c_start: DevBuf, d_c_end: DevBuf,
                       d_c_cn: DevBuf, n_truths: int, d_t_chrom: DevBuf, d_t_start: DevBuf, d_t_end: DevBuf, d_t_cn: DevBuf,
                       d_m_ptr: DevBuf, n_mem: int, d_m_truth: DevBuf, po: float, d_stats: DevBuf):
        """the resident layout of include/goleft_b200.h (gl_cnveval_device); d_stats: S x 12 uint64"""
        self._ck(lib.gl_cnveval_device(self.h, S, d_c_ptr.ptr, n_calls, d_c_chrom.ptr, d_c_start.ptr, d_c_end.ptr, d_c_cn.ptr, n_truths,
                                       d_t_chrom.ptr, d_t_start.ptr, d_t_end.ptr, d_t_cn.ptr, d_m_ptr.ptr, n_mem, d_m_truth.ptr,
                                       float(po), d_stats.ptr))

    # ---- indexcov PCA
    def indexcov_pca(self, x: np.ndarray, k: int = 5, D: Optional[int] = None, want_gram: bool = False):
        """(proj S x k, sv[k], k_out, gram S x S or None) of the uint8 rows of x (columns [0, D) of each row)"""
        x = np.ascontiguousarray(x, np.uint8)
        S, ld = x.shape
        D = ld if D is None else D
        proj, sv, ko = np.empty((S, k), np.float64), np.empty(k, np.float64), C.c_int32(0)
        gram = np.empty((S, S), np.int64) if want_gram else None
        self._ck(lib.gl_indexcov_pca(self.h, _ptr(x), ld, S, D, k, _ptr(proj), _ptr(sv), C.byref(ko), _ptr(gram)))
        return proj, sv, ko.value, gram

    def indexcov_pca_device(self, d_x: DevBuf, ld: int, S: int, D: int, k: int = 5, want_gram: bool = False):
        proj, sv, ko = np.empty((S, k), np.float64), np.empty(k, np.float64), C.c_int32(0)
        gram = np.empty((S, S), np.int64) if want_gram else None
        self._ck(lib.gl_indexcov_pca_device(self.h, d_x.ptr, ld, S, D, k, _ptr(proj), _ptr(sv), C.byref(ko), _ptr(gram)))
        return proj, sv, ko.value, gram

    def indexcov_pca_phases(self):
        """seconds of the last indexcov_pca call: {upload, gram, eigen}"""
        t = (C.c_double * 3)()
        self._ck(lib.gl_indexcov_pca_phases(self.h, t))
        return dict(zip(("upload", "gram", "eigen"), list(t)))

    def sym_tridiag(self, a: np.ndarray, u: Optional[np.ndarray] = None):
        """(d[n], e[n-1], tau[n-2], reflectors n x n, Q u or None) of the symmetric n x n float64 matrix a: the device
        tridiagonalisation indexcov's PCA and dcnv --svd share (gl_sym_tridiag); u: k x n vectors of T"""
        a = _as(a, np.float64)
        if a.ndim != 2 or a.shape[0] != a.shape[1]:
            raise ValueError("sym_tridiag: a must be square")
        n = a.shape[0]
        d, e, tau = np.empty(n, np.float64), np.empty(max(n - 1, 0), np.float64), np.empty(max(n - 2, 0), np.float64)
        refl = np.empty((n, n), np.float64)
        if u is not None:
            u = np.array(u, np.float64, order="C", copy=True)
            if u.ndim != 2 or u.shape[1] != n:
                raise ValueError("sym_tridiag: u must be k x n")
        k = 0 if u is None else u.shape[0]
        self._ck(lib.gl_sym_tridiag(self.h, _ptr(a), n, _ptr(d), _ptr(e), _ptr(tau), _ptr(refl), k, _ptr(u)))
        return d, e, tau, refl, u

    # ---- multi-GPU
    def comm_init(self, id128: bytes, rank: int, world: int):
        buf = (C.c_uint8 * 128).from_buffer_copy(id128)
        self._ck(lib.gl_comm_init(self.h, C.cast(buf, _vp), rank, world))

    def allgather_device(self, d_send: DevBuf, d_recv: DevBuf, nbytes: int):
        self._ck(lib.gl_allgather_device(self.h, d_send.ptr, d_recv.ptr, nbytes))


def comm_unique_id() -> bytes:
    buf = (C.c_uint8 * 128)()
    rc = lib.gl_comm_unique_id(C.cast(buf, _vp))
    if rc != GL_OK:
        raise GlError(rc, lib.gl_last_error(None).decode())
    return bytes(buf)
