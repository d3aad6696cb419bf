"""ctypes loader for libloghisto_b200.so (the C ABI in include/loghisto_b200.h).

There is no CPU fallback: if the shared library is missing it is built with
nvcc; if that is impossible, or no CUDA device is present when a context is
created, the error is raised to the caller.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

LIB_PATH = _build.LIB

LH_OK = 0
LH_ERR_INVALID = -1
LH_ERR_CUDA = -2
LH_ERR_NOMEM = -3
LH_ERR_NO_DEVICE = -4
LH_ERR_STATE = -5
LH_ERR_RANGE = -6
LH_MAX_PERCENTILES = 32


class lh_config(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("device", C.c_int32),
        ("max_histograms", C.c_uint32), ("max_counters", C.c_uint32),
        ("staging_bytes", C.c_uint64), ("staging_slots", C.c_uint32), ("flags", C.c_uint32),
        ("precision", C.c_uint32), ("reserved", C.c_uint32 * 3),
    ]


class lh_staging(C.Structure):
    _fields_ = [("host", C.c_void_p), ("bytes", C.c_uint64), ("slot", C.c_uint32), ("reserved", C.c_uint32)]


class lh_device_view(C.Structure):
    _fields_ = [
        ("d_buckets", C.c_void_p), ("d_counters", C.c_void_p),
        ("n_bucket_words", C.c_uint64), ("n_counter_words", C.c_uint64), ("stream", C.c_void_p),
        ("d_flags", C.c_void_p), ("n_flag_words", C.c_uint64),
    ]


LH_PEER_HANDLE_BYTES = 1024
LH_MAX_RANKS = 16
LH_ROW_ABSENT = 0xFFFFFFFF   # map entry of lh_snapshot_allreduce_rows: this rank has nothing under that row


class lh_comm_stats(C.Structure):
    _fields_ = [
        ("rank", C.c_uint32), ("world", C.c_uint32), ("status", C.c_uint32), ("reserved", C.c_uint32),
        ("allreduces", C.c_uint64), ("last_bytes_from_peers", C.c_uint64),
    ]


class lh_sparse(C.Structure):
    _fields_ = [
        ("offsets", C.POINTER(C.c_uint32)), ("keys", C.POINTER(C.c_int16)),
        ("counts", C.POINTER(C.c_uint64)), ("counter_deltas", C.POINTER(C.c_uint64)),
        ("total_entries", C.c_uint64),
    ]


class lh_stats(C.Structure):
    _fields_ = [
        ("samples", C.c_uint64), ("counter_ops", C.c_uint64), ("dropped", C.c_uint64),
        ("kernel_launches", C.c_uint64), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
        ("snapshots", C.c_uint64),
    ]


class lh_recorder(C.Structure):
    """What device code records through (include/loghisto_b200_device.cuh); passed by value to the caller's kernels."""
    _fields_ = [
        ("d_buckets", C.c_void_p), ("d_flags", C.c_void_p), ("d_counters", C.c_void_p), ("d_dropped", C.c_void_p),
        ("max_histograms", C.c_uint32), ("max_counters", C.c_uint32), ("block_smem_bytes", C.c_uint32),
        ("reserved", C.c_uint32), ("scope", C.c_uint64), ("prec", C.c_uint8 * 48),
    ]


LH_VALUES_F64 = 0      # lh_batch_item.kind: float64 values
LH_VALUES_I64NS = 1    # int64 nanoseconds, recorded as float64(ns)


class lh_batch_item(C.Structure):
    """One (histogram id, device array) item of lh_ingest_batch."""
    _fields_ = [("d_values", C.c_void_p), ("n", C.c_uint64), ("histogram_id", C.c_uint32), ("kind", C.c_uint32)]


class lh_gpu_timer(C.Structure):
    """Opaque handle of a GPU timer (lh_gpu_timer_start)."""
    _fields_ = [("handle", C.c_uint64)]


class lh_certify_form(C.Structure):
    """One (precision, form) row of lh_fastpath_certify."""
    _fields_ = [("samples", C.c_uint64), ("flagged", C.c_uint64), ("wrong", C.c_uint64), ("out_of_range", C.c_uint64),
                ("unflagged_outside", C.c_uint64), ("over_flagged", C.c_uint64), ("input_mismatch", C.c_uint64),
                ("max_err", C.c_double), ("min_margin", C.c_double)]


LH_GRAPH_UNBOUND = 0xFFFFFFFF   # target id of a graph recorder row whose drained counts are dropped and counted


class lh_graph_recorder(C.Structure):
    """A graph recorder (lh_graph_recorder_create): `rec` is passed by value to kernels captured into CUDA graphs."""
    _fields_ = [("handle", C.c_uint64), ("rec", lh_recorder)]


class lh_board_header(C.Structure):
    """Header of a device subscription board (include/loghisto_b200.h)."""
    _fields_ = [("seq", C.c_uint64), ("publishes", C.c_uint64), ("np", C.c_uint32), ("reserved", C.c_uint32 * 3),
                ("percentiles", C.c_double * LH_MAX_PERCENTILES)]


class lh_board_hist_row(C.Structure):
    _fields_ = [("count", C.c_uint64), ("sum", C.c_double), ("avg", C.c_double), ("present", C.c_uint32),
                ("reserved", C.c_uint32), ("pvals", C.c_double * LH_MAX_PERCENTILES),
                ("pkeys", C.c_int32 * LH_MAX_PERCENTILES)]


class lh_board_counter_row(C.Structure):
    _fields_ = [("rate", C.c_uint64), ("total", C.c_uint64), ("present", C.c_uint32), ("reserved", C.c_uint32)]


class lh_board(C.Structure):
    """A device subscription board (lh_board_create): passed by value to the caller's kernels, which read it with
    lh::read_histogram / lh::read_counter."""
    _fields_ = [("handle", C.c_uint64), ("d_board", C.c_void_p), ("k", C.c_uint32), ("kc", C.c_uint32),
                ("bytes", C.c_uint64)]


class lh_raw_row_header(C.Structure):
    """Header of one row of a raw device subscription board (include/loghisto_b200.h)."""
    _fields_ = [("seq", C.c_uint64), ("publishes", C.c_uint64), ("total", C.c_uint64), ("key_lo", C.c_int32),
                ("key_hi", C.c_int32)]


class lh_raw_board(C.Structure):
    """A raw device subscription board (lh_raw_board_create): passed by value to the caller's kernels, which query it
    with lh::raw_percentile / lh::raw_rank / lh::raw_bucket_count."""
    _fields_ = [("handle", C.c_uint64), ("d_rows", C.c_void_p), ("d_decomp", C.c_void_p), ("k", C.c_uint32),
                ("reserved", C.c_uint32), ("prec", C.c_uint8 * 48)]


def LH_RAW_CELLS_OFFSET(k: int) -> int:
    """Byte offset of row 0's running counts from lh_raw_board.d_rows."""
    return (k * 32 + 255) & ~255


LH_RAW_MAX_WINDOW = 4096   # publishes a window board may sum per row (lh_raw_board_create_window)

LH_GAUGE_F64, LH_GAUGE_F32, LH_GAUGE_F16, LH_GAUGE_BF16, LH_GAUGE_I64, LH_GAUGE_I32, LH_GAUGE_U64 = range(7)


class lh_gauge_src(C.Structure):
    """One device gauge of lh_gauges_read: a scalar of dtype LH_GAUGE_* at d_value (include/loghisto_b200.h)."""
    _fields_ = [("d_value", C.c_void_p), ("dtype", C.c_uint32), ("reserved", C.c_uint32)]


class lh_array_src(C.Structure):
    """One array of lh_snapshot_ingest_arrays: n elements of dtype LH_GAUGE_* at d_values, recorded under
    histogram_id (include/loghisto_b200.h)."""
    _fields_ = [("d_values", C.c_void_p), ("n", C.c_uint64), ("dtype", C.c_uint32), ("histogram_id", C.c_uint32)]


_vp, _sz, _u32, _u64, _i32 = C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint64, C.c_int32

# name -> (restype, argtypes); every symbol include/loghisto_b200.h declares
SIGNATURES = {
    "lh_create": (_i32, [C.POINTER(lh_config), C.POINTER(_vp)]),
    "lh_destroy": (_i32, [_vp]),
    "lh_strerror": (C.c_char_p, [_i32]),
    "lh_last_error": (C.c_char_p, [_vp]),
    "lh_abi_version": (_u32, []),
    "lh_ingest_f64": (_i32, [_vp, _u32, _vp, _sz, _vp]),
    "lh_ingest_keyed_f64_u16": (_i32, [_vp, _vp, _vp, _sz, _vp]),
    "lh_ingest_keyed_f64_u32": (_i32, [_vp, _vp, _vp, _sz, _vp]),
    "lh_ingest_keyed_i64ns_u16": (_i32, [_vp, _vp, _vp, _sz, _vp]),
    "lh_ingest_keyed_pair_u16": (_i32, [_vp, _vp, _vp, _sz, _vp, _vp, _sz, _vp]),
    "lh_ingest_batch": (_i32, [_vp, C.POINTER(lh_batch_item), _u32, _vp]),
    "lh_counter_add_u16": (_i32, [_vp, _vp, _vp, _sz, _vp]),
    "lh_counter_add_u32": (_i32, [_vp, _vp, _vp, _sz, _vp]),
    "lh_ingest_keyed_mapped_u16": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32, _sz, _vp]),
    "lh_ingest_keyed_mapped_u32": (_i32, [_vp, _vp, _u32, _vp, _vp, _u32, _sz, _vp]),
    "lh_counter_add_mapped_u16": (_i32, [_vp, _vp, _u32, _vp, _vp, _sz, _vp]),
    "lh_counter_add_mapped_u32": (_i32, [_vp, _vp, _u32, _vp, _vp, _sz, _vp]),
    "lh_ingest_f64_host": (_i32, [_vp, _u32, _vp, _sz]),
    "lh_ingest_keyed_f64_u16_host": (_i32, [_vp, _vp, _vp, _sz]),
    "lh_ingest_keyed_i64ns_u16_host": (_i32, [_vp, _vp, _vp, _sz]),
    "lh_counter_add_u16_host": (_i32, [_vp, _vp, _vp, _sz]),
    "lh_merge_counts_host": (_i32, [_vp, _vp, _vp, _vp, _sz]),
    "lh_staging_acquire": (_i32, [_vp, C.POINTER(lh_staging)]),
    "lh_staging_commit_f64": (_i32, [_vp, C.POINTER(lh_staging), _u32, _sz]),
    "lh_staging_commit_keyed_f64_u16": (_i32, [_vp, C.POINTER(lh_staging), _sz, _u64]),
    "lh_staging_commit_counter_u16": (_i32, [_vp, C.POINTER(lh_staging), _sz, _u64]),
    "lh_staging_abandon": (_i32, [_vp, C.POINTER(lh_staging)]),
    "lh_record_begin": (_i32, [_vp, _vp, C.POINTER(lh_recorder)]),
    "lh_record_end": (_i32, [_vp, C.POINTER(lh_recorder)]),
    "lh_graph_recorder_create": (_i32, [_vp, _u32, _u32, _vp, _vp, C.POINTER(lh_graph_recorder)]),
    "lh_graph_recorder_bind": (_i32, [_vp, C.POINTER(lh_graph_recorder), _vp, _vp]),
    "lh_graph_recorder_ingest": (_i32, [_vp, C.POINTER(lh_graph_recorder), C.POINTER(lh_batch_item), _u32, _vp]),
    "lh_graph_recorder_ingest_keyed_u16": (_i32, [_vp, C.POINTER(lh_graph_recorder), _vp, _vp, _u32, _sz, _vp]),
    "lh_graph_recorder_ingest_keyed_u32": (_i32, [_vp, C.POINTER(lh_graph_recorder), _vp, _vp, _u32, _sz, _vp]),
    "lh_graph_recorder_counter_add_u16": (_i32, [_vp, C.POINTER(lh_graph_recorder), _vp, _vp, _sz, _vp]),
    "lh_graph_recorder_counter_add_u32": (_i32, [_vp, C.POINTER(lh_graph_recorder), _vp, _vp, _sz, _vp]),
    "lh_graph_recorder_timer_start": (_i32, [_vp, C.POINTER(lh_graph_recorder), _u32, _vp]),
    "lh_graph_recorder_timer_stop": (_i32, [_vp, C.POINTER(lh_graph_recorder), _u32, _vp, _vp]),
    "lh_graph_recorder_destroy": (_i32, [_vp, C.POINTER(lh_graph_recorder), _vp]),
    "lh_board_create": (_i32, [_vp, _u32, _u32, C.POINTER(lh_board)]),
    "lh_snapshot_publish": (_i32, [_vp, C.POINTER(lh_board), _vp, _vp, _vp]),
    "lh_board_read": (_i32, [_vp, C.POINTER(lh_board), _vp, _vp]),
    "lh_board_destroy": (_i32, [_vp, C.POINTER(lh_board)]),
    "lh_raw_board_create": (_i32, [_vp, _u32, C.POINTER(lh_raw_board)]),
    "lh_raw_board_create_window": (_i32, [_vp, _u32, _u32, C.POINTER(lh_raw_board)]),
    "lh_snapshot_publish_raw": (_i32, [_vp, C.POINTER(lh_raw_board), _vp]),
    "lh_raw_percentiles": (_i32, [_vp, C.POINTER(lh_raw_board), _vp, _vp, _u32, _vp, _vp, _vp, _vp]),
    "lh_raw_ranks": (_i32, [_vp, C.POINTER(lh_raw_board), _vp, _vp, _u32, _vp, _vp, _vp, _vp]),
    "lh_raw_percentiles_grid": (_i32, [_vp, C.POINTER(lh_raw_board), _vp, _u32, _vp, _vp, _vp, _vp]),
    "lh_raw_ranks_grid": (_i32, [_vp, C.POINTER(lh_raw_board), _vp, _u32, _vp, _vp, _vp, _vp]),
    "lh_raw_board_destroy": (_i32, [_vp, C.POINTER(lh_raw_board)]),
    "lh_gauges_read": (_i32, [_vp, C.POINTER(lh_gauge_src), _u32, _vp]),
    "lh_snapshot_ingest_arrays": (_i32, [_vp, C.POINTER(lh_array_src), _u32]),
    "lh_ingest_arrays": (_i32, [_vp, C.POINTER(lh_array_src), _u32, _vp]),
    "lh_graph_recorder_ingest_arrays": (_i32, [_vp, C.POINTER(lh_graph_recorder), C.POINTER(lh_array_src), _u32, _vp]),
    "lh_gpu_timer_start": (_i32, [_vp, _vp, C.POINTER(lh_gpu_timer)]),
    "lh_gpu_timer_stop": (_i32, [_vp, C.POINTER(lh_gpu_timer), _u32, _vp, _vp]),
    "lh_gpu_timer_release": (_i32, [_vp, C.POINTER(lh_gpu_timer)]),
    "lh_snapshot_begin": (_i32, [_vp]),
    "lh_snapshot_device": (_i32, [_vp, C.POINTER(lh_device_view)]),
    "lh_snapshot_reduce": (_i32, [_vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp]),
    "lh_snapshot_reduce_async": (_i32, [_vp, _vp, _u32, C.POINTER(_u64)]),
    "lh_snapshot_result": (_i32, [_vp, _u64, _vp, _vp, _vp, _vp, _vp]),
    "lh_snapshot_export": (_i32, [_vp, C.POINTER(lh_sparse)]),
    "lh_snapshot_copy_histogram": (_i32, [_vp, _u32, _vp]),
    "lh_snapshot_end": (_i32, [_vp]),
    "lh_reduce_sparse_host": (_i32, [_vp, _u32, _vp, _vp, _vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp]),
    "lh_comm_export": (_i32, [_vp, _vp]),
    "lh_comm_import": (_i32, [_vp, _u32, _u32, _vp]),
    "lh_snapshot_allreduce": (_i32, [_vp, _u32, C.POINTER(_u64)]),
    "lh_comm_allreduce_ms": (_i32, [_vp, _u64, C.POINTER(C.c_float)]),
    "lh_comm_info": (_i32, [_vp, C.POINTER(lh_comm_stats)]),
    "lh_snapshot_rows": (_i32, [_vp, _vp, _vp, C.POINTER(_u32)]),
    "lh_snapshot_allreduce_rows": (_i32, [_vp, _u64, _vp, _u32, _vp, _u32, _vp, C.POINTER(_u64)]),
    "lh_snapshot_row_levels": (_i32, [_vp, _vp]),
    "lh_snapshot_pack_rows": (_i32, [_vp, _u32, _vp, _vp, _u32, _vp, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_u64),
                                     C.POINTER(_vp)]),
    "lh_snapshot_unpack_rows": (_i32, [_vp, _u32]),
    "lh_keyed_kernel_name": (C.c_char_p, [_vp]),
    "lh_compress_f64": (_i32, [_vp, _vp, _sz, _vp, C.c_int, _vp]),
    "lh_decompress_table": (_i32, [_vp, _vp]),
    "lh_fastpath_margin": (_i32, [_vp, _vp, _sz, C.POINTER(C.c_double), C.POINTER(_u64), _vp]),
    "lh_fastpath_margin_detail": (_i32, [_vp, C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "lh_fastpath_certify": (_i32, [_vp, _u32, _u32, C.POINTER(lh_certify_form)]),
    "lh_gen_stream_f64": (_i32, [_vp, C.c_int, _u64, _u64, _sz, _vp, _vp]),
    "lh_gen_ids_u16": (_i32, [_vp, C.c_int, _u64, _u64, _sz, _u32, _vp, _vp]),
    "lh_get_stats": (_i32, [_vp, C.POINTER(lh_stats)]),
    "lh_sync": (_i32, [_vp]),
    "lh_ingest_stream": (_vp, [_vp]),
    "lh_device_alloc": (_i32, [_vp, _sz, C.POINTER(_vp)]),
    "lh_device_free": (_i32, [_vp, _vp]),
    "lh_host_alloc_pinned": (_i32, [_vp, _sz, C.POINTER(_vp)]),
    "lh_host_free_pinned": (_i32, [_vp, _vp]),
    "lh_memcpy_h2d": (_i32, [_vp, _vp, _vp, _sz]),
    "lh_memcpy_d2h": (_i32, [_vp, _vp, _vp, _sz]),
    "lh_tune": (_i32, [_vp, C.c_char_p, C.c_int64]),
    "lh_k1_variant_count": (_i32, []),
    "lh_k1_variant_current": (_i32, [_vp]),
    "lh_k1_variant_name": (C.c_char_p, [_vp, _i32]),
    "lh_last_kernel_ms": (_i32, [_vp, C.POINTER(C.c_float)]),
    "lh_ingest_seq": (_u64, [_vp]),
    "lh_kernel_ms": (_i32, [_vp, _u64, C.POINTER(C.c_float)]),
}

_lib = None


def load(build_if_missing: bool = True) -> C.CDLL:
    """Load (building first when stale/missing) the CUDA library.  Raises on failure."""
    global _lib
    if _lib is not None:
        return _lib
    if build_if_missing and _build.needs_build():
        _build.build()
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: the loghisto_b200 hot path is CUDA-only and has no CPU fallback; "
            "run `python -m loghisto_b200.build`")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if the ABI and the binding drift apart
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib
