"""ctypes mirror of include/tskv_gpu.h (the C-ABI drop-in boundary) and of the host generator ABI.

Nothing here computes: it only declares structs/prototypes and loads the in-tree shared libraries.
A missing library is a hard error (there is no CPU fallback for the product path).
"""
import ctypes as C
import os

import numpy as np

_PKG = os.path.dirname(os.path.abspath(__file__))

# ---- status codes (include/tskv_gpu.h) ---------------------------------------------------------
TSKV_OK = 0
TSKV_ERR_INVALID_ARG = 1
TSKV_ERR_BAD_ENCODING = 2
TSKV_ERR_SHORT_BLOCK = 3
TSKV_ERR_CRC_MISMATCH = 4
TSKV_ERR_BITSET_MISMATCH = 5
TSKV_ERR_UNSUPPORTED = 6
TSKV_ERR_BUCKET_RANGE = 7
TSKV_ERR_CUDA = 8
TSKV_ERR_NCCL = 9
TSKV_ERR_OOM = 10
TSKV_ERR_BAD_LENGTH = 11
TSKV_ERR_PAGE_FORMAT = 12
STATUS_NAMES = {v: k for k, v in list(globals().items()) if k.startswith("TSKV_ERR_") or k == "TSKV_OK"}

TSKV_PT_TIME, TSKV_PT_I64, TSKV_PT_U64, TSKV_PT_F64, TSKV_PT_BOOL = 0, 1, 2, 3, 4
TSKV_ENC_DEFAULT, TSKV_ENC_NULL, TSKV_ENC_DELTA, TSKV_ENC_QUANTILE = 0, 1, 2, 3
TSKV_ENC_GORILLA, TSKV_ENC_BITPACK, TSKV_ENC_DELTA_TS = 6, 10, 11

TSKV_AGG_COUNT, TSKV_AGG_SUM, TSKV_AGG_MIN, TSKV_AGG_MAX = 1, 2, 4, 8
TSKV_AGG_MEAN, TSKV_AGG_FIRST, TSKV_AGG_LAST, TSKV_AGG_ALL = 16, 32, 64, 0x7F
# f64 sum of squared deviations from the cell mean (the variance state; engine.py derives var* / stddev* from it)
TSKV_AGG_M2 = 0x80
AGG_NAMES = {1: "count", 2: "sum", 4: "min", 8: "max", 16: "mean", 32: "first", 64: "last", 128: "m2"}
# column pairs of tskv_query.n_pairs (covariance / correlation state; engine.py derives covar* / corr from it)
TSKV_MAX_PAIRS = 8
# medians: n_medians in bits 8..15 of tskv_query.reserved, operands after the pairs' (see include/tskv_gpu.h)
TSKV_MAX_MEDIANS = 8
TSKV_MAX_MEDIAN_CELLS = 1 << 22


def query_medians(n):
    """TSKV_QUERY_MEDIANS(n): the flags-word bits of n medians."""
    return (int(n) & 0xFF) << 8


def query_n_medians(flags):
    """TSKV_QUERY_N_MEDIANS(flags)."""
    return (int(flags) >> 8) & 0xFF


# increases: n_increases in bits 16..23 of tskv_query.reserved, operands after the medians' (see include/tskv_gpu.h)
TSKV_MAX_INCREASES = 8


def query_increases(n):
    """TSKV_QUERY_INCREASES(n): the flags-word bits of n increases."""
    return (int(n) & 0xFF) << 16


def query_n_increases(flags):
    """TSKV_QUERY_N_INCREASES(flags)."""
    return (int(flags) >> 16) & 0xFF


TSKV_UPLOAD_VERIFY_CRC = 1
TSKV_UPLOAD_HOST_RESIDENT = 2
TSKV_UPLOAD_VERIFY_ON_READ = 4

# numpy view of tskv_page_desc (24 bytes)
PAGE_DESC_DTYPE = np.dtype(
    [("offset", "<u8"), ("size", "<u4"), ("num_values", "<u4"), ("series_id", "<u4"),
     ("column_id", "<u2"), ("phys_type", "u1"), ("reserved", "u1")], align=False)
assert PAGE_DESC_DTYPE.itemsize == 24

# numpy view of tskv_tombstone (24 bytes); series_id / column_id = TSKV_TOMB_ALL: see include/tskv_gpu.h
TSKV_TOMB_ALL = 0xFFFFFFFF
TSKV_QUERY_MULTI_RANK = 1
TOMBSTONE_DTYPE = np.dtype([("series_id", "<u4"), ("column_id", "<u4"), ("min_ts", "<i8"), ("max_ts", "<i8")], align=False)
assert TOMBSTONE_DTYPE.itemsize == 24


def tombstones(entries):
    """[(series_id | None, column_id | None, min_ts, max_ts), ...] -> TOMBSTONE_DTYPE array (None = TSKV_TOMB_ALL)."""
    a = np.zeros(len(entries), dtype=TOMBSTONE_DTYPE)
    for i, (s, c, lo, hi) in enumerate(entries):
        a[i] = (TSKV_TOMB_ALL if s is None else s, TSKV_TOMB_ALL if c is None else c, lo, hi)
    return a


class PageDesc(C.Structure):
    _fields_ = [("offset", C.c_uint64), ("size", C.c_uint32), ("num_values", C.c_uint32),
                ("series_id", C.c_uint32), ("column_id", C.c_uint16), ("phys_type", C.c_uint8),
                ("reserved", C.c_uint8)]


class TimeRange(C.Structure):
    """Closed interval == models::predicate::domain::TimeRange."""
    _fields_ = [("min_ts", C.c_int64), ("max_ts", C.c_int64)]


class AggColumn(C.Structure):
    _fields_ = [("column_id", C.c_uint16), ("phys_type", C.c_uint8), ("agg_mask", C.c_uint8)]


class FieldPredicate(C.Structure):
    _fields_ = [("column_id", C.c_uint16), ("phys_type", C.c_uint8), ("op", C.c_uint8), ("reserved", C.c_uint32),
                ("value", C.c_uint64)]


CMP_OPS = {"==": 0, "=": 0, "!=": 1, "<>": 1, "<": 2, "<=": 3, ">": 4, ">=": 5}


class Query(C.Structure):
    _fields_ = [("series_ids", C.POINTER(C.c_uint32)), ("n_series", C.c_uint32),
                ("n_time_ranges", C.c_uint32), ("time_ranges", C.POINTER(TimeRange)),
                ("origin", C.c_int64), ("width", C.c_int64), ("first_bucket_start", C.c_int64),
                ("n_buckets", C.c_uint32), ("group_by_series", C.c_uint32),
                ("columns", C.POINTER(AggColumn)), ("n_columns", C.c_uint32), ("reserved", C.c_uint32),
                ("predicates", C.POINTER(FieldPredicate)), ("n_predicates", C.c_uint32), ("n_pairs", C.c_uint32)]


class OutputLayout(C.Structure):
    _fields_ = [("n_out", C.c_uint64), ("n_groups", C.c_uint64), ("n_cells", C.c_uint64),
                ("bitmap_stride", C.c_uint64), ("values_bytes", C.c_uint64),
                ("validity_bytes", C.c_uint64)]


class Counters(C.Structure):
    _fields_ = [("page_read_count", C.c_uint64), ("page_read_bytes", C.c_uint64),
                ("points_decoded", C.c_uint64), ("rows_in_range", C.c_uint64),
                ("elapsed_scan_ms", C.c_double), ("elapsed_h2d_ms", C.c_double),
                ("kernel_launches", C.c_uint64), ("elapsed_fused_ms", C.c_double),
                ("dominant_kernel_ms", C.c_double), ("dominant_kernel_bytes", C.c_uint64),
                ("dominant_kernel_bin", C.c_uint64), ("h2d_bytes", C.c_uint64), ("pruned_page_count", C.c_uint64)]


class PartialsView(C.Structure):
    _fields_ = [("sum_i64_ptr", C.c_uint64), ("sum_i64_len", C.c_uint64),
                ("sum_f64_ptr", C.c_uint64), ("sum_f64_len", C.c_uint64),
                ("min_i64_ptr", C.c_uint64), ("min_i64_len", C.c_uint64),
                ("max_i64_ptr", C.c_uint64), ("max_i64_len", C.c_uint64),
                ("sel_val_ptr", C.c_uint64), ("sel_val_len", C.c_uint64),
                ("sel_first_len", C.c_uint64), ("sel_last_len", C.c_uint64)]


# every symbol include/tskv_gpu.h declares (tests check the library exports all of them)
GPU_SYMBOLS = [
    "tskvgpu_ctx_create", "tskvgpu_ctx_destroy", "tskvgpu_last_error", "tskvgpu_last_error_page",
    "tskvgpu_get_counters", "tskvgpu_ctx_stream", "tskvgpu_upload_pages", "tskvgpu_pages_destroy",
    "tskvgpu_pages_series_count", "tskvgpu_pages_set_time_bounds", "tskvgpu_pages_set_tombstones", "tskvgpu_pages_set_chunk_files", "tskvgpu_pages_set_value_stats", "tskvgpu_decode_pages",
    "tskvgpu_query_output_layout", "tskvgpu_comm_unique_id", "tskvgpu_comm_init", "tskvgpu_comm_destroy", "tskvgpu_scan_exchange",
    "tskvgpu_scan_aggregate", "tskvgpu_scan_prepare", "tskvgpu_scan_run", "tskvgpu_scan_enqueue",
    "tskvgpu_scan_sync", "tskvgpu_scan_partials", "tskvgpu_scan_work_list", "tskvgpu_scan_exchange_view", "tskvgpu_scan_merge_gathered",
    "tskvgpu_scan_snapshot_keys", "tskvgpu_scan_mask_values", "tskvgpu_scan_finalize",
    "tskvgpu_scan_finalize_device", "tskvgpu_scan_destroy", "tskvgpu_version",
    "tskvgpu_scan_prepare_sliding", "tskvgpu_scan_aggregate_sliding",
    "tskvgpu_query_output_layout_grouped", "tskvgpu_scan_prepare_grouped", "tskvgpu_scan_aggregate_grouped",
    "tskvgpu_query_output_layout_edges", "tskvgpu_scan_prepare_edges", "tskvgpu_scan_aggregate_edges",
    "tskvgpu_query_output_layout_labels", "tskvgpu_scan_prepare_labels", "tskvgpu_scan_aggregate_labels",
]


TSKV_STATS_MINMAX = 1
VALUE_STATS_DTYPE = np.dtype([("min", "<u8"), ("max", "<u8"), ("flags", "<u4"), ("reserved", "<u4")])  # tskv_value_stats


def gpu_library_path():
    # TSKV_GPU_LIB: developer override to A/B alternative builds of the same library
    return os.environ.get("TSKV_GPU_LIB") or os.path.join(_PKG, "libtskv_gpu.so")


def hostgen_library_path():
    return os.path.join(_PKG, "libtskv_hostgen.so")


_gpu = None
_gen = None


def load_gpu_library():
    """Loads cnosdb_b200/libtskv_gpu.so and types its entry points. Raises if it is missing."""
    global _gpu
    if _gpu is not None:
        return _gpu
    path = gpu_library_path()
    if not os.path.exists(path):
        raise ImportError(
            "cnosdb_b200/libtskv_gpu.so is missing: build it with `python -m cnosdb_b200.build` "
            "(__graft_entry__.build()). There is no CPU fallback for the scan path.")
    lib = C.CDLL(path)
    vp, u8p, u64p = C.c_void_p, C.POINTER(C.c_uint8), C.POINTER(C.c_uint64)
    lib.tskvgpu_version.restype = C.c_char_p
    lib.tskvgpu_ctx_create.argtypes = [C.c_int32, C.POINTER(vp)]
    lib.tskvgpu_ctx_destroy.argtypes = [vp]
    lib.tskvgpu_ctx_destroy.restype = None
    lib.tskvgpu_last_error.argtypes = [vp]
    lib.tskvgpu_last_error.restype = C.c_char_p
    lib.tskvgpu_last_error_page.argtypes = [vp]
    lib.tskvgpu_last_error_page.restype = C.c_int64
    lib.tskvgpu_get_counters.argtypes = [vp, C.POINTER(Counters)]
    lib.tskvgpu_ctx_stream.argtypes = [vp]
    lib.tskvgpu_ctx_stream.restype = C.c_uint64
    lib.tskvgpu_upload_pages.argtypes = [vp, vp, C.c_uint64, vp, C.c_uint64, C.c_uint32, C.POINTER(vp)]
    lib.tskvgpu_pages_destroy.argtypes = [vp, vp]
    lib.tskvgpu_pages_destroy.restype = None
    lib.tskvgpu_pages_series_count.argtypes = [vp]
    lib.tskvgpu_pages_series_count.restype = C.c_uint64
    lib.tskvgpu_pages_set_tombstones.argtypes = [vp, vp, vp, C.c_uint64]
    lib.tskvgpu_pages_set_time_bounds.argtypes = [vp, vp, vp, C.c_uint64]
    lib.tskvgpu_pages_set_chunk_files.argtypes = [vp, vp, vp, C.c_uint64]
    lib.tskvgpu_pages_set_value_stats.argtypes = [vp, vp, vp, C.c_uint64]
    lib.tskvgpu_comm_unique_id.argtypes = [vp]
    lib.tskvgpu_comm_init.argtypes = [vp, vp, C.c_int32, C.c_int32]
    lib.tskvgpu_comm_destroy.argtypes = [vp]
    lib.tskvgpu_comm_destroy.restype = None
    lib.tskvgpu_scan_exchange.argtypes = [vp, vp]
    lib.tskvgpu_decode_pages.argtypes = [vp, vp, C.c_uint64, C.c_uint64, vp, vp]
    lib.tskvgpu_query_output_layout.argtypes = [vp, C.POINTER(Query), C.POINTER(OutputLayout)]
    lib.tskvgpu_scan_aggregate.argtypes = [vp, vp, C.POINTER(Query), vp, vp]
    lib.tskvgpu_scan_prepare.argtypes = [vp, vp, C.POINTER(Query), C.POINTER(vp)]
    lib.tskvgpu_scan_aggregate_sliding.argtypes = [vp, vp, C.POINTER(Query), C.c_int64, vp, vp]
    lib.tskvgpu_scan_prepare_sliding.argtypes = [vp, vp, C.POINTER(Query), C.c_int64, C.POINTER(vp)]
    lib.tskvgpu_query_output_layout_grouped.argtypes = [vp, C.POINTER(Query), vp, C.c_uint32, C.POINTER(OutputLayout)]
    lib.tskvgpu_scan_prepare_grouped.argtypes = [vp, vp, C.POINTER(Query), vp, C.c_uint32, C.c_int64, C.POINTER(vp)]
    lib.tskvgpu_scan_aggregate_grouped.argtypes = [vp, vp, C.POINTER(Query), vp, C.c_uint32, C.c_int64, vp, vp]
    lib.tskvgpu_query_output_layout_edges.argtypes = [vp, C.POINTER(Query), vp, vp, C.c_uint32, C.POINTER(OutputLayout)]
    lib.tskvgpu_scan_prepare_edges.argtypes = [vp, vp, C.POINTER(Query), vp, vp, C.c_uint32, C.POINTER(vp)]
    lib.tskvgpu_scan_aggregate_edges.argtypes = [vp, vp, C.POINTER(Query), vp, vp, C.c_uint32, vp, vp]
    lib.tskvgpu_query_output_layout_labels.argtypes = [vp, C.POINTER(Query), vp, C.c_uint32, vp, vp, C.c_uint32,
                                                       C.POINTER(OutputLayout)]
    lib.tskvgpu_scan_prepare_labels.argtypes = [vp, vp, C.POINTER(Query), vp, C.c_uint32, vp, vp, C.c_uint32, C.POINTER(vp)]
    lib.tskvgpu_scan_aggregate_labels.argtypes = [vp, vp, C.POINTER(Query), vp, C.c_uint32, vp, vp, C.c_uint32, vp, vp]
    lib.tskvgpu_scan_run.argtypes = [vp, vp]
    lib.tskvgpu_scan_enqueue.argtypes = [vp, vp]
    lib.tskvgpu_scan_sync.argtypes = [vp, vp]
    lib.tskvgpu_scan_partials.argtypes = [vp, vp, C.POINTER(PartialsView)]
    lib.tskvgpu_scan_work_list.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    lib.tskvgpu_scan_exchange_view.argtypes = [vp, vp, u64p, u64p]
    lib.tskvgpu_scan_merge_gathered.argtypes = [vp, vp, C.c_uint64, C.c_uint32]
    lib.tskvgpu_scan_snapshot_keys.argtypes = [vp, vp]
    lib.tskvgpu_scan_mask_values.argtypes = [vp, vp]
    lib.tskvgpu_scan_finalize.argtypes = [vp, vp, vp, vp]
    lib.tskvgpu_scan_finalize_device.argtypes = [vp, vp, u64p, u64p]
    lib.tskvgpu_scan_destroy.argtypes = [vp, vp]
    lib.tskvgpu_scan_destroy.restype = None
    for name in GPU_SYMBOLS:
        fn = getattr(lib, name)
        if fn.restype is C.c_int:  # default restype: every other entry point returns tskv_status
            fn.restype = C.c_int32
    _gpu = lib
    return lib


class GenSpec(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("n_series", C.c_uint32), ("first_series_id", C.c_uint32),
                ("series_stride", C.c_uint32), ("n_fields", C.c_uint32), ("n_points", C.c_uint32),
                ("value_kind", C.c_uint32), ("t0", C.c_int64), ("step", C.c_int64),
                ("jitter_permille", C.c_uint32), ("jitter_max", C.c_uint32),
                ("null_page_permille", C.c_uint32), ("null_row_permille", C.c_uint32),
                ("raw_encoding_permille", C.c_uint32), ("reserved", C.c_uint32)]


class GenResult(C.Structure):
    _fields_ = [("arena", C.c_void_p), ("arena_len", C.c_uint64), ("descs", C.c_void_p),
                ("n_descs", C.c_uint64), ("n_points", C.c_uint64)]


def load_hostgen_library():
    global _gen
    if _gen is not None:
        return _gen
    path = hostgen_library_path()
    if not os.path.exists(path):
        raise ImportError("cnosdb_b200/libtskv_hostgen.so is missing: run `python -m cnosdb_b200.build`")
    lib = C.CDLL(path)
    lib.tskvgen_generate.argtypes = [C.POINTER(GenSpec), C.c_int, C.POINTER(GenResult)]
    lib.tskvgen_generate.restype = C.c_int
    lib.tskvgen_free.argtypes = [C.POINTER(GenResult)]
    lib.tskvgen_free.restype = None
    for name in ("tskvw_encode_timestamps", "tskvw_encode_integers", "tskvw_encode_floats",
                 "tskvw_encode_raw", "tskvw_simple8b_pack"):
        fn = getattr(lib, name)
        fn.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
        fn.restype = C.c_int64
    lib.tskvw_build_page.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64]
    lib.tskvw_build_page.restype = C.c_int64
    lib.tskvw_crc32.argtypes = [C.c_void_p, C.c_uint64]
    lib.tskvw_crc32.restype = C.c_uint32
    _gen = lib
    return lib
