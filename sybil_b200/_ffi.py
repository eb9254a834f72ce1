"""ctypes view of include/sybilgpu.h (libsybilgpu.so) and of the block generator.

The structures below must stay field-for-field identical to the header; the
`-m "not gpu"` test `tests/test_abi.py` checks sizes and that every declared
symbol is exported.  There is no fallback: if the CUDA library is missing the
import raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SG_LIB: an alternative build of the same library (kernel experiments: `SG_NVCC_FLAGS=... SG_LIB_OUT=... _build.build_gpu`)
LIB_PATH = os.environ.get("SG_LIB") or os.path.join(_HERE, "csrc", "libsybilgpu.so")
GEN_PATH = os.path.join(_HERE, "csrc", "libsybilblockgen.so")
GOB_PATH = os.path.join(_HERE, "csrc", "libsybilgob.so")

SG_ABI_VERSION = 4
SG_ORDER_COUNT, SG_ORDER_NONE = -1, -2
SG_MAX_FILTERS, SG_MAX_GROUPS, SG_MAX_AGGS, SG_MAX_COLS = 15, 8, 16, 64
SG_BLOCK_ROWS = 65536
SG_MISSING_KEY = 0xFFFFFFFFFFFFFFFF

SG_OK, SG_ERR_INVALID, SG_ERR_CUDA, SG_ERR_UNSUPPORTED, SG_ERR_NOMEM, SG_ERR_NCCL, SG_ERR_STATE = 0, -1, -2, -3, -4, -5, -6
SG_COL_INT, SG_COL_STR, SG_COL_SET = 1, 2, 3
SG_ENC_ABSENT, SG_ENC_BUCKET, SG_ENC_VALUES = 0, 1, 2
SG_OP_GT, SG_OP_LT, SG_OP_EQ, SG_OP_NEQ, SG_OP_RE, SG_OP_NRE, SG_OP_IN, SG_OP_NIN = 0, 1, 2, 3, 4, 5, 6, 7
SG_MODE_AVG, SG_MODE_HIST = 0, 1
SG_HIST_BASIC, SG_HIST_MULTI = 0, 1

OPS = {"gt": SG_OP_GT, "lt": SG_OP_LT, "eq": SG_OP_EQ, "neq": SG_OP_NEQ, "re": SG_OP_RE, "nre": SG_OP_NRE,
       "in": SG_OP_IN, "nin": SG_OP_NIN}


class sg_filter_desc(C.Structure):
    _fields_ = [("col_slot", C.c_int32), ("col_type", C.c_int32), ("op", C.c_int32), ("_pad", C.c_int32),
                ("int_value", C.c_int64), ("str_value", C.c_char_p), ("str_len", C.c_int64)]


class sg_group_desc(C.Structure):
    _fields_ = [("col_slot", C.c_int32), ("col_type", C.c_int32)]


class sg_agg_desc(C.Structure):
    _fields_ = [("col_slot", C.c_int32), ("_pad", C.c_int32), ("info_min", C.c_int64), ("info_max", C.c_int64)]


class sg_query_desc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("op_mode", C.c_int32), ("hist_kind", C.c_int32),
                ("hist_bucket", C.c_int32), ("nfilters", C.c_int32), ("ngroups", C.c_int32), ("naggs", C.c_int32),
                ("time_col_slot", C.c_int32), ("time_bucket", C.c_int64), ("time_min", C.c_int64),
                ("time_max", C.c_int64), ("weight_col_slot", C.c_int32), ("order_by_agg", C.c_int32),
                ("order_asc", C.c_int32), ("weight_carry", C.c_int32), ("limit", C.c_int64),
                ("filters", C.POINTER(sg_filter_desc)), ("groups", C.POINTER(sg_group_desc)),
                ("aggs", C.POINTER(sg_agg_desc))]


class sg_column_desc(C.Structure):
    _fields_ = [("col_slot", C.c_int32), ("col_type", C.c_int32), ("encoding", C.c_int32), ("delta_ids", C.c_int32),
                ("delta_values", C.c_int32), ("nbins", C.c_uint32), ("nrecord_ids", C.c_uint32),
                ("nvalues", C.c_uint32), ("bin_values", C.c_void_p), ("bin_offsets", C.c_void_p),
                ("record_ids", C.c_void_p), ("values_i64", C.c_void_p), ("values_i32", C.c_void_p),
                ("ndict", C.c_uint32), ("id_bits", C.c_int32), ("dict_bytes", C.c_void_p),
                ("dict_offsets", C.c_void_p), ("value_bits", C.c_int32), ("_pad", C.c_int32),
                ("value_base", C.c_int64)]


class sg_int_info(C.Structure):
    _fields_ = [("col_slot", C.c_int32), ("_pad", C.c_int32), ("min", C.c_int64), ("max", C.c_int64)]


class sg_block_desc(C.Structure):
    _fields_ = [("block_index", C.c_int64), ("num_records", C.c_int32), ("ncols", C.c_int32),
                ("cols", C.POINTER(sg_column_desc)), ("ninfo", C.c_int32), ("_pad", C.c_int32),
                ("info", C.POINTER(sg_int_info))]


class sg_hist_view(C.Structure):
    _fields_ = [("count", C.c_int64), ("sum", C.c_int64), ("min", C.c_int64), ("max", C.c_int64),
                ("avg", C.c_double), ("num_buckets", C.c_int32), ("bucket_size", C.c_int32),
                ("nvalues", C.c_int32), ("nsubhists", C.c_int32), ("values", C.POINTER(C.c_int64))]


class sg_stats(C.Structure):
    _fields_ = [("kernel_ms", C.c_double), ("h2d_ms", C.c_double), ("kernel_launches", C.c_int64),
                ("h2d_bytes", C.c_int64), ("d2h_bytes", C.c_int64), ("rows_scanned", C.c_int64),
                ("blocks_scanned", C.c_int64), ("encoded_bytes", C.c_int64)]


# every symbol include/sybilgpu.h declares: name -> (restype, argtypes)
P = C.c_void_p
SYMBOLS = {
    "sg_abi_version": (C.c_int, []),
    "sg_create": (P, [C.c_int, C.POINTER(C.c_int)]),
    "sg_destroy": (None, [P]),
    "sg_last_error": (C.c_char_p, [P]),
    "sg_device_sm_count": (C.c_int, [P]),
    "sg_pinned_alloc": (P, [P, C.c_size_t]),
    "sg_pinned_free": (None, [P, P]),
    "sg_table_create": (P, [P, C.c_int32, C.POINTER(C.c_int32)]),
    "sg_table_free": (None, [P]),
    "sg_table_add_block": (C.c_int, [P, C.POINTER(sg_block_desc)]),
    "sg_table_add_blocks": (C.c_int, [P, P, C.c_int64]),
    "sg_table_sync": (C.c_int, [P]),
    "sg_table_clear": (C.c_int, [P]),
    "sg_table_num_blocks": (C.c_int64, [P]),
    "sg_table_num_rows": (C.c_int64, [P]),
    "sg_table_device_bytes": (C.c_int64, [P]),
    "sg_table_dict_size": (C.c_int64, [P, C.c_int32]),
    "sg_table_dict_get": (C.c_int, [P, C.c_int32, C.c_int64, C.POINTER(P), C.POINTER(C.c_int64)]),
    "sg_table_intdict_size": (C.c_int64, [P, C.c_int32]),
    "sg_table_intdict_get": (C.c_int, [P, C.c_int32, C.c_int64, C.POINTER(C.c_int64)]),
    "sg_table_dict_seed_str": (C.c_int, [P, C.c_int32, P, P, C.c_int64]),
    "sg_table_dict_seed_int": (C.c_int, [P, C.c_int32, P, C.c_int64]),
    "sg_table_encoded_bytes": (C.c_int64, [P]),
    "sg_table_h2d_bytes": (C.c_int64, [P]),
    "sg_query_begin": (P, [P, P, C.POINTER(sg_query_desc)]),
    "sg_query_free": (None, [P]),
    "sg_query_set_str_lut": (C.c_int, [P, C.c_int32, P, C.c_int64]),
    "sg_query_set_str_replace": (C.c_int, [P, C.c_int32, P, P, C.c_int64]),
    "sg_query_set_sparse_groups": (C.c_int, [P, C.c_int32]),
    "sg_query_set_hashed_folds": (C.c_int, [P, C.c_int32]),
    "sg_query_should_load": (C.c_int, [P, C.POINTER(sg_block_desc)]),
    "sg_query_run": (C.c_int, [P]),
    "sg_query_submit_block": (C.c_int, [P, C.POINTER(sg_block_desc)]),
    "sg_query_allreduce": (C.c_int, [P]),
    "sg_query_finish": (C.c_int, [P, C.POINTER(P)]),
    "sg_query_kernel_ms": (C.c_double, [P]),
    "sg_query_kernel_launches": (C.c_int64, [P]),
    "sg_comm_unique_id": (C.c_int, [P, C.c_char_p]),
    "sg_comm_init": (C.c_int, [P, C.c_char_p, C.c_int, C.c_int]),
    "sg_result_free": (None, [P]),
    "sg_result_matched_count": (C.c_int64, [P]),
    "sg_result_num_groups": (C.c_int64, [P]),
    "sg_result_num_groups_total": (C.c_int64, [P]),
    "sg_result_num_broken": (C.c_int64, [P]),
    "sg_result_num_skipped": (C.c_int64, [P]),
    "sg_result_group": (C.c_int, [P, C.c_int64, C.POINTER(C.c_uint64), C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "sg_result_group_key": (C.c_int, [P, C.c_int64, C.POINTER(P), C.POINTER(C.c_int64)]),
    "sg_result_hist": (C.c_int, [P, C.c_int64, C.c_int32, C.POINTER(sg_hist_view)]),
    "sg_result_percentiles": (C.c_int, [P, C.c_int64, C.c_int32, C.POINTER(C.c_int64)]),
    "sg_result_stddev": (C.c_double, [P, C.c_int64, C.c_int32]),
    "sg_result_sparse_buckets": (C.c_int64, [P, C.c_int64, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int64]),
    "sg_result_num_time_buckets": (C.c_int64, [P]),
    "sg_result_time_bucket": (C.c_int64, [P, C.c_int64]),
    "sg_result_time_slice": (P, [P, C.c_int64]),
    "sg_query_stats": (C.c_int, [P, C.POINTER(sg_stats)]),
}

_lib = None


def bind(lib, symbols):
    for name, (res, args) in symbols.items():
        fn = getattr(lib, name)  # AttributeError when the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    return lib


def lib():
    """libsybilgpu.so, loaded once.  Raises if it has not been built: the product has no CPU path."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "libsybilgpu.so is not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'`; "
                "there is no CPU fallback." % LIB_PATH)
        _lib = bind(C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL), SYMBOLS)
    return _lib


# ---- block generator (sybil_b200/csrc/blockgen.cpp) -----------------------------
SBG_UNIFORM, SBG_SUM4, SBG_TIME, SBG_STRKEY = 0, 1, 2, 3


class sbg_col(C.Structure):
    _fields_ = [("col_slot", C.c_int32), ("col_type", C.c_int32), ("kind", C.c_int32), ("null_per_1024", C.c_int32),
                ("lo", C.c_int64), ("span", C.c_int64), ("a", C.c_int64), ("b", C.c_int64), ("prefix", C.c_char * 16)]


class sbg_spec(C.Structure):
    _fields_ = [("seed", C.c_uint64), ("total_rows", C.c_int64), ("block_rows", C.c_int32), ("ncols", C.c_int32),
                ("cardinality_threshold", C.c_int32), ("num_col_slots", C.c_int32), ("cols", C.POINTER(sbg_col)),
                ("narrow", C.c_int32), ("_pad", C.c_int32)]


class sbg_eval_spec(C.Structure):
    _fields_ = [("nfilters", C.c_int32), ("filter_col", C.c_int32 * 8), ("filter_op", C.c_int32 * 8),
                ("filter_val", C.c_int64 * 8), ("ngroups", C.c_int32), ("group_col", C.c_int32 * 4),
                ("time_col", C.c_int32), ("naggs", C.c_int32), ("time_bucket", C.c_int64), ("time_first", C.c_int64),
                ("time_n", C.c_int32), ("nvals", C.c_int32), ("agg_col", C.c_int32 * 16), ("info_min", C.c_int64 * 16),
                ("info_max", C.c_int64 * 16), ("bsize", C.c_int64 * 16)]


GEN_SYMBOLS = {
    "sbg_eval": (C.c_int64, [C.POINTER(sbg_spec), C.POINTER(sbg_eval_spec), C.c_int64, C.c_int64, C.c_int, P, P, P, P]),
    "sbg_generate": (P, [C.POINTER(sbg_spec), C.c_int64, C.c_int64, C.c_int, P, C.c_size_t]),
    "sbg_free": (None, [P]),
    "sbg_num_blocks": (C.c_int64, [P]),
    "sbg_block": (C.POINTER(sg_block_desc), [P, C.c_int64]),
    "sbg_arena_used": (C.c_int64, [P]),
    "sbg_encoded_bytes": (C.c_int64, [P]),
    "sbg_total_blocks": (C.c_int64, [C.POINTER(sbg_spec)]),
    "sbg_cell": (C.c_int64, [C.POINTER(sbg_spec), C.c_int32, C.c_int64, C.POINTER(C.c_int32)]),
}
_gen = None


def gen():
    global _gen
    if _gen is None:
        if not os.path.exists(GEN_PATH):
            raise RuntimeError("libsybilblockgen.so is not built (%s)" % GEN_PATH)
        _gen = bind(C.CDLL(GEN_PATH), GEN_SYMBOLS)
    return _gen


# ---- include/sybilgob.h: sybil block directory -> sg_block_desc (host side, C++) -------------------
GOB_SYMBOLS = {
    "sgob_read_block_dir": (P, [C.c_char_p, C.POINTER(C.c_char_p), C.POINTER(C.c_int32), C.c_int32, C.POINTER(C.c_uint8),
                                C.c_int64, C.c_char_p, C.c_size_t]),
    "sgob_block_desc": (C.POINTER(sg_block_desc), [P]),
    "sgob_set_narrow": (None, [C.c_int]),
    "sgob_block_free": (None, [P]),
    "sgob_block_bytes": (C.c_int64, [P]),
    "sgob_table_open": (P, [C.c_char_p, C.c_char_p, C.c_char_p, C.c_size_t]),
    "sgob_table_free": (None, [P]),
    "sgob_table_num_cols": (C.c_int32, [P]),
    "sgob_table_col_name": (C.c_char_p, [P, C.c_int32]),
    "sgob_table_col_type": (C.c_int32, [P, C.c_int32]),
    "sgob_table_int_info": (C.c_int32, [P, C.c_int32, C.POINTER(C.c_int64), C.POINTER(C.c_int64)]),
    "sgob_table_num_blocks": (C.c_int64, [P]),
    "sgob_table_block_dir": (C.c_char_p, [P, C.c_int64]),
}
_gob = None


def gobread():
    global _gob
    if _gob is None:
        if not os.path.exists(GOB_PATH):
            raise RuntimeError("libsybilgob.so is not built (%s)" % GOB_PATH)
        _gob = bind(C.CDLL(GOB_PATH), GOB_SYMBOLS)
    return _gob
