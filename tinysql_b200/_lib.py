"""ctypes binding of libtinysql_b200.so — the C-ABI declared in include/tinysql_b200.h.

The product path is the CUDA library: if it is missing or no sm_90 GPU is visible every call
fails loudly (TQ_ERR_NO_DEVICE); there is no CPU fallback anywhere in this package.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libtinysql_b200.so")


class TQColumn(C.Structure):
    """tq_column == chunk.Column (util/chunk/column.go:28-34)."""
    _fields_ = [("length", C.c_int64), ("null_bitmap", C.c_void_p), ("offsets", C.c_void_p), ("data", C.c_void_p)]


class TQJoinDesc(C.Structure):
    _fields_ = [("join_type", C.c_int32), ("outer_is_right", C.c_int32), ("n_build_cols", C.c_int32),
                ("build_types", C.POINTER(C.c_int32)), ("n_probe_cols", C.c_int32), ("probe_types", C.POINTER(C.c_int32)),
                ("n_keys", C.c_int32), ("build_key_idx", C.POINTER(C.c_int32)), ("probe_key_idx", C.POINTER(C.c_int32)),
                ("probe_batch_rows", C.c_int64), ("flags", C.c_int32),
                ("default_inner_bits", C.POINTER(C.c_uint64)), ("default_inner_not_null", C.POINTER(C.c_uint8))]


class TQJoinCond(C.Structure):
    _fields_ = [("op", C.c_int32), ("lhs_col", C.c_int32), ("rhs_col", C.c_int32), ("const_type", C.c_int32), ("const_bits", C.c_uint64)]


class TQExprOp(C.Structure):
    _fields_ = [("kind", C.c_int32), ("op", C.c_int32), ("a", C.c_int32), ("b", C.c_int32), ("c", C.c_int32),
                ("a_unsigned", C.c_int32), ("b_unsigned", C.c_int32), ("is_null", C.c_int32), ("imm", C.c_uint64)]


class TQAggFunc(C.Structure):
    _fields_ = [("func", C.c_int32), ("arg_col", C.c_int32)]


class TQAggDesc(C.Structure):
    _fields_ = [("n_input_cols", C.c_int32), ("input_types", C.POINTER(C.c_int32)), ("n_group_by", C.c_int32),
                ("group_by_cols", C.POINTER(C.c_int32)), ("n_funcs", C.c_int32), ("funcs", C.POINTER(TQAggFunc)),
                ("est_groups", C.c_int64)]


class TQAggFinalFunc(C.Structure):
    _fields_ = [("func", C.c_int32), ("arg_col", C.c_int32), ("arg_col2", C.c_int32)]


class TQAggFinalDesc(C.Structure):
    _fields_ = [("n_input_cols", C.c_int32), ("input_types", C.POINTER(C.c_int32)), ("n_group_by", C.c_int32),
                ("group_by_cols", C.POINTER(C.c_int32)), ("n_funcs", C.c_int32), ("funcs", C.POINTER(TQAggFinalFunc)),
                ("est_groups", C.c_int64)]


class TQSortDesc(C.Structure):
    _fields_ = [("n_cols", C.c_int32), ("types", C.POINTER(C.c_int32)), ("n_by", C.c_int32), ("by_cols", C.POINTER(C.c_int32)),
                ("by_desc", C.POINTER(C.c_int32)), ("limit_offset", C.c_int64), ("limit_count", C.c_int64)]


class TQMJoinDesc(C.Structure):
    _fields_ = [("join_type", C.c_int32), ("outer_is_right", C.c_int32), ("n_inner_cols", C.c_int32), ("inner_types", C.POINTER(C.c_int32)),
                ("n_outer_cols", C.c_int32), ("outer_types", C.POINTER(C.c_int32)), ("n_keys", C.c_int32), ("inner_keys", C.POINTER(C.c_int32)),
                ("outer_keys", C.POINTER(C.c_int32)), ("default_inner_bits", C.POINTER(C.c_uint64)), ("default_inner_not_null", C.POINTER(C.c_uint8))]


# every symbol include/tinysql_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
_COL = C.POINTER(TQColumn)
_I32, _I64 = C.c_int32, C.c_int64
SYMBOLS = {
    "tq_init": (_I32, [_I32]), "tq_shutdown": (_I32, []), "tq_last_error": (_I32, [C.c_char_p, _I32]),
    "tq_version": (C.c_char_p, []),
    "tq_pinned_alloc": (_I32, [C.c_size_t, C.POINTER(_P)]), "tq_pinned_free": (_I32, [_P]),
    "tq_device_alloc": (_I32, [C.c_size_t, C.POINTER(_P)]), "tq_device_free": (_I32, [_P]),
    "tq_memcpy_h2d": (_I32, [_P, _P, C.c_size_t]), "tq_memcpy_d2h": (_I32, [_P, _P, C.c_size_t]),
    "tq_memcpy_d2d": (_I32, [_P, _P, C.c_size_t]),
    "tq_memset_device": (_I32, [_P, _I32, C.c_size_t]), "tq_device_synchronize": (_I32, []), "tq_compute_synchronize": (_I32, []),
    "tq_timer_start": (_I32, []), "tq_timer_stop": (_I32, [C.POINTER(C.c_float)]),
    "tq_kernel_launch_count": (_I64, []), "tq_flush_l2": (_I32, []),
    "tq_vec_compare_int": (_I32, [_I32, _I64, _COL, _I32, _COL, _I32, _COL, _I32]),
    "tq_vec_compare_real": (_I32, [_I32, _I64, _COL, _COL, _COL, _I32]),
    "tq_vec_arith_int": (_I32, [_I32, _I64, _COL, _I32, _COL, _I32, _COL, _I32]),
    "tq_vec_arith_real": (_I32, [_I32, _I64, _COL, _COL, _COL, C.POINTER(_I64), _I32]),
    "tq_vec_logic": (_I32, [_I32, _I64, _COL, _COL, _COL, _I32]),
    "tq_vec_unary": (_I32, [_I32, _I64, _COL, _I32, _COL, _I32]),
    "tq_vec_if": (_I32, [_I64, _COL, _COL, _COL, _COL, _I32]),
    "tq_vec_ifnull": (_I32, [_I64, _COL, _COL, _COL, _I32]),
    "tq_vec_compare_string": (_I32, [_I32, _I64, _COL, _COL, _COL, _I32]),
    "tq_vec_string_unary": (_I32, [_I32, _I64, _COL, _COL, _I32]),
    "tq_vec_in_int": (_I32, [_I64, _COL, _I32, _I32, _COL, C.POINTER(_I32), _COL, _I32]),
    "tq_vec_lt_plus_int": (_I32, [_I64, _COL, _COL, _COL, _COL, _I32]),
    "tq_vec_filter_int": (_I32, [_I64, _COL, _P, _I32]),
    "tq_vec_filter_real": (_I32, [_I64, _COL, _P, _I32]),
    "tq_expr_eval": (_I32, [_I64, _I32, _COL, _I32, C.POINTER(TQExprOp), _I32, C.POINTER(_I32), _COL, _P, C.POINTER(_I64), _I32]),
    "tq_vec_in_real": (_I32, [_I64, _COL, _I32, _COL, _COL, _I32]),
    "tq_vec_in_string": (_I32, [_I64, _COL, _I32, _COL, _COL, _I32]),
    "tq_vec_if_string": (_I32, [_I64, _COL, _COL, _COL, _COL, _I32]),
    "tq_vec_ifnull_string": (_I32, [_I64, _COL, _COL, _COL, _I32]),
    "tq_chunk_encoded_size": (_I32, [_I32, C.POINTER(_I32), _COL, C.POINTER(_I64)]),
    "tq_chunk_encode": (_I32, [_I32, C.POINTER(_I32), _COL, _P, _I64, C.POINTER(_I64)]),
    "tq_chunk_decode": (_I32, [_P, _I64, _I32, C.POINTER(_I32), _COL, C.POINTER(_I64)]),
    "tq_join_create": (_I32, [C.POINTER(TQJoinDesc), C.POINTER(_P)]),
    "tq_join_set_other_conditions": (_I32, [_P, _I32, C.POINTER(TQJoinCond)]),
    "tq_join_set_other_program": (_I32, [_P, _I32, C.POINTER(_I32), _I32, C.POINTER(TQExprOp)]),
    "tq_join_warnings": (_I32, [_P, C.POINTER(_I64)]),
    "tq_join_put_build": (_I32, [_P, _COL, _I32]), "tq_join_finalize_build": (_I32, [_P]),
    "tq_join_put_probe": (_I32, [_P, _COL, _P, _I32]), "tq_join_probe_eof": (_I32, [_P]),
    "tq_join_put_probe_segments": (_I32, [_P, _I32, _COL, C.POINTER(_P), _I64]),
    "tq_join_next": (_I32, [_P, _I64, _COL, C.POINTER(_I64), C.POINTER(_I32)]),
    "tq_join_next_device": (_I32, [_P, _COL, C.POINTER(_I64), C.POINTER(_I32)]),
    "tq_join_next_bytes": (_I32, [_P, _I64, C.POINTER(_I64)]),
    "tq_join_stats": (_I32, [_P, C.POINTER(_I64)]), "tq_join_destroy": (_I32, [_P]),
    "tq_chunk_decode_device": (_I32, [_P, _I64, _I32, C.POINTER(_I32), C.POINTER(_P), _COL, C.POINTER(_I64)]),
    "tq_chunk_device_free": (_I32, [_P]),
    "tq_vec_filter_string": (_I32, [_I64, _COL, _P, _I32]),
    "tq_agg_create": (_I32, [C.POINTER(TQAggDesc), C.POINTER(_P)]),
    "tq_agg_create_final": (_I32, [C.POINTER(TQAggFinalDesc), C.POINTER(_P)]),
    "tq_agg_output_type": (_I32, [_P, _I32, C.POINTER(_I32)]),
    "tq_agg_put": (_I32, [_P, _COL, _I32]), "tq_agg_eof": (_I32, [_P]),
    "tq_agg_next": (_I32, [_P, _I64, _COL, C.POINTER(_I64), C.POINTER(_I32)]),
    "tq_agg_next_device": (_I32, [_P, _COL, C.POINTER(_I64), C.POINTER(_I32)]),
    "tq_agg_next_bytes": (_I32, [_P, _I64, C.POINTER(_I64)]),
    "tq_agg_destroy": (_I32, [_P]), "tq_agg_stats": (_I32, [_P, C.POINTER(_I64)]),
    "tq_agg_partial_width": (_I32, [_P, C.POINTER(_I32)]),
    "tq_agg_export_partial": (_I32, [_P, _COL, C.POINTER(_I64)]),
    "tq_agg_merge_partial": (_I32, [_P, _COL, _I32]),
    "tq_sort_create": (_I32, [C.POINTER(TQSortDesc), C.POINTER(_P)]),
    "tq_sort_put": (_I32, [_P, _COL, _I32]), "tq_sort_eof": (_I32, [_P]),
    "tq_sort_next_bytes": (_I32, [_P, _I64, C.POINTER(_I64)]),
    "tq_sort_next": (_I32, [_P, _I64, _COL, C.POINTER(_I64), C.POINTER(_I32)]),
    "tq_sort_next_device": (_I32, [_P, _COL, C.POINTER(_I64), C.POINTER(_I32)]),
    "tq_sort_stats": (_I32, [_P, C.POINTER(_I64)]),
    "tq_sort_destroy": (_I32, [_P]),
    "tq_mjoin_create": (_I32, [C.POINTER(TQMJoinDesc), C.POINTER(_P)]),
    "tq_mjoin_set_other_conditions": (_I32, [_P, _I32, C.POINTER(TQJoinCond)]),
    "tq_mjoin_set_other_program": (_I32, [_P, _I32, C.POINTER(_I32), _I32, C.POINTER(TQExprOp)]),
    "tq_mjoin_warnings": (_I32, [_P, C.POINTER(_I64)]),
    "tq_mjoin_put_inner": (_I32, [_P, _COL, _I32]),
    "tq_mjoin_put_outer": (_I32, [_P, _COL, _P, _I32]),
    "tq_mjoin_finish": (_I32, [_P]),
    "tq_mjoin_next_bytes": (_I32, [_P, _I64, C.POINTER(_I64)]),
    "tq_mjoin_next": (_I32, [_P, _I64, _COL, C.POINTER(_I64), C.POINTER(_I32)]),
    "tq_mjoin_next_device": (_I32, [_P, _COL, C.POINTER(_I64), C.POINTER(_I32)]),
    "tq_mjoin_destroy": (_I32, [_P]),
    "tq_partition_device": (_I32, [_I32, _COL, C.POINTER(_I32), _I32, _I64, _I32, _COL, C.POINTER(_I64)]),
    "tq_enable_peer_access": (_I32, [_I32]),
    "tq_ipc_get_handle": (_I32, [_P, _P]), "tq_ipc_open_handle": (_I32, [_P, C.POINTER(_P)]), "tq_ipc_close_handle": (_I32, [_P]),
    "tq_partition_count_device": (_I32, [_COL, _I64, _I32, C.POINTER(_I64)]),
    "tq_partition_push_device": (_I32, [_I32, _COL, _I32, _I64, _I32, C.POINTER(_P), C.POINTER(_I64)]),
    "tq_partition_push_device_async": (_I32, [_I32, _COL, _I32, _I64, _I32, C.POINTER(_P), C.POINTER(_I64)]),
    "tq_partition_push_wait": (_I32, []),
    "tq_partition_push_regions": (_I32, [_I32, _COL, _I32, _I64, _I32, C.POINTER(_P), C.POINTER(_P), _I64, _I32, C.c_uint64]),
    "tq_region_wait": (_I32, [_P, _I32, C.c_uint64]),
    "tq_partition_push_sync": (_I32, [_I32]),
}

# status codes (include/tinysql_b200.h)
TQ_OK, TQ_ERR_INVALID_ARG, TQ_ERR_UNSUPPORTED_TYPE, TQ_ERR_OVERFLOW_BIGINT, TQ_ERR_OVERFLOW_BIGINT_UNSIGNED = 0, 1, 2, 3, 4
TQ_ERR_OVERFLOW_DOUBLE, TQ_ERR_DIVISION_BY_ZERO, TQ_ERR_CUDA, TQ_ERR_NO_DEVICE, TQ_ERR_OOM, TQ_ERR_STATE = 5, 6, 7, 8, 9, 10
TQ_TYPE_INT64, TQ_TYPE_UINT64, TQ_TYPE_FLOAT64, TQ_TYPE_FLOAT32, TQ_TYPE_BYTES = 1, 2, 3, 4, 5
TQ_TYPE_NOT_NULL = 0x100
TQ_MEM_HOST, TQ_MEM_DEVICE = 0, 1
TQ_JOIN_STABLE_INPUT = 1

_lib = None


def load():
    """Load the CUDA library; raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `make` (or __graft_entry__.build()); tinysql_b200 has no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class TQError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"tinysql_b200 status {status}: {msg}")
        self.status = status


def last_error():
    buf = C.create_string_buffer(512)
    load().tq_last_error(buf, 512)
    return buf.value.decode("utf-8", "replace")


def check(status):
    if status != TQ_OK:
        raise TQError(status, last_error())
