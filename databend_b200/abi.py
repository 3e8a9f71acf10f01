"""ctypes mirror of include/dbx.h (the C-ABI of libdbx).

Keep in lock-step with the header; tests/test_abi.py checks struct sizes against the
library's own `dbx_abi_sizeof` table so that a drift fails loudly.
"""
import ctypes as C

ABI_VERSION = 1

# dbx_status
OK, ERR_INVALID, ERR_CUDA, ERR_BAD_ARGUMENTS, ERR_UNSUPPORTED, ERR_OOM, ERR_STATE, ERR_NO_DEVICE = range(8)

# dbx_dtype
BOOL, I8, I16, I32, I64, U8, U16, U32, U64, F32, F64, VEC_F32, VEC_I8 = range(13)
MEM_HOST, MEM_DEVICE = 0, 1
NULLABLE = 0x100

# dbx_cmp_op / dbx_arith_op / dbx_pred_kind
EQ, NE, LT, LE, GT, GE = range(6)
ARITH_NONE, ARITH_MODULO = 0, 1
PRED_CMP, PRED_AND, PRED_OR, PRED_BOOLCOL, PRED_CONST = range(5)

# dbx_agg_kind
AGG_SUM, AGG_COUNT, AGG_AVG, AGG_MIN, AGG_MAX = range(5)

# dbx_op_kind
OP_FILTER, OP_AGG_PARTIAL, OP_AGG_FINAL, OP_TOPK, OP_JOIN, OP_WINDOW = range(6)

DIST_COSINE, DIST_L2 = 0, 1
JOIN_INNER, JOIN_LEFT_SEMI, JOIN_LEFT_ANTI, JOIN_LEFT = 0, 1, 2, 3
JOIN_RIGHT, JOIN_RIGHT_SEMI, JOIN_RIGHT_ANTI, JOIN_FULL = 4, 5, 6, 7

MAX_PRED_NODES = 16
MAX_AGGS = 8
MAX_GROUP_COLS = 4


class ScalarValue(C.Union):
    _fields_ = [("i64", C.c_int64), ("u64", C.c_uint64), ("f64", C.c_double)]


class Scalar(C.Structure):
    _fields_ = [("dtype", C.c_int32), ("is_null", C.c_int32), ("v", ScalarValue)]


class Column(C.Structure):
    _fields_ = [
        ("dtype", C.c_int32),
        ("mem", C.c_int32),
        ("is_const", C.c_int32),
        ("vec_dim", C.c_int32),
        ("len", C.c_int64),
        ("data", C.c_void_p),
        ("data_bit_offset", C.c_int64),
        ("validity", C.c_void_p),
        ("validity_bit_offset", C.c_int64),
        ("null_count", C.c_int64),
        ("konst", Scalar),
    ]


class Block(C.Structure):
    _fields_ = [
        ("num_rows", C.c_int64),
        ("num_cols", C.c_int32),
        ("reserved", C.c_int32),
        ("cols", C.POINTER(Column)),
        ("meta", C.c_void_p),
        ("owner", C.c_void_p),
    ]


class Operand(C.Structure):
    _fields_ = [
        ("is_const", C.c_int32),
        ("col", C.c_int32),
        ("arith", C.c_int32),
        ("reserved", C.c_int32),
        ("c", Scalar),
    ]


class PredNode(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("cmp", C.c_int32),
        ("n_children", C.c_int32),
        ("value", C.c_int32),
        ("lhs", Operand),
        ("rhs", Operand),
    ]


class Predicate(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("reserved", C.c_int32), ("nodes", PredNode * MAX_PRED_NODES)]


class AggDesc(C.Structure):
    _fields_ = [("kind", C.c_int32), ("arg_col", C.c_int32)]


class AggParams(C.Structure):
    _fields_ = [
        ("n_group_cols", C.c_int32),
        ("group_cols", C.c_int32 * MAX_GROUP_COLS),
        ("n_aggs", C.c_int32),
        ("aggs", AggDesc * MAX_AGGS),
        ("filter", Predicate),
        ("expected_groups", C.c_int64),
    ]


MAX_SORT_KEYS = 4


class TopkParams(C.Structure):
    _fields_ = [
        ("key_col", C.c_int32),
        ("asc", C.c_int32),
        ("nulls_first", C.c_int32),
        ("reserved", C.c_int32),
        ("limit", C.c_int64),
        ("n_extra_keys", C.c_int32),
        ("extra_key_cols", C.c_int32 * (MAX_SORT_KEYS - 1)),
        ("extra_asc", C.c_int32 * (MAX_SORT_KEYS - 1)),
        ("extra_nulls_first", C.c_int32 * (MAX_SORT_KEYS - 1)),
    ]


# dbx_window_kind / dbx_frame_units / dbx_frame_bound
(WIN_ROW_NUMBER, WIN_RANK, WIN_DENSE_RANK, WIN_PERCENT_RANK, WIN_CUME_DIST, WIN_NTILE, WIN_LAG, WIN_LEAD, WIN_NTH_VALUE,
 WIN_AGGREGATE) = range(10)
FRAME_ROWS, FRAME_RANGE = 0, 1
BOUND_UNBOUNDED_PRECEDING, BOUND_PRECEDING, BOUND_CURRENT_ROW, BOUND_FOLLOWING, BOUND_UNBOUNDED_FOLLOWING = range(1, 6)
MAX_WINDOW_FUNCS = 8


class WindowFrame(C.Structure):
    _fields_ = [
        ("units", C.c_int32),
        ("start", C.c_int32),
        ("end", C.c_int32),
        ("reserved", C.c_int32),
        ("start_offset", C.c_int64),
        ("end_offset", C.c_int64),
    ]


class WindowFunc(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("agg_kind", C.c_int32),
        ("arg_col", C.c_int32),
        ("default_col", C.c_int32),
        ("n", C.c_int64),
        ("ignore_nulls", C.c_int32),
        ("distinct", C.c_int32),
        ("frame", WindowFrame),
    ]


class WindowParams(C.Structure):
    _fields_ = [
        ("n_partition_cols", C.c_int32),
        ("partition_cols", C.c_int32 * MAX_SORT_KEYS),
        ("n_order_cols", C.c_int32),
        ("order_cols", C.c_int32 * MAX_SORT_KEYS),
        ("order_asc", C.c_int32 * MAX_SORT_KEYS),
        ("order_nulls_first", C.c_int32 * MAX_SORT_KEYS),
        ("n_funcs", C.c_int32),
        ("reserved", C.c_int32),
        ("funcs", WindowFunc * MAX_WINDOW_FUNCS),
    ]


MAX_JOIN_KEYS = 4


class JoinParams(C.Structure):
    _fields_ = [
        ("kind", C.c_int32),
        ("build_key_col", C.c_int32),
        ("probe_key_col", C.c_int32),
        ("n_build_cols", C.c_int32),
        ("expected_build_rows", C.c_int64),
        ("n_extra_keys", C.c_int32),
        ("extra_build_key_cols", C.c_int32 * (MAX_JOIN_KEYS - 1)),
        ("extra_probe_key_cols", C.c_int32 * (MAX_JOIN_KEYS - 1)),
    ]


RF_MAX_INLIST = 4096


class RuntimeFilterParams(C.Structure):
    _fields_ = [
        ("enable_inlist", C.c_int32),
        ("enable_bloom", C.c_int32),
        ("enable_min_max", C.c_int32),
        ("in_probe", C.c_int32),
        ("inlist_threshold", C.c_int64),
        ("bloom_threshold", C.c_int64),
        ("min_max_threshold", C.c_uint64),
        ("build_table_rows", C.c_int64),
        ("selectivity_threshold", C.c_uint64),
    ]


class RfPartInfo(C.Structure):
    _fields_ = [
        ("has_min_max", C.c_int32),
        ("has_inlist", C.c_int32),
        ("has_bloom", C.c_int32),
        ("key_dtype", C.c_int32),
        ("min", Scalar),
        ("max", Scalar),
        ("inlist_len", C.c_int64),
        ("bloom_bytes", C.c_int64),
    ]


class RfInfo(C.Structure):
    _fields_ = [
        ("n_parts", C.c_int32),
        ("in_probe", C.c_int32),
        ("build_rows", C.c_int64),
        ("apply_rows_checked", C.c_int64),
        ("apply_rows_rejected", C.c_int64),
        ("probe_rows_checked", C.c_int64),
        ("probe_rows_rejected", C.c_int64),
        ("parts", RfPartInfo * MAX_JOIN_KEYS),
    ]


EXPR_COLUMN, EXPR_CONST, EXPR_CAST, EXPR_CALL = 0, 1, 2, 3
(FN_PLUS, FN_MINUS, FN_MULTIPLY, FN_DIVIDE, FN_DIV, FN_MODULO, FN_NEGATE, FN_EQ, FN_NOTEQ, FN_LT, FN_LTE, FN_GT, FN_GTE, FN_AND, FN_OR, FN_NOT,
 FN_IS_NULL, FN_IS_NOT_NULL, FN_IF, FN_ASSUME_NOT_NULL) = range(20)
MAX_EXPR_NODES = 32
MAX_COMPUTED_COLS = 4


class ExprNode(C.Structure):
    _fields_ = [("kind", C.c_int32), ("func", C.c_int32), ("col", C.c_int32), ("cast_to", C.c_int32), ("try_cast", C.c_int32),
                ("reserved", C.c_int32), ("c", Scalar)]


class Expr(C.Structure):
    _fields_ = [("n_nodes", C.c_int32), ("reserved", C.c_int32), ("nodes", ExprNode * MAX_EXPR_NODES)]


# every function include/dbx.h declares (tests check the library exports each one)
EXPORTS = [
    "dbx_abi_version", "dbx_device_count", "dbx_last_error",
    "dbx_host_alloc", "dbx_host_free", "dbx_host_register", "dbx_host_unregister",
    "dbx_device_alloc", "dbx_device_free", "dbx_memcpy_h2d", "dbx_memcpy_d2h", "dbx_memcpy_d2d", "dbx_device_synchronize",
    "dbx_op_create", "dbx_op_destroy", "dbx_op_push", "dbx_op_finish", "dbx_op_pull", "dbx_block_release", "dbx_op_reset", "dbx_op_synchronize",
    "dbx_join_probe", "dbx_join_final_probe", "dbx_agg_final_merge_partial", "dbx_agg_partial_partition", "dbx_agg_final_merge_rows",
    "dbx_agg_exchange_create", "dbx_agg_exchange_local_buffer", "dbx_agg_exchange_connect", "dbx_agg_exchange_scatter",
    "dbx_agg_exchange_merge", "dbx_agg_exchange_destroy", "dbx_agg_exchange_last_error",
    "dbx_hash_partition",
    "dbx_eval_distance", "dbx_knn_create", "dbx_knn_search", "dbx_knn_destroy", "dbx_knn_last_error", "dbx_knn_last_gemm_ms", "dbx_knn_last_stats",
    "dbx_synth_fill", "dbx_kernel_launch_count", "dbx_op_last_kernel_ms", "dbx_op_kernel_ms", "dbx_op_stream",
    "dbx_op_inputs_consumed", "dbx_agg_exchange_phase_ms",
    "dbx_shuffle_create", "dbx_shuffle_local_buffer", "dbx_shuffle_connect", "dbx_shuffle_send", "dbx_shuffle_recv", "dbx_shuffle_last_ms",
    "dbx_shuffle_destroy", "dbx_shuffle_last_error",
    "dbx_block_take", "dbx_block_take_ranges", "dbx_block_scatter", "dbx_block_concat",
    "dbx_eval_scalar", "dbx_op_kernel_variant", "dbx_agg_jit_selftest", "dbx_eval_jit_selftest",
    "dbx_agg_partial_serialize", "dbx_agg_final_merge_serialized",
    "dbx_join_runtime_filter", "dbx_runtime_filter_info", "dbx_runtime_filter_export", "dbx_runtime_filter_apply",
    "dbx_runtime_filter_destroy", "dbx_op_create_computed", "dbx_agg_expr_jit_selftest", "dbx_op_create_join",
]
