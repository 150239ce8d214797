"""ctypes mirror of include/trino_gpu.h.

This is the Python stand-in for the Panama/JNI binding a Trino maintainer would add (INTEGRATION.md):
plain structs, plain pointers.  It loads trino_b200/libtrino_gpu.so and FAILS LOUDLY when the library
is missing — there is no CPU fallback anywhere in the product path.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libtrino_gpu.so")

# ---- enums (include/trino_gpu.h)
TGPU_OK = 0
ERR_INVALID_ARGUMENT, ERR_CUDA, ERR_INSUFFICIENT_RESOURCES, ERR_NUMERIC_VALUE_OUT_OF_RANGE = -1, -2, -3, -4
ERR_DIVISION_BY_ZERO, ERR_NOT_SUPPORTED, ERR_ILLEGAL_STATE, ERR_INVALID_CAST_ARGUMENT = -5, -6, -7, -8
ERR_INVALID_FUNCTION_ARGUMENT = -9

INT64, INT32, INT16, INT8, FLOAT64, UTF8, DICT32, RLE, INT128, FLOAT32 = 1, 2, 3, 4, 5, 7, 8, 9, 10, 11
COL_NULLS_BYTEMAP = 1
PARTITION_HASH_BUCKET, PARTITION_LOCAL = 0, 1
PAGE_DEVICE = 1

EX_MOV, EX_ADD, EX_SUB, EX_MUL, EX_DIV, EX_MOD, EX_NEG = 0, 1, 2, 3, 4, 5, 6
EX_EQ, EX_NE, EX_LT, EX_LE, EX_GT, EX_GE = 10, 11, 12, 13, 14, 15
EX_AND, EX_OR, EX_NOT, EX_IS_NULL, EX_IS_NOT_NULL, EX_BETWEEN = 20, 21, 22, 23, 24, 25
EX_CAST_BIGINT_TO_DOUBLE, EX_CAST_DOUBLE_TO_BIGINT, EX_IN, EX_LIKE = 30, 31, 40, 41
# DECIMAL casts: EX_CAST_TO_DECIMAL reads BIGINT or DECIMAL (its vtype), the other two read DECIMAL
EX_CAST_TO_DECIMAL, EX_CAST_DECIMAL_TO_BIGINT, EX_CAST_DECIMAL_TO_DOUBLE = 32, 33, 34
# string functions over a VARCHAR operand a: LENGTH gives BIGINT, the others VARCHAR; SUBSTR reads BIGINT b (and c, or OPND_NONE)
EX_LENGTH, EX_SUBSTR, EX_LTRIM, EX_RTRIM, EX_TRIM, EX_CONCAT = 50, 51, 52, 53, 54, 55
MAX_CONCAT_PIECES, MAX_VARCHAR_PROJECTIONS = 8, 8
# conditionals: EX_IF(a, b, c) is a ? b : c with BOOLEAN a and vtype the type of b, c and the result; EX_COALESCE(a, b)
EX_IF, EX_COALESCE = 60, 61
V_BIGINT, V_DOUBLE, V_BOOLEAN, V_VARCHAR, V_DECIMAL = 0, 1, 2, 3, 4
MAX_STRINGS, MAX_STRING_BYTES, MAX_LIKE_PATTERNS = 128, 4096, 8
OPND_NONE, OPND_COLUMN, OPND_TEMP, OPND_CONST, OPND_NULL = 0, 1, 2, 3, 4

AGG_COUNT_STAR, AGG_COUNT, AGG_SUM, AGG_AVG, AGG_MIN, AGG_MAX, AGG_SUM_DECIMAL, AGG_AVG_DECIMAL = 0, 1, 2, 3, 4, 5, 6, 7
AGG_VAR_SAMP, AGG_VAR_POP, AGG_STDDEV_SAMP, AGG_STDDEV_POP = 8, 9, 10, 11
STEP_SINGLE, STEP_PARTIAL, STEP_FINAL, STEP_INTERMEDIATE = 0, 1, 2, 3
JOIN_INNER, JOIN_PROBE_OUTER, JOIN_LOOKUP_OUTER, JOIN_FULL_OUTER = 0, 1, 2, 3
COMM_ID_BYTES = 128
IPC_HANDLE_BYTES = 64
NUM_ARENAS = 3


class Column(C.Structure):
    pass


Column._fields_ = [
    ("type", C.c_int32),
    ("flags", C.c_int32),
    ("length", C.c_int64),
    ("data", C.c_void_p),
    ("offsets", C.c_void_p),
    ("validity", C.c_void_p),
    ("dictionary", C.POINTER(Column)),
]


class Page(C.Structure):
    _fields_ = [
        ("num_columns", C.c_int32),
        ("flags", C.c_int32),
        ("num_rows", C.c_int64),
        ("columns", C.POINTER(Column)),
    ]


class Imm(C.Union):
    _fields_ = [("i64", C.c_int64), ("f64", C.c_double)]


class Operand(C.Structure):
    _fields_ = [("kind", C.c_int32), ("index", C.c_int32), ("imm", Imm)]


class ExprInsn(C.Structure):
    _fields_ = [("op", C.c_int32), ("vtype", C.c_int32), ("dst", C.c_int32), ("reserved", C.c_int32),
                ("a", Operand), ("b", Operand), ("c", Operand)]


class InList(C.Structure):
    _fields_ = [("count", C.c_int32), ("values", C.POINTER(C.c_int64))]


class Bytes(C.Structure):
    _fields_ = [("length", C.c_int32), ("data", C.c_void_p)]


class LikePattern(C.Structure):
    _fields_ = [("pattern", Bytes), ("escape", Bytes)]


class Projection(C.Structure):
    _fields_ = [("kind", C.c_int32), ("index", C.c_int32), ("vtype", C.c_int32)]


class DecimalType(C.Structure):
    _fields_ = [("precision", C.c_int8), ("scale", C.c_int8)]


class DecimalSignature(C.Structure):
    """the resolved DECIMAL types of one instruction's operands a, b, c and its result (zero where not DECIMAL)"""
    _fields_ = [("a", DecimalType), ("b", DecimalType), ("c", DecimalType), ("result", DecimalType)]


class ExprProgram(C.Structure):
    _fields_ = [
        ("num_insns", C.c_int32),
        ("insns", C.POINTER(ExprInsn)),
        ("filter_temp", C.c_int32),
        ("num_filter_insns", C.c_int32),
        ("num_projections", C.c_int32),
        ("projections", C.POINTER(Projection)),
        ("num_in_lists", C.c_int32),
        ("in_lists", C.POINTER(InList)),
        ("num_strings", C.c_int32),
        ("strings", C.POINTER(Bytes)),
        ("num_like_patterns", C.c_int32),
        ("like_patterns", C.POINTER(LikePattern)),
        ("decimal_signatures", C.POINTER(DecimalSignature)),
        ("num_decimal_constants", C.c_int32),
        ("decimal_constants", C.POINTER(C.c_int64)),
    ]


class AggFn(C.Structure):
    _fields_ = [("function", C.c_int32), ("input_channel", C.c_int32), ("mask_channel", C.c_int32), ("reserved", C.c_int32)]


class AggSpec(C.Structure):
    _fields_ = [
        ("num_keys", C.c_int32),
        ("key_channels", C.POINTER(C.c_int32)),
        ("step", C.c_int32),
        ("num_aggs", C.c_int32),
        ("aggs", C.POINTER(AggFn)),
        ("expected_groups", C.c_int64),
        ("max_partial_bytes", C.c_int64),
        ("pre", C.POINTER(ExprProgram)),
        ("num_global_group_ids", C.c_int32),
        ("global_group_ids", C.POINTER(C.c_int32)),
        ("group_id_key", C.c_int32),
        ("num_input_channels", C.c_int32),
        ("input_channel_types", C.POINTER(C.c_int32)),
        ("partial_aggregation_controller", C.c_void_p),
    ]


class JoinBuildSpec(C.Structure):
    _fields_ = [
        ("num_key_channels", C.c_int32),
        ("key_channels", C.POINTER(C.c_int32)),
        ("num_output_channels", C.c_int32),
        ("output_channels", C.POINTER(C.c_int32)),
        ("expected_positions", C.c_int64),
    ]


class JoinProbeSpec(C.Structure):
    _fields_ = [
        ("join_type", C.c_int32),
        ("output_single_match", C.c_int32),
        ("num_key_channels", C.c_int32),
        ("key_channels", C.POINTER(C.c_int32)),
        ("num_output_channels", C.c_int32),
        ("output_channels", C.POINTER(C.c_int32)),
    ]


class PartitionSpec(C.Structure):
    _fields_ = [
        ("num_key_channels", C.c_int32),
        ("key_channels", C.POINTER(C.c_int32)),
        ("bucket_count", C.c_int32),
        ("bucket_to_partition", C.POINTER(C.c_int32)),
        ("null_channel", C.c_int32),
        ("replicates_any_row", C.c_int32),
        ("partition_function", C.c_int32),
        ("key_constants", C.c_void_p),
    ]


class Domain(C.Structure):
    _fields_ = [("channel", C.c_int32), ("null_allowed", C.c_int32), ("kind", C.c_int32), ("num_values", C.c_int32),
                ("min", C.c_int64), ("max", C.c_int64), ("values", C.POINTER(C.c_int64))]


DOMAIN_ALL, DOMAIN_NONE, DOMAIN_RANGE, DOMAIN_DISCRETE = 0, 1, 2, 3

VP = C.c_void_p
PP = C.POINTER(Page)

# name -> (restype, argtypes); every symbol include/trino_gpu.h declares
SIGNATURES = {
    "tgpu_ctx_create": (C.c_int, [C.c_int, C.POINTER(VP)]),
    "tgpu_ctx_destroy": (None, [VP]),
    "tgpu_last_error": (C.c_char_p, [VP]),
    "tgpu_status_name": (C.c_char_p, [C.c_int]),
    "tgpu_ctx_synchronize": (C.c_int, [VP]),
    "tgpu_ctx_stream": (VP, [VP]),
    "tgpu_ctx_kernel_launches": (C.c_int64, [VP]),
    "tgpu_device_count": (C.c_int, []),
    "tgpu_ctx_set_l2_fetch_granularity": (C.c_int, [VP, C.c_int]),
    "tgpu_ctx_get_l2_fetch_granularity": (C.c_int, [VP, C.POINTER(C.c_int)]),
    "tgpu_malloc": (C.c_int, [VP, C.c_size_t, C.POINTER(VP)]),
    "tgpu_free": (C.c_int, [VP, VP]),
    "tgpu_memcpy_h2d": (C.c_int, [VP, VP, VP, C.c_size_t]),
    "tgpu_memcpy_d2h": (C.c_int, [VP, VP, VP, C.c_size_t]),
    "tgpu_host_alloc_pinned": (C.c_int, [C.c_size_t, C.POINTER(VP)]),
    "tgpu_host_free_pinned": (C.c_int, [VP]),
    "tgpu_flush_l2": (C.c_int, [VP]),
    "tgpu_timer_start": (C.c_int, [VP]),
    "tgpu_timer_stop_ms": (C.c_int, [VP, C.POINTER(C.c_float)]),
    "tgpu_ctx_last_kernel_ms": (C.c_int, [VP, C.POINTER(C.c_float)]),
    "tgpu_filter_project_create": (C.c_int, [VP, C.POINTER(ExprProgram), C.POINTER(VP)]),
    "tgpu_agg_create": (C.c_int, [VP, C.POINTER(AggSpec), C.POINTER(VP)]),
    "tgpu_aggregation_create": (C.c_int, [VP, C.POINTER(AggSpec), C.POINTER(VP)]),
    "tgpu_agg_group_count": (C.c_int, [VP, C.POINTER(C.c_int64)]),
    "tgpu_agg_rows_with_partial_aggregation_disabled": (C.c_int, [VP, C.POINTER(C.c_int64)]),
    "tgpu_partial_agg_controller_create": (C.c_int, [C.c_int64, C.c_double, C.POINTER(VP)]),
    "tgpu_partial_agg_controller_destroy": (None, [VP]),
    "tgpu_partial_agg_controller_is_disabled": (C.c_int, [VP]),
    "tgpu_partial_agg_controller_on_flush": (None, [VP, C.c_int64, C.c_int64, C.c_int64]),
    "tgpu_jit_selftest_filter_project": (C.c_int, [C.POINTER(ExprProgram), C.POINTER(C.c_int32), C.c_int32, C.c_uint32, C.POINTER(C.c_int64), C.c_char_p, C.c_int64]),
    "tgpu_jit_selftest_join_filter": (C.c_int, [C.POINTER(ExprProgram), C.c_int32, C.POINTER(C.c_int32), C.c_int32, C.c_uint32, C.POINTER(C.c_int64), C.c_char_p,
                                                C.c_int64]),
    "tgpu_jit_selftest_agg": (C.c_int, [C.POINTER(AggSpec), C.POINTER(C.c_int32), C.c_int32, C.c_uint32, C.POINTER(C.c_int64), C.c_char_p, C.c_int64]),
    "tgpu_groupby_hash_create": (C.c_int, [VP, C.c_int32, C.POINTER(C.c_int32), C.c_int64, C.POINTER(VP)]),
    "tgpu_groupby_hash_get_group_ids": (C.c_int, [VP, PP, VP]),
    "tgpu_join_build_create": (C.c_int, [VP, C.POINTER(JoinBuildSpec), C.POINTER(VP)]),
    "tgpu_join_build_create_filtered": (C.c_int, [VP, C.POINTER(JoinBuildSpec), C.POINTER(ExprProgram), C.c_int32, C.POINTER(VP)]),
    "tgpu_join_build_get_lookup": (C.c_int, [VP, C.POINTER(VP)]),
    "tgpu_lookup_release": (None, [VP]),
    "tgpu_lookup_position_count": (C.c_int64, [VP]),
    "tgpu_lookup_memory_bytes": (C.c_int64, [VP]),
    "tgpu_lookup_has_duplicates": (C.c_int, [VP]),
    "tgpu_join_probe_create": (C.c_int, [VP, C.POINTER(JoinProbeSpec), VP, C.POINTER(VP)]),
    "tgpu_lookup_get_join_positions": (C.c_int, [VP, VP, PP, VP]),
    "tgpu_lookup_copy_position_links": (C.c_int, [VP, VP, VP]),
    "tgpu_partition_create": (C.c_int, [VP, C.POINTER(PartitionSpec), C.POINTER(VP)]),
    "tgpu_partition_last_output_partition": (C.c_int, [VP, C.POINTER(C.c_int32)]),
    "tgpu_partition_get_partitions": (C.c_int, [VP, PP, VP]),
    "tgpu_comm_get_unique_id": (C.c_int, [VP]),
    "tgpu_comm_init": (C.c_int, [VP, VP, C.c_int, C.c_int]),
    "tgpu_comm_destroy": (C.c_int, [VP]),
    "tgpu_comm_arena_create": (C.c_int, [VP, C.c_size_t, VP]),
    "tgpu_comm_arena_open": (C.c_int, [VP, VP]),
    "tgpu_exchange_partitioned": (C.c_int, [VP, VP, PP, C.POINTER(PP)]),
    "tgpu_exchange_partitioned_fenced": (C.c_int, [VP, VP, PP, VP, C.POINTER(PP)]),
    "tgpu_exchange_broadcast": (C.c_int, [VP, PP, C.POINTER(PP)]),
    "tgpu_exchange_begin": (C.c_int, [VP, VP, PP, C.POINTER(VP)]),
    "tgpu_exchange_end": (C.c_int, [VP, VP, C.POINTER(PP)]),
    "tgpu_op_needs_input": (C.c_int, [VP, C.POINTER(C.c_int)]),
    "tgpu_op_add_input": (C.c_int, [VP, PP]),
    "tgpu_op_get_output": (C.c_int, [VP, C.POINTER(PP)]),
    "tgpu_op_finish": (C.c_int, [VP]),
    "tgpu_op_is_finished": (C.c_int, [VP, C.POINTER(C.c_int)]),
    "tgpu_op_memory_bytes": (C.c_int64, [VP]),
    "tgpu_op_close": (None, [VP]),
    "tgpu_page_release": (None, [VP, PP]),
    "tgpu_page_copy_to_host": (C.c_int, [VP, PP, PP]),
    "tgpu_page_utf8_bytes": (C.c_int64, [VP, PP, C.c_int32]),
    "tgpu_join_probe_set_passthrough_by_reference": (C.c_int, [VP, C.c_int32]),
    "tgpu_join_outer_create": (C.c_int, [VP, VP, C.POINTER(C.c_int32), C.c_int32, C.POINTER(VP)]),
    "tgpu_semi_join_create": (C.c_int, [VP, VP, C.c_int32, C.POINTER(VP)]),
    "tgpu_lookup_key_domain": (C.c_int, [VP, VP, C.c_int64, C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "tgpu_page_serialized_size_bound": (C.c_int64, [PP]),
    "tgpu_page_serialize": (C.c_int, [VP, PP, VP, C.c_int64, C.POINTER(C.c_int64)]),
    "tgpu_page_deserialize": (C.c_int, [VP, VP, C.c_int64, C.POINTER(C.c_int32), C.c_int32, C.POINTER(PP)]),
    "tgpu_page_passthrough_channel": (C.c_int, [PP, C.c_int32, C.POINTER(C.c_int32)]),
    "tgpu_synth_orders_keys": (C.c_int, [VP, C.c_int64, C.c_int64, C.c_int64, C.c_uint64, C.c_int, VP]),
    "tgpu_synth_lineitem_rows": (C.c_int64, [C.c_int64]),
    "tgpu_synth_lineitem_keys": (C.c_int, [VP, C.c_int64, C.c_int64, C.c_int64, C.c_uint64, C.c_int, VP]),
    "tgpu_synth_lineitem_q1": (C.c_int, [VP, C.c_int64, C.c_int64, C.c_uint64, VP, VP, VP, VP, VP, VP, VP]),
    "tgpu_column_sum": (C.c_int, [VP, VP, C.c_int64, VP]),
    "tgpu_dynamic_filter_create": (C.c_int, [VP, VP, C.c_int32, C.c_double, VP]),
    "tgpu_dynamic_filter_update": (C.c_int, [VP, VP, C.c_int32]),
    "tgpu_dynamic_filter_is_effective": (C.c_int, [VP, C.c_int32, VP]),
    "tgpu_synth_orders_custkeys": (C.c_int, [VP, C.c_int64, C.c_int64, C.c_int64, C.c_uint64, C.c_int, C.c_int64, C.c_uint64, VP]),
    "tgpu_synth_sequence": (C.c_int, [VP, C.c_int64, C.c_int64, VP]),
    "tgpu_synth_sequence32": (C.c_int, [VP, C.c_int32, C.c_int64, VP]),
    "tgpu_synth_store_sales": (C.c_int, [VP, C.c_int64, C.c_int64, C.c_uint64, VP, VP, VP, VP, VP, VP, VP, VP]),
}

_lib = None


class TrinoGpuError(RuntimeError):
    """A negative tgpu_status; .code is the status, .name the Trino StandardErrorCode name."""

    def __init__(self, code, name, message):
        super().__init__(f"{name} ({code}): {message}")
        self.code = code
        self.name = name


def load_library(path=None):
    """dlopen libtrino_gpu.so and bind every declared symbol.  Raises if the library is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.exists(p):
        raise RuntimeError(
            f"{p} is missing: build it with `python -m trino_b200._build` (nvcc, sm_90a). "
            "trino_b200 has no CPU fallback.")
    lib = C.CDLL(p, mode=C.RTLD_GLOBAL)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)   # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if path is None:
        _lib = lib
    return lib
