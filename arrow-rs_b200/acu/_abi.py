"""ctypes mirror of include/arrow_cuda.h (the C ABI) — struct layouts, enums, prototypes.

The same struct types are used by the CPU oracle (oracle/liboracle.so, test infrastructure
only) so that tests can hand both sides identical descriptors.
"""
import ctypes as C
import os

REPO = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
LIB_PATH = os.path.join(REPO, "arrow-rs_b200", "libarrow_cuda.so")

# acu_status
OK = 0
ERR_INVALID_ARGUMENT = 1
ERR_COMPUTE = 2
ERR_ARITHMETIC_OVERFLOW = 3
ERR_DIVIDE_BY_ZERO = 4
ERR_OFFSET_OVERFLOW = 5
ERR_CAST = 6
ERR_NOT_YET_IMPLEMENTED = 7
ERR_PANIC_OUT_OF_BOUNDS = 8
ERR_CUDA = 100
ERR_NCCL = 101
ERR_OUT_OF_MEMORY = 102

# acu_dtype
I8, I16, I32, I64, U8, U16, U32, U64, F32, F64 = range(10)
DTYPE_NAMES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]
DTYPE_SIZE = [1, 2, 4, 8, 1, 2, 4, 8, 4, 8]
# Decimal128's native (16-byte two's complement); accepted only by acu_cmp / acu_filter_plan_create_cmp / acu_neg, so it
# stays out of the per-dtype lists above
I128 = 10

# acu_arith_op (arrow-arith/src/numeric.rs:181-190)
ADD_WRAPPING, ADD, SUB_WRAPPING, SUB, MUL_WRAPPING, MUL, DIV, REM = range(8)
# acu_cmp_op (arrow-ord/src/cmp.rs:40-60)
EQ, NEQ, LT, LT_EQ, GT, GT_EQ, DISTINCT, NOT_DISTINCT = range(8)
# acu_agg_op
SUM, MIN, MAX, PRODUCT, BIT_AND, BIT_OR, BIT_XOR = range(7)
# acu_bitwise_op (arrow-arith/src/bitwise.rs)
BITWISE_AND, BITWISE_OR, BITWISE_XOR, BITWISE_AND_NOT, BITWISE_SHIFT_LEFT, BITWISE_SHIFT_RIGHT, BITWISE_NOT = range(7)
# acu_like_op (arrow-string/src/like.rs `enum Op`)
LIKE, NLIKE, ILIKE, NILIKE, CONTAINS, STARTS_WITH, ENDS_WITH, EQ_IGNORE_ASCII_CASE = range(8)
# acu_length_op (arrow-string/src/length.rs length / bit_length)
LENGTH, BIT_LENGTH = range(2)
# acu_filter_strategy
FILTER_NONE, FILTER_ALL, FILTER_INDEX, FILTER_SLICES = range(4)

NCCL_UNIQUE_ID_BYTES = 128
# acu_kernel_class
K_ARITH, K_CMP, K_CAST, K_FILTER, K_FILTER_PLAN, K_TAKE, K_REDUCE, K_BYTES = range(8)
KERNEL_CLASS_NAMES = ["arith", "cmp", "cast", "filter", "filter_plan", "take", "reduce", "bytes"]


class ErrorDetail(C.Structure):
    _fields_ = [
        ("status", C.c_int32),
        ("cuda_error", C.c_int32),
        ("index", C.c_int64),
        ("lhs_bits", C.c_uint64),
        ("rhs_bits", C.c_uint64),
        ("len", C.c_uint64),
        ("message", C.c_char * 256),
    ]


class Array(C.Structure):
    _fields_ = [
        ("values", C.c_void_p),
        ("values_offset", C.c_int64),
        ("validity", C.c_void_p),
        ("validity_offset", C.c_int64),
        ("len", C.c_int64),
        ("null_count", C.c_int64),
        ("is_scalar", C.c_int32),
        ("reserved", C.c_int32),
    ]


class ArrayOut(C.Structure):
    _fields_ = [
        ("values", C.c_void_p),
        ("validity", C.c_void_p),
        ("len", C.c_int64),
        ("null_count", C.c_int64),
        ("has_validity", C.c_int32),
        ("reserved", C.c_int32),
    ]


class DecimalType(C.Structure):
    """acu_decimal_type: DataType::Decimal32 / 64 / 128(precision, scale) as byte_width 4 / 8 / 16."""
    _fields_ = [("byte_width", C.c_int32), ("precision", C.c_uint8), ("scale", C.c_int8), ("reserved", C.c_uint8 * 2)]


class BytesArray(C.Structure):
    """acu_bytes_array: a Utf8 / Binary operand of acu_cmp_bytes."""
    _fields_ = [("offsets", C.c_void_p), ("data", C.c_void_p), ("nulls", Array)]


class ViewArray(C.Structure):
    """acu_view_array: a Utf8View / BinaryView operand of acu_cmp_byte_view."""
    _fields_ = [("views", C.c_void_p), ("buffers", C.POINTER(C.c_void_p)), ("n_buffers", C.c_int32), ("reserved", C.c_int32), ("nulls", Array)]


LIST, LARGE_LIST, FIXED_SIZE_LIST = range(3)


class ListArray(C.Structure):
    """acu_list_array: one level of a List / LargeList / FixedSizeList column (the child is described separately)."""
    _fields_ = [("kind", C.c_int32), ("list_size", C.c_int32), ("offsets", C.c_void_p), ("nulls", Array), ("child_len", C.c_int64)]


class RunArray(C.Structure):
    """acu_run_array: the run ends of a RunEndEncoded column and its logical slice (the values child is separate)."""
    _fields_ = [("run_end_dtype", C.c_int32), ("reserved", C.c_int32), ("run_ends", C.c_void_p), ("n_runs", C.c_int64),
                ("offset", C.c_int64), ("len", C.c_int64)]


RUN_VALUES_FIXED, RUN_VALUES_BOOLEAN, RUN_VALUES_BYTES, RUN_VALUES_VIEW, RUN_VALUES_NESTED = range(5)


class RunValues(C.Structure):
    """acu_run_values: the values child of a RunEndEncoded column as take's run merge compares it."""
    _fields_ = [("kind", C.c_int32), ("width", C.c_int32), ("array", Array), ("bytes", BytesArray), ("view", ViewArray)]


UNION_SPARSE, UNION_DENSE = range(2)
ZIP_BUFFERS_NONE, ZIP_BUFFERS_TRUTHY, ZIP_BUFFERS_FALSY, ZIP_BUFFERS_BOTH = range(4)  # acu_zip_buffers
UNION_MAX_FIELDS = 128


class UnionArray(C.Structure):
    """acu_union_array: one level of a sparse / dense Union column (the children are described separately)."""
    _fields_ = [("mode", C.c_int32), ("n_fields", C.c_int32), ("field_type_ids", C.c_void_p), ("type_ids", C.c_void_p),
                ("offsets", C.c_void_p), ("len", C.c_int64)]


COL_PRIMITIVE, COL_BOOLEAN, COL_BYTES, COL_FIXED_SIZE_BINARY = range(4)
BOOL_AND, BOOL_OR, BOOL_AND_NOT, BOOL_AND_KLEENE, BOOL_OR_KLEENE, BOOL_NOT, BOOL_IS_NULL, BOOL_IS_NOT_NULL = range(8)
MAX_BATCH_COLUMNS = 64


class Column(C.Structure):
    """acu_column: one column of a RecordBatch (include/arrow_cuda.h)."""
    _fields_ = [
        ("kind", C.c_int32),
        ("width", C.c_int32),
        ("array", Array),
        ("data", C.c_void_p),
    ]


class ColumnOut(C.Structure):
    _fields_ = [
        ("array", ArrayOut),
        ("data", C.c_void_p),
        ("data_capacity", C.c_int64),
        ("data_len", C.c_int64),
    ]


# ---- Arrow C Data Interface / C Device Data Interface (include/arrow_cuda.h) ----------------------
DEVICE_CPU, DEVICE_CUDA, DEVICE_CUDA_HOST = 1, 2, 3


class ArrowSchema(C.Structure):
    pass


ArrowSchema._fields_ = [
    ("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64), ("n_children", C.c_int64),
    ("children", C.POINTER(C.POINTER(ArrowSchema))), ("dictionary", C.POINTER(ArrowSchema)),
    ("release", C.CFUNCTYPE(None, C.POINTER(ArrowSchema))), ("private_data", C.c_void_p),
]


class ArrowArray(C.Structure):
    pass


ArrowArray._fields_ = [
    ("length", C.c_int64), ("null_count", C.c_int64), ("offset", C.c_int64), ("n_buffers", C.c_int64), ("n_children", C.c_int64),
    ("buffers", C.POINTER(C.c_void_p)), ("children", C.POINTER(C.POINTER(ArrowArray))), ("dictionary", C.POINTER(ArrowArray)),
    ("release", C.CFUNCTYPE(None, C.POINTER(ArrowArray))), ("private_data", C.c_void_p),
]


class ArrowDeviceArray(C.Structure):
    _fields_ = [("array", ArrowArray), ("device_id", C.c_int64), ("device_type", C.c_int32), ("sync_event", C.c_void_p),
                ("reserved", C.c_int64 * 3)]


RELEASE_OWNER = C.CFUNCTYPE(None, C.c_void_p)


def bitmap_bytes(n):
    return ((n + 63) // 64) * 8


P = C.POINTER
vp, i32, i64, u64, f32, f64 = C.c_void_p, C.c_int32, C.c_int64, C.c_uint64, C.c_float, C.c_double

# name -> (restype, argtypes). Every symbol include/arrow_cuda.h declares.
PROTOTYPES = {
    "acu_abi_version": (i32, []),
    "acu_abi_sizeof": (i32, [i32]),
    "acu_ctx_create": (i32, [i32, P(vp)]),
    "acu_ctx_destroy": (None, [vp]),
    "acu_ctx_sync": (i32, [vp]),
    "acu_last_error": (P(ErrorDetail), [vp]),
    "acu_launch_count": (i64, [vp]),
    "acu_device_sm_count": (i32, [vp]),
    "acu_malloc": (i32, [vp, C.c_size_t, P(vp)]),
    "acu_free": (i32, [vp, vp]),
    "acu_memset": (i32, [vp, vp, i32, C.c_size_t]),
    "acu_memcpy_h2d": (i32, [vp, vp, vp, C.c_size_t]),
    "acu_memcpy_d2h": (i32, [vp, vp, vp, C.c_size_t]),
    "acu_memcpy_d2d": (i32, [vp, vp, vp, C.c_size_t]),
    "acu_memcpy_h2d_async": (i32, [vp, vp, vp, C.c_size_t]),
    "acu_memcpy_d2h_async": (i32, [vp, vp, vp, C.c_size_t]),
    "acu_host_alloc": (i32, [vp, C.c_size_t, P(vp)]),
    "acu_host_free": (i32, [vp, vp]),
    "acu_bytes_allocated": (i64, [vp]),
    "acu_timer_start": (i32, [vp]),
    "acu_timer_stop": (i32, [vp, P(f32)]),
    "acu_timer_start_slot": (i32, [vp, i32]),
    "acu_timer_stop_slot": (i32, [vp, i32, P(f32)]),
    "acu_kernel_stats": (i32, [vp, i32, P(f64), P(i64)]),
    "acu_kernel_stats_reset": (i32, [vp]),
    "acu_bitmap_count": (i32, [vp, vp, i64, vp, i64, i64, P(i64)]),
    "acu_filter_plan_create": (i32, [vp, P(Array), P(vp)]),
    "acu_filter_plan_create_cmp": (i32, [vp, i32, i32, P(Array), P(Array), P(vp)]),
    "acu_nullif": (i32, [vp, P(Array), P(Array), P(ArrayOut)]),
    "acu_zip": (i32, [vp, i32, P(Array), P(Array), P(Array), P(ArrayOut)]),
    "acu_zip_bytes": (i32, [vp, i32, P(Array), P(BytesArray), P(BytesArray), vp, vp, i64, P(i64), P(ArrayOut)]),
    "acu_zip_byte_view": (i32, [vp, P(Array), P(ViewArray), P(ViewArray), vp, P(ArrayOut), P(i32)]),
    "acu_zip_boolean": (i32, [vp, P(Array), P(Array), P(Array), P(ArrayOut)]),
    "acu_zip_fixed_size_binary": (i32, [vp, i32, P(Array), P(Array), P(Array), P(ArrayOut)]),
    "acu_filter_plan_destroy": (None, [vp, vp]),
    "acu_filter_plan_indices": (i32, [vp, vp, i32, vp]),
    "acu_filter_plan_count": (i64, [vp]),
    "acu_filter_plan_len": (i64, [vp]),
    "acu_filter_plan_strategy": (i32, [vp]),
    "acu_filter_primitive": (i32, [vp, vp, i32, P(Array), P(ArrayOut)]),
    "acu_filter_boolean": (i32, [vp, vp, P(Array), P(ArrayOut)]),
    "acu_filter_bytes": (i32, [vp, vp, i32, vp, vp, P(Array), vp, vp, i64, P(i64), P(ArrayOut)]),
    "acu_take_primitive": (i32, [vp, i32, P(Array), P(Array), i32, i32, P(ArrayOut)]),
    "acu_take_boolean": (i32, [vp, P(Array), P(Array), i32, i32, P(ArrayOut)]),
    "acu_take_bytes": (i32, [vp, i32, vp, vp, P(Array), P(Array), i32, i32, vp, vp, i64, P(i64), P(ArrayOut)]),
    "acu_take_bytes_extend": (i32, [vp, i32, vp, vp, P(Array), P(Array), i32, vp, vp, i64, P(i64), P(ArrayOut)]),
    "acu_filter_list": (i32, [vp, vp, P(ListArray), vp, P(ArrayOut), P(vp)]),
    "acu_take_list": (i32, [vp, P(ListArray), P(Array), i32, i32, i32, vp, P(ArrayOut), i32, vp, i64, P(i64), P(ArrayOut)]),
    "acu_filter_run_end": (i32, [vp, vp, P(RunArray), vp, P(i64), P(i64), P(vp)]),
    "acu_take_run_end": (i32, [vp, P(RunArray), P(RunValues), P(Array), i32, i32, vp, vp, P(i64)]),
    "acu_filter_nulls": (i32, [vp, vp, P(Array), P(ArrayOut)]),
    "acu_take_nulls": (i32, [vp, P(Array), P(Array), i32, i32, P(ArrayOut)]),
    "acu_filter_union": (i32, [vp, vp, P(UnionArray), vp, vp, vp, P(i64)]),
    "acu_take_union": (i32, [vp, P(UnionArray), P(Array), i32, i32, vp, vp, vp, P(i64)]),
    "acu_filter_fixed_size_binary": (i32, [vp, vp, i32, P(Array), P(ArrayOut)]),
    "acu_take_fixed_size_binary": (i32, [vp, i32, P(Array), P(Array), i32, i32, P(ArrayOut)]),
    "acu_arith": (i32, [vp, i32, i32, P(Array), P(Array), P(ArrayOut)]),
    "acu_bitwise": (i32, [vp, i32, i32, P(Array), P(Array), P(ArrayOut)]),
    "acu_neg": (i32, [vp, i32, i32, P(Array), P(ArrayOut)]),
    "acu_decimal_arith": (i32, [vp, i32, P(DecimalType), P(Array), P(DecimalType), P(Array), P(DecimalType), P(ArrayOut)]),
    "acu_cmp": (i32, [vp, i32, i32, P(Array), P(Array), P(ArrayOut)]),
    "acu_cmp_bytes": (i32, [vp, i32, i32, P(BytesArray), P(BytesArray), P(ArrayOut)]),
    "acu_cmp_byte_view": (i32, [vp, i32, P(ViewArray), P(ViewArray), P(ArrayOut)]),
    "acu_like_bytes": (i32, [vp, i32, i32, i32, P(BytesArray), P(BytesArray), P(ArrayOut)]),
    "acu_like_byte_view": (i32, [vp, i32, i32, P(ViewArray), P(ViewArray), P(ArrayOut)]),
    "acu_length_bytes": (i32, [vp, i32, i32, P(BytesArray), P(ArrayOut)]),
    "acu_length_byte_view": (i32, [vp, i32, P(ViewArray), P(ArrayOut)]),
    "acu_length_fixed_size_binary": (i32, [vp, i32, i32, P(Array), P(ArrayOut)]),
    "acu_substring_bytes": (i32, [vp, i32, i32, i64, i32, u64, P(BytesArray), i64, vp, vp, i64, P(i64), P(ArrayOut)]),
    "acu_substring_by_char": (i32, [vp, i32, i64, i32, u64, P(BytesArray), vp, vp, i64, P(i64), P(ArrayOut)]),
    "acu_substring_byte_view": (i32, [vp, i32, i64, i32, u64, P(ViewArray), vp, P(ArrayOut)]),
    "acu_substring_fixed_size_binary": (i32, [vp, i32, i64, i32, u64, P(Array), P(i32), P(ArrayOut)]),
    "acu_concat_elements_bytes": (i32, [vp, i32, P(BytesArray), P(BytesArray), vp, vp, i64, P(i64), P(ArrayOut)]),
    "acu_concat_elements_bytes_many": (i32, [vp, i32, i32, P(BytesArray), vp, vp, i64, P(i64), P(ArrayOut)]),
    "acu_concat_elements_byte_view": (i32, [vp, P(ViewArray), P(ViewArray), vp, vp, i64, P(i64), P(ArrayOut)]),
    "acu_concat_elements_fixed_size_binary": (i32, [vp, i32, P(Array), i32, P(Array), P(i32), P(ArrayOut)]),
    "acu_cast_numeric": (i32, [vp, i32, i32, i32, P(Array), P(ArrayOut)]),
    "acu_cast_decimal": (i32, [vp, P(DecimalType), P(DecimalType), i32, P(Array), P(ArrayOut)]),
    "acu_cast_to_decimal": (i32, [vp, i32, P(DecimalType), i32, P(Array), P(ArrayOut)]),
    "acu_cast_from_decimal": (i32, [vp, P(DecimalType), i32, i32, P(Array), P(ArrayOut)]),
    "acu_boolean": (i32, [vp, i32, P(Array), P(Array), P(ArrayOut)]),
    "acu_aggregate": (i32, [vp, i32, i32, P(Array), P(u64), P(i64)]),
    "acu_aggregate_i128": (i32, [vp, i32, P(Array), P(u64), P(i64)]),
    "acu_sum_checked": (i32, [vp, i32, P(Array), P(u64), P(i64)]),
    "acu_product_checked": (i32, [vp, i32, P(Array), P(u64), P(i64)]),
    "acu_aggregate_bytes": (i32, [vp, i32, i32, P(BytesArray), P(i64), P(i64)]),
    "acu_aggregate_byte_view": (i32, [vp, i32, P(ViewArray), P(i64), P(i64)]),
    "acu_aggregate_fixed_size_binary": (i32, [vp, i32, i32, P(Array), P(i64), P(i64)]),
    "acu_aggregate_boolean": (i32, [vp, i32, P(Array), P(i32), P(i64)]),
    "acu_filter_record_batch": (i32, [vp, vp, i32, P(Column), P(ColumnOut)]),
    "acu_take_record_batch": (i32, [vp, i32, P(Column), P(Array), i32, i32, P(ColumnOut)]),
    "acu_aggregate_columns": (i32, [vp, i32, P(i32), P(i32), P(Array), P(u64), P(i64)]),
    "acu_ipc_stream_open": (i32, [vp, vp, i64, P(vp), P(i32)]),
    "acu_ipc_stream_field": (i32, [vp, i32, P(i32), P(i32), P(i32), P(i32), P(C.c_char_p)]),
    "acu_ipc_stream_next": (i32, [vp, vp, P(Column), P(i64)]),
    "acu_ipc_stream_close": (None, [vp, vp]),
    "acu_concat": (i32, [vp, i32, P(Column), P(ColumnOut)]),
    "acu_concat_batches": (i32, [vp, i32, i32, P(Column), P(ColumnOut), P(i64)]),
    "acu_bitmap_copy": (i32, [vp, vp, i64, vp, i64, i64, P(i64)]),
    "acu_bitmap_fill": (i32, [vp, vp, i64, i64, i32]),
    "acu_offsets_append": (i32, [vp, i32, vp, i64, i64, i64, vp, i64, P(i64), P(i64)]),
    "acu_export_column": (i32, [vp, P(Column), i32, i32, RELEASE_OWNER, vp, P(ArrowDeviceArray), P(ArrowSchema)]),
    "acu_import_column": (i32, [vp, P(ArrowDeviceArray), P(ArrowSchema), P(Column), P(i32)]),
    "acu_comm_get_unique_id": (i32, [vp]),
    "acu_comm_init": (i32, [vp, vp, i32, i32]),
    "acu_comm_destroy": (i32, [vp]),
    "acu_view_bytes_used": (i32, [vp, vp, i64, P(i64)]),
    "acu_view_fit": (i32, [vp, vp, i64, i64, P(i64), P(i64)]),
    "acu_view_copy_strings": (i32, [vp, vp, i64, P(vp), i32, C.c_uint32, vp, i64, i64, vp, P(i64)]),
    "acu_view_rebase": (i32, [vp, vp, i64, C.c_uint32, vp]),
    "acu_filter_plan_slices": (i32, [vp, vp, vp, i64, P(i64)]),
    "acu_async_begin": (i32, [vp]),
    "acu_results_fetch": (i32, [vp]),
    "acu_async_active": (i32, [vp]),
    "acu_comm_allreduce_aggregates": (i32, [vp, i32, i32, P(u64), P(i64), i32]),
    "acu_comm_allreduce_i64_sum": (i32, [vp, P(i64), i32]),
    "acu_aggregate_allreduce": (i32, [vp, i32, i32, P(Array), P(u64), P(i64)]),
}

_lib = None


# Synthetic-input generators of the benchmarks and tests: libarrow_cuda_testgen.so (include/arrow_cuda_testgen.h), test support
# only. Bound onto the same handle object so that callers keep writing lib.acu_generate_*.
TESTGEN_LIB_PATH = os.path.join(os.path.dirname(LIB_PATH), "libarrow_cuda_testgen.so")
TESTGEN_PROTOTYPES = {
    "acu_generate_values": (i32, [vp, i32, u64, i64, u64, vp, i64]),
    "acu_generate_bits": (i32, [vp, u64, i64, f64, vp, i64]),
}


def load_library(path=None):
    """Load libarrow_cuda.so and bind every prototype. Fails loudly if the CUDA extension
    has not been built — there is no CPU fallback behind this ABI."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    path = path or os.environ.get("ACU_LIB_PATH") or LIB_PATH  # ACU_LIB_PATH: tuning builds of the same ABI
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} is missing: build the CUDA extension first (python -c 'import __graft_entry__ as g; g.build()'). "
            "arrow-cuda has no CPU fallback.")
    lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.acu_abi_version() != 1:
        raise RuntimeError("libarrow_cuda.so ABI version mismatch")
    if os.path.exists(TESTGEN_LIB_PATH):
        gen = C.CDLL(TESTGEN_LIB_PATH, mode=C.RTLD_GLOBAL)
        for name, (res, args) in TESTGEN_PROTOTYPES.items():
            fn = getattr(gen, name)
            fn.restype = res
            fn.argtypes = args
            setattr(lib, name, fn)
    _lib = lib
    return lib
