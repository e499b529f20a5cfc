//! 1:1 declarations of `include/arrow_cuda.h`. Uncompiled in this repository (no rustc here):
//! kept to plain `#[repr(C)]` structs and `extern "C"` prototypes so it is correct by inspection.
#![allow(non_camel_case_types)]
use std::os::raw::{c_char, c_void};

pub type acu_status = i32;
pub const ACU_OK: acu_status = 0;
pub const ACU_ERR_INVALID_ARGUMENT: acu_status = 1;
pub const ACU_ERR_COMPUTE: acu_status = 2;
pub const ACU_ERR_ARITHMETIC_OVERFLOW: acu_status = 3;
pub const ACU_ERR_DIVIDE_BY_ZERO: acu_status = 4;
pub const ACU_ERR_OFFSET_OVERFLOW: acu_status = 5;
pub const ACU_ERR_CAST: acu_status = 6;
pub const ACU_ERR_NOT_YET_IMPLEMENTED: acu_status = 7;
pub const ACU_ERR_PANIC_OUT_OF_BOUNDS: acu_status = 8;
pub const ACU_ERR_IPC: acu_status = 9;
pub const ACU_ERR_PARSE: acu_status = 10;
pub const ACU_ERR_CUDA: acu_status = 100;
pub const ACU_ERR_NCCL: acu_status = 101;
pub const ACU_ERR_OUT_OF_MEMORY: acu_status = 102;

// acu_dtype (include/arrow_cuda.h): Int8..Int64 = 0..3, UInt8..UInt64 = 4..7, Float32 = 8, Float64 = 9
pub const ACU_I8: i32 = 0;
pub const ACU_I16: i32 = 1;
pub const ACU_I32: i32 = 2;
pub const ACU_I64: i32 = 3;
pub const ACU_U8: i32 = 4;
pub const ACU_U16: i32 = 5;
pub const ACU_U32: i32 = 6;
pub const ACU_U64: i32 = 7;
pub const ACU_F32: i32 = 8;
pub const ACU_F64: i32 = 9;
// Decimal128's native (16-byte two's complement, 16-byte aligned): acu_cmp, acu_filter_plan_create_cmp and acu_neg only
pub const ACU_I128: i32 = 10;
// acu_arith_op == arrow-arith/src/numeric.rs:181-190 `enum Op`
pub const ACU_ADD_WRAPPING: i32 = 0;
pub const ACU_ADD: i32 = 1;
pub const ACU_SUB_WRAPPING: i32 = 2;
pub const ACU_SUB: i32 = 3;
pub const ACU_MUL_WRAPPING: i32 = 4;
pub const ACU_MUL: i32 = 5;
pub const ACU_DIV: i32 = 6;
pub const ACU_REM: i32 = 7;
// acu_cmp_op == arrow-ord/src/cmp.rs:40-60 `enum Op`
pub const ACU_EQ: i32 = 0;
pub const ACU_NEQ: i32 = 1;
pub const ACU_LT: i32 = 2;
pub const ACU_LT_EQ: i32 = 3;
pub const ACU_GT: i32 = 4;
pub const ACU_GT_EQ: i32 = 5;
pub const ACU_DISTINCT: i32 = 6;
pub const ACU_NOT_DISTINCT: i32 = 7;
// acu_like_op (arrow-string/src/like.rs `enum Op`)
pub const ACU_LIKE: i32 = 0;
pub const ACU_NLIKE: i32 = 1;
pub const ACU_ILIKE: i32 = 2;
pub const ACU_NILIKE: i32 = 3;
pub const ACU_CONTAINS: i32 = 4;
pub const ACU_STARTS_WITH: i32 = 5;
pub const ACU_ENDS_WITH: i32 = 6;
pub const ACU_EQ_IGNORE_ASCII_CASE: i32 = 7;
// acu_length_op (arrow-string/src/length.rs)
pub const ACU_LENGTH: i32 = 0;
pub const ACU_BIT_LENGTH: i32 = 1;
pub const ACU_SUM: i32 = 0;
pub const ACU_MIN: i32 = 1;
pub const ACU_MAX: i32 = 2;
pub const ACU_PRODUCT: i32 = 3;
pub const ACU_BIT_AND: i32 = 4;
pub const ACU_BIT_OR: i32 = 5;
pub const ACU_BIT_XOR: i32 = 6;
// acu_bitwise_op (arrow-arith/src/bitwise.rs)
pub const ACU_BITWISE_AND: i32 = 0;
pub const ACU_BITWISE_OR: i32 = 1;
pub const ACU_BITWISE_XOR: i32 = 2;
pub const ACU_BITWISE_AND_NOT: i32 = 3;
pub const ACU_BITWISE_SHIFT_LEFT: i32 = 4;
pub const ACU_BITWISE_SHIFT_RIGHT: i32 = 5;
pub const ACU_BITWISE_NOT: i32 = 6;
pub const ACU_BOOL_AND: i32 = 0;
pub const ACU_BOOL_OR: i32 = 1;
pub const ACU_BOOL_AND_NOT: i32 = 2;
pub const ACU_BOOL_AND_KLEENE: i32 = 3;
pub const ACU_BOOL_OR_KLEENE: i32 = 4;
pub const ACU_BOOL_NOT: i32 = 5;
pub const ACU_BOOL_IS_NULL: i32 = 6;
pub const ACU_BOOL_IS_NOT_NULL: i32 = 7;
pub const ACU_COL_PRIMITIVE: i32 = 0;
pub const ACU_COL_BOOLEAN: i32 = 1;
pub const ACU_COL_BYTES: i32 = 2;
pub const ACU_COL_FIXED_SIZE_BINARY: i32 = 3;
pub const ACU_MAX_BATCH_COLUMNS: usize = 64;

#[repr(C)]
pub struct acu_ctx { _private: [u8; 0] }
#[repr(C)]
pub struct acu_filter_plan { _private: [u8; 0] }

#[repr(C)]
pub struct acu_error_detail {
    pub status: acu_status,
    pub cuda_error: i32,
    pub index: i64,
    pub lhs_bits: u64,
    pub rhs_bits: u64,
    pub len: u64,
    pub message: [c_char; 256],
}

/// acu_decimal_type: DataType::Decimal32 / 64 / 128(precision, scale) as byte_width 4 / 8 / 16
#[repr(C)]
#[derive(Clone, Copy, Debug, Default)]
pub struct acu_decimal_type {
    pub byte_width: i32,
    pub precision: u8,
    pub scale: i8,
    pub reserved: [u8; 2],
}

#[repr(C)]
#[derive(Clone, Copy)]
pub struct acu_array {
    pub values: *const c_void,
    pub values_offset: i64,
    pub validity: *const u8,
    pub validity_offset: i64,
    pub len: i64,
    pub null_count: i64,
    pub is_scalar: i32,
    pub reserved: i32,
}

#[repr(C)]
#[derive(Clone, Copy)]
pub struct acu_array_out {
    pub values: *mut c_void,
    pub validity: *mut u8,
    pub len: i64,
    pub null_count: i64,
    pub has_validity: i32,
    pub reserved: i32,
}

/// acu_column (include/arrow_cuda.h): one column of a RecordBatch for the record-batch entry points.
#[repr(C)]
#[derive(Clone, Copy)]
pub struct acu_column {
    pub kind: i32,  // 0 primitive, 1 boolean, 2 bytes (Utf8 / Binary)
    pub width: i32, // primitive: element bytes; bytes: offset width (4 | 8)
    pub array: acu_array,
    pub data: *const u8,
}

/// acu_column_out: caller-owned output buffers of one column.
#[repr(C)]
#[derive(Clone, Copy)]
pub struct acu_column_out {
    pub array: acu_array_out,
    pub data: *mut u8,
    pub data_capacity: i64,
    pub data_len: i64,
}

/// acu_list_array: one level of a List / LargeList / FixedSizeList column (the child is described separately).
pub const ACU_LIST: i32 = 0;
pub const ACU_LARGE_LIST: i32 = 1;
pub const ACU_FIXED_SIZE_LIST: i32 = 2;
#[repr(C)]
#[derive(Clone, Copy)]
pub struct acu_list_array {
    pub kind: i32,
    pub list_size: i32,
    pub offsets: *const c_void,
    pub nulls: acu_array,
    pub child_len: i64,
}

/// acu_bytes_array / acu_view_array: operands of acu_cmp_bytes / acu_cmp_byte_view.
#[repr(C)]
#[derive(Clone, Copy)]
pub struct acu_bytes_array {
    pub offsets: *const c_void,
    pub data: *const u8,
    pub nulls: acu_array,
}
#[repr(C)]
#[derive(Clone, Copy)]
pub struct acu_view_array {
    pub views: *const c_void,
    pub buffers: *const *const u8, // HOST array of n_buffers DEVICE pointers
    pub n_buffers: i32,
    pub reserved: i32,
    pub nulls: acu_array,
}

/// acu_run_array: the run ends of a RunEndEncoded column from physical entry 0 and its logical slice; acu_run_values: its
/// values child as take's run merge compares it (the values child itself is filtered / taken separately).
pub const ACU_RUN_VALUES_FIXED: i32 = 0;
pub const ACU_RUN_VALUES_BOOLEAN: i32 = 1;
pub const ACU_RUN_VALUES_BYTES: i32 = 2;
pub const ACU_RUN_VALUES_VIEW: i32 = 3;
pub const ACU_RUN_VALUES_NESTED: i32 = 4;
#[repr(C)]
#[derive(Clone, Copy)]
pub struct acu_run_array {
    pub run_end_dtype: i32,
    pub reserved: i32,
    pub run_ends: *const c_void,
    pub n_runs: i64,
    pub offset: i64,
    pub len: i64,
}
#[repr(C)]
#[derive(Clone, Copy)]
pub struct acu_run_values {
    pub kind: i32,
    pub width: i32,
    pub array: acu_array,
    pub bytes: acu_bytes_array,
    pub view: acu_view_array,
}
/// acu_union_array: one level of a sparse / dense Union column (the children are filtered / taken separately).
pub const ACU_UNION_SPARSE: i32 = 0;
pub const ACU_UNION_DENSE: i32 = 1;
#[repr(C)]
#[derive(Clone, Copy)]
pub struct acu_union_array {
    pub mode: i32,
    pub n_fields: i32,
    pub field_type_ids: *const i8,
    pub type_ids: *const i8,
    pub offsets: *const i32,
    pub len: i64,
}
#[repr(C)]
pub struct acu_ipc_stream { _private: [u8; 0] }

extern "C" {
    pub fn acu_abi_version() -> i32;
    pub fn acu_abi_sizeof(which: i32) -> i32;
    pub fn acu_ctx_create(device: i32, out: *mut *mut acu_ctx) -> acu_status;
    pub fn acu_ctx_destroy(ctx: *mut acu_ctx);
    pub fn acu_ctx_sync(ctx: *mut acu_ctx) -> acu_status;
    pub fn acu_last_error(ctx: *const acu_ctx) -> *const acu_error_detail;
    pub fn acu_malloc(ctx: *mut acu_ctx, bytes: usize, out: *mut *mut c_void) -> acu_status;
    pub fn acu_free(ctx: *mut acu_ctx, dptr: *mut c_void) -> acu_status;
    pub fn acu_memcpy_h2d(ctx: *mut acu_ctx, dst: *mut c_void, src: *const c_void, bytes: usize) -> acu_status;
    pub fn acu_memcpy_d2h(ctx: *mut acu_ctx, dst: *mut c_void, src: *const c_void, bytes: usize) -> acu_status;
    pub fn acu_host_alloc(ctx: *mut acu_ctx, bytes: usize, out: *mut *mut c_void) -> acu_status;
    pub fn acu_host_free(ctx: *mut acu_ctx, host: *mut c_void) -> acu_status;
    pub fn acu_bitmap_count(ctx: *mut acu_ctx, bits: *const u8, offset: i64, validity: *const u8, validity_offset: i64,
                            len: i64, out_count: *mut i64) -> acu_status;
    pub fn acu_filter_plan_create(ctx: *mut acu_ctx, predicate: *const acu_array, out: *mut *mut acu_filter_plan) -> acu_status;
    pub fn acu_filter_plan_destroy(ctx: *mut acu_ctx, plan: *mut acu_filter_plan);
    pub fn acu_filter_plan_count(plan: *const acu_filter_plan) -> i64;
    pub fn acu_filter_plan_len(plan: *const acu_filter_plan) -> i64;
    pub fn acu_filter_plan_strategy(plan: *const acu_filter_plan) -> i32;
    pub fn acu_filter_plan_indices(ctx: *mut acu_ctx, plan: *const acu_filter_plan, index_dtype: i32, out: *mut c_void) -> acu_status;
    pub fn acu_filter_primitive(ctx: *mut acu_ctx, plan: *const acu_filter_plan, elem_bytes: i32, values: *const acu_array,
                                out: *mut acu_array_out) -> acu_status;
    pub fn acu_filter_boolean(ctx: *mut acu_ctx, plan: *const acu_filter_plan, values: *const acu_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_filter_bytes(ctx: *mut acu_ctx, plan: *const acu_filter_plan, offset_bytes: i32, offsets: *const c_void, data: *const u8,
                            nulls_of: *const acu_array, out_offsets: *mut c_void, out_data: *mut u8, out_data_capacity: i64,
                            out_data_len: *mut i64, out_nulls: *mut acu_array_out) -> acu_status;
    pub fn acu_take_primitive(ctx: *mut acu_ctx, elem_bytes: i32, values: *const acu_array, indices: *const acu_array,
                              index_dtype: i32, check_bounds: i32, out: *mut acu_array_out) -> acu_status;
    pub fn acu_take_boolean(ctx: *mut acu_ctx, values: *const acu_array, indices: *const acu_array, index_dtype: i32,
                            check_bounds: i32, out: *mut acu_array_out) -> acu_status;
    pub fn acu_take_bytes(ctx: *mut acu_ctx, offset_bytes: i32, offsets: *const c_void, data: *const u8, nulls_of: *const acu_array,
                          indices: *const acu_array, index_dtype: i32, check_bounds: i32, out_offsets: *mut c_void,
                          out_data: *mut u8, out_data_capacity: i64, out_data_len: *mut i64, out_nulls: *mut acu_array_out) -> acu_status;
    pub fn acu_take_bytes_extend(ctx: *mut acu_ctx, offset_bytes: i32, offsets: *const c_void, data: *const u8, nulls_of: *const acu_array,
                                 indices: *const acu_array, index_dtype: i32, out_offsets: *mut c_void, out_data: *mut u8,
                                 out_data_capacity: i64, out_data_len: *mut i64, out_nulls: *mut acu_array_out) -> acu_status;
    pub fn acu_filter_list(ctx: *mut acu_ctx, plan: *const acu_filter_plan, list: *const acu_list_array, out_offsets: *mut c_void,
                           out_nulls: *mut acu_array_out, out_child_plan: *mut *mut acu_filter_plan) -> acu_status;
    pub fn acu_take_list(ctx: *mut acu_ctx, list: *const acu_list_array, indices: *const acu_array, index_dtype: i32, check_bounds: i32,
                         keep_null_ranges: i32, out_offsets: *mut c_void, out_nulls: *mut acu_array_out, child_index_dtype: i32,
                         out_child_indices: *mut c_void, capacity: i64, out_child_rows: *mut i64,
                         out_child_index_nulls: *mut acu_array_out) -> acu_status;
    pub fn acu_filter_run_end(ctx: *mut acu_ctx, plan: *const acu_filter_plan, ree: *const acu_run_array, out_run_ends: *mut c_void,
                              out_runs: *mut i64, out_values_start: *mut i64, out_values_plan: *mut *mut acu_filter_plan) -> acu_status;
    pub fn acu_take_run_end(ctx: *mut acu_ctx, ree: *const acu_run_array, values: *const acu_run_values, indices: *const acu_array,
                            index_dtype: i32, check_bounds: i32, out_run_ends: *mut c_void, out_value_indices: *mut c_void,
                            out_runs: *mut i64) -> acu_status;
    pub fn acu_filter_nulls(ctx: *mut acu_ctx, plan: *const acu_filter_plan, nulls_of: *const acu_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_take_nulls(ctx: *mut acu_ctx, nulls_of: *const acu_array, indices: *const acu_array, index_dtype: i32, check_bounds: i32,
                          out: *mut acu_array_out) -> acu_status;
    pub fn acu_filter_union(ctx: *mut acu_ctx, plan: *const acu_filter_plan, u: *const acu_union_array, out_type_ids: *mut i8,
                            out_offsets: *mut i32, out_child_rows: *mut i32, out_field_starts: *mut i64) -> acu_status;
    pub fn acu_take_union(ctx: *mut acu_ctx, u: *const acu_union_array, indices: *const acu_array, index_dtype: i32, check_bounds: i32,
                          out_type_ids: *mut i8, out_offsets: *mut i32, out_child_rows: *mut i32, out_field_starts: *mut i64) -> acu_status;
    pub fn acu_filter_fixed_size_binary(ctx: *mut acu_ctx, plan: *const acu_filter_plan, byte_width: i32, values: *const acu_array,
                                        out: *mut acu_array_out) -> acu_status;
    pub fn acu_take_fixed_size_binary(ctx: *mut acu_ctx, byte_width: i32, values: *const acu_array, indices: *const acu_array,
                                      index_dtype: i32, check_bounds: i32, out: *mut acu_array_out) -> acu_status;
    pub fn acu_arith(ctx: *mut acu_ctx, dtype: i32, op: i32, a: *const acu_array, b: *const acu_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_neg(ctx: *mut acu_ctx, dtype: i32, checked: i32, a: *const acu_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_decimal_arith(ctx: *mut acu_ctx, op: i32, lt: *const acu_decimal_type, a: *const acu_array, rt: *const acu_decimal_type,
                             b: *const acu_array, out_type: *mut acu_decimal_type, out: *mut acu_array_out) -> acu_status;
    pub fn acu_cmp(ctx: *mut acu_ctx, dtype: i32, op: i32, a: *const acu_array, b: *const acu_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_cast_numeric(ctx: *mut acu_ctx, from: i32, to: i32, safe: i32, a: *const acu_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_cast_decimal(ctx: *mut acu_ctx, from: *const acu_decimal_type, to: *const acu_decimal_type, safe: i32, a: *const acu_array,
                            out: *mut acu_array_out) -> acu_status;
    pub fn acu_cast_to_decimal(ctx: *mut acu_ctx, from: i32, to: *const acu_decimal_type, safe: i32, a: *const acu_array,
                               out: *mut acu_array_out) -> acu_status;
    pub fn acu_cast_from_decimal(ctx: *mut acu_ctx, from: *const acu_decimal_type, to: i32, safe: i32, a: *const acu_array,
                                 out: *mut acu_array_out) -> acu_status;
    pub fn acu_aggregate(ctx: *mut acu_ctx, dtype: i32, op: i32, a: *const acu_array, out_bits: *mut u64, out_valid: *mut i64) -> acu_status;
    /// out_bits: 2 words (low, high) of the i128 result
    pub fn acu_aggregate_i128(ctx: *mut acu_ctx, op: i32, a: *const acu_array, out_bits: *mut u64, out_valid: *mut i64) -> acu_status;
    pub fn acu_boolean(ctx: *mut acu_ctx, op: i32, a: *const acu_array, b: *const acu_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_filter_record_batch(ctx: *mut acu_ctx, plan: *const acu_filter_plan, n_columns: i32, columns: *const acu_column,
                                   outs: *mut acu_column_out) -> acu_status;
    pub fn acu_take_record_batch(ctx: *mut acu_ctx, n_columns: i32, columns: *const acu_column, indices: *const acu_array,
                                 index_dtype: i32, check_bounds: i32, outs: *mut acu_column_out) -> acu_status;
    pub fn acu_aggregate_columns(ctx: *mut acu_ctx, n_columns: i32, dtypes: *const i32, ops: *const i32, arrays: *const acu_array,
                                 out_bits: *mut u64, out_valid_counts: *mut i64) -> acu_status;
    pub fn acu_sum_checked(ctx: *mut acu_ctx, dtype: i32, a: *const acu_array, out_bits: *mut u64, out_valid: *mut i64) -> acu_status;
    pub fn acu_product_checked(ctx: *mut acu_ctx, dtype: i32, a: *const acu_array, out_bits: *mut u64, out_valid: *mut i64) -> acu_status;
    pub fn acu_bitwise(ctx: *mut acu_ctx, dtype: i32, op: i32, a: *const acu_array, b: *const acu_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_aggregate_bytes(ctx: *mut acu_ctx, offset_bytes: i32, op: i32, a: *const acu_bytes_array, out_row: *mut i64,
                               out_valid: *mut i64) -> acu_status;
    pub fn acu_aggregate_byte_view(ctx: *mut acu_ctx, op: i32, a: *const acu_view_array, out_row: *mut i64, out_valid: *mut i64) -> acu_status;
    pub fn acu_aggregate_fixed_size_binary(ctx: *mut acu_ctx, byte_width: i32, op: i32, a: *const acu_array, out_row: *mut i64,
                                           out_valid: *mut i64) -> acu_status;
    pub fn acu_aggregate_boolean(ctx: *mut acu_ctx, op: i32, a: *const acu_array, out_value: *mut i32, out_valid: *mut i64) -> acu_status;
    pub fn acu_filter_plan_create_cmp(ctx: *mut acu_ctx, dtype: i32, op: i32, a: *const acu_array, b: *const acu_array,
                                      out: *mut *mut acu_filter_plan) -> acu_status;
    pub fn acu_nullif(ctx: *mut acu_ctx, left: *const acu_array, right: *const acu_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_zip(ctx: *mut acu_ctx, elem_bytes: i32, mask: *const acu_array, truthy: *const acu_array, falsy: *const acu_array,
                   out: *mut acu_array_out) -> acu_status;
    pub fn acu_zip_bytes(ctx: *mut acu_ctx, offset_bytes: i32, mask: *const acu_array, truthy: *const acu_bytes_array,
                         falsy: *const acu_bytes_array, out_offsets: *mut c_void, out_data: *mut u8, out_data_capacity: i64,
                         out_data_len: *mut i64, out_nulls: *mut acu_array_out) -> acu_status;
    pub fn acu_zip_byte_view(ctx: *mut acu_ctx, mask: *const acu_array, truthy: *const acu_view_array, falsy: *const acu_view_array,
                             out_views: *mut c_void, out_nulls: *mut acu_array_out, out_buffers: *mut i32) -> acu_status;
    pub fn acu_zip_boolean(ctx: *mut acu_ctx, mask: *const acu_array, truthy: *const acu_array, falsy: *const acu_array,
                           out: *mut acu_array_out) -> acu_status;
    pub fn acu_zip_fixed_size_binary(ctx: *mut acu_ctx, byte_width: i32, mask: *const acu_array, truthy: *const acu_array,
                                     falsy: *const acu_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_cmp_bytes(ctx: *mut acu_ctx, offset_bytes: i32, op: i32, l: *const acu_bytes_array, r: *const acu_bytes_array,
                         out: *mut acu_array_out) -> acu_status;
    pub fn acu_cmp_byte_view(ctx: *mut acu_ctx, op: i32, l: *const acu_view_array, r: *const acu_view_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_like_bytes(ctx: *mut acu_ctx, offset_bytes: i32, is_utf8: i32, op: i32, l: *const acu_bytes_array, r: *const acu_bytes_array,
                          out: *mut acu_array_out) -> acu_status;
    pub fn acu_like_byte_view(ctx: *mut acu_ctx, is_utf8: i32, op: i32, l: *const acu_view_array, r: *const acu_view_array,
                              out: *mut acu_array_out) -> acu_status;
    pub fn acu_length_bytes(ctx: *mut acu_ctx, offset_bytes: i32, op: i32, a: *const acu_bytes_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_length_byte_view(ctx: *mut acu_ctx, op: i32, a: *const acu_view_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_length_fixed_size_binary(ctx: *mut acu_ctx, byte_width: i32, op: i32, a: *const acu_array, out: *mut acu_array_out) -> acu_status;
    pub fn acu_substring_bytes(ctx: *mut acu_ctx, offset_bytes: i32, is_utf8: i32, start: i64, has_length: i32, length: u64,
                               a: *const acu_bytes_array, data_len: i64, out_offsets: *mut c_void, out_data: *mut u8, out_data_capacity: i64,
                               out_data_len: *mut i64, out_nulls: *mut acu_array_out) -> acu_status;
    pub fn acu_substring_by_char(ctx: *mut acu_ctx, offset_bytes: i32, start: i64, has_length: i32, length: u64, a: *const acu_bytes_array,
                                 out_offsets: *mut c_void, out_data: *mut u8, out_data_capacity: i64, out_data_len: *mut i64,
                                 out_nulls: *mut acu_array_out) -> acu_status;
    pub fn acu_substring_byte_view(ctx: *mut acu_ctx, is_utf8: i32, start: i64, has_length: i32, length: u64, a: *const acu_view_array,
                                   out_views: *mut c_void, out_nulls: *mut acu_array_out) -> acu_status;
    pub fn acu_substring_fixed_size_binary(ctx: *mut acu_ctx, byte_width: i32, start: i64, has_length: i32, length: u64, a: *const acu_array,
                                           out_byte_width: *mut i32, out: *mut acu_array_out) -> acu_status;
    pub fn acu_concat_elements_bytes(ctx: *mut acu_ctx, offset_bytes: i32, l: *const acu_bytes_array, r: *const acu_bytes_array,
                                     out_offsets: *mut c_void, out_data: *mut u8, out_data_capacity: i64, out_data_len: *mut i64,
                                     out_nulls: *mut acu_array_out) -> acu_status;
    pub fn acu_concat_elements_bytes_many(ctx: *mut acu_ctx, offset_bytes: i32, n_arrays: i32, arrays: *const acu_bytes_array,
                                          out_offsets: *mut c_void, out_data: *mut u8, out_data_capacity: i64, out_data_len: *mut i64,
                                          out_nulls: *mut acu_array_out) -> acu_status;
    pub fn acu_concat_elements_byte_view(ctx: *mut acu_ctx, l: *const acu_view_array, r: *const acu_view_array, out_views: *mut c_void,
                                         out_data: *mut u8, out_data_capacity: i64, out_data_len: *mut i64,
                                         out_nulls: *mut acu_array_out) -> acu_status;
    pub fn acu_concat_elements_fixed_size_binary(ctx: *mut acu_ctx, l_width: i32, l: *const acu_array, r_width: i32, r: *const acu_array,
                                                 out_byte_width: *mut i32, out: *mut acu_array_out) -> acu_status;
    pub fn acu_concat(ctx: *mut acu_ctx, n_arrays: i32, arrays: *const acu_column, out: *mut acu_column_out) -> acu_status;
    pub fn acu_concat_batches(ctx: *mut acu_ctx, n_batches: i32, n_columns: i32, columns: *const acu_column, outs: *mut acu_column_out,
                              out_rows: *mut i64) -> acu_status;
    pub fn acu_ipc_stream_open(ctx: *mut acu_ctx, stream: *const u8, stream_len: i64, out: *mut *mut acu_ipc_stream, out_n_fields: *mut i32) -> acu_status;
    pub fn acu_ipc_stream_field(s: *const acu_ipc_stream, i: i32, kind: *mut i32, width: *mut i32, dtype: *mut i32, nullable: *mut i32,
                                name: *mut *const c_char) -> acu_status;
    pub fn acu_ipc_stream_next(ctx: *mut acu_ctx, s: *mut acu_ipc_stream, out_columns: *mut acu_column, out_rows: *mut i64) -> acu_status;
    pub fn acu_ipc_stream_close(ctx: *mut acu_ctx, s: *mut acu_ipc_stream);
    pub fn acu_aggregate_allreduce(ctx: *mut acu_ctx, dtype: i32, op: i32, a: *const acu_array, out_bits: *mut u64, out_valid: *mut i64) -> acu_status;
    pub fn acu_filter_plan_slices(ctx: *mut acu_ctx, plan: *const acu_filter_plan, out_pairs: *mut u64, capacity: i64, out_slices: *mut i64) -> acu_status;
    // stream-ordered sections (include/arrow_cuda.h): the entry points listed there only enqueue between the two calls
    pub fn acu_async_begin(ctx: *mut acu_ctx) -> acu_status;
    pub fn acu_results_fetch(ctx: *mut acu_ctx) -> acu_status;
    pub fn acu_async_active(ctx: *const acu_ctx) -> i32;
    // Utf8View / BinaryView buffer management of BatchCoalescer (arrow-select/src/coalesce/byte_view.rs)
    pub fn acu_view_bytes_used(ctx: *mut acu_ctx, views: *const c_void, n: i64, out_total: *mut i64) -> acu_status;
    pub fn acu_view_fit(ctx: *mut acu_ctx, views: *const c_void, n: i64, remaining_capacity: i64, out_views: *mut i64, out_bytes: *mut i64) -> acu_status;
    pub fn acu_view_copy_strings(ctx: *mut acu_ctx, views: *const c_void, n: i64, buffers: *const *const u8, n_buffers: i32, new_buffer_index: u32,
                                 dst: *mut u8, dst_len: i64, dst_capacity: i64, out_views: *mut c_void, out_bytes: *mut i64) -> acu_status;
    pub fn acu_view_rebase(ctx: *mut acu_ctx, views: *const c_void, n: i64, delta: u32, out_views: *mut c_void) -> acu_status;
    pub fn acu_comm_get_unique_id(out_id: *mut u8) -> acu_status;
    pub fn acu_comm_init(ctx: *mut acu_ctx, id: *const u8, rank: i32, world: i32) -> acu_status;
    pub fn acu_comm_destroy(ctx: *mut acu_ctx) -> acu_status;
    pub fn acu_comm_allreduce_aggregates(ctx: *mut acu_ctx, dtype: i32, op: i32, partial_bits: *mut u64, valid_counts: *mut i64, n: i32) -> acu_status;
    pub fn acu_comm_allreduce_i64_sum(ctx: *mut acu_ctx, values: *mut i64, n: i32) -> acu_status;
}
