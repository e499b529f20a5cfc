// internal.cuh — cross-translation-unit internals (not part of the C ABI).
#pragma once
#include "common.cuh"

// f(T()) for T the native type of a numeric dtype (ACU_I8 .. ACU_F64), otherwise(): one dtype -> C++ type mapping
// for the typed entry points, each keeping its own failure for the dtypes it does not take.
template <class F, class G>
auto acu_with_native(acu_dtype dt, F &&f, G &&otherwise) -> decltype(otherwise()) {
  switch (dt) {
    case ACU_I8: return f(int8_t());
    case ACU_I16: return f(int16_t());
    case ACU_I32: return f(int32_t());
    case ACU_I64: return f(int64_t());
    case ACU_U8: return f(uint8_t());
    case ACU_U16: return f(uint16_t());
    case ACU_U32: return f(uint32_t());
    case ACU_U64: return f(uint64_t());
    case ACU_F32: return f(float());
    case ACU_F64: return f(double());
    default: return otherwise();
  }
}

// The operand front end of every entry point over Utf8 / Binary (acu_bytes_array) and view (acu_view_array) columns.
// An entry point that synchronises (one not split into enqueue and finalise) refuses inside a stream-ordered section:
// acu_sync_only is its first check, before any argument check or device work.
acu_status acu_sync_only(acu_ctx *ctx);
acu_status acu_offset_width_check(acu_ctx *ctx, int32_t offset_bytes);  // Utf8 / Binary offsets are 4 or 8 bytes wide
// A view array's data-buffer pointer table goes to acu_view_table_bytes(a) bytes (a multiple of 256) of the caller's one
// acu_scratch request; acu_view_operand queues the copy of a->buffers there on the ctx stream.
struct ViewOperand;
size_t acu_view_table_bytes(const acu_view_array *a);
acu_status acu_view_operand(acu_ctx *ctx, const acu_view_array *a, void *table_space, ViewOperand *out);

struct acu_filter_plan;
const uint64_t *acu_plan_mask(const acu_filter_plan *p);      // normalised mask words (padded to x32)
const uint64_t *acu_plan_tile_off(const acu_filter_plan *p);  // exclusive output offset per 1024-row tile
int64_t acu_plan_n_words_padded(const acu_filter_plan *p);
void **acu_plan_index_cache(const acu_filter_plan *p);        // lazily materialised selected-row ids (bytes.cu)

// The columns of filter / take / sum-min-max, split so that several columns share one stream synchronisation: launch
// queues the kernels of every column, like columns sharing launches (blockIdx.y = column), with popcounts and results
// landing in res[c], column c's device result block; finalize turns the fetched block into the NullBuffer decision.
// The single-array calls are these launchers on one column.
// filter kinds[c]: 0 primitive, 1 boolean, 2 validity only.
acu_status acu_filter_cols_launch(acu_ctx *ctx, const acu_filter_plan *plan, int n, const int *kinds, const int32_t *widths,
                                  const acu_array *const *values, acu_array_out *const *outs, unsigned long long *const *res, int *modes);
void acu_filter_col_finalize(const acu_filter_plan *plan, int mode, const unsigned long long *hres, acu_array_out *out);
acu_status acu_take_cols_launch(acu_ctx *ctx, int n, const int32_t *elem_bytes, const acu_array *const *values, const char *boolean,
                                const char *val_nulls, const acu_array *indices, acu_dtype index_dtype, bool idx_nulls,
                                acu_array_out *const *outs, unsigned long long *const *res, int *modes);
acu_status acu_take_col_finalize(acu_ctx *ctx, const acu_array *values, const acu_array *indices, acu_dtype index_dtype, int mode,
                                 const unsigned long long *hres, acu_array_out *out);
acu_status acu_take_check_bounds(acu_ctx *ctx, const acu_array *indices, acu_dtype index_dtype, bool idx_nulls, int64_t values_len);
int acu_take_index_kind(acu_dtype t);  // -1 for non-integer index types
// sum / min / max / product / bit_and / bit_or / bit_xor: nc[c] = resolved null count; result bits in res[c][RES_AUX0].
// acu_agg_op_check refuses an op outside acu_agg_op, and a bit op of a float dtype, before anything is queued.
acu_status acu_agg_op_check(acu_ctx *ctx, acu_dtype dtype, acu_agg_op op);
size_t acu_reduce_col_scratch(const acu_ctx *ctx);
acu_status acu_reduce_cols_launch(acu_ctx *ctx, int n, const acu_dtype *dtypes, const acu_agg_op *ops, const acu_array *arrays,
                                  const int64_t *nc, uint8_t *scratch, size_t scratch_per_col, unsigned long long *const *res, int *launched);

// Variable-width columns (bytes.cu), same launch / finalize split for the offsets and value bytes. The column's validity
// is queued and finalised by the driver through acu_filter_cols_launch / acu_take_cols_launch, except take's copy of the
// indices' validity when the values have no nulls. `scratch` must hold acu_bytes_col_scratch(output rows) bytes and
// stay untouched until the stream has drained.
struct acu_bytes_col_state {
  bool gathered = false;          // the offsets / bytes gather was queued (output rows > 0)
  bool idx_nulls_copied = false;  // take: the output validity is a copy of the indices' (valid count in RES_COUNT)
  bool extend = false;            // MutableArrayData::extend: null rows keep their bytes, overflow is try_extend_offsets'
  // the gather's arguments, for the finaliser's offset-overflow diagnosis and capacity check
  int32_t ob = 0;
  int kind = 0;
  const void *offsets = nullptr, *idx = nullptr;
  const uint8_t *data = nullptr, *out_valid = nullptr;
  int64_t m = 0, n_src = 0;
  bool detect_oob = false;
  int64_t *block_tot = nullptr;
  void *out_offsets = nullptr;
  uint8_t *out_data = nullptr;
  int64_t out_cap = 0;
};
size_t acu_bytes_col_scratch(int64_t out_rows);
extern const char *const acu_extend_overflow_text;  // try_extend_offsets' InvalidArgumentError (list.cu)
acu_status acu_plan_cached_indices(acu_ctx *ctx, const acu_filter_plan *plan, const void **out_idx, int *out_kind);
acu_status acu_take_bytes_col_launch(acu_ctx *ctx, int32_t ob, const void *offsets, const uint8_t *data, const acu_array *nulls_of,
                                     bool val_nulls, const acu_array *indices, acu_dtype index_dtype, bool idx_nulls,
                                     void *out_offsets, uint8_t *out_data, int64_t out_cap, acu_array_out *out_nulls, void *scratch,
                                     unsigned long long *res, acu_bytes_col_state *st, bool extend = false);
acu_status acu_take_bytes_col_finalize(acu_ctx *ctx, const acu_array *nulls_of, const acu_array *indices, acu_dtype index_dtype,
                                       const acu_bytes_col_state *st, const unsigned long long *hres, int64_t *out_data_len,
                                       acu_array_out *out_nulls);
acu_status acu_filter_bytes_col_launch(acu_ctx *ctx, const acu_filter_plan *plan, int32_t ob, const void *offsets, const uint8_t *data,
                                       const acu_array *nulls_of, void *out_offsets, uint8_t *out_data, int64_t out_cap, void *scratch,
                                       unsigned long long *res, acu_bytes_col_state *st);
acu_status acu_filter_bytes_col_finalize(acu_ctx *ctx, const acu_bytes_col_state *st, const unsigned long long *hres,
                                         int64_t *out_data_len);

// FixedSizeBinary columns (fixed_size_binary.cu) inside the record-batch drivers: the validity, and the values of the
// widths the fixed-width kernels serve, go through acu_filter_cols_launch / acu_take_cols_launch with the kind / element
// width given here; the other widths' values through the row gather the *_values_launch calls queue (errors in RES_ERR2).
int acu_fsb_filter_kind(const acu_filter_plan *plan, int32_t w, const acu_array *values, const acu_array_out *out);  // 0 or 2
acu_status acu_fsb_filter_values_launch(acu_ctx *ctx, const acu_filter_plan *plan, int32_t w, const acu_array *values, acu_array_out *out,
                                        unsigned long long *res);
void acu_fsb_filter_finalize(const acu_filter_plan *plan, int mode, int32_t w, const unsigned long long *hres, acu_array_out *out);
int32_t acu_fsb_take_width(int32_t w, const acu_array *values, const acu_array_out *out);  // w when k_take serves the values, else 0
acu_status acu_fsb_take_values_launch(acu_ctx *ctx, int32_t w, const acu_array *values, const acu_array *indices, acu_dtype index_dtype,
                                      bool idx_nulls, acu_array_out *out, unsigned long long *res);
// mode: acu_take_cols_launch's, -1 when no validity gather was queued
acu_status acu_fsb_take_finalize(acu_ctx *ctx, int32_t w, const acu_array *values, const acu_array *indices, acu_dtype index_dtype,
                                 bool val_nulls, int mode, const unsigned long long *hres, acu_array_out *out);

// compare_op (arrow-ord/src/cmp.rs:220-382), elementwise.cu: the host-side decisions of every comparison, whatever the
// operand type (primitive, Utf8 / Binary, view). The kernels compute is_lt(a, b) or is_eq(a, b) of the swapped operands
// (a, b) at every slot, negate, then fold the validity into the values (distinct / not_distinct) or write it beside them.
enum { FOLD_NONE = 0, FOLD_DISTINCT = 1, FOLD_NOT_DISTINCT = 2 };
struct acu_cmp_decision {
  int64_t len;
  bool all_null;  // a null scalar against an array: BooleanArray::new_null(len), no kernel (cmp.rs:353, :364)
  bool swap;      // gt / lt_eq: a = r, b = l (cmp.rs:481-488)
  int lt, neg, fold;
  int a_scalar, b_scalar;             // a scalar against an array (two scalars compare as arrays of length 1)
  int a_null_scalar, b_null_scalar;   // that scalar's single slot is null
  const uint8_t *av, *bv;             // validity bitmaps the kernel reads, NULL = no nulls
  int64_t aoff, boff;
  bool has_validity;                  // the result carries a NullBuffer (valid count in RES_COUNT)
};
// The length check (cmp.rs:228-232) and the result length.
acu_status acu_cmp_len(acu_ctx *ctx, const acu_array *l, const acu_array *r, int64_t *len);
// acu_cmp_len, then out = an empty result of that length; for len > 0 the operands' null counts are resolved and the
// rest of *d is decided. Issues no device work unless a null count is unknown.
acu_status acu_cmp_decide(acu_ctx *ctx, acu_cmp_op op, const acu_array *l, const acu_array *r, acu_array_out *out,
                          acu_cmp_decision *d);
// has_validity / null_count of the result from its fetched result block
void acu_cmp_finalize(const acu_cmp_decision &d, const unsigned long long *hres, acu_array_out *out);
// PrimitiveArray::new_null / BooleanArray::new_null: `value_bytes` zeroed value bytes, an all-null bitmap, one
// synchronisation.
acu_status acu_new_null(acu_ctx *ctx, int64_t len, size_t value_bytes, acu_array_out *out);

// Fused compare -> filter plan (elementwise.cu): the cmp kernels write the plan's mask words and per-tile counts.
acu_status acu_cmp_into_plan(acu_ctx *ctx, acu_dtype dtype, acu_cmp_op op, const acu_array *a, const acu_array *b, uint64_t *mask,
                             int64_t n_words_padded, uint32_t *tile_count, int64_t n_tiles);

// In-place inclusive scan of n int64 values (bytes.cu); tmp: >= n / 4096 + n / 4096^2 + 4 values of scratch.
acu_status acu_scan_inclusive_i64(acu_ctx *ctx, int64_t *data, int64_t n, int64_t *tmp);
