// recordbatch.cu — RecordBatch-level entry points: every column of a batch goes through the
// same per-column launch code as the single-array calls, but all kernels of all columns are
// queued back to back on the ctx stream and the host synchronises ONCE (each column owns one
// result block of ctx->d_res), instead of once or twice per column. filter_bytes / take_bytes
// are these drivers on one variable-width column.
//
//   filter_record_batch   arrow-select/src/filter.rs:225-244, :459-478 (one predicate, all columns)
//   take_record_batch     arrow-select/src/take.rs:1123-1133 (take_arrays :155-164)
//   sum/min/max           arrow-arith/src/aggregate.rs:943,1012,1027 (one call per column in the reference)
#include <vector>

#include "bitmap.cuh"
#include "internal.cuh"

namespace {

acu_status bad_columns(acu_ctx *ctx, int32_t n) {
  return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, (uint64_t)n, "record batch of %d columns: 0..%d supported per call", n,
                  ACU_MAX_BATCH_COLUMNS);
}

acu_status bad_kind(acu_ctx *ctx, int32_t c, int32_t kind) {
  acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, (uint64_t)c, "column %d: unknown column kind %d", c, kind);
  return ACU_ERR_INVALID_ARGUMENT;
}

acu_status bad_width(acu_ctx *ctx, int32_t c, int32_t width) {
  return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, (uint64_t)c, "column %d: FixedSizeBinary byte width %d < 0", c, width);
}

// A failed launch may leave work queued: wait for it before returning the error (like the reference, the failing
// column's own ArrowError).
acu_status drain(acu_ctx *ctx, acu_status st) {
  cudaStreamSynchronize(ctx->stream);
  acu_kstats_drain(ctx);
  return st;
}

acu_status filter_columns(acu_ctx *ctx, const acu_filter_plan *plan, int32_t n_columns, const acu_column *columns,
                          acu_column_out *outs) {
  if (n_columns < 0 || n_columns > ACU_MAX_BATCH_COLUMNS) return bad_columns(ctx, n_columns);
  if (n_columns == 0) return ACU_OK;  // RecordBatch with no columns keeps only its row count (filter.rs:236-243)
  const int64_t count = acu_filter_plan_count(plan);
  // one scratch allocation carved per variable-width column (acu_scratch may reallocate: call it once)
  const size_t per_col = acu_bytes_col_scratch(count);
  size_t n_bytes_cols = 0;
  for (int32_t c = 0; c < n_columns; ++c) n_bytes_cols += columns[c].kind == ACU_COL_BYTES;
  uint8_t *scratch = nullptr;
  if (n_bytes_cols) ACU_TRY(acu_scratch(ctx, per_col * n_bytes_cols, reinterpret_cast<void **>(&scratch)));
  std::vector<int> mode(n_columns, 0), kinds(n_columns, 0);
  std::vector<int32_t> widths(n_columns, 0);
  std::vector<const acu_array *> vals(n_columns);
  std::vector<acu_array_out *> outp(n_columns);
  std::vector<unsigned long long *> resp(n_columns);
  std::vector<acu_bytes_col_state> bstate(n_columns);
  for (int32_t c = 0; c < n_columns; ++c) {
    const acu_column &col = columns[c];
    if (col.kind < ACU_COL_PRIMITIVE || col.kind > ACU_COL_FIXED_SIZE_BINARY) return bad_kind(ctx, c, col.kind);
    if (col.kind == ACU_COL_FIXED_SIZE_BINARY && col.width < 0) return bad_width(ctx, c, col.width);
    kinds[c] = col.kind == ACU_COL_PRIMITIVE ? 0 : col.kind == ACU_COL_BOOLEAN ? 1 : 2;
    if (col.kind == ACU_COL_FIXED_SIZE_BINARY) kinds[c] = acu_fsb_filter_kind(plan, col.width, &col.array, &outs[c].array);
    widths[c] = col.width;
    vals[c] = &col.array;
    outp[c] = &outs[c].array;
    resp[c] = acu_dres(ctx, c);
  }
  ACU_TRY(acu_res_reset_n(ctx, n_columns));
  {  // values of fixed-width columns + every validity compaction, like columns sharing launches
    acu_status st = acu_filter_cols_launch(ctx, plan, n_columns, kinds.data(), widths.data(), vals.data(), outp.data(), resp.data(), mode.data());
    if (st != ACU_OK) return drain(ctx, st);
  }
  for (int32_t c = 0; c < n_columns; ++c) {  // FixedSizeBinary values the fixed-width kernels do not serve
    if (columns[c].kind != ACU_COL_FIXED_SIZE_BINARY || kinds[c] != 2) continue;
    acu_status st = acu_fsb_filter_values_launch(ctx, plan, columns[c].width, &columns[c].array, &outs[c].array, acu_dres(ctx, c));
    if (st != ACU_OK) return drain(ctx, st);
  }
  size_t k = 0;
  for (int32_t c = 0; c < n_columns; ++c) {
    const acu_column &col = columns[c];
    if (col.kind != ACU_COL_BYTES) continue;
    acu_status st = acu_filter_bytes_col_launch(ctx, plan, col.width, col.array.values, col.data, &col.array, outs[c].array.values, outs[c].data,
                                                outs[c].data_capacity, scratch + per_col * k++, acu_dres(ctx, c), &bstate[c]);
    if (st != ACU_OK) return drain(ctx, st);
  }
  ACU_TRY(acu_res_fetch_n(ctx, n_columns));
  for (int32_t c = 0; c < n_columns; ++c) {
    if (columns[c].kind == ACU_COL_FIXED_SIZE_BINARY) acu_fsb_filter_finalize(plan, mode[c], columns[c].width, acu_hres(ctx, c), &outs[c].array);
    else acu_filter_col_finalize(plan, mode[c], acu_hres(ctx, c), &outs[c].array);
    outs[c].data_len = 0;
    if (columns[c].kind == ACU_COL_BYTES) ACU_TRY(acu_filter_bytes_col_finalize(ctx, &bstate[c], acu_hres(ctx, c), &outs[c].data_len));
  }
  return ACU_OK;
}

acu_status take_columns(acu_ctx *ctx, int32_t n_columns, const acu_column *columns, const acu_array *indices, acu_dtype index_dtype,
                        int32_t check_bounds, acu_column_out *outs, bool extend = false) {
  if (n_columns < 0 || n_columns > ACU_MAX_BATCH_COLUMNS) return bad_columns(ctx, n_columns);
  if (n_columns == 0) return ACU_OK;
  if (acu_take_index_kind(index_dtype) < 0)  // take.rs:103
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Take only supported for integers, got %s", acu_dtype_name(index_dtype));
  acu_status st;
  const int64_t m = indices->len;
  const int64_t inc = acu_resolve_null_count(ctx, indices, &st);
  ACU_TRY(st);
  const bool idx_nulls = indices->validity && inc > 0;
  std::vector<char> val_nulls(n_columns, 0);
  int64_t checked_len = -1;
  for (int32_t c = 0; c < n_columns; ++c) {  // host-visible facts first: anything that needs its own sync
    const int64_t vnc = acu_resolve_null_count(ctx, &columns[c].array, &st);
    ACU_TRY(st);
    val_nulls[c] = columns[c].array.validity && vnc > 0;
    if (check_bounds && columns[c].array.len != checked_len) {  // the columns of a RecordBatch share one length: normally once
      ACU_TRY(acu_take_check_bounds(ctx, indices, index_dtype, idx_nulls, columns[c].array.len));
      checked_len = columns[c].array.len;
    }
  }
  const size_t per_col = acu_bytes_col_scratch(m);
  size_t n_bytes_cols = 0;
  for (int32_t c = 0; c < n_columns; ++c) n_bytes_cols += columns[c].kind == ACU_COL_BYTES;
  uint8_t *scratch = nullptr;
  if (n_bytes_cols) ACU_TRY(acu_scratch(ctx, per_col * n_bytes_cols, reinterpret_cast<void **>(&scratch)));
  std::vector<int> mode(n_columns, -1);  // -1: no validity gather queued for the column
  std::vector<acu_bytes_col_state> bstate(n_columns);
  // fixed-width / boolean columns, and the validity gather of variable-width columns whose values have nulls:
  // like columns share launches
  std::vector<int32_t> eb;
  std::vector<const acu_array *> vals;
  std::vector<char> isbool, vnulls;
  std::vector<acu_array_out *> outp;
  std::vector<unsigned long long *> resp;
  std::vector<int> who;
  for (int32_t c = 0; c < n_columns; ++c) {
    const acu_column &col = columns[c];
    if (col.kind < ACU_COL_PRIMITIVE || col.kind > ACU_COL_FIXED_SIZE_BINARY) return bad_kind(ctx, c, col.kind);
    if (col.kind == ACU_COL_BYTES && !val_nulls[c]) continue;  // nulls = indices.nulls().cloned(): queued with the bytes pass
    int32_t width = col.kind == ACU_COL_PRIMITIVE ? col.width : 0;
    if (col.kind == ACU_COL_FIXED_SIZE_BINARY) {
      if (col.width < 0) return bad_width(ctx, c, col.width);
      width = acu_fsb_take_width(col.width, &col.array, &outs[c].array);
      if (width == 0 && !val_nulls[c] && !indices->validity) continue;  // no validity to gather: the row gather alone
    }
    eb.push_back(width);
    vals.push_back(&col.array);
    isbool.push_back(col.kind == ACU_COL_BOOLEAN);
    vnulls.push_back(val_nulls[c]);
    outp.push_back(&outs[c].array);
    resp.push_back(acu_dres(ctx, c));
    who.push_back(c);
  }
  ACU_TRY(acu_res_reset_n(ctx, n_columns));
  if (!who.empty()) {
    std::vector<int> modes(who.size(), 0);
    st = acu_take_cols_launch(ctx, (int)who.size(), eb.data(), vals.data(), isbool.data(), vnulls.data(), indices, index_dtype, idx_nulls,
                              outp.data(), resp.data(), modes.data());
    if (st != ACU_OK) return drain(ctx, st);
    for (size_t i = 0; i < who.size(); ++i) mode[who[i]] = modes[i];
  }
  for (int32_t c = 0; c < n_columns; ++c) {  // FixedSizeBinary values k_take does not serve
    if (columns[c].kind != ACU_COL_FIXED_SIZE_BINARY) continue;
    st = acu_fsb_take_values_launch(ctx, columns[c].width, &columns[c].array, indices, index_dtype, idx_nulls, &outs[c].array, acu_dres(ctx, c));
    if (st != ACU_OK) return drain(ctx, st);
  }
  size_t k = 0;
  for (int32_t c = 0; c < n_columns; ++c) {
    const acu_column &col = columns[c];
    if (col.kind != ACU_COL_BYTES) continue;
    st = acu_take_bytes_col_launch(ctx, col.width, col.array.values, col.data, &col.array, val_nulls[c], indices, index_dtype, idx_nulls,
                                   outs[c].array.values, outs[c].data, outs[c].data_capacity, &outs[c].array, scratch + per_col * k++,
                                   acu_dres(ctx, c), &bstate[c], extend);
    if (st != ACU_OK) return drain(ctx, st);
  }
  ACU_TRY(acu_res_fetch_n(ctx, n_columns));
  for (int32_t c = 0; c < n_columns; ++c) {
    const acu_column &col = columns[c];
    outs[c].data_len = 0;
    if (col.kind == ACU_COL_FIXED_SIZE_BINARY) {
      ACU_TRY(acu_fsb_take_finalize(ctx, col.width, &col.array, indices, index_dtype, val_nulls[c], mode[c], acu_hres(ctx, c), &outs[c].array));
      continue;
    }
    if (mode[c] >= 0) ACU_TRY(acu_take_col_finalize(ctx, &col.array, indices, index_dtype, mode[c], acu_hres(ctx, c), &outs[c].array));
    if (col.kind == ACU_COL_BYTES)
      ACU_TRY(acu_take_bytes_col_finalize(ctx, &col.array, indices, index_dtype, &bstate[c], acu_hres(ctx, c), &outs[c].data_len, &outs[c].array));
  }
  return ACU_OK;
}

// One Utf8 / Binary array as an ACU_COL_BYTES column: `array` carries the nulls, its values the offsets.
acu_column bytes_column(int32_t offset_bytes, const void *offsets, const uint8_t *data, const acu_array *nulls_of) {
  acu_column col{};
  col.kind = ACU_COL_BYTES;
  col.width = offset_bytes;
  col.array = *nulls_of;
  col.array.values = offsets;
  col.data = data;
  return col;
}

acu_column_out bytes_column_out(void *out_offsets, uint8_t *out_data, int64_t out_data_capacity, const acu_array_out *out_nulls) {
  acu_column_out out{};
  out.array = *out_nulls;
  out.array.values = out_offsets;
  out.data = out_data;
  out.data_capacity = out_data_capacity;
  return out;
}

// What the single-array byte calls return: the data length and the NullBuffer decision.
acu_status bytes_result(const acu_column_out &out, acu_status st, int64_t *out_data_len, acu_array_out *out_nulls) {
  *out_data_len = out.data_len;
  out_nulls->len = out.array.len;
  out_nulls->null_count = out.array.null_count;
  out_nulls->has_validity = out.array.has_validity;
  return st;
}

}  // namespace

extern "C" acu_status acu_filter_record_batch(acu_ctx *ctx, const acu_filter_plan *plan, int32_t n_columns,
                                              const acu_column *columns, acu_column_out *outs) {
  ACU_ENTER(ctx);
  return filter_columns(ctx, plan, n_columns, columns, outs);
}

extern "C" acu_status acu_take_record_batch(acu_ctx *ctx, int32_t n_columns, const acu_column *columns, const acu_array *indices,
                                            acu_dtype index_dtype, int32_t check_bounds, acu_column_out *outs) {
  ACU_ENTER(ctx);
  return take_columns(ctx, n_columns, columns, indices, index_dtype, check_bounds, outs);
}

extern "C" acu_status acu_filter_bytes(acu_ctx *ctx, const acu_filter_plan *plan, int32_t offset_bytes,
                                       const void *offsets, const uint8_t *data, const acu_array *nulls_of,
                                       void *out_offsets, uint8_t *out_data, int64_t out_data_capacity,
                                       int64_t *out_data_len, acu_array_out *out_nulls) {
  ACU_ENTER(ctx);
  const acu_column col = bytes_column(offset_bytes, offsets, data, nulls_of);
  acu_column_out out = bytes_column_out(out_offsets, out_data, out_data_capacity, out_nulls);
  const acu_status st = filter_columns(ctx, plan, 1, &col, &out);
  return bytes_result(out, st, out_data_len, out_nulls);
}

extern "C" acu_status acu_take_bytes(acu_ctx *ctx, int32_t offset_bytes, const void *offsets, const uint8_t *data,
                                     const acu_array *nulls_of, const acu_array *indices, acu_dtype index_dtype,
                                     int32_t check_bounds, void *out_offsets, uint8_t *out_data,
                                     int64_t out_data_capacity, int64_t *out_data_len, acu_array_out *out_nulls) {
  ACU_ENTER(ctx);
  const acu_column col = bytes_column(offset_bytes, offsets, data, nulls_of);
  acu_column_out out = bytes_column_out(out_offsets, out_data, out_data_capacity, out_nulls);
  const acu_status st = take_columns(ctx, 1, &col, indices, index_dtype, check_bounds, &out);
  return bytes_result(out, st, out_data_len, out_nulls);
}

extern "C" acu_status acu_take_bytes_extend(acu_ctx *ctx, int32_t offset_bytes, const void *offsets, const uint8_t *data,
                                            const acu_array *nulls_of, const acu_array *indices, acu_dtype index_dtype, void *out_offsets,
                                            uint8_t *out_data, int64_t out_data_capacity, int64_t *out_data_len, acu_array_out *out_nulls) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  if (indices->validity && indices->len > 0) {
    acu_status st;
    const int64_t nc = acu_resolve_null_count(ctx, indices, &st);
    ACU_TRY(st);
    if (nc > 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "take_bytes_extend: the row map has a null");
  }
  const acu_column col = bytes_column(offset_bytes, offsets, data, nulls_of);
  acu_column_out out = bytes_column_out(out_offsets, out_data, out_data_capacity, out_nulls);
  const acu_status st = take_columns(ctx, 1, &col, indices, index_dtype, 0, &out, true);
  return bytes_result(out, st, out_data_len, out_nulls);
}

extern "C" acu_status acu_aggregate_columns(acu_ctx *ctx, int32_t n_columns, const acu_dtype *dtypes, const acu_agg_op *ops,
                                            const acu_array *arrays, uint64_t *out_bits, int64_t *out_valid_counts) {
  ACU_ENTER(ctx);
  if (n_columns < 0 || n_columns > ACU_MAX_BATCH_COLUMNS) return bad_columns(ctx, n_columns);
  if (n_columns == 0) return ACU_OK;
  acu_status st;
  std::vector<int64_t> nc(n_columns, 0);
  for (int32_t c = 0; c < n_columns; ++c) ACU_TRY(acu_agg_op_check(ctx, dtypes[c], ops[c]));
  for (int32_t c = 0; c < n_columns; ++c) {
    out_bits[c] = 0;
    nc[c] = acu_resolve_null_count(ctx, &arrays[c], &st);
    ACU_TRY(st);
    out_valid_counts[c] = arrays[c].len - nc[c];
  }
  const size_t per_col = (acu_reduce_col_scratch(ctx) + 255) & ~(size_t)255;
  uint8_t *scratch;
  ACU_TRY(acu_scratch(ctx, per_col * n_columns, reinterpret_cast<void **>(&scratch)));
  std::vector<int> launched(n_columns, 0);
  std::vector<unsigned long long *> resp(n_columns);
  for (int32_t c = 0; c < n_columns; ++c) resp[c] = acu_dres(ctx, c);
  ACU_TRY(acu_res_reset_n(ctx, n_columns));
  st = acu_reduce_cols_launch(ctx, n_columns, dtypes, ops, arrays, nc.data(), scratch, per_col, resp.data(), launched.data());
  if (st != ACU_OK) return drain(ctx, st);
  ACU_TRY(acu_res_fetch_n(ctx, n_columns));
  for (int32_t c = 0; c < n_columns; ++c)
    if (launched[c]) out_bits[c] = acu_hres(ctx, c)[RES_AUX0];
  return ACU_OK;
}
