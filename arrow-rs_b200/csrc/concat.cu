// concat.cu — the building blocks of coalescing: append a row range of a source column to an
// in-progress destination column at an arbitrary row position (SURVEY.md §8(f) rank 1:
// BatchCoalescer::push_batch / push_batch_with_filter, arrow-select/src/coalesce.rs:258-533, whose
// InProgressArray::copy_rows appends `len` rows starting at `offset` of the current source).
//
//   values of fixed width  : a device-to-device copy (acu_memcpy_d2d)
//   validity / boolean bits: acu_bitmap_copy — bits [src_off, src_off+len) to [dst_off, dst_off+len),
//                            every other destination bit preserved
//   all-valid ranges       : acu_bitmap_fill
//   Utf8 offsets           : acu_offsets_append — rebased on the destination's running byte total
//
// One thread per destination u64 word; boundary words are merged with atomicOr / atomicAnd so that
// two appends never need the destination to start on a word.
#include <vector>

#include "bitmap.cuh"
#include "internal.cuh"

namespace {

// dst bits [doff, doff+len) = src bits [soff, soff+len); popcount of the copied bits -> res[RES_COUNT]
__global__ void __launch_bounds__(256) k_bitmap_copy(const uint8_t *__restrict__ src, int64_t soff, unsigned long long *__restrict__ dst,
                                                     int64_t doff, int64_t len, unsigned long long *__restrict__ res) {
  const int64_t w0 = doff >> 6, w1 = (doff + len - 1) >> 6;  // destination words touched
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned cnt = 0;
  for (int64_t w = w0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w <= w1; w += stride) {
    const int64_t lo = w << 6;                                  // first destination bit of this word
    const int64_t b0 = lo < doff ? doff : lo;                   // range of this word that is written
    const int64_t b1 = lo + 64 > doff + len ? doff + len : lo + 64;
    const unsigned sh = (unsigned)(b0 - lo);
    const int n = (int)(b1 - b0);
    uint64_t bits = ld_bits64(src, soff + (b0 - doff), soff + len);  // n valid bits (zero beyond the source range)
    if (n < 64) bits &= (1ull << n) - 1ull;
    cnt += __popcll(bits);
    const uint64_t mask = (n == 64 ? ~0ull : ((1ull << n) - 1ull)) << sh;
    if (n == 64) {
      dst[w] = bits;
    } else {  // boundary word: clear the range, then set — other bits (earlier appends) are untouched
      atomicAnd(dst + w, ~mask);
      atomicOr(dst + w, bits << sh);
    }
  }
  if (res) {
    cnt = warp_sum(cnt);
    if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(res + RES_COUNT, (unsigned long long)cnt);
  }
}

__global__ void __launch_bounds__(256) k_bitmap_fill(unsigned long long *__restrict__ dst, int64_t doff, int64_t len, int value) {
  const int64_t w0 = doff >> 6, w1 = (doff + len - 1) >> 6;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t w = w0 + (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w <= w1; w += stride) {
    const int64_t lo = w << 6;
    const int64_t b0 = lo < doff ? doff : lo, b1 = lo + 64 > doff + len ? doff + len : lo + 64;
    const int n = (int)(b1 - b0);
    const uint64_t mask = (n == 64 ? ~0ull : ((1ull << n) - 1ull)) << (unsigned)(b0 - lo);
    if (n == 64) dst[w] = value ? ~0ull : 0ull;
    else if (value) atomicOr(dst + w, mask);
    else atomicAnd(dst + w, ~mask);
  }
}

// dst[dfirst + j] = base + src[first + j] - src[first], j = 0 .. count (count + 1 entries); the first entry
// past `limit` goes to res[RES_ERR_INDEX]; res[RES_AUX0] = src[first], res[RES_AUX1] = src[first + count]
template <class O>
__global__ void __launch_bounds__(256) k_offsets_append(const O *__restrict__ src, int64_t first, int64_t count, int64_t base,
                                                        O *__restrict__ dst, int64_t dfirst, int64_t limit, unsigned long long *__restrict__ res) {
  const int64_t s0 = (int64_t)__ldg(src + first);
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long err = ~0ull;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j <= count; j += stride) {
    const int64_t v = base + ((int64_t)__ldg(src + first + j) - s0);
    if (v > limit && (unsigned long long)j < err) err = (unsigned long long)j;
    dst[dfirst + j] = (O)v;
  }
  if (err != ~0ull) atomicMin(res + RES_ERR_INDEX, err);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    res[RES_AUX0] = (unsigned long long)s0;
    res[RES_AUX1] = (unsigned long long)(int64_t)__ldg(src + first + count);
  }
}

}  // namespace

extern "C" acu_status acu_bitmap_copy(acu_ctx *ctx, const uint8_t *src, int64_t src_offset, uint8_t *dst, int64_t dst_offset, int64_t len,
                                      int64_t *out_set_bits) {
  ACU_ENTER(ctx);
  if (out_set_bits) *out_set_bits = 0;
  if (len <= 0) return ACU_OK;
  if (((uintptr_t)dst & 7) != 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "bitmap_copy: destination must be 8-byte aligned");
  const int64_t words = ((dst_offset + len - 1) >> 6) - (dst_offset >> 6) + 1;
  if (out_set_bits) ACU_TRY(acu_res_reset(ctx));
  ACU_LAUNCH(ctx, k_bitmap_copy, acu_grid(ctx, (words + 255) / 256, 8), 256, 0, src, src_offset, reinterpret_cast<unsigned long long *>(dst),
             dst_offset, len, out_set_bits ? ctx->d_res : nullptr);
  if (out_set_bits) {
    ACU_TRY(acu_res_fetch(ctx));
    *out_set_bits = (int64_t)ctx->h_res[RES_COUNT];
  }
  return ACU_OK;
}

extern "C" acu_status acu_bitmap_fill(acu_ctx *ctx, uint8_t *dst, int64_t dst_offset, int64_t len, int32_t value) {
  ACU_ENTER(ctx);
  if (len <= 0) return ACU_OK;
  if (((uintptr_t)dst & 7) != 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "bitmap_fill: destination must be 8-byte aligned");
  const int64_t words = ((dst_offset + len - 1) >> 6) - (dst_offset >> 6) + 1;
  ACU_LAUNCH(ctx, k_bitmap_fill, acu_grid(ctx, (words + 255) / 256, 8), 256, 0, reinterpret_cast<unsigned long long *>(dst), dst_offset, len, (int)value);
  return ACU_OK;
}

extern "C" acu_status acu_offsets_append(acu_ctx *ctx, int32_t offset_bytes, const void *src_offsets, int64_t first, int64_t count,
                                         int64_t base, void *dst_offsets, int64_t dst_first, int64_t *out_src_begin, int64_t *out_src_end) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_offset_width_check(ctx, offset_bytes));
  if (count < 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "offsets_append: negative count");
  ACU_TRY(acu_res_reset(ctx));
  const int grid = acu_grid(ctx, (count + 1 + 255) / 256, 8);
  if (offset_bytes == 4)
    ACU_LAUNCH(ctx, k_offsets_append<int32_t>, grid, 256, 0, static_cast<const int32_t *>(src_offsets), first, count, base,
               static_cast<int32_t *>(dst_offsets), dst_first, (int64_t)INT32_MAX, ctx->d_res);
  else
    ACU_LAUNCH(ctx, k_offsets_append<int64_t>, grid, 256, 0, static_cast<const int64_t *>(src_offsets), first, count, base,
               static_cast<int64_t *>(dst_offsets), dst_first, INT64_MAX, ctx->d_res);
  ACU_TRY(acu_res_fetch(ctx));
  const int64_t s0 = (int64_t)ctx->h_res[RES_AUX0], s1 = (int64_t)ctx->h_res[RES_AUX1];
  if (out_src_begin) *out_src_begin = s0;
  if (out_src_end) *out_src_end = s1;
  if (ctx->h_res[RES_ERR_INDEX] != ~0ull) {  // the appended values no longer fit the offset type
    const long long total = (long long)(base + (s1 - s0));
    return acu_fail(ctx, ACU_ERR_OFFSET_OVERFLOW, (int64_t)ctx->h_res[RES_ERR_INDEX], 0, 0, (uint64_t)total, "%lld", total);
  }
  return ACU_OK;
}

// ---- concat / concat_batches (arrow-select/src/concat.rs:495-640) ------------------------------------------------------
// concat_primitives / concat_boolean / concat_bytes are builder.append_array per input (concat.rs:334-368):
//   values   : raw copies in input order (bytes under null slots included)                primitive_builder.rs:290-303
//   booleans : bit ranges appended at the running row                                     boolean_builder.rs append_array
//   bytes    : offsets rebased on the running byte total (OffsetOverflowError(shift + last) when the type overflows),
//              each input's value bytes [offsets[0], offsets[len])                        generic_bytes_builder.rs:169-206
//   nulls    : NullBufferBuilder — materialised iff some input has null_count > 0 (null.rs:209-218), then Some(..)
// One input returns array.slice(0, len) in the reference (zero copy, its NullBuffer kept as it is); with caller-owned
// outputs that is a copy that keeps the input's NullBuffer presence.
static acu_status concat_one_field(acu_ctx *ctx, int32_t n, const acu_column *cols, int64_t stride, acu_column_out *out) {
  if (n <= 0)  // concat.rs:496-499
    return acu_fail(ctx, ACU_ERR_COMPUTE, -1, 0, 0, 0, "concat requires input of at least one array");
  const acu_column &c0 = cols[0];
  for (int i = 1; i < n; ++i) {
    const acu_column &c = cols[(size_t)i * stride];
    if (c.kind != c0.kind || c.width != c0.width)  // concat.rs:505-535 (the reference lists the DataTypes; the C ABI only knows kind / width)
      return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, i, 0, 0, 0,
                      "It is not possible to concatenate arrays of different data types (kind %d width %d, kind %d width %d).",
                      c0.kind, c0.width, c.kind, c.width);
  }
  if (c0.kind == ACU_COL_FIXED_SIZE_BINARY)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "concat: FixedSizeBinary columns are not supported");
  if (c0.kind == ACU_COL_BYTES) ACU_TRY(acu_offset_width_check(ctx, c0.width));
  int64_t total = 0;
  bool any_nulls = false;
  int64_t null_total = 0;
  std::vector<int64_t> ncs((size_t)n);
  for (int i = 0; i < n; ++i) {
    const acu_column &c = cols[(size_t)i * stride];
    acu_status st = ACU_OK;
    ncs[i] = c.array.len ? acu_resolve_null_count(ctx, &c.array, &st) : 0;
    ACU_TRY(st);
    any_nulls = any_nulls || ncs[i] > 0;
    null_total += ncs[i];
    total += c.array.len;
  }
  const bool keep_single = n == 1 && c0.array.validity != nullptr;  // slice(0, len): the NullBuffer survives as it is
  out->array.len = total;
  out->array.null_count = 0;
  out->array.has_validity = 0;
  out->data_len = 0;
  int64_t row = 0, bytes = 0;
  if (c0.kind == ACU_COL_BYTES) ACU_CUDA(ctx, cudaMemsetAsync(out->array.values, 0, (size_t)c0.width, ctx->stream));  // offsets[0] = 0
  for (int i = 0; i < n; ++i) {
    const acu_column &c = cols[(size_t)i * stride];
    const int64_t len = c.array.len;
    if (len == 0) continue;
    if (c.kind == ACU_COL_PRIMITIVE) {
      ACU_CUDA(ctx, cudaMemcpyAsync(static_cast<uint8_t *>(out->array.values) + (size_t)row * c.width, c.array.values, (size_t)len * c.width,
                                    cudaMemcpyDeviceToDevice, ctx->stream));
    } else if (c.kind == ACU_COL_BOOLEAN) {
      ACU_TRY(acu_bitmap_copy(ctx, static_cast<const uint8_t *>(c.array.values), c.array.values_offset, static_cast<uint8_t *>(out->array.values),
                              row, len, nullptr));
    } else {
      int64_t sb = 0, se = 0;
      ACU_TRY(acu_offsets_append(ctx, c.width, c.array.values, 0, len, bytes, out->array.values, row, &sb, &se));
      if (bytes + (se - sb) > out->data_capacity)
        return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, (uint64_t)(bytes + (se - sb)), "output data capacity %lld < required %lld",
                        (long long)out->data_capacity, (long long)(bytes + (se - sb)));
      if (se > sb)
        ACU_CUDA(ctx, cudaMemcpyAsync(out->data + bytes, c.data + sb, (size_t)(se - sb), cudaMemcpyDeviceToDevice, ctx->stream));
      bytes += se - sb;
    }
    if (any_nulls || keep_single) {
      if (c.array.validity) ACU_TRY(acu_bitmap_copy(ctx, c.array.validity, c.array.validity_offset, out->array.validity, row, len, nullptr));
      else ACU_TRY(acu_bitmap_fill(ctx, out->array.validity, row, len, 1));
    }
    row += len;
  }
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  out->data_len = bytes;
  if (any_nulls || keep_single) {
    out->array.has_validity = 1;
    out->array.null_count = null_total;
  }
  return ACU_OK;
}

extern "C" acu_status acu_concat(acu_ctx *ctx, int32_t n_arrays, const acu_column *arrays, acu_column_out *out) {
  ACU_ENTER(ctx);
  return concat_one_field(ctx, n_arrays, arrays, 1, out);
}

extern "C" acu_status acu_concat_batches(acu_ctx *ctx, int32_t n_batches, int32_t n_columns, const acu_column *columns, acu_column_out *outs,
                                         int64_t *out_rows) {
  ACU_ENTER(ctx);
  if (out_rows) *out_rows = 0;
  if (n_batches <= 0) {  // RecordBatch::new_empty(schema) (concat.rs:620-622)
    for (int c = 0; c < n_columns; ++c) { outs[c].array.len = 0; outs[c].array.null_count = 0; outs[c].array.has_validity = 0; outs[c].data_len = 0; }
    return ACU_OK;
  }
  for (int c = 0; c < n_columns; ++c) ACU_TRY(concat_one_field(ctx, n_batches, columns + c, n_columns, &outs[c]));
  if (out_rows && n_columns > 0) *out_rows = outs[0].array.len;
  return ACU_OK;
}
