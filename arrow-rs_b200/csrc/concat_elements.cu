// concat_elements.cu — arrow-string/src/concat_elements.rs: the element-wise concatenation of GenericByteArray (Utf8,
// Binary: i32 offsets; LargeUtf8, LargeBinary: i64), GenericByteViewArray (Utf8View, BinaryView) and FixedSizeBinary.
//
//   bytes (two or many operands): row i is operand 0's value i, then operand 1's, ... (null slots included). ConcatRows
//        reads every operand's two offsets of row i from the operand table; the bytes engine (bytes_engine.cuh) scans the
//        totals, writes the offsets and pushes the row's segments one after another. An i32 result whose running end passes
//        i32::MAX is the reference's `from_usize(..).unwrap()` panic at that row (the engine's `limit`).
//   views: ViewConcatRows gives each non-null row whose result is longer than 12 bytes its length (every other row 0), the
//        same engine places those results in row order in ONE new data buffer and copies their two segments; then
//        k_concat_views writes every view (null: zero, <= 12 bytes: inline, longer: prefix, buffer 0, the engine's offset).
//   FixedSizeBinary: a strided copy (k_fsb_concat); null rows are zero bytes.
//
// The output NullBuffer is NullBuffer::union of the operands': the AND of every present validity bitmap, kept only when it
// has a null.
#include <vector>

#include "bitmap.cuh"
#include "bytes_cmp.cuh"
#include "bytes_engine.cuh"
#include "internal.cuh"

namespace {

// One byte-array operand: the offsets of its logical row 0 and its value bytes.
struct ByteSeg {
  const void *offs;
  const uint8_t *data;
};

template <class O>
struct ConcatRows {
  int ob;
  int64_t m;
  int detect_oob;
  const ByteSeg *ops;  // device table of n_ops operands
  int n_ops;
  __device__ __forceinline__ int nsegs() const { return n_ops; }
  __device__ __forceinline__ void ranges4(int64_t j0, int64_t begin[4], uint64_t len[4], unsigned long long *) const {
#pragma unroll
    for (int k = 0; k < 4; ++k) begin[k] = 0, len[k] = 0;
    for (int s = 0; s < n_ops; ++s) {
      const O *offs = static_cast<const O *>(ops[s].offs);
      O o[5];
#pragma unroll
      for (int k = 0; k < 5; ++k) o[k] = j0 + k <= m ? __ldg(offs + j0 + k) : (O)0;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (j0 + k < m) len[k] += (uint64_t)(int64_t)(o[k + 1] - o[k]);
    }
  }
  __device__ __forceinline__ void segment(int64_t row, int s, const uint8_t **p, uint64_t *len) const {
    const O *offs = static_cast<const O *>(ops[s].offs);
    const O b = __ldg(offs + row), e = __ldg(offs + row + 1);
    *p = ops[s].data + b;
    *len = (uint64_t)(int64_t)(e - b);
  }
};

__device__ __forceinline__ bool row_valid(const uint64_t *valid, int64_t i) { return !valid || ((__ldg(valid + (i >> 6)) >> (i & 63)) & 1ull); }

// The rows of the views' new data buffer: a non-null row whose result is longer than 12 bytes has its total length, every
// other row none. A null row's views are never read.
struct ViewConcatRows {
  int ob;
  int64_t m;
  int detect_oob;
  ViewOperand l, r;
  const uint64_t *valid;  // the union, bit offset 0; NULL = no null
  __device__ __forceinline__ int nsegs() const { return 2; }
  __device__ __forceinline__ void ranges4(int64_t j0, int64_t begin[4], uint64_t len[4], unsigned long long *) const {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      begin[k] = 0, len[k] = 0;
      const int64_t i = j0 + k;
      if (i < m && row_valid(valid, i)) {
        const uint64_t t = (uint64_t)l.view(i).x + (uint64_t)r.view(i).x;
        if (t > 12) len[k] = t;
      }
    }
  }
  __device__ __forceinline__ void segment(int64_t row, int s, const uint8_t **p, uint64_t *len) const {
    const BytesItem it = s ? r.item(row) : l.item(row);
    *p = it.p;
    *len = (uint64_t)it.len;
  }
};

struct ViewConcatOut {
  ViewOperand l, r;
  const uint64_t *valid;
  int64_t n;
  const int32_t *offs;   // the engine's offsets: row i's result starts at offs[i] in the new data buffer
  const int64_t *total;  // the new data buffer's length (device)
  int64_t cap;
  uint4 *out;
};

// Up to 12 bytes of p as a little-endian 96-bit value, zero above n.
__device__ __forceinline__ unsigned __int128 ld_upto12(const uint8_t *p, uint32_t n) {
  const uint64_t lo = ld_upto8(p, n < 8 ? n : 8), hi = n > 8 ? ld_upto8(p + 8, n - 8) : 0ull;
  return ((unsigned __int128)hi << 64) | lo;
}

// make_view of every row: all-zero for a null row; the zero-padded bytes for a result of at most 12 bytes; otherwise the
// length, the first 4 bytes (they span both sides when the left value is shorter than 4), buffer 0 and the row's offset.
// Writes nothing (grid-uniformly) when the data buffer overflows i32 or the caller's capacity.
__global__ void __launch_bounds__(256) k_concat_views(const ViewConcatOut p) {
  const int64_t total = __ldg(p.total);
  if (total > INT32_MAX || total > p.cap) return;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += stride) {
    uint4 r = make_uint4(0, 0, 0, 0);
    if (row_valid(p.valid, i)) {
      const BytesItem a = p.l.item(i), b = p.r.item(i);
      const uint32_t la = (uint32_t)a.len, lb = (uint32_t)b.len, L = la + lb;
      if (L <= 12) {
        const unsigned __int128 x = ld_upto12(a.p, la) | (ld_upto12(b.p, lb) << (8 * la));
        r = make_uint4(L, (uint32_t)x, (uint32_t)(x >> 32), (uint32_t)(x >> 64));
      } else {
        uint32_t pre = (uint32_t)ld_upto8(a.p, la < 4 ? la : 4);
        if (la < 4) pre |= (uint32_t)(ld_upto8(b.p, lb < 4 - la ? lb : 4 - la) << (8 * la));
        r = make_uint4(L, pre, 0u, (uint32_t)__ldg(p.offs + i));
      }
    }
    st_stream16(p.out + i, r);
  }
}

// The bytes of one FixedSizeBinary row side into dst; zero bytes for a null row.
__device__ __forceinline__ void fsb_put(uint8_t *dst, const uint8_t *src, int64_t w, bool valid) {
  for (int64_t k = 0; k < w; k += 8) {
    const uint32_t nb = (uint32_t)(w - k < 8 ? w - k : 8);
    const uint64_t v = valid ? ld_upto8(src + k, nb) : 0ull;
    for (uint32_t b = 0; b < nb; ++b) dst[k + b] = (uint8_t)(v >> (8 * b));
  }
}

// One row per thread: output row i = left row i, then right row i (lw + rw bytes apart).
__global__ void __launch_bounds__(256) k_fsb_concat(const uint8_t *__restrict__ l, int64_t lw, const uint8_t *__restrict__ r, int64_t rw,
                                                    const uint64_t *__restrict__ valid, int64_t n, uint8_t *__restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x, w = lw + rw;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const bool v = row_valid(valid, i);
    fsb_put(out + i * w, l + i * lw, lw, v);
    fsb_put(out + i * w + lw, r + i * rw, rw, v);
  }
}

// ---- host side -------------------------------------------------------------------------------------------------------
acu_status check_array(acu_ctx *ctx, const acu_array *nulls) {
  if (nulls->is_scalar) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "concat_elements takes arrays, not scalars");
  if (nulls->len < 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "concat_elements: negative length");
  return ACU_OK;
}

acu_status same_length(acu_ctx *ctx, const acu_array *l, const acu_array *r) {
  if (l->len != r->len)
    return acu_fail(ctx, ACU_ERR_COMPUTE, -1, 0, 0, 0, "Arrays must have the same length: %lld != %lld", (long long)l->len, (long long)r->len);
  return ACU_OK;
}

// NullBuffer::union of the operands into out (bit offset 0), its valid count in RES_COUNT; *valid = out, or NULL when no
// operand has a NullBuffer.
acu_status union_nulls(acu_ctx *ctx, const std::vector<const acu_array *> &ops, int64_t n, uint8_t *out, const uint64_t **valid) {
  std::vector<const acu_array *> with;
  for (const acu_array *a : ops)
    if (a->validity) with.push_back(a);
  *valid = nullptr;
  if (with.empty() || n == 0) return ACU_OK;
  uint64_t *o = reinterpret_cast<uint64_t *>(out);
  const size_t k = with.size();
  const acu_array *b = k > 1 ? with[1] : nullptr;
  ACU_TRY(acu_bitmap_and_launch(ctx, with[0]->validity, with[0]->validity_offset, b ? b->validity : nullptr, b ? b->validity_offset : 0, n, o,
                                k <= 2));
  for (size_t j = 2; j < k; ++j)  // in place: each word is read and written by the same thread
    ACU_TRY(acu_bitmap_and_launch(ctx, out, 0, with[j]->validity, with[j]->validity_offset, n, o, j + 1 == k));
  *valid = o;
  return ACU_OK;
}

// The builder's NullBuffer: present only when the union has a null.
void union_result(const uint64_t *valid, int64_t n, const unsigned long long *h, acu_array_out *out) {
  out->len = n;
  out->null_count = valid ? n - (int64_t)h[RES_COUNT] : 0;
  out->has_validity = out->null_count > 0;
}

template <class O>
acu_status concat_bytes_run(acu_ctx *ctx, const std::vector<const acu_bytes_array *> &arrays, void *out_offsets, uint8_t *out_data,
                            int64_t out_cap, int64_t *out_data_len, acu_array_out *out_nulls) {
  const int64_t n = arrays[0]->nulls.len;
  std::vector<const acu_array *> nulls;
  std::vector<ByteSeg> table;
  for (const acu_bytes_array *a : arrays) {
    nulls.push_back(&a->nulls);
    table.push_back(ByteSeg{a->offsets, a->data});
  }
  const uint64_t *valid;
  ACU_TRY(union_nulls(ctx, nulls, n, out_nulls->validity, &valid));
  if (n > 0) {
    void *scratch;
    const size_t eng = engine_scratch(n);
    ACU_TRY(acu_scratch(ctx, eng + align256(table.size() * sizeof(ByteSeg)), &scratch));
    ByteSeg *d_table = reinterpret_cast<ByteSeg *>(static_cast<uint8_t *>(scratch) + eng);
    ACU_CUDA(ctx, cudaMemcpyAsync(d_table, table.data(), table.size() * sizeof(ByteSeg), cudaMemcpyHostToDevice, ctx->stream));
    ConcatRows<O> rows{(int)sizeof(O), n, 0, d_table, (int)table.size()};
    ACU_TRY(engine_launch(ctx, rows, static_cast<int64_t *>(scratch), out_offsets, out_data, out_cap,
                          sizeof(O) == 4 ? (int64_t)INT32_MAX : INT64_MAX));
  } else {
    ACU_CUDA(ctx, cudaMemsetAsync(out_offsets, 0, sizeof(O), ctx->stream));
  }
  ACU_TRY(acu_res_fetch(ctx));
  const unsigned long long *h = ctx->h_res;
  *out_data_len = 0;
  union_result(valid, n, h, out_nulls);
  if (n == 0) return ACU_OK;
  if (h[RES_ERR2] != ~0ull)  // `T::Offset::from_usize(output_values.len()).unwrap()` at the first row past i32::MAX
    return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, (int64_t)h[RES_ERR2], 0, 0, 0, "called `Option::unwrap()` on a `None` value");
  return finish_bytes(ctx, out_data, out_cap, out_data_len);
}

acu_status concat_bytes(acu_ctx *ctx, int32_t offset_bytes, const std::vector<const acu_bytes_array *> &arrays, void *out_offsets,
                        uint8_t *out_data, int64_t out_cap, int64_t *out_data_len, acu_array_out *out_nulls) {
  if (offset_bytes == 4) return concat_bytes_run<int32_t>(ctx, arrays, out_offsets, out_data, out_cap, out_data_len, out_nulls);
  return concat_bytes_run<int64_t>(ctx, arrays, out_offsets, out_data, out_cap, out_data_len, out_nulls);
}

}  // namespace

// Every entry point starts with acu_res_reset, whose acu_sync_only refuses inside a stream-ordered section before any
// argument check.
extern "C" acu_status acu_concat_elements_bytes(acu_ctx *ctx, int32_t offset_bytes, const acu_bytes_array *l, const acu_bytes_array *r,
                                                void *out_offsets, uint8_t *out_data, int64_t out_data_capacity, int64_t *out_data_len,
                                                acu_array_out *out_nulls) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(acu_offset_width_check(ctx, offset_bytes));
  ACU_TRY(check_array(ctx, &l->nulls));
  ACU_TRY(check_array(ctx, &r->nulls));
  ACU_TRY(same_length(ctx, &l->nulls, &r->nulls));
  return concat_bytes(ctx, offset_bytes, {l, r}, out_offsets, out_data, out_data_capacity, out_data_len, out_nulls);
}

extern "C" acu_status acu_concat_elements_bytes_many(acu_ctx *ctx, int32_t offset_bytes, int32_t n_arrays, const acu_bytes_array *arrays,
                                                     void *out_offsets, uint8_t *out_data, int64_t out_data_capacity, int64_t *out_data_len,
                                                     acu_array_out *out_nulls) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(acu_offset_width_check(ctx, offset_bytes));
  if (n_arrays < 1) return acu_fail(ctx, ACU_ERR_COMPUTE, -1, 0, 0, 0, "concat requires input of at least one array");
  if (!arrays) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "concat_elements: arrays is NULL");
  std::vector<const acu_bytes_array *> ops;
  for (int32_t k = 0; k < n_arrays; ++k) {
    ACU_TRY(check_array(ctx, &arrays[k].nulls));
    ops.push_back(arrays + k);
  }
  const int64_t size = arrays[0].nulls.len;
  for (const acu_bytes_array *a : ops)
    if (a->nulls.len != size) return acu_fail(ctx, ACU_ERR_COMPUTE, -1, 0, 0, 0, "Arrays must have the same length of %lld", (long long)size);
  return concat_bytes(ctx, offset_bytes, ops, out_offsets, out_data, out_data_capacity, out_data_len, out_nulls);
}

extern "C" acu_status acu_concat_elements_byte_view(acu_ctx *ctx, const acu_view_array *l, const acu_view_array *r, void *out_views,
                                                    uint8_t *out_data, int64_t out_data_capacity, int64_t *out_data_len,
                                                    acu_array_out *out_nulls) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(check_array(ctx, &l->nulls));
  ACU_TRY(check_array(ctx, &r->nulls));
  ACU_TRY(same_length(ctx, &l->nulls, &r->nulls));
  const int64_t n = l->nulls.len;
  const uint64_t *valid;
  ACU_TRY(union_nulls(ctx, {&l->nulls, &r->nulls}, n, out_nulls->validity, &valid));
  if (n > 0) {
    void *scratch;
    const size_t eng = engine_scratch(n), offs = align256((size_t)(n + 1) * 4), lt = acu_view_table_bytes(l);
    ACU_TRY(acu_scratch(ctx, eng + offs + lt + acu_view_table_bytes(r), &scratch));
    uint8_t *base = static_cast<uint8_t *>(scratch);
    ViewConcatRows rows{4, n, 0, {}, {}, valid};
    ACU_TRY(acu_view_operand(ctx, l, base + eng + offs, &rows.l));
    ACU_TRY(acu_view_operand(ctx, r, base + eng + offs + lt, &rows.r));
    int32_t *d_offs = reinterpret_cast<int32_t *>(base + eng);
    int64_t *block_tot = reinterpret_cast<int64_t *>(base);
    // the sizing call (out_views == NULL) runs the length pass only: the offsets land in scratch, no byte is copied
    ACU_TRY(engine_launch(ctx, rows, block_tot, d_offs, out_views ? out_data : nullptr, out_data_capacity, (int64_t)INT32_MAX));
    if (out_views) {
      const int64_t blocks = (n + BY_ROWS - 1) / BY_ROWS;
      ViewConcatOut p{rows.l, rows.r, valid, n, d_offs, block_tot + (blocks - 1), out_data_capacity, static_cast<uint4 *>(out_views)};
      ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_concat_views, acu_grid(ctx, (n + 255) / 256, 8), 256, 0, p);
    }
  }
  ACU_TRY(acu_res_fetch(ctx));
  const unsigned long long *h = ctx->h_res;
  *out_data_len = 0;
  union_result(valid, n, h, out_nulls);
  if (n == 0) return ACU_OK;
  if ((int64_t)h[RES_AUX0] > INT32_MAX) return acu_fail(ctx, ACU_ERR_ARITHMETIC_OVERFLOW, -1, 0, 0, h[RES_AUX0], "byte array offset overflow");
  *out_data_len = (int64_t)h[RES_AUX0];
  if (out_views && *out_data_len > out_data_capacity)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, (uint64_t)*out_data_len, "output data capacity %lld < required %lld",
                    (long long)out_data_capacity, (long long)*out_data_len);
  return ACU_OK;
}

extern "C" acu_status acu_concat_elements_fixed_size_binary(acu_ctx *ctx, int32_t l_width, const acu_array *l, int32_t r_width,
                                                            const acu_array *r, int32_t *out_byte_width, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(check_array(ctx, l));
  ACU_TRY(check_array(ctx, r));
  ACU_TRY(same_length(ctx, l, r));
  for (const int32_t w : {l_width, r_width})
    if (w < 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid size of FixedSizeBinaryArray(%d)", (int)w);
  const int64_t w = (int64_t)l_width + r_width;
  if (w > INT32_MAX)  // `output_size as i32` wraps negative: FixedSizeBinaryBuilder::with_capacity panics, rows or not
    return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, -1, 0, 0, 0, "value length (%d) of the array must >= 0", (int)(int32_t)(uint32_t)w);
  *out_byte_width = (int32_t)w;
  const int64_t n = l->len;
  const uint64_t *valid;
  ACU_TRY(union_nulls(ctx, {l, r}, n, out->validity, &valid));
  if (n > 0 && w > 0)
    ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_fsb_concat, acu_grid(ctx, (n + 255) / 256, 8), 256, 0, static_cast<const uint8_t *>(l->values),
                     (int64_t)l_width, static_cast<const uint8_t *>(r->values), (int64_t)r_width, valid, n, static_cast<uint8_t *>(out->values));
  ACU_TRY(acu_res_fetch(ctx));
  union_result(valid, n, ctx->h_res, out);
  return ACU_OK;
}
