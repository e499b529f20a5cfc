// list.cu — filter and take of List / LargeList / FixedSizeList columns, one level per call.
//
//   filter (arrow-select/src/filter.rs:535-625, the MutableArrayData fallback): the list's new offsets are the offsets
//     pass of filter_bytes; the child is filtered with a CHILD PLAN, the parent plan expanded onto child rows by
//     k_list_expand (one thread per 64-bit child word).
//   take (take_list take.rs:646-727, take_fixed_size_list :765-795): the new offsets are the offsets engine's scan of
//     the taken rows' child counts (bytes_engine.cuh with a producer whose "length" is child rows); the child is taken
//     with a CHILD ROW MAP, the absolute child row of every output child row (k_list_row_map, k_fsl_row_map).
//
// Both kernels stay balanced when row lengths are skewed (one row of 1e8 children among millions of empty rows): a
// thread owns a fixed span of child rows and finds the parent row of a span boundary by binary search over the offsets,
// so neither the number of parent rows nor their lengths decide a thread's work.
#include "bitmap.cuh"
#include "bytes_cmp.cuh"
#include "bytes_engine.cuh"
#include "internal.cuh"

const char *const acu_extend_overflow_text =
    "offset overflow: data exceeds the capacity of the offset type. Try splitting into smaller batches or using a larger type "
    "(e.g. LargeStringArray / LargeBinaryArray instead of StringArray / BinaryArray)";

#define RM_ROWS 16  // child rows per lane of the row map (a warp owns 32 x RM_ROWS consecutive rows)

namespace {

// Offset of list row i: ob 4 / 8 reads the offsets, ob 0 is a FixedSizeList (i * size).
__device__ __forceinline__ int64_t list_off(const void *offs, int ob, int64_t size, int64_t i) {
  return ob ? ld_offset(offs, ob, i) : i * size;
}

// The last row r in [lo, n) with off(r) <= c, given off(lo) <= c: for c < off(n) the non-empty row holding child row c.
__device__ __forceinline__ int64_t row_at(const void *offs, int ob, int64_t size, int64_t lo, int64_t n, int64_t c) {
  if (!ob) return c / size;
  if (lo + 1 < n && list_off(offs, ob, size, lo + 1) > c) return lo;  // the common case: still in row lo
  int64_t hi = n;
  while (hi - lo > 1) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if (list_off(offs, ob, size, mid) <= c) lo = mid;
    else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ uint64_t bit_range(int64_t a, int64_t b) {  // bits [a, b) of a word, 0 <= a < b <= 64
  const uint64_t n = (uint64_t)(b - a);
  return (n >= 64 ? ~0ull : ((1ull << n) - 1ull)) << a;
}

// Child predicate: word w covers child rows [64 w, 64 w + 64). Starting at the parent row of its first row, it ORs the
// selected parents' ranges in registers, hopping from range to range (at most 64 hops, each a short search), and stores
// the word once.
__global__ void __launch_bounds__(256) k_list_expand(const uint64_t *__restrict__ pmask, const void *offs, int ob, int64_t size, int64_t n_rows,
                                                     int64_t base, int64_t child_end, uint64_t *__restrict__ cmask, int64_t n_words) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += stride) {
    const int64_t c0 = w << 6, c1 = c0 + 64 < child_end ? c0 + 64 : child_end;
    uint64_t word = 0;
    int64_t c = c0 > base ? c0 : base;
    if (c < c1) {
      int64_t r = row_at(offs, ob, size, 0, n_rows, c);
      while (true) {
        const int64_t e0 = list_off(offs, ob, size, r + 1), e = e0 < c1 ? e0 : c1;
        if ((__ldg(pmask + (r >> 6)) >> (r & 63)) & 1ull) word |= bit_range(c - c0, e - c0);
        c = e;
        if (c >= c1) break;
        r = row_at(offs, ob, size, r + 1, n_rows, c);
      }
    }
    cmask[w] = word;
  }
}

// The offsets engine's producer for take: row j's "length" is the child rows of list row idx[j]; zero for a null index,
// for a null list row unless the ranges of null rows are kept, and for an out-of-bounds index (its row -> *err).
struct ListTakeRows {
  int ob;                  // engine: output offset width (always 8: the row map searches the exact offsets)
  int64_t m;               // output rows
  const uint8_t *data;     // engine: unused (no bytes are copied)
  int detect_oob;
  const void *offs;        // list offsets
  int lob;                 // their width
  const void *idx;
  int kind;                // acu_take_index_kind
  int64_t n_src;           // list rows
  const uint8_t *ivalid;   // index validity (only with nulls), or NULL
  int64_t ivoff;
  const uint8_t *lvalid;   // list validity when null rows get an empty range, or NULL
  int64_t lvoff;
  __device__ __forceinline__ void ranges4(int64_t j0, int64_t begin[4], uint64_t len[4], unsigned long long *err) const {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int64_t j = j0 + k;
      begin[k] = 0;
      len[k] = 0;
      if (j >= m || (ivalid && !ld_bit(ivalid, ivoff + j))) continue;
      const uint64_t ix = ld_index(idx, kind, j);
      if (ix >= (uint64_t)n_src) {
        if ((unsigned long long)j < *err) *err = (unsigned long long)j;
        continue;
      }
      if (lvalid && !ld_bit(lvalid, lvoff + (int64_t)ix)) continue;
      len[k] = (uint64_t)(ld_offset(offs, lob, (int64_t)ix + 1) - ld_offset(offs, lob, (int64_t)ix));
    }
  }
};

// Child row map of a List / LargeList take: output child row c lies in output row r (new_off[r] <= c < new_off[r + 1])
// and maps to src_off[idx[r]] + (c - new_off[r]). Lane rows are c0 + lane + 32 i, so stores coalesce; a lane searches
// again only when it crosses into another row.
template <class OutT>
__global__ void __launch_bounds__(256) k_list_row_map(const int64_t *__restrict__ new_off, int64_t m, const void *offs, int lob,
                                                      const void *idx, int kind, int64_t total, OutT *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t c0 = warp * (32 * RM_ROWS); c0 < total; c0 += nwarps * (32 * RM_ROWS)) {
    int64_t r = -1, end = -1, shift = 0;
#pragma unroll 4
    for (int i = 0; i < RM_ROWS; ++i) {
      const int64_t c = c0 + lane + 32 * i;
      if (c >= total) break;
      if (c >= end) {
        r = row_at(new_off, 8, 0, r < 0 ? 0 : r + 1, m, c);
        end = __ldg(new_off + r + 1);
        shift = ld_offset(offs, lob, (int64_t)ld_index(idx, kind, r)) - __ldg(new_off + r);
      }
      out[c] = (OutT)(c + shift);
    }
  }
}

// FixedSizeList: output child row c = i * size + k maps to (u32)(idx[i] * size) + k (take_value_indices_from_fixed_size_list:
// the reference's `index as i32 * size`, then `as u32`, is the low 32 bits of the product, taken here in u32 arithmetic),
// 0 and null for a null index. The row of c is a 32-bit division while the map fits u32 positions; the validity word of
// 64 child rows walks (i, k) forward from one division.
__global__ void __launch_bounds__(256) k_fsl_row_map(const void *idx, int kind, const uint8_t *ivalid, int64_t ivoff, int64_t size,
                                                     int64_t total, uint32_t *__restrict__ out, uint64_t *__restrict__ out_valid) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const bool narrow = total <= (int64_t)UINT32_MAX;
  const uint32_t s32 = (uint32_t)size;
  for (int64_t c = t0; c < total; c += stride) {
    const int64_t i = narrow ? (int64_t)((uint32_t)c / s32) : c / size;
    uint32_t v = 0;
    if (!ivalid || ld_bit(ivalid, ivoff + i)) v = (uint32_t)ld_index(idx, kind, i) * s32 + (uint32_t)(c - i * size);
    out[c] = v;
  }
  if (!out_valid) return;
  for (int64_t w = t0; w < (total + 63) / 64; w += stride) {
    int64_t i = (w << 6) / size, k = (w << 6) - i * size;
    uint64_t word = 0;
    for (int b = 0; b < 64 && (w << 6) + b < total; ++b) {
      word |= (uint64_t)ld_bit(ivalid, ivoff + i) << b;
      if (++k == size) { k = 0; ++i; }
    }
    out_valid[w] = word;
  }
}

__global__ void k_narrow_offsets(const int64_t *__restrict__ src, int64_t n, int32_t *__restrict__ dst) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = (int32_t)src[i];
}

acu_status check_list(acu_ctx *ctx, const acu_list_array *l) {
  if (l->kind == ACU_FIXED_SIZE_LIST) {
    if (l->list_size < 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "list_size must be >= 0, got %d", (int)l->list_size);
    return ACU_OK;
  }
  if (l->kind != ACU_LIST && l->kind != ACU_LARGE_LIST)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "unknown list kind %d", (int)l->kind);
  const int ob = l->kind == ACU_LIST ? 4 : 8;
  if ((uintptr_t)l->offsets % (uintptr_t)ob != 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "offsets must be %d-byte aligned", ob);
  return ACU_OK;
}

int list_ob(const acu_list_array *l) { return l->kind == ACU_LIST ? 4 : l->kind == ACU_LARGE_LIST ? 8 : 0; }

acu_status read_offset(acu_ctx *ctx, const acu_list_array *l, int64_t i, int64_t *v) {
  const int ob = list_ob(l);
  if (!ob) { *v = i * l->list_size; return ACU_OK; }
  int64_t raw = 0;
  ACU_CUDA(ctx, cudaMemcpy(&raw, static_cast<const uint8_t *>(l->offsets) + (size_t)i * ob, (size_t)ob, cudaMemcpyDeviceToHost));
  *v = ob == 4 ? (int64_t)(int32_t)raw : raw;
  return ACU_OK;
}

}  // namespace

extern "C" acu_status acu_filter_list(acu_ctx *ctx, const acu_filter_plan *plan, const acu_list_array *list, void *out_offsets,
                                      acu_array_out *out_nulls, acu_filter_plan **out_child_plan) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  *out_child_plan = nullptr;
  ACU_TRY(check_list(ctx, list));
  const int ob = list_ob(list);
  if (ob) {  // the offsets pass of filter_bytes: the selected rows' child counts, rebased to 0, and filter_nulls
    int64_t total = 0;
    ACU_TRY(acu_filter_bytes(ctx, plan, ob, list->offsets, nullptr, &list->nulls, out_offsets, nullptr, 0, &total, out_nulls));
  } else {
    ACU_TRY(acu_res_reset(ctx));
    const int kind = 2;
    const int32_t width = 0;
    int mode = 0;
    const acu_array *v = &list->nulls;
    unsigned long long *res = acu_dres(ctx, 0);
    ACU_TRY(acu_filter_cols_launch(ctx, plan, 1, &kind, &width, &v, &out_nulls, &res, &mode));
    ACU_TRY(acu_res_fetch(ctx));
    acu_filter_col_finalize(plan, mode, acu_hres(ctx, 0), out_nulls);
  }
  // the child plan over [0, offsets[plan len])
  const int64_t n = acu_filter_plan_len(plan);
  int64_t base = 0, child_end = 0;
  ACU_TRY(read_offset(ctx, list, 0, &base));
  ACU_TRY(read_offset(ctx, list, n, &child_end));
  const int64_t n_words = (child_end + 63) / 64;
  void *cmask = nullptr;
  ACU_TRY(acu_malloc(ctx, (size_t)n_words * 8 + 8, &cmask));
  if (n > 0 && n_words > 0 && acu_filter_plan_count(plan) > 0) {
    ACU_LAUNCH_TIMED(ctx, ACU_K_FILTER_PLAN, k_list_expand, acu_grid(ctx, (n_words + 255) / 256, 8), 256, 0, acu_plan_mask(plan), list->offsets, ob,
                     (int64_t)list->list_size, n, base, child_end, static_cast<uint64_t *>(cmask), n_words);
  } else {
    ACU_CUDA(ctx, cudaMemsetAsync(cmask, 0, (size_t)n_words * 8 + 8, ctx->stream));
  }
  acu_array pred{};
  pred.values = cmask;
  pred.len = child_end;
  const acu_status st = acu_filter_plan_create(ctx, &pred, out_child_plan);
  acu_kstats_drain(ctx);
  acu_free(ctx, cmask);
  return st;
}

extern "C" acu_status acu_take_list(acu_ctx *ctx, const acu_list_array *list, const acu_array *indices, acu_dtype index_dtype,
                                    int32_t check_bounds, int32_t keep_null_ranges, void *out_offsets, acu_array_out *out_nulls,
                                    acu_dtype child_index_dtype, void *out_child_indices, int64_t capacity, int64_t *out_child_rows,
                                    acu_array_out *out_child_index_nulls) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  *out_child_rows = 0;
  ACU_TRY(check_list(ctx, list));
  const int ob = list_ob(list);
  const int kind = acu_take_index_kind(index_dtype);
  if (kind < 0)  // take.rs:103
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Take only supported for integers, got %s", acu_dtype_name(index_dtype));
  if (child_index_dtype != ACU_U32 && (child_index_dtype != ACU_U64 || !ob))
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "child row map must be UInt32%s", ob ? " or UInt64" : "");
  if (child_index_dtype == ACU_U32 && ob && list->child_len > (int64_t)UINT32_MAX)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "child of %lld rows needs a UInt64 row map", (long long)list->child_len);
  acu_status st;
  const int64_t m = indices->len, n = list->nulls.len;
  const int64_t inc = m > 0 ? acu_resolve_null_count(ctx, indices, &st) : 0;
  if (m > 0) ACU_TRY(st);
  const bool idx_nulls = indices->validity && inc > 0;
  if (keep_null_ranges && idx_nulls) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "take_list: a child step's row map has a null");
  if (check_bounds) ACU_TRY(acu_take_check_bounds(ctx, indices, index_dtype, idx_nulls, n));
  out_nulls->len = m;
  out_nulls->has_validity = 0;
  out_nulls->null_count = 0;
  if (out_child_index_nulls) {
    out_child_index_nulls->has_validity = 0;
    out_child_index_nulls->null_count = 0;
  }
  if (m == 0) {
    if (ob) ACU_CUDA(ctx, cudaMemsetAsync(out_offsets, 0, (size_t)ob, ctx->stream));
    ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return ACU_OK;
  }
  const int64_t lnc = n > 0 ? acu_resolve_null_count(ctx, &list->nulls, &st) : 0;
  if (n > 0) ACU_TRY(st);
  const char val_nulls = list->nulls.validity && lnc > 0;
  // nulls = take_nulls(list.nulls, indices): the validity-only take (with list nulls it also finds a valid out-of-bounds
  // index, take_bits' panic)
  ACU_TRY(acu_res_reset(ctx));
  unsigned long long *res = acu_dres(ctx, 0);
  const int32_t zero = 0;
  const char not_bool = 0;
  const acu_array *lv = &list->nulls;
  int mode = 0;
  ACU_TRY(acu_take_cols_launch(ctx, 1, &zero, &lv, &not_bool, &val_nulls, indices, index_dtype, idx_nulls, &out_nulls, &res, &mode));
  int64_t *off64 = nullptr;
  if (ob) {
    // the new offsets, exact in i64 (for a List narrowed afterwards): the engine's block totals and scan over child counts
    void *scratch = nullptr;
    const size_t eng = engine_scratch(m);
    ACU_TRY(acu_scratch(ctx, eng + (ob == 4 ? align256((size_t)(m + 1) * 8) : 0), &scratch));
    off64 = ob == 8 ? static_cast<int64_t *>(out_offsets) : reinterpret_cast<int64_t *>(static_cast<uint8_t *>(scratch) + eng);
    ListTakeRows rows{8, m, nullptr, 0, list->offsets, ob, indices->values, kind, n,
                      idx_nulls ? indices->validity : nullptr, indices->validity_offset,
                      (val_nulls && !keep_null_ranges) ? list->nulls.validity : nullptr, list->nulls.validity_offset};
    ACU_TRY(engine_launch(ctx, rows, static_cast<int64_t *>(scratch), off64, nullptr, 0, ob == 4 ? (int64_t)INT32_MAX : INT64_MAX));
    if (ob == 4)
      ACU_LAUNCH(ctx, k_narrow_offsets, acu_grid(ctx, (m + 1 + 255) / 256, 8), 256, 0, off64, m + 1, static_cast<int32_t *>(out_offsets));
  }
  ACU_TRY(acu_res_fetch(ctx));
  const unsigned long long *h = acu_hres(ctx, 0);
  const unsigned long long oob = h[RES_ERR_INDEX], ovf = ob == 4 ? h[RES_ERR2] : ~0ull;
  const int64_t total = ob ? (int64_t)h[RES_AUX0] : m * (int64_t)list->list_size;
  // take_nulls -> take_bits -> BooleanBuffer::value (arrow-buffer/src/buffer/boolean.rs). A FixedSizeList takes its child
  // first (take.rs:770-785): the panic is returned by the call that writes the row map, after writing it
  const bool bit_len_panic = oob != ~0ull && val_nulls;
  auto bit_len_fail = [&]() {
    return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, (int64_t)oob, 0, 0, (uint64_t)n, "assertion failed: idx < self.bit_len");
  };
  if (oob != ~0ull && (val_nulls || oob < ovf) && ob) {
    if (val_nulls) return bit_len_fail();
    uint64_t raw = 0;
    const int sz = acu_dtype_size(index_dtype);
    ACU_CUDA(ctx, cudaMemcpy(&raw, static_cast<const uint8_t *>(indices->values) + (size_t)oob * sz, sz, cudaMemcpyDeviceToHost));
    uint64_t ix = raw;  // ToIndices: i8 / i16 sign-extend to u32, i32 reinterprets
    if (index_dtype == ACU_I8) ix = (uint32_t)(int32_t)(int8_t)raw;
    else if (index_dtype == ACU_I16) ix = (uint32_t)(int32_t)(int16_t)raw;
    else if (index_dtype == ACU_I32) ix = (uint32_t)raw;
    // list_offsets[ix] then list_offsets[ix + 1] over a slice of len + 1 offsets
    const unsigned long long bad = ix == (uint64_t)n ? ix + 1 : ix;
    return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, (int64_t)oob, ix, 0, (uint64_t)n, "index out of bounds: the len is %lld but the index is %llu",
                    (long long)n + 1, bad);
  }
  if (ovf != ~0ull) {
    if (keep_null_ranges) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, (int64_t)ovf, 0, 0, 0, "%s", acu_extend_overflow_text);
    return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, (int64_t)ovf, 0, 0, 0, "called `Option::unwrap()` on a `None` value");
  }
  if (!bit_len_panic) {
    // without list nulls take_fixed_size_list reads no list row (is_null of a list without a NullBuffer): a valid index
    // past the list is the child take's to report, or nothing when (u32)(index * size) + k lands back in the child
    unsigned long long hf[RES_SLOTS];
    std::copy(h, h + RES_SLOTS, hf);
    if (!ob && !val_nulls) hf[RES_ERR_INDEX] = ~0ull;
    ACU_TRY(acu_take_col_finalize(ctx, &list->nulls, indices, index_dtype, mode, hf, out_nulls));
    if (!ob && out_nulls->null_count == 0) out_nulls->has_validity = 0;  // NullBuffer::from_unsliced_buffer
  }
  *out_child_rows = total;
  if (out_child_indices == nullptr) return ACU_OK;
  if (total == 0) return bit_len_panic ? bit_len_fail() : ACU_OK;
  if (capacity < total)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, (uint64_t)total, "take_list: capacity %lld < %lld child rows", (long long)capacity,
                    (long long)total);
  if (ob) {
    const int grid = acu_grid(ctx, (total + 32 * RM_ROWS * 8 - 1) / (32 * RM_ROWS * 8), 8);
    if (child_index_dtype == ACU_U32)
      ACU_LAUNCH_TIMED(ctx, ACU_K_TAKE, k_list_row_map<uint32_t>, grid, 256, 0, off64, m, list->offsets, ob, indices->values, kind, total,
                       static_cast<uint32_t *>(out_child_indices));
    else
      ACU_LAUNCH_TIMED(ctx, ACU_K_TAKE, k_list_row_map<uint64_t>, grid, 256, 0, off64, m, list->offsets, ob, indices->values, kind, total,
                       static_cast<uint64_t *>(out_child_indices));
  } else {
    uint64_t *cv = idx_nulls && out_child_index_nulls ? reinterpret_cast<uint64_t *>(out_child_index_nulls->validity) : nullptr;
    ACU_LAUNCH_TIMED(ctx, ACU_K_TAKE, k_fsl_row_map, acu_grid(ctx, (total + 255) / 256, 8), 256, 0, indices->values, kind,
                     idx_nulls ? indices->validity : nullptr, indices->validity_offset, (int64_t)list->list_size, total,
                     static_cast<uint32_t *>(out_child_indices), cv);
    if (cv) {
      out_child_index_nulls->len = total;
      out_child_index_nulls->has_validity = 1;
      out_child_index_nulls->null_count = inc * (int64_t)list->list_size;
    }
  }
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  acu_kstats_drain(ctx);
  return bit_len_panic ? bit_len_fail() : ACU_OK;
}
