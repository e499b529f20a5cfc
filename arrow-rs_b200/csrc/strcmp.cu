// strcmp.cu — arrow-ord/src/cmp.rs on variable-width operands (SURVEY.md §8(f) rank 3):
//
//   eq / neq / lt / lt_eq / gt / gt_eq / distinct / not_distinct over
//     GenericByteArray      (Utf8, Binary: i32 offsets; LargeUtf8, LargeBinary: i64)   ArrayOrd cmp.rs:783-801
//     GenericByteViewArray  (Utf8View, BinaryView)                                      ArrayOrd cmp.rs:803-898
//   and the short-constant fast path of views, eq_inline_scalar                          cmp.rs:282-300, :405-435
//
// compare_op's host-side decisions (length check, null scalars, operand swap, negation, fold, NullBuffer) are made by
// acu_cmp_decide (internal.cuh), as for primitives. Value bits are computed at every slot. One thread per row, 4 rows per
// lane in flight, result bits packed with a warp ballot (lane == bit), lane 0 of each 32-row group owns the group's
// 32-bit value and validity words.
// Roofline: 2 offsets + the compared bytes per side (byte arrays), 16 B per view (views); HBM-bound.
#include "bitmap.cuh"
#include "bytes_cmp.cuh"
#include "internal.cuh"

namespace {

struct RowCmpCommon {
  int64_t n;
  const uint8_t *av, *bv;  // validity of the two (possibly swapped) operands, NULL = no nulls
  int64_t aoff, boff;
  int a_scalar, b_scalar;
  int a_null_scalar, b_null_scalar;
  int lt;                  // 1: is_lt(a, b), 0: is_eq(a, b)
  int neg, fold;
  uint32_t *out_bits, *out_valid;
  unsigned long long *res;
};

__device__ __forceinline__ bool view_is_lt(const ViewOperand &L, const uint4 &l, const uint4 *lslot, const ViewOperand &R, const uint4 &r,
                                           const uint4 *rslot) {  // cmp.rs:864-893
  if (L.n_buffers == 0 && R.n_buffers == 0) return inline_key_lt(l, r);
  if (l.x <= 12u && r.x <= 12u) return inline_key_lt(l, r);
  if (l.y != r.y) return __byte_perm(l.y, 0, 0x0123) < __byte_perm(r.y, 0, 0x0123);
  const BytesItem a = L.item(l, lslot), b = R.item(r, rslot);
  return bytes_lt(a.p, a.len, b.p, b.len);
}

// lane 0 of a 32-row group turns the ballot into the value / validity words (the word-level part of compare_op)
__device__ __forceinline__ void finish_group(const RowCmpCommon &p, int64_t row0, uint32_t v, int lane, unsigned &valid_cnt) {
  if (lane != 0) return;
  const int64_t left = p.n - row0;
  const uint32_t m = left >= 32 ? 0xffffffffu : ((1u << left) - 1u);
  if (p.neg) v = ~v;
  v &= m;
  uint32_t l = p.a_null_scalar ? 0u : m, r = p.b_null_scalar ? 0u : m;
  if (p.av) l &= ld_bits32(p.av, p.aoff + row0, p.aoff + p.n);
  if (p.bv) r &= ld_bits32(p.bv, p.boff + row0, p.boff + p.n);
  if (p.fold == FOLD_DISTINCT) v = (l ^ r) | (l & r & v);                  // cmp.rs:331
  else if (p.fold == FOLD_NOT_DISTINCT) v = (~(l | r) & m) | (l & r & v);  // cmp.rs:341
  p.out_bits[row0 >> 5] = v;
  if (p.out_valid) {
    p.out_valid[row0 >> 5] = l & r;
    valid_cnt += __popc(l & r);
  }
}

constexpr int ROWS_PER_LANE = 4;

// byte arrays compare the items; views compare the view words first and read a value's bytes only when they must
__device__ __forceinline__ BytesItem cmp_scalar(const BytesOperand &s) { return s.item(0); }
__device__ __forceinline__ uint4 cmp_scalar(const ViewOperand &s) { return __ldg(s.views); }
__device__ __forceinline__ BytesItem cmp_load(const BytesOperand &s, int64_t i) { return s.item(i); }
__device__ __forceinline__ uint4 cmp_load(const ViewOperand &s, int64_t i) { return s.view(i); }
__device__ __forceinline__ bool cmp_row(const RowCmpCommon &p, const BytesOperand &, const BytesItem &a, const BytesOperand &, const BytesItem &b,
                                        int64_t) {
  return p.lt ? bytes_lt(a.p, a.len, b.p, b.len) : bytes_eq(a.p, a.len, b.p, b.len);
}
__device__ __forceinline__ bool cmp_row(const RowCmpCommon &p, const ViewOperand &A, const uint4 &a, const ViewOperand &B, const uint4 &b,
                                        int64_t i) {
  const uint4 *as = A.views + (p.a_scalar ? 0 : i), *bs = B.views + (p.b_scalar ? 0 : i);
  return p.lt ? view_is_lt(A, a, as, B, b, bs) : view_is_eq(A, a, as, B, b, bs);
}

// One kernel for both layouts (Op = BytesOperand or ViewOperand): only the row read and the compare differ.
template <class Op>
__global__ void __launch_bounds__(256) k_cmp_rows(const RowCmpCommon p, const Op A, const Op B) {
  using Row = decltype(cmp_load(A, 0));
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t groups = (p.n + 31) >> 5;
  unsigned valid_cnt = 0;
  Row sa{}, sb{};
  if (p.a_scalar) sa = cmp_scalar(A);
  if (p.b_scalar) sb = cmp_scalar(B);
  for (int64_t g0 = warp * ROWS_PER_LANE; g0 < groups; g0 += nwarps * ROWS_PER_LANE) {
    Row ia[ROWS_PER_LANE], ib[ROWS_PER_LANE];
#pragma unroll
    for (int k = 0; k < ROWS_PER_LANE; ++k) {  // the offset / view loads of 4 rows in flight
      const int64_t i = (g0 + k) * 32 + lane;
      const bool live = i < p.n;
      ia[k] = p.a_scalar ? sa : (live ? cmp_load(A, i) : Row{});
      ib[k] = p.b_scalar ? sb : (live ? cmp_load(B, i) : Row{});
    }
#pragma unroll
    for (int k = 0; k < ROWS_PER_LANE; ++k) {
      const int64_t row0 = (g0 + k) * 32;
      if (row0 >= p.n) break;  // warp-uniform
      const int64_t i = row0 + lane;
      bool r = false;
      if (i < p.n) r = cmp_row(p, A, ia[k], B, ib[k], i);
      finish_group(p, row0, __ballot_sync(ACU_FULL_MASK, r), lane, valid_cnt);
    }
  }
  if (p.out_valid && lane == 0 && valid_cnt) atomicAdd(p.res + RES_COUNT, (unsigned long long)valid_cnt);
}

// eq_inline_scalar (cmp.rs:405-435): (view as u64 & significant) == needle at every slot; 8 rows per lane in flight
__global__ void __launch_bounds__(256) k_view_eq_inline(const uint4 *__restrict__ views, int64_t n, uint64_t significant, uint64_t needle, int neg,
                                                        uint32_t *__restrict__ out_bits) {
  constexpr int U = 8;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t groups = (n + 31) >> 5;
  for (int64_t g0 = warp * U; g0 < groups; g0 += nwarps * U) {
    uint64_t lo[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int64_t i = (g0 + k) * 32 + lane;
      lo[k] = i < n ? ld_stream8(views + i) : ~needle;  // the low 64 bits of the view: length + prefix
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const int64_t row0 = (g0 + k) * 32;
      if (row0 >= n) break;
      uint32_t v = __ballot_sync(ACU_FULL_MASK, (lo[k] & significant) == needle);
      if (lane == 0) {
        const int64_t left = n - row0;
        const uint32_t m = left >= 32 ? 0xffffffffu : ((1u << left) - 1u);
        if (neg) v = ~v;
        out_bits[row0 >> 5] = v & m;
      }
    }
  }
}

// ---- host side -------------------------------------------------------------------------------------------------------
RowCmpCommon row_cmp_params(acu_ctx *ctx, const acu_cmp_decision &d, acu_array_out *out) {
  return RowCmpCommon{d.len, d.av, d.bv, d.aoff, d.boff, d.a_scalar, d.b_scalar, d.a_null_scalar, d.b_null_scalar, d.lt, d.neg, d.fold,
                      static_cast<uint32_t *>(out->values), d.has_validity ? reinterpret_cast<uint32_t *>(out->validity) : nullptr,
                      ctx->d_res};
}

int cmp_grid(acu_ctx *ctx, int64_t n, int rows_per_lane) {
  const int64_t groups = (n + 31) / 32;
  return acu_grid(ctx, ((groups + rows_per_lane - 1) / rows_per_lane + 7) / 8, 16);
}

}  // namespace

extern "C" acu_status acu_cmp_bytes(acu_ctx *ctx, int32_t offset_bytes, acu_cmp_op op, const acu_bytes_array *l, const acu_bytes_array *r,
                                    acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  ACU_TRY(acu_offset_width_check(ctx, offset_bytes));
  acu_cmp_decision d;
  ACU_TRY(acu_cmp_decide(ctx, op, &l->nulls, &r->nulls, out, &d));
  if (d.len == 0) return ACU_OK;
  if (d.all_null) return acu_new_null(ctx, d.len, acu_bitmap_bytes(d.len), out);
  const acu_bytes_array *x = d.swap ? r : l, *y = d.swap ? l : r;
  const BytesOperand A{x->offsets, x->data, offset_bytes}, B{y->offsets, y->data, offset_bytes};
  ACU_TRY(acu_res_reset(ctx));
  ACU_LAUNCH_TIMED(ctx, ACU_K_CMP, k_cmp_rows<BytesOperand>, cmp_grid(ctx, d.len, ROWS_PER_LANE), 256, 0, row_cmp_params(ctx, d, out), A, B);
  ACU_TRY(acu_res_fetch(ctx));
  acu_cmp_finalize(d, ctx->h_res, out);
  return ACU_OK;
}

extern "C" acu_status acu_cmp_byte_view(acu_ctx *ctx, acu_cmp_op op, const acu_view_array *l, const acu_view_array *r, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  const bool ls = l->nulls.is_scalar != 0, rs = r->nulls.is_scalar != 0;
  // eq_inline_scalar (cmp.rs:282-300): == / != of an array against a non-null constant of <= 4 bytes
  if ((op == ACU_EQ || op == ACU_NEQ) && ls != rs) {
    const acu_view_array *arr = ls ? r : l, *sc = ls ? l : r;
    acu_status st;
    const int64_t snc = sc->nulls.len >= 1 ? acu_resolve_null_count(ctx, &sc->nulls, &st) : 1;
    if (sc->nulls.len >= 1) ACU_TRY(st);
    if (sc->nulls.len >= 1 && snc == 0) {
      uint64_t low = 0;
      ACU_TRY(acu_memcpy_d2h(ctx, &low, sc->views, 8));
      const uint32_t needle_len = (uint32_t)low;
      if (needle_len <= 4) {
        const uint64_t significant = ~0ull >> (32 - needle_len * 8);
        const int64_t n = arr->nulls.len;
        out->len = n;
        out->has_validity = 0;
        out->null_count = 0;
        if (n == 0) return ACU_OK;
        const int64_t anc = acu_resolve_null_count(ctx, &arr->nulls, &st);
        ACU_TRY(st);
        ACU_LAUNCH_TIMED(ctx, ACU_K_CMP, k_view_eq_inline, cmp_grid(ctx, n, 8), 256, 0, static_cast<const uint4 *>(arr->views), n, significant,
                         low & significant, op == ACU_NEQ ? 1 : 0, static_cast<uint32_t *>(out->values));
        if (arr->nulls.validity && anc > 0) {  // nulls = values_nulls.filter(null_count > 0)
          ACU_TRY(acu_bitmap_and_launch(ctx, arr->nulls.validity, arr->nulls.validity_offset, nullptr, 0, n,
                                        reinterpret_cast<uint64_t *>(out->validity), false));
          out->has_validity = 1;
          out->null_count = anc;
        }
        ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        acu_kstats_drain(ctx);
        return ACU_OK;
      }
    }
  }
  acu_cmp_decision d;
  ACU_TRY(acu_cmp_decide(ctx, op, &l->nulls, &r->nulls, out, &d));
  if (d.len == 0) return ACU_OK;
  if (d.all_null) return acu_new_null(ctx, d.len, acu_bitmap_bytes(d.len), out);
  const acu_view_array *x = d.swap ? r : l, *y = d.swap ? l : r;
  // the data-buffer pointer tables go to the device (scratch): [x buffers][y buffers]
  void *scratch;
  ACU_TRY(acu_scratch(ctx, acu_view_table_bytes(x) + acu_view_table_bytes(y), &scratch));
  ViewOperand A, B;
  ACU_TRY(acu_view_operand(ctx, x, scratch, &A));
  ACU_TRY(acu_view_operand(ctx, y, static_cast<uint8_t *>(scratch) + acu_view_table_bytes(x), &B));
  ACU_TRY(acu_res_reset(ctx));
  ACU_LAUNCH_TIMED(ctx, ACU_K_CMP, k_cmp_rows<ViewOperand>, cmp_grid(ctx, d.len, ROWS_PER_LANE), 256, 0, row_cmp_params(ctx, d, out), A, B);
  ACU_TRY(acu_res_fetch(ctx));
  acu_cmp_finalize(d, ctx->h_res, out);
  return ACU_OK;
}
