// aggregate_bytes.cu — arrow-arith/src/aggregate.rs min / max of variable-width and fixed-width binary columns, and of
// boolean columns, on the device.
//
//   min_max_helper        (aggregate.rs:460-485)  GenericByteArray (Utf8 / Binary, i32 or i64 offsets), FixedSizeBinary
//   min_max_view_helper   (aggregate.rs:491-518)  GenericByteViewArray (Utf8View / BinaryView)
//   min_boolean / max_boolean, bool_and / bool_or (aggregate.rs:372-457, :880-889)
//
// The reference folds the valid rows in ascending order and replaces its accumulator only on a strict < / >, so its answer
// is the LOWEST logical row holding the extremal value. The device returns that row: candidates are ordered by
// (value, row), a total order, so any merge tree gives the same answer for any grid.
//
// Design: the structure of k_reduce (reduce.cu). One streaming pass; lane l owns validity word l of each 2048-row
// super-group; per-lane accumulator -> warp shuffle tree -> per-CTA partial in scratch -> the last CTA (atomic ticket) folds
// the partials. The accumulator is (key, row, bytes, length), the key a 64-bit value that orders like the bytes: the first
// min(len, 8) bytes big endian, zero-padded, for byte arrays and FixedSizeBinary; the 4-byte prefix for views (all a view
// holds for a long value). A smaller key decides alone; on equal keys a value no longer than the key is a prefix of the
// other, so the length decides; only when both are longer are the remaining bytes compared (bytes_lt). Null slots are
// never read: neither their bytes nor their views.
// Algorithmic bytes: byte arrays 2 offsets (shared between neighbours: (N+1) x offset width) + the first <= 8 bytes of each
// valid value + N/8 of validity, plus the tail bytes of key ties; views 16N + N/8, plus the bytes of key ties; fixed width
// min(width, 8) x N + N/8, plus ties. Boolean: one popcount pass of values & validity (acu_bitmap_and_launch).
#include "bitmap.cuh"
#include "bytes_cmp.cuh"
#include "internal.cuh"

namespace {

struct Cand {
  uint64_t key;
  int64_t row;  // -1: no candidate yet
  const uint8_t *p;
  int64_t len;
};

// item accessors: load(i) reads the row's value descriptor and key; KEY_BYTES = how many leading bytes the key holds
struct BytesSrc {
  static constexpr int KEY_BYTES = 8;
  BytesOperand s;
  __device__ __forceinline__ Cand load(int64_t i) const {
    const BytesItem it = s.item(i);
    return Cand{bswap64(ld_upto8(it.p, (uint32_t)(it.len < 8 ? it.len : 8))), i, it.p, it.len};
  }
};
struct FixedSrc {
  static constexpr int KEY_BYTES = 8;
  const uint8_t *data;
  int64_t width;
  __device__ __forceinline__ Cand load(int64_t i) const {
    const uint8_t *p = data + i * width;
    return Cand{bswap64(ld_upto8(p, (uint32_t)(width < 8 ? width : 8))), i, p, width};
  }
};
struct ViewSrc {
  static constexpr int KEY_BYTES = 4;
  ViewOperand s;
  __device__ __forceinline__ Cand load(int64_t i) const {
    const uint4 v = s.view(i);
    const uint32_t nb = v.x < 4u ? v.x : 4u;
    const uint32_t prefix = nb == 4u ? v.y : (v.y & ((1u << (nb * 8u)) - 1u));
    const BytesItem it = s.item(v, s.views + i);  // a long value's bytes are only read on a key tie
    return Cand{(uint64_t)__byte_perm(prefix, 0, 0x0123) << 32, i, it.p, it.len};
  }
};

// true iff c comes strictly before a in the (value, row) order of OP: smaller (MIN) / larger (MAX) value, then lower row
template <int OP, int KB> __device__ __forceinline__ bool wins(const Cand &c, const Cand &a) {
  if (c.row < 0) return false;
  if (a.row < 0) return true;
  if (c.key != a.key) return OP == ACU_MIN ? c.key < a.key : c.key > a.key;
  if (c.len <= KB || a.len <= KB) {  // equal keys: the shorter value is a prefix of the other
    if (c.len != a.len) return OP == ACU_MIN ? c.len < a.len : c.len > a.len;
    return c.row < a.row;
  }
  const uint8_t *cp = c.p + KB, *ap = a.p + KB;
  const int64_t cl = c.len - KB, al = a.len - KB;
  if (c.row < a.row)  // c wins unless a's value is strictly better
    return !(OP == ACU_MIN ? bytes_lt(ap, al, cp, cl) : bytes_lt(cp, cl, ap, al));
  return OP == ACU_MIN ? bytes_lt(cp, cl, ap, al) : bytes_lt(ap, al, cp, cl);
}

__device__ __forceinline__ Cand shfl_down_cand(const Cand &c, int o) {
  Cand r;
  r.key = __shfl_down_sync(ACU_FULL_MASK, (unsigned long long)c.key, o);
  r.row = __shfl_down_sync(ACU_FULL_MASK, (long long)c.row, o);
  r.p = reinterpret_cast<const uint8_t *>(__shfl_down_sync(ACU_FULL_MASK, (unsigned long long)(uintptr_t)c.p, o));
  r.len = __shfl_down_sync(ACU_FULL_MASK, (long long)c.len, o);
  return r;
}

struct ArgArgs {
  int64_t n;
  const uint8_t *valid;     // validity (NULL: no nulls)
  int64_t voff;
  Cand *partial;            // one candidate per CTA
  unsigned long long *res;  // RES_COUNT valid rows, RES_AUX0 the row (~0: None), RES_AUX3 ticket (zero on entry and on exit)
};

template <int OP, class Src>
__global__ void __launch_bounds__(256) k_arg_extreme(const ArgArgs p, const Src src) {
  constexpr int KB = Src::KEY_BYTES;
  constexpr int U = 4;  // strips (64 rows) in flight per warp: 4 x 2 rows per lane
  __shared__ Cand s_part[8];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n = p.n;
  const int64_t sgroups = (n + 2047) >> 11;  // super-group = 32 strips = 2048 rows = 32 validity words
  Cand acc{0, -1, nullptr, 0};
  unsigned valid_cnt = 0;
  for (int64_t sg = warp; sg < sgroups; sg += nwarps) {
    const int64_t sbase = sg << 11;
    const int64_t wrow = sbase + lane * 64;
    const int64_t k = n - wrow;
    uint64_t vw = k >= 64 ? ~0ull : (k <= 0 ? 0ull : ((~0ull) >> (64 - k)));
    if (p.valid) vw &= ld_bits64(p.valid, p.voff + wrow, p.voff + n);
    valid_cnt += __popcll(vw);
#pragma unroll 1
    for (int s0 = 0; s0 < 32; s0 += U) {
      if (sbase + s0 * 64 >= n) break;
      Cand c[U][2];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint64_t w = __shfl_sync(ACU_FULL_MASK, vw, s0 + u);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int64_t i = sbase + (s0 + u) * 64 + h * 32 + lane;
          c[u][h] = ((w >> (h * 32 + lane)) & 1ull) ? src.load(i) : Cand{0, -1, nullptr, 0};
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u)
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (wins<OP, KB>(c[u][h], acc)) acc = c[u][h];
    }
  }
  valid_cnt = warp_sum(valid_cnt);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const Cand other = shfl_down_cand(acc, o);
    if (wins<OP, KB>(other, acc)) acc = other;
  }
  if (lane == 0) {
    s_part[wid] = acc;
    if (valid_cnt) atomicAdd(p.res + RES_COUNT, (unsigned long long)valid_cnt);
  }
  __syncthreads();
  unsigned int *ticket = reinterpret_cast<unsigned int *>(p.res + RES_AUX3);
  if (threadIdx.x == 0) {
    Cand b = s_part[0];
    for (int w = 1; w < 8; ++w)
      if (wins<OP, KB>(s_part[w], b)) b = s_part[w];
    p.partial[blockIdx.x] = b;
    __threadfence();
    s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (s_last && wid == 0) {  // fold of the per-CTA partials
    __threadfence();
    Cand f{0, -1, nullptr, 0};
    for (unsigned i = lane; i < gridDim.x; i += 32) {
      const volatile Cand *q = p.partial + i;
      const Cand x{q->key, q->row, q->p, q->len};
      if (wins<OP, KB>(x, f)) f = x;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const Cand other = shfl_down_cand(f, o);
      if (wins<OP, KB>(other, f)) f = other;
    }
    if (lane == 0) {
      p.res[RES_AUX0] = (unsigned long long)f.row;  // -1 (all ones) when no row is valid
      *ticket = 0;
    }
  }
}

// Shared front end: argument checks, None cases, the null count, one launch, one synchronisation. One scratch request
// holds [table_bytes for make_src][per-CTA partials]; make_src(table_space, &src) builds the source.
template <class Src, class MakeSrc>
acu_status arg_extreme(acu_ctx *ctx, const char *what, acu_agg_op op, const acu_array *nulls, size_t table_bytes, MakeSrc make_src,
                       int64_t *out_row, int64_t *out_valid_count) {
  if (op != ACU_MIN && op != ACU_MAX) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "%s: op must be min or max", what);
  if (nulls->is_scalar) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "%s: the input must be an array, not a scalar", what);
  const int64_t n = nulls->len;
  if (n == 0) return ACU_OK;  // None (aggregate.rs:464)
  acu_status st = ACU_OK;
  // an unknown null count is counted by the kernel itself (RES_COUNT): no extra pass
  const int64_t nc = (nulls->validity && nulls->null_count < 0) ? -1 : acu_resolve_null_count(ctx, nulls, &st);
  ACU_TRY(st);
  if (nc == n) return ACU_OK;  // every row null: None
  ArgArgs a;
  a.n = n;
  a.valid = (nulls->validity && nc != 0) ? nulls->validity : nullptr;
  a.voff = nulls->validity_offset;
  a.res = ctx->d_res;
  const int64_t sgroups = (n + 2047) >> 11;
  const int grid = acu_grid(ctx, (sgroups + 7) / 8, 8);
  void *scratch;
  ACU_TRY(acu_scratch(ctx, table_bytes + (size_t)grid * sizeof(Cand), &scratch));
  a.partial = reinterpret_cast<Cand *>(static_cast<uint8_t *>(scratch) + table_bytes);
  Src src;
  ACU_TRY(make_src(scratch, &src));
  ACU_TRY(acu_res_reset(ctx));
  if (op == ACU_MIN) ACU_LAUNCH_TIMED(ctx, ACU_K_REDUCE, (k_arg_extreme<ACU_MIN, Src>), grid, 256, 0, a, src);
  else ACU_LAUNCH_TIMED(ctx, ACU_K_REDUCE, (k_arg_extreme<ACU_MAX, Src>), grid, 256, 0, a, src);
  ACU_TRY(acu_res_fetch(ctx));
  *out_valid_count = (int64_t)ctx->h_res[RES_COUNT];
  *out_row = *out_valid_count ? (int64_t)ctx->h_res[RES_AUX0] : -1;
  return ACU_OK;
}

}  // namespace

extern "C" acu_status acu_aggregate_bytes(acu_ctx *ctx, int32_t offset_bytes, acu_agg_op op, const acu_bytes_array *a, int64_t *out_row,
                                          int64_t *out_valid_count) {
  ACU_ENTER(ctx);
  *out_row = -1;
  *out_valid_count = 0;
  ACU_TRY(acu_sync_only(ctx));
  ACU_TRY(acu_offset_width_check(ctx, offset_bytes));
  return arg_extreme<BytesSrc>(
      ctx, "acu_aggregate_bytes", op, &a->nulls, 0,
      [&](void *, BytesSrc *src) { return *src = BytesSrc{BytesOperand{a->offsets, a->data, offset_bytes}}, ACU_OK; }, out_row, out_valid_count);
}

extern "C" acu_status acu_aggregate_byte_view(acu_ctx *ctx, acu_agg_op op, const acu_view_array *a, int64_t *out_row,
                                              int64_t *out_valid_count) {
  ACU_ENTER(ctx);
  *out_row = -1;
  *out_valid_count = 0;
  ACU_TRY(acu_sync_only(ctx));
  return arg_extreme<ViewSrc>(
      ctx, "acu_aggregate_byte_view", op, &a->nulls, acu_view_table_bytes(a),
      [&](void *table_space, ViewSrc *src) { return acu_view_operand(ctx, a, table_space, &src->s); }, out_row, out_valid_count);
}

extern "C" acu_status acu_aggregate_fixed_size_binary(acu_ctx *ctx, int32_t byte_width, acu_agg_op op, const acu_array *a, int64_t *out_row,
                                                      int64_t *out_valid_count) {
  ACU_ENTER(ctx);
  *out_row = -1;
  *out_valid_count = 0;
  ACU_TRY(acu_sync_only(ctx));
  if (byte_width < 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "FixedSizeBinary width must be >= 0, got %d", (int)byte_width);
  return arg_extreme<FixedSrc>(
      ctx, "acu_aggregate_fixed_size_binary", op, a, 0,
      [&](void *, FixedSrc *src) { return *src = FixedSrc{static_cast<const uint8_t *>(a->values), (int64_t)byte_width}, ACU_OK; }, out_row,
      out_valid_count);
}

// min_boolean is Some(false) iff a valid slot is false, max_boolean Some(true) iff a valid slot is true: one popcount of
// values & validity (BooleanArray::true_count) against the valid count.
extern "C" acu_status acu_aggregate_boolean(acu_ctx *ctx, acu_agg_op op, const acu_array *a, int32_t *out_value, int64_t *out_valid_count) {
  ACU_ENTER(ctx);
  *out_value = -1;
  *out_valid_count = 0;
  ACU_TRY(acu_sync_only(ctx));
  if (op != ACU_MIN && op != ACU_MAX) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "acu_aggregate_boolean: op must be min or max");
  if (a->is_scalar) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "acu_aggregate_boolean: the input must be an array, not a scalar");
  const int64_t n = a->len;
  if (n == 0) return ACU_OK;
  acu_status st;
  const int64_t nc = acu_resolve_null_count(ctx, a, &st);
  ACU_TRY(st);
  if (nc == n) return ACU_OK;  // aggregate.rs:374-376
  ACU_TRY(acu_res_reset(ctx));
  const int slot = acu_kstats_begin(ctx, ACU_K_REDUCE);
  st = acu_bitmap_and_launch(ctx, static_cast<const uint8_t *>(a->values), a->values_offset, nc ? a->validity : nullptr, a->validity_offset,
                             n, nullptr, true);
  acu_kstats_end(ctx, slot);
  ACU_TRY(st);
  ACU_TRY(acu_res_fetch(ctx));
  const int64_t valid = n - nc, true_valid = (int64_t)ctx->h_res[RES_COUNT];
  *out_valid_count = valid;
  *out_value = op == ACU_MIN ? (true_valid == valid ? 1 : 0) : (true_valid > 0 ? 1 : 0);
  return ACU_OK;
}
