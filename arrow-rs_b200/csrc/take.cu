// take.cu — arrow-select/src/take.rs on the device.
//
//   take_primitive = take_native + take_nulls   (take.rs:405-457)
//   take_bits / take_boolean                     (take.rs:460-496)
//   check_bounds                                 (take.rs:167-209)
//   ToIndices                                    (take.rs:1030-1084)
//
// Design (gather, HBM/sector-bound): persistent CTAs walk index tiles of 2048 indices.
// The NEXT tile's indices are prefetched into shared memory with a 1-D bulk async copy
// (cp.async.bulk + mbarrier, the TMA engine: UBLKCP in SASS) while the current tile is
// gathered, so the index stream never sits on the dependent-load critical path. Each thread
// then issues 8 independent gathers (values + validity bit) before storing; output values
// are written with fully coalesced stores, output validity is packed with a warp ballot
// (lane == output bit), and the null count / out-of-bounds detection ride in the same pass.
#include <stdio.h>
#include <stdlib.h>

#include <type_traits>

#include "bitmap.cuh"
#include "internal.cuh"

#define TAKE_WTILE_DEFAULT 256  // indices per warp tile (8 gathers per lane in flight)

namespace {

// ---- mbarrier + bulk-copy PTX wrappers --------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, unsigned bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

template <int W> struct VecOf;
template <> struct VecOf<1> { using type = uint8_t; };
template <> struct VecOf<2> { using type = uint16_t; };
template <> struct VecOf<4> { using type = uint32_t; };
template <> struct VecOf<8> { using type = uint64_t; };
template <> struct VecOf<16> { using type = uint4; };
struct alignas(16) U32B { uint4 lo, hi; };
template <> struct VecOf<32> { using type = U32B; };

template <class V> __device__ __forceinline__ V zero_of() { V v; memset(&v, 0, sizeof(V)); return v; }
template <class V> __device__ __forceinline__ V gather_ld(const V *p) {
  if constexpr (sizeof(V) == 32) {
    V v;
    v.lo = __ldg(reinterpret_cast<const uint4 *>(p));
    v.hi = __ldg(reinterpret_cast<const uint4 *>(p) + 1);
    return v;
  } else {
    return __ldg(p);
  }
}

struct TakeArgs {
  const void *values;       // NULL for take_nulls-only / take_boolean passes
  int64_t n_values;
  const uint8_t *vvalid;    // values validity to gather (NULL: none)
  int64_t vvoff;
  const uint8_t *vbits;     // boolean VALUES to gather (take_boolean), else NULL
  int64_t vboff;
  const void *idx;
  int64_t m;
  const uint8_t *ivalid;    // index validity (only when it has nulls, or to clone)
  int64_t ivoff;
  int idx_has_nulls;        // indices.null_count() > 0
  void *out;
  uint32_t *out_valid;      // u32 words, bit offset 0 (NULL: none)
  uint32_t *out_bits;       // take_boolean values
  unsigned long long *res;
  int use_bulk;             // idx base 16-B aligned: stage index tiles with cp.async.bulk
};

// ToIndices (take.rs:1030-1084). IT: 0=u8 1=i8 2=u16 3=i16 4=u32/i32 5=u64/i64
template <int IT> struct IdxOf;
template <> struct IdxOf<0> { using raw = uint8_t; };
template <> struct IdxOf<1> { using raw = int8_t; };
template <> struct IdxOf<2> { using raw = uint16_t; };
template <> struct IdxOf<3> { using raw = int16_t; };
template <> struct IdxOf<4> { using raw = uint32_t; };
template <> struct IdxOf<5> { using raw = uint64_t; };
// index after ToIndices: u32 for every source type but (u)int64 -> keeps the gather state in 32-bit registers
template <int IT> struct WideOf { using type = typename std::conditional<IT == 5, uint64_t, uint32_t>::type; };
template <int IT> __device__ __forceinline__ typename WideOf<IT>::type widen(typename IdxOf<IT>::raw v) {
  if constexpr (IT == 1 || IT == 3) return (uint32_t)(int32_t)v;  // `as u32` sign-extends
  else return (typename WideOf<IT>::type)v;
}

// BOOL: take_boolean (bit gather of boolean VALUES, no value gather); else take_primitive.
// Up to TAKE_BATCH_COLS columns per launch (blockIdx.y = column): the columns of a take_record_batch share the
// index array, hence the grid.x size.
constexpr int TAKE_BATCH_COLS = 8;
struct TakeBatch { TakeArgs col[TAKE_BATCH_COLS]; };

// PL = gathers per lane in flight (warp tile = 32 * PL indices), MINB = resident CTAs per SM the register budget is cut for.
template <int W, int IT, bool BOOL, int PL = 8, int MINB = 3>
__global__ void __launch_bounds__(256, MINB) k_take(const TakeBatch batch) {
  constexpr int TAKE_WTILE = 32 * PL;
  constexpr int TAKE_PER_LANE = PL;
  const TakeArgs a = batch.col[blockIdx.y];
  using V = typename VecOf<W>::type;
  using I = typename IdxOf<IT>::raw;
  // warp-private double-buffered index tiles: no CTA-wide barrier anywhere in the loop
  __shared__ __align__(16) I s_idx[8][2][TAKE_WTILE];
  __shared__ __align__(8) uint64_t s_bar[8][2];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const I *idx = static_cast<const I *>(a.idx);
  const int64_t n_tiles = (a.m + TAKE_WTILE - 1) / TAKE_WTILE;
  const bool gather_values = !BOOL && a.values != nullptr;
  unsigned valid_cnt = 0;
  unsigned long long err = ~0ull;

  if (lane == 0) { mbar_init(&s_bar[wid][0], 1); mbar_init(&s_bar[wid][1], 1); }
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncwarp();

  // stage tile `t` into this warp's buffer `b`
  auto stage = [&](int64_t t, int b) {
    const int64_t j0 = t * TAKE_WTILE;
    const int cnt = (int)((a.m - j0) < TAKE_WTILE ? (a.m - j0) : TAKE_WTILE);
    const bool bulk = a.use_bulk && cnt == TAKE_WTILE;  // full tiles only: size % 16 == 0
    if (bulk) {
      if (lane == 0) {
        mbar_expect_tx(&s_bar[wid][b], (unsigned)(TAKE_WTILE * sizeof(I)));
        bulk_g2s(&s_idx[wid][b][0], idx + j0, (unsigned)(TAKE_WTILE * sizeof(I)), &s_bar[wid][b]);
      }
    } else {
      for (int k = lane; k < cnt; k += 32) s_idx[wid][b][k] = __ldg(idx + j0 + k);
    }
    return bulk;
  };

  unsigned phase0 = 0, phase1 = 0;  // mbarrier parity per buffer (scalars: no local-memory array)
  int64_t t = warp;
  bool cur_bulk = false;
  if (t < n_tiles) cur_bulk = stage(t, 0);
  int buf = 0;
  for (; t < n_tiles; t += nwarps) {
    const int64_t tn = t + nwarps;
    bool next_bulk = false;
    if (tn < n_tiles) next_bulk = stage(tn, buf ^ 1);  // prefetch while we gather
    if (cur_bulk) {
      mbar_wait(&s_bar[wid][buf], buf ? phase1 : phase0);
      if (buf) phase1 ^= 1; else phase0 ^= 1;
    }
    else __syncwarp();

    const int64_t j0 = t * TAKE_WTILE;
    typename WideOf<IT>::type ix[TAKE_PER_LANE];
    bool live[TAKE_PER_LANE], inb[TAKE_PER_LANE];
    V v[TAKE_PER_LANE];
    uint32_t bit[TAKE_PER_LANE];
#pragma unroll
    for (int k = 0; k < TAKE_PER_LANE; ++k) {
      const int j = k * 32 + lane;
      live[k] = j0 + j < a.m;
      ix[k] = live[k] ? widen<IT>(s_idx[wid][buf][j]) : 0;
      // take() converts the indices with ToIndices BEFORE take_native (take.rs:100): i32 is REINTERPRETED as u32 and i8 / i16
      // are widened with `as u32`, so `index.as_usize()` (take.rs:442) zero-extends — a negative i32 index is the in-bounds
      // row 2^32 + idx when values.len() exceeds it, exactly as here
      inb[k] = live[k] && (uint64_t)ix[k] < (uint64_t)a.n_values;
    }
    // ---- 8 independent gathers in flight per lane ----
#pragma unroll
    for (int k = 0; k < TAKE_PER_LANE; ++k) {
      if (gather_values) v[k] = inb[k] ? gather_ld<V>(static_cast<const V *>(a.values) + ix[k]) : zero_of<V>();
      uint32_t b = 1u;
      if (a.vvalid) b = inb[k] ? ld_bit(a.vvalid, a.vvoff + (int64_t)ix[k]) : 0u;
      if (BOOL) b |= (inb[k] ? ld_bit(a.vbits, a.vboff + (int64_t)ix[k]) : 0u) << 1;
      bit[k] = b;
    }
#pragma unroll
    for (int k = 0; k < TAKE_PER_LANE; ++k) {
      const int64_t gj = j0 + k * 32 + lane;  // gj - lane is a multiple of 32: lane == output bit
      uint32_t iv = ~0u;
      if (a.ivalid) iv = ld_bits32(a.ivalid, a.ivoff + (gj - lane), a.ivoff + a.m);
      const bool idx_valid = live[k] && ((iv >> lane) & 1u);
      // out-of-bounds at a VALID index slot panics in the reference (take.rs:447,454);
      // at a NULL slot it yields T::default() (already zero)
      const bool counts_as_valid_idx = a.idx_has_nulls ? idx_valid : live[k];
      if (live[k] && !inb[k] && counts_as_valid_idx) { unsigned long long e = (unsigned long long)gj; err = e < err ? e : err; }
      if (gather_values && live[k]) static_cast<V *>(a.out)[gj] = v[k];
      if (a.out_valid) {
        bool ob = live[k];
        if (a.vvalid) ob = ob && (bit[k] & 1u) && counts_as_valid_idx;  // take_bits of values.nulls
        else ob = idx_valid;                                             // indices.nulls().cloned()
        const uint32_t word = __ballot_sync(ACU_FULL_MASK, ob);
        if (lane == 0 && gj < a.m) { a.out_valid[gj >> 5] = word; valid_cnt += __popc(word); }
      }
      if (BOOL) {  // take_bits on boolean values: unset at null indices
        const bool ob = live[k] && counts_as_valid_idx && ((bit[k] >> 1) & 1u);
        const uint32_t word = __ballot_sync(ACU_FULL_MASK, ob);
        if (lane == 0 && gj < a.m) a.out_bits[gj >> 5] = word;
      }
    }
    __syncwarp();  // the whole warp is done with s_idx[wid][buf] before it is refilled
    buf ^= 1;
    cur_bulk = next_bulk;
  }
  if (a.out_valid) {
    if (lane == 0 && valid_cnt) atomicAdd(a.res + RES_COUNT, (unsigned long long)valid_cnt);
  }
  if (err != ~0ull) atomicMin(a.res + RES_ERR_INDEX, err);
}

// check_bounds (take.rs:167-209) on the ORIGINAL index type: lowest offending row.
template <int IT, bool SIGNED>
__global__ void __launch_bounds__(256) k_check_bounds(const void *idx_v, int64_t m, int64_t len,
                                                      const uint8_t *ivalid, int64_t ivoff,
                                                      unsigned long long *res) {
  using I = typename IdxOf<IT>::raw;
  const I *idx = static_cast<const I *>(idx_v);
  unsigned long long err = ~0ull;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += stride) {
    if (ivalid && !ld_bit(ivalid, ivoff + j)) continue;
    bool bad;
    if constexpr (SIGNED) {
      using S = typename std::make_signed<I>::type;
      const int64_t v = (int64_t)(S)idx[j];
      // nullable path only tests `index >= len` (take.rs:183); otherwise also `< 0` (:193-199)
      bad = ivalid ? (v >= len) : (v < 0 || v >= len);
    } else {
      bad = (uint64_t)idx[j] >= (uint64_t)len;
    }
    if (bad && (unsigned long long)j < err) err = (unsigned long long)j;
  }
  if (err != ~0ull) atomicMin(res + RES_ERR_INDEX, err);
}

int index_kind(acu_dtype t) {
  switch (t) {
    case ACU_U8: return 0; case ACU_I8: return 1; case ACU_U16: return 2; case ACU_I16: return 3;
    case ACU_U32: case ACU_I32: return 4; case ACU_U64: case ACU_I64: return 5;
    default: return -1;
  }
}
uint64_t index_max(acu_dtype t) {
  switch (t) {
    case ACU_I8: return INT8_MAX; case ACU_I16: return INT16_MAX; case ACU_I32: return INT32_MAX;
    case ACU_I64: return INT64_MAX; case ACU_U8: return UINT8_MAX; case ACU_U16: return UINT16_MAX;
    case ACU_U32: return UINT32_MAX; default: return UINT64_MAX;
  }
}

template <int W>
acu_status launch_take_w(acu_ctx *ctx, int kind, const TakeBatch &tb, int n_cols) {
  const TakeArgs &ta = tb.col[0];
  constexpr int TAKE_WTILE = TAKE_WTILE_DEFAULT;
  const int64_t tiles = ((ta.m + TAKE_WTILE - 1) / TAKE_WTILE + 7) / 8;  // CTAs: 8 warp tiles each
#define ACU_TAKE_CASE(IT)                                                                                   \
  case IT:                                                                                                                   \
    if (W == 1 && ta.vbits)                                                                                                  \
      ACU_LAUNCH_TIMED(ctx, ACU_K_TAKE, (k_take<1, IT, true>), dim3(acu_wave_grid(ctx, k_take<1, IT, true>, 256, 0, tiles), n_cols), 256, 0, tb); \
    else                                                                                                                     \
      ACU_LAUNCH_TIMED(ctx, ACU_K_TAKE, (k_take<W, IT, false>), dim3(acu_wave_grid(ctx, k_take<W, IT, false>, 256, 0, tiles), n_cols), 256, 0, tb); \
    break;
  switch (kind) {
    ACU_TAKE_CASE(0) ACU_TAKE_CASE(1) ACU_TAKE_CASE(2) ACU_TAKE_CASE(3) ACU_TAKE_CASE(4) ACU_TAKE_CASE(5)
    default: break;
  }
#undef ACU_TAKE_CASE
  return ACU_OK;
}

acu_status launch_take(acu_ctx *ctx, int elem_bytes, int kind, const TakeBatch &tb, int n_cols) {
  switch (elem_bytes) {
    case 1: return launch_take_w<1>(ctx, kind, tb, n_cols);
    case 2: return launch_take_w<2>(ctx, kind, tb, n_cols);
    case 4: return launch_take_w<4>(ctx, kind, tb, n_cols);
    case 8: return launch_take_w<8>(ctx, kind, tb, n_cols);
    case 16: return launch_take_w<16>(ctx, kind, tb, n_cols);
    case 32: return launch_take_w<32>(ctx, kind, tb, n_cols);
    default: return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "take: unsupported element width %d", elem_bytes);
  }
}

acu_status fetch_index(acu_ctx *ctx, const acu_array *indices, acu_dtype t, int64_t j, uint64_t *raw, char *text, size_t n) {
  uint64_t v = 0;
  const int sz = acu_dtype_size(t);
  ACU_CUDA(ctx, cudaMemcpyAsync(&v, static_cast<const uint8_t *>(indices->values) + (size_t)j * sz, sz, cudaMemcpyDeviceToHost, ctx->stream));
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *raw = v;
  if (acu_dtype_is_signed(t)) {
    int64_t s = sz == 1 ? (int8_t)v : sz == 2 ? (int16_t)v : sz == 4 ? (int32_t)v : (int64_t)v;
    snprintf(text, n, "%lld", (long long)s);
  } else {
    snprintf(text, n, "%llu", (unsigned long long)v);
  }
  return ACU_OK;
}

}  // namespace

// take_primitive / take_boolean: the record-batch launcher on one column.
static acu_status take_array(acu_ctx *ctx, int32_t elem_bytes, const acu_array *values, bool boolean_values,
                             const acu_array *indices, acu_dtype index_dtype, int32_t check_bounds, acu_array_out *out) {
  ACU_ENTER(ctx);
  const int kind = index_kind(index_dtype);
  if (kind < 0)  // take.rs:103
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Take only supported for integers, got %s", acu_dtype_name(index_dtype));
  acu_status st;
  const int64_t m = indices->len;
  const int64_t inc = acu_resolve_null_count(ctx, indices, &st);
  ACU_TRY(st);
  const bool idx_nulls = indices->validity && inc > 0;
  if (check_bounds) ACU_TRY(acu_take_check_bounds(ctx, indices, index_dtype, idx_nulls, values->len));
  out->len = m;
  out->has_validity = 0;
  out->null_count = 0;
  if (m == 0) return ACU_OK;  // take_impl: new_empty_array (take.rs:216-218)
  const int64_t vnc = acu_resolve_null_count(ctx, values, &st);
  ACU_TRY(st);
  const char val_nulls = values->validity && vnc > 0;  // take_nulls (take.rs:419-430)
  const char is_bool = boolean_values;
  int mode = 0;
  const int blk = acu_call_begin(ctx, &st);
  ACU_TRY(st);
  unsigned long long *res = acu_dres(ctx, blk);
  ACU_TRY(acu_take_cols_launch(ctx, 1, &elem_bytes, &values, &is_bool, &val_nulls, indices, index_dtype, idx_nulls, &out, &res, &mode));
  const acu_array v = *values, ix = *indices;  // the finaliser may run later (acu_results_fetch): keep copies of the descriptors
  return acu_call_end(ctx, blk, [ctx, v, ix, index_dtype, mode, out](const unsigned long long *h) -> acu_status {
    return acu_take_col_finalize(ctx, &v, &ix, index_dtype, mode, h, out);
  });
}

static TakeArgs take_args(int32_t elem_bytes, const acu_array *values, bool boolean_values, bool val_nulls, const acu_array *indices,
                          acu_dtype /*index_dtype*/, bool idx_nulls, acu_array_out *out, unsigned long long *res) {
  TakeArgs ta{};
  ta.values = (elem_bytes > 0 && !boolean_values) ? values->values : nullptr;
  ta.n_values = values->len;
  if (val_nulls) { ta.vvalid = values->validity; ta.vvoff = values->validity_offset; }
  if (boolean_values) { ta.vbits = static_cast<const uint8_t *>(values->values); ta.vboff = values->values_offset; ta.out_bits = static_cast<uint32_t *>(out->values); }
  ta.idx = indices->values;
  ta.m = indices->len;
  if (idx_nulls || (!val_nulls && indices->validity)) { ta.ivalid = indices->validity; ta.ivoff = indices->validity_offset; }
  ta.idx_has_nulls = idx_nulls;
  ta.out = out->values;
  if (val_nulls || indices->validity) ta.out_valid = reinterpret_cast<uint32_t *>(out->validity);
  ta.res = res;
  ta.use_bulk = ((uintptr_t)indices->values % 16) == 0;
  return ta;
}

// The columns of take / take_record_batch: queue the gathers on the ctx stream without synchronising. Columns that run
// the same kernel instantiation (element width / boolean / validity-only) share a launch. elem_bytes[c] == 0 with
// boolean[c] == 0 is the validity-only gather of a variable-width column. val_nulls / idx_nulls = "has a validity
// buffer with at least one null" (exact, the NullBuffer decision depends on it). modes[c]: bit 0 = an output validity
// was produced, bit 1 = it came from take_bits(values.nulls) (None when it has no nulls).
acu_status acu_take_cols_launch(acu_ctx *ctx, int n, const int32_t *elem_bytes, const acu_array *const *values, const char *boolean,
                                const char *val_nulls, const acu_array *indices, acu_dtype index_dtype, bool idx_nulls,
                                acu_array_out *const *outs, unsigned long long *const *res, int *modes) {
  const int kind = index_kind(index_dtype);
  for (int c = 0; c < n; ++c) {
    modes[c] = 0;
    outs[c]->len = indices->len;
    outs[c]->has_validity = 0;
    outs[c]->null_count = 0;
  }
  if (indices->len == 0) return ACU_OK;
  // kernel instantiation of column c: a column without a value buffer gathers its validity only
  auto klass = [&](int c) { return boolean[c] ? -1 : (elem_bytes[c] > 0 && values[c]->values ? elem_bytes[c] : 0); };
  char done[ACU_MAX_BATCH_COLUMNS] = {0};
  for (int c = 0; c < n; ++c) {
    if (done[c]) continue;
    TakeBatch tb{};
    int k = 0;
    for (int d = c; d < n && k < TAKE_BATCH_COLS; ++d) {
      if (done[d] || klass(d) != klass(c)) continue;
      tb.col[k] = take_args(elem_bytes[d], values[d], boolean[d] != 0, val_nulls[d] != 0, indices, index_dtype, idx_nulls, outs[d], res[d]);
      modes[d] = (tb.col[k].out_valid ? 1 : 0) | (val_nulls[d] ? 2 : 0);
      done[d] = 1;
      ++k;
    }
    ACU_TRY(launch_take(ctx, klass(c) > 0 ? klass(c) : 1, kind, tb, k));
  }
  return ACU_OK;
}

acu_status acu_take_col_finalize(acu_ctx *ctx, const acu_array *values, const acu_array *indices, acu_dtype index_dtype, int mode,
                                 const unsigned long long *hres, acu_array_out *out) {
  const int64_t m = indices->len;
  if (m == 0) return ACU_OK;
  if (hres[RES_ERR_INDEX] != ~0ull) {
    const int64_t j = (int64_t)hres[RES_ERR_INDEX];
    uint64_t raw;
    char text[32];
    ACU_TRY(fetch_index(ctx, indices, index_dtype, j, &raw, text, sizeof text));
    // the reference panics on the index AFTER ToIndices (u32 / u64): take.rs:447
    uint64_t widened = raw;
    switch (index_dtype) {
      case ACU_I8: widened = (uint32_t)(int32_t)(int8_t)raw; break;
      case ACU_I16: widened = (uint32_t)(int32_t)(int16_t)raw; break;
      case ACU_I32: widened = (uint32_t)raw; break;
      default: break;
    }
    return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, j, widened, 0, (uint64_t)values->len, "Out-of-bounds index %llu",
                    (unsigned long long)widened);
  }
  if (mode & 1) {
    const int64_t null_count = m - (int64_t)hres[RES_COUNT];
    if (mode & 2) {  // NullBuffer::from_unsliced_buffer: None when no nulls (null.rs:266-270)
      if (null_count > 0) { out->has_validity = 1; out->null_count = null_count; }
    } else {
      out->has_validity = 1;
      out->null_count = null_count;
    }
  }
  return ACU_OK;
}

// TakeOptions{check_bounds:true} (take.rs:167-209) for one index array against `values_len` rows; synchronises.
acu_status acu_take_check_bounds(acu_ctx *ctx, const acu_array *indices, acu_dtype index_dtype, bool idx_nulls, int64_t values_len) {
  const int kind = index_kind(index_dtype);
  const int64_t m = indices->len;
  if (!(m > 0 && (uint64_t)values_len <= index_max(index_dtype))) return ACU_OK;  // T::Native::from_usize(len)
  ACU_TRY(acu_res_reset(ctx));
  const int grid = acu_grid(ctx, (m + 255) / 256, 8);
  const uint8_t *iv = idx_nulls ? indices->validity : nullptr;
  const bool sgn = acu_dtype_is_signed(index_dtype);
#define ACU_CB_CASE(IT)                                                                                                   \
  case IT:                                                                                                                \
    if (sgn) ACU_LAUNCH(ctx, (k_check_bounds<IT, true>), grid, 256, 0, indices->values, m, values_len, iv, indices->validity_offset, ctx->d_res); \
    else ACU_LAUNCH(ctx, (k_check_bounds<IT, false>), grid, 256, 0, indices->values, m, values_len, iv, indices->validity_offset, ctx->d_res);    \
    break;
  switch (kind) { ACU_CB_CASE(0) ACU_CB_CASE(1) ACU_CB_CASE(2) ACU_CB_CASE(3) ACU_CB_CASE(4) ACU_CB_CASE(5) default: break; }
#undef ACU_CB_CASE
  ACU_TRY(acu_res_fetch(ctx));
  if (ctx->h_res[RES_ERR_INDEX] != ~0ull) {
    const int64_t j = (int64_t)ctx->h_res[RES_ERR_INDEX];
    uint64_t raw;
    char text[32];
    ACU_TRY(fetch_index(ctx, indices, index_dtype, j, &raw, text, sizeof text));
    return acu_fail(ctx, ACU_ERR_COMPUTE, j, raw, 0, (uint64_t)values_len,
                    "Array index out of bounds, cannot get item at index %s from %lld entries", text, (long long)values_len);
  }
  return ACU_OK;
}

int acu_take_index_kind(acu_dtype t) { return index_kind(t); }

extern "C" acu_status acu_take_primitive(acu_ctx *ctx, int32_t elem_bytes, const acu_array *values,
                                         const acu_array *indices, acu_dtype index_dtype,
                                         int32_t check_bounds, acu_array_out *out) {
  return take_array(ctx, elem_bytes, values, false, indices, index_dtype, check_bounds, out);
}

extern "C" acu_status acu_take_boolean(acu_ctx *ctx, const acu_array *values, const acu_array *indices,
                                       acu_dtype index_dtype, int32_t check_bounds, acu_array_out *out) {
  return take_array(ctx, 0, values, true, indices, index_dtype, check_bounds, out);
}
