// reduce.cu — arrow-arith/src/aggregate.rs sum / min / max / product / bit_and / bit_or / bit_xor on the device.
//
// Reference: aggregate() :317-366, accumulators :52-176, sum :943, product :953, min :1012, max :1027,
// bit_and / bit_or / bit_xor :788-875. sum and product wrap for integers (add_wrapping / mul_wrapping)
// and are IEEE for floats; min/max use the totalOrder (arrow-array/src/arithmetic.rs:400-437). Float
// `sum` and `product` are order-dependent in the reference itself (lane count depends on compile-time
// target features, aggregate.rs:303-313), so parity for them is tolerance-based; everything else is
// bit-exact (wrapping multiplication and the bit ops are associative and commutative).
//
// Design: one streaming pass (HBM-bound, 8N + N/8 bytes). Lane l of a warp owns rows l and
// l+32 of each 64-row strip (one validity word per strip), 4 strips in flight. Per-thread
// accumulators -> warp shuffle tree -> per-CTA partial in scratch; the last CTA to finish
// (atomic ticket) folds the partials in a fixed order, so results are deterministic for a
// given grid. Float min/max run on integer totalOrder keys.
#include <limits>
#include <type_traits>

#include "bitmap.cuh"
#include "internal.cuh"

namespace {

template <class T> struct KeyOf { using type = T; };
template <> struct KeyOf<double> { using type = int64_t; };
template <> struct KeyOf<float> { using type = int32_t; };

template <class T> __device__ __forceinline__ typename KeyOf<T>::type to_key(T v) {
  if constexpr (std::is_floating_point<T>::value) return total_key(v);
  else return v;
}
template <class T> __device__ __forceinline__ T from_key(typename KeyOf<T>::type k) {
  if constexpr (sizeof(T) == 8 && std::is_floating_point<T>::value) return __longlong_as_double(k ^ (int64_t)((uint64_t)(k >> 63) >> 1));
  else if constexpr (std::is_floating_point<T>::value) return __int_as_float(k ^ (int32_t)((uint32_t)(k >> 31) >> 1));
  else return k;
}

// accumulator domain: min/max -> totalOrder key; every other op -> T itself
template <class T, int OP> struct AccOf {
  using type = typename std::conditional<OP == ACU_MIN || OP == ACU_MAX, typename KeyOf<T>::type, T>::type;
};

template <class A, int OP> __device__ __forceinline__ A acc_identity() {
  if constexpr (OP == ACU_SUM) return A(0);
  else if constexpr (OP == ACU_MIN) return std::numeric_limits<A>::max();   // MAX_TOTAL_ORDER
  else if constexpr (OP == ACU_MAX) return std::numeric_limits<A>::lowest();  // MIN_TOTAL_ORDER
  else if constexpr (OP == ACU_PRODUCT) return A(1);
  else if constexpr (OP == ACU_BIT_AND) return (A)~(A)0;                   // -1: all ones
  else return A(0);                                                        // bit_or / bit_xor
}
template <class A, int OP> __device__ __forceinline__ A acc_merge(A a, A b) {
  if constexpr (OP == ACU_SUM) {
    if constexpr (std::is_same<A, double>::value) return __dadd_rn(a, b);
    else if constexpr (std::is_same<A, float>::value) return __fadd_rn(a, b);
    else if constexpr (sizeof(A) == 16) return (A)((unsigned __int128)a + (unsigned __int128)b);  // i128 add_wrapping
    else return (A)((typename std::make_unsigned<A>::type)a + (typename std::make_unsigned<A>::type)b);  // add_wrapping
  } else if constexpr (OP == ACU_MIN) {
    return b < a ? b : a;
  } else if constexpr (OP == ACU_MAX) {
    return b > a ? b : a;
  } else if constexpr (OP == ACU_PRODUCT) {
    if constexpr (std::is_same<A, double>::value) return __dmul_rn(a, b);
    else if constexpr (std::is_same<A, float>::value) return __fmul_rn(a, b);
    else {  // mul_wrapping in the unsigned type, at least 32 bits wide (a u16 x u16 would be promoted to int and overflow it)
      using U = typename std::conditional<(sizeof(A) < 4), uint32_t, typename std::make_unsigned<A>::type>::type;
      return (A)((U)a * (U)b);
    }
  } else if constexpr (OP == ACU_BIT_AND) {
    return a & b;
  } else if constexpr (OP == ACU_BIT_OR) {
    return a | b;
  } else {
    return a ^ b;
  }
}
template <class T, int OP> __device__ __forceinline__ typename AccOf<T, OP>::type acc_lift(T v) {
  if constexpr (OP == ACU_MIN || OP == ACU_MAX) return to_key<T>(v);
  else return v;
}

template <class A> __device__ __forceinline__ A shfl_down_any(A v, int o) {
  if constexpr (sizeof(A) == 16) {  // Decimal128: two 64-bit halves
    long long x[2];
    memcpy(x, &v, 16);
    x[0] = __shfl_down_sync(ACU_FULL_MASK, x[0], o);
    x[1] = __shfl_down_sync(ACU_FULL_MASK, x[1], o);
    memcpy(&v, x, 16);
    return v;
  } else if constexpr (sizeof(A) == 8) {
    long long x;
    memcpy(&x, &v, 8);
    x = __shfl_down_sync(ACU_FULL_MASK, x, o);
    memcpy(&v, &x, 8);
    return v;
  } else {
    int x = 0;
    memcpy(&x, &v, sizeof(A));
    x = __shfl_down_sync(ACU_FULL_MASK, x, o);
    memcpy(&v, &x, sizeof(A));
    return v;
  }
}

constexpr int REDUCE_BATCH_COLS = 8;
struct ReduceArgs {
  const void *v;            // values (native type of the launch)
  int64_t n;
  const uint8_t *valid;     // validity (NULL: no nulls)
  int64_t voff;
  void *partial;            // one accumulator per CTA
  unsigned long long *res;  // result block: RES_COUNT valid rows, RES_AUX0 result bits, RES_AUX3 ticket (zero on entry and on exit)
};
struct ReduceBatch { ReduceArgs col[REDUCE_BATCH_COLS]; };

template <class T, int OP>
__global__ void __launch_bounds__(256) k_reduce(const ReduceBatch batch) {
  using A = typename AccOf<T, OP>::type;
  // blockIdx.y = column of the batch (same dtype and op); the ticket is a slot of the column's result block
  const T *__restrict__ v = static_cast<const T *>(batch.col[blockIdx.y].v);
  const int64_t n = batch.col[blockIdx.y].n;
  const uint8_t *__restrict__ valid = batch.col[blockIdx.y].valid;
  const int64_t voff = batch.col[blockIdx.y].voff;
  A *__restrict__ partial = static_cast<A *>(batch.col[blockIdx.y].partial);
  unsigned long long *__restrict__ res = batch.col[blockIdx.y].res;
  unsigned int *__restrict__ ticket = reinterpret_cast<unsigned int *>(res + RES_AUX3);
  constexpr int U = 8;  // strips (64 rows) in flight per warp: 8 x 2 loads per lane
  __shared__ A s_part[8];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t sgroups = (n + 2047) >> 11;  // super-group = 32 strips = 2048 rows = 32 validity words
  A acc = acc_identity<A, OP>();
  unsigned valid_cnt = 0;
  for (int64_t sg = warp; sg < sgroups; sg += nwarps) {
    const int64_t sbase = sg << 11;
    // lane l owns validity word l of the super-group (one coalesced 256-B bitmap access)
    const int64_t wrow = sbase + lane * 64;
    const int64_t k = n - wrow;
    uint64_t vw = k >= 64 ? ~0ull : (k <= 0 ? 0ull : ((~0ull) >> (64 - k)));
    if (valid) vw &= ld_bits64(valid, voff + wrow, voff + n);
    valid_cnt += __popcll(vw);
#pragma unroll 1
    for (int s0 = 0; s0 < 32; s0 += U) {
      if (sbase + s0 * 64 >= n) break;
      T x[U][2];
#pragma unroll
      for (int u = 0; u < U; ++u) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int64_t i = sbase + (s0 + u) * 64 + h * 32 + lane;
          x[u][h] = i < n ? ldg_elem(v + i) : T();
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint64_t w = __shfl_sync(ACU_FULL_MASK, vw, s0 + u);
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if ((w >> (h * 32 + lane)) & 1ull) acc = acc_merge<A, OP>(acc, acc_lift<T, OP>(x[u][h]));
      }
    }
  }
  valid_cnt = warp_sum(valid_cnt);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc = acc_merge<A, OP>(acc, shfl_down_any(acc, o));
  if (lane == 0) {
    s_part[wid] = acc;
    if (valid_cnt) atomicAdd(res + RES_COUNT, (unsigned long long)valid_cnt);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    A b = s_part[0];
    for (int w = 1; w < 8; ++w) b = acc_merge<A, OP>(b, s_part[w]);
    partial[blockIdx.x] = b;
    __threadfence();
    s_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  }
  __syncthreads();
  if (s_last && wid == 0) {  // fixed-order fold of the per-CTA partials
    __threadfence();
    A f = acc_identity<A, OP>();
    for (unsigned i = lane; i < gridDim.x; i += 32) f = acc_merge<A, OP>(f, *(volatile A *)(partial + i));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) f = acc_merge<A, OP>(f, shfl_down_any(f, o));
    if (lane == 0) {
      T r;
      if constexpr (OP == ACU_MIN || OP == ACU_MAX) r = from_key<T>(f);
      else r = f;
      unsigned long long bits[2] = {0, 0};  // an i128 result fills RES_AUX0 (low) and RES_AUX1 (high)
      memcpy(bits, &r, sizeof(T));
      res[RES_AUX0] = bits[0];
      if (sizeof(T) == 16) res[RES_AUX1] = bits[1];
      *ticket = 0;
    }
  }
}

template <class T, int OP>
acu_status reduce_launch(acu_ctx *ctx, const ReduceBatch &rb, int n_cols, int64_t max_len) {
  using A = typename AccOf<T, OP>::type;
  static_assert(sizeof(A) <= 16, "partials must fit the per-column scratch");
  const int64_t strips = (max_len + 63) >> 6;
  const int grid = acu_wave_grid(ctx, k_reduce<T, OP>, 256, 0, (strips / 32 + 1 + 7) / 8);
  ACU_LAUNCH_TIMED(ctx, ACU_K_REDUCE, (k_reduce<T, OP>), dim3(grid, n_cols), 256, 0, rb);
  return ACU_OK;
}

// The (dtype, op) pair has passed acu_agg_op_check; the bit ops are instantiated for integer types only.
template <class T>
acu_status reduce_typed(acu_ctx *ctx, acu_agg_op op, const ReduceBatch &rb, int n_cols, int64_t max_len) {
  constexpr bool INTEGRAL = std::is_integral<T>::value && sizeof(T) <= 8;
  switch (op) {
    case ACU_SUM: return reduce_launch<T, ACU_SUM>(ctx, rb, n_cols, max_len);
    case ACU_MIN: return reduce_launch<T, ACU_MIN>(ctx, rb, n_cols, max_len);
    case ACU_MAX: return reduce_launch<T, ACU_MAX>(ctx, rb, n_cols, max_len);
    default: break;
  }
  if constexpr (sizeof(T) <= 8) {
    if (op == ACU_PRODUCT) return reduce_launch<T, ACU_PRODUCT>(ctx, rb, n_cols, max_len);
  }
  if constexpr (INTEGRAL) {
    if (op == ACU_BIT_AND) return reduce_launch<T, ACU_BIT_AND>(ctx, rb, n_cols, max_len);
    if (op == ACU_BIT_OR) return reduce_launch<T, ACU_BIT_OR>(ctx, rb, n_cols, max_len);
    if (op == ACU_BIT_XOR) return reduce_launch<T, ACU_BIT_XOR>(ctx, rb, n_cols, max_len);
  }
  return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "aggregate: op %d", (int)op);
}

acu_status reduce_dispatch(acu_ctx *ctx, acu_dtype dtype, acu_agg_op op, const ReduceBatch &rb, int n_cols, int64_t max_len) {
  return acu_with_native(
      dtype, [&](auto t) { return reduce_typed<decltype(t)>(ctx, op, rb, n_cols, max_len); },
      [&] { return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "aggregate: dtype %d", (int)dtype); });
}

ReduceArgs reduce_args(const acu_array *a, int64_t nc, void *scratch, unsigned long long *res) {
  ReduceArgs r;
  r.v = a->values;
  r.n = a->len;
  r.valid = (a->validity && nc != 0) ? a->validity : nullptr;  // nc < 0: unknown (counted by the kernel)
  r.voff = a->validity_offset;
  r.partial = scratch;
  r.res = res;
  return r;
}

}  // namespace

// sum / min / max / product take every native dtype, bit_and / bit_or / bit_xor the integer ones (aggregate.rs:788-875)
acu_status acu_agg_op_check(acu_ctx *ctx, acu_dtype dtype, acu_agg_op op) {
  if (op == ACU_SUM || op == ACU_MIN || op == ACU_MAX || op == ACU_PRODUCT) return ACU_OK;
  if (op != ACU_BIT_AND && op != ACU_BIT_OR && op != ACU_BIT_XOR)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "aggregate: op %d", (int)op);
  if (acu_dtype_is_float(dtype))
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "aggregate: bit_and / bit_or / bit_xor of %s", acu_dtype_name(dtype));
  return ACU_OK;
}

// per-column scratch of one queued reduction: one partial per CTA of the widest grid
size_t acu_reduce_col_scratch(const acu_ctx *ctx) { return (size_t)ctx->sm_count * 8 * 8 * 16 + 4096; }

// Queue sum / min / max of columns on the ctx stream (no sync); those with the same (dtype, op) share a launch
// (blockIdx.y = column). The caller has resolved the null counts (nc[c] < 0: unknown, the kernel consults the validity
// and counts): nc[c] == len (or len == 0) means None and nothing is launched for the column (launched[c] = 0). The
// result lands in res[c][RES_AUX0] as the native bit pattern.
acu_status acu_reduce_cols_launch(acu_ctx *ctx, int n, const acu_dtype *dtypes, const acu_agg_op *ops, const acu_array *arrays,
                                  const int64_t *nc, uint8_t *scratch, size_t scratch_per_col, unsigned long long *const *res, int *launched) {
  char done[ACU_MAX_BATCH_COLUMNS] = {0};
  for (int c = 0; c < n; ++c) {
    launched[c] = 0;
    if (arrays[c].len == 0 || nc[c] == arrays[c].len) done[c] = 1;  // None (aggregate.rs:320-323)
  }
  for (int c = 0; c < n; ++c) {
    if (done[c]) continue;
    ReduceBatch rb{};
    int k = 0;
    int64_t max_len = 0;
    for (int d = c; d < n && k < REDUCE_BATCH_COLS; ++d) {
      if (done[d] || dtypes[d] != dtypes[c] || ops[d] != ops[c]) continue;
      rb.col[k++] = reduce_args(&arrays[d], nc[d], scratch + scratch_per_col * d, res[d]);
      if (arrays[d].len > max_len) max_len = arrays[d].len;
      done[d] = 1;
      launched[d] = 1;
    }
    ACU_TRY(reduce_dispatch(ctx, dtypes[c], ops[c], rb, k, max_len));
  }
  return ACU_OK;
}

// acu_aggregate / acu_aggregate_i128 (wide: out_bits[0..1] of an __int128 result)
static acu_status aggregate_one(acu_ctx *ctx, acu_dtype dtype, acu_agg_op op, const acu_array *a, bool wide, uint64_t *out_bits,
                                int64_t *out_valid_count) {
  *out_valid_count = 0;
  if (a->len == 0) return ACU_OK;  // None
  acu_status st = ACU_OK;
  // inside an async section an unknown null count (the array was produced earlier in the same section) is not resolved by
  // a round trip: the kernel consults the validity and counts the valid rows itself (RES_COUNT)
  const bool deferred_nc = ctx->async_on && a->validity && a->null_count < 0;
  const int64_t nc = deferred_nc ? -1 : acu_resolve_null_count(ctx, a, &st);
  ACU_TRY(st);
  if (!deferred_nc) *out_valid_count = a->len - nc;
  const size_t scratch_bytes = acu_reduce_col_scratch(ctx);
  void *scratch;
  ACU_TRY(acu_scratch(ctx, scratch_bytes, &scratch));
  int launched = 0;
  const int blk = acu_call_begin(ctx, &st);
  ACU_TRY(st);
  unsigned long long *res = acu_dres(ctx, blk);
  if (!wide) {
    ACU_TRY(acu_reduce_cols_launch(ctx, 1, &dtype, &op, a, &nc, static_cast<uint8_t *>(scratch), scratch_bytes, &res, &launched));
  } else if (nc != a->len) {  // Decimal128: the same launch on __int128, kept out of the dtype dispatch of acu_aggregate*
    ReduceBatch rb{};
    rb.col[0] = reduce_args(a, nc, scratch, res);
    ACU_TRY(reduce_typed<__int128>(ctx, op, rb, 1, a->len));
    launched = 1;
  }
  if (!launched && !ctx->async_on) return ACU_OK;
  return acu_call_end(ctx, blk, [launched, deferred_nc, wide, out_bits, out_valid_count](const unsigned long long *h) -> acu_status {
    if (!launched) return ACU_OK;
    if (deferred_nc) {
      *out_valid_count = (int64_t)h[RES_COUNT];
      if (*out_valid_count == 0) return ACU_OK;  // every row null: None (aggregate.rs:320-323)
    }
    out_bits[0] = h[RES_AUX0];
    if (wide) out_bits[1] = h[RES_AUX1];
    return ACU_OK;
  });
}

extern "C" acu_status acu_aggregate(acu_ctx *ctx, acu_dtype dtype, acu_agg_op op, const acu_array *a,
                                    uint64_t *out_bits, int64_t *out_valid_count) {
  ACU_ENTER(ctx);
  *out_bits = 0;
  *out_valid_count = 0;
  ACU_TRY(acu_agg_op_check(ctx, dtype, op));
  return aggregate_one(ctx, dtype, op, a, false, out_bits, out_valid_count);
}

extern "C" acu_status acu_aggregate_i128(acu_ctx *ctx, acu_agg_op op, const acu_array *a, uint64_t out_bits[2],
                                         int64_t *out_valid_count) {
  ACU_ENTER(ctx);
  out_bits[0] = out_bits[1] = 0;
  if (op != ACU_SUM && op != ACU_MIN && op != ACU_MAX)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "aggregate: op %d", (int)op);
  if (a->len && (uintptr_t)a->values % 16 != 0)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Int128 values must be 16-byte aligned");
  return aggregate_one(ctx, ACU_I128, op, a, true, out_bits, out_valid_count);
}
