// sumchecked.cu — sum_checked (arrow-arith/src/aggregate.rs:897-937): the reference folds
// `acc.add_checked(v)` over the valid values IN ORDER, so it fails exactly when some running
// prefix of the (unbounded) sum leaves the native type's range — even if the final total fits.
//
// A prefix-range test is associative: a row segment is summarised by (total, lowest prefix,
// highest prefix) in 128-bit arithmetic and  (t1,lo1,hi1) (+) (t2,lo2,hi2) = (t1+t2,
// min(lo1, t1+lo2), max(hi1, t1+hi2)).  Pass 1 reduces contiguous 4096-row chunks to such
// triples (one CTA per chunk, 16 consecutive rows per thread, ordered shuffle tree); pass 2 (one
// CTA) scans the chunk triples, produces the total and the FIRST chunk in which a prefix
// overflows; only then pass 3 walks that one chunk sequentially to rebuild the reference's error
// ("Overflow happened on: {acc:?} + {value:?}", arrow-array/src/arithmetic.rs:163-170).
//
// product_checked (aggregate.rs:963-1001) has the same three passes over a different summary. Before the
// first zero, |running product| never decreases (every factor has |x| >= 1), and a zero absorbs everything
// after it, so the fold fails at the first prefix whose magnitude passes the limit L (2^(w-1) for signed,
// 2^w - 1 for unsigned types) — or, for signed types, whose magnitude equals L = 2^(w-1) while its sign is
// positive. A segment of rows is summarised by
//   (has_zero, B = |product before its first zero| saturated above L, its sign, pos, neg)
// where pos / neg say whether the segment's own running sign is + / - at some row between its last factor
// with |x| >= 2 (its first row if there is none) and its first zero: exactly the rows at which the running
// magnitude equals its final value m*B. A segment entered with magnitude m and sign s (no zero yet) fails iff
// m*B > L, or m*B == L and the flag of sign s is set (pos for s = +, neg for s = -). The pass 3 walk of the
// one failing chunk rebuilds the reference's "Overflow happened on: {acc:?} * {value:?}" (arithmetic.rs:193-200).
#include <stdio.h>

#include <type_traits>

#include "bitmap.cuh"
#include "internal.cuh"

namespace {

typedef __int128 i128;
constexpr int SC_THREADS = 256, SC_ROWS_PER_THREAD = 16, SC_CHUNK = SC_THREADS * SC_ROWS_PER_THREAD;

struct Seg {
  i128 total, lo, hi;  // lo / hi over the prefixes AFTER each add; an empty segment has lo = +INF, hi = -INF
};
__device__ __forceinline__ i128 seg_inf() { return (i128)1 << 120; }  // |any real prefix| < 2^104 (2^40 rows x 2^64)
__device__ __forceinline__ Seg seg_empty() { return Seg{0, seg_inf(), -seg_inf()}; }
__device__ __forceinline__ Seg seg_join(const Seg &a, const Seg &b) {  // a's rows precede b's
  Seg r;
  r.total = a.total + b.total;
  const i128 blo = a.total + b.lo, bhi = a.total + b.hi;
  r.lo = a.lo < blo ? a.lo : blo;
  r.hi = a.hi > bhi ? a.hi : bhi;
  return r;
}
__device__ __forceinline__ i128 shfl_down_i128(i128 v, int o) {
  unsigned long long lo = (unsigned long long)v, hi = (unsigned long long)(v >> 64);
  lo = __shfl_down_sync(ACU_FULL_MASK, lo, o);
  hi = __shfl_down_sync(ACU_FULL_MASK, hi, o);
  return (i128)(((unsigned __int128)hi << 64) | lo);
}
__device__ __forceinline__ Seg shfl_down_seg(const Seg &s, int o) {
  return Seg{shfl_down_i128(s.total, o), shfl_down_i128(s.lo, o), shfl_down_i128(s.hi, o)};
}

template <class T> __device__ __forceinline__ i128 type_min() { return std::is_signed<T>::value ? -((i128)1 << (8 * sizeof(T) - 1)) : (i128)0; }
template <class T> __device__ __forceinline__ i128 type_max() {
  return std::is_signed<T>::value ? ((i128)1 << (8 * sizeof(T) - 1)) - 1 : ((i128)1 << (8 * sizeof(T))) - 1;
}

// pass 1: one CTA per 4096-row chunk
template <class T>
__global__ void __launch_bounds__(SC_THREADS) k_sumchk_chunks(const T *__restrict__ v, int64_t n, const uint8_t *__restrict__ valid, int64_t voff,
                                                              Seg *__restrict__ chunk_seg) {
  __shared__ Seg s_warp[SC_THREADS / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t row0 = (int64_t)blockIdx.x * SC_CHUNK + (int64_t)threadIdx.x * SC_ROWS_PER_THREAD;
  uint32_t bits = 0;
  if (row0 < n) {
    const int64_t left = n - row0;
    bits = left >= SC_ROWS_PER_THREAD ? 0xFFFFu : ((1u << left) - 1u);
    if (valid) bits &= ld_bits32(valid, voff + row0, voff + n);
  }
  Seg s = seg_empty();
  i128 acc = 0;
#pragma unroll
  for (int k = 0; k < SC_ROWS_PER_THREAD; ++k) {
    if ((bits >> k) & 1u) {
      acc += (i128)v[row0 + k];
      if (acc < s.lo) s.lo = acc;
      if (acc > s.hi) s.hi = acc;
    }
  }
  s.total = acc;
  // ordered tree: after step o lane l holds the join of lanes [l, l + 2o)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const Seg r = shfl_down_seg(s, o);
    if (lane + o < 32) s = seg_join(s, r);
  }
  if (lane == 0) s_warp[wid] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    Seg c = s_warp[0];
    for (int w = 1; w < SC_THREADS / 32; ++w) c = seg_join(c, s_warp[w]);
    chunk_seg[blockIdx.x] = c;
  }
}

// pass 2: one CTA over all chunk triples: total, and the first chunk with an out-of-range prefix
template <class T>
__global__ void __launch_bounds__(1024) k_sumchk_scan(const Seg *__restrict__ chunk_seg, int64_t chunks, unsigned long long *__restrict__ res) {
  __shared__ i128 s_tot[1024];
  __shared__ unsigned long long s_first;
  const int t = threadIdx.x;
  const int64_t per = (chunks + 1023) / 1024;
  const int64_t c0 = (int64_t)t * per, c1 = c0 + per < chunks ? c0 + per : chunks;
  i128 mine = 0;
  for (int64_t c = c0; c < c1; ++c) mine += chunk_seg[c].total;
  s_tot[t] = mine;
  if (t == 0) s_first = ~0ull;
  __syncthreads();
  // exclusive prefix of the per-thread totals (1024 entries: a serial pass by one warp lane per 32 is plenty)
  if (t == 0) {
    i128 run = 0;
    for (int i = 0; i < 1024; ++i) {
      const i128 x = s_tot[i];
      s_tot[i] = run;
      run += x;
    }
    const T total = (T)run;  // meaningful only when nothing overflowed
    unsigned long long b = 0;
    memcpy(&b, &total, sizeof(T));
    res[RES_AUX0] = b;
  }
  __syncthreads();
  i128 acc = s_tot[t];
  unsigned long long cand = ~0ull;
  i128 cand_acc = 0;
  const i128 lo = type_min<T>(), hi = type_max<T>();
  for (int64_t c = c0; c < c1; ++c) {
    const Seg s = chunk_seg[c];
    if (acc + s.lo < lo || acc + s.hi > hi) {
      cand = (unsigned long long)c;
      cand_acc = acc;
      break;
    }
    acc += s.total;
  }
  if (cand != ~0ull) atomicMin(&s_first, cand);
  __syncthreads();
  if (cand != ~0ull && cand == s_first) {
    res[RES_ERR_INDEX] = cand;                              // first failing chunk
    const T a = (T)cand_acc;                                // the accumulator on entry to it is still in range
    unsigned long long b = 0;
    memcpy(&b, &a, sizeof(T));
    res[RES_AUX1] = b;
  }
}

// pass 3 (error path only): walk the failing chunk in order
template <class T>
__global__ void k_sumchk_locate(const T *__restrict__ v, int64_t n, const uint8_t *__restrict__ valid, int64_t voff, int64_t chunk,
                                unsigned long long acc_bits, unsigned long long *__restrict__ res) {
  T acc;
  memcpy(&acc, &acc_bits, sizeof(T));
  const int64_t r0 = chunk * SC_CHUNK, r1 = r0 + SC_CHUNK < n ? r0 + SC_CHUNK : n;
  const i128 lo = type_min<T>(), hi = type_max<T>();
  for (int64_t r = r0; r < r1; ++r) {
    if (valid && !ld_bit(valid, voff + r)) continue;
    const i128 s = (i128)acc + (i128)v[r];
    if (s < lo || s > hi) {
      unsigned long long a = 0, b = 0;
      const T x = v[r];
      memcpy(&a, &acc, sizeof(T));
      memcpy(&b, &x, sizeof(T));
      res[RES_AUX2] = (unsigned long long)r;
      res[RES_AUX1] = a;
      res[RES_AUX0] = b;
      return;
    }
    acc = (T)s;
  }
}

// ---- product_checked ----
typedef unsigned __int128 u128;
constexpr u128 PC_SAT = (u128)1 << 64;  // above every limit L (<= 2^64 - 1); magnitudes saturate here

struct PSeg {
  u128 mag;     // |product before the first zero|, saturated at PC_SAT; 1 for an empty segment
  uint32_t f;   // PF_* flags
};
enum { PF_ZERO = 1, PF_NEG = 2, PF_POS_AT_MAX = 4, PF_NEG_AT_MAX = 8 };  // PF_NEG: the pre-zero product is negative

__host__ __device__ __forceinline__ u128 sat_mul(u128 a, u128 b) {
  if ((a >> 64) || (b >> 64)) return PC_SAT;  // both >= 1 before any zero: the product is at least the saturated side
  const u128 m = a * b;                      // < 2^128
  return m > PC_SAT ? PC_SAT : m;
}
__device__ __forceinline__ PSeg pseg_empty() { return PSeg{1, 0}; }
// a's rows precede b's
__device__ __forceinline__ PSeg pseg_join(const PSeg &a, const PSeg &b) {
  if (a.f & PF_ZERO) return a;
  uint32_t bf = b.f & (PF_POS_AT_MAX | PF_NEG_AT_MAX);
  if (a.f & PF_NEG) bf = ((bf & PF_POS_AT_MAX) ? PF_NEG_AT_MAX : 0) | ((bf & PF_NEG_AT_MAX) ? PF_POS_AT_MAX : 0);  // b's signs seen from a's start
  PSeg r;
  r.mag = sat_mul(a.mag, b.mag);
  // b's rows at its own final magnitude are the combined segment's; when b has no |x| >= 2 factor, a's rows at a's
  // final magnitude are too
  r.f = (b.f & PF_ZERO) | ((a.f ^ b.f) & PF_NEG) | bf | (b.mag > 1 ? 0 : (a.f & (PF_POS_AT_MAX | PF_NEG_AT_MAX)));
  return r;
}
template <class T> __host__ __device__ __forceinline__ u128 pc_limit() {
  return std::is_signed<T>::value ? (u128)1 << (8 * sizeof(T) - 1) : ((u128)1 << (8 * sizeof(T))) - 1;
}
// the fold entered with magnitude m and sign `neg` fails inside segment s (m >= 1, no zero before it)
template <class T> __device__ __forceinline__ bool pseg_fails(u128 m, bool neg, const PSeg &s) {
  const u128 p = sat_mul(m, s.mag), L = pc_limit<T>();
  if (p > L) return true;
  return std::is_signed<T>::value && p == L && (s.f & (neg ? PF_NEG_AT_MAX : PF_POS_AT_MAX));
}
__device__ __forceinline__ PSeg shfl_down_pseg(const PSeg &s, int o) {
  unsigned long long lo = (unsigned long long)s.mag, hi = (unsigned long long)(s.mag >> 64);
  lo = __shfl_down_sync(ACU_FULL_MASK, lo, o);
  hi = __shfl_down_sync(ACU_FULL_MASK, hi, o);
  return PSeg{((u128)hi << 64) | lo, __shfl_down_sync(ACU_FULL_MASK, s.f, o)};
}

// pass 1: one CTA per 4096-row chunk (the layout of k_sumchk_chunks)
template <class T>
__global__ void __launch_bounds__(SC_THREADS) k_prodchk_chunks(const T *__restrict__ v, int64_t n, const uint8_t *__restrict__ valid,
                                                               int64_t voff, PSeg *__restrict__ chunk_seg) {
  __shared__ PSeg s_warp[SC_THREADS / 32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t row0 = (int64_t)blockIdx.x * SC_CHUNK + (int64_t)threadIdx.x * SC_ROWS_PER_THREAD;
  uint32_t bits = 0;
  if (row0 < n) {
    const int64_t left = n - row0;
    bits = left >= SC_ROWS_PER_THREAD ? 0xFFFFu : ((1u << left) - 1u);
    if (valid) bits &= ld_bits32(valid, voff + row0, voff + n);
  }
  // every valid row's value is loaded before any is looked at (reading past a zero is harmless): a load gated on the
  // previous row's value would serialise the thread's loads
  T xs[SC_ROWS_PER_THREAD];
#pragma unroll
  for (int k = 0; k < SC_ROWS_PER_THREAD; ++k) xs[k] = ((bits >> k) & 1u) ? v[row0 + k] : T(1);
  PSeg s = pseg_empty();
#pragma unroll
  for (int k = 0; k < SC_ROWS_PER_THREAD; ++k) {
    if (((bits >> k) & 1u) && !(s.f & PF_ZERO)) {
      const T x = xs[k];
      if (x == 0) {
        s.f |= PF_ZERO;
        continue;
      }
      bool xneg = false;
      if constexpr (std::is_signed<T>::value) xneg = x < 0;
      const u128 ax = xneg ? (u128)(0 - (unsigned long long)(long long)x) : (u128)(unsigned long long)x;
      if (xneg) s.f ^= PF_NEG;
      if (ax > 1) {
        s.mag = sat_mul(s.mag, ax);
        s.f &= ~(uint32_t)(PF_POS_AT_MAX | PF_NEG_AT_MAX);  // the rows at the final magnitude start here
      }
      s.f |= (s.f & PF_NEG) ? PF_NEG_AT_MAX : PF_POS_AT_MAX;
    }
  }
  // ordered tree: after step o lane l holds the join of lanes [l, l + 2o)
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const PSeg r = shfl_down_pseg(s, o);
    if (lane + o < 32) s = pseg_join(s, r);
  }
  if (lane == 0) s_warp[wid] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    PSeg c = s_warp[0];
    for (int w = 1; w < SC_THREADS / 32; ++w) c = pseg_join(c, s_warp[w]);
    chunk_seg[blockIdx.x] = c;
  }
}

// pass 2: one CTA over all chunk summaries: the product, and the first chunk in which the fold fails together with the
// accumulator on entry to it
template <class T>
__global__ void __launch_bounds__(1024) k_prodchk_scan(const PSeg *__restrict__ chunk_seg, int64_t chunks, unsigned long long *__restrict__ res) {
  __shared__ PSeg s_pre[1024];
  __shared__ unsigned long long s_first;
  const int t = threadIdx.x;
  const int64_t per = (chunks + 1023) / 1024;
  const int64_t c0 = (int64_t)t * per, c1 = c0 + per < chunks ? c0 + per : chunks;
  PSeg mine = pseg_empty();
  for (int64_t c = c0; c < c1; ++c) mine = pseg_join(mine, chunk_seg[c]);
  s_pre[t] = mine;
  if (t == 0) s_first = ~0ull;
  __syncthreads();
  if (t == 0) {  // exclusive prefix of the per-thread summaries
    PSeg run = pseg_empty();
    for (int i = 0; i < 1024; ++i) {
      const PSeg x = s_pre[i];
      s_pre[i] = run;
      run = pseg_join(run, x);
    }
    // the product when nothing failed: 0 after a zero, else +/- the (then exact) magnitude
    const unsigned long long m = (unsigned long long)run.mag;
    const unsigned long long p = (run.f & PF_ZERO) ? 0ull : (run.f & PF_NEG) ? 0ull - m : m;
    const T total = (T)p;
    unsigned long long b = 0;
    memcpy(&b, &total, sizeof(T));
    res[RES_AUX0] = b;
  }
  __syncthreads();
  PSeg acc = s_pre[t];
  unsigned long long cand = ~0ull;
  PSeg cand_acc = acc;
  for (int64_t c = c0; c < c1 && !(acc.f & PF_ZERO); ++c) {
    const PSeg s = chunk_seg[c];
    if (pseg_fails<T>(acc.mag, acc.f & PF_NEG, s)) {
      cand = (unsigned long long)c;
      cand_acc = acc;
      break;
    }
    acc = pseg_join(acc, s);
  }
  if (cand != ~0ull) atomicMin(&s_first, cand);
  __syncthreads();
  if (cand != ~0ull && cand == s_first) {
    res[RES_ERR_INDEX] = cand;  // first failing chunk
    const unsigned long long m = (unsigned long long)cand_acc.mag;  // in range: nothing failed before this chunk
    const T a = (T)((cand_acc.f & PF_NEG) ? 0ull - m : m);
    unsigned long long b = 0;
    memcpy(&b, &a, sizeof(T));
    res[RES_AUX1] = b;
  }
}

// pass 3 (error path only): walk the failing chunk in order
template <class T>
__global__ void k_prodchk_locate(const T *__restrict__ v, int64_t n, const uint8_t *__restrict__ valid, int64_t voff, int64_t chunk,
                                 unsigned long long acc_bits, unsigned long long *__restrict__ res) {
  T acc;
  memcpy(&acc, &acc_bits, sizeof(T));
  const int64_t r0 = chunk * SC_CHUNK, r1 = r0 + SC_CHUNK < n ? r0 + SC_CHUNK : n;
  for (int64_t r = r0; r < r1; ++r) {
    if (valid && !ld_bit(valid, voff + r)) continue;
    const T x = v[r];
    bool ovf;
    T o;
    if constexpr (sizeof(T) == 8 && !std::is_signed<T>::value) {
      ovf = __umul64hi(acc, x) != 0;
      o = acc * x;
    } else {
      const i128 p = (i128)acc * (i128)x;  // |acc|, |x| <= 2^63: exact
      ovf = p < type_min<T>() || p > type_max<T>();
      o = (T)p;
    }
    if (ovf) {
      unsigned long long a = 0, b = 0;
      memcpy(&a, &acc, sizeof(T));
      memcpy(&b, &x, sizeof(T));
      res[RES_AUX2] = (unsigned long long)r;
      res[RES_AUX1] = a;
      res[RES_AUX0] = b;
      return;
    }
    acc = o;
  }
}

template <class T> void fmt_int(char *buf, size_t n, unsigned long long bits) {  // Rust {:?} of the native integer
  T v;
  memcpy(&v, &bits, sizeof(T));
  if (std::is_signed<T>::value) snprintf(buf, n, "%lld", (long long)v);
  else snprintf(buf, n, "%llu", (unsigned long long)v);
}

// The three passes of one checked fold: PRODUCT picks product_checked's summaries and operator, else sum_checked's.
template <class T, bool PRODUCT>
acu_status checked_fold_typed(acu_ctx *ctx, const acu_array *a, const uint8_t *valid, uint64_t *out_bits) {
  using S = typename std::conditional<PRODUCT, PSeg, Seg>::type;
  const int64_t n = a->len;
  const int64_t chunks = (n + SC_CHUNK - 1) / SC_CHUNK;
  void *scratch;
  ACU_TRY(acu_scratch(ctx, (size_t)chunks * sizeof(S) + 256, &scratch));
  S *segs = static_cast<S *>(scratch);
  const T *v = static_cast<const T *>(a->values);
  ACU_TRY(acu_res_reset(ctx));
  if constexpr (PRODUCT) {
    ACU_LAUNCH_TIMED(ctx, ACU_K_REDUCE, k_prodchk_chunks<T>, (unsigned)chunks, SC_THREADS, 0, v, n, valid, a->validity_offset, segs);
    ACU_LAUNCH_TIMED(ctx, ACU_K_REDUCE, k_prodchk_scan<T>, 1, 1024, 0, segs, chunks, ctx->d_res);
  } else {
    ACU_LAUNCH_TIMED(ctx, ACU_K_REDUCE, k_sumchk_chunks<T>, (unsigned)chunks, SC_THREADS, 0, v, n, valid, a->validity_offset, segs);
    ACU_LAUNCH_TIMED(ctx, ACU_K_REDUCE, k_sumchk_scan<T>, 1, 1024, 0, segs, chunks, ctx->d_res);
  }
  ACU_TRY(acu_res_fetch(ctx));
  if (ctx->h_res[RES_ERR_INDEX] != ~0ull) {
    const int64_t chunk = (int64_t)ctx->h_res[RES_ERR_INDEX];
    const unsigned long long acc_bits = ctx->h_res[RES_AUX1];
    ACU_TRY(acu_res_reset(ctx));
    if constexpr (PRODUCT) ACU_LAUNCH(ctx, k_prodchk_locate<T>, 1, 1, 0, v, n, valid, a->validity_offset, chunk, acc_bits, ctx->d_res);
    else ACU_LAUNCH(ctx, k_sumchk_locate<T>, 1, 1, 0, v, n, valid, a->validity_offset, chunk, acc_bits, ctx->d_res);
    ACU_TRY(acu_res_fetch(ctx));
    char ls[40], rs[40];
    fmt_int<T>(ls, sizeof ls, ctx->h_res[RES_AUX1]);
    fmt_int<T>(rs, sizeof rs, ctx->h_res[RES_AUX0]);
    return acu_fail(ctx, ACU_ERR_ARITHMETIC_OVERFLOW, (int64_t)ctx->h_res[RES_AUX2], ctx->h_res[RES_AUX1], ctx->h_res[RES_AUX0], 0,
                    "Overflow happened on: %s %s %s", ls, PRODUCT ? "*" : "+", rs);
  }
  *out_bits = ctx->h_res[RES_AUX0];
  return ACU_OK;
}

// sum_checked / product_checked: None for an empty or all-null array (aggregate.rs:902-904, :968-970), floats as the
// unchecked aggregate: add_checked / mul_checked are the plain IEEE ops and never fail (arithmetic.rs:317-319); only the
// association order differs from sum / product, which the reference leaves unspecified — same kernel, same tolerance
template <bool PRODUCT>
acu_status checked_fold(acu_ctx *ctx, acu_dtype dtype, const acu_array *a, uint64_t *out_bits, int64_t *out_valid_count) {
  if (dtype == ACU_F32 || dtype == ACU_F64) return acu_aggregate(ctx, dtype, PRODUCT ? ACU_PRODUCT : ACU_SUM, a, out_bits, out_valid_count);
  *out_bits = 0;
  *out_valid_count = 0;
  if (a->len == 0) return ACU_OK;  // Ok(None)
  acu_status st;
  const int64_t nc = acu_resolve_null_count(ctx, a, &st);
  ACU_TRY(st);
  *out_valid_count = a->len - nc;
  if (nc == a->len) return ACU_OK;
  const uint8_t *valid = (a->validity && nc > 0) ? a->validity : nullptr;
  auto fail = [&] {
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "%s: dtype %d", PRODUCT ? "product_checked" : "sum_checked", (int)dtype);
  };
  return acu_with_native(
      dtype,
      [&](auto t) {
        using T = decltype(t);
        if constexpr (std::is_integral<T>::value) return checked_fold_typed<T, PRODUCT>(ctx, a, valid, out_bits);
        else return fail();
      },
      fail);
}

}  // namespace

extern "C" acu_status acu_sum_checked(acu_ctx *ctx, acu_dtype dtype, const acu_array *a, uint64_t *out_bits, int64_t *out_valid_count) {
  ACU_ENTER(ctx);
  return checked_fold<false>(ctx, dtype, a, out_bits, out_valid_count);
}

extern "C" acu_status acu_product_checked(acu_ctx *ctx, acu_dtype dtype, const acu_array *a, uint64_t *out_bits,
                                          int64_t *out_valid_count) {
  ACU_ENTER(ctx);
  *out_bits = 0;
  *out_valid_count = 0;
  ACU_TRY(acu_sync_only(ctx));  // refused whatever the input, before any device work (also for floats and empty inputs)
  return checked_fold<true>(ctx, dtype, a, out_bits, out_valid_count);
}
