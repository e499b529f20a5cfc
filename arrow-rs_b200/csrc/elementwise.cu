// elementwise.cu — numeric::{add,sub,mul,div,rem,neg}(_wrapping), bitwise::*, cmp::*, cast (numeric and decimal).
//
// Reference: arrow-arith/src/numeric.rs:36-374, arrow-arith/src/bitwise.rs, arrow-arith/src/arity.rs:104-135,254-299,
// arrow-array/src/array/primitive_array.rs:916-1103, arrow-array/src/arithmetic.rs:148-437,
// arrow-ord/src/cmp.rs:220-648, arrow-cast/src/cast/mod.rs:2550-2614.
//
// All kernels are single-pass and HBM-bound: each input byte is read once, each output
// byte written once, and the validity AND + popcount ride along in the same pass.
// Every kernel here has one shape: a warp owns 2048-row super-groups = 32 validity words,
// lane l owning word l (one coalesced 256-B bitmap access per super-group). Lane l reads
// elements [l*EPL, (l+1)*EPL) of each 32*EPL-row load: EPL = 16 / sizeof(T) (128-bit
// accesses, 512-B warp requests) when the value pointers are 16-B aligned, EPL = 1 for
// unaligned slices. Warp 0 finishes the ragged tail (< 2048 rows) in 64-row strips after
// its super-groups, so each call is one launch.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <limits>
#include <string>
#include <type_traits>

#include "bitmap.cuh"
#include "internal.cuh"

namespace {

// ---------------------------------------------------------------------------------------
// 128-bit packs
// ---------------------------------------------------------------------------------------
template <class T, int EPL> struct alignas(EPL * sizeof(T) == 16 ? 16 : sizeof(T)) Pack { T v[EPL]; };

template <class T, int EPL>
__device__ __forceinline__ Pack<T, EPL> pack_load(const T *p) {
  Pack<T, EPL> r;
  if constexpr (EPL * sizeof(T) == 16) {
    uint4 x = ld_stream16(p);
    r = *reinterpret_cast<Pack<T, EPL> *>(&x);
  } else {
    static_assert(EPL == 1, "scalar path");
    r.v[0] = __ldg(p);
  }
  return r;
}
template <class T, int EPL>
__device__ __forceinline__ void pack_store(T *p, Pack<T, EPL> r) {
  if constexpr (EPL * sizeof(T) == 16) {
    st_stream16(p, *reinterpret_cast<uint4 *>(&r));
  } else {
    *p = r.v[0];
  }
}

__device__ __forceinline__ uint64_t ones_to(int64_t row, int64_t n) {  // bits [row,row+64) ∩ [0,n)
  int64_t k = n - row;
  return k >= 64 ? ~0ull : (k <= 0 ? 0ull : ((~0ull) >> (64 - k)));
}

// 256-thread CTAs for n rows: 8 warps per CTA, one 2048-row super-group per warp step; a column shorter than 2048 rows
// still gets warp 0, which finishes the ragged tail.
int64_t sg_blocks(int64_t n) { return (n / 2048 + 1 + 7) / 8; }

// ---------------------------------------------------------------------------------------
// Per-element arithmetic (ArrowNativeTypeOp, arithmetic.rs:148-437)
// ---------------------------------------------------------------------------------------
enum { CLS_WRAP = 0, CLS_CHECKED = 1, CLS_DIVREM = 2, CLS_DECIMAL = 3, CLS_BITWISE = 4 };
enum { OP_ADD = 0, OP_SUB = 1, OP_MUL = 2, OP_DIV = 3, OP_REM = 4, OP_NEG = 5 };

template <class T> struct is_fp { static constexpr bool value = std::is_floating_point<T>::value; };

__device__ __forceinline__ double fp_add(double a, double b) { return __dadd_rn(a, b); }  // never contracted
__device__ __forceinline__ double fp_sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double fp_mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double fp_div(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ double fp_rem(double a, double b) { return fmod(a, b); }
__device__ __forceinline__ float fp_add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float fp_sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fp_mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fp_div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float fp_rem(float a, float b) { return fmodf(a, b); }

// returns true when the reference would return Err at this element
template <class T, int CLS>
__device__ __forceinline__ bool apply_op(int op, T l, T r, T &o) {
  if constexpr (is_fp<T>::value) {
    if constexpr (CLS == CLS_DIVREM) {
      o = (op == OP_DIV) ? fp_div(l, r) : fp_rem(l, r);
    } else {
      o = (op == OP_ADD) ? fp_add(l, r) : (op == OP_SUB) ? fp_sub(l, r) : (op == OP_MUL) ? fp_mul(l, r) : -r;
    }
    return false;
  } else {
    using U = typename std::make_unsigned<T>::type;
    constexpr bool SIGNED = std::is_signed<T>::value;
    if constexpr (CLS == CLS_WRAP) {
      U a = (U)l, b = (U)r;
      o = (T)((op == OP_ADD) ? (U)(a + b) : (op == OP_SUB) ? (U)(a - b) : (op == OP_MUL) ? (U)(a * b) : (U)((U)0 - b));
      return false;
    } else if constexpr (CLS == CLS_CHECKED) {
      if constexpr (sizeof(T) < 8) {
        using W = typename std::conditional<SIGNED, int64_t, uint64_t>::type;
        W a = (W)l, b = (W)r;
        W w = (op == OP_ADD) ? a + b : (op == OP_SUB) ? a - b : (op == OP_MUL) ? a * b : (W)0 - b;
        o = (T)w;
        if constexpr (SIGNED) return w < (W)std::numeric_limits<T>::min() || w > (W)std::numeric_limits<T>::max();
        else return (op == OP_SUB) ? (a < b) : (op == OP_NEG ? false : w > (W)std::numeric_limits<T>::max());
      } else if constexpr (SIGNED) {
        int64_t a = l, b = r;
        if (op == OP_NEG) { a = 0; }
        if (op == OP_ADD) {
          int64_t s = (int64_t)((uint64_t)a + (uint64_t)b);
          o = s;
          return ((a ^ s) & (b ^ s)) < 0;
        } else if (op == OP_MUL) {
          int64_t lo = (int64_t)((uint64_t)a * (uint64_t)b);
          int64_t hi = __mul64hi(a, b);
          o = lo;
          return hi != (lo >> 63);
        } else {  // SUB / NEG
          int64_t s = (int64_t)((uint64_t)a - (uint64_t)b);
          o = s;
          return ((a ^ b) & (a ^ s)) < 0;
        }
      } else {
        uint64_t a = l, b = r;
        if (op == OP_ADD) { o = a + b; return o < a; }
        if (op == OP_MUL) { o = a * b; return __umul64hi(a, b) != 0; }
        if (op == OP_NEG) { o = (uint64_t)0 - b; return false; }
        o = a - b;
        return a < b;
      }
    } else {  // CLS_DIVREM: div_checked (arithmetic.rs:204-215) / rem (numeric.rs:345-351)
      o = 0;
      if (r == 0) return true;
      if constexpr (SIGNED) {
        if (r == (T)-1) {
          if (op == OP_DIV) {
            if (l == std::numeric_limits<T>::min()) return true;
            o = (T)(-l);
          }
          return false;  // rem: wrapping_rem(x, -1) == 0
        }
      }
      o = (op == OP_DIV) ? (T)(l / r) : (T)(l % r);
      return false;
    }
  }
}

// bitwise.rs rows (op = acu_bitwise_op), integer T only. Shifts are wrapping_shl / wrapping_shr by b's bit pattern modulo
// the width (bitwise.rs:81-111, :176-207). Narrow values shift in 32 bits: a left shift of a negative signed value is
// undefined, and a narrow unsigned one would be promoted to int.
template <int OP, class T> __device__ __forceinline__ T bitwise_row(T l, T r) {
  using U = typename std::make_unsigned<T>::type;
  using W = typename std::conditional<(sizeof(T) < 4), uint32_t, U>::type;
  using SW = typename std::conditional<(sizeof(T) < 4), int32_t, T>::type;
  const unsigned amt = (unsigned)((U)r & (U)(8 * sizeof(T) - 1));
  if constexpr (OP == ACU_BITWISE_AND) return l & r;
  else if constexpr (OP == ACU_BITWISE_OR) return l | r;
  else if constexpr (OP == ACU_BITWISE_XOR) return l ^ r;
  else if constexpr (OP == ACU_BITWISE_AND_NOT) return l & (T)~r;
  else if constexpr (OP == ACU_BITWISE_SHIFT_LEFT) return (T)((W)(U)l << amt);
  else if constexpr (OP == ACU_BITWISE_SHIFT_RIGHT) {  // arithmetic for signed, logical for unsigned T
    if constexpr (std::is_signed<T>::value) return (T)((SW)l >> amt);
    else return (T)((W)l >> amt);
  } else {
    return (T)~l;  // not
  }
}
// f(integral_constant<op>): one straight-line body per op, so that the op is decided once per strip group and not at
// each of its (up to 64 narrow) elements, which would spill
template <class F> __device__ __forceinline__ void bitwise_dispatch(int op, F &&f) {
  switch (op) {
    case ACU_BITWISE_AND: f(std::integral_constant<int, ACU_BITWISE_AND>()); break;
    case ACU_BITWISE_OR: f(std::integral_constant<int, ACU_BITWISE_OR>()); break;
    case ACU_BITWISE_XOR: f(std::integral_constant<int, ACU_BITWISE_XOR>()); break;
    case ACU_BITWISE_AND_NOT: f(std::integral_constant<int, ACU_BITWISE_AND_NOT>()); break;
    case ACU_BITWISE_SHIFT_LEFT: f(std::integral_constant<int, ACU_BITWISE_SHIFT_LEFT>()); break;
    case ACU_BITWISE_SHIFT_RIGHT: f(std::integral_constant<int, ACU_BITWISE_SHIFT_RIGHT>()); break;
    default: f(std::integral_constant<int, ACU_BITWISE_NOT>()); break;
  }
}
// The rows of 16 bytes of values: the logical ops act on whole 32-bit words, the shifts on each element in turn, so that
// 128-bit packs of narrow values are never unpacked into one register per element (they would spill).
template <int OP, class T> __device__ __forceinline__ uint32_t bitwise_word(uint32_t a, uint32_t b) {
  if constexpr (OP == ACU_BITWISE_SHIFT_LEFT || OP == ACU_BITWISE_SHIFT_RIGHT) {
    constexpr int BITS = 8 * sizeof(T);
    constexpr uint32_t MASK = BITS == 32 ? ~0u : (1u << (BITS & 31)) - 1u;
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 4 / (int)sizeof(T); ++i) {  // element i: bits [BITS*i, BITS*(i+1)) of the word
      const unsigned amt = (b >> (BITS * i)) & (BITS - 1);
      uint32_t r;
      if constexpr (OP == ACU_BITWISE_SHIFT_LEFT) r = (a >> (BITS * i)) << amt;
      else if constexpr (std::is_signed<T>::value) r = (uint32_t)((int32_t)(a << (32 - BITS * (i + 1))) >> (32 - BITS + amt));
      else r = ((a >> (BITS * i)) & MASK) >> amt;
      o |= (r & MASK) << (BITS * i);
    }
    return o;
  } else {
    return bitwise_row<OP, uint32_t>(a, b);
  }
}
template <int OP, class T> __device__ __forceinline__ uint4 bitwise_vec(uint4 a, uint4 b) {
  uint4 o;
  if constexpr (sizeof(T) == 8 && (OP == ACU_BITWISE_SHIFT_LEFT || OP == ACU_BITWISE_SHIFT_RIGHT)) {
    const T r0 = bitwise_row<OP, T>((T)(((uint64_t)a.y << 32) | a.x), (T)(((uint64_t)b.y << 32) | b.x));
    const T r1 = bitwise_row<OP, T>((T)(((uint64_t)a.w << 32) | a.z), (T)(((uint64_t)b.w << 32) | b.z));
    o.x = (uint32_t)(uint64_t)r0; o.y = (uint32_t)((uint64_t)r0 >> 32);
    o.z = (uint32_t)(uint64_t)r1; o.w = (uint32_t)((uint64_t)r1 >> 32);
  } else {
    o.x = bitwise_word<OP, T>(a.x, b.x);
    o.y = bitwise_word<OP, T>(a.y, b.y);
    o.z = bitwise_word<OP, T>(a.z, b.z);
    o.w = bitwise_word<OP, T>(a.w, b.w);
  }
  return o;
}

// One strip group of k_arith's CLS_BITWISE steady state: NL warp-wide loads per operand, all issued before any use, then
// the op decided once for the group. `a` is always an array (acu_bitwise).
template <class T, int EPL, int NL>
__device__ __forceinline__ void bitwise_group(int op, const T *__restrict__ pa, const T *__restrict__ pb, T *__restrict__ po,
                                              int b_scalar, T sb) {
  if constexpr (EPL * sizeof(T) == 16) {
    uint4 va[NL], vb[NL];
#pragma unroll
    for (int k = 0; k < NL; ++k) {
      va[k] = ld_stream16(pa + k * 32 * EPL);
      if (!b_scalar) vb[k] = ld_stream16(pb + k * 32 * EPL);
    }
    uint4 sv;  // the scalar in every element
    if constexpr (sizeof(T) == 8) {
      sv.x = sv.z = (uint32_t)(uint64_t)sb;
      sv.y = sv.w = (uint32_t)((uint64_t)sb >> 32);
    } else {
      sv.x = sv.y = sv.z = sv.w = (uint32_t)(typename std::make_unsigned<T>::type)sb * (sizeof(T) == 1 ? 0x01010101u : sizeof(T) == 2 ? 0x00010001u : 1u);
    }
    bitwise_dispatch(op, [&](auto c) {
#pragma unroll
      for (int k = 0; k < NL; ++k) st_stream16(po + k * 32 * EPL, bitwise_vec<decltype(c)::value, T>(va[k], b_scalar ? sv : vb[k]));
    });
  } else {
    static_assert(EPL == 1, "scalar path");
    T va[NL], vb[NL];
#pragma unroll
    for (int k = 0; k < NL; ++k) {
      va[k] = __ldg(pa + k * 32);
      if (!b_scalar) vb[k] = __ldg(pb + k * 32);
    }
    bitwise_dispatch(op, [&](auto c) {
#pragma unroll
      for (int k = 0; k < NL; ++k) po[k * 32] = bitwise_row<decltype(c)::value, T>(va[k], b_scalar ? sb : vb[k]);
    });
  }
}

template <class T> __device__ __forceinline__ T bitwise_apply(int op, T l, T r) {
  T o;
  bitwise_dispatch(op, [&](auto c) { o = bitwise_row<decltype(c)::value, T>(l, r); });
  return o;
}

// ---------------------------------------------------------------------------------------
// Decimal rows (decimal_op, numeric.rs:970-1107) on the natives int32_t / int64_t / __int128. Every step is checked
// (arithmetic.rs:148-300). Under strict C++17 std::is_signed / make_unsigned do not cover __int128, hence own traits.
// Host and device share these functions: the error finaliser replays the failing row with them.
// ---------------------------------------------------------------------------------------
template <class T> struct dec_unsigned { using type = typename std::make_unsigned<T>::type; };
template <> struct dec_unsigned<__int128> { using type = unsigned __int128; };
template <class T> __host__ __device__ __forceinline__ T dec_min() {
  return (T)((typename dec_unsigned<T>::type)1 << (8 * sizeof(T) - 1));
}

__host__ __device__ __forceinline__ uint64_t umul64hi(uint64_t a, uint64_t b) {
#ifdef __CUDA_ARCH__
  return __umul64hi(a, b);
#else
  return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
__host__ __device__ __forceinline__ int64_t mul64hi(int64_t a, int64_t b) {
#ifdef __CUDA_ARCH__
  return __mul64hi(a, b);
#else
  return (int64_t)(((__int128)a * b) >> 64);
#endif
}

// each returns true when the checked op overflows
template <class T> __host__ __device__ __forceinline__ bool add_ovf(T a, T b, T &o) {
  using U = typename dec_unsigned<T>::type;
  const T s = (T)((U)a + (U)b);
  o = s;
  return ((a ^ s) & (b ^ s)) < 0;
}
template <class T> __host__ __device__ __forceinline__ bool sub_ovf(T a, T b, T &o) {
  using U = typename dec_unsigned<T>::type;
  const T s = (T)((U)a - (U)b);
  o = s;
  return ((a ^ b) & (a ^ s)) < 0;
}
__host__ __device__ __forceinline__ bool mul_ovf(int32_t a, int32_t b, int32_t &o) {
  const int64_t w = (int64_t)a * b;
  o = (int32_t)w;
  return w != (int64_t)o;
}
__host__ __device__ __forceinline__ bool mul_ovf(int64_t a, int64_t b, int64_t &o) {
  const int64_t lo = (int64_t)((uint64_t)a * (uint64_t)b);
  o = lo;
  return mul64hi(a, b) != (lo >> 63);
}
// i128 x i128 with 64-bit limbs. Two operands that fit in i64 cannot overflow (one 64 x 64 -> 128 product);
// otherwise the magnitudes are multiplied and range-checked for the sign of the result.
__host__ __device__ __forceinline__ bool mul_ovf(__int128 a, __int128 b, __int128 &o) {
  const int64_t a64 = (int64_t)a, b64 = (int64_t)b;
  if ((__int128)a64 == a && (__int128)b64 == b) {
    const uint64_t lo = (uint64_t)a64 * (uint64_t)b64;
    o = (__int128)(((unsigned __int128)(uint64_t)mul64hi(a64, b64) << 64) | lo);
    return false;
  }
  using U = unsigned __int128;
  const bool neg = (a < 0) != (b < 0);
  const U ua = a < 0 ? (U)0 - (U)a : (U)a, ub = b < 0 ? (U)0 - (U)b : (U)b;
  const uint64_t ah = (uint64_t)(ua >> 64), al = (uint64_t)ua, bh = (uint64_t)(ub >> 64), bl = (uint64_t)ub;
  if (ah && bh) return true;
  const uint64_t x = ah ? ah : bh, y = ah ? bl : al;  // the one cross term that can be non-zero
  if (umul64hi(x, y)) return true;
  const uint64_t cross = x * y;
  const uint64_t hi = umul64hi(al, bl) + cross;
  if (hi < cross) return true;
  const U m = ((U)hi << 64) | (U)(al * bl);
  if (m > ((U)1 << 127) - (neg ? 0 : 1)) return true;
  o = neg ? (__int128)((U)0 - m) : (__int128)m;
  return false;
}
// div_checked / mod_checked: zero divisor, MIN / -1 and MIN % -1 fail; div truncates toward zero
template <class T> __host__ __device__ __forceinline__ bool divrem_ovf(bool is_div, T l, T r, T &o) {
  o = T();
  if (r == T()) return true;
  if (r == (T)-1) {
    if (l == dec_min<T>()) return true;
    if (is_div) o = (T)(T() - l);
    return false;
  }
  if constexpr (sizeof(T) == 16) {  // 64-bit division when both operands allow it; __int128 `/` is a software routine
    const int64_t l64 = (int64_t)l, r64 = (int64_t)r;
    if ((__int128)l64 == l && (__int128)r64 == r) {
      o = is_div ? l64 / r64 : l64 % r64;
      return false;
    }
  }
  o = is_div ? (T)(l / r) : (T)(l % r);
  return false;
}
// One row: add / sub / div / rem = l.mul_checked(l_mul)?.op(r.mul_checked(r_mul)?) (a multiplier of 1 is skipped: it
// cannot fail), mul = l.mul_checked(r), neg = r.neg_checked().
template <class T> __host__ __device__ __forceinline__ bool dec_apply(int op, T l, T r, T l_mul, T r_mul, T &o) {
  o = T();
  if (op == OP_NEG) return sub_ovf<T>(T(), r, o);
  if (op == OP_MUL) return mul_ovf(l, r, o);
  if (l_mul != (T)1 && mul_ovf(l, l_mul, l)) return true;
  if (r_mul != (T)1 && mul_ovf(r, r_mul, r)) return true;
  if (op == OP_ADD) return add_ovf<T>(l, r, o);
  if (op == OP_SUB) return sub_ovf<T>(l, r, o);
  return divrem_ovf<T>(op == OP_DIV, l, r, o);
}

// ---------------------------------------------------------------------------------------
// Binary / unary arithmetic kernel
// ---------------------------------------------------------------------------------------
template <class T>
struct ArithParams {
  const T *a, *b;
  T *out;
  int64_t n;
  const uint8_t *av, *bv;  // input validity bitmaps taking part in the union (or NULL)
  int64_t aoff, boff;
  uint64_t *out_valid;     // NULL => no NullBuffer in the result
  unsigned long long *res;
  int op;
  int a_scalar, b_scalar;
  int zero_nulls;          // try_binary / try_unary: zero under nulls, op only at valid slots
  T l_mul, r_mul;          // CLS_DECIMAL: rescale multipliers of add / sub / div / rem
};

template <class T, int CLS>
__device__ __forceinline__ bool row_op(const ArithParams<T> &p, T l, T r, T &o) {
  if constexpr (CLS == CLS_DECIMAL) return dec_apply<T>(p.op, l, r, p.l_mul, p.r_mul, o);
  else if constexpr (CLS == CLS_BITWISE) { o = bitwise_apply<T>(p.op, l, r); return false; }
  else return apply_op<T, CLS>(p.op, l, r, o);
}

// Steady state: a warp owns "super-groups" of 2048 rows = 32 validity words (lane l <-> word
// l: ONE coalesced 256-B bitmap access per operand per super-group), processed as groups of
// U strips whose loads are all issued before any use. The ragged remainder (< 2048 rows) is
// finished element-wise by warp 0 so that bounds-checked code stays out of the streaming loop.
// Decimal128 rows are 16 B per operand: U = 4 strips keep 128 B per operand and lane in flight, two CTAs per SM give
// the checked i128 steps their registers.
template <class T, int CLS, int EPL>
__global__ void __launch_bounds__(256, ((CLS == CLS_WRAP || CLS == CLS_BITWISE) ? 4 : (CLS == CLS_DECIMAL && sizeof(T) == 16) ? 2 : 3))
    k_arith(const ArithParams<T> p) {
  constexpr bool WIDE = CLS == CLS_DECIMAL && sizeof(T) == 16;
  constexpr int R = (32 * EPL > 64) ? 32 * EPL : 64;  // rows per strip
  constexpr int LPS = R / (32 * EPL);                 // loads per lane per strip
  constexpr int U = (LPS >= 2 && !WIDE) ? 2 : 4;      // strips in flight per warp
  constexpr int GROUP = U * R;                        // rows per group
  constexpr int SG = 2048;                            // rows per super-group
  constexpr int GPS = SG / GROUP;                     // groups per super-group
  constexpr bool fallible = (CLS != CLS_WRAP && CLS != CLS_BITWISE) && !is_fp<T>::value;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n = p.n;
  const int64_t sgroups = n / SG;
  const bool has_valid = p.out_valid != nullptr;
  T sa = T(), sb = T();
  if (p.a_scalar) sa = ldg_elem(p.a);
  if (p.b_scalar) sb = ldg_elem(p.b);
  unsigned valid_cnt = 0;
  unsigned long long err = ~0ull;

  for (int64_t sg = warp; sg < sgroups; sg += nwarps) {
    const int64_t sbase = sg * SG;
    uint64_t vw = ~0ull;  // lane l owns validity word l of the super-group
    if (has_valid) {
      const int64_t row = sbase + lane * 64;
      if (p.av) vw &= ld_bits64(p.av, p.aoff + row, p.aoff + n);
      if (p.bv) vw &= ld_bits64(p.bv, p.boff + row, p.boff + n);
      p.out_valid[row >> 6] = vw;
      valid_cnt += __popcll(vw);
    }
#pragma unroll 1
    for (int gi = 0; gi < GPS; ++gi) {
      const int64_t base = sbase + gi * GROUP;
      const T *__restrict__ pa = p.a + base + lane * EPL;
      const T *__restrict__ pb = p.b + base + lane * EPL;
      if constexpr (CLS == CLS_BITWISE) {  // `a` is always an array here (acu_bitwise)
        T *__restrict__ po = p.out + base + lane * EPL;
        bitwise_group<T, EPL, U * LPS>(p.op, pa, pb, po, p.b_scalar, sb);
        continue;
      }
      Pack<T, EPL> va[U * LPS], vb[U * LPS];
      // ---- every load of the group is issued before any use (memory-level parallelism) ----
#pragma unroll
      for (int k = 0; k < U * LPS; ++k) {
        if (!p.a_scalar) va[k] = pack_load<T, EPL>(pa + k * 32 * EPL);
        if (!p.b_scalar) vb[k] = pack_load<T, EPL>(pb + k * 32 * EPL);
      }
      // ---- compute + store ----
      T *__restrict__ po = p.out + base + lane * EPL;
#pragma unroll
      for (int k = 0; k < U * LPS; ++k) {
        uint32_t bits = ~0u;
        if (fallible && p.zero_nulls) {
          const int pos = gi * GROUP + k * 32 * EPL + lane * EPL;  // row inside the super-group
          const uint64_t w = __shfl_sync(ACU_FULL_MASK, vw, pos >> 6);
          bits = (uint32_t)(w >> (pos & 63));
        }
        Pack<T, EPL> o;
#pragma unroll
        for (int e = 0; e < EPL; ++e) {
          const T l = p.a_scalar ? sa : va[k].v[e];
          const T r = p.b_scalar ? sb : vb[k].v[e];
          T x;
          const bool bad = row_op<T, CLS>(p, l, r, x);
          if (fallible) {
            if (!((bits >> e) & 1u)) x = T();
            else if (bad) {
              const unsigned long long i = (unsigned long long)(base + k * 32 * EPL + lane * EPL + e);
              err = i < err ? i : err;
            }
          }
          o.v[e] = x;
        }
        pack_store<T, EPL>(po + k * 32 * EPL, o);
      }
    }
  }

  // ---- ragged remainder: 64-row strips, lane owns rows l and l+32 ----
  if (warp == 0) {
    for (int64_t row = sgroups * SG; row < n; row += 64) {
      uint64_t vw = ones_to(row, n);
      if (has_valid) {
        if (p.av) vw &= ld_bits64(p.av, p.aoff + row, p.aoff + n);
        if (p.bv) vw &= ld_bits64(p.bv, p.boff + row, p.boff + n);
        if (lane == 0) { p.out_valid[row >> 6] = vw; valid_cnt += __popcll(vw); }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t i = row + h * 32 + lane;
        if (i >= n) continue;
        const T l = p.a_scalar ? sa : ldg_elem(p.a + i);
        const T r = p.b_scalar ? sb : ldg_elem(p.b + i);
        T x;
        const bool bad = row_op<T, CLS>(p, l, r, x);
        if (fallible) {
          const bool live = !p.zero_nulls || ((vw >> (h * 32 + lane)) & 1ull);
          if (!live) x = T();
          else if (bad) err = (unsigned long long)i < err ? (unsigned long long)i : err;
        }
        p.out[i] = x;
      }
    }
  }
  if (has_valid) {
    valid_cnt = warp_sum(valid_cnt);
    if (lane == 0 && valid_cnt) atomicAdd(p.res + RES_COUNT, (unsigned long long)valid_cnt);
  }
  if (fallible && err != ~0ull) atomicMin(p.res + RES_ERR_INDEX, err);
}

template <class T, int CLS>
acu_status launch_arith(acu_ctx *ctx, const ArithParams<T> &p) {
  constexpr int EPLV = 16 / sizeof(T);
  bool aligned = ((uintptr_t)p.out % 16 == 0) && (p.a_scalar || (uintptr_t)p.a % 16 == 0) &&
                 (p.b_scalar || (uintptr_t)p.b % 16 == 0);
  const int64_t blocks = sg_blocks(p.n);
  if (aligned)
    ACU_LAUNCH_TIMED(ctx, ACU_K_ARITH, (k_arith<T, CLS, EPLV>), acu_wave_grid(ctx, k_arith<T, CLS, EPLV>, 256, 0, blocks), 256, 0, p);
  else
    ACU_LAUNCH_TIMED(ctx, ACU_K_ARITH, (k_arith<T, CLS, 1>), acu_wave_grid(ctx, k_arith<T, CLS, 1>, 256, 0, blocks), 256, 0, p);
  return ACU_OK;
}

const char *op_symbol(acu_arith_op op) {  // numeric.rs:192-202
  switch (op) {
    case ACU_ADD_WRAPPING: case ACU_ADD: return "+";
    case ACU_SUB_WRAPPING: case ACU_SUB: return "-";
    case ACU_MUL_WRAPPING: case ACU_MUL: return "*";
    case ACU_DIV: return "/";
    default: return "%";
  }
}

// Rust {:?} of i128: snprintf has no 128-bit conversion
void fmt_i128(char *buf, size_t n, __int128 v) {
  char tmp[48];
  int k = 0;
  unsigned __int128 m = v < 0 ? (unsigned __int128)0 - (unsigned __int128)v : (unsigned __int128)v;
  do { tmp[k++] = (char)('0' + (int)(m % 10)); m /= 10; } while (m);
  size_t j = 0;
  if (v < 0 && j + 1 < n) buf[j++] = '-';
  while (k && j + 1 < n) buf[j++] = tmp[--k];
  buf[j] = 0;
}
template <class T> void fmt_native(char *buf, size_t n, T v) {  // Rust {:?} of integers
  if constexpr (sizeof(T) == 16) fmt_i128(buf, n, v);
  else if constexpr (std::is_floating_point<T>::value) snprintf(buf, n, "%.17g", (double)v);
  else if constexpr (std::is_signed<T>::value) snprintf(buf, n, "%lld", (long long)v);
  else snprintf(buf, n, "%llu", (unsigned long long)v);
}
// bit pattern for acu_error_detail (the low 64 bits of an i128)
template <class T> uint64_t bits_of(T v) { uint64_t b = 0; memcpy(&b, &v, sizeof(T) < 8 ? sizeof(T) : 8); return b; }

// The rescale multipliers and result type of one decimal_op call (numeric.rs:991-1104).
template <class T> struct DecArgs {
  T l_mul, r_mul;
  int max_precision, max_scale;
  uint8_t precision;
  int8_t scale;
};

// with_precision_and_scale / validate_decimal_precision_and_scale (arrow-array/src/types.rs:1442-1472)
acu_status decimal_validate(acu_ctx *ctx, int max_precision, int max_scale, int precision, int scale) {
  if (precision == 0)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "precision cannot be 0, has to be between [1, %d]", max_precision);
  if (precision > max_precision)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "precision %d is greater than max %d", precision, max_precision);
  if (scale > max_scale)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "scale %d is greater than max %d", scale, max_scale);
  if (scale > 0 && scale > precision)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "scale %d is greater than precision %d", scale, precision);
  return ACU_OK;
}

// Fetch the operands at the lowest failing row and rebuild the reference's error. Decimal rows are replayed step by
// step with the device's own checked ops, so the message names the step that failed and its (rescaled) operands.
template <class T>
acu_status arith_error(acu_ctx *ctx, acu_arith_op op, bool is_neg, const acu_array *a, const acu_array *b, int64_t idx,
                       const DecArgs<T> *dec = nullptr) {
  T l = T(), r = T();
  if (a) ACU_CUDA(ctx, cudaMemcpyAsync(&l, static_cast<const T *>(a->values) + (a->is_scalar ? 0 : idx), sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
  ACU_CUDA(ctx, cudaMemcpyAsync(&r, static_cast<const T *>(b->values) + (b->is_scalar ? 0 : idx), sizeof(T), cudaMemcpyDeviceToHost, ctx->stream));
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const uint64_t lb = bits_of(l), rb = bits_of(r);
  T x = l, y = r;  // the operands of the failing step
  const char *sym = op_symbol(op);
  bool rescale_failed = false;
  if constexpr (std::is_same<T, int32_t>::value || std::is_same<T, int64_t>::value || sizeof(T) == 16) {
    if (dec && !is_neg && op != ACU_MUL && op != ACU_MUL_WRAPPING) {
      T t;
      if (dec->l_mul != (T)1 && mul_ovf(l, dec->l_mul, t)) {
        y = dec->l_mul, rescale_failed = true;
      } else {
        if (dec->l_mul != (T)1) x = t;
        if (dec->r_mul != (T)1 && mul_ovf(r, dec->r_mul, t)) x = r, y = dec->r_mul, rescale_failed = true;
        else if (dec->r_mul != (T)1) y = t;
      }
      if (rescale_failed) sym = "*";
    }
  }
  if ((op == ACU_DIV || op == ACU_REM) && !is_neg && !rescale_failed && y == T())
    return acu_fail(ctx, ACU_ERR_DIVIDE_BY_ZERO, idx, lb, rb, 0, "Divide by zero error");
  char ls[48], rs[48];
  fmt_native(ls, sizeof ls, x);
  fmt_native(rs, sizeof rs, y);
  if (is_neg)
    return acu_fail(ctx, ACU_ERR_ARITHMETIC_OVERFLOW, idx, rb, 0, 0, "Overflow happened on: - %s", rs);
  return acu_fail(ctx, ACU_ERR_ARITHMETIC_OVERFLOW, idx, lb, rb, 0, "Overflow happened on: %s %s %s", ls, sym, rs);
}

template <class T> acu_status launch_bitwise(acu_ctx *ctx, const ArithParams<T> &p) {
  if constexpr (std::is_integral<T>::value) return launch_arith<T, CLS_BITWISE>(ctx, p);
  else return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "bitwise operation on a non-integer type");
}

// DEC: decimal_op rows (every op checked, CLS_DECIMAL) with dec's multipliers, then its result-type validation.
// bitwise_op >= 0: a bitwise.rs op (acu_bitwise_op, CLS_BITWISE) through the same binary / unary rules as the wrapping ops;
// `op` is then unused.
template <class T, bool DEC = false>
acu_status arith_typed(acu_ctx *ctx, acu_arith_op op, const acu_array *a, const acu_array *b, acu_array_out *out,
                       const DecArgs<T> *dec = nullptr, int bitwise_op = -1) {
  const bool bitwise = bitwise_op >= 0;
  const bool checked = DEC || (!bitwise && !is_fp<T>::value && (op == ACU_ADD || op == ACU_SUB || op == ACU_MUL || op == ACU_DIV || op == ACU_REM));
  DecArgs<T> dv{};
  if constexpr (DEC) dv = *dec;
  auto validate = [ctx, dv]() -> acu_status {
    return DEC ? decimal_validate(ctx, dv.max_precision, dv.max_scale, dv.precision, dv.scale) : ACU_OK;
  };
  const bool a_s = a->is_scalar != 0, b_s = b->is_scalar != 0;
  acu_status st;
  ArithParams<T> p{};
  p.a = static_cast<const T *>(a->values);
  p.b = static_cast<const T *>(b->values);
  p.out = static_cast<T *>(out->values);
  p.res = ctx->d_res;
  p.a_scalar = a_s && !b_s;
  p.b_scalar = b_s && !a_s;
  switch (op) {
    case ACU_ADD_WRAPPING: case ACU_ADD: p.op = OP_ADD; break;
    case ACU_SUB_WRAPPING: case ACU_SUB: p.op = OP_SUB; break;
    case ACU_MUL_WRAPPING: case ACU_MUL: p.op = OP_MUL; break;
    case ACU_DIV: p.op = OP_DIV; break;
    default: p.op = OP_REM; break;
  }
  if (bitwise) p.op = bitwise_op;
  p.l_mul = DEC ? dv.l_mul : T();
  p.r_mul = DEC ? dv.r_mul : T();
  out->has_validity = 0;
  out->null_count = 0;
  int64_t len;
  if (a_s != b_s) {  // op!/try_op! scalar arms (numeric.rs:278-317)
    const acu_array *s = a_s ? a : b, *arr = a_s ? b : a;
    len = arr->len;
    int64_t snc = acu_resolve_null_count(ctx, s, &st);
    ACU_TRY(st);
    if (snc != 0) {
      ACU_TRY(acu_new_null(ctx, len, (size_t)len * sizeof(T), out));
      return validate();
    }
    out->len = len;
    if (len == 0) { out->has_validity = arr->validity != nullptr; return validate(); }
    if (arr->validity) {  // nulls().cloned()
      (a_s ? p.bv : p.av) = arr->validity;
      (a_s ? p.boff : p.aoff) = arr->validity_offset;
      p.out_valid = reinterpret_cast<uint64_t *>(out->validity);
      p.zero_nulls = checked;
    }
  } else {  // binary / try_binary (arity.rs:104-135, :254-299)
    if (a->len != b->len)
      return acu_fail(ctx, ACU_ERR_COMPUTE, -1, 0, 0, 0,
                      checked ? "Cannot perform a binary operation on arrays of different length"
                              : "Cannot perform binary operation on arrays of different length");
    len = a->len;
    out->len = len;
    if (len == 0) return validate();
    int64_t an = acu_resolve_null_count(ctx, a, &st);
    ACU_TRY(st);
    int64_t bn = acu_resolve_null_count(ctx, b, &st);
    ACU_TRY(st);
    // NullBuffer::union (null.rs:79-87)
    if (a->validity && b->validity && (an > 0 || bn > 0)) {
      p.av = a->validity; p.aoff = a->validity_offset;
      p.bv = b->validity; p.boff = b->validity_offset;
    } else if (a->validity && !b->validity && an > 0) {
      p.av = a->validity; p.aoff = a->validity_offset;
    } else if (b->validity && !a->validity && bn > 0) {
      p.bv = b->validity; p.boff = b->validity_offset;
    }
    if (p.av || p.bv) {
      p.out_valid = reinterpret_cast<uint64_t *>(out->validity);
      p.zero_nulls = checked;
    }
  }
  p.n = len;
  const int blk = acu_call_begin(ctx, &st);
  ACU_TRY(st);
  p.res = acu_dres(ctx, blk);
  if constexpr (DEC) {
    ACU_TRY((launch_arith<T, CLS_DECIMAL>(ctx, p)));
  } else if (bitwise) {
    ACU_TRY(launch_bitwise<T>(ctx, p));
  } else if (is_fp<T>::value) {
    if (op == ACU_DIV || op == ACU_REM) ACU_TRY((launch_arith<T, CLS_DIVREM>(ctx, p)));
    else ACU_TRY((launch_arith<T, CLS_WRAP>(ctx, p)));
  } else if (op == ACU_DIV || op == ACU_REM) {
    ACU_TRY((launch_arith<T, CLS_DIVREM>(ctx, p)));
  } else if (checked) {
    ACU_TRY((launch_arith<T, CLS_CHECKED>(ctx, p)));
  } else {
    ACU_TRY((launch_arith<T, CLS_WRAP>(ctx, p)));
  }
  const acu_array ca = *a, cb = *b;  // the finaliser may run later (acu_results_fetch)
  const bool has_valid = p.out_valid != nullptr;
  return acu_call_end(ctx, blk, [ctx, op, checked, ca, cb, has_valid, len, out, dv, validate](const unsigned long long *h) -> acu_status {
    if (checked && h[RES_ERR_INDEX] != ~0ull) return arith_error<T>(ctx, op, false, &ca, &cb, (int64_t)h[RES_ERR_INDEX], DEC ? &dv : nullptr);
    if (has_valid) {
      out->has_validity = 1;
      out->null_count = len - (int64_t)h[RES_COUNT];
    }
    return validate();
  });
}

// Decimal128 (T = __int128) is always neg_checked, on the decimal class, and stream-ordered inside sections.
template <class T>
acu_status neg_typed(acu_ctx *ctx, int32_t checked_in, const acu_array *a, acu_array_out *out) {
  constexpr bool DEC = sizeof(T) == 16;
  const bool checked = DEC || (checked_in && !is_fp<T>::value);
  int64_t len = a->len;
  out->len = len;
  out->has_validity = a->validity != nullptr;
  out->null_count = 0;
  if (len == 0) return ACU_OK;
  ArithParams<T> p{};
  p.a = static_cast<const T *>(a->values);  // ignored by OP_NEG (a_scalar => one broadcast load)
  p.b = static_cast<const T *>(a->values);
  p.out = static_cast<T *>(out->values);
  p.res = ctx->d_res;
  p.a_scalar = 1;
  p.op = OP_NEG;
  p.n = len;
  if (a->validity) {  // unary / try_unary: nulls().cloned()
    p.bv = a->validity;
    p.boff = a->validity_offset;
    p.out_valid = reinterpret_cast<uint64_t *>(out->validity);
    p.zero_nulls = checked;
  }
  if constexpr (DEC) {
    acu_status st;
    const int blk = acu_call_begin(ctx, &st);
    ACU_TRY(st);
    p.res = acu_dres(ctx, blk);
    p.l_mul = p.r_mul = 1;
    ACU_TRY((launch_arith<T, CLS_DECIMAL>(ctx, p)));
    const acu_array ca = *a;
    const bool has_valid = p.out_valid != nullptr;
    return acu_call_end(ctx, blk, [ctx, ca, has_valid, len, out](const unsigned long long *h) -> acu_status {
      if (h[RES_ERR_INDEX] != ~0ull) return arith_error<T>(ctx, ACU_SUB, true, nullptr, &ca, (int64_t)h[RES_ERR_INDEX]);
      if (has_valid) out->null_count = len - (int64_t)h[RES_COUNT];
      return ACU_OK;
    });
  } else {
    ACU_TRY(acu_res_reset(ctx));
    if (checked) ACU_TRY((launch_arith<T, CLS_CHECKED>(ctx, p)));
    else ACU_TRY((launch_arith<T, CLS_WRAP>(ctx, p)));
    ACU_TRY(acu_res_fetch(ctx));
    if (checked && ctx->h_res[RES_ERR_INDEX] != ~0ull)
      return arith_error<T>(ctx, ACU_SUB, true, nullptr, a, (int64_t)ctx->h_res[RES_ERR_INDEX]);
    if (p.out_valid) out->null_count = len - (int64_t)ctx->h_res[RES_COUNT];
    return ACU_OK;
  }
}

// ---------------------------------------------------------------------------------------
// cmp — one result bit per row (collect_bool, cmp.rs:580-611)
// ---------------------------------------------------------------------------------------
template <class T>
struct CmpParams {
  const T *a, *b;
  int64_t n;
  const uint8_t *av, *bv;
  int64_t aoff, boff;
  int a_scalar, b_scalar;
  int a_null_scalar, b_null_scalar;  // scalar side whose single slot is null
  int neg, fold;
  uint64_t *out_bits, *out_valid;
  unsigned long long *res;
  // fused compare -> filter plan (acu_filter_plan_create_cmp): out_bits is the plan's mask and receives result & validity;
  // tile_count[t] = selected rows of 1024-row tile t
  int fuse;
  uint32_t *tile_count;
};

template <class T> __device__ __forceinline__ bool pred_eq(T l, T r) {
  if constexpr (sizeof(T) == 8 && is_fp<T>::value) return __double_as_longlong(l) == __double_as_longlong(r);
  else if constexpr (is_fp<T>::value) return __float_as_int(l) == __float_as_int(r);
  else return l == r;
}
template <class T> __device__ __forceinline__ bool pred_lt(T l, T r) {
  if constexpr (is_fp<T>::value) return total_key(l) < total_key(r);
  else return l < r;
}

// A super-group's 2048 rows are read as 2048 / (32*EPL) warp-wide loads; lane l holds rows [l*EPL, (l+1)*EPL) of
// each. `bits` has one bit per such row (bit e = row l*EPL + e). The rows of load `load` fill EPL 32-bit halves of the
// super-group's bit string, and each half is ONE warp OR-reduction (redux.sync) of the lanes' shifted bits. Half h goes
// to lane h/2, so lane l ends up owning word l of the super-group (rows [l*64, l*64+64)) as (lo, hi).
template <int EPL>
__device__ __forceinline__ void pack_lane_bits(uint32_t bits, int load, uint32_t &lo, uint32_t &hi) {
  const int lane = threadIdx.x & 31;
  bits <<= (lane * EPL) & 31;              // where this lane's EPL bits land inside their 32-bit half
  const int my_half = (lane * EPL) >> 5;   // which half of the load's bit string they belong to
#pragma unroll
  for (int hh = 0; hh < EPL; ++hh) {
    const uint32_t half = __reduce_or_sync(ACU_FULL_MASK, my_half == hh ? bits : 0u);
    const int h = load * EPL + hh;         // 32-bit half inside the super-group
    if (lane == (h >> 1)) { if (h & 1) hi = half; else lo = half; }
  }
}

// A warp owns 2048-row super-groups = 32 result words. Every lane reads EPL elements per warp-wide load (128-bit
// vectors when the value pointers are 16-B aligned, one element otherwise), 4 loads in flight, and ends up owning
// result word l and validity word l: one coalesced 256-B store each per super-group. The ragged tail (< 2048 rows) is
// finished by warp 0 in 64-row strips: lane l compares rows l and l+32, two ballots give the packed word. In fuse mode
// it also writes the tail's (at most two) tile counts.
template <class T, bool LT, int EPL>
__global__ void __launch_bounds__(256, 4) k_cmp(const CmpParams<T> p) {
  constexpr int RPL = 32 * EPL;          // rows per warp-wide load
  constexpr int LOADS = 2048 / RPL;      // loads per super-group
  constexpr int U = LOADS < 4 ? LOADS : 4;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n = p.n;
  const int64_t sgroups = n >> 11;
  T sa = T(), sb = T();
  if (p.a_scalar) sa = ldg_elem(p.a);
  if (p.b_scalar) sb = ldg_elem(p.b);
  unsigned valid_cnt = 0;
  for (int64_t sg = warp; sg < sgroups; sg += nwarps) {
    const int64_t sbase = sg << 11;
    uint64_t lw = ~0ull, rw = ~0ull;  // lane-owned validity words
    if (p.a_null_scalar) lw = 0;
    if (p.b_null_scalar) rw = 0;
    const int64_t wrow = sbase + lane * 64;
    if (p.av) lw &= ld_bits64(p.av, p.aoff + wrow, p.aoff + n);
    if (p.bv) rw &= ld_bits64(p.bv, p.boff + wrow, p.boff + n);
    uint32_t my_lo = 0, my_hi = 0;    // lane-owned result word
#pragma unroll 1
    for (int l0 = 0; l0 < LOADS; l0 += U) {
      Pack<T, EPL> va[U], vb[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i0 = sbase + (int64_t)(l0 + u) * RPL + lane * EPL;
        if (!p.a_scalar) va[u] = pack_load<T, EPL>(p.a + i0);
        if (!p.b_scalar) vb[u] = pack_load<T, EPL>(p.b + i0);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        uint32_t x = 0;
#pragma unroll
        for (int e = 0; e < EPL; ++e) {
          const T l = p.a_scalar ? sa : va[u].v[e];
          const T r = p.b_scalar ? sb : vb[u].v[e];
          x |= (uint32_t)(LT ? pred_lt(l, r) : pred_eq(l, r)) << e;
        }
        pack_lane_bits<EPL>(x, l0 + u, my_lo, my_hi);
      }
    }
    uint64_t v = (uint64_t)my_lo | ((uint64_t)my_hi << 32);
    if (p.neg) v = ~v;
    if (p.fold == FOLD_DISTINCT) v = (lw ^ rw) | (lw & rw & v);
    else if (p.fold == FOLD_NOT_DISTINCT) v = ~(lw | rw) | (lw & rw & v);
    if (p.fuse) {
      if (p.fold == FOLD_NONE) v &= lw & rw;
      unsigned c = __popcll(v);
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) c += __shfl_xor_sync(ACU_FULL_MASK, c, o);  // sum inside each 16-lane half = one 1024-row tile
      if ((lane & 15) == 0) p.tile_count[(sbase >> 10) + (lane >> 4)] = c;
    }
    p.out_bits[(sbase >> 6) + lane] = v;
    if (p.out_valid) {
      p.out_valid[(sbase >> 6) + lane] = lw & rw;
      valid_cnt += __popcll(lw & rw);
    }
  }

  if (warp == 0) {
    unsigned tile_cnt = 0;
    for (int64_t row = sgroups << 11; row < n; row += 64) {
      uint64_t v = 0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t i = row + h * 32 + lane;
        const T l = (!p.a_scalar && i < n) ? ldg_elem(p.a + i) : sa;
        const T r = (!p.b_scalar && i < n) ? ldg_elem(p.b + i) : sb;
        v |= (uint64_t)__ballot_sync(ACU_FULL_MASK, LT ? pred_lt(l, r) : pred_eq(l, r)) << (h * 32);
      }
      if (p.neg) v = ~v;
      if (lane == 0) {
        const uint64_t m = ones_to(row, n);
        v &= m;
        uint64_t lw = p.a_null_scalar ? 0ull : m, rw = p.b_null_scalar ? 0ull : m;
        if (p.av) lw &= ld_bits64(p.av, p.aoff + row, p.aoff + n);
        if (p.bv) rw &= ld_bits64(p.bv, p.boff + row, p.boff + n);
        if (p.fold == FOLD_DISTINCT) v = (lw ^ rw) | (lw & rw & v);              // cmp.rs:331
        else if (p.fold == FOLD_NOT_DISTINCT) v = (~(lw | rw) & m) | (lw & rw & v);  // cmp.rs:341
        else if (p.fuse) v &= lw & rw;  // a null result selects nothing (filter.rs:167-171)
        p.out_bits[row >> 6] = v;
        if (p.out_valid) {
          p.out_valid[row >> 6] = lw & rw;
          valid_cnt += __popcll(lw & rw);
        }
        if (p.fuse) {  // a tile ends every 16 words and at the last word
          tile_cnt += __popcll(v);
          if (row + 64 >= n || ((row + 64) & 1023) == 0) { p.tile_count[row >> 10] = tile_cnt; tile_cnt = 0; }
        }
      }
    }
  }
  if (p.out_valid) {
    valid_cnt = warp_sum(valid_cnt);
    if (lane == 0 && valid_cnt) atomicAdd(p.res + RES_COUNT, (unsigned long long)valid_cnt);
  }
}

template <class T, int EPL>
acu_status launch_cmp(acu_ctx *ctx, bool lt, const CmpParams<T> &p) {
  const int64_t blocks = sg_blocks(p.n);
  if (lt) ACU_LAUNCH_TIMED(ctx, ACU_K_CMP, (k_cmp<T, true, EPL>), acu_wave_grid(ctx, k_cmp<T, true, EPL>, 256, 0, blocks), 256, 0, p);
  else ACU_LAUNCH_TIMED(ctx, ACU_K_CMP, (k_cmp<T, false, EPL>), acu_wave_grid(ctx, k_cmp<T, false, EPL>, 256, 0, blocks), 256, 0, p);
  return ACU_OK;
}

struct CmpFuse {  // destination of a fused compare -> filter plan
  uint64_t *mask;
  int64_t n_words_padded;
  uint32_t *tile_count;
  int64_t n_tiles;
};

template <class T>
acu_status cmp_typed(acu_ctx *ctx, acu_cmp_op op, const acu_array *l, const acu_array *r, acu_array_out *out, const CmpFuse *fuse = nullptr) {
  acu_array_out scratch_out{};
  if (fuse) out = &scratch_out;
  acu_cmp_decision d;
  ACU_TRY(acu_cmp_decide(ctx, op, l, r, out, &d));
  const int64_t len = d.len;
  if (len == 0) return ACU_OK;
  if (fuse) {  // words past the data (the plan pads its mask to a multiple of 32 words) select nothing
    const int64_t used = (len + 63) / 64;
    if (fuse->n_words_padded > used)
      ACU_CUDA(ctx, cudaMemsetAsync(fuse->mask + used, 0, (size_t)(fuse->n_words_padded - used) * 8, ctx->stream));
  }
  if (d.all_null) {
    if (fuse) {  // an all-null predicate selects nothing
      ACU_CUDA(ctx, cudaMemsetAsync(fuse->mask, 0, (size_t)fuse->n_words_padded * 8, ctx->stream));
      ACU_CUDA(ctx, cudaMemsetAsync(fuse->tile_count, 0, (size_t)fuse->n_tiles * 4, ctx->stream));
      return ACU_OK;
    }
    return acu_new_null(ctx, len, acu_bitmap_bytes(len), out);
  }
  CmpParams<T> p{};
  p.a = static_cast<const T *>((d.swap ? r : l)->values);
  p.b = static_cast<const T *>((d.swap ? l : r)->values);
  p.n = len;
  p.av = d.av; p.aoff = d.aoff;
  p.bv = d.bv; p.boff = d.boff;
  p.a_scalar = d.a_scalar; p.a_null_scalar = d.a_null_scalar;
  p.b_scalar = d.b_scalar; p.b_null_scalar = d.b_null_scalar;
  p.neg = d.neg;
  p.fold = d.fold;
  p.out_bits = fuse ? fuse->mask : static_cast<uint64_t *>(out->values);
  if (d.has_validity && !fuse) p.out_valid = reinterpret_cast<uint64_t *>(out->validity);
  p.res = ctx->d_res;
  if (fuse) { p.fuse = 1; p.tile_count = fuse->tile_count; }
  int blk = 0;
  if (!fuse) {
    acu_status st;
    blk = acu_call_begin(ctx, &st);
    ACU_TRY(st);
    p.res = acu_dres(ctx, blk);
  }
  // 128-bit loads when both non-scalar value pointers are 16-B aligned, one element per lane otherwise
  const bool aligned = (p.a_scalar || (uintptr_t)p.a % 16 == 0) && (p.b_scalar || (uintptr_t)p.b % 16 == 0);
  if (aligned) ACU_TRY((launch_cmp<T, 16 / sizeof(T)>(ctx, d.lt, p)));
  else ACU_TRY((launch_cmp<T, 1>(ctx, d.lt, p)));
  if (fuse) return ACU_OK;  // stream-ordered: the plan's scan kernels follow on the same stream
  return acu_call_end(ctx, blk, [d, out](const unsigned long long *h) -> acu_status {
    acu_cmp_finalize(d, h, out);
    return ACU_OK;
  });
}

// ---------------------------------------------------------------------------------------
// cast (numeric): unary_opt / try_unary over num_traits::cast (num-traits 0.2.19)
// ---------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ int clz64(uint64_t x) {
#ifdef __CUDA_ARCH__
  return __clzll((long long)x);
#else
  return x ? __builtin_clzll(x) : 64;
#endif
}
// An integral double with |v| < 2^127 as i128 (exact: the value has at most 53 significant bits).
__host__ __device__ __forceinline__ __int128 f64_to_i128(double v) {
  if (v > -9.2e18 && v < 9.2e18) return (__int128)(int64_t)v;
  int e;
  const double fr = frexp(fabs(v), &e);  // |v| = fr * 2^e, fr in [0.5, 1), e >= 63 > 53
  const unsigned __int128 m = (unsigned __int128)(uint64_t)ldexp(fr, 53) << (e - 53);
  return v < 0 ? (__int128)((unsigned __int128)0 - m) : (__int128)m;
}

template <class I, class O>
__host__ __device__ __forceinline__ bool num_cast(I v, O &o) {
  if constexpr (sizeof(O) == 16) {  // f64 -> i128 (num_traits to_i128): -2^127 <= v < 2^127
    static_assert(is_fp<I>::value, "integer -> i128 is a widening, not a num_cast");
    if (!(v >= -1.7014118346046923e38 && v < 1.7014118346046923e38)) return false;
    o = f64_to_i128((double)v);
    return true;
  } else if constexpr (is_fp<O>::value) {
    o = (O)v;  // cvt.rn: int->float RNE, f64->f32 RNE (overflow -> inf), always Some
    return true;
  } else if constexpr (is_fp<I>::value) {
    if (v != v) return false;
    constexpr bool OS = std::is_signed<O>::value;
    if constexpr (sizeof(I) > sizeof(O)) {
      const I lo = OS ? (I)std::numeric_limits<O>::min() - (I)1 : (I)-1;
      const I hi = (I)std::numeric_limits<O>::max() + (I)1;
      if (!(v > lo && v < hi)) return false;
    } else {
      const I hi = (I)std::numeric_limits<O>::max();
      if constexpr (OS) { if (!(v >= (I)std::numeric_limits<O>::min() && v < hi)) return false; }
      else { if (!(v > (I)-1 && v < hi)) return false; }
    }
    o = (O)v;  // truncates toward zero for in-range values
    return true;
  } else {
    constexpr bool IS = std::is_signed<I>::value, OS = std::is_signed<O>::value;
    if constexpr (IS == OS) {
      if (v < std::numeric_limits<O>::min() || v > std::numeric_limits<O>::max()) return false;
    } else if constexpr (IS) {
      if (v < 0) return false;
      if ((typename std::make_unsigned<I>::type)v > std::numeric_limits<O>::max()) return false;
    } else {
      if (v > (typename std::make_unsigned<O>::type)std::numeric_limits<O>::max()) return false;
    }
    o = (O)v;
    return true;
  }
}

// Casts that cannot fail (anything -> float, widening integer casts) compile without the failure bookkeeping.
template <class I, class O> struct cast_infallible {
  static constexpr bool value = is_fp<O>::value ||
      (!is_fp<I>::value && ((std::is_signed<I>::value == std::is_signed<O>::value && sizeof(O) >= sizeof(I)) ||
                            (!std::is_signed<I>::value && std::is_signed<O>::value && sizeof(O) > sizeof(I))));
};
template <class O, int EPL> struct alignas((sizeof(O) * EPL >= 16) ? 16 : sizeof(O) * EPL) OutPack { O v[EPL]; };

// The layout of k_cmp: 2048-row super-groups, EPL input elements per lane and load (128-bit vectors when both pointers
// are 16-B aligned, one element otherwise), lane-owned validity words, ragged tail finished by warp 0. unary_opt /
// try_unary: the cast runs at valid slots only, zero elsewhere. A valid slot whose value does not fit O becomes null
// (`safe`) or reports its row, the lowest one winning (atomicMin).
template <class I, class O, int EPL>
__global__ void __launch_bounds__(256, 4) k_cast(const I *__restrict__ in, O *__restrict__ out, const int64_t n,
                                                 const uint8_t *__restrict__ iv, const int64_t ioff, uint64_t *__restrict__ out_valid,
                                                 const int safe, unsigned long long *__restrict__ res) {
  constexpr bool fallible = !cast_infallible<I, O>::value;
  constexpr int RPL = 32 * EPL;
  constexpr int LOADS = 2048 / RPL;
  constexpr int U = LOADS < 4 ? LOADS : 4;
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t sgroups = n >> 11;
  unsigned valid_cnt = 0;
  unsigned long long err = ~0ull;
  for (int64_t sg = warp; sg < sgroups; sg += nwarps) {
    const int64_t sbase = sg << 11;
    uint64_t vw = ~0ull;
    if (iv) vw = ld_bits64(iv, ioff + sbase + lane * 64, ioff + n);
    uint32_t bad_lo = 0, bad_hi = 0;  // lane-owned word: valid slots whose value does not fit O
#pragma unroll 1
    for (int l0 = 0; l0 < LOADS; l0 += U) {
      Pack<I, EPL> v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = pack_load<I, EPL>(in + sbase + (int64_t)(l0 + u) * RPL + lane * EPL);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int pos = (l0 + u) * RPL + lane * EPL;
        const uint64_t w = __shfl_sync(ACU_FULL_MASK, vw, pos >> 6);
        const uint32_t bits = (uint32_t)(w >> (pos & 63));
        OutPack<O, EPL> o;
        uint32_t bad = 0;
#pragma unroll
        for (int e = 0; e < EPL; ++e) {
          O x = O();
          if (((bits >> e) & 1u) && !num_cast<I, O>(v[u].v[e], x)) bad |= 1u << e;
          o.v[e] = x;
        }
        *reinterpret_cast<OutPack<O, EPL> *>(out + sbase + pos) = o;
        if (fallible && __any_sync(ACU_FULL_MASK, bad)) pack_lane_bits<EPL>(bad, l0 + u, bad_lo, bad_hi);  // failures are rare
      }
    }
    const uint64_t bad = (uint64_t)bad_lo | ((uint64_t)bad_hi << 32);
    if (fallible && bad) {
      if (safe) vw &= ~bad;  // unrepresentable => null
      else err = min(err, (unsigned long long)(sbase + lane * 64 + __ffsll((long long)bad) - 1));
    }
    if (out_valid) { out_valid[(sbase >> 6) + lane] = vw; valid_cnt += __popcll(vw); }
  }

  if (warp == 0) {
    for (int64_t row = sgroups << 11; row < n; row += 64) {
      uint64_t vw = ones_to(row, n);
      if (iv) vw &= ld_bits64(iv, ioff + row, ioff + n);
      uint64_t bad = 0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t i = row + h * 32 + lane;
        O x = O();
        const bool b = ((vw >> (h * 32 + lane)) & 1ull) && !num_cast<I, O>(__ldg(in + i), x);
        if (i < n) out[i] = x;
        if constexpr (fallible) bad |= (uint64_t)__ballot_sync(ACU_FULL_MASK, b) << (h * 32);
      }
      if (fallible && bad) {
        if (safe) vw &= ~bad;
        else err = min(err, (unsigned long long)(row + __ffsll((long long)bad) - 1));
      }
      if (out_valid && lane == 0) { out_valid[row >> 6] = vw; valid_cnt += __popcll(vw); }
    }
  }
  if (out_valid) {
    valid_cnt = warp_sum(valid_cnt);
    if (lane == 0 && valid_cnt) atomicAdd(res + RES_COUNT, (unsigned long long)valid_cnt);
  }
  if (fallible && err != ~0ull) atomicMin(res + RES_ERR_INDEX, err);
}

// ACU_I128 values are read and written as 16-byte vectors: the pointers must have the alignment of i128.
acu_status i128_aligned(acu_ctx *ctx, const void *x, const void *y) {
  if (((uintptr_t)x | (uintptr_t)y) % 16 != 0)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Int128 values must be 16-byte aligned");
  return ACU_OK;
}

// ---------------------------------------------------------------------------------------
// decimal_op's result type and multipliers (numeric.rs:991-1104), in Rust's i8 / u8 arithmetic. Where the reference's
// i8 subtractions overflow (debug builds panic) this wraps, as a release build does.
// ---------------------------------------------------------------------------------------
int8_t i8_wrap(int v) { return (int8_t)(uint8_t)(v & 0xff); }
int8_t i8_sat(int v) { return (int8_t)(v < -128 ? -128 : v > 127 ? 127 : v); }
uint8_t u8_sat(int v) { return (uint8_t)(v > 255 ? 255 : v); }
uint8_t u8_of(int8_t v) { return (uint8_t)v; }                  // `as u8`
uint32_t u32_of(int8_t v) { return (uint32_t)(int32_t)v; }      // `as u32` (sign-extending)

template <class T> bool pow10_checked(uint32_t exp, T *out) {  // 10.checked_pow(exp)
  T v = 1;
  for (uint32_t i = 0; i < exp; ++i)
    if (mul_ovf(v, (T)10, v)) return false;
  *out = v;
  return true;
}
template <class T> T pow10_wrapping(uint32_t exp) {  // 10.wrapping_pow(exp): 2^exp divides 10^exp, so 0 from exp = bits
  using U = typename dec_unsigned<T>::type;
  if (exp >= 8 * sizeof(T)) return T();
  U v = 1;
  for (uint32_t i = 0; i < exp; ++i) v *= 10;
  return (T)v;
}

const char *decimal_name(int width) { return width == 4 ? "Decimal32" : width == 8 ? "Decimal64" : "Decimal128"; }

template <class T>
acu_status decimal_typed(acu_ctx *ctx, acu_arith_op op, const acu_decimal_type &lt, const acu_array *a, const acu_decimal_type &rt,
                         const acu_array *b, acu_decimal_type *out_type, acu_array_out *out) {
  constexpr int MP = sizeof(T) == 4 ? 9 : sizeof(T) == 8 ? 18 : 38;  // MAX_PRECISION = MAX_SCALE
  const int p1 = lt.precision, p2 = rt.precision, s1 = lt.scale, s2 = rt.scale;
  DecArgs<T> d{};
  d.l_mul = d.r_mul = 1;
  d.max_precision = d.max_scale = MP;
  uint32_t le = 0, re = 0;  // exponents of the checked multipliers
  bool pow_l = false, pow_r = false;
  switch (op) {
    case ACU_ADD: case ACU_ADD_WRAPPING: case ACU_SUB: case ACU_SUB_WRAPPING: case ACU_REM: {
      const int8_t rs = (int8_t)(s1 > s2 ? s1 : s2);
      const int8_t d1 = i8_wrap(p1 - s1), d2 = i8_wrap(p2 - s2);
      if (op == ACU_REM) {
        d.precision = (uint8_t)std::min<int>(u8_of(i8_sat(rs + std::min(d1, d2))), MP);
        d.l_mul = pow10_wrapping<T>(u32_of(i8_wrap(rs - s1)));
        d.r_mul = pow10_wrapping<T>(u32_of(i8_wrap(rs - s2)));
      } else {
        d.precision = (uint8_t)std::min<int>(u8_sat(u8_of(i8_sat(rs + std::max(d1, d2))) + 1), MP);
        le = u32_of(i8_wrap(rs - s1));
        re = u32_of(i8_wrap(rs - s2));
        pow_l = pow_r = true;
      }
      d.scale = rs;
      break;
    }
    case ACU_MUL: case ACU_MUL_WRAPPING: {
      d.precision = (uint8_t)std::min<int>(u8_sat(p1 + p2 + 1), MP);
      d.scale = i8_sat(s1 + s2);
      if (d.scale > MP)
        return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Output scale of %s(%d, %d) * %s(%d, %d) would exceed max scale of %d",
                        decimal_name(lt.byte_width), p1, s1, decimal_name(rt.byte_width), p2, s2, MP);
      break;
    }
    case ACU_DIV: {
      const int8_t rs = (int8_t)std::min<int>(i8_sat(s1 + 4), MP);
      const int8_t mul_pow = i8_wrap(i8_wrap(rs - s1) + s2);
      d.precision = (uint8_t)std::min<int>(u8_of(i8_sat(mul_pow + p1)), MP);
      d.scale = rs;
      if (mul_pow > 0) { le = u32_of(mul_pow); pow_l = true; }
      else if (mul_pow < 0) { re = u32_of(i8_wrap(-mul_pow)); pow_r = true; }
      break;
    }
    default:
      return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid arithmetic operation: op %d", (int)op);
  }
  if (pow_l && !pow10_checked<T>(le, &d.l_mul))
    return acu_fail(ctx, ACU_ERR_ARITHMETIC_OVERFLOW, -1, 0, 0, 0, "Overflow happened on: 10 ^ %u", le);
  if (pow_r && !pow10_checked<T>(re, &d.r_mul))
    return acu_fail(ctx, ACU_ERR_ARITHMETIC_OVERFLOW, -1, 0, 0, 0, "Overflow happened on: 10 ^ %u", re);
  out_type->byte_width = lt.byte_width;
  out_type->precision = d.precision;
  out_type->scale = d.scale;
  out_type->reserved[0] = out_type->reserved[1] = 0;
  return arith_typed<T, true>(ctx, op, a, b, out, &d);
}

// ---------------------------------------------------------------------------------------
// Decimal casts (arrow-cast/src/cast/decimal.rs:161-529, :836-1004; mod.rs:86-92, :366-444). One row function per kind,
// shared by the device and the host replay of a failing row. Every per-call constant (10^k, the rounding half, the output
// precision's bounds, the powi multiplier) is computed once on the host. cast_launch launches and finalises these and
// the numeric casts (DK_NUM: k_cast over num_cast).
// ---------------------------------------------------------------------------------------
// decimal / integer / float -> decimal, decimal -> integer / float, numeric -> numeric
enum { DK_DEC = 0, DK_INT = 1, DK_FLOAT = 2, DK_TO_INT = 3, DK_TO_FLOAT = 4, DK_NUM = 5 };
enum { DM_UNARY = 0, DM_OPT = 1, DM_TRY = 2 };  // unary (every slot; a failure is the unwrap panic), unary_opt / builder (valid slots; failure -> null), try_unary (valid slots; failure -> error)
enum { DR_OK = 0, DR_NONE = 1, DR_MUL = 2, DR_PRECISION = 3 };  // row outcome: the conversion returned None / the checked multiply failed / outside the output precision

struct DcastArgs {
  __int128 k;       // 10^delta: the multiplier or divisor, in the native that applies it
  __int128 half;    // k / 2 (downscale rounding)
  __int128 lo, hi;  // MIN / MAX_FOR_EACH_PRECISION[p_out]; lo > hi when p_out exceeds MAX_PRECISION (nothing fits)
  double fk;        // 10_f64.powi(scale)
  uint32_t chunk[5];  // k = product of these powers of ten (each <= 10^9): the full-width i128 division
  int nchunk;
  int down;   // DK_DEC: divide by k and round; DK_INT / DK_TO_INT: divide by k (else multiply)
  int zero;   // the all-zero shortcuts
  int wrap;   // the infallible upscale multiplies wrapping
  int check;  // is_valid_decimal_precision after the conversion
};

// O::from_decimal / NumCast / integer_to_decimal_native: does the (integral) value fit O?
template <class O, class T> __host__ __device__ __forceinline__ bool fits_in(T v) {
  if constexpr (sizeof(O) == 16) return true;  // every source native fits i128
  else if constexpr (sizeof(T) == 16) {
    if constexpr (std::is_signed<O>::value)
      return v >= (__int128)std::numeric_limits<O>::min() && v <= (__int128)std::numeric_limits<O>::max();
    else return v >= 0 && v <= (__int128)std::numeric_limits<O>::max();
  } else {
    O o;
    return num_cast<T, O>(v, o);
  }
}

// u128 / d for d < 2^32: long division over 32-bit limbs, three 64-bit divisions.
__host__ __device__ __forceinline__ unsigned __int128 udiv_u32(unsigned __int128 x, uint32_t d) {
  const uint64_t hi = (uint64_t)(x >> 64), lo = (uint64_t)x;
  const uint64_t qh = hi / d;
  uint64_t t = ((hi % d) << 32) | (lo >> 32);
  const uint64_t q1 = t / d;
  t = ((t % d) << 32) | (lo & 0xffffffffull);
  return ((unsigned __int128)qh << 64) | (q1 << 32) | (t / d);
}

// Magnitude quotient and remainder by k = 10^delta. A value below 2^64 with k below 2^64 takes one 64-bit division; a
// full-width i128 is divided by k's <= 10^9 factors in turn (floor(floor(x / a) / b) = floor(x / ab)).
template <class I>
__host__ __device__ __forceinline__ void udivmod_k(typename dec_unsigned<I>::type m, const DcastArgs &a, typename dec_unsigned<I>::type &q,
                                                   typename dec_unsigned<I>::type &r) {
  using U = typename dec_unsigned<I>::type;
  const U k = (U)a.k;
  if constexpr (sizeof(I) == 16) {
    if ((m >> 64) == 0 && (k >> 64) == 0) {
      q = (uint64_t)m / (uint64_t)k;
    } else {
      q = m;
      for (int c = 0; c < a.nchunk; ++c) q = udiv_u32(q, a.chunk[c]);
    }
  } else {
    q = m / k;
  }
  r = m - q * k;
}

__host__ __device__ __forceinline__ double i128_to_f64(__int128 v) {  // `as f64`: round to nearest, ties to even
  const int64_t v64 = (int64_t)v;
  if ((__int128)v64 == v) return (double)v64;
  using U = unsigned __int128;
  const U m = v < 0 ? (U)0 - (U)v : (U)v;
  const int bits = 128 - clz64((uint64_t)(m >> 64));  // >= 64
  const int sh = bits - 64;
  // the top 64 bits with every lower bit folded into a sticky bit 0: one RNE conversion rounds exactly as the whole value
  uint64_t top = (uint64_t)(m >> sh);
  if (sh > 0 && (m & ((U(1) << sh) - 1)) != 0) top |= 1;
  const double d = ldexp((double)top, sh);
  return v < 0 ? -d : d;
}
__host__ __device__ __forceinline__ double dmul_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}
__host__ __device__ __forceinline__ double ddiv_rn(double a, double b) {
#ifdef __CUDA_ARCH__
  return __ddiv_rn(a, b);
#else
  return a / b;
#endif
}

// One row. `mid` receives the value a message prints: the narrowed value whose multiply failed (DK_INT), the scaled
// value (DK_TO_INT), the value outside the output precision.
template <class I, class O, int KIND>
__host__ __device__ __forceinline__ int dcast_row(const DcastArgs &a, I v, O &o, __int128 &mid) {
  if (a.zero) { o = O(); return DR_OK; }
  if constexpr (KIND == DK_DEC || KIND == DK_INT) {
    if (a.down) {
      // decimal downscale: div_wrapping / mod_wrapping in I, rounded half away from zero (decimal.rs:237-249);
      // integer to a negative scale: div_checked in I (mod.rs:398-401)
      using U = typename dec_unsigned<I>::type;
      const bool neg = v < I();
      const U m = neg ? (U)0 - (U)v : (U)v;
      U q, r;
      udivmod_k<I>(m, a, q, r);
      if (KIND == DK_DEC && r >= (U)a.half) q += 1;
      const I d = neg ? (I)((U)0 - q) : (I)q;
      if (!fits_in<O>(d)) return DR_NONE;
      o = (O)d;
    } else {
      if (!fits_in<O>(v)) return DR_NONE;  // from_decimal / integer_to_decimal_native
      const O x = (O)v, k = (O)a.k;
      using U = typename dec_unsigned<O>::type;
      if (a.wrap) { o = (O)((U)x * (U)k); return DR_OK; }  // infallible: mul_wrapping
      if (k != (O)1 && mul_ovf(x, k, o)) { mid = (__int128)x; return KIND == DK_INT ? DR_MUL : DR_NONE; }
      if (k == (O)1) o = x;
    }
  } else if constexpr (KIND == DK_FLOAT) {
    // single_float_to_decimal: (mul * v).round() (one IEEE multiply, round half away from zero), then to_i32 / i64 / i128
    const double x = round(dmul_rn(a.fk, (double)v));
    if (!num_cast<double, O>(x, o)) return DR_NONE;
  } else if constexpr (KIND == DK_TO_INT) {
    I s;
    if (a.down) {  // div_checked by 10^scale: truncates toward zero
      using U = typename dec_unsigned<I>::type;
      const bool neg = v < I();
      const U m = neg ? (U)0 - (U)v : (U)v;
      U q, r;
      udivmod_k<I>(m, a, q, r);
      s = neg ? (I)((U)0 - q) : (I)q;
    } else if (mul_ovf(v, (I)a.k, s)) {
      mid = (__int128)v;
      return DR_MUL;
    }
    mid = (__int128)s;
    if (!fits_in<O>(s)) return DR_NONE;
    o = (O)s;
    return DR_OK;
  } else {  // DK_TO_FLOAT: (x as f64) / 10_f64.powi(scale), `as f32` after for Float32
    double x;
    if constexpr (sizeof(I) == 16) x = i128_to_f64(v);
    else x = (double)v;
    o = (O)ddiv_rn(x, a.fk);
    return DR_OK;
  }
  if constexpr (KIND != DK_TO_INT && KIND != DK_TO_FLOAT) {
    if (a.check && !((O)a.lo <= o && o <= (O)a.hi)) { mid = (__int128)o; return DR_PRECISION; }
  }
  return DR_OK;
}

template <class I, class O>
struct DcastParams {
  const I *in;
  O *out;
  int64_t n;
  const uint8_t *iv;
  int64_t ioff;
  uint64_t *out_valid;
  unsigned long long *res;
  int mode;
  DcastArgs a;
};

// k_cast's layout, one element per lane and load (rows are 4-16 B, so a warp-wide load is already one coalesced
// 128-512 B request): 2048-row super-groups, lane-owned validity words, the ragged tail finished by warp 0, the lowest
// failing row by atomicMin. A sibling of k_cast rather than k_cast over this row function: ptxas (CUDA 12.9, sm_90a) gives
// the merged kernel more registers either way its parameters are passed. With one parameter struct, 95 of the 170
// numeric casts grow (up to +6, e.g. i32 -> i8 48 -> 54); with k_cast's separate parameters, 15 of these 69 do
// (i128 -> Decimal32 rescale 72 -> 96, i8 -> Decimal64 40 -> 48).
template <class I, class O, int KIND>
__global__ void __launch_bounds__(256, (sizeof(I) == 16 || sizeof(O) == 16) ? 2 : 4) k_dcast(const DcastParams<I, O> p) {
  constexpr int U = 4;  // loads in flight per lane
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t n = p.n;
  const int64_t sgroups = n >> 11;
  const bool every = p.mode == DM_UNARY;
  unsigned valid_cnt = 0;
  unsigned long long err = ~0ull;
  for (int64_t sg = warp; sg < sgroups; sg += nwarps) {
    const int64_t sbase = sg << 11;
    uint64_t vw = ~0ull;
    if (p.iv) vw = ld_bits64(p.iv, p.ioff + sbase + lane * 64, p.ioff + n);
    const uint64_t live = every ? ~0ull : vw;  // rows the cast runs at
    uint32_t bad_lo = 0, bad_hi = 0;
#pragma unroll 1
    for (int l0 = 0; l0 < 64; l0 += U) {
      I v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) v[u] = ldg_elem(p.in + sbase + (int64_t)(l0 + u) * 32 + lane);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int pos = (l0 + u) * 32 + lane;
        const uint64_t w = __shfl_sync(ACU_FULL_MASK, live, pos >> 6);
        O x = O();
        bool bad = false;
        if ((w >> (pos & 63)) & 1ull) {
          __int128 mid;
          bad = dcast_row<I, O, KIND>(p.a, v[u], x, mid) != DR_OK;
          if (bad) x = O();
        }
        p.out[sbase + pos] = x;
        if (__any_sync(ACU_FULL_MASK, bad)) pack_lane_bits<1>(bad, l0 + u, bad_lo, bad_hi);  // failures are rare
      }
    }
    const uint64_t bad = (uint64_t)bad_lo | ((uint64_t)bad_hi << 32);
    if (bad) {
      if (p.mode == DM_OPT) vw &= ~bad;
      else err = min(err, (unsigned long long)(sbase + lane * 64 + __ffsll((long long)bad) - 1));
    }
    if (p.out_valid) { p.out_valid[(sbase >> 6) + lane] = vw; valid_cnt += __popcll(vw); }
  }

  if (warp == 0) {
    for (int64_t row = sgroups << 11; row < n; row += 64) {
      uint64_t vw = ones_to(row, n);
      if (p.iv) vw &= ld_bits64(p.iv, p.ioff + row, p.ioff + n);
      const uint64_t live = every ? ones_to(row, n) : vw;
      uint64_t bad = 0;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t i = row + h * 32 + lane;
        O x = O();
        bool b = false;
        if ((live >> (h * 32 + lane)) & 1ull) {
          __int128 mid;
          b = dcast_row<I, O, KIND>(p.a, ldg_elem(p.in + i), x, mid) != DR_OK;
          if (b) x = O();
        }
        if (i < n) p.out[i] = x;
        bad |= (uint64_t)__ballot_sync(ACU_FULL_MASK, b) << (h * 32);
      }
      if (bad) {
        if (p.mode == DM_OPT) vw &= ~bad;
        else err = min(err, (unsigned long long)(row + __ffsll((long long)bad) - 1));
      }
      if (p.out_valid && lane == 0) { p.out_valid[row >> 6] = vw; valid_cnt += __popcll(vw); }
    }
  }
  if (p.out_valid) {
    valid_cnt = warp_sum(valid_cnt);
    if (lane == 0 && valid_cnt) atomicAdd(p.res + RES_COUNT, (unsigned long long)valid_cnt);
  }
  if (err != ~0ull) atomicMin(p.res + RES_ERR_INDEX, err);
}

int dec_max_precision(int width) { return width == 4 ? 9 : width == 8 ? 18 : 38; }
__int128 pow10_i128(int k) {
  __int128 v = 1;
  for (int i = 0; i < k; ++i) v *= 10;
  return v;
}
// O::MIN / MAX_FOR_EACH_PRECISION[p] (arrow-data/src/decimal.rs), or an empty range when p is past the table
void precision_bounds(int width, int p, DcastArgs &a) {
  if (p > dec_max_precision(width)) { a.lo = 1; a.hi = 0; return; }
  a.hi = pow10_i128(p) - 1;
  a.lo = -a.hi;
}
// 10^k as factors of at most 10^9, for the full-width division
void set_k(DcastArgs &a, int k) {
  a.k = pow10_i128(k);
  a.half = a.k / 2;
  a.nchunk = 0;
  for (int left = k; left > 0; left -= 9) a.chunk[a.nchunk++] = (uint32_t)pow10_i128(left < 9 ? left : 9);
}
// 10_f64.powi(e): compiler-builtins' `pow` (what llvm.powi calls for a runtime exponent): repeated squaring, then 1 / r
// for a negative exponent. Not always the correctly rounded 10^e (it differs at e = 33, 34, 37 and most e <= -23).
double powi10(int e) {
  double a = 10.0, r = 1.0;
  const bool recip = e < 0;
  uint32_t k = recip ? (uint32_t)0 - (uint32_t)e : (uint32_t)e;
  for (;;) {
    if (k & 1) r *= a;
    k >>= 1;
    if (!k) break;
    a *= a;
  }
  return recip ? 1.0 / r : r;
}

// format_decimal_str_internal (arrow-data/src/decimal.rs:1137-1167), truncation quirk included
void fmt_decimal_str(char *buf, size_t n, const char *value, int precision, int scale, bool safe) {
  const bool neg = value[0] == '-';
  const char *rest = neg ? value + 1 : value;
  const size_t rlen = strlen(rest);
  const size_t bound = safe ? std::min<size_t>((size_t)precision, rlen) + (neg ? 1 : 0) : strlen(value);
  char v[64];
  snprintf(v, sizeof v, "%.*s", (int)bound, value);
  const size_t vlen = strlen(v);
  const std::string zeros(scale < 0 ? (size_t)-scale : (size_t)scale - std::min<size_t>(rlen, (size_t)scale), '0');
  if (scale == 0) snprintf(buf, n, "%s", v);
  else if (scale < 0) snprintf(buf, n, "%s%s", v, zeros.c_str());
  else if (rlen > (size_t)scale) snprintf(buf, n, "%.*s.%s", (int)(vlen - scale), v, v + vlen - scale);
  else snprintf(buf, n, "%s0.%s%s", neg ? "-" : "", zeros.c_str(), rest);
}
// validate_decimal{32,64,}_precision's error (arrow-data/src/decimal.rs:1030ff)
acu_status precision_error(acu_ctx *ctx, int width, __int128 v, int p, int s, int64_t idx, uint64_t bits) {
  const char *name = decimal_name(width);
  const int mp = dec_max_precision(width);
  if (p > mp) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, idx, bits, 0, 0, "Max precision of a %s is %d, but got %d", name, mp, p);
  const __int128 hi = p ? pow10_i128(p) - 1 : 0;
  char vs[48], bs[48], a[96], b[96];
  fmt_i128(vs, sizeof vs, v);
  fmt_i128(bs, sizeof bs, v > hi ? hi : -hi);
  fmt_decimal_str(a, sizeof a, vs, p, s, false);
  fmt_decimal_str(b, sizeof b, bs, p, s, true);
  return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, idx, bits, 0, 0, "%s is too %s to store in a %s of precision %d. %s is %s", a,
                  v > hi ? "large" : "small", name, p, v > hi ? "Max" : "Min", b);
}

// Rust's `{:?}` of f32 / f64: the shortest digits that round-trip in the value's own type; plain notation with at least one
// fractional digit when 1e-4 <= |v| < 1e16 or v == 0, else `1e40` / `1.5e-7`.
void fmt_float_debug(char *buf, size_t n, double v, bool f32) {
  if (v != v) { snprintf(buf, n, "NaN"); return; }
  if (std::isinf(v)) { snprintf(buf, n, v < 0 ? "-inf" : "inf"); return; }
  if (v == 0) { snprintf(buf, n, std::signbit(v) ? "-0.0" : "0.0"); return; }
  char t[64];
  for (int prec = 0; prec <= 17; ++prec) {
    snprintf(t, sizeof t, "%.*e", prec, v);
    if (f32 ? strtof(t, nullptr) == (float)v : strtod(t, nullptr) == v) break;
  }
  char digits[32];
  int nd = 0;
  const char *c = t + (t[0] == '-');
  for (; *c != 'e'; ++c) if (*c != '.') digits[nd++] = *c;
  const int e = atoi(c + 1);
  while (nd > 1 && digits[nd - 1] == '0') --nd;
  digits[nd] = 0;
  const double a = fabs(v);
  const bool expo = f32 ? (a < (double)1e-4f || a >= (double)1e16f) : (a < 1e-4 || a >= 1e16);
  char out[96];
  int k = 0;
  if (v < 0) out[k++] = '-';
  if (expo) {
    out[k++] = digits[0];
    if (nd > 1) { out[k++] = '.'; for (int i = 1; i < nd; ++i) out[k++] = digits[i]; }
    k += snprintf(out + k, sizeof out - k, "e%d", e);
  } else if (e >= 0) {
    for (int i = 0; i <= e; ++i) out[k++] = i < nd ? digits[i] : '0';
    out[k++] = '.';
    if (nd > e + 1) for (int i = e + 1; i < nd; ++i) out[k++] = digits[i];
    else out[k++] = '0';
  } else {
    out[k++] = '0';
    out[k++] = '.';
    for (int i = 0; i < -e - 1; ++i) out[k++] = '0';
    for (int i = 0; i < nd; ++i) out[k++] = digits[i];
  }
  out[k] = 0;
  snprintf(buf, n, "%s", out);
}

template <class T> void fmt_value(char *buf, size_t n, T v) {
  if constexpr (std::is_floating_point<T>::value) fmt_float_debug(buf, n, (double)v, sizeof(T) == 4);
  else fmt_native(buf, n, v);
}

// What a failing row turns into; `what` names the output type of the messages ("Decimal32(9, 2)").
struct DcastCall {
  int kind;
  int mode;
  int safe;
  int out_width;        // decimal outputs: 4 / 8 / 16
  uint8_t precision;    // decimal outputs
  int8_t scale;
  acu_dtype out_dtype;  // integer / float outputs
  bool builder;         // decimal -> integer: a NullBuffer only when some row is null
};

template <class I, class O, int KIND>
acu_status cast_launch(acu_ctx *ctx, const DcastCall &c, const DcastArgs &args, const acu_array *a, acu_array_out *out) {
  const int64_t len = a->len;
  out->len = len;
  out->null_count = 0;
  // unary_opt (numeric_cast when safe) always carries a NullBuffer; unary / try_unary clone the input's; the builder
  // decides after the rows
  out->has_validity = c.mode == DM_OPT || (a->validity != nullptr);
  if (len == 0) {
    if (c.builder) out->has_validity = 0;
    return ACU_OK;
  }
  const I *in = static_cast<const I *>(a->values);
  O *dst = static_cast<O *>(out->values);
  uint64_t *ov = out->has_validity ? reinterpret_cast<uint64_t *>(out->validity) : nullptr;
  ACU_TRY(acu_res_reset(ctx));
  const int64_t blocks = sg_blocks(len);
  if constexpr (KIND == DK_NUM) {
    // An 8-byte input read one element per lane is already one coalesced 256-B warp request; on an H100 that beats 16-B
    // vectors for these casts (f64 -> i32 and i64 -> f64 at 1e8 and 1e9 rows), so only narrower inputs are vectorised.
    constexpr int EPLV = sizeof(I) == 8 ? 1 : 16 / sizeof(I);
    if ((uintptr_t)in % 16 == 0 && (uintptr_t)dst % 16 == 0)
      ACU_LAUNCH_TIMED(ctx, ACU_K_CAST, (k_cast<I, O, EPLV>), acu_wave_grid(ctx, k_cast<I, O, EPLV>, 256, 0, blocks), 256, 0,
                       in, dst, len, a->validity, a->validity_offset, ov, c.safe, ctx->d_res);
    else
      ACU_LAUNCH_TIMED(ctx, ACU_K_CAST, (k_cast<I, O, 1>), acu_wave_grid(ctx, k_cast<I, O, 1>, 256, 0, blocks), 256, 0,
                       in, dst, len, a->validity, a->validity_offset, ov, c.safe, ctx->d_res);
  } else {
    const DcastParams<I, O> p{in, dst, len, a->validity, a->validity_offset, ov, ctx->d_res, c.mode, args};
    ACU_LAUNCH_TIMED(ctx, ACU_K_CAST, (k_dcast<I, O, KIND>), acu_wave_grid(ctx, k_dcast<I, O, KIND>, 256, 0, blocks), 256, 0, p);
  }
  ACU_TRY(acu_res_fetch(ctx));
  if (ctx->h_res[RES_ERR_INDEX] != ~0ull) {
    const int64_t idx = (int64_t)ctx->h_res[RES_ERR_INDEX];
    I v;
    ACU_CUDA(ctx, cudaMemcpyAsync(&v, in + idx, sizeof(I), cudaMemcpyDeviceToHost, ctx->stream));
    ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const uint64_t bits = bits_of(v);
    if constexpr (KIND == DK_NUM) {  // try_numeric_cast: num_traits::cast returned None
      char s[40];
      fmt_native(s, sizeof s, v);
      return acu_fail(ctx, ACU_ERR_CAST, idx, bits, 0, 0, "Can't cast value %s to type %s", s, acu_dtype_name(c.out_dtype));
    } else {
      if (c.mode == DM_UNARY)  // from_decimal(x).unwrap() / f_fallible(x).unwrap() on a slot that does not convert
        return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, idx, bits, 0, 0, "called `Option::unwrap()` on a `None` value");
      O o;
      __int128 mid = 0;
      const int r = dcast_row<I, O, KIND>(args, v, o, mid);
      char vs[64], ms[48], ks[48];
      fmt_value(vs, sizeof vs, v);
      fmt_i128(ms, sizeof ms, mid);
      fmt_i128(ks, sizeof ks, args.k);
      if (r == DR_PRECISION) return precision_error(ctx, c.out_width, mid, c.precision, c.scale, idx, bits);
      if (r == DR_MUL) return acu_fail(ctx, ACU_ERR_ARITHMETIC_OVERFLOW, idx, bits, 0, 0, "Overflow happened on: %s * %s", ms, ks);
      if (KIND == DK_TO_INT)
        return acu_fail(ctx, ACU_ERR_CAST, idx, bits, 0, 0, "value of %s is out of range %s", ms, acu_dtype_name(c.out_dtype));
      return acu_fail(ctx, ACU_ERR_CAST, idx, bits, 0, 0, "Cannot cast to %s(%d, %d). Overflowing on %s", decimal_name(c.out_width),
                      (int)c.precision, (int)c.scale, vs);
    }
  }
  if (ov) out->null_count = len - (int64_t)ctx->h_res[RES_COUNT];
  if (c.builder && out->null_count == 0) out->has_validity = 0;
  return ACU_OK;
}

template <class I, class O, int KIND>
acu_status dcast_to_decimal(acu_ctx *ctx, const DcastCall &c, const DcastArgs &args, const acu_array *a, acu_array_out *out) {
  ACU_TRY((cast_launch<I, O, KIND>(ctx, c, args, a, out)));
  const int mp = dec_max_precision(c.out_width);
  return decimal_validate(ctx, mp, mp, c.precision, c.scale);  // with_precision_and_scale, after the rows
}

template <class I, int KIND>
acu_status dcast_to_width(acu_ctx *ctx, const DcastCall &c, const DcastArgs &args, const acu_array *a, acu_array_out *out) {
  if (c.out_width == 4) return dcast_to_decimal<I, int32_t, KIND>(ctx, c, args, a, out);
  if (c.out_width == 8) return dcast_to_decimal<I, int64_t, KIND>(ctx, c, args, a, out);
  return dcast_to_decimal<I, __int128, KIND>(ctx, c, args, a, out);
}

// decimal -> decimal: cast_decimal_to_decimal(_same_type), decimal.rs:448-529 with make_upscaler / make_downscaler
template <class I>
acu_status cast_decimal_typed(acu_ctx *ctx, const acu_decimal_type &from, const acu_decimal_type &to, int32_t safe,
                              const acu_array *a, acu_array_out *out) {
  const int p_in = from.precision, s_in = from.scale, p_out = to.precision, s_out = to.scale;
  DcastCall c{DK_DEC, DM_UNARY, safe, to.byte_width, to.precision, to.scale, ACU_I8, false};
  DcastArgs args{};
  precision_bounds(to.byte_width, p_out, args);
  if (from.byte_width == to.byte_width && s_in == s_out && p_in <= p_out) {
    // array.clone() (decimal.rs:461), decided in u8 before any i8 arithmetic: the same bytes, the input's nulls. Run as the
    // identity unary (multiply by 1), which reproduces them exactly.
    set_k(args, 0);
    c.mode = DM_UNARY, args.wrap = 1;
  } else if (s_in <= s_out) {
    const int8_t delta = i8_wrap(s_out - s_in);
    if (delta < 0 || delta > dec_max_precision(to.byte_width))  // O::MAX_FOR_EACH_PRECISION.get(delta as usize) misses
      return acu_fail(ctx, ACU_ERR_CAST, -1, 0, 0, 0, "Cannot cast to %s(%d, %d). Value overflows for output scale",
                      decimal_name(to.byte_width), p_out, s_out);
    set_k(args, delta);
    if (i8_wrap((int8_t)p_in + delta) <= (int8_t)p_out) c.mode = DM_UNARY, args.wrap = 1;
    else c.mode = safe ? DM_OPT : DM_TRY, args.check = 1;
  } else {
    const int8_t delta = i8_wrap(s_in - s_out);
    if (delta < 0 || delta > dec_max_precision(from.byte_width)) {  // past I's table: every value rounds to zero
      args.zero = 1;
    } else {
      set_k(args, delta);
      args.down = 1;
      if (i8_wrap((int8_t)p_in - delta) < (int8_t)p_out) c.mode = DM_UNARY;
      else c.mode = safe ? DM_OPT : DM_TRY, args.check = 1;
    }
  }
  return dcast_to_width<I, DK_DEC>(ctx, c, args, a, out);
}

// integer -> decimal: cast_integer_to_decimal, mod.rs:366-444
template <class I>
acu_status cast_int_to_decimal(acu_ctx *ctx, const acu_decimal_type &to, int32_t safe, const acu_array *a, acu_array_out *out) {
  DcastCall c{DK_INT, safe ? DM_OPT : DM_TRY, safe, to.byte_width, to.precision, to.scale, ACU_I8, false};
  DcastArgs args{};
  precision_bounds(to.byte_width, to.precision, args);
  args.check = 1;
  const uint32_t e = to.scale < 0 ? (uint32_t)(-(int)to.scale) : (uint32_t)to.scale;
  if (to.scale < 0) {  // 10^|scale| in the source type
    if (!pow10_checked<__int128>(e, &args.k) || !fits_in<I>(args.k)) {
      args.zero = 1, c.mode = DM_UNARY;  // a factor beyond the source type: every quotient is 0 (unary)
    } else {
      set_k(args, (int)e);
      args.down = 1;
    }
  } else {
    bool ok;
    if (to.byte_width == 4) { int32_t k; ok = pow10_checked<int32_t>(e, &k); }
    else if (to.byte_width == 8) { int64_t k; ok = pow10_checked<int64_t>(e, &k); }
    else { __int128 k; ok = pow10_checked<__int128>(e, &k); }
    if (!ok)
      return acu_fail(ctx, ACU_ERR_CAST, -1, 0, 0, 0, "Cannot cast to \"%s\"(%d, %d). The scale causes overflow.",
                      decimal_name(to.byte_width), (int)to.precision, (int)to.scale);
    set_k(args, (int)e);
  }
  return dcast_to_width<I, DK_INT>(ctx, c, args, a, out);
}

// float -> decimal: cast_floating_point_to_decimal, decimal.rs:836-885
template <class I>
acu_status cast_float_to_decimal(acu_ctx *ctx, const acu_decimal_type &to, int32_t safe, const acu_array *a, acu_array_out *out) {
  DcastCall c{DK_FLOAT, safe ? DM_OPT : DM_TRY, safe, to.byte_width, to.precision, to.scale, ACU_I8, false};
  DcastArgs args{};
  precision_bounds(to.byte_width, to.precision, args);
  args.check = 1;
  args.fk = powi10(to.scale);
  return dcast_to_width<I, DK_FLOAT>(ctx, c, args, a, out);
}

// decimal -> integer / float: cast_decimal_to_integer / cast_decimal_to_float, decimal.rs:887-1004
template <class I, class O>
acu_status cast_from_decimal_typed(acu_ctx *ctx, const acu_decimal_type &from, acu_dtype to, int32_t safe, const acu_array *a,
                                   acu_array_out *out) {
  DcastArgs args{};
  if constexpr (is_fp<O>::value) {
    DcastCall c{DK_TO_FLOAT, DM_UNARY, safe, 0, 0, 0, to, false};
    args.fk = powi10(from.scale);
    return cast_launch<I, O, DK_TO_FLOAT>(ctx, c, args, a, out);
  } else {
    DcastCall c{DK_TO_INT, safe ? DM_OPT : DM_TRY, safe, 0, 0, 0, to, true};
    const uint32_t e = from.scale < 0 ? (uint32_t)(-(int)from.scale) : (uint32_t)from.scale;
    I k;
    if (!pow10_checked<I>(e, &k))
      return acu_fail(ctx, ACU_ERR_CAST, -1, 0, 0, 0, "Cannot cast to \"%s\". The scale %d causes overflow.",
                      decimal_name(from.byte_width), (int)from.scale);
    set_k(args, (int)e);
    args.down = from.scale >= 0;
    return cast_launch<I, O, DK_TO_INT>(ctx, c, args, a, out);
  }
}

template <class I>
acu_status cast_from_decimal_to(acu_ctx *ctx, const acu_decimal_type &from, acu_dtype to, int32_t safe, const acu_array *a,
                                acu_array_out *out) {
  return acu_with_native(
      to, [&](auto o) { return cast_from_decimal_typed<I, decltype(o)>(ctx, from, to, safe, a, out); },
      [&] {
        return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, -1, 0, 0, 0, "cast from %s to dtype %d", decimal_name(from.byte_width), (int)to);
      });
}

// the operand's decimal type is an array's: refused like an invalid type (with_precision_and_scale) at call time
acu_status decimal_type_ok(acu_ctx *ctx, const acu_decimal_type *t) {
  const int w = t->byte_width;
  if (w != 4 && w != 8 && w != 16)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid decimal type: byte width %d", (int)w);
  const int mp = dec_max_precision(w);
  return decimal_validate(ctx, mp, mp, t->precision, t->scale);
}

}  // namespace

extern "C" acu_status acu_arith(acu_ctx *ctx, acu_dtype dtype, acu_arith_op op, const acu_array *a,
                                const acu_array *b, acu_array_out *out) {
  ACU_ENTER(ctx);
  return acu_with_native(
      dtype, [&](auto t) { return arith_typed<decltype(t)>(ctx, op, a, b, out); },
      [&] { return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid arithmetic operation: dtype %d", (int)dtype); });
}

extern "C" acu_status acu_neg(acu_ctx *ctx, acu_dtype dtype, int32_t checked, const acu_array *a, acu_array_out *out) {
  ACU_ENTER(ctx);
  if (checked && (dtype == ACU_U8 || dtype == ACU_U16 || dtype == ACU_U32 || dtype == ACU_U64))  // numeric.rs:174-176
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid arithmetic operation: !%s", acu_dtype_name(dtype));
  if (dtype == ACU_I128) {
    ACU_TRY(i128_aligned(ctx, a->values, out->values));
    return neg_typed<__int128>(ctx, 1, a, out);
  }
  return acu_with_native(
      dtype, [&](auto t) { return neg_typed<decltype(t)>(ctx, checked, a, out); },
      [&] { return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid arithmetic operation: dtype %d", (int)dtype); });
}

// bitwise.rs: array-array ops through `binary`, the _scalar forms and not through `unary` (arith_typed's scalar arm with
// the array's nulls cloned; not reads its operand as both sides, the scalar side ignored by the row).
extern "C" acu_status acu_bitwise(acu_ctx *ctx, acu_dtype dtype, acu_bitwise_op op, const acu_array *a, const acu_array *b,
                                  acu_array_out *out) {
  ACU_ENTER(ctx);
  if (dtype < ACU_I8 || dtype > ACU_U64)  // PrimitiveArray<T> with T::Native: BitAnd + ... : the integer types only
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid bitwise operation: dtype %d", (int)dtype);
  if (op < ACU_BITWISE_AND || op > ACU_BITWISE_NOT)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid bitwise operation: op %d", (int)op);
  if (a->is_scalar) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "bitwise: the left operand must be an array");
  acu_array self_b;
  if (op == ACU_BITWISE_NOT) {
    self_b = *a;
    self_b.validity = nullptr;
    self_b.null_count = 0;
    self_b.len = 1;
    self_b.is_scalar = 1;
    b = &self_b;
  } else if (!b) {
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "bitwise: op %d needs a right operand", (int)op);
  } else if (b->is_scalar) {
    if (op == ACU_BITWISE_AND_NOT) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "bitwise: and_not has no scalar form");
    acu_status st;
    const int64_t snc = acu_resolve_null_count(ctx, b, &st);
    ACU_TRY(st);
    if (snc != 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "bitwise: the scalar operand is a T::Native and cannot be null");
  }
  return acu_with_native(
      dtype, [&](auto t) { return arith_typed<decltype(t)>(ctx, ACU_ADD_WRAPPING, a, b, out, nullptr, (int)op); },
      [&] { return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid bitwise operation: dtype %d", (int)dtype); });
}

extern "C" acu_status acu_cmp(acu_ctx *ctx, acu_dtype dtype, acu_cmp_op op, const acu_array *a,
                              const acu_array *b, acu_array_out *out) {
  ACU_ENTER(ctx);
  if (dtype == ACU_I128) {
    ACU_TRY(i128_aligned(ctx, a->values, b->values));
    return cmp_typed<__int128>(ctx, op, a, b, out);
  }
  return acu_with_native(
      dtype, [&](auto t) { return cmp_typed<decltype(t)>(ctx, op, a, b, out); },
      [&] { return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid comparison operation: dtype %d", (int)dtype); });
}

acu_status acu_cmp_len(acu_ctx *ctx, const acu_array *l, const acu_array *r, int64_t *len) {
  const bool ls = l->is_scalar != 0, rs = r->is_scalar != 0;
  if (l->len != r->len && !ls && !rs)  // cmp.rs:228-232
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0,
                    "Cannot compare arrays of different lengths, got %lld vs %lld", (long long)l->len, (long long)r->len);
  *len = ls ? r->len : l->len;
  return ACU_OK;
}

acu_status acu_cmp_decide(acu_ctx *ctx, acu_cmp_op op, const acu_array *l, const acu_array *r, acu_array_out *out,
                          acu_cmp_decision *d) {
  *d = acu_cmp_decision{};
  ACU_TRY(acu_cmp_len(ctx, l, r, &d->len));
  out->len = d->len;
  out->has_validity = 0;
  out->null_count = 0;
  if (d->len == 0) return ACU_OK;
  acu_status st;
  const int64_t lnc = acu_resolve_null_count(ctx, l, &st);
  ACU_TRY(st);
  const int64_t rnc = acu_resolve_null_count(ctx, r, &st);
  ACU_TRY(st);
  const bool ls = l->is_scalar != 0, rs = r->is_scalar != 0;
  const bool ln = lnc > 0, rn = rnc > 0;  // logical_nulls().filter(null_count > 0)
  const bool fold = op == ACU_DISTINCT || op == ACU_NOT_DISTINCT;
  d->all_null = !fold && ((ls && ln) || (rs && rn)) && !(ls && rs);
  if (d->all_null) return ACU_OK;
  d->swap = op == ACU_GT || op == ACU_LT_EQ;
  const acu_array *x = d->swap ? r : l, *y = d->swap ? l : r;
  const bool xs = d->swap ? rs : ls, ys = d->swap ? ls : rs;
  const bool xn = d->swap ? rn : ln, yn = d->swap ? ln : rn;
  d->lt = !(op == ACU_EQ || op == ACU_NEQ || fold);
  d->neg = op == ACU_NEQ || op == ACU_DISTINCT || op == ACU_LT_EQ || op == ACU_GT_EQ;
  d->fold = op == ACU_DISTINCT ? FOLD_DISTINCT : op == ACU_NOT_DISTINCT ? FOLD_NOT_DISTINCT : FOLD_NONE;
  d->a_scalar = xs && !ys;
  d->b_scalar = ys && !xs;
  if (xn) { if (d->a_scalar) d->a_null_scalar = 1; else { d->av = x->validity; d->aoff = x->validity_offset; } }
  if (yn) { if (d->b_scalar) d->b_null_scalar = 1; else { d->bv = y->validity; d->boff = y->validity_offset; } }
  d->has_validity = !fold && (xn || yn);
  return ACU_OK;
}

void acu_cmp_finalize(const acu_cmp_decision &d, const unsigned long long *hres, acu_array_out *out) {
  if (!d.has_validity) return;
  out->has_validity = 1;
  out->null_count = d.len - (int64_t)hres[RES_COUNT];
}

acu_status acu_new_null(acu_ctx *ctx, int64_t len, size_t value_bytes, acu_array_out *out) {
  if (value_bytes) ACU_CUDA(ctx, cudaMemsetAsync(out->values, 0, value_bytes, ctx->stream));
  if (len) ACU_CUDA(ctx, cudaMemsetAsync(out->validity, 0, acu_bitmap_bytes(len), ctx->stream));
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  out->len = len;
  out->has_validity = 1;
  out->null_count = len;
  return ACU_OK;
}

// The comparison of acu_cmp written straight into a filter plan's mask / tile counts (compact.cu: acu_filter_plan_create_cmp).
// Stream-ordered, no synchronisation.
acu_status acu_cmp_into_plan(acu_ctx *ctx, acu_dtype dtype, acu_cmp_op op, const acu_array *a, const acu_array *b, uint64_t *mask,
                             int64_t n_words_padded, uint32_t *tile_count, int64_t n_tiles) {
  CmpFuse f{mask, n_words_padded, tile_count, n_tiles};
  const CmpFuse *fuse = &f;
  acu_array_out *out = nullptr;
  if (dtype == ACU_I128) {
    ACU_TRY(i128_aligned(ctx, a->values, b->values));
    return cmp_typed<__int128>(ctx, op, a, b, out, fuse);
  }
  return acu_with_native(
      dtype, [&](auto t) { return cmp_typed<decltype(t)>(ctx, op, a, b, out, fuse); },
      [&] { return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid comparison operation: dtype %d", (int)dtype); });
}

extern "C" acu_status acu_cast_numeric(acu_ctx *ctx, acu_dtype from, acu_dtype to, int32_t safe,
                                       const acu_array *a, acu_array_out *out) {
  ACU_ENTER(ctx);
  // numeric_cast (unary_opt: a value that does not fit O is null) / try_numeric_cast (try_unary: it is an error)
  const DcastCall c{DK_NUM, safe ? DM_OPT : DM_TRY, safe, 0, 0, 0, to, false};
  return acu_with_native(
      from,
      [&](auto i) {
        return acu_with_native(
            to, [&](auto o) { return cast_launch<decltype(i), decltype(o), DK_NUM>(ctx, c, DcastArgs{}, a, out); },
            [&] { return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, -1, 0, 0, 0, "cast to dtype %d", (int)to); });
      },
      [&] { return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, -1, 0, 0, 0, "cast from dtype %d", (int)from); });
}

extern "C" acu_status acu_decimal_arith(acu_ctx *ctx, acu_arith_op op, const acu_decimal_type *lt, const acu_array *a,
                                        const acu_decimal_type *rt, const acu_array *b, acu_decimal_type *out_type,
                                        acu_array_out *out) {
  ACU_ENTER(ctx);
  const int w = lt->byte_width;
  if ((w != 4 && w != 8 && w != 16) || rt->byte_width != w)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid decimal operation: byte widths %d and %d", (int)w, (int)rt->byte_width);
  const int mp = w == 4 ? 9 : w == 8 ? 18 : 38;
  ACU_TRY(decimal_validate(ctx, mp, mp, lt->precision, lt->scale));
  ACU_TRY(decimal_validate(ctx, mp, mp, rt->precision, rt->scale));
  if (w == 4) return decimal_typed<int32_t>(ctx, op, *lt, a, *rt, b, out_type, out);
  if (w == 8) return decimal_typed<int64_t>(ctx, op, *lt, a, *rt, b, out_type, out);
  ACU_TRY(i128_aligned(ctx, a->values, b->values));
  ACU_TRY(i128_aligned(ctx, out->values, nullptr));
  return decimal_typed<__int128>(ctx, op, *lt, a, *rt, b, out_type, out);
}

extern "C" acu_status acu_cast_decimal(acu_ctx *ctx, const acu_decimal_type *from, const acu_decimal_type *to, int32_t safe,
                                       const acu_array *a, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(decimal_type_ok(ctx, from));
  if (to->byte_width != 4 && to->byte_width != 8 && to->byte_width != 16)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid decimal type: byte width %d", (int)to->byte_width);
  if (from->byte_width == 16) ACU_TRY(i128_aligned(ctx, a->values, nullptr));
  if (to->byte_width == 16) ACU_TRY(i128_aligned(ctx, out->values, nullptr));
  if (from->byte_width == 4) return cast_decimal_typed<int32_t>(ctx, *from, *to, safe, a, out);
  if (from->byte_width == 8) return cast_decimal_typed<int64_t>(ctx, *from, *to, safe, a, out);
  return cast_decimal_typed<__int128>(ctx, *from, *to, safe, a, out);
}

extern "C" acu_status acu_cast_to_decimal(acu_ctx *ctx, acu_dtype from, const acu_decimal_type *to, int32_t safe,
                                          const acu_array *a, acu_array_out *out) {
  ACU_ENTER(ctx);
  if (to->byte_width != 4 && to->byte_width != 8 && to->byte_width != 16)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid decimal type: byte width %d", (int)to->byte_width);
  if (to->byte_width == 16) ACU_TRY(i128_aligned(ctx, out->values, nullptr));
  return acu_with_native(
      from,
      [&](auto i) {
        using I = decltype(i);
        if constexpr (is_fp<I>::value) return cast_float_to_decimal<I>(ctx, *to, safe, a, out);
        else return cast_int_to_decimal<I>(ctx, *to, safe, a, out);
      },
      [&] {
        return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, -1, 0, 0, 0, "cast from dtype %d to %s", (int)from, decimal_name(to->byte_width));
      });
}

extern "C" acu_status acu_cast_from_decimal(acu_ctx *ctx, const acu_decimal_type *from, acu_dtype to, int32_t safe,
                                            const acu_array *a, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(decimal_type_ok(ctx, from));
  if (from->byte_width == 4) return cast_from_decimal_to<int32_t>(ctx, *from, to, safe, a, out);
  if (from->byte_width == 8) return cast_from_decimal_to<int64_t>(ctx, *from, to, safe, a, out);
  ACU_TRY(i128_aligned(ctx, a->values, nullptr));
  return cast_from_decimal_to<__int128>(ctx, *from, to, safe, a, out);
}
