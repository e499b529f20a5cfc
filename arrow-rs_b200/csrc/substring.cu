// substring.cu — arrow-string/src/length.rs (length / bit_length) and arrow-string/src/substring.rs (substring,
// substring_by_char) over GenericByteArray (Utf8, Binary: i32 offsets; LargeUtf8, LargeBinary: i64), GenericByteViewArray
// (Utf8View, BinaryView) and FixedSizeBinary.
//
//   length / bit_length: one streaming kernel per layout; the input's NullBuffer is cloned (normalised to bit offset 0).
//   substring (bytes):   each row's (begin, len) comes from its own two offsets (SubstrRows), the bytes engine
//                        (bytes_engine.cuh) scans the lengths, writes the offsets and copies the ranges.
//   substring_by_char:   k_char_bounds walks each row's UTF-8 once and stores its byte range; rows longer than LONG_ROW
//                        bytes are walked by one warp each (k_char_long); the same engine then copies the ranges (RangeRows).
//   substring (views):   a 16 B -> 16 B map (k_substr_view): results of <= 12 bytes are rebuilt inline, longer ones keep
//                        pointing into the input's data buffers (offset advanced, new prefix); no byte is copied.
//   FixedSizeBinary:     a strided copy (k_fsb_substr).
//
// Errors are found on the device as the lowest failing key (atomicMin); the host recomputes the failing row's offsets
// with the same __host__ __device__ range functions to build the reference's message.
#include <algorithm>
#include <type_traits>

#include "bitmap.cuh"
#include "bytes_cmp.cuh"
#include "bytes_engine.cuh"
#include "internal.cuh"

namespace {

constexpr int64_t LONG_ROW = 512;    // bytes a by_char row may walk before it goes to the warp-per-row kernel
constexpr unsigned long long PANIC_KEY = 1ull << 62;  // byte arrays: every boundary error precedes every slice panic

__host__ __device__ __forceinline__ bool is_cont(uint8_t b) { return (b & 0xC0u) == 0x80u; }

// ---- the reference's range rules ----------------------------------------------------------------------------------
// byte_substring (substring.rs:319-397) in the offset type O, wrapping like a release build.
template <class O>
__host__ __device__ __forceinline__ void byte_range(O p0, O p1, O start, bool has_len, O length, O *s, O *e) {
  using U = typename std::make_unsigned<O>::type;
  if (start > 0) {
    const O x = (O)((U)p0 + (U)start);
    *s = x < p1 ? x : p1;
  } else if (start == 0) {
    *s = p0;
  } else {
    const O x = (O)((U)p1 + (U)start);
    *s = x > p0 ? x : p0;
  }
  if (has_len) {
    const O x = (O)((U)length + (U)*s);
    *e = x < p1 ? x : p1;
  } else {
    *e = p1;
  }
}

// view_substring_range (substring.rs:254-271): offsets relative to the value, in i64 (length as i64).
__host__ __device__ __forceinline__ void view_range(int64_t L, int64_t start, bool has_len, uint64_t length, int64_t *s, int64_t *e) {
  *s = start > 0 ? (start < L ? start : L) : start == 0 ? 0 : (L + start > 0 ? L + start : 0);
  if (has_len) {
    const int64_t l = (int64_t)length;
    const int64_t x = (l > 0 && *s > INT64_MAX - l) ? INT64_MAX : *s + l;  // saturating_add
    *e = x < L ? x : L;
  } else {
    *e = L;
  }
}

// str::is_char_boundary at a usize position of the n bytes at p: reads p[pos] only when pos < n.
__device__ __forceinline__ bool char_boundary(const uint8_t *p, uint64_t pos, uint64_t n) {
  if (pos == 0 || pos == n) return true;
  if (pos > n) return false;
  return !is_cont(__ldg(p + pos));
}

// ---- length / bit_length (length.rs:26-200) -------------------------------------------------------------------------
__device__ __forceinline__ void ld4(const int32_t *p, int32_t o[4]) {
  const int4 q = __ldg(reinterpret_cast<const int4 *>(p));
  o[0] = q.x, o[1] = q.y, o[2] = q.z, o[3] = q.w;
}
__device__ __forceinline__ void ld4(const int64_t *p, int64_t o[4]) {
  const longlong2 a = __ldg(reinterpret_cast<const longlong2 *>(p)), b = __ldg(reinterpret_cast<const longlong2 *>(p) + 1);
  o[0] = a.x, o[1] = a.y, o[2] = b.x, o[3] = b.y;
}
__device__ __forceinline__ void st4(int32_t *p, const int32_t r[4]) { *reinterpret_cast<int4 *>(p) = make_int4(r[0], r[1], r[2], r[3]); }
__device__ __forceinline__ void st4(int64_t *p, const int64_t r[4]) {
  reinterpret_cast<longlong2 *>(p)[0] = make_longlong2(r[0], r[1]);
  reinterpret_cast<longlong2 *>(p)[1] = make_longlong2(r[2], r[3]);
}

// out[i] = (offs[i+1] - offs[i]) << shift, wrapping, at every slot. A thread owns 4 consecutive rows: one vector load of
// offsets [j0, j0+4), one scalar load of offsets[j0+4], one vector store (vec: both pointers 16-byte aligned).
template <class O>
__global__ void __launch_bounds__(256) k_length_bytes(const O *__restrict__ offs, int64_t n, int shift, int vec, O *__restrict__ out) {
  using U = typename std::make_unsigned<O>::type;
  const int64_t groups = (n + 3) >> 2, stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += stride) {
    const int64_t j0 = g << 2;
    O o[5], r[4];
    if (vec && j0 + 4 <= n) {
      ld4(offs + j0, o);
      o[4] = __ldg(offs + j0 + 4);
#pragma unroll
      for (int k = 0; k < 4; ++k) r[k] = (O)(((U)o[k + 1] - (U)o[k]) << shift);
      st4(out + j0, r);
    } else {
      for (int64_t j = j0; j < n && j < j0 + 4; ++j) out[j] = (O)(((U)__ldg(offs + j + 1) - (U)__ldg(offs + j)) << shift);
    }
  }
}

// views: the low 32 bits of every view, null views included (`*view as i32`, then wrapping_mul(8)).
__global__ void __launch_bounds__(256) k_length_view(const uint32_t *__restrict__ words, int64_t n, int shift, int32_t *__restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = (int32_t)(__ldg(words + 4 * i) << shift);
}

__global__ void __launch_bounds__(256) k_fill_i32(int32_t *__restrict__ out, int64_t n, int32_t v) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = v;
}

// ---- substring of a byte array: the producers of bytes_engine.cuh ----------------------------------------------------
// Failure key of row j: 2j (start offset not a char boundary), 2j + 1 (end offset), PANIC_KEY | j (the slice panics).
template <class O, bool UTF8>
struct SubstrRows {
  int ob;
  int64_t m;
  const uint8_t *data;
  int detect_oob;
  const O *offs;
  int64_t data_len;  // the whole value-data buffer: its end is a char boundary and is never read
  O start, length;
  int has_len;
  __device__ __forceinline__ void ranges4(int64_t j0, int64_t begin[4], uint64_t len[4], unsigned long long *err) const {
    O o[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) o[k] = j0 + k <= m ? __ldg(offs + j0 + k) : (O)0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      begin[k] = 0;
      len[k] = 0;
      if (j0 + k >= m) continue;
      O s, e;
      byte_range<O>(o[k], o[k + 1], start, has_len != 0, length, &s, &e);
      const unsigned long long row = (unsigned long long)(j0 + k);
      unsigned long long key = ~0ull;
      // as_usize of a negative offset is huge: never a boundary
      if (UTF8 && start != 0 && !char_boundary(data, (uint64_t)(int64_t)s, (uint64_t)data_len)) key = 2 * row;
      else if (UTF8 && has_len && !char_boundary(data, (uint64_t)(int64_t)e, (uint64_t)data_len)) key = 2 * row + 1;
      else if (s < 0 || e < s) key = PANIC_KEY | row;  // e >= s >= 0 keeps e <= p1 <= data_len
      if (key != ~0ull) {
        if (key < *err) *err = key;
        continue;
      }
      begin[k] = (int64_t)s;
      len[k] = (uint64_t)(int64_t)(e - s);
    }
  }
};

// Precomputed ranges (substring_by_char).
struct RangeRows {
  int ob;
  int64_t m;
  const uint8_t *data;
  int detect_oob;
  const int64_t *rb, *rl;
  __device__ __forceinline__ void ranges4(int64_t j0, int64_t begin[4], uint64_t len[4], unsigned long long *) const {
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const bool in = j0 + k < m;
      begin[k] = in ? __ldg(rb + j0 + k) : 0;
      len[k] = in ? (uint64_t)__ldg(rl + j0 + k) : 0;
    }
  }
};

// ---- substring_by_char: utf8_bounds (substring.rs:219-251) -----------------------------------------------------------
// The position of the k-th (0-based) char start in p[from, to), `to` when there are k or fewer. WARP: the warp walks the
// row 32 bytes at a time (ballot on the non-continuation bytes); otherwise one byte at a time.
template <bool WARP>
__device__ __forceinline__ int64_t nth_fwd(const uint8_t *p, int64_t from, int64_t to, uint64_t k, int lane) {
  constexpr int W = WARP ? 32 : 1;
  for (int64_t base = from; base < to; base += W) {
    const int64_t x = base + (WARP ? lane : 0);
    const bool st = x < to && !is_cont(__ldg(p + x));
    uint32_t b = WARP ? __ballot_sync(ACU_FULL_MASK, st) : (uint32_t)st;
    const uint32_t c = __popc(b);
    if (k < c) {
      for (uint32_t t = 0; t < (uint32_t)k; ++t) b &= b - 1;
      return base + __ffs(b) - 1;
    }
    k -= c;
  }
  return to;
}
// The position of the k-th (0-based) char start of p[0, to) counted from the end, -1 when there are k or fewer.
template <bool WARP>
__device__ __forceinline__ int64_t nth_back(const uint8_t *p, int64_t to, uint64_t k, int lane) {
  constexpr int W = WARP ? 32 : 1;
  for (int64_t base = to - 1; base >= 0; base -= W) {
    const int64_t x = base - (WARP ? lane : 0);
    const bool st = x >= 0 && !is_cont(__ldg(p + x));
    uint32_t b = WARP ? __ballot_sync(ACU_FULL_MASK, st) : (uint32_t)st;
    const uint32_t c = __popc(b);
    if (k < c) {
      for (uint32_t t = 0; t < (uint32_t)k; ++t) b &= b - 1;
      return base - (__ffs(b) - 1);
    }
    k -= c;
  }
  return -1;
}

template <bool WARP>
__device__ __forceinline__ void char_bounds(const uint8_t *p, int64_t L, int64_t start, bool has_len, uint64_t length, int lane,
                                            int64_t *s, int64_t *e) {
  if (start >= 0) {
    *s = nth_fwd<WARP>(p, 0, L, (uint64_t)start, lane);
  } else {
    const uint64_t back = (uint64_t)0 - (uint64_t)start;  // unsigned_abs
    const int64_t x = nth_back<WARP>(p, L, back - 1, lane);
    *s = x < 0 ? 0 : x;
  }
  *e = (!has_len || length >= (uint64_t)(L - *s)) ? L : nth_fwd<WARP>(p, *s, L, length, lane);
}

struct CharParams {
  BytesOperand src;
  const uint8_t *valid;  // NULL = no nulls
  int64_t voff, n;
  int64_t start;
  int has_len;
  uint64_t length;
  int64_t *rb, *rl;       // out: absolute begin and length of every row (null rows: 0, 0)
  int64_t *long_rows;       // room for every row: each long row is queued
  unsigned long long *res;  // RES_AUX0: queued long rows
};

__global__ void __launch_bounds__(256) k_char_bounds(const CharParams p) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += stride) {
    int64_t b = 0, l = 0;
    if (!p.valid || ld_bit(p.valid, p.voff + i)) {  // null slots become empty
      const int64_t p0 = ld_offset(p.src.offs, p.src.ob, i), p1 = ld_offset(p.src.offs, p.src.ob, i + 1);
      const int64_t L = p1 - p0;
      if (L > LONG_ROW) {
        p.long_rows[atomicAdd(p.res + RES_AUX0, 1ull)] = i;
      } else {
        int64_t s, e;
        char_bounds<false>(p.src.data + p0, L, p.start, p.has_len != 0, p.length, 0, &s, &e);
        b = p0 + s, l = e - s;
      }
    }
    p.rb[i] = b;
    p.rl[i] = l;
  }
}

// The queue's length is read on the device, so no host round trip sits between the two kernels.
__global__ void __launch_bounds__(256) k_char_long(const CharParams p) {
  const int64_t count = (int64_t)*(volatile const unsigned long long *)(p.res + RES_AUX0);
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t k = warp; k < count; k += nwarps) {
    const int64_t i = p.long_rows[k];
    const int64_t p0 = ld_offset(p.src.offs, p.src.ob, i), p1 = ld_offset(p.src.offs, p.src.ob, i + 1);
    int64_t s, e;
    char_bounds<true>(p.src.data + p0, p1 - p0, p.start, p.has_len != 0, p.length, lane, &s, &e);
    if (lane == 0) p.rb[i] = p0 + s, p.rl[i] = e - s;
  }
}

// ---- substring of a view array (substring.rs:254-317) -----------------------------------------------------------------
// Failure key of row j: 4j (start offset not a char boundary), 4j + 1 (end offset), 4j + 2 (the slice panics).
struct ViewSubstr {
  ViewOperand src;
  const uint8_t *valid;
  int64_t voff, n;
  int64_t start;
  int has_len;
  uint64_t length;
  uint4 *out;
  unsigned long long *res;  // RES_ERR_INDEX: lowest failure key
};

template <bool UTF8>
__global__ void __launch_bounds__(256) k_substr_view(const ViewSubstr p) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long err = ~0ull;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < p.n; i += stride) {
    uint4 r = make_uint4(0, 0, 0, 0);  // a null slot: append_null's all-zero view
    if (!p.valid || ld_bit(p.valid, p.voff + i)) {
      const uint4 v = p.src.view(i);
      const BytesItem it = p.src.item(v, p.src.views + i);
      const int64_t L = it.len;
      const uint8_t *val = it.p;
      int64_t s, e;
      view_range(L, p.start, p.has_len != 0, p.length, &s, &e);
      unsigned long long key = ~0ull;
      if (UTF8 && !char_boundary(val, (uint64_t)s, (uint64_t)L)) key = 4 * (unsigned long long)i;
      else if (UTF8 && !char_boundary(val, (uint64_t)e, (uint64_t)L)) key = 4 * (unsigned long long)i + 1;
      else if (e < s) key = 4 * (unsigned long long)i + 2;
      if (key != ~0ull) {
        if (key < err) err = key;
      } else {
        const uint32_t nl = (uint32_t)(e - s);
        const uint8_t *q = val + s;
        if (nl <= 12) {
          const uint64_t lo = ld_upto8(q, nl < 8 ? nl : 8), hi = nl > 8 ? ld_upto8(q + 8, nl - 8) : 0ull;
          r = make_uint4(nl, (uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi);
        } else {  // still in the input's buffer: same buffer index, offset advanced, new prefix
          r = make_uint4(nl, (uint32_t)ld_upto8(q, 4), v.z, v.w + (uint32_t)s);
        }
      }
    }
    st_stream16(p.out + i, r);
  }
  if (err != ~0ull) atomicMin(p.res + RES_ERR_INDEX, err);
}

// ---- substring of a FixedSizeBinary array (substring.rs:399-459): every row's [new_start, new_start + new_len) ---------
// One row per thread: 8-byte pieces of the source row (ld_upto8) leave as bytes, since the output rows are new_len apart.
__global__ void __launch_bounds__(256) k_fsb_substr(const uint8_t *__restrict__ in, int64_t w, int64_t new_start, int64_t new_len, int64_t n,
                                                    uint8_t *__restrict__ out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const uint8_t *src = in + i * w + new_start;
    uint8_t *dst = out + i * new_len;
    for (int64_t k = 0; k < new_len; k += 8) {
      const uint32_t nb = (uint32_t)(new_len - k < 8 ? new_len - k : 8);
      const uint64_t v = ld_upto8(src + k, nb);
      for (uint32_t b = 0; b < nb; ++b) dst[k + b] = (uint8_t)(v >> (8 * b));
    }
  }
}

// ---- host side -------------------------------------------------------------------------------------------------------
acu_status check_input(acu_ctx *ctx, const acu_array *nulls, const char *what) {
  if (nulls->is_scalar) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "%s takes an array, not a scalar", what);
  if (nulls->len < 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "%s: negative length", what);
  return ACU_OK;
}

// The input's validity normalised to bit offset 0 into out->validity; its valid count lands in RES_COUNT (block 0).
acu_status copy_validity(acu_ctx *ctx, const acu_array *nulls, acu_array_out *out) {
  if (!nulls->validity || nulls->len == 0) return ACU_OK;
  return acu_bitmap_and_launch(ctx, nulls->validity, nulls->validity_offset, nullptr, 0, nulls->len,
                               reinterpret_cast<uint64_t *>(out->validity), true, ctx->d_res);
}

// NullBuffer::from_unsliced_buffer: the copied bitmap is kept only when it has a null.
void unsliced_nulls(const acu_array *nulls, const unsigned long long *h, acu_array_out *out) {
  out->len = nulls->len;
  out->null_count = nulls->validity && nulls->len ? nulls->len - (int64_t)h[RES_COUNT] : 0;
  out->has_validity = out->null_count > 0;
}

// Rust's panic texts for data[s..e] over a buffer of n bytes.
acu_status slice_panic(acu_ctx *ctx, int64_t row, uint64_t s, uint64_t e, uint64_t n) {
  if (s > e) return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, row, s, e, n, "slice index starts at %llu but ends at %llu",
                             (unsigned long long)s, (unsigned long long)e);
  return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, row, s, e, n, "range end index %llu out of range for slice of length %llu",
                  (unsigned long long)e, (unsigned long long)n);
}
acu_status boundary_error(acu_ctx *ctx, int64_t row, uint64_t off) {
  return acu_fail(ctx, ACU_ERR_COMPUTE, row, off, 0, 0, "The offset %llu is at an invalid utf-8 boundary.", (unsigned long long)off);
}

template <class O>
acu_status substring_bytes_run(acu_ctx *ctx, int32_t is_utf8, int64_t start, bool has_len, uint64_t length, const acu_bytes_array *a,
                               int64_t data_len, void *out_offsets, uint8_t *out_data, int64_t out_cap, int64_t *out_data_len,
                               acu_array_out *out_nulls) {
  const int64_t n = a->nulls.len;
  const O st = (O)start, ln = (O)length;  // `start as i32`, `length as i32` for i32 offsets
  ACU_TRY(copy_validity(ctx, &a->nulls, out_nulls));
  if (n > 0) {
    void *scratch;
    ACU_TRY(acu_scratch(ctx, engine_scratch(n), &scratch));
    const O *offs = static_cast<const O *>(a->offsets);
    if (is_utf8) {
      SubstrRows<O, true> r{(int)sizeof(O), n, a->data, 0, offs, data_len, st, ln, has_len};
      ACU_TRY(engine_launch(ctx, r, static_cast<int64_t *>(scratch), out_offsets, out_data, out_cap, INT64_MAX));
    } else {
      SubstrRows<O, false> r{(int)sizeof(O), n, a->data, 0, offs, data_len, st, ln, has_len};
      ACU_TRY(engine_launch(ctx, r, static_cast<int64_t *>(scratch), out_offsets, out_data, out_cap, INT64_MAX));
    }
  } else {
    ACU_CUDA(ctx, cudaMemsetAsync(out_offsets, 0, sizeof(O), ctx->stream));
  }
  ACU_TRY(acu_res_fetch(ctx));
  const unsigned long long *h = ctx->h_res;
  *out_data_len = 0;
  unsliced_nulls(&a->nulls, h, out_nulls);
  if (n == 0) return ACU_OK;
  const unsigned long long key = h[RES_ERR_INDEX];
  if (key != ~0ull) {  // the failing row's offsets, recomputed as the kernel did
    const int64_t row = (int64_t)(key >= PANIC_KEY ? key - PANIC_KEY : key / 2);
    O o[2];
    ACU_TRY(acu_memcpy_d2h(ctx, o, static_cast<const O *>(a->offsets) + row, sizeof o));
    O s, e;
    byte_range<O>(o[0], o[1], st, has_len, ln, &s, &e);
    const uint64_t us = (uint64_t)(int64_t)s, ue = (uint64_t)(int64_t)e;  // as_usize
    if (key >= PANIC_KEY) return slice_panic(ctx, row, us, ue, (uint64_t)data_len);
    return boundary_error(ctx, row, key % 2 ? ue : us);
  }
  return finish_bytes(ctx, out_data, out_cap, out_data_len);
}

acu_status substring_by_char_run(acu_ctx *ctx, int32_t ob, int64_t start, bool has_len, uint64_t length, const acu_bytes_array *a,
                                 void *out_offsets, uint8_t *out_data, int64_t out_cap, int64_t *out_data_len, acu_array_out *out_nulls) {
  const int64_t n = a->nulls.len;
  if (n > 0) {
    void *scratch;
    const size_t eng = engine_scratch(n), ranges = align256((size_t)n * 8);
    ACU_TRY(acu_scratch(ctx, eng + 2 * ranges + ranges, &scratch));
    uint8_t *base = static_cast<uint8_t *>(scratch);
    CharParams p{BytesOperand{a->offsets, a->data, ob}, a->nulls.validity, a->nulls.validity_offset, n, start, has_len, length,
                 reinterpret_cast<int64_t *>(base + eng), reinterpret_cast<int64_t *>(base + eng + ranges),
                 reinterpret_cast<int64_t *>(base + eng + 2 * ranges), ctx->d_res};
    ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_char_bounds, acu_grid(ctx, (n + 255) / 256, 8), 256, 0, p);
    ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_char_long, acu_grid(ctx, (n + 7) / 8, 16), 256, 0, p);  // one warp per queued row
    RangeRows r{ob, n, a->data, 0, p.rb, p.rl};
    ACU_TRY(engine_launch(ctx, r, reinterpret_cast<int64_t *>(base), out_offsets, out_data, out_cap, INT64_MAX));
  } else {
    ACU_CUDA(ctx, cudaMemsetAsync(out_offsets, 0, (size_t)ob, ctx->stream));
  }
  ACU_TRY(copy_validity(ctx, &a->nulls, out_nulls));
  ACU_TRY(acu_res_fetch(ctx));
  *out_data_len = 0;
  unsliced_nulls(&a->nulls, ctx->h_res, out_nulls);
  if (n == 0) return ACU_OK;
  return finish_bytes(ctx, out_data, out_cap, out_data_len);
}

}  // namespace

// Every entry point starts with acu_res_reset, whose acu_sync_only refuses inside a stream-ordered section before any
// argument check.
extern "C" acu_status acu_length_bytes(acu_ctx *ctx, int32_t offset_bytes, acu_length_op op, const acu_bytes_array *a, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(acu_offset_width_check(ctx, offset_bytes));
  if (op != ACU_LENGTH && op != ACU_BIT_LENGTH) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "invalid length op %d", (int)op);
  ACU_TRY(check_input(ctx, &a->nulls, "length"));
  const int64_t n = a->nulls.len;
  const int shift = op == ACU_BIT_LENGTH ? 3 : 0;
  const int vec = ((uintptr_t)a->offsets % 16 == 0) && ((uintptr_t)out->values % 16 == 0);
  if (n > 0) {
    const int grid = acu_grid(ctx, ((n + 3) / 4 + 255) / 256, 8);
    if (offset_bytes == 4)
      ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_length_bytes<int32_t>, grid, 256, 0, static_cast<const int32_t *>(a->offsets), n, shift, vec,
                       static_cast<int32_t *>(out->values));
    else
      ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_length_bytes<int64_t>, grid, 256, 0, static_cast<const int64_t *>(a->offsets), n, shift, vec,
                       static_cast<int64_t *>(out->values));
  }
  ACU_TRY(copy_validity(ctx, &a->nulls, out));
  ACU_TRY(acu_res_fetch(ctx));
  out->len = n;
  out->has_validity = a->nulls.validity != nullptr;  // nulls.cloned()
  out->null_count = out->has_validity && n ? n - (int64_t)ctx->h_res[RES_COUNT] : 0;
  return ACU_OK;
}

extern "C" acu_status acu_length_byte_view(acu_ctx *ctx, acu_length_op op, const acu_view_array *a, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  if (op != ACU_LENGTH && op != ACU_BIT_LENGTH) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "invalid length op %d", (int)op);
  ACU_TRY(check_input(ctx, &a->nulls, "length"));
  const int64_t n = a->nulls.len;
  if (n > 0)
    ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_length_view, acu_grid(ctx, (n + 255) / 256, 8), 256, 0, static_cast<const uint32_t *>(a->views), n,
                     op == ACU_BIT_LENGTH ? 3 : 0, static_cast<int32_t *>(out->values));
  ACU_TRY(copy_validity(ctx, &a->nulls, out));
  ACU_TRY(acu_res_fetch(ctx));
  out->len = n;
  out->has_validity = a->nulls.validity != nullptr;
  out->null_count = out->has_validity && n ? n - (int64_t)ctx->h_res[RES_COUNT] : 0;
  return ACU_OK;
}

extern "C" acu_status acu_length_fixed_size_binary(acu_ctx *ctx, int32_t byte_width, acu_length_op op, const acu_array *a, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  if (op != ACU_LENGTH && op != ACU_BIT_LENGTH) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "invalid length op %d", (int)op);
  if (byte_width < 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "negative FixedSizeBinary value length");
  ACU_TRY(check_input(ctx, a, "length"));
  const int64_t n = a->len;
  const int32_t v = (int32_t)((uint32_t)byte_width << (op == ACU_BIT_LENGTH ? 3 : 0));  // `len * 8`, wrapping
  if (n > 0) ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_fill_i32, acu_grid(ctx, (n + 255) / 256, 8), 256, 0, static_cast<int32_t *>(out->values), n, v);
  ACU_TRY(copy_validity(ctx, a, out));
  ACU_TRY(acu_res_fetch(ctx));
  out->len = n;
  out->has_validity = a->validity != nullptr;
  out->null_count = out->has_validity && n ? n - (int64_t)ctx->h_res[RES_COUNT] : 0;
  return ACU_OK;
}

extern "C" acu_status acu_substring_bytes(acu_ctx *ctx, int32_t offset_bytes, int32_t is_utf8, int64_t start, int32_t has_length,
                                          uint64_t length, const acu_bytes_array *a, int64_t data_len, void *out_offsets, uint8_t *out_data,
                                          int64_t out_data_capacity, int64_t *out_data_len, acu_array_out *out_nulls) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(acu_offset_width_check(ctx, offset_bytes));
  ACU_TRY(check_input(ctx, &a->nulls, "substring"));
  if (data_len < 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "substring: negative data length");
  if (offset_bytes == 4)
    return substring_bytes_run<int32_t>(ctx, is_utf8, start, has_length != 0, length, a, data_len, out_offsets, out_data, out_data_capacity,
                                        out_data_len, out_nulls);
  return substring_bytes_run<int64_t>(ctx, is_utf8, start, has_length != 0, length, a, data_len, out_offsets, out_data, out_data_capacity,
                                      out_data_len, out_nulls);
}

extern "C" acu_status acu_substring_by_char(acu_ctx *ctx, int32_t offset_bytes, int64_t start, int32_t has_length, uint64_t length,
                                            const acu_bytes_array *a, void *out_offsets, uint8_t *out_data, int64_t out_data_capacity,
                                            int64_t *out_data_len, acu_array_out *out_nulls) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(acu_offset_width_check(ctx, offset_bytes));
  ACU_TRY(check_input(ctx, &a->nulls, "substring_by_char"));
  return substring_by_char_run(ctx, offset_bytes, start, has_length != 0, length, a, out_offsets, out_data, out_data_capacity, out_data_len,
                               out_nulls);
}

extern "C" acu_status acu_substring_byte_view(acu_ctx *ctx, int32_t is_utf8, int64_t start, int32_t has_length, uint64_t length,
                                              const acu_view_array *a, void *out_views, acu_array_out *out_nulls) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(check_input(ctx, &a->nulls, "substring"));
  const int64_t n = a->nulls.len;
  if (n > 0) {
    void *scratch;
    ACU_TRY(acu_scratch(ctx, acu_view_table_bytes(a), &scratch));
    ViewSubstr p{{}, a->nulls.validity, a->nulls.validity_offset, n, start, has_length, length, static_cast<uint4 *>(out_views), ctx->d_res};
    ACU_TRY(acu_view_operand(ctx, a, scratch, &p.src));
    const int grid = acu_grid(ctx, (n + 255) / 256, 8);
    if (is_utf8) ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_substr_view<true>, grid, 256, 0, p);
    else ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_substr_view<false>, grid, 256, 0, p);
  }
  ACU_TRY(copy_validity(ctx, &a->nulls, out_nulls));
  ACU_TRY(acu_res_fetch(ctx));
  unsliced_nulls(&a->nulls, ctx->h_res, out_nulls);  // the builder's NullBuffer: None without nulls
  const unsigned long long key = ctx->h_res[RES_ERR_INDEX];
  if (n == 0 || key == ~0ull) return ACU_OK;
  const int64_t row = (int64_t)(key / 4);
  uint32_t v[4];
  ACU_TRY(acu_memcpy_d2h(ctx, v, static_cast<const uint4 *>(a->views) + row, sizeof v));
  int64_t s, e;
  view_range(v[0], start, has_length != 0, length, &s, &e);
  if (key % 4 == 2) return slice_panic(ctx, row, (uint64_t)s, (uint64_t)e, v[0]);
  return boundary_error(ctx, row, key % 4 ? (uint64_t)e : (uint64_t)s);  // relative to the value
}

extern "C" acu_status acu_substring_fixed_size_binary(acu_ctx *ctx, int32_t byte_width, int64_t start, int32_t has_length, uint64_t length,
                                                      const acu_array *a, int32_t *out_byte_width, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  if (byte_width < 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "negative FixedSizeBinary value length");
  ACU_TRY(check_input(ctx, a, "substring"));
  const int64_t n = a->len, w = byte_width;
  const uint64_t back = (uint64_t)0 - (uint64_t)start;
  const int64_t new_start = start > 0 ? std::min<int64_t>(start, w) : start == 0 ? 0 : (back >= (uint64_t)w ? 0 : w - (int64_t)back);
  const int64_t new_len = has_length ? (int64_t)std::min<uint64_t>(length, (uint64_t)(w - new_start)) : w - new_start;
  *out_byte_width = (int32_t)new_len;
  if (n > 0 && new_len > 0)
    ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_fsb_substr, acu_grid(ctx, (n + 255) / 256, 8), 256, 0, static_cast<const uint8_t *>(a->values), w,
                     new_start, new_len, n, static_cast<uint8_t *>(out->values));
  ACU_TRY(copy_validity(ctx, a, out));
  ACU_TRY(acu_res_fetch(ctx));
  unsliced_nulls(a, ctx->h_res, out);
  if (new_len == 0 && !out->has_validity) {  // substring.rs:444-450: an all-valid NullBuffer keeps the length
    out->has_validity = 1;
    out->null_count = 0;
    if (n > 0) {
      ACU_CUDA(ctx, cudaMemsetAsync(out->validity, 0xff, acu_bitmap_bytes(n), ctx->stream));
      ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    }
  }
  return ACU_OK;
}
