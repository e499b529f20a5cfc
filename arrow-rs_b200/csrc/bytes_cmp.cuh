// bytes_cmp.cuh — the one operand path of variable-width columns on the device: BytesOperand (Utf8 / Binary, i32 or i64
// offsets) and ViewOperand (Utf8View / BinaryView) and their row reads, and the helpers that order and match the values.
// Shared by the comparison kernels (strcmp.cu), the min / max reductions (aggregate_bytes.cu), the LIKE family (like.cu),
// length / substring (substring.cu), the run merge of a RunEndEncoded take (run_end.cu) and the gathers (bytes.cu,
// ld_offset only). The host builds the operands through
// internal.cuh's front end (acu_offset_width_check, acu_view_operand), after acu_sync_only.
//
// Order: Rust's `Ord` for `&[u8]` (lexicographic on unsigned bytes, a proper prefix sorts first); `&str` orders the same.
#pragma once
#include "common.cuh"

__device__ __forceinline__ int64_t ld_offset(const void *offs, int ob, int64_t i) {
  return ob == 4 ? (int64_t)__ldg(static_cast<const int32_t *>(offs) + i) : __ldg(static_cast<const int64_t *>(offs) + i);
}

// One value: its bytes and length; pre = a view's 4-byte prefix word (0 for byte arrays)
struct BytesItem {
  const uint8_t *p;
  int64_t len;
  uint32_t pre;
};

struct BytesOperand {
  const void *offs;
  const uint8_t *data;
  int ob;
  __device__ __forceinline__ BytesItem item(int64_t i) const {
    const int64_t b = ld_offset(offs, ob, i), e = ld_offset(offs, ob, i + 1);
    return BytesItem{data + b, e - b, 0u};
  }
};

// views (arrow-data/src/byte_view.rs): x = length, y = prefix / inline[0..4), z, w = inline[4..12) or (buffer index, offset)
struct ViewOperand {
  const uint4 *views;
  const uint8_t *const *buffers;  // device array of device pointers
  int n_buffers;
  __device__ __forceinline__ uint4 view(int64_t i) const { return ld_stream16(views + i); }
  // the value of view v held at `slot`: inline values are read from the slot itself, not from a data buffer
  __device__ __forceinline__ BytesItem item(const uint4 &v, const uint4 *slot) const {
    return BytesItem{v.x <= 12u ? reinterpret_cast<const uint8_t *>(slot) + 4 : buffers[v.z] + v.w, (int64_t)v.x, v.y};
  }
  __device__ __forceinline__ BytesItem item(int64_t i) const { return item(view(i), views + i); }
};

// Up to 8 bytes of p[0 .. nb) as a little-endian u64, zero above nb: aligned 8-byte loads that contain a requested byte.
__device__ __forceinline__ uint64_t ld_upto8(const uint8_t *__restrict__ p, uint32_t nb) {
  const uintptr_t addr = (uintptr_t)p;
  const uint64_t *q = reinterpret_cast<const uint64_t *>(addr & ~(uintptr_t)7);
  const uint32_t sh = (uint32_t)(addr & 7u) * 8u;
  uint64_t lo = 0, hi = 0;
  if (nb) lo = __ldg(q);
  if (sh + nb * 8u > 64u) hi = __ldg(q + 1);
  const uint64_t w = (lo >> sh) | ((hi << 1) << (63u - sh));
  return w & (nb >= 8u ? ~0ull : ((1ull << (nb * 8u)) - 1ull));
}

__device__ __forceinline__ uint64_t bswap64(uint64_t x) {
  const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
  return ((uint64_t)__byte_perm(lo, 0, 0x0123) << 32) | (uint64_t)__byte_perm(hi, 0, 0x0123);
}

// u8::to_ascii_lowercase on each of 8 bytes: 'A'..='Z' gain 0x20, every other byte (non-ASCII included) stays
__device__ __forceinline__ uint64_t ascii_lower8(uint64_t x) {
  const uint64_t h = x & 0x7f7f7f7f7f7f7f7full;
  const uint64_t ge_a = h + 0x3f3f3f3f3f3f3f3full;  // bit 7 set where h >= 'A'
  const uint64_t gt_z = h + 0x2525252525252525ull;  // bit 7 set where h > 'Z'
  return x | (((ge_a & ~gt_z & ~x) & 0x8080808080808080ull) >> 2);
}

// n bytes of a and b equal; ICASE: u8::eq_ignore_ascii_case per byte
template <bool ICASE>
__device__ __forceinline__ bool bytes_range_eq(const uint8_t *a, const uint8_t *b, int64_t n) {
  for (int64_t k = 0; k < n; k += 8) {
    const uint32_t nb = (uint32_t)((n - k) < 8 ? (n - k) : 8);
    uint64_t x = ld_upto8(a + k, nb), y = ld_upto8(b + k, nb);
    if (ICASE) x = ascii_lower8(x), y = ascii_lower8(y);
    if (x != y) return false;
  }
  return true;
}

// `&[u8]` equality / ordering of Rust (lexicographic on unsigned bytes, then length)
__device__ __forceinline__ bool bytes_eq(const uint8_t *a, int64_t la, const uint8_t *b, int64_t lb) {
  return la == lb && bytes_range_eq<false>(a, b, la);
}
// view equality (cmp.rs:810-862): the 16 view bytes when no value lives in a data buffer, else length and prefix first
__device__ __forceinline__ bool view_bits_eq(const uint4 &a, const uint4 &b) { return a.x == b.x && a.y == b.y && a.z == b.z && a.w == b.w; }
__device__ __forceinline__ bool view_is_eq(const ViewOperand &L, const uint4 &l, const uint4 *lslot, const ViewOperand &R, const uint4 &r,
                                           const uint4 *rslot) {
  if (L.n_buffers == 0 && R.n_buffers == 0) return view_bits_eq(l, r);
  if (view_bits_eq(l, r) && l.x <= 12u) return true;
  if (l.x != r.x) return false;
  if (l.x == 0u) return true;
  if (l.y != r.y) return false;
  if (l.x <= 12u) return false;
  const BytesItem a = L.item(l, lslot), b = R.item(r, rslot);
  return bytes_eq(a.p, a.len, b.p, b.len);
}
__device__ __forceinline__ bool bytes_lt(const uint8_t *a, int64_t la, const uint8_t *b, int64_t lb) {
  const int64_t n = la < lb ? la : lb;
  for (int64_t k = 0; k < n; k += 8) {
    const uint32_t nb = (uint32_t)((n - k) < 8 ? (n - k) : 8);
    const uint64_t x = ld_upto8(a + k, nb), y = ld_upto8(b + k, nb);
    if (x != y) return bswap64(x) < bswap64(y);  // first differing byte decides
  }
  return la < lb;
}

// GenericByteViewArray::inline_key_fast (byte_view_array.rs:872-874): (raw.swap_bytes() << 32) | len, compared as u128
__device__ __forceinline__ bool inline_key_lt(const uint4 &a, const uint4 &b) {
  // the key's 128 bits, most significant first: inline bytes 0..11 in order (big endian), then the length
  const uint32_t ak[4] = {__byte_perm(a.y, 0, 0x0123), __byte_perm(a.z, 0, 0x0123), __byte_perm(a.w, 0, 0x0123), a.x};
  const uint32_t bk[4] = {__byte_perm(b.y, 0, 0x0123), __byte_perm(b.z, 0, 0x0123), __byte_perm(b.w, 0, 0x0123), b.x};
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (ak[k] != bk[k]) return ak[k] < bk[k];
  return false;
}
