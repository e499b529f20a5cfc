// zip.cu — zip(mask, truthy, falsy) (arrow-select/src/zip.rs) of Utf8 / Binary (i32 offsets), LargeUtf8 / LargeBinary (i64),
// Utf8View / BinaryView, Boolean and FixedSizeBinary(W) columns. acu_zip (select.cu) keeps the fixed-width primitives.
//
// The reference takes one of three paths, and so does every call here:
//   zip_impl (zip.rs:148-210)        at least one side an array, and Boolean / FixedSizeBinary with two scalars
//                                    (FallbackImpl, zip.rs:318-336): MutableArrayData copies row i of the chosen side,
//                                    bytes and bits under nulls included (a null scalar's own bytes too); a NullBuffer is
//                                    built iff some input has a null and dropped again when the result has none.
//   BytesScalarImpl (zip.rs:439-660) two Utf8 / Binary scalars: no NullBuffer when both are valid; with one null scalar an
//                                    unselected row is empty and the NullBuffer is the predicate (or its negation).
//   ByteViewScalarImpl (:673-860)    two view scalars: one view repeated, with the buffer lists decided on the host.
// A mask null counts as false (maybe_prep_null_mask_filter, zip.rs:662-671) everywhere.
//
// Kernels:
//   bytes    ZipRows, a producer for bytes_engine.cuh: row j's one segment is the chosen side's range (or the scalar's, or
//            nothing). The engine's two passes size, scan, write the offsets and copy; its `limit` finds the first row whose
//            end passes i32::MAX. The validity is k_zip_bits without values.
//   views    k_zip_views: one 16-byte select per row. A falsy array view longer than 12 bytes gets its buffer index raised
//            by truthy's buffer count (wrapping u32), nulls included (transform/mod.rs:222-239, :721-735). Data buffers are
//            never read.
//   Boolean  k_zip_bits: one thread per 64-row output word, (sel & t) | (~sel & f); a scalar side is a broadcast word.
//   FixedSizeBinary  k_zip_fsb: positional, so a thread owns 16-byte output chunks aligned to the output address; the byte
//            select mask comes from the rows the chunk touches (first row by a multiply-high division by W). A scalar side
//            is read from a staged copy of its W bytes followed by its first 16 bytes again, at phase pos mod W.
// Every kernel computes the output validity as k_zip does: ((sel & t_valid) | (~sel & f_valid)), each 64-row word written
// by the thread that owns its first row, valid rows counted into RES_COUNT.
#include "bytes_engine.cuh"

#define ZIP_THREADS 256  // k_zip_bits / k_zip_views / k_zip_fsb: 256-thread blocks
#define ZIP_PER_SM 16    // grid = acu_grid(ctx, blocks, ZIP_PER_SM), grid-stride
#define ZIP_FSB_CHUNKS 2 // k_zip_fsb: 16-byte chunks per thread and round

namespace {

enum { ZIP_BUFFERS_NONE = 0, ZIP_BUFFERS_TRUTHY = 1, ZIP_BUFFERS_FALSY = 2, ZIP_BUFFERS_BOTH = 3 };

// The mask and the validity of the two sides, shared by every kernel.
struct ZipSel {
  const uint8_t *mv;  // mask values
  int64_t moff;
  const uint8_t *mn;  // mask validity when it holds a null, else NULL
  int64_t mnoff;
  const uint8_t *tn, *fn;  // validity of an array side with nulls, else NULL (then t_all / f_all)
  int64_t tnoff, fnoff;
  int t_all, f_all;        // validity of a side without a bitmap: all valid (1) / all null (0)
  int64_t len;
  uint64_t *out_valid;     // NULL: no validity produced
  unsigned long long *res;
  __device__ __forceinline__ uint64_t sel(int64_t pos) const {
    uint64_t s = ld_bits64(mv, moff + pos, moff + len);
    if (mn) s &= ld_bits64(mn, mnoff + pos, mnoff + len);
    return s;
  }
  // the validity word of rows pos .. pos + 63 (pos a multiple of 64) given their selection bits; returns its popcount
  __device__ __forceinline__ unsigned put_valid(int64_t pos, uint64_t s) const {
    const int64_t left = len - pos;
    const uint64_t lenmask = left >= 64 ? ~0ull : ((1ull << left) - 1ull);
    const uint64_t tw = tn ? ld_bits64(tn, tnoff + pos, tnoff + len) : (t_all ? ~0ull : 0ull);
    const uint64_t fw = fn ? ld_bits64(fn, fnoff + pos, fnoff + len) : (f_all ? ~0ull : 0ull);
    const uint64_t v = ((s & tw) | (~s & fw)) & lenmask;
    out_valid[pos >> 6] = v;
    return (unsigned)__popcll(v);
  }
};

__device__ __forceinline__ void count_valid(const ZipSel &z, unsigned cnt) {
  cnt = warp_sum(cnt);
  if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(z.res + RES_COUNT, (unsigned long long)cnt);
}

// ---- Boolean (and the validity of the byte zips) -------------------------------------------------------------------
struct BitSide {
  const uint8_t *v;  // array side's value bits, NULL for a scalar
  int64_t off;
  uint64_t word;     // scalar: its value bit broadcast
};

// out == NULL: the validity alone.
__global__ void __launch_bounds__(ZIP_THREADS) k_zip_bits(const ZipSel z, const BitSide t, const BitSide f, uint64_t *out) {
  const int64_t words = (z.len + 63) >> 6;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned cnt = 0;
  for (int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; w < words; w += stride) {
    const int64_t pos = w << 6;
    const uint64_t s = z.sel(pos);
    if (out) {
      const int64_t left = z.len - pos;
      const uint64_t lenmask = left >= 64 ? ~0ull : ((1ull << left) - 1ull);
      const uint64_t tw = t.v ? ld_bits64(t.v, t.off + pos, t.off + z.len) : t.word;
      const uint64_t fw = f.v ? ld_bits64(f.v, f.off + pos, f.off + z.len) : f.word;
      out[w] = ((s & tw) | (~s & fw)) & lenmask;
    }
    if (z.out_valid) cnt += z.put_valid(pos, s);
  }
  if (z.out_valid) count_valid(z, cnt);
}

// ---- Utf8 / Binary: the bytes engine's producer --------------------------------------------------------------------
// An array side reads its offsets (logical row 0 on); a scalar side is one fixed range (length 0 for an empty row).
template <class O>
struct ZipRows {
  int ob;
  int64_t m;
  int detect_oob;
  const uint8_t *mv;
  int64_t moff;
  const uint8_t *mn;
  int64_t mnoff;
  const O *t_offs, *f_offs;   // NULL: scalar side
  const uint8_t *t_data, *f_data;
  const uint8_t *ts, *fs;     // scalar sides: the value's first byte
  uint64_t ts_len, fs_len;
  __device__ __forceinline__ int nsegs() const { return 1; }
  __device__ __forceinline__ uint32_t sel4(int64_t j0) const {
    uint64_t s = ld_bits64(mv, moff + j0, moff + m);
    if (mn) s &= ld_bits64(mn, mnoff + j0, mnoff + m);
    return (uint32_t)s & 15u;
  }
  __device__ __forceinline__ void ranges4(int64_t j0, int64_t begin[4], uint64_t len[4], unsigned long long *) const {
    const uint32_t s = sel4(j0);
    O to[5], fo[5];
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      to[k] = t_offs && j0 + k <= m ? __ldg(t_offs + j0 + k) : (O)0;
      fo[k] = f_offs && j0 + k <= m ? __ldg(f_offs + j0 + k) : (O)0;
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      begin[k] = 0;
      const uint64_t tl = t_offs ? (uint64_t)(int64_t)(to[k + 1] - to[k]) : ts_len;
      const uint64_t fl = f_offs ? (uint64_t)(int64_t)(fo[k + 1] - fo[k]) : fs_len;
      len[k] = j0 + k < m ? ((s >> k) & 1u ? tl : fl) : 0;
    }
  }
  __device__ __forceinline__ void segment(int64_t row, int, const uint8_t **p, uint64_t *len) const {
    uint64_t s = ld_bits64(mv, moff + row, moff + m) & 1ull;
    if (mn) s &= ld_bits64(mn, mnoff + row, mnoff + m);
    if (s & 1ull) {
      if (t_offs) { const O b = __ldg(t_offs + row), e = __ldg(t_offs + row + 1); *p = t_data + b; *len = (uint64_t)(int64_t)(e - b); }
      else { *p = ts; *len = ts_len; }
    } else {
      if (f_offs) { const O b = __ldg(f_offs + row), e = __ldg(f_offs + row + 1); *p = f_data + b; *len = (uint64_t)(int64_t)(e - b); }
      else { *p = fs; *len = fs_len; }
    }
  }
};

// ---- views ---------------------------------------------------------------------------------------------------------
struct ViewSide {
  const uint4 *v;  // array side, NULL for a scalar
  uint4 s;         // scalar side's view (already re-based by the host)
  uint32_t fix;    // added to the buffer index of an array view longer than 12 bytes
};

__global__ void __launch_bounds__(ZIP_THREADS) k_zip_views(const ZipSel z, const ViewSide t, const ViewSide f, uint4 *out) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned cnt = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < z.len; i += stride) {
    const int64_t wpos = i & ~(int64_t)63;
    const uint64_t s = z.sel(wpos);
    const bool pick_t = (s >> (i & 63)) & 1ull;
    const uint4 *src = pick_t ? t.v : f.v;
    uint4 v = pick_t ? t.s : f.s;
    if (src) {
      v = ld_stream16(src + i);
      if (v.x > 12u) v.z += pick_t ? t.fix : f.fix;
    }
    st_stream16(out + i, v);
    if (z.out_valid && (i & 63) == 0) cnt += z.put_valid(wpos, s);
  }
  if (z.out_valid) count_valid(z, cnt);
}

// ---- FixedSizeBinary ------------------------------------------------------------------------------------------------
struct FsbSide {
  const uint8_t *p;  // array side at logical row 0, or the scalar's staged pattern (W bytes, then its first 16 again)
  int scalar;
};

struct ZipFsbArgs {
  uint64_t w;        // >= 1
  DivW div;          // p / w
  uint8_t *out;      // any alignment
};

// bytes [b0, b1) of a 16-byte chunk (0 <= b0 <= b1 <= 16) as a 128-bit mask
__device__ __forceinline__ unsigned __int128 byte_range_mask(uint32_t b0, uint32_t b1) {
  const unsigned __int128 ones = ~(unsigned __int128)0;
  const unsigned __int128 hi = b1 >= 16u ? ones : ((((unsigned __int128)1) << (8u * b1)) - 1u);
  const unsigned __int128 lo = b0 >= 16u ? ones : ((((unsigned __int128)1) << (8u * b0)) - 1u);
  return hi & ~lo;
}

// The nb bytes of one side at output positions p .. p + nb (row p / W, phase p mod W for a scalar).
__device__ __forceinline__ unsigned __int128 side_bytes(const FsbSide &s, uint64_t p, uint64_t phase, uint32_t nb) {
  uint64_t x0, x1;
  load_upto16(s.p, (int64_t)(s.scalar ? phase : p), nb, &x0, &x1);
  return ((unsigned __int128)x1 << 64) | x0;
}

// MAXR: rows one 16-byte chunk can touch (15 / W + 2).
template <int MAXR>
__global__ void __launch_bounds__(ZIP_THREADS) k_zip_fsb(const ZipSel z, const FsbSide t, const FsbSide f, const ZipFsbArgs a) {
  const uint64_t lead = (uintptr_t)a.out & 15u;
  const uint64_t total = (uint64_t)z.len * a.w;
  const int64_t n_chunks = (int64_t)((lead + total + 15) >> 4);
  uint8_t *base = a.out - lead;  // chunk g is base + 16 g, output bytes 16 g - lead ..
  unsigned cnt = 0;
  for (int64_t r0 = (int64_t)blockIdx.x * ZIP_THREADS * ZIP_FSB_CHUNKS; r0 < n_chunks;
       r0 += (int64_t)gridDim.x * ZIP_THREADS * ZIP_FSB_CHUNKS) {
    unsigned __int128 tv[ZIP_FSB_CHUNKS], fv[ZIP_FSB_CHUNKS];
    uint64_t pl[ZIP_FSB_CHUNKS], ph[ZIP_FSB_CHUNKS], row0[ZIP_FSB_CHUNKS];
    // ---- issue: both sides' bytes of every chunk ----
#pragma unroll
    for (int k = 0; k < ZIP_FSB_CHUNKS; ++k) {
      const int64_t g = r0 + (int64_t)k * ZIP_THREADS + threadIdx.x;
      const uint64_t end = (uint64_t)g * 16 + 16 - lead;
      pl[k] = g == 0 ? 0 : (uint64_t)g * 16 - lead;
      ph[k] = end < total ? end : total;
      tv[k] = fv[k] = 0;
      row0[k] = 0;
      if (g < n_chunks) {
        row0[k] = div_by(a.div, pl[k]);
        const uint64_t phase = pl[k] - row0[k] * a.w;
        const uint32_t nb = (uint32_t)(ph[k] - pl[k]);
        tv[k] = side_bytes(t, pl[k], phase, nb);
        fv[k] = side_bytes(f, pl[k], phase, nb);
      }
    }
    // ---- select and store ----
#pragma unroll
    for (int k = 0; k < ZIP_FSB_CHUNKS; ++k) {
      const int64_t g = r0 + (int64_t)k * ZIP_THREADS + threadIdx.x;
      if (g >= n_chunks) continue;
      const int64_t wpos = (int64_t)row0[k] & ~(int64_t)63;
      // the selection bits of rows row0 .. row0 + MAXR - 1, which may run into the next 64-row word
      const uint64_t s_lo = z.sel(wpos), sh = row0[k] & 63u;
      uint64_t s = s_lo >> sh;
      if (sh + MAXR > 64u) s |= z.sel(wpos + 64) << (64u - sh);
      unsigned __int128 m = 0;
#pragma unroll
      for (int q = 0; q < MAXR; ++q) {
        const uint64_t rs = (row0[k] + q) * a.w;  // the row's first output byte
        if (rs >= ph[k]) break;
        if ((s >> q) & 1ull) {
          const uint64_t b0 = rs > pl[k] ? rs : pl[k], b1 = rs + a.w < ph[k] ? rs + a.w : ph[k];
          m |= byte_range_mask((uint32_t)(b0 - pl[k]), (uint32_t)(b1 - pl[k]));
        }
      }
      const unsigned __int128 o = (tv[k] & m) | (fv[k] & ~m);
      const uint64_t lo = (uint64_t)o, hi = (uint64_t)(o >> 64);
      const uint32_t first = g == 0 ? (uint32_t)lead : 0u;
      const uint32_t last = first + (uint32_t)(ph[k] - pl[k]);
      uint8_t *dst = base + (size_t)g * 16;
      if (first == 0u && last == 16u) {
        st_stream16(dst, make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32)));
      } else {
        for (uint32_t b = first; b < last; ++b) {
          const uint32_t x = b - first;
          dst[b] = (uint8_t)((x < 8u ? lo >> (8u * x) : hi >> (8u * (x - 8u))) & 0xffu);
        }
      }
      // the chunk holding the first byte of row 64 k owns validity word k
      if (z.out_valid) {
        const uint64_t first_row = row0[k] * a.w >= pl[k] ? row0[k] : row0[k] + 1;  // first row starting in the chunk
        const uint64_t q = (first_row + 63) & ~(uint64_t)63;
        if (q < (uint64_t)z.len && q * a.w < ph[k]) cnt += z.put_valid((int64_t)q, z.sel((int64_t)q));
      }
    }
  }
  if (z.out_valid) count_valid(z, cnt);
}

// ---- host side -------------------------------------------------------------------------------------------------------
acu_status check_lengths(acu_ctx *ctx, const acu_array *mask, const acu_array *t, const acu_array *f) {
  // zip.rs:123-145 (ScalarZipper::try_new, zip.rs:288-297, uses the same text for scalars)
  const bool ts = t->is_scalar != 0, fs = f->is_scalar != 0;
  if (ts && t->len != 1) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "scalar arrays must have 1 element");
  if (!ts && t->len != mask->len) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "all arrays should have the same length");
  if (fs && f->len != 1) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "scalar arrays must have 1 element");
  if (!fs && f->len != mask->len) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "all arrays should have the same length");
  return ACU_OK;
}

struct NullCounts {
  int64_t m, t, f;
};

acu_status resolve(acu_ctx *ctx, const acu_array *mask, const acu_array *t, const acu_array *f, NullCounts *nc) {
  acu_status st;
  nc->m = acu_resolve_null_count(ctx, mask, &st);
  ACU_TRY(st);
  nc->t = acu_resolve_null_count(ctx, t, &st);
  ACU_TRY(st);
  nc->f = acu_resolve_null_count(ctx, f, &st);
  return st;
}

// The mask and, for zip_impl, the validity of both sides: a NullBuffer iff some input has a null (transform/mod.rs:470).
ZipSel zip_impl_sel(const acu_array *mask, const acu_array *t, const acu_array *f, const NullCounts &nc, uint8_t *out_valid,
                    unsigned long long *res) {
  ZipSel z{};
  z.mv = static_cast<const uint8_t *>(mask->values);
  z.moff = mask->values_offset;
  if (mask->validity && nc.m > 0) { z.mn = mask->validity; z.mnoff = mask->validity_offset; }
  z.len = mask->len;
  z.res = res;
  z.t_all = nc.t > 0 && t->is_scalar ? 0 : 1;
  z.f_all = nc.f > 0 && f->is_scalar ? 0 : 1;
  if (!t->is_scalar && t->validity && nc.t > 0) { z.tn = t->validity; z.tnoff = t->validity_offset; }
  if (!f->is_scalar && f->validity && nc.f > 0) { z.fn = f->validity; z.fnoff = f->validity_offset; }
  if (nc.t > 0 || nc.f > 0) z.out_valid = reinterpret_cast<uint64_t *>(out_valid);
  return z;
}

// The builder's NullBuffer from the fetched valid count: zip_impl drops one without nulls (freeze); the scalar zippers with
// a null scalar always keep theirs (`always`).
void finish_nulls(const ZipSel &z, bool always, const unsigned long long *h, acu_array_out *out) {
  out->len = z.len;
  out->null_count = z.out_valid ? z.len - (int64_t)h[RES_COUNT] : 0;
  out->has_validity = z.out_valid && (always || out->null_count > 0) ? 1 : 0;
}

acu_status launch_bits(acu_ctx *ctx, int cls, const ZipSel &z, const BitSide &t, const BitSide &f, uint64_t *out) {
  if (z.len == 0 || (!out && !z.out_valid)) return ACU_OK;
  const int64_t words = (z.len + 63) >> 6;
  ACU_LAUNCH_TIMED(ctx, cls, k_zip_bits, acu_grid(ctx, (words + ZIP_THREADS - 1) / ZIP_THREADS, ZIP_PER_SM), ZIP_THREADS, 0, z, t, f, out);
  return ACU_OK;
}

template <class O>
acu_status zip_bytes_run(acu_ctx *ctx, const acu_array *mask, const acu_bytes_array *t, const acu_bytes_array *f, void *out_offsets,
                         uint8_t *out_data, int64_t out_cap, int64_t *out_data_len, acu_array_out *out_nulls) {
  const int64_t n = mask->len;
  NullCounts nc;
  ACU_TRY(resolve(ctx, mask, &t->nulls, &f->nulls, &nc));
  const bool ts = t->nulls.is_scalar != 0, fs = f->nulls.is_scalar != 0;
  const bool both = ts && fs, t_null = ts && nc.t > 0, f_null = fs && nc.f > 0;
  // a scalar's value range
  O tr[2] = {0, 0}, fr[2] = {0, 0};
  if (ts) ACU_CUDA(ctx, cudaMemcpyAsync(tr, t->offsets, 2 * sizeof(O), cudaMemcpyDeviceToHost, ctx->stream));
  if (fs) ACU_CUDA(ctx, cudaMemcpyAsync(fr, f->offsets, 2 * sizeof(O), cudaMemcpyDeviceToHost, ctx->stream));
  if (ts || fs) ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  ZipSel z = zip_impl_sel(mask, &t->nulls, &f->nulls, nc, out_nulls->validity, acu_dres(ctx, 0));
  ZipRows<O> rows{};
  rows.ob = (int)sizeof(O);
  rows.m = n;
  rows.mv = z.mv; rows.moff = z.moff; rows.mn = z.mn; rows.mnoff = z.mnoff;
  if (!ts) { rows.t_offs = static_cast<const O *>(t->offsets); rows.t_data = t->data; }
  if (!fs) { rows.f_offs = static_cast<const O *>(f->offsets); rows.f_data = f->data; }
  rows.ts = t->data + (int64_t)tr[0];
  rows.ts_len = (uint64_t)(int64_t)(tr[1] - tr[0]);
  rows.fs = f->data + (int64_t)fr[0];
  rows.fs_len = (uint64_t)(int64_t)(fr[1] - fr[0]);
  bool always = false;
  if (both) {
    // BytesScalarImpl::create_output (zip.rs:622-660): a null scalar's rows are empty and null
    z.tn = z.fn = nullptr;
    z.t_all = !t_null;
    z.f_all = !f_null;
    if (t_null) rows.ts_len = 0;
    if (f_null) rows.fs_len = 0;
    z.out_valid = t_null || f_null ? reinterpret_cast<uint64_t *>(out_nulls->validity) : nullptr;
    always = true;
  }
  if (n > 0) {
    void *scratch;
    ACU_TRY(acu_scratch(ctx, engine_scratch(n), &scratch));
    ACU_TRY(engine_launch(ctx, rows, static_cast<int64_t *>(scratch), out_offsets, out_data, out_cap,
                          sizeof(O) == 4 ? (int64_t)INT32_MAX : INT64_MAX));
    ACU_TRY(launch_bits(ctx, ACU_K_BYTES, z, BitSide{}, BitSide{}, nullptr));
  } else {
    ACU_CUDA(ctx, cudaMemsetAsync(out_offsets, 0, sizeof(O), ctx->stream));
  }
  ACU_TRY(acu_res_fetch(ctx));
  const unsigned long long *h = ctx->h_res;
  *out_data_len = 0;
  finish_nulls(z, always, h, out_nulls);
  if (n == 0) return ACU_OK;
  if (h[RES_ERR2] != ~0ull) {
    if (!both)  // try_extend_offsets (transform/utils.rs:33-60) at the first row whose end passes i32::MAX
      return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, (int64_t)h[RES_ERR2], 0, 0, 0, "%s", acu_extend_overflow_text);
    if (t_null || f_null)  // OffsetBuffer::from_lengths (arrow-buffer/src/buffer/offset.rs)
      return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, -1, 0, 0, 0, "offset overflow");
    int64_t selected = 0;  // all one side: from_repeated_length; mixed: OffsetBufferBuilder::finish (builder/offset.rs)
    ACU_TRY(acu_bitmap_count(ctx, z.mv, z.moff, z.mn, z.mnoff, n, &selected));
    return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, -1, 0, 0, 0, "%s", selected == 0 || selected == n ? "offset overflow" : "overflow");
  }
  return finish_bytes(ctx, out_data, out_cap, out_data_len);
}

acu_status read_view(acu_ctx *ctx, const acu_view_array *a, uint4 *v) {
  ACU_CUDA(ctx, cudaMemcpyAsync(v, a->views, 16, cudaMemcpyDeviceToHost, ctx->stream));
  return ACU_OK;
}

acu_status launch_views(acu_ctx *ctx, const ZipSel &z, const ViewSide &t, const ViewSide &f, void *out) {
  if (z.len == 0) return ACU_OK;
  ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_zip_views, acu_grid(ctx, (z.len + ZIP_THREADS - 1) / ZIP_THREADS, ZIP_PER_SM), ZIP_THREADS, 0, z, t, f,
                   static_cast<uint4 *>(out));
  return ACU_OK;
}

template <int MAXR>
acu_status launch_fsb_r(acu_ctx *ctx, const ZipSel &z, const FsbSide &t, const FsbSide &f, const ZipFsbArgs &a) {
  const int64_t n_chunks = (int64_t)((((uintptr_t)a.out & 15u) + (uint64_t)z.len * a.w + 15) >> 4);
  const int64_t per_block = (int64_t)ZIP_THREADS * ZIP_FSB_CHUNKS;
  ACU_LAUNCH_TIMED(ctx, ACU_K_ARITH, k_zip_fsb<MAXR>, acu_grid(ctx, (n_chunks + per_block - 1) / per_block, ZIP_PER_SM), ZIP_THREADS, 0, z, t,
                   f, a);
  return ACU_OK;
}

// A scalar side's pattern in `stage` (w + 16 bytes): its w bytes, then its first 16 bytes again (w < 16: repeated).
acu_status stage_scalar(acu_ctx *ctx, const acu_array *s, int64_t w, uint8_t *stage) {
  ACU_CUDA(ctx, cudaMemcpyAsync(stage, s->values, (size_t)w, cudaMemcpyDeviceToDevice, ctx->stream));
  uint8_t head[16], tail[16];
  const int64_t nh = w < 16 ? w : 16;
  ACU_CUDA(ctx, cudaMemcpyAsync(head, s->values, (size_t)nh, cudaMemcpyDeviceToHost, ctx->stream));
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < 16; ++i) tail[i] = head[i % nh];
  ACU_CUDA(ctx, cudaMemcpyAsync(stage + w, tail, 16, cudaMemcpyHostToDevice, ctx->stream));
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // `tail` lives on this stack frame
  return ACU_OK;
}

}  // namespace

// Every entry point starts with acu_res_reset, whose acu_sync_only refuses inside a stream-ordered section before any
// argument check.
extern "C" acu_status acu_zip_bytes(acu_ctx *ctx, int32_t offset_bytes, const acu_array *mask, const acu_bytes_array *truthy,
                                    const acu_bytes_array *falsy, void *out_offsets, uint8_t *out_data, int64_t out_data_capacity,
                                    int64_t *out_data_len, acu_array_out *out_nulls) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(acu_offset_width_check(ctx, offset_bytes));
  ACU_TRY(check_lengths(ctx, mask, &truthy->nulls, &falsy->nulls));
  for (const void *p : {truthy->offsets, falsy->offsets, (const void *)out_offsets})
    if ((uintptr_t)p % (uintptr_t)offset_bytes)
      return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "offsets must be %d-byte aligned", (int)offset_bytes);
  if (offset_bytes == 4) return zip_bytes_run<int32_t>(ctx, mask, truthy, falsy, out_offsets, out_data, out_data_capacity, out_data_len, out_nulls);
  return zip_bytes_run<int64_t>(ctx, mask, truthy, falsy, out_offsets, out_data, out_data_capacity, out_data_len, out_nulls);
}

extern "C" acu_status acu_zip_byte_view(acu_ctx *ctx, const acu_array *mask, const acu_view_array *truthy, const acu_view_array *falsy,
                                        void *out_views, acu_array_out *out_nulls, int32_t *out_buffers) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(check_lengths(ctx, mask, &truthy->nulls, &falsy->nulls));
  for (const void *p : {truthy->views, falsy->views, (const void *)out_views})
    if ((uintptr_t)p % 16u) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "views must be 16-byte aligned");
  const int64_t n = mask->len;
  NullCounts nc;
  ACU_TRY(resolve(ctx, mask, &truthy->nulls, &falsy->nulls, &nc));
  const bool ts = truthy->nulls.is_scalar != 0, fs = falsy->nulls.is_scalar != 0;
  const uint32_t nt = (uint32_t)(truthy->n_buffers > 0 ? truthy->n_buffers : 0), nf = (uint32_t)(falsy->n_buffers > 0 ? falsy->n_buffers : 0);
  uint4 tv = make_uint4(0, 0, 0, 0), fv = make_uint4(0, 0, 0, 0);
  if (ts) ACU_TRY(read_view(ctx, truthy, &tv));
  if (fs) ACU_TRY(read_view(ctx, falsy, &fv));
  ZipSel z = zip_impl_sel(mask, &truthy->nulls, &falsy->nulls, nc, out_nulls->validity, acu_dres(ctx, 0));
  ViewSide t{ts ? nullptr : static_cast<const uint4 *>(truthy->views), tv, 0u};
  ViewSide f{fs ? nullptr : static_cast<const uint4 *>(falsy->views), fv, nt};
  bool always = false;
  int32_t buffers = ZIP_BUFFERS_BOTH;  // zip_impl: truthy's buffers, then falsy's (transform/mod.rs:683-690)
  if (ts || fs) ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (!(ts && fs)) {
    if (fs && f.s.x > 12u) f.s.z += nt;  // build_extend_view: only a view that is not inline
  } else {
    // ByteViewScalarImpl::create_output (zip.rs:820-860), decided from the number of selected rows
    int64_t selected = 0;
    if (n > 0) ACU_TRY(acu_bitmap_count(ctx, z.mv, z.moff, z.mn, z.mnoff, n, &selected));
    ACU_TRY(acu_res_reset(ctx));
    const bool t_null = nc.t > 0, f_null = nc.f > 0;
    z.tn = z.fn = nullptr;
    z.out_valid = nullptr;
    if (!t_null && !f_null) {
      if (selected == 0) {
        t.s = fv;
        buffers = ZIP_BUFFERS_FALSY;
      } else if (selected == n) {
        f.s = tv;
        buffers = ZIP_BUFFERS_TRUTHY;
      } else if (nf > 0) {
        f.s.z += nt;  // re-based even when the falsy view is inline (zip.rs:759-769)
      } else {
        buffers = ZIP_BUFFERS_TRUTHY;
      }
    } else {
      // one valid scalar: its view in every row and nulls = the predicate (or its negation); nothing selected, or two null
      // scalars: zero views, no buffers, all null
      z.out_valid = reinterpret_cast<uint64_t *>(out_nulls->validity);
      always = true;
      const int64_t hits = t_null ? n - selected : selected;
      if ((t_null && f_null) || hits == 0) {
        t.s = f.s = make_uint4(0, 0, 0, 0);
        z.t_all = z.f_all = 0;
        buffers = ZIP_BUFFERS_NONE;
      } else if (!t_null) {
        f.s = tv;
        z.t_all = 1;
        z.f_all = 0;
        buffers = ZIP_BUFFERS_TRUTHY;
      } else {
        t.s = fv;
        z.t_all = 0;
        z.f_all = 1;
        buffers = ZIP_BUFFERS_FALSY;
      }
    }
    f.fix = 0;
  }
  ACU_TRY(launch_views(ctx, z, t, f, out_views));
  ACU_TRY(acu_res_fetch(ctx));
  finish_nulls(z, always, ctx->h_res, out_nulls);
  if (out_buffers) *out_buffers = buffers;
  return ACU_OK;
}

extern "C" acu_status acu_zip_boolean(acu_ctx *ctx, const acu_array *mask, const acu_array *truthy, const acu_array *falsy,
                                      acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(check_lengths(ctx, mask, truthy, falsy));
  NullCounts nc;
  ACU_TRY(resolve(ctx, mask, truthy, falsy, &nc));
  const ZipSel z = zip_impl_sel(mask, truthy, falsy, nc, out->validity, acu_dres(ctx, 0));
  BitSide t{static_cast<const uint8_t *>(truthy->values), truthy->values_offset, 0}, f{static_cast<const uint8_t *>(falsy->values),
                                                                                      falsy->values_offset, 0};
  for (BitSide *s : {&t, &f}) {
    const acu_array *a = s == &t ? truthy : falsy;
    if (!a->is_scalar) continue;
    uint8_t byte = 0;  // the scalar's value bit, also under a null (MutableArrayData copies it)
    ACU_CUDA(ctx, cudaMemcpyAsync(&byte, static_cast<const uint8_t *>(a->values) + (a->values_offset >> 3), 1, cudaMemcpyDeviceToHost,
                                  ctx->stream));
    ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    s->word = (byte >> (a->values_offset & 7)) & 1u ? ~0ull : 0ull;
    s->v = nullptr;
  }
  ACU_TRY(launch_bits(ctx, ACU_K_ARITH, z, t, f, reinterpret_cast<uint64_t *>(out->values)));
  ACU_TRY(acu_res_fetch(ctx));
  finish_nulls(z, false, ctx->h_res, out);
  return ACU_OK;
}

extern "C" acu_status acu_zip_fixed_size_binary(acu_ctx *ctx, int32_t byte_width, const acu_array *mask, const acu_array *truthy,
                                                const acu_array *falsy, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(check_lengths(ctx, mask, truthy, falsy));
  if (byte_width < 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid size of FixedSizeBinaryArray(%d)", (int)byte_width);
  NullCounts nc;
  ACU_TRY(resolve(ctx, mask, truthy, falsy, &nc));
  const ZipSel z = zip_impl_sel(mask, truthy, falsy, nc, out->validity, acu_dres(ctx, 0));
  const int64_t w = byte_width, n = mask->len;
  if (n > 0 && w == 0) {
    ACU_TRY(launch_bits(ctx, ACU_K_ARITH, z, BitSide{}, BitSide{}, nullptr));  // no bytes: the validity alone
  } else if (n > 0) {
    FsbSide t{static_cast<const uint8_t *>(truthy->values), 0}, f{static_cast<const uint8_t *>(falsy->values), 0};
    if (truthy->is_scalar || falsy->is_scalar) {
      const size_t one = ((size_t)w + 16 + 255) & ~(size_t)255;
      void *scratch;
      ACU_TRY(acu_scratch(ctx, 2 * one, &scratch));
      uint8_t *st = static_cast<uint8_t *>(scratch);
      if (truthy->is_scalar) { ACU_TRY(stage_scalar(ctx, truthy, w, st)); t = FsbSide{st, 1}; }
      if (falsy->is_scalar) { ACU_TRY(stage_scalar(ctx, falsy, w, st + one)); f = FsbSide{st + one, 1}; }
    }
    ZipFsbArgs a{};
    a.w = (uint64_t)w;
    a.div = make_div_w(a.w);
    a.out = static_cast<uint8_t *>(out->values);
    switch (w >= 16 ? 2 : w >= 8 ? 3 : w >= 4 ? 5 : w >= 2 ? 9 : 17) {
      case 2: ACU_TRY(launch_fsb_r<2>(ctx, z, t, f, a)); break;
      case 3: ACU_TRY(launch_fsb_r<3>(ctx, z, t, f, a)); break;
      case 5: ACU_TRY(launch_fsb_r<5>(ctx, z, t, f, a)); break;
      case 9: ACU_TRY(launch_fsb_r<9>(ctx, z, t, f, a)); break;
      default: ACU_TRY(launch_fsb_r<17>(ctx, z, t, f, a)); break;
    }
  }
  ACU_TRY(acu_res_fetch(ctx));
  finish_nulls(z, false, ctx->h_res, out);
  return ACU_OK;
}
