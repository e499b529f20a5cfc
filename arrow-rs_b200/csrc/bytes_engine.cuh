// bytes_engine.cuh — the offsets-and-copy stage of the variable-width kernels: a producer gives each row's source byte
// range, the engine sums them per CTA (k_bytes_block_totals), and after a device-wide scan of the CTA totals writes the new
// offsets and copies the bytes (k_bytes_offsets_copy). take / filter (bytes.cu), substring (substring.cu) and concat_elements
// (concat_elements.cu) differ only in the producer.
//
// A producer `R` is a trivially copyable struct with
//   int ob; int64_t m;            // offset width, output rows
//   const uint8_t *data;          // the source value bytes the ranges point into
//   int detect_oob;               // k_bytes_block_totals: *err of the first pass goes to res[RES_ERR_INDEX] (atomicMin)
//   void ranges4(int64_t j0, int64_t begin[4], uint64_t len[4], unsigned long long *err) const;
// where ranges4 gives the byte ranges of rows j0 .. j0+3 (zero length past m) and lowers *err to a failing row's key.
//
// A multi-segment producer (concat_elements.cu) builds each row from K >= 1 source segments, each with its own pointer (a
// different operand's buffer, or a view slot's inline bytes). Instead of `data` it has
//   int nsegs() const;                                                   // K
//   void segment(int64_t row, int s, const uint8_t **p, uint64_t *len) const;
// its ranges4 gives each row's total length (begin unused), and the copy pushes the segments of every non-empty row one
// after another through the same staging / direct paths.
#pragma once
#include <type_traits>

#include "internal.cuh"

#define BY_THREADS 512                 // CTA of the bytes kernels: 512 threads x 4 consecutive rows,
#define BY_ROWS (BY_THREADS * 4)       // two CTAs resident per SM so that one loads while the other assembles
#define BY_STAGE_CAP (48 * 1024)

namespace {

template <class R, class = void>
struct has_segments : std::false_type {};
template <class R>
struct has_segments<R, std::void_t<decltype(std::declval<const R &>().nsegs())>> : std::true_type {};

// kind: acu_take_index_kind of the index type
__device__ __forceinline__ uint64_t ld_index(const void *idx, int kind, int64_t j) {
  switch (kind) {
    case 0: return __ldg(static_cast<const uint8_t *>(idx) + j);
    case 1: return (uint64_t)(uint32_t)(int32_t)__ldg(static_cast<const int8_t *>(idx) + j);
    case 2: return __ldg(static_cast<const uint16_t *>(idx) + j);
    case 3: return (uint64_t)(uint32_t)(int32_t)__ldg(static_cast<const int16_t *>(idx) + j);
    case 4: return __ldg(static_cast<const uint32_t *>(idx) + j);
    default: return __ldg(static_cast<const uint64_t *>(idx) + j);
  }
}

// CTA-wide exclusive scan of one u64 per thread (up to 1024 threads); returns the thread's exclusive
// prefix, *total = the CTA total. Two barriers.
__device__ __forceinline__ uint64_t cta_scan_excl(uint64_t v, uint64_t *warp_tot /* [33] shared */, uint64_t *total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  uint64_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint64_t y = __shfl_up_sync(ACU_FULL_MASK, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    const uint64_t w = lane < (int)(blockDim.x >> 5) ? warp_tot[lane] : 0ull;
    uint64_t wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint64_t y = __shfl_up_sync(ACU_FULL_MASK, wi, o);
      if (lane >= o) wi += y;
    }
    warp_tot[lane] = wi - w;
    if (lane == 31) warp_tot[32] = wi;
  }
  __syncthreads();
  *total = warp_tot[32];
  return warp_tot[wid] + incl - v;
}

// pass 1: total value bytes of each CTA's 4096 rows (+ out-of-bounds detection)
template <class R>
__global__ void __launch_bounds__(BY_THREADS) k_bytes_block_totals(const R a, int64_t *__restrict__ block_tot,
                                                             unsigned long long *__restrict__ res) {
  __shared__ uint64_t warp_tot[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t j0 = (int64_t)blockIdx.x * BY_ROWS + (int64_t)threadIdx.x * 4;
  int64_t begin[4];
  uint64_t len[4];
  unsigned long long err = ~0ull;
  a.ranges4(j0, begin, len, &err);
  uint64_t sum = len[0] + len[1] + len[2] + len[3];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(ACU_FULL_MASK, sum, o);
  if (lane == 0) warp_tot[wid] = sum;
  __syncthreads();
  if (wid == 0) {
    uint64_t t = lane < BY_THREADS / 32 ? warp_tot[lane] : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(ACU_FULL_MASK, t, o);
    if (lane == 0) block_tot[blockIdx.x] = (int64_t)t;
  }
  if (a.detect_oob && err != ~0ull) atomicMin(res + RES_ERR_INDEX, err);
}

// Byte stream of one thread into the CTA's staging buffer: bytes are queued in a small
// accumulator (fewer than 4 pending bytes between pushes) and leave as whole aligned 32-bit
// words. A word shared with a neighbouring thread (the first one when the thread's output does
// not start on a word boundary, and the last partial one) is merged with atomicOr into the
// zero-initialised buffer; every other word is exclusively this thread's and is stored plainly.
// push8 is branch-free apart from the two predicated stores.
struct WordEmitter {
  uint32_t *w;
  uint32_t acc;   // pending bytes (low nacc bytes valid, rest zero)
  uint32_t nacc;  // 0..3
  bool shared_first;
  __device__ __forceinline__ void init(uint8_t *stage, uint32_t pos) {
    w = reinterpret_cast<uint32_t *>(stage) + (pos >> 2);
    nacc = pos & 3u;
    acc = 0;
    shared_first = nacc != 0;
  }
  __device__ __forceinline__ void store(uint32_t v) {
    if (shared_first) { atomicOr(w, v); shared_first = false; }
    else *w = v;
    ++w;
  }
  // v: up to 8 bytes (bytes at positions >= nb are zero), nb in 0..8
  __device__ __forceinline__ void push8(uint64_t v, uint32_t nb) {
    const uint32_t sh = nacc * 8u;                       // 0, 8, 16, 24
    const uint32_t vlo = (uint32_t)v, vhi = (uint32_t)(v >> 32);
    const uint32_t x0 = acc | (vlo << sh);
    const uint32_t x1 = __funnelshift_l(vlo, vhi, sh);   // (vhi:vlo << sh) >> 32
    const uint32_t x2 = __funnelshift_l(vhi, 0u, sh);    // bytes pushed past 64 bits (zero when sh == 0)
    const uint32_t t = nacc + nb;                        // 0..11 bytes available
    if (t >= 4u) store(x0);
    if (t >= 8u) store(x1);
    acc = t >= 8u ? x2 : (t >= 4u ? x1 : x0);
    nacc = t & 3u;
  }
  __device__ __forceinline__ void finish() {
    if (acc != 0u) atomicOr(w, acc);
  }
};

// Up to 8 bytes of data[pos .. pos+nb) (nb in 0..8) as a little-endian u64, zero above nb. Only
// aligned 8-byte words that contain at least one requested byte are read.
__device__ __forceinline__ uint64_t load_upto8(const uint8_t *__restrict__ data, int64_t pos, uint32_t nb) {
  const uintptr_t addr = (uintptr_t)data + (uintptr_t)pos;
  const uint64_t *p = reinterpret_cast<const uint64_t *>(addr & ~(uintptr_t)7);
  const uint32_t sh = (uint32_t)(addr & 7u) * 8u;
  uint64_t lo = 0, hi = 0;
  if (nb) lo = __ldg(p);
  if (sh + nb * 8u > 64u) hi = __ldg(p + 1);
  uint64_t w = (lo >> sh) | ((hi << 1) << (63u - sh));
  const uint64_t mask = nb >= 8u ? ~0ull : ((1ull << (nb * 8u)) - 1ull);
  return w & mask;
}

// The first nb (0..16) bytes of data[pos ..) as two little-endian u64 (zero above nb): three aligned
// 8-byte loads, each predicated on containing a requested byte, shared by both halves.
__device__ __forceinline__ void load_upto16(const uint8_t *__restrict__ data, int64_t pos, uint32_t nb, uint64_t *w0, uint64_t *w1) {
  const uintptr_t addr = (uintptr_t)data + (uintptr_t)pos;
  const uint64_t *p = reinterpret_cast<const uint64_t *>(addr & ~(uintptr_t)7);
  const uint32_t sh = (uint32_t)(addr & 7u) * 8u, bits = sh + nb * 8u;
  uint64_t x = 0, y = 0, z = 0;
  if (nb) x = __ldg(p);
  if (bits > 64u) y = __ldg(p + 1);
  if (bits > 128u) z = __ldg(p + 2);
  const uint64_t lo = (x >> sh) | ((y << 1) << (63u - sh));
  const uint64_t hi = (y >> sh) | ((z << 1) << (63u - sh));
  const uint32_t n0 = nb < 8u ? nb : 8u, n1 = nb - n0;
  *w0 = lo & (n0 >= 8u ? ~0ull : ((1ull << (n0 * 8u)) - 1ull));
  *w1 = hi & (n1 >= 8u ? ~0ull : ((1ull << (n1 * 8u)) - 1ull));
}

// The bytes data[pos .. pos+len) into the emitter: the first 16 without branches (short strings are the common case), then
// the rest of a long range 8 at a time. The single-range producers keep these lines inline in k_bytes_offsets_copy: called
// through this helper, their kernels compile to different SASS.
__device__ __forceinline__ void emit_range(WordEmitter &em, const uint8_t *data, int64_t pos, uint64_t len) {
  const uint32_t l32 = len > 16 ? 16u : (uint32_t)len;
  const uint32_t n0 = l32 < 8u ? l32 : 8u, n1 = l32 - n0;
  uint64_t w0, w1;
  load_upto16(data, pos, l32, &w0, &w1);
  em.push8(w0, n0);
  em.push8(w1, n1);
  for (uint64_t c = 16; c < len; c += 8) {
    const uint32_t nb = (uint32_t)((len - c) < 8 ? (len - c) : 8);
    em.push8(load_upto8(data, pos + (int64_t)c, nb), nb);
  }
}

__device__ __forceinline__ void copy_row_direct(uint8_t *__restrict__ dst, const uint8_t *__restrict__ data, int64_t src, uint64_t len) {
  for (uint64_t c = 0; c < len; c += 8) {
    const uint64_t w = ld_bits64(data, (src + (int64_t)c) << 3, (src + (int64_t)len) << 3);
    const int nb = (int)((len - c) < 8 ? (len - c) : 8);
#pragma unroll
    for (int bidx = 0; bidx < 8; ++bidx)
      if (bidx < nb) dst[c + bidx] = (uint8_t)(w >> (8 * bidx));
  }
}

// Skips the byte copy (grid-uniformly: out_data becomes NULL) when the total does not fit the caller's buffer or the offset
// type: decided on the device so that no host round trip sits between the sizing pass and the copy.
__device__ __forceinline__ void skip_copy_if_too_large(uint8_t *__restrict__ &out_data, const int64_t *total_ptr, int64_t out_cap, int64_t limit) {
  if (out_data != nullptr && total_ptr != nullptr) {
    const int64_t total = __ldg(total_ptr);
    if (total > out_cap || total > limit) out_data = nullptr;
  }
}

// pass 2 (after the inclusive scan of the CTA totals): offsets + byte copy. Source bytes are
// fetched 8 at a time with two aligned loads + funnel shift (ld_bits64 on a byte position). The
// CTA's output bytes [cta_begin, cta_end) are assembled in shared memory laid out relative to the
// 16-B aligned global address and written back as whole 128-bit stores (STAGED); CTAs whose
// output does not fit the staging buffer store bytes directly.
template <class R>
__global__ void __launch_bounds__(BY_THREADS, 2) k_bytes_offsets_copy(const R a, const int64_t *__restrict__ block_incl,
                                                             int64_t first_block, void *out_offs, uint8_t *__restrict__ out_data,
                                                             int64_t limit, int64_t probe_row, unsigned long long *res,
                                                             int stage_cap, const int64_t *__restrict__ total_ptr, int64_t out_cap) {
  extern __shared__ __align__(16) uint8_t s_out[];
  __shared__ uint64_t warp_tot[33];
  skip_copy_if_too_large(out_data, total_ptr, out_cap, limit);
  const int64_t blk = first_block + blockIdx.x;
  const int64_t cta_begin = blk ? block_incl[blk - 1] : 0, cta_end = block_incl[blk];
  const int64_t stage_origin = cta_begin - (int64_t)((uintptr_t)(out_data + cta_begin) & 15);  // global byte that maps to s_out[0]
  const bool staged = out_data != nullptr && probe_row < 0 && (cta_end - stage_origin) <= (int64_t)stage_cap;
  const uint32_t nbytes = staged ? (uint32_t)(cta_end - stage_origin) : 0u;  // staged span, starts 16-B aligned in global memory
  const uint32_t lead = (uint32_t)(cta_begin - stage_origin);                // bytes of the first chunk owned by the previous CTA
  if (staged) {  // zero the words the emitters OR into
    const uint32_t chunks = (nbytes + 15) >> 4;
    for (uint32_t c = threadIdx.x; c < chunks; c += BY_THREADS) reinterpret_cast<uint4 *>(s_out)[c] = make_uint4(0, 0, 0, 0);
  }
  const int64_t j0 = blk * BY_ROWS + (int64_t)threadIdx.x * 4;
  int64_t begin[4];
  uint64_t len[4];
  unsigned long long oob = ~0ull;
  a.ranges4(j0, begin, len, &oob);
  uint64_t cta_total;
  const uint64_t rel = cta_scan_excl(len[0] + len[1] + len[2] + len[3], warp_tot, &cta_total);  // also orders the zeroing before the emitters
  int64_t end[4];
  end[0] = cta_begin + (int64_t)(rel + len[0]);
  end[1] = end[0] + (int64_t)len[1];
  end[2] = end[1] + (int64_t)len[2];
  end[3] = end[2] + (int64_t)len[3];
  unsigned long long err = ~0ull;
#pragma unroll
  for (int k = 3; k >= 0; --k)
    if (j0 + k < a.m && end[k] > limit) err = (unsigned long long)(j0 + k);
  if (probe_row >= 0) {
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (probe_row == j0 + k) res[RES_AUX1] = (unsigned long long)end[k];
    return;
  }
  if (err != ~0ull) atomicMin(res + RES_ERR2, err);
  // new offsets: out[j0] = end of the previous row, out[j0+1..j0+3] = the first three ends;
  // the thread holding the last row also writes out[m]
  if (j0 <= a.m) {
    const int64_t first = cta_begin + (int64_t)rel;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (j0 + k <= a.m) {
        const int64_t v = k == 0 ? first : end[k - 1];
        if (a.ob == 4) static_cast<int32_t *>(out_offs)[j0 + k] = (int32_t)v;
        else static_cast<int64_t *>(out_offs)[j0 + k] = v;
      }
    if (j0 + 4 == a.m) {
      if (a.ob == 4) static_cast<int32_t *>(out_offs)[a.m] = (int32_t)end[3];
      else static_cast<int64_t *>(out_offs)[a.m] = end[3];
    }
  }
  if (out_data == nullptr) return;  // grid-uniform
  if (staged) {
    WordEmitter em;
    em.init(s_out, lead + (uint32_t)rel);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if constexpr (has_segments<R>::value) {
        if (len[k])
          for (int s = 0; s < a.nsegs(); ++s) {
            const uint8_t *p;
            uint64_t l;
            a.segment(j0 + k, s, &p, &l);
            emit_range(em, p, 0, l);
          }
      } else {
        // the first 16 bytes of every row without branches (short strings are the common case) ...
        const uint32_t l32 = len[k] > 16 ? 16u : (uint32_t)len[k];
        const uint32_t n0 = l32 < 8u ? l32 : 8u, n1 = l32 - n0;
        uint64_t w0, w1;
        load_upto16(a.data, begin[k], l32, &w0, &w1);
        em.push8(w0, n0);
        em.push8(w1, n1);
        // ... the rest of a long row 8 bytes at a time
        for (uint64_t c = 16; c < len[k]; c += 8) {
          const uint32_t nb = (uint32_t)((len[k] - c) < 8 ? (len[k] - c) : 8);
          em.push8(load_upto8(a.data, begin[k] + (int64_t)c, nb), nb);
        }
      }
    }
    em.finish();
    __syncthreads();
    uint8_t *g = out_data + stage_origin;
    const uint32_t chunks = (nbytes + 15) >> 4;
    for (uint32_t c = threadIdx.x; c < chunks; c += BY_THREADS) {
      const uint32_t b0 = c << 4;
      if (b0 >= lead && b0 + 16 <= nbytes) {
        *reinterpret_cast<uint4 *>(g + b0) = *reinterpret_cast<const uint4 *>(s_out + b0);
      } else {  // partial first / last chunk: only this CTA's bytes
        for (uint32_t x = b0 < lead ? lead : b0; x < b0 + 16 && x < nbytes; ++x) g[x] = s_out[x];
      }
    }
  } else {
    int64_t pos = cta_begin + (int64_t)rel;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if constexpr (has_segments<R>::value) {
        int64_t at = pos;
        if (len[k])
          for (int s = 0; s < a.nsegs(); ++s) {
            const uint8_t *p;
            uint64_t l;
            a.segment(j0 + k, s, &p, &l);
            if (l) copy_row_direct(out_data + at, p, 0, l);
            at += (int64_t)l;
          }
      } else {
        if (len[k]) copy_row_direct(out_data + pos, a.data, begin[k], len[k]);
      }
      pos += (int64_t)len[k];
    }
  }
}

// p / w for every 64-bit p by one multiply-high (Granlund-Montgomery round-up multiplier), for the kernels that find the row
// of a byte position in FixedSizeBinary(w) data (fixed_size_binary.cu, zip.cu): t = umulhi(magic, p), (t + ((p - t) >> sh1)) >> sh2.
struct DivW {
  uint64_t magic;
  int sh1, sh2;
};
__device__ __forceinline__ uint64_t div_by(const DivW &d, uint64_t p) {
  const uint64_t t = __umul64hi(d.magic, p);
  return (t + ((p - t) >> d.sh1)) >> d.sh2;
}
inline DivW make_div_w(uint64_t w) {  // w >= 1
  int l = 0;
  while (l < 64 && (1ull << l) < w) ++l;
  return DivW{(uint64_t)((((unsigned __int128)((l < 64 ? (1ull << l) : 0ull) - w)) << 64) / w) + 1, l < 1 ? l : 1, l > 1 ? l - 1 : 0};
}

// ---- host side: the launch sequence shared by substring.cu and concat_elements.cu ------------------------------------
inline size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

// block totals -> scan -> offsets (+ bytes when out_data != NULL and the total fits out_cap and `limit`); RES_AUX0 = the
// total, RES_ERR2 = the lowest row whose end passes `limit` (the largest value the output offset type holds).
template <class R>
acu_status engine_launch(acu_ctx *ctx, R rows, int64_t *block_tot, void *out_offsets, uint8_t *out_data, int64_t out_cap, int64_t limit) {
  const int64_t blocks = (rows.m + BY_ROWS - 1) / BY_ROWS;
  rows.detect_oob = 1;
  ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_bytes_block_totals<R>, (unsigned)blocks, BY_THREADS, 0, rows, block_tot, ctx->d_res);
  ACU_TRY(acu_scan_inclusive_i64(ctx, block_tot, blocks, block_tot + blocks));
  ACU_CUDA(ctx, cudaMemcpyAsync(ctx->d_res + RES_AUX0, block_tot + (blocks - 1), 8, cudaMemcpyDeviceToDevice, ctx->stream));
  rows.detect_oob = 0;
  const int stage_cap = BY_STAGE_CAP;
  ACU_CUDA(ctx, cudaFuncSetAttribute(k_bytes_offsets_copy<R>, cudaFuncAttributeMaxDynamicSharedMemorySize, stage_cap));
  ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_bytes_offsets_copy<R>, (unsigned)blocks, BY_THREADS, stage_cap, rows, block_tot, (int64_t)0, out_offsets,
                   out_data, limit, (int64_t)-1, ctx->d_res, stage_cap, block_tot + (blocks - 1), out_cap);
  return ACU_OK;
}
inline size_t engine_scratch(int64_t m) {
  const int64_t blocks = (m + BY_ROWS - 1) / BY_ROWS;
  return align256((size_t)(blocks + blocks / 4096 + 64) * 8);
}

inline acu_status finish_bytes(acu_ctx *ctx, uint8_t *out_data, int64_t out_cap, int64_t *out_data_len) {
  *out_data_len = (int64_t)ctx->h_res[RES_AUX0];
  if (out_data && *out_data_len > out_cap)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, (uint64_t)*out_data_len, "output data capacity %lld < required %lld",
                    (long long)out_cap, (long long)*out_data_len);
  return ACU_OK;
}

}  // namespace
