// bytes.cu — variable-width (Utf8 / Binary, i32 or i64 offsets) filter and take.
//
//   take_bytes   (arrow-select/src/take.rs:499-627)  — also Dictionary<K,Utf8> -> Utf8 cast,
//                which the reference implements as take(dict_values, keys)
//                (arrow-cast/src/cast/dictionary.rs:310-317)
//   filter_bytes (arrow-select/src/filter.rs:893-928)
//
// Both are a gather of source rows (filter gathers the plan's selected rows):
//   1. nulls first (take_nulls / filter_nulls), exactly like the reference;
//   2. len[j] = offsets[idx+1]-offsets[idx] for valid output slots, 0 for null slots
//      (take.rs:556-583; filter copies null slots too, filter.rs:891-892);
//   3. pass 1 sums the bytes of every 2048-row block, and a device-wide inclusive scan of the
//      block totals gives each block its first output byte;
//   4. pass 2 writes the new offsets (an i32 overflow reports the first row whose end passes
//      i32::MAX, take.rs:520-523) and copies the bytes. It runs one of three kernels:
//      k_dict_copy           i32 offsets, 32-bit indices with a 16-byte aligned base, a source of
//                            1 .. 8192 rows none longer than 16 bytes, and at least 65536 output
//                            rows: the source is kept in shared memory;
//      k_gather_copy         any other source with i32 offsets and 32-bit indices with a 16-byte
//                            aligned base;
//      k_bytes_offsets_copy  everything else: i64 offsets, 8-, 16- or 64-bit indices, or an
//                            index base that is not 16-byte aligned (bytes_engine.cuh).
#include <stdio.h>
#include <stdlib.h>

#include "bitmap.cuh"
#include "bytes_cmp.cuh"
#include "bytes_engine.cuh"
#include "internal.cuh"

#define SCAN_ELEMS 4096
#define PLAN_TILE_WORDS 64
#define PLAN_SCAN_CHUNK 4096

namespace {

// ---- device-wide inclusive scan of int64 (in place) ------------------------------------
__global__ void __launch_bounds__(1024) k_scan_block(int64_t *__restrict__ data, int64_t n, int64_t *__restrict__ block_tot) {
  __shared__ uint64_t warp_tot[33];
  const int64_t base = (int64_t)blockIdx.x * SCAN_ELEMS + (int64_t)threadIdx.x * 4;
  int64_t c[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) c[k] = (base + k < n) ? data[base + k] : 0;
  c[1] += c[0]; c[2] += c[1]; c[3] += c[2];
  uint64_t total;
  const int64_t excl = (int64_t)cta_scan_excl((uint64_t)c[3], warp_tot, &total);
  if (threadIdx.x == 0 && block_tot) block_tot[blockIdx.x] = (int64_t)total;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (base + k < n) data[base + k] = excl + c[k];
}

__global__ void __launch_bounds__(1024) k_scan_add(int64_t *__restrict__ data, int64_t n, const int64_t *__restrict__ block_incl) {
  if (blockIdx.x == 0) return;
  const int64_t add = block_incl[blockIdx.x - 1];
  const int64_t base = (int64_t)blockIdx.x * SCAN_ELEMS + (int64_t)threadIdx.x * 4;
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (base + k < n) data[base + k] += add;
}

acu_status scan_inclusive(acu_ctx *ctx, int64_t *data, int64_t n, int64_t *tmp /* >= blocks + blocks/4096 + 2 */) {
  if (n <= 0) return ACU_OK;
  const int64_t blocks = (n + SCAN_ELEMS - 1) / SCAN_ELEMS;
  ACU_LAUNCH(ctx, k_scan_block, (unsigned)blocks, 1024, 0, data, n, blocks > 1 ? tmp : nullptr);
  if (blocks > 1) {
    ACU_TRY(scan_inclusive(ctx, tmp, blocks, tmp + blocks));
    ACU_LAUNCH(ctx, k_scan_add, (unsigned)blocks, 1024, 0, data, n, tmp);
  }
  return ACU_OK;
}

// Indices(Vec<usize>) of FilterBuilder::optimize (filter.rs:285-298): selected row ids, u64.
template <class OutT>
__global__ void __launch_bounds__(256) k_plan_indices(const uint64_t *__restrict__ mask, const uint64_t *__restrict__ tile_off,
                                                      int64_t n_words_padded, OutT *__restrict__ out_idx) {
  // one lane per mask word; a warp covers 32 consecutive words (= two 1024-row tiles)
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w0 = warp * 32; w0 < n_words_padded; w0 += nwarps * 32) {
    uint64_t m = __ldg(mask + w0 + lane);
    const uint32_t c = __popcll(m);
    uint32_t incl = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t y = __shfl_up_sync(ACU_FULL_MASK, incl, o);
      if (lane >= o) incl += y;
    }
    if (__shfl_sync(ACU_FULL_MASK, incl, 31) == 0) continue;
    uint64_t k = __ldg(tile_off + (w0 >> 4)) + incl - c;
    const uint64_t row = (uint64_t)(w0 + lane) << 6;
    while (m) {
      const int b = __ffsll((long long)m) - 1;
      m &= m - 1;
      out_idx[k++] = (OutT)(row + b);
    }
  }
}

// ---- fused lengths / scan / offsets / copy -------------------------------------------------
// CTA = BY_THREADS threads x 4 CONSECUTIVE rows (BY_ROWS rows): a thread's four indices are
// one 128-bit load (FAST), its four validity bits a nibble of one u32, and the CTA-wide scan
// runs once over per-thread sums (two barriers) instead of once per row round. All eight
// source-offset loads of a thread are issued before any is used.
// FAST = i32 offsets + 32-bit indices with a 16-B aligned index buffer.
struct BytesArgs {
  const void *offs;        // source offsets (i32 or i64)
  const uint8_t *data;     // source value bytes
  const void *idx;         // source row of each output row
  int kind;                // index kind (see ld_index)
  int ob;                  // offset width
  int64_t m;               // output rows
  int64_t n_src;           // source rows (out-of-bounds detection)
  const uint32_t *out_valid;  // output validity (bit offset 0) or NULL: null slots get zero length
  int detect_oob;          // report an out-of-bounds index at a valid slot through res[RES_ERR_INDEX]
};

// Source byte range of the four rows j0 .. j0+3 (j0 % 4 == 0): begin[k], len[k] (0 for rows past the
// end, null output slots and out-of-bounds indices, whose lowest row goes to *oob_row).
template <bool FAST>
__device__ __forceinline__ void rows4(const BytesArgs &a, int64_t j0, int64_t begin[4], uint64_t len[4], unsigned long long *oob_row) {
  uint32_t vbits = 0xFu;
  if (a.out_valid && j0 < a.m) vbits = (__ldg(a.out_valid + (j0 >> 5)) >> (j0 & 31)) & 0xFu;
  if constexpr (FAST) {  // 32-bit indices, i32 offsets: everything per row in 32 bits
    uint32_t ix[4] = {0, 0, 0, 0};
    const int rows = a.m - j0 >= 4 ? 4 : (a.m > j0 ? (int)(a.m - j0) : 0);
    if (rows == 4) {
      const uint4 q = __ldg(reinterpret_cast<const uint4 *>(static_cast<const uint32_t *>(a.idx) + j0));
      ix[0] = q.x; ix[1] = q.y; ix[2] = q.z; ix[3] = q.w;
    } else {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (k < rows) ix[k] = __ldg(static_cast<const uint32_t *>(a.idx) + j0 + k);
    }
    const uint32_t n32 = a.n_src > (int64_t)0xffffffffll ? 0xffffffffu : (uint32_t)a.n_src;  // n_src >= 2^32: no u32 index is out of bounds
    const bool all_in = a.n_src > (int64_t)0xffffffffll;
    const int32_t *offs = static_cast<const int32_t *>(a.offs);
    int32_t s[4], e[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      bool use = (k < rows) && ((vbits >> k) & 1u);
      if (use && !all_in && ix[k] >= n32) {
        use = false;
        if ((unsigned long long)(j0 + k) < *oob_row) *oob_row = (unsigned long long)(j0 + k);
      }
      s[k] = 0;
      e[k] = 0;
      if (use) {
        s[k] = __ldg(offs + ix[k]);
        e[k] = __ldg(offs + ix[k] + 1);
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      begin[k] = s[k];
      len[k] = (uint32_t)(e[k] - s[k]);
    }
    return;
  }
  uint64_t ix[4] = {0, 0, 0, 0};
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (j0 + k < a.m) ix[k] = ld_index(a.idx, a.kind, j0 + k);
  bool use[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    use[k] = (j0 + k < a.m) && ((vbits >> k) & 1u);
    if (use[k] && ix[k] >= (uint64_t)a.n_src) {
      use[k] = false;
      if ((unsigned long long)(j0 + k) < *oob_row) *oob_row = (unsigned long long)(j0 + k);
    }
  }
  int64_t s[4], e[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {  // all loads first
    s[k] = 0;
    e[k] = 0;
    if (use[k]) {
      s[k] = ld_offset(a.offs, a.ob, (int64_t)ix[k]);
      e[k] = ld_offset(a.offs, a.ob, (int64_t)ix[k] + 1);
    }
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    begin[k] = s[k];
    len[k] = (uint64_t)(e[k] - s[k]);
  }
}

// The take / filter producer of bytes_engine.cuh.
template <bool FAST>
struct GatherRows : BytesArgs {
  __device__ __forceinline__ void ranges4(int64_t j0, int64_t begin[4], uint64_t len[4], unsigned long long *err) const {
    rows4<FAST>(*this, j0, begin, len, err);
  }
};

// ---- dictionary gather: take_bytes from a SMALL source (Dictionary<Int32,Utf8> -> Utf8, cast/dictionary.rs:310-317) ----
// A gather of 32 random dictionary rows through global memory costs 32 L1 wavefronts per load instruction whatever its
// width (one 128-byte line per lane): with two offset loads and the value bytes per row that alone is ~5 cycles per row
// per SM. Here the dictionary is first re-laid out as a table of
// 16-byte zero-padded entries + one length byte per entry (k_dict_table; sources with an entry longer than 16 bytes keep
// the generic path) and every CTA keeps that table in shared memory (D x 17 bytes: 70 KB for D = 4096): the gathers become
// LDS.128 / LDS.U8.
//   pass 1 (k_dict_block_totals): a WARP owns a 2048-row block — 16 x (one 128-bit load of 4 keys per lane, 4 LDS.U8),
//     one redux.sync, no CTA barrier.
//   pass 2 (k_dict_copy): a CTA owns a 2048-row block per round (see the round skeleton below), lane == row % 32 so that
//     the 32 rows of an instruction land ~8 bytes apart: ~2-way bank conflicts. A row's bytes reach their position in the
//     round's image by funnel shifts + predicated ATOMS.OR. All positions inside a round are 32-bit. The first version of
//     this path (warp-private rings, 64-bit positions, bytewise head / tail per warp) was issue-bound.
#define DG_THREADS 512
#define DG_WARPS (DG_THREADS / 32)
#define DG_WROWS (BY_ROWS / DG_WARPS)   // 128 rows per warp and round
#define DG_ITERS (DG_WROWS / 32)        // 4 x 32 rows
#define DG_IMG_BYTES (BY_ROWS * 16 + 32)  // image of one CTA round: <= 2048 x 16 bytes + alignment slack
#define DG_MAX_ENTRIES 8192
static_assert(DG_ITERS == 4, "round_place packs the four 32-row scans of a warp into two registers");

// ---- the round skeleton of k_dict_copy and k_gather_copy ---------------------------------------------------------------------
// A CTA of DG_WARPS warps owns one 2048-row block per round; a lane's rows are r0 + 32 i (r0 = warp * 128 + lane, i < 4).
// With the rows' lengths known, the four 32-row scans of a warp run as two packed 16-bit scans (round_place), the new
// offsets follow (round_offsets), the rows' bytes are ORed into a zeroed 32-KB shared-memory IMAGE of the round's output
// that mirrors the output's 16-byte alignment (each kernel's own code), and the image leaves as coalesced 128-bit stores,
// re-zeroed on the way (image_flush).
__device__ __forceinline__ uint32_t round_rows(int64_t m, int64_t blk) {
  const int64_t left = m - blk * BY_ROWS;
  return left < BY_ROWS ? (uint32_t)left : (uint32_t)BY_ROWS;
}

// A lane's four 32-bit indices of round `blk` (~0 for rows past the end) and, in lanes i < 4, the validity word of the
// warp's i-th 32-row group (all ones without a bitmap, 0 past the end).
__device__ __forceinline__ void round_load(const uint32_t *idx, const uint32_t *out_valid, int64_t m, int64_t blk, uint32_t ix[DG_ITERS], uint32_t &vw) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t base = blk * BY_ROWS;
  const uint32_t rows_here = round_rows(m, blk);
  const uint32_t r0 = wid * DG_WROWS + lane;
  const uint32_t *ip = idx + base + r0;
#pragma unroll
  for (int i = 0; i < DG_ITERS; ++i) ix[i] = (r0 + i * 32 < rows_here) ? __ldg(ip + i * 32) : 0xffffffffu;
  vw = 0xffffffffu;
  if (out_valid) vw = (lane < DG_ITERS && wid * DG_WROWS + lane * 32 < rows_here) ? __ldg(out_valid + (base >> 5) + wid * DG_ITERS + lane) : 0u;
}

// pre[i] = the first byte of row r0 + 32 i within its warp's bytes, wbase = the bytes of the warps before this one; returns
// the round's byte total. Every 32-row total must fit 16 bits (rows of at most 16 bytes, or a round of at most 32 KB).
// One barrier; s_wtot holds DG_WARPS words.
__device__ __forceinline__ uint32_t round_place(const uint32_t len[DG_ITERS], uint32_t *s_wtot, uint32_t pre[DG_ITERS], uint32_t &wbase) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t p01 = len[0] | (len[1] << 16), p23 = len[2] | (len[3] << 16);
  uint32_t i01 = p01, i23 = p23;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t y01 = __shfl_up_sync(ACU_FULL_MASK, i01, o), y23 = __shfl_up_sync(ACU_FULL_MASK, i23, o);
    if (lane >= (uint32_t)o) { i01 += y01; i23 += y23; }
  }
  const uint32_t t01 = __shfl_sync(ACU_FULL_MASK, i01, 31), t23 = __shfl_sync(ACU_FULL_MASK, i23, 31);
  const uint32_t e01 = i01 - p01, e23 = i23 - p23;  // exclusive (no borrow between the fields: each inclusive field >= its own term)
  const uint32_t tot0 = t01 & 0xffffu, tot1 = t01 >> 16, tot2 = t23 & 0xffffu;
  pre[0] = e01 & 0xffffu;
  pre[1] = tot0 + (e01 >> 16);
  pre[2] = tot0 + tot1 + (e23 & 0xffffu);
  pre[3] = tot0 + tot1 + tot2 + (e23 >> 16);
  if (lane == 0) s_wtot[wid] = tot0 + tot1 + tot2 + (t23 >> 16);
  __syncthreads();
  const uint32_t wv = lane < DG_WARPS ? s_wtot[lane] : 0u;
  wbase = __reduce_add_sync(ACU_FULL_MASK, lane < wid ? wv : 0u);
  return __reduce_add_sync(ACU_FULL_MASK, wv);
}

// The new offsets of a round's rows (32-bit wrapping arithmetic on the truncated base: an overflow is reported, not stored),
// the lowest row whose end passes `limit` into err (take.rs:521 "offset overflow"), and offsets[m] from the lane holding
// the last row.
__device__ __forceinline__ void round_offsets(int32_t *out_offs, int64_t m, int64_t base, uint32_t r0, uint32_t rows_here, int64_t cta_begin,
                                              uint32_t T, uint32_t wbase, const uint32_t pre[DG_ITERS], const uint32_t len[DG_ITERS], int64_t limit,
                                              unsigned long long &err) {
  const uint32_t o32 = (uint32_t)cta_begin + wbase;
  uint32_t *op = reinterpret_cast<uint32_t *>(out_offs) + base + r0;
#pragma unroll
  for (int i = 0; i < DG_ITERS; ++i)
    if (r0 + i * 32 < rows_here) op[i * 32] = o32 + pre[i];
  if (cta_begin + T > limit) {
    const int64_t o0 = cta_begin + wbase;
#pragma unroll
    for (int i = 0; i < DG_ITERS; ++i)
      if (r0 + i * 32 < rows_here && o0 + pre[i] + len[i] > limit && (unsigned long long)(base + r0 + i * 32) < err)
        err = (unsigned long long)(base + r0 + i * 32);
  }
  if (base + rows_here == m) {
#pragma unroll
    for (int i = 0; i < DG_ITERS; ++i)
      if (r0 + i * 32 + 1 == rows_here) reinterpret_cast<uint32_t *>(out_offs)[m] = o32 + pre[i] + len[i];
  }
}

// OR `x` into the shared-memory word at byte address `saddr + OFF` (RED: no return value)
template <int OFF>
__device__ __forceinline__ void red_or(uint32_t saddr, uint32_t x) {
  asm volatile("red.shared.or.b32 [%0+%2], %1;" ::"r"(saddr), "r"(x), "n"(OFF) : "memory");
}

// After a barrier (every row is in the image): the round's T bytes, image bytes A .. A + T (A = the output's misalignment
// at cta_begin), to out_data + cta_begin. The first / last chunk is shared with the neighbouring rounds' bytes: it is
// written by whole words, then single bytes. Every chunk read is zeroed again.
__device__ __forceinline__ void image_flush(uint4 *img4, uint8_t *out_data, int64_t cta_begin, uint32_t A, uint32_t T) {
  __syncthreads();
  const uint32_t end = A + T;
  const uint32_t chunks = (end + 15u) >> 4;
  const uint32_t first_full = (A + 15u) >> 4, n_full = (end >> 4) > first_full ? (end >> 4) - first_full : 0u;
  uint8_t *gb = out_data + cta_begin - A;  // 16-byte aligned
  for (uint32_t c = threadIdx.x; c < chunks; c += DG_THREADS) {
    const uint4 q = img4[c];
    img4[c] = make_uint4(0, 0, 0, 0);
    if (c - first_full < n_full) {
      reinterpret_cast<uint4 *>(gb)[c] = q;
    } else {
      const uint32_t qw[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (uint32_t w4 = 0; w4 < 4; ++w4) {
        const uint32_t lo = (c << 4) + 4u * w4;
        if (lo >= A && lo + 4u <= end) {
          *reinterpret_cast<uint32_t *>(gb + lo) = qw[w4];
        } else {
#pragma unroll
          for (uint32_t b = 0; b < 4; ++b)
            if (lo + b >= A && lo + b < end) gb[lo + b] = (uint8_t)(qw[w4] >> (8u * b));
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_dict_table(const int32_t *__restrict__ offs, const uint8_t *__restrict__ data, int64_t n_src,
                                                    uint4 *__restrict__ table, uint8_t *__restrict__ lens, int *__restrict__ too_long) {
  const int64_t d = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n_src) return;
  const int32_t s = __ldg(offs + d), e = __ldg(offs + d + 1);
  const int32_t len = e - s;
  uint32_t w[4] = {0, 0, 0, 0};
  if (len < 0 || len > 16) {
    atomicOr(too_long, 1);
  } else {
    for (int k = 0; k < len; ++k) w[k >> 2] |= (uint32_t)__ldg(data + s + k) << (8 * (k & 3));
  }
  table[d] = make_uint4(w[0], w[1], w[2], w[3]);
  lens[d] = (uint8_t)(len < 0 || len > 16 ? 0 : len);
}

struct DictArgs {
  const uint32_t *keys;       // 32-bit keys (ToIndices of i32 / u32), 16-byte aligned
  int64_t m;                  // output rows
  uint32_t n_src;             // dictionary entries (<= DG_MAX_ENTRIES)
  const uint32_t *out_valid;  // output validity (bit offset 0) or NULL: null slots get zero length
  int detect_oob;
  const uint4 *table;
  const uint8_t *lens;
  const int *too_long;        // set by k_dict_table: the kernels return immediately and the generic path runs
};

// pass 1: byte total of every 2048-row block (+ out-of-bounds keys at valid slots); a warp per block
__global__ void __launch_bounds__(DG_THREADS) k_dict_block_totals(const DictArgs a, int64_t blocks, int64_t *__restrict__ block_tot,
                                                                  unsigned long long *__restrict__ res) {
  extern __shared__ __align__(16) uint8_t s_dyn[];
  if (*a.too_long) return;
  uint8_t *s_len = s_dyn;
  for (uint32_t i = threadIdx.x; i < a.n_src; i += DG_THREADS) s_len[i] = a.lens[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * DG_THREADS + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * DG_THREADS) >> 5;
  const uint32_t n_src = a.n_src;
  unsigned long long err = ~0ull;
  for (int64_t blk = warp; blk < blocks; blk += nwarps) {
    const int64_t base = blk * BY_ROWS;
    uint32_t sum = 0;
    if (base + BY_ROWS <= a.m) {  // a whole block: 16 x (4 keys per lane)
      const uint4 *kp = reinterpret_cast<const uint4 *>(a.keys + base) + lane;
      const uint32_t *vp = a.out_valid ? a.out_valid + (base >> 5) + (lane >> 3) : nullptr;
      const int vsh = (lane & 7) * 4;
#pragma unroll 1
      for (int it0 = 0; it0 < BY_ROWS / 128; it0 += 8) {  // 8 x 128-bit key loads (+ 8 validity words) in flight per lane
        uint4 k[8];
        uint32_t vb[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          k[u] = __ldg(kp + (it0 + u) * 32);
          vb[u] = vp ? __ldg(vp + (it0 + u) * 4) : 0xffffffffu;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const uint32_t v4 = (vb[u] >> vsh) & 0xfu;
          const uint32_t kk[4] = {k[u].x, k[u].y, k[u].z, k[u].w};
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            if ((v4 >> e) & 1u) {
              if (kk[e] < n_src) sum += s_len[kk[e]];
              else {
                const unsigned long long j = (unsigned long long)(base + (it0 + u) * 128 + lane * 4 + e);
                if (j < err) err = j;
              }
            }
          }
        }
      }
    } else {  // the ragged last block
      for (int r = lane; r < BY_ROWS; r += 32) {
        const int64_t j = base + r;
        if (j >= a.m) break;
        const uint32_t key = __ldg(a.keys + j);
        bool use = true;
        if (a.out_valid) use = (__ldg(a.out_valid + (j >> 5)) >> (j & 31)) & 1u;
        if (use) {
          if (key < n_src) sum += s_len[key];
          else if ((unsigned long long)j < err) err = (unsigned long long)j;
        }
      }
    }
    sum = __reduce_add_sync(ACU_FULL_MASK, sum);
    if (lane == 0) block_tot[blk] = (int64_t)sum;
  }
  if (a.detect_oob && err != ~0ull) atomicMin(res + RES_ERR_INDEX, err);
}

// pass 2: new offsets + bytes. A CTA round is a dependent chain (keys -> lengths -> scan -> barrier -> image -> barrier ->
// flush -> barrier) with only two CTAs per SM, so the NEXT round's keys, validity words and base offset are loaded at the
// top of the current round (software prefetch): without it every round exposes a full DRAM latency.
struct DictRound {
  uint32_t key[DG_ITERS];  // raw keys (~0 for rows past the end)
  uint32_t vw;             // lane i < 4: validity word of the warp's i-th 32-row group (all ones without a bitmap)
  int64_t cta_begin;
  uint32_t rows_here;
};

__device__ __forceinline__ void dict_round_load(const DictArgs &a, const int64_t *__restrict__ block_incl, int64_t blk, DictRound &r) {
  r.rows_here = round_rows(a.m, blk);
  r.cta_begin = blk ? __ldg(block_incl + blk - 1) : 0;
  round_load(a.keys, a.out_valid, a.m, blk, r.key, r.vw);
}

__global__ void __launch_bounds__(DG_THREADS, 2) k_dict_copy(const DictArgs a, const int64_t *__restrict__ block_incl, int64_t blocks,
                                                             int32_t *__restrict__ out_offs, uint8_t *__restrict__ out_data, int64_t limit,
                                                             unsigned long long *res, const int64_t *__restrict__ total_ptr, int64_t out_cap) {
  extern __shared__ __align__(16) uint8_t s_dyn[];
  __shared__ uint32_t s_wtot[DG_WARPS];
  if (*a.too_long) return;
  skip_copy_if_too_large(out_data, total_ptr, out_cap, limit);
  const uint32_t n_src = a.n_src;  // the shared-memory table has n_src + 1 entries: the last one is the empty string
  uint4 *s_tab = reinterpret_cast<uint4 *>(s_dyn);
  uint8_t *s_len = s_dyn + ((size_t)n_src + 1) * 16;
  uint32_t *s_img = reinterpret_cast<uint32_t *>(s_dyn + ((size_t)n_src + 1) * 16 + ((n_src + 16u) & ~15u));
  DictRound cur;
  if ((int64_t)blockIdx.x < blocks) dict_round_load(a, block_incl, blockIdx.x, cur);
  for (uint32_t i = threadIdx.x; i < n_src; i += DG_THREADS) { s_tab[i] = a.table[i]; s_len[i] = a.lens[i]; }
  if (threadIdx.x == 0) { s_tab[n_src] = make_uint4(0, 0, 0, 0); s_len[n_src] = 0; }
  for (uint32_t i = threadIdx.x; i < DG_IMG_BYTES / 16; i += DG_THREADS) reinterpret_cast<uint4 *>(s_img)[i] = make_uint4(0, 0, 0, 0);
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t r0 = wid * DG_WROWS + lane;  // this lane's rows of a round: r0 + 32 i
  const uint32_t img = (uint32_t)__cvta_generic_to_shared(s_img);
  unsigned long long err = ~0ull;
  for (int64_t blk = blockIdx.x; blk < blocks; blk += gridDim.x) {
    const int64_t base = blk * BY_ROWS;
    const uint32_t rows_here = cur.rows_here;
    const int64_t cta_begin = cur.cta_begin;
    uint32_t key[DG_ITERS], len[DG_ITERS];
#pragma unroll
    for (int i = 0; i < DG_ITERS; ++i) {
      const uint32_t vw = __shfl_sync(ACU_FULL_MASK, cur.vw, i);
      const bool use = ((vw >> lane) & 1u) && cur.key[i] < n_src;  // (a row past the end has key ~0; OOB keys were reported by pass 1)
      key[i] = use ? cur.key[i] : n_src;                            // entry n_src = the empty string
      len[i] = s_len[key[i]];
    }
    if (blk + gridDim.x < blocks) dict_round_load(a, block_incl, blk + gridDim.x, cur);  // in flight during this round
    uint32_t pre[DG_ITERS], wbase;
    const uint32_t T = round_place(len, s_wtot, pre, wbase);
    round_offsets(out_offs, a.m, base, r0, rows_here, cta_begin, T, wbase, pre, len, limit, err);
    // ---- bytes: rows -> image (predicated RED.OR), image -> global (128-bit stores) ----
    if (out_data != nullptr) {
      const uint32_t A = (uint32_t)((uintptr_t)(out_data + cta_begin) & 15);
#pragma unroll
      for (int i = 0; i < DG_ITERS; ++i) {
        const uint4 e = s_tab[key[i]];  // zero beyond the entry's length
        const uint32_t d = A + wbase + pre[i];
        const uint32_t dsh = (d & 3u) * 8u;
        const uint32_t w = img + (d & ~3u);
        // (ptxas turns a predicated shared-memory RED into branch + BSSY/BSYNC, 5 instructions per word: the first four
        // words are ORed unconditionally — a zero is harmless — and the fifth, non-zero only for rows longer than 12 bytes
        // that start off a word boundary, hides behind one warp vote)
        red_or<0>(w, e.x << dsh);
        red_or<4>(w, __funnelshift_l(e.x, e.y, dsh));
        red_or<8>(w, __funnelshift_l(e.y, e.z, dsh));
        red_or<12>(w, __funnelshift_l(e.z, e.w, dsh));
        const uint32_t x4 = __funnelshift_l(e.w, 0u, dsh);
        if (__any_sync(ACU_FULL_MASK, x4 != 0u)) red_or<16>(w, x4);
      }
      image_flush(reinterpret_cast<uint4 *>(s_img), out_data, cta_begin, A, T);
    }
    __syncthreads();  // the image is zero again, s_wtot can be rewritten
  }
  if (err != ~0ull) atomicMin(res + RES_ERR2, err);
}

// ---- generic gather, FAST case (i32 offsets, 32-bit indices) -------------------------------------------------------------
// The round skeleton applied to an arbitrary source. Where a row's bytes come from differs from the dictionary kernel —
// two scattered offset loads, then up to 16 bytes by three predicated aligned 8-byte loads (rows longer than 16 bytes loop
// in 8-byte pieces) — and those loads are software-pipelined over THREE rounds (indices of round r + 2, offsets of round
// r + 1, bytes of round r in flight together), because a round is one dependent chain of three DRAM round trips. A block
// whose bytes do not fit the image (T > 32 KB, i.e. rows averaging more than 16 bytes) takes a slow direct-copy path in the
// same kernel.
#define GC_IMG_BYTES (BY_ROWS * 16)

// stage 2 (one round ahead): source byte range of this lane's four rows (0 / 0 for rows past the end, null slots and
// out-of-bounds indices) + the block's first output byte and its byte count (saturated to 32 bits)
__device__ __forceinline__ void gather_load_offsets(const BytesArgs &a, const int64_t *__restrict__ block_incl, int64_t blk, const uint32_t idx[DG_ITERS],
                                                    uint32_t vw_lanes, int32_t s[DG_ITERS], int32_t e[DG_ITERS], int64_t &cta_begin, uint32_t &T32) {
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t r0 = wid * DG_WROWS + lane;
  const uint32_t rows_here = round_rows(a.m, blk);
  const bool all_in = a.n_src > (int64_t)0xffffffffll;
  const uint32_t n32 = all_in ? 0xffffffffu : (uint32_t)a.n_src;
  const int32_t *offs = static_cast<const int32_t *>(a.offs);
#pragma unroll
  for (int i = 0; i < DG_ITERS; ++i) {
    const uint32_t vw = __shfl_sync(ACU_FULL_MASK, vw_lanes, i);
    const bool use = (r0 + i * 32 < rows_here) && ((vw >> lane) & 1u) && (all_in || idx[i] < n32);  // OOB: reported by pass 1
    s[i] = 0;
    e[i] = 0;
    if (use) {
      s[i] = __ldg(offs + idx[i]);
      e[i] = __ldg(offs + idx[i] + 1);
    }
  }
  cta_begin = blk ? __ldg(block_incl + blk - 1) : 0;
  const int64_t t = __ldg(block_incl + blk) - cta_begin;
  T32 = t > (int64_t)0xffffffffll ? 0xffffffffu : (uint32_t)t;
}

__global__ void __launch_bounds__(DG_THREADS, 2) k_gather_copy(const BytesArgs a, const int64_t *__restrict__ block_incl, int64_t blocks,
                                                               int32_t *__restrict__ out_offs, uint8_t *__restrict__ out_data, int64_t limit,
                                                               unsigned long long *res, const int64_t *__restrict__ total_ptr, int64_t out_cap) {
  extern __shared__ __align__(16) uint8_t s_dyn[];
  __shared__ uint32_t s_wtot[DG_WARPS];
  __shared__ unsigned long long s_wtot64[DG_WARPS];
  skip_copy_if_too_large(out_data, total_ptr, out_cap, limit);
  uint32_t *s_img = reinterpret_cast<uint32_t *>(s_dyn);
  uint4 *img4 = reinterpret_cast<uint4 *>(s_dyn);
  for (uint32_t i = threadIdx.x; i < (GC_IMG_BYTES + 32) / 16; i += DG_THREADS) img4[i] = make_uint4(0, 0, 0, 0);
  const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const uint32_t r0 = wid * DG_WROWS + lane;
  const uint32_t img = (uint32_t)__cvta_generic_to_shared(s_img);
  const uint32_t *idx = static_cast<const uint32_t *>(a.idx);
  const uint8_t *__restrict__ data = a.data;
  unsigned long long err = ~0ull;
  // pipeline state: (s, e, first output byte, byte count) of the current round, (indices, validity words) of the next one
  int32_t s[DG_ITERS], e[DG_ITERS];
  uint32_t idx_n[DG_ITERS], vw_n = 0, T_c = 0;
  int64_t begin_c = 0;
  const int64_t stride = gridDim.x;
  int64_t blk = blockIdx.x;
  if (blk < blocks) {
    uint32_t idx0[DG_ITERS], vw0;
    round_load(idx, a.out_valid, a.m, blk, idx0, vw0);
    gather_load_offsets(a, block_incl, blk, idx0, vw0, s, e, begin_c, T_c);
    if (blk + stride < blocks) round_load(idx, a.out_valid, a.m, blk + stride, idx_n, vw_n);
  }
  __syncthreads();
  for (; blk < blocks; blk += stride) {
    const int64_t base = blk * BY_ROWS;
    const uint32_t rows_here = round_rows(a.m, blk);
    const int64_t cta_begin = begin_c;
    const uint32_t Tblk = T_c;
    uint32_t len[DG_ITERS];
    int32_t sc[DG_ITERS];
#pragma unroll
    for (int i = 0; i < DG_ITERS; ++i) {
      sc[i] = s[i];
      len[i] = (uint32_t)(e[i] - s[i]);
    }
    // next round's offsets (its indices arrived during the previous round) and the round after's indices
    if (blk + stride < blocks) {
      gather_load_offsets(a, block_incl, blk + stride, idx_n, vw_n, s, e, begin_c, T_c);
      if (blk + 2 * stride < blocks) round_load(idx, a.out_valid, a.m, blk + 2 * stride, idx_n, vw_n);
    }
    if (Tblk <= (uint32_t)GC_IMG_BYTES) {
      // ---- the first 16 bytes of every row: three predicated aligned 8-byte loads each, all issued before the scan ----
      uint64_t w[DG_ITERS][3];
      uint32_t sh[DG_ITERS];
      if (out_data != nullptr) {
#pragma unroll
        for (int i = 0; i < DG_ITERS; ++i) {
          const uintptr_t addr = (uintptr_t)data + (uintptr_t)(int64_t)sc[i];
          const uint64_t *p = reinterpret_cast<const uint64_t *>(addr & ~(uintptr_t)7);
          const uint32_t l16 = len[i] > 16u ? 16u : len[i];
          sh[i] = (uint32_t)(addr & 7u) * 8u;
          const uint32_t bits = sh[i] + l16 * 8u;
          w[i][0] = l16 ? __ldg(p) : 0ull;
          w[i][1] = bits > 64u ? __ldg(p + 1) : 0ull;
          w[i][2] = bits > 128u ? __ldg(p + 2) : 0ull;
        }
      }
      uint32_t pre[DG_ITERS], wbase;
      round_place(len, s_wtot, pre, wbase);  // (the round's total is Tblk: T <= 32 KB, so every partial sum fits 16 bits)
      round_offsets(out_offs, a.m, base, r0, rows_here, cta_begin, Tblk, wbase, pre, len, limit, err);
      if (out_data != nullptr) {
        const uint32_t A = (uint32_t)((uintptr_t)(out_data + cta_begin) & 15);
#pragma unroll
        for (int i = 0; i < DG_ITERS; ++i) {
          const uint32_t l16 = len[i] > 16u ? 16u : len[i];
          // 16 source bytes from the three aligned words, zero beyond the row
          uint64_t lo = (w[i][0] >> sh[i]) | ((w[i][1] << 1) << (63u - sh[i]));
          uint64_t hi = (w[i][1] >> sh[i]) | ((w[i][2] << 1) << (63u - sh[i]));
          const uint32_t n0 = l16 < 8u ? l16 : 8u, n1 = l16 - n0;
          lo &= n0 >= 8u ? ~0ull : ((1ull << (n0 * 8u)) - 1ull);
          hi &= n1 >= 8u ? ~0ull : ((1ull << (n1 * 8u)) - 1ull);
          const uint32_t ex = (uint32_t)lo, ey = (uint32_t)(lo >> 32), ez = (uint32_t)hi, ew = (uint32_t)(hi >> 32);
          const uint32_t d = A + wbase + pre[i];
          const uint32_t dsh = (d & 3u) * 8u;
          const uint32_t wa = img + (d & ~3u);
          red_or<0>(wa, ex << dsh);
          red_or<4>(wa, __funnelshift_l(ex, ey, dsh));
          red_or<8>(wa, __funnelshift_l(ey, ez, dsh));
          const uint32_t x3 = __funnelshift_l(ez, ew, dsh), x4 = __funnelshift_l(ew, 0u, dsh);
          if (__any_sync(ACU_FULL_MASK, (x3 | x4) != 0u)) {
            red_or<12>(wa, x3);
            red_or<16>(wa, x4);
          }
          // the rest of a long row, 8 bytes at a time
          for (uint32_t c = 16; c < len[i]; c += 8) {
            const uint32_t nb = len[i] - c < 8u ? len[i] - c : 8u;
            const uint64_t v = load_upto8(data, (int64_t)sc[i] + c, nb);
            const uint32_t dd = d + c;
            const uint32_t ds2 = (dd & 3u) * 8u;
            const uint32_t w2 = img + (dd & ~3u);
            const uint32_t vx = (uint32_t)v, vy = (uint32_t)(v >> 32);
            red_or<0>(w2, vx << ds2);
            red_or<4>(w2, __funnelshift_l(vx, vy, ds2));
            red_or<8>(w2, __funnelshift_l(vy, 0u, ds2));
          }
        }
        image_flush(img4, out_data, cta_begin, A, Tblk);
      }
      __syncthreads();
    } else {
      // ---- a block of long rows: 64-bit scans, direct copies (correct for any length; rows average > 16 bytes here) ----
      unsigned long long pre64[DG_ITERS], run = 0;
#pragma unroll
      for (int i = 0; i < DG_ITERS; ++i) {
        unsigned long long inc = len[i];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned long long y = __shfl_up_sync(ACU_FULL_MASK, inc, o);
          if (lane >= (uint32_t)o) inc += y;
        }
        pre64[i] = run + inc - len[i];
        run += __shfl_sync(ACU_FULL_MASK, inc, 31);
      }
      if (lane == 0) s_wtot64[wid] = run;
      __syncthreads();
      unsigned long long wbase = 0;
      for (uint32_t w2 = 0; w2 < wid; ++w2) wbase += s_wtot64[w2];
      const int64_t o0 = cta_begin + (int64_t)wbase;
#pragma unroll
      for (int i = 0; i < DG_ITERS; ++i) {
        if (r0 + i * 32 < rows_here) {
          const int64_t start = o0 + (int64_t)pre64[i];
          out_offs[base + r0 + i * 32] = (int32_t)start;
          if (start + (int64_t)len[i] > limit && (unsigned long long)(base + r0 + i * 32) < err) err = (unsigned long long)(base + r0 + i * 32);
          if (r0 + i * 32 + 1 == rows_here && base + rows_here == a.m) out_offs[a.m] = (int32_t)(start + (int64_t)len[i]);
          if (out_data != nullptr && len[i]) copy_row_direct(out_data + start, data, (int64_t)sc[i], (uint64_t)len[i]);
        }
      }
      __syncthreads();
    }
  }
  if (err != ~0ull) atomicMin(res + RES_ERR2, err);
}

// lengths -> CTA totals -> scan -> offsets (+ byte copy when out_data != NULL and it fits), queued
// on the ctx stream without synchronising; gather_finalize reads the fetched result block:
// RES_ERR_INDEX = lowest out-of-bounds row (detect_oob), RES_AUX0 = total value bytes,
// RES_ERR2 = lowest row whose running total exceeds the offset type.
size_t gather_block_bytes(int64_t m) {
  const int64_t blocks = (m + BY_ROWS - 1) / BY_ROWS;
  return (((size_t)(2 * blocks + blocks / SCAN_ELEMS + 4096) * 8) + 255) & ~(size_t)255;
}
// block totals / scan scratch + the dictionary table of the small-source path (16-byte entries, length bytes, flag)
size_t gather_scratch_bytes(int64_t m) { return gather_block_bytes(m) + (size_t)DG_MAX_ENTRIES * 17 + 256; }

// Grid of a round kernel with `smem` bytes of dynamic shared memory: one CTA per 2048-row block, at most as many as are
// resident at once (a CTA loops over blocks). The dictionary kernel's shared memory depends on the source's size.
template <class K>
acu_status round_grid(acu_ctx *ctx, K kernel, size_t smem, int64_t blocks, int *grid) {
  ACU_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int per_sm = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, DG_THREADS, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  *grid = acu_grid(ctx, blocks, per_sm);
  return ACU_OK;
}

acu_status gather_launch(acu_ctx *ctx, int32_t ob, const void *offsets, const uint8_t *data, const void *idx, int kind,
                         int64_t m, int64_t n_src, const uint8_t *out_valid, bool detect_oob, void *out_offsets,
                         uint8_t *out_data, int64_t out_cap, void *scratch, unsigned long long *res, acu_bytes_col_state *gs) {
  const int64_t blocks = (m + BY_ROWS - 1) / BY_ROWS;
  int64_t *block_tot = static_cast<int64_t *>(scratch);
  BytesArgs a{offsets, data, idx, kind, (int)ob, m, n_src, reinterpret_cast<const uint32_t *>(out_valid), detect_oob ? 1 : 0};
  // pass 1 of the fast kernels reads four indices as one 128-bit load
  const bool fast = ob == 4 && kind == 4 && ((uintptr_t)idx % 16 == 0);
  const int64_t limit = ob == 4 ? (int64_t)INT32_MAX : INT64_MAX;
  gs->gathered = true;
  gs->ob = ob;
  gs->kind = kind;
  gs->offsets = offsets;
  gs->idx = idx;
  gs->data = data;
  gs->out_valid = out_valid;
  gs->m = m;
  gs->n_src = n_src;
  gs->detect_oob = detect_oob;
  gs->block_tot = block_tot;
  gs->out_offsets = out_offsets;
  gs->out_data = out_data;
  gs->out_cap = out_cap;
  // small source (a dictionary): table in shared memory, see k_dict_copy
  if (fast && n_src <= DG_MAX_ENTRIES && n_src > 0 && m >= 65536) {
    uint8_t *extra = static_cast<uint8_t *>(scratch) + gather_block_bytes(m);
    uint4 *table = reinterpret_cast<uint4 *>(extra);
    uint8_t *lens = extra + (size_t)DG_MAX_ENTRIES * 16;
    int *flag = reinterpret_cast<int *>(extra + (size_t)DG_MAX_ENTRIES * 17);
    ACU_CUDA(ctx, cudaMemsetAsync(flag, 0, 4, ctx->stream));
    ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_dict_table, (unsigned)((n_src + 255) / 256), 256, 0, static_cast<const int32_t *>(offsets), data, n_src, table, lens, flag);
    int too_long = 0;
    ACU_CUDA(ctx, cudaMemcpyAsync(&too_long, flag, 4, cudaMemcpyDeviceToHost, ctx->stream));
    ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // entries longer than 16 bytes: the generic kernels below
    if (!too_long) {
      DictArgs da{static_cast<const uint32_t *>(idx), m, (uint32_t)n_src, reinterpret_cast<const uint32_t *>(out_valid), detect_oob ? 1 : 0, table, lens, flag};
      const size_t smem1 = (size_t)n_src, smem2 = ((size_t)n_src + 1) * 16 + (((size_t)n_src + 16) & ~(size_t)15) + DG_IMG_BYTES;
      int g2 = 0;
      ACU_TRY(round_grid(ctx, k_dict_copy, smem2, blocks, &g2));
      const int g1 = acu_grid(ctx, (blocks + DG_WARPS - 1) / DG_WARPS, 4);
      ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_dict_block_totals, g1, DG_THREADS, smem1, da, blocks, block_tot, res);
      ACU_TRY(scan_inclusive(ctx, block_tot, blocks, block_tot + blocks));
      ACU_CUDA(ctx, cudaMemcpyAsync(res + RES_AUX0, block_tot + (blocks - 1), 8, cudaMemcpyDeviceToDevice, ctx->stream));
      da.detect_oob = 0;
      ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_dict_copy, g2, DG_THREADS, smem2, da, block_tot, blocks, static_cast<int32_t *>(out_offsets), out_data, limit, res,
                       block_tot + (blocks - 1), out_cap);
      return ACU_OK;
    }
  }
  if (fast) ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_bytes_block_totals<GatherRows<true>>, (unsigned)blocks, BY_THREADS, 0, GatherRows<true>{a}, block_tot, res);
  else ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_bytes_block_totals<GatherRows<false>>, (unsigned)blocks, BY_THREADS, 0, GatherRows<false>{a}, block_tot, res);
  ACU_TRY(scan_inclusive(ctx, block_tot, blocks, block_tot + blocks));
  ACU_CUDA(ctx, cudaMemcpyAsync(res + RES_AUX0, block_tot + (blocks - 1), 8, cudaMemcpyDeviceToDevice, ctx->stream));
  a.detect_oob = 0;
  if (fast) {
    const size_t smem = GC_IMG_BYTES + 32;
    int grid = 0;
    ACU_TRY(round_grid(ctx, k_gather_copy, smem, blocks, &grid));
    ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_gather_copy, grid, DG_THREADS, smem, a, block_tot, blocks, static_cast<int32_t *>(out_offsets), out_data, limit, res,
                     block_tot + (blocks - 1), out_cap);
  } else {
    const int stage_cap = BY_STAGE_CAP;
    ACU_CUDA(ctx, cudaFuncSetAttribute(k_bytes_offsets_copy<GatherRows<false>>, cudaFuncAttributeMaxDynamicSharedMemorySize, stage_cap));
    ACU_LAUNCH_TIMED(ctx, ACU_K_BYTES, k_bytes_offsets_copy<GatherRows<false>>, (unsigned)blocks, BY_THREADS, stage_cap, GatherRows<false>{a}, block_tot, (int64_t)0, out_offsets,
                     out_data, limit, (int64_t)-1, res, stage_cap, block_tot + (blocks - 1), out_cap);
  }
  return ACU_OK;
}

// *oob_row >= 0: an out-of-bounds index at a valid slot (the caller raises the panic status).
acu_status gather_finalize(acu_ctx *ctx, const acu_bytes_col_state &gs, const unsigned long long *hres, int64_t *out_len, int64_t *oob_row) {
  if (oob_row) *oob_row = -1;
  if (gs.detect_oob && hres[RES_ERR_INDEX] != ~0ull) {
    if (oob_row) *oob_row = (int64_t)hres[RES_ERR_INDEX];
    return ACU_OK;
  }
  *out_len = (int64_t)hres[RES_AUX0];
  if (hres[RES_ERR2] != ~0ull) {  // T::Offset::from_usize(capacity) failed (take.rs:520-523)
    const int64_t j = (int64_t)hres[RES_ERR2];
    const BytesArgs a{gs.offsets, gs.data, gs.idx, gs.kind, (int)gs.ob, gs.m, gs.n_src, reinterpret_cast<const uint32_t *>(gs.out_valid), 0};
    ACU_TRY(acu_res_reset(ctx));
    ACU_LAUNCH(ctx, k_bytes_offsets_copy<GatherRows<false>>, 1, BY_THREADS, 0, GatherRows<false>{a}, gs.block_tot, j / BY_ROWS, gs.out_offsets, static_cast<uint8_t *>(nullptr),
               INT64_MAX, j, ctx->d_res, 0, static_cast<const int64_t *>(nullptr), (int64_t)0);
    ACU_TRY(acu_res_fetch(ctx));
    const long long cap = (long long)ctx->h_res[RES_AUX1];
    if (gs.extend)  // try_extend_offsets (arrow-data/src/transform/utils.rs)
      return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, j, 0, 0, (uint64_t)cap, "%s", acu_extend_overflow_text);
    return acu_fail(ctx, ACU_ERR_OFFSET_OVERFLOW, j, 0, 0, (uint64_t)cap, "%lld", cap);
  }
  if (gs.out_data && *out_len > gs.out_cap)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, (uint64_t)*out_len,
                    "output data capacity %lld < required %lld", (long long)gs.out_cap, (long long)*out_len);
  return ACU_OK;
}

// Every kernel reads and writes offsets as whole ob-byte words (ob already checked to be 4 or 8).
acu_status offsets_aligned(acu_ctx *ctx, int32_t ob, const void *offsets, const void *out_offsets) {
  if (((uintptr_t)offsets | (uintptr_t)out_offsets) % (uintptr_t)ob != 0)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "offsets must be %d-byte aligned", (int)ob);
  return ACU_OK;
}

acu_status zero_first_offset(acu_ctx *ctx, void *out_offsets, int ob) {
  ACU_CUDA(ctx, cudaMemsetAsync(out_offsets, 0, (size_t)ob, ctx->stream));
  return ACU_OK;
}

}  // namespace

// In-place inclusive scan of n int64 values on the ctx stream (views.cu); tmp holds >= n / 4096 + n / 4096^2 + 4 values.
acu_status acu_scan_inclusive_i64(acu_ctx *ctx, int64_t *data, int64_t n, int64_t *tmp) { return scan_inclusive(ctx, data, n, tmp); }


extern "C" acu_status acu_filter_plan_indices(acu_ctx *ctx, const acu_filter_plan *plan, acu_dtype index_dtype,
                                              void *out_indices) {
  ACU_ENTER(ctx);
  if (index_dtype != ACU_U32 && index_dtype != ACU_U64)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "plan indices must be UInt32 or UInt64");
  if (index_dtype == ACU_U32 && acu_filter_plan_len(plan) > (int64_t)UINT32_MAX)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "predicate too long for UInt32 indices");
  if (acu_filter_plan_count(plan) == 0) return ACU_OK;
  const int64_t nwp = acu_plan_n_words_padded(plan);
  const int grid = acu_grid(ctx, (nwp / 32 + 7) / 8, 8);
  if (index_dtype == ACU_U32)
    ACU_LAUNCH_TIMED(ctx, ACU_K_FILTER_PLAN, k_plan_indices<uint32_t>, grid, 256, 0, acu_plan_mask(plan), acu_plan_tile_off(plan),
                     nwp, static_cast<uint32_t *>(out_indices));
  else
    ACU_LAUNCH_TIMED(ctx, ACU_K_FILTER_PLAN, k_plan_indices<uint64_t>, grid, 256, 0, acu_plan_mask(plan), acu_plan_tile_off(plan),
                     nwp, static_cast<uint64_t *>(out_indices));
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  acu_kstats_drain(ctx);
  return ACU_OK;
}

// ---- IterationStrategy::Slices (FilterBuilder::optimize, filter.rs:285-298) = SlicesIterator (filter.rs:44-77) --------------
// Runs of selected rows as [start, end) pairs in ascending order. A run starts at a set bit whose predecessor is clear and
// ends after a set bit whose successor is clear; both are word-local tests once the neighbouring word's edge bit is known
// (the plan's mask is normalised to bit offset 0 and zero padded). The k-th start and the k-th end belong to the same run,
// so two independent scans of the per-word counts place them.
__global__ void __launch_bounds__(256) k_plan_slice_counts(const uint64_t *__restrict__ mask, int64_t n_words, int64_t *__restrict__ n_starts,
                                                           int64_t *__restrict__ n_ends) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += stride) {
    const uint64_t m = __ldg(mask + i);
    const uint64_t prev = i ? (__ldg(mask + i - 1) >> 63) : 0ull, next = i + 1 < n_words ? (__ldg(mask + i + 1) & 1ull) : 0ull;
    n_starts[i] = __popcll(m & ~((m << 1) | prev));
    n_ends[i] = __popcll(m & ~((m >> 1) | (next << 63)));
  }
}

__global__ void __launch_bounds__(256) k_plan_slices_emit(const uint64_t *__restrict__ mask, int64_t n_words, const int64_t *__restrict__ incl_starts,
                                                          const int64_t *__restrict__ incl_ends, int64_t capacity, uint64_t *__restrict__ out_pairs) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += stride) {
    const uint64_t m = __ldg(mask + i);
    if (!m) continue;
    const uint64_t prev = i ? (__ldg(mask + i - 1) >> 63) : 0ull, next = i + 1 < n_words ? (__ldg(mask + i + 1) & 1ull) : 0ull;
    uint64_t st = m & ~((m << 1) | prev), en = m & ~((m >> 1) | (next << 63));
    int64_t ks = incl_starts[i] - __popcll(st), ke = incl_ends[i] - __popcll(en);
    for (; st; st &= st - 1, ++ks)
      if (ks < capacity) out_pairs[2 * ks] = (uint64_t)(i << 6) + (uint64_t)(__ffsll((long long)st) - 1);
    for (; en; en &= en - 1, ++ke)
      if (ke < capacity) out_pairs[2 * ke + 1] = (uint64_t)(i << 6) + (uint64_t)__ffsll((long long)en);
  }
}

extern "C" acu_status acu_filter_plan_slices(acu_ctx *ctx, const acu_filter_plan *plan, uint64_t *out_pairs, int64_t capacity,
                                             int64_t *out_slices) {
  ACU_ENTER(ctx);
  *out_slices = 0;
  if (acu_filter_plan_len(plan) == 0 || acu_filter_plan_count(plan) == 0) return ACU_OK;
  const int64_t n_words = acu_plan_n_words_padded(plan);
  void *scratch;
  const size_t one = ((size_t)n_words + (size_t)n_words / 4096 + 64) * 8;
  ACU_TRY(acu_scratch(ctx, 3 * one, &scratch));
  int64_t *ns = static_cast<int64_t *>(scratch), *ne = ns + one / 8, *tmp = ne + one / 8;
  const int grid = acu_grid(ctx, (n_words + 255) / 256, 8);
  ACU_LAUNCH(ctx, k_plan_slice_counts, grid, 256, 0, acu_plan_mask(plan), n_words, ns, ne);
  ACU_TRY(scan_inclusive(ctx, ns, n_words, tmp));
  ACU_TRY(scan_inclusive(ctx, ne, n_words, tmp));
  int64_t total = 0;
  ACU_CUDA(ctx, cudaMemcpyAsync(&total, ns + (n_words - 1), 8, cudaMemcpyDeviceToHost, ctx->stream));
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  *out_slices = total;
  if (out_pairs == nullptr || total == 0) return ACU_OK;  // sizing call
  if (capacity < total)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, (uint64_t)total, "filter_plan_slices: capacity %lld < %lld slices", (long long)capacity,
                    (long long)total);
  ACU_LAUNCH_TIMED(ctx, ACU_K_FILTER_PLAN, k_plan_slices_emit, grid, 256, 0, acu_plan_mask(plan), n_words, ns, ne, capacity, out_pairs);
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  acu_kstats_drain(ctx);
  return ACU_OK;
}

// The selected row ids of a plan (the reference's IterationStrategy::Indices, filter.rs:285-298), materialised once per
// plan and shared by every variable-width column filtered with it: UInt32 when the predicate is short enough, else UInt64.
acu_status acu_plan_cached_indices(acu_ctx *ctx, const acu_filter_plan *plan, const void **out_idx, int *out_kind) {
  void **slot = acu_plan_index_cache(plan);
  const bool narrow = acu_filter_plan_len(plan) <= (int64_t)UINT32_MAX;
  *out_kind = narrow ? 4 : 5;
  if (*slot == nullptr) {
    void *mem = nullptr;
    ACU_TRY(acu_malloc(ctx, (size_t)acu_filter_plan_count(plan) * (narrow ? 4 : 8), &mem));
    const int64_t nwp = acu_plan_n_words_padded(plan);
    const int grid = acu_grid(ctx, (nwp / 32 + 7) / 8, 8);
    if (narrow)
      ACU_LAUNCH_TIMED(ctx, ACU_K_FILTER_PLAN, k_plan_indices<uint32_t>, grid, 256, 0, acu_plan_mask(plan), acu_plan_tile_off(plan), nwp,
                       static_cast<uint32_t *>(mem));
    else
      ACU_LAUNCH_TIMED(ctx, ACU_K_FILTER_PLAN, k_plan_indices<uint64_t>, grid, 256, 0, acu_plan_mask(plan), acu_plan_tile_off(plan), nwp,
                       static_cast<uint64_t *>(mem));
    *slot = mem;
  }
  *out_idx = *slot;
  return ACU_OK;
}

size_t acu_bytes_col_scratch(int64_t out_rows) { return gather_scratch_bytes(out_rows); }

// ---- one variable-width column of take / take_record_batch ------------------------------------
acu_status acu_take_bytes_col_launch(acu_ctx *ctx, int32_t ob, const void *offsets, const uint8_t *data, const acu_array *nulls_of,
                                     bool val_nulls, const acu_array *indices, acu_dtype index_dtype, bool idx_nulls,
                                     void *out_offsets, uint8_t *out_data, int64_t out_cap, acu_array_out *out_nulls, void *scratch,
                                     unsigned long long *res, acu_bytes_col_state *st, bool extend) {
  *st = acu_bytes_col_state();
  st->extend = extend;
  ACU_TRY(acu_offset_width_check(ctx, ob));
  ACU_TRY(offsets_aligned(ctx, ob, offsets, out_offsets));
  const int64_t m = indices->len;
  out_nulls->len = m;
  out_nulls->has_validity = 0;
  out_nulls->null_count = 0;
  if (m == 0) return zero_first_offset(ctx, out_offsets, ob);
  const uint8_t *ov = nullptr;
  if (val_nulls) {
    if (!extend) ov = out_nulls->validity;  // take_bits(values.nulls), gathered by acu_take_cols_launch
  } else if (indices->validity) {
    // values without nulls: take_nulls = indices.nulls().cloned() (take.rs:429) is a bitmap copy, and the
    // out-of-bounds check rides in the first bytes pass — no separate gather pass.
    ACU_TRY(acu_bitmap_and_launch(ctx, indices->validity, indices->validity_offset, nullptr, 0, m,
                                  reinterpret_cast<uint64_t *>(out_nulls->validity), true, res));
    st->idx_nulls_copied = true;
    if (idx_nulls) ov = out_nulls->validity;
  }
  // with value nulls the take kernel of the validity gather reports an out-of-bounds index
  return gather_launch(ctx, ob, offsets, data, indices->values, acu_take_index_kind(index_dtype), m, nulls_of->len, ov, !val_nulls, out_offsets,
                       out_data, out_cap, scratch, res, st);
}

acu_status acu_take_bytes_col_finalize(acu_ctx *ctx, const acu_array *nulls_of, const acu_array *indices, acu_dtype index_dtype,
                                       const acu_bytes_col_state *st, const unsigned long long *hres, int64_t *out_data_len,
                                       acu_array_out *out_nulls) {
  *out_data_len = 0;
  const int64_t m = indices->len;
  if (!st->gathered) return ACU_OK;
  int64_t oob_row = -1;
  ACU_TRY(gather_finalize(ctx, *st, hres, out_data_len, &oob_row));
  if (oob_row >= 0) {  // the reference panics on a bounds-checked slice index (take.rs:517)
    uint64_t raw = 0;
    const int sz = acu_dtype_size(index_dtype);
    ACU_TRY(acu_memcpy_d2h(ctx, &raw, static_cast<const uint8_t *>(indices->values) + (size_t)oob_row * sz, sz));
    uint64_t widened = raw;
    if (index_dtype == ACU_I8) widened = (uint32_t)(int32_t)(int8_t)raw;
    else if (index_dtype == ACU_I16) widened = (uint32_t)(int32_t)(int16_t)raw;
    else if (index_dtype == ACU_I32) widened = (uint32_t)raw;
    return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, oob_row, widened, 0, (uint64_t)nulls_of->len, "Out-of-bounds index %llu",
                    (unsigned long long)widened);
  }
  if (st->idx_nulls_copied) {
    out_nulls->has_validity = 1;
    out_nulls->null_count = m - (int64_t)hres[RES_COUNT];
  }
  return ACU_OK;
}

// ---- one variable-width column of filter / filter_record_batch ---------------------------------
acu_status acu_filter_bytes_col_launch(acu_ctx *ctx, const acu_filter_plan *plan, int32_t ob, const void *offsets, const uint8_t *data,
                                       const acu_array *nulls_of, void *out_offsets, uint8_t *out_data, int64_t out_cap, void *scratch,
                                       unsigned long long *res, acu_bytes_col_state *st) {
  *st = acu_bytes_col_state();
  ACU_TRY(acu_offset_width_check(ctx, ob));
  ACU_TRY(offsets_aligned(ctx, ob, offsets, out_offsets));
  const int64_t count = acu_filter_plan_count(plan);
  if (count == 0) return zero_first_offset(ctx, out_offsets, ob);
  const void *idx;
  int kind;
  ACU_TRY(acu_plan_cached_indices(ctx, plan, &idx, &kind));
  // null slots are copied too (filter.rs:891-892): no output-validity masking of the lengths
  return gather_launch(ctx, ob, offsets, data, idx, kind, count, nulls_of->len, nullptr, false, out_offsets, out_data, out_cap, scratch,
                       res, st);
}

acu_status acu_filter_bytes_col_finalize(acu_ctx *ctx, const acu_bytes_col_state *st, const unsigned long long *hres,
                                         int64_t *out_data_len) {
  *out_data_len = 0;
  if (!st->gathered) return ACU_OK;
  return gather_finalize(ctx, *st, hres, out_data_len, nullptr);
}
