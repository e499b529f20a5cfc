// compact.cu — arrow-select/src/filter.rs on the device (stream compaction).
//
//   FilterBuilder::new/optimize/build  (filter.rs:254-324)  -> acu_filter_plan_create
//   FilterPredicate::filter            (filter.rs:449-452)  -> acu_filter_primitive / _boolean
//   filter_native / filter_bits / filter_nulls (filter.rs:512-533, :680-788)
//
// Design (HBM-bound):
//   plan:     one pass over the predicate bits (N/8 bytes): mask = values & validity
//             normalised to bit offset 0, popcount per 1024-row tile, two-level exclusive scan
//             -> tile_off[t] = first output row of tile t (u64). The plan is reused by every
//             column of a RecordBatch (FilterPredicate::filter_record_batch, filter.rs:459-478).
//   values:   k_filter_fused<W, ALIGNED>: warp-centric, no CTA barrier. A warp owns a 1024-row
//             tile; the NEXT tile's mask words/offsets are prefetched while this tile's values
//             are in flight. Each lane owns 16-byte chunks; their loads are PREDICATED on "this
//             chunk holds a selected row", so at low selectivity most 32-B DRAM sectors are never
//             fetched (real traffic < algorithmic bytes), and land in a warp-private shared-memory
//             buffer (cp.async for 16-B aligned values, 8-, 4- or 1-byte loads for zero-copy
//             slices). rank = prefix + popc(mask below) -> stored straight to its final position
//             (neighbouring ranks land in the same sectors and merge in L2). Below 4 % selectivity
//             16-B aligned values go through k_filter_values_async<W>, the same compaction
//             without the validity.
//   validity: at >= 4 % selectivity the same warp compacts the tile's validity bits (software
//             PEXT) in the value pass. Below that, and for boolean VALUES (filter_bits /
//             filter_boolean), k_compress_bits: one lane per 64-bit mask word extracts the
//             selected source bits, a warp scan places them, a warp-private shared-memory
//             window assembles output words (atomicOr only on the two boundary words), and
//             the popcount gives filter_nulls' null count.
#include <vector>

#include "bitmap.cuh"
#include "internal.cuh"

#define TILE_ROWS 1024
#define TILE_WORDS (TILE_ROWS / 64)
#define SCAN_CHUNK 4096  // tiles per scan block

struct acu_filter_plan {
  int64_t len = 0;
  int64_t count = 0;
  int32_t strategy = ACU_FILTER_NONE;
  int64_t n_tiles = 0;
  uint64_t *mask = nullptr;       // n_tiles * TILE_WORDS words padded to a multiple of 32, zero padded
  uint64_t *tile_off = nullptr;   // n_tiles + 1 exclusive output offsets (padded)
  uint32_t *tile_count = nullptr; // scratch of the scan
  uint64_t *chunk_total = nullptr;
  void *storage = nullptr;
  mutable void *index_cache = nullptr;  // selected row ids (u32 / u64), built on first use by a variable-width column
};

namespace {

// ---- plan kernels ----------------------------------------------------------------------
// One lane per mask word; a warp covers two tiles (2 x 16 words).
__global__ void __launch_bounds__(256) k_plan_mask(const uint8_t *__restrict__ pv, int64_t poff,
                                                   const uint8_t *__restrict__ nv, int64_t noff,
                                                   int64_t len, int64_t n_words_padded, uint64_t *__restrict__ mask,
                                                   uint32_t *__restrict__ tile_count, int64_t n_tiles) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t w0 = warp * 32; w0 < n_words_padded; w0 += nwarps * 32) {
    const int64_t w = w0 + lane;
    const int64_t row = w << 6;
    uint64_t m = ld_bits64(pv, poff + row, poff + len);
    if (nv) m &= ld_bits64(nv, noff + row, noff + len);  // prep_null_mask_filter
    mask[w] = m;
    unsigned c = __popcll(m);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) c += __shfl_xor_sync(ACU_FULL_MASK, c, o);  // sum inside each 16-lane half
    const int64_t t = w >> 4;
    if ((lane & 15) == 0 && t < n_tiles) tile_count[t] = c;
  }
}

// Block-wide exclusive scan of up to SCAN_CHUNK tile counts (1024 threads x 4) -> tile_off (chunk-local)
__global__ void __launch_bounds__(1024) k_plan_scan_chunks(const uint32_t *__restrict__ tile_count, int64_t n_tiles,
                                                           uint64_t *__restrict__ tile_off,
                                                           uint64_t *__restrict__ chunk_total) {
  __shared__ uint32_t warp_tot[32];
  const int64_t base = (int64_t)blockIdx.x * SCAN_CHUNK + (int64_t)threadIdx.x * 4;
  uint32_t c[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) c[k] = (base + k < n_tiles) ? tile_count[base + k] : 0u;
  uint32_t mine = c[0] + c[1] + c[2] + c[3];
  uint32_t incl = mine;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    uint32_t y = __shfl_up_sync(ACU_FULL_MASK, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    uint32_t w = warp_tot[lane], wi = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t y = __shfl_up_sync(ACU_FULL_MASK, wi, o);
      if (lane >= o) wi += y;
    }
    warp_tot[lane] = wi - w;  // exclusive
    if (lane == 31) chunk_total[blockIdx.x] = wi;
  }
  __syncthreads();
  uint32_t excl = warp_tot[wid] + incl - mine;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (base + k < n_tiles) tile_off[base + k] = excl;
    excl += c[k];
  }
}

// Single block: exclusive scan of the chunk totals (u64), grand total -> res[RES_COUNT].
__global__ void __launch_bounds__(1024) k_plan_scan_top(uint64_t *__restrict__ chunk_total, int64_t n_chunks,
                                                        unsigned long long *__restrict__ res) {
  __shared__ uint64_t warp_tot[32];
  __shared__ uint64_t carry_s;
  if (threadIdx.x == 0) carry_s = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int64_t base = 0; base < n_chunks; base += 1024) {
    const int64_t i = base + threadIdx.x;
    uint64_t v = i < n_chunks ? chunk_total[i] : 0ull, incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint64_t y = __shfl_up_sync(ACU_FULL_MASK, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    if (wid == 0) {
      uint64_t w = warp_tot[lane], wi = w;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        uint64_t y = __shfl_up_sync(ACU_FULL_MASK, wi, o);
        if (lane >= o) wi += y;
      }
      warp_tot[lane] = wi - w;
    }
    __syncthreads();
    const uint64_t carry = carry_s;
    if (i < n_chunks) chunk_total[i] = carry + warp_tot[wid] + incl - v;
    __syncthreads();
    if (threadIdx.x == 1023) carry_s = carry + warp_tot[31] + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) res[RES_COUNT] = carry_s;
}

// tile_off[t] += chunk offset; tile_off[n_tiles .. padded) = total
__global__ void __launch_bounds__(256) k_plan_finalize(uint64_t *__restrict__ tile_off, int64_t n_tiles, int64_t n_padded,
                                                       const uint64_t *__restrict__ chunk_off,
                                                       const unsigned long long *__restrict__ res) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < n_padded; t += stride)
    tile_off[t] = t < n_tiles ? tile_off[t] + chunk_off[t / SCAN_CHUNK] : res[RES_COUNT];
}

// ---- value compaction ------------------------------------------------------------------
struct FilterArgs {
  const uint8_t *values;
  uint8_t *out;
  const uint64_t *mask;
  const uint64_t *tile_off;
  int64_t n_tiles;
  // fused validity compaction: source validity bitmap (NULL = none: no validity, or it goes through k_compress_bits),
  // its bit offset, the predicate length, the compacted output bitmap (zeroed by the host wrapper) and the result block
  // for the popcount
  const uint8_t *vsrc;
  int64_t voff;
  int64_t vlen;
  uint32_t *vout;
  unsigned long long *res;
};

// Up to BATCH_COLS columns per launch: blockIdx.y selects the column (all columns of a record batch share the plan,
// hence the grid.x size), so a filter_record_batch costs one launch per element width instead of one per column.
constexpr int BATCH_COLS = 8;
struct FilterBatch { FilterArgs col[BATCH_COLS]; };

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// The 16-byte chunk at p of a value buffer whose base is not 16-byte aligned (a zero-copy slice): two 8-byte loads for
// W >= 8, four 4-byte loads for W = 4, byte loads below; each load only when its row is selected (bit e of `bits` =
// row e of the chunk). Unloaded parts are zero.
template <int W>
__device__ __forceinline__ uint4 ld_chunk_unaligned(const uint8_t *p, uint32_t bits) {
  uint4 v;
  if constexpr (W >= 8) {
    const uint64_t *q = reinterpret_cast<const uint64_t *>(p);
    const uint64_t lo = (bits & 1u) ? __ldg(q) : 0ull;
    const uint64_t hi = (bits & (W == 8 ? 2u : 1u)) ? __ldg(q + 1) : 0ull;  // W >= 16: both halves belong to the one row
    v = make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
  } else if constexpr (W == 4) {
    const uint32_t *q = reinterpret_cast<const uint32_t *>(p);
    v.x = (bits & 1u) ? __ldg(q) : 0u;
    v.y = (bits & 2u) ? __ldg(q + 1) : 0u;
    v.z = (bits & 4u) ? __ldg(q + 2) : 0u;
    v.w = (bits & 8u) ? __ldg(q + 3) : 0u;
  } else {
    uint8_t *vb = reinterpret_cast<uint8_t *>(&v);
#pragma unroll
    for (int e = 0; e < 16; ++e) vb[e] = ((bits >> (e / W)) & 1u) ? __ldg(p + e) : (uint8_t)0;
  }
  return v;
}

__device__ __forceinline__ uint64_t pext64_sparse(uint64_t v, uint64_t m, uint32_t cnt) {
  // PEXT(v, m) looping over the RARER kind of selected bit (validity bitmaps are mostly ones).
  const uint64_t ones = m & v, zeros = m & ~v;
  const bool clear_mode = __popcll(zeros) <= __popcll(ones);
  uint64_t it = clear_mode ? zeros : ones, acc = 0;
  while (it) {
    const int b = __ffsll((long long)it) - 1;
    it &= it - 1;
    acc |= 1ull << __popcll(m & ((1ull << b) - 1ull));
  }
  const uint64_t full = cnt == 64 ? ~0ull : ((1ull << cnt) - 1ull);
  return clear_mode ? (full & ~acc) : acc;
}

// A tile is compacted in passes of PASS_BYTES per warp (the landing buffer, 4 KB). Chunk c of a pass
// (c = j*32 + lane) covers rows row_base + j*RPJ + lr, lr = lane*RPC/CPR. For W <= 8 a chunk round spans whole mask
// words, so the word / 32-bit half / bit position of a lane's chunk differ from round to round only by a compile-time
// amount; for W = 16 / 32 a round is a fraction of one word. Everything below is 32-bit arithmetic on 32-bit halves of
// the mask words.
template <int W> struct FilterCfg {
  static constexpr int PASS_BYTES = (TILE_ROWS * W < 4096) ? TILE_ROWS * W : 4096;
  static constexpr int PASS_ROWS = PASS_BYTES / W;
  static constexpr int PASSES = TILE_ROWS / PASS_ROWS;
  static constexpr int CPP = PASS_BYTES / 16;                      // 16-byte chunks per pass
  static constexpr int ITERS = CPP / 32;                           // chunk rounds per pass
  static constexpr int RPC = W <= 16 ? 16 / W : 1;                 // rows per chunk (W = 32: two chunks per row)
  static constexpr int CPR = W <= 16 ? 1 : W / 16;                 // chunks per row
  static constexpr int RPJ = 32 * RPC / CPR;                       // rows per chunk round
  static constexpr uint32_t CHUNK_MASK = RPC == 32 ? 0xffffffffu : ((1u << RPC) - 1u);
};

// k_filter_fused<W, ALIGNED>: filter_native (and, with vsrc set, filter_nulls) of one tile per warp.
// Values: every needed 16-byte chunk of a pass goes in flight into the warp's landing buffer before any is used. With a
// 16-byte aligned values base the loads are cp.async (LDGSTS), which keeps ALL of a pass's sectors in flight without
// holding them in registers, as a latency-bound sparse read needs; a zero-copy slice (ALIGNED = false) loads through
// registers with ld_chunk_unaligned (all of a pass's loads are issued before the first is staged, so a lane holds up to
// 8 chunks: 80 registers, 3 CTAs/SM, without spills). Each lane then ranks and stores the selected elements of its own
// chunks. The mask / rank bookkeeping is strength-reduced to 32-bit operations on lane-constant positions: a lane's
// selection bits of a whole pass are packed into one register at issue time and reused by the consume phase.
// Validity: FilterPredicate::filter_nulls (filter.rs:512-533) is fused in. The warp that owns a tile already holds its
// mask and popcount prefix, so lanes 0..15 PEXT the source validity words with them and OR the bits into the output
// bitmap (zeroed by the host before the launch); the popcount (= the filtered null count) goes to the column's result
// block. The mask is read ONCE for values and validity.
template <int W, bool ALIGNED>
__global__ void __launch_bounds__(256, ALIGNED ? 5 : 3) k_filter_fused(const FilterBatch batch) {
  const FilterArgs &a = batch.col[blockIdx.y];
  using F = FilterCfg<W>;
  constexpr int RPC = F::RPC, CPR = F::CPR, RPJ = F::RPJ;
  static_assert(RPC * F::ITERS <= 32, "the per-pass selection bits of a lane must fit one register");
  extern __shared__ __align__(16) uint8_t s_raw[];
  __shared__ uint32_t s_h[8][2 * TILE_WORDS];   // the tile's mask as 32-bit halves ...
  __shared__ uint32_t s_hp[8][2 * TILE_WORDS];  // ... and the exclusive popcount prefix of every half
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int lr = lane * RPC / CPR;               // lane's row offset inside a chunk round
  const int lr_half = lr >> 5, lr_bit = lr & 31; // (W <= 8: fixed for every round; W >= 16: lr < 32, lr_half = 0)
  uint4 *lbuf = reinterpret_cast<uint4 *>(s_raw + (size_t)wid * F::PASS_BYTES) + lane;  // the lane's slot of round 0
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const uint8_t *__restrict__ vsrc = a.vsrc;
  const bool v_aligned = vsrc && (((uintptr_t)vsrc & 7) == 0) && ((a.voff & 63) == 0);  // validity words are plain aligned u64 loads
  unsigned valid_cnt = 0;

  int64_t t = warp;
  uint64_t m_next = 0, off_next = 0, end_next = 0;
  if (t < a.n_tiles) {
    if (lane < TILE_WORDS) m_next = __ldg(a.mask + t * TILE_WORDS + lane);
    off_next = __ldg(a.tile_off + t);
    end_next = __ldg(a.tile_off + t + 1);
  }
  for (; t < a.n_tiles; t += nwarps) {
    const uint64_t m = m_next, out0 = off_next, cnt = end_next - off_next;
    const int64_t tn = t + nwarps;
    if (tn < a.n_tiles) {
      m_next = (lane < TILE_WORDS) ? __ldg(a.mask + tn * TILE_WORDS + lane) : 0ull;
      off_next = __ldg(a.tile_off + tn);
      end_next = __ldg(a.tile_off + tn + 1);
    }
    if (cnt == 0) continue;  // warp-uniform
    // lane h owns half h of the tile's 32 halves: its popcount prefix is one 32-lane scan
    const uint32_t src_lo = __shfl_sync(ACU_FULL_MASK, (uint32_t)m, lane >> 1);
    const uint32_t src_hi = __shfl_sync(ACU_FULL_MASK, (uint32_t)(m >> 32), lane >> 1);
    const uint32_t hv = (lane & 1) ? src_hi : src_lo;
    const uint32_t hc = __popc(hv);
    uint32_t hincl = hc;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(ACU_FULL_MASK, hincl, o);
      if (lane >= o) hincl += y;
    }
    s_h[wid][lane] = hv;
    s_hp[wid][lane] = hincl - hc;
    // the validity word of the tile goes in flight before the value loads (consumed after them)
    uint64_t v = 0;
    if (vsrc && m) {
      if (v_aligned) v = __ldg(reinterpret_cast<const uint64_t *>(vsrc) + ((a.voff + t * TILE_ROWS) >> 6) + lane);  // bits past vlen: masked by m
      else v = ld_bits64(vsrc, a.voff + t * TILE_ROWS + (int64_t)lane * 64, a.voff + a.vlen);
    }
    __syncwarp();
    const uint8_t *src = a.values + (size_t)t * TILE_ROWS * W;
    uint8_t *dst = a.out + (size_t)out0 * W;
#pragma unroll 1
    for (int pass = 0; pass < F::PASSES; ++pass) {
      const int half_base = (pass * F::PASS_ROWS) >> 5;  // first 32-bit half of the pass
      const uint8_t *psrc = src + ((size_t)pass * F::CPP + lane) * 16;
      asm volatile("" : "+l"(psrc));  // keep the lane's source address in registers: every round is [psrc + immediate]
      const uint32_t *hh = &s_h[wid][half_base + lr_half];
      uint32_t sel = 0;  // RPC selection bits per round, packed
      uint4 x[ALIGNED ? 1 : F::ITERS];  // unaligned loads: registers first, so that all of them are in flight at once
      // ---- issue: every needed chunk of the pass goes in flight (coalesced: lane <-> consecutive 16-byte chunks) ----
#pragma unroll
      for (int j = 0; j < F::ITERS; ++j) {
        const int r0 = j * RPJ;                                  // compile-time row offset of the round inside the pass
        const uint32_t bits = (hh[r0 >> 5] >> ((r0 & 31) + lr_bit)) & F::CHUNK_MASK;
        sel |= bits << (j * RPC);
        if constexpr (ALIGNED) {
          if (bits) cp_async16(lbuf + j * 32, psrc + (size_t)j * 512);
        } else {
          x[j] = ld_chunk_unaligned<W>(psrc + (size_t)j * 512, bits);
        }
      }
      if constexpr (ALIGNED) {
        cp_async_wait_all();
      } else {
#pragma unroll
        for (int j = 0; j < F::ITERS; ++j) lbuf[j * 32] = x[j];
      }
      __syncwarp();
      // ---- consume: rank and store the selected elements (no branch: every store is predicated) ----
      const uint32_t *hp = &s_hp[wid][half_base + lr_half];
#pragma unroll
      for (int j = 0; j < F::ITERS; ++j) {
        const uint32_t bits = (sel >> (j * RPC)) & F::CHUNK_MASK;
        const int r0 = j * RPJ;
        const int sh = (r0 & 31) + lr_bit;
        const uint32_t rank = hp[r0 >> 5] + __popc(hh[r0 >> 5] & ((1u << sh) - 1u));
        const uint4 x = lbuf[j * 32];
        if constexpr (W == 8) {
          uint64_t *o = reinterpret_cast<uint64_t *>(dst) + rank;
          if (bits & 1u) o[0] = (uint64_t)x.x | ((uint64_t)x.y << 32);
          if (bits & 2u) o[bits & 1u] = (uint64_t)x.z | ((uint64_t)x.w << 32);
        } else if constexpr (W == 4) {
          uint32_t *o = reinterpret_cast<uint32_t *>(dst) + rank;
          if (bits & 1u) *o++ = x.x;
          if (bits & 2u) *o++ = x.y;
          if (bits & 4u) *o++ = x.z;
          if (bits & 8u) *o = x.w;
        } else if constexpr (W == 2) {
          uint16_t *o = reinterpret_cast<uint16_t *>(dst) + rank;
          const uint16_t *ve = reinterpret_cast<const uint16_t *>(&x);
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if ((bits >> e) & 1u) *o++ = ve[e];
        } else if constexpr (W == 1) {
          uint8_t *o = dst + rank;
          const uint8_t *ve = reinterpret_cast<const uint8_t *>(&x);
#pragma unroll
          for (int e = 0; e < 16; ++e)
            if ((bits >> e) & 1u) *o++ = ve[e];
        } else {
          if (bits) {
            const int half = lane % CPR;  // (j*32 + lane) % CPR, CPR divides 32
            uint64_t *o = reinterpret_cast<uint64_t *>(dst + (size_t)rank * W + half * 16);
            o[0] = (uint64_t)x.x | ((uint64_t)x.y << 32);
            o[1] = (uint64_t)x.z | ((uint64_t)x.w << 32);
          }
        }
      }
      __syncwarp();  // the landing buffer is reused by the next pass / tile
    }
    // ---- validity: PEXT(source validity, mask) per word; the (<= 3) output words a lane touches are merged with RED.OR ----
    // (fire-and-forget into the zeroed bitmap: no shared-memory window, no warp barriers, no dependent latency)
    if (vsrc) {
      const uint32_t c = __popcll(m);               // lanes >= 16 hold m = 0
      if (c) {
        const uint64_t bits = pext64_sparse(v, m, c);
        valid_cnt += __popcll(bits);
        const uint64_t p = out0 + s_hp[wid][(2 * lane) & 31];  // first output bit of this word's selected rows
        const uint32_t sh = (uint32_t)p & 31u;
        uint32_t *o = a.vout + (p >> 5);
        const uint32_t w0 = (uint32_t)(bits << sh);
        const uint64_t rest = sh ? (bits >> (32u - sh)) : (bits >> 32);
        if (w0) atomicOr(o, w0);
        if ((uint32_t)rest) atomicOr(o + 1, (uint32_t)rest);
        if ((uint32_t)(rest >> 32)) atomicOr(o + 2, (uint32_t)(rest >> 32));
      }
      __syncwarp();  // s_hp is rewritten by the next tile
    }
  }
  if (vsrc && a.res) {
    valid_cnt = warp_sum(valid_cnt);
    if (lane == 0 && valid_cnt) atomicAdd(a.res + RES_COUNT, (unsigned long long)valid_cnt);
  }
}

// k_filter_values_async<W>: the value compaction of k_filter_fused<W, true> without the validity, kept for sparse
// predicates (< 4 % selected) over 16-byte aligned values, where almost no value bytes move: it holds the tile's mask as
// 64-bit words, runs 6 CTAs/SM and sizes its grid to every resident slot. On an H100 it measured faster there than
// k_filter_fused<8, true> without validity: filter i64 at s = 0.001 0.63 against 0.86 ms, at s = 0.01 1.01 against
// 1.19 ms (1e9 rows, plan + value + validity kernels).
template <int W>
__global__ void __launch_bounds__(256, 6) k_filter_values_async(const FilterBatch batch) {
  const FilterArgs &a = batch.col[blockIdx.y];
  using F = FilterCfg<W>;
  constexpr int RPC = F::RPC, CPR = F::CPR, RPJ = F::RPJ;
  extern __shared__ __align__(16) uint8_t s_raw[];
  __shared__ uint64_t s_m[8][TILE_WORDS];   // the tile's mask words ...
  __shared__ uint32_t s_p[8][TILE_WORDS];   // ... and their exclusive popcount prefix (LDS broadcast beats 3 SHFL per round)
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int lr = lane * RPC / CPR;           // lane's row offset inside a chunk round
  uint4 *buf = reinterpret_cast<uint4 *>(s_raw + (size_t)wid * F::PASS_BYTES);
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;

  int64_t t = warp;
  uint64_t m_next = 0, off_next = 0, end_next = 0;
  if (t < a.n_tiles) {
    if (lane < TILE_WORDS) m_next = __ldg(a.mask + t * TILE_WORDS + lane);
    off_next = __ldg(a.tile_off + t);
    end_next = __ldg(a.tile_off + t + 1);
  }
  for (; t < a.n_tiles; t += nwarps) {
    const uint64_t m = m_next, out0 = off_next, cnt = end_next - off_next;
    const int64_t tn = t + nwarps;
    if (tn < a.n_tiles) {
      m_next = (lane < TILE_WORDS) ? __ldg(a.mask + tn * TILE_WORDS + lane) : 0ull;
      off_next = __ldg(a.tile_off + tn);
      end_next = __ldg(a.tile_off + tn + 1);
    }
    if (cnt == 0) continue;
    const uint32_t c = __popcll(m);
    uint32_t incl = c;
#pragma unroll
    for (int o = 1; o < TILE_WORDS; o <<= 1) {
      uint32_t y = __shfl_up_sync(ACU_FULL_MASK, incl, o);
      if (lane >= o) incl += y;
    }
    if (lane < TILE_WORDS) { s_m[wid][lane] = m; s_p[wid][lane] = incl - c; }
    __syncwarp();
    const uint8_t *src = a.values + (size_t)t * TILE_ROWS * W;
    uint8_t *dst = a.out + (size_t)out0 * W;
#pragma unroll 1
    for (int pass = 0; pass < F::PASSES; ++pass) {
      const int row_base = pass * F::PASS_ROWS;
      const uint8_t *psrc = src + ((size_t)pass * F::CPP + lane) * 16;
      // ---- issue: every needed chunk of the pass goes in flight ----
#pragma unroll
      for (int j = 0; j < F::ITERS; ++j) {
        const int r = row_base + j * RPJ + lr;
        const uint32_t bits = (uint32_t)(s_m[wid][r >> 6] >> (r & 63)) & ((1u << RPC) - 1u);
        if (bits) cp_async16(buf + j * 32 + lane, psrc + (size_t)j * 512);
      }
      cp_async_wait_all();
      __syncwarp();
      // ---- consume: rank and store the selected elements ----
#pragma unroll
      for (int j = 0; j < F::ITERS; ++j) {
        const int r = row_base + j * RPJ + lr;
        const uint64_t word = s_m[wid][r >> 6];
        const uint32_t bits = (uint32_t)(word >> (r & 63)) & ((1u << RPC) - 1u);
        if (!bits) continue;
        const uint32_t rank = s_p[wid][r >> 6] + __popcll(word & ((1ull << (r & 63)) - 1ull));
        const uint4 v = buf[j * 32 + lane];
        if constexpr (W == 8) {
          uint64_t *o = reinterpret_cast<uint64_t *>(dst) + rank;
          if (bits & 1u) *o++ = (uint64_t)v.x | ((uint64_t)v.y << 32);
          if (bits & 2u) *o = (uint64_t)v.z | ((uint64_t)v.w << 32);
        } else if constexpr (W == 4) {
          uint32_t *o = reinterpret_cast<uint32_t *>(dst) + rank;
          if (bits & 1u) *o++ = v.x;
          if (bits & 2u) *o++ = v.y;
          if (bits & 4u) *o++ = v.z;
          if (bits & 8u) *o = v.w;
        } else if constexpr (W == 2) {
          uint16_t *o = reinterpret_cast<uint16_t *>(dst) + rank;
          const uint16_t *ve = reinterpret_cast<const uint16_t *>(&v);
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if ((bits >> e) & 1u) *o++ = ve[e];
        } else if constexpr (W == 1) {
          uint8_t *o = dst + rank;
          const uint8_t *ve = reinterpret_cast<const uint8_t *>(&v);
#pragma unroll
          for (int e = 0; e < 16; ++e)
            if ((bits >> e) & 1u) *o++ = ve[e];
        } else {
          const int half = lane % CPR;  // (j*32 + lane) % CPR, CPR divides 32
          uint64_t *o = reinterpret_cast<uint64_t *>(dst + (size_t)rank * W + half * 16);
          o[0] = (uint64_t)v.x | ((uint64_t)v.y << 32);
          o[1] = (uint64_t)v.z | ((uint64_t)v.w << 32);
        }
      }
      __syncwarp();  // the buffers are reused by the next pass / tile
    }
  }
}

// ---- bit compaction (validity / boolean values): software PEXT --------------------------
// One lane per mask word; a warp covers 32 consecutive words (two tiles).
struct CompressArgs {
  const uint8_t *src;       // bitmap to compact (validity or boolean values)
  int64_t soff;             // its bit offset
  uint32_t *out;            // compacted bits (bit offset 0), zeroed by k_zero_outputs
  unsigned long long *res;  // result block for the popcount, or NULL
  uint64_t out_bytes;       // bytes of `out` to zero
  const uint64_t *count_ptr;  // pending plan (async section): the selected-row count is still on the device
};
struct CompressBatch { CompressArgs col[BATCH_COLS]; };

// zero the outputs of a compress batch (the compaction ORs into boundary words)
__global__ void __launch_bounds__(256) k_zero_outputs(const CompressBatch batch) {
  const CompressArgs &c = batch.col[blockIdx.y];
  uint64_t *o = reinterpret_cast<uint64_t *>(c.out);  // bitmaps are whole u64 words (acu_bitmap_bytes)
  const uint64_t words = c.count_ptr ? ((*c.count_ptr + 63) >> 6) : (c.out_bytes >> 3);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (uint64_t)gridDim.x * blockDim.x) o[i] = 0ull;
}
// the same for one bitmap whose length (rows) is read from the device: zeroing the validity output of a fused filter
// whose plan is pending, without touching more than the caller sized for the rows actually selected
__global__ void __launch_bounds__(256) k_zero_bitmap_dev(uint64_t *__restrict__ o, const uint64_t *__restrict__ count_ptr) {
  const uint64_t words = (*count_ptr + 63) >> 6;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < words; i += (uint64_t)gridDim.x * blockDim.x) o[i] = 0ull;
}

__global__ void __launch_bounds__(256, 8) k_compress_bits(const CompressBatch batch, int64_t len, const uint64_t *__restrict__ mask,
                                                       const uint64_t *__restrict__ tile_off, int64_t n_words_padded) {
  const uint8_t *__restrict__ src = batch.col[blockIdx.y].src;
  const int64_t soff = batch.col[blockIdx.y].soff;
  uint32_t *__restrict__ out = batch.col[blockIdx.y].out;
  unsigned long long *__restrict__ res = batch.col[blockIdx.y].res;
  __shared__ uint32_t s_win[8][68];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  unsigned valid_cnt = 0;
  for (int64_t w0 = warp * 32; w0 < n_words_padded; w0 += nwarps * 32) {
    const int64_t w = w0 + lane;
    uint64_t m = __ldg(mask + w);
    const uint32_t cnt = __popcll(m);
    uint32_t incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      uint32_t y = __shfl_up_sync(ACU_FULL_MASK, incl, o);
      if (lane >= o) incl += y;
    }
    const uint32_t total = __shfl_sync(ACU_FULL_MASK, incl, 31);
    if (total == 0) continue;  // warp-uniform
    const uint64_t base = __ldg(tile_off + (w0 >> 4));  // first output bit of this 32-word group
    uint64_t bits = 0;
    if (m) {
      // PEXT(v, m). The loop runs over the RARER kind of selected bit: validity bitmaps are
      // mostly ones, so start from all-ones and clear the (few) selected-and-unset rows; data
      // that is mostly zeros starts from zero and sets. rank(b) = popc(m below bit b).
      const uint64_t v = ld_bits64(src, soff + (w << 6), soff + len);
      const uint64_t ones = m & v, zeros = m & ~v;
      const bool clear_mode = __popcll(zeros) <= __popcll(ones);
      uint64_t it = clear_mode ? zeros : ones, acc = 0;
      while (it) {
        const int b = __ffsll((long long)it) - 1;
        it &= it - 1;
        acc |= 1ull << __popcll(m & ((1ull << b) - 1ull));
      }
      const uint64_t full = cnt == 64 ? ~0ull : ((1ull << cnt) - 1ull);
      bits = clear_mode ? (full & ~acc) : acc;
    }
    valid_cnt += __popcll(bits);
    // assemble in a warp-private window aligned to the first output word
    const uint32_t lead = (uint32_t)(base & 31);
    const uint32_t nwords = (lead + total + 31) >> 5;  // <= 65
    for (uint32_t i = lane; i < nwords; i += 32) s_win[wid][i] = 0;
    __syncwarp();
    if (cnt) {
      const uint32_t p = lead + incl - cnt;  // bit position inside the window
      const uint32_t sh = p & 31;
      atomicOr(&s_win[wid][p >> 5], (uint32_t)(bits << sh));
      if (sh + cnt > 32) {
        const uint64_t rest = bits >> (32 - sh);  // sh == 0 -> bits >> 32
        atomicOr(&s_win[wid][(p >> 5) + 1], (uint32_t)rest);
        if (sh + cnt > 64) atomicOr(&s_win[wid][(p >> 5) + 2], (uint32_t)(rest >> 32));
      }
    }
    __syncwarp();
    uint32_t *o = out + (base >> 5);
    for (uint32_t i = lane; i < nwords; i += 32) {
      const uint32_t word = s_win[wid][i];
      if (i == 0 || i == nwords - 1) { if (word) atomicOr(o + i, word); }  // shared with neighbouring groups
      else o[i] = word;
    }
    __syncwarp();
  }
  if (res) {
    valid_cnt = warp_sum(valid_cnt);
    if (lane == 0 && valid_cnt) atomicAdd(res + RES_COUNT, (unsigned long long)valid_cnt);
  }
}

acu_status check_len(acu_ctx *ctx, const acu_filter_plan *plan, int64_t values_len) {
  if (plan->len > values_len)  // filter.rs:536-542
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, (uint64_t)values_len,
                    "Filter predicate of length %lld is larger than target array of length %lld",
                    (long long)plan->len, (long long)values_len);
  return ACU_OK;
}

bool aligned16(const void *p) { return ((uintptr_t)p % 16) == 0; }

// `fused`: the predicate is dense enough for the value kernel to compact the validity too (fuses_validity)
template <int W>
acu_status launch_filter(acu_ctx *ctx, const FilterBatch &fb, int n_cols, bool fused) {
  const FilterArgs &fa = fb.col[0];  // the columns of a batch share the plan and the values' alignment class
  constexpr size_t smem = 8 * (size_t)FilterCfg<W>::PASS_BYTES;  // 8 warps x per-warp landing buffer
  const bool al = aligned16(fa.values);
  void (*kernel)(const FilterBatch) = !al ? k_filter_fused<W, false> : fused ? k_filter_fused<W, true> : k_filter_values_async<W>;
  if (ctx->occupancy.find(reinterpret_cast<const void *>(kernel)) == ctx->occupancy.end())  // first use on this device
    ACU_CUDA(ctx, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if (al && !fused) {
    const int gx = acu_wave_grid(ctx, kernel, 256, smem, (fa.n_tiles + 7) / 8);
    ACU_LAUNCH_TIMED(ctx, ACU_K_FILTER, kernel, dim3(gx, n_cols), 256, smem, fb);
    return ACU_OK;
  }
  // every warp should own several tiles (the next tile's mask / offsets are prefetched while the current one is in
  // flight): with the columns of a record batch in blockIdx.y the x-grid is divided by the column count
  constexpr int tiles_per_warp = 4;
  const int64_t want = (fa.n_tiles + 8 * (int64_t)tiles_per_warp - 1) / (8 * (int64_t)tiles_per_warp);
  int gx = acu_wave_grid(ctx, kernel, 256, smem, (fa.n_tiles + 7) / 8);
  gx = (gx + n_cols - 1) / n_cols;
  if (gx > want) gx = (int)(want < 1 ? 1 : want);
  ACU_LAUNCH_TIMED(ctx, ACU_K_FILTER, kernel, dim3(gx, n_cols), 256, smem, fb);
  return ACU_OK;
}

acu_status launch_filter_width(acu_ctx *ctx, int32_t elem_bytes, const FilterBatch &fb, int n_cols, bool fused) {
  switch (elem_bytes) {
    case 1: return launch_filter<1>(ctx, fb, n_cols, fused);
    case 2: return launch_filter<2>(ctx, fb, n_cols, fused);
    case 4: return launch_filter<4>(ctx, fb, n_cols, fused);
    case 8: return launch_filter<8>(ctx, fb, n_cols, fused);
    case 16: return launch_filter<16>(ctx, fb, n_cols, fused);
    case 32: return launch_filter<32>(ctx, fb, n_cols, fused);
    default:
      return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "filter: unsupported element width %d", elem_bytes);
  }
}

// out (zeroed here) = bits of each `src` selected by the plan; optional popcounts into the columns' result blocks.
acu_status launch_compress(acu_ctx *ctx, const acu_filter_plan *plan, const CompressBatch &cb, int n_cols) {
  const int64_t n_words_padded = ((plan->n_tiles * TILE_WORDS + 31) / 32) * 32;
  const int64_t words = (int64_t)acu_bitmap_bytes(plan->count < 0 ? plan->len : plan->count) / 8;
  ACU_LAUNCH(ctx, k_zero_outputs, dim3(acu_grid(ctx, (words + 255) / 256, 4), n_cols), 256, 0, cb);
  const int gx = acu_wave_grid(ctx, k_compress_bits, 256, 0, (n_words_padded / 32 + 7) / 8);
  ACU_LAUNCH_TIMED(ctx, ACU_K_FILTER, k_compress_bits, dim3(gx, n_cols), 256, 0, cb, plan->len, plan->mask, plan->tile_off, n_words_padded);
  return ACU_OK;
}

CompressArgs compress_args(const acu_filter_plan *plan, const uint8_t *src, int64_t soff, void *out, unsigned long long *res) {
  CompressArgs c;
  c.src = src;
  c.soff = soff;
  c.out = static_cast<uint32_t *>(out);
  c.res = res;
  c.out_bytes = acu_bitmap_bytes(plan->count < 0 ? plan->len : plan->count);
  c.count_ptr = plan->count < 0 ? plan->tile_off + plan->n_tiles : nullptr;  // pending (async section): tile_off[n_tiles] = count
  return c;
}

// The value kernel compacts the validity in the same pass unless the predicate is very sparse (< 4 % selected: almost
// no value bytes move, the per-tile validity work dominates and k_compress_bits beside it is faster there; 16-byte
// aligned values then go through k_filter_values_async).
bool fuses_validity(const acu_filter_plan *plan) {
  return plan->count < 0 || plan->count * 25 >= plan->len;  // count < 0: not fetched yet (async section)
}

FilterArgs filter_args(const acu_filter_plan *plan, const acu_array *values, acu_array_out *out, bool has_nulls,
                       unsigned long long *res) {
  FilterArgs fa{};
  fa.values = static_cast<const uint8_t *>(values->values);
  fa.out = static_cast<uint8_t *>(out->values);
  fa.mask = plan->mask;
  fa.tile_off = plan->tile_off;
  fa.n_tiles = plan->n_tiles;
  if (has_nulls && fuses_validity(plan)) {  // FilterPredicate::filter_nulls in the same pass (filter.rs:512-533)
    fa.vsrc = values->validity;
    fa.voff = values->validity_offset;
    fa.vlen = plan->len;
    fa.vout = reinterpret_cast<uint32_t *>(out->validity);
    fa.res = res;
  }
  return fa;
}

}  // namespace

extern "C" {

// Allocate the plan's device storage for a predicate of `len` rows.
static acu_status plan_alloc(acu_ctx *ctx, int64_t len, acu_filter_plan **out_plan) {
  acu_filter_plan *plan = new acu_filter_plan();
  plan->len = len;
  *out_plan = plan;
  if (len == 0) return ACU_OK;
  const int64_t n_tiles = (len + TILE_ROWS - 1) / TILE_ROWS;
  const int64_t n_chunks = (n_tiles + SCAN_CHUNK - 1) / SCAN_CHUNK;
  const int64_t n_words_padded = ((n_tiles * TILE_WORDS + 31) / 32) * 32;
  const int64_t n_off_padded = n_words_padded / TILE_WORDS + 2;
  plan->n_tiles = n_tiles;
  auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
  const size_t mask_b = up((size_t)n_words_padded * 8), off_b = up((size_t)n_off_padded * 8),
               cnt_b = up((size_t)n_tiles * 4), ch_b = up((size_t)n_chunks * 8);
  void *mem = nullptr;
  acu_status st = acu_malloc(ctx, mask_b + off_b + cnt_b + ch_b, &mem);
  if (st != ACU_OK) { delete plan; *out_plan = nullptr; return st; }
  uint8_t *p = static_cast<uint8_t *>(mem);
  plan->storage = mem;
  plan->mask = reinterpret_cast<uint64_t *>(p);
  plan->tile_off = reinterpret_cast<uint64_t *>(p + mask_b);
  plan->tile_count = reinterpret_cast<uint32_t *>(p + mask_b + off_b);
  plan->chunk_total = reinterpret_cast<uint64_t *>(p + mask_b + off_b + cnt_b);
  return ACU_OK;
}

// mask + tile_count are queued on the stream: scan them into tile offsets, fetch the count, pick the strategy.
static acu_status plan_finish(acu_ctx *ctx, acu_filter_plan *plan, int kslot, int blk) {
  const int64_t len = plan->len, n_tiles = plan->n_tiles;
  const int64_t n_chunks = (n_tiles + SCAN_CHUNK - 1) / SCAN_CHUNK;
  const int64_t n_words_padded = ((n_tiles * TILE_WORDS + 31) / 32) * 32;
  const int64_t n_off_padded = n_words_padded / TILE_WORDS + 2;
  unsigned long long *res = acu_dres(ctx, blk);
  k_plan_scan_chunks<<<(unsigned)n_chunks, 1024, 0, ctx->stream>>>(plan->tile_count, n_tiles, plan->tile_off, plan->chunk_total);
  k_plan_scan_top<<<1, 1024, 0, ctx->stream>>>(plan->chunk_total, n_chunks, res);
  k_plan_finalize<<<acu_grid(ctx, (n_off_padded + 255) / 256, 8), 256, 0, ctx->stream>>>(plan->tile_off, n_tiles, n_off_padded,
                                                                                     plan->chunk_total, res);
  if (kslot >= 0) acu_kstats_end(ctx, kslot);
  ctx->launches += 3;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return acu_cuda_fail(ctx, e, "filter plan kernels");
  // inside an async section the count stays on the device until acu_results_fetch: the plan is usable at once (the value
  // kernels read tile_off on the device), count / strategy are filled in by the finaliser
  plan->count = -1;
  plan->strategy = ACU_FILTER_INDEX;
  return acu_call_end(ctx, blk, [plan, len](const unsigned long long *h) -> acu_status {
    plan->count = (int64_t)h[RES_COUNT];
    // IterationStrategy::default_strategy (filter.rs:346-364)
    if (plan->count == 0) plan->strategy = ACU_FILTER_NONE;
    else if (plan->count == len) plan->strategy = ACU_FILTER_ALL;
    else if ((double)plan->count / (double)len > 0.8) plan->strategy = ACU_FILTER_SLICES;
    else plan->strategy = ACU_FILTER_INDEX;
    return ACU_OK;
  });
}

acu_status acu_filter_plan_create(acu_ctx *ctx, const acu_array *pred, acu_filter_plan **out_plan) {
  *out_plan = nullptr;
  ACU_ENTER(ctx);
  const int64_t len = pred->len;
  acu_status st = ACU_OK;
  int64_t nc = 0;
  if (len > 0) {
    nc = acu_resolve_null_count(ctx, pred, &st);
    ACU_TRY(st);
  }
  acu_filter_plan *plan = nullptr;
  ACU_TRY(plan_alloc(ctx, len, &plan));
  if (len == 0) { *out_plan = plan; return ACU_OK; }
  auto bail = [&](acu_status s) { acu_free(ctx, plan->storage); delete plan; return s; };
  const int64_t n_words_padded = ((plan->n_tiles * TILE_WORDS + 31) / 32) * 32;
  const uint8_t *nv = (pred->validity && nc > 0) ? pred->validity : nullptr;  // filter.rs:261-264
  const int blk = acu_call_begin(ctx, &st);
  if (st != ACU_OK) return bail(st);
  const int slot = acu_kstats_begin(ctx, ACU_K_FILTER_PLAN);
  k_plan_mask<<<acu_grid(ctx, (n_words_padded / 32 + 7) / 8, 8), 256, 0, ctx->stream>>>(
      static_cast<const uint8_t *>(pred->values), pred->values_offset, nv, pred->validity_offset, len, n_words_padded,
      plan->mask, plan->tile_count, plan->n_tiles);
  ctx->launches += 1;
  st = plan_finish(ctx, plan, slot, blk);
  if (st != ACU_OK) return bail(st);
  *out_plan = plan;
  return ACU_OK;
}

// FilterBuilder::new(&cmp::op(a, b)?) fused: the comparison kernels write mask + tile counts (see include/arrow_cuda.h).
acu_status acu_filter_plan_create_cmp(acu_ctx *ctx, acu_dtype dtype, acu_cmp_op op, const acu_array *a, const acu_array *b,
                                      acu_filter_plan **out_plan) {
  *out_plan = nullptr;
  ACU_ENTER(ctx);
  int64_t len = 0;
  ACU_TRY(acu_cmp_len(ctx, a, b, &len));
  acu_filter_plan *plan = nullptr;
  ACU_TRY(plan_alloc(ctx, len, &plan));
  if (len == 0) { *out_plan = plan; return ACU_OK; }
  auto bail = [&](acu_status s) { acu_free(ctx, plan->storage); delete plan; return s; };
  const int64_t n_words_padded = ((plan->n_tiles * TILE_WORDS + 31) / 32) * 32;
  acu_status st = ACU_OK;
  const int blk = acu_call_begin(ctx, &st);
  if (st != ACU_OK) return bail(st);
  st = acu_cmp_into_plan(ctx, dtype, op, a, b, plan->mask, n_words_padded, plan->tile_count, plan->n_tiles);
  if (st != ACU_OK) return bail(st);
  st = plan_finish(ctx, plan, -1, blk);
  if (st != ACU_OK) return bail(st);
  *out_plan = plan;
  return ACU_OK;
}

void acu_filter_plan_destroy(acu_ctx *ctx, acu_filter_plan *plan) {
  if (!plan) return;
  if (plan->storage) acu_free(ctx, plan->storage);
  if (plan->index_cache) acu_free(ctx, plan->index_cache);
  delete plan;
}
int64_t acu_filter_plan_count(const acu_filter_plan *plan) { return plan->count; }
int64_t acu_filter_plan_len(const acu_filter_plan *plan) { return plan->len; }
int32_t acu_filter_plan_strategy(const acu_filter_plan *plan) { return plan->strategy; }

// filter of one primitive (kind 0) or boolean (kind 1) array: the record-batch launcher on one column.
static acu_status filter_array(acu_ctx *ctx, const acu_filter_plan *plan, int kind, int32_t elem_bytes, const acu_array *values,
                               acu_array_out *out) {
  ACU_ENTER(ctx);
  int mode = 0;
  acu_status st = ACU_OK;
  const int blk = acu_call_begin(ctx, &st);
  ACU_TRY(st);
  unsigned long long *res = acu_dres(ctx, blk);
  ACU_TRY(acu_filter_cols_launch(ctx, plan, 1, &kind, &elem_bytes, &values, &out, &res, &mode));
  return acu_call_end(ctx, blk, [plan, mode, out](const unsigned long long *h) -> acu_status {
    acu_filter_col_finalize(plan, mode, h, out);
    return ACU_OK;
  });
}

acu_status acu_filter_primitive(acu_ctx *ctx, const acu_filter_plan *plan, int32_t elem_bytes,
                                const acu_array *values, acu_array_out *out) {
  return filter_array(ctx, plan, 0, elem_bytes, values, out);
}

acu_status acu_filter_boolean(acu_ctx *ctx, const acu_filter_plan *plan, const acu_array *values,
                              acu_array_out *out) {
  return filter_array(ctx, plan, 1, 0, values, out);
}

}  // extern "C"

// IterationStrategy::All: values.slice(0, count) (filter.rs:546) of one column; the slice keeps its NullBuffer (mode 2).
static acu_status filter_slice_col(acu_ctx *ctx, const acu_filter_plan *plan, int kind, int32_t elem_bytes, const acu_array *values,
                                   acu_array_out *out, unsigned long long *res, int *mode) {
  if (kind == 0)
    ACU_CUDA(ctx, cudaMemcpyAsync(out->values, values->values, (size_t)plan->count * elem_bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  else if (kind == 1)
    ACU_TRY(acu_bitmap_and_launch(ctx, static_cast<const uint8_t *>(values->values), values->values_offset, nullptr, 0,
                                  plan->count, static_cast<uint64_t *>(out->values), false));
  if (values->validity) {
    ACU_TRY(acu_bitmap_and_launch(ctx, values->validity, values->validity_offset, nullptr, 0, plan->count,
                                  reinterpret_cast<uint64_t *>(out->validity), true, res));
    *mode = 2;
  }
  return ACU_OK;
}

// The columns of filter / filter_record_batch (kinds[c]: 0 primitive of widths[c] bytes, 1 boolean, 2 validity only):
// queue the value kernels and the validity compactions on the ctx stream WITHOUT synchronising. The value kernels of
// equal-width columns and all the bit compactions share launches (blockIdx.y = column); res[c] = result block of column c.
// modes[c] tells acu_filter_col_finalize how to read that block: 0 = no validity work, 1 = compacted validity + popcount,
// 2 = IterationStrategy::All slice, 3 = compacted with a pending plan.
acu_status acu_filter_cols_launch(acu_ctx *ctx, const acu_filter_plan *plan, int n, const int *kinds, const int32_t *widths,
                                  const acu_array *const *values, acu_array_out *const *outs, unsigned long long *const *res, int *modes) {
  for (int c = 0; c < n; ++c) {
    modes[c] = 0;
    ACU_TRY(check_len(ctx, plan, values[c]->len));
    outs[c]->len = plan->count;
    outs[c]->has_validity = 0;
    outs[c]->null_count = 0;
  }
  const bool pending = plan->count < 0;  // async section: the count is still on the device, outputs are sized for plan->len
  if (!pending && (plan->strategy == ACU_FILTER_NONE || plan->count == 0)) return ACU_OK;
  if (plan->strategy == ACU_FILTER_ALL) {
    for (int c = 0; c < n; ++c) ACU_TRY(filter_slice_col(ctx, plan, kinds[c], widths[c], values[c], outs[c], res[c], &modes[c]));
    return ACU_OK;
  }
  // a validity buffer with a cached null_count of 0 is dropped (filter.rs:513-516); an unknown
  // null_count (-1) is compacted and counted: the result is the same, NullBuffer-wise
  // (a pending plan may turn out to select everything, where the reference slices and KEEPS the NullBuffer even without
  // nulls: the validity is then compacted whenever it exists and the finaliser decides, mode 3)
  auto has_nulls = [&](int c) { return values[c]->validity != nullptr && (values[c]->null_count != 0 || pending); };
  const int compacted_mode = pending ? 3 : 1;
  // value kernels grouped by (element width, alignment class)
  std::vector<char> done(n, 0);
  for (int c = 0; c < n; ++c) {
    if (kinds[c] != 0 || done[c]) continue;
    FilterBatch fb{};
    int k = 0;
    const bool al = aligned16(values[c]->values);
    for (int d = c; d < n && k < BATCH_COLS; ++d) {
      if (kinds[d] != 0 || done[d] || widths[d] != widths[c] || aligned16(values[d]->values) != al) continue;
      fb.col[k] = filter_args(plan, values[d], outs[d], has_nulls(d), res[d]);
      if (fb.col[k].vsrc) {  // the kernel ORs boundary words into the bitmap
        if (pending)
          ACU_LAUNCH(ctx, k_zero_bitmap_dev, acu_grid(ctx, (plan->len / 64 + 255) / 256, 2), 256, 0,
                     reinterpret_cast<uint64_t *>(outs[d]->validity), plan->tile_off + plan->n_tiles);
        else
          ACU_CUDA(ctx, cudaMemsetAsync(outs[d]->validity, 0, acu_bitmap_bytes(plan->count), ctx->stream));
        modes[d] = compacted_mode;
      }
      ++k;
      done[d] = 1;
    }
    ACU_TRY(launch_filter_width(ctx, widths[c], fb, k, fuses_validity(plan)));
  }
  // bit compactions: boolean values and every validity buffer that may hold nulls (FilterPredicate::filter_nulls,
  // filter.rs:512-533) unless the value kernel compacted it
  CompressBatch cb{};
  int k = 0;
  auto flush = [&]() -> acu_status {
    if (k) ACU_TRY(launch_compress(ctx, plan, cb, k));
    k = 0;
    return ACU_OK;
  };
  for (int c = 0; c < n; ++c) {
    if (kinds[c] == 1) {
      cb.col[k++] = compress_args(plan, static_cast<const uint8_t *>(values[c]->values), values[c]->values_offset, outs[c]->values, nullptr);
      if (k == BATCH_COLS) ACU_TRY(flush());
    }
    if (has_nulls(c) && !(kinds[c] == 0 && fuses_validity(plan))) {
      cb.col[k++] = compress_args(plan, values[c]->validity, values[c]->validity_offset, outs[c]->validity, res[c]);
      modes[c] = compacted_mode;
      if (k == BATCH_COLS) ACU_TRY(flush());
    }
  }
  return flush();
}

void acu_filter_col_finalize(const acu_filter_plan *plan, int mode, const unsigned long long *hres, acu_array_out *out) {
  out->len = plan->count;  // (known only now when the call was queued in an async section)
  out->has_validity = 0;
  out->null_count = 0;
  if (mode == 1) {  // None when the filtered validity has no nulls (filter.rs:523-525)
    const int64_t null_count = plan->count - (int64_t)hres[RES_COUNT];
    if (null_count > 0) { out->has_validity = 1; out->null_count = null_count; }
  } else if (mode == 3) {  // queued with a pending plan: IterationStrategy::All keeps the NullBuffer, the others drop an empty one
    const int64_t null_count = plan->count - (int64_t)hres[RES_COUNT];
    if (null_count > 0 || (plan->count == plan->len && plan->count > 0)) { out->has_validity = 1; out->null_count = null_count; }
  } else if (mode == 2) {  // the slice keeps its NullBuffer
    out->has_validity = 1;
    out->null_count = plan->count - (int64_t)hres[RES_COUNT];
  }
}

// Internal accessors for bytes.cu (filter_bytes materialises the selected row indices).
const uint64_t *acu_plan_mask(const acu_filter_plan *p) { return p->mask; }
const uint64_t *acu_plan_tile_off(const acu_filter_plan *p) { return p->tile_off; }
void **acu_plan_index_cache(const acu_filter_plan *p) { return &p->index_cache; }
int64_t acu_plan_n_words_padded(const acu_filter_plan *p) { return ((p->n_tiles * TILE_WORDS + 31) / 32) * 32; }
