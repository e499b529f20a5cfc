// fixed_size_binary.cu — filter and take of FixedSizeBinary(W) columns of any width W >= 0.
//
//   filter_fixed_size_binary (arrow-select/src/filter.rs:946-996), take_fixed_size_binary (take.rs:802-862).
//
//   Routing, by an input property: the widths the fixed-width kernels already serve keep them, with the same semantics.
//     filter: W in {1, 2, 4, 8, 16, 32} (values and output aligned to min(W, 8)) -> k_filter_fused, as filter_primitive;
//             IterationStrategy::All -> values.slice(0, count), a copy of the first count * W bytes;
//     take:   W in {1, 2, 4, 8, 16} (values and output aligned to W) -> k_take: take_fixed_size is take_native byte for byte;
//     W == 0: no bytes move, only the validity.
//     Every other case -> k_fsb_gather, below. The validity of every case is the validity-only filter / take column of
//     compact.cu / take.cu (FilterPredicate::filter_nulls, take_nulls + NullBuffer::union).
//
//   k_fsb_gather: output row j copies source row src(j) (the widened index for take, the plan's selected row for filter).
//     A thread owns 16-byte output chunks aligned to the absolute output address; a chunk covers output rows
//     floor(p / W) .. floor((p + 15) / W), at most 15 / W + 2 of them (2 when W >= 16). The chunk's first row comes from one
//     multiply-high division by W (per-launch magic), the rest by walking. Each row piece (<= 16 bytes) is fetched with
//     load_upto16 of bytes_engine.cuh (aligned 8-byte loads + funnel shifts) and shifted into place; FSB_CHUNKS chunks per
//     thread and round, all index and source loads issued before the first store; full chunks leave as st.global.cs.v4,
//     the partial first / last chunk byte by byte. Byte positions are 64-bit everywhere.
//     take_fixed_size_binary_buffer_dynamic_length (take.rs:827-861): a null index gives W zero bytes and is never read;
//     a valid index reads values[idx*W .. idx*W + W] with usize arithmetic that wraps (a release build), and a slice out of
//     order or past the buffer reads nothing and sends its output row to res[RES_ERR2] (atomicMin: the lowest row, whatever
//     the grid); the host rebuilds core's slice panic from the fetched index.
//     `native` (the k_take widths whose buffers are not aligned for it): take_fixed_size (take.rs:876-926) instead: an
//     in-bounds null index gathers its row, an out-of-bounds null index gives zeros, a valid one panics.
#include <algorithm>

#include "bytes_engine.cuh"

#define FSB_THREADS 256  // k_fsb_gather: 256-thread blocks
#define FSB_PER_SM 8     // grid = acu_grid(ctx, blocks of FSB_THREADS * chunks-per-thread chunks, FSB_PER_SM), grid-stride

namespace {

struct FsbArgs {
  const uint8_t *src;     // values at logical row 0 (any alignment)
  uint64_t n_rows;        // values' rows
  uint64_t n_bytes;       // n_rows * w
  uint64_t w;             // >= 1
  DivW div;               // p / w (bytes_engine.cuh)
  const void *idx;        // ld_index kind `kind`
  int kind;
  const uint8_t *ivalid;  // validity of the indices when it holds a null, else NULL
  int64_t ivoff;
  int native;             // take_fixed_size: a null in-bounds index still gathers
  int64_t m;              // output rows
  uint8_t *out;           // any alignment
  unsigned long long *res;
};

// Rows a 16-byte chunk can touch, and chunks per thread and round, by instantiation.
template <int MAXR> struct FsbCfg { static constexpr int CHUNKS = MAXR <= 3 ? 4 : MAXR <= 5 ? 2 : 1; };

// The source byte of row r's first byte, or ~0 when the row reads nothing (zeros); *err lowered on a panicking row.
__device__ __forceinline__ uint64_t row_source(const FsbArgs &a, int64_t r, unsigned long long *err) {
  const uint64_t ix = ld_index(a.idx, a.kind, r);
  const bool valid = a.ivalid == nullptr || ld_bit(a.ivalid, a.ivoff + r);
  const uint64_t start = ix * a.w, end = start + a.w;  // usize arithmetic: wraps
  const bool ok = a.native ? ix < a.n_rows : (start <= end && end <= a.n_bytes);
  if (!ok && valid && (unsigned long long)r < *err) *err = (unsigned long long)r;
  return ok && (valid || a.native) ? start : ~0ull;
}

// A piece x1:x0 of nb bytes ORed into the chunk lo:hi at byte offset o (o + nb <= 16).
__device__ __forceinline__ void place(uint64_t x0, uint64_t x1, uint32_t o, uint64_t *lo, uint64_t *hi) {
  const uint32_t s = 8u * (o & 7u);
  const uint64_t a0 = x0 << s, a1 = (x1 << s) | ((x0 >> 1) >> (63u - s));
  if (o < 8u) {
    *lo |= a0;
    *hi |= a1;
  } else {
    *hi |= a0;
  }
}

template <int MAXR>
__global__ void __launch_bounds__(FSB_THREADS) k_fsb_gather(const FsbArgs a) {
  constexpr int K = FsbCfg<MAXR>::CHUNKS;
  const uint64_t lead = (uintptr_t)a.out & 15u;
  const uint64_t total = (uint64_t)a.m * a.w;
  const int64_t n_chunks = (int64_t)((lead + total + 15) >> 4);
  uint8_t *base = a.out - lead;  // chunk g is base + 16 g, output bytes 16 g - lead ..
  unsigned long long err = ~0ull;
  for (int64_t r0 = (int64_t)blockIdx.x * FSB_THREADS * K; r0 < n_chunks; r0 += (int64_t)gridDim.x * FSB_THREADS * K) {
    uint64_t lo[K], hi[K];
    uint64_t src[K][MAXR];
    int64_t row0[K];
    // ---- issue: every row's index, then every piece's source words ----
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int64_t g = r0 + (int64_t)k * FSB_THREADS + threadIdx.x;
      const uint64_t p0 = (uint64_t)g * 16 - lead;  // may wrap below 0 for g == 0: only compared through pl
      const uint64_t pl = g == 0 ? 0 : p0, ph = (uint64_t)g * 16 + 16 - lead < total ? (uint64_t)g * 16 + 16 - lead : total;
      row0[k] = g < n_chunks ? (int64_t)div_by(a.div, pl) : 0;
#pragma unroll
      for (int q = 0; q < MAXR; ++q) {
        const int64_t r = row0[k] + q;
        src[k][q] = g < n_chunks && (uint64_t)r * a.w < ph ? row_source(a, r, &err) : ~0ull;
      }
    }
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int64_t g = r0 + (int64_t)k * FSB_THREADS + threadIdx.x;
      const uint64_t p0 = (uint64_t)g * 16 - lead;
      const uint64_t pl = g == 0 ? 0 : p0, ph = (uint64_t)g * 16 + 16 - lead < total ? (uint64_t)g * 16 + 16 - lead : total;
      lo[k] = hi[k] = 0;
#pragma unroll
      for (int q = 0; q < MAXR; ++q) {
        const uint64_t rs = (uint64_t)(row0[k] + q) * a.w;  // the row's first output byte
        if (g >= n_chunks || rs >= ph) continue;
        const uint64_t b0 = rs > pl ? rs : pl, b1 = rs + a.w < ph ? rs + a.w : ph;
        if (src[k][q] == ~0ull) continue;
        uint64_t x0, x1;
        load_upto16(a.src, (int64_t)(src[k][q] + (b0 - rs)), (uint32_t)(b1 - b0), &x0, &x1);
        place(x0, x1, (uint32_t)(b0 - p0), &lo[k], &hi[k]);
      }
    }
    // ---- store ----
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const int64_t g = r0 + (int64_t)k * FSB_THREADS + threadIdx.x;
      if (g >= n_chunks) continue;
      const uint32_t first = g == 0 ? (uint32_t)lead : 0u;
      const uint64_t end = (uint64_t)g * 16 + 16 - lead;
      const uint32_t last = end <= total ? 16u : (uint32_t)(16u - (end - total));
      uint8_t *dst = base + (size_t)g * 16;
      if (first == 0u && last == 16u) {
        st_stream16(dst, make_uint4((uint32_t)lo[k], (uint32_t)(lo[k] >> 32), (uint32_t)hi[k], (uint32_t)(hi[k] >> 32)));
      } else {
        for (uint32_t b = first; b < last; ++b) dst[b] = (uint8_t)((b < 8u ? lo[k] >> (8u * b) : hi[k] >> (8u * (b - 8u))) & 0xffu);
      }
    }
  }
  if (err != ~0ull) atomicMin(a.res + RES_ERR2, err);
}

int max_rows(int64_t w) { return w >= 16 ? 2 : w >= 8 ? 3 : w >= 4 ? 5 : w >= 2 ? 9 : 17; }

template <int MAXR>
acu_status launch_gather_r(acu_ctx *ctx, int cls, const FsbArgs &a) {
  const int64_t n_chunks = (int64_t)((((uintptr_t)a.out & 15u) + (uint64_t)a.m * a.w + 15) >> 4);
  const int64_t per_block = (int64_t)FSB_THREADS * FsbCfg<MAXR>::CHUNKS;
  const int grid = acu_grid(ctx, (n_chunks + per_block - 1) / per_block, FSB_PER_SM);
  ACU_LAUNCH_TIMED(ctx, cls, k_fsb_gather<MAXR>, grid, FSB_THREADS, 0, a);
  return ACU_OK;
}

// m output rows of width w from src, row j from source row idx[j] (ld_index kind); nothing when m * w == 0.
acu_status launch_gather(acu_ctx *ctx, int cls, int64_t w, const acu_array *values, const void *idx, int kind, const uint8_t *ivalid,
                         int64_t ivoff, bool native, int64_t m, void *out, unsigned long long *res) {
  if (m == 0 || w == 0) return ACU_OK;
  FsbArgs a{};
  a.src = static_cast<const uint8_t *>(values->values);
  a.n_rows = (uint64_t)values->len;
  a.n_bytes = (uint64_t)values->len * (uint64_t)w;
  a.w = (uint64_t)w;
  a.div = make_div_w(a.w);
  a.idx = idx;
  a.kind = kind;
  a.ivalid = ivalid;
  a.ivoff = ivoff;
  a.native = native;
  a.m = m;
  a.out = static_cast<uint8_t *>(out);
  a.res = res;
  switch (max_rows(w)) {
    case 2: return launch_gather_r<2>(ctx, cls, a);
    case 3: return launch_gather_r<3>(ctx, cls, a);
    case 5: return launch_gather_r<5>(ctx, cls, a);
    case 9: return launch_gather_r<9>(ctx, cls, a);
    default: return launch_gather_r<17>(ctx, cls, a);
  }
}

bool aligned_to(const void *p, int64_t a) { return ((uintptr_t)p % (uintptr_t)a) == 0; }

bool take_native_width(int32_t w) { return w == 1 || w == 2 || w == 4 || w == 8 || w == 16; }

// Route of a take column: k_take serves it (values and output aligned to w).
bool take_by_ktake(int32_t w, const acu_array *values, const acu_array_out *out) {
  return take_native_width(w) && aligned_to(values->values, w) && aligned_to(out->values, w);
}

}  // namespace

int acu_fsb_filter_kind(const acu_filter_plan *plan, int32_t w, const acu_array *values, const acu_array_out *out) {
  if (acu_filter_plan_strategy(plan) == ACU_FILTER_ALL) return 0;  // values.slice(0, count): the first count * w bytes
  const bool primitive = w == 1 || w == 2 || w == 4 || w == 8 || w == 16 || w == 32;
  const int64_t al = w < 8 ? w : 8;
  return primitive && aligned_to(values->values, al) && aligned_to(out->values, al) ? 0 : 2;
}

acu_status acu_fsb_filter_values_launch(acu_ctx *ctx, const acu_filter_plan *plan, int32_t w, const acu_array *values, acu_array_out *out,
                                        unsigned long long *res) {
  const int32_t strategy = acu_filter_plan_strategy(plan);
  if (w == 0 || strategy == ACU_FILTER_NONE || strategy == ACU_FILTER_ALL || acu_filter_plan_count(plan) == 0) return ACU_OK;
  const void *idx = nullptr;
  int kind = 0;
  ACU_TRY(acu_plan_cached_indices(ctx, plan, &idx, &kind));
  return launch_gather(ctx, ACU_K_FILTER, w, values, idx, kind, nullptr, 0, true, acu_filter_plan_count(plan), out->values, res);
}

void acu_fsb_filter_finalize(const acu_filter_plan *plan, int mode, int32_t w, const unsigned long long *hres, acu_array_out *out) {
  acu_filter_col_finalize(plan, mode, hres, out);
  // FixedSizeBinaryArray::try_new of width 0 takes its length from the NullBuffer (fixed_size_binary_array.rs:178-201);
  // the All slice keeps its length
  if (w == 0 && !out->has_validity && acu_filter_plan_strategy(plan) != ACU_FILTER_ALL) out->len = 0;
}

int32_t acu_fsb_take_width(int32_t w, const acu_array *values, const acu_array_out *out) {
  return take_by_ktake(w, values, out) ? w : 0;
}

acu_status acu_fsb_take_values_launch(acu_ctx *ctx, int32_t w, const acu_array *values, const acu_array *indices, acu_dtype index_dtype,
                                      bool idx_nulls, acu_array_out *out, unsigned long long *res) {
  if (w == 0 || take_by_ktake(w, values, out)) return ACU_OK;
  return launch_gather(ctx, ACU_K_TAKE, w, values, indices->values, acu_take_index_kind(index_dtype), idx_nulls ? indices->validity : nullptr,
                       indices->validity_offset, take_native_width(w), indices->len, out->values, res);
}

acu_status acu_fsb_take_finalize(acu_ctx *ctx, int32_t w, const acu_array *values, const acu_array *indices, acu_dtype index_dtype,
                                 bool val_nulls, int mode, const unsigned long long *hres, acu_array_out *out) {
  const int64_t m = indices->len;
  out->len = m;
  out->has_validity = 0;
  out->null_count = 0;
  if (m == 0) return ACU_OK;
  unsigned long long h[RES_SLOTS];
  std::copy(hres, hres + RES_SLOTS, h);
  const bool ktake = take_by_ktake(w, values, out);
  if (!ktake && h[RES_ERR2] != ~0ull) {  // the value step's panic
    const int64_t j = (int64_t)h[RES_ERR2];
    const int sz = acu_dtype_size(index_dtype);
    uint64_t raw = 0;
    ACU_CUDA(ctx, cudaMemcpyAsync(&raw, static_cast<const uint8_t *>(indices->values) + (size_t)j * sz, sz, cudaMemcpyDeviceToHost, ctx->stream));
    ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    uint64_t ix = raw;  // ToIndices (take.rs:1030-1084): i8 / i16 `as u32` sign-extend, i32 is reinterpreted as u32
    if (index_dtype == ACU_I8) ix = (uint32_t)(int32_t)(int8_t)raw;
    else if (index_dtype == ACU_I16) ix = (uint32_t)(int32_t)(int16_t)raw;
    else if (index_dtype == ACU_I32) ix = (uint32_t)raw;
    if (take_native_width(w))  // take_fixed_size
      return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, j, ix, 0, (uint64_t)values->len, "Out-of-bounds index %llu", (unsigned long long)ix);
    // core's slice indexing (Range<usize>::index -> slice_index_fail(start, end, len), Rust 1.97): the start against the
    // length first, then the end, then the order of the range
    const uint64_t s = ix * (uint64_t)w, e = s + (uint64_t)w, n = (uint64_t)values->len * (uint64_t)w;
    if (s > n)
      return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, j, s, e, n, "range start index %llu out of range for slice of length %llu",
                      (unsigned long long)s, (unsigned long long)n);
    if (e > n)
      return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, j, s, e, n, "range end index %llu out of range for slice of length %llu",
                      (unsigned long long)e, (unsigned long long)n);
    return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, j, s, e, n, "slice index starts at %llu but ends at %llu", (unsigned long long)s,
                    (unsigned long long)e);
  }
  unsigned long long bits_oob = ~0ull;
  if (!ktake) {  // a valid index past the values reaches the validity gather only through take_bits (below)
    bits_oob = h[RES_ERR_INDEX];
    h[RES_ERR_INDEX] = ~0ull;
  }
  if (mode >= 0) ACU_TRY(acu_take_col_finalize(ctx, values, indices, index_dtype, mode, h, out));
  if (val_nulls && bits_oob != ~0ull)  // BooleanBuffer::value in take_bits (arrow-buffer/src/buffer/boolean.rs)
    return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, (int64_t)bits_oob, 0, 0, (uint64_t)values->len, "assertion failed: idx < self.bit_len");
  if (out->null_count == 0) out->has_validity = 0;  // NullBuffer::union: a buffer only when a side has a null (null.rs:79-87)
  if (w == 0 && !out->has_validity) out->len = 0;   // try_new of width 0: the length of the NullBuffer
  return ACU_OK;
}

extern "C" acu_status acu_filter_fixed_size_binary(acu_ctx *ctx, const acu_filter_plan *plan, int32_t byte_width, const acu_array *values,
                                                   acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  acu_column col{};
  col.kind = ACU_COL_FIXED_SIZE_BINARY;
  col.width = byte_width;
  col.array = *values;
  acu_column_out o{};
  o.array = *out;
  const acu_status st = acu_filter_record_batch(ctx, plan, 1, &col, &o);
  out->len = o.array.len;
  out->has_validity = o.array.has_validity;
  out->null_count = o.array.null_count;
  return st;
}

extern "C" acu_status acu_take_fixed_size_binary(acu_ctx *ctx, int32_t byte_width, const acu_array *values, const acu_array *indices,
                                                 acu_dtype index_dtype, int32_t check_bounds, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  acu_column col{};
  col.kind = ACU_COL_FIXED_SIZE_BINARY;
  col.width = byte_width;
  col.array = *values;
  acu_column_out o{};
  o.array = *out;
  const acu_status st = acu_take_record_batch(ctx, 1, &col, indices, index_dtype, check_bounds, &o);
  out->len = o.array.len;
  out->has_validity = o.array.has_validity;
  out->null_count = o.array.null_count;
  return st;
}
