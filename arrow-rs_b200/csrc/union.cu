// union.cu — filter and take of sparse / dense Union columns, and the NullBuffer of a Struct's filter / take. The children
// and fields are filtered / taken by the caller through the entry point of their type, with the plan / indices / child
// row map these calls leave.
//
//   type ids (and dense offsets): the existing filter / take of 1- and 4-byte fixed-width columns (filter_primitive,
//     take_native).
//   dense partition: the M output rows are partitioned by type id, stably, in two passes whatever the field count:
//     k_union_count counts every tile's rows per field (a shared-memory histogram over the id -> field table),
//     k_union_scan turns each field's tile counts into exclusive tile bases, k_union_starts sums the fields into the
//     field starts, and k_union_scatter gives every row its position (field start + tile base + the rows of earlier
//     rounds, earlier warps and lower lanes with the same field, from __match_any_sync), writes its source offset there in
//     the child row map and replaces it by its rank within the field, the new offset. No atomic decides a position.
//   The reference's literal dense take (take.rs:346-382) filters the offsets once per field and ranks the type ids once
//     more; that is one pass over the type ids per field, 128 at 128 fields.
//   Struct nulls: the validity-only filter / take column of compact.cu / take.cu, as acu_filter_list / acu_take_list use.
#include <vector>

#include "bitmap.cuh"
#include "internal.cuh"

#define UN_THREADS 256    // every partition kernel: 256-thread blocks
#define UN_TILE_ROWS 4096 // rows per tile: a block walks its tile in rounds of UN_THREADS rows, one row per thread
#define UN_PER_SM 8       // tile kernels run on acu_grid(ctx, tiles, UN_PER_SM) blocks, grid-stride over tiles

namespace {

constexpr int kWarps = UN_THREADS / 32;
constexpr int kMaxFields = ACU_UNION_MAX_FIELDS;

union FieldTable {  // type id (0..127) -> field, -1 for an id that names no field
  int8_t f[kMaxFields];
  uint32_t w[kMaxFields / 4];
};

__device__ __forceinline__ int field_of(const int8_t *s_tab, int8_t id) { return id >= 0 ? s_tab[id] : -1; }

// Word i of the table by thread i, with constant indices so that the table is read from the kernel parameters in place.
__device__ __forceinline__ void load_table(int8_t *s_tab, const FieldTable &tab) {
#pragma unroll
  for (int i = 0; i < kMaxFields / 4; ++i)
    if (threadIdx.x == i) reinterpret_cast<uint32_t *>(s_tab)[i] = tab.w[i];
}

// counts[f * n_tiles + tile] = the tile's rows of field f; rows whose id names no field are added to res[RES_AUX0].
__global__ void __launch_bounds__(UN_THREADS) k_union_count(const int8_t *__restrict__ ids, int64_t m, FieldTable tab, int nf,
                                                            int64_t n_tiles, int64_t *__restrict__ counts, unsigned long long *res) {
  __shared__ __align__(4) int8_t s_tab[kMaxFields];
  __shared__ unsigned s_cnt[kMaxFields];
  load_table(s_tab, tab);
  const int lane = threadIdx.x & 31;
  unsigned long long unknown = 0;
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    for (int t = threadIdx.x; t < nf; t += UN_THREADS) s_cnt[t] = 0;
    __syncthreads();
    const int64_t r_end = (tile + 1) * UN_TILE_ROWS < m ? (tile + 1) * UN_TILE_ROWS : m;
    for (int64_t r0 = tile * UN_TILE_ROWS; r0 < r_end; r0 += UN_THREADS) {
      const int64_t r = r0 + threadIdx.x;
      const int f = r < r_end ? field_of(s_tab, __ldg(ids + r)) : -2;
      const unsigned peers = __match_any_sync(ACU_FULL_MASK, f);
      if (lane == __ffs(peers) - 1) {
        if (f >= 0) atomicAdd(&s_cnt[f], (unsigned)__popc(peers));
        else if (f == -1) unknown += (unsigned)__popc(peers);
      }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < nf; t += UN_THREADS) counts[(int64_t)t * n_tiles + tile] = s_cnt[t];
    __syncthreads();
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) unknown += __shfl_xor_sync(ACU_FULL_MASK, unknown, o);
  if (lane == 0 && unknown) atomicAdd(res + RES_AUX0, unknown);
}

// Block f: exclusive scan of field f's tile counts in place; totals[f] = its rows.
__global__ void __launch_bounds__(UN_THREADS) k_union_scan(int64_t *__restrict__ counts, int64_t n_tiles, int64_t *__restrict__ totals) {
  __shared__ int64_t s_warp[kWarps];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int64_t *c = counts + (int64_t)blockIdx.x * n_tiles;
  int64_t carry = 0;
  for (int64_t i0 = 0; i0 < n_tiles; i0 += UN_THREADS) {
    const int64_t i = i0 + threadIdx.x;
    const int64_t v = i < n_tiles ? c[i] : 0;
    int64_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int64_t y = __shfl_up_sync(ACU_FULL_MASK, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) s_warp[warp] = x;
    __syncthreads();
    int64_t below = 0, all = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      below += w < warp ? s_warp[w] : 0;
      all += s_warp[w];
    }
    if (i < n_tiles) c[i] = carry + below + x - v;
    carry += all;
    __syncthreads();
  }
  if (threadIdx.x == 0) totals[blockIdx.x] = carry;
}

// starts[f] = rows of the fields before f, starts[nf] = rows of every field.
__global__ void k_union_starts(const int64_t *__restrict__ totals, int nf, int64_t *__restrict__ starts) {
  int64_t s = 0;
  for (int f = 0; f < nf; ++f) {
    starts[f] = s;
    s += totals[f];
  }
  starts[nf] = s;
}

// Row r of field f goes to map position starts[f] + base(f, tile) + (rows of f in earlier rounds of the tile) + (rows of
// f in lower warps of this round) + (rows of f in lower lanes of this warp); map[pos] = offs[r], offs[r] = pos - starts[f].
// A row whose id names no field gets offset 0 and no map entry.
__global__ void __launch_bounds__(UN_THREADS) k_union_scatter(const int8_t *__restrict__ ids, int32_t *__restrict__ offs, int64_t m,
                                                              FieldTable tab, int nf, int64_t n_tiles, const int64_t *__restrict__ base,
                                                              const int64_t *__restrict__ starts, int32_t *__restrict__ map) {
  __shared__ __align__(4) int8_t s_tab[kMaxFields];
  __shared__ int64_t s_start[kMaxFields];
  __shared__ int64_t s_run[kMaxFields];
  __shared__ unsigned s_w[kWarps][kMaxFields];
  load_table(s_tab, tab);
  for (int t = threadIdx.x; t < nf; t += UN_THREADS) s_start[t] = __ldg(starts + t);
  for (int t = threadIdx.x; t < kWarps * kMaxFields; t += UN_THREADS) s_w[t / kMaxFields][t % kMaxFields] = 0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned lt = (1u << lane) - 1u;
  __syncthreads();
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    for (int t = threadIdx.x; t < nf; t += UN_THREADS) s_run[t] = s_start[t] + __ldg(base + (int64_t)t * n_tiles + tile);
    __syncthreads();
    const int64_t r_end = (tile + 1) * UN_TILE_ROWS < m ? (tile + 1) * UN_TILE_ROWS : m;
    for (int64_t r0 = tile * UN_TILE_ROWS; r0 < r_end; r0 += UN_THREADS) {
      const int64_t r = r0 + threadIdx.x;
      const int f = r < r_end ? field_of(s_tab, __ldg(ids + r)) : -2;
      const unsigned peers = __match_any_sync(ACU_FULL_MASK, f);
      if (f >= 0 && lane == __ffs(peers) - 1) s_w[warp][f] = (unsigned)__popc(peers);
      __syncthreads();
      if (f >= 0) {
        int64_t pos = s_run[f] + __popc(peers & lt);
        for (int w = 0; w < warp; ++w) pos += s_w[w][f];
        map[pos] = offs[r];
        // the rank is an i32 offset: past i32::MAX rows of one field it wraps (two's complement) as the reference's i32
        // running count does in a release build; acu_take_union then reports try_new's offset error
        offs[r] = (int32_t)(uint32_t)(pos - s_start[f]);
      } else if (f == -1) {
        offs[r] = 0;
      }
      __syncthreads();
      for (int t = threadIdx.x; t < nf; t += UN_THREADS) {
        int64_t add = 0;
#pragma unroll
        for (int w = 0; w < kWarps; ++w) {
          add += s_w[w][t];
          s_w[w][t] = 0;
        }
        s_run[t] += add;
      }
      __syncthreads();
    }
  }
}

struct DevBufs {  // acu_malloc'ed buffers freed on every return (the nested entry points use the ctx scratch)
  acu_ctx *ctx;
  std::vector<void *> p;
  acu_status get(size_t bytes, void **out) {
    ACU_TRY(acu_malloc(ctx, bytes, out));
    p.push_back(*out);
    return ACU_OK;
  }
  ~DevBufs() {
    for (void *q : p) acu_free(ctx, q);
  }
};

acu_status check_union(acu_ctx *ctx, const acu_union_array *u, FieldTable *tab) {
  if (u->mode != ACU_UNION_SPARSE && u->mode != ACU_UNION_DENSE)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "unknown union mode %d", (int)u->mode);
  if (u->n_fields < 1 || u->n_fields > kMaxFields || !u->field_type_ids)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "a union needs 1 to %d fields, got %d", kMaxFields, (int)u->n_fields);
  if (u->len < 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "union length must be >= 0");
  if (u->mode == ACU_UNION_DENSE && (uintptr_t)u->offsets % 4 != 0)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "dense union offsets must be 4-byte aligned");
  for (int i = 0; i < kMaxFields; ++i) tab->f[i] = -1;
  for (int f = 0; f < u->n_fields; ++f) {
    const int id = u->field_type_ids[f];
    if (id < 0 || tab->f[id] >= 0)
      return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "union field type ids must be distinct and in [0, 127], got %d", id);
    tab->f[id] = (int8_t)f;
  }
  return ACU_OK;
}

// The dense partition of the m rows `ids` / `offs` (offs: source offsets in, new offsets out) into `map`; the field
// starts go to starts_host. Sparse unions pass offs == nullptr: the rows are only counted. *unknown = rows whose id names
// no field.
acu_status union_partition(acu_ctx *ctx, int cls, const int8_t *ids, int32_t *offs, int64_t m, const FieldTable &tab, int nf,
                           int32_t *map, int64_t *starts_host, unsigned long long *unknown) {
  *unknown = 0;
  if (starts_host)
    for (int f = 0; f <= nf; ++f) starts_host[f] = 0;
  if (m == 0) return ACU_OK;
  const int64_t n_tiles = (m + UN_TILE_ROWS - 1) / UN_TILE_ROWS;
  DevBufs bufs{ctx};
  void *counts = nullptr, *totals = nullptr, *starts = nullptr;
  ACU_TRY(bufs.get((size_t)nf * n_tiles * 8 + 16, &counts));
  ACU_TRY(bufs.get((size_t)(2 * nf + 2) * 8, &totals));
  starts = static_cast<int64_t *>(totals) + nf;
  ACU_TRY(acu_res_reset(ctx));
  const int grid = acu_grid(ctx, n_tiles, UN_PER_SM);
  int64_t *cnt = static_cast<int64_t *>(counts);
  ACU_LAUNCH_TIMED(ctx, cls, k_union_count, grid, UN_THREADS, 0, ids, m, tab, nf, n_tiles, cnt, acu_dres(ctx, 0));
  if (offs) {
    int64_t *tot = static_cast<int64_t *>(totals), *st = static_cast<int64_t *>(starts);
    ACU_LAUNCH_TIMED(ctx, cls, k_union_scan, nf, UN_THREADS, 0, cnt, n_tiles, tot);
    ACU_LAUNCH_TIMED(ctx, cls, k_union_starts, 1, 1, 0, tot, nf, st);
    ACU_LAUNCH_TIMED(ctx, cls, k_union_scatter, grid, UN_THREADS, 0, ids, offs, m, tab, nf, n_tiles, cnt, st, map);
    ACU_CUDA(ctx, cudaMemcpyAsync(starts_host, st, (size_t)(nf + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
  }
  ACU_TRY(acu_res_fetch(ctx));
  acu_kstats_drain(ctx);
  *unknown = acu_hres(ctx, 0)[RES_AUX0];
  return ACU_OK;
}

}  // namespace

extern "C" acu_status acu_filter_nulls(acu_ctx *ctx, const acu_filter_plan *plan, const acu_array *nulls_of, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  const int64_t plen = acu_filter_plan_len(plan);
  if (plen > nulls_of->len)  // filter.rs:536-542
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Filter predicate of length %lld is larger than target array of length %lld",
                    (long long)plen, (long long)nulls_of->len);
  ACU_TRY(acu_res_reset(ctx));
  const int kind = 2;
  const int32_t width = 0;
  int mode = 0;
  unsigned long long *res = acu_dres(ctx, 0);
  ACU_TRY(acu_filter_cols_launch(ctx, plan, 1, &kind, &width, &nulls_of, &out, &res, &mode));
  ACU_TRY(acu_res_fetch(ctx));
  acu_filter_col_finalize(plan, mode, acu_hres(ctx, 0), out);
  acu_kstats_drain(ctx);
  return ACU_OK;
}

extern "C" acu_status acu_take_nulls(acu_ctx *ctx, const acu_array *nulls_of, const acu_array *indices, acu_dtype index_dtype,
                                     int32_t check_bounds, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  if (acu_take_index_kind(index_dtype) < 0)  // take.rs:103
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Take only supported for integers, got %s", acu_dtype_name(index_dtype));
  acu_status st = ACU_OK;
  const int64_t m = indices->len, n = nulls_of->len;
  const int64_t inc = m > 0 ? acu_resolve_null_count(ctx, indices, &st) : 0;
  if (m > 0) ACU_TRY(st);
  const bool idx_nulls = indices->validity && inc > 0;
  if (check_bounds) ACU_TRY(acu_take_check_bounds(ctx, indices, index_dtype, idx_nulls, n));
  out->len = m;
  out->has_validity = 0;
  out->null_count = 0;
  if (m == 0) return ACU_OK;
  // array.is_valid(index) reads the struct's validity buffer whenever there is one, with or without nulls in it
  const char read_valid = nulls_of->validity != nullptr;
  ACU_TRY(acu_res_reset(ctx));
  unsigned long long *res = acu_dres(ctx, 0);
  const int32_t zero = 0;
  const char not_bool = 0;
  int mode = 0;
  ACU_TRY(acu_take_cols_launch(ctx, 1, &zero, &nulls_of, &not_bool, &read_valid, indices, index_dtype, idx_nulls, &out, &res, &mode));
  ACU_TRY(acu_res_fetch(ctx));
  acu_kstats_drain(ctx);
  unsigned long long h[RES_SLOTS];
  std::copy(acu_hres(ctx, 0), acu_hres(ctx, 0) + RES_SLOTS, h);
  const unsigned long long oob = h[RES_ERR_INDEX];
  h[RES_ERR_INDEX] = ~0ull;  // a valid index past the struct is read only through its validity buffer (below)
  ACU_TRY(acu_take_col_finalize(ctx, nulls_of, indices, index_dtype, mode, h, out));
  if (out->null_count == 0) out->has_validity = 0;  // StructArray::try_new: nulls.filter(|n| n.null_count() > 0)
  if (read_valid && oob != ~0ull)  // BooleanBuffer::value (arrow-buffer/src/buffer/boolean.rs), after the fields' takes
    return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, (int64_t)oob, 0, 0, (uint64_t)n, "assertion failed: idx < self.bit_len");
  return ACU_OK;
}

extern "C" acu_status acu_filter_union(acu_ctx *ctx, const acu_filter_plan *plan, const acu_union_array *u, int8_t *out_type_ids,
                                       int32_t *out_offsets, int32_t *out_child_rows, int64_t *out_field_starts) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  FieldTable tab;
  ACU_TRY(check_union(ctx, u, &tab));
  const int64_t plen = acu_filter_plan_len(plan);
  if (plen > u->len)  // filter.rs:536-542
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Filter predicate of length %lld is larger than target array of length %lld",
                    (long long)plen, (long long)u->len);
  const int32_t strategy = acu_filter_plan_strategy(plan);
  if (strategy == ACU_FILTER_NONE || strategy == ACU_FILTER_ALL) return ACU_OK;  // filter.rs:545-546, the caller's
  const int64_t count = acu_filter_plan_count(plan);
  DevBufs bufs{ctx};
  void *scratch_valid = nullptr;
  ACU_TRY(bufs.get(acu_bitmap_bytes(count) + 8, &scratch_valid));
  acu_array ta{};
  ta.values = u->type_ids;
  ta.len = u->len;
  acu_array_out o{};
  o.values = out_type_ids;
  o.validity = static_cast<uint8_t *>(scratch_valid);
  ACU_TRY(acu_filter_primitive(ctx, plan, 1, &ta, &o));
  if (u->mode == ACU_UNION_SPARSE) return ACU_OK;
  acu_array oa{};
  oa.values = u->offsets;
  oa.len = u->len;
  o.values = out_offsets;
  ACU_TRY(acu_filter_primitive(ctx, plan, 4, &oa, &o));
  unsigned long long unknown = 0;  // only a malformed union: those rows go into no child
  return union_partition(ctx, ACU_K_FILTER_PLAN, out_type_ids, out_offsets, count, tab, u->n_fields, out_child_rows, out_field_starts,
                         &unknown);
}

extern "C" acu_status acu_take_union(acu_ctx *ctx, const acu_union_array *u, const acu_array *indices, acu_dtype index_dtype,
                                     int32_t check_bounds, int8_t *out_type_ids, int32_t *out_offsets, int32_t *out_child_rows,
                                     int64_t *out_field_starts) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  FieldTable tab;
  ACU_TRY(check_union(ctx, u, &tab));
  const int64_t m = indices->len;
  DevBufs bufs{ctx};
  void *scratch_valid = nullptr;
  ACU_TRY(bufs.get(acu_bitmap_bytes(m) + 8, &scratch_valid));
  // take_native of the type ids, then of the offsets (take.rs:334-351): acu_take_primitive's bounds check and panics
  acu_array ta{};
  ta.values = u->type_ids;
  ta.len = u->len;
  acu_array_out o{};
  o.values = out_type_ids;
  o.validity = static_cast<uint8_t *>(scratch_valid);
  ACU_TRY(acu_take_primitive(ctx, 1, &ta, indices, index_dtype, check_bounds, &o));
  const bool dense = u->mode == ACU_UNION_DENSE;
  if (dense) {
    acu_array oa{};
    oa.values = u->offsets;
    oa.len = u->len;
    o.values = out_offsets;
    ACU_TRY(acu_take_primitive(ctx, 4, &oa, indices, index_dtype, 0, &o));
  }
  unsigned long long unknown = 0;
  ACU_TRY(union_partition(ctx, ACU_K_TAKE, out_type_ids, dense ? out_offsets : nullptr, m, tab, u->n_fields, out_child_rows,
                          dense ? out_field_starts : nullptr, &unknown));
  if (unknown)  // UnionArray::try_new (union_array.rs:208-218), after the children
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Type Ids values must match one of the field type ids");
  if (dense)  // a field of more than i32::MAX rows: its wrapped offsets fail try_new's next check (union_array.rs:221-229)
    for (int f = 0; f < u->n_fields; ++f)
      if (out_field_starts[f + 1] - out_field_starts[f] > (int64_t)INT32_MAX)
        return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Offsets must be non-negative and within the length of the Array");
  return ACU_OK;
}
