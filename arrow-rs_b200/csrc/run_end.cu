// run_end.cu — filter and take of RunEndEncoded columns. The run ends are handled here; the values child is filtered /
// taken by the caller through the entry point of its type, with the plan / value indices these calls return.
//
//   filter (filter_run_end_array, arrow-select/src/filter.rs:628-677): k_ree_bounds finds the physical range of the slice
//     (get_start_physical_index / get_end_physical_index, arrow-buffer/src/buffer/run.rs:232-267); k_ree_filter_runs gives
//     every run of it rank(clipped end), the selected rows below its end, read from the filter plan's mask and tile offsets,
//     and keeps it iff that rank exceeds its predecessor's. The keep bits become the values plan (acu_filter_plan_create) and
//     the kept runs' ranks, compacted with it by the filter kernel, are the new run ends.
//   take (take_run, arrow-select/src/take.rs:948-995): k_ree_take_map converts every index (ToIndices), reduces the largest
//     value, null slots included (get_physical_indices' bounds error, run.rs:321-378), and binary-searches its physical run;
//     k_ree_run_ends marks every output position q that ends a run (q == M, or the physical runs of rows q - 1 and q differ
//     and their values do not compare equal). That bitmap is a plan whose selected positions are the new run ends
//     (acu_filter_plan_indices) and which compacts the physical rows into the value indices (the filter kernel).
#include <vector>

#include "bitmap.cuh"
#include "bytes_cmp.cuh"
#include "bytes_engine.cuh"
#include "internal.cuh"

#define RE_THREADS 256  // every kernel here: 256-thread blocks on acu_grid(ctx, blocks, RE_PER_SM), grid-stride inside
#define RE_PER_SM 8

namespace {

// RunEndBuffer::get_physical_index (run.rs:232-241) of absolute logical row x: the number of run ends <= x, clamped to a
// physical run so that a malformed buffer is never read past its end
template <class R>
__device__ int64_t physical_index(const R *re, int64_t n, int64_t x) {
  int64_t lo = 0, hi = n;
  while (lo < hi) {
    const int64_t mid = lo + ((hi - lo) >> 1);
    if ((int64_t)__ldg(re + mid) <= x) lo = mid + 1;
    else hi = mid;
  }
  return lo < n ? lo : (n > 0 ? n - 1 : 0);
}

// start / end physical index of the slice -> res[RES_AUX1] / res[RES_AUX2] (one thread)
template <class R>
__global__ void k_ree_bounds(const R *re, int64_t n, int64_t offset, int64_t len, unsigned long long *res) {
  int64_t start = 0, end = 0;
  if (len > 0) {
    if (offset != 0) start = physical_index(re, n, offset);
    end = (int64_t)__ldg(re + n - 1) == offset + len ? n - 1 : physical_index(re, n, offset + len - 1);
  }
  res[RES_AUX1] = (unsigned long long)start;
  res[RES_AUX2] = (unsigned long long)end;
}

// Selected rows of the plan in [0, x), x <= plan len: the tile's output offset plus the popcounts of the tile's words below
// x (at most 16 words) and of the partial word.
__device__ __forceinline__ int64_t plan_rank(const uint64_t *__restrict__ mask, const uint64_t *__restrict__ tile_off, int64_t x) {
  int64_t r = (int64_t)__ldg(tile_off + (x >> 10));
  const int64_t w = x >> 6;
  for (int64_t k = (x >> 10) << 4; k < w; ++k) r += __popcll(__ldg(mask + k));
  if (x & 63) r += __popcll(__ldg(mask + w) & ((1ull << (x & 63)) - 1ull));
  return r;
}

// A lane owns physical run start + j, clipped to end = min(run_end - offset, plen) (saturating at 0); it takes its
// predecessor's rank from the lane below, lane 0 computes it. keep = a selected row in [previous end, end).
template <class R>
__global__ void __launch_bounds__(RE_THREADS) k_ree_filter_runs(const R *__restrict__ re, int64_t start, int64_t pl, int64_t offset,
                                                                int64_t plen, const uint64_t *__restrict__ mask,
                                                                const uint64_t *__restrict__ tile_off, uint32_t *__restrict__ keep,
                                                                R *__restrict__ ranks) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  auto clipped_rank = [&](int64_t p) {
    int64_t e = (int64_t)__ldg(re + p) - offset;
    e = e < 0 ? 0 : (e < plen ? e : plen);
    return plan_rank(mask, tile_off, e);
  };
  for (int64_t j0 = warp * 32; j0 < pl; j0 += nwarps * 32) {
    const int64_t j = j0 + lane;
    const int64_t rk = j < pl ? clipped_rank(start + j) : 0;
    int64_t prev = __shfl_up_sync(ACU_FULL_MASK, rk, 1);
    if (lane == 0) prev = j0 == 0 ? 0 : clipped_rank(start + j0 - 1);
    const unsigned bits = __ballot_sync(ACU_FULL_MASK, j < pl && rk > prev);
    if (lane == 0) keep[j0 >> 5] = bits;
    if (j < pl) ranks[j] = (R)rk;
  }
}

// Output row j's physical run: the first run whose end exceeds offset + ToIndices(idx[j]), written to phys[j + 1] (the
// run-end plan selects position q = j + 1 for a run ending at row j). The largest index value -> res[RES_AUX0].
template <class R, class IdxT>
__global__ void __launch_bounds__(RE_THREADS) k_ree_take_map(const R *__restrict__ re, int64_t n, int64_t offset, const void *idx, int kind,
                                                             int64_t m, IdxT *__restrict__ phys, unsigned long long *res) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  unsigned long long mx = 0;
  for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < m; j += stride) {
    const uint64_t x = ld_index(idx, kind, j);
    mx = x > mx ? x : mx;
    phys[j + 1] = (IdxT)physical_index(re, n, (int64_t)(x + (uint64_t)offset));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long y = __shfl_xor_sync(ACU_FULL_MASK, mx, o);
    mx = y > mx ? y : mx;
  }
  if ((threadIdx.x & 31) == 0 && mx) atomicMax(res + RES_AUX0, mx);
}

// make_comparator's equality of two physical rows (SortOptions::default(): two nulls are equal, a null never equals a value)
template <class V>
struct NullsThen {
  V v;
  const uint8_t *valid;
  int64_t voff;
  __device__ __forceinline__ bool eq(int64_t a, int64_t b) const {
    if (valid) {
      const uint32_t va = ld_bit(valid, voff + a), vb = ld_bit(valid, voff + b);
      if (!(va & vb)) return va == vb;
    }
    return v.eq(a, b);
  }
};
template <class T>
struct FixedEq {  // integers, decimals and floats under total_cmp: equal iff the bits are
  const T *v;
  __device__ __forceinline__ bool eq(int64_t a, int64_t b) const { return ldg_elem(v + a) == ldg_elem(v + b); }
};
struct BoolEq {
  const uint8_t *bits;
  int64_t off;
  __device__ __forceinline__ bool eq(int64_t a, int64_t b) const { return ld_bit(bits, off + a) == ld_bit(bits, off + b); }
};
struct BytesEq {
  BytesOperand s;
  __device__ __forceinline__ bool eq(int64_t a, int64_t b) const {
    const BytesItem x = s.item(a), y = s.item(b);
    return bytes_eq(x.p, x.len, y.p, y.len);
  }
};
struct ViewEq {
  ViewOperand s;
  __device__ __forceinline__ bool eq(int64_t a, int64_t b) const { return view_is_eq(s, s.view(a), s.views + a, s, s.view(b), s.views + b); }
};

// Bit q of [0, M] (ballot-packed u32 words): q ends a run of the output. phys[q] is the physical run of output row q - 1.
template <class Src, class IdxT>
__global__ void __launch_bounds__(RE_THREADS) k_ree_run_ends(const IdxT *__restrict__ phys, int64_t m, Src src, uint32_t *__restrict__ bits) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t q0 = warp * 32; q0 <= m; q0 += nwarps * 32) {
    const int64_t q = q0 + lane;
    bool end = q == m;
    if (q >= 1 && q < m) {
      const IdxT a = phys[q + 1], b = phys[q];
      end = a != b && !src.eq((int64_t)a, (int64_t)b);
    }
    const unsigned w = __ballot_sync(ACU_FULL_MASK, end);
    if (lane == 0) bits[q0 >> 5] = w;
  }
}

__global__ void __launch_bounds__(RE_THREADS) k_ree_narrow16(const uint32_t *__restrict__ src, int64_t n, int16_t *__restrict__ dst) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) dst[i] = (int16_t)src[i];
}

int re_grid(const acu_ctx *ctx, int64_t threads) { return acu_grid(ctx, (threads + RE_THREADS - 1) / RE_THREADS, RE_PER_SM); }

template <class F>
acu_status with_run_end(acu_dtype dt, F &&f) {
  switch (dt) {
    case ACU_I16: return f(int16_t());
    case ACU_I32: return f(int32_t());
    default: return f(int64_t());
  }
}

acu_status check_run_array(acu_ctx *ctx, const acu_run_array *r) {
  const acu_dtype dt = (acu_dtype)r->run_end_dtype;
  if (dt != ACU_I16 && dt != ACU_I32 && dt != ACU_I64)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "run ends must be Int16, Int32 or Int64, got %s", acu_dtype_name(dt));
  const int w = acu_dtype_size(dt);
  if ((uintptr_t)r->run_ends % (uintptr_t)w != 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "run ends must be %d-byte aligned", w);
  if (r->offset < 0 || r->len < 0 || r->n_runs < 0)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "RunArray offset, length and run count must be >= 0");
  if (r->n_runs == 0 && r->len > 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "a RunArray of length > 0 needs a run");
  return ACU_OK;
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

}  // namespace

extern "C" acu_status acu_filter_run_end(acu_ctx *ctx, const acu_filter_plan *plan, const acu_run_array *ree, void *out_run_ends,
                                         int64_t *out_runs, int64_t *out_values_start, acu_filter_plan **out_values_plan) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  *out_runs = 0;
  *out_values_start = 0;
  *out_values_plan = nullptr;
  ACU_TRY(check_run_array(ctx, ree));
  const int64_t plen = acu_filter_plan_len(plan);
  if (plen > ree->len)  // filter.rs:536-542
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Filter predicate of length %lld is larger than target array of length %lld",
                    (long long)plen, (long long)ree->len);
  const int32_t strategy = acu_filter_plan_strategy(plan);
  if (strategy == ACU_FILTER_NONE || strategy == ACU_FILTER_ALL) return ACU_OK;  // filter.rs:545-546, the caller's
  return with_run_end((acu_dtype)ree->run_end_dtype, [&](auto r0) -> acu_status {
    using R = decltype(r0);
    const R *re = static_cast<const R *>(ree->run_ends);
    ACU_TRY(acu_res_reset(ctx));
    ACU_LAUNCH_TIMED(ctx, ACU_K_FILTER_PLAN, k_ree_bounds<R>, 1, 1, 0, re, ree->n_runs, ree->offset, ree->len, acu_dres(ctx, 0));
    ACU_TRY(acu_res_fetch(ctx));
    const int64_t start = (int64_t)acu_hres(ctx, 0)[RES_AUX1];
    int64_t end = (int64_t)acu_hres(ctx, 0)[RES_AUX2];
    if (end < start) end = start;  // only a malformed buffer
    const int64_t pl = end - start + 1;
    DevBufs bufs{ctx};
    void *keep = nullptr, *ranks = nullptr;
    ACU_TRY(bufs.get((size_t)(pl + 63) / 64 * 8 + 16, &keep));
    ACU_TRY(bufs.get((size_t)pl * sizeof(R) + 16, &ranks));
    ACU_LAUNCH_TIMED(ctx, ACU_K_FILTER_PLAN, k_ree_filter_runs<R>, re_grid(ctx, (pl + 31) / 32 * 32), RE_THREADS, 0, re, start, pl, ree->offset,
                     plen, acu_plan_mask(plan), acu_plan_tile_off(plan), static_cast<uint32_t *>(keep), static_cast<R *>(ranks));
    acu_array kp{};
    kp.values = keep;
    kp.len = pl;
    acu_filter_plan *vplan = nullptr;
    ACU_TRY(acu_filter_plan_create(ctx, &kp, &vplan));
    acu_array ra{};
    ra.values = ranks;
    ra.len = pl;
    acu_array_out o{};
    o.values = out_run_ends;
    const acu_status st = acu_filter_primitive(ctx, vplan, (int32_t)sizeof(R), &ra, &o);
    acu_kstats_drain(ctx);
    if (st != ACU_OK) {
      acu_filter_plan_destroy(ctx, vplan);
      return st;
    }
    *out_runs = acu_filter_plan_count(vplan);
    *out_values_start = start;
    *out_values_plan = vplan;
    return ACU_OK;
  });
}

extern "C" acu_status acu_take_run_end(acu_ctx *ctx, const acu_run_array *ree, const acu_run_values *values, const acu_array *indices,
                                       acu_dtype index_dtype, int32_t check_bounds, void *out_run_ends, void *out_value_indices,
                                       int64_t *out_runs) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  *out_runs = 0;
  ACU_TRY(check_run_array(ctx, ree));
  const int vk = values->kind;
  const int w = values->width;
  if (vk == ACU_RUN_VALUES_FIXED && w != 1 && w != 2 && w != 4 && w != 8 && w != 16)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "fixed-width values must be 1, 2, 4, 8 or 16 bytes wide, got %d", w);
  if (vk == ACU_RUN_VALUES_BYTES) ACU_TRY(acu_offset_width_check(ctx, w));
  if (vk < ACU_RUN_VALUES_FIXED || vk > ACU_RUN_VALUES_NESTED)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "unknown RunEndEncoded values kind %d", vk);
  const int kind = acu_take_index_kind(index_dtype);
  if (kind < 0)  // take.rs:103
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Take only supported for integers, got %s", acu_dtype_name(index_dtype));
  const int64_t m = indices->len;
  acu_status st = ACU_OK;
  const int64_t inc = m > 0 ? acu_resolve_null_count(ctx, indices, &st) : 0;
  if (m > 0) ACU_TRY(st);
  if (check_bounds) ACU_TRY(acu_take_check_bounds(ctx, indices, index_dtype, indices->validity && inc > 0, ree->len));
  if (m == 0) return ACU_OK;
  const bool wide = kind == 5;  // ToIndices: Int64 / UInt64 -> UInt64, every other index type -> UInt32
  if (!wide && ree->n_runs > (int64_t)UINT32_MAX + 1)
    return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, -1, 0, 0, 0, "take of more than 2^32 runs with UInt32 indices is not yet implemented");
  const int iw = wide ? 8 : 4;
  return with_run_end((acu_dtype)ree->run_end_dtype, [&](auto r0) -> acu_status {
    using R = decltype(r0);
    const R *re = static_cast<const R *>(ree->run_ends);
    DevBufs bufs{ctx};
    void *phys = nullptr, *bits = nullptr;
    ACU_TRY(bufs.get((size_t)(m + 1) * iw + 16, &phys));
    ACU_TRY(bufs.get((size_t)(m + 1 + 63) / 64 * 8 + 16, &bits));
    ACU_TRY(acu_res_reset(ctx));
    const int grid = re_grid(ctx, m);
    if (wide)
      ACU_LAUNCH_TIMED(ctx, ACU_K_TAKE, (k_ree_take_map<R, uint64_t>), grid, RE_THREADS, 0, re, ree->n_runs, ree->offset, indices->values, kind, m,
                       static_cast<uint64_t *>(phys), acu_dres(ctx, 0));
    else
      ACU_LAUNCH_TIMED(ctx, ACU_K_TAKE, (k_ree_take_map<R, uint32_t>), grid, RE_THREADS, 0, re, ree->n_runs, ree->offset, indices->values, kind, m,
                       static_cast<uint32_t *>(phys), acu_dres(ctx, 0));
    ACU_TRY(acu_res_fetch(ctx));
    const unsigned long long mx = acu_hres(ctx, 0)[RES_AUX0];
    if (mx >= (unsigned long long)ree->len)  // run_array.rs:343-356
      return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, mx, 0, (uint64_t)ree->len, "Logical index %llu is out of bounds for RunArray of length %lld",
                      mx, (long long)ree->len);
    // make_comparator comes next in take_run (take.rs:963-967): here nested values are not compared yet
    if (vk == ACU_RUN_VALUES_NESTED)
      return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, -1, 0, 0, 0, "take of a RunEndEncoded column with nested values is not yet implemented");
    // the last run end pushed is M, the largest: some from_usize(..).unwrap() fails iff M does not fit the run-end type
    if (m > (int64_t)std::numeric_limits<R>::max())
      return acu_fail(ctx, ACU_ERR_PANIC_OUT_OF_BOUNDS, -1, 0, 0, (uint64_t)m, "called `Option::unwrap()` on a `None` value");
    // the run-end bitmap, typed on the values child
    void *table = nullptr;
    if (vk == ACU_RUN_VALUES_VIEW) ACU_TRY(bufs.get(acu_view_table_bytes(&values->view) + 16, &table));
    const int bgrid = re_grid(ctx, (m + 1 + 31) / 32 * 32);
    uint32_t *bw = static_cast<uint32_t *>(bits);
    auto launch = [&](auto src) -> acu_status {
      if (wide)
        ACU_LAUNCH_TIMED(ctx, ACU_K_TAKE, (k_ree_run_ends<decltype(src), uint64_t>), bgrid, RE_THREADS, 0, static_cast<const uint64_t *>(phys), m, src, bw);
      else
        ACU_LAUNCH_TIMED(ctx, ACU_K_TAKE, (k_ree_run_ends<decltype(src), uint32_t>), bgrid, RE_THREADS, 0, static_cast<const uint32_t *>(phys), m, src, bw);
      return ACU_OK;
    };
    const acu_array &a = values->array;
    if (vk == ACU_RUN_VALUES_FIXED) {
      const void *v = a.values;
      if (w == 1) ACU_TRY(launch(NullsThen<FixedEq<uint8_t>>{{static_cast<const uint8_t *>(v)}, a.validity, a.validity_offset}));
      else if (w == 2) ACU_TRY(launch(NullsThen<FixedEq<uint16_t>>{{static_cast<const uint16_t *>(v)}, a.validity, a.validity_offset}));
      else if (w == 4) ACU_TRY(launch(NullsThen<FixedEq<uint32_t>>{{static_cast<const uint32_t *>(v)}, a.validity, a.validity_offset}));
      else if (w == 8) ACU_TRY(launch(NullsThen<FixedEq<uint64_t>>{{static_cast<const uint64_t *>(v)}, a.validity, a.validity_offset}));
      else {
        if ((uintptr_t)v % 16 != 0) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "16-byte values must be 16-byte aligned");
        ACU_TRY(launch(NullsThen<FixedEq<unsigned __int128>>{{static_cast<const unsigned __int128 *>(v)}, a.validity, a.validity_offset}));
      }
    } else if (vk == ACU_RUN_VALUES_BOOLEAN) {
      ACU_TRY(launch(NullsThen<BoolEq>{{static_cast<const uint8_t *>(a.values), a.values_offset}, a.validity, a.validity_offset}));
    } else if (vk == ACU_RUN_VALUES_BYTES) {
      const acu_bytes_array &b = values->bytes;
      ACU_TRY(launch(NullsThen<BytesEq>{{BytesOperand{b.offsets, b.data, w}}, b.nulls.validity, b.nulls.validity_offset}));
    } else {
      ViewOperand vo{};
      ACU_TRY(acu_view_operand(ctx, &values->view, table, &vo));
      ACU_TRY(launch(NullsThen<ViewEq>{{vo}, values->view.nulls.validity, values->view.nulls.validity_offset}));
    }
    acu_array ba{};
    ba.values = bits;
    ba.len = m + 1;
    acu_filter_plan *plan = nullptr;
    ACU_TRY(acu_filter_plan_create(ctx, &ba, &plan));
    struct PlanGuard {
      acu_ctx *c;
      acu_filter_plan *p;
      ~PlanGuard() { acu_filter_plan_destroy(c, p); }
    } guard{ctx, plan};
    const int64_t runs = acu_filter_plan_count(plan);
    // run ends: the selected positions themselves
    if (sizeof(R) == 2) {
      void *tmp = nullptr;
      ACU_TRY(bufs.get((size_t)runs * 4 + 16, &tmp));
      ACU_TRY(acu_filter_plan_indices(ctx, plan, ACU_U32, tmp));
      ACU_LAUNCH_TIMED(ctx, ACU_K_TAKE, k_ree_narrow16, re_grid(ctx, runs), RE_THREADS, 0, static_cast<const uint32_t *>(tmp), runs,
                       static_cast<int16_t *>(out_run_ends));
    } else {
      ACU_TRY(acu_filter_plan_indices(ctx, plan, sizeof(R) == 4 ? ACU_U32 : ACU_U64, out_run_ends));
    }
    // value indices: phys[q] (the physical run of output row q - 1) at every run end q
    acu_array pa{};
    pa.values = phys;
    pa.len = m + 1;
    acu_array_out o{};
    o.values = out_value_indices;
    ACU_TRY(acu_filter_primitive(ctx, plan, iw, &pa, &o));
    acu_kstats_drain(ctx);
    *out_runs = runs;
    return ACU_OK;
  });
}
