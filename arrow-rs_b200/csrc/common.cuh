// common.cuh — shared device/host helpers for the sm_90a arrow::compute kernels.
//
// Layout conventions (arrow-buffer, see include/arrow_cuda.h): LSB-first bitmaps with an
// arbitrary bit offset on INPUT, bit offset 0 and whole-u64-word stores on OUTPUT.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <functional>
#include <unordered_map>
#include <vector>

#include "../../include/arrow_cuda.h"

#define ACU_FULL_MASK 0xffffffffu

// ---------------------------------------------------------------------------------------
// Host-side context
// ---------------------------------------------------------------------------------------
enum {  // slots of the device/pinned result block
  RES_COUNT = 0,     // popcounts / valid counts
  RES_ERR_INDEX = 1, // lowest failing row (atomicMin), init UINT64_MAX
  RES_AUX0 = 2,
  RES_AUX1 = 3,
  RES_AUX2 = 4,
  RES_AUX3 = 5,
  RES_ERR2 = 6,      // second lowest-failing-row slot (atomicMin), init UINT64_MAX
  RES_SLOTS = 16,
  RES_BLOCKS = 64    // result blocks: one per column of a record-batch call (block 0 for single-array calls)
};

struct acu_ctx {
  int device = 0;
  int sm_count = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
  acu_error_detail err{};
  int64_t launches = 0;
  int64_t bytes_allocated = 0;
  std::unordered_map<void *, size_t> allocs;
  std::unordered_map<const void *, int> occupancy;  // resident CTAs per SM, per kernel
  unsigned long long *d_res = nullptr;  // RES_BLOCKS x RES_SLOTS u64 on the device
  unsigned long long *h_res = nullptr;  // pinned mirror
  bool res_clean = false;               // the result blocks hold their initial values (see acu_res_reset_n)
  int res_dirty_blocks = RES_BLOCKS;
  // stream-ordered section (acu_async_begin ... acu_results_fetch): calls enqueue only, one result block each
  bool async_on = false;
  int async_blocks = 0;
  std::vector<std::function<acu_status(const unsigned long long *)>> async_fin;  // finalisers, in call order
  std::vector<int> async_blk;
  void *d_scratch = nullptr;            // grows on demand (block partials, scans)
  size_t scratch_bytes = 0;
  // NCCL (loaded with dlopen, see comm.cu)
  void *nccl_comm = nullptr;
  int rank = 0, world = 1;
  // timers (acu_timer_*_slot) and per-kernel-class device time (acu_kernel_stats)
  cudaEvent_t tev[ACU_TIMER_SLOTS][2] = {};
  static constexpr int KEV_PAIRS = 64;
  cudaEvent_t kev[KEV_PAIRS][2] = {};
  int kev_class[KEV_PAIRS] = {};
  int kev_pending = 0;
  double kstat_ms[ACU_K_CLASSES] = {};
  int64_t kstat_n[ACU_K_CLASSES] = {};
};

// Drain the timed-launch events (call after the stream has been synchronised).
void acu_kstats_drain(acu_ctx *ctx);
// Begin / end a timed kernel launch of class `cls` (records a CUDA event pair on the stream).
int acu_kstats_begin(acu_ctx *ctx, int cls);
void acu_kstats_end(acu_ctx *ctx, int slot);

acu_status acu_fail(acu_ctx *ctx, acu_status st, int64_t index, uint64_t lhs, uint64_t rhs,
                    uint64_t len, const char *fmt, ...) __attribute__((format(printf, 7, 8)));
acu_status acu_cuda_fail(acu_ctx *ctx, cudaError_t e, const char *what);
acu_status acu_scratch(acu_ctx *ctx, size_t bytes, void **out);  // >= bytes, 256-B aligned
acu_status acu_res_reset(acu_ctx *ctx);                          // zero slots, ERR_INDEX = ~0
acu_status acu_res_fetch(acu_ctx *ctx);                          // D2H + stream sync
acu_status acu_res_reset_n(acu_ctx *ctx, int blocks);            // the same for the first `blocks` result blocks
acu_status acu_res_fetch_n(acu_ctx *ctx, int blocks);
// One call = acu_call_begin (its result block: block 0 after a reset, or the next free block of an async section)
// ... kernels ... acu_call_end(fin): synchronous mode fetches and runs `fin` on the pinned block now; inside an async
// section `fin` is queued for acu_results_fetch. `fin` turns the block into null counts / errors.
int acu_call_begin(acu_ctx *ctx, acu_status *st);
acu_status acu_call_end(acu_ctx *ctx, int block, std::function<acu_status(const unsigned long long *)> fin);
static inline unsigned long long *acu_dres(acu_ctx *ctx, int block) { return ctx->d_res + (size_t)block * RES_SLOTS; }
static inline const unsigned long long *acu_hres(const acu_ctx *ctx, int block) { return ctx->h_res + (size_t)block * RES_SLOTS; }
int64_t acu_resolve_null_count(acu_ctx *ctx, const acu_array *a, acu_status *st);

#define ACU_CUDA(ctx, expr)                                         \
  do {                                                              \
    cudaError_t _e = (expr);                                        \
    if (_e != cudaSuccess) return acu_cuda_fail((ctx), _e, #expr);  \
  } while (0)

// Every C-ABI entry point first makes the ctx's device current on the calling host thread
// (a ctx may be driven from any thread; new threads default to device 0).
#define ACU_ENTER(ctx)                                                                      \
  do {                                                                                      \
    cudaError_t _e = cudaSetDevice((ctx)->device);                                          \
    if (_e != cudaSuccess) return acu_cuda_fail((ctx), _e, "cudaSetDevice");                \
  } while (0)

#define ACU_TRY(expr)                  \
  do {                                 \
    acu_status _s = (expr);            \
    if (_s != ACU_OK) return _s;       \
  } while (0)

// Launch on the ctx stream, count it, surface launch-config errors immediately.
#define ACU_LAUNCH(ctx, kernel, grid, block, smem, ...)                            \
  do {                                                                             \
    kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);               \
    (ctx)->launches++;                                                             \
    cudaError_t _e = cudaGetLastError();                                           \
    if (_e != cudaSuccess) return acu_cuda_fail((ctx), _e, "launch " #kernel);     \
  } while (0)

// Same as ACU_LAUNCH, bracketed by an event pair accumulated into class `cls`.
#define ACU_LAUNCH_TIMED(ctx, cls, kernel, grid, block, smem, ...)                 \
  do {                                                                             \
    int _slot = acu_kstats_begin((ctx), (cls));                                    \
    kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);               \
    (ctx)->launches++;                                                             \
    cudaError_t _e = cudaGetLastError();                                           \
    acu_kstats_end((ctx), _slot);                                                  \
    if (_e != cudaSuccess) return acu_cuda_fail((ctx), _e, "launch " #kernel);     \
  } while (0)

static inline int acu_dtype_size(acu_dtype t) {
  switch (t) {
    case ACU_I8: case ACU_U8: return 1;
    case ACU_I16: case ACU_U16: return 2;
    case ACU_I32: case ACU_U32: case ACU_F32: return 4;
    default: return 8;
  }
}
static inline bool acu_dtype_is_float(acu_dtype t) { return t == ACU_F32 || t == ACU_F64; }
static inline bool acu_dtype_is_signed(acu_dtype t) { return t <= ACU_I64; }
static inline const char *acu_dtype_name(acu_dtype t) {
  static const char *n[] = {"Int8", "Int16", "Int32", "Int64", "UInt8", "UInt16", "UInt32", "UInt64", "Float32", "Float64", "Int128"};
  return (int)t >= 0 && (int)t <= (int)ACU_I128 ? n[(int)t] : "unknown";
}

// Persistent-style grid: enough CTAs to fill every SM `per_sm` times, never more than the work.
static inline int acu_grid(const acu_ctx *ctx, int64_t work_items, int per_sm) {
  int64_t g = (int64_t)ctx->sm_count * per_sm;
  if (g > work_items) g = work_items;
  if (g < 1) g = 1;
  return (int)g;
}

#ifdef __CUDACC__
// Persistent grid sized from the kernel's real occupancy: SMs x resident CTAs per SM
// (one full wave, grid-stride inside), never more CTAs than work items.
template <class K>
static inline int acu_wave_grid(acu_ctx *ctx, K kernel, int block, size_t smem, int64_t work_blocks) {
  const void *key = reinterpret_cast<const void *>(kernel);
  auto it = ctx->occupancy.find(key);
  int per_sm;
  if (it == ctx->occupancy.end()) {
    per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, block, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
    ctx->occupancy[key] = per_sm;
  } else {
    per_sm = it->second;
  }
  // 8 waves of CTAs: the hardware scheduler evens out per-SM imbalance (tools/arith_sweep.cu compares
  // waves and occupancy points on the streaming add)
  return acu_grid(ctx, work_blocks, per_sm * 8);
}

// ---------------------------------------------------------------------------------------
// Device helpers
// ---------------------------------------------------------------------------------------

// 64 bits of a bitmap starting at absolute bit position `pos` (relative to `base`);
// bits at positions >= end read as zero. Uses aligned 8-byte loads (base may be any byte
// address; the enclosing aligned words are always inside the allocation granule).
__device__ __forceinline__ uint64_t ld_bits64(const uint8_t *__restrict__ base, int64_t pos, int64_t end) {
  int64_t n = end - pos;
  if (n <= 0) return 0ull;
  uintptr_t addr = (uintptr_t)base + (uintptr_t)(pos >> 3);
  uintptr_t al = addr & ~(uintptr_t)7;
  unsigned shift = (unsigned)((addr & 7) << 3) + (unsigned)(pos & 7);
  const uint64_t *p = reinterpret_cast<const uint64_t *>(al);
  uint64_t w = __ldg(p) >> shift;
  if (shift != 0 && (int64_t)(64 - shift) < n) w |= __ldg(p + 1) << (64 - shift);
  if (n < 64) w &= (~0ull) >> (64 - n);
  return w;
}

// 32 bits starting at `pos`, zero past `end`.
__device__ __forceinline__ uint32_t ld_bits32(const uint8_t *__restrict__ base, int64_t pos, int64_t end) {
  int64_t n = end - pos;
  if (n <= 0) return 0u;
  uintptr_t addr = (uintptr_t)base + (uintptr_t)(pos >> 3);
  uintptr_t al = addr & ~(uintptr_t)3;
  unsigned shift = (unsigned)((addr & 3) << 3) + (unsigned)(pos & 7);
  const uint32_t *p = reinterpret_cast<const uint32_t *>(al);
  uint32_t w = __ldg(p) >> shift;
  if (shift != 0 && (int64_t)(32 - shift) < n) w |= __ldg(p + 1) << (32 - shift);
  if (n < 32) w &= (~0u) >> (32 - n);
  return w;
}

__device__ __forceinline__ uint32_t ld_bit(const uint8_t *__restrict__ base, int64_t pos) {
  return (__ldg(base + (pos >> 3)) >> (pos & 7)) & 1u;
}

// Streaming 128-bit accesses: the hot kernels touch every byte exactly once, so bypass
// L1 allocation (ld.global.nc.L1::no_allocate) and mark stores streaming (st.global.cs).
__device__ __forceinline__ uint4 ld_stream16(const void *p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream16(void *p, uint4 v) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ uint64_t ld_stream8(const void *p) {
  uint64_t r;
  asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(r) : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream8(void *p, uint64_t v) {
  asm volatile("st.global.cs.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// __ldg of one element of any native width; __int128 (Decimal128, 16-byte aligned) has no __ldg overload.
template <class T> __device__ __forceinline__ T ldg_elem(const T *p) {
  if constexpr (sizeof(T) == 16) {
    const longlong2 v = __ldg(reinterpret_cast<const longlong2 *>(p));
    T r;
    memcpy(&r, &v, 16);
    return r;
  } else {
    return __ldg(p);
  }
}

template <class T> __device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(ACU_FULL_MASK, v, o);
  return v;
}

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

// IEEE-754 totalOrder keys (Rust f64::total_cmp; arrow-array/src/arithmetic.rs:400-410)
__device__ __forceinline__ int64_t total_key(double x) {
  int64_t b = __double_as_longlong(x);
  return b ^ (int64_t)((uint64_t)(b >> 63) >> 1);
}
__device__ __forceinline__ int32_t total_key(float x) {
  int32_t b = __float_as_int(x);
  return b ^ (int32_t)((uint32_t)(b >> 31) >> 1);
}
#endif  // __CUDACC__
