// ctx.cu — acu_ctx (device + stream + scratch), DeviceBuffer allocation, copies, timing,
// error detail, synthetic input generators, and the operand front end of the Utf8 / Binary / view entry points
// (internal.cuh). Boundary: include/arrow_cuda.h.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>

#include <new>

#include "bytes_cmp.cuh"
#include "internal.cuh"

acu_status acu_fail(acu_ctx *ctx, acu_status st, int64_t index, uint64_t lhs, uint64_t rhs,
                    uint64_t len, const char *fmt, ...) {
  acu_error_detail &e = ctx->err;
  e.status = st;
  e.cuda_error = 0;
  e.index = index;
  e.lhs_bits = lhs;
  e.rhs_bits = rhs;
  e.len = len;
  // message = Display of the ArrowError variant (arrow-schema/src/error.rs:96-137)
  const char *prefix = "";
  switch (st) {
    case ACU_ERR_INVALID_ARGUMENT: prefix = "Invalid argument error: "; break;
    case ACU_ERR_COMPUTE: prefix = "Compute error: "; break;
    case ACU_ERR_ARITHMETIC_OVERFLOW: prefix = "Arithmetic overflow: "; break;
    case ACU_ERR_OFFSET_OVERFLOW: prefix = "Offset overflow error: "; break;
    case ACU_ERR_CAST: prefix = "Cast error: "; break;
    case ACU_ERR_NOT_YET_IMPLEMENTED: prefix = "Not yet implemented: "; break;
    case ACU_ERR_IPC: prefix = "Ipc error: "; break;
    case ACU_ERR_PARSE: prefix = "Parser error: "; break;
    default: break;
  }
  size_t n = strlen(prefix);
  memcpy(e.message, prefix, n);
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(e.message + n, sizeof(e.message) - n, fmt, ap);
  va_end(ap);
  return st;
}

acu_status acu_cuda_fail(acu_ctx *ctx, cudaError_t e, const char *what) {
  acu_status st = (e == cudaErrorMemoryAllocation) ? ACU_ERR_OUT_OF_MEMORY : ACU_ERR_CUDA;
  acu_fail(ctx, st, -1, 0, 0, 0, "CUDA error %d (%s) in %s", (int)e, cudaGetErrorString(e), what);
  ctx->err.cuda_error = (int32_t)e;
  cudaGetLastError();  // clear sticky-less errors
  return st;
}

acu_status acu_scratch(acu_ctx *ctx, size_t bytes, void **out) {
  if (bytes > ctx->scratch_bytes) {
    size_t want = (bytes + (1u << 20)) & ~(size_t)((1u << 20) - 1);
    if (ctx->d_scratch) {
      ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
      ACU_CUDA(ctx, cudaFree(ctx->d_scratch));
      ctx->d_scratch = nullptr;
      ctx->scratch_bytes = 0;
    }
    ACU_CUDA(ctx, cudaMalloc(&ctx->d_scratch, want));
    ctx->scratch_bytes = want;
  }
  *out = ctx->d_scratch;
  return ACU_OK;
}

acu_status acu_sync_only(acu_ctx *ctx) {
  if (ctx->async_on)
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0,
                    "this entry point synchronises and is not available between acu_async_begin and acu_results_fetch");
  return ACU_OK;
}

acu_status acu_offset_width_check(acu_ctx *ctx, int32_t offset_bytes) {
  if (offset_bytes != 4 && offset_bytes != 8) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "offset width must be 4 or 8");
  return ACU_OK;
}

size_t acu_view_table_bytes(const acu_view_array *a) {
  return ((size_t)(a->n_buffers > 0 ? a->n_buffers : 0) * sizeof(void *) + 255) & ~(size_t)255;
}

acu_status acu_view_operand(acu_ctx *ctx, const acu_view_array *a, void *table_space, ViewOperand *out) {
  const uint8_t *const *table = nullptr;
  if (a->n_buffers > 0) {
    ACU_CUDA(ctx, cudaMemcpyAsync(table_space, a->buffers, (size_t)a->n_buffers * sizeof(void *), cudaMemcpyHostToDevice, ctx->stream));
    table = static_cast<const uint8_t *const *>(table_space);
  }
  *out = ViewOperand{static_cast<const uint4 *>(a->views), table, a->n_buffers};
  return ACU_OK;
}

__global__ void k_res_reset(unsigned long long *res, int slots) {
  int i = threadIdx.x;
  if (i < slots) res[i] = ((i % RES_SLOTS) == RES_ERR_INDEX || (i % RES_SLOTS) == RES_ERR2) ? ~0ull : 0ull;
}

// The result blocks are kept CLEAN between calls: every fetch queues their re-initialisation right behind its D2H copy
// (off the critical path of the next call), so a call's "reset" is normally free — no launch in front of its kernels.
// res_clean is dropped by the first reset after a fetch; a call that failed between its reset and its fetch leaves
// res_clean false and the next reset launches k_res_reset itself. res_dirty_blocks = blocks possibly written since.
acu_status acu_res_reset_n(acu_ctx *ctx, int blocks) {
  ACU_TRY(acu_sync_only(ctx));  // entry points that have not been split into enqueue + finalise would synchronise here
  if (blocks < 1) blocks = 1;
  if (blocks > RES_BLOCKS) blocks = RES_BLOCKS;
  if (!ctx->res_clean) {
    const int n = blocks > ctx->res_dirty_blocks ? blocks : ctx->res_dirty_blocks;
    ACU_LAUNCH(ctx, k_res_reset, 1, n * RES_SLOTS, 0, ctx->d_res, n * RES_SLOTS);
  }
  ctx->res_clean = false;
  ctx->res_dirty_blocks = blocks;
  return ACU_OK;
}

acu_status acu_res_fetch_n(acu_ctx *ctx, int blocks) {
  if (blocks < 1) blocks = 1;
  if (blocks > RES_BLOCKS) blocks = RES_BLOCKS;
  ACU_CUDA(ctx, cudaMemcpyAsync(ctx->h_res, ctx->d_res, (size_t)blocks * RES_SLOTS * sizeof(unsigned long long),
                                cudaMemcpyDeviceToHost, ctx->stream));
  const int n = blocks > ctx->res_dirty_blocks ? blocks : ctx->res_dirty_blocks;
  ACU_LAUNCH(ctx, k_res_reset, 1, n * RES_SLOTS, 0, ctx->d_res, n * RES_SLOTS);  // stream-ordered behind the copy
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  ctx->res_clean = true;
  ctx->res_dirty_blocks = 0;
  acu_kstats_drain(ctx);
  return ACU_OK;
}

int acu_call_begin(acu_ctx *ctx, acu_status *st) {
  if (!ctx->async_on) {
    *st = acu_res_reset(ctx);
    return 0;
  }
  if (ctx->async_blocks >= RES_BLOCKS) {
    *st = acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "more than %d calls queued in one async section", (int)RES_BLOCKS);
    return 0;
  }
  *st = ACU_OK;
  return ctx->async_blocks++;
}

acu_status acu_call_end(acu_ctx *ctx, int block, std::function<acu_status(const unsigned long long *)> fin) {
  if (!ctx->async_on) {
    ACU_TRY(acu_res_fetch(ctx));
    return fin(acu_hres(ctx, 0));
  }
  ctx->async_fin.push_back(std::move(fin));
  ctx->async_blk.push_back(block);
  return ACU_OK;
}

extern "C" acu_status acu_async_begin(acu_ctx *ctx) {
  ACU_ENTER(ctx);
  if (ctx->async_on) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "acu_async_begin: a section is already open");
  ACU_TRY(acu_res_reset_n(ctx, RES_BLOCKS));  // every block clean (free when the last fetch left them so)
  ctx->async_on = true;
  ctx->async_blocks = 0;
  ctx->async_fin.clear();
  ctx->async_blk.clear();
  return ACU_OK;
}

extern "C" acu_status acu_results_fetch(acu_ctx *ctx) {
  ACU_ENTER(ctx);
  if (!ctx->async_on) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "acu_results_fetch: no async section is open");
  ctx->async_on = false;
  acu_status first = acu_res_fetch_n(ctx, ctx->async_blocks > 0 ? ctx->async_blocks : 1);  // ONE D2H copy + ONE synchronisation
  acu_error_detail first_err = ctx->err;
  if (first == ACU_OK) {
    for (size_t i = 0; i < ctx->async_fin.size(); ++i) {  // in call order: a plan's count is known before its filters finalise
      const acu_status st = ctx->async_fin[i](acu_hres(ctx, ctx->async_blk[i]));
      if (st != ACU_OK && first == ACU_OK) {
        first = st;
        first_err = ctx->err;
      }
    }
  }
  if (first != ACU_OK) ctx->err = first_err;
  ctx->async_fin.clear();
  ctx->async_blk.clear();
  ctx->async_blocks = 0;
  return first;
}

extern "C" int32_t acu_async_active(const acu_ctx *ctx) { return ctx->async_on ? 1 : 0; }

acu_status acu_res_reset(acu_ctx *ctx) { return acu_res_reset_n(ctx, 1); }
acu_status acu_res_fetch(acu_ctx *ctx) { return acu_res_fetch_n(ctx, 1); }

// ---- per-kernel-class device time ---------------------------------------------------------
int acu_kstats_begin(acu_ctx *ctx, int cls) {
  if (ctx->kev_pending == acu_ctx::KEV_PAIRS) {  // ring full: wait for the oldest work, drain
    cudaEventSynchronize(ctx->kev[acu_ctx::KEV_PAIRS - 1][1]);
    acu_kstats_drain(ctx);
  }
  const int slot = ctx->kev_pending++;
  ctx->kev_class[slot] = cls;
  cudaEventRecord(ctx->kev[slot][0], ctx->stream);
  return slot;
}
void acu_kstats_end(acu_ctx *ctx, int slot) { cudaEventRecord(ctx->kev[slot][1], ctx->stream); }
void acu_kstats_drain(acu_ctx *ctx) {
  for (int i = 0; i < ctx->kev_pending; ++i) {
    float ms = 0.f;
    if (cudaEventSynchronize(ctx->kev[i][1]) == cudaSuccess &&
        cudaEventElapsedTime(&ms, ctx->kev[i][0], ctx->kev[i][1]) == cudaSuccess) {
      ctx->kstat_ms[ctx->kev_class[i]] += ms;
      ctx->kstat_n[ctx->kev_class[i]] += 1;
    }
  }
  ctx->kev_pending = 0;
}

extern "C" {

int32_t acu_abi_version(void) { return ACU_ABI_VERSION; }
int32_t acu_abi_sizeof(int32_t which) {
  switch (which) {
    case 0: return (int32_t)sizeof(acu_array);
    case 1: return (int32_t)sizeof(acu_array_out);
    case 2: return (int32_t)sizeof(acu_error_detail);
    case 3: return (int32_t)sizeof(acu_column);
    case 4: return (int32_t)sizeof(acu_column_out);
    default: return -1;
  }
}

acu_status acu_ctx_create(int32_t device, acu_ctx **out) {
  *out = nullptr;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || device < 0 || device >= count) return ACU_ERR_CUDA;  // no CPU fallback
  if (cudaSetDevice(device) != cudaSuccess) return ACU_ERR_CUDA;
  acu_ctx *ctx = new (std::nothrow) acu_ctx();
  if (!ctx) return ACU_ERR_OUT_OF_MEMORY;
  ctx->device = device;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete ctx; return ACU_ERR_CUDA; }
  ctx->sm_count = prop.multiProcessorCount;
  bool ok = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) == cudaSuccess &&
            cudaEventCreate(&ctx->ev_start) == cudaSuccess &&
            cudaEventCreate(&ctx->ev_stop) == cudaSuccess &&
            cudaMalloc(&ctx->d_res, (size_t)RES_BLOCKS * RES_SLOTS * sizeof(unsigned long long)) == cudaSuccess &&
            cudaHostAlloc(&ctx->h_res, (size_t)RES_BLOCKS * RES_SLOTS * sizeof(unsigned long long), cudaHostAllocDefault) == cudaSuccess;
  for (int i = 0; ok && i < ACU_TIMER_SLOTS; ++i)
    ok = cudaEventCreate(&ctx->tev[i][0]) == cudaSuccess && cudaEventCreate(&ctx->tev[i][1]) == cudaSuccess;
  for (int i = 0; ok && i < acu_ctx::KEV_PAIRS; ++i)
    ok = cudaEventCreate(&ctx->kev[i][0]) == cudaSuccess && cudaEventCreate(&ctx->kev[i][1]) == cudaSuccess;
  if (!ok) { acu_ctx_destroy(ctx); return ACU_ERR_CUDA; }
  // keep freed blocks in the stream-ordered pool (no OS round trip between calls)
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t thr = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  // L2 fill granularity. Sparse kernels (filter at low selectivity, take) only need the 32-B
  // sectors they touch; the default granularity fills whole 128-B lines from HBM (at 10 % selectivity
  // a 128-B line of 8-B values holds a selected row with probability 1 - 0.9^16 = 81.5 %).
  cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
  cudaGetLastError();
  ctx->err.status = ACU_OK;
  ctx->err.index = -1;
  *out = ctx;
  return ACU_OK;
}

acu_status acu_comm_destroy(acu_ctx *ctx);

void acu_ctx_destroy(acu_ctx *ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  if (ctx->nccl_comm) acu_comm_destroy(ctx);
  if (ctx->stream) cudaStreamSynchronize(ctx->stream);
  for (auto &kv : ctx->allocs) cudaFree(kv.first);
  if (ctx->d_scratch) cudaFree(ctx->d_scratch);
  if (ctx->d_res) cudaFree(ctx->d_res);
  if (ctx->h_res) cudaFreeHost(ctx->h_res);
  if (ctx->ev_start) cudaEventDestroy(ctx->ev_start);
  if (ctx->ev_stop) cudaEventDestroy(ctx->ev_stop);
  for (int i = 0; i < ACU_TIMER_SLOTS; ++i)
    for (int j = 0; j < 2; ++j)
      if (ctx->tev[i][j]) cudaEventDestroy(ctx->tev[i][j]);
  for (int i = 0; i < acu_ctx::KEV_PAIRS; ++i)
    for (int j = 0; j < 2; ++j)
      if (ctx->kev[i][j]) cudaEventDestroy(ctx->kev[i][j]);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  delete ctx;
}

acu_status acu_ctx_sync(acu_ctx *ctx) {
  ACU_ENTER(ctx);
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  acu_kstats_drain(ctx);
  return ACU_OK;
}

const acu_error_detail *acu_last_error(const acu_ctx *ctx) { return &ctx->err; }
int64_t acu_launch_count(const acu_ctx *ctx) { return ctx->launches; }
int32_t acu_device_sm_count(const acu_ctx *ctx) { return ctx->sm_count; }
int64_t acu_bytes_allocated(const acu_ctx *ctx) { return ctx->bytes_allocated; }

acu_status acu_malloc(acu_ctx *ctx, size_t bytes, void **out) {
  *out = nullptr;
  size_t rounded = (bytes + 255) & ~(size_t)255;
  if (rounded == 0) rounded = 256;
  void *p = nullptr;
  ACU_CUDA(ctx, cudaSetDevice(ctx->device));
  ACU_CUDA(ctx, cudaMallocAsync(&p, rounded, ctx->stream));
  ctx->allocs[p] = rounded;
  ctx->bytes_allocated += (int64_t)rounded;
  *out = p;
  return ACU_OK;
}

acu_status acu_free(acu_ctx *ctx, void *dptr) {
  ACU_ENTER(ctx);
  if (!dptr) return ACU_OK;
  auto it = ctx->allocs.find(dptr);
  if (it == ctx->allocs.end())
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "acu_free: pointer not owned by this ctx");
  ctx->bytes_allocated -= (int64_t)it->second;
  ctx->allocs.erase(it);
  ACU_CUDA(ctx, cudaFreeAsync(dptr, ctx->stream));
  return ACU_OK;
}

acu_status acu_memset(acu_ctx *ctx, void *dptr, int32_t byte, size_t bytes) {
  ACU_ENTER(ctx);
  if (bytes) ACU_CUDA(ctx, cudaMemsetAsync(dptr, byte, bytes, ctx->stream));
  return ACU_OK;
}

acu_status acu_memcpy_h2d(acu_ctx *ctx, void *dst, const void *src, size_t bytes) {
  ACU_ENTER(ctx);
  if (bytes) ACU_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return ACU_OK;
}
acu_status acu_memcpy_d2h(acu_ctx *ctx, void *dst, const void *src, size_t bytes) {
  ACU_ENTER(ctx);
  if (bytes) ACU_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return ACU_OK;
}
acu_status acu_memcpy_d2d(acu_ctx *ctx, void *dst, const void *src, size_t bytes) {
  ACU_ENTER(ctx);
  if (bytes) ACU_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, ctx->stream));
  return ACU_OK;
}
acu_status acu_memcpy_h2d_async(acu_ctx *ctx, void *dst, const void *src, size_t bytes) {
  ACU_ENTER(ctx);
  if (bytes) ACU_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return ACU_OK;
}
acu_status acu_memcpy_d2h_async(acu_ctx *ctx, void *dst, const void *src, size_t bytes) {
  ACU_ENTER(ctx);
  if (bytes) ACU_CUDA(ctx, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  return ACU_OK;
}
acu_status acu_host_alloc(acu_ctx *ctx, size_t bytes, void **out) {
  ACU_ENTER(ctx);
  ACU_CUDA(ctx, cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
  return ACU_OK;
}
acu_status acu_host_free(acu_ctx *ctx, void *host) {
  ACU_ENTER(ctx);
  if (host) ACU_CUDA(ctx, cudaFreeHost(host));
  return ACU_OK;
}

acu_status acu_timer_start_slot(acu_ctx *ctx, int32_t slot) {
  ACU_ENTER(ctx);
  if (slot < 0 || slot >= ACU_TIMER_SLOTS) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "timer slot %d", slot);
  ACU_CUDA(ctx, cudaEventRecord(ctx->tev[slot][0], ctx->stream));
  return ACU_OK;
}
acu_status acu_timer_stop_slot(acu_ctx *ctx, int32_t slot, float *out_ms) {
  ACU_ENTER(ctx);
  if (slot < 0 || slot >= ACU_TIMER_SLOTS) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "timer slot %d", slot);
  ACU_CUDA(ctx, cudaEventRecord(ctx->tev[slot][1], ctx->stream));
  ACU_CUDA(ctx, cudaEventSynchronize(ctx->tev[slot][1]));
  ACU_CUDA(ctx, cudaEventElapsedTime(out_ms, ctx->tev[slot][0], ctx->tev[slot][1]));
  acu_kstats_drain(ctx);
  return ACU_OK;
}
acu_status acu_timer_start(acu_ctx *ctx) { return acu_timer_start_slot(ctx, 0); }
acu_status acu_timer_stop(acu_ctx *ctx, float *out_ms) { return acu_timer_stop_slot(ctx, 0, out_ms); }

acu_status acu_kernel_stats(acu_ctx *ctx, int32_t cls, double *out_total_ms, int64_t *out_launches) {
  if (cls < 0 || cls >= ACU_K_CLASSES) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "kernel class %d", cls);
  *out_total_ms = ctx->kstat_ms[cls];
  *out_launches = ctx->kstat_n[cls];
  return ACU_OK;
}
acu_status acu_kernel_stats_reset(acu_ctx *ctx) {
  for (int i = 0; i < ACU_K_CLASSES; ++i) { ctx->kstat_ms[i] = 0; ctx->kstat_n[i] = 0; }
  return ACU_OK;
}

}  // extern "C"
