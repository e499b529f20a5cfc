// comm.cu — multi-GPU plumbing: row-range shards need no data-path collective; NCCL is used
// only for the final reduction of per-shard scalar aggregates (sum/min/max) and row counts
// (SURVEY.md §8(e)). NCCL is resolved at run time with dlopen so that the library has no
// link-time NCCL dependency and shares the copy already loaded in the process (e.g. the one
// bundled with torch when bench.py uses torch.distributed for rendezvous).
#include <dlfcn.h>
#include <stdio.h>

#include "internal.cuh"

namespace {

typedef struct { char internal[ACU_NCCL_UNIQUE_ID_BYTES]; } nccl_unique_id;
typedef void *nccl_comm_t;
enum { NCCL_SUM = 0, NCCL_MAX = 2, NCCL_MIN = 3 };
enum { NCCL_INT64 = 4, NCCL_UINT64 = 5, NCCL_FLOAT32 = 7, NCCL_FLOAT64 = 8 };

struct NcclApi {
  void *handle = nullptr;
  int (*GetUniqueId)(nccl_unique_id *) = nullptr;
  int (*CommInitRank)(nccl_comm_t *, int, nccl_unique_id, int) = nullptr;
  int (*CommDestroy)(nccl_comm_t) = nullptr;
  int (*AllReduce)(const void *, void *, size_t, int, int, nccl_comm_t, cudaStream_t) = nullptr;
  int (*GroupStart)() = nullptr;
  int (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(int) = nullptr;
};

NcclApi *nccl_api() {
  static NcclApi api;
  static bool tried = false;
  if (!tried) {
    tried = true;
    const char *names[] = {"libnccl.so.2", "libnccl.so", nullptr};
    // a copy already in the process (e.g. the one torch bundles) wins; otherwise load the system one
    // privately (RTLD_LOCAL) so that it can never satisfy another library's NCCL symbols
    for (int i = 0; names[i] && !api.handle; ++i) api.handle = dlopen(names[i], RTLD_NOW | RTLD_NOLOAD);
    for (int i = 0; names[i] && !api.handle; ++i) api.handle = dlopen(names[i], RTLD_NOW | RTLD_LOCAL);
    if (api.handle) {
      api.GetUniqueId = (int (*)(nccl_unique_id *))dlsym(api.handle, "ncclGetUniqueId");
      api.CommInitRank = (int (*)(nccl_comm_t *, int, nccl_unique_id, int))dlsym(api.handle, "ncclCommInitRank");
      api.CommDestroy = (int (*)(nccl_comm_t))dlsym(api.handle, "ncclCommDestroy");
      api.AllReduce = (int (*)(const void *, void *, size_t, int, int, nccl_comm_t, cudaStream_t))dlsym(api.handle, "ncclAllReduce");
      api.GroupStart = (int (*)())dlsym(api.handle, "ncclGroupStart");
      api.GroupEnd = (int (*)())dlsym(api.handle, "ncclGroupEnd");
      api.GetErrorString = (const char *(*)(int))dlsym(api.handle, "ncclGetErrorString");
      if (!api.GetUniqueId || !api.CommInitRank || !api.CommDestroy || !api.AllReduce || !api.GroupStart || !api.GroupEnd) {
        dlclose(api.handle);
        api.handle = nullptr;
      }
    }
  }
  return api.handle ? &api : nullptr;
}

acu_status nccl_fail(acu_ctx *ctx, int rc, const char *what) {
  NcclApi *api = nccl_api();
  acu_fail(ctx, ACU_ERR_NCCL, -1, 0, 0, 0, "NCCL error %d (%s) in %s", rc,
           (api && api->GetErrorString) ? api->GetErrorString(rc) : "?", what);
  ctx->err.cuda_error = rc;
  return ACU_ERR_NCCL;
}

#define ACU_NCCL(ctx, expr)                                \
  do {                                                     \
    int _rc = (expr);                                      \
    if (_rc != 0) return nccl_fail((ctx), _rc, #expr);     \
  } while (0)

__host__ __device__ inline int64_t key64(uint64_t bits, acu_dtype t) {  // native bits -> order-preserving int64 key
  switch (t) {
    case ACU_I8: return (int8_t)bits;
    case ACU_I16: return (int16_t)bits;
    case ACU_I32: return (int32_t)bits;
    case ACU_I64: return (int64_t)bits;
    case ACU_F32: { int32_t b = (int32_t)(uint32_t)bits; return (int64_t)(b ^ (int32_t)((uint32_t)(b >> 31) >> 1)); }
    case ACU_F64: { int64_t b = (int64_t)bits; return b ^ (int64_t)((uint64_t)(b >> 63) >> 1); }
    default: return (int64_t)bits;  // unsigned: reduced as uint64
  }
}
__host__ __device__ inline uint64_t unkey64(int64_t k, acu_dtype t) {
  switch (t) {
    case ACU_I8: return (uint8_t)k;
    case ACU_I16: return (uint16_t)k;
    case ACU_I32: return (uint32_t)k;
    case ACU_F32: { int32_t b = (int32_t)k; return (uint32_t)(b ^ (int32_t)((uint32_t)(b >> 31) >> 1)); }
    case ACU_F64: return (uint64_t)(k ^ (int64_t)((uint64_t)(k >> 63) >> 1));
    default: return (uint64_t)k;
  }
}


// Encode a shard's partial aggregate for the all-reduce (what acu_comm_allreduce_aggregates does on the host): identity for
// a shard without valid rows, sign extension for narrow signed sums, totalOrder keys for signed / float min / max.
__host__ __device__ inline uint64_t encode_partial(uint64_t bits, bool empty, acu_dtype dtype, acu_agg_op op) {
  const bool is_unsigned = dtype == ACU_U8 || dtype == ACU_U16 || dtype == ACU_U32 || dtype == ACU_U64;
  if (op == ACU_SUM) {
    uint64_t v = dtype == ACU_F32 ? (empty ? 0 : (bits & 0xffffffffull)) : (empty ? 0 : bits);
    if (dtype != ACU_F32 && dtype != ACU_F64 && !is_unsigned) v = (uint64_t)key64(v, dtype);
    return v;
  }
  if (is_unsigned) return empty ? (op == ACU_MIN ? ~0ull : 0ull) : bits;
  return (uint64_t)(empty ? (op == ACU_MIN ? INT64_MAX : INT64_MIN) : key64(bits, dtype));
}

__global__ void k_stage_partial(const unsigned long long *res, int launched, long long valid_count, int dtype, int op, uint64_t *buf) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (valid_count < 0) valid_count = launched ? (long long)res[RES_COUNT] : 0;  // counted by k_reduce (unknown on the host)
  const uint64_t bits = launched ? res[RES_AUX0] : 0ull;
  buf[0] = encode_partial(bits, valid_count == 0, (acu_dtype)dtype, (acu_agg_op)op);
  buf[1] = (uint64_t)valid_count;
}

// The partial encodings and NCCL ops above exist for sum / min / max only; NCCL has no product or bitwise reduction.
acu_status allreduce_op_ok(acu_ctx *ctx, acu_agg_op op) {
  if (op == ACU_SUM || op == ACU_MIN || op == ACU_MAX) return ACU_OK;
  return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, -1, 0, 0, 0, "all-reduce of aggregate op %d", (int)op);
}
}  // namespace

extern "C" {

acu_status acu_comm_get_unique_id(uint8_t out_id[ACU_NCCL_UNIQUE_ID_BYTES]) {
  NcclApi *api = nccl_api();
  if (!api) return ACU_ERR_NCCL;
  nccl_unique_id id;
  if (api->GetUniqueId(&id) != 0) return ACU_ERR_NCCL;
  memcpy(out_id, id.internal, ACU_NCCL_UNIQUE_ID_BYTES);
  return ACU_OK;
}

acu_status acu_comm_init(acu_ctx *ctx, const uint8_t id_bytes[ACU_NCCL_UNIQUE_ID_BYTES], int32_t rank, int32_t world) {
  NcclApi *api = nccl_api();
  if (!api) return acu_fail(ctx, ACU_ERR_NCCL, -1, 0, 0, 0, "libnccl.so.2 could not be loaded");
  nccl_unique_id id;
  memcpy(id.internal, id_bytes, ACU_NCCL_UNIQUE_ID_BYTES);
  ACU_CUDA(ctx, cudaSetDevice(ctx->device));
  nccl_comm_t comm = nullptr;
  ACU_NCCL(ctx, api->CommInitRank(&comm, world, id, rank));
  ctx->nccl_comm = comm;
  ctx->rank = rank;
  ctx->world = world;
  return ACU_OK;
}

acu_status acu_comm_destroy(acu_ctx *ctx) {
  NcclApi *api = nccl_api();
  if (api && ctx->nccl_comm) {
    cudaStreamSynchronize(ctx->stream);
    api->CommDestroy(ctx->nccl_comm);
  }
  ctx->nccl_comm = nullptr;
  ctx->world = 1;
  ctx->rank = 0;
  return ACU_OK;
}

acu_status acu_comm_allreduce_i64_sum(acu_ctx *ctx, int64_t *values, int32_t n) {
  ACU_ENTER(ctx);
  if (ctx->world <= 1 || !ctx->nccl_comm || n <= 0) return ACU_OK;
  NcclApi *api = nccl_api();
  void *buf;
  ACU_TRY(acu_scratch(ctx, (size_t)n * 8, &buf));
  ACU_CUDA(ctx, cudaMemcpyAsync(buf, values, (size_t)n * 8, cudaMemcpyHostToDevice, ctx->stream));
  ACU_NCCL(ctx, api->AllReduce(buf, buf, (size_t)n, NCCL_INT64, NCCL_SUM, ctx->nccl_comm, ctx->stream));
  ACU_CUDA(ctx, cudaMemcpyAsync(values, buf, (size_t)n * 8, cudaMemcpyDeviceToHost, ctx->stream));
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return ACU_OK;
}

acu_status acu_comm_allreduce_aggregates(acu_ctx *ctx, acu_dtype dtype, acu_agg_op op, uint64_t *partial_bits,
                                         int64_t *valid_counts, int32_t n) {
  ACU_ENTER(ctx);
  ACU_TRY(allreduce_op_ok(ctx, op));
  if (ctx->world <= 1 || !ctx->nccl_comm || n <= 0) return ACU_OK;
  NcclApi *api = nccl_api();
  if (n > 32) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "at most 32 aggregates per all-reduce");
  // staging lives in the upper half of the ctx result blocks: pinned on the host side, so both copies are
  // truly asynchronous; layout [n x 8 B values][n x int64 counts]
  uint64_t *stage = reinterpret_cast<uint64_t *>(ctx->h_res + (size_t)(RES_BLOCKS / 2) * RES_SLOTS);
  uint8_t *buf = reinterpret_cast<uint8_t *>(ctx->d_res + (size_t)(RES_BLOCKS / 2) * RES_SLOTS);
  ctx->res_clean = false;  // the staging overwrites result blocks: the next reset re-initialises all of them
  ctx->res_dirty_blocks = RES_BLOCKS;
  const bool is_unsigned = dtype == ACU_U8 || dtype == ACU_U16 || dtype == ACU_U32 || dtype == ACU_U64;
  int nccl_type, nccl_op;
  for (int i = 0; i < n; ++i) {
    const bool empty = valid_counts[i] == 0;  // a shard with no valid rows contributes the identity
    if (op == ACU_SUM) {
      if (dtype == ACU_F32) stage[i] = empty ? 0 : (partial_bits[i] & 0xffffffffull);
      else stage[i] = empty ? 0 : partial_bits[i];
      if (dtype != ACU_F32 && dtype != ACU_F64 && !is_unsigned) stage[i] = (uint64_t)key64(stage[i], dtype);  // sign-extend
    } else if (is_unsigned) {
      stage[i] = empty ? (op == ACU_MIN ? ~0ull : 0ull) : partial_bits[i];
    } else {
      int64_t k = empty ? (op == ACU_MIN ? INT64_MAX : INT64_MIN) : key64(partial_bits[i], dtype);
      stage[i] = (uint64_t)k;
    }
    stage[n + i] = (uint64_t)valid_counts[i];
  }
  if (op == ACU_SUM) {
    nccl_op = NCCL_SUM;
    nccl_type = dtype == ACU_F64 ? NCCL_FLOAT64 : dtype == ACU_F32 ? NCCL_FLOAT32 : NCCL_INT64;  // two's complement: one sum for both signs
  } else {
    nccl_op = op == ACU_MIN ? NCCL_MIN : NCCL_MAX;
    nccl_type = is_unsigned ? NCCL_UINT64 : NCCL_INT64;
  }
  ACU_CUDA(ctx, cudaMemcpyAsync(buf, stage, (size_t)n * 16, cudaMemcpyHostToDevice, ctx->stream));
  if (nccl_op == NCCL_SUM && nccl_type == NCCL_INT64) {
    // integer sums and the valid counts are both int64 sums: ONE all-reduce over 2n words
    ACU_NCCL(ctx, api->AllReduce(buf, buf, (size_t)n * 2, NCCL_INT64, NCCL_SUM, ctx->nccl_comm, ctx->stream));
  } else {
    ACU_NCCL(ctx, api->GroupStart());
    if (nccl_type == NCCL_FLOAT32) {
      // f32 partials occupy the low 4 bytes of each 8-byte slot: reduce 2n floats (the high
      // halves are zero and stay zero under sum)
      ACU_NCCL(ctx, api->AllReduce(buf, buf, (size_t)n * 2, NCCL_FLOAT32, nccl_op, ctx->nccl_comm, ctx->stream));
    } else {
      ACU_NCCL(ctx, api->AllReduce(buf, buf, (size_t)n, nccl_type, nccl_op, ctx->nccl_comm, ctx->stream));
    }
    ACU_NCCL(ctx, api->AllReduce(buf + (size_t)n * 8, buf + (size_t)n * 8, (size_t)n, NCCL_INT64, NCCL_SUM, ctx->nccl_comm, ctx->stream));
    ACU_NCCL(ctx, api->GroupEnd());
  }
  ACU_CUDA(ctx, cudaMemcpyAsync(stage, buf, (size_t)n * 16, cudaMemcpyDeviceToHost, ctx->stream));
  ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int i = 0; i < n; ++i) {
    valid_counts[i] = (int64_t)stage[n + i];
    if (op == ACU_SUM) {
      const int sz = acu_dtype_size(dtype);
      partial_bits[i] = sz == 8 ? stage[i] : (stage[i] & ((1ull << (8 * sz)) - 1ull));  // wrapping sum in native width
    } else if (is_unsigned) {
      partial_bits[i] = stage[i];
    } else {
      partial_bits[i] = unkey64((int64_t)stage[i], dtype);
    }
  }
  return ACU_OK;
}

// sum / min / max of this rank's shard combined over all ranks with ONE synchronisation (see include/arrow_cuda.h). The
// all-reduce runs in place on slots 8..9 of the call's own result block, so the combined value travels to the host with
// the block (the call's fetch, or acu_results_fetch at the end of an async section): no host bounce.
acu_status acu_aggregate_allreduce(acu_ctx *ctx, acu_dtype dtype, acu_agg_op op, const acu_array *a, uint64_t *out_bits,
                                   int64_t *out_valid_count) {
  ACU_TRY(allreduce_op_ok(ctx, op));
  if (ctx->world <= 1 || !ctx->nccl_comm) return acu_aggregate(ctx, dtype, op, a, out_bits, out_valid_count);
  ACU_ENTER(ctx);
  NcclApi *api = nccl_api();
  *out_bits = 0;
  *out_valid_count = 0;
  acu_status st = ACU_OK;
  const bool deferred_nc = ctx->async_on && a->len && a->validity && a->null_count < 0;
  const int64_t nc = deferred_nc ? -1 : (a->len ? acu_resolve_null_count(ctx, a, &st) : 0);
  ACU_TRY(st);
  const int64_t valid = deferred_nc ? -1 : a->len - nc;
  const size_t scratch_bytes = acu_reduce_col_scratch(ctx);
  void *scratch;
  ACU_TRY(acu_scratch(ctx, scratch_bytes, &scratch));
  int launched = 0;
  const int blk = acu_call_begin(ctx, &st);
  ACU_TRY(st);
  unsigned long long *res = acu_dres(ctx, blk);
  ACU_TRY(acu_reduce_cols_launch(ctx, 1, &dtype, &op, a, &nc, static_cast<uint8_t *>(scratch), scratch_bytes, &res, &launched));
  constexpr int SLOT = 8;  // slots 8..9 of the block: {combined value, combined valid count}
  uint64_t *buf = reinterpret_cast<uint64_t *>(acu_dres(ctx, blk) + SLOT);
  ACU_LAUNCH(ctx, k_stage_partial, 1, 32, 0, acu_dres(ctx, blk), launched, (long long)valid, (int)dtype, (int)op, buf);
  const bool is_unsigned = dtype == ACU_U8 || dtype == ACU_U16 || dtype == ACU_U32 || dtype == ACU_U64;
  if (op == ACU_SUM && dtype != ACU_F32 && dtype != ACU_F64) {
    ACU_NCCL(ctx, api->AllReduce(buf, buf, 2, NCCL_INT64, NCCL_SUM, ctx->nccl_comm, ctx->stream));  // value and count: one int64 sum
  } else {
    ACU_NCCL(ctx, api->GroupStart());
    if (op == ACU_SUM && dtype == ACU_F32) ACU_NCCL(ctx, api->AllReduce(buf, buf, 2, NCCL_FLOAT32, NCCL_SUM, ctx->nccl_comm, ctx->stream));
    else if (op == ACU_SUM) ACU_NCCL(ctx, api->AllReduce(buf, buf, 1, NCCL_FLOAT64, NCCL_SUM, ctx->nccl_comm, ctx->stream));
    else ACU_NCCL(ctx, api->AllReduce(buf, buf, 1, is_unsigned ? NCCL_UINT64 : NCCL_INT64, op == ACU_MIN ? NCCL_MIN : NCCL_MAX, ctx->nccl_comm, ctx->stream));
    ACU_NCCL(ctx, api->AllReduce(buf + 1, buf + 1, 1, NCCL_INT64, NCCL_SUM, ctx->nccl_comm, ctx->stream));
    ACU_NCCL(ctx, api->GroupEnd());
  }
  return acu_call_end(ctx, blk, [dtype, op, is_unsigned, out_bits, out_valid_count](const unsigned long long *h) -> acu_status {
    const uint64_t v = h[SLOT];
    *out_valid_count = (int64_t)h[SLOT + 1];
    if (op == ACU_SUM) {
      const int sz = acu_dtype_size(dtype);
      *out_bits = sz == 8 ? v : (v & ((1ull << (8 * sz)) - 1ull));
    } else if (is_unsigned) {
      *out_bits = v;
    } else {
      *out_bits = unkey64((int64_t)v, dtype);
    }
    return ACU_OK;
  });
}

}  // extern "C"
