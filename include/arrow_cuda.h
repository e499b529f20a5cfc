/*
 * arrow_cuda.h — C ABI of the H100-native arrow::compute hot path.
 *
 * This is the drop-in boundary (SURVEY.md §8(b)): one extern "C" entry point per
 * reference kernel, taking raw DEVICE pointers + explicit lengths / bit offsets, so
 * that a thin Rust `arrow-cuda` crate (rust/arrow-cuda, source only — no rustc in
 * this image) or the C++ host mirror (arrow-rs_b200/host/arrow_cuda.hpp) can wrap
 * them with the reference's own signatures over ArrayRef / RecordBatch.
 *
 * Layout contract (mirrors arrow-buffer; reference file:line in brackets):
 *   - values buffer: contiguous little-endian natives, pointer already advanced to
 *     logical element 0                      [arrow-buffer/src/buffer/scalar.rs:29-46]
 *   - validity / boolean bitmap: bytes, bit i of the logical array at byte
 *     (off+i)>>3, bit (off+i)&7, LSB first, 1 = valid / true
 *                                            [arrow-buffer/src/util/bit_util.rs:52-66,
 *                                             arrow-buffer/src/buffer/boolean.rs:97-104]
 *   - null_count is cached beside the bitmap  [arrow-buffer/src/buffer/null.rs:34-37]
 *
 * Every OUTPUT bitmap is written with bit offset 0 and must have a capacity of
 * acu_bitmap_bytes(len) = 8*ceil(len/64) bytes (kernels store whole 64-bit words);
 * bits at positions >= len are unspecified, exactly as in the reference
 * (arrow-ord/src/cmp.rs:598-608).
 *
 * Calls are synchronous with respect to the host: every entry point that returns a
 * host-visible scalar (count, null_count, error index) synchronises the ctx stream
 * before returning (stream-ordered sections, acu_async_begin below, defer that to ONE
 * synchronisation for a chain of calls). One acu_ctx = one device + one stream + scratch; a ctx must not
 * be used from two host threads at once, distinct ctxs are independent (the
 * reference kernels are pure, re-entrant functions: arrow-array/src/array/mod.rs:99).
 *
 * There is NO CPU fallback behind this ABI: if no CUDA device is present
 * acu_ctx_create fails with ACU_ERR_CUDA.
 */
#ifndef ARROW_CUDA_H
#define ARROW_CUDA_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ACU_ABI_VERSION 1

/* ------------------------------------------------------------------------- */
/* Status codes — one per ArrowError variant the hot path can produce        */
/* (arrow-schema/src/error.rs:26-67), plus the reference's panics, plus      */
/* device-side failures.                                                     */
/* ------------------------------------------------------------------------- */
typedef int32_t acu_status;
enum {
  ACU_OK = 0,
  ACU_ERR_INVALID_ARGUMENT = 1,    /* ArrowError::InvalidArgumentError          */
  ACU_ERR_COMPUTE = 2,             /* ArrowError::ComputeError                  */
  ACU_ERR_ARITHMETIC_OVERFLOW = 3, /* ArrowError::ArithmeticOverflow            */
  ACU_ERR_DIVIDE_BY_ZERO = 4,      /* ArrowError::DivideByZero                  */
  ACU_ERR_OFFSET_OVERFLOW = 5,     /* ArrowError::OffsetOverflowError(usize)    */
  ACU_ERR_CAST = 6,                /* ArrowError::CastError                     */
  ACU_ERR_NOT_YET_IMPLEMENTED = 7, /* ArrowError::NotYetImplemented             */
  ACU_ERR_PANIC_OUT_OF_BOUNDS = 8, /* the reference panics (take.rs:447,454)    */
  ACU_ERR_IPC = 9,                 /* ArrowError::IpcError                      */
  ACU_ERR_PARSE = 10,              /* ArrowError::ParseError                    */
  ACU_ERR_CUDA = 100,              /* CUDA runtime error (detail.cuda_error)    */
  ACU_ERR_NCCL = 101,              /* NCCL error                                */
  ACU_ERR_OUT_OF_MEMORY = 102
};

/* Filled on every non-OK return; lets the host shim rebuild the reference's exact
 * message, e.g. "Overflow happened on: {lhs} + {rhs}" (arrow-array/src/arithmetic.rs:163-170)
 * or "Array index out of bounds, cannot get item at index {index} from {len} entries"
 * (arrow-select/src/take.rs:186-188). `message` already holds that text. */
typedef struct acu_error_detail {
  acu_status status;
  int32_t cuda_error;   /* cudaError_t / ncclResult_t when status >= 100 */
  int64_t index;        /* lowest offending logical row, -1 if n/a        */
  uint64_t lhs_bits;    /* operand bit patterns at `index`                */
  uint64_t rhs_bits;
  uint64_t len;         /* array length / capacity relevant to the error  */
  char message[256];
} acu_error_detail;

typedef struct acu_ctx acu_ctx;

/* Native types (arrow-array/src/types.rs:67-80, ArrowPrimitiveType::Native).
 * ACU_I128 is the native of Decimal128: 16-byte little-endian two's complement values whose pointer must be 16-byte
 * aligned (the alignment of i128; a misaligned pointer => ACU_ERR_INVALID_ARGUMENT). Only acu_cmp (and through it
 * acu_filter_plan_create_cmp) and acu_neg accept it; every other entry point taking an acu_dtype rejects it as it
 * rejects an unknown dtype. Decimal32 / Decimal64 columns ARE Int32 / Int64 columns to acu_cmp, acu_filter_plan_create_cmp,
 * acu_aggregate and acu_aggregate_columns: the reference compares and aggregates decimals as their native integers, so
 * ACU_I32 / ACU_I64 give Decimal32 / Decimal64 exactly the reference's results. */
typedef enum acu_dtype {
  ACU_I8 = 0, ACU_I16 = 1, ACU_I32 = 2, ACU_I64 = 3,
  ACU_U8 = 4, ACU_U16 = 5, ACU_U32 = 6, ACU_U64 = 7,
  ACU_F32 = 8, ACU_F64 = 9,
  ACU_I128 = 10
} acu_dtype;

/* arrow-arith/src/numeric.rs:181-190 `enum Op` — same order. */
typedef enum acu_arith_op {
  ACU_ADD_WRAPPING = 0, ACU_ADD = 1,
  ACU_SUB_WRAPPING = 2, ACU_SUB = 3,
  ACU_MUL_WRAPPING = 4, ACU_MUL = 5,
  ACU_DIV = 6, ACU_REM = 7
} acu_arith_op;

/* arrow-ord/src/cmp.rs:40-60 `enum Op`. */
typedef enum acu_cmp_op {
  ACU_EQ = 0, ACU_NEQ = 1, ACU_LT = 2, ACU_LT_EQ = 3, ACU_GT = 4, ACU_GT_EQ = 5,
  ACU_DISTINCT = 6, ACU_NOT_DISTINCT = 7
} acu_cmp_op;

/* arrow-arith/src/aggregate.rs:943,1012,1027 (sum / min / max), :953 (product), :850-875 (bit_and / bit_or / bit_xor). */
typedef enum acu_agg_op {
  ACU_SUM = 0, ACU_MIN = 1, ACU_MAX = 2,
  ACU_PRODUCT = 3, ACU_BIT_AND = 4, ACU_BIT_OR = 5, ACU_BIT_XOR = 6
} acu_agg_op;

/* arrow-arith/src/bitwise.rs: bitwise_and / or / xor / and_not / shift_left / shift_right / not. */
typedef enum acu_bitwise_op {
  ACU_BITWISE_AND = 0, ACU_BITWISE_OR = 1, ACU_BITWISE_XOR = 2, ACU_BITWISE_AND_NOT = 3,
  ACU_BITWISE_SHIFT_LEFT = 4, ACU_BITWISE_SHIFT_RIGHT = 5, ACU_BITWISE_NOT = 6
} acu_bitwise_op;

/* A borrowed, immutable view of a primitive / boolean array in HBM
 * (PrimitiveArray{values,nulls} arrow-array/src/array/primitive_array.rs:596-601;
 *  BooleanArray{values,nulls} arrow-array/src/array/boolean_array.rs:68-71). */
typedef struct acu_array {
  const void *values;       /* device ptr to logical element 0 (for boolean arrays: bitmap bytes) */
  int64_t values_offset;    /* boolean arrays only: bit offset of logical row 0 in `values`      */
  const uint8_t *validity;  /* device ptr to validity bytes, NULL = no NullBuffer                */
  int64_t validity_offset;  /* bit offset of logical row 0 in `validity`                         */
  int64_t len;              /* logical length                                                    */
  int64_t null_count;       /* cached null count; -1 = unknown (counted on device)               */
  int32_t is_scalar;        /* Datum::get().1 (arrow-array/src/scalar.rs:78-152): len must be 1  */
  int32_t reserved;
} acu_array;

/* Caller-owned output. `values` capacity: len*width bytes (boolean results:
 * acu_bitmap_bytes(len)); `validity` capacity: acu_bitmap_bytes(len).
 * On return: len, null_count, has_validity (0 => the reference returns nulls = None
 * and the validity buffer content is unspecified). */
typedef struct acu_array_out {
  void *values;
  uint8_t *validity;
  int64_t len;
  int64_t null_count;
  int32_t has_validity;
  int32_t reserved;
} acu_array_out;

static inline size_t acu_bitmap_bytes(int64_t len) { return (size_t)((len + 63) / 64) * 8; }

/* ------------------------------------------------------------------------- */
/* Context, memory, timing                                                   */
/* ------------------------------------------------------------------------- */
int32_t acu_abi_version(void);
/* sizeof() of the ABI structs as this library was compiled, for binding self-checks:
 * 0 acu_array, 1 acu_array_out, 2 acu_error_detail, 3 acu_column, 4 acu_column_out; -1 otherwise. */
int32_t acu_abi_sizeof(int32_t which);
acu_status acu_ctx_create(int32_t device, acu_ctx **out);
void acu_ctx_destroy(acu_ctx *ctx);
acu_status acu_ctx_sync(acu_ctx *ctx);
/* Detail of the last failing call on this ctx (never NULL once ctx exists). */
const acu_error_detail *acu_last_error(const acu_ctx *ctx);
/* Number of kernels this ctx has launched since creation (bench.py: gpu_launches). */
int64_t acu_launch_count(const acu_ctx *ctx);
int32_t acu_device_sm_count(const acu_ctx *ctx);

/* DeviceBuffer allocation: 256-B aligned, stream-ordered (cudaMallocAsync pool);
 * mirrors arrow-buffer's 128-B aligned host allocation (src/alloc/alignment.rs:38). */
acu_status acu_malloc(acu_ctx *ctx, size_t bytes, void **out_dptr);
acu_status acu_free(acu_ctx *ctx, void *dptr);
acu_status acu_memset(acu_ctx *ctx, void *dptr, int32_t byte, size_t bytes);
acu_status acu_memcpy_h2d(acu_ctx *ctx, void *dst_dptr, const void *src_host, size_t bytes);
acu_status acu_memcpy_d2h(acu_ctx *ctx, void *dst_host, const void *src_dptr, size_t bytes);
acu_status acu_memcpy_d2d(acu_ctx *ctx, void *dst_dptr, const void *src_dptr, size_t bytes);
/* Asynchronous variants (ordered on the ctx stream; host memory must be pinned). */
acu_status acu_memcpy_h2d_async(acu_ctx *ctx, void *dst_dptr, const void *src_host, size_t bytes);
acu_status acu_memcpy_d2h_async(acu_ctx *ctx, void *dst_host, const void *src_dptr, size_t bytes);
acu_status acu_host_alloc(acu_ctx *ctx, size_t bytes, void **out_host);   /* pinned */
acu_status acu_host_free(acu_ctx *ctx, void *host);
/* Bytes currently allocated through acu_malloc on this ctx (observability; the
 * reference's MemoryPool tracking, arrow-buffer/src/pool.rs:73-85). */
int64_t acu_bytes_allocated(const acu_ctx *ctx);

/* ---- Stream-ordered sections -------------------------------------------------------------------------------------
 * The reference functions are synchronous (arrow-array/src/array/mod.rs:99) and so is every entry point by default. A
 * caller that chains several kernels (filter -> take -> add -> sum) can instead open a SECTION: between acu_async_begin
 * and acu_results_fetch the entry points listed below only ENQUEUE their kernels on the ctx stream and return at once;
 * each call owns one of the ctx's 64 result blocks (count, null count, lowest failing row stay in HBM).
 * acu_results_fetch copies all blocks to the host in ONE transfer with ONE synchronisation, then finalises the queued
 * calls in call order: it fills the acu_array_out / scalar outputs the calls were given (len, has_validity, null_count,
 * aggregate bits), fills acu_filter_plan count / strategy, and returns the FIRST error in call order with its exact
 * reference text (the outputs of the calls after a failed one are unspecified, as after any failed call).
 *   - stream-ordered inside a section: acu_filter_plan_create, acu_filter_plan_create_cmp, acu_filter_primitive,
 *     acu_filter_boolean, acu_take_primitive / acu_take_boolean (check_bounds = 0), acu_arith, acu_bitwise,
 *     acu_decimal_arith, acu_cmp (ACU_I128 included), acu_neg (ACU_I128 only), acu_aggregate, acu_aggregate_i128, acu_aggregate_allreduce. Any other
 *     entry point fails with ACU_ERR_INVALID_ARGUMENT (it would synchronise).
 *   - every output descriptor, scalar output pointer and plan passed to a queued call must stay alive until the fetch;
 *     input arrays must carry their cached null_count (-1 would need a device count = a synchronisation), except for
 *     acu_aggregate*, which then counts the valid rows on the device (an array produced earlier in the same section);
 *   - a plan created inside the section can be used by filters queued after it: their outputs must then be sized for
 *     plan LEN rows (the count is still on the device); out->len is set by the fetch;
 *   - at most 64 calls per section. */
acu_status acu_async_begin(acu_ctx *ctx);
acu_status acu_results_fetch(acu_ctx *ctx);
int32_t acu_async_active(const acu_ctx *ctx);

/* CUDA-event timers on the ctx stream (events see exactly the stream kernels run on).
 * ACU_TIMER_SLOTS independent slots so that a step timer can bracket per-op timers. */
#define ACU_TIMER_SLOTS 8
acu_status acu_timer_start(acu_ctx *ctx);                /* slot 0 */
acu_status acu_timer_stop(acu_ctx *ctx, float *out_ms);  /* slot 0; records + synchronises */
acu_status acu_timer_start_slot(acu_ctx *ctx, int32_t slot);
acu_status acu_timer_stop_slot(acu_ctx *ctx, int32_t slot, float *out_ms);

/* Per-kernel device time, always on: every launch of a hot kernel is bracketed by a pair of
 * CUDA events on the ctx stream and its elapsed time is accumulated per kernel class when
 * the call synchronises. bench.py derives roofline.achieved from these (kernel-only) times. */
typedef enum acu_kernel_class {
  ACU_K_ARITH = 0, ACU_K_CMP = 1, ACU_K_CAST = 2, ACU_K_FILTER = 3, ACU_K_FILTER_PLAN = 4,
  ACU_K_TAKE = 5, ACU_K_REDUCE = 6, ACU_K_BYTES = 7, ACU_K_CLASSES = 8
} acu_kernel_class;
acu_status acu_kernel_stats(acu_ctx *ctx, int32_t kernel_class, double *out_total_ms, int64_t *out_launches);
acu_status acu_kernel_stats_reset(acu_ctx *ctx);


/* ------------------------------------------------------------------------- */
/* Bitmaps                                                                   */
/* ------------------------------------------------------------------------- */
/* popcount of bits [offset, offset+len)  — BooleanBuffer::count_set_bits
 * (arrow-buffer/src/buffer/boolean.rs) / BooleanArray::true_count when `validity`
 * is non-NULL (arrow-array/src/array/boolean_array.rs:175-187). */
acu_status acu_bitmap_count(acu_ctx *ctx, const uint8_t *bits, int64_t offset,
                            const uint8_t *validity, int64_t validity_offset, int64_t len,
                            int64_t *out_count);

/* ------------------------------------------------------------------------- */
/* filter — arrow-select/src/filter.rs                                       */
/* ------------------------------------------------------------------------- */
/* FilterBuilder::new + optimize + build (filter.rs:254-324): folds predicate nulls
 * into the mask (prep_null_mask_filter :167-171), counts selected rows, and keeps a
 * device-resident plan (normalised mask words + per-tile output offsets) that can be
 * applied to any number of columns (FilterPredicate, filter.rs:442-533). */
typedef struct acu_filter_plan acu_filter_plan;
typedef enum acu_filter_strategy {  /* IterationStrategy, filter.rs:328-365 */
  ACU_FILTER_NONE = 0, ACU_FILTER_ALL = 1, ACU_FILTER_INDEX = 2, ACU_FILTER_SLICES = 3
} acu_filter_strategy;

acu_status acu_filter_plan_create(acu_ctx *ctx, const acu_array *predicate /* boolean array */,
                                  acu_filter_plan **out_plan);
void acu_filter_plan_destroy(acu_ctx *ctx, acu_filter_plan *plan);
/* FilterBuilder::optimize (filter.rs:285-298): materialise IterationStrategy::Indices — the
 * selected row ids in ascending order, as index_dtype ACU_U32 or ACU_U64 (count entries). */
acu_status acu_filter_plan_indices(acu_ctx *ctx, const acu_filter_plan *plan, acu_dtype index_dtype,
                                   void *out_indices);
/* FilterBuilder::optimize for dense predicates: IterationStrategy::Slices(Vec<(usize, usize)>) = SlicesIterator
 * (filter.rs:44-77, :285-298): the runs of selected rows as [start, end) pairs in ascending order, out_pairs[2k] = start,
 * out_pairs[2k + 1] = end of run k. *out_slices = number of runs; out_pairs == NULL sizes only. Null predicate slots select
 * nothing (the plan's mask is prep_null_mask_filter'ed). */
acu_status acu_filter_plan_slices(acu_ctx *ctx, const acu_filter_plan *plan, uint64_t *out_pairs, int64_t capacity,
                                  int64_t *out_slices);
int64_t acu_filter_plan_count(const acu_filter_plan *plan);      /* FilterPredicate::count */
int64_t acu_filter_plan_len(const acu_filter_plan *plan);        /* predicate length       */
int32_t acu_filter_plan_strategy(const acu_filter_plan *plan);   /* acu_filter_strategy    */

/* filter_primitive / filter_native + filter_nulls (filter.rs:732-788, :512-533).
 * elem_bytes in {1,2,4,8,16,32}. Error if plan len > values.len (filter.rs:536-542).
 * out->values capacity: count*elem_bytes. out->has_validity = 0 when the source has no
 * nulls or the filtered result has none (filter.rs:518-526). */
acu_status acu_filter_primitive(acu_ctx *ctx, const acu_filter_plan *plan, int32_t elem_bytes,
                                const acu_array *values, acu_array_out *out);
/* filter_boolean / filter_bits (filter.rs:680-729): `values` is a boolean array. */
acu_status acu_filter_boolean(acu_ctx *ctx, const acu_filter_plan *plan, const acu_array *values,
                              acu_array_out *out);
/* filter_bytes for Utf8/Binary (offset_bytes = 4) and Large* (8) (filter.rs:893-928).
 * Two-phase: out_offsets (count+1 entries) is always written and *out_data_len returned;
 * value bytes are copied only if out_data != NULL (capacity out_data_capacity). `offsets` and
 * `out_offsets` must be aligned to offset_bytes (a misaligned pointer => ACU_ERR_INVALID_ARGUMENT,
 * and out_offsets is not written). */
acu_status acu_filter_bytes(acu_ctx *ctx, const acu_filter_plan *plan, int32_t offset_bytes,
                            const void *offsets, const uint8_t *data, const acu_array *nulls_of,
                            void *out_offsets, uint8_t *out_data, int64_t out_data_capacity,
                            int64_t *out_data_len, acu_array_out *out_nulls);

/* FilterBuilder::new(&cmp::op(a, b)?) without the BooleanArray in between (SURVEY.md §8(f) rank 2: arrow-ord/src/cmp.rs:220-382
 * feeding arrow-select/src/filter.rs:254-273): the comparison writes the plan's normalised mask (result & result validity —
 * a null comparison result selects nothing, prep_null_mask_filter filter.rs:167-171) and the per-tile counts directly;
 * the 2 x N/8-byte result bitmaps are never written to or re-read from HBM. The plan is identical to
 * acu_filter_plan_create(acu_cmp(dtype, op, a, b)). Errors as acu_cmp. */
acu_status acu_filter_plan_create_cmp(acu_ctx *ctx, acu_dtype dtype, acu_cmp_op op, const acu_array *a,
                                      const acu_array *b, acu_filter_plan **out_plan);

/* ------------------------------------------------------------------------- */
/* nullif / zip — arrow-select/src/nullif.rs, zip.rs                         */
/* ------------------------------------------------------------------------- */
/* nullif(left, right) (nullif.rs:44-113): the result shares left's value buffers; only the validity changes:
 * out->validity = left.validity & !(right.values & right.validity) (bit offset 0), out->null_count, out->has_validity = 0
 * when no slot is null (ArrayDataBuilder::build drops an all-valid NullBuffer). `left` may be an array of any kind: only
 * its validity / len are read; out->values is not touched. Length mismatch => ACU_ERR_COMPUTE. */
acu_status acu_nullif(acu_ctx *ctx, const acu_array *left, const acu_array *right /* boolean */, acu_array_out *out);

/* zip(mask, truthy, falsy) (zip.rs:99-226) for fixed-width values of elem_bytes in {1,2,4,8,16,32}: out[i] = truthy[i] where
 * mask[i] is Some(true), else falsy[i]; either side may be a scalar (is_scalar, len 1); value bytes are copied blindly from
 * the chosen side (also under nulls); the result carries a validity buffer iff some input has nulls and the result has at
 * least one. Both sides scalar = ScalarZipper (zip.rs:248-440): with one null scalar every slot holds the other value and
 * the validity (always present) is the mask / its negation. ACU_ERR_INVALID_ARGUMENT "all arrays should have the same
 * length" / "scalar arrays must have 1 element". */
acu_status acu_zip(acu_ctx *ctx, int32_t elem_bytes, const acu_array *mask /* boolean */, const acu_array *truthy,
                   const acu_array *falsy, acu_array_out *out);

/* zip of Utf8 / Binary (offset_bytes 4), LargeUtf8 / LargeBinary (8), Utf8View / BinaryView, Boolean and
 * FixedSizeBinary(byte_width) columns. Scalars, lengths, texts and mask nulls as acu_zip; masks, validity and operands may
 * start at any bit offset or pointer alignment, with two exceptions: offsets are aligned to offset_bytes, as for the other
 * byte calls, and views (truthy's, falsy's and out_views) to 16 bytes, the alignment of the u128 views buffer
 * (ScalarBuffer<u128>); a misaligned views pointer => ACU_ERR_INVALID_ARGUMENT "views must be 16-byte aligned". The caller checks that
 * both sides have one data type ("arguments need to have the same data type"). Three paths, as the reference:
 *   - at least one side an array, and Boolean / FixedSizeBinary with two scalars (zip_impl over MutableArrayData,
 *     zip.rs:148-210, FallbackImpl zip.rs:318-336): row i is row i of the chosen side (row 0 of a scalar), its bytes and bits
 *     under nulls included; has_validity iff some input has a null and the result has one. Byte offsets are rebased on the
 *     running total: an i32 end past i32::MAX is ACU_ERR_INVALID_ARGUMENT "offset overflow: data exceeds the capacity of the
 *     offset type. ..." (try_extend_offsets) with detail.index = the first such row. A falsy view longer than 12 bytes gets
 *     buffer_index += truthy->n_buffers (wrapping u32), nulls included, and *out_buffers = ACU_ZIP_BUFFERS_BOTH.
 *   - two Utf8 / Binary scalars (BytesScalarImpl, zip.rs:439-660): both valid: no NullBuffer; one valid: its value where the
 *     predicate (its negation for a valid falsy) holds, empty null rows elsewhere, has_validity = 1; both null: empty rows,
 *     all null. An i32 overflow is the reference's panic, ACU_ERR_PANIC_OUT_OF_BOUNDS "offset overflow" (one value in every
 *     row, or one valid scalar) or "overflow" (a mixed mask of two valid scalars), detail.index = -1.
 *   - two view scalars (ByteViewScalarImpl, zip.rs:673-860): both valid: an all-true mask gives the truthy view and
 *     buffers, an all-false one the falsy's, a mixed one the truthy buffers and, when falsy has any, falsy's after them, its
 *     view's buffer index raised by truthy->n_buffers even when the view is inline; no NullBuffer. One valid: its view in
 *     every row, its buffers, nulls = the predicate (negated for falsy), or zero views and no buffers when no row is
 *     selected. Both null: zero views, no buffers, all null.
 * acu_zip_bytes is two-phase like acu_filter_bytes: out_offsets (mask->len + 1 entries) always written, *out_data_len
 * returned, bytes copied only when out_data != NULL; an offset overflow is reported by the sizing call already. acu_zip_byte_view
 * writes mask->len views; of each side's data buffers it reads only n_buffers (neither `buffers` nor the bytes they point
 * at, so a caller may pass buffers = NULL). Boolean results are a bitmap at bit offset 0; FixedSizeBinary
 * results have mask->len x byte_width bytes at any alignment (byte_width < 0 => ACU_ERR_INVALID_ARGUMENT). Synchronous
 * (refused inside a stream-ordered section); kernel time in ACU_K_BYTES (bytes, views) / ACU_K_ARITH (Boolean,
 * FixedSizeBinary). */
typedef enum acu_zip_buffers {  /* which data-buffer list a view zip result references */
  ACU_ZIP_BUFFERS_NONE = 0, ACU_ZIP_BUFFERS_TRUTHY = 1, ACU_ZIP_BUFFERS_FALSY = 2, ACU_ZIP_BUFFERS_BOTH = 3
} acu_zip_buffers;
struct acu_bytes_array;
struct acu_view_array;
acu_status acu_zip_bytes(acu_ctx *ctx, int32_t offset_bytes, const acu_array *mask, const struct acu_bytes_array *truthy,
                         const struct acu_bytes_array *falsy, void *out_offsets, uint8_t *out_data, int64_t out_data_capacity,
                         int64_t *out_data_len, acu_array_out *out_nulls);
acu_status acu_zip_byte_view(acu_ctx *ctx, const acu_array *mask, const struct acu_view_array *truthy,
                             const struct acu_view_array *falsy, void *out_views, acu_array_out *out_nulls, int32_t *out_buffers);
acu_status acu_zip_boolean(acu_ctx *ctx, const acu_array *mask, const acu_array *truthy, const acu_array *falsy,
                           acu_array_out *out);
acu_status acu_zip_fixed_size_binary(acu_ctx *ctx, int32_t byte_width, const acu_array *mask, const acu_array *truthy,
                                     const acu_array *falsy, acu_array_out *out);

/* ------------------------------------------------------------------------- */
/* take — arrow-select/src/take.rs                                           */
/* ------------------------------------------------------------------------- */
/* take_primitive = take_native + take_nulls (take.rs:405-457). `indices.values`
 * has native type index_dtype (any integer type; ToIndices take.rs:1030-1084:
 * i8/i16 sign-extend to u32, i32/i64 reinterpret). check_bounds != 0 =>
 * TakeOptions{check_bounds:true} (take.rs:167-209): ACU_ERR_COMPUTE with the lowest
 * offending index. Otherwise an out-of-bounds VALID index returns
 * ACU_ERR_PANIC_OUT_OF_BOUNDS (the reference panics) and an out-of-bounds index in a
 * NULL slot yields T::default() = 0 (take.rs:442-448). */
acu_status acu_take_primitive(acu_ctx *ctx, int32_t elem_bytes, const acu_array *values,
                              const acu_array *indices, acu_dtype index_dtype,
                              int32_t check_bounds, acu_array_out *out);
/* take_boolean / take_bits (take.rs:460-496). */
acu_status acu_take_boolean(acu_ctx *ctx, const acu_array *values, const acu_array *indices,
                            acu_dtype index_dtype, int32_t check_bounds, acu_array_out *out);
/* take_bytes (take.rs:499-627); also Dictionary<K,Utf8> -> Utf8 cast =
 * unpack_dictionary (arrow-cast/src/cast/dictionary.rs:310-317) with values = the
 * dictionary and indices = the keys. i32 offset overflow => ACU_ERR_OFFSET_OVERFLOW
 * (take.rs:520-523). Two-phase like acu_filter_bytes, with the same alignment rule for
 * `offsets` and `out_offsets`. `nulls_of` carries the
 * validity/len/null_count of the byte array (its `values` member is ignored). */
acu_status acu_take_bytes(acu_ctx *ctx, int32_t offset_bytes, const void *offsets,
                          const uint8_t *data, const acu_array *nulls_of,
                          const acu_array *indices, acu_dtype index_dtype, int32_t check_bounds,
                          void *out_offsets, uint8_t *out_data, int64_t out_data_capacity,
                          int64_t *out_data_len, acu_array_out *out_nulls);

/* ------------------------------------------------------------------------- */
/* filter / take of List, LargeList and FixedSizeList columns                */
/* ------------------------------------------------------------------------- */
/* One level of a list column (GenericListArray / FixedSizeListArray). The child is NOT described here: the calls work on one
 * level at a time and the caller filters / takes the child with the plan / row map they return, through any filter / take
 * entry point (or these calls again for a nested list).
 *   kind      ACU_LIST (i32 offsets), ACU_LARGE_LIST (i64) or ACU_FIXED_SIZE_LIST (list_size >= 0 children per row);
 *   offsets   LIST / LARGE_LIST: nulls.len + 1 entries from logical row 0, ABSOLUTE child rows (a sliced list has
 *             offsets[0] != 0), aligned to their width; ignored for FIXED_SIZE_LIST, whose row i is the child rows
 *             [i * list_size, (i + 1) * list_size) (the child is already advanced to the list's logical row 0);
 *   nulls     len / validity / validity_offset / null_count of the list (`values` ignored);
 *   child_len rows of the child. */
typedef enum acu_list_kind { ACU_LIST = 0, ACU_LARGE_LIST = 1, ACU_FIXED_SIZE_LIST = 2 } acu_list_kind;
typedef struct acu_list_array {
  int32_t kind;
  int32_t list_size;
  const void *offsets;
  acu_array nulls;
  int64_t child_len;
} acu_list_array;

/* filter of a list (filter.rs:535-625: the MutableArrayData fallback). Every selected row keeps its whole child range, null
 * rows included. out_offsets (LIST / LARGE_LIST only, count + 1 entries of the list's width, starting at 0) and out_nulls
 * (filter_nulls: a NullBuffer only when the result has a null; capacity acu_bitmap_bytes(count)). *out_child_plan is a new
 * plan over the child rows [0, offsets[plan len]) selecting the selected rows' ranges; the caller filters the child with it
 * and destroys it. Predicate longer than the list => ACU_ERR_INVALID_ARGUMENT "Filter predicate of length {p} is larger
 * than target array of length {n}". Strategy NONE / ALL: the reference returns an empty array / values.slice(0, count);
 * here the offsets are rebased to 0 and the child is cut to the selected range, which arrow-data's equality treats as the
 * same array, and the NullBuffer presence is that of acu_filter_primitive (ALL keeps the list's NullBuffer as it is).
 * Synchronous (not available inside a stream-ordered section); the child plan's expansion counts in ACU_K_FILTER_PLAN. */
acu_status acu_filter_list(acu_ctx *ctx, const acu_filter_plan *plan, const acu_list_array *list, void *out_offsets,
                           acu_array_out *out_nulls, acu_filter_plan **out_child_plan);

/* take of a list. Two-phase: out_child_indices == NULL sizes only (writes out_offsets, out_nulls and *out_child_rows); the
 * second call also writes the child row map, out_child_indices[k] = the child row that becomes output child row k, as
 * child_index_dtype ACU_U32 or ACU_U64 (ACU_U32 needs child_len <= UINT32_MAX; FIXED_SIZE_LIST takes ACU_U32 only, as the
 * reference does); capacity < *out_child_rows => ACU_ERR_INVALID_ARGUMENT. The caller then takes the child with that map.
 * keep_null_ranges = 0 is take_list (take.rs:646-727) / take_fixed_size_list (:765-795):
 *   - out_nulls = take_nulls(list.nulls, indices) (a NullBuffer only when some row is null for FIXED_SIZE_LIST);
 *   - LIST / LARGE_LIST: a null output row gets an empty range, out_offsets start at 0, the map has no nulls;
 *   - FIXED_SIZE_LIST: row i maps to the u32 child rows (u32)(index * list_size) + k, wrapping, and a null index to
 *     list_size null child rows (out_child_index_nulls, capacity acu_bitmap_bytes(rows); has_validity iff an index is null);
 *   - check_bounds != 0: ACU_ERR_COMPUTE "Array index out of bounds, cannot get item at index {i} from {len} entries";
 *   - otherwise a valid out-of-bounds index is the reference's panic, ACU_ERR_PANIC_OUT_OF_BOUNDS at the lowest such row:
 *     "assertion failed: idx < self.bit_len" (take_bits) when the list has a null, else "index out of bounds: the len is
 *     {len + 1} but the index is {i}" (the offsets slice). A FIXED_SIZE_LIST takes its child before it reads the list's
 *     validity: its sizing call succeeds and the call that writes the row map writes it, then returns the take_bits panic,
 *     so that the caller can take the child first and report the child's own error ahead of it;
 *   - LIST: the first output row whose end passes i32::MAX is from_usize(..).unwrap()'s panic: ACU_ERR_PANIC_OUT_OF_BOUNDS
 *     "called `Option::unwrap()` on a `None` value" (without list nulls the lower of this row and an out-of-bounds row).
 * keep_null_ranges = 1 is the child step of a parent list's take (MutableArrayData::extend, arrow-data/src/transform/
 * list.rs): every row keeps its range, null rows included; the indices carry no nulls; the nulls are those of take_nulls;
 * an i32 offset overflow is ACU_ERR_INVALID_ARGUMENT "offset overflow: data exceeds the capacity of the offset type. ..."
 * (try_extend_offsets) at the first such row. Synchronous; the row map's kernels count in ACU_K_TAKE and the offsets pass
 * in ACU_K_BYTES, like every user of the offsets engine. */
acu_status acu_take_list(acu_ctx *ctx, const acu_list_array *list, const acu_array *indices, acu_dtype index_dtype,
                         int32_t check_bounds, int32_t keep_null_ranges, void *out_offsets, acu_array_out *out_nulls,
                         acu_dtype child_index_dtype, void *out_child_indices, int64_t capacity, int64_t *out_child_rows,
                         acu_array_out *out_child_index_nulls);

/* The Utf8 / Binary child of a list take: MutableArrayData::extend of every row of `indices` (a child row map without
 * nulls), so null rows keep their bytes, unlike acu_take_bytes. Nulls as take_nulls (a NullBuffer only when some row is
 * null). An i32 offset overflow => ACU_ERR_INVALID_ARGUMENT "offset overflow: data exceeds the capacity of the offset type.
 * Try splitting into smaller batches or using a larger type (e.g. LargeStringArray / LargeBinaryArray instead of
 * StringArray / BinaryArray)", detail.index = the first row whose end passes i32::MAX. Indices with a null =>
 * ACU_ERR_INVALID_ARGUMENT. Two-phase like acu_take_bytes; synchronous; kernel time in ACU_K_BYTES. */
acu_status acu_take_bytes_extend(acu_ctx *ctx, int32_t offset_bytes, const void *offsets, const uint8_t *data,
                                 const acu_array *nulls_of, const acu_array *indices, acu_dtype index_dtype, void *out_offsets,
                                 uint8_t *out_data, int64_t out_data_capacity, int64_t *out_data_len, acu_array_out *out_nulls);

/* ------------------------------------------------------------------------- */
/* numeric — arrow-arith/src/numeric.rs, arity.rs                            */
/* ------------------------------------------------------------------------- */
/* add/add_wrapping/sub/sub_wrapping/mul/mul_wrapping/div/rem (numeric.rs:36-81).
 * a and b have native type `dtype`; either may be a scalar (is_scalar, len 1).
 * Floats: every op is the IEEE single operation (no FMA contraction), never errors.
 * Integers: wrapping ops via `binary` (op evaluated at every slot), checked ops via
 * `try_binary` (zero under nulls, first failing valid index reported)
 * (arity.rs:104-135, :254-299). Length mismatch => ACU_ERR_COMPUTE.
 * In place (binary_mut / try_binary_mut / unary_mut / try_unary_mut, arity.rs:137-252,301-363): out->values may BE a->values
 * (or b->values), and out->validity an input validity buffer whose bit offset is 0 — every element / bitmap word is read
 * before the same element / word is written. A failed checked op leaves the buffer partially overwritten (the reference's
 * try_binary_mut consumes its input as well). */
acu_status acu_arith(acu_ctx *ctx, acu_dtype dtype, acu_arith_op op, const acu_array *a,
                     const acu_array *b, acu_array_out *out);
/* neg (checked != 0) / neg_wrapping (numeric.rs:103-186). ACU_I128 (Decimal128) is always neg_checked, whatever
 * `checked` says: the reference's neg_wrapping falls back to neg for every non-integer type (numeric.rs:181-186). For the
 * same reason a Decimal32 / Decimal64 negation is acu_neg(ACU_I32 / ACU_I64, checked = 1). */
acu_status acu_neg(acu_ctx *ctx, acu_dtype dtype, int32_t checked, const acu_array *a,
                   acu_array_out *out);

/* ------------------------------------------------------------------------- */
/* bitwise — arrow-arith/src/bitwise.rs                                      */
/* ------------------------------------------------------------------------- */
/* bitwise_and / or / xor / and_not / shift_left / shift_right (array-array, through `binary`, arity.rs:104-135), their
 * _scalar forms (b->is_scalar; and_not has none) and bitwise_not (b == NULL), through `unary`, for the integer dtypes
 * ACU_I8 .. ACU_U64:
 *   - the op is evaluated at every slot, so the values under nulls are op(a[i], b[i]); the result's NullBuffer is the
 *     union of the inputs' (array-array) or a's (scalar forms, not); an empty array-array result has no NullBuffer;
 *   - shifts are wrapping_shl / wrapping_shr by b's two's-complement bit pattern modulo the bit width (a u64 shifted by
 *     u64::MAX shifts by 63); shift_right is arithmetic for signed and logical for unsigned types;
 *   - length mismatch => ACU_ERR_COMPUTE "Cannot perform binary operation on arrays of different length";
 *   - a scalar `a`, a null scalar `b`, a scalar and_not, b == NULL for any op but NOT, a float or ACU_I128 dtype, or an op
 *     outside acu_bitwise_op => ACU_ERR_INVALID_ARGUMENT.
 * In place as acu_arith; stream-ordered inside a section like acu_arith; kernel time counts in ACU_K_ARITH. */
acu_status acu_bitwise(acu_ctx *ctx, acu_dtype dtype, acu_bitwise_op op, const acu_array *a, const acu_array *b,
                       acu_array_out *out);

/* ------------------------------------------------------------------------- */
/* decimal arithmetic — decimal_op (arrow-arith/src/numeric.rs:970-1107)     */
/* ------------------------------------------------------------------------- */
/* DataType::Decimal32 / 64 / 128(precision, scale): byte_width 4 / 8 / 16 (values ACU_I32 / ACU_I64 / ACU_I128).
 * Decimal256 is not supported. */
typedef struct acu_decimal_type {
  int32_t byte_width;
  uint8_t precision;
  int8_t scale;
  uint8_t reserved[2];
} acu_decimal_type;

/* add / sub / mul / div / rem of two decimal operands of the same width, with the reference's Hive precision / scale rules
 * (MAX_PRECISION = MAX_SCALE = 9 / 18 / 38 for widths 4 / 8 / 16). *out_type receives the result type; out->values holds
 * byte_width bytes per row.
 *   - add, sub (s = max(s1, s2)): l * 10^(s - s1) +/- r * 10^(s - s2), each multiplication checked, left before right;
 *     mul: l * r checked, scale s1 + s2; div (scale min(s1 + 4, MAX_SCALE)): l * l_mul / r * r_mul, truncated toward zero;
 *     rem: l * l_mul % r * r_mul with the multipliers of add computed WRAPPING (pow_wrapping), and MIN % -1 an overflow
 *     (mod_checked, not the integer rem's 0). The wrapping ops are checked like the others.
 *   - rows are evaluated only where both sides are valid (try_binary / try_unary: zero under nulls); a scalar (is_scalar)
 *     is rescaled per row, so its overflow is reported at the lowest valid row of the array and not at all when no row is
 *     valid; a null scalar gives an all-null result. The error of the lowest failing valid row is returned:
 *     ACU_ERR_ARITHMETIC_OVERFLOW "Overflow happened on: {a} {op} {b}" with the operands of the failing step (a rescale
 *     prints the rescaled operand and its multiplier, "10 * 100000000000000000000000000000000000000"), or
 *     ACU_ERR_DIVIDE_BY_ZERO "Divide by zero error". detail.index = that row, lhs_bits / rhs_bits = the low 64 bits of
 *     the row's raw operands.
 *   - before any row is read, also for empty arrays: ACU_ERR_ARITHMETIC_OVERFLOW "Overflow happened on: 10 ^ {exp}" when
 *     a multiplier does not fit the native type; ACU_ERR_INVALID_ARGUMENT "Output scale of Decimal128(3, 3) *
 *     Decimal128(37, 37) would exceed max scale of 38" for mul. After the rows (a row error wins), the result type is
 *     validated like with_precision_and_scale: ACU_ERR_INVALID_ARGUMENT "precision cannot be 0, has to be between [1,
 *     {MAX}]", "scale {s} is greater than max {MAX}", "scale {s} is greater than precision {p}".
 *   - The result type follows Rust's i8 / u8 arithmetic (saturating_add, `as u8`, .min(MAX_PRECISION)). Where the
 *     reference's `p as i8 - s` or a scale difference leaves the i8 range (a scale below -89), the reference panics in
 *     debug builds and wraps in release builds; this library wraps, like a release build: the difference is taken
 *     modulo 256 and a negative exponent reads as a huge u32 (so the multiplier overflows, or is 0 for rem).
 *   - an operand type that validate_decimal_precision_and_scale rejects (precision 0 or above MAX_PRECISION, scale above
 *     MAX_SCALE or above a positive precision), byte widths that differ or are not 4 / 8 / 16, an ACU_I128 pointer that is
 *     not 16-byte aligned, or op outside acu_arith_op => ACU_ERR_INVALID_ARGUMENT at call time; lengths that differ =>
 *     ACU_ERR_COMPUTE "Cannot perform a binary operation on arrays of different length".
 * Stream-ordered inside a section (the result-type validation then reports at the fetch); kernel time counts in
 * ACU_K_ARITH. In place as acu_arith. */
acu_status acu_decimal_arith(acu_ctx *ctx, acu_arith_op op, const acu_decimal_type *lt, const acu_array *a,
                             const acu_decimal_type *rt, const acu_array *b, acu_decimal_type *out_type,
                             acu_array_out *out);

/* ------------------------------------------------------------------------- */
/* cmp — arrow-ord/src/cmp.rs                                                */
/* ------------------------------------------------------------------------- */
/* eq/neq/lt/lt_eq/gt/gt_eq/distinct/not_distinct (cmp.rs:79-202). Result is a boolean
 * array: out->values = bit-packed results. Floats compare by IEEE-754 totalOrder
 * (arrow-array/src/arithmetic.rs:400-410). ACU_I128 (Decimal128) compares as signed i128; decimals compare as their
 * native integers, so the reference's refusal of operands whose decimal types differ ("Invalid comparison operation:
 * {l_t} {op} {r_t}", cmp.rs:260-263) belongs to the caller, which knows the logical types. */
acu_status acu_cmp(acu_ctx *ctx, acu_dtype dtype, acu_cmp_op op, const acu_array *a,
                   const acu_array *b, acu_array_out *out);

/* The same eight comparisons on variable-width operands (SURVEY.md §8(f) rank 3).
 * acu_bytes_array = GenericByteArray (Utf8 / Binary: offset_bytes 4, LargeUtf8 / LargeBinary: 8; ArrayOrd cmp.rs:783-801):
 * `offsets` points at the offset of logical row 0 (nulls.len + 1 entries), `nulls` carries len / validity / null_count /
 * is_scalar (its `values` member is ignored). acu_view_array = GenericByteViewArray (Utf8View / BinaryView; ArrayOrd
 * cmp.rs:803-898): `views` = 16 bytes per row (length u32, then 12 inline bytes, or 4-byte prefix + buffer index u32 + offset
 * u32: arrow-data/src/byte_view.rs), `buffers` = a HOST array of n_buffers DEVICE pointers to the data buffers. Bytes compare
 * like Rust's `&[u8]` (lexicographic on unsigned bytes, then length). Equality of a view array against a non-null constant of
 * at most 4 bytes takes the reference's short-constant path (eq_inline_scalar, cmp.rs:405-435: one masked 64-bit compare per
 * view). Null handling, result layout and errors exactly as acu_cmp. */
typedef struct acu_bytes_array {
  const void *offsets;
  const uint8_t *data;
  acu_array nulls;
} acu_bytes_array;
typedef struct acu_view_array {
  const void *views;
  const uint8_t *const *buffers;
  int32_t n_buffers;
  int32_t reserved;
  acu_array nulls;
} acu_view_array;
acu_status acu_cmp_bytes(acu_ctx *ctx, int32_t offset_bytes, acu_cmp_op op, const acu_bytes_array *l,
                         const acu_bytes_array *r, acu_array_out *out);
acu_status acu_cmp_byte_view(acu_ctx *ctx, acu_cmp_op op, const acu_view_array *l, const acu_view_array *r,
                             acu_array_out *out);

/* ------------------------------------------------------------------------- */
/* filter / take of RunEndEncoded columns                                    */
/* ------------------------------------------------------------------------- */
/* The run ends of a RunArray (arrow-array/src/array/run_array.rs, RunEndBuffer arrow-buffer/src/buffer/run.rs). The values
 * child is NOT described here: the calls return a plan / value indices and the caller filters / takes the values child with
 * them through the entry point of its type, as for a list's child.
 *   run_end_dtype ACU_I16, ACU_I32 or ACU_I64;
 *   run_ends      n_runs entries from physical entry 0 (not advanced by `offset`), aligned to their width;
 *   offset, len   the logical slice: logical row i is the first physical run whose end is > offset + i.
 * A malformed run-ends buffer (not strictly increasing, or not covering offset + len) gives an unspecified result, but
 * every search is clamped to [0, n_runs). n_runs == 0 with len > 0, a negative offset / len or an unaligned pointer =>
 * ACU_ERR_INVALID_ARGUMENT. */
typedef struct acu_run_array {
  int32_t run_end_dtype;
  int32_t reserved;
  const void *run_ends;
  int64_t n_runs;
  int64_t offset;
  int64_t len;
} acu_run_array;

/* filter of a RunArray (filter_run_end_array, arrow-select/src/filter.rs:628-677). Predicate longer than the logical length =>
 * ACU_ERR_INVALID_ARGUMENT "Filter predicate of length {p} is larger than target array of length {n}"; a shorter one drops the
 * runs past it. Strategy NONE / ALL: nothing is written, *out_runs = 0 and *out_values_plan = NULL; the reference returns an
 * empty RunArray / values.slice(0, count) (the run ends and values as they are, logical length count). Otherwise, over the
 * physical runs [start, end] of the slice (get_start_physical_index / get_end_physical_index, run.rs:232-267), a run is kept
 * iff a selected row lies in [previous clipped end, min(run_end - offset, p)), and its new end is the number of selected
 * rows below that clipped end: out_run_ends (capacity min(count, n_runs) entries of the run-end type) gets the *out_runs
 * kept runs' ends, *out_values_start = start, and *out_values_plan is a new plan over the values rows [start, end] (length
 * end - start + 1) selecting the kept runs. The caller filters values.slice(start, end - start + 1) with it (a top-level
 * filter of the values child, with that plan's own strategy) and destroys it. Synchronous; the physical bounds and the
 * keep / rank pass count in ACU_K_FILTER_PLAN, the run-end compaction in ACU_K_FILTER. */
acu_status acu_filter_run_end(acu_ctx *ctx, const acu_filter_plan *plan, const acu_run_array *ree, void *out_run_ends,
                              int64_t *out_runs, int64_t *out_values_start, acu_filter_plan **out_values_plan);

/* The values child of a RunArray as take_run's merge compares it (make_comparator with SortOptions::default(), arrow-ord/src/
 * ord.rs): two nulls are equal, a null never equals a valid value, two valid values are equal iff
 *   ACU_RUN_VALUES_FIXED   their `width` (1, 2, 4, 8 or 16) bytes are equal: integers, Decimal32/64/128, and floats under
 *                          total_cmp (so -0.0 != 0.0 and NaNs with different payloads differ); `array` from physical row 0;
 *   ACU_RUN_VALUES_BOOLEAN their bits are equal; `array` (values bitmap at values_offset) from physical row 0;
 *   ACU_RUN_VALUES_BYTES   their bytes are equal; `bytes` with offsets of `width` 4 (Utf8 / Binary) or 8 (Large*);
 *   ACU_RUN_VALUES_VIEW    their bytes are equal; `view` (Utf8View / BinaryView).
 * ACU_RUN_VALUES_NESTED (a list or other nested child) is refused by acu_take_run_end (below); any other kind or width =>
 * ACU_ERR_INVALID_ARGUMENT. */
typedef enum acu_run_values_kind {
  ACU_RUN_VALUES_FIXED = 0, ACU_RUN_VALUES_BOOLEAN = 1, ACU_RUN_VALUES_BYTES = 2, ACU_RUN_VALUES_VIEW = 3,
  ACU_RUN_VALUES_NESTED = 4
} acu_run_values_kind;
typedef struct acu_run_values {
  int32_t kind;
  int32_t width;
  acu_array array;
  acu_bytes_array bytes;
  acu_view_array view;
} acu_run_values;

/* take of a RunArray (take_run, arrow-select/src/take.rs:948-995). In order:
 *   - a non-integer index type => ACU_ERR_INVALID_ARGUMENT "Take only supported for integers, got {type}";
 *   - check_bounds != 0 (take.rs:167-209, null slots ignored): ACU_ERR_COMPUTE "Array index out of bounds, cannot get item
 *     at index {i} from {len} entries";
 *   - no indices: *out_runs = 0 (new_empty_array);
 *   - the indices converted by ToIndices (take.rs:1030-1084: Int8 / Int16 sign-extend to UInt32, Int32 reinterprets as UInt32,
 *     Int64 as UInt64), their largest VALUE, null slots included, at least len => ACU_ERR_INVALID_ARGUMENT "Logical index
 *     {max} is out of bounds for RunArray of length {len}" (get_physical_indices, run.rs:321-378, run_array.rs:343-356);
 *   - a nested values child, where take_run builds its comparator => ACU_ERR_NOT_YET_IMPLEMENTED "take of a RunEndEncoded
 *     column with nested values is not yet implemented";
 *   - more output rows than the run-end type holds (from_usize(..).unwrap()) => ACU_ERR_PANIC_OUT_OF_BOUNDS "called
 *     `Option::unwrap()` on a `None` value".
 * Output row ix >= 1 starts a new run iff its physical run differs from row ix - 1's and their values are not equal under
 * `values` (above). out_run_ends gets the *out_runs run ends (the last is indices.len) in the run-end type; out_value_indices
 * the physical row of each run's last row, UInt32 for indices that convert to UInt32 and UInt64 for Int64 / UInt64 (more than
 * 2^32 runs with UInt32 indices => ACU_ERR_NOT_YET_IMPLEMENTED). Both need capacity indices.len entries. The caller then
 * takes the values child with out_value_indices (no nulls) through the take entry point of its type. Synchronous; kernel
 * time counts in ACU_K_TAKE, the boundary plan and its compaction in ACU_K_FILTER_PLAN / ACU_K_FILTER. */
acu_status acu_take_run_end(acu_ctx *ctx, const acu_run_array *ree, const acu_run_values *values, const acu_array *indices,
                            acu_dtype index_dtype, int32_t check_bounds, void *out_run_ends, void *out_value_indices,
                            int64_t *out_runs);

/* ------------------------------------------------------------------------- */
/* filter / take of Struct, sparse Union and dense Union columns             */
/* ------------------------------------------------------------------------- */
/* A struct's fields are filtered / taken one by one through the entry point of their type; these two calls produce the
 * struct's own NullBuffer. `nulls_of` carries the struct's len / validity / validity_offset / null_count (`values` ignored).
 *
 * acu_filter_nulls: predicate.filter_nulls(array.nulls()) (filter_struct, arrow-select/src/filter.rs:1010-1030): out
 * (capacity acu_bitmap_bytes(count)) holds the selected rows' validity, with a NullBuffer only when one of them is null;
 * strategy ALL keeps the NullBuffer as it is (values.slice(0, count)), NONE has none. Predicate longer than the struct =>
 * ACU_ERR_INVALID_ARGUMENT "Filter predicate of length {p} is larger than target array of length {n}". Synchronous; kernel
 * time in ACU_K_FILTER.
 *
 * acu_take_nulls: the validity of take_impl's Struct arm (take.rs:270-298): row j is valid iff index j is valid and
 * array.is_valid(index j). A NullBuffer only when a row is null (StructArray::try_new drops one without nulls; an
 * empty-field struct keeps it, which is the caller's to build: out->validity is then written whenever the indices or the
 * struct have a validity buffer). In order: a non-integer index type => ACU_ERR_INVALID_ARGUMENT "Take only supported for
 * integers, got {type}"; check_bounds != 0 => ACU_ERR_COMPUTE "Array index out of bounds, cannot get item at index {i} from
 * {len} entries"; then out is written. Unlike take_nulls, is_valid reads a validity buffer that has no null in the slice:
 * when nulls_of has a validity buffer, a valid index >= len is BooleanBuffer::value's panic, ACU_ERR_PANIC_OUT_OF_BOUNDS
 * "assertion failed: idx < self.bit_len" at the lowest such row. The reference takes the fields before it reads the
 * validity, so that panic is returned after out is written: the caller takes the fields first and reports a field's own
 * error ahead of it. Without a validity buffer no row is read. Synchronous; kernel time in ACU_K_TAKE. */
acu_status acu_filter_nulls(acu_ctx *ctx, const acu_filter_plan *plan, const acu_array *nulls_of, acu_array_out *out);
acu_status acu_take_nulls(acu_ctx *ctx, const acu_array *nulls_of, const acu_array *indices, acu_dtype index_dtype,
                          int32_t check_bounds, acu_array_out *out);

/* One level of a union column (UnionArray, arrow-array/src/array/union_array.rs). The children are NOT described here: the
 * caller filters / takes each child through the entry point of its type, as for a list's child.
 *   mode            ACU_UNION_SPARSE or ACU_UNION_DENSE;
 *   n_fields        1..ACU_UNION_MAX_FIELDS;
 *   field_type_ids  host array of n_fields distinct type ids in [0, 127], in field order;
 *   type_ids        Int8, on the device, from logical row 0;
 *   offsets         Int32, dense only, on the device, from logical row 0, 4-byte aligned;
 *   len             logical rows.
 * A type id that names no field, or a dense offset outside its child, is malformed input: the result is then unspecified,
 * but no access leaves the buffers. A bad mode, field count, field type id or alignment => ACU_ERR_INVALID_ARGUMENT. */
#define ACU_UNION_MAX_FIELDS 128
typedef enum acu_union_mode { ACU_UNION_SPARSE = 0, ACU_UNION_DENSE = 1 } acu_union_mode;
typedef struct acu_union_array {
  int32_t mode;
  int32_t n_fields;
  const int8_t *field_type_ids;
  const int8_t *type_ids;
  const int32_t *offsets;
  int64_t len;
} acu_union_array;

/* filter of a union. Sparse (filter_sparse_union, filter.rs:1033-1054): out_type_ids (count entries) = filter_primitive of
 * the type ids; the caller filters every child with the same plan. Dense (the MutableArrayData fallback, filter.rs:597-622,
 * build_extend_dense in arrow-data/src/transform/union.rs): out_type_ids as above; out_offsets (count entries) = for every
 * selected row, the number of earlier selected rows of its type id; out_child_rows (capacity count Int32 entries) = the
 * selected rows' source offsets grouped by field in field order, each group in output order; out_field_starts (host,
 * n_fields + 1 entries): field f's rows are [starts[f], starts[f + 1]). The caller extends child f with those rows as ACU_I32
 * indices (MutableArrayData::extend, the child step of a list take). Predicate longer than the union =>
 * ACU_ERR_INVALID_ARGUMENT "Filter predicate of length {p} is larger than target array of length {n}". Strategy NONE / ALL:
 * nothing is written (the reference returns new_empty_array / values.slice(0, count); a dense slice keeps its children
 * whole, a sparse one slices them). Synchronous; the compaction counts in ACU_K_FILTER, the partition in ACU_K_FILTER_PLAN. */
acu_status acu_filter_union(acu_ctx *ctx, const acu_filter_plan *plan, const acu_union_array *u, int8_t *out_type_ids,
                            int32_t *out_offsets, int32_t *out_child_rows, int64_t *out_field_starts);

/* take of a union (take.rs:334-382). In order:
 *   - the index type, check_bounds and take_native's out-of-bounds panics exactly as acu_take_primitive (type ids first,
 *     then the dense offsets); a null index gathers the type id / offset when it is in bounds and 0 when it is not;
 *   - every output is written: out_type_ids (indices.len entries); for a dense union out_offsets (the running count per
 *     type id), out_child_rows (capacity indices.len Int32 entries) and out_field_starts (host, n_fields + 1 entries), laid
 *     out as in acu_filter_union; the caller takes child f with rows [starts[f], starts[f + 1]) as ACU_I32 indices (plain
 *     take), or every child of a sparse union with the indices themselves;
 *   - a taken type id that names no field (reachable: a null out-of-bounds index yields 0) => ACU_ERR_INVALID_ARGUMENT
 *     "Type Ids values must match one of the field type ids" (UnionArray::try_new, union_array.rs:177-242), returned after
 *     the outputs are written, so that the caller takes the children first and reports a child's error ahead of it;
 *   - then, for a dense union, a field with more than i32::MAX output rows => ACU_ERR_INVALID_ARGUMENT "Offsets must be
 *     non-negative and within the length of the Array", also after the outputs are written.
 * The new offsets are i32: past i32::MAX rows of one field they wrap (two's complement), in acu_filter_union as well, as the
 * reference's i32 running counts do in a release build.
 * Synchronous; the gathers and the partition count in ACU_K_TAKE. */
acu_status acu_take_union(acu_ctx *ctx, const acu_union_array *u, const acu_array *indices, acu_dtype index_dtype,
                          int32_t check_bounds, int8_t *out_type_ids, int32_t *out_offsets, int32_t *out_child_rows,
                          int64_t *out_field_starts);

/* ------------------------------------------------------------------------- */
/* like — arrow-string/src/like.rs                                           */
/* ------------------------------------------------------------------------- */
/* arrow-string/src/like.rs `enum Op` */
typedef enum acu_like_op {
  ACU_LIKE = 0, ACU_NLIKE = 1, ACU_ILIKE = 2, ACU_NILIKE = 3,
  ACU_CONTAINS = 4, ACU_STARTS_WITH = 5, ACU_ENDS_WITH = 6, ACU_EQ_IGNORE_ASCII_CASE = 7
} acu_like_op;
/* like / nlike / ilike / nilike / contains / starts_with / ends_with / eq_ignore_ascii_case (like.rs:83-216, like_op
 * :218-296). l = the haystack, r = the pattern / needle; either may be a scalar (nulls.is_scalar), with the column layouts
 * of acu_cmp_bytes / acu_cmp_byte_view. is_utf8 = 1 for Utf8 / LargeUtf8 / Utf8View, 0 for Binary / LargeBinary /
 * BinaryView, which accept only contains / starts_with / ends_with (binary_like.rs:34-47).
 * Result (a boolean array, as acu_cmp):
 *   - r a null scalar: every row null (BooleanArray::new_null);
 *   - r a non-null scalar (op_scalar): the predicate runs at every slot of l, null slots included, and the result carries
 *     l's NullBuffer as it is (present iff l->nulls.validity != NULL);
 *   - otherwise (op_binary, l an array or a scalar): a row with a null side is null with value bit 0, and the result has a
 *     NullBuffer iff some row is null.
 * LIKE patterns: `\x` is a literal x (a trailing `\` a literal backslash), `%` any run of characters, `_` one character
 * (one UTF-8 scalar), anchored at both ends; ilike folds like the reference's regex (simple case folding: an ASCII letter
 * matches both cases, k / K also U+212A and s / S also U+017F). Errors: lengths differ => ACU_ERR_INVALID_ARGUMENT "Cannot
 * compare arrays of different lengths, got {l} vs {r}"; a binary column with another op => ACU_ERR_INVALID_ARGUMENT
 * "Invalid binary operation: {OP}" (LIKE, NILIKE, EQ_IGNORE_ASCII_CASE, ...).
 * Not reproduced:
 *   - an ilike / nilike pattern with a non-ASCII character fails with ACU_ERR_NOT_YET_IMPLEMENTED wherever the reference
 *     would compile it: a non-null scalar pattern (detail.index = -1), or a per-row pattern in a row whose two sides are
 *     non-null (detail.index = the lowest such row);
 *   - the reference fails to compile the regex of a huge pattern (its regex size limit); the device matches it.
 * Synchronous (not available inside a stream-ordered section); kernel time is counted in ACU_K_CMP. */
acu_status acu_like_bytes(acu_ctx *ctx, int32_t offset_bytes, int32_t is_utf8, acu_like_op op, const acu_bytes_array *l,
                          const acu_bytes_array *r, acu_array_out *out);
acu_status acu_like_byte_view(acu_ctx *ctx, int32_t is_utf8, acu_like_op op, const acu_view_array *l,
                              const acu_view_array *r, acu_array_out *out);

/* ------------------------------------------------------------------------- */
/* length / substring — arrow-string/src/length.rs, substring.rs             */
/* ------------------------------------------------------------------------- */
typedef enum acu_length_op { ACU_LENGTH = 0, ACU_BIT_LENGTH = 1 } acu_length_op;
/* length / bit_length (length.rs:26-200). The value is computed at EVERY slot, null slots included, and the result carries
 * the input's NullBuffer as it is (nulls.cloned(): present iff nulls.validity != NULL, even without nulls), normalised to
 * bit offset 0.
 *   - acu_length_bytes: Utf8 / Binary (offset_bytes 4) give Int32, LargeUtf8 / LargeBinary (8) give Int64:
 *     offsets[i+1] - offsets[i], wrapping; bit_length multiplies by 8, wrapping. out->values: len x offset_bytes bytes.
 *   - acu_length_byte_view: Int32, the low 32 bits of each view (`*view as i32`; also for null views, whose bytes may be
 *     anything); bit_length wrapping_mul(8). out->values: len x 4 bytes.
 *   - acu_length_fixed_size_binary: Int32, byte_width (bit_length byte_width * 8, wrapping) at every slot; byte_width < 0
 *     => ACU_ERR_INVALID_ARGUMENT.
 * A scalar input or an op outside acu_length_op => ACU_ERR_INVALID_ARGUMENT. */
acu_status acu_length_bytes(acu_ctx *ctx, int32_t offset_bytes, acu_length_op op, const acu_bytes_array *a, acu_array_out *out);
acu_status acu_length_byte_view(acu_ctx *ctx, acu_length_op op, const acu_view_array *a, acu_array_out *out);
acu_status acu_length_fixed_size_binary(acu_ctx *ctx, int32_t byte_width, acu_length_op op, const acu_array *a, acu_array_out *out);

/* filter / take of a FixedSizeBinary(byte_width) column (filter_fixed_size_binary filter.rs:946-996, take_fixed_size_binary
 * take.rs:802-862). `values->values` points at logical row 0 (values->len rows of byte_width bytes, any alignment);
 * out->values has capacity (output rows) x byte_width bytes, any alignment; out->validity acu_bitmap_bytes(output rows) + 8.
 * byte_width < 0 => ACU_ERR_INVALID_ARGUMENT.
 *   - filter: the selected rows' bytes in row order, bytes under null slots included; the NullBuffer as for
 *     acu_filter_primitive (FilterPredicate::filter_nulls; IterationStrategy::All keeps the input's).
 *   - take: check_bounds and "Take only supported for integers" as for acu_take_primitive. Widths 1, 2, 4, 8 and 16 follow
 *     take_fixed_size (take_native byte for byte): an in-bounds null index still gathers its row, an out-of-bounds null
 *     index gives zeros, a valid out-of-bounds index is ACU_ERR_PANIC_OUT_OF_BOUNDS "Out-of-bounds index {index}". Every
 *     other width (0 and 32 included) follows the dynamic-length path: a null index gives byte_width zero bytes and is never
 *     read; a valid index reads values[index * byte_width .. + byte_width] in wrapping 64-bit arithmetic, so an index whose
 *     product wraps into the buffer reads those bytes; a slice past the buffer or out of order is ACU_ERR_PANIC_OUT_OF_BOUNDS
 *     at the lowest such row, checked in this order: "range start index {s} out of range for slice of length
 *     {len * byte_width}", "range end index {e} out of range for slice of length {len * byte_width}", "slice index starts
 *     at {s} but ends at {e}" (lhs_bits = s, rhs_bits = e). Then, when the values have a null, a valid index past them
 *     is the validity gather's ACU_ERR_PANIC_OUT_OF_BOUNDS "assertion failed: idx < self.bit_len".
 *     NullBuffer::union(take_nulls(values), indices.nulls()): has_validity = 1 only when the result has a null (unlike
 *     acu_take_primitive, indices whose NullBuffer has no null give none).
 *   - byte_width 0 (FixedSizeBinaryArray::try_new takes the length from the NullBuffer): a take, or a filter that is not
 *     IterationStrategy::All, whose result has no NullBuffer has out->len = 0.
 * Synchronous (refused inside a stream-ordered section); kernel time in ACU_K_FILTER / ACU_K_TAKE. */
acu_status acu_filter_fixed_size_binary(acu_ctx *ctx, const acu_filter_plan *plan, int32_t byte_width, const acu_array *values,
                                        acu_array_out *out);
acu_status acu_take_fixed_size_binary(acu_ctx *ctx, int32_t byte_width, const acu_array *values, const acu_array *indices,
                                      acu_dtype index_dtype, int32_t check_bounds, acu_array_out *out);

/* substring(array, start, length) (substring.rs:73-459): has_length = 0 is `None`, else `Some(length)`.
 *
 * acu_substring_bytes — byte_substring (:319-397) for Utf8 / LargeUtf8 (is_utf8 = 1) and Binary / LargeBinary (0).
 *   `data_len` is the length of the whole value-data buffer `a->data` points at (value_data().len(), also for a slice).
 *   - i32 offsets take `start as i32` and `length as i32` and add in i32, wrapping as in a release build; i64 offsets take
 *     `length as i64`. Row i: new_start = min(offsets[i] + start, offsets[i+1]) for start > 0, offsets[i] for start == 0,
 *     max(offsets[i+1] + start, offsets[i]) for start < 0; new_end = min(length + new_start, offsets[i+1]), or offsets[i+1].
 *   - the rule runs at every slot, null slots included (a null slot keeps the substring of the bytes under it).
 *   - Utf8 checks each new offset with is_char_boundary against the whole value-data buffer (offsets are absolute; the end
 *     of the buffer is a boundary; a negative offset reads as its huge usize): new_start when start != 0, new_end when a
 *     length is given, rows in order, start before end. The first failure is ACU_ERR_COMPUTE "The offset {offset} is at an
 *     invalid utf-8 boundary." (detail.index = the row, lhs_bits = the offset).
 *   - otherwise, where wrapping leaves a row whose slice data[new_start..new_end] is out of order or out of the buffer, the
 *     reference panics: ACU_ERR_PANIC_OUT_OF_BOUNDS at the lowest such row, "slice index starts at {s} but ends at {e}" or
 *     "range end index {e} out of range for slice of length {data_len}" (lhs_bits = s, rhs_bits = e as usize).
 *   - out_offsets: len + 1 entries starting at 0 (also for a sliced input). Two-phase like acu_filter_bytes: out_data == NULL
 *     writes only the offsets and *out_data_len; otherwise the bytes go to out_data (capacity out_data_capacity; too small
 *     => ACU_ERR_INVALID_ARGUMENT, no byte written).
 *   - out_nulls (validity capacity acu_bitmap_bytes(len)): NullBuffer::from_unsliced_buffer, so has_validity = 0 when the
 *     input has no null (unlike length).
 * acu_substring_by_char — substring_by_char (:144-251) for Utf8 / LargeUtf8: start and length count chars (utf8_bounds:
 *   nth / nth_back for the start, nth for the end); null slots become empty; never fails. Output as acu_substring_bytes.
 *   Both two-phase calls compute every row's range and run the offsets pass, the sizing call as well as the copy call.
 * acu_substring_byte_view — string_view_substring / binary_view_substring (:254-317): null slots become all-zero views (as
 *   append_null writes them); offsets are relative to the value (view_substring_range, length as i64); Utf8View
 *   (is_utf8 = 1) checks both ends of every non-null row, and its error message gives the RELATIVE offset. A row whose slice
 *   panics (length >= 2^63) => ACU_ERR_PANIC_OUT_OF_BOUNDS as above, relative to the value. out_views: 16 bytes per row,
 *   16-byte aligned; out_nulls as the builder's: has_validity = 0 when the result has no null.
 *   Buffer layout (differs on purpose from the reference's StringViewBuilder; the logical values are equal): a result of at
 *   most 12 bytes is an inline view, zero padded; a longer one points into the INPUT's data buffers (same buffer_index,
 *   offset advanced by new_start, the new 4-byte prefix), so the result shares a->buffers and no byte is copied.
 * acu_substring_fixed_size_binary — fixed_size_binary_substring (:399-459): one output width *out_byte_width = new_len for
 *   the whole column; row i = data[i*byte_width + new_start ..][..new_len], null rows too (out->values: len x new_len
 *   bytes). Nulls as from_unsliced_buffer, except that new_len == 0 without nulls gives an all-valid NullBuffer.
 * A scalar input, a negative byte_width or data_len, or an offset width other than 4 / 8 => ACU_ERR_INVALID_ARGUMENT.
 * Synchronous (not available inside a stream-ordered section); kernel time is counted in ACU_K_BYTES. */
acu_status acu_substring_bytes(acu_ctx *ctx, int32_t offset_bytes, int32_t is_utf8, int64_t start, int32_t has_length, uint64_t length,
                               const acu_bytes_array *a, int64_t data_len, void *out_offsets, uint8_t *out_data,
                               int64_t out_data_capacity, int64_t *out_data_len, acu_array_out *out_nulls);
acu_status acu_substring_by_char(acu_ctx *ctx, int32_t offset_bytes, int64_t start, int32_t has_length, uint64_t length,
                                 const acu_bytes_array *a, void *out_offsets, uint8_t *out_data, int64_t out_data_capacity,
                                 int64_t *out_data_len, acu_array_out *out_nulls);
acu_status acu_substring_byte_view(acu_ctx *ctx, int32_t is_utf8, int64_t start, int32_t has_length, uint64_t length,
                                   const acu_view_array *a, void *out_views, acu_array_out *out_nulls);
acu_status acu_substring_fixed_size_binary(acu_ctx *ctx, int32_t byte_width, int64_t start, int32_t has_length, uint64_t length,
                                           const acu_array *a, int32_t *out_byte_width, acu_array_out *out);

/* ------------------------------------------------------------------------- */
/* concat_elements — arrow-string/src/concat_elements.rs                     */
/* ------------------------------------------------------------------------- */
/* The element-wise concatenation of equally long arrays (concat_elements.rs:31-407). Row i of the result is the operands'
 * values at row i, one after another. Nulls are NullBuffer::union of the operands': out_nulls / out carries a validity
 * (normalised to bit offset 0, capacity acu_bitmap_bytes(len)) only when some row is null, also when an operand has a
 * NullBuffer without nulls. Lengths that differ => ACU_ERR_COMPUTE "Arrays must have the same length: {l} != {r}".
 *
 * acu_concat_elements_bytes — concat_elements_bytes / _utf8 / concat_element_binary (:31-104) for Utf8 / Binary
 *   (offset_bytes 4) and LargeUtf8 / LargeBinary (8); no byte is validated, so one entry point serves both. Every row is
 *   concatenated, null rows included (the bytes under a null slot are copied). out_offsets: len + 1 entries starting at 0
 *   (also for sliced operands, which may be sliced differently). With i32 offsets, the first row whose end passes i32::MAX
 *   is the reference's `from_usize(..).unwrap()` panic: ACU_ERR_PANIC_OUT_OF_BOUNDS "called `Option::unwrap()` on a `None`
 *   value", detail.index = that row. Two-phase like acu_substring_bytes: out_data == NULL writes the offsets and
 *   *out_data_len only; both calls run the offsets pass and the overflow check. A copy call whose out_data_capacity is
 *   below the total => ACU_ERR_INVALID_ARGUMENT, no byte written.
 * acu_concat_elements_bytes_many — concat_elements_utf8_many (:113-173) over n_arrays >= 1 operands, `arrays` a HOST array
 *   of descriptors; output as above. n_arrays < 1 => ACU_ERR_COMPUTE "concat requires input of at least one array"; an
 *   operand whose length differs from arrays[0]'s => ACU_ERR_COMPUTE "Arrays must have the same length of {len}".
 * acu_concat_elements_byte_view — concat_elements_string_view_array / binary_view_array (:230-407), with the reference's
 *   layout bit for bit: a null row is an all-zero view and its operands' views are never read; a result of at most 12 bytes
 *   is an inline view, zero padded; a longer one is appended, in row order, to ONE new data buffer (out_data) and its view
 *   is (length, first 4 bytes, buffer 0, offset). The result has that one data buffer when *out_data_len > 0 and none
 *   otherwise. Two-phase: out_views == NULL is the sizing call (*out_data_len = the bytes of the non-null results longer
 *   than 12 bytes); the copy call writes out_views (16 bytes per row, 16-byte aligned) and out_data. A data buffer longer
 *   than i32::MAX => ACU_ERR_ARITHMETIC_OVERFLOW "byte array offset overflow" before any row is written; a copy call whose
 *   out_data_capacity is below *out_data_len => ACU_ERR_INVALID_ARGUMENT, nothing written.
 * acu_concat_elements_fixed_size_binary — concat_elements_fixed_size_binary (:181-228): *out_byte_width = l_width + r_width,
 *   row i = left row i then right row i; a null row is zero bytes (append_null). After the length check, a negative width
 *   => ACU_ERR_INVALID_ARGUMENT "Invalid size of FixedSizeBinaryArray({w})", left before right; a sum past i32::MAX is the
 *   reference's builder panic, also with zero rows: ACU_ERR_PANIC_OUT_OF_BOUNDS "value length ({sum as i32}) of the array
 *   must >= 0". out->values: len x (l_width + r_width) bytes.
 * Type dispatch (concat_elements_dyn, :419-476) belongs to the typed host layers. A scalar operand or an offset width other
 * than 4 / 8 => ACU_ERR_INVALID_ARGUMENT. Synchronous (not available inside a stream-ordered section); kernel time is
 * counted in ACU_K_BYTES. */
acu_status acu_concat_elements_bytes(acu_ctx *ctx, int32_t offset_bytes, const acu_bytes_array *l, const acu_bytes_array *r,
                                     void *out_offsets, uint8_t *out_data, int64_t out_data_capacity, int64_t *out_data_len,
                                     acu_array_out *out_nulls);
acu_status acu_concat_elements_bytes_many(acu_ctx *ctx, int32_t offset_bytes, int32_t n_arrays, const acu_bytes_array *arrays,
                                          void *out_offsets, uint8_t *out_data, int64_t out_data_capacity, int64_t *out_data_len,
                                          acu_array_out *out_nulls);
acu_status acu_concat_elements_byte_view(acu_ctx *ctx, const acu_view_array *l, const acu_view_array *r, void *out_views,
                                         uint8_t *out_data, int64_t out_data_capacity, int64_t *out_data_len, acu_array_out *out_nulls);
acu_status acu_concat_elements_fixed_size_binary(acu_ctx *ctx, int32_t l_width, const acu_array *l, int32_t r_width,
                                                 const acu_array *r, int32_t *out_byte_width, acu_array_out *out);

/* Utf8View / BinaryView buffer management for BatchCoalescer (InProgressByteViewArray, arrow-select/src/coalesce/
 * byte_view.rs). The reference decides per source array whether its data buffers are compacted ("gc": when they hold more
 * than twice the bytes its views use, :366-381) and how output buffers are sized (BufferSource, :526-559); that policy stays
 * on the host (host/arrow_cuda.hpp, acu/coalesce.py). The per-view work runs on the device:
 *   acu_view_bytes_used   = GenericByteViewArray::total_buffer_bytes_used (arrow-array/src/array/byte_view_array.rs:749-761):
 *                           sum of the lengths of the views longer than 12 bytes (null slots included, as in the reference).
 *   acu_view_fit          = the "copy as many views as fit the current buffer" loop (:259-271): *out_views = leading views
 *                           that fit `remaining_capacity` (EVERY view's length is compared with what is left, only the long
 *                           ones consume it — the reference's loop), *out_bytes = bytes of the long views among them.
 *   acu_view_copy_strings = append_views_and_copy_strings_inner (:298-354): out_views[i] = views[i], every view longer than
 *                           12 bytes rewritten to {buffer_index = new_buffer_index, offset = position in dst} with its bytes
 *                           copied to dst[dst_len ...] in view order (null slots too); *out_bytes = bytes appended. `buffers` =
 *                           HOST array of n_buffers DEVICE pointers (the source's data buffers).
 *   acu_view_rebase       = append_views_and_update_buffer_index (:176-216): buffer_index += delta for the long views.
 * views / out_views: 16 bytes per row, 16-byte aligned; out_views may alias views. */
acu_status acu_view_bytes_used(acu_ctx *ctx, const void *views, int64_t n, int64_t *out_total);
acu_status acu_view_fit(acu_ctx *ctx, const void *views, int64_t n, int64_t remaining_capacity, int64_t *out_views,
                        int64_t *out_bytes);
acu_status acu_view_copy_strings(acu_ctx *ctx, const void *views, int64_t n, const uint8_t *const *buffers,
                                 int32_t n_buffers, uint32_t new_buffer_index, uint8_t *dst, int64_t dst_len,
                                 int64_t dst_capacity, void *out_views, int64_t *out_bytes);
acu_status acu_view_rebase(acu_ctx *ctx, const void *views, int64_t n, uint32_t delta, void *out_views);

/* ------------------------------------------------------------------------- */
/* cast — arrow-cast/src/cast/mod.rs                                         */
/* ------------------------------------------------------------------------- */
/* cast_numeric_arrays (mod.rs:2550-2614). safe != 0 => numeric_cast (unrepresentable
 * value -> null, output always has a validity buffer: primitive_array.rs:1065-1103);
 * safe == 0 => try_numeric_cast (ACU_ERR_CAST "Can't cast value {v} to type {T}"). */
acu_status acu_cast_numeric(acu_ctx *ctx, acu_dtype from, acu_dtype to, int32_t safe,
                            const acu_array *a, acu_array_out *out);

/* Decimal casts (arrow-cast/src/cast/decimal.rs, the decimal arms of cast_with_options in mod.rs), under
 * CastOptions{safe: safe != 0}. Decimal32 / 64 / 128 values are ACU_I32 / ACU_I64 / ACU_I128 natives (acu_decimal_type);
 * out->values holds the output native per row. Synchronous, like acu_cast_numeric (not stream-ordered inside a section);
 * kernel time counts in ACU_K_CAST. Decimal128 pointers, input and output, must be 16-byte aligned, and the input decimal
 * type must pass validate_decimal_precision_and_scale (ACU_ERR_INVALID_ARGUMENT otherwise, at call time).
 *
 * Which array the reference builds decides values under nulls and the NullBuffer:
 *   - unary (the infallible casts): the value is computed at EVERY slot, null slots included; the input's nulls are kept.
 *   - unary_opt (safe, fallible): valid slots only, 0 under nulls and where the cast fails (-> null); the result ALWAYS has
 *     a NullBuffer.
 *   - try_unary (unsafe, fallible): valid slots only, 0 under nulls, the input's nulls kept; the lowest failing valid row
 *     is the error (detail.index, detail.lhs_bits = the low 64 bits of its raw input).
 *   - decimal -> integer (PrimitiveBuilder): 0 under nulls, a NullBuffer only when some row is null.
 *
 * acu_cast_decimal, decimal -> decimal (cast_decimal_to_decimal(_same_type), decimal.rs:161-529):
 *   - delta = s_out - s_in (upscale, s_in <= s_out) or s_in - s_out (downscale), in i8 arithmetic that wraps like a release
 *     build; a negative delta misses MAX_FOR_EACH_PRECISION. Upscale: x converted to the output native, times 10^delta.
 *     Downscale: x / 10^delta in the INPUT native, rounded half away from zero, then converted.
 *   - infallible (unary) when p_in + delta <= p_out (upscale) or p_in - delta < p_out (downscale), computed in i8: the
 *     infallible upscale multiplies wrapping; a slot whose value does not convert to the output native (a valid value that
 *     breaks its own precision, or bytes under a null) is the reference's `unwrap()` panic: ACU_ERR_PANIC_OUT_OF_BOUNDS
 *     "called `Option::unwrap()` on a `None` value" at the lowest such slot. Same scale, same width and p_in <= p_out is
 *     the reference's array.clone(), decided in u8 ahead of the i8 test (so p_out above 127 still clones and only the
 *     closing type check fails): the same bytes, nulls and null slots included.
 *   - otherwise fallible: a failed rescale or a value outside p_out is null (safe), or ACU_ERR_CAST "Cannot cast to
 *     Decimal64(18, 18). Overflowing on {x}" (the input value) / the precision error below (unsafe).
 *   - an upscale delta past the output's table: ACU_ERR_CAST "Cannot cast to Decimal128(p, s). Value overflows for output
 *     scale", safe or not, also for an empty array. A downscale delta past the input's table: every value 0, the input's
 *     nulls kept.
 * acu_cast_to_decimal, from ACU_I8 .. ACU_U64, ACU_F32, ACU_F64:
 *   - integers (cast_integer_to_decimal, mod.rs:366-444): scale < 0 divides by 10^-scale in the SOURCE type first (a
 *     factor that overflows the source type gives all zeros, the input's nulls kept); scale >= 0 multiplies by 10^scale,
 *     computed checked in the output native before any row (ACU_ERR_CAST "Cannot cast to \"Decimal32\"(9, 10). The scale
 *     causes overflow."). A failing row (unsafe): the value does not fit the output native (or any failure at a negative
 *     scale) => ACU_ERR_CAST "Cannot cast to Decimal32(9, 0). Overflowing on {v}" with the input; the checked multiply
 *     fails => ACU_ERR_ARITHMETIC_OVERFLOW "Overflow happened on: {v} * {10^scale}" with the narrowed value.
 *   - floats (cast_floating_point_to_decimal, decimal.rs:836-885): (mul * v).round() with mul = 10_f64.powi(scale), one
 *     IEEE multiply (no FMA), rounded half away from zero, then to_i32 / to_i64 / to_i128 (NaN, +-inf or out of range =>
 *     None). powi is repeated squaring with 1 / r for a negative exponent (the `pow` of Rust's compiler-builtins, which a
 *     runtime-exponent llvm.powi calls), not the correctly rounded 10^scale. A failing row (unsafe): ACU_ERR_CAST
 *     "Cannot cast to Decimal128(38, 10). Overflowing on {v:?}" with Rust's Debug of the f32 / f64 (shortest round-trip
 *     digits; 1e-4 <= |v| < 1e16 or 0 in plain notation with a fractional digit, else "1e40"; NaN, inf, -inf).
 * acu_cast_from_decimal, to ACU_I8 .. ACU_U64, ACU_F32, ACU_F64:
 *   - integers (cast_decimal_to_integer, decimal.rs:887-987): 10^|scale| computed checked in the decimal native before any
 *     row (ACU_ERR_CAST "Cannot cast to \"Decimal32\". The scale 10 causes overflow."); scale >= 0 divides truncating,
 *     scale < 0 multiplies checked (unsafe: ACU_ERR_ARITHMETIC_OVERFLOW "Overflow happened on: {v} * {10^k}"); then
 *     NumCast to the integer type (unsafe: ACU_ERR_CAST "value of {v} is out of range Int8", v scaled).
 *   - floats (cast_decimal_to_float, mod.rs:86-92): unary (x as f64) / 10_f64.powi(scale); i128 -> f64 rounds to nearest,
 *     ties to even; Float32 is that f64 `as f32` (two roundings, as the reference). Never fails.
 * In every cast to a decimal, an unsafe row outside the output precision is validate_decimal{32,64,}_precision's
 * ACU_ERR_INVALID_ARGUMENT "1234567.89 is too large to store in a Decimal128 of precision 6. Max is 9999.99" (or "too small
 * ... Min is", or "Max precision of a Decimal128 is 38, but got 40"), the value formatted by format_decimal_str_internal
 * with its truncation rule. Type-level errors come before any row, row errors before the closing with_precision_and_scale
 * check of the output type (ACU_ERR_INVALID_ARGUMENT, as acu_decimal_arith's). Not reproduced: Decimal256, Float16,
 * strings, temporal types, Null and dictionary inputs. */
acu_status acu_cast_decimal(acu_ctx *ctx, const acu_decimal_type *from, const acu_decimal_type *to, int32_t safe,
                            const acu_array *a, acu_array_out *out);
acu_status acu_cast_to_decimal(acu_ctx *ctx, acu_dtype from, const acu_decimal_type *to, int32_t safe,
                               const acu_array *a, acu_array_out *out);
acu_status acu_cast_from_decimal(acu_ctx *ctx, const acu_decimal_type *from, acu_dtype to, int32_t safe,
                                 const acu_array *a, acu_array_out *out);

/* ------------------------------------------------------------------------- */
/* boolean — arrow-arith/src/boolean.rs (predicate construction before filter) */
/* ------------------------------------------------------------------------- */
typedef enum acu_bool_op {
  ACU_BOOL_AND = 0,         /* and        boolean.rs:256  values a&b at every slot, nulls = union */
  ACU_BOOL_OR = 1,          /* or         boolean.rs:273 */
  ACU_BOOL_AND_NOT = 2,     /* and_not    boolean.rs:291  a & !b */
  ACU_BOOL_AND_KLEENE = 3,  /* and_kleene boolean.rs:60   false AND null = false */
  ACU_BOOL_OR_KLEENE = 4,   /* or_kleene  boolean.rs:156  true OR null = true */
  ACU_BOOL_NOT = 5,         /* not        boolean.rs:310  (b == NULL) */
  ACU_BOOL_IS_NULL = 6,     /* is_null    boolean.rs:327  any array kind: only a's validity/len are read; b == NULL */
  ACU_BOOL_IS_NOT_NULL = 7  /* is_not_null boolean.rs:347 */
} acu_bool_op;
/* a, b: BooleanArrays (values = bitmaps with bit offsets). out->values receives the result
 * bitmap (bit offset 0, whole u64 words, bits >= len zero). The result carries a validity
 * buffer exactly when the reference's does: and/or/and_not/kleene when either input has
 * one (even without nulls), not when `a` has one, is_null/is_not_null never. Length
 * mismatch => ACU_ERR_COMPUTE "Cannot perform bitwise operation on arrays of different
 * length". */
acu_status acu_boolean(acu_ctx *ctx, acu_bool_op op, const acu_array *a, const acu_array *b,
                       acu_array_out *out);

/* ------------------------------------------------------------------------- */
/* aggregate — arrow-arith/src/aggregate.rs                                  */
/* ------------------------------------------------------------------------- */
/* sum/min/max (aggregate.rs:943,1012,1027): *out_bits = the native result's bit
 * pattern (zero-extended), *out_valid_count = number of non-null rows; the reference
 * returns None iff out_valid_count == 0 (aggregate.rs:320-323).
 * product (aggregate.rs:953) wraps for integers (mul_wrapping) and is IEEE for floats (association order unspecified, as
 * for sum); bit_and / bit_or / bit_xor (aggregate.rs:788-875) take the integer dtypes only (a float =>
 * ACU_ERR_INVALID_ARGUMENT). An op outside acu_agg_op => ACU_ERR_INVALID_ARGUMENT. */
acu_status acu_aggregate(acu_ctx *ctx, acu_dtype dtype, acu_agg_op op, const acu_array *a,
                         uint64_t *out_bits, int64_t *out_valid_count);
/* sum / min / max of a Decimal128 (ACU_I128) column: out_bits[0] = low, out_bits[1] = high 64 bits of the i128 result;
 * sum wraps (add_wrapping in i128), min / max use the signed i128 order; None iff *out_valid_count == 0. Decimal32 /
 * Decimal64 columns use acu_aggregate with ACU_I32 / ACU_I64. Stream-ordered inside a section like acu_aggregate. */
acu_status acu_aggregate_i128(acu_ctx *ctx, acu_agg_op op, const acu_array *a, uint64_t out_bits[2],
                              int64_t *out_valid_count);

/* sum_checked (aggregate.rs:897-937): the in-order checked fold. Integers:
 * ACU_ERR_ARITHMETIC_OVERFLOW "Overflow happened on: {acc} + {value}" at the first valid
 * row whose running sum leaves the native range (index = that row) — also when the final
 * total would fit. Floats never fail (add_checked is the plain add): same as ACU_SUM. */
acu_status acu_sum_checked(acu_ctx *ctx, acu_dtype dtype, const acu_array *a, uint64_t *out_bits,
                           int64_t *out_valid_count);
/* product_checked (aggregate.rs:963-1001): the in-order fold acc.mul_checked(v) from 1. Integers:
 * ACU_ERR_ARITHMETIC_OVERFLOW "Overflow happened on: {acc} * {value}" at the first valid row whose running product
 * leaves the native range (index = that row, lhs_bits / rhs_bits = acc / value) — also when a later zero would bring the
 * product back to 0. Floats never fail (mul_checked is the plain multiply): same as ACU_PRODUCT. Contract otherwise as
 * acu_sum_checked. Synchronous: inside a stream-ordered section every call, float and empty inputs included, fails with
 * ACU_ERR_INVALID_ARGUMENT before any device work. Kernel time in ACU_K_REDUCE. */
acu_status acu_product_checked(acu_ctx *ctx, acu_dtype dtype, const acu_array *a, uint64_t *out_bits,
                               int64_t *out_valid_count);

/* min / max of Utf8 / Binary (offset_bytes 4), LargeUtf8 / LargeBinary (8), Utf8View / BinaryView and FixedSizeBinary
 * columns: min_max_helper / min_max_view_helper (aggregate.rs:460-518) behind min_string, max_binary_view,
 * min_fixed_size_binary ... (:520-568). Values order like Rust's `&[u8]` (lexicographic on unsigned bytes, a proper prefix
 * first). op = ACU_MIN | ACU_MAX (ACU_SUM => ACU_ERR_INVALID_ARGUMENT). *out_row = the LOWEST logical row holding the
 * extremal value (the reference folds in row order and replaces only on a strict < / >), -1 = None (every row null, or
 * len == 0); *out_valid_count = non-null rows. Null slots are never read. The column layouts are those of acu_cmp_bytes /
 * acu_cmp_byte_view; a FixedSizeBinary column is an acu_array whose `values` holds len x byte_width bytes (byte_width >= 0,
 * negative => ACU_ERR_INVALID_ARGUMENT). is_scalar inputs => ACU_ERR_INVALID_ARGUMENT. Synchronous (not available inside a
 * stream-ordered section); kernel time is counted in ACU_K_REDUCE. */
acu_status acu_aggregate_bytes(acu_ctx *ctx, int32_t offset_bytes, acu_agg_op op, const acu_bytes_array *a,
                               int64_t *out_row, int64_t *out_valid_count);
acu_status acu_aggregate_byte_view(acu_ctx *ctx, acu_agg_op op, const acu_view_array *a, int64_t *out_row,
                                   int64_t *out_valid_count);
acu_status acu_aggregate_fixed_size_binary(acu_ctx *ctx, int32_t byte_width, acu_agg_op op, const acu_array *a,
                                           int64_t *out_row, int64_t *out_valid_count);
/* min_boolean / bool_and (ACU_MIN), max_boolean / bool_or (ACU_MAX) (aggregate.rs:372-457, :880-889): *out_value 0 | 1,
 * -1 = None; *out_valid_count = non-null rows. `values` is the value bitmap with bit offset values_offset. Synchronous, as
 * above. */
acu_status acu_aggregate_boolean(acu_ctx *ctx, acu_agg_op op, const acu_array *a, int32_t *out_value,
                                 int64_t *out_valid_count);

/* ------------------------------------------------------------------------- */
/* RecordBatch level — filter_record_batch / take_record_batch / per-column   */
/* aggregates with ONE stream synchronisation per call                        */
/* ------------------------------------------------------------------------- */
/* A column of a RecordBatch (arrow-array/src/record_batch.rs:224). PRIMITIVE: `array`
 * as for acu_filter_primitive with element width `width`; BOOLEAN: `array.values` is a
 * bitmap; BYTES (Utf8/Binary/LargeUtf8/LargeBinary): `array.values` = the offsets
 * buffer (i32 if width == 4, i64 if width == 8, array.len + 1 entries), `data` = the
 * value bytes, `array.validity/len/null_count` the nulls. */
/* FIXED_SIZE_BINARY (filter / take record-batch calls only): `array` as for acu_filter_fixed_size_binary with byte width
 * `width`; acu_concat, acu_concat_batches and export refuse it with ACU_ERR_INVALID_ARGUMENT. */
typedef enum acu_column_kind { ACU_COL_PRIMITIVE = 0, ACU_COL_BOOLEAN = 1, ACU_COL_BYTES = 2, ACU_COL_FIXED_SIZE_BINARY = 3 } acu_column_kind;

typedef struct acu_column {
  int32_t kind;          /* acu_column_kind */
  int32_t width;         /* PRIMITIVE: element bytes (1,2,4,8,16,32); BYTES: offset bytes (4|8) */
  acu_array array;
  const uint8_t *data;   /* BYTES only */
} acu_column;

/* Caller-owned output of one column. `array.values` receives the values (PRIMITIVE /
 * BOOLEAN) or the new offsets (BYTES, rows + 1 entries); `data` (capacity
 * `data_capacity`) the value bytes; `data_len` is set to the bytes required/written.
 * BYTES offsets, in and out, must be aligned to `width`, as for acu_take_bytes. */
typedef struct acu_column_out {
  acu_array_out array;
  uint8_t *data;
  int64_t data_capacity;
  int64_t data_len;
} acu_column_out;

/* filter_record_batch (filter.rs:225-244) / FilterPredicate::filter_record_batch
 * (filter.rs:459-478): every column filtered with the same plan (the predicate is
 * scanned once), all kernels queued back to back, one synchronisation. Columns keep
 * their order; on error the status/detail of the first failing column is returned (the
 * reference propagates that column's ArrowError). At most ACU_MAX_BATCH_COLUMNS columns. */
#define ACU_MAX_BATCH_COLUMNS 64
acu_status acu_filter_record_batch(acu_ctx *ctx, const acu_filter_plan *plan, int32_t n_columns,
                                   const acu_column *columns, acu_column_out *outs);

/* take_record_batch (take.rs:1123-1133) / take_arrays (take.rs:155-164): every column
 * gathered with the same indices; check_bounds as in acu_take_primitive. Null counts of
 * the columns and of the indices should be cached (>= 0); unknown ones are counted
 * first (one extra synchronisation each). */
acu_status acu_take_record_batch(acu_ctx *ctx, int32_t n_columns, const acu_column *columns,
                                 const acu_array *indices, acu_dtype index_dtype, int32_t check_bounds,
                                 acu_column_out *outs);

/* sum/min/max of n columns (acu_aggregate semantics per column) with one
 * synchronisation: dtypes[i]/ops[i] describe arrays[i]. */
acu_status acu_aggregate_columns(acu_ctx *ctx, int32_t n_columns, const acu_dtype *dtypes,
                                 const acu_agg_op *ops, const acu_array *arrays, uint64_t *out_bits,
                                 int64_t *out_valid_counts);

/* ------------------------------------------------------------------------- */
/* appending row ranges — the pieces of BatchCoalescer / concat               */
/* (arrow-select/src/coalesce.rs:258-533 InProgressArray::copy_rows)          */
/* ------------------------------------------------------------------------- */
/* Values of a fixed-width column append with acu_memcpy_d2d. Bits (validity, boolean
 * values): dst bits [dst_offset, dst_offset+len) = src bits [src_offset, ..+len), every
 * other bit of dst preserved (dst 8-byte aligned, capacity a whole number of u64 words).
 * *out_set_bits (optional; forces a synchronisation) = number of set bits copied. */
acu_status acu_bitmap_copy(acu_ctx *ctx, const uint8_t *src, int64_t src_offset, uint8_t *dst,
                           int64_t dst_offset, int64_t len, int64_t *out_set_bits);
/* dst bits [dst_offset, dst_offset+len) = value (0 | 1), other bits preserved. */
acu_status acu_bitmap_fill(acu_ctx *ctx, uint8_t *dst, int64_t dst_offset, int64_t len, int32_t value);
/* Utf8/Binary offsets of `count` rows starting at source row `first`, rebased so that the
 * first one equals `base` (the destination's byte total so far):
 * dst[dst_first + j] = base + src[first + j] - src[first], j = 0..count. Returns the source
 * byte range [*out_src_begin, *out_src_end) to append with acu_memcpy_d2d.
 * ACU_ERR_OFFSET_OVERFLOW when the running total leaves the offset type. */
acu_status acu_offsets_append(acu_ctx *ctx, int32_t offset_bytes, const void *src_offsets, int64_t first,
                              int64_t count, int64_t base, void *dst_offsets, int64_t dst_first,
                              int64_t *out_src_begin, int64_t *out_src_end);

/* concat (arrow-select/src/concat.rs:495-577): n columns of the same kind / width appended in order into the caller-owned
 * `out` (capacities: total rows * width; boolean / validity bitmaps acu_bitmap_bytes(total rows); BYTES: total rows + 1
 * offsets and out->data_capacity value bytes). Values and the bytes under null slots are copied as they are; the result
 * carries a validity buffer iff some input has nulls (NullBufferBuilder semantics) — a single input keeps its NullBuffer
 * presence (the reference returns array.slice(0, len)). Errors: no input => ACU_ERR_COMPUTE "concat requires input of at
 * least one array"; mixed kinds / widths => ACU_ERR_INVALID_ARGUMENT; i32 offsets overflowing => ACU_ERR_OFFSET_OVERFLOW
 * (generic_bytes_builder.rs:185-189). Inputs without a cached null_count cost one count each. */
acu_status acu_concat(acu_ctx *ctx, int32_t n_arrays, const acu_column *arrays, acu_column_out *out);
/* concat_batches (concat.rs:607-640): columns[b * n_columns + c] = column c of batch b; outs[c] = concat of field c over the
 * batches; *out_rows = rows of the result. No batch => every field is empty. */
acu_status acu_concat_batches(acu_ctx *ctx, int32_t n_batches, int32_t n_columns, const acu_column *columns,
                              acu_column_out *outs, int64_t *out_rows);

/* ------------------------------------------------------------------------- */
/* Arrow C Data Interface / C Device Data Interface                           */
/* ------------------------------------------------------------------------- */
/* The structs of the Arrow specification (the reference's FFI_ArrowArray / FFI_ArrowSchema,
 * arrow-data/src/ffi.rs:37-69, arrow-schema/src/ffi.rs). Guarded like the specification's
 * own header so that they can coexist with <arrow/c/abi.h>. */
#ifndef ARROW_C_DATA_INTERFACE
#define ARROW_C_DATA_INTERFACE
struct ArrowSchema {
  const char *format;
  const char *name;
  const char *metadata;
  int64_t flags;
  int64_t n_children;
  struct ArrowSchema **children;
  struct ArrowSchema *dictionary;
  void (*release)(struct ArrowSchema *);
  void *private_data;
};
struct ArrowArray {
  int64_t length;
  int64_t null_count;
  int64_t offset;
  int64_t n_buffers;
  int64_t n_children;
  const void **buffers;
  struct ArrowArray **children;
  struct ArrowArray *dictionary;
  void (*release)(struct ArrowArray *);
  void *private_data;
};
#endif
#ifndef ARROW_C_DEVICE_DATA_INTERFACE
#define ARROW_C_DEVICE_DATA_INTERFACE
typedef int32_t ArrowDeviceType;
#define ARROW_DEVICE_CPU 1
#define ARROW_DEVICE_CUDA 2
#define ARROW_DEVICE_CUDA_HOST 3
struct ArrowDeviceArray {
  struct ArrowArray array;
  int64_t device_id;
  ArrowDeviceType device_type;
  void *sync_event;
  int64_t reserved[3];
};
#endif
/* Export a column (no copy): buffers[0] = validity, [1] = values | offsets, [2] = bytes, one
 * logical offset (= the validity / boolean bit offset; `values` pointers are stepped back by
 * it, so the column must be a slice of a buffer whose row 0 is addressable — true of every
 * array this library or Arrow produces). `dtype` names the primitive type for the schema
 * format. The consumer's call of out_array->array.release invokes release_owner(owner) exactly
 * once. ctx may be NULL only for ARROW_DEVICE_CPU columns. For device columns the ctx stream is
 * synchronised first and sync_event is NULL. On any error out_array->array.release is NULL (nothing to release). */
acu_status acu_export_column(acu_ctx *ctx, const acu_column *col, acu_dtype dtype, int32_t device_type,
                             void (*release_owner)(void *), void *owner,
                             struct ArrowDeviceArray *out_array, struct ArrowSchema *out_schema);
/* View an imported (device or host) array as an acu_column: pointers into the producer's
 * buffers, valid until the caller invokes in->array.release. Flat primitive / boolean /
 * (large) utf8 / binary formats; anything else => ACU_ERR_NOT_YET_IMPLEMENTED.
 * Device rules of the C Device Data Interface: for ARROW_DEVICE_CUDA / CUDA_HOST arrays `ctx` is required, a CUDA array's
 * device_id must be the ctx's device (ACU_ERR_INVALID_ARGUMENT otherwise), and a non-NULL sync_event (a cudaEvent_t*) is
 * waited on by the ctx stream before any later kernel of this ctx can touch the buffers. ARROW_DEVICE_CPU arrays yield HOST
 * pointers (in->device_type tells the caller; ctx may be NULL); other device types => ACU_ERR_NOT_YET_IMPLEMENTED. */
acu_status acu_import_column(acu_ctx *ctx, const struct ArrowDeviceArray *in, const struct ArrowSchema *schema,
                             acu_column *out, acu_dtype *out_dtype);

/* ------------------------------------------------------------------------- */
/* Arrow IPC stream -> HBM (arrow-ipc/src/reader.rs StreamReader)            */
/* ------------------------------------------------------------------------- */
/* StreamReader::try_new (reader.rs:1587-1640) over an in-memory IPC stream (`stream` must stay valid until close): reads the
 * schema message. Flat primitive / boolean / Utf8 / Binary / LargeUtf8 / LargeBinary fields, uncompressed little-endian
 * bodies; anything else => ACU_ERR_NOT_YET_IMPLEMENTED naming the field. Errors keep the reference's texts ("Expected schema
 * message, found empty stream.", "Expected a schema as the first message in the stream, got: RecordBatch", ...). */
typedef struct acu_ipc_stream acu_ipc_stream;
acu_status acu_ipc_stream_open(acu_ctx *ctx, const uint8_t *stream, int64_t stream_len, acu_ipc_stream **out,
                               int32_t *out_n_fields);
/* Field i of the schema: kind (acu_column_kind), width (element / offset bytes), dtype (acu_dtype, -1 for boolean and byte
 * fields), nullable, name (owned by the stream). */
acu_status acu_ipc_stream_field(const acu_ipc_stream *s, int32_t i, int32_t *kind, int32_t *width, int32_t *dtype,
                                int32_t *nullable, const char **name);
/* StreamReader::next (maybe_next, reader.rs:1646-1671): decodes the next RecordBatch message. Its body goes to HBM with ONE
 * host->device copy into a buffer owned by the stream, and out_columns[0..n_fields) are VIEWS into that buffer (IPC body
 * buffers are 8-byte aligned Arrow buffers: nothing is re-laid out); they stay valid until the next call or close. The
 * validity pointer is NULL when the field node's null_count is 0 (reader.rs:271). *out_rows = -1 at the end of the stream. */
acu_status acu_ipc_stream_next(acu_ctx *ctx, acu_ipc_stream *s, acu_column *out_columns, int64_t *out_rows);
void acu_ipc_stream_close(acu_ctx *ctx, acu_ipc_stream *s);

/* ------------------------------------------------------------------------- */
/* multi-GPU: row-range shards, NCCL only for the final scalar reduce        */
/* ------------------------------------------------------------------------- */
#define ACU_NCCL_UNIQUE_ID_BYTES 128
acu_status acu_comm_get_unique_id(uint8_t out_id[ACU_NCCL_UNIQUE_ID_BYTES]);
acu_status acu_comm_init(acu_ctx *ctx, const uint8_t id[ACU_NCCL_UNIQUE_ID_BYTES], int32_t rank,
                         int32_t world_size);
acu_status acu_comm_destroy(acu_ctx *ctx);
/* All-reduce `n` per-shard partial aggregates of one (dtype, op) in one NCCL call.
 * partial_bits[i] / valid_counts[i] are what acu_aggregate returned on this rank;
 * on return they hold the global result. Float min/max are reduced on their
 * totalOrder integer keys (NCCL's float min/max are IEEE, not totalOrder). */
acu_status acu_comm_allreduce_aggregates(acu_ctx *ctx, acu_dtype dtype, acu_agg_op op,
                                         uint64_t *partial_bits, int64_t *valid_counts,
                                         int32_t n);
/* acu_aggregate over this rank's shard combined over all ranks in ONE call with ONE synchronisation: the partial stays in
 * HBM, a one-thread kernel re-encodes it (identity for a shard without valid rows, totalOrder key for float / signed
 * min / max), NCCL reduces {value, valid_count} in place on the ctx stream, and only the final pair crosses to the host
 * (no host bounce between the reduction kernel and the collective). Without a communicator it is acu_aggregate.
 * Both all-reduce entry points take ACU_SUM / ACU_MIN / ACU_MAX only: any other op => ACU_ERR_NOT_YET_IMPLEMENTED before
 * any collective runs, with or without a communicator (NCCL has no product or bitwise reduction). */
acu_status acu_aggregate_allreduce(acu_ctx *ctx, acu_dtype dtype, acu_agg_op op, const acu_array *a,
                                   uint64_t *out_bits, int64_t *out_valid_count);
/* Sum int64 scalars across ranks (row counts, null counts). */
acu_status acu_comm_allreduce_i64_sum(acu_ctx *ctx, int64_t *values, int32_t n);

#ifdef __cplusplus
}
#endif
#endif /* ARROW_CUDA_H */
