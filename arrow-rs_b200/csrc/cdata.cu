// cdata.cu — Arrow C Data Interface / C Device Data Interface for the columns this library works
// on (SURVEY.md §8(f) rank 4: the format either side of the path).
//
// The reference speaks the C Data Interface (FFI_ArrowArray, arrow-data/src/ffi.rs:37-69;
// FFI_ArrowSchema, arrow-schema/src/ffi.rs; to_ffi / from_ffi, arrow-array/src/ffi.rs:237-271)
// but has no ArrowDeviceArray. A device-resident result leaves here as an ArrowDeviceArray
// (device_type = ARROW_DEVICE_CUDA, device_id = the ctx's device, sync_event = NULL after a
// stream synchronisation) whose embedded ArrowArray has exactly the reference's layout:
// buffers[0] = validity, buffers[1] = values | offsets, buffers[2] = value bytes, one logical
// `offset` for all of them. Pure host code: no kernels, no copies — ownership moves through the
// release callback (the consumer calls it exactly once, arrow-data/src/ffi.rs:69-98).
#include <stdlib.h>
#include <string.h>

#include "common.cuh"

namespace {

struct ExportPrivate {
  const void *buffers[3];
  void (*release_owner)(void *);
  void *owner;
};

void release_exported_array(struct ArrowArray *array) {
  if (!array || !array->release) return;
  ExportPrivate *p = static_cast<ExportPrivate *>(array->private_data);
  if (p) {
    if (p->release_owner) p->release_owner(p->owner);
    free(p);
  }
  array->release = nullptr;  // marks the structure released (Arrow C Data Interface)
}

void release_exported_schema(struct ArrowSchema *schema) {
  if (!schema || !schema->release) return;
  schema->release = nullptr;  // format / name point to static strings: nothing to free
}

const char *format_of(int32_t kind, int32_t width, acu_dtype dtype) {
  if (kind == ACU_COL_BOOLEAN) return "b";
  if (kind == ACU_COL_BYTES) return width == 8 ? "U" : "u";
  static const char *f[] = {"c", "s", "i", "l", "C", "S", "I", "L", "f", "g"};
  return f[(int)dtype];
}

bool parse_format(const char *fmt, int32_t *kind, int32_t *width, acu_dtype *dtype) {
  if (!fmt || !fmt[0] || fmt[1]) return false;
  *dtype = ACU_U8;
  switch (fmt[0]) {
    case 'b': *kind = ACU_COL_BOOLEAN; *width = 0; return true;
    case 'u': case 'z': *kind = ACU_COL_BYTES; *width = 4; return true;
    case 'U': case 'Z': *kind = ACU_COL_BYTES; *width = 8; return true;
    default: break;
  }
  static const char codes[] = "csilCSILfg";
  const char *p = strchr(codes, fmt[0]);
  if (!p) return false;
  *kind = ACU_COL_PRIMITIVE;
  *dtype = (acu_dtype)(p - codes);
  *width = acu_dtype_size(*dtype);
  return true;
}

}  // namespace

extern "C" acu_status acu_export_column(acu_ctx *ctx, const acu_column *col, acu_dtype dtype, int32_t device_type,
                                        void (*release_owner)(void *), void *owner, struct ArrowDeviceArray *out_array,
                                        struct ArrowSchema *out_schema) {
  if (!col || !out_array) return ctx ? acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "export: NULL argument") : ACU_ERR_INVALID_ARGUMENT;
  out_array->array.release = nullptr;  // stays NULL on every error path: the caller of a failed export has nothing to release
  if (col->kind == ACU_COL_FIXED_SIZE_BINARY)
    return ctx ? acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "export: FixedSizeBinary columns are not supported") : ACU_ERR_INVALID_ARGUMENT;
  if (device_type != ARROW_DEVICE_CPU) {
    // a device column needs the ctx: no event is handed over (sync_event = NULL), so the data must be complete when this
    // returns — synchronise BEFORE anything is allocated or published
    if (!ctx) return ACU_ERR_INVALID_ARGUMENT;
    ACU_ENTER(ctx);
    ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  }
  const acu_array &a = col->array;
  // one logical offset for every buffer: the bit offset of the validity (and of boolean values)
  int64_t offset = a.validity ? a.validity_offset : 0;
  if (col->kind == ACU_COL_BOOLEAN) {
    if (a.validity && a.validity_offset != a.values_offset) {
      if (!ctx) return ACU_ERR_INVALID_ARGUMENT;
      return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "export: boolean values and validity must share one offset (got %lld / %lld)",
                      (long long)a.values_offset, (long long)a.validity_offset);
    }
    offset = a.values_offset;
  }
  ExportPrivate *p = static_cast<ExportPrivate *>(calloc(1, sizeof(ExportPrivate)));
  if (!p) return ACU_ERR_OUT_OF_MEMORY;
  p->release_owner = release_owner;
  p->owner = owner;
  const int64_t elem = col->kind == ACU_COL_PRIMITIVE ? col->width : col->kind == ACU_COL_BYTES ? col->width : 0;
  p->buffers[0] = a.validity;
  // `values` already points at logical row 0: step back so that buffers[1] + offset * width is row 0 again
  p->buffers[1] = col->kind == ACU_COL_BOOLEAN ? a.values : static_cast<const uint8_t *>(a.values) - (size_t)offset * (size_t)elem;
  p->buffers[2] = col->kind == ACU_COL_BYTES ? col->data : nullptr;
  memset(out_array, 0, sizeof(*out_array));
  struct ArrowArray *arr = &out_array->array;
  arr->length = a.len;
  arr->null_count = a.validity ? a.null_count : 0;  // -1 = unknown, as in the C Data Interface
  arr->offset = offset;
  arr->n_buffers = col->kind == ACU_COL_BYTES ? 3 : 2;
  arr->n_children = 0;
  arr->buffers = p->buffers;
  arr->children = nullptr;
  arr->dictionary = nullptr;
  arr->release = release_exported_array;
  arr->private_data = p;
  out_array->device_type = device_type;
  out_array->device_id = (device_type == ARROW_DEVICE_CPU || !ctx) ? -1 : ctx->device;
  out_array->sync_event = nullptr;
  if (out_schema) {
    memset(out_schema, 0, sizeof(*out_schema));
    out_schema->format = format_of(col->kind, col->width, dtype);
    out_schema->name = "";
    out_schema->metadata = nullptr;
    out_schema->flags = 2;  // ARROW_FLAG_NULLABLE
    out_schema->release = release_exported_schema;
  }
  return ACU_OK;
}

extern "C" acu_status acu_import_column(acu_ctx *ctx, const struct ArrowDeviceArray *in, const struct ArrowSchema *schema, acu_column *out,
                                        acu_dtype *out_dtype) {
  if (!in || !schema || !out || !in->array.release || !schema->release)
    return ctx ? acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "import: NULL argument or released array") : ACU_ERR_INVALID_ARGUMENT;
  // Arrow C Device Data Interface: the consumer must know where the buffers live and must wait on a non-NULL sync_event
  // before touching them
  if (in->device_type == ARROW_DEVICE_CUDA || in->device_type == ARROW_DEVICE_CUDA_HOST) {
    if (!ctx) return ACU_ERR_INVALID_ARGUMENT;  // device memory cannot be consumed without a stream to order against
    ACU_ENTER(ctx);
    if (in->device_type == ARROW_DEVICE_CUDA && in->device_id != ctx->device)
      return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "import: array lives on CUDA device %lld, this context drives device %d",
                      (long long)in->device_id, ctx->device);
    if (in->sync_event) ACU_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, *static_cast<cudaEvent_t *>(in->sync_event), 0));
  } else if (in->device_type != ARROW_DEVICE_CPU) {
    return ctx ? acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, -1, 0, 0, 0, "import: ArrowDeviceType %d", (int)in->device_type) : ACU_ERR_NOT_YET_IMPLEMENTED;
  }
  int32_t kind, width;
  acu_dtype dtype;
  if (!parse_format(schema->format, &kind, &width, &dtype)) return ACU_ERR_NOT_YET_IMPLEMENTED;  // nested / temporal / decimal formats
  const struct ArrowArray &a = in->array;
  if (a.n_children != 0 || a.dictionary != nullptr) return ACU_ERR_NOT_YET_IMPLEMENTED;
  if (a.n_buffers != (kind == ACU_COL_BYTES ? 3 : 2)) return ACU_ERR_INVALID_ARGUMENT;
  memset(out, 0, sizeof(*out));
  out->kind = kind;
  out->width = width;
  out->array.len = a.length;
  out->array.validity = static_cast<const uint8_t *>(a.buffers[0]);
  out->array.validity_offset = a.buffers[0] ? a.offset : 0;
  out->array.null_count = a.buffers[0] ? a.null_count : 0;
  if (kind == ACU_COL_BOOLEAN) {
    out->array.values = a.buffers[1];
    out->array.values_offset = a.offset;
  } else {
    out->array.values = static_cast<const uint8_t *>(a.buffers[1]) + (size_t)a.offset * (size_t)width;
    if (kind == ACU_COL_BYTES) out->data = static_cast<const uint8_t *>(a.buffers[2]);
  }
  if (out_dtype) *out_dtype = dtype;
  return ACU_OK;
}
