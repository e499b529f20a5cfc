// ipc.cu — Arrow IPC *stream* decode straight into HBM (SURVEY.md §8(f) rank 4: the step before the hot path).
//
// Reference: arrow-ipc/src/reader.rs — StreamReader::try_new (:1587-1640), maybe_next (:1646-1671), MessageReader framing
// (:1872-1958: optional 0xFFFFFFFF continuation marker, i32 metadata length, 0 = end of stream, a bare EOF is a valid
// end), RecordBatchDecoder::create_primitive_array (:264-297: validity buffer used only when null_count > 0), and the
// flatbuffers tables of arrow-ipc/src/gen/{Message,Schema}.rs (vtable slots cited below).
//
// Design: the reference copies every IPC buffer into its own host allocation; here a RecordBatch message costs ONE
// host->device copy of its whole body, and the columns handed to the kernels are *views* into that device buffer (IPC
// body buffers are 8-byte aligned and already in Arrow layout: values, LSB-first bitmaps, offsets — nothing to re-lay
// out). The metadata (a few hundred bytes of flatbuffers) is walked on the host by the small reader below; no flatbuffers
// library is needed for the handful of tables involved.
// Scope: flat fields of primitive / boolean / Utf8 / Binary / LargeUtf8 / LargeBinary type, uncompressed bodies, little
// endian. Dictionary-encoded, nested, view and compressed batches => ACU_ERR_NOT_YET_IMPLEMENTED (named in the message).
#include <string>
#include <vector>

#include "common.cuh"

namespace {

// ---- a minimal flatbuffers reader (little endian; every access bounds-checked against the metadata block) ----
struct Fb {
  const uint8_t *base;
  int64_t size;
  bool ok = true;
  template <class T> T rd(int64_t pos) {
    if (pos < 0 || pos + (int64_t)sizeof(T) > size) { ok = false; return T(); }
    T v;
    memcpy(&v, base + pos, sizeof(T));
    return v;
  }
  int64_t root() { return (int64_t)rd<uint32_t>(0); }
  // position of field `vt_off` (the VT_* constant of the generated code) inside table `t`, or -1 when absent
  int64_t field(int64_t t, int vt_off) {
    const int64_t vt = t - (int64_t)rd<int32_t>(t);
    const uint16_t vt_size = rd<uint16_t>(vt);
    if (!ok || vt_off + 2 > vt_size) return -1;
    const uint16_t off = rd<uint16_t>(vt + vt_off);
    return off ? t + off : -1;
  }
  template <class T> T scalar(int64_t t, int vt_off, T dflt) {
    const int64_t p = field(t, vt_off);
    return p < 0 ? dflt : rd<T>(p);
  }
  int64_t indirect(int64_t t, int vt_off) {  // offset field -> position of the referenced table / vector / string
    const int64_t p = field(t, vt_off);
    return p < 0 ? -1 : p + (int64_t)rd<uint32_t>(p);
  }
  int64_t vec_len(int64_t v) { return v < 0 ? 0 : (int64_t)rd<uint32_t>(v); }
  int64_t vec_table(int64_t v, int64_t i) {  // element i of a vector of tables
    const int64_t p = v + 4 + 4 * i;
    return p + (int64_t)rd<uint32_t>(p);
  }
  std::string str(int64_t s) {
    if (s < 0) return std::string();
    const int64_t n = vec_len(s);
    if (!ok || s + 4 + n > size) { ok = false; return std::string(); }
    return std::string(reinterpret_cast<const char *>(base + s + 4), (size_t)n);
  }
};

// Schema.fbs `Type` union tags (arrow-ipc/src/gen/Schema.rs:798-821)
enum { T_NULL = 1, T_INT = 2, T_FLOAT = 3, T_BINARY = 4, T_UTF8 = 5, T_BOOL = 6, T_LARGEBINARY = 19, T_LARGEUTF8 = 20 };
// Message.fbs `MessageHeader` union tags
enum { H_NONE = 0, H_SCHEMA = 1, H_DICTIONARY = 2, H_RECORDBATCH = 3, H_TENSOR = 4, H_SPARSETENSOR = 5 };
const char *header_name(int h) {
  static const char *n[] = {"NONE", "Schema", "DictionaryBatch", "RecordBatch", "Tensor", "SparseTensor"};
  return (h >= 0 && h <= 5) ? n[h] : "?";
}

struct FieldInfo {
  std::string name;
  int kind = ACU_COL_PRIMITIVE;  // acu_column_kind
  int width = 0;                 // element bytes (PRIMITIVE) / offset bytes (BYTES)
  int dtype = -1;                // acu_dtype for numeric fields
  int nullable = 1;
  int n_buffers = 2;             // IPC buffers of the field: validity + values (+ data)
};

struct Message {
  int header_type = H_NONE;
  int64_t meta_pos = 0, meta_len = 0;  // the flatbuffer
  int64_t body_pos = 0, body_len = 0;
};

}  // namespace

struct acu_ipc_stream {
  const uint8_t *data = nullptr;
  int64_t len = 0, pos = 0;
  std::vector<FieldInfo> fields;
  bool finished = false;
  void *d_body = nullptr;  // device copy of the current batch's body
  size_t d_body_cap = 0;
};

namespace {

// MessageReader::maybe_next (reader.rs:1872-1958). *eos = end of stream (marker, zero length or a clean EOF).
acu_status next_message(acu_ctx *ctx, acu_ipc_stream *s, Message *m, bool *eos) {
  *eos = false;
  if (s->pos + 4 > s->len) { *eos = true; return ACU_OK; }  // EOF without the 0xFFFFFFFF 0x00000000 terminator is valid
  uint32_t word;
  memcpy(&word, s->data + s->pos, 4);
  s->pos += 4;
  if (word == 0xFFFFFFFFu) {  // continuation marker: the size follows
    if (s->pos + 4 > s->len) return acu_fail(ctx, ACU_ERR_IPC, -1, 0, 0, 0, "failed to fill whole buffer");
    memcpy(&word, s->data + s->pos, 4);
    s->pos += 4;
  }
  const int32_t meta_len = (int32_t)word;
  if (meta_len == 0) { *eos = true; return ACU_OK; }
  if (meta_len < 0) return acu_fail(ctx, ACU_ERR_PARSE, -1, 0, 0, 0, "Invalid metadata length: %d", meta_len);
  if (s->pos + meta_len > s->len) return acu_fail(ctx, ACU_ERR_IPC, -1, 0, 0, 0, "failed to fill whole buffer");
  m->meta_pos = s->pos;
  m->meta_len = meta_len;
  s->pos += meta_len;
  Fb fb{s->data + m->meta_pos, m->meta_len};
  const int64_t msg = fb.root();
  m->header_type = fb.scalar<uint8_t>(msg, 6 /* VT_HEADER_TYPE */, 0);
  m->body_len = fb.scalar<int64_t>(msg, 10 /* VT_BODYLENGTH */, 0);
  if (!fb.ok) return acu_fail(ctx, ACU_ERR_PARSE, -1, 0, 0, 0, "Unable to get root as message: truncated flatbuffer");
  if (m->body_len < 0 || s->pos + m->body_len > s->len) return acu_fail(ctx, ACU_ERR_IPC, -1, 0, 0, 0, "failed to fill whole buffer");
  m->body_pos = s->pos;
  s->pos += m->body_len;
  return ACU_OK;
}

acu_status parse_schema(acu_ctx *ctx, acu_ipc_stream *s, const Message &m) {
  Fb fb{s->data + m.meta_pos, m.meta_len};
  const int64_t msg = fb.root();
  const int64_t schema = fb.indirect(msg, 8 /* VT_HEADER */);
  if (schema < 0 || !fb.ok) return acu_fail(ctx, ACU_ERR_PARSE, -1, 0, 0, 0, "Failed to parse schema from message header");
  if (fb.scalar<int16_t>(schema, 4 /* VT_ENDIANNESS */, 0) != 0)
    return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, -1, 0, 0, 0, "big-endian IPC streams");
  const int64_t fields = fb.indirect(schema, 6 /* VT_FIELDS */);
  const int64_t n = fb.vec_len(fields);
  for (int64_t i = 0; i < n; ++i) {
    const int64_t f = fb.vec_table(fields, i);
    FieldInfo fi;
    fi.name = fb.str(fb.indirect(f, 4 /* VT_NAME */));
    fi.nullable = fb.scalar<uint8_t>(f, 6 /* VT_NULLABLE */, 0);
    const int type_type = fb.scalar<uint8_t>(f, 8 /* VT_TYPE_TYPE */, 0);
    const int64_t type = fb.indirect(f, 10 /* VT_TYPE_ */);
    if (fb.field(f, 12 /* VT_DICTIONARY */) >= 0)
      return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, i, 0, 0, 0, "IPC field '%s': dictionary-encoded fields", fi.name.c_str());
    if (fb.vec_len(fb.indirect(f, 14 /* VT_CHILDREN */)) > 0)
      return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, i, 0, 0, 0, "IPC field '%s': nested types", fi.name.c_str());
    switch (type_type) {
      case T_INT: {
        const int bits = fb.scalar<int32_t>(type, 4 /* VT_BITWIDTH */, 0);
        const bool sgn = fb.scalar<uint8_t>(type, 6 /* VT_IS_SIGNED */, 0) != 0;
        fi.kind = ACU_COL_PRIMITIVE;
        fi.width = bits / 8;
        switch (bits) {
          case 8: fi.dtype = sgn ? ACU_I8 : ACU_U8; break;
          case 16: fi.dtype = sgn ? ACU_I16 : ACU_U16; break;
          case 32: fi.dtype = sgn ? ACU_I32 : ACU_U32; break;
          case 64: fi.dtype = sgn ? ACU_I64 : ACU_U64; break;
          default: return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, i, 0, 0, 0, "IPC field '%s': Int of %d bits", fi.name.c_str(), bits);
        }
        break;
      }
      case T_FLOAT: {
        const int prec = fb.scalar<int16_t>(type, 4 /* VT_PRECISION */, 0);  // HALF 0, SINGLE 1, DOUBLE 2
        if (prec != 1 && prec != 2) return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, i, 0, 0, 0, "IPC field '%s': Float16", fi.name.c_str());
        fi.kind = ACU_COL_PRIMITIVE;
        fi.width = prec == 1 ? 4 : 8;
        fi.dtype = prec == 1 ? ACU_F32 : ACU_F64;
        break;
      }
      case T_BOOL: fi.kind = ACU_COL_BOOLEAN; fi.width = 0; break;
      case T_UTF8: case T_BINARY: fi.kind = ACU_COL_BYTES; fi.width = 4; fi.n_buffers = 3; break;
      case T_LARGEUTF8: case T_LARGEBINARY: fi.kind = ACU_COL_BYTES; fi.width = 8; fi.n_buffers = 3; break;
      default:
        return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, i, 0, 0, 0, "IPC field '%s': type tag %d", fi.name.c_str(), type_type);
    }
    if (!fb.ok) return acu_fail(ctx, ACU_ERR_PARSE, -1, 0, 0, 0, "Failed to parse schema from message header");
    s->fields.push_back(fi);
  }
  return ACU_OK;
}

}  // namespace

extern "C" {

acu_status acu_ipc_stream_open(acu_ctx *ctx, const uint8_t *stream, int64_t stream_len, acu_ipc_stream **out, int32_t *out_n_fields) {
  ACU_ENTER(ctx);
  *out = nullptr;
  acu_ipc_stream *s = new acu_ipc_stream();
  s->data = stream;
  s->len = stream_len;
  Message m;
  bool eos = false;
  acu_status st = next_message(ctx, s, &m, &eos);
  if (st == ACU_OK && eos) st = acu_fail(ctx, ACU_ERR_IPC, -1, 0, 0, 0, "Expected schema message, found empty stream.");  // reader.rs:1593-1597
  if (st == ACU_OK && m.header_type != H_SCHEMA)
    st = acu_fail(ctx, ACU_ERR_IPC, -1, 0, 0, 0, "Expected a schema as the first message in the stream, got: %s", header_name(m.header_type));
  if (st == ACU_OK) st = parse_schema(ctx, s, m);
  if (st != ACU_OK) { delete s; return st; }
  if (out_n_fields) *out_n_fields = (int32_t)s->fields.size();
  *out = s;
  return ACU_OK;
}

acu_status acu_ipc_stream_field(const acu_ipc_stream *s, int32_t i, int32_t *kind, int32_t *width, int32_t *dtype, int32_t *nullable,
                                const char **name) {
  if (!s || i < 0 || (size_t)i >= s->fields.size()) return ACU_ERR_INVALID_ARGUMENT;
  const FieldInfo &f = s->fields[(size_t)i];
  if (kind) *kind = f.kind;
  if (width) *width = f.width;
  if (dtype) *dtype = f.dtype;
  if (nullable) *nullable = f.nullable;
  if (name) *name = f.name.c_str();
  return ACU_OK;
}

acu_status acu_ipc_stream_next(acu_ctx *ctx, acu_ipc_stream *s, acu_column *out_columns, int64_t *out_rows) {
  ACU_ENTER(ctx);
  *out_rows = -1;
  if (s->finished) return ACU_OK;
  for (;;) {
    Message m;
    bool eos = false;
    ACU_TRY(next_message(ctx, s, &m, &eos));
    if (eos) { s->finished = true; return ACU_OK; }
    if (m.header_type == H_SCHEMA)  // reader.rs:1661-1665
      return acu_fail(ctx, ACU_ERR_IPC, -1, 0, 0, 0, "Expected a record batch, but found a schema");
    if (m.header_type == H_DICTIONARY) continue;  // no field of a supported schema references a dictionary
    if (m.header_type != H_RECORDBATCH)
      return acu_fail(ctx, ACU_ERR_PARSE, -1, 0, 0, 0, "Unsupported message header type in IPC stream: '%s'", header_name(m.header_type));
    Fb fb{s->data + m.meta_pos, m.meta_len};
    const int64_t msg = fb.root();
    const int64_t rb = fb.indirect(msg, 8 /* VT_HEADER */);
    if (rb < 0) return acu_fail(ctx, ACU_ERR_IPC, -1, 0, 0, 0, "Unable to read IPC message as record batch");
    if (fb.field(rb, 10 /* VT_COMPRESSION */) >= 0) return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, -1, 0, 0, 0, "compressed IPC record batches");
    const int64_t rows = fb.scalar<int64_t>(rb, 4 /* VT_LENGTH */, 0);
    const int64_t nodes = fb.indirect(rb, 6 /* VT_NODES */), buffers = fb.indirect(rb, 8 /* VT_BUFFERS */);
    if (nodes < 0) return acu_fail(ctx, ACU_ERR_IPC, -1, 0, 0, 0, "Unable to get field nodes from IPC RecordBatch");
    if (buffers < 0) return acu_fail(ctx, ACU_ERR_IPC, -1, 0, 0, 0, "Unable to get buffers from IPC RecordBatch");
    const int64_t n_nodes = fb.vec_len(nodes), n_bufs = fb.vec_len(buffers);
    int64_t need_bufs = 0;
    for (const FieldInfo &f : s->fields) need_bufs += f.n_buffers;
    if (n_nodes != (int64_t)s->fields.size() || n_bufs < need_bufs)
      return acu_fail(ctx, ACU_ERR_IPC, -1, 0, 0, 0, "Buffer count mismatched with metadata");
    // the whole body in one host -> device copy
    if ((size_t)m.body_len > s->d_body_cap) {
      if (s->d_body) ACU_TRY(acu_free(ctx, s->d_body));
      s->d_body = nullptr;
      s->d_body_cap = 0;
      ACU_TRY(acu_malloc(ctx, (size_t)m.body_len + 64, &s->d_body));
      s->d_body_cap = (size_t)m.body_len;
    }
    if (m.body_len) ACU_CUDA(ctx, cudaMemcpyAsync(s->d_body, s->data + m.body_pos, (size_t)m.body_len, cudaMemcpyHostToDevice, ctx->stream));
    // FieldNode { length: i64, null_count: i64 } and Buffer { offset: i64, length: i64 } are inline 16-byte structs
    int64_t b = 0;
    for (size_t c = 0; c < s->fields.size(); ++c) {
      const FieldInfo &f = s->fields[c];
      const int64_t node = nodes + 4 + 16 * (int64_t)c;
      const int64_t len = fb.rd<int64_t>(node), nulls = fb.rd<int64_t>(node + 8);
      int64_t boff[3] = {0, 0, 0}, blen[3] = {0, 0, 0};
      for (int k = 0; k < f.n_buffers; ++k, ++b) {
        boff[k] = fb.rd<int64_t>(buffers + 4 + 16 * b);
        blen[k] = fb.rd<int64_t>(buffers + 4 + 16 * b + 8);
        if (boff[k] < 0 || blen[k] < 0 || boff[k] + blen[k] > m.body_len) return acu_fail(ctx, ACU_ERR_IPC, (int64_t)c, 0, 0, 0, "Buffer count mismatched with metadata");
      }
      if (!fb.ok) return acu_fail(ctx, ACU_ERR_IPC, -1, 0, 0, 0, "Unable to read IPC message as record batch");
      uint8_t *body = static_cast<uint8_t *>(s->d_body);
      acu_column &col = out_columns[c];
      col = acu_column{};
      col.kind = f.kind;
      col.width = f.width;
      col.array.len = len;
      col.array.null_count = nulls;
      // reader.rs:271: the validity buffer is used only when null_count > 0 (writers may send an empty one otherwise)
      col.array.validity = (nulls > 0 && blen[0] > 0) ? body + boff[0] : nullptr;
      col.array.values = body + boff[1];
      if (f.kind == ACU_COL_BYTES) col.data = body + boff[2];
      if (len != rows) return acu_fail(ctx, ACU_ERR_IPC, (int64_t)c, 0, 0, 0, "Buffer count mismatched with metadata");
    }
    ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // the host bytes may be released after the call
    *out_rows = rows;
    return ACU_OK;
  }
}

void acu_ipc_stream_close(acu_ctx *ctx, acu_ipc_stream *s) {
  if (!s) return;
  if (s->d_body) acu_free(ctx, s->d_body);
  delete s;
}

}  // extern "C"
