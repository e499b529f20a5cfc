// arrow_cuda.hpp — C++17 host-side mirror of the arrow-rs compute API over the C ABI.
//
// The reference's host language is Rust; there is no Rust toolchain in this image, so this
// header plays the role of the `arrow-cuda` crate: the same type and function names, argument
// order and error text as the reference, every call forwarded to libarrow_cuda.so
// (include/arrow_cuda.h). Arrays own DeviceBuffers (HBM) with arrow-buffer's layout: values
// buffer + LSB-first validity bitmap + bit offset + cached null_count.
//
//   arrow-rs                                              here
//   ----------------------------------------------------  -------------------------------------------
//   arrow_schema::ArrowError          (error.rs:26-67)    arrow_cuda::ArrowError
//   Result<T, ArrowError>                                 arrow_cuda::Result<T>  (.unwrap(), .unwrap_err())
//   arrow_buffer::Buffer / NullBuffer (immutable.rs:83)   arrow_cuda::Buffer / NullBuffer
//   ArrayRef = Arc<dyn Array>         (array/mod.rs:446)  ArrayRef = std::shared_ptr<Array>
//   PrimitiveArray<T>, BooleanArray, StringArray          same names
//   Scalar<T> / Datum                 (scalar.rs:78-152)  Scalar / Datum
//   RecordBatch                       (record_batch.rs)   RecordBatch
//   arrow::compute::{filter, take, cast, ...}             arrow_cuda::compute::{...}
//   arrow::compute::kernels::{numeric, cmp}::*            arrow_cuda::compute::kernels::{numeric, cmp}::*
//
// No CPU fallback: Context::get() throws if no CUDA device / library is available.
#pragma once

#include <algorithm>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <optional>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <variant>
#include <vector>

#include "../../include/arrow_cuda.h"

namespace arrow_cuda {

// ---------------------------------------------------------------------------------------
// ArrowError / Result
// ---------------------------------------------------------------------------------------
struct ArrowError {
  acu_status status = ACU_OK;
  std::string message;  // == the reference's Display output
  int64_t index = -1;
  const std::string &to_string() const { return message; }
};

template <class T>
class Result {
 public:
  Result(T v) : v_(std::move(v)) {}            // NOLINT(google-explicit-constructor)
  Result(ArrowError e) : v_(std::move(e)) {}   // NOLINT(google-explicit-constructor)
  bool is_ok() const { return v_.index() == 0; }
  bool is_err() const { return !is_ok(); }
  T unwrap() {
    if (!is_ok()) throw std::runtime_error("called `Result::unwrap()` on an `Err` value: " + std::get<1>(v_).message);
    return std::move(std::get<0>(v_));
  }
  ArrowError unwrap_err() const {
    if (is_ok()) throw std::runtime_error("called `Result::unwrap_err()` on an `Ok` value");
    return std::get<1>(v_);
  }
 private:
  std::variant<T, ArrowError> v_;
};

// ---------------------------------------------------------------------------------------
// Context: one acu_ctx per device (the reference kernels are pure functions; the ctx is
// the implicit "where does this run")
// ---------------------------------------------------------------------------------------
class Context {
 public:
  static Context &get(int device = 0) {
    static std::map<int, std::unique_ptr<Context>> ctxs;
    auto it = ctxs.find(device);
    if (it == ctxs.end()) it = ctxs.emplace(device, std::unique_ptr<Context>(new Context(device))).first;
    return *it->second;
  }
  acu_ctx *raw() const { return ctx_; }
  ArrowError last_error(acu_status st) const {
    const acu_error_detail *d = acu_last_error(ctx_);
    return ArrowError{st, d->message, d->index};
  }
  ~Context() { acu_ctx_destroy(ctx_); }
 private:
  explicit Context(int device) {
    if (acu_ctx_create(device, &ctx_) != ACU_OK)
      throw std::runtime_error("arrow-cuda: no usable CUDA device (there is no CPU fallback)");
  }
  acu_ctx *ctx_ = nullptr;
};

// ---------------------------------------------------------------------------------------
// DeviceBuffer (arrow_buffer::Buffer): Arc-owned allocation + byte length
// ---------------------------------------------------------------------------------------
class Buffer {
 public:
  Buffer() = default;
  static Buffer allocate(size_t bytes, int device = 0) {
    Buffer b;
    void *p = nullptr;
    acu_ctx *ctx = Context::get(device).raw();
    if (acu_malloc(ctx, bytes + 16, &p) != ACU_OK) throw std::bad_alloc();
    b.mem_ = std::shared_ptr<void>(p, [ctx](void *q) { acu_free(ctx, q); });
    b.len_ = bytes;
    return b;
  }
  static Buffer from_host(const void *src, size_t bytes, int device = 0) {
    Buffer b = allocate(bytes, device);
    if (bytes) acu_memcpy_h2d(Context::get(device).raw(), b.mem_.get(), src, bytes);
    return b;
  }
  void to_host(void *dst, size_t bytes, int device = 0) const {
    if (bytes) acu_memcpy_d2h(Context::get(device).raw(), dst, mem_.get(), bytes);
  }
  void *data() const { return mem_.get(); }
  size_t len() const { return len_; }
 private:
  std::shared_ptr<void> mem_;
  size_t len_ = 0;
};

// NullBuffer { buffer: BooleanBuffer, null_count } (arrow-buffer/src/buffer/null.rs:34-37)
struct NullBuffer {
  Buffer buffer;
  int64_t offset = 0;  // bit offset
  int64_t len = 0;
  int64_t null_count = 0;
};

inline std::vector<uint8_t> pack_bits(const std::vector<bool> &bits) {
  std::vector<uint8_t> out(acu_bitmap_bytes((int64_t)bits.size()) + 8, 0);
  for (size_t i = 0; i < bits.size(); ++i)
    if (bits[i]) out[i >> 3] |= (uint8_t)(1u << (i & 7));
  return out;
}

// ---------------------------------------------------------------------------------------
// DataType / native type traits (arrow-array/src/types.rs:67-80)
// ---------------------------------------------------------------------------------------
enum class DataType { Int8, Int16, Int32, Int64, UInt8, UInt16, UInt32, UInt64, Float32, Float64, Boolean, Utf8, Decimal32, Decimal64, Decimal128,
                      List, LargeList, FixedSizeList, RunEndEncoded, Struct, Union, FixedSizeBinary };

template <class T> struct NativeOf;
#define ACU_NATIVE(T, DT, CODE) \
  template <> struct NativeOf<T> { static constexpr DataType data_type = DataType::DT; static constexpr acu_dtype code = CODE; };
ACU_NATIVE(int8_t, Int8, ACU_I8) ACU_NATIVE(int16_t, Int16, ACU_I16) ACU_NATIVE(int32_t, Int32, ACU_I32)
ACU_NATIVE(int64_t, Int64, ACU_I64) ACU_NATIVE(uint8_t, UInt8, ACU_U8) ACU_NATIVE(uint16_t, UInt16, ACU_U16)
ACU_NATIVE(uint32_t, UInt32, ACU_U32) ACU_NATIVE(uint64_t, UInt64, ACU_U64) ACU_NATIVE(float, Float32, ACU_F32)
ACU_NATIVE(double, Float64, ACU_F64)
#undef ACU_NATIVE

inline int dtype_code(DataType t) { return (int)t; }  // numeric DataTypes share acu_dtype's numbering
inline int dtype_width(DataType t) {
  switch (t) {
    case DataType::Int8: case DataType::UInt8: return 1;
    case DataType::Int16: case DataType::UInt16: return 2;
    case DataType::Int32: case DataType::UInt32: case DataType::Float32: return 4;
    case DataType::Int64: case DataType::UInt64: case DataType::Float64: return 8;
    default: return 0;
  }
}

// ---------------------------------------------------------------------------------------
// Arrays
// ---------------------------------------------------------------------------------------
class Array {
 public:
  virtual ~Array() = default;
  virtual DataType data_type() const = 0;
  int64_t len() const { return len_; }
  bool is_empty() const { return len_ == 0; }
  const std::optional<NullBuffer> &nulls() const { return nulls_; }
  int64_t null_count() const { return nulls_ ? nulls_->null_count : 0; }
  // acu_array view (borrowed)
  acu_array view(bool scalar = false) const {
    acu_array a{};
    a.values = values_ptr();
    a.values_offset = values_bit_offset();
    a.validity = nulls_ ? static_cast<const uint8_t *>(nulls_->buffer.data()) : nullptr;
    a.validity_offset = nulls_ ? nulls_->offset : 0;
    a.len = len_;
    a.null_count = nulls_ ? nulls_->null_count : 0;
    a.is_scalar = scalar ? 1 : 0;
    return a;
  }
  std::vector<bool> valid_mask() const {
    std::vector<bool> v((size_t)len_, true);
    if (nulls_) {
      std::vector<uint8_t> bits(acu_bitmap_bytes(nulls_->offset + len_) + 8);
      nulls_->buffer.to_host(bits.data(), std::min(bits.size(), nulls_->buffer.len()));
      for (int64_t i = 0; i < len_; ++i) v[(size_t)i] = (bits[(size_t)((nulls_->offset + i) >> 3)] >> ((nulls_->offset + i) & 7)) & 1;
    }
    return v;
  }
  bool is_null(int64_t i) const { return !valid_mask()[(size_t)i]; }
  bool is_valid(int64_t i) const { return !is_null(i); }
 protected:
  virtual const void *values_ptr() const = 0;
  virtual int64_t values_bit_offset() const { return 0; }
  int64_t len_ = 0;
  std::optional<NullBuffer> nulls_;
};
using ArrayRef = std::shared_ptr<Array>;

inline std::optional<NullBuffer> nulls_from_mask(const std::vector<bool> &valid, bool force = false) {
  int64_t nc = 0;
  for (bool b : valid) nc += !b;
  if (nc == 0 && !force) return std::nullopt;
  auto bits = pack_bits(valid);
  return NullBuffer{Buffer::from_host(bits.data(), bits.size()), 0, (int64_t)valid.size(), nc};
}

template <class T>
class PrimitiveArray : public Array {
 public:
  using Native = T;
  PrimitiveArray() = default;
  // PrimitiveArray::new(values, nulls)
  PrimitiveArray(Buffer values, int64_t len, std::optional<NullBuffer> nulls, int64_t elem_offset = 0)
      : values_(std::move(values)), elem_offset_(elem_offset) { len_ = len; nulls_ = std::move(nulls); }
  // From<Vec<T>> / From<Vec<Option<T>>>
  static PrimitiveArray from(const std::vector<T> &v) {
    return PrimitiveArray(Buffer::from_host(v.data(), v.size() * sizeof(T)), (int64_t)v.size(), std::nullopt);
  }
  static PrimitiveArray from(const std::vector<std::optional<T>> &v) {
    std::vector<T> vals(v.size(), T());
    std::vector<bool> valid(v.size(), true);
    for (size_t i = 0; i < v.size(); ++i) { if (v[i]) vals[i] = *v[i]; else valid[i] = false; }
    return PrimitiveArray(Buffer::from_host(vals.data(), vals.size() * sizeof(T)), (int64_t)v.size(), nulls_from_mask(valid));
  }
  static PrimitiveArray new_null(int64_t len) {
    std::vector<std::optional<T>> v((size_t)len, std::nullopt);
    auto a = from(v);
    if (!a.nulls_) a.nulls_ = nulls_from_mask(std::vector<bool>((size_t)len, false), true);
    return a;
  }
  DataType data_type() const override { return NativeOf<T>::data_type; }
  // Array::slice — zero copy (pointer + bit-offset arithmetic)
  PrimitiveArray slice(int64_t offset, int64_t length) const {
    PrimitiveArray out(values_, length, nulls_, elem_offset_ + offset);
    if (out.nulls_) {
      out.nulls_->offset += offset;
      out.nulls_->len = length;
      out.nulls_->null_count = -1;  // recounted on device on first use
    }
    return out;
  }
  std::vector<T> values() const {
    std::vector<T> v((size_t)len_);
    if (len_) acu_memcpy_d2h(Context::get().raw(), v.data(), values_ptr(), (size_t)len_ * sizeof(T));
    return v;
  }
  T value(int64_t i) const { return values()[(size_t)i]; }
  const Buffer &buffer() const { return values_; }
  int64_t elem_offset() const { return elem_offset_; }
  std::vector<std::optional<T>> to_vec() const {
    auto vals = values();
    auto valid = valid_mask();
    std::vector<std::optional<T>> out((size_t)len_);
    for (size_t i = 0; i < out.size(); ++i) if (valid[i]) out[i] = vals[i];
    return out;
  }
 protected:
  const void *values_ptr() const override { return static_cast<const T *>(values_.data()) + elem_offset_; }
 private:
  Buffer values_;
  int64_t elem_offset_ = 0;
};
using Int8Array = PrimitiveArray<int8_t>;
using Int16Array = PrimitiveArray<int16_t>;
using Int32Array = PrimitiveArray<int32_t>;
using Int64Array = PrimitiveArray<int64_t>;
using UInt8Array = PrimitiveArray<uint8_t>;
using UInt16Array = PrimitiveArray<uint16_t>;
using UInt32Array = PrimitiveArray<uint32_t>;
using UInt64Array = PrimitiveArray<uint64_t>;
using Float32Array = PrimitiveArray<float>;
using Float64Array = PrimitiveArray<double>;

// Decimal32 / Decimal64 / Decimal128 (arrow-array/src/types.rs DecimalType): natives int32_t / int64_t / __int128, with the
// type's precision and scale. Decimal256 is not supported.
template <class T> struct DecimalTraits;
template <> struct DecimalTraits<int32_t> {
  static constexpr DataType data_type = DataType::Decimal32; static constexpr acu_dtype code = ACU_I32;
  static constexpr uint8_t max_precision = 9; static constexpr int8_t default_scale = 2; static constexpr const char *prefix = "Decimal32";
};
template <> struct DecimalTraits<int64_t> {
  static constexpr DataType data_type = DataType::Decimal64; static constexpr acu_dtype code = ACU_I64;
  static constexpr uint8_t max_precision = 18; static constexpr int8_t default_scale = 6; static constexpr const char *prefix = "Decimal64";
};
template <> struct DecimalTraits<__int128> {
  static constexpr DataType data_type = DataType::Decimal128; static constexpr acu_dtype code = ACU_I128;
  static constexpr uint8_t max_precision = 38; static constexpr int8_t default_scale = 10; static constexpr const char *prefix = "Decimal128";
};

// validate_decimal_precision_and_scale (arrow-array/src/types.rs:1442-1472): the error's Display text, empty when valid
inline std::string decimal_type_error(int max_precision, int precision, int scale) {
  const std::string p = "Invalid argument error: ";
  if (precision == 0) return p + "precision cannot be 0, has to be between [1, " + std::to_string(max_precision) + "]";
  if (precision > max_precision) return p + "precision " + std::to_string(precision) + " is greater than max " + std::to_string(max_precision);
  if (scale > max_precision) return p + "scale " + std::to_string(scale) + " is greater than max " + std::to_string(max_precision);
  if (scale > 0 && scale > precision) return p + "scale " + std::to_string(scale) + " is greater than precision " + std::to_string(precision);
  return "";
}

template <class T>
class DecimalArray : public Array {
 public:
  using Native = T;
  using Traits = DecimalTraits<T>;
  DecimalArray() = default;
  DecimalArray(Buffer values, int64_t len, std::optional<NullBuffer> nulls, int64_t elem_offset = 0,
               uint8_t precision = Traits::max_precision, int8_t scale = Traits::default_scale)
      : values_(std::move(values)), elem_offset_(elem_offset), precision_(precision), scale_(scale) { len_ = len; nulls_ = std::move(nulls); }
  // From<Vec<T>> / From<Vec<Option<T>>>: the default type Decimal*(MAX_PRECISION, DEFAULT_SCALE)
  static DecimalArray from(const std::vector<T> &v) {
    return DecimalArray(Buffer::from_host(v.data(), v.size() * sizeof(T)), (int64_t)v.size(), std::nullopt);
  }
  static DecimalArray from(const std::vector<std::optional<T>> &v) {
    std::vector<T> vals(v.size(), T());
    std::vector<bool> valid(v.size(), true);
    for (size_t i = 0; i < v.size(); ++i) { if (v[i]) vals[i] = *v[i]; else valid[i] = false; }
    return DecimalArray(Buffer::from_host(vals.data(), vals.size() * sizeof(T)), (int64_t)v.size(), nulls_from_mask(valid));
  }
  // PrimitiveArray::with_precision_and_scale (primitive_array.rs:1665-1671)
  Result<DecimalArray> with_precision_and_scale(uint8_t precision, int8_t scale) const {
    const std::string e = decimal_type_error(Traits::max_precision, precision, scale);
    if (!e.empty()) return ArrowError{ACU_ERR_INVALID_ARGUMENT, e};
    return DecimalArray(values_, len_, nulls_, elem_offset_, precision, scale);
  }
  DataType data_type() const override { return Traits::data_type; }
  uint8_t precision() const { return precision_; }
  int8_t scale() const { return scale_; }
  acu_decimal_type decimal_type() const { return acu_decimal_type{(int32_t)sizeof(T), precision_, scale_, {0, 0}}; }
  std::string type_display() const {  // Display of DataType::Decimal*(p, s)
    return std::string(Traits::prefix) + "(" + std::to_string((int)precision_) + ", " + std::to_string((int)scale_) + ")";
  }
  DecimalArray slice(int64_t offset, int64_t length) const {
    DecimalArray out(values_, length, nulls_, elem_offset_ + offset, precision_, scale_);
    if (out.nulls_) {
      out.nulls_->offset += offset;
      out.nulls_->len = length;
      out.nulls_->null_count = -1;
    }
    return out;
  }
  std::vector<T> values() const {
    std::vector<T> v((size_t)len_);
    if (len_) acu_memcpy_d2h(Context::get().raw(), v.data(), values_ptr(), (size_t)len_ * sizeof(T));
    return v;
  }
  std::vector<std::optional<T>> to_vec() const {
    auto vals = values();
    auto valid = valid_mask();
    std::vector<std::optional<T>> out((size_t)len_);
    for (size_t i = 0; i < out.size(); ++i) if (valid[i]) out[i] = vals[i];
    return out;
  }
 protected:
  const void *values_ptr() const override { return static_cast<const T *>(values_.data()) + elem_offset_; }
 private:
  Buffer values_;
  int64_t elem_offset_ = 0;
  uint8_t precision_ = Traits::max_precision;
  int8_t scale_ = Traits::default_scale;
};
using Decimal32Array = DecimalArray<int32_t>;
using Decimal64Array = DecimalArray<int64_t>;
using Decimal128Array = DecimalArray<__int128>;
template <class A> struct is_decimal_array : std::false_type {};
template <class T> struct is_decimal_array<DecimalArray<T>> : std::true_type {};

class BooleanArray : public Array {
 public:
  BooleanArray() = default;
  BooleanArray(Buffer bits, int64_t bit_offset, int64_t len, std::optional<NullBuffer> nulls)
      : bits_(std::move(bits)), bit_offset_(bit_offset) { len_ = len; nulls_ = std::move(nulls); }
  static BooleanArray from(const std::vector<bool> &v) {
    auto bits = pack_bits(v);
    return BooleanArray(Buffer::from_host(bits.data(), bits.size()), 0, (int64_t)v.size(), std::nullopt);
  }
  static BooleanArray from(const std::vector<std::optional<bool>> &v) {
    std::vector<bool> vals(v.size(), false), valid(v.size(), true);
    for (size_t i = 0; i < v.size(); ++i) { if (v[i]) vals[i] = *v[i]; else valid[i] = false; }
    auto bits = pack_bits(vals);
    return BooleanArray(Buffer::from_host(bits.data(), bits.size()), 0, (int64_t)v.size(), nulls_from_mask(valid));
  }
  DataType data_type() const override { return DataType::Boolean; }
  BooleanArray slice(int64_t offset, int64_t length) const {
    BooleanArray out(bits_, bit_offset_ + offset, length, nulls_);
    if (out.nulls_) { out.nulls_->offset += offset; out.nulls_->len = length; out.nulls_->null_count = -1; }
    return out;
  }
  std::vector<bool> values() const {
    std::vector<uint8_t> bits(acu_bitmap_bytes(bit_offset_ + len_) + 8);
    bits_.to_host(bits.data(), std::min(bits.size(), bits_.len()));
    std::vector<bool> v((size_t)len_);
    for (int64_t i = 0; i < len_; ++i) v[(size_t)i] = (bits[(size_t)((bit_offset_ + i) >> 3)] >> ((bit_offset_ + i) & 7)) & 1;
    return v;
  }
  bool value(int64_t i) const { return values()[(size_t)i]; }
  const Buffer &bits() const { return bits_; }
  std::vector<std::optional<bool>> to_vec() const {
    auto vals = values();
    auto valid = valid_mask();
    std::vector<std::optional<bool>> out((size_t)len_);
    for (size_t i = 0; i < out.size(); ++i) if (valid[i]) out[i] = (bool)vals[i];
    return out;
  }
  int64_t true_count() const {  // boolean_array.rs:175-187
    acu_array a = view();
    int64_t c = 0;
    acu_bitmap_count(Context::get().raw(), static_cast<const uint8_t *>(a.values), a.values_offset, a.validity, a.validity_offset, len_, &c);
    return c;
  }
 protected:
  const void *values_ptr() const override { return bits_.data(); }
  int64_t values_bit_offset() const override { return bit_offset_; }
 private:
  Buffer bits_;
  int64_t bit_offset_ = 0;
};

// GenericByteArray<Utf8> (arrow-array/src/array/byte_array.rs:87-92): i32 offsets + value bytes
class StringArray : public Array {
 public:
  StringArray() = default;
  StringArray(Buffer offsets, Buffer data, int64_t len, std::optional<NullBuffer> nulls)
      : offsets_(std::move(offsets)), data_(std::move(data)) { len_ = len; nulls_ = std::move(nulls); }
  static StringArray from(const std::vector<std::optional<std::string>> &v) {
    std::vector<int32_t> offs(v.size() + 1, 0);
    std::string bytes;
    std::vector<bool> valid(v.size(), true);
    for (size_t i = 0; i < v.size(); ++i) {
      if (v[i]) bytes += *v[i]; else valid[i] = false;
      offs[i + 1] = (int32_t)bytes.size();
    }
    return StringArray(Buffer::from_host(offs.data(), offs.size() * 4), Buffer::from_host(bytes.data(), bytes.size()),
                       (int64_t)v.size(), nulls_from_mask(valid));
  }
  static StringArray from(const std::vector<std::string> &v) {
    std::vector<std::optional<std::string>> o(v.begin(), v.end());
    return from(o);
  }
  DataType data_type() const override { return DataType::Utf8; }
  const Buffer &offsets() const { return offsets_; }
  const Buffer &value_data() const { return data_; }
  std::vector<std::optional<std::string>> to_vec() const {
    std::vector<int32_t> offs((size_t)len_ + 1);
    offsets_.to_host(offs.data(), offs.size() * 4);
    std::string bytes((size_t)offs.back(), '\0');
    data_.to_host(bytes.data(), bytes.size());
    auto valid = valid_mask();
    std::vector<std::optional<std::string>> out((size_t)len_);
    for (size_t i = 0; i < out.size(); ++i)
      if (valid[i]) out[i] = bytes.substr((size_t)offs[i], (size_t)(offs[i + 1] - offs[i]));
    return out;
  }
 protected:
  const void *values_ptr() const override { return nullptr; }
 private:
  Buffer offsets_, data_;
};

// GenericListArray<O> (arrow-array/src/array/list_array.rs): len + 1 offsets from logical row 0, ABSOLUTE rows of the child
// `values` (a slice keeps the whole child), and the nulls. ListArray = i32 offsets, LargeListArray = i64.
template <class O>
class GenericListArray : public Array {
 public:
  GenericListArray(Buffer offsets, ArrayRef values, int64_t len, std::optional<NullBuffer> nulls)
      : offsets_(std::move(offsets)), values_(std::move(values)) { len_ = len; nulls_ = std::move(nulls); }
  // GenericListArray::new(field, OffsetBuffer, values, nulls)
  static GenericListArray from(const std::vector<O> &offsets, ArrayRef values, const std::vector<bool> &valid = {}) {
    return GenericListArray(Buffer::from_host(offsets.data(), offsets.size() * sizeof(O)), std::move(values), (int64_t)offsets.size() - 1,
                            valid.empty() ? std::nullopt : nulls_from_mask(valid));
  }
  DataType data_type() const override { return sizeof(O) == 4 ? DataType::List : DataType::LargeList; }
  const Buffer &offsets() const { return offsets_; }
  const ArrayRef &values() const { return values_; }
  std::vector<O> value_offsets() const {
    std::vector<O> v((size_t)len_ + 1);
    offsets_.to_host(v.data(), v.size() * sizeof(O));
    return v;
  }
  GenericListArray slice(int64_t offset, int64_t length) const {  // Array::slice
    GenericListArray out(Buffer(), values_, length, nulls_);
    std::vector<O> o = value_offsets();
    out.offsets_ = Buffer::from_host(o.data() + offset, (size_t)(length + 1) * sizeof(O));
    if (out.nulls_) { out.nulls_->offset += offset; out.nulls_->len = length; out.nulls_->null_count = -1; }
    return out;
  }
 protected:
  const void *values_ptr() const override { return nullptr; }
 private:
  Buffer offsets_;
  ArrayRef values_;
};
using ListArray = GenericListArray<int32_t>;
using LargeListArray = GenericListArray<int64_t>;

// FixedSizeListArray (arrow-array/src/array/fixed_size_list_array.rs): row i is values rows [i * size, (i + 1) * size).
class FixedSizeListArray : public Array {
 public:
  FixedSizeListArray(int32_t size, ArrayRef values, int64_t len, std::optional<NullBuffer> nulls)
      : size_(size), values_(std::move(values)) { len_ = len; nulls_ = std::move(nulls); }
  // FixedSizeListArray::new(field, size, values, nulls)
  static FixedSizeListArray from(int32_t size, ArrayRef values, const std::vector<bool> &valid = {}) {
    const int64_t len = size ? values->len() / size : (int64_t)valid.size();
    return FixedSizeListArray(size, std::move(values), len, valid.empty() ? std::nullopt : nulls_from_mask(valid));
  }
  DataType data_type() const override { return DataType::FixedSizeList; }
  int32_t value_length() const { return size_; }
  const ArrayRef &values() const { return values_; }
 protected:
  const void *values_ptr() const override { return nullptr; }
 private:
  int32_t size_;
  ArrayRef values_;
};

// RunArray<R> (arrow-array/src/array/run_array.rs): the run ends (RunEndBuffer, arrow-buffer/src/buffer/run.rs) from
// physical entry 0, a logical window (offset, len) over them, and the values child, one row per physical run.
// Int16RunArray / Int32RunArray / Int64RunArray.
template <class R>
class RunArray : public Array {
 public:
  RunArray(Buffer run_ends, int64_t n_runs, ArrayRef values, int64_t offset, int64_t len)
      : run_ends_(std::move(run_ends)), n_runs_(n_runs), values_(std::move(values)), offset_(offset) { len_ = len; }
  // RunArray::try_new(run_ends, values): the logical length is the last run end
  static RunArray from(const std::vector<R> &run_ends, ArrayRef values) {
    return RunArray(Buffer::from_host(run_ends.data(), run_ends.size() * sizeof(R)), (int64_t)run_ends.size(), std::move(values), 0,
                    run_ends.empty() ? 0 : (int64_t)run_ends.back());
  }
  DataType data_type() const override { return DataType::RunEndEncoded; }
  // RunEndBuffer::values: every physical run end (not advanced by the offset)
  std::vector<R> run_ends() const {
    std::vector<R> v((size_t)n_runs_);
    run_ends_.to_host(v.data(), v.size() * sizeof(R));
    return v;
  }
  const Buffer &run_ends_buffer() const { return run_ends_; }
  int64_t num_runs() const { return n_runs_; }
  int64_t offset() const { return offset_; }
  const ArrayRef &values() const { return values_; }
  // RunArray::slice: only the logical window moves (RunEndBuffer::slice, run.rs:269-285)
  RunArray slice(int64_t offset, int64_t length) const {
    if (offset + length > len_) throw std::runtime_error("the length + offset of the sliced RunEndBuffer cannot exceed the existing length");
    return RunArray(run_ends_, n_runs_, values_, offset_ + offset, length);
  }
  // RunArray::get_physical_indices (run_array.rs:343-356, RunEndBuffer::get_physical_indices run.rs:321-378), on the host:
  // the run of every logical index, or the largest index when it is out of bounds
  template <class I>
  Result<std::vector<size_t>> get_physical_indices(const std::vector<I> &logical) const {
    std::vector<size_t> out(logical.size());
    if (logical.empty()) return out;
    const I mx = *std::max_element(logical.begin(), logical.end());
    if ((uint64_t)mx >= (uint64_t)len_)
      return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: Logical index " + std::to_string((uint64_t)mx) +
                                                      " is out of bounds for RunArray of length " + std::to_string(len_)};
    const std::vector<R> ends = run_ends();
    for (size_t j = 0; j < logical.size(); ++j)
      out[j] = (size_t)(std::upper_bound(ends.begin(), ends.end(), (int64_t)(offset_ + (int64_t)logical[j]),
                                         [](int64_t x, R e) { return x < (int64_t)e; }) - ends.begin());
    return out;
  }
  acu_run_array run_view() const {
    acu_run_array r{};
    r.run_end_dtype = sizeof(R) == 2 ? ACU_I16 : sizeof(R) == 4 ? ACU_I32 : ACU_I64;
    r.run_ends = run_ends_.data();
    r.n_runs = n_runs_;
    r.offset = offset_;
    r.len = len_;
    return r;
  }
 protected:
  const void *values_ptr() const override { return nullptr; }
 private:
  Buffer run_ends_;
  int64_t n_runs_;
  ArrayRef values_;
  int64_t offset_;
};
using Int16RunArray = RunArray<int16_t>;
using Int32RunArray = RunArray<int32_t>;
using Int64RunArray = RunArray<int64_t>;

// StructArray (arrow-array/src/array/struct_array.rs): columns of the struct's length from its logical row 0, and the
// nulls. Every field is nullable here.
// FixedSizeBinaryArray (arrow-array/src/array/fixed_size_binary_array.rs): `value_length` bytes per row, the rows from
// row `row_offset` of `values`.
class FixedSizeBinaryArray : public Array {
 public:
  FixedSizeBinaryArray(int32_t value_length, Buffer values, int64_t len, std::optional<NullBuffer> nulls, int64_t row_offset = 0)
      : value_length_(value_length), values_(std::move(values)), row_offset_(row_offset) {
    len_ = len;
    nulls_ = std::move(nulls);
  }
  // FixedSizeBinaryArray::try_new (:170-201): of width 0 the length comes from the NullBuffer (0 without one)
  static Result<FixedSizeBinaryArray> try_new(int32_t value_length, Buffer values, std::optional<NullBuffer> nulls) {
    if (value_length < 0)
      return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: Value length cannot be negative, got " + std::to_string(value_length)};
    int64_t len;
    if (value_length == 0) {
      if (values.len() != 0)
        return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: Buffer cannot have non-zero length if the value length is zero"};
      len = nulls ? nulls->len : 0;
    } else {
      len = (int64_t)values.len() / value_length;
      if (nulls && nulls->len != len)
        return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: Incorrect length of null buffer for FixedSizeBinaryArray, expected " +
                                                        std::to_string(len) + " got " + std::to_string(nulls->len)};
    }
    return FixedSizeBinaryArray(value_length, std::move(values), len, std::move(nulls));
  }
  // try_from_sparse_iter_with_size: a null row's bytes are zero
  static FixedSizeBinaryArray from(const std::vector<std::optional<std::vector<uint8_t>>> &rows, int32_t value_length) {
    std::vector<uint8_t> bytes(rows.size() * (size_t)value_length, 0);
    std::vector<bool> valid(rows.size(), true);
    for (size_t i = 0; i < rows.size(); ++i) {
      if (!rows[i]) { valid[i] = false; continue; }
      if (rows[i]->size() != (size_t)value_length) throw std::invalid_argument("FixedSizeBinaryArray::from: a row of the wrong width");
      std::copy(rows[i]->begin(), rows[i]->end(), bytes.begin() + i * value_length);
    }
    return FixedSizeBinaryArray(value_length, Buffer::from_host(bytes.data(), bytes.size()), (int64_t)rows.size(), nulls_from_mask(valid));
  }
  DataType data_type() const override { return DataType::FixedSizeBinary; }
  int32_t value_length() const { return value_length_; }
  std::vector<uint8_t> value(int64_t i) const {
    if (i < 0 || i >= len_) throw std::out_of_range("FixedSizeBinaryArray::value: index out of bounds");
    std::vector<uint8_t> v((size_t)value_length_);
    if (value_length_)
      acu_memcpy_d2h(Context::get().raw(), v.data(), static_cast<const uint8_t *>(values_ptr()) + (size_t)i * value_length_, v.size());
    return v;
  }
  // Array::slice: zero copy
  FixedSizeBinaryArray slice(int64_t offset, int64_t length) const {
    FixedSizeBinaryArray out(value_length_, values_, length, nulls_, row_offset_ + offset);
    if (out.nulls_) {
      out.nulls_->offset += offset;
      out.nulls_->len = length;
      out.nulls_->null_count = -1;  // recounted on device on first use
    }
    return out;
  }
  const Buffer &values() const { return values_; }
 protected:
  const void *values_ptr() const override { return static_cast<const uint8_t *>(values_.data()) + (size_t)row_offset_ * value_length_; }
 private:
  int32_t value_length_ = 0;
  Buffer values_;
  int64_t row_offset_ = 0;
};

class StructArray : public Array {
 public:
  StructArray(std::vector<ArrayRef> columns, int64_t len, std::optional<NullBuffer> nulls) : columns_(std::move(columns)) {
    len_ = len;
    nulls_ = std::move(nulls);
  }
  // StructArray::new(fields, arrays, nulls): try_new drops a NullBuffer without nulls
  static StructArray from(std::vector<ArrayRef> columns, const std::vector<bool> &valid = {}) {
    const int64_t len = columns.at(0)->len();
    return StructArray(std::move(columns), len, valid.empty() ? std::nullopt : nulls_from_mask(valid));
  }
  // StructArray::new_empty_fields(len, nulls): no columns, the NullBuffer kept as given
  static StructArray new_empty_fields(int64_t len, const std::vector<bool> &valid = {}) {
    return StructArray({}, len, valid.empty() ? std::nullopt : nulls_from_mask(valid, true));
  }
  DataType data_type() const override { return DataType::Struct; }
  const std::vector<ArrayRef> &columns() const { return columns_; }
  const ArrayRef &column(size_t i) const { return columns_.at(i); }
  size_t num_columns() const { return columns_.size(); }
 protected:
  const void *values_ptr() const override { return nullptr; }
 private:
  std::vector<ArrayRef> columns_;
};

// UnionArray (arrow-array/src/array/union_array.rs): the fields' type ids in field order, one Int8 type id per row and, for
// a dense union, one Int32 offset per row into the row's child. A sparse union's children have the union's length. A union
// has no NullBuffer.
class UnionArray : public Array {
 public:
  UnionArray(std::vector<int8_t> field_type_ids, Buffer type_ids, std::optional<Buffer> offsets, std::vector<ArrayRef> children, int64_t len)
      : field_type_ids_(std::move(field_type_ids)), type_ids_(std::move(type_ids)), offsets_(std::move(offsets)), children_(std::move(children)) {
    len_ = len;
  }
  // UnionArray::try_new (union_array.rs:177-242)
  static Result<UnionArray> try_new(std::vector<int8_t> field_type_ids, const std::vector<int8_t> &type_ids,
                                    std::optional<std::vector<int32_t>> offsets, std::vector<ArrayRef> children) {
    auto fail = [](const char *m) { return ArrowError{ACU_ERR_INVALID_ARGUMENT, std::string("Invalid argument error: ") + m}; };
    if (field_type_ids.size() != children.size()) return fail("Union fields length must match child arrays length");
    if (offsets && offsets->size() != type_ids.size()) return fail("Type Ids and Offsets lengths must match");
    if (!offsets)
      for (const auto &c : children)
        if (c->len() != (int64_t)type_ids.size()) return fail("Sparse union child arrays must be equal in length to the length of the union");
    std::map<int, int64_t> lens;
    for (size_t f = 0; f < field_type_ids.size(); ++f) lens[field_type_ids[f]] = children[f]->len();
    for (int8_t t : type_ids)
      if (!lens.count(t)) return fail("Type Ids values must match one of the field type ids");
    if (offsets)
      for (size_t i = 0; i < type_ids.size(); ++i)
        if ((*offsets)[i] < 0 || (*offsets)[i] >= lens[type_ids[i]]) return fail("Offsets must be non-negative and within the length of the Array");
    std::optional<Buffer> ob;
    if (offsets) ob = Buffer::from_host(offsets->data(), offsets->size() * 4);
    return UnionArray(std::move(field_type_ids), Buffer::from_host(type_ids.data(), type_ids.size()), std::move(ob), std::move(children),
                      (int64_t)type_ids.size());
  }
  DataType data_type() const override { return DataType::Union; }
  bool is_dense() const { return offsets_.has_value(); }
  const std::vector<int8_t> &field_type_ids() const { return field_type_ids_; }
  const std::vector<ArrayRef> &children() const { return children_; }
  const ArrayRef &child(int8_t type_id) const {
    for (size_t f = 0; f < field_type_ids_.size(); ++f)
      if (field_type_ids_[f] == type_id) return children_[f];
    throw std::runtime_error("invalid union type id");
  }
  const Buffer &type_ids_buffer() const { return type_ids_; }
  const std::optional<Buffer> &offsets_buffer() const { return offsets_; }
  std::vector<int8_t> type_ids() const {
    std::vector<int8_t> v((size_t)len_);
    type_ids_.to_host(v.data(), v.size());
    return v;
  }
  std::vector<int32_t> value_offsets() const {
    std::vector<int32_t> v(offsets_ ? (size_t)len_ : 0);
    if (offsets_) offsets_->to_host(v.data(), v.size() * 4);
    return v;
  }
  acu_union_array union_view() const {
    acu_union_array u{};
    u.mode = offsets_ ? ACU_UNION_DENSE : ACU_UNION_SPARSE;
    u.n_fields = (int32_t)field_type_ids_.size();
    u.field_type_ids = field_type_ids_.data();
    u.type_ids = static_cast<const int8_t *>(type_ids_.data());
    u.offsets = offsets_ ? static_cast<const int32_t *>(offsets_->data()) : nullptr;
    u.len = len_;
    return u;
  }
 protected:
  const void *values_ptr() const override { return nullptr; }
 private:
  std::vector<int8_t> field_type_ids_;
  Buffer type_ids_;
  std::optional<Buffer> offsets_;
  std::vector<ArrayRef> children_;
};

// Datum (arrow-array/src/scalar.rs:78-152): an array, or a Scalar wrapping a 1-element array
template <class A>
struct Scalar {
  A array;
  explicit Scalar(A a) : array(std::move(a)) {}
};
template <class T> Scalar<PrimitiveArray<T>> new_scalar(T v) { return Scalar<PrimitiveArray<T>>(PrimitiveArray<T>::from(std::vector<T>{v})); }
template <class T> Scalar<PrimitiveArray<T>> new_null_scalar() { return Scalar<PrimitiveArray<T>>(PrimitiveArray<T>::new_null(1)); }

template <class A> const A &datum_array(const A &a) { return a; }
template <class A> const A &datum_array(const Scalar<A> &s) { return s.array; }
template <class A> bool datum_is_scalar(const A &) { return false; }
template <class A> bool datum_is_scalar(const Scalar<A> &) { return true; }

// ---------------------------------------------------------------------------------------
// RecordBatch (arrow-array/src/record_batch.rs:224-232)
// ---------------------------------------------------------------------------------------
struct Field { std::string name; DataType data_type; bool nullable = true; };
using Schema = std::vector<Field>;

class RecordBatch {
 public:
  static Result<RecordBatch> try_new(Schema schema, std::vector<ArrayRef> columns) {
    if (schema.size() != columns.size())
      return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: number of columns(" + std::to_string(columns.size()) +
                                                       ") must match number of fields(" + std::to_string(schema.size()) + ") in schema"};
    int64_t rows = columns.empty() ? 0 : columns[0]->len();
    for (auto &c : columns)
      if (c->len() != rows) return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: all columns in a record batch must have the same length"};
    return RecordBatch(std::move(schema), std::move(columns), rows);
  }
  RecordBatch(Schema schema, std::vector<ArrayRef> columns, int64_t rows)
      : schema_(std::move(schema)), columns_(std::move(columns)), rows_(rows) {}
  const Schema &schema() const { return schema_; }
  const std::vector<ArrayRef> &columns() const { return columns_; }
  const ArrayRef &column(size_t i) const { return columns_[i]; }
  int64_t num_rows() const { return rows_; }
  size_t num_columns() const { return columns_.size(); }
 private:
  Schema schema_;
  std::vector<ArrayRef> columns_;
  int64_t rows_ = 0;
};

// ---------------------------------------------------------------------------------------
// compute
// ---------------------------------------------------------------------------------------
namespace compute {
namespace detail {

// DataType Display of an operand (decimals carry their precision and scale)
template <class A> std::string type_text(const A &a);

inline acu_array_out make_out(Buffer &values, Buffer &validity, size_t value_bytes, int64_t rows) {
  values = Buffer::allocate(value_bytes);
  validity = Buffer::allocate(acu_bitmap_bytes(rows));
  acu_array_out o{};
  o.values = values.data();
  o.validity = static_cast<uint8_t *>(validity.data());
  return o;
}
// drop_empty_nulls: MutableArrayData::freeze keeps a NullBuffer only if it has a null (arrow-data/src/transform/mod.rs:936)
inline std::optional<NullBuffer> out_nulls(const acu_array_out &o, Buffer validity, bool drop_empty_nulls = false) {
  if (!o.has_validity || (drop_empty_nulls && o.null_count == 0)) return std::nullopt;
  return NullBuffer{std::move(validity), 0, o.len, o.null_count};
}

template <class T>
ArrayRef wrap_primitive(DataType dt, Buffer values, int64_t len, std::optional<NullBuffer> nulls) {
  (void)dt;
  return std::make_shared<PrimitiveArray<T>>(std::move(values), len, std::move(nulls));
}
inline ArrayRef make_primitive(DataType dt, Buffer values, int64_t len, std::optional<NullBuffer> nulls) {
  switch (dt) {
    case DataType::Int8: return wrap_primitive<int8_t>(dt, std::move(values), len, std::move(nulls));
    case DataType::Int16: return wrap_primitive<int16_t>(dt, std::move(values), len, std::move(nulls));
    case DataType::Int32: return wrap_primitive<int32_t>(dt, std::move(values), len, std::move(nulls));
    case DataType::Int64: return wrap_primitive<int64_t>(dt, std::move(values), len, std::move(nulls));
    case DataType::UInt8: return wrap_primitive<uint8_t>(dt, std::move(values), len, std::move(nulls));
    case DataType::UInt16: return wrap_primitive<uint16_t>(dt, std::move(values), len, std::move(nulls));
    case DataType::UInt32: return wrap_primitive<uint32_t>(dt, std::move(values), len, std::move(nulls));
    case DataType::UInt64: return wrap_primitive<uint64_t>(dt, std::move(values), len, std::move(nulls));
    case DataType::Float32: return wrap_primitive<float>(dt, std::move(values), len, std::move(nulls));
    default: return wrap_primitive<double>(dt, std::move(values), len, std::move(nulls));
  }
}
inline const char *dtype_display(DataType t) {
  static const char *n[] = {"Int8", "Int16", "Int32", "Int64", "UInt8", "UInt16", "UInt32", "UInt64", "Float32", "Float64", "Boolean", "Utf8",
                            "Decimal32", "Decimal64", "Decimal128", "List", "LargeList", "FixedSizeList", "RunEndEncoded", "Struct", "Union", "FixedSizeBinary"};
  return n[(int)t];
}
template <class A> std::string type_text(const A &a) {
  if constexpr (is_decimal_array<A>::value) return a.type_display();
  else return dtype_display(a.data_type());
}
// One acu_column per column of a RecordBatch (include/arrow_cuda.h: acu_column)
inline acu_column column_view(const Array &a) {
  acu_column c{};
  c.array = a.view();
  if (a.data_type() == DataType::Boolean) {
    c.kind = ACU_COL_BOOLEAN;
  } else if (a.data_type() == DataType::Utf8) {
    const auto &s = static_cast<const StringArray &>(a);
    c.kind = ACU_COL_BYTES;
    c.width = 4;
    c.array.values = s.offsets().data();
    c.array.values_offset = 0;
    c.data = static_cast<const uint8_t *>(s.value_data().data());
  } else if (a.data_type() == DataType::FixedSizeBinary) {
    c.kind = ACU_COL_FIXED_SIZE_BINARY;
    c.width = static_cast<const FixedSizeBinaryArray &>(a).value_length();
  } else {
    c.kind = ACU_COL_PRIMITIVE;
    c.width = dtype_width(a.data_type());
  }
  return c;
}

// Output buffers of a record-batch call: values / offsets, validity and (Utf8) value bytes per column.
struct BatchOutputs {
  std::vector<Buffer> values, validity, data;
  std::vector<acu_column_out> outs;
  void allocate(const std::vector<ArrayRef> &cols, int64_t rows, const std::vector<int64_t> &data_caps) {
    const size_t n = cols.size();
    values.resize(n);
    validity.resize(n);
    data.resize(n);
    outs.assign(n, acu_column_out{});
    for (size_t i = 0; i < n; ++i) {
      const DataType dt = cols[i]->data_type();
      const size_t w = dt == DataType::FixedSizeBinary ? (size_t) static_cast<const FixedSizeBinaryArray &>(*cols[i]).value_length() : dtype_width(dt);
      const size_t vbytes = dt == DataType::Boolean ? acu_bitmap_bytes(rows) : dt == DataType::Utf8 ? (size_t)(rows + 1) * 4 : (size_t)rows * w;
      values[i] = Buffer::allocate(vbytes);
      validity[i] = Buffer::allocate(acu_bitmap_bytes(rows));
      outs[i].array.values = values[i].data();
      outs[i].array.validity = static_cast<uint8_t *>(validity[i].data());
      if (dt == DataType::Utf8 && data_caps[i] >= 0) {
        data[i] = Buffer::allocate((size_t)data_caps[i]);
        outs[i].data = static_cast<uint8_t *>(data[i].data());
        outs[i].data_capacity = data_caps[i];
      }
    }
  }
  std::vector<ArrayRef> wrap(const std::vector<ArrayRef> &cols) {
    std::vector<ArrayRef> res;
    for (size_t i = 0; i < cols.size(); ++i) {
      const DataType dt = cols[i]->data_type();
      const acu_array_out &o = outs[i].array;
      if (dt == DataType::Boolean) res.push_back(std::make_shared<BooleanArray>(values[i], 0, o.len, out_nulls(o, validity[i])));
      else if (dt == DataType::Utf8) res.push_back(std::make_shared<StringArray>(values[i], data[i], o.len, out_nulls(o, validity[i])));
      else if (dt == DataType::FixedSizeBinary)
        res.push_back(std::make_shared<FixedSizeBinaryArray>(static_cast<const FixedSizeBinaryArray &>(*cols[i]).value_length(), values[i], o.len,
                                                             out_nulls(o, validity[i])));
      else res.push_back(make_primitive(dt, values[i], o.len, out_nulls(o, validity[i])));
    }
    return res;
  }
};
}  // namespace detail

// ---- filter (arrow-select/src/filter.rs) ------------------------------------------------
// FilterPredicate (filter.rs:442-533): owns the device-resident plan, reusable across columns.
class FilterPredicate {
 public:
  FilterPredicate() = default;
  explicit FilterPredicate(acu_filter_plan *p) : plan_(p, [](acu_filter_plan *q) { acu_filter_plan_destroy(Context::get().raw(), q); }) {}
  // acu_filter_plan_create of a predicate (FilterBuilder::new(filter).build())
  static Result<FilterPredicate> try_new(const BooleanArray &filter) {
    Context &c = Context::get();
    acu_array p = filter.view();
    acu_filter_plan *plan = nullptr;
    acu_status st = acu_filter_plan_create(c.raw(), &p, &plan);
    if (st != ACU_OK) return c.last_error(st);
    return FilterPredicate(plan);
  }
  acu_filter_plan *raw() const { return plan_.get(); }
  int64_t count() const { return acu_filter_plan_count(plan_.get()); }
  // IterationStrategy::Slices of FilterBuilder::optimize = SlicesIterator::new(&filter).collect() (filter.rs:44-77,285-298):
  // the runs of selected rows as [start, end), computed on the device
  Result<std::vector<std::pair<size_t, size_t>>> slices() const {
    Context &c = Context::get();
    int64_t n = 0;
    acu_status st = acu_filter_plan_slices(c.raw(), plan_.get(), nullptr, 0, &n);
    if (st != ACU_OK) return c.last_error(st);
    std::vector<std::pair<size_t, size_t>> out((size_t)n);
    if (n == 0) return out;
    Buffer pairs = Buffer::allocate((size_t)n * 16);
    if ((st = acu_filter_plan_slices(c.raw(), plan_.get(), static_cast<uint64_t *>(pairs.data()), n, &n)) != ACU_OK) return c.last_error(st);
    std::vector<uint64_t> host((size_t)n * 2);
    pairs.to_host(host.data(), host.size() * 8);
    for (int64_t k = 0; k < n; ++k) out[(size_t)k] = {(size_t)host[2 * k], (size_t)host[2 * k + 1]};
    return out;
  }
  // FilterPredicate::filter (filter.rs:480-483): any array, at any nesting
  Result<ArrayRef> filter(const Array &values) const;
  // FilterPredicate::filter_record_batch (filter.rs:459-478): one plan, every column, ONE synchronisation
  // (acu_filter_record_batch queues the kernels of all columns back to back).
  Result<RecordBatch> filter_record_batch(const RecordBatch &batch) const {
    Context &c = Context::get();
    const auto &cols = batch.columns();
    if (cols.empty()) return RecordBatch(batch.schema(), {}, count());
    std::vector<acu_column> in;
    std::vector<int64_t> caps;
    for (const auto &col : cols) {
      in.push_back(detail::column_view(*col));
      // a filtered Utf8 column never holds more bytes than its source
      caps.push_back(col->data_type() == DataType::Utf8 ? (int64_t) static_cast<const StringArray &>(*col).value_data().len() : -1);
    }
    detail::BatchOutputs out;
    out.allocate(cols, count(), caps);
    std::vector<ArrayRef> res;
    for (size_t first = 0; first < cols.size(); first += ACU_MAX_BATCH_COLUMNS) {
      const int32_t n = (int32_t)std::min<size_t>(ACU_MAX_BATCH_COLUMNS, cols.size() - first);
      acu_status st = acu_filter_record_batch(c.raw(), plan_.get(), n, in.data() + first, out.outs.data() + first);
      if (st != ACU_OK) return c.last_error(st);
    }
    return RecordBatch(batch.schema(), out.wrap(cols), count());
  }
 private:
  std::shared_ptr<acu_filter_plan> plan_;
};

class FilterBuilder {  // filter.rs:254-324
 public:
  explicit FilterBuilder(const BooleanArray &filter) {
    auto p = FilterPredicate::try_new(filter);
    if (p.is_err()) throw std::runtime_error(p.unwrap_err().message);
    pred_ = p.unwrap();
  }
  FilterBuilder &optimize() { return *this; }  // the device plan is always materialised
  FilterPredicate build() { return pred_; }
  // FilterBuilder::new(&cmp::OP(l, r)?).build() with the comparison fused into the plan pass: the BooleanArray is never
  // materialised (acu_filter_plan_create_cmp). l / r: PrimitiveArray<T> or Scalar<PrimitiveArray<T>> of one type.
  template <class L, class R>
  static Result<FilterPredicate> from_cmp(acu_cmp_op op, const L &lhs, const R &rhs) {
    const auto &l = datum_array(lhs);
    const auto &r = datum_array(rhs);
    if (l.data_type() != r.data_type() || dtype_width(l.data_type()) == 0)
      return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: Invalid comparison operation"};
    acu_array a = l.view(datum_is_scalar(lhs)), b = r.view(datum_is_scalar(rhs));
    acu_filter_plan *plan = nullptr;
    Context &c = Context::get();
    acu_status st = acu_filter_plan_create_cmp(c.raw(), (acu_dtype)dtype_code(l.data_type()), op, &a, &b, &plan);
    if (st != ACU_OK) return c.last_error(st);
    return FilterPredicate(plan);
  }
 private:
  FilterPredicate pred_;
};

// ---- take (arrow-select/src/take.rs) ----------------------------------------------------
struct TakeOptions { bool check_bounds = false; };  // take.rs:388-394

// ---- filter / take of every array type (filter.rs:174-199, take.rs:89-105) ------------------------------------------
// filter_any / take_any have one arm per DataType. A nested array makes one C call per level, which returns the plan or
// row map of the level below, and each child goes through the arm of its own type:
// - List / LargeList / FixedSizeList (filter.rs:535-625, take.rs:646-795): acu_filter_list / acu_take_list. A List's child
//   is extended (MutableArrayData: a Utf8 child keeps the bytes under its null rows, acu_take_bytes_extend); a
//   FixedSizeList's child is taken. Not reproduced here: when a List's i32 offsets and its child's both overflow, this
//   mirror reports the List's unwrap panic (the Python layer reports the child's error first, as the reference does).
// - Struct, sparse Union and dense Union (filter.rs:597-622, :1010-1054, take.rs:270-298, :334-382): a struct's columns,
//   then acu_filter_nulls / acu_take_nulls for its NullBuffer. acu_filter_union / acu_take_union give a union's type ids
//   and, for a dense union, its new offsets and a child row map grouped by field; child f is then taken (take) or extended
//   (filter, the child step of a list take) with its slice of the map.
// - RunEndEncoded (filter_run_end_array filter.rs:628-677, take_run take.rs:948-995), at the top level only:
//   acu_filter_run_end / acu_take_run_end write the new run ends and return the values child's plan / value indices.
//   Values: primitive, Boolean and Utf8 (and lists, filter only). As in the Python layer, a RunEndEncoded array below
//   another level is refused (MutableArrayData does not extend one).
namespace detail {
// take.rs:103: the indices must be integers
inline std::optional<ArrowError> index_type_error(DataType it) {
  if ((int)it <= (int)DataType::UInt64) return std::nullopt;
  return ArrowError{ACU_ERR_INVALID_ARGUMENT, std::string("Invalid argument error: Take only supported for integers, got ") + dtype_display(it)};
}
// an output of `rows` rows that receives a validity bitmap only
inline acu_array_out validity_out(Buffer &validity, int64_t rows) {
  validity = Buffer::allocate(acu_bitmap_bytes(rows));
  acu_array_out o{};
  o.validity = static_cast<uint8_t *>(validity.data());
  return o;
}
// A Utf8 output of `rows` rows in two calls of `call(offsets, data, capacity, &total, &out)`: the first (no data buffer)
// sizes the value bytes, the second writes them.
template <class F>
Result<ArrayRef> bytes_out(int64_t rows, bool drop_empty_nulls, F call) {
  Context &c = Context::get();
  Buffer offs = Buffer::allocate((size_t)(rows + 1) * 4), nb;
  acu_array_out o = validity_out(nb, rows);
  int64_t total = 0;
  acu_status st = call(offs.data(), nullptr, 0, &total, &o);
  if (st != ACU_OK) return c.last_error(st);
  Buffer data = Buffer::allocate((size_t)total);
  if ((st = call(offs.data(), static_cast<uint8_t *>(data.data()), total, &total, &o)) != ACU_OK) return c.last_error(st);
  return ArrayRef(std::make_shared<StringArray>(offs, data, o.len, out_nulls(o, nb, drop_empty_nulls)));
}

inline acu_list_array list_view(const Array &a) {
  acu_list_array l{};
  l.nulls = a.view();
  l.nulls.values = nullptr;
  if (a.data_type() == DataType::FixedSizeList) {
    const auto &f = static_cast<const FixedSizeListArray &>(a);
    l.kind = ACU_FIXED_SIZE_LIST;
    l.list_size = f.value_length();
    l.child_len = f.values()->len();
  } else if (a.data_type() == DataType::List) {
    const auto &g = static_cast<const ListArray &>(a);
    l.kind = ACU_LIST;
    l.offsets = g.offsets().data();
    l.child_len = g.values()->len();
  } else {
    const auto &g = static_cast<const LargeListArray &>(a);
    l.kind = ACU_LARGE_LIST;
    l.offsets = g.offsets().data();
    l.child_len = g.values()->len();
  }
  return l;
}
inline const ArrayRef &list_values(const Array &a) {
  if (a.data_type() == DataType::FixedSizeList) return static_cast<const FixedSizeListArray &>(a).values();
  if (a.data_type() == DataType::List) return static_cast<const ListArray &>(a).values();
  return static_cast<const LargeListArray &>(a).values();
}
inline ArrayRef list_like(const Array &a, Buffer offsets, ArrayRef child, int64_t len, std::optional<NullBuffer> nulls) {
  if (a.data_type() == DataType::FixedSizeList)
    return std::make_shared<FixedSizeListArray>(static_cast<const FixedSizeListArray &>(a).value_length(), std::move(child), len, std::move(nulls));
  if (a.data_type() == DataType::List) return std::make_shared<ListArray>(std::move(offsets), std::move(child), len, std::move(nulls));
  return std::make_shared<LargeListArray>(std::move(offsets), std::move(child), len, std::move(nulls));
}

template <class T> ArrayRef slice_prim(const Array &a, int64_t off, int64_t len) {
  return std::make_shared<PrimitiveArray<T>>(static_cast<const PrimitiveArray<T> &>(a).slice(off, len));
}
// Array::slice of the RunArray value types
inline ArrayRef slice_any(const Array &a, int64_t off, int64_t len) {
  std::optional<NullBuffer> nulls = a.nulls();
  if (nulls) { nulls->offset += off; nulls->len = len; nulls->null_count = -1; }
  switch (a.data_type()) {
    case DataType::Int8: return slice_prim<int8_t>(a, off, len);
    case DataType::Int16: return slice_prim<int16_t>(a, off, len);
    case DataType::Int32: return slice_prim<int32_t>(a, off, len);
    case DataType::Int64: return slice_prim<int64_t>(a, off, len);
    case DataType::UInt8: return slice_prim<uint8_t>(a, off, len);
    case DataType::UInt16: return slice_prim<uint16_t>(a, off, len);
    case DataType::UInt32: return slice_prim<uint32_t>(a, off, len);
    case DataType::UInt64: return slice_prim<uint64_t>(a, off, len);
    case DataType::Float32: return slice_prim<float>(a, off, len);
    case DataType::Float64: return slice_prim<double>(a, off, len);
    case DataType::Boolean: return std::make_shared<BooleanArray>(static_cast<const BooleanArray &>(a).slice(off, len));
    case DataType::List: return std::make_shared<ListArray>(static_cast<const ListArray &>(a).slice(off, len));
    case DataType::LargeList: return std::make_shared<LargeListArray>(static_cast<const LargeListArray &>(a).slice(off, len));
    case DataType::FixedSizeList: {
      const auto &f = static_cast<const FixedSizeListArray &>(a);
      return std::make_shared<FixedSizeListArray>(f.value_length(), slice_any(*f.values(), off * f.value_length(), len * f.value_length()), len,
                                                  nulls);
    }
    case DataType::Utf8: {  // the offsets from the new row 0; the value bytes are shared
      const auto &s = static_cast<const StringArray &>(a);
      std::vector<int32_t> o((size_t)a.len() + 1);
      s.offsets().to_host(o.data(), o.size() * 4);
      return std::make_shared<StringArray>(Buffer::from_host(o.data() + off, (size_t)(len + 1) * 4), s.value_data(), len, nulls);
    }
    case DataType::FixedSizeBinary:
      return std::make_shared<FixedSizeBinaryArray>(static_cast<const FixedSizeBinaryArray &>(a).slice(off, len));
    case DataType::Struct: {
      std::vector<ArrayRef> cols;
      for (const auto &col : static_cast<const StructArray &>(a).columns()) cols.push_back(slice_any(*col, off, len));
      return std::make_shared<StructArray>(std::move(cols), len, nulls);
    }
    default: throw std::runtime_error(std::string("RunArray values of type ") + dtype_display(a.data_type()) + " are not supported by this mirror");
  }
}
template <class T> ArrayRef empty_prim() { return std::make_shared<PrimitiveArray<T>>(PrimitiveArray<T>::from(std::vector<T>{})); }
// new_empty_array: no rows and no NullBuffer
inline ArrayRef empty_like(const Array &a) {
  switch (a.data_type()) {
    case DataType::Int8: return empty_prim<int8_t>();
    case DataType::Int16: return empty_prim<int16_t>();
    case DataType::Int32: return empty_prim<int32_t>();
    case DataType::Int64: return empty_prim<int64_t>();
    case DataType::UInt8: return empty_prim<uint8_t>();
    case DataType::UInt16: return empty_prim<uint16_t>();
    case DataType::UInt32: return empty_prim<uint32_t>();
    case DataType::UInt64: return empty_prim<uint64_t>();
    case DataType::Float32: return empty_prim<float>();
    case DataType::Float64: return empty_prim<double>();
    case DataType::Boolean: return std::make_shared<BooleanArray>(BooleanArray::from(std::vector<bool>{}));
    case DataType::Utf8: return std::make_shared<StringArray>(StringArray::from(std::vector<std::string>{}));
    case DataType::List: return std::make_shared<ListArray>(ListArray::from({0}, empty_like(*list_values(a))));
    case DataType::LargeList: return std::make_shared<LargeListArray>(LargeListArray::from({0}, empty_like(*list_values(a))));
    case DataType::FixedSizeList:
      return std::make_shared<FixedSizeListArray>(static_cast<const FixedSizeListArray &>(a).value_length(), empty_like(*list_values(a)), 0,
                                                  std::nullopt);
    case DataType::FixedSizeBinary:
      return std::make_shared<FixedSizeBinaryArray>(static_cast<const FixedSizeBinaryArray &>(a).value_length(), Buffer::allocate(0), 0, std::nullopt);
    default: throw std::runtime_error(std::string("RunArray values of type ") + dtype_display(a.data_type()) + " are not supported by this mirror");
  }
}
// f(run) with the RunArray<R> behind a RunEndEncoded array
template <class F>
Result<ArrayRef> with_run_array(const Array &a, F f) {
  if (const auto *r = dynamic_cast<const RunArray<int16_t> *>(&a)) return f(*r);
  if (const auto *r = dynamic_cast<const RunArray<int32_t> *>(&a)) return f(*r);
  return f(dynamic_cast<const RunArray<int64_t> &>(a));
}

inline acu_array nulls_view(const Array &a) {
  acu_array v = a.view();
  v.values = nullptr;
  return v;
}
inline ArrayRef i32_slice(const Buffer &map, int64_t start, int64_t len) {
  return std::make_shared<PrimitiveArray<int32_t>>(map, len, std::nullopt, start);
}
// the first `len` rows of a union: the type ids (and offsets) move, a dense union keeps its children whole, a sparse one
// slices them
inline ArrayRef union_head(const UnionArray &u, int64_t len) {
  std::vector<int8_t> t = u.type_ids();
  std::optional<Buffer> ob;
  std::vector<ArrayRef> children = u.children();
  if (u.is_dense()) {
    std::vector<int32_t> o = u.value_offsets();
    ob = Buffer::from_host(o.data(), (size_t)len * 4);
  } else {
    for (auto &c : children) c = slice_any(*c, 0, len);
  }
  return std::make_shared<UnionArray>(u.field_type_ids(), Buffer::from_host(t.data(), (size_t)len), std::move(ob), std::move(children), len);
}

// keep: `values` is the child step of a List take (MutableArrayData::extend: every row keeps its range or bytes).
inline Result<ArrayRef> take_any(const Array &values, const Array &indices, int cb, bool keep);

// child_step: `values` is a child of a list whose top level was filtered with a plan other than All (nullopt at the top).
// The reference builds those levels with MutableArrayData (filter.rs:600), which drops a NullBuffer without nulls even
// where the level's own plan selects every row; under a top-level All it slices every level as it is.
inline Result<ArrayRef> filter_any(const Array &values, const FilterPredicate &pred, std::optional<bool> child_step = std::nullopt) {
  Context &c = Context::get();
  acu_filter_plan *plan = pred.raw();
  const int64_t n = pred.count();
  const bool step = child_step.value_or(false);
  const acu_array v = values.view();
  Buffer vb, nb;
  acu_status st;
  switch (values.data_type()) {
    case DataType::Boolean: {
      acu_array_out o = make_out(vb, nb, acu_bitmap_bytes(n), n);
      if ((st = acu_filter_boolean(c.raw(), plan, &v, &o)) != ACU_OK) return c.last_error(st);
      return ArrayRef(std::make_shared<BooleanArray>(vb, 0, o.len, out_nulls(o, nb, step)));
    }
    case DataType::Utf8: {
      const auto &s = static_cast<const StringArray &>(values);
      return bytes_out(n, step, [&](void *offs, uint8_t *data, int64_t cap, int64_t *total, acu_array_out *o) {
        return acu_filter_bytes(c.raw(), plan, 4, s.offsets().data(), static_cast<const uint8_t *>(s.value_data().data()), &v, offs, data, cap,
                                total, o);
      });
    }
    case DataType::FixedSizeBinary: {  // filter_fixed_size_binary (filter.rs:946-996)
      const int32_t w = static_cast<const FixedSizeBinaryArray &>(values).value_length();
      acu_array_out o = make_out(vb, nb, (size_t)n * w, n);
      if ((st = acu_filter_fixed_size_binary(c.raw(), plan, w, &v, &o)) != ACU_OK) return c.last_error(st);
      // MutableArrayData keeps every extended row of a FixedSizeBinary(0) child (try_new's length rule is the top level's)
      return ArrayRef(std::make_shared<FixedSizeBinaryArray>(w, vb, step ? n : o.len, out_nulls(o, nb, step)));
    }
    case DataType::List: case DataType::LargeList: case DataType::FixedSizeList: {
      const acu_list_array l = list_view(values);
      Buffer offs = Buffer::allocate((size_t)(n + 1) * (l.kind == ACU_LIST ? 4 : 8));
      acu_array_out o = validity_out(nb, n);
      acu_filter_plan *child_plan = nullptr;
      if ((st = acu_filter_list(c.raw(), plan, &l, offs.data(), &o, &child_plan)) != ACU_OK) return c.last_error(st);
      const FilterPredicate cp(child_plan);
      auto child = filter_any(*list_values(values), cp, child_step ? *child_step : n != acu_filter_plan_len(plan));
      if (child.is_err()) return child.unwrap_err();
      return list_like(values, offs, child.unwrap(), o.len, out_nulls(o, nb, step));
    }
    case DataType::Struct: {  // filter_struct: every column, then filter_nulls
      std::vector<ArrayRef> cols;
      for (const auto &col : static_cast<const StructArray &>(values).columns()) {
        auto r = filter_any(*col, pred, child_step);
        if (r.is_err()) return r.unwrap_err();
        cols.push_back(r.unwrap());
      }
      const acu_array nv = nulls_view(values);
      acu_array_out o = validity_out(nb, n);
      if ((st = acu_filter_nulls(c.raw(), plan, &nv, &o)) != ACU_OK) return c.last_error(st);
      return ArrayRef(std::make_shared<StructArray>(std::move(cols), n, out_nulls(o, nb, step)));
    }
    case DataType::Union: {
      const auto &u = static_cast<const UnionArray &>(values);
      const int32_t strategy = acu_filter_plan_strategy(plan);
      if (u.is_dense() && step && strategy == ACU_FILTER_ALL) {
        // a list's child step extends every row even when its plan selects them all: the rows of a take of 0 .. n
        std::vector<uint64_t> ids((size_t)n);
        for (int64_t i = 0; i < n; ++i) ids[(size_t)i] = (uint64_t)i;
        return take_any(values, PrimitiveArray<uint64_t>::from(ids), 0, true);
      }
      const acu_union_array uv = u.union_view();
      const size_t nf = u.field_type_ids().size();
      Buffer tids = Buffer::allocate((size_t)n), offs = Buffer::allocate((size_t)n * 4), map = Buffer::allocate((size_t)n * 4);
      std::vector<int64_t> starts(nf + 1, 0);
      if ((st = acu_filter_union(c.raw(), plan, &uv, static_cast<int8_t *>(tids.data()), static_cast<int32_t *>(offs.data()),
                                 static_cast<int32_t *>(map.data()), starts.data())) != ACU_OK)
        return c.last_error(st);
      std::vector<ArrayRef> children;
      if (u.is_dense()) {
        if (strategy == ACU_FILTER_ALL) return union_head(u, n);  // values.slice(0, count)
        for (size_t f = 0; f < nf; ++f) {  // build_extend_dense: each child extended row by row
          auto r = take_any(*u.children()[f], *i32_slice(map, starts[f], starts[f + 1] - starts[f]), 0, true);
          if (r.is_err()) return r.unwrap_err();
          children.push_back(r.unwrap());
        }
        return ArrayRef(std::make_shared<UnionArray>(u.field_type_ids(), tids, offs, std::move(children), n));
      }
      for (const auto &ch : u.children()) {
        auto r = filter_any(*ch, pred, child_step);
        if (r.is_err()) return r.unwrap_err();
        children.push_back(r.unwrap());
      }
      if (strategy == ACU_FILTER_NONE || strategy == ACU_FILTER_ALL) {
        std::vector<int8_t> t = u.type_ids();
        tids = Buffer::from_host(t.data(), (size_t)n);
      }
      return ArrayRef(std::make_shared<UnionArray>(u.field_type_ids(), tids, std::nullopt, std::move(children), n));
    }
    case DataType::RunEndEncoded:
      return ArrowError{ACU_ERR_NOT_YET_IMPLEMENTED, "Not yet implemented: filter of a RunEndEncoded array below the top level"};
    default: {
      const int w = dtype_width(values.data_type());
      acu_array_out o = make_out(vb, nb, (size_t)n * w, n);
      if ((st = acu_filter_primitive(c.raw(), plan, w, &v, &o)) != ACU_OK) return c.last_error(st);
      return make_primitive(values.data_type(), vb, o.len, out_nulls(o, nb, step));
    }
  }
}

inline Result<ArrayRef> take_any(const Array &values, const Array &indices, int cb, bool keep) {
  Context &c = Context::get();
  const int64_t m = indices.len();
  const acu_array v = values.view(), ix = indices.view();
  const acu_dtype it = (acu_dtype)dtype_code(indices.data_type());
  Buffer vb, nb;
  acu_status st;
  std::optional<ArrowError> deferred;
  std::vector<ArrayRef> children;
  switch (values.data_type()) {
    case DataType::Boolean: {
      acu_array_out o = make_out(vb, nb, acu_bitmap_bytes(m), m);
      if ((st = acu_take_boolean(c.raw(), &v, &ix, it, cb, &o)) != ACU_OK) return c.last_error(st);
      return ArrayRef(std::make_shared<BooleanArray>(vb, 0, o.len, out_nulls(o, nb)));
    }
    case DataType::Utf8: {
      const auto &s = static_cast<const StringArray &>(values);
      const uint8_t *src = static_cast<const uint8_t *>(s.value_data().data());
      return bytes_out(m, false, [&](void *offs, uint8_t *data, int64_t cap, int64_t *total, acu_array_out *o) {
        if (keep) return acu_take_bytes_extend(c.raw(), 4, s.offsets().data(), src, &v, &ix, it, offs, data, cap, total, o);
        return acu_take_bytes(c.raw(), 4, s.offsets().data(), src, &v, &ix, it, cb, offs, data, cap, total, o);
      });
    }
    case DataType::FixedSizeBinary: {  // take_fixed_size_binary (take.rs:802-862)
      const int32_t w = static_cast<const FixedSizeBinaryArray &>(values).value_length();
      acu_array_out o = make_out(vb, nb, (size_t)m * w, m);
      if ((st = acu_take_fixed_size_binary(c.raw(), w, &v, &ix, it, cb, &o)) != ACU_OK) return c.last_error(st);
      // MutableArrayData keeps every extended row of a FixedSizeBinary(0) child (try_new's length rule is the top level's)
      return ArrayRef(std::make_shared<FixedSizeBinaryArray>(w, vb, keep ? m : o.len, out_nulls(o, nb)));
    }
    case DataType::List: case DataType::LargeList: case DataType::FixedSizeList: {
      const acu_list_array l = list_view(values);
      const bool fixed = l.kind == ACU_FIXED_SIZE_LIST;
      const acu_dtype cdt = fixed || l.child_len <= (int64_t)UINT32_MAX ? ACU_U32 : ACU_U64;
      Buffer offs = Buffer::allocate((size_t)(m + 1) * (l.kind == ACU_LIST ? 4 : 8));
      acu_array_out o = validity_out(nb, m), cn{};
      int64_t rows = 0;
      if ((st = acu_take_list(c.raw(), &l, &ix, it, cb, keep ? 1 : 0, offs.data(), &o, cdt, nullptr, 0, &rows, &cn)) != ACU_OK) return c.last_error(st);
      Buffer map = Buffer::allocate((size_t)rows * (cdt == ACU_U32 ? 4 : 8)), cnb = Buffer::allocate(acu_bitmap_bytes(rows));
      cn.validity = static_cast<uint8_t *>(cnb.data());
      if ((st = acu_take_list(c.raw(), &l, &ix, it, cb, keep ? 1 : 0, offs.data(), &o, cdt, map.data(), rows, &rows, &cn)) != ACU_OK) {
        // take_fixed_size_list: the child is taken before the list's validity is read
        if (!fixed || st != ACU_ERR_PANIC_OUT_OF_BOUNDS) return c.last_error(st);
        deferred = c.last_error(st);
      }
      std::optional<NullBuffer> map_nulls;
      if (cn.has_validity) map_nulls = NullBuffer{cnb, 0, rows, cn.null_count};
      ArrayRef rm = cdt == ACU_U32 ? ArrayRef(std::make_shared<PrimitiveArray<uint32_t>>(map, rows, map_nulls))
                                   : ArrayRef(std::make_shared<PrimitiveArray<uint64_t>>(map, rows, map_nulls));
      auto child = take_any(*list_values(values), *rm, 0, keep || !fixed);
      if (child.is_err()) return child.unwrap_err();
      if (deferred) return *deferred;
      return list_like(values, offs, child.unwrap(), o.len, out_nulls(o, nb));
    }
    case DataType::Struct: {
      // take_impl's Struct arm: check_bounds first, then the columns, then the validity (whose panic comes after them)
      const acu_array nv = nulls_view(values);
      acu_array_out o = validity_out(nb, m);
      if ((st = acu_take_nulls(c.raw(), &nv, &ix, it, cb, &o)) != ACU_OK) {
        if (st != ACU_ERR_PANIC_OUT_OF_BOUNDS) return c.last_error(st);
        deferred = c.last_error(st);
      }
      for (const auto &col : static_cast<const StructArray &>(values).columns()) {
        auto r = take_any(*col, indices, 0, keep);
        if (r.is_err()) return r.unwrap_err();
        children.push_back(r.unwrap());
      }
      if (deferred) return *deferred;
      std::optional<NullBuffer> nulls = out_nulls(o, nb);
      if (children.empty() && !keep && !nulls) nulls = nulls_from_mask(std::vector<bool>((size_t)m, true), true);  // new_empty_fields
      return ArrayRef(std::make_shared<StructArray>(std::move(children), m, std::move(nulls)));
    }
    case DataType::Union: {
      const auto &u = static_cast<const UnionArray &>(values);
      const acu_union_array uv = u.union_view();
      const size_t nf = u.field_type_ids().size();
      Buffer tids = Buffer::allocate((size_t)m), offs = Buffer::allocate((size_t)m * 4), map = Buffer::allocate((size_t)m * 4);
      std::vector<int64_t> starts(nf + 1, 0);
      if ((st = acu_take_union(c.raw(), &uv, &ix, it, cb, static_cast<int8_t *>(tids.data()), static_cast<int32_t *>(offs.data()),
                               static_cast<int32_t *>(map.data()), starts.data())) != ACU_OK) {
        ArrowError e = c.last_error(st);
        // UnionArray::try_new validates after the children are taken
        if (e.message.find("Type Ids values must match one of the field type ids") == std::string::npos &&
            e.message.find("Offsets must be non-negative and within the length of the Array") == std::string::npos)
          return e;
        deferred = e;
      }
      for (size_t f = 0; f < nf; ++f) {
        auto r = u.is_dense() ? take_any(*u.children()[f], *i32_slice(map, starts[f], starts[f + 1] - starts[f]), 0, keep)
                              : take_any(*u.children()[f], indices, 0, keep);
        if (r.is_err()) return r.unwrap_err();
        children.push_back(r.unwrap());
      }
      if (deferred) return *deferred;
      std::optional<Buffer> ob;
      if (u.is_dense()) ob = offs;
      return ArrayRef(std::make_shared<UnionArray>(u.field_type_ids(), tids, std::move(ob), std::move(children), m));
    }
    case DataType::RunEndEncoded:
      return ArrowError{ACU_ERR_NOT_YET_IMPLEMENTED, "Not yet implemented: take of a RunEndEncoded array below the top level"};
    default: {
      const int w = dtype_width(values.data_type());
      acu_array_out o = make_out(vb, nb, (size_t)m * w, m);
      if ((st = acu_take_primitive(c.raw(), w, &v, &ix, it, cb, &o)) != ACU_OK) return c.last_error(st);
      return make_primitive(values.data_type(), vb, o.len, out_nulls(o, nb));
    }
  }
}

template <class R>
Result<ArrayRef> filter_run_end(const RunArray<R> &values, const FilterPredicate &pred) {
  Context &c = Context::get();
  acu_filter_plan *plan = pred.raw();
  const acu_run_array r = values.run_view();
  const int64_t count = pred.count();
  Buffer ends = Buffer::allocate((size_t)std::max<int64_t>(std::min(count, values.num_runs()), 1) * sizeof(R));
  int64_t runs = 0, start = 0;
  acu_filter_plan *vplan = nullptr;
  acu_status st = acu_filter_run_end(c.raw(), plan, &r, ends.data(), &runs, &start, &vplan);
  if (st != ACU_OK) return c.last_error(st);
  if (!vplan) {
    if (acu_filter_plan_strategy(plan) == ACU_FILTER_ALL) return ArrayRef(std::make_shared<RunArray<R>>(values.slice(0, count)));
    return ArrayRef(std::make_shared<RunArray<R>>(Buffer::allocate(0), 0, empty_like(*values.values()), 0, 0));
  }
  const FilterPredicate vpred(vplan);
  auto v = filter_any(*slice_any(*values.values(), start, acu_filter_plan_len(vplan)), vpred);
  if (v.is_err()) return v.unwrap_err();
  std::vector<R> host((size_t)runs);
  ends.to_host(host.data(), host.size() * sizeof(R));
  return ArrayRef(std::make_shared<RunArray<R>>(ends, runs, v.unwrap(), 0, (int64_t)host.back()));  // the last new run end
}

template <class R>
Result<ArrayRef> take_run_end(const RunArray<R> &values, const Array &indices, int cb) {
  Context &c = Context::get();
  const DataType it = indices.data_type();
  const Array &vals = *values.values();
  acu_run_values rv{};
  switch (vals.data_type()) {
    case DataType::Boolean: rv.kind = ACU_RUN_VALUES_BOOLEAN; rv.array = vals.view(); break;
    case DataType::Utf8: {
      const auto &s = static_cast<const StringArray &>(vals);
      rv.kind = ACU_RUN_VALUES_BYTES;
      rv.width = 4;
      rv.bytes.offsets = s.offsets().data();
      rv.bytes.data = static_cast<const uint8_t *>(s.value_data().data());
      rv.bytes.nulls = vals.view();
      break;
    }
    case DataType::List: case DataType::LargeList: case DataType::FixedSizeList: case DataType::Struct: case DataType::Union:
    case DataType::FixedSizeBinary:  // the run merge would need a value_length-byte comparator
      rv.kind = ACU_RUN_VALUES_NESTED;
      break;
    default:
      if (dtype_width(vals.data_type()) == 0)
        throw std::runtime_error(std::string("RunArray values of type ") + dtype_display(vals.data_type()) + " are not supported by this mirror");
      rv.kind = ACU_RUN_VALUES_FIXED;
      rv.width = dtype_width(vals.data_type());
      rv.array = vals.view();
  }
  const int64_t m = indices.len();
  const bool wide = it == DataType::Int64 || it == DataType::UInt64;  // ToIndices: UInt64 value indices
  const acu_run_array r = values.run_view();
  const acu_array ix = indices.view();
  Buffer ends = Buffer::allocate((size_t)std::max<int64_t>(m, 1) * sizeof(R)), vi = Buffer::allocate((size_t)std::max<int64_t>(m, 1) * (wide ? 8 : 4));
  int64_t runs = 0;
  acu_status st = acu_take_run_end(c.raw(), &r, &rv, &ix, (acu_dtype)dtype_code(it), cb, ends.data(), vi.data(), &runs);
  if (st != ACU_OK) return c.last_error(st);
  if (m == 0) return ArrayRef(std::make_shared<RunArray<R>>(Buffer::allocate(0), 0, empty_like(vals), 0, 0));
  ArrayRef vix = wide ? ArrayRef(std::make_shared<PrimitiveArray<uint64_t>>(vi, runs, std::nullopt))
                      : ArrayRef(std::make_shared<PrimitiveArray<uint32_t>>(vi, runs, std::nullopt));
  auto v = take_any(vals, *vix, 0, false);
  if (v.is_err()) return v.unwrap_err();
  return ArrayRef(std::make_shared<RunArray<R>>(ends, runs, v.unwrap(), 0, m));
}
}  // namespace detail

inline Result<ArrayRef> FilterPredicate::filter(const Array &values) const {
  if (values.data_type() == DataType::RunEndEncoded)
    return detail::with_run_array(values, [&](const auto &run) { return detail::filter_run_end(run, *this); });
  return detail::filter_any(values, *this);
}

// arrow::compute::filter (filter.rs:201-213)
inline Result<ArrayRef> filter(const Array &values, const BooleanArray &predicate) {
  auto pred = FilterPredicate::try_new(predicate);
  if (pred.is_err()) return pred.unwrap_err();
  return pred.unwrap().filter(values);
}
inline Result<RecordBatch> filter_record_batch(const RecordBatch &batch, const BooleanArray &predicate) {
  return FilterBuilder(predicate).optimize().build().filter_record_batch(batch);
}

// arrow::compute::take (take.rs:89-105)
inline Result<ArrayRef> take(const Array &values, const Array &indices, std::optional<TakeOptions> options = std::nullopt) {
  if (auto e = detail::index_type_error(indices.data_type())) return *e;
  const int cb = options && options->check_bounds ? 1 : 0;
  if (values.data_type() == DataType::RunEndEncoded)
    return detail::with_run_array(values, [&](const auto &run) { return detail::take_run_end(run, indices, cb); });
  return detail::take_any(values, indices, cb, false);
}

// take.rs:1123-1133: every column gathered with the same indices, one synchronisation per (up to 64-column) call.
// Utf8 columns are sized by a first pass without a byte buffer (duplicated indices can grow a column beyond its source).
inline Result<RecordBatch> take_record_batch(const RecordBatch &batch, const Array &indices) {
  Context &c = Context::get();
  const DataType it = indices.data_type();
  if (auto e = detail::index_type_error(it)) return *e;
  const auto &cols = batch.columns();
  const int64_t m = indices.len();
  if (cols.empty()) return RecordBatch(batch.schema(), {}, m);
  std::vector<acu_column> in;
  bool any_utf8 = false;
  for (const auto &col : cols) {
    in.push_back(detail::column_view(*col));
    any_utf8 = any_utf8 || col->data_type() == DataType::Utf8;
  }
  acu_array ix = indices.view();
  std::vector<int64_t> caps(cols.size(), -1);
  auto run = [&](detail::BatchOutputs &out) -> acu_status {
    for (size_t first = 0; first < cols.size(); first += ACU_MAX_BATCH_COLUMNS) {
      const int32_t n = (int32_t)std::min<size_t>(ACU_MAX_BATCH_COLUMNS, cols.size() - first);
      acu_status st = acu_take_record_batch(c.raw(), n, in.data() + first, &ix, (acu_dtype)dtype_code(it), 0, out.outs.data() + first);
      if (st != ACU_OK) return st;
    }
    return ACU_OK;
  };
  if (any_utf8) {  // sizing pass (offsets + nulls only)
    detail::BatchOutputs sizing;
    sizing.allocate(cols, m, caps);
    acu_status st = run(sizing);
    if (st != ACU_OK) return c.last_error(st);
    for (size_t i = 0; i < cols.size(); ++i)
      if (cols[i]->data_type() == DataType::Utf8) caps[i] = sizing.outs[i].data_len;
  }
  detail::BatchOutputs out;
  out.allocate(cols, m, caps);
  acu_status st = run(out);
  if (st != ACU_OK) return c.last_error(st);
  return RecordBatch(batch.schema(), out.wrap(cols), m);
}

// ---- BatchCoalescer (arrow-select/src/coalesce.rs:148-590) -----------------------------------
// Output batches hold exactly target_batch_size rows, in input order; in-progress columns live in HBM at
// their final capacity and rows are appended in place (InProgressArray::copy_rows): fixed-width values by
// device-to-device copy, validity / boolean bits by acu_bitmap_copy at the current bit position (nothing is
// materialised until the first null arrives, like NullBufferBuilder), Utf8 by acu_offsets_append + byte copy.
class BatchCoalescer {
 public:
  BatchCoalescer(Schema schema, int64_t target_batch_size) : schema_(std::move(schema)), target_(target_batch_size) {
    for (const auto &f : schema_) cols_.push_back(fresh(f.data_type));
  }
  const Schema &schema() const { return schema_; }
  int64_t get_buffered_rows() const { return buffered_; }
  bool is_empty() const { return buffered_ == 0 && completed_.empty(); }
  bool has_completed_batch() const { return !completed_.empty(); }
  std::optional<RecordBatch> next_completed_batch() {
    if (completed_.empty()) return std::nullopt;
    RecordBatch b = std::move(completed_.front());
    completed_.erase(completed_.begin());
    return b;
  }
  // coalesce.rs:325-533
  Result<int64_t> push_batch(const RecordBatch &batch) {
    if (batch.num_columns() != cols_.size())
      return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: Batch has " + std::to_string(batch.num_columns()) +
                                                       " columns but BatchCoalescer expects " + std::to_string(cols_.size())};
    int64_t num_rows = batch.num_rows(), offset = 0;
    while (num_rows > target_ - buffered_) {
      const int64_t remaining = target_ - buffered_;
      for (size_t c = 0; c < cols_.size(); ++c) {
        auto st = copy_rows(cols_[c], *batch.column(c), offset, remaining);
        if (st.is_err()) return st.unwrap_err();
      }
      buffered_ += remaining;
      offset += remaining;
      num_rows -= remaining;
      finish_buffered_batch();
    }
    if (num_rows > 0)
      for (size_t c = 0; c < cols_.size(); ++c) {
        auto st = copy_rows(cols_[c], *batch.column(c), offset, num_rows);
        if (st.is_err()) return st.unwrap_err();
      }
    buffered_ += num_rows;
    if (buffered_ >= target_) finish_buffered_batch();
    return buffered_;
  }
  // "semantically equivalent of calling push_batch with the results from filter_record_batch" (coalesce.rs:236-237)
  Result<int64_t> push_batch_with_filter(const RecordBatch &batch, const BooleanArray &filter) {
    auto f = filter_record_batch(batch, filter);
    if (f.is_err()) return f.unwrap_err();
    return push_batch(f.unwrap());
  }
  Result<int64_t> push_batch_with_indices(const RecordBatch &batch, const Array &indices) {  // coalesce.rs:289-298
    auto t = take_record_batch(batch, indices);
    if (t.is_err()) return t.unwrap_err();
    return push_batch(t.unwrap());
  }
  void finish_buffered_batch() {  // coalesce.rs:547-570
    if (buffered_ == 0) return;
    std::vector<ArrayRef> arrays;
    for (size_t c = 0; c < cols_.size(); ++c) {
      InProgress &p = cols_[c];
      std::optional<NullBuffer> nulls;
      if (p.materialised && p.null_count > 0) nulls = NullBuffer{p.valid, 0, buffered_, p.null_count};
      if (p.dt == DataType::Boolean) arrays.push_back(std::make_shared<BooleanArray>(p.values, 0, buffered_, nulls));
      else if (p.dt == DataType::Utf8) arrays.push_back(std::make_shared<StringArray>(p.values, p.data, buffered_, nulls));
      else arrays.push_back(detail::make_primitive(p.dt, p.values, buffered_, nulls));
      p = fresh(p.dt);
    }
    completed_.push_back(RecordBatch(schema_, std::move(arrays), buffered_));
    buffered_ = 0;
  }

 private:
  struct InProgress {
    DataType dt;
    Buffer values, valid, data;
    bool materialised = false;
    int64_t null_count = 0, data_len = 0, data_cap = 0;
  };
  InProgress fresh(DataType dt) const {
    InProgress p;
    p.dt = dt;
    p.valid = Buffer::allocate(acu_bitmap_bytes(target_));
    if (dt == DataType::Boolean) p.values = Buffer::allocate(acu_bitmap_bytes(target_));
    else if (dt == DataType::Utf8) {
      p.values = Buffer::allocate((size_t)(target_ + 1) * 4);
      p.data_cap = 1 << 16;
      p.data = Buffer::allocate((size_t)p.data_cap);
      const int32_t zero = 0;
      acu_memcpy_h2d(Context::get().raw(), p.values.data(), &zero, 4);
    } else p.values = Buffer::allocate((size_t)target_ * dtype_width(dt));
    return p;
  }
  Result<int64_t> copy_rows(InProgress &p, const Array &src, int64_t offset, int64_t n) {
    Context &c = Context::get();
    acu_ctx *h = c.raw();
    const acu_array v = src.view();
    acu_status st;
    int64_t nulls_here = 0;
    if (v.validity && v.null_count != 0) {
      int64_t set = 0;
      if ((st = acu_bitmap_count(h, v.validity, v.validity_offset + offset, nullptr, 0, n, &set)) != ACU_OK) return c.last_error(st);
      nulls_here = n - set;
    }
    uint8_t *valid = static_cast<uint8_t *>(p.valid.data());
    if (nulls_here) {
      if (!p.materialised) {
        if ((st = acu_bitmap_fill(h, valid, 0, buffered_, 1)) != ACU_OK) return c.last_error(st);
        p.materialised = true;
      }
      if ((st = acu_bitmap_copy(h, v.validity, v.validity_offset + offset, valid, buffered_, n, nullptr)) != ACU_OK) return c.last_error(st);
      p.null_count += nulls_here;
    } else if (p.materialised) {
      if ((st = acu_bitmap_fill(h, valid, buffered_, n, 1)) != ACU_OK) return c.last_error(st);
    }
    if (p.dt == DataType::Boolean) {
      st = acu_bitmap_copy(h, static_cast<const uint8_t *>(v.values), v.values_offset + offset, static_cast<uint8_t *>(p.values.data()), buffered_, n, nullptr);
    } else if (p.dt == DataType::Utf8) {
      const auto &s = static_cast<const StringArray &>(src);
      int64_t s0 = 0, s1 = 0;
      if ((st = acu_offsets_append(h, 4, s.offsets().data(), offset, n, p.data_len, p.values.data(), buffered_, &s0, &s1)) != ACU_OK) return c.last_error(st);
      const int64_t nbytes = s1 - s0;
      if (p.data_len + nbytes > p.data_cap) {
        while (p.data_cap < p.data_len + nbytes) p.data_cap *= 2;
        Buffer bigger = Buffer::allocate((size_t)p.data_cap);
        if (p.data_len) acu_memcpy_d2d(h, bigger.data(), p.data.data(), (size_t)p.data_len);
        acu_ctx_sync(h);  // the old bytes buffer is released when `p.data` is reassigned
        p.data = bigger;
      }
      st = acu_memcpy_d2d(h, static_cast<uint8_t *>(p.data.data()) + p.data_len, static_cast<const uint8_t *>(s.value_data().data()) + s0, (size_t)nbytes);
      p.data_len += nbytes;
    } else {
      const int w = dtype_width(p.dt);
      st = acu_memcpy_d2d(h, static_cast<uint8_t *>(p.values.data()) + (size_t)buffered_ * w, static_cast<const uint8_t *>(v.values) + (size_t)offset * w, (size_t)n * w);
    }
    if (st != ACU_OK) return c.last_error(st);
    return n;
  }
  Schema schema_;
  int64_t target_;
  std::vector<InProgress> cols_;
  int64_t buffered_ = 0;
  std::vector<RecordBatch> completed_;
};

// ---- Utf8View / BinaryView columns: GenericByteViewArray + BatchCoalescer's InProgressByteViewArray ----------------------
// (arrow-array/src/array/byte_view_array.rs; arrow-select/src/coalesce/byte_view.rs:39-559). A view = 16 bytes: length u32 |
// 12 inline bytes, or length | 4-byte prefix | buffer index u32 | offset u32. The policy below (gc decision, BufferSource,
// "fill the current buffer, then start a new one") is the reference's; the per-view work runs on the device (acu_view_*).
struct ViewDataBuffer {
  Buffer buffer;
  size_t len = 0, capacity = 0;  // Buffer::len() / Buffer::capacity()
};

class StringViewArray {
 public:
  StringViewArray() = default;
  StringViewArray(Buffer views, int64_t offset, int64_t len, std::vector<ViewDataBuffer> buffers, std::vector<bool> valid)
      : views_(std::move(views)), offset_(offset), len_(len), buffers_(std::move(buffers)), valid_(std::move(valid)) {}
  // StringViewBuilder::with_fixed_block_size(block_size): long values fill blocks of `block_size` bytes
  static StringViewArray from(const std::vector<std::optional<std::string>> &v, size_t block_size = 8192) {
    std::vector<uint8_t> views(v.size() * 16 + 16, 0);
    std::vector<std::string> blocks;
    std::string cur;
    std::vector<bool> valid(v.size(), true);
    for (size_t i = 0; i < v.size(); ++i) {
      if (!v[i]) { valid[i] = false; continue; }
      const std::string &sv = *v[i];
      const uint32_t len = (uint32_t)sv.size();
      memcpy(&views[16 * i], &len, 4);
      if (len <= 12) {
        memcpy(&views[16 * i + 4], sv.data(), len);
      } else {
        if (cur.size() + len > block_size && !cur.empty()) { blocks.push_back(cur); cur.clear(); }
        const uint32_t bi = (uint32_t)blocks.size(), off = (uint32_t)cur.size();
        memcpy(&views[16 * i + 4], sv.data(), 4);
        memcpy(&views[16 * i + 8], &bi, 4);
        memcpy(&views[16 * i + 12], &off, 4);
        cur += sv;
      }
    }
    if (!cur.empty()) blocks.push_back(cur);
    std::vector<ViewDataBuffer> bufs;
    for (const auto &b : blocks) bufs.push_back(ViewDataBuffer{Buffer::from_host(b.data(), b.size()), b.size(), std::max(block_size, b.size())});
    return StringViewArray(Buffer::from_host(views.data(), v.size() * 16), 0, (int64_t)v.size(), std::move(bufs), std::move(valid));
  }
  int64_t len() const { return len_; }
  const void *views_ptr() const { return static_cast<const uint8_t *>(views_.data()) + 16 * offset_; }
  const std::vector<ViewDataBuffer> &data_buffers() const { return buffers_; }
  const std::vector<bool> &valid() const { return valid_; }  // validity of rows [0, len) (host side: the test mirror)
  bool has_nulls() const { return std::find(valid_.begin(), valid_.end(), false) != valid_.end(); }
  StringViewArray slice(int64_t offset, int64_t len) const {
    return StringViewArray(views_, offset_ + offset, len, buffers_, std::vector<bool>(valid_.begin() + offset, valid_.begin() + offset + len));
  }
  // GenericByteViewArray::total_buffer_bytes_used (byte_view_array.rs:749-761)
  Result<int64_t> total_buffer_bytes_used() const {
    int64_t total = 0;
    Context &c = Context::get();
    const acu_status st = acu_view_bytes_used(c.raw(), views_ptr(), len_, &total);
    if (st != ACU_OK) return c.last_error(st);
    return total;
  }
  std::vector<std::optional<std::string>> to_vec() const {
    std::vector<uint8_t> views((size_t)len_ * 16 + 16);
    if (len_) acu_memcpy_d2h(Context::get().raw(), views.data(), views_ptr(), (size_t)len_ * 16);
    std::vector<std::string> data;
    for (const auto &b : buffers_) {
      std::string sdat(b.len, '\0');
      b.buffer.to_host(sdat.data(), b.len);
      data.push_back(std::move(sdat));
    }
    std::vector<std::optional<std::string>> out((size_t)len_);
    for (int64_t i = 0; i < len_; ++i) {
      if (!valid_[(size_t)i]) continue;
      uint32_t len, bi, off;
      memcpy(&len, &views[16 * i], 4);
      if (len <= 12) out[(size_t)i] = std::string(reinterpret_cast<const char *>(&views[16 * i + 4]), len);
      else {
        memcpy(&bi, &views[16 * i + 8], 4);
        memcpy(&off, &views[16 * i + 12], 4);
        out[(size_t)i] = data[bi].substr(off, len);
      }
    }
    return out;
  }
 private:
  Buffer views_;
  int64_t offset_ = 0, len_ = 0;
  std::vector<ViewDataBuffer> buffers_;
  std::vector<bool> valid_;
};

namespace coalesce {

// BufferSource (byte_view.rs:526-559): 8 KiB doubling to 1 MiB, or the size asked for when larger
class BufferSource {
 public:
  size_t next_size(size_t min_size) {
    if (current_ < kMax) current_ *= 2;
    if (current_ >= min_size) return current_;
    while (current_ <= min_size && current_ < kMax) current_ *= 2;
    return std::max(current_, min_size);
  }
 private:
  static constexpr size_t kMax = 1024 * 1024;
  size_t current_ = 4 * 1024;
};

class InProgressByteViewArray {
 public:
  explicit InProgressByteViewArray(int64_t batch_size) : batch_size_(batch_size) {}
  // set_source (:357-391)
  Result<int64_t> set_source(std::optional<StringViewArray> source) {
    source_ = std::move(source);
    need_gc_ = false;
    ideal_ = 0;
    if (source_ && !source_->data_buffers().empty()) {
      auto used = source_->total_buffer_bytes_used();
      if (used.is_err()) return used.unwrap_err();
      ideal_ = (size_t)used.unwrap();
      size_t actual = 0;
      for (const auto &b : source_->data_buffers()) actual += b.capacity;
      need_gc_ = ideal_ != 0 && actual > ideal_ * 2;
    }
    return (int64_t)ideal_;
  }
  bool source_needs_gc() const { return need_gc_; }
  // copy_rows (:393-436)
  Result<int64_t> copy_rows(int64_t offset, int64_t len) {
    if (!source_) return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: Internal Error: InProgressByteViewArray: source not set"};
    if (!views_.data()) views_ = Buffer::allocate((size_t)batch_size_ * 16);
    const StringViewArray piece = source_->slice(offset, len);
    valid_.insert(valid_.end(), piece.valid().begin(), piece.valid().end());
    Context &c = Context::get();
    acu_status st = ACU_OK;
    if (ideal_ == 0) {
      st = acu_view_rebase(c.raw(), piece.views_ptr(), len, 0, out_at(n_views_));
    } else if (need_gc_) {
      auto r = append_views_and_copy_strings(piece, ideal_);
      if (r.is_err()) return r;
    } else {  // append_views_and_update_buffer_index (:176-216)
      finish_current();
      const uint32_t starting = (uint32_t)completed_.size();
      for (const auto &b : piece.data_buffers()) completed_.push_back(b);
      st = acu_view_rebase(c.raw(), piece.views_ptr(), len, starting, out_at(n_views_));
    }
    if (st != ACU_OK) return c.last_error(st);
    n_views_ += len;
    return len;
  }
  // finish (:490-520)
  StringViewArray finish() {
    finish_current();
    StringViewArray out(views_, 0, n_views_, std::move(completed_), std::move(valid_));
    views_ = Buffer();
    n_views_ = 0;
    completed_.clear();
    valid_.clear();
    return out;
  }

 private:
  void *out_at(int64_t row) const { return static_cast<uint8_t *>(views_.data()) + 16 * row; }
  void finish_current() {
    if (current_) { completed_.push_back(*current_); current_.reset(); }
  }
  ViewDataBuffer next_buffer(size_t min_size) {
    const size_t cap = source_sizes_.next_size(min_size);
    return ViewDataBuffer{Buffer::allocate(cap), 0, cap};
  }
  // append_views_and_copy_strings (:228-291)
  Result<int64_t> append_views_and_copy_strings(const StringViewArray &piece, size_t view_buffer_size) {
    if (!current_) return copy_inner(piece, 0, piece.len(), next_buffer(view_buffer_size));
    const size_t remaining = current_->capacity - current_->len;
    if (view_buffer_size <= remaining) {
      ViewDataBuffer cur = *current_;
      current_.reset();
      return copy_inner(piece, 0, piece.len(), cur);
    }
    Context &c = Context::get();
    int64_t num_to_current = 0, bytes_to_current = 0;
    const acu_status st = acu_view_fit(c.raw(), piece.views_ptr(), piece.len(), (int64_t)remaining, &num_to_current, &bytes_to_current);
    if (st != ACU_OK) return c.last_error(st);
    ViewDataBuffer cur = *current_;
    current_.reset();
    auto r = copy_inner(piece, 0, num_to_current, cur);
    if (r.is_err()) return r;
    finish_current();
    return copy_inner(piece, num_to_current, piece.len() - num_to_current, next_buffer(view_buffer_size - (size_t)bytes_to_current));
  }
  // append_views_and_copy_strings_inner (:298-354)
  Result<int64_t> copy_inner(const StringViewArray &piece, int64_t first, int64_t n, ViewDataBuffer dst) {
    if (n > 0) {
      Context &c = Context::get();
      std::vector<const uint8_t *> table;
      for (const auto &b : piece.data_buffers()) table.push_back(static_cast<const uint8_t *>(b.buffer.data()));
      int64_t bytes = 0;
      const acu_status st = acu_view_copy_strings(c.raw(), static_cast<const uint8_t *>(piece.views_ptr()) + 16 * first, n, table.data(), (int32_t)table.size(),
                                                  (uint32_t)completed_.size(), static_cast<uint8_t *>(dst.buffer.data()), (int64_t)dst.len,
                                                  (int64_t)dst.capacity, out_at(n_views_ + first), &bytes);
      if (st != ACU_OK) return c.last_error(st);
      dst.len += (size_t)bytes;
    }
    current_ = dst;
    return n;
  }
  int64_t batch_size_;
  std::optional<StringViewArray> source_;
  bool need_gc_ = false;
  size_t ideal_ = 0;
  Buffer views_;
  int64_t n_views_ = 0;
  std::vector<bool> valid_;
  std::optional<ViewDataBuffer> current_;
  std::vector<ViewDataBuffer> completed_;
  BufferSource source_sizes_;
};

}  // namespace coalesce

// ---- kernels::numeric (arrow-arith/src/numeric.rs) ---------------------------------------
namespace kernels {
namespace numeric {
namespace detail2 {
// decimal_op (numeric.rs:970-1107): the result type comes from the device call
template <class T>
Result<ArrayRef> decimal_arith(acu_arith_op op, const DecimalArray<T> &l, bool ls, const DecimalArray<T> &r, bool rs) {
  Context &c = Context::get();
  const int64_t n = ls && !rs ? r.len() : l.len();
  Buffer vb, nb;
  acu_array a = l.view(ls), b = r.view(rs);
  acu_decimal_type lt = l.decimal_type(), rt = r.decimal_type(), ot{};
  acu_array_out o = compute::detail::make_out(vb, nb, (size_t)std::max<int64_t>(n, 1) * sizeof(T), n);
  acu_status st = acu_decimal_arith(c.raw(), op, &lt, &a, &rt, &b, &ot, &o);
  if (st != ACU_OK) return c.last_error(st);
  return ArrayRef(std::make_shared<DecimalArray<T>>(vb, o.len, compute::detail::out_nulls(o, nb), 0, ot.precision, ot.scale));
}
template <class T> Result<ArrayRef> decimal_neg(const DecimalArray<T> &a) {  // neg_checked at every width (numeric.rs:116-136)
  Context &c = Context::get();
  Buffer vb, nb;
  acu_array v = a.view();
  acu_array_out o = compute::detail::make_out(vb, nb, (size_t)std::max<int64_t>(a.len(), 1) * sizeof(T), a.len());
  acu_status st = acu_neg(c.raw(), DecimalTraits<T>::code, 1, &v, &o);
  if (st != ACU_OK) return c.last_error(st);
  return ArrayRef(std::make_shared<DecimalArray<T>>(vb, o.len, compute::detail::out_nulls(o, nb), 0, a.precision(), a.scale()));
}

template <class L, class R>
Result<ArrayRef> arithmetic_op(acu_arith_op op, const char *sym, const L &lhs, const R &rhs) {
  const auto &l = datum_array(lhs);
  const auto &r = datum_array(rhs);
  const bool ls = datum_is_scalar(lhs), rs = datum_is_scalar(rhs);
  using LA = std::decay_t<decltype(l)>;
  using RA = std::decay_t<decltype(r)>;
  if constexpr (is_decimal_array<LA>::value || is_decimal_array<RA>::value) {  // (Decimal*, Decimal*) arms, numeric.rs:257-260
    if constexpr (std::is_same<LA, RA>::value) return decimal_arith(op, l, ls, r, rs);
    else return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: Invalid arithmetic operation: " + compute::detail::type_text(l) +
                                                         " " + sym + " " + compute::detail::type_text(r)};
  } else {
  if (l.data_type() != r.data_type() || dtype_width(l.data_type()) == 0)  // numeric.rs:270-272
    return ArrowError{ACU_ERR_INVALID_ARGUMENT, std::string("Invalid argument error: Invalid arithmetic operation: ") +
                                                     compute::detail::dtype_display(l.data_type()) + " " + sym + " " +
                                                     compute::detail::dtype_display(r.data_type())};
  Context &c = Context::get();
  const int64_t n = ls && !rs ? r.len() : l.len();
  Buffer vb, nb;
  acu_array a = l.view(ls), b = r.view(rs);
  acu_array_out o = compute::detail::make_out(vb, nb, (size_t)std::max<int64_t>(n, 1) * dtype_width(l.data_type()), n);
  acu_status st = acu_arith(c.raw(), (acu_dtype)dtype_code(l.data_type()), op, &a, &b, &o);
  if (st != ACU_OK) return c.last_error(st);
  return compute::detail::make_primitive(l.data_type(), vb, o.len, compute::detail::out_nulls(o, nb));
  }
}
}  // namespace detail2
#define ACU_NUMERIC(NAME, OP, SYM) \
  template <class L, class R> Result<ArrayRef> NAME(const L &lhs, const R &rhs) { return detail2::arithmetic_op(OP, SYM, lhs, rhs); }
ACU_NUMERIC(add, ACU_ADD, "+") ACU_NUMERIC(add_wrapping, ACU_ADD_WRAPPING, "+") ACU_NUMERIC(sub, ACU_SUB, "-")
ACU_NUMERIC(sub_wrapping, ACU_SUB_WRAPPING, "-") ACU_NUMERIC(mul, ACU_MUL, "*") ACU_NUMERIC(mul_wrapping, ACU_MUL_WRAPPING, "*")
ACU_NUMERIC(div, ACU_DIV, "/") ACU_NUMERIC(rem, ACU_REM, "%")
#undef ACU_NUMERIC

inline Result<ArrayRef> neg_impl(const Array &a, int checked) {
  // decimals: neg_wrapping falls back to neg (numeric.rs:181-186)
  if (auto d = dynamic_cast<const Decimal32Array *>(&a)) return detail2::decimal_neg(*d);
  if (auto d = dynamic_cast<const Decimal64Array *>(&a)) return detail2::decimal_neg(*d);
  if (auto d = dynamic_cast<const Decimal128Array *>(&a)) return detail2::decimal_neg(*d);
  Context &c = Context::get();
  Buffer vb, nb;
  acu_array v = a.view();
  acu_array_out o = compute::detail::make_out(vb, nb, (size_t)std::max<int64_t>(a.len(), 1) * dtype_width(a.data_type()), a.len());
  acu_status st = acu_neg(c.raw(), (acu_dtype)dtype_code(a.data_type()), checked, &v, &o);
  if (st != ACU_OK) return c.last_error(st);
  return compute::detail::make_primitive(a.data_type(), vb, o.len, compute::detail::out_nulls(o, nb));
}
inline Result<ArrayRef> neg(const Array &a) { return neg_impl(a, 1); }
inline Result<ArrayRef> neg_wrapping(const Array &a) { return neg_impl(a, 0); }
}  // namespace numeric

// ---- kernels::cmp (arrow-ord/src/cmp.rs) ---------------------------------------------------
namespace cmp {
namespace detail3 {
template <class L, class R>
Result<BooleanArray> compare_op(acu_cmp_op op, const char *sym, const L &lhs, const R &rhs) {
  const auto &l = datum_array(lhs);
  const auto &r = datum_array(rhs);
  const bool ls = datum_is_scalar(lhs), rs = datum_is_scalar(rhs);
  using LA = std::decay_t<decltype(l)>;
  acu_dtype code = (acu_dtype)dtype_code(l.data_type());
  if constexpr (is_decimal_array<LA>::value) {  // decimals compare as their natives; the DataTypes must be equal, precision included
    if (!ls && !rs && l.len() != r.len())  // cmp.rs:228-232 comes first
      return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: Cannot compare arrays of different lengths, got " +
                                                      std::to_string(l.len()) + " vs " + std::to_string(r.len())};
    if (compute::detail::type_text(l) != compute::detail::type_text(r))
      return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: Invalid comparison operation: " + compute::detail::type_text(l) +
                                                      " " + sym + " " + compute::detail::type_text(r)};
    code = DecimalTraits<typename LA::Native>::code;
  }
  if (l.data_type() != r.data_type())  // cmp.rs:260-264
    return ArrowError{ACU_ERR_INVALID_ARGUMENT, std::string("Invalid argument error: Invalid comparison operation: ") +
                                                     compute::detail::dtype_display(l.data_type()) + " " + sym + " " +
                                                     compute::detail::dtype_display(r.data_type())};
  Context &c = Context::get();
  const int64_t n = ls ? r.len() : l.len();
  Buffer vb, nb;
  acu_array a = l.view(ls), b = r.view(rs);
  acu_array_out o = compute::detail::make_out(vb, nb, acu_bitmap_bytes(std::max<int64_t>(n, 1)), std::max<int64_t>(n, 1));
  acu_status st = acu_cmp(c.raw(), code, op, &a, &b, &o);
  if (st != ACU_OK) return c.last_error(st);
  return BooleanArray(vb, 0, o.len, compute::detail::out_nulls(o, nb));
}
}  // namespace detail3
// GenericByteArray operands (cmp.rs:783-801): Utf8 arrays and scalars through acu_cmp_bytes
inline acu_bytes_array bytes_view(const StringArray &a, bool scalar) {
  acu_bytes_array b{};
  b.offsets = a.offsets().data();
  b.data = static_cast<const uint8_t *>(a.value_data().data());
  b.nulls = a.view(scalar);
  return b;
}
inline Result<BooleanArray> compare_strings(acu_cmp_op op, const StringArray &l, bool ls, const StringArray &r, bool rs) {
  Context &c = Context::get();
  const int64_t n = ls ? r.len() : l.len();
  Buffer vb, nb;
  acu_bytes_array a = bytes_view(l, ls), b = bytes_view(r, rs);
  acu_array_out o = compute::detail::make_out(vb, nb, acu_bitmap_bytes(std::max<int64_t>(n, 1)), std::max<int64_t>(n, 1));
  acu_status st = acu_cmp_bytes(c.raw(), 4, op, &a, &b, &o);
  if (st != ACU_OK) return c.last_error(st);
  return BooleanArray(vb, 0, o.len, compute::detail::out_nulls(o, nb));
}
#define ACU_CMP(NAME, OP, SYM) \
  inline Result<BooleanArray> NAME(const StringArray &l, const StringArray &r) { return compare_strings(OP, l, false, r, false); } \
  inline Result<BooleanArray> NAME(const StringArray &l, const Scalar<StringArray> &r) { return compare_strings(OP, l, false, r.array, true); } \
  inline Result<BooleanArray> NAME(const Scalar<StringArray> &l, const StringArray &r) { return compare_strings(OP, l.array, true, r, false); } \
  template <class L, class R> Result<BooleanArray> NAME(const L &lhs, const R &rhs) { return detail3::compare_op(OP, SYM, lhs, rhs); }
ACU_CMP(eq, ACU_EQ, "==") ACU_CMP(neq, ACU_NEQ, "!=") ACU_CMP(lt, ACU_LT, "<") ACU_CMP(lt_eq, ACU_LT_EQ, "<=")
ACU_CMP(gt, ACU_GT, ">") ACU_CMP(gt_eq, ACU_GT_EQ, ">=") ACU_CMP(distinct, ACU_DISTINCT, "IS DISTINCT FROM")
ACU_CMP(not_distinct, ACU_NOT_DISTINCT, "IS NOT DISTINCT FROM")
#undef ACU_CMP
}  // namespace cmp

// ---- kernels::boolean (arrow-arith/src/boolean.rs) -------------------------------------------
// `and`, `or`, `not` are reserved alternative tokens in C++: the mirror appends an underscore.
namespace boolean {
namespace detail4 {
inline Result<BooleanArray> boolean_op(acu_bool_op op, const Array &a, const Array *b) {
  Context &c = Context::get();
  const int64_t n = a.len();
  Buffer vb, nb;
  acu_array av = a.view(), bv{};
  if (b) bv = b->view();
  acu_array_out o = compute::detail::make_out(vb, nb, acu_bitmap_bytes(std::max<int64_t>(n, 1)), std::max<int64_t>(n, 1));
  acu_status st = acu_boolean(c.raw(), op, &av, b ? &bv : nullptr, &o);
  if (st != ACU_OK) return c.last_error(st);
  return BooleanArray(vb, 0, o.len, compute::detail::out_nulls(o, nb));
}
}  // namespace detail4
inline Result<BooleanArray> and_(const BooleanArray &l, const BooleanArray &r) { return detail4::boolean_op(ACU_BOOL_AND, l, &r); }
inline Result<BooleanArray> or_(const BooleanArray &l, const BooleanArray &r) { return detail4::boolean_op(ACU_BOOL_OR, l, &r); }
inline Result<BooleanArray> and_not(const BooleanArray &l, const BooleanArray &r) { return detail4::boolean_op(ACU_BOOL_AND_NOT, l, &r); }
inline Result<BooleanArray> and_kleene(const BooleanArray &l, const BooleanArray &r) { return detail4::boolean_op(ACU_BOOL_AND_KLEENE, l, &r); }
inline Result<BooleanArray> or_kleene(const BooleanArray &l, const BooleanArray &r) { return detail4::boolean_op(ACU_BOOL_OR_KLEENE, l, &r); }
inline Result<BooleanArray> not_(const BooleanArray &a) { return detail4::boolean_op(ACU_BOOL_NOT, a, nullptr); }
inline Result<BooleanArray> is_null(const Array &a) { return detail4::boolean_op(ACU_BOOL_IS_NULL, a, nullptr); }
inline Result<BooleanArray> is_not_null(const Array &a) { return detail4::boolean_op(ACU_BOOL_IS_NOT_NULL, a, nullptr); }
}  // namespace boolean

// ---- kernels::bitwise (arrow-arith/src/bitwise.rs) -------------------------------------------
// Integer PrimitiveArrays only (the reference's trait bounds exclude floats): the op at every slot, NullBuffer::union of
// the operands (array forms) or the left operand's nulls (scalar forms, not). Shifts wrap the amount modulo the width.
namespace bitwise {
namespace detail5 {
template <class T>
Result<PrimitiveArray<T>> bitwise_op(acu_bitwise_op op, const PrimitiveArray<T> &l, const PrimitiveArray<T> *r, const T *scalar) {
  static_assert(std::is_integral<T>::value, "bitwise operations take integer arrays");
  Context &c = Context::get();
  const int64_t n = l.len();
  Buffer vb, nb;
  acu_array a = l.view(), b{};
  std::optional<PrimitiveArray<T>> s;
  if (r) b = r->view();
  if (scalar) {
    s = PrimitiveArray<T>::from(std::vector<T>{*scalar});
    b = s->view(true);
  }
  acu_array_out o = compute::detail::make_out(vb, nb, (size_t)std::max<int64_t>(n, 1) * sizeof(T), n);
  acu_status st = acu_bitwise(c.raw(), NativeOf<T>::code, op, &a, (r || scalar) ? &b : nullptr, &o);
  if (st != ACU_OK) return c.last_error(st);
  return PrimitiveArray<T>(vb, o.len, compute::detail::out_nulls(o, nb));
}
}  // namespace detail5
#define ACU_BITWISE(NAME, OP)                                                                                          \
  template <class T> Result<PrimitiveArray<T>> NAME(const PrimitiveArray<T> &l, const PrimitiveArray<T> &r) {        \
    return detail5::bitwise_op<T>(OP, l, &r, nullptr);                                                               \
  }
#define ACU_BITWISE_SCALAR(NAME, OP)                                                                                   \
  template <class T> Result<PrimitiveArray<T>> NAME(const PrimitiveArray<T> &l, T scalar) {                          \
    return detail5::bitwise_op<T>(OP, l, nullptr, &scalar);                                                          \
  }
ACU_BITWISE(bitwise_and, ACU_BITWISE_AND) ACU_BITWISE(bitwise_or, ACU_BITWISE_OR) ACU_BITWISE(bitwise_xor, ACU_BITWISE_XOR)
ACU_BITWISE(bitwise_and_not, ACU_BITWISE_AND_NOT) ACU_BITWISE(bitwise_shift_left, ACU_BITWISE_SHIFT_LEFT)
ACU_BITWISE(bitwise_shift_right, ACU_BITWISE_SHIFT_RIGHT)
ACU_BITWISE_SCALAR(bitwise_and_scalar, ACU_BITWISE_AND) ACU_BITWISE_SCALAR(bitwise_or_scalar, ACU_BITWISE_OR)
ACU_BITWISE_SCALAR(bitwise_xor_scalar, ACU_BITWISE_XOR) ACU_BITWISE_SCALAR(bitwise_shift_left_scalar, ACU_BITWISE_SHIFT_LEFT)
ACU_BITWISE_SCALAR(bitwise_shift_right_scalar, ACU_BITWISE_SHIFT_RIGHT)
#undef ACU_BITWISE
#undef ACU_BITWISE_SCALAR
template <class T> Result<PrimitiveArray<T>> bitwise_not(const PrimitiveArray<T> &a) {
  return detail5::bitwise_op<T>(ACU_BITWISE_NOT, a, nullptr, nullptr);
}
}  // namespace bitwise
}  // namespace kernels

// ---- cast (arrow-cast/src/cast/mod.rs) -------------------------------------------------------
struct CastOptions { bool safe = true; };  // mod.rs:96-111
// A decimal cast target: DataType::Decimal32 / Decimal64 / Decimal128(precision, scale)
struct DecimalDataType { DataType data_type; uint8_t precision; int8_t scale; };

namespace detail {
inline bool decimal_type_of(const Array &a, acu_decimal_type *t) {
  if (auto d = dynamic_cast<const DecimalArray<int32_t> *>(&a)) { *t = d->decimal_type(); return true; }
  if (auto d = dynamic_cast<const DecimalArray<int64_t> *>(&a)) { *t = d->decimal_type(); return true; }
  if (auto d = dynamic_cast<const DecimalArray<__int128> *>(&a)) { *t = d->decimal_type(); return true; }
  return false;
}
inline int decimal_width(DataType t) { return t == DataType::Decimal32 ? 4 : t == DataType::Decimal64 ? 8 : t == DataType::Decimal128 ? 16 : 0; }
}  // namespace detail

// The decimal arms of cast_with_options (mod.rs:980-1219): decimal -> decimal, integer / float -> decimal. The result is
// Decimal*Array::with_precision_and_scale(precision, scale) of the cast values.
inline Result<ArrayRef> cast_with_options(const Array &array, const DecimalDataType &to, const CastOptions &opt) {
  const int w = detail::decimal_width(to.data_type);
  acu_decimal_type from{}, tt{w, to.precision, to.scale, {0, 0}};
  const bool from_decimal = detail::decimal_type_of(array, &from);
  if (w == 0 || (!from_decimal && dtype_width(array.data_type()) == 0))
    return ArrowError{ACU_ERR_CAST, std::string("Cast error: Casting from ") + detail::dtype_display(array.data_type()) + " to " +
                                        detail::dtype_display(to.data_type) + " not supported"};
  Context &c = Context::get();
  Buffer vb, nb;
  acu_array v = array.view();
  acu_array_out o = detail::make_out(vb, nb, (size_t)std::max<int64_t>(array.len(), 1) * w, array.len());
  acu_status st = from_decimal ? acu_cast_decimal(c.raw(), &from, &tt, opt.safe ? 1 : 0, &v, &o)
                               : acu_cast_to_decimal(c.raw(), (acu_dtype)dtype_code(array.data_type()), &tt, opt.safe ? 1 : 0, &v, &o);
  if (st != ACU_OK) return c.last_error(st);
  auto nulls = detail::out_nulls(o, nb);
  if (w == 4) return ArrayRef(std::make_shared<DecimalArray<int32_t>>(vb, o.len, nulls, 0, to.precision, to.scale));
  if (w == 8) return ArrayRef(std::make_shared<DecimalArray<int64_t>>(vb, o.len, nulls, 0, to.precision, to.scale));
  return ArrayRef(std::make_shared<DecimalArray<__int128>>(vb, o.len, nulls, 0, to.precision, to.scale));
}

inline Result<ArrayRef> cast_with_options(const Array &array, DataType to_type, const CastOptions &opt) {
  acu_decimal_type from{};
  if (detail::decimal_type_of(array, &from) && dtype_width(to_type) != 0) {  // decimal -> integer / float
    Context &c = Context::get();
    Buffer vb, nb;
    acu_array v = array.view();
    acu_array_out o = detail::make_out(vb, nb, (size_t)std::max<int64_t>(array.len(), 1) * dtype_width(to_type), array.len());
    acu_status st = acu_cast_from_decimal(c.raw(), &from, (acu_dtype)dtype_code(to_type), opt.safe ? 1 : 0, &v, &o);
    if (st != ACU_OK) return c.last_error(st);
    return detail::make_primitive(to_type, vb, o.len, detail::out_nulls(o, nb));
  }
  if (dtype_width(array.data_type()) == 0 || dtype_width(to_type) == 0)
    return ArrowError{ACU_ERR_CAST, std::string("Cast error: Casting from ") + detail::dtype_display(array.data_type()) + " to " +
                                        detail::dtype_display(to_type) + " not supported"};
  Context &c = Context::get();
  Buffer vb, nb;
  acu_array v = array.view();
  acu_array_out o = detail::make_out(vb, nb, (size_t)std::max<int64_t>(array.len(), 1) * dtype_width(to_type), array.len());
  acu_status st = acu_cast_numeric(c.raw(), (acu_dtype)dtype_code(array.data_type()), (acu_dtype)dtype_code(to_type), opt.safe ? 1 : 0, &v, &o);
  if (st != ACU_OK) return c.last_error(st);
  return detail::make_primitive(to_type, vb, o.len, detail::out_nulls(o, nb));
}
inline Result<ArrayRef> cast(const Array &array, DataType to_type) { return cast_with_options(array, to_type, CastOptions{}); }

// Dictionary<Int32, Utf8> -> Utf8 (arrow-cast/src/cast/dictionary.rs:310-317): take(dict values, keys)
inline Result<ArrayRef> cast_dictionary_to_utf8(const Int32Array &keys, const StringArray &dictionary) { return take(dictionary, keys, std::nullopt); }

// ---- aggregate (arrow-arith/src/aggregate.rs) ------------------------------------------------
namespace detail {
template <class T>
std::optional<T> aggregate(acu_agg_op op, const PrimitiveArray<T> &a) {
  uint64_t bits = 0;
  int64_t valid = 0;
  acu_array v = a.view();
  acu_status st = acu_aggregate(Context::get().raw(), NativeOf<T>::code, op, &v, &bits, &valid);
  if (st != ACU_OK) throw std::runtime_error(Context::get().last_error(st).message);
  if (valid == 0) return std::nullopt;
  T out;
  std::memcpy(&out, &bits, sizeof(T));
  return out;
}
// decimals: sum wraps in the native, min / max in its order (acu_aggregate_i128 for Decimal128)
template <class T>
std::optional<T> aggregate_decimal(acu_agg_op op, const DecimalArray<T> &a) {
  uint64_t bits[2] = {0, 0};
  int64_t valid = 0;
  acu_array v = a.view();
  acu_status st = sizeof(T) == 16 ? acu_aggregate_i128(Context::get().raw(), op, &v, bits, &valid)
                                  : acu_aggregate(Context::get().raw(), DecimalTraits<T>::code, op, &v, bits, &valid);
  if (st != ACU_OK) throw std::runtime_error(Context::get().last_error(st).message);
  if (valid == 0) return std::nullopt;
  T out;
  std::memcpy(&out, bits, sizeof(T));
  return out;
}
}  // namespace detail
template <class T> std::optional<T> sum(const DecimalArray<T> &a) { return detail::aggregate_decimal(ACU_SUM, a); }
template <class T> std::optional<T> min(const DecimalArray<T> &a) { return detail::aggregate_decimal(ACU_MIN, a); }
template <class T> std::optional<T> max(const DecimalArray<T> &a) { return detail::aggregate_decimal(ACU_MAX, a); }
template <class T> std::optional<T> sum(const PrimitiveArray<T> &a) { return detail::aggregate(ACU_SUM, a); }
template <class T> std::optional<T> min(const PrimitiveArray<T> &a) { return detail::aggregate(ACU_MIN, a); }
template <class T> std::optional<T> max(const PrimitiveArray<T> &a) { return detail::aggregate(ACU_MAX, a); }
// product (aggregate.rs:953): mul_wrapping for integers; bit_and / bit_or / bit_xor (aggregate.rs:788-875): integers only
template <class T> std::optional<T> product(const PrimitiveArray<T> &a) { return detail::aggregate(ACU_PRODUCT, a); }
template <class T> std::optional<T> bit_and(const PrimitiveArray<T> &a) { return detail::aggregate(ACU_BIT_AND, a); }
template <class T> std::optional<T> bit_or(const PrimitiveArray<T> &a) { return detail::aggregate(ACU_BIT_OR, a); }
template <class T> std::optional<T> bit_xor(const PrimitiveArray<T> &a) { return detail::aggregate(ACU_BIT_XOR, a); }
namespace detail {
template <class T>
Result<std::optional<T>> checked_fold(acu_status (*fn)(acu_ctx *, acu_dtype, const acu_array *, uint64_t *, int64_t *),
                                      const PrimitiveArray<T> &a) {
  uint64_t bits = 0;
  int64_t valid = 0;
  acu_array v = a.view();
  acu_status st = fn(Context::get().raw(), NativeOf<T>::code, &v, &bits, &valid);
  if (st != ACU_OK) return Context::get().last_error(st);
  if (valid == 0) return std::optional<T>(std::nullopt);
  T out;
  std::memcpy(&out, &bits, sizeof(T));
  return std::optional<T>(out);
}
}  // namespace detail
// sum_checked (aggregate.rs:897-937): Ok(None) when every row is null, Err(ArithmeticOverflow) at the first overflowing add
template <class T> Result<std::optional<T>> sum_checked(const PrimitiveArray<T> &a) { return detail::checked_fold(acu_sum_checked, a); }
// product_checked (aggregate.rs:963-1001): Err(ArithmeticOverflow) at the first valid row whose running product overflows
template <class T> Result<std::optional<T>> product_checked(const PrimitiveArray<T> &a) { return detail::checked_fold(acu_product_checked, a); }

// min_string / max_string, min_string_view / max_string_view (aggregate.rs:520-568): the device returns the lowest row
// holding the extremal value; its bytes are copied out (an owned value where the reference borrows from the array).
namespace detail {
inline std::optional<std::string> string_extreme(acu_agg_op op, const StringArray &a) {
  acu_bytes_array b{};
  b.offsets = a.offsets().data();
  b.data = static_cast<const uint8_t *>(a.value_data().data());
  b.nulls = a.view();
  int64_t row = -1, valid = 0;
  Context &c = Context::get();
  const acu_status st = acu_aggregate_bytes(c.raw(), 4, op, &b, &row, &valid);
  if (st != ACU_OK) throw std::runtime_error(c.last_error(st).message);
  if (row < 0) return std::nullopt;
  int32_t se[2];
  acu_memcpy_d2h(c.raw(), se, static_cast<const int32_t *>(a.offsets().data()) + row, sizeof se);
  std::string out((size_t)(se[1] - se[0]), '\0');
  if (!out.empty()) acu_memcpy_d2h(c.raw(), out.data(), static_cast<const uint8_t *>(a.value_data().data()) + se[0], out.size());
  return out;
}
inline std::optional<std::string> string_view_extreme(acu_agg_op op, const StringViewArray &a) {
  Context &c = Context::get();
  std::vector<const uint8_t *> ptrs;
  for (const auto &b : a.data_buffers()) ptrs.push_back(static_cast<const uint8_t *>(b.buffer.data()));
  std::optional<NullBuffer> nulls = nulls_from_mask(a.valid());  // the mirror keeps view validity on the host
  acu_view_array v{};
  v.views = a.views_ptr();
  v.buffers = ptrs.data();
  v.n_buffers = (int32_t)ptrs.size();
  v.nulls.len = a.len();
  if (nulls) {
    v.nulls.validity = static_cast<const uint8_t *>(nulls->buffer.data());
    v.nulls.null_count = nulls->null_count;
  }
  int64_t row = -1, valid = 0;
  const acu_status st = acu_aggregate_byte_view(c.raw(), op, &v, &row, &valid);
  if (st != ACU_OK) throw std::runtime_error(c.last_error(st).message);
  if (row < 0) return std::nullopt;
  return a.slice(row, 1).to_vec()[0];
}
inline std::optional<bool> boolean_extreme(acu_agg_op op, const BooleanArray &a) {
  acu_array v = a.view();
  int32_t value = -1;
  int64_t valid = 0;
  Context &c = Context::get();
  const acu_status st = acu_aggregate_boolean(c.raw(), op, &v, &value, &valid);
  if (st != ACU_OK) throw std::runtime_error(c.last_error(st).message);
  if (value < 0) return std::nullopt;
  return value != 0;
}
}  // namespace detail
inline std::optional<std::string> min_string(const StringArray &a) { return detail::string_extreme(ACU_MIN, a); }
inline std::optional<std::string> max_string(const StringArray &a) { return detail::string_extreme(ACU_MAX, a); }
inline std::optional<std::string> min_string_view(const StringViewArray &a) { return detail::string_view_extreme(ACU_MIN, a); }
inline std::optional<std::string> max_string_view(const StringViewArray &a) { return detail::string_view_extreme(ACU_MAX, a); }
// min_boolean / max_boolean (aggregate.rs:372-457); bool_and / bool_or are the same functions (:880-889)
inline std::optional<bool> min_boolean(const BooleanArray &a) { return detail::boolean_extreme(ACU_MIN, a); }
inline std::optional<bool> max_boolean(const BooleanArray &a) { return detail::boolean_extreme(ACU_MAX, a); }
inline std::optional<bool> bool_and(const BooleanArray &a) { return min_boolean(a); }
inline std::optional<bool> bool_or(const BooleanArray &a) { return max_boolean(a); }

// ---- like (arrow-string/src/like.rs) --------------------------------------------------------------------------
// like / nlike / ilike / nilike / contains / starts_with / ends_with / eq_ignore_ascii_case on Utf8 and Utf8View arrays
// and scalars (the haystack first), through acu_like_bytes / acu_like_byte_view.
namespace like {
namespace detail {
inline Result<BooleanArray> like_strings(acu_like_op op, const StringArray &l, bool ls, const StringArray &r, bool rs) {
  Context &c = Context::get();
  const int64_t n = ls ? r.len() : l.len();
  Buffer vb, nb;
  acu_bytes_array a = kernels::cmp::bytes_view(l, ls), b = kernels::cmp::bytes_view(r, rs);
  acu_array_out o = compute::detail::make_out(vb, nb, acu_bitmap_bytes(std::max<int64_t>(n, 1)), std::max<int64_t>(n, 1));
  const acu_status st = acu_like_bytes(c.raw(), 4, 1, op, &a, &b, &o);
  if (st != ACU_OK) return c.last_error(st);
  return BooleanArray(vb, 0, o.len, compute::detail::out_nulls(o, nb));
}
struct ViewDesc {  // an acu_view_array with the buffer pointer table and the validity it points at
  std::vector<const uint8_t *> ptrs;
  std::optional<NullBuffer> nulls;
  acu_view_array v{};
  ViewDesc(const StringViewArray &a, bool scalar) : nulls(nulls_from_mask(a.valid())) {
    for (const auto &b : a.data_buffers()) ptrs.push_back(static_cast<const uint8_t *>(b.buffer.data()));
    v.views = a.views_ptr();
    v.buffers = ptrs.data();
    v.n_buffers = (int32_t)ptrs.size();
    v.nulls.len = a.len();
    v.nulls.is_scalar = scalar ? 1 : 0;
    if (nulls) {
      v.nulls.validity = static_cast<const uint8_t *>(nulls->buffer.data());
      v.nulls.null_count = nulls->null_count;
    }
  }
};
inline Result<BooleanArray> like_views(acu_like_op op, const StringViewArray &l, bool ls, const StringViewArray &r, bool rs) {
  Context &c = Context::get();
  const int64_t n = ls ? r.len() : l.len();
  Buffer vb, nb;
  const ViewDesc a(l, ls), b(r, rs);
  acu_array_out o = compute::detail::make_out(vb, nb, acu_bitmap_bytes(std::max<int64_t>(n, 1)), std::max<int64_t>(n, 1));
  const acu_status st = acu_like_byte_view(c.raw(), 1, op, &a.v, &b.v, &o);
  if (st != ACU_OK) return c.last_error(st);
  return BooleanArray(vb, 0, o.len, compute::detail::out_nulls(o, nb));
}
}  // namespace detail
#define ACU_LIKE_FN(NAME, OP)                                                                                                     \
  inline Result<BooleanArray> NAME(const StringArray &l, const StringArray &r) { return detail::like_strings(OP, l, false, r, false); } \
  inline Result<BooleanArray> NAME(const StringArray &l, const Scalar<StringArray> &r) { return detail::like_strings(OP, l, false, r.array, true); } \
  inline Result<BooleanArray> NAME(const Scalar<StringArray> &l, const StringArray &r) { return detail::like_strings(OP, l.array, true, r, false); } \
  inline Result<BooleanArray> NAME(const Scalar<StringArray> &l, const Scalar<StringArray> &r) { return detail::like_strings(OP, l.array, true, r.array, true); } \
  inline Result<BooleanArray> NAME(const StringViewArray &l, const StringViewArray &r) { return detail::like_views(OP, l, false, r, false); } \
  inline Result<BooleanArray> NAME(const StringViewArray &l, const Scalar<StringViewArray> &r) { return detail::like_views(OP, l, false, r.array, true); } \
  inline Result<BooleanArray> NAME(const Scalar<StringViewArray> &l, const StringViewArray &r) { return detail::like_views(OP, l.array, true, r, false); } \
  inline Result<BooleanArray> NAME(const Scalar<StringViewArray> &l, const Scalar<StringViewArray> &r) { return detail::like_views(OP, l.array, true, r.array, true); }
ACU_LIKE_FN(like, ACU_LIKE) ACU_LIKE_FN(nlike, ACU_NLIKE) ACU_LIKE_FN(ilike, ACU_ILIKE) ACU_LIKE_FN(nilike, ACU_NILIKE)
ACU_LIKE_FN(contains, ACU_CONTAINS) ACU_LIKE_FN(starts_with, ACU_STARTS_WITH) ACU_LIKE_FN(ends_with, ACU_ENDS_WITH)
ACU_LIKE_FN(eq_ignore_ascii_case, ACU_EQ_IGNORE_ASCII_CASE)
#undef ACU_LIKE_FN
}  // namespace like

// ---- length / substring (arrow-string/src/length.rs, substring.rs) ----------------------------------------------
// length / bit_length / substring on Utf8 (StringArray) and Utf8View (StringViewArray) arrays, substring_by_char on Utf8,
// through acu_length_bytes / acu_length_byte_view / acu_substring_bytes / acu_substring_by_char / acu_substring_byte_view.
// A view result shares the input's data buffers (a long value keeps its buffer index with an advanced offset); the
// reference's StringViewBuilder copies it into new buffers, and the logical values are equal.
namespace detail {
inline Result<Int32Array> length_strings(acu_length_op op, const StringArray &a) {
  Context &c = Context::get();
  Buffer vb, nb;
  const acu_bytes_array x = kernels::cmp::bytes_view(a, false);
  acu_array_out o = make_out(vb, nb, (size_t)std::max<int64_t>(a.len(), 1) * 4, a.len());
  const acu_status st = acu_length_bytes(c.raw(), 4, op, &x, &o);
  if (st != ACU_OK) return c.last_error(st);
  return Int32Array(vb, o.len, out_nulls(o, nb));
}
inline Result<Int32Array> length_views(acu_length_op op, const StringViewArray &a) {
  Context &c = Context::get();
  Buffer vb, nb;
  const like::detail::ViewDesc x(a, false);
  acu_array_out o = make_out(vb, nb, (size_t)std::max<int64_t>(a.len(), 1) * 4, a.len());
  const acu_status st = acu_length_byte_view(c.raw(), op, &x.v, &o);
  if (st != ACU_OK) return c.last_error(st);
  return Int32Array(vb, o.len, out_nulls(o, nb));
}
// The two-phase byte-array call: the offsets and the byte count, then the bytes.
template <class F>
inline Result<StringArray> substring_two_phase(const StringArray &a, F call) {
  Context &c = Context::get();
  const acu_bytes_array x = kernels::cmp::bytes_view(a, false);
  Buffer offs = Buffer::allocate((size_t)(a.len() + 1) * 4), nb = Buffer::allocate(acu_bitmap_bytes(std::max<int64_t>(a.len(), 1)));
  acu_array_out o{};
  o.validity = static_cast<uint8_t *>(nb.data());
  int64_t total = 0;
  acu_status st = call(&x, offs.data(), nullptr, 0, &total, &o);
  if (st != ACU_OK) return c.last_error(st);
  Buffer data = Buffer::allocate((size_t)total);
  st = call(&x, offs.data(), static_cast<uint8_t *>(data.data()), total, &total, &o);
  if (st != ACU_OK) return c.last_error(st);
  return StringArray(offs, data, o.len, out_nulls(o, nb));
}
}  // namespace detail
inline Result<Int32Array> length(const StringArray &a) { return detail::length_strings(ACU_LENGTH, a); }
inline Result<Int32Array> bit_length(const StringArray &a) { return detail::length_strings(ACU_BIT_LENGTH, a); }
inline Result<Int32Array> length(const StringViewArray &a) { return detail::length_views(ACU_LENGTH, a); }
inline Result<Int32Array> bit_length(const StringViewArray &a) { return detail::length_views(ACU_BIT_LENGTH, a); }

// substring(array, start, length) (substring.rs:73-118); start / length count bytes.
inline Result<StringArray> substring(const StringArray &a, int64_t start, std::optional<uint64_t> length = std::nullopt) {
  const int64_t data_len = (int64_t)a.value_data().len();
  return detail::substring_two_phase(a, [&](const acu_bytes_array *x, void *offs, uint8_t *data, int64_t cap, int64_t *total, acu_array_out *o) {
    return acu_substring_bytes(Context::get().raw(), 4, 1, start, length.has_value(), length.value_or(0), x, data_len, offs, data, cap, total, o);
  });
}
inline Result<StringViewArray> substring(const StringViewArray &a, int64_t start, std::optional<uint64_t> length = std::nullopt) {
  Context &c = Context::get();
  const like::detail::ViewDesc x(a, false);
  Buffer views = Buffer::allocate((size_t)std::max<int64_t>(a.len(), 1) * 16), nb = Buffer::allocate(acu_bitmap_bytes(std::max<int64_t>(a.len(), 1)));
  acu_array_out o{};
  o.validity = static_cast<uint8_t *>(nb.data());
  const acu_status st = acu_substring_byte_view(c.raw(), 1, start, length.has_value(), length.value_or(0), &x.v, views.data(), &o);
  if (st != ACU_OK) return c.last_error(st);
  return StringViewArray(views, 0, a.len(), a.data_buffers(), a.valid());  // null slots stay null
}
// substring_by_char(array, start, length) (substring.rs:144-165); start / length count chars.
inline Result<StringArray> substring_by_char(const StringArray &a, int64_t start, std::optional<uint64_t> length = std::nullopt) {
  return detail::substring_two_phase(a, [&](const acu_bytes_array *x, void *offs, uint8_t *data, int64_t cap, int64_t *total, acu_array_out *o) {
    return acu_substring_by_char(Context::get().raw(), 4, start, length.has_value(), length.value_or(0), x, offs, data, cap, total, o);
  });
}

// ---- concat_elements (arrow-string/src/concat_elements.rs) -------------------------------------------------------
// concat_elements_utf8 / concat_elements_utf8_many on Utf8 (StringArray), concat_elements_string_view_array on Utf8View
// (StringViewArray) and concat_elements_dyn, through acu_concat_elements_bytes / _bytes_many / _byte_view. A view result
// has the reference's layout: one new data buffer, none when no result is longer than 12 bytes.
namespace detail {
// The two-phase byte-array call over n rows: the offsets and the byte count, then the bytes.
template <class F>
inline Result<StringArray> concat_two_phase(int64_t n, F call) {
  Context &c = Context::get();
  Buffer offs = Buffer::allocate((size_t)(n + 1) * 4), nb = Buffer::allocate(acu_bitmap_bytes(std::max<int64_t>(n, 1)));
  acu_array_out o{};
  o.validity = static_cast<uint8_t *>(nb.data());
  int64_t total = 0;
  acu_status st = call(offs.data(), nullptr, 0, &total, &o);
  if (st != ACU_OK) return c.last_error(st);
  Buffer data = Buffer::allocate((size_t)std::max<int64_t>(total, 1));
  st = call(offs.data(), static_cast<uint8_t *>(data.data()), total, &total, &o);
  if (st != ACU_OK) return c.last_error(st);
  return StringArray(offs, data, o.len, out_nulls(o, nb));
}
}  // namespace detail

inline Result<StringArray> concat_elements_utf8(const StringArray &left, const StringArray &right) {
  const acu_bytes_array l = kernels::cmp::bytes_view(left, false), r = kernels::cmp::bytes_view(right, false);
  return detail::concat_two_phase(left.len(), [&](void *offs, uint8_t *data, int64_t cap, int64_t *total, acu_array_out *o) {
    return acu_concat_elements_bytes(Context::get().raw(), 4, &l, &r, offs, data, cap, total, o);
  });
}

inline Result<StringArray> concat_elements_utf8_many(const std::vector<const StringArray *> &arrays) {
  std::vector<acu_bytes_array> xs;
  for (const StringArray *a : arrays) xs.push_back(kernels::cmp::bytes_view(*a, false));
  return detail::concat_two_phase(arrays.empty() ? 0 : arrays[0]->len(), [&](void *offs, uint8_t *data, int64_t cap, int64_t *total, acu_array_out *o) {
    return acu_concat_elements_bytes_many(Context::get().raw(), 4, (int32_t)xs.size(), xs.data(), offs, data, cap, total, o);
  });
}

inline Result<StringViewArray> concat_elements_string_view_array(const StringViewArray &left, const StringViewArray &right) {
  Context &c = Context::get();
  const like::detail::ViewDesc l(left, false), r(right, false);
  const int64_t n = left.len();
  Buffer views = Buffer::allocate((size_t)std::max<int64_t>(n, 1) * 16), nb = Buffer::allocate(acu_bitmap_bytes(std::max<int64_t>(n, 1)));
  acu_array_out o{};
  o.validity = static_cast<uint8_t *>(nb.data());
  int64_t total = 0;
  acu_status st = acu_concat_elements_byte_view(c.raw(), &l.v, &r.v, nullptr, nullptr, 0, &total, &o);
  if (st != ACU_OK) return c.last_error(st);
  Buffer data = Buffer::allocate((size_t)std::max<int64_t>(total, 1));
  st = acu_concat_elements_byte_view(c.raw(), &l.v, &r.v, views.data(), static_cast<uint8_t *>(data.data()), total, &total, &o);
  if (st != ACU_OK) return c.last_error(st);
  std::vector<bool> valid((size_t)o.len, true);
  if (o.has_validity) {
    std::vector<uint8_t> bits(acu_bitmap_bytes(o.len));
    nb.to_host(bits.data(), bits.size());
    for (size_t i = 0; i < valid.size(); ++i) valid[i] = (bits[i >> 3] >> (i & 7)) & 1;
  }
  std::vector<ViewDataBuffer> bufs;
  if (total > 0) bufs.push_back(ViewDataBuffer{data, (size_t)total, (size_t)total});
  return StringViewArray(views, 0, o.len, std::move(bufs), std::move(valid));
}

// concat_elements_dyn (concat_elements.rs:419-476): Utf8 operands; any other pair fails as the reference does.
inline Result<ArrayRef> concat_elements_dyn(const Array &left, const Array &right) {
  if (left.data_type() != right.data_type())
    return ArrowError{ACU_ERR_COMPUTE, std::string("Compute error: Cannot concat arrays of different types: ") + detail::dtype_display(left.data_type()) +
                                           " != " + detail::dtype_display(right.data_type())};
  if (left.data_type() != DataType::Utf8)
    return ArrowError{ACU_ERR_NOT_YET_IMPLEMENTED, std::string("Not yet implemented: concat not supported for ") + detail::dtype_display(left.data_type())};
  auto r = concat_elements_utf8(static_cast<const StringArray &>(left), static_cast<const StringArray &>(right));
  if (r.is_err()) return r.unwrap_err();
  return ArrayRef(std::make_shared<StringArray>(r.unwrap()));
}
inline Result<StringViewArray> concat_elements_dyn(const StringViewArray &left, const StringViewArray &right) {
  return concat_elements_string_view_array(left, right);
}


// ---- nullif / zip (arrow-select/src/nullif.rs:44-113, zip.rs:99-226) -------------------------------------------
namespace detail {
// The same buffers with another NullBuffer (ArrayData::into_builder().nulls(..): nullif shares the value buffers)
inline ArrayRef with_nulls(const Array &a, std::optional<NullBuffer> nulls);
}  // namespace detail

// nullif(left, right): validity &= !(right is Some(true)); values shared (zero copy)
inline Result<ArrayRef> nullif(const Array &left, const BooleanArray &right) {
  Context &c = Context::get();
  Buffer vb, nb;
  acu_array l = left.view(), r = right.view();
  acu_array_out o = detail::make_out(vb, nb, 16, std::max<int64_t>(left.len(), 1));
  acu_status st = acu_nullif(c.raw(), &l, &r, &o);
  if (st != ACU_OK) return c.last_error(st);
  if (left.len() == 0) return detail::with_nulls(left, left.nulls());
  return detail::with_nulls(left, detail::out_nulls(o, nb));
}

namespace detail {
// zip of Utf8 (StringArray), Boolean and FixedSizeBinary operands: acu_zip_bytes / acu_zip_boolean / acu_zip_fixed_size_binary
template <class A> struct zip_column : std::false_type {};
template <> struct zip_column<StringArray> : std::true_type {};
template <> struct zip_column<BooleanArray> : std::true_type {};
template <> struct zip_column<FixedSizeBinaryArray> : std::true_type {};
template <class D> using datum_array_t = std::decay_t<decltype(datum_array(std::declval<const D &>()))>;

inline Result<ArrayRef> zip_column_impl(const BooleanArray &mask, const StringArray &t, bool ts, const StringArray &f, bool fs) {
  const acu_bytes_array tb = kernels::cmp::bytes_view(t, ts), fb = kernels::cmp::bytes_view(f, fs);
  const acu_array m = mask.view();
  const int64_t n = mask.len();
  Context &c = Context::get();
  Buffer offs = Buffer::allocate((size_t)(n + 1) * 4), nb = Buffer::allocate(acu_bitmap_bytes(std::max<int64_t>(n, 1)));
  acu_array_out o{};
  o.validity = static_cast<uint8_t *>(nb.data());
  int64_t total = 0;
  acu_status st = acu_zip_bytes(c.raw(), 4, &m, &tb, &fb, offs.data(), nullptr, 0, &total, &o);
  if (st != ACU_OK) return c.last_error(st);
  Buffer data = Buffer::allocate((size_t)std::max<int64_t>(total, 1));
  st = acu_zip_bytes(c.raw(), 4, &m, &tb, &fb, offs.data(), static_cast<uint8_t *>(data.data()), total, &total, &o);
  if (st != ACU_OK) return c.last_error(st);
  return ArrayRef(std::make_shared<StringArray>(offs, data, o.len, out_nulls(o, nb)));
}

inline Result<ArrayRef> zip_column_impl(const BooleanArray &mask, const BooleanArray &t, bool ts, const BooleanArray &f, bool fs) {
  Context &c = Context::get();
  const int64_t n = mask.len();
  Buffer vb, nb;
  acu_array m = mask.view(), tv = t.view(ts), fv = f.view(fs);
  acu_array_out o = make_out(vb, nb, acu_bitmap_bytes(std::max<int64_t>(n, 1)), std::max<int64_t>(n, 1));
  acu_status st = acu_zip_boolean(c.raw(), &m, &tv, &fv, &o);
  if (st != ACU_OK) return c.last_error(st);
  return ArrayRef(std::make_shared<BooleanArray>(vb, 0, o.len, out_nulls(o, nb)));
}

inline Result<ArrayRef> zip_column_impl(const BooleanArray &mask, const FixedSizeBinaryArray &t, bool ts, const FixedSizeBinaryArray &f,
                                        bool fs) {
  if (t.value_length() != f.value_length())  // FixedSizeBinary(4) vs (5): zip.rs:117-121
    return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: arguments need to have the same data type"};
  Context &c = Context::get();
  const int64_t n = mask.len();
  Buffer vb, nb;
  acu_array m = mask.view(), tv = t.view(ts), fv = f.view(fs);
  acu_array_out o = make_out(vb, nb, (size_t)std::max<int64_t>(n, 1) * t.value_length(), std::max<int64_t>(n, 1));
  acu_status st = acu_zip_fixed_size_binary(c.raw(), t.value_length(), &m, &tv, &fv, &o);
  if (st != ACU_OK) return c.last_error(st);
  return ArrayRef(std::make_shared<FixedSizeBinaryArray>(t.value_length(), vb, o.len, out_nulls(o, nb)));
}
}  // namespace detail

// zip(mask, truthy, falsy) for arrays / scalars of one type: primitive, Utf8 (StringArray), Boolean or FixedSizeBinary
template <class L, class R>
Result<ArrayRef> zip(const BooleanArray &mask, const L &truthy, const R &falsy) {
  if constexpr (detail::zip_column<detail::datum_array_t<L>>::value)
    return detail::zip_column_impl(mask, datum_array(truthy), datum_is_scalar(truthy), datum_array(falsy), datum_is_scalar(falsy));
  const auto &t = datum_array(truthy);
  const auto &f = datum_array(falsy);
  if (t.data_type() != f.data_type())  // zip.rs:117-121
    return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Invalid argument error: arguments need to have the same data type"};
  Context &c = Context::get();
  const int64_t n = mask.len();
  Buffer vb, nb;
  acu_array m = mask.view(), tv = t.view(datum_is_scalar(truthy)), fv = f.view(datum_is_scalar(falsy));
  acu_array_out o = detail::make_out(vb, nb, (size_t)std::max<int64_t>(n, 1) * dtype_width(t.data_type()), std::max<int64_t>(n, 1));
  acu_status st = acu_zip(c.raw(), dtype_width(t.data_type()), &m, &tv, &fv, &o);
  if (st != ACU_OK) return c.last_error(st);
  return detail::make_primitive(t.data_type(), vb, o.len, detail::out_nulls(o, nb));
}

// zip of Utf8View operands (StringViewArray, a data-buffer list of its own): the result references truthy's buffers,
// falsy's, both (truthy's first) or none, as acu_zip_byte_view reports
namespace detail {
inline Result<StringViewArray> zip_views(const BooleanArray &mask, const StringViewArray &t, bool ts, const StringViewArray &f, bool fs) {
  Context &c = Context::get();
  const like::detail::ViewDesc tv(t, ts), fv(f, fs);
  const acu_array m = mask.view();
  const int64_t n = mask.len();
  Buffer views = Buffer::allocate((size_t)std::max<int64_t>(n, 1) * 16), nb = Buffer::allocate(acu_bitmap_bytes(std::max<int64_t>(n, 1)));
  acu_array_out o{};
  o.validity = static_cast<uint8_t *>(nb.data());
  int32_t which = ACU_ZIP_BUFFERS_NONE;
  const acu_status st = acu_zip_byte_view(c.raw(), &m, &tv.v, &fv.v, views.data(), &o, &which);
  if (st != ACU_OK) return c.last_error(st);
  std::vector<bool> valid((size_t)o.len, true);
  if (o.has_validity) {
    std::vector<uint8_t> bits(acu_bitmap_bytes(o.len));
    nb.to_host(bits.data(), bits.size());
    for (size_t i = 0; i < valid.size(); ++i) valid[i] = (bits[i >> 3] >> (i & 7)) & 1;
  }
  std::vector<ViewDataBuffer> bufs;
  if (which == ACU_ZIP_BUFFERS_TRUTHY || which == ACU_ZIP_BUFFERS_BOTH) bufs = t.data_buffers();
  if (which == ACU_ZIP_BUFFERS_FALSY || which == ACU_ZIP_BUFFERS_BOTH)
    bufs.insert(bufs.end(), f.data_buffers().begin(), f.data_buffers().end());
  return StringViewArray(views, 0, o.len, std::move(bufs), std::move(valid));
}
}  // namespace detail
inline Result<StringViewArray> zip(const BooleanArray &mask, const StringViewArray &t, const StringViewArray &f) {
  return detail::zip_views(mask, t, false, f, false);
}
inline Result<StringViewArray> zip(const BooleanArray &mask, const Scalar<StringViewArray> &t, const StringViewArray &f) {
  return detail::zip_views(mask, t.array, true, f, false);
}
inline Result<StringViewArray> zip(const BooleanArray &mask, const StringViewArray &t, const Scalar<StringViewArray> &f) {
  return detail::zip_views(mask, t, false, f.array, true);
}
inline Result<StringViewArray> zip(const BooleanArray &mask, const Scalar<StringViewArray> &t, const Scalar<StringViewArray> &f) {
  return detail::zip_views(mask, t.array, true, f.array, true);
}

// ---- concat / concat_batches (arrow-select/src/concat.rs:495-640) -----------------------------------------------
inline Result<ArrayRef> concat(const std::vector<const Array *> &arrays) {
  Context &c = Context::get();
  if (arrays.empty()) return ArrowError{ACU_ERR_COMPUTE, "Compute error: concat requires input of at least one array"};
  const DataType dt = arrays[0]->data_type();
  for (const Array *a : arrays)
    if (a->data_type() != dt)  // concat.rs:505-535
      return ArrowError{ACU_ERR_INVALID_ARGUMENT, std::string("Invalid argument error: It is not possible to concatenate arrays of different data types (") +
                                                       detail::dtype_display(dt) + ", " + detail::dtype_display(a->data_type()) + ")."};
  std::vector<acu_column> cols;
  int64_t rows = 0, bytes = 0;
  for (const Array *a : arrays) {
    cols.push_back(detail::column_view(*a));
    rows += a->len();
    if (dt == DataType::Utf8) bytes += (int64_t)static_cast<const StringArray *>(a)->value_data().len();
  }
  std::vector<ArrayRef> proto{detail::with_nulls(*arrays[0], arrays[0]->nulls())};
  detail::BatchOutputs outs;
  outs.allocate(proto, std::max<int64_t>(rows, 1), {bytes});
  acu_status st = acu_concat(c.raw(), (int32_t)cols.size(), cols.data(), outs.outs.data());
  if (st != ACU_OK) return c.last_error(st);
  return outs.wrap(proto)[0];
}

inline Result<RecordBatch> concat_batches(const Schema &schema, const std::vector<const RecordBatch *> &batches) {
  if (batches.empty()) {  // RecordBatch::new_empty(schema)
    std::vector<ArrayRef> empty;
    for (const Field &f : schema) {
      if (f.data_type == DataType::Boolean) empty.push_back(std::make_shared<BooleanArray>(BooleanArray::from(std::vector<bool>{})));
      else if (f.data_type == DataType::Utf8) empty.push_back(std::make_shared<StringArray>(StringArray::from(std::vector<std::string>{})));
      else empty.push_back(detail::make_primitive(f.data_type, Buffer::allocate(16), 0, std::nullopt));
    }
    return RecordBatch(schema, std::move(empty), 0);
  }
  std::vector<ArrayRef> cols;
  for (size_t i = 0; i < schema.size(); ++i) {
    std::vector<const Array *> field;
    for (const RecordBatch *b : batches) field.push_back(b->column(i).get());
    auto r = concat(field);
    if (r.is_err()) return r.unwrap_err();
    cols.push_back(r.unwrap());
  }
  return RecordBatch::try_new(schema, std::move(cols));
}
}  // namespace compute

// downcast helpers (as_primitive::<T>() etc.)
template <class T> const PrimitiveArray<T> &as_primitive(const ArrayRef &a) { return dynamic_cast<const PrimitiveArray<T> &>(*a); }
inline const BooleanArray &as_boolean(const ArrayRef &a) { return dynamic_cast<const BooleanArray &>(*a); }
inline const StringArray &as_string(const ArrayRef &a) { return dynamic_cast<const StringArray &>(*a); }


namespace compute { namespace detail {
inline ArrayRef with_nulls(const Array &a, std::optional<NullBuffer> nulls) {
  if (a.data_type() == DataType::Boolean) {
    const auto &b = static_cast<const BooleanArray &>(a);
    acu_array v = b.view();
    return std::make_shared<BooleanArray>(b.bits(), v.values_offset, b.len(), std::move(nulls));
  }
  if (a.data_type() == DataType::Utf8) {
    const auto &s = static_cast<const StringArray &>(a);
    return std::make_shared<StringArray>(s.offsets(), s.value_data(), s.len(), std::move(nulls));
  }
  switch (a.data_type()) {
#define ACU_WN(DT, T) case DataType::DT: { const auto &p = static_cast<const PrimitiveArray<T> &>(a); \
    return std::make_shared<PrimitiveArray<T>>(p.buffer(), p.len(), std::move(nulls), p.elem_offset()); }
    ACU_WN(Int8, int8_t) ACU_WN(Int16, int16_t) ACU_WN(Int32, int32_t) ACU_WN(Int64, int64_t) ACU_WN(UInt8, uint8_t)
    ACU_WN(UInt16, uint16_t) ACU_WN(UInt32, uint32_t) ACU_WN(UInt64, uint64_t) ACU_WN(Float32, float)
#undef ACU_WN
    default: { const auto &p = static_cast<const PrimitiveArray<double> &>(a);
      return std::make_shared<PrimitiveArray<double>>(p.buffer(), p.len(), std::move(nulls), p.elem_offset()); }
  }
}
} }  // namespace compute::detail

// ---------------------------------------------------------------------------------------
// ipc::StreamReader (arrow-ipc/src/reader.rs:1529-1671): record batches decoded straight into HBM.
// Every batch's body is ONE host->device copy; the columns own a share of that device buffer.
// ---------------------------------------------------------------------------------------
namespace ipc {
class StreamReader {
 public:
  // StreamReader::try_new(reader, None) over an in-memory stream
  static Result<StreamReader> try_new(std::vector<uint8_t> stream) {
    StreamReader r;
    r.bytes_ = std::make_shared<std::vector<uint8_t>>(std::move(stream));
    Context &c = Context::get();
    acu_ipc_stream *s = nullptr;
    int32_t n = 0;
    acu_status st = acu_ipc_stream_open(c.raw(), r.bytes_->data(), (int64_t)r.bytes_->size(), &s, &n);
    if (st != ACU_OK) return c.last_error(st);
    r.stream_ = std::shared_ptr<acu_ipc_stream>(s, [](acu_ipc_stream *q) { acu_ipc_stream_close(Context::get().raw(), q); });
    for (int32_t i = 0; i < n; ++i) {
      int32_t kind, width, dtype, nullable;
      const char *name;
      acu_ipc_stream_field(s, i, &kind, &width, &dtype, &nullable, &name);
      Field f;
      f.name = name;
      f.nullable = nullable != 0;
      if (kind == ACU_COL_BOOLEAN) f.data_type = DataType::Boolean;
      else if (kind == ACU_COL_BYTES && width == 4) f.data_type = DataType::Utf8;
      else if (kind == ACU_COL_PRIMITIVE) f.data_type = (DataType)dtype;
      else return ArrowError{ACU_ERR_NOT_YET_IMPLEMENTED, "Not yet implemented: IPC field '" + f.name + "': LargeUtf8 in the C++ mirror"};
      r.schema_.push_back(f);
    }
    return r;
  }
  const Schema &schema() const { return schema_; }
  bool is_finished() const { return finished_; }
  // Iterator::next: Ok(None) at the end of the stream
  Result<std::optional<RecordBatch>> next() {
    Context &c = Context::get();
    std::vector<acu_column> cols(schema_.size());
    int64_t rows = -1;
    acu_status st = acu_ipc_stream_next(c.raw(), stream_.get(), cols.data(), &rows);
    if (st != ACU_OK) return c.last_error(st);
    if (rows < 0) { finished_ = true; return std::optional<RecordBatch>(); }
    // the views point into the stream's device buffer, which the next call reuses: give the batch its own copy
    std::vector<ArrayRef> out;
    for (size_t i = 0; i < cols.size(); ++i) {
      const acu_column &col = cols[i];
      const DataType dt = schema_[i].data_type;
      std::optional<NullBuffer> nulls;
      if (col.array.validity) {
        Buffer nb = Buffer::allocate(acu_bitmap_bytes(rows));
        acu_memcpy_d2d(c.raw(), nb.data(), col.array.validity, (size_t)((rows + 7) / 8));
        nulls = NullBuffer{nb, 0, rows, col.array.null_count};
      }
      if (dt == DataType::Boolean) {
        Buffer vb = Buffer::allocate(acu_bitmap_bytes(rows));
        acu_memcpy_d2d(c.raw(), vb.data(), col.array.values, (size_t)((rows + 7) / 8));
        out.push_back(std::make_shared<BooleanArray>(vb, 0, rows, nulls));
      } else if (dt == DataType::Utf8) {
        Buffer ob = Buffer::allocate((size_t)(rows + 1) * 4);
        acu_memcpy_d2d(c.raw(), ob.data(), col.array.values, (size_t)(rows + 1) * 4);
        int32_t last = 0;
        if (rows > 0) acu_memcpy_d2h(c.raw(), &last, static_cast<const int32_t *>(col.array.values) + rows, 4);
        Buffer db = Buffer::allocate((size_t)last);
        if (last) acu_memcpy_d2d(c.raw(), db.data(), col.data, (size_t)last);
        out.push_back(std::make_shared<StringArray>(ob, db, rows, nulls));
      } else {
        const size_t bytes = (size_t)rows * dtype_width(dt);
        Buffer vb = Buffer::allocate(bytes);
        if (bytes) acu_memcpy_d2d(c.raw(), vb.data(), col.array.values, bytes);
        out.push_back(compute::detail::make_primitive(dt, vb, rows, nulls));
      }
    }
    return std::optional<RecordBatch>(RecordBatch(schema_, std::move(out), rows));
  }
 private:
  std::shared_ptr<std::vector<uint8_t>> bytes_;
  std::shared_ptr<acu_ipc_stream> stream_;
  Schema schema_;
  bool finished_ = false;
};
}  // namespace ipc

// ---------------------------------------------------------------------------------------
// parquet::arrow::arrow_reader::{ArrowPredicate, ArrowPredicateFn, RowFilter} (parquet/src/arrow/arrow_reader/filter.rs:29-200):
// the caller of the hot path. Predicates are applied in order, each one to the rows that survived the previous ones (late
// materialisation: evaluate_predicate, parquet/src/arrow/arrow_reader/mod.rs), `false` and `null` both drop the row; the
// final selection is applied to the projected batch with filter_record_batch. Here every intermediate lives in HBM.
// ---------------------------------------------------------------------------------------
namespace parquet {
class ArrowPredicate {
 public:
  virtual ~ArrowPredicate() = default;
  // columns (indices into the batch) this predicate needs: ProjectionMask
  virtual const std::vector<size_t> &projection() const = 0;
  // must return a BooleanArray of batch.num_rows() rows
  virtual Result<BooleanArray> evaluate(const RecordBatch &batch) = 0;
};
class ArrowPredicateFn : public ArrowPredicate {
 public:
  using Fn = std::function<Result<BooleanArray>(const RecordBatch &)>;
  ArrowPredicateFn(std::vector<size_t> projection, Fn f) : projection_(std::move(projection)), f_(std::move(f)) {}
  const std::vector<size_t> &projection() const override { return projection_; }
  Result<BooleanArray> evaluate(const RecordBatch &batch) override { return f_(batch); }
 private:
  std::vector<size_t> projection_;
  Fn f_;
};
class RowFilter {
 public:
  explicit RowFilter(std::vector<std::shared_ptr<ArrowPredicate>> predicates) : predicates_(std::move(predicates)) {}
  // Decode-time filtering of one (already decoded, device-resident) batch: returns the rows for which every predicate is true.
  Result<RecordBatch> apply(const RecordBatch &batch) const {
    RecordBatch cur = batch;
    for (const auto &p : predicates_) {
      Schema ps;
      std::vector<ArrayRef> pc;
      for (size_t i : p->projection()) { ps.push_back(cur.schema()[i]); pc.push_back(cur.column(i)); }
      RecordBatch projected(ps, pc, cur.num_rows());
      auto mask = p->evaluate(projected);
      if (mask.is_err()) return mask.unwrap_err();
      BooleanArray m = mask.unwrap();
      if (m.len() != cur.num_rows())  // arrow_reader/mod.rs: "ArrowPredicate predicate returned {} rows, expected {}"
        return ArrowError{ACU_ERR_INVALID_ARGUMENT, "Parquet argument error: General error: ArrowPredicate predicate returned " +
                                                         std::to_string(m.len()) + " rows, expected " + std::to_string(cur.num_rows())};
      auto next = compute::filter_record_batch(cur, m);  // prep_null_mask_filter: null selects nothing
      if (next.is_err()) return next.unwrap_err();
      cur = next.unwrap();
    }
    return cur;
  }
 private:
  std::vector<std::shared_ptr<ArrowPredicate>> predicates_;
};
}  // namespace parquet

}  // namespace arrow_cuda
