// test_host.cpp — the reference's unit tests, re-expressed against the C++ host mirror
// (arrow_cuda.hpp). Each test cites the arrow-rs test it transcribes; assertions are on the
// same values and the same error strings. Runs on a CUDA device (no CPU fallback).
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host   (exit code 0 = all passed)
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <functional>
#include <limits>

#include "arrow_cuda.hpp"

using namespace arrow_cuda;
using namespace arrow_cuda::compute;
namespace numeric = arrow_cuda::compute::kernels::numeric;
namespace cmpk = arrow_cuda::compute::kernels::cmp;

static int g_failed = 0, g_checks = 0;
#define CHECK(cond)                                                                    \
  do {                                                                                 \
    ++g_checks;                                                                        \
    if (!(cond)) { ++g_failed; std::printf("  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); } \
  } while (0)
#define CHECK_EQ(a, b) CHECK((a) == (b))

template <class T> using O = std::optional<T>;
static const std::nullopt_t N = std::nullopt;

// arrow-select/src/filter.rs:1177 test_filter_array_slice
static void test_filter_array_slice() {
  auto a = Int32Array::from(std::vector<int32_t>{5, 6, 7, 8, 9}).slice(1, 4);
  auto b = BooleanArray::from(std::vector<bool>{true, false, false, true});
  auto c = filter(a, b).unwrap();
  const auto &d = as_primitive<int32_t>(c);
  CHECK_EQ(2, d.len());
  CHECK_EQ(6, d.value(0));
  CHECK_EQ(9, d.value(1));
}

// filter.rs:1191 test_filter_array_low_density
static void test_filter_array_low_density() {
  std::vector<int32_t> data;
  std::vector<bool> pred;
  for (int i = 1; i <= 65; ++i) { data.push_back(i); pred.push_back(i % 65 == 0); }
  data.push_back(66); data.push_back(67);
  pred.push_back(false); pred.push_back(true);
  auto c = filter(Int32Array::from(data), BooleanArray::from(pred)).unwrap();
  const auto &d = as_primitive<int32_t>(c);
  CHECK_EQ(2, d.len());
  CHECK_EQ(65, d.value(0));
  CHECK_EQ(67, d.value(1));
}

// filter.rs:1208 test_filter_array_high_density
static void test_filter_array_high_density() {
  std::vector<O<int32_t>> data;
  std::vector<bool> pred;
  for (int i = 1; i <= 65; ++i) { data.push_back(i); pred.push_back(i % 65 != 0); }
  data[1] = N;
  for (O<int32_t> v : {O<int32_t>(66), O<int32_t>(N), O<int32_t>(67), O<int32_t>(N)}) data.push_back(v);
  for (bool b : {false, true, true, true}) pred.push_back(b);
  auto c = filter(Int32Array::from(data), BooleanArray::from(pred)).unwrap();
  const auto &d = as_primitive<int32_t>(c);
  CHECK_EQ(67, d.len());
  CHECK_EQ(3, d.null_count());
  CHECK_EQ(1, d.value(0));
  CHECK(d.is_null(1));
  CHECK_EQ(64, d.value(63));
  CHECK(d.is_null(64));
  CHECK_EQ(67, d.value(65));
}

// filter.rs:1233 / :1254 test_filter_string_array_simple / _with_null
static void test_filter_string_array() {
  auto a = StringArray::from(std::vector<std::string>{"hello", " ", "world", "!"});
  auto c = filter(a, BooleanArray::from(std::vector<bool>{true, false, true, false})).unwrap();
  auto d = as_string(c).to_vec();
  CHECK_EQ(2u, d.size());
  CHECK(d[0] == O<std::string>("hello"));
  CHECK(d[1] == O<std::string>("world"));
  auto a2 = StringArray::from(std::vector<O<std::string>>{std::string("hello"), N, std::string("world"), N});
  auto c2 = filter(a2, BooleanArray::from(std::vector<bool>{true, false, false, true})).unwrap();
  auto d2 = as_string(c2).to_vec();
  CHECK(d2[0] == O<std::string>("hello"));
  CHECK(!d2[1].has_value());
}

// filter.rs:1718 test_null_mask, :1738 test_fast_path
static void test_null_mask_and_fast_path() {
  auto a = Int64Array::from(std::vector<O<int64_t>>{1, 2, N});
  auto mask1 = BooleanArray::from(std::vector<O<bool>>{true, true, N});
  auto out = filter(a, mask1).unwrap();
  CHECK(as_primitive<int64_t>(out).to_vec() == (std::vector<O<int64_t>>{1, 2}));
  auto all = filter(a, BooleanArray::from(std::vector<bool>{true, true, true})).unwrap();
  CHECK(as_primitive<int64_t>(all).to_vec() == (std::vector<O<int64_t>>{1, 2, N}));
  auto none = filter(a, BooleanArray::from(std::vector<bool>{false, false, false})).unwrap();
  CHECK_EQ(0, none->len());
  CHECK(none->data_type() == DataType::Int64);
}

// filter.rs:536-542 error text
static void test_filter_predicate_too_long() {
  auto r = filter(Int32Array::from(std::vector<int32_t>{1, 2}), BooleanArray::from(std::vector<bool>{true, false, true}));
  CHECK(r.is_err());
  CHECK_EQ(r.unwrap_err().to_string(), std::string("Invalid argument error: Filter predicate of length 3 is larger than target array of length 2"));
}

// filter.rs:225-244, :459-478 filter_record_batch: one predicate, every column
static void test_filter_record_batch() {
  Schema schema{{"a", DataType::Int32}, {"b", DataType::Utf8}, {"c", DataType::Float64}};
  std::vector<ArrayRef> cols{
      std::make_shared<Int32Array>(Int32Array::from(std::vector<O<int32_t>>{1, N, 3, 4})),
      std::make_shared<StringArray>(StringArray::from(std::vector<std::string>{"w", "x", "y", "z"})),
      std::make_shared<Float64Array>(Float64Array::from(std::vector<double>{0.5, 1.5, 2.5, 3.5}))};
  auto batch = RecordBatch::try_new(schema, cols).unwrap();
  auto out = filter_record_batch(batch, BooleanArray::from(std::vector<bool>{true, true, false, true})).unwrap();
  CHECK_EQ(3, out.num_rows());
  CHECK(as_primitive<int32_t>(out.column(0)).to_vec() == (std::vector<O<int32_t>>{1, N, 4}));
  CHECK(as_string(out.column(1)).to_vec() == (std::vector<O<std::string>>{std::string("w"), std::string("x"), std::string("z")}));
  CHECK(as_primitive<double>(out.column(2)).to_vec() == (std::vector<O<double>>{0.5, 1.5, 3.5}));
}

// take.rs:1123-1133 take_record_batch (doc example take.rs:1108-1121): every column, same indices; here with a
// repeated index (a Utf8 column that grows) and a null index
static void test_take_record_batch() {
  Schema schema{{"a", DataType::Int32}, {"b", DataType::Utf8}, {"c", DataType::Boolean}};
  std::vector<ArrayRef> cols{
      std::make_shared<Int32Array>(Int32Array::from(std::vector<O<int32_t>>{1, N, 3, 4})),
      std::make_shared<StringArray>(StringArray::from(std::vector<O<std::string>>{std::string("w"), std::string("xx"), N, std::string("zzzz")})),
      std::make_shared<BooleanArray>(BooleanArray::from(std::vector<bool>{true, false, true, false}))};
  auto batch = RecordBatch::try_new(schema, cols).unwrap();
  auto idx = UInt32Array::from(std::vector<O<uint32_t>>{3, 3, N, 0, 1, 2});
  auto out = take_record_batch(batch, idx).unwrap();
  CHECK_EQ(6, out.num_rows());
  CHECK(as_primitive<int32_t>(out.column(0)).to_vec() == (std::vector<O<int32_t>>{4, 4, N, 1, N, 3}));
  CHECK(as_string(out.column(1)).to_vec() ==
        (std::vector<O<std::string>>{std::string("zzzz"), std::string("zzzz"), N, std::string("w"), std::string("xx"), N}));
  CHECK(as_boolean(out.column(2)).to_vec() == (std::vector<O<bool>>{false, false, N, true, false, true}));
  // filter -> take -> same rows as filtering the taken batch's source positions
  auto f = filter_record_batch(batch, BooleanArray::from(std::vector<bool>{true, false, true, true})).unwrap();
  auto t = take_record_batch(f, UInt32Array::from(std::vector<uint32_t>{2, 0})).unwrap();
  CHECK(as_primitive<int32_t>(t.column(0)).to_vec() == (std::vector<O<int32_t>>{4, 1}));
  CHECK(as_string(t.column(1)).to_vec() == (std::vector<O<std::string>>{std::string("zzzz"), std::string("w")}));
}

// arrow-arith/src/boolean.rs:473 test_bool_array_and_kleene_nulls, :514 or_kleene, :422 or, :631 not (sliced), :835 is_null
static void test_boolean_kernels() {
  using namespace arrow_cuda::compute::kernels::boolean;
  using OB = O<bool>;
  auto a = BooleanArray::from(std::vector<OB>{N, N, N, false, false, false, true, true, true});
  auto b = BooleanArray::from(std::vector<OB>{N, false, true, N, false, true, N, false, true});
  CHECK(and_kleene(a, b).unwrap().to_vec() == (std::vector<OB>{N, false, N, false, false, false, N, false, true}));
  CHECK(or_kleene(a, b).unwrap().to_vec() == (std::vector<OB>{N, N, true, N, false, true, true, true, true}));
  CHECK(or_(a, b).unwrap().to_vec() == (std::vector<OB>{N, N, N, N, false, true, N, true, true}));
  CHECK(and_(a, b).unwrap().to_vec() == (std::vector<OB>{N, N, N, N, false, false, N, false, true}));
  auto s = BooleanArray::from(std::vector<OB>{N, true, false, N, true}).slice(1, 4);
  CHECK(not_(s).unwrap().to_vec() == (std::vector<OB>{false, true, N, false}));
  auto i = Int32Array::from(std::vector<O<int32_t>>{1, N, 3, N});
  auto r = is_null(i).unwrap();
  CHECK(r.to_vec() == (std::vector<OB>{false, true, false, true}));
  CHECK(!r.nulls().has_value());
  CHECK(is_not_null(i).unwrap().to_vec() == (std::vector<OB>{true, false, true, false}));
  auto e = and_(BooleanArray::from(std::vector<bool>{true, false}), BooleanArray::from(std::vector<bool>{true}));
  CHECK(e.is_err());
  CHECK_EQ(e.unwrap_err().to_string(), std::string("Compute error: Cannot perform bitwise operation on arrays of different length"));
  // the predicate never leaves the device: cmp -> and_kleene -> filter
  auto x = Int32Array::from(std::vector<O<int32_t>>{5, 1, N, 7, 2});
  auto m = and_kleene(arrow_cuda::compute::kernels::cmp::gt(x, new_scalar<int32_t>(1)).unwrap(), BooleanArray::from(std::vector<bool>{true, true, true, false, true})).unwrap();
  CHECK(as_primitive<int32_t>(filter(x, m).unwrap()).to_vec() == (std::vector<O<int32_t>>{5, 2}));
}

// aggregate.rs:1993 test_sum_checked_overflow (+ the wrapping twin :1985)
static void test_sum_checked() {
  auto a = Int32Array::from(std::vector<int32_t>{2147483647, 1});
  CHECK_EQ(sum(a).value(), (int32_t)-2147483648LL);
  auto r = sum_checked(a);
  CHECK(r.is_err());
  CHECK_EQ(r.unwrap_err().to_string(), std::string("Arithmetic overflow: Overflow happened on: 2147483647 + 1"));
  auto ok = sum_checked(Int64Array::from(std::vector<O<int64_t>>{5, N, 7})).unwrap();
  CHECK(ok.has_value() && *ok == 12);
  CHECK(!sum_checked(Int64Array::from(std::vector<O<int64_t>>{N, N})).unwrap().has_value());
}

// arrow-select/src/coalesce.rs:42-110 (struct doc example), :239-257 (push_batch_with_filter), :271-288 (push_batch_with_indices)
static void test_batch_coalescer() {
  Schema schema{{"a", DataType::Int32}};
  auto rb = [&](std::vector<O<int32_t>> v) {
    return RecordBatch::try_new(schema, {std::make_shared<Int32Array>(Int32Array::from(v))}).unwrap();
  };
  BatchCoalescer co(schema, 4);
  co.push_batch(rb({1, 2, 3})).unwrap();
  CHECK(!co.next_completed_batch().has_value());
  co.push_batch(rb({4, 5, 6})).unwrap();
  auto b = co.next_completed_batch();
  CHECK(b.has_value());
  CHECK(as_primitive<int32_t>(b->column(0)).to_vec() == (std::vector<O<int32_t>>{1, 2, 3, 4}));
  CHECK(!co.next_completed_batch().has_value());
  co.finish_buffered_batch();
  CHECK(as_primitive<int32_t>(co.next_completed_batch()->column(0)).to_vec() == (std::vector<O<int32_t>>{5, 6}));
  CHECK(co.is_empty());

  BatchCoalescer cf(schema, 1000);
  auto filter = BooleanArray::from(std::vector<bool>{true, false, true});
  cf.push_batch_with_filter(rb({1, N, 3}), filter).unwrap();
  cf.push_batch_with_filter(rb({4, 5, 6}), filter).unwrap();
  cf.finish_buffered_batch();
  auto fb = cf.next_completed_batch();
  CHECK(as_primitive<int32_t>(fb->column(0)).to_vec() == (std::vector<O<int32_t>>{1, 3, 4, 6}));
  CHECK(!fb->column(0)->nulls().has_value());  // the only null was filtered out: NullBufferBuilder never materialised

  BatchCoalescer ci(schema, 1000);
  ci.push_batch(rb({0, 0, 0})).unwrap();
  ci.push_batch_with_indices(rb({1, 1, 4, 5, 1, 4}), UInt64Array::from(std::vector<uint64_t>{0, 1, 4, 2, 5, 3})).unwrap();
  ci.finish_buffered_batch();
  CHECK(as_primitive<int32_t>(ci.next_completed_batch()->column(0)).to_vec() == (std::vector<O<int32_t>>{0, 0, 0, 1, 1, 1, 4, 4, 5}));

  // strings + nulls across an output boundary
  Schema s2{{"s", DataType::Utf8}, {"b", DataType::Boolean}};
  BatchCoalescer cs(s2, 3);
  auto sb = [&](std::vector<O<std::string>> v, std::vector<O<bool>> w) {
    return RecordBatch::try_new(s2, {std::make_shared<StringArray>(StringArray::from(v)), std::make_shared<BooleanArray>(BooleanArray::from(w))}).unwrap();
  };
  cs.push_batch(sb({std::string("ab"), N}, {true, N})).unwrap();
  cs.push_batch(sb({std::string("cde"), std::string(""), std::string("f")}, {false, true, N})).unwrap();
  cs.finish_buffered_batch();
  auto b1 = cs.next_completed_batch(), b2 = cs.next_completed_batch();
  CHECK(as_string(b1->column(0)).to_vec() == (std::vector<O<std::string>>{std::string("ab"), N, std::string("cde")}));
  CHECK(as_boolean(b1->column(1)).to_vec() == (std::vector<O<bool>>{true, N, false}));
  CHECK(as_string(b2->column(0)).to_vec() == (std::vector<O<std::string>>{std::string(""), std::string("f")}));
  CHECK(as_boolean(b2->column(1)).to_vec() == (std::vector<O<bool>>{true, N}));
  auto bad = cs.push_batch(rb({1}));
  CHECK(bad.is_err());
  CHECK_EQ(bad.unwrap_err().to_string(), std::string("Invalid argument error: Batch has 1 columns but BatchCoalescer expects 2"));
}

// arrow-select/src/take.rs:1371-1440 test_take_primitive
template <class T>
static void take_primitive_case() {
  auto index = UInt32Array::from(std::vector<O<uint32_t>>{3, N, 1, 3, 2});
  auto values = PrimitiveArray<T>::from(std::vector<O<T>>{T(0), N, T(2), T(3), N});
  auto out = take(values, index, std::nullopt).unwrap();
  CHECK(as_primitive<T>(out).to_vec() == (std::vector<O<T>>{T(3), N, N, T(3), T(2)}));
}
static void test_take_primitive() {
  take_primitive_case<int8_t>();
  take_primitive_case<int16_t>();
  take_primitive_case<int32_t>();
  take_primitive_case<int64_t>();
  take_primitive_case<uint8_t>();
  take_primitive_case<uint16_t>();
  take_primitive_case<uint32_t>();
  take_primitive_case<uint64_t>();
  take_primitive_case<float>();
  take_primitive_case<double>();
}

// take.rs:1331 test_take_primitive_nullable_indices_non_null_values_with_offset
static void test_take_with_offset() {
  auto index = UInt32Array::from(std::vector<O<uint32_t>>{0, 1, 2, 3, N, N}).slice(2, 4);
  auto values = Int64Array::from(std::vector<int64_t>{0, 10, 20, 30, 40, 50});
  auto out = take(values, index, std::nullopt).unwrap();
  CHECK(as_primitive<int64_t>(out).to_vec() == (std::vector<O<int64_t>>{20, 30, N, N}));
}

// take.rs:1627 test_take_bool
static void test_take_bool() {
  auto index = UInt32Array::from(std::vector<O<uint32_t>>{3, N, 1, 3, 2});
  auto values = BooleanArray::from(std::vector<O<bool>>{false, N, true, false, N});
  auto out = take(values, index, std::nullopt).unwrap();
  CHECK(as_boolean(out).to_vec() == (std::vector<O<bool>>{false, N, N, false, true}));
}

// take.rs:2408 test_take_out_of_bounds, :2455-2465 message, :2423 panic
static void test_take_out_of_bounds() {
  auto index = UInt32Array::from(std::vector<O<uint32_t>>{3, N, 1, 3, 6});
  auto values = Int64Array::from(std::vector<O<int64_t>>{0, N, 2, 3, N});
  auto r = take(values, index, TakeOptions{true});
  CHECK(r.is_err());
  CHECK_EQ(r.unwrap_err().to_string(), std::string("Compute error: Array index out of bounds, cannot get item at index 6 from 5 entries"));
  auto p = take(Int64Array::from(std::vector<int64_t>{0, 1, 2, 3}), UInt32Array::from(std::vector<uint32_t>{1000}), std::nullopt);
  CHECK(p.is_err());
  CHECK_EQ(p.unwrap_err().status, (acu_status)ACU_ERR_PANIC_OUT_OF_BOUNDS);  // the reference panics here
}

// take.rs:76-88 doc example; take.rs:2719 test_take_bytes_null_indices; dictionary.rs:310-317
static void test_take_strings_and_dictionary() {
  auto values = StringArray::from(std::vector<std::string>{"zero", "one", "two"});
  auto taken = take(values, UInt32Array::from(std::vector<uint32_t>{2, 1}), std::nullopt).unwrap();
  CHECK(as_string(taken).to_vec() == (std::vector<O<std::string>>{std::string("two"), std::string("one")}));
  auto dict = StringArray::from(std::vector<O<std::string>>{std::string("one"), N, std::string("three")});
  auto keys = Int32Array::from(std::vector<O<int32_t>>{0, 1, 2, N, 0, 2});
  auto flat = cast_dictionary_to_utf8(keys, dict).unwrap();
  CHECK(as_string(flat).to_vec() ==
        (std::vector<O<std::string>>{std::string("one"), N, std::string("three"), N, std::string("one"), std::string("three")}));
}

// arrow-arith/src/numeric.rs:1296-1361 test_integer
static void test_integer() {
  auto a = Int32Array::from(std::vector<int32_t>{4, 3, 5, -6, 100});
  auto b = Int32Array::from(std::vector<int32_t>{6, 2, 5, -7, 3});
  CHECK(as_primitive<int32_t>(numeric::add(a, b).unwrap()).values() == (std::vector<int32_t>{10, 5, 10, -13, 103}));
  CHECK(as_primitive<int32_t>(numeric::sub(a, b).unwrap()).values() == (std::vector<int32_t>{-2, 1, 0, 1, 97}));
  CHECK(as_primitive<int32_t>(numeric::div(a, b).unwrap()).values() == (std::vector<int32_t>{0, 1, 1, 0, 33}));
  CHECK(as_primitive<int32_t>(numeric::mul(a, b).unwrap()).values() == (std::vector<int32_t>{24, 6, 25, 42, 300}));
  CHECK(as_primitive<int32_t>(numeric::rem(a, b).unwrap()).values() == (std::vector<int32_t>{4, 1, 0, -6, 1}));

  auto a8 = Int8Array::from(std::vector<O<int8_t>>{int8_t(2), N, int8_t(45)});
  auto b8 = Int8Array::from(std::vector<O<int8_t>>{int8_t(5), int8_t(3), N});
  CHECK(as_primitive<int8_t>(numeric::add(a8, b8).unwrap()).to_vec() == (std::vector<O<int8_t>>{int8_t(7), N, N}));

  auto ua = UInt8Array::from(std::vector<uint8_t>{56, 5, 3});
  auto ub = UInt8Array::from(std::vector<uint8_t>{200, 2, 5});
  CHECK_EQ(numeric::add(ua, ub).unwrap_err().to_string(), std::string("Arithmetic overflow: Overflow happened on: 56 + 200"));
  CHECK(as_primitive<uint8_t>(numeric::add_wrapping(ua, ub).unwrap()).values() == (std::vector<uint8_t>{0, 7, 8}));
  auto uc = UInt8Array::from(std::vector<uint8_t>{34, 5, 3});
  CHECK_EQ(numeric::sub(uc, ub).unwrap_err().to_string(), std::string("Arithmetic overflow: Overflow happened on: 34 - 200"));
  CHECK(as_primitive<uint8_t>(numeric::sub_wrapping(uc, ub).unwrap()).values() == (std::vector<uint8_t>{90, 3, 254}));
  CHECK_EQ(numeric::mul(uc, ub).unwrap_err().to_string(), std::string("Arithmetic overflow: Overflow happened on: 34 * 200"));
  CHECK(as_primitive<uint8_t>(numeric::mul_wrapping(uc, ub).unwrap()).values() == (std::vector<uint8_t>{144, 10, 15}));

  auto mn = Int16Array::from(std::vector<int16_t>{std::numeric_limits<int16_t>::min()});
  auto m1 = Int16Array::from(std::vector<int16_t>{-1});
  CHECK_EQ(numeric::div(mn, m1).unwrap_err().to_string(), std::string("Arithmetic overflow: Overflow happened on: -32768 / -1"));
  CHECK(as_primitive<int16_t>(numeric::rem(mn, m1).unwrap()).values() == (std::vector<int16_t>{0}));
  auto x = Int16Array::from(std::vector<int16_t>{21});
  auto z = Int16Array::from(std::vector<int16_t>{0});
  CHECK_EQ(numeric::div(x, z).unwrap_err().to_string(), std::string("Divide by zero error"));
  CHECK_EQ(numeric::rem(x, z).unwrap_err().to_string(), std::string("Divide by zero error"));
}

// numeric.rs:1364-1397 test_float
static void test_float() {
  const float MAX = std::numeric_limits<float>::max(), INF = std::numeric_limits<float>::infinity();
  auto a = Float32Array::from(std::vector<float>{1.f, MAX, 6.f, -4.f, -1.f, 0.f});
  auto b = Float32Array::from(std::vector<float>{1.f, MAX, MAX, -3.f, 45.f, 0.f});
  CHECK(as_primitive<float>(numeric::add(a, b).unwrap()).values() == (std::vector<float>{2.f, INF, MAX, -7.f, 44.f, 0.f}));
  CHECK(as_primitive<float>(numeric::sub(a, b).unwrap()).values() == (std::vector<float>{0.f, 0.f, -MAX, -1.f, -46.f, 0.f}));
  CHECK(as_primitive<float>(numeric::mul(a, b).unwrap()).values() == (std::vector<float>{1.f, INF, INF, 12.f, -45.f, 0.f}));
  auto d = as_primitive<float>(numeric::div(a, b).unwrap()).values();
  CHECK_EQ(d[0], 1.f);
  CHECK_EQ(d[1], 1.f);
  CHECK(d[2] < std::numeric_limits<float>::epsilon());
  CHECK_EQ(d[3], -4.f / -3.f);
  CHECK(std::isnan(d[5]));
  auto r = as_primitive<float>(numeric::rem(a, b).unwrap()).values();
  CHECK((std::vector<float>(r.begin(), r.begin() + 5)) == (std::vector<float>{0.f, 0.f, 6.f, -1.f, -1.f}));
  CHECK(std::isnan(r[5]));
}

// numeric.rs:1152-1185 test_neg; scalar arms numeric.rs:278-317
static void test_neg_and_scalars() {
  CHECK(as_primitive<int64_t>(numeric::neg(Int64Array::from(std::vector<int64_t>{1, -5, 2, 693, 3929})).unwrap()).values() ==
        (std::vector<int64_t>{-1, 5, -2, -693, -3929}));
  CHECK_EQ(numeric::neg(Int32Array::from(std::vector<int32_t>{std::numeric_limits<int32_t>::min()})).unwrap_err().to_string(),
           std::string("Arithmetic overflow: Overflow happened on: - -2147483648"));
  CHECK_EQ(as_primitive<int64_t>(numeric::neg_wrapping(Int64Array::from(std::vector<int64_t>{std::numeric_limits<int64_t>::min()})).unwrap()).value(0),
           std::numeric_limits<int64_t>::min());
  CHECK_EQ(numeric::neg(UInt32Array::from(std::vector<uint32_t>{1})).unwrap_err().to_string(),
           std::string("Invalid argument error: Invalid arithmetic operation: !UInt32"));
  auto arr = Int64Array::from(std::vector<O<int64_t>>{1, N, 3});
  CHECK(as_primitive<int64_t>(numeric::add(arr, new_scalar<int64_t>(10)).unwrap()).to_vec() == (std::vector<O<int64_t>>{11, N, 13}));
  CHECK(as_primitive<int64_t>(numeric::sub(new_scalar<int64_t>(10), arr).unwrap()).to_vec() == (std::vector<O<int64_t>>{9, N, 7}));
  CHECK(as_primitive<int64_t>(numeric::add(arr, new_null_scalar<int64_t>()).unwrap()).to_vec() == (std::vector<O<int64_t>>{N, N, N}));
  CHECK_EQ(numeric::add(Int32Array::from(std::vector<int32_t>{1}), Int64Array::from(std::vector<int64_t>{1})).unwrap_err().to_string(),
           std::string("Invalid argument error: Invalid arithmetic operation: Int32 + Int64"));
}

// arrow-ord/src/comparison.rs:2475-2571 (NaN totalOrder), :3558-3575 test_floating_zeros
static void test_cmp_total_order() {
  const double NaN = std::numeric_limits<double>::quiet_NaN();
  auto a1 = Float64Array::from(std::vector<double>{NaN, 7.0, 8.0, 8.0, 10.0});
  auto a2 = Float64Array::from(std::vector<double>{NaN, NaN, 8.0, 8.0, 10.0});
  CHECK(cmpk::eq(a1, a2).unwrap().values() == (std::vector<bool>{true, false, true, true, true}));
  CHECK(cmpk::neq(a1, a2).unwrap().values() == (std::vector<bool>{false, true, false, false, false}));
  auto b1 = Float64Array::from(std::vector<double>{NaN, 7.0, 8.0, 8.0, 11.0, NaN});
  auto b2 = Float64Array::from(std::vector<double>{NaN, NaN, 8.0, 9.0, 10.0, 1.0});
  CHECK(cmpk::lt(b1, b2).unwrap().values() == (std::vector<bool>{false, true, false, true, false, false}));
  CHECK(cmpk::lt_eq(b1, b2).unwrap().values() == (std::vector<bool>{true, true, true, true, false, false}));
  CHECK(cmpk::gt(b1, b2).unwrap().values() == (std::vector<bool>{false, false, false, false, true, true}));
  CHECK(cmpk::gt_eq(b1, b2).unwrap().values() == (std::vector<bool>{true, false, true, false, true, true}));
  CHECK(cmpk::eq(a1, new_scalar<double>(NaN)).unwrap().values() == (std::vector<bool>{true, false, false, false, false}));
  auto za = Float32Array::from(std::vector<float>{0.0f, -0.0f});
  auto zb = Float32Array::from(std::vector<float>{-0.0f, 0.0f});
  CHECK(cmpk::eq(za, zb).unwrap().values() == (std::vector<bool>{false, false}));
  CHECK(cmpk::eq(za, new_scalar<float>(0.0f)).unwrap().values() == (std::vector<bool>{true, false}));
  CHECK(cmpk::eq(za, new_scalar<float>(-0.0f)).unwrap().values() == (std::vector<bool>{false, true}));
}

// arrow-ord/src/cmp.rs:1044-1116 is_distinct_from_nulls, test_distinct_scalar
static void test_distinct() {
  auto l = Int32Array::from(std::vector<O<int32_t>>{0, 0, N, 3, 0, 0});
  auto r = Int32Array::from(std::vector<O<int32_t>>{0, N, N, N, 0, N});
  CHECK(cmpk::distinct(l, r).unwrap().to_vec() == (std::vector<O<bool>>{false, true, false, true, false, true}));
  CHECK(cmpk::not_distinct(l, r).unwrap().to_vec() == (std::vector<O<bool>>{true, false, true, false, true, false}));
  auto a = Int32Array::from(std::vector<O<int32_t>>{N, N, 2, 3});
  auto b = new_null_scalar<int32_t>();
  CHECK(cmpk::distinct(a, b).unwrap().to_vec() == (std::vector<O<bool>>{false, false, true, true}));
  CHECK(cmpk::not_distinct(b, a).unwrap().to_vec() == (std::vector<O<bool>>{true, true, false, false}));
  CHECK(cmpk::eq(a, b).unwrap().null_count() == 4);
  CHECK_EQ(cmpk::eq(Int32Array::from(std::vector<int32_t>{1, 2, 3}), Int32Array::from(std::vector<int32_t>{1, 2})).unwrap_err().to_string(),
           std::string("Invalid argument error: Cannot compare arrays of different lengths, got 3 vs 2"));
}

// arrow-cast/src/cast/mod.rs:8449-8569 test_cast_from_int64
static void test_cast_from_int64() {
  const int64_t I64MIN = std::numeric_limits<int64_t>::min(), I64MAX = std::numeric_limits<int64_t>::max();
  auto a = Int64Array::from(std::vector<int64_t>{I64MIN, INT32_MIN, INT16_MIN, INT8_MIN, 0, INT8_MAX, INT16_MAX, INT32_MAX, I64MAX});
  auto f = as_primitive<double>(cast(a, DataType::Float64).unwrap()).values();
  CHECK(f == (std::vector<double>{-9223372036854775808.0, -2147483648.0, -32768.0, -128.0, 0.0, 127.0, 32767.0, 2147483647.0, 9223372036854775808.0}));
  auto i32 = as_primitive<int32_t>(cast(a, DataType::Int32).unwrap()).to_vec();
  CHECK(i32 == (std::vector<O<int32_t>>{N, INT32_MIN, INT16_MIN, INT8_MIN, 0, INT8_MAX, INT16_MAX, INT32_MAX, N}));
  auto i16 = as_primitive<int16_t>(cast(a, DataType::Int16).unwrap()).to_vec();
  CHECK(i16 == (std::vector<O<int16_t>>{N, N, int16_t(INT16_MIN), int16_t(INT8_MIN), int16_t(0), int16_t(INT8_MAX), int16_t(INT16_MAX), N, N}));
  auto e = cast_with_options(Int64Array::from(std::vector<int64_t>{1, I64MAX}), DataType::Int32, CastOptions{false});
  CHECK_EQ(e.unwrap_err().to_string(), std::string("Cast error: Can't cast value 9223372036854775807 to type Int32"));
}

// arrow-arith/src/aggregate.rs:1039-1137, :1299-1416, :1985
static void test_aggregates() {
  CHECK(sum(Int32Array::from(std::vector<int32_t>{1, 2, 3, 4, 5})) == O<int32_t>(15));
  CHECK(sum(Float64Array::from(std::vector<double>{1.1, 2.2, 3.3, 4.4, 5.5})) == O<double>(16.5));
  CHECK(!sum(Int32Array::from(std::vector<O<int32_t>>{N, N, N})).has_value());
  CHECK(sum(Int32Array::from(std::vector<int32_t>{INT32_MAX, 1})) == O<int32_t>(INT32_MIN));  // test_sum_overflow: wraps
  auto a = Int32Array::from(std::vector<O<int32_t>>{5, N, N, 8, 9});
  CHECK(min(a) == O<int32_t>(5));
  CHECK(max(a) == O<int32_t>(9));
  const double NaN = std::numeric_limits<double>::quiet_NaN(), INF = std::numeric_limits<double>::infinity();
  auto f = Float64Array::from(std::vector<double>{-INF, NaN, INF, -NaN});
  auto mx = *max(f), mn = *min(f);
  CHECK(std::isnan(mx) && !std::signbit(mx));  // test_primitive_min_max_float_negative_nan
  CHECK(std::isnan(mn) && std::signbit(mn));
}


// arrow-select/src/nullif.rs:127 test_nullif_int_array, :466 test_nullif_no_nulls
static void test_nullif() {
  auto a = Int32Array::from(std::vector<O<int32_t>>{15, N, 8, 1, 9});
  auto comp = BooleanArray::from(std::vector<O<bool>>{false, N, true, false, N});
  auto res = nullif(a, comp).unwrap();
  CHECK((as_primitive<int32_t>(res).to_vec() == std::vector<O<int32_t>>{15, N, N, 1, 9}));
  auto b = Int32Array::from(std::vector<int32_t>{15, 7, 8, 1, 9});
  res = nullif(b, comp).unwrap();
  CHECK((as_primitive<int32_t>(res).to_vec() == std::vector<O<int32_t>>{15, 7, N, 1, 9}));
  CHECK((as_primitive<int32_t>(res).values() == std::vector<int32_t>{15, 7, 8, 1, 9}));  // values are shared untouched
  auto err = nullif(b, BooleanArray::from(std::vector<bool>{true})).unwrap_err();
  CHECK_EQ(err.message, std::string("Compute error: Cannot perform comparison operation on arrays of different length"));
}

// arrow-select/src/zip.rs:870 test_zip_kernel_one, :892 scalar_falsy_1, :975 primitive_scalar_none_1
static void test_zip() {
  auto a = Int32Array::from(std::vector<O<int32_t>>{5, N, 7, N, 1});
  auto b = Int32Array::from(std::vector<O<int32_t>>{N, 3, 6, 7, 3});
  auto mask = BooleanArray::from(std::vector<bool>{true, true, false, false, true});
  auto out = zip(mask, a, b).unwrap();
  CHECK((as_primitive<int32_t>(out).to_vec() == std::vector<O<int32_t>>{5, N, 6, 7, 1}));
  out = zip(mask, a, new_scalar<int32_t>(42)).unwrap();
  CHECK((as_primitive<int32_t>(out).to_vec() == std::vector<O<int32_t>>{5, N, 42, 42, 1}));
  out = zip(mask, new_scalar<int32_t>(42), new_null_scalar<int32_t>()).unwrap();
  CHECK((as_primitive<int32_t>(out).to_vec() == std::vector<O<int32_t>>{42, 42, N, N, 42}));
  auto err = zip(mask, Int32Array::from(std::vector<int32_t>{1, 2}), b).unwrap_err();
  CHECK_EQ(err.message, std::string("Invalid argument error: all arrays should have the same length"));
}

// arrow-select/src/concat.rs:880 test_concat_primitive_arrays, :832 test_concat_string_arrays, :698 test_concat_empty_vec
static void test_concat() {
  auto a = Int64Array::from(std::vector<O<int64_t>>{-1, -1, 2, N, N});
  auto b = Int64Array::from(std::vector<O<int64_t>>{101, 102, 103, N});
  auto c = Int64Array::from(std::vector<int64_t>{256, 512, 1024});
  auto arr = concat({&a, &b, &c}).unwrap();
  CHECK((as_primitive<int64_t>(arr).to_vec() == std::vector<O<int64_t>>{-1, -1, 2, N, N, 101, 102, 103, N, 256, 512, 1024}));
  auto sa = a.slice(1, 3), sb = b.slice(1, 3);
  arr = concat({&sa, &sb}).unwrap();
  CHECK((as_primitive<int64_t>(arr).to_vec() == std::vector<O<int64_t>>{-1, 2, N, 102, 103, N}));
  auto s1 = StringArray::from(std::vector<std::string>{"hello", "world"});
  auto s2 = StringArray::from(std::vector<std::string>{"2", "3", "4"});
  auto s3 = StringArray::from(std::vector<O<std::string>>{std::string("foo"), std::string("bar"), N, std::string("baz")});
  arr = concat({&s1, &s2, &s3}).unwrap();
  CHECK((as_string(arr).to_vec() == std::vector<O<std::string>>{std::string("hello"), std::string("world"), std::string("2"), std::string("3"),
                                                                std::string("4"), std::string("foo"), std::string("bar"), N, std::string("baz")}));
  CHECK_EQ(concat({}).unwrap_err().message, std::string("Compute error: concat requires input of at least one array"));
  Schema schema{{"a", DataType::Int64, true}, {"s", DataType::Utf8, true}};
  auto b1 = RecordBatch::try_new(schema, {std::make_shared<Int64Array>(c), std::make_shared<StringArray>(StringArray::from(std::vector<std::string>{"x", "y", "z"}))}).unwrap();
  auto b2 = RecordBatch::try_new(schema, {std::make_shared<Int64Array>(b), std::make_shared<StringArray>(s3)}).unwrap();
  auto cb = concat_batches(schema, {&b1, &b2}).unwrap();
  CHECK_EQ(7, cb.num_rows());
  CHECK((as_primitive<int64_t>(cb.column(0)).to_vec() == std::vector<O<int64_t>>{256, 512, 1024, 101, 102, 103, N}));
}

// arrow-ord/src/comparison.rs:1246 test_utf8_array_eq, :1318 test_utf8_array_lt, :1147 test_utf8_eq_scalar_on_slice
static void test_cmp_utf8() {
  auto l = StringArray::from(std::vector<std::string>{"arrow", "arrow", "arrow", "arrow"});
  auto r = StringArray::from(std::vector<std::string>{"arrow", "parquet", "datafusion", "flight"});
  CHECK((cmpk::eq(l, r).unwrap().to_vec() == std::vector<O<bool>>{true, false, false, false}));
  CHECK((cmpk::neq(l, r).unwrap().to_vec() == std::vector<O<bool>>{false, true, true, true}));
  auto l2 = StringArray::from(std::vector<std::string>{"arrow", "datafusion", "flight", "parquet"});
  auto f = StringArray::from(std::vector<std::string>{"flight", "flight", "flight", "flight"});
  CHECK((cmpk::lt(l2, f).unwrap().to_vec() == std::vector<O<bool>>{true, true, false, false}));
  CHECK((cmpk::gt_eq(l2, f).unwrap().to_vec() == std::vector<O<bool>>{false, false, true, true}));
  auto sc = Scalar<StringArray>(StringArray::from(std::vector<std::string>{"flight"}));
  CHECK((cmpk::lt_eq(l2, sc).unwrap().to_vec() == std::vector<O<bool>>{true, true, true, false}));
  auto withnull = StringArray::from(std::vector<O<std::string>>{N, std::string("hello"), std::string("world"), std::string("")});
  auto hello = Scalar<StringArray>(StringArray::from(std::vector<std::string>{"hello"}));
  CHECK((cmpk::eq(withnull, hello).unwrap().to_vec() == std::vector<O<bool>>{N, true, false, false}));
}

// parquet/src/arrow/arrow_reader/filter.rs:63-106 (ArrowPredicateFn doc example "b > 0") + RowFilter semantics :138-170
static void test_row_filter() {
  Schema schema{{"a", DataType::Int64, true}, {"b", DataType::Int64, true}};
  auto a = std::make_shared<Int64Array>(Int64Array::from(std::vector<O<int64_t>>{1, 2, 3, N, 5, 6}));
  auto b = std::make_shared<Int64Array>(Int64Array::from(std::vector<O<int64_t>>{-1, 4, 0, 7, N, 9}));
  auto batch = RecordBatch::try_new(schema, {a, b}).unwrap();
  auto p1 = std::make_shared<parquet::ArrowPredicateFn>(std::vector<size_t>{1}, [](const RecordBatch &rb) {
    return cmpk::gt(as_primitive<int64_t>(rb.column(0)), new_scalar<int64_t>(0));  // b > 0 (null => dropped)
  });
  auto p2 = std::make_shared<parquet::ArrowPredicateFn>(std::vector<size_t>{0}, [](const RecordBatch &rb) {
    return cmpk::lt(as_primitive<int64_t>(rb.column(0)), new_scalar<int64_t>(6));  // a < 6, evaluated on the surviving rows only
  });
  auto out = parquet::RowFilter({p1, p2}).apply(batch).unwrap();
  CHECK_EQ(1, out.num_rows());  // rows with b > 0: (2,4) (null,7) (6,9); of those a < 6: (2,4) — a null `a` is dropped
  CHECK((as_primitive<int64_t>(out.column(0)).to_vec() == std::vector<O<int64_t>>{2}));
  CHECK((as_primitive<int64_t>(out.column(1)).to_vec() == std::vector<O<int64_t>>{4}));
  // the same first predicate with the comparison fused into the filter plan (no BooleanArray in HBM)
  auto fused = FilterBuilder::from_cmp(ACU_GT, as_primitive<int64_t>(batch.column(1)), new_scalar<int64_t>(0)).unwrap();
  auto fb = fused.filter_record_batch(batch).unwrap();
  CHECK_EQ(3, fb.num_rows());
  CHECK((as_primitive<int64_t>(fb.column(1)).to_vec() == std::vector<O<int64_t>>{4, 7, 9}));
  auto bad = std::make_shared<parquet::ArrowPredicateFn>(std::vector<size_t>{0}, [](const RecordBatch &) {
    return Result<BooleanArray>(BooleanArray::from(std::vector<bool>{true}));
  });
  CHECK(parquet::RowFilter({bad}).apply(batch).is_err());
}

// arrow-ipc/src/reader.rs:1587-1671 StreamReader over a stream written by another Arrow implementation (the Python test
// writes it with pyarrow into $ACU_TEST_IPC_FILE: a: int64 [1, null, 3], s: utf8 ["x", null, "hello"], b: bool [true,
// false, null], f: float32 [1.5, 2.5, 3.5]; then a second batch = rows 1..3 of the first)
static void test_ipc_stream_reader() {
  const char *path = std::getenv("ACU_TEST_IPC_FILE");
  if (!path) { std::printf("  (ACU_TEST_IPC_FILE not set: ipc stream test skipped)\n"); return; }
  std::FILE *fp = std::fopen(path, "rb");
  CHECK(fp != nullptr);
  if (!fp) return;
  std::vector<uint8_t> bytes;
  uint8_t buf[4096];
  size_t n;
  while ((n = std::fread(buf, 1, sizeof buf, fp)) > 0) bytes.insert(bytes.end(), buf, buf + n);
  std::fclose(fp);
  auto reader = ipc::StreamReader::try_new(bytes).unwrap();
  CHECK_EQ(4u, reader.schema().size());
  CHECK_EQ(std::string("s"), reader.schema()[1].name);
  auto b1 = reader.next().unwrap();
  CHECK(b1.has_value());
  CHECK_EQ(3, b1->num_rows());
  CHECK((as_primitive<int64_t>(b1->column(0)).to_vec() == std::vector<O<int64_t>>{1, N, 3}));
  CHECK((as_string(b1->column(1)).to_vec() == std::vector<O<std::string>>{std::string("x"), N, std::string("hello")}));
  CHECK((as_boolean(b1->column(2)).to_vec() == std::vector<O<bool>>{true, false, N}));
  CHECK((as_primitive<float>(b1->column(3)).to_vec() == std::vector<O<float>>{1.5f, 2.5f, 3.5f}));
  CHECK(!b1->column(3)->nulls().has_value());  // null_count 0 => no NullBuffer (reader.rs:271)
  auto b2 = reader.next().unwrap();
  CHECK(b2.has_value());
  CHECK_EQ(2, b2->num_rows());
  CHECK((as_primitive<int64_t>(b2->column(0)).to_vec() == std::vector<O<int64_t>>{N, 3}));
  CHECK((as_string(b2->column(1)).to_vec() == std::vector<O<std::string>>{N, std::string("hello")}));
  // the decoded batch feeds the hot path directly: filter by (a is not null)
  auto kept = filter_record_batch(*b2, arrow_cuda::compute::kernels::boolean::is_not_null(*b2->column(0)).unwrap()).unwrap();
  CHECK_EQ(1, kept.num_rows());
  auto end = reader.next().unwrap();
  CHECK(!end.has_value());
  CHECK(reader.is_finished());
  CHECK_EQ(ipc::StreamReader::try_new(std::vector<uint8_t>{}).unwrap_err().message, std::string("Ipc error: Expected schema message, found empty stream."));
}

// arrow-select/src/coalesce.rs:1079-1167,1230-1304 (test_string_view_batch_large_no_compact, _large_slice_compact,
// _many_small_compact, _many_small_boundary): expected data-buffer layouts of the coalesced StringViewArray
static void test_string_view_coalesce() {
  using arrow_cuda::compute::StringViewArray;
  using arrow_cuda::compute::coalesce::InProgressByteViewArray;
  auto repeated = [](size_t n, std::vector<O<std::string>> items) {
    std::vector<O<std::string>> v;
    for (size_t i = 0; i < n; ++i) v.push_back(items[i % items.size()]);
    return StringViewArray::from(v, 8192);
  };
  auto layout = [](const StringViewArray &a) {
    std::vector<std::pair<size_t, size_t>> l;
    for (const auto &b : a.data_buffers()) l.push_back({b.len, b.capacity});
    return l;
  };
  using L = std::vector<std::pair<size_t, size_t>>;
  const std::string long_s = "This string is longer than 12 bytes";
  auto large = repeated(1000, {long_s});
  CHECK_EQ(5u, large.data_buffers().size());
  {  // full buffers: adopted, not copied
    InProgressByteViewArray ip(1000);
    ip.set_source(large).unwrap();
    CHECK(!ip.source_needs_gc());
    ip.copy_rows(0, 1000).unwrap();
    auto out = ip.finish();
    CHECK((layout(out) == L{{8190, 8192}, {8190, 8192}, {8190, 8192}, {8190, 8192}, {2240, 8192}}));
    CHECK(out.to_vec() == large.to_vec());
  }
  {  // a 22-row slice of it uses 770 of 40960 buffer bytes: garbage-collected into one 8 KiB buffer
    InProgressByteViewArray ip(1000);
    auto sl = large.slice(11, 22);
    ip.set_source(sl).unwrap();
    CHECK(ip.source_needs_gc());
    ip.copy_rows(0, 22).unwrap();
    auto out = ip.finish();
    CHECK((layout(out) == L{{770, 8192}}));
    CHECK(out.to_vec() == sl.to_vec());
  }
  {  // ten batches of 100 long (28 bytes) + 100 short strings: buffers of 8, 16, 32 KiB filled in turn
    auto b = repeated(200, {std::string("This string is 28 bytes long"), std::string("small string")});
    InProgressByteViewArray ip(8000);
    std::vector<O<std::string>> expect;
    for (int k = 0; k < 10; ++k) {
      ip.set_source(b).unwrap();
      ip.copy_rows(0, 200).unwrap();
      auto v = b.to_vec();
      expect.insert(expect.end(), v.begin(), v.end());
    }
    auto out = ip.finish();
    CHECK((layout(out) == L{{8176, 8192}, {16380, 16384}, {3444, 32768}}));
    CHECK(out.to_vec() == expect);
  }
  {  // strings that fill power-of-two buffers exactly; output batches of 900 rows cut the 100-row inputs
    auto b = repeated(100, {std::string("This string is a power of two=32")});
    InProgressByteViewArray ip(900);
    int64_t buffered = 0;
    std::vector<StringViewArray> outs;
    for (int k = 0; k < 20; ++k) {
      ip.set_source(b).unwrap();
      int64_t n = 100, off = 0;
      while (n > 900 - buffered) {
        const int64_t rem = 900 - buffered;
        ip.copy_rows(off, rem).unwrap();
        off += rem; n -= rem; buffered = 0;
        outs.push_back(ip.finish());
      }
      if (n > 0) { ip.copy_rows(off, n).unwrap(); buffered += n; }
      if (buffered >= 900) { outs.push_back(ip.finish()); buffered = 0; }
    }
    if (buffered) outs.push_back(ip.finish());
    CHECK_EQ(3u, outs.size());
    CHECK_EQ(900, outs[0].len());
    CHECK_EQ(200, outs[2].len());
    CHECK((layout(outs[0]) == L{{8192, 8192}, {16384, 16384}, {4224, 32768}}));
  }
  {  // nulls and inline-only arrays
    auto small = StringViewArray::from({std::string("foo"), N, std::string("bar")});
    InProgressByteViewArray ip(16);
    ip.set_source(small).unwrap();
    ip.copy_rows(1, 2).unwrap();
    auto out = ip.finish();
    CHECK(out.data_buffers().empty());
    CHECK((out.to_vec() == std::vector<O<std::string>>{N, std::string("bar")}));
  }
}

// arrow-select/src/filter.rs:1640-1678 test_slice_iterator_bits / _bits1 / _chunk_and_bits
static void test_slice_iterator() {
  using P = std::vector<std::pair<size_t, size_t>>;
  auto bools = [](size_t n, std::function<bool(size_t)> f) {
    std::vector<O<bool>> v;
    for (size_t i = 0; i < n; ++i) v.push_back(f(i));
    return BooleanArray::from(v);
  };
  CHECK((FilterBuilder(bools(64, [](size_t i) { return i == 1; })).build().slices().unwrap() == P{{1, 2}}));
  CHECK((FilterBuilder(bools(64, [](size_t i) { return i != 1; })).build().slices().unwrap() == P{{0, 1}, {2, 64}}));
  auto pred = FilterBuilder(bools(130, [](size_t i) { return i % 62 != 0; })).build();
  CHECK((pred.slices().unwrap() == P{{1, 62}, {63, 124}, {125, 130}}));
  CHECK_EQ(61 + 61 + 5, pred.count());
}

// Primitive, Boolean and Utf8 arrays reached through an ArrayRef (as RecordBatch::column returns them) give the results of
// the concrete-type calls in filter, FilterPredicate::filter and take
template <class A>
static void check_array_ref(const A &a) {
  const ArrayRef ref = std::make_shared<A>(a);
  auto same = [](Result<ArrayRef> got, const ArrayRef &want) {
    if (got.is_err()) return false;
    const ArrayRef g = got.unwrap();
    return g->data_type() == want->data_type() && static_cast<const A &>(*g).to_vec() == static_cast<const A &>(*want).to_vec();
  };
  const auto p = BooleanArray::from(std::vector<bool>{true, false, true, true});
  const auto idx = Int64Array::from(std::vector<O<int64_t>>{3, N, 0, 0});
  const ArrayRef f = filter(a, p).unwrap(), t = take(a, idx).unwrap();
  CHECK(same(filter(*ref, p), f));
  CHECK(same(FilterBuilder(p).build().filter(*ref), f));
  CHECK(same(take(*ref, idx), t));
}
static void test_array_ref() {
  check_array_ref(Int16Array::from(std::vector<O<int16_t>>{1, N, -3, 4}));
  check_array_ref(Float64Array::from(std::vector<double>{1.5, 2.5, -3.5, 4.5}));
  check_array_ref(BooleanArray::from(std::vector<O<bool>>{true, N, false, true}));
  check_array_ref(StringArray::from(std::vector<O<std::string>>{"a", N, "ccc", ""}));
}

int main() {
  try {
    Context::get(0);
  } catch (const std::exception &e) {
    std::printf("arrow-cuda host tests need a CUDA device: %s\n", e.what());
    return 77;
  }
  struct T { const char *name; std::function<void()> fn; };
  std::vector<T> tests = {
      {"filter_array_slice", test_filter_array_slice},
      {"filter_array_low_density", test_filter_array_low_density},
      {"filter_array_high_density", test_filter_array_high_density},
      {"filter_string_array", test_filter_string_array},
      {"null_mask_and_fast_path", test_null_mask_and_fast_path},
      {"filter_predicate_too_long", test_filter_predicate_too_long},
      {"filter_record_batch", test_filter_record_batch},
      {"take_record_batch", test_take_record_batch},
      {"boolean_kernels", test_boolean_kernels},
      {"sum_checked", test_sum_checked},
      {"batch_coalescer", test_batch_coalescer},
      {"take_primitive", test_take_primitive},
      {"take_with_offset", test_take_with_offset},
      {"take_bool", test_take_bool},
      {"take_out_of_bounds", test_take_out_of_bounds},
      {"take_strings_and_dictionary", test_take_strings_and_dictionary},
      {"integer", test_integer},
      {"float", test_float},
      {"neg_and_scalars", test_neg_and_scalars},
      {"cmp_total_order", test_cmp_total_order},
      {"distinct", test_distinct},
      {"cast_from_int64", test_cast_from_int64},
      {"aggregates", test_aggregates},
      {"nullif", test_nullif},
      {"zip", test_zip},
      {"concat", test_concat},
      {"cmp_utf8", test_cmp_utf8},
      {"row_filter", test_row_filter},
      {"ipc_stream_reader", test_ipc_stream_reader},
      {"string_view_coalesce", test_string_view_coalesce},
      {"slice_iterator", test_slice_iterator},
      {"array_ref", test_array_ref},
  };
  for (auto &t : tests) {
    int before = g_failed;
    try {
      t.fn();
    } catch (const std::exception &e) {
      ++g_failed;
      std::printf("  EXCEPTION in %s: %s\n", t.name, e.what());
    }
    std::printf("test %s ... %s\n", t.name, g_failed == before ? "ok" : "FAILED");
  }
  std::printf("%zu tests, %d checks, %d failed\n", tests.size(), g_checks, g_failed);
  return g_failed ? 1 : 0;
}
