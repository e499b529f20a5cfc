// test_host_fixed_size_binary.cpp — the reference's FixedSizeBinary filter / take tests (arrow-select/src/filter.rs:1341-1411;
// arrow-select/src/take.rs:2242-2294) re-expressed against the C++ host mirror (arrow_cuda.hpp), with the width-0 length rule,
// the dynamic-length path's slice panics and the nested and record-batch forms. Runs on a CUDA device (no CPU fallback);
// exits 77 when there is none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_fixed_size_binary   (exit code 0 = all passed)
#include <cstdio>

#include "arrow_cuda.hpp"

using namespace arrow_cuda;
using namespace arrow_cuda::compute;

static int g_failed = 0, g_checks = 0;
#define CHECK(cond)                                                                    \
  do {                                                                                 \
    ++g_checks;                                                                        \
    if (!(cond)) { ++g_failed; std::printf("  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); } \
  } while (0)

using Bytes = std::vector<uint8_t>;
using Rows = std::vector<std::optional<Bytes>>;
static const FixedSizeBinaryArray &fsb(const ArrayRef &a) { return static_cast<const FixedSizeBinaryArray &>(*a); }
static BooleanArray pred(const std::vector<bool> &b) { return BooleanArray::from(b); }

static void test_filter_fixed_binary() {
  const Bytes v1{1, 2}, v2{3, 4}, v3{5, 6};
  const auto a = FixedSizeBinaryArray::from({v1, v2, v3}, 2);
  auto c = filter(a, pred({true, false, true})).unwrap();
  CHECK(c->len() == 2 && fsb(c).value(0) == v1 && fsb(c).value(1) == v3);
  auto c2 = FilterBuilder(pred({true, false, true})).optimize().build().filter(a).unwrap();
  CHECK(c2->len() == 2 && fsb(c2).value(0) == v1 && fsb(c2).value(1) == v3);
  CHECK(filter(a, pred({false, false, false})).unwrap()->len() == 0);
  c = filter(a, pred({true, true, true})).unwrap();
  CHECK(c->len() == 3 && fsb(c).value(0) == v1 && fsb(c).value(1) == v2 && fsb(c).value(2) == v3);
  c = filter(a, pred({false, false, true})).unwrap();
  CHECK(c->len() == 1 && fsb(c).value(0) == v3);
}

static void take_with_nulls_indices(int32_t w) {
  Rows rows;
  for (uint8_t k = 1; k <= 4; ++k) {
    Bytes r((size_t)w, k);
    if (w == 5) r[4] = 1;
    rows.push_back(r);
  }
  const auto values = FixedSizeBinaryArray::from(rows, w);
  const auto indices = PrimitiveArray<uint32_t>::from(std::vector<std::optional<uint32_t>>{0u, std::nullopt, std::nullopt, 3u});
  auto r = take(values, indices).unwrap();
  CHECK(r->len() == 4 && r->null_count() == 2);
  CHECK((r->valid_mask() == std::vector<bool>{true, false, false, true}));
  CHECK(fsb(r).value(0) == *rows[0] && fsb(r).value(3) == *rows[3]);
  if (w == 5) CHECK(fsb(r).value(1) == Bytes(5, 0));  // the dynamic-length path zeroes a null index's bytes
}

static void test_width_zero_length_rule() {
  // FixedSizeBinaryArray::try_new of width 0: the length comes from the NullBuffer
  CHECK(FixedSizeBinaryArray::try_new(0, Buffer::allocate(0), std::nullopt).unwrap().len() == 0);
  CHECK(FixedSizeBinaryArray::try_new(0, Buffer::allocate(0), nulls_from_mask({true, false, true})).unwrap().len() == 3);
  CHECK(FixedSizeBinaryArray::try_new(-1, Buffer::allocate(0), std::nullopt).is_err());
  const auto z = FixedSizeBinaryArray::from({Bytes{}, Bytes{}, Bytes{}}, 0);
  CHECK(filter(z, pred({true, false, true})).unwrap()->len() == 0);
  CHECK(filter(z, pred({true, true, true})).unwrap()->len() == 3);  // All: values.slice(0, count)
  const auto zn = FixedSizeBinaryArray::from({Bytes{}, std::nullopt, Bytes{}}, 0);
  CHECK(filter(zn, pred({true, true, false})).unwrap()->len() == 2);
  CHECK(take(z, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{2, 0, 9})).unwrap()->len() == 0);
  auto r = take(zn, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{1, 0}));
  CHECK(r.unwrap()->len() == 2);
  r = take(zn, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{0, 9}));
  CHECK(r.is_err() && r.unwrap_err().message == "assertion failed: idx < self.bit_len");
}

static void test_take_panics_and_wrap() {
  Bytes b(40);
  for (size_t i = 0; i < b.size(); ++i) b[i] = (uint8_t)i;
  const auto a = FixedSizeBinaryArray::from({Bytes(b.begin(), b.begin() + 20), Bytes(b.begin() + 20, b.end())}, 20);
  // idx * 20 wraps to 0 for idx = 2^62: the reference reads row 0
  auto r = take(a, PrimitiveArray<uint64_t>::from(std::vector<uint64_t>{1ull << 62, 1}));
  CHECK(r.is_ok());
  if (r.is_ok()) {
    auto t = r.unwrap();
    CHECK(fsb(t).value(0) == Bytes(b.begin(), b.begin() + 20) && fsb(t).value(1) == Bytes(b.begin() + 20, b.end()));
  }
  r = take(a, PrimitiveArray<int64_t>::from(std::vector<int64_t>{0, -1}));
  CHECK(r.is_err() && r.unwrap_err().message == "range start index 18446744073709551596 out of range for slice of length 40" &&
        r.unwrap_err().index == 1);
  r = take(a, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{2}));
  CHECK(r.is_err() && r.unwrap_err().message == "range end index 60 out of range for slice of length 40");
  r = take(a, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{3}));
  CHECK(r.is_err() && r.unwrap_err().message == "range start index 60 out of range for slice of length 40");
  const auto n4 = FixedSizeBinaryArray::from({Bytes{1, 2, 3, 4}}, 4);
  r = take(n4, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{0, 7}));
  CHECK(r.is_err() && r.unwrap_err().message == "Out-of-bounds index 7");
  r = take(n4, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{7}), TakeOptions{true});
  CHECK(r.is_err() && r.unwrap_err().message == "Compute error: Array index out of bounds, cannot get item at index 7 from 1 entries");
}

static void test_slice_and_nesting() {
  const auto a = FixedSizeBinaryArray::from({Bytes{1, 1, 1}, std::nullopt, Bytes{3, 3, 3}, Bytes{4, 4, 4}, Bytes{5, 5, 5}}, 3);
  const auto s = a.slice(1, 3);
  CHECK(s.len() == 3 && s.value(1) == (Bytes{3, 3, 3}) && s.is_null(0));
  auto f = filter(s, pred({true, false, true})).unwrap();
  CHECK(f->len() == 2 && f->is_null(0) && fsb(f).value(1) == (Bytes{4, 4, 4}));
  // a list of FixedSizeBinary: the child is extended (every row kept, an empty NullBuffer dropped)
  const auto child = std::make_shared<FixedSizeBinaryArray>(FixedSizeBinaryArray::from({Bytes{1, 2, 3}, Bytes{4, 5, 6}, Bytes{7, 8, 9}}, 3));
  const auto l = ListArray::from({0, 1, 3}, child);
  auto lf = filter(l, pred({false, true})).unwrap();
  const auto &lc = fsb(detail::list_values(*lf));
  CHECK(lc.len() == 2 && lc.value(0) == (Bytes{4, 5, 6}) && lc.value(1) == (Bytes{7, 8, 9}) && !lc.nulls());
  // a struct field
  const auto st = StructArray::from({std::make_shared<FixedSizeBinaryArray>(a), std::make_shared<PrimitiveArray<int32_t>>(
                                                                                     PrimitiveArray<int32_t>::from(std::vector<int32_t>{1, 2, 3, 4, 5}))});
  auto t = take(st, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{4, 1})).unwrap();
  const auto &tf = fsb(static_cast<const StructArray &>(*t).column(0));
  CHECK(tf.len() == 2 && tf.value(0) == (Bytes{5, 5, 5}) && tf.is_null(1));
}

static void test_record_batches() {
  const auto a = std::make_shared<FixedSizeBinaryArray>(FixedSizeBinaryArray::from({Bytes(20, 1), std::nullopt, Bytes(20, 3)}, 20));
  const auto b = std::make_shared<PrimitiveArray<int32_t>>(PrimitiveArray<int32_t>::from(std::vector<int32_t>{10, 20, 30}));
  Schema schema{{"a", DataType::FixedSizeBinary}, {"b", DataType::Int32}};
  const auto batch = RecordBatch::try_new(schema, {a, b}).unwrap();
  auto f = filter_record_batch(batch, pred({false, true, true})).unwrap();
  CHECK(f.num_rows() == 2 && f.column(0)->is_null(0) && fsb(f.column(0)).value(1) == Bytes(20, 3));
  auto t = take_record_batch(batch, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{2, 0})).unwrap();
  CHECK(t.num_rows() == 2 && fsb(t.column(0)).value(0) == Bytes(20, 3) && fsb(t.column(0)).value(1) == Bytes(20, 1) && !t.column(0)->nulls());
}

// FixedSizeBinary arrays of any width reached through an ArrayRef (as RecordBatch::column returns them) give the results of
// the concrete-type calls in filter, FilterPredicate::filter and take
static void test_array_ref() {
  for (int32_t w : {0, 3, 16}) {
    Rows rows;
    for (uint8_t k = 1; k <= 4; ++k) rows.push_back(k == 2 ? std::nullopt : std::optional<Bytes>(Bytes((size_t)w, k)));
    const auto a = FixedSizeBinaryArray::from(rows, w);
    const ArrayRef ref = std::make_shared<FixedSizeBinaryArray>(a);
    auto bytes = [](const ArrayRef &r) {
      Rows out;
      for (int64_t i = 0; i < r->len(); ++i) out.push_back(r->is_null(i) ? std::nullopt : std::optional<Bytes>(fsb(r).value(i)));
      return out;
    };
    auto same = [&](Result<ArrayRef> got, const ArrayRef &want) {
      if (got.is_err()) return false;
      const ArrayRef g = got.unwrap();
      return g->data_type() == DataType::FixedSizeBinary && fsb(g).value_length() == w && g->len() == want->len() && bytes(g) == bytes(want);
    };
    const auto p = pred({true, true, false, true});
    const auto idx = UInt32Array::from(std::vector<uint32_t>{3, 1, 0});
    const ArrayRef f = filter(a, p).unwrap(), t = take(a, idx).unwrap();
    CHECK(same(filter(*ref, p), f));
    CHECK(same(FilterBuilder(p).build().filter(*ref), f));
    CHECK(same(take(*ref, idx), t));
  }
}

int main() {
  try {
    Context::get();
  } catch (const std::exception &e) {
    std::printf("SKIP: %s (no CPU fallback)\n", e.what());
    return 77;
  }
  test_filter_fixed_binary();
  take_with_nulls_indices(4);  // test_take_fixed_size_binary_with_nulls_indices
  take_with_nulls_indices(5);  // test_take_fixed_size_binary_with_nulls_indices_not_optimized_length
  test_width_zero_length_rule();
  test_take_panics_and_wrap();
  test_slice_and_nesting();
  test_record_batches();
  test_array_ref();
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
