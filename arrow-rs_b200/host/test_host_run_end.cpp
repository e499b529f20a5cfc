// test_host_run_end.cpp — the reference's RunEndEncoded filter / take tests (arrow-select/src/filter.rs:1429-1535;
// arrow-select/src/take.rs:2605-2660, :2912-3030) and RunArray::get_physical_indices (arrow-array/src/array/run_array.rs)
// re-expressed against the C++ host mirror (arrow_cuda.hpp). Runs on a CUDA device (no CPU fallback); exits 77 when there is
// none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_run_end   (exit code 0 = all passed)
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

template <class T> using O = std::optional<T>;

template <class T> static ArrayRef prim(const std::vector<T> &v) { return std::make_shared<PrimitiveArray<T>>(PrimitiveArray<T>::from(v)); }
static ArrayRef strs(const std::vector<std::string> &v) { return std::make_shared<StringArray>(StringArray::from(v)); }

// PrimitiveRunBuilder / StringRunBuilder::extend: equal neighbours share a run
template <class R, class V> static std::pair<std::vector<R>, std::vector<V>> runs(const std::vector<V> &logical) {
  std::vector<R> ends;
  std::vector<V> vals;
  for (size_t i = 0; i < logical.size(); ++i) {
    if (!vals.empty() && vals.back() == logical[i]) ends.back() = (R)(i + 1);
    else { ends.push_back((R)(i + 1)); vals.push_back(logical[i]); }
  }
  return {ends, vals};
}

template <class R> static const RunArray<R> &as_run(const ArrayRef &a) { return static_cast<const RunArray<R> &>(*a); }
template <class T> static std::vector<O<T>> prim_values(const ArrayRef &a) { return static_cast<const PrimitiveArray<T> &>(*a).to_vec(); }

// the logical values of a RunArray with primitive values
template <class R, class T> static std::vector<T> logical(const RunArray<R> &a) {
  const auto ends = a.run_ends();
  const auto vals = prim_values<T>(a.values());
  std::vector<T> out;
  for (int64_t i = 0; i < a.len(); ++i) {
    const size_t p = (size_t)(std::upper_bound(ends.begin(), ends.end(), a.offset() + i, [](int64_t x, R e) { return x < (int64_t)e; }) - ends.begin());
    out.push_back(*vals[p]);
  }
  return out;
}

// test_filter_run_end_encoding_array (filter.rs:1429)
static void test_filter_run_end_encoding_array() {
  auto a = Int64RunArray::from({2, 3, 8}, prim<int64_t>({7, -2, 9}));
  auto c = filter(a, BooleanArray::from(std::vector<bool>{true, false, true, false, true, false, true, false})).unwrap();
  const auto &r = as_run<int64_t>(c);
  CHECK(r.len() == 4);
  CHECK((r.run_ends() == std::vector<int64_t>{1, 2, 4}));
  CHECK((prim_values<int64_t>(r.values()) == std::vector<O<int64_t>>{7, -2, 9}));
}

// test_filter_run_end_encoding_array_sliced (filter.rs:1449)
static void test_filter_run_end_encoding_array_sliced() {
  auto a = Int64RunArray::from({2, 3, 8}, prim<int64_t>({7, -2, 9})).slice(2, 3);
  auto c = filter(a, BooleanArray::from(std::vector<bool>{true, false, true})).unwrap();
  CHECK((logical<int64_t, int64_t>(as_run<int64_t>(c)) == std::vector<int64_t>{-2, 9}));
}

// test_filter_run_end_encoding_array_remove_value (filter.rs:1466)
static void test_filter_run_end_encoding_array_remove_value() {
  auto a = Int32RunArray::from({2, 3, 8, 10}, prim<int32_t>({7, -2, 9, -8}));
  auto c = filter(a, BooleanArray::from(std::vector<bool>{false, true, false, false, true, false, true, false, false, false})).unwrap();
  const auto &r = as_run<int32_t>(c);
  CHECK(r.len() == 3);
  CHECK((r.run_ends() == std::vector<int32_t>{1, 3}));
  CHECK((prim_values<int32_t>(r.values()) == std::vector<O<int32_t>>{7, 9}));
}

// test_filter_run_end_encoding_array_remove_all_but_one (filter.rs:1486)
static void test_filter_run_end_encoding_array_remove_all_but_one() {
  auto a = Int16RunArray::from({2, 3, 8, 10}, prim<int16_t>({7, -2, 9, -8}));
  auto c = filter(a, BooleanArray::from(std::vector<bool>{false, false, false, false, false, false, true, false, false, false})).unwrap();
  const auto &r = as_run<int16_t>(c);
  CHECK(r.len() == 1);
  CHECK((r.run_ends() == std::vector<int16_t>{1}));
  CHECK((prim_values<int16_t>(r.values()) == std::vector<O<int16_t>>{9}));
}

// test_filter_run_end_encoding_array_empty (filter.rs:1505)
static void test_filter_run_end_encoding_array_empty() {
  auto a = Int64RunArray::from({2, 3, 8, 10}, prim<int64_t>({7, -2, 9, -8}));
  auto c = filter(a, BooleanArray::from(std::vector<bool>(10, false))).unwrap();
  CHECK(as_run<int64_t>(c).len() == 0);
  CHECK(as_run<int64_t>(c).values()->len() == 0);
}

// test_filter_run_end_encoding_array_max_value_gt_predicate_len (filter.rs:1518)
static void test_filter_run_end_encoding_array_max_value_gt_predicate_len() {
  auto a = Int64RunArray::from({2, 3, 8, 10}, prim<int64_t>({7, -2, 9, -8}));
  auto c = filter(a, BooleanArray::from(std::vector<bool>{false, true, true})).unwrap();
  const auto &r = as_run<int64_t>(c);
  CHECK(r.len() == 2);
  CHECK((r.run_ends() == std::vector<int64_t>{1, 2}));
  CHECK((prim_values<int64_t>(r.values()) == std::vector<O<int64_t>>{7, -2}));
}

// filter_array's length check (filter.rs:536-542)
static void test_filter_predicate_too_long() {
  auto a = Int32RunArray::from({2, 3}, prim<int32_t>({1, 2}));
  auto e = filter(a, BooleanArray::from(std::vector<bool>(4, true))).unwrap_err();
  CHECK(e.message == "Invalid argument error: Filter predicate of length 4 is larger than target array of length 3");
}

// test_take_runs (take.rs:2605)
static void test_take_runs() {
  auto rv = runs<int32_t, int32_t>({1, 1, 2, 2, 1, 1, 1, 2, 2, 1, 1, 2, 2});
  auto a = Int32RunArray::from(rv.first, prim<int32_t>(rv.second));
  auto c = take(a, Int32Array::from(std::vector<int32_t>{7, 2, 3, 7, 11, 4, 6})).unwrap();
  const auto &r = as_run<int32_t>(c);
  CHECK(r.len() == 7);
  CHECK((r.run_ends() == std::vector<int32_t>{5, 7}));
  CHECK((prim_values<int32_t>(r.values()) == std::vector<O<int32_t>>{2, 1}));
}

// test_take_runs_sliced (take.rs:2631)
static void test_take_runs_sliced() {
  auto rv = runs<int32_t, int32_t>({1, 1, 2, 2, 3, 3, 3, 4, 4, 5, 5, 6, 6});
  auto a = Int32RunArray::from(rv.first, prim<int32_t>(rv.second)).slice(4, 6);
  auto c = take(a, Int32Array::from(std::vector<int32_t>{0, 5, 5, 1, 4})).unwrap();
  const auto &r = as_run<int32_t>(c);
  CHECK((r.run_ends() == std::vector<int32_t>{1, 3, 4, 5}));
  CHECK((logical<int32_t, int32_t>(r) == std::vector<int32_t>{3, 5, 5, 3, 4}));
}

// test_take_run_empty_indices (take.rs:2912)
static void test_take_run_empty_indices() {
  auto rv = runs<int32_t, int32_t>({1, 1, 2, 2});
  auto a = Int32RunArray::from(rv.first, prim<int32_t>(rv.second));
  auto c = take(a, Int32Array::from(std::vector<int32_t>{})).unwrap();
  CHECK(c->len() == 0 && c->null_count() == 0);
  CHECK(as_run<int32_t>(c).run_ends().empty() && as_run<int32_t>(c).values()->len() == 0);
}

// test_take_run_end_encoded_merges_identical_runs (take.rs:2936)
static void test_take_merges_identical_runs() {
  auto rv = runs<int32_t, int32_t>({1, 1, 0, 0, 1, 1});
  auto a = Int32RunArray::from(rv.first, prim<int32_t>(rv.second));
  auto c = take(a, Int32Array::from(std::vector<int32_t>{0, 1, 4, 5})).unwrap();
  const auto &r = as_run<int32_t>(c);
  CHECK((r.run_ends() == std::vector<int32_t>{4}));
  CHECK((logical<int32_t, int32_t>(r) == std::vector<int32_t>{1, 1, 1, 1}));
}

// the logical values of a RunArray with Utf8 values
static std::vector<std::string> logical_strs(const RunArray<int32_t> &a) {
  const auto ends = a.run_ends();
  const auto vals = static_cast<const StringArray &>(*a.values()).to_vec();
  std::vector<std::string> out;
  for (int64_t i = 0; i < a.len(); ++i)
    out.push_back(*vals[(size_t)(std::upper_bound(ends.begin(), ends.end(), (int32_t)(a.offset() + i)) - ends.begin())]);
  return out;
}

// test_take_run_end_encoded_merges_identical_string_runs (take.rs:2964)
static void test_take_merges_identical_string_runs() {
  auto rv = runs<int32_t, std::string>({"bob", "bob", "alice", "alice", "bob", "bob"});
  auto a = Int32RunArray::from(rv.first, strs(rv.second));
  auto c = take(a, Int32Array::from(std::vector<int32_t>{0, 1, 4, 5})).unwrap();
  const auto &r = as_run<int32_t>(c);
  CHECK((r.run_ends() == std::vector<int32_t>{4}));
  CHECK((logical_strs(r) == std::vector<std::string>{"bob", "bob", "bob", "bob"}));
}

// test_take_run_end_encoded_mixed_runs (take.rs:2993)
static void test_take_mixed_runs() {
  auto rv = runs<int32_t, std::string>({"bob", "bob", "alice", "alice", "bob", "bob", "eve", "eve"});
  auto a = Int32RunArray::from(rv.first, strs(rv.second));
  auto c = take(a, Int32Array::from(std::vector<int32_t>{0, 0, 1, 4, 5, 2, 3, 2, 6, 7, 6})).unwrap();
  const auto &r = as_run<int32_t>(c);
  CHECK((r.run_ends() == std::vector<int32_t>{5, 8, 11}));
  CHECK((logical_strs(r) == std::vector<std::string>{"bob", "bob", "bob", "bob", "bob", "alice", "alice", "alice", "eve", "eve", "eve"}));
}

// RunArray::get_physical_indices (run_array.rs:1195-1292): every logical index, shuffled and repeated, at every slice; an
// index past the length names the largest index
static void test_get_physical_indices() {
  std::vector<int32_t> ends;
  int32_t e = 0;
  for (int k = 0; e < 80; ++k) { e = std::min(80, e + 1 + (k * 7) % 5); ends.push_back(e); }
  std::vector<int32_t> vals(ends.size());
  for (size_t k = 0; k < vals.size(); ++k) vals[k] = (int32_t)k;
  auto a = Int32RunArray::from(ends, prim<int32_t>(vals));
  for (int64_t off = 0; off < 80; ++off) {
    for (int64_t len = 1; off + len <= 80; len += 9) {
      auto s = a.slice(off, len);
      std::vector<uint32_t> ix;
      for (int64_t i = len - 1; i >= 0; --i) { ix.push_back((uint32_t)i); ix.push_back((uint32_t)((i * 5) % len)); }
      auto p = s.get_physical_indices(ix).unwrap();
      bool ok = true;
      for (size_t j = 0; j < ix.size(); ++j) {
        const int64_t x = off + ix[j];
        ok = ok && (p[j] == 0 ? 0 : ends[p[j] - 1]) <= x && x < ends[p[j]];
      }
      CHECK(ok);
      // the device take maps the same indices to the same runs: its values are those runs' values
      auto t = take(s, UInt32Array::from(ix)).unwrap();
      std::vector<int32_t> want;
      for (size_t j = 0; j < ix.size(); ++j) want.push_back((int32_t)p[j]);
      CHECK((logical<int32_t, int32_t>(as_run<int32_t>(t)) == want));
    }
  }
  auto err = a.slice(3, 20).get_physical_indices(std::vector<uint32_t>{0, 25, 19, 40, 2}).unwrap_err();
  CHECK(err.message == "Invalid argument error: Logical index 40 is out of bounds for RunArray of length 20");
}

// take_run's errors: the largest index value (null slots included) past the length, check_bounds, the Int16 unwrap panic
static void test_take_errors() {
  auto a = Int16RunArray::from({3, 5}, prim<int8_t>({1, 2}));
  auto null_over_oob = UInt32Array::from(std::vector<O<uint32_t>>{0, std::nullopt, 4});
  CHECK(take(a, null_over_oob).is_ok());
  auto e = take(a, UInt32Array::from(std::vector<uint32_t>{0, 9, 4})).unwrap_err();
  CHECK(e.message == "Invalid argument error: Logical index 9 is out of bounds for RunArray of length 5");
  e = take(a, Int32Array::from(std::vector<int32_t>{0, -1}), TakeOptions{true}).unwrap_err();
  CHECK(e.message == "Compute error: Array index out of bounds, cannot get item at index -1 from 5 entries");
  CHECK(take(a, UInt16Array::from(std::vector<uint16_t>(32767, 1))).is_ok());
  e = take(a, UInt16Array::from(std::vector<uint16_t>(32768, 1))).unwrap_err();
  CHECK(e.status == ACU_ERR_PANIC_OUT_OF_BOUNDS && e.message == "called `Option::unwrap()` on a `None` value");
}

// A RunArray of every run-end type reached through an ArrayRef (as RecordBatch::column and every child accessor return
// it) takes the run-end path in filter, FilterPredicate::filter and take, with the results of the concrete-type calls
template <class R>
static void check_array_ref() {
  const auto a = RunArray<R>::from({2, 3, 8}, prim<int32_t>({7, -2, 9}));
  const ArrayRef ref = std::make_shared<RunArray<R>>(a);
  auto same = [](Result<ArrayRef> got, const ArrayRef &want) {
    if (got.is_err()) return false;
    const ArrayRef g = got.unwrap();
    return g->data_type() == DataType::RunEndEncoded && logical<R, int32_t>(as_run<R>(g)) == logical<R, int32_t>(as_run<R>(want));
  };
  const auto p = BooleanArray::from(std::vector<bool>{true, false, true, false, true, false, true, false});
  const auto idx = UInt32Array::from(std::vector<uint32_t>{7, 2, 0, 0});
  const ArrayRef f = filter(a, p).unwrap(), t = take(a, idx).unwrap();
  CHECK(same(filter(*ref, p), f));
  CHECK(same(FilterBuilder(p).build().filter(*ref), f));
  CHECK(same(take(*ref, idx), t));
}

// RunEndEncoded is filtered and taken at the top level only: below a struct or a list it is refused
static void test_nested_run_end_refused() {
  const ArrayRef run = std::make_shared<Int32RunArray>(Int32RunArray::from({2, 3}, prim<int32_t>({1, 2})));
  const auto p = BooleanArray::from(std::vector<bool>{true, false, true});
  const auto idx = UInt32Array::from(std::vector<uint32_t>{2, 0});
  const std::string f = "Not yet implemented: filter of a RunEndEncoded array below the top level";
  const std::string t = "Not yet implemented: take of a RunEndEncoded array below the top level";
  auto refused = [](Result<ArrayRef> r, const std::string &msg) {
    return r.is_err() && r.unwrap_err().status == ACU_ERR_NOT_YET_IMPLEMENTED && r.unwrap_err().message == msg;
  };
  const auto s = StructArray::from({run});
  CHECK(refused(filter(s, p), f));
  CHECK(refused(take(s, idx), t));
  const auto l = ListArray::from({0, 1, 3}, run);
  CHECK(refused(filter(l, BooleanArray::from(std::vector<bool>{false, true})), f));
  CHECK(refused(take(l, idx.slice(1, 1)), t));
}

int main() {
  try {
    Context::get();
  } catch (const std::exception &e) {
    std::printf("SKIP: %s (no CPU fallback)\n", e.what());
    return 77;
  }
  test_filter_run_end_encoding_array();
  test_filter_run_end_encoding_array_sliced();
  test_filter_run_end_encoding_array_remove_value();
  test_filter_run_end_encoding_array_remove_all_but_one();
  test_filter_run_end_encoding_array_empty();
  test_filter_run_end_encoding_array_max_value_gt_predicate_len();
  test_filter_predicate_too_long();
  test_take_runs();
  test_take_runs_sliced();
  test_take_run_empty_indices();
  test_take_merges_identical_runs();
  test_take_merges_identical_string_runs();
  test_take_mixed_runs();
  test_get_physical_indices();
  test_take_errors();
  check_array_ref<int16_t>();
  check_array_ref<int32_t>();
  check_array_ref<int64_t>();
  test_nested_run_end_refused();
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
