// test_host_list.cpp — the reference's list filter / take tests (arrow-select/src/filter.rs:1559, :2017, :2055;
// arrow-select/src/take.rs:1827-2115, :2186, :2298, :2532-2600, :2702) re-expressed against the C++ host mirror
// (arrow_cuda.hpp). Runs on a CUDA device (no CPU fallback); exits 77 when there is none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_list   (exit code 0 = all passed)
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
using Row = O<std::vector<O<int32_t>>>;
using Rows = std::vector<Row>;

static ArrayRef ints(const std::vector<O<int32_t>> &v) { return std::make_shared<Int32Array>(Int32Array::from(v)); }
static std::vector<O<int32_t>> iv(std::initializer_list<int32_t> v) { return std::vector<O<int32_t>>(v.begin(), v.end()); }

// the logical rows of a list of Int32 (any of the three list types)
static Rows rows_of(const Array &a) {
  const auto &child = static_cast<const Int32Array &>(*compute::detail::list_values(a));
  const auto vals = child.to_vec();
  const auto valid = a.valid_mask();
  Rows out((size_t)a.len());
  for (int64_t i = 0; i < a.len(); ++i) {
    int64_t s, e;
    if (a.data_type() == DataType::FixedSizeList) {
      const int64_t w = static_cast<const FixedSizeListArray &>(a).value_length();
      s = i * w; e = s + w;
    } else if (a.data_type() == DataType::List) {
      const auto o = static_cast<const ListArray &>(a).value_offsets();
      s = o[(size_t)i]; e = o[(size_t)i + 1];
    } else {
      const auto o = static_cast<const LargeListArray &>(a).value_offsets();
      s = o[(size_t)i]; e = o[(size_t)i + 1];
    }
    if (valid[(size_t)i]) out[(size_t)i] = std::vector<O<int32_t>>(vals.begin() + s, vals.begin() + e);
  }
  return out;
}

template <class O_>
static std::vector<int64_t> offsets_of(const Array &a) {
  const auto o = static_cast<const GenericListArray<O_> &>(a).value_offsets();
  return std::vector<int64_t>(o.begin(), o.end());
}

// test_filter_list_array (filter.rs:1559)
static void test_filter_list_array() {
  auto a = LargeListArray::from({0, 3, 6, 8, 8}, ints(iv({0, 1, 2, 3, 4, 5, 6, 7})), {true, true, true, false});
  auto r = filter(a, BooleanArray::from(std::vector<bool>{false, true, false, true})).unwrap();
  CHECK((rows_of(*r) == Rows{iv({3, 4, 5}), std::nullopt}));
  CHECK((offsets_of<int64_t>(*r) == std::vector<int64_t>{0, 3, 3}));
}

// test_filter_fixed_size_list_arrays (:2017) and _with_null (:2055)
static void test_filter_fixed_size_list() {
  auto a = FixedSizeListArray::from(3, ints(iv({0, 1, 2, 3, 4, 5, 6, 7, 8})));
  CHECK((rows_of(*filter(a, BooleanArray::from(std::vector<bool>{true, false, false})).unwrap()) == Rows{iv({0, 1, 2})}));
  CHECK((rows_of(*filter(a, BooleanArray::from(std::vector<bool>{true, false, true})).unwrap()) == Rows{iv({0, 1, 2}), iv({6, 7, 8})}));
  auto n = FixedSizeListArray::from(2, ints(iv({0, 1, 2, 3, 4, 5, 6, 7, 8, 9})), {true, false, false, true, true});
  auto r = filter(n, BooleanArray::from(std::vector<bool>{true, true, false, true, false})).unwrap();
  CHECK((rows_of(*r) == Rows{iv({0, 1}), std::nullopt, iv({6, 7})}));
}

// test_take_list / _with_value_nulls / _with_nulls (take.rs:1827-2115), for List and LargeList
template <class L, class O_>
static void test_take_list_macros() {
  const auto idx = UInt32Array::from(std::vector<O<uint32_t>>{3, std::nullopt, 1, 2, 0});
  auto a = L::from({0, 3, 6, 6, 8}, ints(iv({0, 0, 0, -1, -2, -1, 2, 3})));
  auto r = take(a, idx).unwrap();
  CHECK((rows_of(*r) == Rows{iv({2, 3}), std::nullopt, iv({-1, -2, -1}), iv({}), iv({0, 0, 0})}));
  CHECK((offsets_of<O_>(*r) == std::vector<int64_t>{0, 2, 2, 5, 5, 8}));

  const auto idx2 = UInt32Array::from(std::vector<O<uint32_t>>{2, std::nullopt, 1, 3, 0});
  auto b = L::from({0, 3, 6, 7, 9}, ints({0, std::nullopt, 0, -1, -2, 3, std::nullopt, 5, std::nullopt}), {true, true, true, true});
  r = take(b, idx2).unwrap();
  CHECK((rows_of(*r) == Rows{std::vector<O<int32_t>>{std::nullopt}, std::nullopt, iv({-1, -2, 3}), std::vector<O<int32_t>>{5, std::nullopt},
                             std::vector<O<int32_t>>{0, std::nullopt, 0}}));
  CHECK((offsets_of<O_>(*r) == std::vector<int64_t>{0, 1, 1, 4, 6, 9}));

  auto c = L::from({0, 3, 6, 6, 8}, ints({0, std::nullopt, 0, -1, -2, 3, 5, std::nullopt}), {true, true, false, true});
  r = take(c, idx2).unwrap();
  CHECK((rows_of(*r) == Rows{std::nullopt, std::nullopt, iv({-1, -2, 3}), std::vector<O<int32_t>>{5, std::nullopt},
                             std::vector<O<int32_t>>{0, std::nullopt, 0}}));
  CHECK((offsets_of<O_>(*r) == std::vector<int64_t>{0, 0, 0, 3, 5, 8}));
  CHECK((r->valid_mask() == std::vector<bool>{false, false, true, true, true}));
}

// test_take_list_out_of_bounds (:2298)
static void test_take_list_out_of_bounds() {
  auto a = ListArray::from({0, 3, 6, 8}, ints(iv({0, 0, 0, -1, -2, -1, 2, 3})));
  auto e = take(a, UInt32Array::from(std::vector<uint32_t>{1000}));
  CHECK(e.is_err() && e.unwrap_err().status == ACU_ERR_PANIC_OUT_OF_BOUNDS &&
        e.unwrap_err().to_string() == "index out of bounds: the len is 4 but the index is 1000");
}

// test_take_sliced_list / _large_list / _with_value_nulls (:2532-2600)
template <class L>
static void test_take_sliced() {
  const auto idx = UInt32Array::from(std::vector<O<uint32_t>>{3, 0, std::nullopt, 2, 1});
  auto a = L::from({0, 2, 5, 5, 5, 7, 8}, ints(iv({0, 1, 2, 3, 4, 5, 6, 7})), {true, true, false, true, true, true}).slice(1, 4);
  CHECK((rows_of(*take(a, idx).unwrap()) == Rows{iv({5, 6}), iv({2, 3, 4}), std::nullopt, iv({}), std::nullopt}));
  const auto idx2 = UInt32Array::from(std::vector<O<uint32_t>>{2, 0, std::nullopt, 3, 1});
  auto b = L::from({0, 1, 3, 3, 5, 5, 6}, ints({10, std::nullopt, 1, 2, std::nullopt, 3}), {true, true, false, true, true, true}).slice(1, 4);
  CHECK((rows_of(*take(b, idx2).unwrap()) == Rows{std::vector<O<int32_t>>{2, std::nullopt}, std::vector<O<int32_t>>{std::nullopt, 1},
                                                 std::nullopt, iv({}), std::nullopt}));
}

// test_take_fixed_size_list (:2186, the Int32 case) and test_take_fixed_size_list_null_indices (:2702)
static void test_take_fixed_size_list() {
  auto a = FixedSizeListArray::from(3, ints({std::nullopt, 1, 2, 3, 4, std::nullopt, 6, 7, 8}));
  CHECK((rows_of(*take(a, UInt32Array::from(std::vector<uint32_t>{2, 1, 0})).unwrap()) ==
         Rows{iv({6, 7, 8}), std::vector<O<int32_t>>{3, 4, std::nullopt}, std::vector<O<int32_t>>{std::nullopt, 1, 2}}));
  auto b = FixedSizeListArray::from(2, ints(iv({0, 1, 2, 3})));
  auto r = take(b, Int32Array::from(std::vector<O<int32_t>>{0, std::nullopt})).unwrap();
  const auto child = static_cast<const Int32Array &>(*static_cast<const FixedSizeListArray &>(*r).values()).to_vec();
  CHECK((child == std::vector<O<int32_t>>{0, 1, std::nullopt, std::nullopt}));
}

// A List filtered with a plan other than All goes through MutableArrayData (filter.rs:600), whose freeze keeps the
// child's NullBuffer only if the result has a null (arrow-data/src/transform/mod.rs:936): here the unselected row is
// empty, so the child plan selects all of [0, 4), and the child's only null lies past it. Under a top-level All the
// reference slices, and the child keeps its NullBuffer.
static void test_filter_child_plan_all() {
  auto a = ListArray::from({0, 2, 2, 4}, ints({0, 1, 2, 3, 4, 5, std::nullopt}));
  auto r = filter(a, BooleanArray::from(std::vector<bool>{true, false, true})).unwrap();
  CHECK((rows_of(*r) == Rows{iv({0, 1}), iv({2, 3})}));
  CHECK(!compute::detail::list_values(*r)->nulls().has_value());
  r = filter(a, BooleanArray::from(std::vector<bool>{true, true, true})).unwrap();
  CHECK(compute::detail::list_values(*r)->nulls().has_value());
}

// Every list type reached through an ArrayRef (as RecordBatch::column and every child accessor return it) takes the list
// path in filter, FilterPredicate::filter and take, with the results of the concrete-type calls
static bool same_list(Result<ArrayRef> got, const ArrayRef &want) {
  if (got.is_err()) return false;
  const ArrayRef g = got.unwrap();
  return g->data_type() == want->data_type() && rows_of(*g) == rows_of(*want);
}
template <class L>
static void check_array_ref(const L &a) {
  const ArrayRef ref = std::make_shared<L>(a);
  const auto p = BooleanArray::from(std::vector<bool>{true, false, true, true});
  const auto idx = UInt32Array::from(std::vector<uint32_t>{3, 0, 0});
  const ArrayRef f = filter(a, p).unwrap(), t = take(a, idx).unwrap();
  CHECK(same_list(filter(*ref, p), f));
  CHECK(same_list(FilterBuilder(p).build().filter(*ref), f));
  CHECK(same_list(take(*ref, idx), t));
}
static void test_array_ref() {
  check_array_ref(ListArray::from({0, 2, 2, 5, 6}, ints(iv({0, 1, 2, 3, 4, 5})), {true, false, true, true}));
  check_array_ref(LargeListArray::from({0, 2, 2, 5, 6}, ints(iv({0, 1, 2, 3, 4, 5}))));
  check_array_ref(FixedSizeListArray::from(2, ints(iv({0, 1, 2, 3, 4, 5, 6, 7}))));
}

int main() {
  try {
    Context::get();
  } catch (const std::exception &e) {
    std::printf("SKIP: %s (no CPU fallback)\n", e.what());
    return 77;
  }
  test_filter_list_array();
  test_filter_fixed_size_list();
  test_filter_child_plan_all();
  test_take_list_macros<ListArray, int32_t>();
  test_take_list_macros<LargeListArray, int64_t>();
  test_take_list_out_of_bounds();
  test_take_sliced<ListArray>();
  test_take_sliced<LargeListArray>();
  test_take_fixed_size_list();
  test_array_ref();
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
