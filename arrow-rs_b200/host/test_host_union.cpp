// test_host_union.cpp — the reference's Struct and Union filter / take tests (arrow-select/src/filter.rs:2081-2370;
// arrow-select/src/take.rs:2343-2405, :2731-2871) re-expressed against the C++ host mirror (arrow_cuda.hpp). Runs on a
// CUDA device (no CPU fallback); exits 77 when there is none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_union   (exit code 0 = all passed)
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

template <class T> static ArrayRef prim(const std::vector<O<T>> &v) { return std::make_shared<PrimitiveArray<T>>(PrimitiveArray<T>::from(v)); }
static ArrayRef strs(const std::vector<O<std::string>> &v) { return std::make_shared<StringArray>(StringArray::from(v)); }
template <class T> static std::vector<O<T>> vals(const ArrayRef &a) { return static_cast<const PrimitiveArray<T> &>(*a).to_vec(); }
static std::vector<O<std::string>> svals(const ArrayRef &a) { return static_cast<const StringArray &>(*a).to_vec(); }
static const UnionArray &as_union(const ArrayRef &a) { return static_cast<const UnionArray &>(*a); }
static const StructArray &as_struct(const ArrayRef &a) { return static_cast<const StructArray &>(*a); }
static BooleanArray pred(const std::vector<bool> &b) { return BooleanArray::from(b); }

// UnionBuilder::new_dense / new_sparse with fields A: Int32 (type id 0) and B: Float64 (type id 1); a row is (0, a) or (1, b)
struct Row { int8_t t; O<double> v; };
static UnionArray ab_union(const std::vector<Row> &rows, bool dense) {
  std::vector<int8_t> tids;
  std::vector<int32_t> offs;
  std::vector<O<int32_t>> a;
  std::vector<O<double>> b;
  for (const Row &r : rows) {
    tids.push_back(r.t);
    if (dense) {
      offs.push_back(r.t == 0 ? (int32_t)a.size() : (int32_t)b.size());
      if (r.t == 0) a.push_back(r.v ? O<int32_t>((int32_t)*r.v) : std::nullopt);
      else b.push_back(r.v);
    } else {
      a.push_back(r.t == 0 && r.v ? O<int32_t>((int32_t)*r.v) : std::nullopt);
      b.push_back(r.t == 1 ? r.v : std::nullopt);
    }
  }
  return UnionArray::try_new({0, 1}, tids, dense ? O<std::vector<int32_t>>(offs) : std::nullopt, {prim<int32_t>(a), prim<double>(b)}).unwrap();
}
// compare_union_arrays (filter.rs:2187-2227): the type id and the slot's value (or null) of every row
static std::vector<Row> union_rows(const UnionArray &u) {
  const auto t = u.type_ids();
  const auto o = u.value_offsets();
  const auto a = vals<int32_t>(u.child(0));
  const auto b = vals<double>(u.child(1));
  std::vector<Row> out;
  for (size_t i = 0; i < t.size(); ++i) {
    const size_t k = u.is_dense() ? (size_t)o[i] : i;
    if (t[i] == 0) out.push_back({0, a[k] ? O<double>(*a[k]) : std::nullopt});
    else out.push_back({1, b[k]});
  }
  return out;
}
static bool same_rows(const std::vector<Row> &x, const std::vector<Row> &y) {
  if (x.size() != y.size()) return false;
  for (size_t i = 0; i < x.size(); ++i)
    if (x[i].t != y[i].t || x[i].v != y[i].v) return false;
  return true;
}

// test_filter_union_array (filter.rs:2081-2111) over the dense and the sparse builder
static void test_filter_union_array(bool dense) {
  const UnionArray u = ab_union({{0, 1}, {1, 3.2}, {0, 34}}, dense);
  CHECK(same_rows(union_rows(as_union(filter(u, pred({true, false, false})).unwrap())), {{0, 1}}));
  CHECK(same_rows(union_rows(as_union(filter(u, pred({true, false, true})).unwrap())), {{0, 1}, {0, 34}}));
  CHECK(same_rows(union_rows(as_union(filter(u, pred({true, true, false})).unwrap())), {{0, 1}, {1, 3.2}}));
}

// test_filter_run_union_array_dense: to_data() equality with the builder's A 1, A 3
static void test_filter_run_union_array_dense() {
  const UnionArray u = UnionArray::try_new({0}, {0, 0, 0}, std::vector<int32_t>{0, 1, 2}, {prim<int32_t>({1, 3, 34})}).unwrap();
  const auto r = filter(u, pred({true, true, false})).unwrap();
  CHECK((as_union(r).type_ids() == std::vector<int8_t>{0, 0}));
  CHECK((as_union(r).value_offsets() == std::vector<int32_t>{0, 1}));
  CHECK((vals<int32_t>(as_union(r).child(0)) == std::vector<O<int32_t>>{1, 3}));
}

// test_filter_union_array_dense_with_nulls / test_filter_union_array_sparse_with_nulls
static void test_filter_union_array_with_nulls(bool dense) {
  const UnionArray u = ab_union({{0, 1}, {1, 3.2}, {1, std::nullopt}, {0, 34}}, dense);
  if (dense) CHECK(same_rows(union_rows(as_union(filter(u, pred({true, true, false, false})).unwrap())), {{0, 1}, {1, 3.2}}));
  CHECK(same_rows(union_rows(as_union(filter(u, pred({true, false, true, false})).unwrap())), {{0, 1}, {1, std::nullopt}}));
}

// test_filter_struct (filter.rs:2250-2318)
static void test_filter_struct() {
  const auto p = pred({true, false, true, false});
  const ArrayRef a = strs({"hello", " ", "world", "!"}), b = prim<int32_t>({5, 6, 7, 8});
  for (int with_b = 0; with_b < 2; ++with_b) {
    for (int with_nulls = 0; with_nulls < 2; ++with_nulls) {
      const std::vector<ArrayRef> cols = with_b ? std::vector<ArrayRef>{a, b} : std::vector<ArrayRef>{a};
      const StructArray s = StructArray::from(cols, with_nulls ? std::vector<bool>{true, false, false, true} : std::vector<bool>{});
      const auto r = filter(s, p).unwrap();
      const auto &rs = as_struct(r);
      CHECK(rs.len() == 2);
      CHECK((svals(rs.column(0)) == std::vector<O<std::string>>{"hello", "world"}));
      if (with_b) CHECK((vals<int32_t>(rs.column(1)) == std::vector<O<int32_t>>{5, 7}));
      CHECK(rs.nulls().has_value() == (with_nulls == 1));
      if (with_nulls) CHECK((rs.valid_mask() == std::vector<bool>{true, false}));
    }
  }
}

// test_filter_empty_struct (filter.rs:2321-2370)
static void test_filter_empty_struct() {
  const ArrayRef c = std::make_shared<StructArray>(StructArray::new_empty_fields(3, {true, true, true}));
  const StructArray a = StructArray::from({prim<int64_t>({std::nullopt, std::nullopt, std::nullopt}), c}, {true, true, true});
  const auto r = filter(a, pred({true, false, true})).unwrap();
  CHECK(r->len() == 2);
  CHECK(as_struct(r).column(1)->len() == 2);
}

// create_test_struct (take.rs:1236-1260): a: Boolean, b: Int32; a null row is null in both columns
static StructArray test_struct(const std::vector<O<std::pair<bool, int32_t>>> &rows) {
  std::vector<O<bool>> a;
  std::vector<O<int32_t>> b;
  std::vector<bool> valid;
  for (const auto &r : rows) {
    a.push_back(r ? O<bool>(r->first) : std::nullopt);
    b.push_back(r ? O<int32_t>(r->second) : std::nullopt);
    valid.push_back(r.has_value());
  }
  return StructArray::from({std::make_shared<BooleanArray>(BooleanArray::from(a)), prim<int32_t>(b)}, valid);
}
static std::vector<O<std::pair<bool, int32_t>>> struct_rows(const StructArray &s) {
  const auto a = static_cast<const BooleanArray &>(*s.column(0)).to_vec();
  const auto b = vals<int32_t>(s.column(1));
  const auto v = s.valid_mask();
  std::vector<O<std::pair<bool, int32_t>>> out;
  for (size_t i = 0; i < v.size(); ++i) out.push_back(v[i] ? O<std::pair<bool, int32_t>>({*a[i], *b[i]}) : std::nullopt);
  return out;
}
static const std::vector<O<std::pair<bool, int32_t>>> kStruct{{{true, 42}}, {{false, 28}}, {{false, 19}}, {{true, 31}}, std::nullopt};

// test_take_struct (take.rs:2343-2377)
static void test_take_struct() {
  const StructArray s = test_struct(kStruct);
  const auto r = take(s, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{0, 3, 1, 0, 2, 4})).unwrap();
  CHECK(r->len() == 6);
  CHECK(r->null_count() == 1);
  CHECK((struct_rows(as_struct(r)) == std::vector<O<std::pair<bool, int32_t>>>{{{true, 42}}, {{true, 31}}, {{false, 28}}, {{true, 42}},
                                                                               {{false, 19}}, std::nullopt}));
  const StructArray e = StructArray::new_empty_fields(6, {false, true, false, true, false, true});
  const auto re = take(e, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{0, 2, 1, 4})).unwrap();
  CHECK(re->len() == 4);
  CHECK((re->valid_mask() == std::vector<bool>{false, false, true, false}));
}

// test_take_struct_with_null_indices (take.rs:2380-2405)
static void test_take_struct_with_null_indices() {
  const StructArray s = test_struct(kStruct);
  const auto idx = PrimitiveArray<uint32_t>::from(std::vector<O<uint32_t>>{std::nullopt, 3, 1, std::nullopt, 0, 4});
  const auto r = take(s, idx).unwrap();
  CHECK(r->null_count() == 3);
  CHECK((struct_rows(as_struct(r)) == std::vector<O<std::pair<bool, int32_t>>>{std::nullopt, {{true, 31}}, {{false, 28}}, std::nullopt,
                                                                               {{true, 42}}, std::nullopt}));
}

// test_take_union_sparse (take.rs:2731-2768)
static void test_take_union_sparse() {
  const ArrayRef structs = std::make_shared<StructArray>(test_struct(kStruct));
  const ArrayRef strings = strs({"a", std::nullopt, "c", std::nullopt, "d"});
  const UnionArray u = UnionArray::try_new({0, 1}, {1, 1, 1, 1, 1}, std::nullopt, {structs, strings}).unwrap();
  const auto r = take(u, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{0, 3, 1, 0, 2, 4})).unwrap();
  CHECK((svals(as_union(r).child(1)) == std::vector<O<std::string>>{"a", std::nullopt, std::nullopt, "a", "c", "d"}));
}

// test_take_union_dense (take.rs:2771-2826)
static void test_take_union_dense() {
  const UnionArray u = UnionArray::try_new({0, 1}, {0, 1, 1, 0, 0, 1, 0}, std::vector<int32_t>{0, 0, 1, 1, 2, 2, 3},
                                           {prim<uint32_t>({10, 20, 30, 40}), strs({"a", std::nullopt, "c", "d"})}).unwrap();
  const auto r = take(u, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{0, 3, 1, 0, 2, 4})).unwrap();
  CHECK((as_union(r).value_offsets() == std::vector<int32_t>{0, 1, 0, 2, 1, 3}));
  CHECK((as_union(r).type_ids() == std::vector<int8_t>{0, 0, 1, 0, 1, 0}));
  CHECK((vals<uint32_t>(as_union(r).child(0)) == std::vector<O<uint32_t>>{10, 20, 10, 30}));
  CHECK((svals(as_union(r).child(1)) == std::vector<O<std::string>>{"a", std::nullopt}));
}

// test_take_union_dense_using_builder (take.rs:2829-2852)
static void test_take_union_dense_using_builder() {
  const UnionArray u = ab_union({{0, 1}, {1, 3.0}, {0, 4}, {0, 5}, {1, 2.0}}, true);
  const auto r = take(u, PrimitiveArray<uint32_t>::from(std::vector<uint32_t>{2, 0, 1, 2})).unwrap();
  const UnionArray e = ab_union({{0, 4}, {0, 1}, {1, 3.0}, {0, 4}}, true);
  CHECK(as_union(r).type_ids() == e.type_ids());
  CHECK(as_union(r).value_offsets() == e.value_offsets());
  CHECK(vals<int32_t>(as_union(r).child(0)) == vals<int32_t>(e.child(0)));
  CHECK(vals<double>(as_union(r).child(1)) == vals<double>(e.child(1)));
}

// test_take_union_dense_all_match_issue_6206 (take.rs:2855-2871)
static void test_take_union_dense_all_match_issue_6206() {
  const UnionArray u = UnionArray::try_new({0}, {0, 0, 0, 0, 0}, std::vector<int32_t>{0, 1, 2, 3, 4}, {prim<int64_t>({1, 2, 3, 4, 5})}).unwrap();
  const auto r = take(u, PrimitiveArray<int64_t>::from(std::vector<int64_t>{0, 2, 4})).unwrap();
  CHECK(r->len() == 3);
  CHECK((vals<int64_t>(as_union(r).child(0)) == std::vector<O<int64_t>>{1, 3, 5}));
}

// UnionArray::try_new's validation: a null out-of-bounds index takes type id 0, which names no field here
static void test_take_union_type_id_validation() {
  const UnionArray u = UnionArray::try_new({3, 7}, {3, 7}, std::vector<int32_t>{0, 0}, {prim<int32_t>({1}), prim<int32_t>({2})}).unwrap();
  const std::vector<uint32_t> raw{0, 99};  // index 1 is null and out of bounds: take_native gives it type id 0
  const PrimitiveArray<uint32_t> idx(Buffer::from_host(raw.data(), raw.size() * 4), 2, nulls_from_mask({true, false}));
  const auto r = take(u, idx);
  CHECK(r.is_err() && r.unwrap_err().message == "Invalid argument error: Type Ids values must match one of the field type ids");
  CHECK(UnionArray::try_new({0}, {1}, std::nullopt, {prim<int32_t>({1})}).is_err());
}

// Struct and Union arrays reached through an ArrayRef (as RecordBatch::column and every child accessor return them) take
// their own paths in filter, FilterPredicate::filter and take, with the results of the concrete-type calls
template <class A, class Rows>
static void check_array_ref(const A &a, const BooleanArray &p, const UInt32Array &idx, Rows rows) {
  const ArrayRef ref = std::make_shared<A>(a);
  auto same = [&](Result<ArrayRef> got, const ArrayRef &want) {
    if (got.is_err()) return false;
    const ArrayRef g = got.unwrap();
    return g->data_type() == a.data_type() && rows(g) == rows(want);
  };
  const ArrayRef f = filter(a, p).unwrap(), t = take(a, idx).unwrap();
  CHECK(same(filter(*ref, p), f));
  CHECK(same(FilterBuilder(p).build().filter(*ref), f));
  CHECK(same(take(*ref, idx), t));
}
static void test_array_ref() {
  const auto idx = UInt32Array::from(std::vector<uint32_t>{2, 0, 2});
  for (bool dense : {true, false}) {
    auto rows = [](const ArrayRef &r) {
      std::vector<std::pair<int8_t, O<double>>> out;
      for (const Row &x : union_rows(as_union(r))) out.push_back({x.t, x.v});
      return out;
    };
    check_array_ref(ab_union({{0, 1}, {1, 3.2}, {0, 34}}, dense), pred({true, false, true}), idx, rows);
  }
  check_array_ref(test_struct(kStruct), pred({true, false, true, false, true}), idx, [](const ArrayRef &r) { return struct_rows(as_struct(r)); });
}

int main() {
  try {
    Context::get();
  } catch (const std::exception &e) {
    std::printf("SKIP: %s (no CPU fallback)\n", e.what());
    return 77;
  }
  test_filter_union_array(true);
  test_filter_union_array(false);
  test_filter_run_union_array_dense();
  test_filter_union_array_with_nulls(true);
  test_filter_union_array_with_nulls(false);
  test_filter_struct();
  test_filter_empty_struct();
  test_take_struct();
  test_take_struct_with_null_indices();
  test_take_union_sparse();
  test_take_union_dense();
  test_take_union_dense_using_builder();
  test_take_union_dense_all_match_issue_6206();
  test_take_union_type_id_validation();
  test_array_ref();
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
