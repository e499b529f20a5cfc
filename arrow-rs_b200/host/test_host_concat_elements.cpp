// test_host_concat_elements.cpp — the reference's concat_elements tests (arrow-string/src/concat_elements.rs:478-956) on
// Utf8 and Utf8View, re-expressed against the C++ host mirror (arrow_cuda.hpp). Runs on a CUDA device (no CPU
// fallback); exits 77 when there is none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_concat_elements   (exit code 0 = all passed)
#include <cstdio>
#include <functional>

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
using S = std::vector<O<std::string>>;

static S strs(std::initializer_list<const char *> v) {
  S out;
  for (const char *s : v) out.push_back(s ? O<std::string>(s) : std::nullopt);
  return out;
}

static std::vector<O<std::string>> dyn_vec(const StringArray &l, const StringArray &r) {
  return static_cast<const StringArray &>(*concat_elements_dyn(l, r).unwrap()).to_vec();
}

// test_string_concat, _empty_string, _no_null, _error (:484-543)
static void test_string_concat() {
  CHECK(dyn_vec(StringArray::from(strs({"foo", "bar", nullptr})), StringArray::from(strs({nullptr, "yyy", "zzz"}))) ==
        strs({nullptr, "baryyy", nullptr}));
  CHECK(dyn_vec(StringArray::from(strs({"foo", "", "bar"})), StringArray::from(strs({"baz", "", ""}))) == strs({"foobaz", "", "bar"}));
  CHECK(dyn_vec(StringArray::from(strs({"foo", "bar"})), StringArray::from(strs({"bar", "baz"}))) == strs({"foobar", "barbaz"}));
  auto e = concat_elements_dyn(StringArray::from(strs({"foo", "bar"})), StringArray::from(strs({"baz"})));
  CHECK(e.is_err() && e.unwrap_err().to_string() == "Compute error: Arrays must have the same length: 2 != 1");
}

// test_string_concat_error_empty, _one, _many (:590-624)
static void test_many() {
  auto e = concat_elements_utf8_many({});
  CHECK(e.is_err() && e.unwrap_err().to_string() == "Compute error: concat requires input of at least one array");
  const StringArray one = StringArray::from(strs({nullptr, "baryyy", nullptr}));
  auto r1 = concat_elements_utf8_many({&one}).unwrap();
  CHECK(r1.to_vec() == one.to_vec() && r1.null_count() == 2);
  const StringArray foo = StringArray::from(strs({"f", "o", "o", nullptr})), bar = StringArray::from(strs({nullptr, "b", "a", "r"})),
                    baz = StringArray::from(strs({"b", nullptr, "a", "z"}));
  CHECK(concat_elements_utf8_many({&foo, &bar, &baz}).unwrap().to_vec() == strs({nullptr, nullptr, "oaa", nullptr}));
  const StringArray two = StringArray::from(strs({"a", "b"}));
  auto e2 = concat_elements_utf8_many({&foo, &two});
  CHECK(e2.is_err() && e2.unwrap_err().to_string() == "Compute error: Arrays must have the same length of 4");
}

// test_string_view_concat (:725-788)
static void test_string_view_concat() {
  const char *lg = "ThisStringIsLongerThan12Bytes";
  const std::string L(lg);
  auto r = concat_elements_string_view_array(StringViewArray::from(strs({"foo", "bar", nullptr, "foofoofoo", "foo", lg, lg})),
                                             StringViewArray::from(strs({nullptr, "yyy", "zzz", "barbarbar", lg, "bar", lg})))
               .unwrap();
  const std::string e4 = "foo" + L, e5 = L + "bar", e6 = L + L;
  CHECK(r.to_vec() == strs({nullptr, "baryyy", nullptr, "foofoofoobarbarbar", e4.c_str(), e5.c_str(), e6.c_str()}));
  // the reference's layout: one data buffer holding the long results in row order
  CHECK(r.data_buffers().size() == 1 && r.data_buffers()[0].len == 18 + e4.size() + e5.size() + e6.size());
  auto r2 = concat_elements_dyn(StringViewArray::from(strs({"a", "b", "foofoofoo", "a", lg, lg})),
                                StringViewArray::from(strs({"c", "d", "barbarbar", lg, "d", lg})))
                .unwrap();
  const std::string f3 = "a" + L, f4 = L + "d";
  CHECK(r2.to_vec() == strs({"ac", "bd", "foofoofoobarbarbar", f3.c_str(), f4.c_str(), e6.c_str()}));
  auto inl = concat_elements_string_view_array(StringViewArray::from(strs({"ab", nullptr})), StringViewArray::from(strs({"c", "d"}))).unwrap();
  CHECK(inl.data_buffers().empty() && inl.to_vec() == strs({"abc", nullptr}));
  auto e = concat_elements_string_view_array(StringViewArray::from(strs({"foo", "bar"})), StringViewArray::from(strs({"baz"})));
  CHECK(e.is_err() && e.unwrap_err().to_string() == "Compute error: Arrays must have the same length: 2 != 1");
}

// test_concat_dyn_different_type (:945-955), with an Int32 column for the Utf8 side
static void test_dyn_errors() {
  auto e = concat_elements_dyn(StringArray::from(strs({"foo"})), Int32Array::from(std::vector<int32_t>{1}));
  CHECK(e.is_err() && e.unwrap_err().to_string() == "Compute error: Cannot concat arrays of different types: Utf8 != Int32");
  auto n = concat_elements_dyn(Int32Array::from(std::vector<int32_t>{1}), Int32Array::from(std::vector<int32_t>{2}));
  CHECK(n.is_err() && n.unwrap_err().to_string() == "Not yet implemented: concat not supported for Int32");
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
      {"string_concat", test_string_concat},
      {"many", test_many},
      {"string_view_concat", test_string_view_concat},
      {"dyn_errors", test_dyn_errors},
  };
  for (const auto &t : tests) {
    const int before = g_failed;
    t.fn();
    std::printf("%s %s\n", g_failed == before ? "ok  " : "FAIL", t.name);
  }
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
