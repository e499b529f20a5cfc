// test_host_zip.cpp — the reference's byte and view zip tests (arrow-select/src/zip.rs) re-expressed against the C++ host
// mirror (arrow_cuda.hpp), with Boolean and FixedSizeBinary cases of FallbackImpl. Runs on a CUDA device (no CPU
// fallback); exits 77 when there is none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_zip   (exit code 0 = all passed)
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

using S = std::optional<std::string>;
using Strs = std::vector<S>;
static const StringArray &str(const ArrayRef &a) { return static_cast<const StringArray &>(*a); }
static BooleanArray mask(const std::vector<bool> &b) { return BooleanArray::from(b); }
static Scalar<StringArray> sscalar(S v) { return Scalar<StringArray>{StringArray::from(Strs{v})}; }
static Scalar<StringViewArray> vscalar(S v) { return Scalar<StringViewArray>{StringViewArray::from(Strs{v})}; }
static BooleanArray null_mask_6() {
  return BooleanArray::from(std::vector<std::optional<bool>>{true, true, false, std::nullopt, false, false});
}

static void test_zip_string_array_with_nulls_is_mask_should_be_treated_as_false() {
  const auto t = StringArray::from(std::vector<std::string>{"1", "2", "3", "4", "5", "6"});
  const auto f = StringArray::from(std::vector<std::string>{"7", "8", "9", "10", "11", "12"});
  auto out = zip(null_mask_6(), t, f).unwrap();
  CHECK(str(out).to_vec() == (Strs{"1", "2", "9", "10", "11", "12"}));
  CHECK(!out->nulls());
}

static void test_zip_kernel_bytes_scalar_none() {
  const auto m = mask({true, true, false, false, true});
  auto a = zip(m, sscalar("hello"), sscalar(std::nullopt)).unwrap();
  CHECK(str(a).to_vec() == (Strs{"hello", "hello", std::nullopt, std::nullopt, "hello"}));
  auto b = zip(m, sscalar(std::nullopt), sscalar("hello")).unwrap();
  CHECK(str(b).to_vec() == (Strs{std::nullopt, std::nullopt, "hello", "hello", std::nullopt}));
}

static void test_zip_kernel_bytes_scalar_both() {
  auto out = zip(mask({true, true, false, true, false, false}), sscalar("test"), sscalar("something else")).unwrap();
  CHECK(str(out).to_vec() == (Strs{"test", "test", "something else", "test", "something else", "something else"}));
  CHECK(!out->nulls());
}

static void test_zip_scalar_bytes_only_taking_one_side() {
  const auto t5 = mask(std::vector<bool>(5, true)), f5 = mask(std::vector<bool>(5, false));
  const Strs nulls(5, std::nullopt), tests(5, S("test")), elses(5, S("something else"));
  CHECK(str(zip(t5, sscalar(std::nullopt), sscalar("test")).unwrap()).to_vec() == nulls);
  CHECK(str(zip(f5, sscalar(std::nullopt), sscalar("test")).unwrap()).to_vec() == tests);
  CHECK(str(zip(t5, sscalar("test"), sscalar(std::nullopt)).unwrap()).to_vec() == tests);
  CHECK(str(zip(f5, sscalar("test"), sscalar(std::nullopt)).unwrap()).to_vec() == nulls);
  CHECK(str(zip(t5, sscalar("test"), sscalar("something else")).unwrap()).to_vec() == tests);
  CHECK(str(zip(f5, sscalar("test"), sscalar("something else")).unwrap()).to_vec() == elses);
  CHECK(str(zip(mask({true, false, true, false, true}), sscalar(std::nullopt), sscalar(std::nullopt)).unwrap()).to_vec() == nulls);
}

static void test_zip_kernel_scalar_strings_and_array_scalar() {
  auto out = zip(mask({true, false, true, false, true}), sscalar("hello"), sscalar("world")).unwrap();
  CHECK(str(out).to_vec() == (Strs{"hello", "world", "hello", "world", "hello"}));
  const auto a = StringArray::from(Strs{"a", std::nullopt, "ccc"});
  out = zip(mask({false, true, true}), a, sscalar("zz")).unwrap();
  CHECK(str(out).to_vec() == (Strs{"zz", std::nullopt, "ccc"}));
}

static void test_zip_views() {
  const std::string l1 = "longer than 12 bytes", l2 = "another longer than 12 bytes";
  CHECK(zip(mask({true, false, true, false}), vscalar("hello"), vscalar("world")).unwrap().to_vec() == (Strs{"hello", "world", "hello", "world"}));
  CHECK(zip(mask({true, true, false, false, true}), vscalar("hello"), vscalar(std::nullopt)).unwrap().to_vec() ==
        (Strs{"hello", "hello", std::nullopt, std::nullopt, "hello"}));
  CHECK(zip(mask({true, true}), vscalar(std::nullopt), vscalar(std::nullopt)).unwrap().to_vec() == (Strs{std::nullopt, std::nullopt}));
  CHECK(zip(mask({false, false}), vscalar("hello"), vscalar("world")).unwrap().to_vec() == (Strs{"world", "world"}));
  CHECK(zip(mask({true, false}), vscalar(l1), vscalar(l2)).unwrap().to_vec() == (Strs{l1, l2}));
  CHECK(zip(mask({true, false, true, false}), vscalar("hello"), vscalar(l1)).unwrap().to_vec() == (Strs{"hello", l1, "hello", l1}));
  CHECK(zip(mask({true, true}), vscalar(l1), vscalar(l2)).unwrap().to_vec() == (Strs{l1, l1}));
  CHECK(zip(mask({false, false}), vscalar(l1), vscalar(l2)).unwrap().to_vec() == (Strs{l2, l2}));
  // arrays: falsy's long views move past truthy's buffers
  const auto t = StringViewArray::from(Strs{l1, "x", std::nullopt}, 16), f = StringViewArray::from(Strs{l2, l1, "y"}, 16);
  CHECK(zip(mask({false, true, false}), t, f).unwrap().to_vec() == (Strs{l2, "x", "y"}));
}

static void test_boolean_and_fixed_size_binary_fallback() {
  using Rows = std::vector<std::optional<std::vector<uint8_t>>>;
  const std::vector<uint8_t> abc{'a', 'b', 'c'}, xyz{'x', 'y', 'z'};
  const auto t = Scalar<FixedSizeBinaryArray>{FixedSizeBinaryArray::from(Rows{abc}, 3)};
  const auto f = Scalar<FixedSizeBinaryArray>{FixedSizeBinaryArray::from(Rows{std::nullopt}, 3)};
  auto out = zip(mask({true, true, true}), t, f).unwrap();
  CHECK(!out->nulls());  // FallbackImpl: no NullBuffer when only the valid scalar is selected
  out = zip(mask({true, false, true}), t, f).unwrap();
  const auto &fo = static_cast<const FixedSizeBinaryArray &>(*out);
  CHECK(fo.value(0) == abc && out->nulls() && out->nulls()->null_count == 1);
  const auto w4 = FixedSizeBinaryArray::from(Rows{std::vector<uint8_t>(4, 1)}, 4);
  CHECK(zip(mask({true}), Scalar<FixedSizeBinaryArray>{w4}, t).is_err());
  const auto bt = Scalar<BooleanArray>{BooleanArray::from(std::vector<bool>{true})};
  const auto bf = Scalar<BooleanArray>{BooleanArray::from(std::vector<std::optional<bool>>{std::nullopt})};
  auto b = zip(mask({true, false, true}), bt, bf).unwrap();
  CHECK(static_cast<const BooleanArray &>(*b).to_vec() == (std::vector<std::optional<bool>>{true, std::nullopt, true}));
}

int main() {
  try {
    Context::get();
  } catch (const std::exception &e) {
    std::printf("SKIP: %s (no CPU fallback)\n", e.what());
    return 77;
  }
  test_zip_string_array_with_nulls_is_mask_should_be_treated_as_false();
  test_zip_kernel_bytes_scalar_none();
  test_zip_kernel_bytes_scalar_both();
  test_zip_scalar_bytes_only_taking_one_side();
  test_zip_kernel_scalar_strings_and_array_scalar();
  test_zip_views();
  test_boolean_and_fixed_size_binary_fallback();
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
