// test_host_aggregate.cpp — the reference's min / max tests of string, string-view and boolean columns
// (arrow-arith/src/aggregate.rs), re-expressed against the C++ host mirror (arrow_cuda.hpp). Runs on a CUDA device (no CPU
// fallback); exits 77 when there is none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_aggregate   (exit code 0 = all passed)
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
static const std::nullopt_t N = std::nullopt;
using S = std::vector<O<std::string>>;
using B = std::vector<O<bool>>;

// test_string! (aggregate.rs:1598-1615): the same case on StringArray and StringViewArray
static void check_string(const S &input, O<std::string> mn, O<std::string> mx) {
  const StringArray s = StringArray::from(input);
  CHECK(min_string(s) == mn);
  CHECK(max_string(s) == mx);
  const StringViewArray v = StringViewArray::from(input, 16);  // small blocks: long values spread over several buffers
  CHECK(min_string_view(v) == mn);
  CHECK(max_string_view(v) == mx);
}

static void test_string_min_max() {
  // aggregate.rs:1617-1629 test_string_min_max_with_nulls
  check_string(S{std::string("b012345678901234"), N, N, std::string("a"), std::string("c"), std::string("b0123xxxxxxxxxxx")},
               std::string("a"), std::string("c"));
  // :1631-1641 test_string_min_max_no_null
  check_string(S{std::string("b"), std::string("b012345678901234"), std::string("a"), std::string("b012xxxxxxxxxxxx")},
               std::string("a"), std::string("b012xxxxxxxxxxxx"));
  // :1643-1648 test_string_min_max_all_nulls
  check_string(S{N, N}, N, N);
  // :1650-1661 test_string_min_max_1
  check_string(S{N, std::string("c12345678901234"), N, std::string("b"), std::string("c1234xxxxxxxxxx")}, std::string("b"),
               std::string("c1234xxxxxxxxxx"));
  // :1663-1668 test_string_min_max_empty
  check_string(S{}, N, N);
  // :1941-1961 test_min_max_sliced_string (unsliced form; the sliced form runs on the view array)
  check_string(S{N, std::string("foo")}, std::string("foo"), std::string("foo"));
  const StringViewArray sliced = StringViewArray::from(S{N, N, N, N, N, std::string("foo")}).slice(4, 2);
  CHECK(min_string_view(sliced) == O<std::string>("foo"));
  CHECK(max_string_view(sliced) == O<std::string>("foo"));
}

static void check_boolean(const BooleanArray &a, O<bool> mn, O<bool> mx) {
  CHECK(min_boolean(a) == mn);
  CHECK(max_boolean(a) == mx);
  CHECK(bool_and(a) == mn);
  CHECK(bool_or(a) == mx);
}

static void test_bool_and_or() {  // aggregate.rs:1263-1297
  check_boolean(BooleanArray::from(std::vector<bool>{true, false, true, false, true}), false, true);
  check_boolean(BooleanArray::from(B{N, true, true, N, true}), true, true);
  check_boolean(BooleanArray::from(B{N, N, N}), N, N);
  check_boolean(BooleanArray::from(B{N, false, false, N, false}), false, false);
}

static void test_boolean_min_max() {  // aggregate.rs:1671-1740
  check_boolean(BooleanArray::from(B{}), N, N);
  check_boolean(BooleanArray::from(B{N, N}), N, N);
  check_boolean(BooleanArray::from(B{true, false, true}), false, true);
  check_boolean(BooleanArray::from(B{true, true, N, false, N}), false, true);
  check_boolean(BooleanArray::from(B{N, true, N, false, N}), false, true);
  check_boolean(BooleanArray::from(B{false, true, N, false, N}), false, true);
  check_boolean(BooleanArray::from(B{true, N}), true, true);
  check_boolean(BooleanArray::from(B{false, N}), false, false);
  check_boolean(BooleanArray::from(B{true}), true, true);
  check_boolean(BooleanArray::from(B{false}), false, false);
  check_boolean(BooleanArray::from(B{N, false}), false, false);
  check_boolean(BooleanArray::from(B{N, true}), true, true);
}

static B repeat(B v, O<bool> x, int n) {
  v.insert(v.end(), (size_t)n, x);
  return v;
}

static void test_boolean_min_max_64_96() {  // aggregate.rs:1742-1826
  check_boolean(BooleanArray::from(repeat(repeat(B{}, true, 64), false, 64)), false, true);
  check_boolean(BooleanArray::from(repeat(repeat(repeat(repeat(repeat(B{}, true, 31), N, 1), true, 32), false, 1), N, 63)), false, true);
  check_boolean(BooleanArray::from(repeat(repeat(B{}, false, 64), true, 64)), false, true);
  check_boolean(BooleanArray::from(repeat(repeat(repeat(repeat(repeat(B{}, false, 31), N, 1), false, 32), true, 1), N, 63)), false, true);
  check_boolean(BooleanArray::from(repeat(B{}, true, 96)), true, true);
  check_boolean(BooleanArray::from(repeat(repeat(repeat(repeat(B{}, true, 31), N, 1), true, 63), N, 1)), true, true);
  check_boolean(BooleanArray::from(repeat(B{}, false, 96)), false, false);
  check_boolean(BooleanArray::from(repeat(repeat(repeat(repeat(B{}, false, 31), N, 1), false, 63), N, 1)), false, false);
}

static void test_min_max_sliced_boolean() {  // aggregate.rs:1919-1938
  check_boolean(BooleanArray::from(B{N, true}), true, true);
  check_boolean(BooleanArray::from(B{N, N, N, N, N, true}).slice(4, 2), true, true);
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
      {"string_min_max", test_string_min_max},
      {"bool_and_or", test_bool_and_or},
      {"boolean_min_max", test_boolean_min_max},
      {"boolean_min_max_64_96", test_boolean_min_max_64_96},
      {"min_max_sliced_boolean", test_min_max_sliced_boolean},
  };
  for (const auto &t : tests) {
    const int before = g_failed;
    t.fn();
    std::printf("%s %s\n", g_failed == before ? "ok  " : "FAIL", t.name);
  }
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
