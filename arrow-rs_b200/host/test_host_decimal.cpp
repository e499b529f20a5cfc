// test_host_decimal.cpp — the reference's decimal tests (arrow-arith/src/numeric.rs test_decimal and the decimal cases of
// test_neg, arrow-ord/src/comparison.rs test_decimal32/64/128 and the _scalar variants), re-expressed against the C++ host
// mirror (arrow_cuda.hpp), plus sum / min / max edge cases (the reference has no literal decimal aggregate tests). Runs on a
// CUDA device (no CPU fallback); exits 77 when there is none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_decimal   (exit code 0 = all passed)
#include <cstdio>
#include <functional>
#include <limits>

#include "arrow_cuda.hpp"

using namespace arrow_cuda;
using namespace arrow_cuda::compute;
using namespace arrow_cuda::compute::kernels;

static int g_failed = 0, g_checks = 0;
#define CHECK(cond)                                                                    \
  do {                                                                                 \
    ++g_checks;                                                                        \
    if (!(cond)) { ++g_failed; std::printf("  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); } \
  } while (0)

template <class T> using O = std::optional<T>;
static const std::nullopt_t N = std::nullopt;
using i128 = __int128;
static const i128 I128_MAX = (i128)(((unsigned __int128)1 << 127) - 1);
static const i128 I128_MIN = -I128_MAX - 1;

template <class T> static DecimalArray<T> typed(const std::vector<T> &v, uint8_t p, int8_t s) {
  return DecimalArray<T>::from(v).with_precision_and_scale(p, s).unwrap();
}
template <class T> static const DecimalArray<T> &as_decimal(const ArrayRef &a) {
  return *std::dynamic_pointer_cast<DecimalArray<T>>(a);
}
template <class T> static std::vector<T> vals(const ArrayRef &a) { return as_decimal<T>(a).values(); }
static std::vector<O<bool>> bools(const Result<BooleanArray> &r) { return Result<BooleanArray>(r).unwrap().to_vec(); }
template <class R> static std::string err(R r) { return r.unwrap_err().message; }

// numeric.rs:1400-1480 test_decimal
static void test_decimal() {
  const auto a = typed<i128>({15, 0, -577, 334, -78, 3}, 12, 3);  // 0.015 7.842 -0.577 0.334 -0.078 0.003
  const auto b = typed<i128>({54, 34, -356, 3, 6, 745}, 12, 1);   // 5.4 0 -35.6 0.3 0.6 7.45
  auto r = numeric::add(a, b).unwrap();
  CHECK(as_decimal<i128>(r).type_display() == "Decimal128(15, 3)");
  CHECK(vals<i128>(r) == (std::vector<i128>{5415, 3400, -36177, 634, 522, 74503}));
  r = numeric::sub(a, b).unwrap();
  CHECK(as_decimal<i128>(r).type_display() == "Decimal128(15, 3)");
  CHECK(vals<i128>(r) == (std::vector<i128>{-5385, -3400, 35023, 34, -678, -74497}));
  r = numeric::mul(a, b).unwrap();
  CHECK(as_decimal<i128>(r).type_display() == "Decimal128(25, 4)");
  CHECK(vals<i128>(r) == (std::vector<i128>{810, 0, 205412, 1002, -468, 2235}));
  r = numeric::div(a, b).unwrap();
  CHECK(as_decimal<i128>(r).type_display() == "Decimal128(17, 7)");
  CHECK(vals<i128>(r) == (std::vector<i128>{27777, 0, 162078, 11133333, -1300000, 402}));
  r = numeric::rem(a, b).unwrap();
  CHECK(as_decimal<i128>(r).type_display() == "Decimal128(12, 3)");
  CHECK(vals<i128>(r) == (std::vector<i128>{15, 0, -577, 34, -78, 3}));

  auto a1 = typed<i128>({1}, 3, 3);
  const auto b1 = typed<i128>({1}, 37, 37);
  CHECK(err(numeric::mul(a1, b1)) ==
        "Invalid argument error: Output scale of Decimal128(3, 3) * Decimal128(37, 37) would exceed max scale of 38");
  a1 = typed<i128>({1}, 3, -2);
  CHECK(err(numeric::add(a1, b1)) == "Arithmetic overflow: Overflow happened on: 10 ^ 39");
  a1 = typed<i128>({10}, 3, -1);
  CHECK(err(numeric::add(a1, b1)) == "Arithmetic overflow: Overflow happened on: 10 * 100000000000000000000000000000000000000");
  const auto z = typed<i128>({0}, 1, 1);
  CHECK(err(numeric::div(a1, z)) == "Divide by zero error");
  CHECK(err(numeric::rem(a1, z)) == "Divide by zero error");
}

// numeric.rs:1197-1228 test_neg, the decimal cases: the type is kept
template <class T> static void check_neg() {
  const auto a = typed<T>({1, 3, -44, 2, 4}, 9, 6);
  auto r = numeric::neg(a).unwrap();
  CHECK(as_decimal<T>(r).type_display() == a.type_display());
  CHECK(vals<T>(r) == (std::vector<T>{-1, -3, 44, -2, -4}));
  r = numeric::neg_wrapping(a).unwrap();  // neg_wrapping falls back to neg for decimals
  CHECK(vals<T>(r) == (std::vector<T>{-1, -3, 44, -2, -4}));
  const T mn = std::is_same<T, i128>::value ? (T)I128_MIN : std::numeric_limits<T>::min();
  CHECK(err(numeric::neg_wrapping(typed<T>({1, mn}, 9, 0))).rfind("Arithmetic overflow: Overflow happened on: - ", 0) == 0);
}
static void test_neg() { check_neg<int32_t>(); check_neg<int64_t>(); check_neg<i128>(); }

// comparison.rs:3294-3415 test_decimal32 / 64 / 128
template <class T> static void check_cmp() {
  const auto a = DecimalArray<T>::from(std::vector<T>{1, 2, 4, 5});
  const auto b = DecimalArray<T>::from(std::vector<T>{7, -3, 4, 3});
  CHECK(bools(cmp::eq(a, b)) == (std::vector<O<bool>>{false, false, true, false}));
  CHECK(bools(cmp::lt(a, b)) == (std::vector<O<bool>>{true, false, false, false}));
  CHECK(bools(cmp::lt_eq(a, b)) == (std::vector<O<bool>>{true, false, true, false}));
  CHECK(bools(cmp::gt(a, b)) == (std::vector<O<bool>>{false, true, false, true}));
  CHECK(bools(cmp::gt_eq(a, b)) == (std::vector<O<bool>>{false, true, true, true}));
}
// comparison.rs:3319-3364 / 3416-3460 test_decimal32_scalar / test_decimal128_scalar
template <class T> static void check_cmp_scalar() {
  const auto a = DecimalArray<T>::from(std::vector<O<T>>{1, 2, 3, N, 4, 5});
  const Scalar<DecimalArray<T>> b(DecimalArray<T>::from(std::vector<T>{3}));
  CHECK(bools(cmp::eq(a, b)) == (std::vector<O<bool>>{false, false, true, N, false, false}));
  CHECK(bools(cmp::neq(a, b)) == (std::vector<O<bool>>{true, true, false, N, true, true}));
  CHECK(bools(cmp::lt(a, b)) == (std::vector<O<bool>>{true, true, false, N, false, false}));
  CHECK(bools(cmp::lt_eq(a, b)) == (std::vector<O<bool>>{true, true, true, N, false, false}));
  CHECK(bools(cmp::gt(a, b)) == (std::vector<O<bool>>{false, false, false, N, true, true}));
  CHECK(bools(cmp::gt_eq(a, b)) == (std::vector<O<bool>>{false, false, true, N, true, true}));
}
static void test_cmp() {
  check_cmp<int32_t>(); check_cmp<int64_t>(); check_cmp<i128>();
  check_cmp_scalar<int32_t>(); check_cmp_scalar<i128>();
  // compare_op refuses DataTypes that differ, precision included (cmp.rs:260-263)
  const auto a = typed<i128>({1, 2}, 9, 0), b = typed<i128>({1, 2}, 10, 0);
  CHECK(err(cmp::lt(a, b)) == "Invalid argument error: Invalid comparison operation: Decimal128(9, 0) < Decimal128(10, 0)");
}

static void test_with_precision_and_scale() {
  CHECK(err(Decimal32Array::from(std::vector<int32_t>{1}).with_precision_and_scale(10, 0)) ==
        "Invalid argument error: precision 10 is greater than max 9");
  CHECK(err(Decimal128Array::from(std::vector<i128>{1}).with_precision_and_scale(0, 0)) ==
        "Invalid argument error: precision cannot be 0, has to be between [1, 38]");
  CHECK(err(Decimal64Array::from(std::vector<int64_t>{1}).with_precision_and_scale(5, 6)) ==
        "Invalid argument error: scale 6 is greater than precision 5");
  CHECK(Decimal128Array::from(std::vector<i128>{1}).type_display() == "Decimal128(38, 10)");
}

// sum wraps (add_wrapping), min / max in the native order, None without valid rows
static void test_aggregates() {
  auto a = Decimal128Array::from(std::vector<O<i128>>{I128_MAX, 1});
  CHECK(sum(a) == O<i128>(I128_MIN) && min(a) == O<i128>(1) && max(a) == O<i128>(I128_MAX));
  a = Decimal128Array::from(std::vector<O<i128>>{0, I128_MIN, N, I128_MAX, -5});
  CHECK(sum(a) == O<i128>(-6) && min(a) == O<i128>(I128_MIN) && max(a) == O<i128>(I128_MAX));
  a = Decimal128Array::from(std::vector<O<i128>>{N, N});
  CHECK(!sum(a) && !min(a) && !max(a));
  CHECK(!sum(Decimal128Array::from(std::vector<i128>{})));
  CHECK(sum(a.slice(0, 0)) == std::nullopt);
  const auto d32 = Decimal32Array::from(std::vector<O<int32_t>>{2147483647, 1, N, 5});  // 2^31 + 5 wraps in i32
  CHECK(sum(d32) == O<int32_t>(-2147483643) && min(d32) == O<int32_t>(1) && max(d32) == O<int32_t>(2147483647));
  const auto d64 = Decimal64Array::from(std::vector<O<int64_t>>{5, N, -3});
  CHECK(sum(d64) == O<int64_t>(2) && min(d64) == O<int64_t>(-3) && max(d64) == O<int64_t>(5));
}

// a zero-copy slice keeps the i128 values aligned and moves the validity bit offset
static void test_sliced() {
  const auto a = Decimal128Array::from(std::vector<O<i128>>{1, N, 3, 4, N, 6, 7}).with_precision_and_scale(20, 2).unwrap();
  const auto b = Decimal128Array::from(std::vector<O<i128>>{10, 20, N, 40, 50, 60, 70}).with_precision_and_scale(20, 0).unwrap();
  const auto as = a.slice(1, 5), bs = b.slice(1, 5);
  const auto r = numeric::add(as, bs).unwrap();
  CHECK(as_decimal<i128>(r).to_vec() == (std::vector<O<i128>>{N, N, 4004, N, 6006}));
  CHECK(bools(cmp::gt(as, Scalar<Decimal128Array>(typed<i128>({3}, 20, 2)))) == (std::vector<O<bool>>{N, false, true, N, true}));
  CHECK(sum(as) == O<i128>(13) && min(as) == O<i128>(3) && max(as) == O<i128>(6));
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
      {"decimal", test_decimal},
      {"neg", test_neg},
      {"cmp", test_cmp},
      {"with_precision_and_scale", test_with_precision_and_scale},
      {"aggregates", test_aggregates},
      {"sliced", test_sliced},
  };
  for (const auto &t : tests) {
    const int before = g_failed;
    t.fn();
    std::printf("%s %s\n", g_failed == before ? "ok  " : "FAIL", t.name);
  }
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
