// test_host_decimal_cast.cpp — a handful of the reference's decimal cast tests (arrow-cast/src/cast/mod.rs tests module)
// re-expressed against the C++ host mirror's cast_with_options (arrow_cuda.hpp). Runs on a CUDA device (no CPU fallback);
// exits 77 when there is none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_decimal_cast   (exit code 0 = all passed)
#include <cstdio>
#include <functional>
#include <limits>

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
using i128 = __int128;
static const CastOptions SAFE{true}, UNSAFE{false};

template <class T> static DecimalArray<T> typed(const std::vector<O<T>> &v, uint8_t p, int8_t s) {
  return DecimalArray<T>::from(v).with_precision_and_scale(p, s).unwrap();
}
template <class T> static std::vector<O<T>> dec_list(const ArrayRef &a) {
  const auto &d = *std::dynamic_pointer_cast<DecimalArray<T>>(a);
  const auto v = d.values();
  std::vector<O<T>> out;
  for (int64_t i = 0; i < d.len(); ++i) out.push_back(d.is_null(i) ? O<T>() : O<T>(v[(size_t)i]));
  return out;
}
template <class R> static std::string err(R r) { return r.unwrap_err().message; }

// test_cast_decimal_to_decimal_round / test_cast_decimal32_to_decimal32_overflow / _large_scale_reduction
static void test_decimal_to_decimal() {
  const auto a = typed<i128>({1123454, 2123456, -3123453, -3123456, N}, 20, 4);
  auto r = cast_with_options(a, DecimalDataType{DataType::Decimal128, 20, 3}, SAFE).unwrap();
  CHECK(dec_list<i128>(r) == (std::vector<O<i128>>{112345, 212346, -312345, -312346, N}));
  const auto m = typed<int32_t>({std::numeric_limits<int32_t>::max()}, 9, 3);
  CHECK(err(cast_with_options(m, DecimalDataType{DataType::Decimal32, 9, 9}, UNSAFE)) ==
        "Cast error: Cannot cast to Decimal32(9, 9). Overflowing on 2147483647");
  const auto l = typed<int32_t>({-999999999, 0, 999999999, N}, 9, 3);
  r = cast_with_options(l, DecimalDataType{DataType::Decimal32, 9, -6}, SAFE).unwrap();
  CHECK(dec_list<int32_t>(r) == (std::vector<O<int32_t>>{-1, 0, 1, N}));
  r = cast_with_options(l, DecimalDataType{DataType::Decimal32, 9, -7}, SAFE).unwrap();
  CHECK(dec_list<int32_t>(r) == (std::vector<O<int32_t>>{0, 0, 0, N}));
  // test_decimal_to_decimal_throw_error_on_precision_overflow_same_scale / _greater_scale, across widths
  const auto p = typed<i128>({123456789}, 24, 2);
  CHECK(err(cast_with_options(p, DecimalDataType{DataType::Decimal128, 6, 2}, UNSAFE)) ==
        "Invalid argument error: 1234567.89 is too large to store in a Decimal128 of precision 6. Max is 9999.99");
  CHECK(err(cast_with_options(p, DecimalDataType{DataType::Decimal64, 6, 3}, UNSAFE)) ==
        "Invalid argument error: 1234567.890 is too large to store in a Decimal64 of precision 6. Max is 999.999");
}

// test_cast_decimal_error_output / test_cast_integer_to_decimal32_does_not_truncate / test_cast_f64_to_decimal128
static void test_to_decimal() {
  CHECK(err(cast_with_options(Int64Array::from(std::vector<int64_t>{1}), DecimalDataType{DataType::Decimal32, 1, 1}, UNSAFE)) ==
        "Invalid argument error: 1.0 is too large to store in a Decimal32 of precision 1. Max is 0.9");
  CHECK(err(cast_with_options(Int64Array::from(std::vector<int64_t>{-1}), DecimalDataType{DataType::Decimal32, 1, 1}, UNSAFE)) ==
        "Invalid argument error: -1.0 is too small to store in a Decimal32 of precision 1. Min is -0.9");
  const auto big = Int64Array::from(std::vector<int64_t>{5000000000, 10000000000, 42});
  auto r = cast_with_options(big, DecimalDataType{DataType::Decimal32, 9, 0}, SAFE).unwrap();
  CHECK(dec_list<int32_t>(r) == (std::vector<O<int32_t>>{N, N, 42}));
  CHECK(err(cast_with_options(big, DecimalDataType{DataType::Decimal32, 9, 0}, UNSAFE)) ==
        "Cast error: Cannot cast to Decimal32(9, 0). Overflowing on 5000000000");
  r = cast_with_options(Int64Array::from(std::vector<int64_t>{5000000000}), DecimalDataType{DataType::Decimal32, 9, -1}, UNSAFE).unwrap();
  CHECK(dec_list<int32_t>(r) == (std::vector<O<int32_t>>{500000000}));
  const auto f = Float64Array::from(std::vector<double>{0.0699999999, 0.0659999999, 0.0650000000, 0.0649999999});
  r = cast_with_options(f, DecimalDataType{DataType::Decimal128, 18, 2}, SAFE).unwrap();
  CHECK(dec_list<i128>(r) == (std::vector<O<i128>>{7, 7, 7, 6}));
  r = cast_with_options(f, DecimalDataType{DataType::Decimal128, 18, 3}, SAFE).unwrap();
  CHECK(dec_list<i128>(r) == (std::vector<O<i128>>{70, 66, 65, 65}));
}

// test_cast_decimal_to_numeric_negative_scale (Decimal32 parts), and decimal -> Float64
static void test_from_decimal() {
  auto r = cast_with_options(typed<int32_t>({125, 225, 325, N, 525}, 8, -2), DataType::Int64, SAFE).unwrap();
  const auto &i = *std::dynamic_pointer_cast<Int64Array>(r);
  CHECK(i.to_vec() == (std::vector<O<int64_t>>{12500, 22500, 32500, N, 52500}));
  r = cast_with_options(typed<i128>({12345, -5, N}, 10, 2), DataType::Float64, SAFE).unwrap();
  const auto &d = *std::dynamic_pointer_cast<Float64Array>(r);
  CHECK(d.to_vec() == (std::vector<O<double>>{123.45, -0.05, N}));
  CHECK(err(cast_with_options(typed<int32_t>({1}, 9, -10), DataType::Int64, SAFE)) ==
        "Cast error: Cannot cast to \"Decimal32\". The scale -10 causes overflow.");
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
      {"decimal_to_decimal", test_decimal_to_decimal},
      {"to_decimal", test_to_decimal},
      {"from_decimal", test_from_decimal},
  };
  for (const auto &t : tests) {
    const int before = g_failed;
    t.fn();
    std::printf("%s %s\n", g_failed == before ? "ok  " : "FAIL", t.name);
  }
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
