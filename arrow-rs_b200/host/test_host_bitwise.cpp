// test_host_bitwise.cpp — the reference's bitwise tests (arrow-arith/src/bitwise.rs:211-392) and its product /
// product_checked / bit_and / bit_or / bit_xor tests (arrow-arith/src/aggregate.rs:1051-1110, :1209-1260) re-expressed
// against the C++ host mirror (arrow_cuda.hpp). Runs on a CUDA device (no CPU fallback); exits 77 when there is none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_bitwise   (exit code 0 = all passed)
#include <cstdio>
#include <functional>
#include <limits>

#include "arrow_cuda.hpp"

using namespace arrow_cuda;
using namespace arrow_cuda::compute;
using namespace arrow_cuda::compute::kernels::bitwise;

static int g_failed = 0, g_checks = 0;
#define CHECK(cond)                                                                    \
  do {                                                                                 \
    ++g_checks;                                                                        \
    if (!(cond)) { ++g_failed; std::printf("  FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); } \
  } while (0)

template <class T> using O = std::optional<T>;
static const std::nullopt_t N = std::nullopt;
using U64 = std::vector<O<uint64_t>>;
using I32 = std::vector<O<int32_t>>;

static void test_bitwise_and_array() {  // bitwise.rs:211
  CHECK(bitwise_and(UInt64Array::from(U64{1, 2, N, 4}), UInt64Array::from(U64{5, 10, 8, 12})).unwrap().to_vec() == (U64{1, 2, N, 4}));
  CHECK(bitwise_and(Int32Array::from(I32{1, 2, N, 4}), Int32Array::from(I32{5, -10, 8, 12})).unwrap().to_vec() == (I32{1, 2, N, 4}));
}

static void test_bitwise_shift() {  // bitwise.rs:229-263
  const auto l = UInt64Array::from(U64{1, 2, N, 4, 8});
  CHECK(bitwise_shift_left(l, UInt64Array::from(U64{5, 10, 8, 12, std::numeric_limits<uint64_t>::max()})).unwrap().to_vec() ==
        (U64{32, 2048, N, 16384, 0}));
  CHECK(bitwise_shift_left_scalar(l, (uint64_t)2).unwrap().to_vec() == (U64{4, 8, N, 16, 32}));
  const auto r = UInt64Array::from(U64{32, 2048, N, 16384, 3});
  CHECK(bitwise_shift_right(r, UInt64Array::from(U64{5, 10, 8, 12, 65})).unwrap().to_vec() == (U64{1, 2, N, 4, 1}));
  CHECK(bitwise_shift_right_scalar(r, (uint64_t)2).unwrap().to_vec() == (U64{8, 512, N, 4096, 0}));
}

static void test_bitwise_and_array_scalar() {  // bitwise.rs:265
  CHECK(bitwise_and_scalar(UInt64Array::from(U64{15, 2, N, 4}), (uint64_t)7).unwrap().to_vec() == (U64{7, 2, N, 4}));
  CHECK(bitwise_and_scalar(Int32Array::from(I32{1, 2, N, 4}), -20).unwrap().to_vec() == (I32{0, 0, N, 4}));
}

static void test_bitwise_or() {  // bitwise.rs:282, :343
  CHECK(bitwise_or(UInt64Array::from(U64{1, 2, N, 4}), UInt64Array::from(U64{7, 5, 8, 13})).unwrap().to_vec() == (U64{7, 7, N, 13}));
  CHECK(bitwise_or(Int32Array::from(I32{1, 2, N, 4}), Int32Array::from(I32{-7, -5, 8, 13})).unwrap().to_vec() == (I32{-7, -5, N, 13}));
  CHECK(bitwise_or_scalar(UInt64Array::from(U64{15, 2, N, 4}), (uint64_t)7).unwrap().to_vec() == (U64{15, 7, N, 7}));
  CHECK(bitwise_or_scalar(Int32Array::from(I32{1, 2, N, 4}), 20).unwrap().to_vec() == (I32{21, 22, N, 20}));
}

static void test_bitwise_not_and_not() {  // bitwise.rs:299, :318
  CHECK(bitwise_not(UInt64Array::from(U64{1, 2, N, 4})).unwrap().to_vec() ==
        (U64{18446744073709551614ull, 18446744073709551613ull, N, 18446744073709551611ull}));
  CHECK(bitwise_not(Int32Array::from(I32{1, 2, N, 4})).unwrap().to_vec() == (I32{-2, -3, N, -5}));
  const auto l = UInt64Array::from(U64{8, 2, N, 4}), r = UInt64Array::from(U64{7, 5, 8, 13});
  const auto res = bitwise_and_not(l, r).unwrap();
  CHECK(res.to_vec() == (U64{8, 2, N, 0}));
  CHECK(bitwise_and(l, bitwise_not(r).unwrap()).unwrap().to_vec() == res.to_vec());
  const auto li = Int32Array::from(I32{2, 1, N, 3}), ri = Int32Array::from(I32{-7, -5, 8, 13});
  const auto resi = bitwise_and_not(li, ri).unwrap();
  CHECK(resi.to_vec() == (I32{2, 0, N, 2}));
  CHECK(bitwise_and(li, bitwise_not(ri).unwrap()).unwrap().to_vec() == resi.to_vec());
}

static void test_bitwise_xor() {  // bitwise.rs:360, :377
  CHECK(bitwise_xor(UInt64Array::from(U64{1, 2, N, 4}), UInt64Array::from(U64{7, 5, 8, 13})).unwrap().to_vec() == (U64{6, 7, N, 9}));
  CHECK(bitwise_xor(Int32Array::from(I32{1, 2, N, 4}), Int32Array::from(I32{-7, 5, 8, -13})).unwrap().to_vec() == (I32{-8, 7, N, -9}));
  CHECK(bitwise_xor_scalar(UInt64Array::from(U64{15, 2, N, 4}), (uint64_t)7).unwrap().to_vec() == (U64{8, 5, N, 3}));
  CHECK(bitwise_xor_scalar(Int32Array::from(I32{1, 2, N, 4}), -20).unwrap().to_vec() == (I32{-19, -18, N, -24}));
}

static void test_binary_length_mismatch() {  // arity.rs:104-135: the `binary` text, without the "a" of try_binary
  auto r = bitwise_and(Int32Array::from(I32{1, 2}), Int32Array::from(I32{1}));
  CHECK(!r.is_ok());
  if (!r.is_ok()) CHECK(r.unwrap_err().message == "Compute error: Cannot perform binary operation on arrays of different length");
}

static void test_product() {  // aggregate.rs:1051-1110
  CHECK(product(Int32Array::from(I32{1, 2, 3, 4, 5})) == O<int32_t>(120));
  CHECK(product(Float64Array::from(std::vector<double>{1.0, 2.0, 3.0, 4.0, 5.0})) == O<double>(120.0));
  CHECK(product(Int32Array::from(I32{N, 2, 3, N, 5})) == O<int32_t>(30));
  CHECK(product(Int32Array::from(I32{N, N, N})) == std::nullopt);
  CHECK(product(Int32Array::from(std::vector<int32_t>{})) == std::nullopt);
  CHECK(product_checked(Int32Array::from(I32{1, 2, 3, 4, 5})).unwrap() == O<int32_t>(120));
  CHECK(product_checked(Int32Array::from(I32{N, 2, 3, N, 5})).unwrap() == O<int32_t>(30));
  CHECK(product_checked(Int32Array::from(I32{N, N, N})).unwrap() == std::nullopt);
  const auto ovf = Int32Array::from(std::vector<int32_t>{std::numeric_limits<int32_t>::max(), 2});
  CHECK(product(ovf) == O<int32_t>(-2));
  auto r = product_checked(ovf);
  CHECK(!r.is_ok());
  if (!r.is_ok()) CHECK(r.unwrap_err().message == "Arithmetic overflow: Overflow happened on: 2147483647 * 2");
}

static void test_bit_aggregates() {  // aggregate.rs:1209-1260
  CHECK(bit_and(Int32Array::from(I32{1, 2, 3, 4, 5})) == O<int32_t>(0));
  CHECK(bit_and(Int32Array::from(I32{N, 2, 3, N, N})) == O<int32_t>(2));
  CHECK(bit_and(Int32Array::from(I32{N, N, N})) == std::nullopt);
  CHECK(bit_or(Int32Array::from(I32{1, 2, 3, 4, 5})) == O<int32_t>(7));
  CHECK(bit_or(Int32Array::from(I32{N, 2, 3, N, 5})) == O<int32_t>(7));
  CHECK(bit_or(Int32Array::from(I32{N, N, N})) == std::nullopt);
  CHECK(bit_xor(Int32Array::from(I32{1, 2, 3, 4, 5})) == O<int32_t>(1));
  CHECK(bit_xor(Int32Array::from(I32{N, 2, 3, N, 5})) == O<int32_t>(4));
  CHECK(bit_xor(Int32Array::from(I32{N, N, N})) == std::nullopt);
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
      {"bitwise_and_array", test_bitwise_and_array},
      {"bitwise_shift", test_bitwise_shift},
      {"bitwise_and_array_scalar", test_bitwise_and_array_scalar},
      {"bitwise_or", test_bitwise_or},
      {"bitwise_not_and_not", test_bitwise_not_and_not},
      {"bitwise_xor", test_bitwise_xor},
      {"binary_length_mismatch", test_binary_length_mismatch},
      {"product", test_product},
      {"bit_aggregates", test_bit_aggregates},
  };
  for (const auto &t : tests) {
    const int before = g_failed;
    t.fn();
    std::printf("%s %s\n", g_failed == before ? "ok  " : "FAIL", t.name);
  }
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
