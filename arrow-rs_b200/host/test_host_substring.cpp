// test_host_substring.cpp — the reference's length / substring doc examples and a few of its tests
// (arrow-string/src/length.rs, substring.rs) re-expressed against the C++ host mirror (arrow_cuda.hpp). Runs on a CUDA
// device (no CPU fallback); exits 77 when there is none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_substring   (exit code 0 = all passed)
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
using I = std::vector<O<int32_t>>;

static S strs(std::initializer_list<const char *> v) {
  S out;
  for (const char *s : v) out.push_back(s ? O<std::string>(s) : N);
  return out;
}

// substring.rs:46-53 and :127-135, the doc examples
static void test_doc_examples() {
  const S in = strs({"arrow", nullptr, "rust"});
  CHECK(substring(StringArray::from(in), 1, 4).unwrap().to_vec() == strs({"rrow", nullptr, "ust"}));
  CHECK(substring(StringViewArray::from(in, 16), 1, 4).unwrap().to_vec() == strs({"rrow", nullptr, "ust"}));
  CHECK(substring_by_char(StringArray::from(strs({"arrow", nullptr, "Γ ⊢x:T"})), 1, 4).unwrap().to_vec() ==
        strs({"rrow", nullptr, " ⊢x:"}));
  // substring.rs:66-71: "E=mc²" cut inside the 2-byte '²'
  auto r = substring(StringArray::from(strs({"E=mc²"})), 0, 5);
  CHECK(r.is_err() && r.unwrap_err().message.find("invalid utf-8 boundary") != std::string::npos);
}

// without_nulls_generic_string (substring.rs:782-821), a few rows of its table
static void test_without_nulls_string() {
  const S in = strs({"hello", "", "word"});
  struct Row { int64_t start; O<uint64_t> len; S expected; };
  const std::vector<Row> rows = {
      {0, N, in}, {1, N, strs({"ello", "", "ord"})}, {-1, N, strs({"o", "", "d"})}, {-10, N, in},
      {1, 2, strs({"el", "", "or"})}, {-3, 4, strs({"llo", "", "ord"})}, {10, N, strs({"", "", ""})}};
  for (const auto &row : rows) {
    CHECK(substring(StringArray::from(in), row.start, row.len).unwrap().to_vec() == row.expected);
    CHECK(substring(StringViewArray::from(in, 16), row.start, row.len).unwrap().to_vec() == row.expected);
  }
}

// without_nulls_generic_string_by_char (substring.rs:881-919), a few rows
static void test_by_char() {
  const S in = strs({"hello", "", "Γ ⊢x:T"});
  CHECK(substring_by_char(StringArray::from(in), -4, 2).unwrap().to_vec() == strs({"el", "", "⊢x"}));
  CHECK(substring_by_char(StringArray::from(in), 2, N).unwrap().to_vec() == strs({"llo", "", "⊢x:T"}));
  CHECK(substring_by_char(StringArray::from(in), 1, UINT64_MAX).unwrap().to_vec() == strs({"ello", "", " ⊢x:T"}));
}

// string_view_matches_utf8 (substring.rs:1117-1148): a view result equals the Utf8 one, also past 12 bytes
static void test_view_matches_utf8() {
  const S in = strs({"hello world", "", nullptr, "a", "this one is definitely longer than twelve bytes"});
  const std::vector<std::pair<int64_t, O<uint64_t>>> params = {{0, N}, {0, 5}, {1, 3}, {5, N}, {100, 2}, {-3, N}, {-100, 4}};
  for (const auto &p : params)
    CHECK(substring(StringViewArray::from(in, 16), p.first, p.second).unwrap().to_vec() ==
          substring(StringArray::from(in), p.first, p.second).unwrap().to_vec());
  // string_view_rejects_an_invalid_char_boundary: the message gives the offset relative to the value
  auto r = substring(StringViewArray::from(strs({"héllo"})), 2, N);
  CHECK(r.is_err() && r.unwrap_err().message == "Compute error: The offset 2 is at an invalid utf-8 boundary.");
}

// length.rs: length_test_string / bit_length_test_string / length_null_string, on Utf8 and Utf8View
static void test_length() {
  const S in = strs({"hello", " ", nullptr, "💖"});
  CHECK(length(StringArray::from(in)).unwrap().to_vec() == (I{5, 1, N, 4}));
  CHECK(bit_length(StringArray::from(in)).unwrap().to_vec() == (I{40, 8, N, 32}));
  CHECK(length(StringViewArray::from(in)).unwrap().to_vec() == (I{5, 1, N, 4}));
  CHECK(bit_length(StringViewArray::from(in)).unwrap().to_vec() == (I{40, 8, N, 32}));
  // nulls.cloned(): an input without a NullBuffer gives none
  CHECK(length(StringArray::from(strs({"one", "two"}))).unwrap().nulls() == std::nullopt);
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
      {"doc_examples", test_doc_examples},
      {"without_nulls_string", test_without_nulls_string},
      {"by_char", test_by_char},
      {"view_matches_utf8", test_view_matches_utf8},
      {"length", test_length},
  };
  for (const auto &t : tests) {
    const int before = g_failed;
    t.fn();
    std::printf("%s %s\n", g_failed == before ? "ok  " : "FAIL", t.name);
  }
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
