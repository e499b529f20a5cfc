// test_host_like.cpp — a few of the reference's LIKE-family tests (arrow-string/src/like.rs, predicate.rs) re-expressed
// against the C++ host mirror (arrow_cuda.hpp). Runs on a CUDA device (no CPU fallback); exits 77 when there is none.
//
// Build: see arrow-rs_b200/host/Makefile.  Run: ./test_host_like   (exit code 0 = all passed)
#include <cstdio>
#include <functional>

#include "arrow_cuda.hpp"

using namespace arrow_cuda;
using namespace arrow_cuda::compute;
namespace L = arrow_cuda::compute::like;  // arrow_string::like

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

static S strs(std::initializer_list<const char *> v) {
  S out;
  for (const char *s : v) out.push_back(s ? O<std::string>(s) : N);
  return out;
}
static B bools(std::initializer_list<bool> v) { return B(v.begin(), v.end()); }

using Fn = std::function<Result<BooleanArray>(const StringArray &, const StringArray &)>;
using FnS = std::function<Result<BooleanArray>(const StringArray &, const Scalar<StringArray> &)>;
using FnV = std::function<Result<BooleanArray>(const StringViewArray &, const StringViewArray &)>;
using FnVS = std::function<Result<BooleanArray>(const StringViewArray &, const Scalar<StringViewArray> &)>;

// test_utf8! (like.rs:466-494): both sides arrays, on StringArray and StringViewArray
static void check_arrays(const S &l, const S &r, Fn f, FnV fv, const B &expected) {
  CHECK(f(StringArray::from(l), StringArray::from(r)).unwrap().to_vec() == expected);
  CHECK(fv(StringViewArray::from(l, 16), StringViewArray::from(r, 16)).unwrap().to_vec() == expected);
}
// test_utf8_scalar! (like.rs:557-589): a scalar pattern
static void check_scalar(const S &l, const std::string &r, FnS f, FnVS fv, const B &expected) {
  CHECK(f(StringArray::from(l), Scalar<StringArray>(StringArray::from(S{r}))).unwrap().to_vec() == expected);
  CHECK(fv(StringViewArray::from(l, 16), Scalar<StringViewArray>(StringViewArray::from(S{r}))).unwrap().to_vec() == expected);
}
#define F(NAME) [](const auto &a, const auto &b) { return L::NAME(a, b); }

static void test_utf8_array_like() {  // like.rs:646-663
  check_arrays(strs({"arrow", "arrow_long_string_more than 12 bytes", "arrow", "arrow", "arrow", "arrows", "arrow", "arrow"}),
               strs({"arrow", "ar%", "%ro%", "foo", "arr", "arrow_", "arrow_", ".*"}), F(like), F(like),
               bools({true, true, true, false, false, true, false, false}));
}

static void test_utf8_array_like_scalar() {  // like.rs:695-721, :807-834
  const S hay = strs({"arrow", "parrow", "arrows", "arr", "arrow long string longer than 12 bytes"});
  check_scalar(hay, "arrow%", F(like), F(like), bools({true, false, true, false, true}));
  check_scalar(strs({"arrow", "arrows", "parrow", "arr", "arrow long string longer than 12 bytes"}), "arrow_", F(like), F(like),
               bools({false, true, false, false, false}));
  check_scalar(hay, "arrow%", F(nlike), F(nlike), bools({false, true, false, true, false}));
}

static void test_utf8_array_ilike_unicode() {  // like.rs:1063-1081: simple case folding (ﬀ is not FF, ß is not SS)
  check_scalar(strs({"FFkoß", "FFkoSS", "FFkoss", "FFkoS", "FFkos", "ﬀkoSS", "ﬀkoß", "FFKoSS", "longer than 12 bytes FFKoSS"}), "FFkoSS",
               F(ilike), F(ilike), bools({false, true, true, false, false, false, false, true, false}));
}

static void test_starts_ends_contains() {  // like.rs:725-805, :1155-1175
  const S hay = strs({"arrow", "parrow", "arrows", "arr", "arrow long string longer than 12 bytes"});
  check_scalar(hay, "arrow", F(starts_with), F(starts_with), bools({true, false, true, false, true}));
  check_scalar(hay, "arrow", F(ends_with), F(ends_with), bools({true, true, false, false, false}));
  check_scalar(strs({"sdlkdfFkoßsdfs", "sdlkdFFkoSSdggs", "FkoS", "😃sadlksFFkoSSsh😃klF", "longer than 12 bytes FFKoSS"}), "FFkoSS",
               F(contains), F(contains), bools({false, true, false, true, false}));
  check_arrays(strs({"arrow", "rs", "arrow-rS", "Parquet"}), strs({"ARROW", "rS", "ARROW-rs", "arrow"}), F(eq_ignore_ascii_case),
               F(eq_ignore_ascii_case), bools({true, true, true, false}));  // like.rs:194-210 (doc example)
}

static void test_like_escape() {  // like.rs:1598-1838 (a few rows)
  struct Row { const char *v, *p; bool e; };
  for (const Row &t : {Row{"", "", true}, Row{"\\", "\\", true}, Row{"_", "\\_", true}, Row{"a", "\\%", false},
                       Row{"\\a", "\\\\%", true}, Row{"xyza\\c", "%a\\\\c", true}}) {
    const StringArray v = StringArray::from(S{std::string(t.v)}), p = StringArray::from(S{std::string(t.p)});
    CHECK(L::like(v, p).unwrap().to_vec() == B{t.e});
    CHECK(L::ilike(Scalar<StringArray>(v), Scalar<StringArray>(p)).unwrap().to_vec() == B{t.e});
    CHECK(L::nilike(StringViewArray::from(S{std::string(t.v)}), StringViewArray::from(S{std::string(t.p)})).unwrap().to_vec() == B{!t.e});
  }
}

static void test_nulls() {  // like.rs:1340-1363, :1532-1563
  check_scalar(S{std::string("Earth"), std::string("Fire"), std::string("Water"), std::string("Air"), N, std::string("Air"),
                 std::string("bbbbb\nAir")},
               "Air", F(like), F(like), B{false, false, false, true, N, true, false});
  const Scalar<StringArray> null_pattern(StringArray::from(S{N}));
  const BooleanArray r = L::like(StringArray::from(S{std::string("a")}), null_pattern).unwrap();
  CHECK(r.len() == 1 && r.to_vec() == B{N});
  CHECK(L::ilike(Scalar<StringArray>(StringArray::from(S{N})), StringArray::from(S{std::string("%a%b_c_d%e")})).unwrap().to_vec() == B{N});
}

static void test_errors() {
  const auto e = L::like(StringArray::from(S{std::string("a"), std::string("b")}), StringArray::from(S{std::string("a")})).unwrap_err();
  CHECK(e.status == ACU_ERR_INVALID_ARGUMENT && e.message.find("Cannot compare arrays of different lengths, got 2 vs 1") != std::string::npos);
  const auto f = L::ilike(StringArray::from(S{std::string("a")}), Scalar<StringArray>(StringArray::from(S{std::string("é%")}))).unwrap_err();
  CHECK(f.status == ACU_ERR_NOT_YET_IMPLEMENTED);
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
      {"utf8_array_like", test_utf8_array_like},
      {"utf8_array_like_scalar", test_utf8_array_like_scalar},
      {"utf8_array_ilike_unicode", test_utf8_array_ilike_unicode},
      {"starts_ends_contains", test_starts_ends_contains},
      {"like_escape", test_like_escape},
      {"nulls", test_nulls},
      {"errors", test_errors},
  };
  for (const auto &t : tests) {
    const int before = g_failed;
    t.fn();
    std::printf("%s %s\n", g_failed == before ? "ok  " : "FAIL", t.name);
  }
  std::printf("%d checks, %d failed\n", g_checks, g_failed);
  return g_failed ? 1 : 0;
}
