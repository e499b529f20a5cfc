// like.cu — arrow-string/src/like.rs: like / nlike / ilike / nilike / contains / starts_with / ends_with /
// eq_ignore_ascii_case over GenericByteArray (Utf8, Binary: i32 offsets; LargeUtf8, LargeBinary: i64) and
// GenericByteViewArray (Utf8View, BinaryView).
//
// A LIKE pattern is the glob of predicate.rs's regex_like: `\x` a literal x (a trailing `\` a literal backslash), `%` any
// run of scalars, `_` one UTF-8 scalar, anchored at both ends; ilike folds an ASCII letter to both cases plus U+212A (k)
// and U+017F (s), the simple case folds that reach ASCII. Every element matches one scalar, so a segment's leftmost start
// is also its leftmost end and the matcher needs no backtracking. The host classifies a scalar pattern once
// (Predicate::like's Eq / StartsWith / EndsWith / Contains); per-row patterns use the glob on the row's bytes. Row layout
// as k_cmp_rows; rows whose match scans more than LONG_ROW bytes are matched by one warp each (k_like_long).
#include <algorithm>
#include <string>
#include <type_traits>

#include "bitmap.cuh"
#include "bytes_cmp.cuh"
#include "internal.cuh"

namespace {

enum LikeMode : int {
  LM_EQ = 0, LM_PREFIX = 1, LM_SUFFIX = 2, LM_CONTAINS = 3,  // byte-wise against an (unescaped) needle
  LM_IEQ = 4, LM_IPREFIX = 5, LM_ISUFFIX = 6,                 // the same with u8::eq_ignore_ascii_case
  LM_GLOB = 7                                                  // the LIKE pattern itself, case-folded when icase
};
enum { P_PCT = -1, P_ANY = -2 };
constexpr int ROWS_PER_LANE = 4;
constexpr int64_t LONG_ROW = 512;   // bytes a row's match may scan before it goes to the warp-per-row kernel
constexpr int64_t LONG_CAP = 16384; // queued long rows per call; rows beyond it are matched in place

struct LikeParams {
  int64_t n;
  int mode, icase, neg;
  int binary;                 // op_binary: a row with a null side is null with value bit 0; else op_scalar (values everywhere)
  int l_bcast, r_bcast;       // the haystack (op_binary) / the pattern (op_scalar) is one value for every row
  const uint8_t *needle;      // r_bcast: the classified pattern / needle bytes (device)
  int64_t needle_len;
  const uint8_t *lv, *rv;     // validity bitmaps read, NULL = none
  int64_t loff, roff;
  int check_ascii;            // per-row ilike: the lowest evaluated row whose pattern is not ASCII goes to RES_ERR_INDEX
  uint32_t *out_bits, *out_valid;
  unsigned long long *res;    // RES_COUNT valid rows, RES_AUX0 queued long rows
  int64_t *long_rows;
};

__device__ __forceinline__ bool is_cont(uint8_t b) { return (b & 0xC0u) == 0x80u; }

// ---- byte compares and substring search (Predicate::Eq / StartsWith / EndsWith / Contains / I*Ascii) -------------------
template <bool WARP>
__device__ __forceinline__ bool range_eq(const uint8_t *a, const uint8_t *b, int64_t n, bool icase, int lane) {
  if (!WARP) return icase ? bytes_range_eq<true>(a, b, n) : bytes_range_eq<false>(a, b, n);
  bool ok = true;
  for (int64_t k = (int64_t)lane * 8; k < n; k += 256) {
    const uint32_t nb = (uint32_t)((n - k) < 8 ? (n - k) : 8);
    uint64_t x = ld_upto8(a + k, nb), y = ld_upto8(b + k, nb);
    if (icase) x = ascii_lower8(x), y = ascii_lower8(y);
    ok &= x == y;
  }
  return __all_sync(ACU_FULL_MASK, ok);
}

template <bool WARP>
__device__ __forceinline__ bool contains(const uint8_t *h, int64_t hl, const uint8_t *nd, int64_t nl, int lane) {
  if (nl == 0) return true;
  if (nl > hl) return false;
  const uint8_t first = __ldg(nd);
  if (WARP) {
    for (int64_t base = 0; base + nl <= hl; base += 32) {
      const int64_t s = base + lane;
      const bool f = s + nl <= hl && __ldg(h + s) == first && bytes_range_eq<false>(h + s, nd, nl);
      if (__any_sync(ACU_FULL_MASK, f)) return true;
    }
    return false;
  }
  if (hl <= 16 && nl <= 8) {  // the whole row in two registers: shift the window, one compare per start
    const uint64_t lo = ld_upto8(h, (uint32_t)(hl < 8 ? hl : 8)), hi = hl > 8 ? ld_upto8(h + 8, (uint32_t)(hl - 8)) : 0ull;
    const uint64_t mask = nl == 8 ? ~0ull : ((1ull << (nl * 8)) - 1ull), w = ld_upto8(nd, (uint32_t)nl);
    for (int s = 0; s + nl <= hl; ++s) {
      const uint64_t win = s == 0 ? lo : s < 8 ? ((lo >> (8 * s)) | (hi << (64 - 8 * s))) : (hi >> (8 * (s - 8)));
      if ((win & mask) == w) return true;
    }
    return false;
  }
  for (int64_t s = 0; s + nl <= hl; ++s)
    if (__ldg(h + s) == first && bytes_range_eq<false>(h + s, nd, nl)) return true;
  return false;
}

// ---- the glob matcher (regex_like) ------------------------------------------------------------------------------------
// The next pattern element at q: a literal byte, P_PCT or P_ANY.
__device__ __forceinline__ int pat_next(const uint8_t *P, int64_t pl, int64_t &q) {
  const uint8_t c = __ldg(P + q++);
  if (c == '\\') return q < pl ? (int)__ldg(P + q++) : (int)'\\';
  if (c == '%') return P_PCT;
  if (c == '_') return P_ANY;
  return c;
}

// One element against the scalar at haystack byte x: the byte after that scalar, -1 = no match.
__device__ __forceinline__ int64_t elem_match(int e, const uint8_t *H, int64_t hl, int64_t x, bool icase) {
  if (x >= hl) return -1;
  const uint8_t b = __ldg(H + x);
  if (e == P_ANY) {  // one whole UTF-8 scalar
    ++x;
    while (x < hl && is_cont(__ldg(H + x))) ++x;
    return x;
  }
  if (b == (uint8_t)e) return x + 1;
  if (icase) {
    const uint8_t lc = (uint8_t)e | 0x20u;
    if (lc >= 'a' && lc <= 'z') {
      if ((b | 0x20u) == lc) return x + 1;
      if (lc == 'k' && x + 2 < hl && b == 0xE2 && __ldg(H + x + 1) == 0x84 && __ldg(H + x + 2) == 0xAA) return x + 3;  // U+212A
      if (lc == 's' && x + 1 < hl && b == 0xC5 && __ldg(H + x + 1) == 0xBF) return x + 2;                               // U+017F
    }
  }
  return -1;
}

// The segment [qs, qe) (no unescaped %) matched from haystack byte x: the byte after the match, -1 = no match.
__device__ __forceinline__ int64_t seg_match(const uint8_t *P, int64_t pl, int64_t qs, int64_t qe, const uint8_t *H, int64_t hl, int64_t x,
                                             bool icase) {
  for (int64_t q = qs; q < qe && x >= 0;) x = elem_match(pat_next(P, pl, q), H, hl, x, icase);
  return x;
}

// The segment starting at qs: *qe = the unescaped % that ends it (or pl), *m = the scalars it matches.
__device__ __forceinline__ void seg_scan(const uint8_t *P, int64_t pl, int64_t qs, int64_t *qe, int64_t *m) {
  int64_t q = qs, k = 0;
  while (q < pl) {
    const int64_t q0 = q;
    const int e = pat_next(P, pl, q);
    if (e == P_PCT) {
      q = q0;
      break;
    }
    if (e == P_ANY || !is_cont((uint8_t)e)) ++k;
  }
  *qe = q;
  *m = k;
}

template <bool WARP>
__device__ __forceinline__ bool glob_match(const uint8_t *P, int64_t pl, const uint8_t *H, int64_t hl, bool icase, int lane) {
  int64_t q = 0, x = 0;
  bool pct = false;
  while (q < pl) {  // the head segment, anchored at the start
    const int e = pat_next(P, pl, q);
    if (e == P_PCT) {
      pct = true;
      break;
    }
    x = elem_match(e, H, hl, x, icase);
    if (x < 0) return false;
  }
  if (!pct) return x == hl;
  for (;;) {
    while (q < pl && __ldg(P + q) == '%') ++q;
    if (q >= pl) return true;  // the pattern ends with %
    int64_t qe, m;
    seg_scan(P, pl, q, &qe, &m);
    if (qe == pl) {  // the tail segment, anchored at the end: it starts m scalars before it
      int64_t t = hl;
      for (int64_t k = 0; k < m; ++k) {
        if (t <= x) return false;
        --t;
        while (t > x && is_cont(__ldg(H + t))) --t;
      }
      return seg_match(P, pl, q, qe, H, hl, t, icase) == hl;
    }
    // a middle segment: its leftmost match at a scalar boundary >= x
    int64_t end = -1;
    if (WARP) {
      for (int64_t base = x; base < hl; base += 32) {
        const int64_t s = base + lane;
        int64_t e = -1;
        if (s < hl && (s == x || !is_cont(__ldg(H + s)))) e = seg_match(P, pl, q, qe, H, hl, s, icase);
        const unsigned b = __ballot_sync(ACU_FULL_MASK, e >= 0);
        if (b) {
          end = __shfl_sync(ACU_FULL_MASK, e, __ffs(b) - 1);
          break;
        }
      }
    } else {
      for (int64_t s = x; s < hl && end < 0;) {
        end = seg_match(P, pl, q, qe, H, hl, s, icase);
        ++s;
        while (s < hl && is_cont(__ldg(H + s))) ++s;
      }
    }
    if (end < 0) return false;
    x = end;
    q = qe + 1;
  }
}

template <bool WARP>
__device__ __forceinline__ bool like_row(int mode, bool icase, const BytesItem &h, const BytesItem &nd, int lane) {
  switch (mode) {
    case LM_EQ: case LM_IEQ: return h.len == nd.len && range_eq<WARP>(h.p, nd.p, nd.len, mode == LM_IEQ, lane);
    case LM_PREFIX: case LM_IPREFIX: return h.len >= nd.len && range_eq<WARP>(h.p, nd.p, nd.len, mode == LM_IPREFIX, lane);
    case LM_SUFFIX: case LM_ISUFFIX:
      return h.len >= nd.len && range_eq<WARP>(h.p + (h.len - nd.len), nd.p, nd.len, mode == LM_ISUFFIX, lane);
    case LM_CONTAINS: return contains<WARP>(h.p, h.len, nd.p, nd.len, lane);
    default: return glob_match<WARP>(nd.p, nd.len, h.p, h.len, icase, lane);
  }
}

// Bytes a row's match may read beyond its first word.
__device__ __forceinline__ int64_t row_work(int mode, int64_t hl, int64_t nl) {
  switch (mode) {
    case LM_EQ: case LM_IEQ: return hl == nl ? nl : 0;
    case LM_CONTAINS: case LM_GLOB: return hl;
    default: return hl >= nl ? nl : 0;
  }
}

__device__ __forceinline__ bool has_non_ascii(const uint8_t *p, int64_t n) {
  for (int64_t k = 0; k < n; k += 8)
    if (ld_upto8(p + k, (uint32_t)((n - k) < 8 ? (n - k) : 8)) & 0x8080808080808080ull) return true;
  return false;
}

template <class Op, int MODE>
__device__ __forceinline__ bool row_eval(const LikeParams &p, const BytesItem &h, const BytesItem &nd, int64_t i) {
  if (MODE == LM_GLOB && p.check_ascii && has_non_ascii(nd.p, nd.len)) {
    atomicMin(p.res + RES_ERR_INDEX, (unsigned long long)i);
    return false;
  }
  constexpr int mode = MODE;
  if (std::is_same<Op, ViewOperand>::value && h.len > 12 && mode != LM_CONTAINS && mode != LM_GLOB && mode != LM_SUFFIX && mode != LM_ISUFFIX) {
    // equal / prefix of an out-of-line view: the length and the view's 4-byte prefix decide before any data buffer is read
    const bool eq = mode == LM_EQ || mode == LM_IEQ, fold = mode == LM_IEQ || mode == LM_IPREFIX;
    if (eq ? h.len != nd.len : h.len < nd.len) return false;
    const uint32_t k = (uint32_t)(nd.len < 4 ? nd.len : 4);
    uint64_t a = h.pre & (uint32_t)(k == 4 ? 0xffffffffu : ((1u << (8 * k)) - 1u)), b = ld_upto8(nd.p, k);
    if (fold) a = ascii_lower8(a), b = ascii_lower8(b);
    if (a != b) return false;
    if (!eq && nd.len <= 4) return true;
  }
  if (row_work(mode, h.len, nd.len) > LONG_ROW) {
    const unsigned long long slot = atomicAdd(p.res + RES_AUX0, 1ull);
    if (slot < (unsigned long long)LONG_CAP) {
      p.long_rows[slot] = i;
      return false;  // provisional: k_like_long flips the bit when the row matches
    }
  }
  return like_row<false>(MODE, p.icase != 0, h, nd, 0);
}

// One instantiation per mode: the mode's matcher inlined with no dispatch; the glob keeps one copy of its matcher.
template <class Op, int MODE>
__global__ void __launch_bounds__(256, MODE == LM_GLOB ? 1 : 3) k_like(const LikeParams p, const Op L, const Op R) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int64_t groups = (p.n + 31) >> 5;
  unsigned valid_cnt = 0;
  BytesItem sl{nullptr, 0, 0u};
  const BytesItem sr{p.needle, p.needle_len, 0u};
  if (p.l_bcast) sl = L.item(0);
  for (int64_t g0 = warp * ROWS_PER_LANE; g0 < groups; g0 += nwarps * ROWS_PER_LANE) {
    BytesItem ih[ROWS_PER_LANE], in[ROWS_PER_LANE];
#pragma unroll
    for (int k = 0; k < ROWS_PER_LANE; ++k) {  // the offset / view loads of 4 rows in flight
      const int64_t i = (g0 + k) * 32 + lane;
      const bool live = i < p.n;
      ih[k] = p.l_bcast ? sl : (live ? L.item(i) : BytesItem{nullptr, 0, 0u});
      in[k] = p.r_bcast ? sr : (live ? R.item(i) : BytesItem{nullptr, 0, 0u});
    }
#pragma unroll (MODE == LM_GLOB ? 1 : ROWS_PER_LANE)
    for (int k = 0; k < ROWS_PER_LANE; ++k) {  // row k's items picked out of the registers
      const int64_t row0 = (g0 + k) * 32;
      if (row0 >= p.n) break;  // warp-uniform
      BytesItem h = ih[0], nd = in[0];
#pragma unroll
      for (int j = 1; j < ROWS_PER_LANE; ++j)
        if (k == j) h = ih[j], nd = in[j];
      const int64_t left = p.n - row0;
      const uint32_t m = left >= 32 ? 0xffffffffu : ((1u << left) - 1u);
      uint32_t lw = m, rw = m;
      if (p.lv) lw &= ld_bits32(p.lv, p.loff + row0, p.loff + p.n);
      if (p.rv) rw &= ld_bits32(p.rv, p.roff + row0, p.roff + p.n);
      const uint32_t valid = p.binary ? (lw & rw) : lw;
      const bool eval = ((p.binary ? valid : m) >> lane) & 1u;
      const bool r = eval && row_eval<Op, MODE>(p, h, nd, row0 + lane);
      uint32_t v = __ballot_sync(ACU_FULL_MASK, r);
      if (lane == 0) {
        if (p.neg) v = ~v;
        p.out_bits[row0 >> 5] = v & (p.binary ? valid : m);
        if (p.out_valid) {
          p.out_valid[row0 >> 5] = valid;
          valid_cnt += __popc(valid);
        }
      }
    }
  }
  if (p.out_valid && lane == 0 && valid_cnt) atomicAdd(p.res + RES_COUNT, (unsigned long long)valid_cnt);
}

// The queued long rows, one warp each; the provisional bit (no match) is flipped where the row matches.
template <class Op, int MODE>
__global__ void __launch_bounds__(256, 1) k_like_long(const LikeParams p, const Op L, const Op R, int64_t count) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t k = warp; k < count; k += nwarps) {
    const int64_t i = p.long_rows[k];
    const BytesItem h = L.item(p.l_bcast ? 0 : i);
    const BytesItem nd = p.r_bcast ? BytesItem{p.needle, p.needle_len, 0u} : R.item(i);
    if (like_row<true>(MODE, p.icase != 0, h, nd, lane) && lane == 0) atomicXor(p.out_bits + (i >> 5), 1u << (i & 31));
  }
}

// GenericByteViewArray::is_ascii (byte_view_array.rs:1177-1188): a valid slot holding a byte >= 0x80 sets RES_AUX1.
template <class Op>
__global__ void __launch_bounds__(256) k_view_non_ascii(const Op V, int64_t n, const uint8_t *valid, int64_t voff,
                                                        unsigned long long *res) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    if (valid && !ld_bit(valid, voff + i)) continue;
    const BytesItem it = V.item(i);
    if (has_non_ascii(it.p, it.len)) atomicOr(res + RES_AUX1, 1ull);
  }
}

// ---- host side -------------------------------------------------------------------------------------------------------
const char *const OP_NAMES[] = {"LIKE", "NLIKE", "ILIKE", "NILIKE", "CONTAINS", "STARTS_WITH", "ENDS_WITH", "EQ_IGNORE_ASCII_CASE"};
const int OP_MODE[] = {LM_GLOB, LM_GLOB, LM_GLOB, LM_GLOB, LM_CONTAINS, LM_PREFIX, LM_SUFFIX, LM_IEQ};  // before classify_like

bool has_like_wildcard(const std::string &s) { return s.find_first_of("%_\\") != std::string::npos; }  // contains_like_pattern

// Predicate::like (predicate.rs:46-61) on the unescaped pattern: a pattern without `_` whose `%` are all leading and / or
// trailing is an equality, prefix, suffix or substring test of the literal between them; anything else is LM_GLOB.
int classify_like(const std::string &pat, std::string *needle) {
  std::vector<int> el;
  for (size_t q = 0; q < pat.size();) {
    const unsigned char c = (unsigned char)pat[q++];
    if (c == '\\') el.push_back(q < pat.size() ? (unsigned char)pat[q++] : '\\');
    else el.push_back(c == '%' ? P_PCT : c == '_' ? P_ANY : (int)c);
  }
  size_t a = 0, b = el.size();
  while (a < b && el[a] == P_PCT) ++a;
  while (b > a && el[b - 1] == P_PCT) --b;
  const bool lead = a > 0, trail = b < el.size();
  needle->clear();
  for (size_t k = a; k < b; ++k) {
    if (el[k] < 0) return LM_GLOB;
    needle->push_back((char)el[k]);
  }
  if (lead && a == el.size()) return LM_PREFIX;  // only %: every value matches
  return lead ? (trail ? LM_CONTAINS : LM_SUFFIX) : (trail ? LM_PREFIX : LM_EQ);
}

// Predicate::ilike's ASCII fast paths (predicate.rs:68-82) on the raw pattern, -1 = none.
int ilike_ascii_shape(const std::string &pat, std::string *needle) {
  if (!has_like_wildcard(pat)) return *needle = pat, LM_IEQ;
  const size_t n = pat.size();
  if (pat[n - 1] == '%' && !has_like_wildcard(pat.substr(0, n - 1))) return *needle = pat.substr(0, n - 1), LM_IPREFIX;
  if (pat[0] == '%' && !has_like_wildcard(pat.substr(1))) return *needle = pat.substr(1), LM_ISUFFIX;
  return -1;
}

// The bytes of row 0 of a scalar operand, read in stream order.
acu_status scalar_bytes(acu_ctx *ctx, int ob, const acu_bytes_array *s, std::string *out) {
  int64_t o[2] = {0, 0};
  if (ob == 4) {
    int32_t o32[2];
    ACU_TRY(acu_memcpy_d2h(ctx, o32, s->offsets, sizeof o32));
    o[0] = o32[0], o[1] = o32[1];
  } else {
    ACU_TRY(acu_memcpy_d2h(ctx, o, s->offsets, sizeof o));
  }
  out->assign((size_t)(o[1] - o[0]), '\0');
  return acu_memcpy_d2h(ctx, &(*out)[0], s->data + o[0], out->size());
}
acu_status scalar_bytes(acu_ctx *ctx, int, const acu_view_array *s, std::string *out) {
  uint32_t v[4];
  ACU_TRY(acu_memcpy_d2h(ctx, v, s->views, sizeof v));
  out->assign(v[0], '\0');
  if (v[0] <= 12) return memcpy(&(*out)[0], reinterpret_cast<const char *>(v) + 4, v[0]), ACU_OK;
  if (v[2] >= (uint32_t)s->n_buffers) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "view buffer index out of range");
  return acu_memcpy_d2h(ctx, &(*out)[0], s->buffers[v[2]] + v[3], out->size());
}

// The device operands; the view pointer tables go to `*cursor` (scratch).
size_t table_bytes(const acu_bytes_array *) { return 0; }
size_t table_bytes(const acu_view_array *a) { return acu_view_table_bytes(a); }
acu_status make_operand(acu_ctx *, int ob, const acu_bytes_array *a, uint8_t **, BytesOperand *op) {
  *op = BytesOperand{a->offsets, a->data, ob};
  return ACU_OK;
}
acu_status make_operand(acu_ctx *ctx, int, const acu_view_array *a, uint8_t **cursor, ViewOperand *op) {
  ACU_TRY(acu_view_operand(ctx, a, *cursor, op));
  *cursor += acu_view_table_bytes(a);
  return ACU_OK;
}

// k_like (count < 0) or k_like_long over `count` queued rows, instantiated for p.mode
template <class Op>
acu_status launch_like(acu_ctx *ctx, const LikeParams &p, const Op &L, const Op &R, int grid, int64_t count) {
#define LIKE_CASE(M)                                                                             \
  case M:                                                                                        \
    if (count < 0) ACU_LAUNCH_TIMED(ctx, ACU_K_CMP, (k_like<Op, M>), grid, 256, 0, p, L, R);         \
    else ACU_LAUNCH_TIMED(ctx, ACU_K_CMP, (k_like_long<Op, M>), grid, 256, 0, p, L, R, count);        \
    return ACU_OK;
  switch (p.mode) {
    LIKE_CASE(LM_EQ) LIKE_CASE(LM_PREFIX) LIKE_CASE(LM_SUFFIX) LIKE_CASE(LM_CONTAINS)
    LIKE_CASE(LM_IEQ) LIKE_CASE(LM_IPREFIX) LIKE_CASE(LM_ISUFFIX) LIKE_CASE(LM_GLOB)
  }
#undef LIKE_CASE
  return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "invalid like mode %d", p.mode);
}

int like_grid(acu_ctx *ctx, int64_t n) {
  const int64_t groups = (n + 31) / 32;
  return acu_grid(ctx, ((groups + ROWS_PER_LANE - 1) / ROWS_PER_LANE + 7) / 8, 16);
}

// like_op (like.rs:218-296) with string_apply / binary_apply, op_scalar and op_binary.
template <class Arr>
acu_status like_run(acu_ctx *ctx, int ob, int32_t is_utf8, acu_like_op op, const Arr *l, const Arr *r, acu_array_out *out) {
  if ((int)op < 0 || (int)op > 7) return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "invalid like op %d", (int)op);
  int64_t len;
  ACU_TRY(acu_cmp_len(ctx, &l->nulls, &r->nulls, &len));
  if (!is_utf8 && op != ACU_CONTAINS && op != ACU_STARTS_WITH && op != ACU_ENDS_WITH)  // binary_like.rs:34-47
    return acu_fail(ctx, ACU_ERR_INVALID_ARGUMENT, -1, 0, 0, 0, "Invalid binary operation: %s", OP_NAMES[op]);
  out->len = len;
  out->has_validity = 0;
  out->null_count = 0;
  const bool ls = l->nulls.is_scalar != 0, rs = r->nulls.is_scalar != 0;
  const bool ilike = op == ACU_ILIKE || op == ACU_NILIKE;
  acu_status st = ACU_OK;
  LikeParams p{};
  p.n = len;
  p.neg = op == ACU_NLIKE || op == ACU_NILIKE;
  p.icase = ilike;
  std::string needle;
  bool quirk = false;  // views: Predicate::ilike's ASCII fast path, decided by is_ascii over the valid slots
  std::string quirk_needle;
  int quirk_mode = -1;
  int64_t lnc = 0;
  if (rs) {  // op_scalar (like.rs:349-368), or a null scalar: BooleanArray::new_null (:314-316)
    const int64_t rnc = acu_resolve_null_count(ctx, &r->nulls, &st);
    ACU_TRY(st);
    if (rnc > 0) return len ? acu_new_null(ctx, len, acu_bitmap_bytes(len), out) : ACU_OK;
    std::string pat;
    ACU_TRY(scalar_bytes(ctx, ob, r, &pat));
    if (ilike) {
      for (unsigned char c : pat)
        if (c >= 0x80)
          return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, -1, 0, 0, 0, "%s with a non-ASCII pattern (full Unicode case folding)", OP_NAMES[op]);
    }
    if (len == 0) return ACU_OK;
    p.mode = OP_MODE[op];
    needle = pat;
    if (op == ACU_LIKE || op == ACU_NLIKE) {
      std::string lit;
      const int m = classify_like(pat, &lit);
      if (m != LM_GLOB) p.mode = m, needle = lit;
    }
    lnc = acu_resolve_null_count(ctx, &l->nulls, &st);
    ACU_TRY(st);
    // Only a view with null slots can tell the fast path from the regex: a valid slot decides is_ascii, and where every
    // valid slot is ASCII both agree on the valid slots.
    if (ilike && std::is_same<Arr, acu_view_array>::value && lnc > 0) {
      quirk_mode = ilike_ascii_shape(pat, &quirk_needle);
      quirk = quirk_mode >= 0;
    }
    p.r_bcast = 1;
    p.lv = l->nulls.validity;
    p.loff = l->nulls.validity_offset;
    out->has_validity = l->nulls.validity != nullptr;  // from_unary: nulls = the haystack's logical_nulls()
  } else {  // op_binary (like.rs:385-432): a row is null where either side is
    if (len == 0) return ACU_OK;
    lnc = acu_resolve_null_count(ctx, &l->nulls, &st);
    ACU_TRY(st);
    const int64_t rnc = acu_resolve_null_count(ctx, &r->nulls, &st);
    ACU_TRY(st);
    if (ls && lnc > 0) return acu_new_null(ctx, len, acu_bitmap_bytes(len), out);
    p.binary = 1;
    p.l_bcast = ls;
    p.mode = OP_MODE[op];
    p.check_ascii = ilike;
    if (!ls && lnc > 0) p.lv = l->nulls.validity, p.loff = l->nulls.validity_offset;
    if (rnc > 0) p.rv = r->nulls.validity, p.roff = r->nulls.validity_offset;
    out->has_validity = lnc > 0 || rnc > 0;
  }
  // scratch: [view pointer tables][needle][queued long rows]
  const size_t tb = table_bytes(l) + table_bytes(r);
  const size_t nb = (std::max(needle.size(), quirk_needle.size()) + 256) & ~(size_t)255;
  void *scratch;
  ACU_TRY(acu_scratch(ctx, tb + nb + (size_t)LONG_CAP * sizeof(int64_t), &scratch));
  uint8_t *cursor = static_cast<uint8_t *>(scratch);
  using Op = typename std::conditional<std::is_same<Arr, acu_view_array>::value, ViewOperand, BytesOperand>::type;
  Op L, R;
  ACU_TRY(make_operand(ctx, ob, l, &cursor, &L));
  ACU_TRY(make_operand(ctx, ob, r, &cursor, &R));
  uint8_t *d_needle = cursor;
  p.long_rows = reinterpret_cast<int64_t *>(cursor + nb);
  if (quirk) {
    ACU_TRY(acu_res_reset(ctx));
    ACU_LAUNCH_TIMED(ctx, ACU_K_CMP, k_view_non_ascii<Op>, acu_grid(ctx, (len + 255) / 256, 8), 256, 0, L, len, l->nulls.validity,
                     l->nulls.validity_offset, ctx->d_res);
    ACU_TRY(acu_res_fetch(ctx));
    if (ctx->h_res[RES_AUX1] == 0) p.mode = quirk_mode, needle = quirk_needle;
  }
  if (!needle.empty()) ACU_CUDA(ctx, cudaMemcpyAsync(d_needle, needle.data(), needle.size(), cudaMemcpyHostToDevice, ctx->stream));
  p.needle = d_needle;
  p.needle_len = (int64_t)needle.size();
  p.out_bits = static_cast<uint32_t *>(out->values);
  p.out_valid = out->has_validity ? reinterpret_cast<uint32_t *>(out->validity) : nullptr;
  p.res = ctx->d_res;
  ACU_TRY(acu_res_reset(ctx));
  ACU_TRY(launch_like(ctx, p, L, R, like_grid(ctx, len), -1));
  ACU_TRY(acu_res_fetch(ctx));
  const unsigned long long *h = ctx->h_res;
  if (h[RES_ERR_INDEX] != ~0ull)
    return acu_fail(ctx, ACU_ERR_NOT_YET_IMPLEMENTED, (int64_t)h[RES_ERR_INDEX], 0, 0, (uint64_t)len,
                    "%s with a non-ASCII pattern (full Unicode case folding)", OP_NAMES[op]);
  if (out->has_validity) out->null_count = len - (int64_t)h[RES_COUNT];
  const int64_t queued = (int64_t)std::min<unsigned long long>(h[RES_AUX0], (unsigned long long)LONG_CAP);
  if (queued > 0) {
    ACU_TRY(launch_like(ctx, p, L, R, acu_grid(ctx, (queued + 7) / 8, 16), queued));
    ACU_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    acu_kstats_drain(ctx);
  }
  return ACU_OK;
}

}  // namespace

extern "C" acu_status acu_like_bytes(acu_ctx *ctx, int32_t offset_bytes, int32_t is_utf8, acu_like_op op, const acu_bytes_array *l,
                                     const acu_bytes_array *r, acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  ACU_TRY(acu_offset_width_check(ctx, offset_bytes));
  return like_run(ctx, offset_bytes, is_utf8, op, l, r, out);
}

extern "C" acu_status acu_like_byte_view(acu_ctx *ctx, int32_t is_utf8, acu_like_op op, const acu_view_array *l, const acu_view_array *r,
                                         acu_array_out *out) {
  ACU_ENTER(ctx);
  ACU_TRY(acu_sync_only(ctx));
  return like_run(ctx, 0, is_utf8, op, l, r, out);
}
