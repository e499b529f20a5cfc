"""The variable-width kernels at the points where a row changes path, against the Python oracles at the usual bar
(offsets, value bytes, validity bits, null_count, NullBuffer presence, error status / text / row):

  like.cu        a row whose match scans more than LONG_ROW bytes is queued for k_like_long (one warp per row), which
                 flips a provisional bit (written negated for NLIKE / NILIKE); past LONG_CAP queued rows the rest are
                 matched in place by one thread. Rows of row_work 511 / 512 / 513 in every mode, and LONG_CAP, LONG_CAP + 1
                 and LONG_CAP + 3000 long rows spread among short ones.
  substring.cu   a by_char row longer than LONG_ROW bytes is walked 32 bytes at a time by one warp (k_char_long, SMs x 16
                 CTAs of 8 warps); rows of 512 / 513 bytes with a char start or a multi-byte char at window positions
                 31 / 32 / 33 from either end, and more long rows than one round of k_char_long.
  bytes_engine   a 2048-row CTA whose output span (its bytes plus `lead`, the 16-B misalignment of its first output byte)
                 fits BY_STAGE_CAP is assembled in shared memory, otherwise stored directly; spans of 49152 / 49153 at
                 leads 0 / 1 / 15, partial last chunks, empty and single-row CTAs, through substring and concat_elements
                 called with an output 0 / 1 / 15 bytes into a sentinel-filled allocation.

Long columns are built from a few dozen distinct values: the oracle runs on those and its result is expanded by row
index. Every test asserts that its rows sit where it says they do."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from acu import BOOL, HostArray, Utf8Column, ViewColumn, bitmap_bytes, pack_bits
from acu import _abi as abi

from like_util import column
from oracle_concat_elements import ConcatElementsOracle
from oracle_like import LikeOracle
from oracle_substring import SubstringOracle, bytes_column, nulls_unsliced
from substring_util import bytes_col, nulls_of, sliced
from test_gpu_concat_elements import assert_result as assert_concat
from test_gpu_like import same as like_same
from test_gpu_substring import assert_result as assert_substring
from test_gpu_substring import same as substring_same
from test_gpu_parity import assert_same

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "arrow-rs_b200", "csrc")

# Mirrors of the kernels' constants (pinned by test_constants_pinned).
LONG_ROW = 512            # like.cu and substring.cu: bytes a row may scan / walk before it goes to a warp
LONG_CAP = 16384          # like.cu: queued long rows per call
BY_THREADS = 512          # bytes_engine.cuh: threads per CTA
BY_ROWS = BY_THREADS * 4  # rows per CTA
BY_STAGE_CAP = 48 * 1024  # bytes a CTA may assemble in shared memory
CHAR_LONG_CTAS_PER_SM, CHAR_LONG_WARPS_PER_CTA = 16, 8  # k_char_long's grid
SENTINEL = 0xA5

LIKE_ORACLE, SUBSTRING_ORACLE, CONCAT_ORACLE = LikeOracle(), SubstringOracle(), ConcatElementsOracle()
STRING_TYPES = ["utf8", "large_utf8", "utf8_view"]
LIKE, NLIKE, ILIKE, NILIKE = abi.LIKE, abi.NLIKE, abi.ILIKE, abi.NILIKE
CONTAINS, STARTS_WITH, ENDS_WITH, IEQ_OP = abi.CONTAINS, abi.STARTS_WITH, abi.ENDS_WITH, abi.EQ_IGNORE_ASCII_CASE


# ---- 0. the constants the placements depend on -------------------------------------------------------------------------
def _source(name):
    with open(os.path.join(CSRC, name), encoding="utf-8") as f:
        return f.read()


def test_constants_pinned():
    """A retune of any of these moves every boundary away from the rows placed on it: update the mirrors above (and the
    placements) together with the kernels."""
    like, sub, eng = _source("like.cu"), _source("substring.cu"), _source("bytes_engine.cuh")
    assert re.search(r"constexpr int64_t LONG_ROW = (\d+);", like).group(1) == str(LONG_ROW)
    assert re.search(r"constexpr int64_t LONG_CAP = (\d+);", like).group(1) == str(LONG_CAP)
    assert "if (row_work(mode, h.len, nd.len) > LONG_ROW)" in like
    assert re.search(r"constexpr int64_t LONG_ROW = (\d+);", sub).group(1) == str(LONG_ROW)
    assert "if (L > LONG_ROW)" in sub
    assert re.search(r"k_char_long, acu_grid\(ctx, \(n \+ 7\) / 8, (\d+)\), 256,", sub).group(1) == str(CHAR_LONG_CTAS_PER_SM)
    assert 256 // 32 == CHAR_LONG_WARPS_PER_CTA
    assert re.search(r"#define BY_THREADS (\d+)\s", eng).group(1) == str(BY_THREADS)
    assert re.search(r"#define BY_ROWS \(BY_THREADS \* (\d+)\)", eng).group(1) == str(BY_ROWS // BY_THREADS)
    a, b = re.search(r"#define BY_STAGE_CAP \((\d+) \* (\d+)\)", eng).groups()
    assert int(a) * int(b) == BY_STAGE_CAP
    assert "(cta_end - stage_origin) <= (int64_t)stage_cap" in eng


# ---- A. like: row_work at 511 / 512 / 513 ------------------------------------------------------------------------------
LM_EQ, LM_PREFIX, LM_SUFFIX, LM_CONTAINS, LM_IEQ, LM_IPREFIX, LM_ISUFFIX, LM_GLOB = range(8)
MODE_NAMES = ["EQ", "PREFIX", "SUFFIX", "CONTAINS", "IEQ", "IPREFIX", "ISUFFIX", "GLOB"]
OP_MODE = {LIKE: LM_GLOB, NLIKE: LM_GLOB, ILIKE: LM_GLOB, NILIKE: LM_GLOB, CONTAINS: LM_CONTAINS, STARTS_WITH: LM_PREFIX,
           ENDS_WITH: LM_SUFFIX, IEQ_OP: LM_IEQ}


def classify_like(pat):
    """like.cu's classify_like on pattern bytes: (mode, needle)."""
    el, q = [], 0
    while q < len(pat):
        c = pat[q]
        q += 1
        if c == 0x5C:
            el.append(pat[q] if q < len(pat) else 0x5C)
            q += q < len(pat)
        else:
            el.append(-1 if c == 0x25 else -2 if c == 0x5F else c)
    a, b = 0, len(el)
    while a < b and el[a] == -1:
        a += 1
    while b > a and el[b - 1] == -1:
        b -= 1
    if any(e < 0 for e in el[a:b]):
        return LM_GLOB, pat
    needle, lead, trail = bytes(el[a:b]), a > 0, b < len(el)
    if lead and a == len(el):
        return LM_PREFIX, needle
    return (LM_CONTAINS if trail else LM_SUFFIX) if lead else (LM_PREFIX if trail else LM_EQ), needle


def ilike_ascii_shape(pat):
    """like.cu's ilike_ascii_shape: the view is_ascii quirk's mode, or None."""
    wild = lambda s: any(c in s for c in b"%_\\")
    if not wild(pat):
        return LM_IEQ, pat
    if pat.endswith(b"%") and not wild(pat[:-1]):
        return LM_IPREFIX, pat[:-1]
    if pat.startswith(b"%") and not wild(pat[1:]):
        return LM_ISUFFIX, pat[1:]
    return None


def device_mode(op, pat, scalar):
    if scalar and op in (LIKE, NLIKE):
        return classify_like(pat)
    return OP_MODE[op], pat


def row_work(mode, hl, nl):
    if mode in (LM_EQ, LM_IEQ):
        return nl if hl == nl else 0
    if mode in (LM_CONTAINS, LM_GLOB):
        return hl
    return nl if hl >= nl else 0


def reaches_queue(mode, hay, nd, view):
    """False where the view's length / 4-byte prefix shortcut (like.cu row_eval) decides before the queue test."""
    if not view or len(hay) <= 12 or mode not in (LM_EQ, LM_IEQ, LM_PREFIX, LM_IPREFIX):
        return True
    eq, fold = mode in (LM_EQ, LM_IEQ), mode in (LM_IEQ, LM_IPREFIX)
    if (len(hay) != len(nd)) if eq else (len(hay) < len(nd)):
        return False
    k = min(len(nd), 4)
    a, b = hay[:k], nd[:k]
    if fold:
        a, b = a.lower(), b.lower()
    return a == b and (eq or len(nd) > 4)


WIDE = {1: "abcdKxyz", 2: "éßΓ¿ÿ", 3: "€⊢日￿", 4: "😈🎉\U00010000"}
OTHER = {"a": "c", "b": "d", "c": "a", "d": "b", "K": "L", "x": "w", "y": "v", "z": "u", "é": "è", "ß": "à", "Γ": "Δ",
         "¿": "¾", "ÿ": "þ", "€": "₭", "⊢": "⊣", "日": "月", "￿": "￾", "😈": "😉", "🎉": "🎊",
         "\U00010000": "\U00010001", "q": "r", "Q": "R", "m": "n", "M": "N"}


def fill(nbytes, widths, rng):
    """A str of exactly `nbytes` UTF-8 bytes: chars of the given byte widths in turn, ASCII where the next one does not fit."""
    out, k, used = [], 0, 0
    while used < nbytes:
        w = widths[k % len(widths)]
        if used + w > nbytes:
            w = 1
        pool = WIDE[w]
        out.append(pool[int(rng.integers(0, len(pool)))])
        used += w
        k += 1
    return "".join(out)


def char_at(s, pos):
    """(index, char) of the char of s covering UTF-8 byte `pos`."""
    at = 0
    for j, ch in enumerate(s):
        w = len(ch.encode())
        if at <= pos < at + w:
            return j, ch
        at += w
    raise IndexError(pos)


def swap_at(s, pos):
    """s with the char covering byte `pos` replaced by another char of the same width (differing in its last byte)."""
    j, ch = char_at(s, pos)
    return s[:j] + OTHER[ch] + s[j + 1:]


def case_swapped(s):
    return s.swapcase() if s.isascii() else "".join(c.swapcase() if c.isascii() else c for c in s)


def bodies(W, rng):
    """Haystack / needle bodies of exactly W bytes, no LIKE wildcards: ASCII (with letters at both ends), and mixed ones whose
    last char is 2 / 3 / 4 bytes wide, so that for W = 513 a multi-byte scalar straddles byte 512."""
    asc = "Kq" + fill(W - 4, (1,), rng) + "mQ"
    out = {"ascii": asc}
    for w in (2, 3, 4):
        out[f"mixed{w}"] = "Kq" + fill(W - 2 - w, (1, 2, 3, 4), rng) + WIDE[w][0]
    for name, s in out.items():
        assert len(s.encode()) == W, name
    return out


def boundary_rows(W, rng):
    """(hay rows, needle bodies) of one width: each body, near-misses in its last byte, in byte 512 and in byte 0, a
    case-swapped copy, one byte longer at either end, one char shorter, and its last multi-byte char spelled as ASCII."""
    b = bodies(W, rng)
    rows, owner = [], []
    for name, s in b.items():
        mine = [s, swap_at(s, W - 1), swap_at(s, 0), case_swapped(s), s + "z", "z" + s, s[:-1], "Kq" + s[2:]]
        if W > 512:
            mine.append(swap_at(s, 512))
        if W > 511:
            mine.append(swap_at(s, 511))
        last = s[-1]
        if not last.isascii():
            mine.append(s[:-1] + "y" * len(last.encode()))  # same bytes, more scalars: `_` at the end no longer fits
        rows += mine
        owner += [name] * len(mine)
    return rows + [None, "ab", ""], owner + ["ascii"] * 3, b


def scalar_cases(b):
    """(op, pattern) pairs whose device mode covers EQ, IEQ, PREFIX, SUFFIX, CONTAINS and GLOB on W-byte needles / rows."""
    cases = []
    asc = b["ascii"]
    for name, s in b.items():
        tail3, j512 = s[-3:], None
        cases += [(LIKE, s), (IEQ_OP, s), (LIKE, s + "%"), (LIKE, "%" + s), (STARTS_WITH, s), (ENDS_WITH, s),
                  (LIKE, "%" + tail3 + "%"), (CONTAINS, tail3), (LIKE, "%" + s[-2] + "_"), (LIKE, "%" + s[-3] + "_%"),
                  (LIKE, s[:2] + "%" + s[-1]), (LIKE, "_" + s[1:])]
    cases += [(ILIKE, asc), (ILIKE, asc.lower() + "%"), (ILIKE, "%" + asc.upper()), (ILIKE, "%k_%"), (ILIKE, "%mq")]
    out = []
    for op, p in cases:  # each positive op with its negation
        out.append((op, p))
        if op in (LIKE, ILIKE):
            out.append((op + 1, p))
    return out


def placements(op, typ, hays, pats, scalar):
    """{mode: set of row_work} over the rows that reach the queue test (evaluated rows only)."""
    got = {}
    view = typ == "utf8_view"
    for i, h in enumerate(hays):
        p = pats[0] if scalar else pats[i]
        if (h is None and not scalar) or p is None:
            continue
        hb, pb = (h or "").encode(), p.encode()
        mode, nd = device_mode(op, pb, scalar)
        if reaches_queue(mode, hb, nd, view):
            got.setdefault(mode, set()).add(row_work(mode, len(hb), len(nd)))
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("typ", STRING_TYPES)
def test_like_row_work_boundary(gpu, typ):
    """row_work 511 / 512 / 513 in every mode, matches and near-misses at the last byte, at byte 512 and in a multi-byte
    scalar across it, every positive op with its negation; op_scalar and op_binary."""
    rng = np.random.default_rng(512)
    seen = {}
    for W in (511, 512, 513):
        hays, owner, b = boundary_rows(W, rng)
        hc = column(typ, hays)
        for op, p in scalar_cases(b):
            like_same(gpu, op, typ, hc, column(typ, [p], scalar=True), f"W={W} op={op} {p[:8]!r}..{p[-4:]!r}")
            for m, w in placements(op, typ, hays, [p], True).items():
                seen.setdefault(m, set()).update(w)
        # op_binary: each row against the body it was made from (and the ASCII one for ilike, whose patterns must be ASCII)
        for op in range(8):
            for shape in ("", "%", "pre"):
                if op in (ILIKE, NILIKE):
                    src = [b["ascii"]] * len(hays)
                else:
                    src = [b[o] for o in owner]
                pats = [s if shape == "" else (s + "%" if shape == "%" else "%" + s[-5:]) for s in src]
                pats[-1] = None
                like_same(gpu, op, typ, hc, column(typ, pats), f"W={W} per-row op={op} shape={shape!r}")
                for m, w in placements(op, typ, hays, pats, False).items():
                    seen.setdefault(m, set()).update(w)
    for m in (LM_EQ, LM_IEQ, LM_PREFIX, LM_SUFFIX, LM_CONTAINS, LM_GLOB):
        assert {511, 512, 513} <= seen.get(m, set()), f"{MODE_NAMES[m]}: row_work {sorted(seen.get(m, set()))[-6:]}"


@pytest.mark.gpu
def test_like_prefix_suffix_longer_haystack(gpu):
    """PREFIX / SUFFIX: nl of 511 / 512 / 513 with hl == nl and hl > nl, for each of the three string types."""
    rng = np.random.default_rng(77)
    for W in (511, 512, 513):
        nd = bodies(W, rng)["mixed3"]
        hays = [nd, nd + "tail€", "head😈" + nd, swap_at(nd, W - 1) + "t", "h" + swap_at(nd, 0), nd[:-1]]
        for typ in STRING_TYPES:
            hc = column(typ, hays)
            for op, p, mode in [(STARTS_WITH, nd, LM_PREFIX), (LIKE, nd + "%", LM_PREFIX), (NLIKE, nd + "%", LM_PREFIX),
                                (ENDS_WITH, nd, LM_SUFFIX), (LIKE, "%" + nd, LM_SUFFIX), (NLIKE, "%" + nd, LM_SUFFIX)]:
                assert device_mode(op, p.encode(), True)[0] == mode
                works = [(len(h.encode()), row_work(mode, len(h.encode()), W)) for h in hays]
                assert (W, W) in works and any(hl > W and w == W for hl, w in works)
                like_same(gpu, op, typ, hc, column(typ, [p], scalar=True), f"W={W} {typ} op={op} mode={MODE_NAMES[mode]}")


def long_null_columns(typ, value, n_valid):
    """A column whose null slots hold `value` (long): Utf8 / LargeUtf8 keep the bytes under the slot, views a view of it."""
    items = [value if i % 3 == 0 else None for i in range(n_valid * 3)] + ["x"]
    if typ == "utf8_view":
        col = ViewColumn.from_values([None if x is None else x.encode() for x in items], 1 << 16)
        under = col.views[0].copy()  # row 0 is valid and holds `value` out of line
        col.views[[i for i, x in enumerate(items) if x is None]] = under
        return col
    return bytes_col([None if x is None else x.encode() for x in items], np.int64 if typ == "large_utf8" else np.int32,
                     garbage=value.encode())


@pytest.mark.gpu
@pytest.mark.parametrize("typ", STRING_TYPES)
def test_like_long_match_under_null(gpu, typ):
    """op_scalar computes a value at every slot: a long matching haystack under a null slot is queued and its flipped bit
    (negated for NLIKE) must be there."""
    rng = np.random.default_rng(3)
    value = "ab" + fill(600, (1, 2, 3), rng) + "Kq"
    col = long_null_columns(typ, value, 40)
    assert col.nulls.null_count > 0
    for op, p in [(LIKE, "%K_"), (NLIKE, "%K_"), (LIKE, "%" + value[300:310] + "%"), (NLIKE, "%" + value[300:310] + "%"),
                  (LIKE, "ab%_q"), (NLIKE, "ab%_q"), (CONTAINS, "Kq"), (ILIKE, "%kQ"), (NILIKE, "AB%")]:
        mode, nd = device_mode(op, p.encode(), True)
        assert row_work(mode, len(value.encode()), len(nd)) > LONG_ROW
        like_same(gpu, op, typ, col, column(typ, [p], scalar=True), f"{typ} under null op={op} {p[:12]!r}")


@pytest.mark.gpu
def test_like_view_shortcut_and_is_ascii_quirk(gpu):
    """Views: long values whose length or 4-byte prefix decides EQ / IEQ / PREFIX before the queue; ilike through the
    is_ascii quirk (IEQ / IPREFIX / ISUFFIX on 511 / 512 / 513-byte needles) and, with one non-ASCII valid value, the glob."""
    rng = np.random.default_rng(8)
    for W in (511, 512, 513):
        asc = bodies(W, rng)["ascii"]
        rows = [asc, asc.swapcase(), swap_at(asc, 0), swap_at(asc, W - 1), swap_at(asc, 4), asc + "z", "z" + asc, asc[:-1],
                "KQ" + asc[2:], None, "kq", None]
        for non_ascii in (False, True):
            items = rows + (["é" * 300] if non_ascii else [])
            col = column("utf8_view", items)
            for op, p in [(LIKE, asc), (IEQ_OP, asc), (LIKE, asc + "%"), (STARTS_WITH, asc), (STARTS_WITH, "Kq"),
                          (LIKE, "KqA%"), (ILIKE, asc), (NILIKE, asc), (ILIKE, asc.lower() + "%"), (NILIKE, asc.upper() + "%"),
                          (ILIKE, "%" + asc.lower()), (NILIKE, "%" + asc), (ILIKE, "kq%"), (NILIKE, "%Q")]:
                if op in (ILIKE, NILIKE) and not non_ascii:
                    mode = ilike_ascii_shape(p.encode())[0]
                    assert mode in (LM_IEQ, LM_IPREFIX, LM_ISUFFIX)
                    nl = len(ilike_ascii_shape(p.encode())[1])
                    assert nl <= 4 or nl == W
                like_same(gpu, op, "utf8_view", col, column("utf8_view", [p], scalar=True), f"W={W} non_ascii={non_ascii} op={op}")
            # the prefix shortcut decides the rows that differ in their first 4 bytes or in length
            decided = [not reaches_queue(LM_EQ, (h or "").encode(), asc.encode(), True) for h in items]
            assert sum(decided) >= 5


# ---- A. like: the LONG_CAP queue ----------------------------------------------------------------------------------------
def cap_values(rng):
    """Distinct values: 30 long ones (520..700 bytes, all containing "Kq", half "ab€d"), 8 short ones, and a null."""
    longs = []
    for k in range(30):
        n = int(rng.integers(520, 700))
        core = fill(n - 8, (1, 1, 2, 3, 4), rng)
        mid = len(core) // 2
        s = core[:mid] + ("ab€d" if k % 2 else "ab€e") + core[mid:]
        longs.append(s[: len(s) - 4] + "Kq" + s[len(s) - 4:] if k % 3 else "Kq" + s)
    shorts = ["", "Kq", "ab€d", "xKqx", "abcd", "é", "q" * 40, "ab€dKq"]
    for s in longs:
        assert len(s.encode()) > LONG_ROW
    for s in shorts:
        assert len(s.encode()) <= 40
    return longs + shorts + [None], len(longs)


def expand_like(small, idx):
    """The oracle's result on the distinct values, expanded to the rows idx."""
    vals = small.value_array()[idx]
    if small.validity is None:
        return HostArray(BOOL, pack_bits(vals), len(idx), None, 0, 0, 0)
    valid = small.valid_mask()[idx]
    return HostArray(BOOL, pack_bits(vals), len(idx), pack_bits(valid), 0, 0, int(len(idx) - valid.sum()))


@pytest.mark.gpu
@pytest.mark.parametrize("typ", STRING_TYPES)
def test_like_long_cap(gpu, typ):
    """Exactly LONG_CAP, LONG_CAP + 1 and LONG_CAP + 3000 long rows, interleaved with short and null rows over the whole
    column: which rows overflow the queue depends on scheduling, and every row's bit must be right either way."""
    rng = np.random.default_rng(16384)
    distinct, n_long_distinct = cap_values(rng)
    small_col = column(typ, distinct)
    ops = [(CONTAINS, "Kq"), (NLIKE, "%Kq%"), (LIKE, "%ab_d%"), (NILIKE, "%AB_D%")]
    small = {(op, p): LIKE_ORACLE.like_view(op, small_col, column(typ, [p], scalar=True)) if typ == "utf8_view" else
             LIKE_ORACLE.like_bytes(op, small_col, column(typ, [p], scalar=True)) for op, p in ops}
    for n_long in (LONG_CAP, LONG_CAP + 1, LONG_CAP + 3000):
        n_short, n_null = n_long // 2, n_long // 8
        idx = np.concatenate([rng.integers(0, n_long_distinct, n_long), rng.integers(n_long_distinct, len(distinct) - 1, n_short),
                              np.full(n_null, len(distinct) - 1)])
        idx = idx[rng.permutation(len(idx))]
        assert set(np.unique(idx).tolist()) == set(range(len(distinct)))
        items = [distinct[i] for i in idx]
        col = column(typ, items, block=1 << 22)
        lens = np.array([len(d.encode()) if d is not None else 0 for d in distinct])[idx]
        assert int((lens > LONG_ROW).sum()) == n_long  # CONTAINS / GLOB: row_work = hl; null slots are empty
        assert int((idx[: len(idx) // 4] < n_long_distinct).sum()) > 0 and int((idx[-len(idx) // 4:] < n_long_distinct).sum()) > 0
        for op, p in ops:
            assert device_mode(op, p.encode(), True)[0] in (LM_CONTAINS, LM_GLOB)
            exp = expand_like(small[(op, p)], idx)
            got = gpu.like_view(op, col, column(typ, [p], scalar=True)) if typ == "utf8_view" else \
                gpu.like_bytes(op, col, column(typ, [p], scalar=True))
            assert_same(got, exp, f"{typ} long rows={n_long} op={op} {p!r}")
        # CONTAINS "Kq" matches every long row, so a queued row left unflipped shows
        assert small[(CONTAINS, "Kq")].value_array()[:n_long_distinct].all()


# ---- B. substring_by_char: the warp window and k_char_long's rounds ----------------------------------------------------
def char_starts(b):
    return [k for k, x in enumerate(b) if not 0x80 <= x <= 0xBF]


def by_char_templates(rng):
    """Rows of exactly 512 and 513 bytes of 1-, 2-, 3- and 4-byte chars, shifted by an ASCII lead so that every residue
    puts a char start or a multi-byte char's continuation at window positions 31 / 32 / 33 from either end."""
    out = []
    for L in (512, 513):
        for widths in ((1,), (2,), (3,), (4,), (1, 2, 3, 4), (4, 3, 2, 1)):
            for front in range(max(widths)):
                s = "A" * front + fill(L - front, widths, rng)
                b = s.encode()
                assert len(b) == L
                out.append(b)
    return out


def by_char_params(b):
    """Starts 0, 1, k and -k on either side of a 32-byte window boundary (and deep in the row), -(chars + 1); for each the
    lengths None, the exact remaining char count, one less, and 2^64 - 1."""
    st = char_starts(b)
    nch, L = len(st), len(b)
    fwd = [next(j for j, p in enumerate(st) if p >= bound) for bound in (32, 64, 480)]
    back = [sum(1 for p in st if p >= L - bound) for bound in (32, 64, 480)]
    starts = {0, 1, nch, -(nch + 1)} | {k for j in fwd for k in (j - 1, j)} | {-k for c in back for k in (c, c + 1)}
    out = []
    for s in sorted(starts):
        first = s if s >= 0 else max(nch + s, 0)
        rem = max(nch - first, 0)
        for ln in {None, rem, rem - 1, 2**64 - 1}:
            if ln is None or ln >= 0:
                out.append((s, ln))
    return out


@pytest.mark.gpu
def test_by_char_window_boundaries(gpu):
    """512-byte rows (one thread) and 513-byte rows (one warp) with starts and lengths across the 32-byte windows of
    nth_fwd / nth_back; i32 and i64 offsets, plain and sliced; a null row holding 700 bytes must stay empty."""
    rng = np.random.default_rng(513)
    tmpl = by_char_templates(rng)
    for L in (512, 513):
        for pos in (31, 32, 33):
            for p in (pos, L - 1 - pos):
                assert any(len(t) == L and not 0x80 <= t[p] <= 0xBF for t in tmpl), (L, p)
                assert any(len(t) == L and 0x80 <= t[p] <= 0xBF for t in tmpl), (L, p)
    for t in tmpl:
        items = [t, None, "aé".encode()]
        params = by_char_params(t)
        for dtype in (np.int32, np.int64):
            plain = bytes_col(items, dtype, garbage=b"N" * 700)
            full = bytes_col([b"x", "ÿ".encode()] + items + [b"z"], dtype, garbage=b"N" * 700)
            for col in (plain, sliced(full, 2, len(items))):
                for s, ln in params:
                    substring_same(gpu, lambda be: be.substring_by_char(col, s, ln), f"L={len(t)} {t[:6]!r} start={s} length={ln}")


def expand_by_char(small, idx, col):
    """The oracle's by_char result on the distinct values (valid rows only), expanded to rows idx (null rows: empty)."""
    vals = [bytes(small.data[int(small.offsets[j]): int(small.offsets[j + 1])]) for j in range(small.length)]
    m = col.nulls.valid_mask()
    return bytes_column([vals[j] if ok else b"" for j, ok in zip(idx, m)], col.offsets.dtype, *nulls_unsliced(col))


@pytest.mark.gpu
def test_by_char_long_rounds(gpu):
    """More than 1.2 x one round of k_char_long (SMs x 16 CTAs x 8 warps, one row per warp) long rows, with null rows of
    700 bytes among them (empty, never queued); i32 and i64 offsets, plain and sliced."""
    sms = gpu.lib.acu_device_sm_count(gpu.h)
    round_rows = sms * CHAR_LONG_CTAS_PER_SM * CHAR_LONG_WARPS_PER_CTA
    rng = np.random.default_rng(128)
    longs = [fill(int(rng.integers(513, 640)), w, rng).encode() for w in [(1,), (2,), (3,), (4,), (1, 2, 3, 4)] * 5]
    shorts = [b"", "é".encode(), b"ab", fill(512, (1, 2, 3, 4), rng).encode(), fill(40, (3, 1), rng).encode()]
    distinct = longs + shorts
    n_long = int(1.2 * round_rows) + 101
    n = n_long + n_long // 3 + n_long // 10
    kind = rng.permutation(np.concatenate([np.zeros(n_long, int), np.ones(n_long // 3, int), np.full(n_long // 10, 2)]))
    idx = np.where(kind == 0, rng.integers(0, len(longs), n), rng.integers(len(longs), len(distinct), n))
    valid = kind != 2
    garbage = b"N" * 700
    chunks = [distinct[j] if ok else garbage for j, ok in zip(idx, valid)]
    lens = np.array([len(c) for c in chunks], dtype=np.int64)
    data = np.frombuffer(b"".join(chunks), dtype=np.uint8).copy()
    assert int(((lens > LONG_ROW) & valid).sum()) == n_long > 1.2 * round_rows
    assert int(((lens > LONG_ROW) & ~valid).sum()) > 0
    assert (n + 7) // 8 >= sms * CHAR_LONG_CTAS_PER_SM  # k_char_long's grid is full, so a second round is needed
    small_col = bytes_col(distinct, np.int64)
    for dtype in (np.int32, np.int64):
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(dtype)
        full = Utf8Column(offs, data, nulls_of(valid))
        for col, sel in ((full, idx), (sliced(full, 3, n - 5), idx[3:n - 2])):
            for s, ln in [(0, None), (1, 2**64 - 1), (40, 300), (-100, None), (-37, 33), (513, None)]:
                exp = expand_by_char(SUBSTRING_ORACLE.substring_by_char(small_col, s, ln), sel, col)
                got = gpu.substring_by_char(col, s, ln)
                assert_substring(got, exp, f"by_char rounds {np.dtype(dtype).name} n={col.length} start={s} length={ln}")


# ---- C. the copy engine's staging limit -----------------------------------------------------------------------------------
def cta_rows(total, rng, mode="spread"):
    """BY_ROWS row lengths summing to total: spread (varied, some empty), empty, or one row holding everything."""
    if mode == "one":
        lens = np.zeros(BY_ROWS, np.int64)
        lens[int(rng.integers(1, BY_ROWS - 1))] = total
        return lens
    if total == 0:
        return np.zeros(BY_ROWS, np.int64)
    return rng.multinomial(total, rng.dirichlet(np.full(BY_ROWS, 0.7))).astype(np.int64)


STAGED_PAIRS = [(0, BY_STAGE_CAP), (0, BY_STAGE_CAP + 1), (1, BY_STAGE_CAP), (1, BY_STAGE_CAP + 1), (15, BY_STAGE_CAP),
                (15, BY_STAGE_CAP + 1)]
PARTIAL_TAILS = [(0, BY_STAGE_CAP - 15), (15, BY_STAGE_CAP - 1), (1, BY_STAGE_CAP - 1)]  # staged, last chunk of 1 / 15 bytes


def engine_plan(d, rng, extras=True):
    """CTA totals that put every target (lead, span) on a CTA when out_data is d bytes past a 16-B boundary: a CTA's span is
    its bytes plus its lead, and the next CTA's lead is that span mod 16, so small filler CTAs set the leads in between.
    CTA 0 is a full staged buffer at lead d. Returns the row lengths."""
    targets = [(d, BY_STAGE_CAP)] + STAGED_PAIRS + (PARTIAL_TAILS + ["empty", "one"] if extras else ["empty"])
    totals, modes, lead = [], [], d
    for tg in targets:
        if tg in ("empty", "one"):
            t = 60_000 if tg == "one" else 0
            totals.append(t), modes.append(tg if tg == "one" else "spread")
            lead = (lead + t) % 16
            continue
        want, span = tg
        if lead != want:
            t = (want - lead) % 16 + 16 * int(rng.integers(30, 60))
            totals.append(t), modes.append("spread")
            lead = want
        totals.append(span - want), modes.append("spread")
        lead = span % 16
    rows = [cta_rows(t, rng, m) for t, m in zip(totals, modes)]
    rows.append(rng.integers(0, 30, 777))  # a partial last CTA
    return np.concatenate(rows)


def check_engine_placement(lens, d, extras=True):
    """The (lead, span, staged) of every CTA from the actual row lengths, and the placements the plan promised."""
    n = len(lens)
    starts = np.arange(0, n, BY_ROWS)
    totals = np.add.reduceat(lens, starts)
    begins = np.concatenate([[0], np.cumsum(totals)[:-1]])
    leads = (d + begins) % 16
    spans = totals + leads
    got = set(zip(leads.tolist(), spans.tolist()))
    assert leads[0] == d and spans[0] == BY_STAGE_CAP
    for tg in STAGED_PAIRS + (PARTIAL_TAILS if extras else []):
        assert tg in got, tg
    staged = spans <= BY_STAGE_CAP
    assert staged.any() and (~staged).any()
    if extras:
        assert {int(s % 16) for s, st in zip(spans, staged) if st} >= {1, 15}  # partial last chunks of 1 and 15 bytes
        nonempty = totals > 0
        assert any(not nonempty[k] and nonempty[:k].any() and nonempty[k + 1:].any() for k in range(len(totals)))
        per_cta = [lens[s:s + BY_ROWS] for s in starts]
        assert any((c > 0).sum() == 1 and c.sum() > BY_STAGE_CAP for c in per_cta)
    return int(lens.sum())


def run_two_phase(gpu, call, n, ob, d, expected_total):
    """Both phases of an offsets-and-copy entry point through ctypes: the sizing call (no data buffer), then the copy into
    an output d bytes past the start of a sentinel-filled allocation, with a capacity of exactly the total. The bytes
    before the output and after the total must keep the sentinel."""
    lib, h = gpu.lib, gpu.h
    owned = []
    try:
        d_off = gpu.malloc((n + 1) * ob + 16)
        owned.append(d_off)
        out = gpu.alloc_out(0, n)
        owned += [out.values, out.validity]
        total = C.c_int64(-1)
        gpu.check(call(d_off, None, 0, C.byref(total), C.byref(out)))
        assert total.value == expected_total
        size = d + total.value + 64
        base = gpu.malloc(size)
        owned.append(base)
        assert base % 16 == 0
        gpu.check(lib.acu_memset(h, base, SENTINEL, size))
        gpu.check(lib.acu_memset(h, d_off, 0xEE, (n + 1) * ob))
        again = C.c_int64(-1)
        gpu.check(call(d_off, base + d, total.value, C.byref(again), C.byref(out)))
        assert again.value == total.value
        raw = gpu.d2h(base, size)
        assert (raw[:d] == SENTINEL).all(), "bytes before the output were written"
        assert (raw[d + total.value:] == SENTINEL).all(), "bytes after the output were written"
        offs = gpu.d2h(d_off, (n + 1) * ob, np.int32 if ob == 4 else np.int64)
        validity = gpu.d2h(out.validity, bitmap_bytes(n)) if out.has_validity else None
        nulls = HostArray(abi.U8, np.zeros(0, np.uint8), n, validity, 0, 0, out.null_count if out.has_validity else 0)
        return Utf8Column(offs, raw[d:d + total.value].copy(), nulls)
    finally:
        for p in owned:
            gpu.free(p)


def binary_col(lens, dtype, rng, null_p=0.02):
    offs = np.concatenate([[0], np.cumsum(lens)]).astype(dtype)
    data = rng.integers(0, 256, int(offs[-1]) + 16, dtype=np.uint8)
    return Utf8Column(offs, data, nulls_of(rng.random(len(lens)) >= null_p))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.int32, np.int64])
@pytest.mark.parametrize("d", [0, 1, 15])
def test_engine_staging_substring(gpu, dtype, d):
    """substring(Binary, 0, None) copies every row: CTAs at spans 49152 (staged, buffer exactly full) and 49153 (direct)
    with leads 0 / 1 / 15, partial last chunks of 1 and 15 bytes, a CTA of empty rows, a CTA of one 60 KB row."""
    rng = np.random.default_rng(100 * d + np.dtype(dtype).itemsize)
    lens = engine_plan(d, rng)
    total = check_engine_placement(lens, d)
    col = binary_col(lens, dtype, rng)
    ob, lib, h = np.dtype(dtype).itemsize, gpu.lib, gpu.h
    owned = []
    try:
        dc = gpu._upload_bytes_col(col, owned)
        got = run_two_phase(gpu, lambda oo, od, cap, tot, out: lib.acu_substring_bytes(h, ob, 0, 0, 0, 0, C.byref(dc), col.data.nbytes, oo, od,
                                                                                      cap, tot, out), col.length, ob, d, total)
    finally:
        for p in owned:
            gpu.free(p)
    assert_substring(got, SUBSTRING_ORACLE.substring(col, 0, None, is_utf8=False), f"substring d={d}")


def split_cols(lens, k, dtype, rng, max_seg=None):
    """k operands whose row lengths add up to lens (each segment 0..max_seg bytes when given)."""
    n = len(lens)
    if max_seg is None:
        cut = (rng.random(n) * (lens + 1)).astype(np.int64)
        parts = [cut, lens - cut]
    else:  # a row's bytes go to lens[i] random slots of k x max_seg
        assert lens.max() <= k * max_seg
        rank = rng.random((n, k * max_seg)).argsort(axis=1).argsort(axis=1)
        parts = list((rank < lens[:, None]).reshape(n, k, max_seg).sum(axis=2).T.astype(np.int64))
    return [binary_col(p, dtype, rng, null_p=0.01) for p in parts]


def fit_rows(lens, cap, rng):
    """lens with every row capped at `cap` bytes and the excess moved to other rows of the same CTA (CTA totals kept)."""
    out = lens.copy()
    for s in range(0, len(out), BY_ROWS):
        c = out[s:s + BY_ROWS]
        excess = int(np.maximum(c - cap, 0).sum())
        np.minimum(c, cap, out=c)
        while excess:
            room = np.flatnonzero(c < cap)
            pick = rng.choice(room, min(excess, len(room)), replace=False)
            c[pick] += 1
            excess -= len(pick)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.int32, np.int64])
@pytest.mark.parametrize("d", [0, 1, 15])
def test_engine_staging_concat(gpu, dtype, d):
    """concat_elements of two Binary columns at the same CTA placements as the substring test."""
    rng = np.random.default_rng(200 * d + np.dtype(dtype).itemsize)
    lens = engine_plan(d, rng)
    total = check_engine_placement(lens, d)
    l, r = split_cols(lens, 2, dtype, rng)
    ob, lib, h = np.dtype(dtype).itemsize, gpu.lib, gpu.h
    owned = []
    try:
        dl, dr = gpu._upload_bytes_col(l, owned), gpu._upload_bytes_col(r, owned)
        got = run_two_phase(gpu, lambda oo, od, cap, tot, out: lib.acu_concat_elements_bytes(h, ob, C.byref(dl), C.byref(dr), oo, od, cap, tot, out),
                            l.length, ob, d, total)
    finally:
        for p in owned:
            gpu.free(p)
    assert_concat(got, CONCAT_ORACLE.concat_elements(l, r, is_utf8=False), f"concat d={d}")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.int32, np.int64])
@pytest.mark.parametrize("d", [1, 15])
def test_engine_staging_concat_many(gpu, dtype, d):
    """concat_elements_utf8_many of 17 operands of 0..3 bytes a row: every row pushes many tiny segments, at the staged /
    direct pair placements."""
    rng = np.random.default_rng(300 * d + np.dtype(dtype).itemsize)
    lens = fit_rows(engine_plan(d, rng, extras=False), 17 * 3, rng)
    total = check_engine_placement(lens, d, extras=False)
    cols = split_cols(lens, 17, dtype, rng, max_seg=3)
    ob, lib, h = np.dtype(dtype).itemsize, gpu.lib, gpu.h
    owned = []
    try:
        arr = (abi.BytesArray * 17)(*[gpu._upload_bytes_col(c, owned) for c in cols])
        got = run_two_phase(gpu, lambda oo, od, cap, tot, out: lib.acu_concat_elements_bytes_many(h, ob, 17, arr, oo, od, cap, tot, out),
                            cols[0].length, ob, d, total)
    finally:
        for p in owned:
            gpu.free(p)
    assert_concat(got, CONCAT_ORACLE.concat_elements_utf8_many(cols), f"concat many d={d}")
