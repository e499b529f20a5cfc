"""like / nlike / ilike / nilike / contains / starts_with / ends_with / eq_ignore_ascii_case on the device vs the oracle
(tests/oracle_like.py), bit for bit: value bits at every slot (including under nulls), validity, null_count, NullBuffer
presence, and error status / text / row. Reference: arrow-string/src/like.rs, predicate.rs, binary_like.rs. The oracle
itself is pinned by the reference's literal vectors (tests/test_oracle_like.py)."""
import numpy as np
import pytest

import acu
from acu import HostArray, Utf8Column, ViewColumn
from acu import _abi as abi

from like_util import column, golden_cases, rand_utf8, run, run_form
from oracle_like import LikeOracle
from test_gpu_parity import assert_same, expect_same_error

pytestmark = pytest.mark.gpu

ORACLE = LikeOracle()
ROW_CASES = [c for c in golden_cases() if "op" in c]
ALL_OPS = list(range(8))
STRING_TYPES = ["utf8", "large_utf8", "utf8_view"]
SIZES = [0, 1, 31, 33, 64, 129, 1000, 4097]
# haystack scalars: 1-4 byte UTF-8, the simple folds that reach ASCII (K U+212A, ſ U+017F) and one that does not (ı U+0131)
HAY = ["a", "b", "c", "A", "B", "k", "K", "K", "s", "S", "ſ", "ı", "i", "é", "€", "😈", "%", "_", "\\"]
PAT = ["a", "b", "c", "A", "k", "s", "i", "%", "%", "_", "\\", "é", "😈"]


def same(gpu, op, typ, l, r, what):
    got, exp = expect_same_error(gpu, ORACLE, lambda be: run(be, op, typ, l, r))
    if got is not None:
        assert_same(got, exp, what)


@pytest.mark.parametrize("case", ROW_CASES, ids=[c["id"] for c in ROW_CASES])
def test_like_golden(gpu, case):
    for form in case["forms"]:
        got, exp = run_form(gpu, case, form), run_form(ORACLE, case, form)
        assert_same(got, exp, f"{case['id']} on {form}")
        assert got.to_list() == case["expected"]


def sliced(col, off, n):
    """Array::slice of a Utf8Column: offsets start mid-buffer (offsets[0] != 0)."""
    return Utf8Column(col.offsets[off:off + n + 1], col.data, col.nulls.slice(off, n))


def view_garbage(rng):
    """Inline views of valid UTF-8 (lengths <= 12) to leave under null slots."""
    g = np.zeros((5, 16), dtype=np.uint8)
    for k, s in enumerate(["K", "kſ", "ıK", "abc", "😈_%"]):
        b = s.encode()
        g[k, 0] = len(b)
        g[k, 4:4 + len(b)] = np.frombuffer(b, dtype=np.uint8)
    return g


@pytest.mark.parametrize("op", ALL_OPS)
def test_like_fuzz(gpu, op):
    rng = np.random.default_rng(4100 + op)
    garbage = view_garbage(rng)
    for n in SIZES:
        for null_p in (None, 0.1, 0.5):
            hay = rand_utf8(rng, n + 3, HAY, 16, null_p)
            pats = rand_utf8(rng, n + 3, PAT, 5, null_p)
            for typ in STRING_TYPES:
                if typ == "utf8_view":
                    l = ViewColumn.from_values([None if x is None else x.encode() for x in hay[:n]], 48, garbage_under_nulls=garbage)
                    r = column(typ, pats[:n])
                else:
                    l, r = sliced(column(typ, hay), 3, n), sliced(column(typ, pats), 3, n)
                same(gpu, op, typ, l, r, f"array/array n={n} op={op} {typ} nulls={null_p}")
                if n:
                    for p in ["", "%", "ab%", "%ab", "%a%", "a_c", "%a_c%", "_%_", "%K%", "k%", "%s", "\\%%", "a\\", "%😈_é%", "%__"]:
                        same(gpu, op, typ, l, column(typ, [p], scalar=True), f"array/scalar n={n} op={op} {typ} {p!r}")
                    same(gpu, op, typ, l, column(typ, [None], scalar=True), f"array/null scalar n={n} op={op} {typ}")
                    for h in ["abc", None, "Kabcſ"]:
                        same(gpu, op, typ, column(typ, [h], scalar=True), r, f"scalar/array n={n} op={op} {typ} {h!r}")


def test_like_multi_round_grid(gpu):
    """Sizes that make k_like run at least two grid-stride rounds (grid = SMs x 16 CTAs of 8 warps, 4 x 32 rows per warp)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 2 * sms * 16 * 8 * 4 * 32 + 4097
    rng = np.random.default_rng(11)
    lens = rng.integers(0, 13, n)
    offs = np.zeros(n + 1, dtype=np.int32)
    offs[1:] = np.cumsum(lens)
    data = np.frombuffer(b"abcK", dtype=np.uint8)[rng.integers(0, 4, int(offs[-1]))].copy()
    mask = rng.random(n) >= 0.05
    nulls = HostArray(abi.U8, np.zeros(0, np.uint8), n, acu.pack_bits(mask), 0, 0, int(n - mask.sum()))
    col = Utf8Column(offs, np.concatenate([data, np.zeros(16, np.uint8)]), nulls)
    views = np.zeros((n, 16), dtype=np.uint8)
    views[:, :4] = lens.astype(np.uint32).view(np.uint8).reshape(n, 4)
    for k in range(12):
        sel = lens > k
        views[sel, 4 + k] = data[offs[:-1][sel] + k]
    vcol = ViewColumn(views, [], nulls)
    for op, pat in [(abi.STARTS_WITH, "ab"), (abi.CONTAINS, "bK"), (abi.LIKE, "%c")]:
        sc = column("utf8", [pat], scalar=True)
        assert_same(gpu.like_bytes(op, col, sc), ORACLE.like_bytes(op, col, sc), f"multi-round utf8 op={op}")
        vs = column("utf8_view", [pat], scalar=True)
        assert_same(gpu.like_view(op, vcol, vs), ORACLE.like_view(op, vcol, vs), f"multi-round view op={op}")


def test_like_view_is_ascii_quirk(gpu):
    """Valid slots all ASCII: ilike's IEqAscii / IStartsWithAscii / IEndsWithAscii run at the null slots too."""
    rng = np.random.default_rng(5)
    garbage = view_garbage(rng)
    for valid_non_ascii in (False, True):
        items = [None if i % 3 == 1 else ("K" if valid_non_ascii and i == 6 else "kab") for i in range(70)]
        items += ["k" * 20, None]
        v = ViewColumn.from_values([None if x is None else x.encode() for x in items], 64, garbage_under_nulls=garbage)
        for op in (abi.ILIKE, abi.NILIKE):
            for p in ["k", "K", "kab", "k%", "%k", "%s", "ab%", "%k%", "k_b", "%"]:
                same(gpu, op, "utf8_view", v, column("utf8_view", [p], scalar=True), f"quirk {p!r} non_ascii={valid_non_ascii}")


def test_like_binary_non_utf8(gpu):
    rng = np.random.default_rng(6)
    for typ in ["binary", "large_binary", "binary_view"]:
        for n in [1, 100, 3000]:
            items = [None if rng.random() < 0.1 else bytes(rng.integers(0, 256, int(rng.integers(0, 20)), dtype=np.uint8))
                     for _ in range(n)]
            needles = [bytes(rng.integers(0, 256, int(rng.integers(0, 3)), dtype=np.uint8)) for _ in range(n)]
            l, r = column(typ, items), column(typ, needles)
            for op in (abi.CONTAINS, abi.STARTS_WITH, abi.ENDS_WITH):
                same(gpu, op, typ, l, r, f"{typ} array/array n={n} op={op}")
                for nd in [b"", b"\xff", b"\x00\xfe", items[0] or b"\x80"]:
                    same(gpu, op, typ, l, column(typ, [nd], scalar=True), f"{typ} array/scalar n={n} op={op} {nd!r}")
            for op in (abi.LIKE, abi.NLIKE, abi.ILIKE, abi.NILIKE, abi.EQ_IGNORE_ASCII_CASE):
                same(gpu, op, typ, l, column(typ, [b"a"], scalar=True), f"{typ} invalid op={op}")


def test_like_long_rows(gpu):
    """A few rows of 1e5+ bytes among short ones: the warp-per-row kernel (k_like_long)."""
    big = "ab" * 50000
    items = ["x", big + "K", None, big + "a😈c" + big, "abc", big[:-1] + "ſ", big, "K" * 40000]
    mid = big[5:400]
    for typ in ["utf8", "utf8_view"]:
        l = column(typ, items, block=1 << 20)
        for op in ALL_OPS:
            for p in ["%bK", "%a_c%", "%b", "ab%", "%abc%", "%K%", "%S", big, "%" + mid + "%", "a%b%a%😈%", "%k", "%" + mid + "_%b"]:
                same(gpu, op, typ, l, column(typ, [p], scalar=True), f"long {typ} op={op} {p[:20]!r}")
            same(gpu, op, typ, l, column(typ, [big + "k", "%a%", None, "%😈_" + big, "%", "ab%ſ", big, "%kk"]),
                 f"long {typ} per-row op={op}")
            same(gpu, op, typ, column(typ, [big + "K"], scalar=True), column(typ, ["%b_", big + "k", "%"]), f"long {typ} scalar hay op={op}")


def test_like_errors(gpu):
    for typ in STRING_TYPES:
        same(gpu, abi.LIKE, typ, column(typ, ["a", "b"]), column(typ, ["a"]), "length mismatch")
        same(gpu, abi.CONTAINS, typ, column(typ, []), column(typ, ["a"]), "length mismatch 0 vs 1")
        for op in (abi.ILIKE, abi.NILIKE):
            same(gpu, op, typ, column(typ, ["a"]), column(typ, ["é%"], scalar=True), "non-ASCII scalar ilike pattern")
            same(gpu, op, typ, column(typ, []), column(typ, ["é%"], scalar=True), "non-ASCII scalar ilike pattern, empty")
            same(gpu, op, typ, column(typ, ["a", None, "c", "d", "e"]), column(typ, ["a", "é", None, "ü", "ö"]), "non-ASCII per-row")
            same(gpu, op, typ, column(typ, [None], scalar=True), column(typ, ["é", "ü"]), "non-ASCII per-row, null haystack")
    for typ in ["binary", "large_binary", "binary_view"]:
        same(gpu, abi.LIKE, typ, column(typ, ["a", "b"]), column(typ, ["a"]), "binary length mismatch before the op check")
