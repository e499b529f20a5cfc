"""length / bit_length / substring / substring_by_char on the device vs the oracle (tests/oracle_substring.py), bit for
bit: offsets, value bytes, validity bits, NullBuffer presence, null_count, and error status / text / row. View results
are compared logically, and bit-exactly for null views, inline views and the 4-byte prefix of long views (the device keeps
long results in the input's buffers, the reference's builder copies them; include/arrow_cuda.h). Reference:
arrow-string/src/length.rs, substring.rs."""
import numpy as np
import pytest

import acu
from acu import FixedSizeBinaryColumn, HostArray, Utf8Column, ViewColumn, column_value

from oracle_substring import SubstringOracle
from substring_util import (bytes_col, decode, golden_cases, golden_inputs, nulls_of, rand_items, run_case, sliced, values)
from test_gpu_parity import assert_same, expect_same_error

pytestmark = pytest.mark.gpu

ORACLE = SubstringOracle()
CASES = golden_cases()
STARTS = [-2**63, -2**31 - 1, -2**31, -7, -1, 0, 1, 2, 5, 2**31 - 1, 2**31, 2**32 + 1]
LENGTHS = [None, 0, 1, 3, 2**31 - 1, 2**31, 2**32 + 1, 2**63, 2**64 - 1]


def assert_nulls(g, e, what):
    assert (g.validity is None) == (e.validity is None), f"{what}: NullBuffer presence"
    if e.validity is not None:
        assert np.array_equal(g.valid_mask(), e.valid_mask()), f"{what}: validity bits"
        assert g.null_count == e.null_count, f"{what}: null_count {g.null_count} != {e.null_count}"


def assert_result(got, exp, what):
    if isinstance(exp, HostArray):
        assert_same(got, exp, what)
    elif isinstance(exp, Utf8Column):
        assert np.array_equal(got.offsets, exp.offsets), f"{what}: offsets"
        assert bytes(got.data) == bytes(exp.data), f"{what}: bytes"
        assert_nulls(got.nulls, exp.nulls, what)
    elif isinstance(exp, FixedSizeBinaryColumn):
        assert got.values.shape == exp.values.shape and np.array_equal(got.values, exp.values), f"{what}: values"
        assert_nulls(got.nulls, exp.nulls, what)
    else:
        assert_nulls(got.nulls, exp.nulls, what)
        m = exp.nulls.valid_mask()
        for i in range(exp.length):
            gv, ev = got.views[i], exp.views[i]
            if not m[i]:
                assert not gv.any(), f"{what}: null view {i} not zeroed"
                continue
            assert column_value(got, i) == column_value(exp, i), f"{what}: row {i}"
            if ev[0] <= 12 and not ev[1:4].any():
                assert np.array_equal(gv, ev), f"{what}: inline view {i}"
            else:
                assert np.array_equal(gv[:8], ev[:8]), f"{what}: length / prefix of view {i}"


def same(gpu, fn, what):
    got, exp = expect_same_error(gpu, ORACLE, fn)
    if exp is not None:
        assert_result(got, exp, what)
    return exp


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_substring_golden(gpu, case):
    for typ, utf8, col in golden_inputs(case):
        exp = same(gpu, lambda be: run_case(be, case, col, utf8), f"{case['id']} {typ}")
        if exp is None:
            continue
        if case["fn"] in ("length", "bit_length"):
            assert run_case(gpu, case, col, utf8).to_list() == case["expected"]
        elif "expected" in case:
            assert values(run_case(gpu, case, col, utf8)) == decode(case["expected"])


@pytest.mark.parametrize("dtype", [np.int32, np.int64])
@pytest.mark.parametrize("utf8", [True, False])
def test_substring_bytes_fuzz(gpu, dtype, utf8):
    """Every start / length of the extreme grid, wrapping panics and boundary errors included, on plain and sliced
    columns with bytes under the null slots."""
    rng = np.random.default_rng(7 + (dtype == np.int64) + 2 * utf8)
    items = rand_items(rng, 700, 9, 0.15)
    full = bytes_col(items, dtype, garbage="é".encode())
    for col in (full, sliced(full, 13, 600)):
        for s in STARTS:
            for ln in LENGTHS:
                same(gpu, lambda be: be.substring(col, s, ln, is_utf8=utf8), f"start={s} length={ln}")


def test_substring_bytes_panic_and_boundary_rows(gpu):
    """The lowest failing row wins; every boundary error precedes every panic; a boundary error under a null slot
    counts for Utf8 (the rule runs at every slot) but not for Utf8View (null slots are skipped)."""
    items = [b"abc", None, b"xyz", "dé".encode()]
    col = bytes_col(items, np.int32, garbage="é".encode())  # the null slot holds 0xC3 0xA9
    exp = same(gpu, lambda be: be.substring(col, 1, 1), "boundary under a null slot")
    assert exp is None
    with pytest.raises(acu.ArrowError) as e:
        gpu.substring(col, 1, 1)
    assert e.value.index == 1 and "invalid utf-8 boundary" in str(e.value)
    view = ViewColumn.from_values([b"abc", None, b"xyz", b"d"], garbage_under_nulls=[np.array([2, 0xC3, 0xA9] + [0] * 13, np.uint8)])
    same(gpu, lambda be: be.substring(view, 1, 1), "view null slot skipped")
    for s, ln in [(2**31 - 1, None), (1, 2**31 - 1), (-1, 2**32 - 1), (0, 2**64 - 1)]:
        for utf8 in (True, False):
            same(gpu, lambda be: be.substring(bytes_col([b"ab", b"", b"cd", b"e"], np.int32), s, ln, is_utf8=utf8), f"{s} {ln}")


def test_substring_boundary_at_0xbf(gpu):
    """0xBF is the last continuation byte: an offset on it is not a char boundary, for Utf8 (absolute offset) and Utf8View
    (relative), at either end of the range; by_char steps over it."""
    items = ["aÿb".encode(), "¿?".encode(), "x\uffffy".encode()]
    col, view = bytes_col(items, np.int32), ViewColumn.from_values(items)
    for s, ln in [(2, None), (1, 1), (-2, None), (0, 2), (2, 1)]:
        for c in (col, view):
            exp = same(gpu, lambda be: be.substring(c, s, ln), f"0xBF {s} {ln}")
            if (s, ln) in [(2, None), (0, 2)]:
                assert exp is None  # an error on both sides
        same(gpu, lambda be: be.substring_by_char(col, s, ln), f"0xBF by_char {s} {ln}")


def test_substring_by_char_fuzz(gpu):
    rng = np.random.default_rng(21)
    for dtype in (np.int32, np.int64):
        items = rand_items(rng, 500, 10, 0.2)
        items[::37] = [rand_items(rng, 1, 1500, 0)[0] * 2 for _ in items[::37]]  # rows past the warp threshold
        full = bytes_col(items, dtype, garbage=b"\xff\xfe")
        for col in (full, sliced(full, 5, 480)):
            for s in STARTS + [-600, 600]:
                for ln in [None, 0, 1, 3, 700, 2**63, 2**64 - 1]:
                    same(gpu, lambda be: be.substring_by_char(col, s, ln), f"by_char start={s} length={ln}")


@pytest.mark.parametrize("utf8", [True, False])
def test_substring_view_fuzz(gpu, utf8):
    rng = np.random.default_rng(33 + utf8)
    items = rand_items(rng, 600, 12, 0.15)
    garbage = [np.frombuffer(np.array([0xFFFFFFF0, 1, 2, 3], dtype=np.uint32).tobytes(), dtype=np.uint8)]
    col = ViewColumn.from_values(items, block_size=256, garbage_under_nulls=garbage)  # several data buffers
    assert len(col.buffers) > 4
    for s in STARTS + [-13, 13]:
        for ln in LENGTHS + [12, 13]:
            same(gpu, lambda be: be.substring(col, s, ln, is_utf8=utf8), f"view start={s} length={ln}")


def test_length_fuzz(gpu):
    rng = np.random.default_rng(44)
    items = rand_items(rng, 3000, 20, 0.2)
    garbage = [np.frombuffer(np.array([0xDEADBEEF, 5, 6, 7], dtype=np.uint32).tobytes(), dtype=np.uint8)]
    cols = [bytes_col(items, np.int32), bytes_col(items, np.int64), sliced(bytes_col(items, np.int32), 3, 2900),
            ViewColumn.from_values(items, garbage_under_nulls=garbage),
            FixedSizeBinaryColumn.from_values([None if x is None else b"abcdefg" for x in items], 7)]
    # wrapping lengths: offsets that are not monotonic
    cols.append(Utf8Column(np.array([0, 2**31 - 1, -2**31, 5], dtype=np.int32), np.zeros(8, np.uint8), nulls_of([True] * 3, force=True)))
    for col in cols:
        for fn in ("length", "bit_length"):
            same(gpu, lambda be: getattr(be, fn)(col), f"{fn} {type(col).__name__}")


def test_grid_rounds(gpu):
    """Sizes past one grid-stride round of the length (SMs x 8 CTAs x 256 threads x 4 rows), view and by_char kernels
    (SMs x 8 x 256 rows); not a multiple of 64."""
    sms = gpu.lib.acu_device_sm_count(gpu.h)
    rng = np.random.default_rng(55)
    n = int(sms * 8 * 256 * 1.3) + 37
    items = rand_items(rng, n, 4, 0.1)
    v = ViewColumn.from_values(items, block_size=1 << 16)
    same(gpu, lambda be: be.substring(v, 1, 13), "view rounds")
    b = bytes_col(items, np.int32)
    same(gpu, lambda be: be.substring_by_char(b, -2, 1), "by_char rounds")
    same(gpu, lambda be: be.substring(b, 1, 2, is_utf8=False), "bytes")
    nl = int(sms * 8 * 256 * 4 * 1.2) + 37
    offs = np.cumsum(np.concatenate([[0], rng.integers(0, 5, nl)])).astype(np.int64)
    big = Utf8Column(offs, np.zeros(int(offs[-1]), np.uint8), nulls_of(rng.random(nl) > 0.1))
    same(gpu, lambda be: be.length(big), "length rounds")


def test_empty_and_all_null(gpu):
    for dtype in (np.int32, np.int64):
        for items in ([], [None] * 70):
            col = bytes_col(items, dtype, garbage=b"zz")
            for fn in (lambda be: be.substring(col, 1, 1), lambda be: be.substring_by_char(col, 1, 1), lambda be: be.length(col)):
                same(gpu, fn, f"{len(items)} rows")
    for items in ([], [None] * 70):
        v = ViewColumn.from_values(items)
        same(gpu, lambda be: be.substring(v, 0, 2), "view")
        same(gpu, lambda be: be.length(v), "view length")


def test_fixed_size_binary(gpu):
    for width in (0, 1, 5, 16):
        for items in ([b"a" * width] * 3, [None, b"b" * width, None], []):
            col = FixedSizeBinaryColumn.from_values(items, width)
            for s in (-2**63, -3, -1, 0, 1, 2, 100):
                for ln in (None, 0, 1, 2**64 - 1):
                    same(gpu, lambda be: be.substring(col, s, ln), f"fsb w={width} {s} {ln}")
            same(gpu, lambda be: be.length(col), "fsb length")
            same(gpu, lambda be: be.bit_length(col), "fsb bit_length")
    # new_len == 0 without nulls: an all-valid NullBuffer
    got = gpu.substring(FixedSizeBinaryColumn.from_values([b"abc"] * 3, 3), 3, None)
    assert got.nulls.validity is not None and got.nulls.null_count == 0 and got.values.shape == (3, 0)


def test_two_phase_capacity(gpu):
    col = bytes_col([b"hello", b"world", None], np.int32)
    same(gpu, lambda be: be.substring(col, 1, 3, data_capacity=100), "larger capacity")
    same(gpu, lambda be: be.substring(col, 1, 3, data_capacity=5), "too small")
    same(gpu, lambda be: be.substring_by_char(col, 1, 3, data_capacity=0), "too small by char")
