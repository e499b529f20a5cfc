"""CPU: the length / substring oracle (tests/oracle_substring.py) pinned against the reference's literal vectors
(tests/golden/substring_vectors.json: length.rs and substring.rs test tables), then, as a secondary cross-check only,
against Python slicing on ASCII and valid UTF-8 data."""
import numpy as np
import pytest

import acu

from oracle_substring import SubstringOracle, char_bounds, view_range
from substring_util import decode, golden_cases, golden_inputs, rand_items, run_case, values

ORACLE = SubstringOracle()
CASES = golden_cases()


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_oracle_golden(case):
    results = []
    for typ, utf8, col in golden_inputs(case):
        if "error" in case:
            with pytest.raises(acu.ArrowError) as e:
                run_case(ORACLE, case, col, utf8)
            assert case["error"] in str(e.value)
            continue
        got = run_case(ORACLE, case, col, utf8)
        if case["fn"] in ("length", "bit_length"):
            assert got.to_list() == case["expected"], typ
        elif case["kind"] == "view_matches":
            results.append(values(got))
        else:
            assert values(got) == decode(case["expected"]), typ
    if case["kind"] == "view_matches":
        assert results[0] == results[1]


def test_oracle_golden_count():
    assert len(CASES) == 158


def test_oracle_nulls_rules():
    """length clones the NullBuffer (present without nulls); substring drops it (from_unsliced_buffer)."""
    from substring_util import nulls_of
    col = acu.Utf8Column(np.array([0, 1, 3], dtype=np.int32), np.frombuffer(b"abc", dtype=np.uint8).copy(), nulls_of([True, True], force=True))
    assert ORACLE.length(col).validity is not None
    assert ORACLE.substring(col, 1).nulls.validity is None


def test_oracle_wrapping_panic():
    """start = 2^31 - 1 on i32 offsets: p0 + start wraps negative; Binary panics on the slice, Utf8 fails the boundary."""
    from substring_util import bytes_col
    col = bytes_col([b"ab", b"cd"], np.int32)
    with pytest.raises(acu.ArrowError) as e:
        ORACLE.substring(col, 2**31 - 1, None, is_utf8=False)
    assert e.value.status == 8 and e.value.index == 1
    with pytest.raises(acu.ArrowError) as e:
        ORACLE.substring(col, 2**31 - 1, None, is_utf8=True)
    assert e.value.status == 2 and str(e.value) == f"Compute error: The offset {2**64 - 2**31 + 1} is at an invalid utf-8 boundary."


# ---- secondary cross-check: Python slicing --------------------------------------------------------------------------
def py_byte_substring(b, start, length):
    L = len(b)
    s = min(start, L) if start > 0 else 0 if start == 0 else max(L + start, 0)
    e = L if length is None else min(s + length, L)
    return b[s:e]


def py_char_substring(b, start, length):
    t = b.decode()
    s = t[start:] if start >= 0 else t[max(len(t) + start, 0):]
    return (s if length is None else s[:length]).encode()


@pytest.mark.parametrize("seed", range(4))
def test_cross_check_python_slicing(seed):
    rng = np.random.default_rng(seed)
    from substring_util import bytes_col
    ascii_items = [None if rng.random() < 0.1 else bytes(rng.integers(97, 123, int(rng.integers(0, 20))).astype(np.uint8)) for _ in range(200)]
    utf8_items = rand_items(rng, 200, 12, 0.1)
    for start in (-30, -5, -1, 0, 1, 3, 30):
        for length in (None, 0, 1, 4, 100):
            got = values(ORACLE.substring(bytes_col(ascii_items, np.int64), start, length))
            assert got == [None if x is None else py_byte_substring(x, start, length) for x in ascii_items]
            got = values(ORACLE.substring_by_char(bytes_col(utf8_items, np.int32), start, length))
            assert got == [None if x is None else py_char_substring(x, start, length) for x in utf8_items]


def test_range_helpers():
    assert view_range(5, -100, 4) == (0, 4)
    assert view_range(5, 2, 2**64 - 1) == (2, 1)  # length as i64 = -1: the slice panics
    assert char_bounds("Γ ⊢x:T".encode(), -4, 2) == (len("Γ ".encode()), len("Γ ⊢x".encode()))
