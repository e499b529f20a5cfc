"""CPU: the concat_elements oracle (tests/oracle_concat_elements.py) pinned against the reference's literal vectors
(tests/golden/concat_elements_vectors.json: the concat_elements.rs test module), its null / layout / overflow rules, and,
as a secondary cross-check only, pyarrow's binary_join_element_wise on the valid rows."""
import numpy as np
import pytest

import acu
from acu import FixedSizeBinaryColumn, HostArray, ViewColumn
from acu import _abi as abi

from concat_util import column, golden_cases, run_case
from oracle_concat_elements import ConcatElementsOracle, I32_MAX, first_overflow_row
from substring_util import bytes_col, decode, nulls_of, rand_items, values

ORACLE = ConcatElementsOracle()
CASES = golden_cases()


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_oracle_golden(case):
    if "error" in case:
        with pytest.raises(acu.ArrowError) as e:
            run_case(ORACLE, case)
        assert str(e.value) == case["error"] and e.value.status == case["status"]
        return
    assert values(run_case(ORACLE, case)) == decode(case["expected"])


def test_oracle_golden_count():
    assert len(CASES) == 28


def test_bytes_under_nulls_and_union():
    l = bytes_col([b"ab", None, b"c"], np.int32, garbage=b"XY")
    r = bytes_col([b"1", b"2", None], np.int32, garbage=b"Z")
    out = ORACLE.concat_elements(l, r)
    assert list(out.offsets) == [0, 3, 6, 8] and bytes(out.data) == b"ab1XY2cZ"
    assert out.nulls.null_count == 2 and list(out.nulls.valid_mask()) == [True, False, False]
    # a NullBuffer without nulls on both sides: the union is None
    l2, r2 = bytes_col([b"a"], np.int64), bytes_col([b"b"], np.int64)
    l2.nulls, r2.nulls = nulls_of([True], force=True), nulls_of([True], force=True)
    assert ORACLE.concat_elements(l2, r2).nulls.validity is None


def test_view_layout():
    l = ViewColumn.from_values([b"abc", b"", None, b"x" * 12, b"ab"])
    r = ViewColumn.from_values([b"defghijklm", b"", b"q", b"", b"cdefghijklmno"])
    out = ORACLE.concat_elements(l, r, is_utf8=False)
    v = out.views
    assert bytes(v[0]) == (13).to_bytes(4, "little") + b"abcd" + bytes(4) + bytes(4)          # 13 bytes: long, offset 0
    assert bytes(v[1]) == bytes(16)                                                          # empty inline view
    assert bytes(v[2]) == bytes(16)                                                          # null
    assert bytes(v[3]) == (12).to_bytes(4, "little") + b"x" * 12                             # exactly 12: inline
    assert bytes(v[4]) == (15).to_bytes(4, "little") + b"abcd" + bytes(4) + (13).to_bytes(4, "little")  # prefix spans both
    assert len(out.buffers) == 1 and bytes(out.buffers[0]) == b"abcdefghijklm" + b"abcdefghijklmno"
    assert out.nulls.null_count == 1
    inline = ORACLE.concat_elements(ViewColumn.from_values([b"a"]), ViewColumn.from_values([b"b"]))
    assert inline.buffers == []


def test_fsb_rules():
    l = FixedSizeBinaryColumn.from_values([b"ab", None], 2)
    r = FixedSizeBinaryColumn.from_values([b"c", b"d"], 1)
    out = ORACLE.concat_elements(l, r)
    assert out.values.tobytes() == b"abc" + bytes(3) and out.nulls.null_count == 1
    big_l = FixedSizeBinaryColumn(np.zeros((0, 2**31 - 1), np.uint8), nulls_of([]))
    big_r = FixedSizeBinaryColumn(np.zeros((0, 2), np.uint8), nulls_of([]))
    with pytest.raises(acu.ArrowError) as e:
        ORACLE.concat_elements(big_l, big_r)
    assert e.value.status == abi.ERR_PANIC_OUT_OF_BOUNDS and str(e.value) == "value length (-2147483647) of the array must >= 0"


def test_unwrap_row_rule():
    assert first_overflow_row([I32_MAX]) is None
    assert first_overflow_row([5, I32_MAX - 5, 1, 0]) == 2
    assert first_overflow_row([2**30, 2**30 - 1, 0, 1]) == 3


def test_dyn_errors():
    with pytest.raises(acu.ArrowError) as e:
        ORACLE.concat_elements(ViewColumn.from_values([b"a"]), bytes_col([b"a"], np.int32))
    assert str(e.value) == "Compute error: Cannot concat arrays of different types: Utf8View != Utf8"
    a = HostArray.from_list(abi.I32, [1, 2])
    with pytest.raises(acu.ArrowError) as e:
        ORACLE.concat_elements(a, a)
    assert e.value.status == abi.ERR_NOT_YET_IMPLEMENTED and str(e.value) == "Not yet implemented: concat not supported for Int32"


@pytest.mark.parametrize("seed", range(4))
def test_oracle_vs_pyarrow(seed):
    """Secondary check: the valid rows against pyarrow.compute.binary_join_element_wise(a, b, "")."""
    pa = pytest.importorskip("pyarrow")
    pc = pytest.importorskip("pyarrow.compute")
    rng = np.random.default_rng(seed)
    n = 200
    a, b = rand_items(rng, n, 20, 0.2), rand_items(rng, n, 20, 0.2)
    exp = pc.binary_join_element_wise(pa.array([None if x is None else x.decode() for x in a], pa.string()),
                                      pa.array([None if x is None else x.decode() for x in b], pa.string()), "").to_pylist()
    for typ in ("utf8", "large_utf8", "utf8_view"):
        got = values(ORACLE.concat_elements(column(typ, a), column(typ, b)))
        assert [None if g is None else g.decode() for g in got] == exp, typ
