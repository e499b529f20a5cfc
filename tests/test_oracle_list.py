"""The filter / take oracle (tests/oracle_filter_take.py) of list and flat columns against the reference's literal cases,
and its own rules on small inputs."""
import numpy as np
import pytest

from acu import BOOL, HostArray, ListColumn, Utf8Column
from acu import _abi as abi

import oracle_filter_take as oft
from list_util import check, golden_cases, run_case
from oracle_filter_take import nulls_of as _nulls


@pytest.mark.parametrize("case", golden_cases(), ids=lambda c: c["name"])
def test_golden(case):
    check(case, lambda: run_case(case, lambda c, p: oft.filter(c, oft.filter_mask(p)), oft.take_host), oft.OracleError)


def test_filter_keeps_null_ranges_take_empties_them():
    child = Utf8Column(np.array([0, 2, 4, 7], np.int32), np.frombuffer(b"abcdefg", np.uint8).copy(), _nulls([True, False, True]))
    col = ListColumn(np.array([1, 2, 3], np.int32), child, _nulls([False, True]))
    f = oft.filter(col, np.array([True, True]))
    assert [int(x) for x in f.offsets] == [0, 1, 2] and oft.describe(f.child)[2] == b"cdefg"
    t = oft.take_host(col, HostArray.from_numpy(abi.U32, [0, 1]))
    assert [int(x) for x in t.offsets] == [0, 0, 1]
    # the Utf8 child of a list take keeps the bytes under its null rows
    t = oft.take_host(ListColumn(np.array([0, 3], np.int32), child, _nulls([True])), HostArray.from_numpy(abi.U32, [0]))
    assert oft.describe(t.child)[2] == b"abcdefg" and t.child.nulls.validity is not None


def test_unchecked_panics():
    col = ListColumn(np.array([0, 1, 2], np.int32), HostArray.from_numpy(abi.I32, [5, 6]), _nulls([True, True]))
    with pytest.raises(oft.OracleError) as e:
        oft.take_host(col, HostArray.from_numpy(abi.U32, [0, 2]))
    assert e.value.message == "index out of bounds: the len is 3 but the index is 3" and e.value.index == 1
    col.nulls = _nulls([True, False])
    with pytest.raises(oft.OracleError) as e:
        oft.take_host(col, HostArray.from_numpy(abi.U32, [0, 2]))
    assert e.value.message == "assertion failed: idx < self.bit_len"


def _null_over(dtype, items, value):
    """Indices `items` whose null slots hold `value`."""
    h = HostArray.from_list(dtype, items)
    h.values[[i for i, x in enumerate(items) if x is None]] = value
    return h


# take of a flat column: take_bits sets only the valid indices' bits; take_primitive's value gather panics before take_nulls
# (take.rs:405-416); check_bounds returns Ok when the length does not fit the index type (take.rs:174-180)
FLAT_TAKES = [
    ("boolean under a null index", HostArray.from_list(BOOL, [True, True, None]), _null_over(abi.U32, [0, None, 1], 1), False,
     ("flat", 3, [True, False, True], [True, False, True])),
    ("gather before take_nulls", HostArray.from_list(abi.I32, [1, None, 3]), HostArray.from_list(abi.U32, [0, 7]), False,
     (abi.ERR_PANIC_OUT_OF_BOUNDS, "Out-of-bounds index 7", 1)),
    ("check_bounds skipped past the index type", HostArray.from_numpy(abi.I32, np.arange(300)), HostArray.from_list(abi.I8, [-1]), True,
     (abi.ERR_PANIC_OUT_OF_BOUNDS, "Out-of-bounds index 4294967295", 0)),
]


@pytest.mark.parametrize("name,col,idx,check_bounds,expect", FLAT_TAKES, ids=[c[0] for c in FLAT_TAKES])
def test_flat_take(name, col, idx, check_bounds, expect):
    if expect[0] == "flat":
        assert oft.describe(oft.take_host(col, idx, check_bounds)) == expect
        return
    with pytest.raises(oft.OracleError) as e:
        oft.take_host(col, idx, check_bounds)
    assert (e.value.status, e.value.message, e.value.index) == expect
