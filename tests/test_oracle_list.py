"""The list oracle (tests/oracle_list.py) against the reference's literal cases, and its own rules on small inputs."""
import numpy as np
import pytest

from acu import HostArray, ListColumn, Utf8Column
from acu import _abi as abi

import oracle_list as ol
from list_util import check, golden_cases, run_case


@pytest.mark.parametrize("case", golden_cases(), ids=lambda c: c["name"])
def test_golden(case):
    check(case, lambda: run_case(case, lambda c, p: ol.filter(c, ol.filter_mask(p)), ol.take_host), ol.OracleError)


def _nulls(mask):
    h = HostArray.from_list(abi.U8, [0 if v else None for v in mask])
    h.values = np.zeros(0, np.uint8)
    return h


def test_filter_keeps_null_ranges_take_empties_them():
    child = Utf8Column(np.array([0, 2, 4, 7], np.int32), np.frombuffer(b"abcdefg", np.uint8).copy(), _nulls([True, False, True]))
    col = ListColumn(np.array([1, 2, 3], np.int32), child, _nulls([False, True]))
    f = ol.filter(col, np.array([True, True]))
    assert [int(x) for x in f.offsets] == [0, 1, 2] and ol.describe(f.child)[2] == b"cdefg"
    t = ol.take_host(col, HostArray.from_numpy(abi.U32, [0, 1]))
    assert [int(x) for x in t.offsets] == [0, 0, 1]
    # the Utf8 child of a list take keeps the bytes under its null rows
    t = ol.take_host(ListColumn(np.array([0, 3], np.int32), child, _nulls([True])), HostArray.from_numpy(abi.U32, [0]))
    assert ol.describe(t.child)[2] == b"abcdefg" and t.child.nulls.validity is not None


def test_unchecked_panics():
    col = ListColumn(np.array([0, 1, 2], np.int32), HostArray.from_numpy(abi.I32, [5, 6]), _nulls([True, True]))
    with pytest.raises(ol.OracleError) as e:
        ol.take_host(col, HostArray.from_numpy(abi.U32, [0, 2]))
    assert e.value.message == "index out of bounds: the len is 3 but the index is 3" and e.value.index == 1
    col.nulls = _nulls([True, False])
    with pytest.raises(ol.OracleError) as e:
        ol.take_host(col, HostArray.from_numpy(abi.U32, [0, 2]))
    assert e.value.message == "assertion failed: idx < self.bit_len"
