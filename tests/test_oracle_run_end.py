"""The RunEndEncoded oracle (tests/oracle_run_end.py) against the reference's literal cases, and against the property tests
of arrow-array/src/array/run_array.rs:1195-1292 (every logical index, shuffled and repeated, at every slice)."""
import numpy as np
import pytest

from acu import HostArray, RunEndColumn
from acu import _abi as abi

import oracle_run_end as ore
from run_end_util import check, golden_cases, run_case


@pytest.mark.parametrize("case", golden_cases(), ids=lambda c: c["name"])
def test_golden(case):
    check(case, run_case(case, lambda c, p: ore.filter(c, ore.ol.filter_mask(p)), ore.take))


def _random_run_array(rng, n_logical=80):
    lens = []
    while sum(lens) < n_logical:
        lens.append(int(rng.integers(1, 8)))
    lens[-1] -= sum(lens) - n_logical
    ends = np.cumsum(lens).astype(np.int32)
    vals = HostArray.from_numpy(abi.I32, np.arange(len(ends)) * 10)
    return RunEndColumn(ends, vals)


def test_get_physical_indices_every_slice():
    """run_array.rs:1195-1245: logical indices shuffled and repeated map to the run that holds them, at every slice."""
    rng = np.random.default_rng(7)
    col = _random_run_array(rng)
    ends = [int(x) for x in col.run_ends]
    for off in range(80):
        for ln in range(0, 80 - off + 1, 7 if off % 5 else 1):
            s = col.slice(off, ln)
            ix = list(range(ln)) * 2
            rng.shuffle(ix)
            phys = ore.get_physical_indices(s, ix)
            for x, p in zip(ix, phys):
                assert (ends[p - 1] if p else 0) <= off + x < ends[p]
            if ln:
                assert ore.start_physical(s) == phys[ix.index(0)] and ore.end_physical(s) == phys[ix.index(ln - 1)]


def test_get_physical_indices_names_the_largest_index():
    """run_array.rs:1247-1292: an index past the length fails naming the largest index value, null slots included."""
    col = _random_run_array(np.random.default_rng(1)).slice(3, 20)
    with pytest.raises(ore.OracleError) as e:
        ore.get_physical_indices(col, [0, 25, 19, 40, 2])
    assert e.value.message == "Invalid argument error: Logical index 40 is out of bounds for RunArray of length 20"
    idx = HostArray.from_list(abi.U32, [0, None, 1])
    idx.values[1] = 21  # a null slot over an out-of-bounds value
    with pytest.raises(ore.OracleError) as e:
        ore.take(col, idx)
    assert e.value.message == "Invalid argument error: Logical index 21 is out of bounds for RunArray of length 20"


def test_take_logical_values_every_slice():
    rng = np.random.default_rng(3)
    col = _random_run_array(rng)
    for off in range(0, 80, 3):
        for ln in sorted({min(1, 80 - off), min(5, 80 - off), 80 - off} - {0}):
            s = col.slice(off, ln)
            ix = rng.integers(0, ln, 30)
            got = ore.take(s, HostArray.from_numpy(abi.I64, ix))
            full = ore.logical(s)
            assert ore.logical(got) == [full[i] for i in ix]
            # merged runs: no two neighbouring runs hold equal values
            vals = got.values.to_list()
            assert all(a != b for a, b in zip(vals, vals[1:]))


def test_filter_logical_values_every_slice():
    rng = np.random.default_rng(5)
    col = _random_run_array(rng)
    for off in range(0, 80, 3):
        for ln in sorted({min(1, 80 - off), min(9, 80 - off), 80 - off} - {0}):
            s = col.slice(off, ln)
            for p in (ln, max(ln - 3, 0)):
                mask = rng.random(p) < 0.3
                got = ore.filter(s, mask)
                full = ore.logical(s)
                assert ore.logical(got) == [full[i] for i in range(p) if mask[i]]


def test_merge_rules():
    """Two nulls are equal, a null never equals a value, floats compare by total_cmp (bits)."""
    vals = HostArray.from_list(abi.F64, [1.0, None, None, 2.0, -0.0, 0.0, float("nan")])
    vals.values[6] = np.frombuffer(np.uint64(0x7FF8000000000001).tobytes(), np.float64)[0]
    col = RunEndColumn(np.arange(1, 8, dtype=np.int16), vals)
    got = ore.take(col, HostArray.from_numpy(abi.U8, [1, 2, 3, 4, 5, 6, 0]))
    assert [int(x) for x in got.run_ends] == [2, 3, 4, 5, 6, 7]


def test_int16_run_end_unwrap():
    col = RunEndColumn(np.array([40000], np.int64), HostArray.from_list(abi.I8, [1]))
    col16 = RunEndColumn(np.array([32767], np.int16), HostArray.from_list(abi.I8, [1]))
    assert [int(x) for x in ore.take(col16, HostArray.from_numpy(abi.U16, np.zeros(32767, np.uint16))).run_ends] == [32767]
    col16 = RunEndColumn(np.array([2], np.int16), HostArray.from_list(abi.I8, [1]))
    with pytest.raises(ore.OracleError) as e:
        ore.take(col16, HostArray.from_numpy(abi.U16, np.zeros(32768, np.uint16)))
    assert e.value.status == abi.ERR_PANIC_OUT_OF_BOUNDS and e.value.message == ore.UNWRAP_NONE
    assert ore.take(col, HostArray.from_numpy(abi.U16, np.zeros(32768, np.uint16))).length == 32768
