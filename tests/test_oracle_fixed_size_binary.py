"""tests/oracle_fixed_size_binary.py against the reference's literal FixedSizeBinary filter / take cases and the
hand-derived ones (tests/golden/fixed_size_binary_vectors.json), on the CPU. The device tests run the same cases."""
import json
import os

import numpy as np
import pytest

from acu import HostArray
from acu import _abi as abi

import oracle_fixed_size_binary as of
import oracle_list as ol

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fixed_size_binary_vectors.json")
with open(GOLDEN) as f:
    CASES = json.load(f)
DTYPES = {"u32": abi.U32, "u64": abi.U64, "i64": abi.I64}
NP = {abi.U32: np.uint32, abi.U64: np.uint64, abi.I64: np.int64}


def build_column(d):
    w, rows = d["width"], d["values"]
    vals = np.frombuffer(b"".join(bytes.fromhex(r) if r is not None else bytes(w) for r in rows), np.uint8).reshape(len(rows), w)
    valid = None if all(r is not None for r in rows) else [r is not None for r in rows]
    return of.column(vals, valid)


def build_indices(d):
    """(raw values, valid mask, has a NullBuffer, acu dtype, HostArray)."""
    dt = DTYPES[d["dtype"]]
    raw = d.get("raw") or [0 if v is None else v for v in d["values"]]
    valid = [v is not None for v in d["values"]]
    arr = np.array([x % (1 << 64) if dt == abi.U64 else x for x in raw], dtype=NP[dt])
    h = HostArray.from_numpy(dt, arr, np.array(valid) if d["buffer"] else None)
    return arr, np.array(valid), d["buffer"], dt, h


def run_case(case, filter_fn, take_fn):
    """filter_fn(col, predicate list) / take_fn(col, indices tuple) -> column or raises an error with status and message."""
    col = build_column(case["column"])
    if case["op"] == "filter":
        return filter_fn(col, case["predicate"])
    return take_fn(col, build_indices(case["indices"]))


def check(case, run):
    exp = case["expect"]
    if "error" in exp:
        with pytest.raises(Exception) as e:
            run()
        assert e.value.status == getattr(abi, "ERR_" + exp["error"]) and e.value.message == exp["message"]
        return
    r = run()
    assert r.length == exp["length"]
    rows = [None if v is None else bytes.fromhex(v) for v in exp["values"]]
    assert r.values.shape == (exp["length"], case["column"]["width"])
    valid = of.valid_mask(r)
    assert [None if not valid[i] else bytes(r.values[i]) for i in range(r.length)] == rows[:r.length]
    assert of.has_buffer(r) == exp["nulls"]
    if "under_nulls" in case:  # every row's bytes, null rows included
        assert [bytes(r.values[i]).hex() for i in range(r.length)] == case["under_nulls"]


def oracle_filter(col, pred):
    return of.filter(col, ol.filter_mask(HostArray.bool_from_numpy(np.array(pred, bool))))


def oracle_take(col, ix):
    raw, valid, buf, dt, _ = ix
    return of.take(col, raw, valid, buf, dt)


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{c['name']}-{k}" for k, c in enumerate(CASES)])
def test_oracle_matches_golden(i):
    case = CASES[i]
    check(case, lambda: run_case(case, oracle_filter, oracle_take))


def test_golden_covers_every_reference_test():
    names = {c["name"] for c in CASES}
    assert {"test_filter_fixed_binary", "test_take_fixed_size_binary_with_nulls_indices",
            "test_take_fixed_size_binary_with_nulls_indices_not_optimized_length"} <= names


def test_check_bounds_comes_before_the_value_step():
    col = of.column(np.arange(12, dtype=np.uint8).reshape(2, 6), None)
    with pytest.raises(ol.OracleError) as e:
        of.take(col, np.array([5], np.int32), None, False, abi.I32, check_bounds=True)
    assert e.value.status == abi.ERR_COMPUTE and e.value.message.endswith("Array index out of bounds, cannot get item at index 5 from 2 entries")


def test_child_step_keeps_width_zero_rows_and_drops_an_empty_null_buffer():
    col = of.column(np.zeros((3, 0), np.uint8), [True, True, False])
    r = of.filter(col, np.array([True, True, False]), child_step=True)
    assert r.length == 2 and not of.has_buffer(r)
