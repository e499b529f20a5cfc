"""Builds the columns of tests/golden/list_vectors.json and runs a case through the oracle or the device."""
import json
import os

import numpy as np

from acu import FixedSizeListColumn, HostArray, ListColumn
from acu import _abi as abi

import oracle_list as ol

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "list_vectors.json")
DTYPES = {"u32": abi.U32, "i32": abi.I32, "i64": abi.I64, "u8": abi.U8, "u64": abi.U64}


def golden_cases():
    with open(GOLDEN) as f:
        return json.load(f)


def build(d):
    child = HostArray.from_list(DTYPES[d.get("child_type", "i32")], d["child"])
    n = len(d["offsets"]) - 1 if "offsets" in d else len(d["child"]) // d["size"]
    nulls = HostArray.from_list(abi.U8, [0] * n) if d["nulls"] is None else \
        HostArray.from_list(abi.U8, [0 if v else None for v in d["nulls"]])
    nulls.values = np.zeros(0, np.uint8)
    if d["kind"] == "fixed_size_list":
        col = FixedSizeListColumn(d["size"], child, nulls)
    else:
        col = ListColumn(np.array(d["offsets"], np.int64 if d["kind"] == "large_list" else np.int32), child, nulls)
    if "slice" in d:  # Array::slice: offsets from the new row 0, the validity's bit offset advanced
        off, ln = d["slice"]
        assert d["kind"] != "fixed_size_list"
        nl = nulls.slice(off, ln)
        nl.values = np.zeros(0, np.uint8)
        col = ListColumn(col.offsets[off:off + ln + 1].copy(), child, nl)
    return col


def run_case(case, filter_fn, take_fn):
    """filter_fn(col, predicate) / take_fn(col, indices) -> column; returns the column."""
    col = build(case["list"])
    if case["op"] == "filter":
        return filter_fn(col, HostArray.bool_from_numpy(np.array(case["predicate"], bool)))
    return take_fn(col, HostArray.from_list(DTYPES[case["index_dtype"]], case["indices"]))


def check(case, run, error_type):
    exp = case.get("expect")
    if isinstance(exp, dict):
        try:
            run()
        except error_type as e:
            assert e.status == getattr(abi, "ERR_" + exp["error"]) and e.message == exp["message"]
            return
        raise AssertionError(f"{case['name']}: no error")
    got = run()
    if exp is not None:
        assert ol.to_pylist(got) == exp, case["name"]
    if "expect_child" in case:
        assert ol.to_pylist(got.child) == case["expect_child"], case["name"]
    if "expect_offsets" in case:
        assert [int(x) for x in got.offsets] == case["expect_offsets"]
