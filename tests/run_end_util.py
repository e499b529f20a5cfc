"""Builds the columns of tests/golden/run_end_vectors.json and runs a case through the oracle or the device."""
import json
import os

import numpy as np

from acu import HostArray, RunEndColumn, Utf8Column
from acu import _abi as abi

import oracle_run_end as ore

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "run_end_vectors.json")
DTYPES = {"i8": abi.I8, "u8": abi.U8, "i16": abi.I16, "u16": abi.U16, "i32": abi.I32, "u32": abi.U32, "i64": abi.I64, "u64": abi.U64}
NP = {"i16": np.int16, "i32": np.int32, "i64": np.int64}


def golden_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def utf8(items):
    data = b"".join(s.encode() for s in items)
    offs = np.zeros(len(items) + 1, np.int32)
    offs[1:] = np.cumsum([len(s.encode()) for s in items])
    nulls = HostArray.from_list(abi.U8, [0] * len(items))
    nulls.values = np.zeros(0, np.uint8)
    return Utf8Column(offs, np.frombuffer(data, np.uint8).copy(), nulls)


def build(case):
    vals = utf8(case["values"]) if case["values_type"] == "utf8" else HostArray.from_list(DTYPES[case["values_type"]], case["values"])
    col = RunEndColumn(np.array(case["run_ends"], NP[case["run_end_type"]]), vals)
    if "slice" in case:
        col = col.slice(*case["slice"])
    return col


def run_case(case, filter_fn, take_fn):
    col = build(case)
    if case["op"] == "filter":
        return filter_fn(col, HostArray.bool_from_numpy(np.array(case["predicate"], bool)))
    return take_fn(col, HostArray.from_list(DTYPES[case["index_dtype"]], case["indices"]))


def check(case, got):
    name = case["name"]
    if "expect_len" in case:
        assert got.length == case["expect_len"], name
    if "expect_run_ends" in case:
        assert [int(x) for x in got.run_ends] == case["expect_run_ends"], name
        assert got.offset == 0
    if "expect_values" in case:
        vals = ore.ol.to_pylist(got.values)
        if case["values_type"] == "utf8":
            vals = [v.decode() for v in vals]
        assert vals == case["expect_values"], name
    if "expect_logical" in case:
        vals = ore.logical(got)
        if case["values_type"] == "utf8":
            vals = [v.decode() for v in vals]
        assert vals == case["expect_logical"], name
