"""Builds the columns of tests/golden/union_vectors.json and checks a case's result against its expectations."""
import json
import os

import numpy as np

from acu import BOOL, HostArray, StructColumn, UnionColumn, Utf8Column
from acu import _abi as abi

import oracle_filter_take as oft
from oracle_filter_take import nulls_of

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "union_vectors.json")
DTYPES = {"i32": abi.I32, "u32": abi.U32, "i64": abi.I64, "f64": abi.F64, "u8": abi.U8, "u64": abi.U64}


def golden_cases():
    with open(GOLDEN) as f:
        return json.load(f)


def build(d):
    t = d["type"]
    if t == "struct":
        fields = [build(f) for f in d["fields"]]
        n = fields[0].length if fields else len(d["nulls"])
        return StructColumn(fields, nulls_of([True] * n) if d["nulls"] is None else nulls_of(d["nulls"], force=True))
    if t == "union":
        mode = abi.UNION_DENSE if d["mode"] == "dense" else abi.UNION_SPARSE
        return UnionColumn(mode, d["field_type_ids"], [build(c) for c in d["children"]], d["type_ids"], d.get("offsets"))
    if t == "utf8":
        vals = d["values"]
        data = b"".join((v or "").encode() for v in vals)
        offs = np.zeros(len(vals) + 1, np.int32)
        offs[1:] = np.cumsum([len((v or "").encode()) for v in vals])
        return Utf8Column(offs, np.frombuffer(data + b"\0", np.uint8).copy(), nulls_of([v is not None for v in vals]))
    if t == "bool":
        return HostArray.from_list(BOOL, d["values"])
    return HostArray.from_list(DTYPES[t], d["values"])


def run_case(case, filter_fn, take_fn):
    col = build(case["column"])
    if case["op"] == "filter":
        return filter_fn(col, HostArray.bool_from_numpy(np.array(case["predicate"], bool)))
    return take_fn(col, HostArray.from_list(DTYPES[case["index_dtype"]], case["indices"]))


def _decode(v):
    return v.decode() if isinstance(v, bytes) else v


def _plain(x):
    if isinstance(x, list):
        return [_plain(y) for y in x]
    return _decode(x)


def check(case, got):
    name = case["name"]
    if "expect" in case:
        assert _plain(oft.to_pylist(got)) == case["expect"], name
    if "expect_len" in case:
        assert got.length == case["expect_len"], name
    if "expect_type_ids" in case:
        assert [int(x) for x in got.type_ids] == case["expect_type_ids"], name
    if "expect_offsets" in case:
        assert [int(x) for x in got.offsets] == case["expect_offsets"], name
    if "expect_children" in case:
        for c, exp in zip(got.children, case["expect_children"]):
            if exp is not None:
                assert _plain(oft.to_pylist(c)) == exp, name
    if "expect_fields" in case:
        assert [_plain(oft.to_pylist(f)) for f in got.fields] == case["expect_fields"], name
    if "expect_nulls" in case:
        exp = case["expect_nulls"]
        assert (got.nulls.validity is None) == (exp is None), name
        if exp is not None:
            assert [bool(b) for b in got.nulls.valid_mask()] == exp, name
    if "expect_null_count" in case:
        assert int(sum(not b for b in got.nulls.valid_mask())) == case["expect_null_count"], name
