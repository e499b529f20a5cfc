#!/usr/bin/env python
"""Transcribes the reference's literal min / max tests of byte, view, fixed-size-binary and boolean columns
(arrow-arith/src/aggregate.rs, apache/arrow-rs @ cd7c6b83) into tests/golden/aggregate_vectors.json.

Nothing here runs the reference: every case is a literal input -> literal expected output copied from the cited test, with
the builder calls of the Rust test (`append_slice(&[true; 64])`, `append_nulls(63)`, `.slice(4, 2)`) re-evaluated in Python.
Run `python tests/golden/make_golden_aggregate.py` to regenerate the committed JSON.

Encoding: "kind" is "binary" (values are hex strings), "string" (UTF-8 strings) or "boolean"; null = Arrow null. "forms"
lists the array types the reference test runs the case on (the test_binary! / test_string! macros):
  binary:  Binary, LargeBinary, BinaryView, and FixedSizeBinary with every value zero-padded to the longest one
           (pad_inputs_and_test_fixed_size_binary, aggregate.rs:1501-1536);
  string:  Utf8, LargeUtf8, Utf8View.
"slice" = [offset, length] applied to the built array (Array::slice). "min" / "max" = the expected results (the boolean
cases also pin bool_and = min_boolean and bool_or = max_boolean, aggregate.rs:880-889).
"""
import json
import os

cases = []
BINARY_FORMS = ["binary", "large_binary", "binary_view", "fixed_size_binary"]
STRING_FORMS = ["utf8", "large_utf8", "utf8_view"]


def hx(b):
    return None if b is None else b.hex()


def binary_case(id, ref, data, mn, mx, slice=None):
    c = {"id": id, "ref": ref, "kind": "binary", "forms": BINARY_FORMS if slice is None else ["binary"],
         "data": [hx(x) for x in data], "min": hx(mn), "max": hx(mx)}
    if slice is not None:
        c["slice"] = list(slice)
    cases.append(c)


def string_case(id, ref, data, mn, mx, slice=None):
    c = {"id": id, "ref": ref, "kind": "string", "forms": STRING_FORMS if slice is None else ["utf8"], "data": data, "min": mn, "max": mx}
    if slice is not None:
        c["slice"] = list(slice)
    cases.append(c)


def boolean_case(id, ref, data, mn, mx, slice=None):
    c = {"id": id, "ref": ref, "kind": "boolean", "data": data, "min": mn, "max": mx}
    if slice is not None:
        c["slice"] = list(slice)
    cases.append(c)


A = "arrow-arith/src/aggregate.rs"

# ---- test_binary! (aggregate.rs:1536-1596) --------------------------------------------------------------------------
binary_case("test_binary_min_max_with_nulls", A + ":1557-1569",
            [b"b01234567890123", None, None, b"a", b"c", b"abcdedfg0123456"], b"a", b"c")
binary_case("test_binary_min_max_no_null", A + ":1571-1581",
            [b"b", b"abcdefghijklmnopqrst", b"c", b"b01234567890123"], b"abcdefghijklmnopqrst", b"c")
binary_case("test_binary_min_max_all_nulls", A + ":1582", [None, None], None, None)
binary_case("test_binary_min_max_1", A + ":1585-1596",
            [None, b"b01234567890123435", None, b"b0123xxxxxxxxxxx", b"a"], b"a", b"b0123xxxxxxxxxxx")

# ---- test_string! (aggregate.rs:1598-1668) --------------------------------------------------------------------------
string_case("test_string_min_max_with_nulls", A + ":1617-1629",
            ["b012345678901234", None, None, "a", "c", "b0123xxxxxxxxxxx"], "a", "c")
string_case("test_string_min_max_no_null", A + ":1631-1641",
            ["b", "b012345678901234", "a", "b012xxxxxxxxxxxx"], "a", "b012xxxxxxxxxxxx")
string_case("test_string_min_max_all_nulls", A + ":1643-1648", [None, None], None, None)
string_case("test_string_min_max_1", A + ":1650-1661", [None, "c12345678901234", None, "b", "c1234xxxxxxxxxx"], "b", "c1234xxxxxxxxxx")
string_case("test_string_min_max_empty", A + ":1663-1668", [], None, None)

# ---- bool_and / bool_or (aggregate.rs:1263-1297) --------------------------------------------------------------------
boolean_case("test_primitive_array_bool_and", A + ":1263-1267", [True, False, True, False, True], False, True)
boolean_case("test_primitive_array_bool_and_with_nulls", A + ":1269-1273", [None, True, True, None, True], True, True)
boolean_case("test_primitive_array_bool_and_all_nulls", A + ":1275-1279", [None, None, None], None, None)
boolean_case("test_primitive_array_bool_or", A + ":1281-1285", [True, False, True, False, True], False, True)
boolean_case("test_primitive_array_bool_or_with_nulls", A + ":1287-1291", [None, False, False, None, False], False, False)
boolean_case("test_primitive_array_bool_or_all_nulls", A + ":1293-1297", [None, None, None], None, None)

# ---- test_boolean_min_max* (aggregate.rs:1671-1826) -----------------------------------------------------------------
boolean_case("test_boolean_min_max_empty", A + ":1671-1676", [], None, None)
boolean_case("test_boolean_min_max_all_null", A + ":1678-1683", [None, None], None, None)
boolean_case("test_boolean_min_max_no_null", A + ":1685-1690", [True, False, True], False, True)
for k, (data, mn, mx) in enumerate([
        ([True, True, None, False, None], False, True),
        ([None, True, None, False, None], False, True),
        ([False, True, None, False, None], False, True),
        ([True, None], True, True),
        ([False, None], False, False),
        ([True], True, True),
        ([False], False, False)]):
    boolean_case(f"test_boolean_min_max_{k}", A + ":1692-1721", data, mn, mx)
for k, (data, mn, mx) in enumerate([
        ([False], False, False),
        ([None, False], False, False),
        ([None, True], True, True),
        ([True], True, True)]):
    boolean_case(f"test_boolean_min_max_smaller_{k}", A + ":1723-1740", data, mn, mx)
boolean_case("test_boolean_min_max_64_true_64_false_no_nulls", A + ":1742-1762", [True] * 64 + [False] * 64, False, True)
boolean_case("test_boolean_min_max_64_true_64_false_with_nulls", A + ":1742-1762",
             [True] * 31 + [None] + [True] * 32 + [False] + [None] * 63, False, True)
boolean_case("test_boolean_min_max_64_false_64_true_no_nulls", A + ":1764-1784", [False] * 64 + [True] * 64, False, True)
boolean_case("test_boolean_min_max_64_false_64_true_with_nulls", A + ":1764-1784",
             [False] * 31 + [None] + [False] * 32 + [True] + [None] * 63, False, True)
boolean_case("test_boolean_min_max_96_true_no_nulls", A + ":1786-1805", [True] * 96, True, True)
boolean_case("test_boolean_min_max_96_true_with_nulls", A + ":1786-1805",
             [True] * 31 + [None] + [True] * 32 + [True] * 31 + [None], True, True)
boolean_case("test_boolean_min_max_96_false_no_nulls", A + ":1807-1826", [False] * 96, False, False)
boolean_case("test_boolean_min_max_96_false_with_nulls", A + ":1807-1826",
             [False] * 31 + [None] + [False] * 32 + [False] * 31 + [None], False, False)

# ---- test_min_max_sliced_* (aggregate.rs:1919-1983) -----------------------------------------------------------------
boolean_case("test_min_max_sliced_boolean", A + ":1919-1938", [None, True], True, True)
boolean_case("test_min_max_sliced_boolean_sliced", A + ":1919-1938", [None, None, None, None, None, True], True, True, slice=(4, 2))
string_case("test_min_max_sliced_string", A + ":1941-1961", [None, "foo"], "foo", "foo")
string_case("test_min_max_sliced_string_sliced", A + ":1941-1961", [None, None, None, None, None, "foo"], "foo", "foo", slice=(4, 2))
binary_case("test_min_max_sliced_binary", A + ":1963-1983", [None, bytes([5])], bytes([5]), bytes([5]))
binary_case("test_min_max_sliced_binary_sliced", A + ":1963-1983", [None, None, None, None, None, bytes([5])], bytes([5]), bytes([5]),
            slice=(4, 2))

if __name__ == "__main__":
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "aggregate_vectors.json")
    with open(out, "w") as f:
        json.dump({"source": "apache/arrow-rs @ cd7c6b83, " + A, "cases": cases}, f, indent=1)
        f.write("\n")
    print(f"{len(cases)} cases -> {out}")
