"""Writes list_vectors.json: every literal case of the reference's list filter / take tests, transcribed as data.

  filter: arrow-select/src/filter.rs test_filter_list_array (:1559), test_filter_fixed_size_list_arrays (:2017) and
          _with_null (:2055)
  take:   arrow-select/src/take.rs test_take_list / _large_list, _with_value_nulls, _with_nulls (macros :1827, :1882,
          :1950; tests :2090-2115), test_take_fixed_size_list (:2186), test_take_list_out_of_bounds (:2298),
          test_take_sliced_list* (:2532-2600), test_take_value_index_from_fixed_list (:2660),
          test_take_fixed_size_list_null_indices (:2702)

A list is {"kind": "list" | "large_list" | "fixed_size_list", "offsets" | "size", "child": [values, None = null],
"child_type": "i32" (default) | "u8" | "u64", "nulls": [bool] or null, "slice": [offset, length] (optional, list.slice)}.
"indices" may hold None (a null index). "expect" is the logical result (None = a null row) or {"error": status name,
"message": text}; "expect_offsets" the result's offsets, "expect_child" its child's values (None = null)."""
import json
import os


def nested(rows):
    """Offsets, flat child values and row validity of a list built from Option<Vec<Option<v>>> rows."""
    offs, child, nulls = [0], [], []
    for r in rows:
        nulls.append(r is not None)
        child += r or []
        offs.append(len(child))
    return offs, child, nulls


def fixed(rows, size):
    """FixedSizeListArray::from_iter_primitive: a null row holds `size` null children."""
    child, nulls = [], []
    for r in rows:
        nulls.append(r is not None)
        child += r if r is not None else [None] * size
    return child, nulls


def take_list_cases():
    out = []
    for kind in ("list", "large_list"):
        out.append({"name": f"test_take_{kind}", "op": "take",
                    "list": {"kind": kind, "offsets": [0, 3, 6, 6, 8], "child": [0, 0, 0, -1, -2, -1, 2, 3], "nulls": None},
                    "indices": [3, None, 1, 2, 0], "index_dtype": "u32",
                    "expect": [[2, 3], None, [-1, -2, -1], [], [0, 0, 0]],
                    "expect_offsets": [0, 2, 2, 5, 5, 8], "expect_child": [2, 3, -1, -2, -1, 0, 0, 0]})
        out.append({"name": f"test_take_{kind}_with_value_nulls", "op": "take",
                    "list": {"kind": kind, "offsets": [0, 3, 6, 7, 9], "child": [0, None, 0, -1, -2, 3, None, 5, None],
                             "nulls": [True, True, True, True]},
                    "indices": [2, None, 1, 3, 0], "index_dtype": "u32",
                    "expect": [[None], None, [-1, -2, 3], [5, None], [0, None, 0]],
                    "expect_offsets": [0, 1, 1, 4, 6, 9], "expect_child": [None, -1, -2, 3, 5, None, 0, None, 0]})
        out.append({"name": f"test_take_{kind}_with_nulls", "op": "take",
                    "list": {"kind": kind, "offsets": [0, 3, 6, 6, 8], "child": [0, None, 0, -1, -2, 3, 5, None],
                             "nulls": [True, True, False, True]},
                    "indices": [2, None, 1, 3, 0], "index_dtype": "u32",
                    "expect": [None, None, [-1, -2, 3], [5, None], [0, None, 0]],
                    "expect_offsets": [0, 0, 0, 3, 5, 8], "expect_child": [-1, -2, 3, 5, None, 0, None, 0]})
        offs, child, nulls = nested([[0, 1], [2, 3, 4], None, [], [5, 6], [7]])
        out.append({"name": f"test_take_sliced_{kind}", "op": "take",
                    "list": {"kind": kind, "offsets": offs, "child": child, "nulls": nulls, "slice": [1, 4]},
                    "indices": [3, 0, None, 2, 1], "index_dtype": "u32",
                    "expect": [[5, 6], [2, 3, 4], None, [], None]})
        offs, child, nulls = nested([[10], [None, 1], None, [2, None], [], [3]])
        out.append({"name": f"test_take_sliced_{kind}_with_value_nulls", "op": "take",
                    "list": {"kind": kind, "offsets": offs, "child": child, "nulls": nulls, "slice": [1, 4]},
                    "indices": [2, 0, None, 3, 1], "index_dtype": "u32",
                    "expect": [[2, None], [None, 1], None, [], None]})
    return out


def fixed_cases():
    out = []
    for name, size, ct, rows, idx, exp in [
        ("test_take_fixed_size_list/Int32", 3, "i32", [[None, 1, 2], [3, 4, None], [6, 7, 8]], [2, 1, 0],
         [[6, 7, 8], [3, 4, None], [None, 1, 2]]),
        ("test_take_fixed_size_list/UInt8", 1, "u8", [[1], [2], [3], [4], [5], [6], [7], [8]], [2, 7, 0], [[3], [8], [1]]),
        ("test_take_fixed_size_list/UInt64", 3, "u64", [[10, 11, 12], [13, 14, 15], None, [16, 17, 18]], [3, 2, 1, 2, 0],
         [[16, 17, 18], None, [13, 14, 15], None, [10, 11, 12]]),
    ]:
        child, nulls = fixed(rows, size)
        out.append({"name": name, "op": "take", "list": {"kind": "fixed_size_list", "size": size, "child": child,
                                                         "child_type": ct, "nulls": nulls},
                    "indices": idx, "index_dtype": "u32", "expect": exp})
    # take_value_indices_from_fixed_size_list: over an identity child the taken child IS the child row map
    for idx, exp in [([2, 1, 0], [6, 7, 8, 3, 4, 5, 0, 1, 2]), ([3, 2, 1, 2, 0], [9, 10, 11, 6, 7, 8, 3, 4, 5, 6, 7, 8, 0, 1, 2])]:
        out.append({"name": f"test_take_value_index_from_fixed_list/{len(idx)}", "op": "take",
                    "list": {"kind": "fixed_size_list", "size": 3, "child": list(range(12)), "nulls": [True, True, False, True]},
                    "indices": idx, "index_dtype": "u32", "expect_child": exp})
    out.append({"name": "test_take_fixed_size_list_null_indices", "op": "take",
                "list": {"kind": "fixed_size_list", "size": 2, "child": [0, 1, 2, 3], "nulls": None},
                "indices": [0, None], "index_dtype": "i32", "expect": [[0, 1], None], "expect_child": [0, 1, None, None]})
    return out


CASES = [
    {"name": "test_filter_list_array", "op": "filter",
     "list": {"kind": "large_list", "offsets": [0, 3, 6, 8, 8], "child": list(range(8)), "nulls": [True, True, True, False]},
     "predicate": [False, True, False, True],
     "expect": [[3, 4, 5], None], "expect_offsets": [0, 3, 3]},
    {"name": "test_filter_fixed_size_list_arrays/1", "op": "filter",
     "list": {"kind": "fixed_size_list", "size": 3, "child": list(range(9)), "nulls": None},
     "predicate": [True, False, False], "expect": [[0, 1, 2]]},
    {"name": "test_filter_fixed_size_list_arrays/2", "op": "filter",
     "list": {"kind": "fixed_size_list", "size": 3, "child": list(range(9)), "nulls": None},
     "predicate": [True, False, True], "expect": [[0, 1, 2], [6, 7, 8]]},
    {"name": "test_filter_fixed_size_list_arrays_with_null", "op": "filter",
     "list": {"kind": "fixed_size_list", "size": 2, "child": list(range(10)), "nulls": [True, False, False, True, True]},
     "predicate": [True, True, False, True, False], "expect": [[0, 1], None, [6, 7]]},
    {"name": "test_take_list_out_of_bounds", "op": "take",
     "list": {"kind": "list", "offsets": [0, 3, 6, 8], "child": [0, 0, 0, -1, -2, -1, 2, 3], "nulls": None},
     "indices": [1000], "index_dtype": "u32",
     "expect": {"error": "PANIC_OUT_OF_BOUNDS", "message": "index out of bounds: the len is 4 but the index is 1000"}},
] + take_list_cases() + fixed_cases()

if __name__ == "__main__":
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "list_vectors.json"), "w") as f:
        json.dump(CASES, f, indent=1)
        f.write("\n")
