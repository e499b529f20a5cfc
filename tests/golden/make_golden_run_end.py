"""Writes run_end_vectors.json: the literal cases of the reference's RunEndEncoded filter / take tests, transcribed as data.

  filter: arrow-select/src/filter.rs test_filter_run_end_encoding_array (:1429), _sliced (:1449), _remove_value (:1466),
          _remove_all_but_one (:1486), _empty (:1505), _max_value_gt_predicate_len (:1518)
  take:   arrow-select/src/take.rs test_take_runs (:2605), test_take_runs_sliced (:2631), test_take_run_empty_indices (:2912),
          test_take_run_end_encoded_merges_identical_runs (:2936), _merges_identical_string_runs (:2964), _mixed_runs (:2993)

A case is {"name", "op": "filter" | "take", "run_ends", "run_end_type": "i16" | "i32" | "i64", "values", "values_type": "i16" |
"i32" | "i64" | "utf8", "slice": [offset, length] (optional, RunArray::slice), "predicate" (filter) or "indices" and
"index_dtype" (take)}. The expectations are what each test asserts: "expect_len" (the logical length), "expect_run_ends",
"expect_values" (the physical values child) and "expect_logical" (the logical values); a missing key is not asserted."""
import json
import os


def runs(logical):
    """PrimitiveRunBuilder / StringRunBuilder::extend: equal neighbours share a run."""
    ends, vals = [], []
    for i, v in enumerate(logical):
        if vals and vals[-1] == v:
            ends[-1] = i + 1
        else:
            ends.append(i + 1)
            vals.append(v)
    return ends, vals


def filter_cases():
    t, f = True, False
    return [
        {"name": "test_filter_run_end_encoding_array", "op": "filter", "run_ends": [2, 3, 8], "run_end_type": "i64",
         "values": [7, -2, 9], "values_type": "i64", "predicate": [t, f, t, f, t, f, t, f],
         "expect_len": 4, "expect_run_ends": [1, 2, 4], "expect_values": [7, -2, 9]},
        {"name": "test_filter_run_end_encoding_array_sliced", "op": "filter", "run_ends": [2, 3, 8], "run_end_type": "i64",
         "values": [7, -2, 9], "values_type": "i64", "slice": [2, 3], "predicate": [t, f, t], "expect_logical": [-2, 9]},
        {"name": "test_filter_run_end_encoding_array_remove_value", "op": "filter", "run_ends": [2, 3, 8, 10], "run_end_type": "i32",
         "values": [7, -2, 9, -8], "values_type": "i32", "predicate": [f, t, f, f, t, f, t, f, f, f],
         "expect_len": 3, "expect_run_ends": [1, 3], "expect_values": [7, 9]},
        {"name": "test_filter_run_end_encoding_array_remove_all_but_one", "op": "filter", "run_ends": [2, 3, 8, 10],
         "run_end_type": "i16", "values": [7, -2, 9, -8], "values_type": "i16", "predicate": [f, f, f, f, f, f, t, f, f, f],
         "expect_len": 1, "expect_run_ends": [1], "expect_values": [9]},
        {"name": "test_filter_run_end_encoding_array_empty", "op": "filter", "run_ends": [2, 3, 8, 10], "run_end_type": "i64",
         "values": [7, -2, 9, -8], "values_type": "i64", "predicate": [f] * 10, "expect_len": 0},
        {"name": "test_filter_run_end_encoding_array_max_value_gt_predicate_len", "op": "filter", "run_ends": [2, 3, 8, 10],
         "run_end_type": "i64", "values": [7, -2, 9, -8], "values_type": "i64", "predicate": [f, t, t],
         "expect_len": 2, "expect_run_ends": [1, 2], "expect_values": [7, -2]},
    ]


def take_cases():
    out = []
    ends, vals = runs([1, 1, 2, 2, 1, 1, 1, 2, 2, 1, 1, 2, 2])
    out.append({"name": "test_take_runs", "op": "take", "run_ends": ends, "run_end_type": "i32", "values": vals, "values_type": "i32",
                "indices": [7, 2, 3, 7, 11, 4, 6], "index_dtype": "i32",
                "expect_len": 7, "expect_run_ends": [5, 7], "expect_values": [2, 1]})
    ends, vals = runs([1, 1, 2, 2, 3, 3, 3, 4, 4, 5, 5, 6, 6])
    out.append({"name": "test_take_runs_sliced", "op": "take", "run_ends": ends, "run_end_type": "i32", "values": vals,
                "values_type": "i32", "slice": [4, 6], "indices": [0, 5, 5, 1, 4], "index_dtype": "i32",
                "expect_run_ends": [1, 3, 4, 5], "expect_logical": [3, 5, 5, 3, 4]})
    ends, vals = runs([1, 1, 2, 2])
    out.append({"name": "test_take_run_empty_indices", "op": "take", "run_ends": ends, "run_end_type": "i32", "values": vals,
                "values_type": "i32", "indices": [], "index_dtype": "i32", "expect_len": 0, "expect_run_ends": [], "expect_values": []})
    ends, vals = runs([1, 1, 0, 0, 1, 1])
    out.append({"name": "test_take_run_end_encoded_merges_identical_runs", "op": "take", "run_ends": ends, "run_end_type": "i32",
                "values": vals, "values_type": "i32", "indices": [0, 1, 4, 5], "index_dtype": "i32",
                "expect_run_ends": [4], "expect_logical": [1, 1, 1, 1]})
    ends, vals = runs(["bob", "bob", "alice", "alice", "bob", "bob"])
    out.append({"name": "test_take_run_end_encoded_merges_identical_string_runs", "op": "take", "run_ends": ends,
                "run_end_type": "i32", "values": vals, "values_type": "utf8", "indices": [0, 1, 4, 5], "index_dtype": "i32",
                "expect_run_ends": [4], "expect_logical": ["bob"] * 4})
    ends, vals = runs(["bob", "bob", "alice", "alice", "bob", "bob", "eve", "eve"])
    out.append({"name": "test_take_run_end_encoded_mixed_runs", "op": "take", "run_ends": ends, "run_end_type": "i32",
                "values": vals, "values_type": "utf8", "indices": [0, 0, 1, 4, 5, 2, 3, 2, 6, 7, 6], "index_dtype": "i32",
                "expect_run_ends": [5, 8, 11], "expect_logical": ["bob"] * 5 + ["alice"] * 3 + ["eve"] * 3})
    return out


if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "run_end_vectors.json")
    with open(path, "w") as f:
        json.dump({"cases": filter_cases() + take_cases()}, f, indent=1)
        f.write("\n")
