"""Writes union_vectors.json: the literal cases of the reference's struct and union filter / take tests, as data.

  filter.rs  test_filter_union_array_dense / _sparse (and their shared helper's three predicates),
             test_filter_run_union_array_dense, test_filter_union_array_dense_with_nulls / _sparse_with_nulls,
             test_filter_struct, test_filter_empty_struct
  take.rs    test_take_struct, test_take_struct_with_null_indices, test_take_union_sparse, test_take_union_dense,
             test_take_union_dense_using_builder, test_take_union_dense_all_match_issue_6206

A column is {"type": "i32" | "u32" | "i64" | "f64" | "bool" | "utf8", "values": [...]} (null = None),
{"type": "struct", "fields": [...], "nulls": [valid bits] | null} or {"type": "union", "mode": "sparse" | "dense",
"field_type_ids": [...], "children": [...], "type_ids": [...], "offsets": [...] (dense)}. A union's expected logical values
are [type id, child value] pairs, a struct's are lists of field values (None for a null row)."""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def prim(t, values):
    return {"type": t, "values": values}


def dense(ids, children, tids, offs):
    return {"type": "union", "mode": "dense", "field_type_ids": ids, "children": children, "type_ids": tids, "offsets": offs}


def sparse(ids, children, tids):
    return {"type": "union", "mode": "sparse", "field_type_ids": ids, "children": children, "type_ids": tids}


def struct(fields, nulls):
    return {"type": "struct", "fields": fields, "nulls": nulls}


def test_struct(rows):
    """create_test_struct (take.rs:1236-1260): fields a: Boolean, b: Int32; a null row is null in both fields."""
    a = [None if r is None else r[0] for r in rows]
    b = [None if r is None else r[1] for r in rows]
    return struct([prim("bool", a), prim("i32", b)], [r is not None for r in rows])


cases = []

# test_filter_union_array (filter.rs:2081-2111) over the dense and the sparse builder's A 1, B 3.2, A 34
ab_dense = dense([0, 1], [prim("i32", [1, 34]), prim("f64", [3.2])], [0, 1, 0], [0, 0, 1])
ab_sparse = sparse([0, 1], [prim("i32", [1, None, 34]), prim("f64", [None, 3.2, None])], [0, 1, 0])
for name, col in (("test_filter_union_array_dense", ab_dense), ("test_filter_union_array_sparse", ab_sparse)):
    for pred, exp in (([True, False, False], [[0, 1]]), ([True, False, True], [[0, 1], [0, 34]]),
                      ([True, True, False], [[0, 1], [1, 3.2]])):
        cases.append({"name": name, "op": "filter", "column": col, "predicate": pred, "expect": exp})

# test_filter_run_union_array_dense: to_data() equality with the builder's A 1, A 3
cases.append({"name": "test_filter_run_union_array_dense", "op": "filter",
              "column": dense([0], [prim("i32", [1, 3, 34])], [0, 0, 0], [0, 1, 2]), "predicate": [True, True, False],
              "expect": [[0, 1], [0, 3]], "expect_type_ids": [0, 0], "expect_offsets": [0, 1], "expect_children": [[1, 3]]})

# test_filter_union_array_dense_with_nulls / _sparse_with_nulls: A 1, B 3.2, B null, A 34
abn_dense = dense([0, 1], [prim("i32", [1, 34]), prim("f64", [3.2, None])], [0, 1, 1, 0], [0, 0, 1, 1])
abn_sparse = sparse([0, 1], [prim("i32", [1, None, None, 34]), prim("f64", [None, 3.2, None, None])], [0, 1, 1, 0])
cases.append({"name": "test_filter_union_array_dense_with_nulls", "op": "filter", "column": abn_dense,
              "predicate": [True, True, False, False], "expect": [[0, 1], [1, 3.2]]})
for name, col in (("test_filter_union_array_dense_with_nulls", abn_dense), ("test_filter_union_array_sparse_with_nulls", abn_sparse)):
    cases.append({"name": name, "op": "filter", "column": col, "predicate": [True, False, True, False], "expect": [[0, 1], [1, None]]})

# test_filter_struct (filter.rs:2250-2318)
a = prim("utf8", ["hello", " ", "world", "!"])
b = prim("i32", [5, 6, 7, 8])
for fields, exp_fields in (([a], [["hello", "world"]]), ([a, b], [["hello", "world"], [5, 7]])):
    for nulls, exp_nulls in ((None, None), ([True, False, False, True], [True, False])):
        cases.append({"name": "test_filter_struct", "op": "filter", "column": struct(fields, nulls), "predicate": [True, False, True, False],
                      "expect_fields": exp_fields, "expect_nulls": exp_nulls})

# test_filter_empty_struct (filter.rs:2321-2370): a {b: Int64, c: {}}; StructArray::new drops a's all-valid NullBuffer,
# new_empty_fields keeps c's
cases.append({"name": "test_filter_empty_struct", "op": "filter",
              "column": struct([prim("i64", [None, None, None]), struct([], [True, True, True])], None),
              "predicate": [True, False, True], "expect_len": 2})

# test_take_struct (take.rs:2343-2377)
ts = [(True, 42), (False, 28), (False, 19), (True, 31), None]
cases.append({"name": "test_take_struct", "op": "take", "column": test_struct(ts), "indices": [0, 3, 1, 0, 2, 4], "index_dtype": "u32",
              "expect": [[True, 42], [True, 31], [False, 28], [True, 42], [False, 19], None], "expect_null_count": 1})
cases.append({"name": "test_take_struct", "op": "take", "column": struct([], [False, True, False, True, False, True]),
              "indices": [0, 2, 1, 4], "index_dtype": "u32", "expect_nulls": [False, False, True, False]})
# test_take_struct_with_null_indices (take.rs:2380-2405)
cases.append({"name": "test_take_struct_with_null_indices", "op": "take", "column": test_struct(ts),
              "indices": [None, 3, 1, None, 0, 4], "index_dtype": "u32",
              "expect": [None, [True, 31], [False, 28], None, [True, 42], None], "expect_null_count": 3})

# test_take_union_sparse (take.rs:2731-2768): a struct child (id 0) and a Utf8 child (id 1), every row of type 1
cases.append({"name": "test_take_union_sparse", "op": "take",
              "column": sparse([0, 1], [test_struct(ts), prim("utf8", ["a", None, "c", None, "d"])], [1] * 5),
              "indices": [0, 3, 1, 0, 2, 4], "index_dtype": "u32",
              "expect_children": [None, ["a", None, None, "a", "c", "d"]]})
# test_take_union_dense (take.rs:2771-2826)
cases.append({"name": "test_take_union_dense", "op": "take",
              "column": dense([0, 1], [prim("u32", [10, 20, 30, 40]), prim("utf8", ["a", None, "c", "d"])], [0, 1, 1, 0, 0, 1, 0],
                              [0, 0, 1, 1, 2, 2, 3]),
              "indices": [0, 3, 1, 0, 2, 4], "index_dtype": "u32",
              "expect_type_ids": [0, 0, 1, 0, 1, 0], "expect_offsets": [0, 1, 0, 2, 1, 3], "expect_children": [[10, 20, 10, 30], ["a", None]]})
# test_take_union_dense_using_builder (take.rs:2829-2852): a 1, b 3.0, a 4, a 5, b 2.0 taken at [2, 0, 1, 2]
cases.append({"name": "test_take_union_dense_using_builder", "op": "take",
              "column": dense([0, 1], [prim("i32", [1, 4, 5]), prim("f64", [3.0, 2.0])], [0, 1, 0, 0, 1], [0, 0, 1, 2, 1]),
              "indices": [2, 0, 1, 2], "index_dtype": "u32",
              "expect": [[0, 4], [0, 1], [1, 3.0], [0, 4]], "expect_type_ids": [0, 0, 1, 0], "expect_offsets": [0, 1, 0, 2],
              "expect_children": [[4, 1, 4], [3.0]]})
# test_take_union_dense_all_match_issue_6206 (take.rs:2855-2871)
cases.append({"name": "test_take_union_dense_all_match_issue_6206", "op": "take",
              "column": dense([0], [prim("i64", [1, 2, 3, 4, 5])], [0] * 5, [0, 1, 2, 3, 4]),
              "indices": [0, 2, 4], "index_dtype": "i64", "expect_len": 3, "expect": [[0, 1], [0, 3], [0, 5]]})

if __name__ == "__main__":
    with open(os.path.join(HERE, "union_vectors.json"), "w") as f:
        json.dump(cases, f, indent=1)
        f.write("\n")
    print(f"{len(cases)} cases")
