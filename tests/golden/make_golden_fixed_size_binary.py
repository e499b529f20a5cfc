"""Writes fixed_size_binary_vectors.json: the literal cases of the reference's FixedSizeBinary filter / take tests, as data,
and hand-derived cases for the rules those tests do not reach.

  filter.rs  test_filter_fixed_binary (its four predicates)
  take.rs    test_take_fixed_size_binary_with_nulls_indices (width 4, take_fixed_size)
             test_take_fixed_size_binary_with_nulls_indices_not_optimized_length (width 5, the dynamic-length path)
  derived    width 0 (FixedSizeBinaryArray::try_new takes the length from the NullBuffer), indices whose NullBuffer has no
             null (NullBuffer::union drops it, take_primitive keeps it), a UInt64 index whose index * width wraps into the
             buffer, Int64 -1 (the start passes the buffer: core's start panic), a valid index one row past the buffer (the end
             panic), a valid index further past it (the start panic), a null out-of-bounds index on the dynamic path (never
             read), and an in-bounds null index on take_fixed_size (gathered under the null).

A column is {"width": W, "values": [hex or null]} (a null row's bytes are zero). Indices are {"dtype": "u32" | "u64" |
"i64", "values": [int or null], "buffer": bool}. "expect" is {"values": [hex or null], "length": n, "nulls": bool} or
{"error": status name, "message": text}."""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def col(w, rows):
    return {"width": w, "values": [None if r is None else bytes(r).hex() for r in rows]}


def ok(rows, nulls, length=None):
    return {"values": [None if r is None else bytes(r).hex() for r in rows], "length": len(rows) if length is None else length,
            "nulls": nulls}


def err(status, message):
    return {"error": status, "message": message}


cases = []
v = col(2, [[1, 2], [3, 4], [5, 6]])
for pred, exp in (([True, False, True], ok([[1, 2], [5, 6]], False)), ([False, False, False], ok([], False)),
                  ([True, True, True], ok([[1, 2], [3, 4], [5, 6]], False)), ([False, False, True], ok([[5, 6]], False))):
    cases.append({"name": "test_filter_fixed_binary", "op": "filter", "column": v, "predicate": pred, "expect": exp})

for w, name in ((4, "test_take_fixed_size_binary_with_nulls_indices"),
                (5, "test_take_fixed_size_binary_with_nulls_indices_not_optimized_length")):
    rows = [[k] * 4 + ([1] if w == 5 else []) for k in (1, 2, 3, 4)]
    if w == 5:
        rows[0][4] = 1
    cases.append({"name": name, "op": "take", "column": col(w, rows), "indices": {"dtype": "u32", "values": [0, None, None, 3], "buffer": True},
                  "expect": ok([rows[0], None, None, rows[3]], True)})

z = col(0, [[], None, [], []])
cases += [
    {"name": "width0_filter_no_nulls_has_length_0", "op": "filter", "column": col(0, [[], [], []]), "predicate": [True, False, True],
     "expect": ok([], False, 0)},
    {"name": "width0_filter_with_a_null_keeps_its_length", "op": "filter", "column": z, "predicate": [True, True, False, False],
     "expect": ok([[], None], True)},
    {"name": "width0_filter_all_keeps_its_length", "op": "filter", "column": col(0, [[], []]), "predicate": [True, True],
     "expect": ok([[], []], False)},
    {"name": "width0_take_no_nulls_has_length_0", "op": "take", "column": col(0, [[], []]),
     "indices": {"dtype": "u32", "values": [1, 0, 7], "buffer": False}, "expect": ok([], False, 0)},
    {"name": "width0_take_with_a_null", "op": "take", "column": z, "indices": {"dtype": "u32", "values": [1, 0], "buffer": False},
     "expect": ok([None, []], True)},
    {"name": "width0_take_bits_panics_past_values_with_nulls", "op": "take", "column": z,
     "indices": {"dtype": "u32", "values": [0, 9], "buffer": False}, "expect": err("PANIC_OUT_OF_BOUNDS", "assertion failed: idx < self.bit_len")},
    {"name": "empty_null_buffer_of_indices_is_dropped", "op": "take", "column": col(3, [[1, 2, 3], [4, 5, 6]]),
     "indices": {"dtype": "u32", "values": [1, 0], "buffer": True}, "expect": ok([[4, 5, 6], [1, 2, 3]], False)},
    {"name": "empty_null_buffer_of_indices_is_dropped_native_width", "op": "take", "column": col(4, [[1, 2, 3, 4], [5, 6, 7, 8]]),
     "indices": {"dtype": "u32", "values": [1], "buffer": True}, "expect": ok([[5, 6, 7, 8]], False)},
    {"name": "u64_index_wraps_into_the_buffer", "op": "take", "column": col(20, [list(range(20)), list(range(20, 40))]),
     "indices": {"dtype": "u64", "values": [2 ** 62, 1], "buffer": False}, "expect": ok([list(range(20)), list(range(20, 40))], False)},
    {"name": "u64_index_wraps_to_an_unaligned_byte", "op": "take", "column": col(3, [[1, 2, 3], [4, 5, 6]]),
     "indices": {"dtype": "u64", "values": [pow(3, -1, 2 ** 64)], "buffer": False}, "expect": ok([[2, 3, 4]], False)},
    {"name": "i64_minus_one_is_the_start_panic", "op": "take", "column": col(20, [list(range(20))]),
     "indices": {"dtype": "i64", "values": [0, -1], "buffer": False},
     "expect": err("PANIC_OUT_OF_BOUNDS", f"range start index {2 ** 64 - 20} out of range for slice of length 20")},
    {"name": "valid_index_two_rows_past_the_buffer_is_the_start_panic", "op": "take", "column": col(6, [[1] * 6, [2] * 6]),
     "indices": {"dtype": "u32", "values": [0, 3], "buffer": False},
     "expect": err("PANIC_OUT_OF_BOUNDS", "range start index 18 out of range for slice of length 12")},
    {"name": "valid_index_past_the_buffer_is_the_end_panic", "op": "take", "column": col(6, [[1] * 6, [2] * 6]),
     "indices": {"dtype": "u32", "values": [1, 2], "buffer": False},
     "expect": err("PANIC_OUT_OF_BOUNDS", "range end index 18 out of range for slice of length 12")},
    {"name": "null_index_past_the_buffer_is_never_read", "op": "take", "column": col(6, [[1] * 6, [2] * 6]),
     "indices": {"dtype": "u32", "values": [None, 1], "buffer": True, "raw": [99, 1]}, "expect": ok([None, [2] * 6], True)},
    {"name": "native_width_valid_index_past_the_values_panics", "op": "take", "column": col(2, [[1, 2], [3, 4]]),
     "indices": {"dtype": "u32", "values": [None, 9], "buffer": True, "raw": [1, 9]},
     "expect": err("PANIC_OUT_OF_BOUNDS", "Out-of-bounds index 9")},
    {"name": "native_width_null_index_in_bounds_gathers_its_row", "op": "take", "column": col(2, [[1, 2], [3, 4]]),
     "indices": {"dtype": "u32", "values": [None, 0], "buffer": True, "raw": [1, 0]}, "expect": ok([None, [1, 2]], True),
     "under_nulls": ["0304", "0102"]},
]

with open(os.path.join(HERE, "fixed_size_binary_vectors.json"), "w") as f:
    json.dump(cases, f, indent=1)
    f.write("\n")
