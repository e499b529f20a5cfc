"""Writes zip_vectors.json: the literal cases of the reference's byte and view zip tests (arrow-select/src/zip.rs, the Utf8,
LargeUtf8, Binary, LargeBinary, Utf8View and BinaryView ones), as data, and hand-derived Boolean and FixedSizeBinary cases.

  zip.rs   test_zip_string_array_with_nulls_is_mask_should_be_treated_as_false
           test_zip_kernel_large_string_scalar_with_boolean_array_mask_with_nulls_should_be_treated_as_false
           test_zip_kernel_bytes_scalar_none_1 / _2, test_zip_kernel_bytes_scalar_both
           test_zip_scalar_bytes_only_taking_one_side (its seven cases)
           test_zip_kernel_scalar_strings / _binary / _large_binary
           test_zip_kernel_scalar_strings_array_view / _binary_array_view / _strings_array_view_with_nulls
           test_zip_kernel_scalar_strings_array_view_all_true_null / _all_false_null
           test_zip_kernel_scalar_string_array_view_all_true / _all_false
           test_zip_kernel_scalar_strings_large_strings / _array_view_large_short_strings / _array_view_large_all_true /
           _array_view_large_all_false
  derived  Boolean and FixedSizeBinary(3): arrays with nulls (bits and bytes under nulls come from the chosen side), an array
           against a null scalar (the scalar's own value under its null rows), and two scalars with one null over an
           all-true and a mixed mask. Two scalars go through FallbackImpl = zip_impl: the unselected rows hold the null
           scalar's value, and no NullBuffer is left when the mask selects only the valid scalar. acu_zip's
           PrimitiveScalarImpl would instead write the valid value in every row and always keep a NullBuffer.

A side is {"scalar": bool, "values": [hex or null], "raw": [hex] (optional: the bytes under nulls)}. A mask is {"values":
[bool], "valid": [bool] or null}. "expect" is {"values": [hex or null], "nulls": bool (a NullBuffer is present), "raw":
[hex] (optional: every row's bytes, nulls included)}."""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def h(x):
    return None if x is None else (x.encode() if isinstance(x, str) else bytes(x)).hex()


def side(values, scalar=False, raw=None):
    d = {"scalar": scalar, "values": [h(v) for v in values]}
    if raw is not None:
        d["raw"] = [h(v) for v in raw]
    return d


def mask(values, valid=None):
    return {"values": list(values), "valid": None if valid is None else list(valid)}


def expect(values, nulls, raw=None):
    d = {"values": [h(v) for v in values], "nulls": nulls}
    if raw is not None:
        d["raw"] = [h(v) for v in raw]
    return d


cases = []


def case(name, typ, m, t, f, e, width=None):
    c = {"name": name, "type": typ, "mask": m, "truthy": t, "falsy": f, "expect": e}
    if width is not None:
        c["width"] = width
    cases.append(c)


NULL_MASK = mask([True, True, False, True, False, False], [True, True, True, False, True, True])
case("test_zip_string_array_with_nulls_is_mask_should_be_treated_as_false", "utf8", NULL_MASK,
     side(["1", "2", "3", "4", "5", "6"]), side(["7", "8", "9", "10", "11", "12"]),
     expect(["1", "2", "9", "10", "11", "12"], False))
case("test_zip_kernel_large_string_scalar_with_boolean_array_mask_with_nulls_should_be_treated_as_false", "large_utf8", NULL_MASK,
     side(["test"], True), side(["something else"], True),
     expect(["test", "test"] + ["something else"] * 4, False))
M5 = mask([True, True, False, False, True])
case("test_zip_kernel_bytes_scalar_none_1", "utf8", M5, side(["hello"], True), side([None], True),
     expect(["hello", "hello", None, None, "hello"], True))
case("test_zip_kernel_bytes_scalar_none_2", "utf8", M5, side([None], True), side(["hello"], True),
     expect([None, None, "hello", "hello", None], True))
case("test_zip_kernel_bytes_scalar_both", "utf8", mask([True, True, False, True, False, False]), side(["test"], True),
     side(["something else"], True), expect(["test", "test", "something else", "test", "something else", "something else"], False))
ALL_T, ALL_F = mask([True] * 5), mask([False] * 5)
NUL, S1, S2 = side([None], True), side(["test"], True), side(["something else"], True)
one_side = "test_zip_scalar_bytes_only_taking_one_side"
case(one_side + "[1]", "utf8", ALL_T, NUL, S1, expect([None] * 5, True))
case(one_side + "[2]", "utf8", ALL_F, NUL, S1, expect(["test"] * 5, True))
case(one_side + "[3]", "utf8", ALL_T, S1, NUL, expect(["test"] * 5, True))
case(one_side + "[4]", "utf8", ALL_F, S1, NUL, expect([None] * 5, True))
case(one_side + "[5]", "utf8", ALL_T, S1, S2, expect(["test"] * 5, False))
case(one_side + "[6]", "utf8", ALL_F, S1, S2, expect(["something else"] * 5, False))
case(one_side + "[7]", "utf8", mask([True, False, True, False, True]), NUL, NUL, expect([None] * 5, True))
ALT5 = mask([True, False, True, False, True])
case("test_zip_kernel_scalar_strings", "utf8", ALT5, side(["hello"], True), side(["world"], True),
     expect(["hello", "world", "hello", "world", "hello"], False))
TB, FB = b"\xFF\xFE\xFD", b"world"
case("test_zip_kernel_scalar_binary", "binary", ALT5, side([TB], True), side([FB], True), expect([TB, FB, TB, FB, TB], False))
case("test_zip_kernel_scalar_large_binary", "large_binary", ALT5, side([b"hey"], True), side([FB], True),
     expect([b"hey", FB, b"hey", FB, b"hey"], False))
case("test_zip_kernel_scalar_strings_array_view", "utf8view", mask([True, False, True, False]), side(["hello"], True),
     side(["world"], True), expect(["hello", "world", "hello", "world"], False))
case("test_zip_kernel_scalar_binary_array_view", "binaryview", mask([True, False]), side([b"hello"], True), side([b"world"], True),
     expect([b"hello", b"world"], False))
case("test_zip_kernel_scalar_strings_array_view_with_nulls", "utf8view", M5, side(["hello"], True), side([None], True),
     expect(["hello", "hello", None, None, "hello"], True))
case("test_zip_kernel_scalar_strings_array_view_all_true_null", "utf8view", mask([True, True]), side([None], True), side([None], True),
     expect([None, None], True))
case("test_zip_kernel_scalar_strings_array_view_all_false_null", "utf8view", mask([False, False]), side([None], True),
     side([None], True), expect([None, None], True))
case("test_zip_kernel_scalar_string_array_view_all_true", "utf8view", mask([True, True]), side(["hello"], True), side(["world"], True),
     expect(["hello", "hello"], False))
case("test_zip_kernel_scalar_string_array_view_all_false", "utf8view", mask([False, False]), side(["hello"], True),
     side(["world"], True), expect(["world", "world"], False))
L1, L2 = "longer than 12 bytes", "another longer than 12 bytes"
case("test_zip_kernel_scalar_strings_large_strings", "utf8view", mask([True, False]), side([L1], True), side([L2], True),
     expect([L1, L2], False))
case("test_zip_kernel_scalar_strings_array_view_large_short_strings", "utf8view", mask([True, False, True, False]),
     side(["hello"], True), side([L1], True), expect(["hello", L1, "hello", L1], False))
case("test_zip_kernel_scalar_strings_array_view_large_all_true", "utf8view", mask([True, True]), side([L1], True), side([L2], True),
     expect([L1, L1], False))
case("test_zip_kernel_scalar_strings_array_view_large_all_false", "utf8view", mask([False, False]), side([L1], True), side([L2], True),
     expect([L2, L2], False))

# ---- hand-derived: Boolean (a value is b"\x01" / b"\x00") ----
T, F = b"\x01", b"\x00"
MIX4 = mask([True, False, True, False], [True, True, False, True])  # row 2: a null mask slot counts as false
case("derived_boolean_arrays_with_nulls", "boolean", MIX4, side([T, None, T, F], raw=[T, T, T, F]), side([F, T, None, F], raw=[F, T, T, F]),
     expect([T, T, None, F], True, raw=[T, T, T, F]))
case("derived_boolean_array_against_null_scalar", "boolean", mask([True, False, True]), side([F, T, F]), side([None], True, raw=[T]),
     expect([F, None, F], True, raw=[F, T, F]))
case("derived_boolean_two_scalars_one_null_all_true", "boolean", mask([True, True, True]), side([T], True), side([None], True, raw=[F]),
     expect([T, T, T], False, raw=[T, T, T]))
case("derived_boolean_two_scalars_one_null_mixed", "boolean", mask([True, False, True]), side([T], True), side([None], True, raw=[F]),
     expect([T, None, T], True, raw=[T, F, T]))
case("derived_boolean_arrays_without_nulls", "boolean", mask([False, True]), side([T, F]), side([F, T]), expect([F, F], False))

# ---- hand-derived: FixedSizeBinary(3) ----
A, B, C, D = b"abc", b"def", b"ghi", b"jkl"
X, Y = b"xyz", b"uvw"
case("derived_fsb_arrays_with_nulls", "fsb", MIX4, side([A, None, C, D], raw=[A, B, C, D]), side([X, Y, None, X], raw=[X, Y, Y, X]),
     expect([A, Y, None, X], True, raw=[A, Y, Y, X]), 3)
case("derived_fsb_array_against_null_scalar", "fsb", mask([True, False, True]), side([A, B, C]), side([None], True, raw=[X]),
     expect([A, None, C], True, raw=[A, X, C]), 3)
case("derived_fsb_two_scalars_one_null_all_true", "fsb", mask([True, True, True]), side([A], True), side([None], True, raw=[X]),
     expect([A, A, A], False, raw=[A, A, A]), 3)
case("derived_fsb_two_scalars_one_null_mixed", "fsb", mask([True, False, True]), side([A], True), side([None], True, raw=[X]),
     expect([A, None, A], True, raw=[A, X, A]), 3)
case("derived_fsb_null_truthy_scalar_mixed", "fsb", mask([True, False]), side([None], True, raw=[Y]), side([B], True),
     expect([None, B], True, raw=[Y, B]), 3)
case("derived_fsb_two_valid_scalars", "fsb", mask([False, True, True]), side([A], True), side([B], True), expect([B, A, A], False), 3)

if __name__ == "__main__":
    with open(os.path.join(HERE, "zip_vectors.json"), "w") as out:
        json.dump(cases, out, indent=1)
        out.write("\n")
