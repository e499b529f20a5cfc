"""Writes tests/golden/decimal_cast_vectors.json: the literal inputs, outputs and error texts of the reference's decimal cast
tests (arrow-cast/src/cast/mod.rs tests module, and the rescale_decimal tests of arrow-cast/src/cast/decimal.rs), without
the Decimal256, Float16, string and dictionary cases. Run from the repository root: python tests/golden/make_golden_decimal_cast.py

A case: kind "dec" (decimal -> decimal), "to_dec" (integer / float -> decimal) or "from_dec" (decimal -> integer / float);
"in" = {width, precision, scale} or {dtype}, with "values" (null = None); "to" likewise; "safe"; then "expected" (the
result's values, nulls as None; null where the reference only asserts the cast succeeds) or "error" (the error's Display
text; "*" where the reference only asserts an error) or "error_contains" (a substring the reference asserts).

Cases the reference runs through Decimal256 as well (run_decimal_cast_test_case_between_multiple_types) are kept for
Decimal128 -> Decimal128 only; the reference's Float16 and Decimal256 arrays are left out. Where a reference test only asserts
`is_ok()` for the safe variant of an unsafe error case, the safe variant is left out (its values are not stated)."""
import json
import os

I8, I16, I32, I64, U8, U16, U32, U64, F32, F64 = range(10)


def dec(width, p, s, values=None):
    d = {"width": width, "precision": p, "scale": s}
    if values is not None:
        d["values"] = values
    return d


def prim(dtype, values=None):
    d = {"dtype": dtype}
    if values is not None:
        d["values"] = values
    return d


def case(name, kind, src, to, safe, expected=None, error=None, error_contains=None):
    c = {"name": name, "kind": kind, "in": src, "to": to, "safe": safe}
    if error is not None:
        c["error"] = error
    elif error_contains is not None:
        c["error_contains"] = error_contains
    else:
        c["expected"] = expected
    return c


def coverage(name, rows):
    """DecimalCastTestConfig rows (input_prec, input_scale, input_repr, output_prec, output_scale, Ok value or Err text),
    cast with safe = false, Decimal128 -> Decimal128; "{}" in an error is the output type's prefix."""
    out = []
    for i, (pi, si, v, po, so, r) in enumerate(rows):
        if isinstance(r, str):
            out.append(case(f"{name}_{i}", "dec", dec(16, pi, si, [v]), dec(16, po, so), False, error=r.replace("{}", "Decimal128")))
        else:
            out.append(case(f"{name}_{i}", "dec", dec(16, pi, si, [v]), dec(16, po, so), False, [r]))
    return out


E = "Invalid argument error: "
UNSIGNED_AND_SIGNED = [U8, U16, U32, U64, I8, I16, I32, I64]
D2N_IN = [125, 225, 325, None, 525]


ROUND_IN = [1123454, 2123456, -3123453, -3123456, None]
ROUND_OUT = [112345, 212346, -312345, -312346, None]

CASES = [
    # test_cast_decimal_to_decimal_round
    case("test_cast_decimal_to_decimal_round", "dec", dec(16, 20, 4, ROUND_IN), dec(16, 20, 3), True, ROUND_OUT),
    # test_cast_decimal32_to_decimal32_overflow / 64 / 128
    case("test_cast_decimal32_to_decimal32_overflow", "dec", dec(4, 9, 3, [2 ** 31 - 1]), dec(4, 9, 9), False,
         error="Cast error: Cannot cast to Decimal32(9, 9). Overflowing on 2147483647"),
    case("test_cast_decimal64_to_decimal64_overflow", "dec", dec(8, 18, 3, [2 ** 63 - 1]), dec(8, 18, 18), False,
         error="Cast error: Cannot cast to Decimal64(18, 18). Overflowing on 9223372036854775807"),
    case("test_cast_decimal128_to_decimal128_overflow", "dec", dec(16, 38, 3, [2 ** 127 - 1]), dec(16, 38, 38), False,
         error="Cast error: Cannot cast to Decimal128(38, 38). Overflowing on 170141183460469231731687303715884105727"),
    # test_cast_decimal32/64_to_decimal32/64_large_scale_reduction
    case("test_cast_decimal32_to_decimal32_large_scale_reduction", "dec", dec(4, 9, 3, [-999999999, 0, 999999999, None]),
         dec(4, 9, -6), True, [-1, 0, 1, None]),
    case("test_cast_decimal32_to_decimal32_large_scale_reduction_zero", "dec", dec(4, 9, 3, [-999999999, 0, 999999999, None]),
         dec(4, 9, -7), True, [0, 0, 0, None]),
    case("test_cast_decimal64_to_decimal64_large_scale_reduction", "dec",
         dec(8, 18, 3, [-999999999999999999, 0, 999999999999999999, None]), dec(8, 18, -15), True, [-1, 0, 1, None]),
    case("test_cast_decimal64_to_decimal64_large_scale_reduction_zero", "dec",
         dec(8, 18, 3, [-999999999999999999, 0, 999999999999999999, None]), dec(8, 18, -16), True, [0, 0, 0, None]),
    # test_decimal_to_decimal_throw_error_on_precision_overflow_* and _same_scale
    case("test_decimal_to_decimal_throw_error_on_precision_overflow_same_scale", "dec", dec(16, 24, 2, [123456789]),
         dec(16, 6, 2), False,
         error="Invalid argument error: 1234567.89 is too large to store in a Decimal128 of precision 6. Max is 9999.99"),
    case("test_decimal_to_decimal_throw_error_on_precision_overflow_lower_scale", "dec", dec(16, 24, 4, [123456789]),
         dec(16, 6, 2), False,
         error="Invalid argument error: 12345.68 is too large to store in a Decimal128 of precision 6. Max is 9999.99"),
    case("test_decimal_to_decimal_throw_error_on_precision_overflow_greater_scale", "dec", dec(16, 24, 2, [123456789]),
         dec(16, 6, 3), False,
         error="Invalid argument error: 1234567.890 is too large to store in a Decimal128 of precision 6. Max is 999.999"),
    case("test_decimal_to_decimal_same_scale", "dec", dec(16, 4, 2, [520]), dec(16, 3, 2), False, [520]),
    case("test_decimal_to_decimal_same_scale_zero", "dec", dec(16, 3, 0, [0]), dec(16, 2, 0), True, [0]),
    # test_cast_decimal_error_output
    case("test_cast_decimal_error_output_large", "to_dec", prim(I64, [1]), dec(4, 1, 1), False,
         error="Invalid argument error: 1.0 is too large to store in a Decimal32 of precision 1. Max is 0.9"),
    case("test_cast_decimal_error_output_small", "to_dec", prim(I64, [-1]), dec(4, 1, 1), False,
         error="Invalid argument error: -1.0 is too small to store in a Decimal32 of precision 1. Min is -0.9"),
    # test_cast_decimal_to_numeric_negative_scale (Decimal128 / Decimal32 parts)
    case("test_cast_decimal_to_numeric_negative_scale_d32", "from_dec", dec(4, 8, -2, [125, 225, 325, None, 525]), prim(I64),
         True, [12500, 22500, 32500, None, 52500]),
    case("test_cast_decimal_to_numeric_negative_scale_d32_s9", "from_dec", dec(4, 9, -9, [2, 1, None]), prim(I64), True,
         [2000000000, 1000000000, None]),
    # test_cast_f64_to_decimal128
    case("test_cast_f64_to_decimal128_s2", "to_dec", prim(F64, [0.0699999999, 0.0659999999, 0.0650000000, 0.0649999999]),
         dec(16, 18, 2), True, [7, 7, 7, 6]),
    case("test_cast_f64_to_decimal128_s3", "to_dec", prim(F64, [0.0699999999, 0.0659999999, 0.0650000000, 0.0649999999]),
         dec(16, 18, 3), True, [70, 66, 65, 65]),
    # test_cast_integer_to_decimal32_does_not_truncate
    case("test_cast_integer_to_decimal32_does_not_truncate_safe", "to_dec", prim(I64, [5000000000, 10000000000, 42]),
         dec(4, 9, 0), True, [None, None, 42]),
    case("test_cast_integer_to_decimal32_does_not_truncate_unsafe", "to_dec", prim(I64, [5000000000, 10000000000, 42]),
         dec(4, 9, 0), False, error="Cast error: Cannot cast to Decimal32(9, 0). Overflowing on 5000000000"),
    case("test_cast_integer_to_decimal32_does_not_truncate_d128", "to_dec", prim(I64, [5000000000, 10000000000, 42]),
         dec(16, 9, 0), True, [None, None, 42]),
    # test_cast_integer_to_decimal32_scales_before_narrowing
    case("test_cast_integer_to_decimal32_scales_before_narrowing_safe", "to_dec", prim(I64, [5000000000]), dec(4, 9, -1), True,
         [500000000]),
    case("test_cast_integer_to_decimal32_scales_before_narrowing_unsafe", "to_dec", prim(I64, [5000000000]), dec(4, 9, -1),
         False, [500000000]),
    # test_cast_uint_to_decimal32_does_not_wrap / test_cast_uint64_max_to_decimal64_does_not_wrap
    case("test_cast_uint_to_decimal32_does_not_wrap_safe", "to_dec", prim(U32, [4000000000]), dec(4, 9, 0), True, [None]),
    case("test_cast_uint_to_decimal32_does_not_wrap_unsafe", "to_dec", prim(U32, [4000000000]), dec(4, 9, 0), False,
         error="Cast error: Cannot cast to Decimal32(9, 0). Overflowing on 4000000000"),
    case("test_cast_uint_to_decimal32_does_not_wrap_d128", "to_dec", prim(U32, [4000000000]), dec(16, 9, 0), True, [None]),
    case("test_cast_uint64_max_to_decimal64_does_not_wrap", "to_dec", prim(U64, [2 ** 64 - 1]), dec(8, 18, 0), False,
         error="Cast error: Cannot cast to Decimal64(18, 0). Overflowing on 18446744073709551615"),
    # rescale_decimal tests (decimal.rs): one-row casts with the same outcome (None = a null under safe casting)
    case("test_rescale_decimal_upscale_within_precision", "dec", dec(16, 5, 2, [12345]), dec(16, 8, 5), True, [12345000]),
    case("test_rescale_decimal_downscale_rounds_half_away_from_zero", "dec", dec(16, 5, 3, [1050, -1050]), dec(16, 5, 1), True,
         [11, -11]),
    case("test_rescale_decimal_downscale_large_delta_returns_zero", "dec", dec(4, 9, 9, [12345]), dec(4, 9, 4), True, [0]),
    case("test_rescale_decimal_upscale_overflow_returns_none", "dec", dec(4, 4, 0, [9999]), dec(4, 5, 2), True, [None]),
]

# test_decimal_to_decimal_coverage / _increase_scale_and_precision_unchecked / _decrease_scale_and_precision_unchecked
CASES += coverage("test_decimal_to_decimal_coverage", [
    (5, 1, 99999, 10, 6, 9999900000),
    (5, 1, 99, 7, 6, 9900000),
    (5, 1, 99999, 7, 6, E + "9999.900000 is too large to store in a {} of precision 7. Max is 9.999999"),
    (5, 3, 99999, 10, 2, 10000),
    (5, 3, 99994, 10, 2, 9999),
    (5, 3, 99999, 10, 3, 99999),
    (10, 5, 999999, 8, 7, 99999900),
    (10, 5, 9999999, 8, 7, E + "99.9999900 is too large to store in a {} of precision 8. Max is 9.9999999"),
    (7, 4, 9999999, 6, 2, 100000),
    (10, 5, 12345678, 8, 3, 123457),
    (10, 5, 9999999, 4, 3, E + "100.000 is too large to store in a {} of precision 4. Max is 9.999"),
    (10, 5, 999999, 6, 5, 999999),
    (10, 5, 9999999, 6, 5, E + "99.99999 is too large to store in a {} of precision 6. Max is 9.99999"),
    (7, 4, 12345, 7, 6, 1234500),
    (7, 4, 123456, 7, 6, E + "12.345600 is too large to store in a {} of precision 7. Max is 9.999999"),
    (7, 5, 1234567, 7, 4, 123457),
    (7, 5, 9999999, 7, 5, 9999999),
    (7, 0, 1234567, 8, 0, 1234567),
    (7, 0, 1234567, 6, 0, E + "1234567 is too large to store in a {} of precision 6. Max is 999999"),
    (7, 0, 123456, 6, 0, 123456),
])
CASES += coverage("test_decimal_to_decimal_increase_scale_and_precision_unchecked", [
    (5, 0, 99999, 10, 5, 9999900000),
    (5, 0, -99999, 10, 5, -9999900000),
    (5, 2, 99999, 10, 5, 99999000),
    (5, -2, -99999, 10, 3, -9999900000),
    (5, 3, -12345, 6, 5, E + "-12.34500 is too small to store in a {} of precision 6. Min is -9.99999"),
])
CASES += coverage("test_decimal_to_decimal_decrease_scale_and_precision_unchecked", [
    (5, 0, 99999, 3, -3, 100),
    (5, 0, -99999, 1, -5, -1),
    (10, 2, 123456789, 5, -2, 12346),
    (10, 4, -9876543210, 7, 0, -987654),
    (7, 4, 9999999, 6, 3, E + "1000.000 is too large to store in a {} of precision 6. Max is 999.999"),
])

# test_cast_decimal32/64/128_to_decimal32/64/128 (Decimal256 arms left out)
for w, p in ((4, 9), (8, 17), (16, 20)):
    name = f"test_cast_decimal{8 * w}_to_decimal{8 * w}"
    CASES.append(case(name, "dec", dec(w, p, 3, [1123456, 2123456, 3123456, None]), dec(w, p, 4), True,
                      [11234560, 21234560, 31234560, None]))
    CASES.append(case(name + "_precision_error", "dec", dec(w, {4: 9, 8: 9, 16: 10}[w], 0, [123456, None]), dec(w, 2, 2), False,
                      error=f"{E}123456.00 is too large to store in a Decimal{8 * w} of precision 2. Max is 0.99"))
# test_cast_decimal128_to_decimal128_negative_scale / _negative
CASES.append(case("test_cast_decimal128_to_decimal128_negative_scale", "dec", dec(16, 20, 0, [1123450, 2123455, 3123456, None]),
                  dec(16, 20, -1), True, [112345, 212346, 312346, None]))
CASES.append(case("test_cast_decimal128_to_decimal128_negative_123", "dec", dec(16, 10, -1, [123]), dec(16, 10, -2), True, [12]))
CASES.append(case("test_cast_decimal128_to_decimal128_negative_125", "dec", dec(16, 10, -1, [125]), dec(16, 10, -2), True, [13]))
# (test_decimal_to_decimal_throw_error_on_precision_overflow_diff_type casts to Decimal256: left out)
# test_cast_decimal32/64/128_to_numeric (generate_decimal_to_numeric_cast_test_case; the Float16 arm left out)
for w, p in ((4, 8), (8, 8), (16, 38)):
    for t in UNSIGNED_AND_SIGNED:
        CASES.append(case(f"test_cast_decimal{8 * w}_to_numeric_{t}", "from_dec", dec(w, p, 2, D2N_IN), prim(t), True,
                          [1, 2, 3, None, 5]))
    for t in (F32, F64):
        CASES.append(case(f"test_cast_decimal{8 * w}_to_numeric_{t}", "from_dec", dec(w, p, 2, D2N_IN), prim(t), True,
                          [1.25, 2.25, 3.25, None, 5.25]))
CASES += [
    case("test_cast_decimal128_to_numeric_u8_unsafe", "from_dec", dec(16, 38, 2, [51300]), prim(U8), False,
         error="Cast error: value of 513 is out of range UInt8"),
    case("test_cast_decimal128_to_numeric_u8_safe", "from_dec", dec(16, 38, 2, [51300]), prim(U8), True, [None]),
    case("test_cast_decimal128_to_numeric_i8_unsafe", "from_dec", dec(16, 38, 2, [24400]), prim(I8), False,
         error="Cast error: value of 244 is out of range Int8"),
    case("test_cast_decimal128_to_numeric_i8_safe", "from_dec", dec(16, 38, 2, [24400]), prim(I8), True, [None]),
    case("test_cast_decimal128_to_numeric_f32", "from_dec", dec(16, 38, 2, [125, 225, 325, None, 525, 112345678, 112345679]),
         prim(F32), True, [1.25, 2.25, 3.25, None, 5.25, 1123456.75, 1123456.75]),
    case("test_cast_decimal128_to_numeric_f64", "from_dec",
         dec(16, 38, 2, [125, 225, 325, None, 525, 112345678901234568, 112345678901234560]), prim(F64), True,
         [1.25, 2.25, 3.25, None, 5.25, 1123456789012345.6, 1123456789012345.6]),
]
# test_cast_decimal_to_numeric_negative_scale (the Decimal64 / Decimal128 / Decimal32 error parts)
CASES += [
    case("test_cast_decimal_to_numeric_negative_scale_d64_s3", "from_dec", dec(8, 18, -3, D2N_IN), prim(I64), True,
         [125000, 225000, 325000, None, 525000]),
    case("test_cast_decimal_to_numeric_negative_scale_d64_s10", "from_dec", dec(8, 18, -10, [12, 34, None]), prim(I64), True,
         [120000000000, 340000000000, None]),
    case("test_cast_decimal_to_numeric_negative_scale_d128_s4", "from_dec", dec(16, 38, -4, D2N_IN), prim(I64), True,
         [1250000, 2250000, 3250000, None, 5250000]),
    case("test_cast_decimal_to_numeric_negative_scale_d128_s18", "from_dec", dec(16, 38, -18, [9, 1, None]), prim(I64), True,
         [9000000000000000000, 1000000000000000000, None]),
    case("test_cast_decimal_to_numeric_negative_scale_mul_overflow", "from_dec", dec(4, 9, -1, [999999999]), prim(I64), False,
         error="Arithmetic overflow: Overflow happened on: 999999999 * 10"),
    case("test_cast_decimal_to_numeric_negative_scale_mul_overflow_safe", "from_dec", dec(4, 9, -1, [999999999]), prim(I64), True,
         [None]),
    case("test_cast_decimal_to_numeric_negative_scale_out_of_range", "from_dec", dec(8, 18, -1, [13]), prim(I8), False,
         error="Cast error: value of 130 is out of range Int8"),
    case("test_cast_decimal_to_numeric_negative_scale_out_of_range_safe", "from_dec", dec(8, 18, -1, [13]), prim(I8), True, [None]),
]
# test_cast_numeric_to_decimal128 and its _overflow / _negative / _precision_overflow variants
for t in UNSIGNED_AND_SIGNED:
    CASES.append(case(f"test_cast_numeric_to_decimal128_{t}", "to_dec", prim(t, [1, 2, 3, None, 5]), dec(16, 38, 6), True,
                      [1000000, 2000000, 3000000, None, 5000000]))
CASES += [
    case("test_cast_numeric_to_decimal128_u8_null_4", "to_dec", prim(U8, [1, 2, 3, 4, 100]), dec(16, 3, 1), True,
         [10, 20, 30, 40, None]),
    case("test_cast_numeric_to_decimal128_i8_null_4", "to_dec", prim(I8, [1, 2, 3, 4, 100]), dec(16, 3, 1), True,
         [10, 20, 30, 40, None]),
    case("test_cast_numeric_to_decimal128_f32", "to_dec", prim(F32, [1.1, 2.2, 4.4, None, 1.1234564, 1.1234567]), dec(16, 38, 6),
         True, [1100000, 2200000, 4400000, None, 1123456, 1123457]),
    case("test_cast_numeric_to_decimal128_f64", "to_dec",
         prim(F64, [1.1, 2.2, 4.4, None, 1.1234564891234, 1.1234567891234, 1.1234564890123456, 1.1234567890123456]),
         dec(16, 38, 6), True, [1100000, 2200000, 4400000, None, 1123456, 1123457, 1123456, 1123457]),
    case("test_cast_numeric_to_decimal128_overflow_safe", "to_dec", prim(I64, [2 ** 63 - 1]), dec(16, 38, 30), True, [None]),
    case("test_cast_numeric_to_decimal128_overflow_unsafe", "to_dec", prim(I64, [2 ** 63 - 1]), dec(16, 38, 30), False, error="*"),
    case("test_cast_numeric_to_decimal128_negative_i32", "to_dec", prim(I32, [1123456, 2123456, 3123456]), dec(16, 38, -1), True,
         [112345, 212345, 312345]),
    case("test_cast_numeric_to_decimal128_negative_f32", "to_dec", prim(F32, [1123.456, 2123.456, 3123.456]), dec(16, 38, -1), True,
         [112, 212, 312]),
    case("test_cast_numeric_to_decimal128_precision_overflow_safe", "to_dec", prim(I64, [1234567]), dec(16, 7, 3), True, [None]),
    case("test_cast_numeric_to_decimal128_precision_overflow_unsafe", "to_dec", prim(I64, [1234567]), dec(16, 7, 3), False,
         error=E + "1234567.000 is too large to store in a Decimal128 of precision 7. Max is 9999.999"),
]
# test_cast_floating_to_decimals (the reference asserts only that the unsafe cast succeeds), and
# test_cast_floating_point_to_decimal128_precision_overflow / _overflow
for w in (4, 8, 16):
    CASES.append(case(f"test_cast_floating_to_decimals_{8 * w}", "to_dec", prim(F64, [1.1]), dec(w, 9, 3), False, None))
CASES += [
    case("test_cast_floating_point_to_decimal128_precision_overflow_safe", "to_dec", prim(F64, [1.1]), dec(16, 2, 2), True, [None]),
    case("test_cast_floating_point_to_decimal128_precision_overflow_unsafe", "to_dec", prim(F64, [1.1]), dec(16, 2, 2), False,
         error_contains=E + "1.10 is too large to store in a Decimal128 of precision 2. Max is 0.99"),
    case("test_cast_floating_point_to_decimal128_overflow_safe", "to_dec", prim(F64, [1.7976931348623157e308]), dec(16, 38, 30),
         True, [None]),
    case("test_cast_floating_point_to_decimal128_overflow_unsafe", "to_dec", prim(F64, [1.7976931348623157e308]),
         dec(16, 38, 30), False, error_contains="Cast error: Cannot cast to Decimal128(38, 30)"),
]


def main():
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "decimal_cast_vectors.json")
    with open(path, "w") as f:
        json.dump({"cases": CASES}, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
