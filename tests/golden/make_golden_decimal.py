"""Writes tests/golden/decimal_vectors.json: the reference's literal decimal test vectors, transcribed by hand.

Sources (apache/arrow-rs):
  - arrow-arith/src/numeric.rs `test_decimal` (:1400-1480): values, result types and the four error texts;
  - arrow-arith/src/numeric.rs `test_neg` (:1197-1228): the Decimal32 / 64 / 128 cases;
  - arrow-ord/src/comparison.rs `test_decimal32/64/128` and `test_decimal32/128_scalar` (:3294-3460);
  - arrow-select/src/take.rs `test_take_decimal128*` (:1263-1300), which pin the 16-byte take path.
The reference has no literal decimal sum / min / max vectors, so `aggregate` holds hand-derived edge cases (a wrap at
2^127, i128::MIN / MAX, all-null, empty); their expectations are exact integer arithmetic: sum wraps in i128.

Run: python tests/golden/make_golden_decimal.py
"""
import json
import os

I128_MAX = (1 << 127) - 1
I128_MIN = -(1 << 127)


def dec(w, p, s, values):
    return {"width": w, "precision": p, "scale": s, "values": values}


def arith():
    a = dec(16, 12, 3, [15, 0, -577, 334, -78, 3])
    b = dec(16, 12, 1, [54, 34, -356, 3, 6, 745])
    cases = [
        {"op": "add", "a": a, "b": b, "type": [15, 3], "values": [5415, 3400, -36177, 634, 522, 74503]},
        {"op": "sub", "a": a, "b": b, "type": [15, 3], "values": [-5385, -3400, 35023, 34, -678, -74497]},
        {"op": "mul", "a": a, "b": b, "type": [25, 4], "values": [810, 0, 205412, 1002, -468, 2235]},
        {"op": "div", "a": a, "b": b, "type": [17, 7], "values": [27777, 0, 162078, 11133333, -1300000, 402]},
        {"op": "rem", "a": a, "b": b, "type": [12, 3], "values": [15, 0, -577, 34, -78, 3]},
    ]
    b37 = dec(16, 37, 37, [1])
    cases += [
        {"op": "mul", "a": dec(16, 3, 3, [1]), "b": b37, "error": "InvalidArgument",
         "message": "Invalid argument error: Output scale of Decimal128(3, 3) * Decimal128(37, 37) would exceed max scale of 38"},
        {"op": "add", "a": dec(16, 3, -2, [1]), "b": b37, "error": "ArithmeticOverflow",
         "message": "Arithmetic overflow: Overflow happened on: 10 ^ 39"},
        {"op": "add", "a": dec(16, 3, -1, [10]), "b": b37, "error": "ArithmeticOverflow",
         "message": "Arithmetic overflow: Overflow happened on: 10 * 100000000000000000000000000000000000000"},
        {"op": "div", "a": dec(16, 3, -1, [10]), "b": dec(16, 1, 1, [0]), "error": "DivideByZero",
         "message": "Divide by zero error"},
        {"op": "rem", "a": dec(16, 3, -1, [10]), "b": dec(16, 1, 1, [0]), "error": "DivideByZero",
         "message": "Divide by zero error"},
    ]
    return cases


def neg():
    return [{"a": dec(w, 9, 6, [1, 3, -44, 2, 4]), "values": [-1, -3, 44, -2, -4]} for w in (4, 8, 16)]


def cmp():
    out = []
    for w in (4, 8, 16):  # test_decimal32 / 64 / 128
        a, b = [1, 2, 4, 5], [7, -3, 4, 3]
        for op, e in (("eq", [False, False, True, False]), ("lt", [True, False, False, False]),
                      ("lt_eq", [True, False, True, False]), ("gt", [False, True, False, True]),
                      ("gt_eq", [False, True, True, True])):
            out.append({"width": w, "op": op, "a": a, "b": b, "b_scalar": False, "expected": e})
    for w in (4, 16):  # test_decimal32_scalar / test_decimal128_scalar
        a = [1, 2, 3, None, 4, 5]
        for op, e in (("eq", [False, False, True, None, False, False]), ("neq", [True, True, False, None, True, True]),
                      ("lt", [True, True, False, None, False, False]), ("lt_eq", [True, True, True, None, False, False]),
                      ("gt", [False, False, False, None, True, True]), ("gt_eq", [False, False, True, None, True, True])):
            out.append({"width": w, "op": op, "a": a, "b": [3], "b_scalar": True, "expected": e})
    return out


def take():
    return [
        {"precision": 10, "scale": 5, "values": [None, 3, 5, 2, 3, None], "indices": [0, 5, 3, 1, 4, 2],
         "expected": [None, None, 2, 3, 3, 5]},
        {"precision": 10, "scale": 5, "values": [0, 1, 2, 3, 4], "indices": [3, None, 1, 3, 2],
         "expected": [3, None, 1, 3, 2]},
    ]


def aggregate():
    return [
        {"name": "wrap at 2^127", "values": [I128_MAX, 1], "sum": I128_MIN, "min": 1, "max": I128_MAX},
        {"name": "wrap below -2^127", "values": [I128_MIN, -1, None], "sum": I128_MAX, "min": I128_MIN, "max": -1},
        {"name": "min and max of i128", "values": [0, I128_MIN, None, I128_MAX, -5], "sum": -6, "min": I128_MIN, "max": I128_MAX},
        {"name": "all null", "values": [None, None, None], "sum": None, "min": None, "max": None},
        {"name": "empty", "values": [], "sum": None, "min": None, "max": None},
        {"name": "single", "values": [-(10 ** 37)], "sum": -(10 ** 37), "min": -(10 ** 37), "max": -(10 ** 37)},
    ]


def main():
    doc = {"arith": arith(), "neg": neg(), "cmp": cmp(), "take": take(), "aggregate": aggregate()}
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "decimal_vectors.json")
    with open(path, "w") as f:
        json.dump(doc, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
