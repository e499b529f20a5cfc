"""Writes tests/golden/bitwise_vectors.json: the literal cases of the reference's bitwise tests (arrow-arith/src/bitwise.rs
test module) and of its product / product_checked / bit_and / bit_or / bit_xor tests (arrow-arith/src/aggregate.rs),
transcribed as data with the file:line of each. Values are integers or floats (None = null); `expected` is what the
reference asserts; an `error` case only asserts that an error is returned.

    python tests/golden/make_golden_bitwise.py
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
U64MAX = 2**64 - 1
I32MAX = 2**31 - 1


def bw(src, fn, dtype, left, right, expected, scalar=None):
    return {"src": "arrow-arith/src/bitwise.rs:" + str(src), "fn": fn, "dtype": dtype, "left": left, "right": right,
            "scalar": scalar, "expected": expected}


def agg(src, fn, dtype, values, expected=None, error=False):
    return {"src": "arrow-arith/src/aggregate.rs:" + str(src), "fn": fn, "dtype": dtype, "values": values,
            "expected": expected, "error": error}


def build():
    n = None
    bitwise = [
        bw(213, "and", "uint64", [1, 2, n, 4], [5, 10, 8, 12], [1, 2, n, 4]),
        bw(220, "and", "int32", [1, 2, n, 4], [5, -10, 8, 12], [1, 2, n, 4]),
        bw(230, "shift_left", "uint64", [1, 2, n, 4, 8], [5, 10, 8, 12, U64MAX], [32, 2048, n, 16384, 0]),
        bw(239, "shift_left", "uint64", [1, 2, n, 4, 8], None, [4, 8, n, 16, 32], scalar=2),
        bw(248, "shift_right", "uint64", [32, 2048, n, 16384, 3], [5, 10, 8, 12, 65], [1, 2, n, 4, 1]),
        bw(257, "shift_right", "uint64", [32, 2048, n, 16384, 3], None, [8, 512, n, 4096, 0], scalar=2),
        bw(267, "and", "uint64", [15, 2, n, 4], None, [7, 2, n, 4], scalar=7),
        bw(274, "and", "int32", [1, 2, n, 4], None, [0, 0, n, 4], scalar=-20),
        bw(284, "or", "uint64", [1, 2, n, 4], [7, 5, 8, 13], [7, 7, n, 13]),
        bw(291, "or", "int32", [1, 2, n, 4], [-7, -5, 8, 13], [-7, -5, n, 13]),
        bw(301, "not", "uint64", [1, 2, n, 4], None, [18446744073709551614, 18446744073709551613, n, 18446744073709551611]),
        bw(311, "not", "int32", [1, 2, n, 4], None, [-2, -3, n, -5]),
        bw(320, "and_not", "uint64", [8, 2, n, 4], [7, 5, 8, 13], [8, 2, n, 0]),
        bw(331, "and_not", "int32", [2, 1, n, 3], [-7, -5, 8, 13], [2, 0, n, 2]),
        bw(345, "or", "uint64", [15, 2, n, 4], None, [15, 7, n, 7], scalar=7),
        bw(352, "or", "int32", [1, 2, n, 4], None, [21, 22, n, 20], scalar=20),
        bw(362, "xor", "uint64", [1, 2, n, 4], [7, 5, 8, 13], [6, 7, n, 9]),
        bw(369, "xor", "int32", [1, 2, n, 4], [-7, 5, 8, -13], [-8, 7, n, -9]),
        bw(379, "xor", "uint64", [15, 2, n, 4], None, [8, 5, n, 3], scalar=7),
        bw(386, "xor", "int32", [1, 2, n, 4], None, [-19, -18, n, -24], scalar=-20),
    ]
    aggregates = [
        agg(1052, "product", "int32", [1, 2, 3, 4, 5], 120),
        agg(1058, "product", "float64", [1.0, 2.0, 3.0, 4.0, 5.0], 120.0),
        agg(1064, "product", "int32", [n, 2, 3, n, 5], 30),
        agg(1070, "product", "int32", [n, n, n], None),
        agg(1076, "product", "int32", [], None),
        agg(1082, "product_checked", "int32", [1, 2, 3, 4, 5], 120),
        agg(1088, "product_checked", "int32", [n, 2, 3, n, 5], 30),
        agg(1094, "product_checked", "int32", [n, n, n], None),
        agg(1100, "product", "int32", [I32MAX, 2], -2),
        agg(1107, "product_checked", "int32", [I32MAX, 2], error=True),
        agg(1210, "bit_and", "int32", [1, 2, 3, 4, 5], 0),
        agg(1216, "bit_and", "int32", [n, 2, 3, n, n], 2),
        agg(1222, "bit_and", "int32", [n, n, n], None),
        agg(1228, "bit_or", "int32", [1, 2, 3, 4, 5], 7),
        agg(1234, "bit_or", "int32", [n, 2, 3, n, 5], 7),
        agg(1240, "bit_or", "int32", [n, n, n], None),
        agg(1246, "bit_xor", "int32", [1, 2, 3, 4, 5], 1),
        agg(1252, "bit_xor", "int32", [n, 2, 3, n, 5], 4),
        agg(1258, "bit_xor", "int32", [n, n, n], None),
    ]
    return {"bitwise": bitwise, "aggregate": aggregates}


if __name__ == "__main__":
    with open(os.path.join(HERE, "bitwise_vectors.json"), "w") as f:
        json.dump(build(), f, indent=1)
        f.write("\n")
