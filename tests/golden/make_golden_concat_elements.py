"""Writes tests/golden/concat_elements_vectors.json: every literal case of the reference's concat_elements tests
(arrow-string/src/concat_elements.rs test module), transcribed as data. Values are lists of hex strings (None = null);
`expected` is what the reference asserts (logical values). Error cases keep the reference's asserted `to_string()` text
(the ArrowError Display), and its ArrowError variant as `status`.

Case fields: `fn` is "dyn" (concat_elements_dyn of `left` / `right`, typed `types` = [left type, right type]) or "many"
(concat_elements_utf8_many of `arrays`); `slices` ([offset, length] per operand) slices the operands first; FixedSizeBinary
operands carry their widths in `widths`.

    python tests/golden/make_golden_concat_elements.py
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
COMPUTE, NOT_YET_IMPLEMENTED = 2, 7


def h(items):
    return [None if x is None else (x.encode() if isinstance(x, str) else bytes(x)).hex() for x in items]


def dyn(cid, typ, left, right, expected=None, error=None, widths=None, slices=None, rtyp=None):
    c = {"id": cid, "fn": "dyn", "types": [typ, rtyp or typ], "left": h(left), "right": h(right)}
    if widths is not None:
        c["widths"] = widths
    if slices is not None:
        c["slices"] = slices
    if error is not None:
        c["error"], c["status"] = error
    else:
        c["expected"] = h(expected)
    return c


def many(cid, arrays, expected=None, error=None):
    c = {"id": cid, "fn": "many", "types": ["utf8"], "arrays": [h(a) for a in arrays]}
    if error is not None:
        c["error"], c["status"] = error
    else:
        c["expected"] = h(expected)
    return c


def build():
    long = "ThisStringIsLongerThan12Bytes"
    fbb = ["foo", "bar", None]
    nyz = [None, "yyy", "zzz"]
    n_baryyy_n = [None, "baryyy", None]
    view_l = ["foo", "bar", None, "foofoofoo", "foo", long, long]
    view_r = [None, "yyy", "zzz", "barbarbar", long, "bar", long]
    view_e = [None, "baryyy", None, "foofoofoobarbarbar", "foo" + long, long + "bar", long + long]
    len_err = ("Compute error: Arrays must have the same length: 2 != 1", COMPUTE)
    return [
        dyn("string_concat", "utf8", fbb, nyz, n_baryyy_n),
        dyn("string_concat_empty_string", "utf8", ["foo", "", "bar"], ["baz", "", ""], ["foobaz", "", "bar"]),
        dyn("string_concat_no_null", "utf8", ["foo", "bar"], ["bar", "baz"], ["foobar", "barbaz"]),
        dyn("string_concat_error", "utf8", ["foo", "bar"], ["baz"], error=len_err),
        dyn("string_concat_slice_1", "utf8", [None, "foo", "bar", "baz"], ["boo", None, "far", "faz"], [None, "foofar", "barfaz"],
            slices=[[0, 3], [1, 3]]),
        dyn("string_concat_slice_2", "utf8", [None, "foo", "bar", "baz"], ["boo", None, "far", "faz"], [None, "bazfar"],
            slices=[[2, 2], [1, 2]]),
        many("string_concat_error_empty", [], error=("Compute error: concat requires input of at least one array", COMPUTE)),
        many("string_concat_one", [n_baryyy_n], n_baryyy_n),
        many("string_concat_many", [["f", "o", "o", None], [None, "b", "a", "r"], ["b", None, "a", "z"]], [None, None, "oaa", None]),
        dyn("fixed_size_binary_concat", "fixed_size_binary", fbb, nyz, n_baryyy_n, widths=[3, 3]),
        dyn("mixed_fixed_size_binary_concat", "fixed_size_binary", ["foobar", "barbaz", None], nyz, [None, "barbazyyy", None],
            widths=[6, 3]),
        dyn("fixed_size_binary_concat_no_null", "fixed_size_binary", ["ab", "cd"], ["12", "34"], ["ab12", "cd34"], widths=[2, 2]),
        dyn("fixed_size_binary_concat_error", "fixed_size_binary", ["ab", "cd"], ["12"], error=len_err, widths=[2, 2]),
        dyn("fixed_size_binary_concat_empty", "fixed_size_binary", [], [], [], widths=[0, 0]),
        dyn("binary_view_concat", "binary_view", view_l, view_r, view_e),
        dyn("string_view_concat_1", "utf8_view", view_l, view_r, view_e),
        dyn("string_view_concat_2", "utf8_view", ["a", "b", "foofoofoo", "a", long, long], ["c", "d", "barbarbar", long, "d", long],
            ["ac", "bd", "foofoofoobarbarbar", "a" + long, long + "d", long + long]),
        dyn("binary_view_concat_no_null", "binary_view", ["foo", "bar", "", "baz"], ["bar", "baz", "", ""], ["foobar", "barbaz", "", "baz"]),
        dyn("binary_view_concat_error", "binary_view", ["foo", "bar"], ["baz"], error=len_err),
        dyn("binary_view_concat_empty", "binary_view", [], [], []),
        dyn("concat_dyn_same_type_utf8", "utf8", fbb, nyz, n_baryyy_n),
        dyn("concat_dyn_same_type_large_utf8", "large_utf8", fbb, nyz, n_baryyy_n),
        dyn("concat_dyn_same_type_binary", "binary", fbb, nyz, n_baryyy_n),
        dyn("concat_dyn_same_type_large_binary", "large_binary", fbb, nyz, n_baryyy_n),
        dyn("concat_dyn_same_type_binary_view", "binary_view", view_l, view_r, view_e),
        dyn("concat_dyn_same_type_utf8_view", "utf8_view", view_l, view_r, view_e),
        dyn("concat_dyn_same_type_fixed_size_binary", "fixed_size_binary", fbb, nyz, n_baryyy_n, widths=[3, 3]),
        dyn("concat_dyn_different_type", "utf8", fbb, [None, "1", "2"], rtyp="large_utf8",
            error=("Compute error: Cannot concat arrays of different types: Utf8 != LargeUtf8", COMPUTE)),
    ]


if __name__ == "__main__":
    cases = build()
    with open(os.path.join(HERE, "concat_elements_vectors.json"), "w") as f:
        json.dump({"source": "arrow-string/src/concat_elements.rs (tests :478-956)", "cases": cases}, f, indent=1)
        f.write("\n")
    print(f"{len(cases)} cases")
