"""Writes tests/golden/substring_vectors.json: the literal tables of the reference's length / bit_length / substring /
substring_by_char tests (arrow-string/src/length.rs and substring.rs test modules), transcribed as data. Values are
lists of hex strings (None = null); `expected` is what the reference asserts (logical values). Error cases keep the
reference's message text.

    python tests/golden/make_golden_substring.py
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))


def h(items):
    return [None if x is None else (x.encode() if isinstance(x, str) else bytes(x)).hex() for x in items]


def grid(kind, typ, fn, inp, rows):
    return [{"kind": kind, "types": typ, "fn": fn, "input": h(inp), "start": s, "length": ln, "expected": h(exp)}
            for s, ln, exp in rows]


def build():
    cases = []
    # substring.rs with_nulls_generic_binary / without_nulls_generic_binary (Binary, LargeBinary)
    bn = [b"hello", None, bytes([0xf8, 0xf9, 0xff, 0xfa])]
    cases += grid("bytes", ["binary", "large_binary"], "substring", [None, None, None], [(-1, 1, [None, None, None])])
    cases += grid("bytes", ["binary", "large_binary"], "substring", bn, [
        (0, None, bn), (0, 0, [b"", None, b""]), (1000, 0, [b"", None, b""]), (-1000, None, bn), (0, 1000, bn)])
    bw = [b"hello", b"", bytes([0xf8, 0xf9, 0xff, 0xfa])]
    cases += grid("bytes", ["binary", "large_binary"], "substring", [b"", b"", b""], [(2, 1, [b"", b"", b""])])
    cases += grid("bytes", ["binary", "large_binary"], "substring", bw, [
        (0, None, bw), (1, None, [b"ello", b"", bytes([0xf9, 0xff, 0xfa])]), (2, None, [b"llo", b"", bytes([0xff, 0xfa])]),
        (3, None, [b"lo", b"", bytes([0xfa])]), (10, None, [b"", b"", b""]), (-1, None, [b"o", b"", bytes([0xfa])]),
        (-2, None, [b"lo", b"", bytes([0xff, 0xfa])]), (-3, None, [b"llo", b"", bytes([0xf9, 0xff, 0xfa])]), (-10, None, bw),
        (1, 1, [b"e", b"", bytes([0xf9])]), (1, 2, [b"el", b"", bytes([0xf9, 0xff])]), (1, 3, [b"ell", b"", bytes([0xf9, 0xff, 0xfa])]),
        (1, 4, [b"ello", b"", bytes([0xf9, 0xff, 0xfa])]), (-3, 1, [b"l", b"", bytes([0xf9])]), (-3, 2, [b"ll", b"", bytes([0xf9, 0xff])]),
        (-3, 3, [b"llo", b"", bytes([0xf9, 0xff, 0xfa])]), (-3, 4, [b"llo", b"", bytes([0xf9, 0xff, 0xfa])])])
    # with_nulls_generic_string / without_nulls_generic_string (Utf8, LargeUtf8)
    sn = ["hello", None, "word"]
    cases += grid("bytes", ["utf8", "large_utf8"], "substring", [None, None, None], [(0, None, [None, None, None])])
    cases += grid("bytes", ["utf8", "large_utf8"], "substring", sn, [
        (0, None, sn), (0, 0, ["", None, ""]), (1000, 0, ["", None, ""]), (-1000, None, sn), (0, 1000, sn)])
    sw = ["hello", "", "word"]
    cases += grid("bytes", ["utf8", "large_utf8"], "substring", ["", "", ""], [(0, None, ["", "", ""])])
    cases += grid("bytes", ["utf8", "large_utf8"], "substring", sw, [
        (0, None, sw), (1, None, ["ello", "", "ord"]), (2, None, ["llo", "", "rd"]), (3, None, ["lo", "", "d"]),
        (10, None, ["", "", ""]), (-1, None, ["o", "", "d"]), (-2, None, ["lo", "", "rd"]), (-3, None, ["llo", "", "ord"]),
        (-10, None, sw), (1, 1, ["e", "", "o"]), (1, 2, ["el", "", "or"]), (1, 3, ["ell", "", "ord"]), (1, 4, ["ello", "", "ord"]),
        (-3, 1, ["l", "", "o"]), (-3, 2, ["ll", "", "or"]), (-3, 3, ["llo", "", "ord"]), (-3, 4, ["llo", "", "ord"])])
    # substring_by_char: with_nulls / without_nulls / ascii (Utf8, LargeUtf8)
    cn = ["hello", None, "Γ ⊢x:T"]
    cases += grid("bytes", ["utf8", "large_utf8"], "substring_by_char", [None, None, None], [(0, None, [None, None, None])])
    cases += grid("bytes", ["utf8", "large_utf8"], "substring_by_char", cn, [
        (0, None, cn), (0, 0, ["", None, ""]), (1000, 0, ["", None, ""]), (-1000, None, cn), (0, 1000, cn)])
    cw = ["hello", "", "Γ ⊢x:T"]
    cases += grid("bytes", ["utf8", "large_utf8"], "substring_by_char", ["", "", ""], [(0, None, ["", "", ""])])
    cases += grid("bytes", ["utf8", "large_utf8"], "substring_by_char", cw, [
        (0, None, cw), (1, None, ["ello", "", " ⊢x:T"]), (2, None, ["llo", "", "⊢x:T"]), (3, None, ["lo", "", "x:T"]),
        (10, None, ["", "", ""]), (-1, None, ["o", "", "T"]), (-2, None, ["lo", "", ":T"]), (-4, None, ["ello", "", "⊢x:T"]),
        (-10, None, cw), (1, 1, ["e", "", " "]), (1, 2, ["el", "", " ⊢"]), (1, 3, ["ell", "", " ⊢x"]), (1, 6, ["ello", "", " ⊢x:T"]),
        (-4, 1, ["e", "", "⊢"]), (-4, 2, ["el", "", "⊢x"]), (-4, 3, ["ell", "", "⊢x:"]), (-4, 4, ["ello", "", "⊢x:T"])])
    ca = ["hello", None, "", "rust"]
    cases += grid("bytes", ["utf8", "large_utf8"], "substring_by_char", ca, [
        (0, None, ca), (1, None, ["ello", None, "", "ust"]), (4, None, ["o", None, "", ""]), (1000, None, ["", None, "", ""]),
        (-1, None, ["o", None, "", "t"]), (-4, None, ["ello", None, "", "rust"]), (-1000, None, ca), (0, 0, ["", None, "", ""]),
        (1, 2, ["el", None, "", "us"]), (-4, 2, ["el", None, "", "ru"]), (0, 1000, ca), (1, 2**64 - 1, ["ello", None, "", "ust"])])
    # FixedSizeBinary: with_nulls / without_nulls
    fn_ = [b"cat", None, bytes([0xf8, 0xf9, 0xff])]
    cases += grid("fsb", ["fixed_size_binary"], "substring", [None, None, None], [(3, 2, [None, None, None])])
    fw = [b"cat", b"dog", bytes([0xf8, 0xf9, 0xff])]
    for inp in (fn_, fw):
        f = lambda k: [None if x is None else x[k] for x in inp]  # noqa: E731
        cases += grid("fsb", ["fixed_size_binary"], "substring", inp, [
            (0, None, inp), (1, None, f(slice(1, None))), (2, None, f(slice(2, None))), (3, None, f(slice(3, None))),
            (10, None, f(slice(3, None))), (-1, None, f(slice(2, None))), (-2, None, f(slice(1, None))), (-3, None, inp),
            (-10, None, inp), (1, 1, f(slice(1, 2))), (1, 2, f(slice(1, 3))), (1, 3, f(slice(1, 3))), (-3, 1, f(slice(0, 1))),
            (-3, 2, f(slice(0, 2))), (-3, 3, inp), (-3, 4, inp)])
    cases += grid("fsb", ["fixed_size_binary"], "substring", [b"", b"", b""], [(1, 2, [b"", b"", b""])])
    # *_with_non_zero_offset: the array [v0, v1, v2] with validity 0b101, sliced to rows 1..3
    for typ, fn, vals, offs, start, exp in [
            (["binary", "large_binary"], "substring", list(range(15)), [0, 5, 10, 15], 1, [None, bytes([11, 12, 13, 14])]),
            (["utf8", "large_utf8"], "substring", list(b"hellotherearrow"), [0, 5, 10, 15], 1, [None, b"rrow"]),
            (["utf8", "large_utf8"], "substring_by_char", list("S→T = Πx:S.T".encode()), [0, 5, 8, 15], 1,
             [None, "x:S.T"])]:
        cases.append({"kind": "sliced", "types": typ, "fn": fn, "data": bytes(vals).hex(), "offsets": offs, "valid": [True, False, True],
                      "slice": [1, 2], "start": start, "length": None, "expected": h(exp)})
    cases.append({"kind": "fsb_sliced", "types": ["fixed_size_binary"], "fn": "substring", "data": b"hellotherearrow".hex(), "width": 5,
                  "valid": [True, False, True], "slice": [1, 2], "start": 1, "length": None, "expected": h([None, b"rrow"])})
    # check_start_index / check_length / non_utf8_bytes
    for s, ln in [(-1, None), (0, 5)]:
        cases.append({"kind": "bytes", "types": ["utf8"], "fn": "substring", "input": h(["E=mc²", "ascii"]), "start": s, "length": ln,
                      "error": "invalid utf-8 boundary"})
    cases += grid("bytes", ["binary"], "substring", [bytes([0xE4, 0xBD, 0xA0, 0xE5, 0xA5, 0xBD, 0xE8, 0xAF, 0xAD])],
                  [(0, 5, [bytes([0xE4, 0xBD, 0xA0, 0xE5, 0xA5])])])
    # string_view_matches_utf8 / binary_view_matches_binary: the view result equals the Utf8 / Binary one
    vs = ["hello world", "", None, "a", "this one is definitely longer than twelve bytes"]
    for s, ln in [(0, None), (0, 0), (0, 5), (0, 1000), (1, 3), (5, None), (100, 2), (100, None), (-3, None), (-3, 2), (-100, 4), (-100, None)]:
        cases.append({"kind": "view_matches", "types": ["utf8"], "fn": "substring", "input": h(vs), "start": s, "length": ln})
    vb = [b"hello world", b"", None, b"abc", b"this one is definitely longer than twelve bytes"]
    for s, ln in [(0, None), (0, 5), (2, 3), (-3, None), (100, 2)]:
        cases.append({"kind": "view_matches", "types": ["binary"], "fn": "substring", "input": h(vb), "start": s, "length": ln})
    vm = ["héllo wörld", "日本語", None]
    for s, ln in [(0, 3), (3, 3), (0, 6), (-3, None), (-6, 3)]:
        cases.append({"kind": "view_matches", "types": ["utf8"], "fn": "substring", "input": h(vm), "start": s, "length": ln})
    # string_view_rejects_an_invalid_char_boundary: "héllo" starts 'h', then the 2-byte 'é'
    cases.append({"kind": "view", "types": ["utf8_view"], "fn": "substring", "input": h(["héllo"]), "start": 2, "length": None,
                  "error": "The offset 2 is at an invalid utf-8 boundary."})
    # length.rs: length / bit_length case tables
    for typ in (["utf8", "large_utf8", "binary", "large_binary", "utf8_view", "binary_view"],):
        cases.append({"kind": "length", "types": typ, "fn": "length", "input": h(["hello", " ", None]), "expected": [5, 1, None]})
        cases.append({"kind": "length", "types": typ, "fn": "length", "input": h(["one", "on", "o", ""]), "expected": [3, 2, 1, 0]})
        cases.append({"kind": "length", "types": typ, "fn": "length", "input": h(["💖"]), "expected": [4]})
        cases.append({"kind": "length", "types": typ, "fn": "bit_length", "input": h(["one", "on", "o", ""]), "expected": [24, 16, 8, 0]})
        cases.append({"kind": "length", "types": typ, "fn": "bit_length", "input": h(["one", None, "", "two"]), "expected": [24, None, 0, 24]})
        cases.append({"kind": "length", "types": typ, "fn": "bit_length", "input": h(["💖"]), "expected": [32]})
    cases.append({"kind": "length", "types": ["fixed_size_binary"], "fn": "length", "input": h([b"one", None, b"two"]), "expected": [3, None, 3]})
    cases.append({"kind": "length", "types": ["fixed_size_binary"], "fn": "bit_length", "input": h([b"one", None, b"two"]),
                  "expected": [24, None, 24]})
    # length_offsets_string / bit_length_offsets_string: ["hello", " ", "world", null].slice(1, 3)
    for fn, exp in [("length", [1, 5, None]), ("bit_length", [8, 40, None])]:
        cases.append({"kind": "length_sliced", "types": ["utf8", "large_utf8", "binary", "large_binary"], "fn": fn,
                      "input": h(["hello", " ", "world", None]), "slice": [1, 3], "expected": exp})
    for i, c in enumerate(cases):
        c["id"] = f"{c['fn']}-{c['kind']}-{i}"
    return cases


if __name__ == "__main__":
    out = os.path.join(HERE, "substring_vectors.json")
    with open(out, "w") as f:
        json.dump({"source": "arrow-string/src/length.rs, arrow-string/src/substring.rs test modules", "cases": build()}, f, indent=0)
        f.write("\n")
    print(out)
