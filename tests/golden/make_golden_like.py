#!/usr/bin/env python
"""Transcribes the reference's literal LIKE-family tests (arrow-string/src/like.rs and predicate.rs, apache/arrow-rs @
cd7c6b83) into tests/golden/like_vectors.json.

Nothing here runs the reference: every case is a literal input -> literal expected output copied from the cited test.
The tables are long (like_escape_many alone has 729 rows), so they are read out of the Rust test source rather than retyped:
`python tests/golden/make_golden_like.py <arrow-rs checkout>` regenerates the committed JSON.

The JSON keeps the literal tables as the tests write them (null = Arrow null); tests/like_util.py expands them into cases
with the array forms each reference test runs them on (dictionary forms left out).
"""
import json
import os
import re
import sys

L = "arrow-string/src/like.rs"
P = "arrow-string/src/predicate.rs"
STR_TYPES = ["utf8", "large_utf8", "utf8_view"]
BIN_TYPES = ["binary", "large_binary"]


# ---- a reader for the Rust literals these tests use --------------------------------------------------------------------
def rust_string(src, i):
    """(value, next index) of the string literal at src[i]: "...", r"..." or r#"..."#."""
    if src.startswith('r#"', i):
        j = src.index('"#', i + 3)
        return src[i + 3:j], j + 2
    if src.startswith('r"', i):
        j = src.index('"', i + 2)
        return src[i + 2:j], j + 1
    assert src[i] == '"', src[i:i + 20]
    out, j = [], i + 1
    while src[j] != '"':
        c = src[j]
        if c == "\\":
            e = src[j + 1]
            if e == "u":
                k = src.index("}", j)
                out.append(chr(int(src[j + 3:k], 16)))
                j = k + 1
                continue
            out.append({"n": "\n", "t": "\t", "r": "\r", "0": "\0", "\\": "\\", '"': '"', "'": "'"}[e])
            j += 2
            continue
        out.append(c)
        j += 1
    return "".join(out), j + 1


TOKEN = re.compile(r'\s*(r#?"|"|Some\(|None|true|false|vec!\[|\[|\]|\(|\)|,|[A-Za-z_][A-Za-z0-9_]*|//[^\n]*)')


def parse_value(src, i):
    """(value, next index): a string, bool, None, Some(x) (= x) or a vec![...] / [...] list."""
    while True:
        m = TOKEN.match(src, i)
        t = m.group(1)
        if t.startswith("//"):
            i = m.end()
            continue
        break
    if t in ('"', 'r"', 'r#"'):
        return rust_string(src, m.start(1))
    if t == "Some(":
        v, i = parse_value(src, m.end())
        return v, expect(src, i, ")")
    if t == "None":
        return None, m.end()
    if t in ("true", "false"):
        return t == "true", m.end()
    if t in ("vec![", "[", "("):
        close = ")" if t == "(" else "]"
        out, i = [], m.end()
        while True:
            if peek(src, i) == close:
                return (tuple(out) if close == ")" else out), expect(src, i, close)
            v, i = parse_value(src, i)
            out.append(v)
            if peek(src, i) == ",":
                i = expect(src, i, ",")
    return t, m.end()  # an identifier (the op)


def peek(src, i):
    while True:
        m = TOKEN.match(src, i)
        if not m.group(1).startswith("//"):
            return m.group(1)
        i = m.end()


def expect(src, i, tok):
    while True:
        m = TOKEN.match(src, i)
        if m.group(1).startswith("//"):
            i = m.end()
            continue
        assert m.group(1) == tok, (tok, src[i:i + 40])
        return m.end()


def line_of(src, i):
    return src.count("\n", 0, i) + 1


def main(root):
    like = open(os.path.join(root, L), encoding="utf-8").read()
    pred = open(os.path.join(root, P), encoding="utf-8").read()
    base = like.index("mod tests")
    out = {"source": f"apache/arrow-rs @ cd7c6b83, {L}, {P}"}

    # test_utf8! / test_utf8_and_binary! / test_utf8_scalar! / test_utf8_and_binary_scalar!: [name, line, macro, op, left, right, expected]
    out["macros"] = []
    for m in re.finditer(r"\n    (test_utf8\w*)!\(\s*(#\[[^\]]*\]\s*)?", like[base:]):
        args, i = [], m.end()
        for k in range(5):
            v, i = parse_value(like[base:], i)
            args.append(v)
            if k < 4:
                i = expect(like[base:], i, ",")
        out["macros"].append([args[0], line_of(like, base + m.start() + 1), m.group(1), args[3], args[1], args[2], args[4]])

    # string_null_like_pattern / string_view_null_like_pattern: the patterns each run against a null haystack
    k = like.index("fn string_null_like_pattern()")
    out["null_haystack_patterns"], _ = parse_value(like, like.index("for pattern in &", k) + len("for pattern in &"))

    # like_escape: (value, pattern, expected) rows; like_escape_many: every value against every pattern, pattern-major
    k = like.index("fn like_escape()")
    out["like_escape"], _ = parse_value(like, like.index("let test_cases = ", k) + len("let test_cases = "))
    k = like.index("fn like_escape_many()")
    table, _ = parse_value(like, like.index("let test_cases = ", k) + len("let test_cases = "))
    values = list(dict.fromkeys(v for v, _, _ in table))
    patterns = list(dict.fromkeys(p for _, p, _ in table))
    assert [(v, p) for v, p, _ in table] == [(v, p) for p in patterns for v in values]
    out["like_escape_many"] = {"values": values, "patterns": patterns, "expected": "".join("1" if e else "0" for _, _, e in table)}

    # predicate.rs tests: assert!(Predicate::X(needle).evaluate(haystack)) / assert!(!...) -> [kind, needle, haystack, expected, line]
    kinds = {"contains": "contains", "StartsWith": "starts_with", "EndsWith": "ends_with", "IStartsWithAscii": "istarts_with_ascii",
             "IEndsWithAscii": "iends_with_ascii"}
    out["predicates"] = []
    for m in re.finditer(r"assert!\((!?)Predicate::(contains|StartsWith|EndsWith|IStartsWithAscii|IEndsWithAscii)\(", pred):
        needle, i = parse_value(pred, m.end())
        i = expect(pred, i, ")")
        assert pred[i:].startswith(".evaluate(")
        hay, i = parse_value(pred, i + len(".evaluate("))
        out["predicates"].append([kinds[m.group(2)], needle, hay, m.group(1) != "!", line_of(pred, m.start())])
    # test_regex_like: [pattern, regex]
    k = pred.index("fn test_regex_like()")
    out["regex_like"], _ = parse_value(pred, pred.index("let test_cases = ", k) + len("let test_cases = "))

    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "like_vectors.json")
    with open(path, "w", encoding="utf-8") as f:  # one entry per line
        f.write("{\n" + ",\n".join(f"{json.dumps(key)}: " + (json.dumps(v, ensure_ascii=False) if not isinstance(v, list) else
                "[\n" + ",\n".join(json.dumps(x, ensure_ascii=False) for x in v) + "]") for key, v in out.items()) + "\n}\n")
    print(f"-> {path}")


if __name__ == "__main__":
    main(sys.argv[1])
