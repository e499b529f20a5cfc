"""Builders shared by the LIKE-family tests: golden forms -> columns, random string / pattern generators."""
import json
import os

import numpy as np

from acu import ViewColumn

from oracle_like import OPS
from test_oracle_cmp_bytes import utf8_column

STRING_FORMS = ["utf8", "large_utf8", "utf8_view"]
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "like_vectors.json")


def golden_cases():
    """The reference's literal cases (tests/golden/like_vectors.json) as dicts: a row case has op / left / right / forms
    ("<type>:<shape>", shape = array_array | array_scalar | scalar_array | scalar_scalar) / expected rows; a predicate case
    has predicate / needle / haystack / expected; a regex case has regex_like / regex."""
    with open(GOLDEN, encoding="utf-8") as f:
        g = json.load(f)
    L, P = "arrow-string/src/like.rs", "arrow-string/src/predicate.rs"
    cases = []
    for name, line, macro, op, left, right, expected in g["macros"]:  # like.rs:466-644
        scalar = macro.endswith("_scalar")
        types = STRING_FORMS + (["binary", "large_binary"] if "binary" in macro else [])
        cases.append({"id": name, "ref": f"{L}:{line}", "op": op, "left": left, "right": [right] if scalar else right,
                      "forms": [f"{t}:{'array_scalar' if scalar else 'array_array'}" for t in types], "expected": expected})
    every_shape = ("scalar_scalar", "scalar_array", "array_array", "array_scalar")
    for t, fn in (("utf8", "string"), ("utf8_view", "string_view")):  # like.rs:1438-1596
        for op in ("like", "ilike", "nlike", "nilike"):
            for p in g["null_haystack_patterns"]:
                cases.append({"id": f"{fn}_null_like_pattern_{op}_{p!r}", "ref": L, "op": op, "left": [None], "right": [p],
                              "forms": [f"{t}:{s}" for s in every_shape], "expected": [None]})
            cases.append({"id": f"{fn}_like_scalar_null_{op}", "ref": L, "op": op, "left": ["a"], "right": [None],
                          "forms": [f"{t}:{s}" for s in every_shape], "expected": [None]})
    many = g["like_escape_many"]
    rows = [(v, p) for p in many["patterns"] for v in many["values"]]
    for op, neg in (("like", False), ("ilike", False), ("nlike", True), ("nilike", True)):  # like.rs:1598-2607
        for j, (v, p, e) in enumerate(g["like_escape"]):
            cases.append({"id": f"like_escape_{op}_{j}", "ref": L, "op": op, "left": [v], "right": [p],
                          "forms": [f"{t}:{s}" for t in STRING_FORMS for s in ("array_array", "scalar_scalar")], "expected": [e != neg]})
        cases.append({"id": f"like_escape_many_{op}", "ref": L, "op": op, "left": [v for v, _ in rows], "right": [p for _, p in rows],
                      "forms": [f"{t}:array_array" for t in STRING_FORMS], "expected": [(e == "1") != neg for e in many["expected"]]})
    for kind, needle, hay, expected, line in g["predicates"]:
        cases.append({"id": f"predicate_{kind}_{line}", "ref": f"{P}:{line}", "predicate": kind, "needle": needle, "haystack": hay,
                      "expected": expected})
    for j, (pat, rx) in enumerate(g["regex_like"]):
        cases.append({"id": f"regex_like_{j}", "ref": P, "regex_like": pat, "regex": rx})
    return cases


def enc(items):
    return [None if x is None else (x.encode() if isinstance(x, str) else bytes(x)) for x in items]


def column(typ, items, scalar=False, block=64):
    """A Utf8Column / ViewColumn of `typ` (utf8, large_utf8, utf8_view, binary, large_binary, binary_view)."""
    items = enc(items)
    if typ.endswith("view"):
        return ViewColumn.from_values(items, block, scalar=scalar)
    return utf8_column(items, typ.startswith("large"), scalar)


def run(backend, op, typ, l, r):
    """like_bytes / like_view of `backend` on two columns of `typ`."""
    is_utf8 = typ.endswith("utf8") or typ == "utf8_view"
    if typ.endswith("view"):
        return backend.like_view(op, l, r, is_utf8)
    return backend.like_bytes(op, l, r, is_utf8)


def run_form(backend, case, form):
    """The golden case on one of its forms ("<type>:<shape>")."""
    typ, shape = form.split(":")
    ls, rs = shape.startswith("scalar"), shape.endswith("scalar")
    left = case["left"][:1] if ls else case["left"]
    right = case["right"][:1] if rs else case["right"]
    return run(backend, OPS[case["op"]], typ, column(typ, left, ls), column(typ, right, rs))


def rand_utf8(rng, n, alphabet, max_len, null_p=None):
    out = []
    for _ in range(n):
        if null_p is not None and rng.random() < null_p:
            out.append(None)
            continue
        k = int(rng.integers(0, max_len + 1))
        out.append("".join(alphabet[int(j)] for j in rng.integers(0, len(alphabet), k)))
    return out
