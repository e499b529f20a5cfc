"""CPU: the LIKE-family oracle (tests/oracle_like.py) pinned against the reference's literal vectors
(tests/golden/like_vectors.json: like.rs's test macros, like_escape / like_escape_many, the null tests, predicate.rs),
against the reference's case-folding examples, and, as a cross-check only, case-sensitive LIKE on ASCII data against
Python's `re` running regex_like's translation of the pattern."""
import re

import numpy as np
import pytest

import acu
from acu import _abi as abi

from like_util import column, golden_cases, rand_utf8, run, run_form
from oracle_like import LikeOracle, evaluate, glob_match, regex_like

ORACLE = LikeOracle()
CASES = golden_cases()
ROW_CASES = [c for c in CASES if "op" in c]


@pytest.mark.parametrize("case", ROW_CASES, ids=[c["id"] for c in ROW_CASES])
def test_oracle_golden_rows(case):
    for form in case["forms"]:
        got = run_form(ORACLE, case, form).to_list()
        assert got == case["expected"], f"{case['id']} on {form}"


def test_oracle_golden_predicates_and_regex_translation():
    n = 0
    for c in CASES:
        if "predicate" in c:
            assert evaluate((c["predicate"], c["needle"]), c["haystack"].encode()) == c["expected"], c["id"]
            n += 1
        elif "regex_like" in c:
            assert regex_like(c["regex_like"]) == c["regex"], c["id"]
            n += 1
    assert n == 81


def test_oracle_simple_case_folding():
    """like.rs:1063-1198 (loose matching: ﬀ is not FF, ß is not SS) and the simple folds that reach ASCII."""
    assert glob_match("k", "K", True) and glob_match("K", "K", True)
    assert glob_match("s", "ſ", True) and glob_match("%S%", "xſy", True)
    assert not glob_match("i", "ı", True)  # ı folds with status T only, though "ı".upper() == "I"
    assert not glob_match("ss", "ß", True) and not glob_match("ff", "ﬀ", True)
    assert not glob_match("k", "K", False)
    assert glob_match("_", "😈", False) and not glob_match("__", "😈", False)


@pytest.mark.parametrize("seed", range(3))
def test_oracle_like_matches_python_re_on_ascii(seed):
    """Cross-check only: the glob restatement against Python's re on regex_like's literal translation (ASCII data)."""
    rng = np.random.default_rng(seed)
    pats = rand_utf8(rng, 300, ["a", "b", "%", "_", "\\", ".", "*", "$"], 7)
    hays = rand_utf8(rng, 60, ["a", "b", ".", "*", "\\", "$", "\n", "%", "_"], 8)
    for p in pats:
        rx = re.compile(regex_like(p, r"\Z"), re.DOTALL)
        for h in hays:
            assert glob_match(p, h, False) == (rx.search(h) is not None), (p, h)


def test_oracle_view_is_ascii_quirk():
    """A view whose valid slots are ASCII takes ilike's IEqAscii fast path at the null slots too: a null K (U+212A) gives
    value bit 0 against 'k', where the regex (and any Utf8 array holding it) gives 1."""
    items = ["k", None, "K"]
    v = acu.ViewColumn.from_values([x.encode() if x else None for x in items], garbage_under_nulls=None)
    v.views[1] = v.views[0]
    v.views[1, 0] = 3
    v.views[1, 4:7] = np.frombuffer("K".encode(), dtype=np.uint8)
    pat = column("utf8_view", ["k"], scalar=True)
    res = ORACLE.like_view(abi.ILIKE, v, pat)
    assert res.value_array().tolist() == [True, False, True] and res.to_list() == [True, None, True]
    v.views[2] = v.views[1]  # a valid non-ASCII slot: the regex everywhere
    assert ORACLE.like_view(abi.ILIKE, v, pat).value_array().tolist() == [True, True, True]
    u = column("utf8", ["k", "K", "K"])
    u.nulls = acu.HostArray.from_list(abi.U8, [0, None, 0])
    u.nulls.values = np.zeros(0, np.uint8)
    assert ORACLE.like_bytes(abi.ILIKE, u, column("utf8", ["k"], scalar=True)).value_array().tolist() == [True, True, True]


def test_oracle_errors():
    a, b = column("utf8", ["a", "b"]), column("utf8", ["a"])
    with pytest.raises(acu.ArrowError, match="Cannot compare arrays of different lengths, got 2 vs 1"):
        ORACLE.like_bytes(abi.LIKE, a, b)
    for op, name in [(abi.LIKE, "LIKE"), (abi.NILIKE, "NILIKE"), (abi.EQ_IGNORE_ASCII_CASE, "EQ_IGNORE_ASCII_CASE")]:
        with pytest.raises(acu.ArrowError, match=f"Invalid binary operation: {name}$"):
            run(ORACLE, op, "binary", column("binary", ["a"]), column("binary", ["a"], scalar=True))
    with pytest.raises(acu.ArrowError) as e:
        ORACLE.like_bytes(abi.ILIKE, column("utf8", ["a"]), column("utf8", ["é%"], scalar=True))
    assert e.value.status == 7 and e.value.index == -1
    with pytest.raises(acu.ArrowError) as e:
        ORACLE.like_bytes(abi.NILIKE, column("utf8", ["a", None, "c", "d"]), column("utf8", ["a", "é", None, "ü"]))
    assert e.value.status == 7 and e.value.index == 3
