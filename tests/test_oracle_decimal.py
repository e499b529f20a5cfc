"""CPU checks of tests/oracle_decimal.py: it reproduces the reference's literal decimal vectors
(tests/golden/decimal_vectors.json) and, over a grid of operand types with negative scales and the MAX_SCALE edges, the
Hive precision / scale rules of decimal_op written out in plain integers."""
import json
import os

import pytest

import oracle_decimal as od

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "decimal_vectors.json")
OPS = {"add": od.ADD, "sub": od.SUB, "mul": od.MUL, "div": od.DIV, "rem": od.REM}
CMP_OPS = {"eq": od.EQ, "neq": od.NEQ, "lt": od.LT, "lt_eq": od.LT_EQ, "gt": od.GT, "gt_eq": od.GT_EQ}


def golden():
    with open(GOLDEN) as f:
        return json.load(f)


def operand(d, scalar=False):
    vals = [0 if v is None else v for v in d["values"]]
    validity = None if all(v is not None for v in d["values"]) else [v is not None for v in d["values"]]
    return od.Operand(d["width"], d["precision"], d["scale"], vals, validity, scalar)


def test_golden_file_is_current():
    import importlib.util
    spec = importlib.util.spec_from_file_location("make_golden_decimal", os.path.join(os.path.dirname(GOLDEN), "make_golden_decimal.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    assert golden() == {"arith": m.arith(), "neg": m.neg(), "cmp": m.cmp(), "take": m.take(), "aggregate": m.aggregate()}


@pytest.mark.parametrize("i", range(len(golden()["arith"])))
def test_oracle_reproduces_numeric_rs_test_decimal(i):
    c = golden()["arith"][i]
    a, b = operand(c["a"]), operand(c["b"])
    if "error" in c:
        with pytest.raises(od.DecimalError) as e:
            od.decimal_op(OPS[c["op"]], a, b)
        assert e.value.status == c["error"] and e.value.message == c["message"]
    else:
        r = od.decimal_op(OPS[c["op"]], a, b)
        assert [r.precision, r.scale] == c["type"] and r.values == c["values"]


def test_oracle_reproduces_test_neg():
    for c in golden()["neg"]:
        r = od.neg(operand(c["a"]))
        assert r.values == c["values"] and (r.precision, r.scale) == (9, 6)


def test_oracle_reproduces_comparison_rs():
    for c in golden()["cmp"]:
        a = od.Operand(c["width"], 10, 0, [0 if v is None else v for v in c["a"]],
                       None if None not in c["a"] else [v is not None for v in c["a"]])
        b = od.Operand(c["width"], 10, 0, c["b"], None, c["b_scalar"])
        vals, validity = od.cmp(CMP_OPS[c["op"]], a, b)
        got = [v if validity is None or validity[i] else None for i, v in enumerate(vals)]
        assert got == c["expected"], c


def test_oracle_aggregates_pin_the_edge_cases():
    for c in golden()["aggregate"]:
        a = od.Operand(16, 38, 0, [0 if v is None else v for v in c["values"]], [v is not None for v in c["values"]])
        for kind in ("sum", "min", "max"):
            assert od.aggregate(kind, a) == c[kind], (c["name"], kind)


# ---- the type rules, written out as in the reference's comments -------------------------------------------------------
def textual(op, w, p1, s1, p2, s2):
    """The Hive rules as the reference's comments state them, for operand types whose i8 arithmetic cannot overflow."""
    mp = od.MAX_PRECISION[w]
    if op in (od.ADD, od.SUB):
        s = max(s1, s2)
        return min(s + max(p1 - s1, p2 - s2) + 1, mp), s, (s - s1, s - s2)
    if op == od.MUL:
        return min(p1 + p2 + 1, mp), s1 + s2, None
    if op == od.DIV:  # p1 - s1 + s2 + result_scale; a negative sum is `as u8` of a negative i8, i.e. >= 128
        s = min(s1 + 4, mp)
        p = p1 - s1 + s2 + s
        return (min(p, mp) if p >= 0 else mp), s, s - s1 + s2
    s = max(s1, s2)
    return min(s + min(p1 - s1, p2 - s2), mp), s, None


GRID_SCALES = [-128, -90, -89, -40, -5, -1, 0, 1, 2, 5]


def grid(w):
    mp = od.MAX_PRECISION[w]
    precisions = sorted({1, 2, mp // 2, mp - 1, mp})
    scales = sorted(set(GRID_SCALES + [mp - 1, mp]))
    for p in precisions:
        for s in scales:
            if od.validate_type(w, p, s) is None:
                yield p, s


@pytest.mark.parametrize("w", [4, 8, 16])
def test_type_rules_match_the_textual_rules(w):
    mp = od.MAX_PRECISION[w]
    types = list(grid(w))
    checked = 0
    for p1, s1 in types:
        for p2, s2 in types:
            in_range = all(-128 <= x <= 127 for x in (p1 - s1, p2 - s2, max(s1, s2) - s1, max(s1, s2) - s2))
            for op in (od.ADD, od.SUB, od.MUL, od.DIV, od.REM):
                try:
                    rp, rs, lm, rm = od.result_type(op, w, p1, s1, p2, s2)
                    err = None
                except od.DecimalError as e:
                    err = e
                if not in_range:
                    continue
                tp, ts, extra = textual(op, w, p1, s1, p2, s2)
                if op == od.MUL:
                    if ts > mp:
                        assert err is not None and err.status == "InvalidArgument"
                        continue
                    ts = max(-128, ts)
                if op in (od.ADD, od.SUB):
                    exps = extra
                    if max(exps) > mp:
                        assert err is not None and err.message == f"Arithmetic overflow: Overflow happened on: 10 ^ {exps[0] if exps[0] > mp else exps[1]}"
                        continue
                    assert (lm, rm) == (10 ** exps[0], 10 ** exps[1])
                if op == od.DIV:
                    if abs(extra) > mp:
                        assert err is not None and err.message == f"Arithmetic overflow: Overflow happened on: 10 ^ {abs(extra)}"
                        continue
                    assert (lm, rm) == ((10 ** extra, 1) if extra >= 0 else (1, 10 ** -extra))
                assert err is None, (op, p1, s1, p2, s2, err.message)
                assert (rp, rs) == (tp, ts), (op, p1, s1, p2, s2)
                checked += 1
    assert checked > 500


def test_i8_overflow_wraps_like_a_release_build():
    # p - s = 38 - (-100) = 138 leaves i8: a debug build panics, a release build wraps to -118; rem's precision is then
    # (0 + min(-118, 10)) as u8 = 138, capped at 38
    rp, rs, lm, rm = od.result_type(od.REM, 16, 38, -100, 10, 0)
    assert (rp, rs) == (38, 0)
    # the scale difference 0 - (-100) = 100 fits; 38 - (-100) = 138 wraps to -118 and reads as a huge u32 exponent
    with pytest.raises(od.DecimalError) as e:
        od.result_type(od.ADD, 16, 10, -100, 10, 38)
    assert e.value.message == f"Arithmetic overflow: Overflow happened on: 10 ^ {(-118) % (1 << 32)}"
    # rem computes its multipliers wrapping: a huge exponent gives 0, so every valid row divides by zero
    _, _, lm, rm = od.result_type(od.REM, 16, 10, -100, 10, 38)
    assert lm == 0 and rm == 1
    # div: mul_pow = 38 - 38 + (-128) = -128, whose neg_wrapping stays -128
    with pytest.raises(od.DecimalError) as e:
        od.result_type(od.DIV, 16, 38, 38, 1, -128)
    assert e.value.message == f"Arithmetic overflow: Overflow happened on: 10 ^ {(-128) % (1 << 32)}"


def test_evaluation_order_and_rem_overflow():
    w = 16
    mn = -(1 << 127)
    # MIN % -1 is an overflow for decimals (mod_checked), where the integer rem gives 0
    with pytest.raises(od.DecimalError) as e:
        od.decimal_op(od.REM, od.Operand(w, 38, 0, [mn]), od.Operand(w, 38, 0, [-1]))
    assert e.value.status == "ArithmeticOverflow" and e.value.message == f"Arithmetic overflow: Overflow happened on: {mn} % -1"
    # the receiver's rescale fails before the zero divisor is seen
    with pytest.raises(od.DecimalError) as e:
        od.decimal_op(od.DIV, od.Operand(w, 38, 0, [10 ** 36]), od.Operand(w, 38, 0, [0]))
    assert e.value.message == f"Arithmetic overflow: Overflow happened on: {10 ** 36} * 10000"
    # a scalar's rescale fails at the lowest valid row, and not at all without valid rows
    s = od.Operand(w, 3, -1, [10], None, True)
    b = od.Operand(w, 37, 37, [1, 2], [False, True])
    with pytest.raises(od.DecimalError) as e:
        od.decimal_op(od.ADD, s, b)
    assert e.value.index == 1
    r = od.decimal_op(od.ADD, s, od.Operand(w, 37, 37, [1, 2], [False, False]))
    assert r.values == [0, 0] and r.null_count == 2
