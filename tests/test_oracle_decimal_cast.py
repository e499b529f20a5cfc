"""tests/oracle_decimal_cast.py against the reference's literal decimal cast vectors (tests/golden/decimal_cast_vectors.json)
and the rules its header states. CPU only."""
import json
import math
import os

import pytest

import oracle_decimal as od
import oracle_decimal_cast as oc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "decimal_cast_vectors.json")


def golden_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def operand(d):
    vals = d["values"]
    validity = None if all(v is not None for v in vals) else [v is not None for v in vals]
    return od.Operand(d["width"], d["precision"], d["scale"], [0 if v is None else v for v in vals], validity)


def prim(d):
    vals = d["values"]
    validity = None if all(v is not None for v in vals) else [v is not None for v in vals]
    zero = 0.0 if d["dtype"] in (oc.F32, oc.F64) else 0
    return oc.Prim(d["dtype"], [zero if v is None else v for v in vals], validity)


def run_oracle(c):
    t = c["to"]
    if c["kind"] == "dec":
        return oc.cast_decimal(operand(c["in"]), t["width"], t["precision"], t["scale"], c["safe"])
    if c["kind"] == "to_dec":
        return oc.cast_to_decimal(prim(c["in"]), t["width"], t["precision"], t["scale"], c["safe"])
    return oc.cast_from_decimal(operand(c["in"]), t["dtype"], c["safe"])


def as_list(out):
    return [v if out.validity is None or out.validity[i] else None for i, v in enumerate(out.values)]


@pytest.mark.parametrize("c", golden_cases(), ids=lambda c: c["name"])
def test_oracle_matches_reference_vectors(c):
    if "error" in c or "error_contains" in c:
        with pytest.raises(oc.CastError) as e:
            run_oracle(c)
        assert e.value.message == c["error"] if c.get("error", "*") != "*" else c.get("error_contains", "") in e.value.message
    elif c["expected"] is None:  # the reference asserts only that the cast succeeds
        run_oracle(c)
    else:
        assert as_list(run_oracle(c)) == c["expected"]


def test_powi_differs_from_correctly_rounded_where_stated():
    """The powi loop is not the correctly rounded 10^k at k = 33, 34, 37 and at -23 (checked with exact rationals)."""
    from fractions import Fraction

    def nearest(k):
        return float(Fraction(10) ** k)
    differ = [k for k in range(-128, 39) if oc.powi10(k) != nearest(k)]
    assert {33, 34, 37, -23} <= set(differ)
    assert all(k <= -23 for k in differ if k < 0) and [k for k in differ if k >= 0] == [33, 34, 37]


def test_round_half_away_from_zero():
    assert [oc.round_half_away(x) for x in (0.5, 1.5, 2.5, -0.5, -2.5, 0.49999999999999994, 4503599627370495.5)] == \
        [1.0, 2.0, 3.0, -1.0, -3.0, 0.0, 4503599627370496.0]


def test_float_debug():
    assert [oc.float_debug(x, False) for x in (0.0, -0.0, 1.0, 0.1, 1e16, 1e15, 1e-4, 1e-5, 1.5e-7, 1e40, math.nan, math.inf,
                                                -math.inf, 123.456, -2.5)] == \
        ["0.0", "-0.0", "1.0", "0.1", "1e16", "1000000000000000.0", "0.0001", "1e-5", "1.5e-7", "1e40", "NaN", "inf", "-inf",
         "123.456", "-2.5"]
    assert oc.float_debug(oc.f32(0.1), True) == "0.1" and oc.float_debug(oc.f32(3.4e38), True) == "3.4e38"


def test_format_decimal_str_internal():
    f = oc.format_decimal_str_internal
    assert f("123456789", 6, 2, False) == "1234567.89" and f("999999", 6, 2, True) == "9999.99"
    assert f("-5", 3, 3, False) == "-0.005" and f("12", 3, -2, False) == "1200" and f("0", 0, 2, True) == "0.00"


def test_infallible_test_is_i8():
    """p_out above 127 reads negative as i8. Decimal128(38, 0) -> (200, 1) is therefore fallible, so the unsafe row reports
    the precision error of the row instead of the closing type validation; so is Decimal64(18, 0) -> Decimal128(200, 0)."""
    for a, w, s in ((od.Operand(16, 38, 0, [5]), 16, 1), (od.Operand(8, 18, 0, [5]), 16, 0)):
        with pytest.raises(oc.CastError) as e:
            oc.cast_decimal(a, w, 200, s, False)
        assert e.value.message == "Invalid argument error: Max precision of a Decimal128 is 38, but got 200" and e.value.index == 0
        with pytest.raises(oc.CastError) as e:
            oc.cast_decimal(a, w, 200, s, True)
        assert e.value.message == "Invalid argument error: precision 200 is greater than max 38" and e.value.index == -1


def test_same_type_clone_is_decided_before_the_i8_test():
    """cast_decimal_to_decimal_same_type clones when the scales match and p_in <= p_out in u8 (decimal.rs:461): Decimal128(38,
    0) -> (200, 0) runs no row, and with_precision_and_scale reports the type, safe or not."""
    a = od.Operand(16, 38, 0, [5, 2 ** 100], [True, False])
    for safe in (True, False):
        with pytest.raises(oc.CastError) as e:
            oc.cast_decimal(a, 16, 200, 0, safe)
        assert e.value.message == "Invalid argument error: precision 200 is greater than max 38" and e.value.index == -1
    r = oc.cast_decimal(a, 16, 38, 0, False)  # the clone keeps the bytes under the null
    assert r.values == [5, 2 ** 100] and r.validity == [True, False] and r.null_count == 1
