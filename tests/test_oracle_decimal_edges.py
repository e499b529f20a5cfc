"""The decimal oracles (tests/oracle_decimal.py, tests/oracle_decimal_cast.py) against the closed forms of
tests/decimal_edges_util.py on every boundary family: each ok row's value, and each failing row failing at its own index
after a prefix of ok rows (an error with safe = False; a null with safe = True, unless the cast is the unary one, whose
failure does not depend on `safe`). The GPU tests compare the kernels with the oracle on the same families, so together
they check the kernels against these closed forms."""
import struct

import numpy as np
import pytest

import decimal_edges_util as du
import oracle_decimal as od
import oracle_decimal_cast as oc

FAMILIES = du.all_families()


def operand(w, p, s, vals, validity=None):
    return od.Operand(w, p, s, list(vals), validity)


def run(fam, rows, safe):
    """The oracle's result of `fam` on input rows `rows`: (values, validity or None)."""
    k, a = fam.kind, fam.args
    if k == "arith":
        op, w, p1, s1, p2, s2 = a
        r = od.decimal_op(op, operand(w, p1, s1, [x[0] for x in rows]), operand(w, p2, s2, [x[1] for x in rows]))
    elif k == "neg":
        r = od.neg(operand(*a, rows))
    elif k == "dec":
        wi, p_in, s_in, wo, p_out, s_out = a
        r = oc.cast_decimal(operand(wi, p_in, s_in, rows), wo, p_out, s_out, safe)
    elif k == "to_dec":
        dt, w, p, s = a
        r = oc.cast_to_decimal(oc.Prim(dt, list(rows)), w, p, s, safe)
    else:
        w, p, s, to = a
        r = oc.cast_from_decimal(operand(w, p, s, rows), to, safe)
    return r.values, r.validity


def bits(v):
    return struct.pack("<d", v) if isinstance(v, float) else v


@pytest.mark.parametrize("group", list(FAMILIES))
def test_families_against_closed_forms(group):
    checked = 0
    for fam in FAMILIES[group]:
        for safe in (False, True) if fam.kind in ("dec", "to_dec", "from_dec") else (False,):
            if fam.ok:
                vals, validity = run(fam, fam.ok, safe)
                assert [bits(v) for v in vals] == [bits(v) for v in fam.exp], fam.name
                assert validity is None or all(validity), fam.name
            for x in fam.fail:
                rows = fam.prefix() + [x]
                i = len(rows) - 1
                if safe and not fam.unary:
                    vals, validity = run(fam, rows, safe)
                    assert validity is not None and not validity[i] and all(validity[:i]) and vals[i] == 0, (fam.name, x)
                    continue
                with pytest.raises((od.DecimalError, oc.CastError)) as e:
                    run(fam, rows, safe)
                assert e.value.index == i, (fam.name, x, e.value.message)
                assert (e.value.status == "Panic") == fam.unary, (fam.name, x, e.value.message)
            checked += len(fam.ok) + len(fam.fail)
    assert checked > 50


def test_families_cover_the_switch_points():
    """The families reach the thresholds they are built for."""
    fams = FAMILIES
    dec = {f.args: f for f in fams["decimal -> decimal"]}
    for wi in du.WIDTHS:  # every scale change the width pair allows
        for wo in du.WIDTHS:
            mi, mo = du.MAXP[wi], du.MAXP[wo]
            deltas = {a[2] - a[5] for a in dec if a[0] == wi and a[3] == wo and a[1] == mi}
            assert deltas == set(range(-mo, mi + 1))
    # downscales of Decimal128 by 19 and 20 digits (the single 64-bit division against the chunked one), with full-width
    # dividends and exact ties among the ok rows
    for k in (9, 10, 18, 19, 20, 27, 28, 36, 37, 38):
        f = dec[(16, 38, k, 16, 38, 0)]
        assert any(abs(x) >= 2 ** 120 for x in f.ok) and any(x % 10 ** k == 10 ** k // 2 for x in f.ok if x > 0), k
    mul = [f for f in fams["mul"] if f.args[1] == 16][0]
    assert (2 ** 127 - 1, 1) in mul.ok and (-(2 ** 64), 2 ** 63) in mul.ok and (2 ** 64, 2 ** 63) in mul.fail
    assert (2 ** 65 - 1, 2 ** 64 - 1) in mul.fail and (2 ** 96, 2 ** 32) in mul.fail and (2 ** 96, -(2 ** 31)) in mul.ok
    for w in (4, 8):
        m = [f for f in fams["mul"] if f.args[1] == w][0]
        lo, hi = du.native(w)
        products = {a * b for a, b in m.fail}
        assert lo in m.exp and hi in m.exp and hi + 1 in products and lo - 1 in products, w
    to_f64 = [f for f in fams["decimal -> float"] if f.args[3] == du.F64][0]
    assert {abs(x).bit_length() for x in to_f64.ok} >= set(range(63, 128))


@pytest.mark.parametrize("values", du.aggregate_sets(), ids=lambda v: f"n{len(v)}")
def test_aggregate_sets(values):
    op = od.Operand(16, 38, 0, [0 if v is None else v for v in values], [v is not None for v in values])
    assert tuple(od.aggregate(k, op) for k in ("sum", "min", "max")) == du.aggregate_closed(values)


def test_float_ties_are_exact():
    """The float families hold exact ties (x * 10^s is exactly k + 1/2 before any rounding) and products that round to a
    tie; every such row rounds away from zero."""
    from fractions import Fraction
    exact = 0
    for fam in FAMILIES["float -> decimal"]:
        dt, w, p, s = fam.args
        for x, v in zip(fam.ok, fam.exp):
            m = x * du.f64_scale(s)
            if np.isfinite(m) and Fraction(m).denominator == 2:
                assert v == (int(m + 0.5) if m > 0 else int(m - 0.5)), (fam.name, x)
                exact += s >= 0 and Fraction(m) == Fraction(x) * 10 ** s
    assert exact > 100
