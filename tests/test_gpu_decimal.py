"""Decimal32 / Decimal64 / Decimal128 arithmetic, negation, comparison, sum / min / max, filter and take on the device
against tests/oracle_decimal.py, bit for bit: values (0 under nulls), validity, null_count, NullBuffer presence, result
type, status, message and error row.

The multi-round size is sized() of test_gpu_elementwise_rounds: at least 1.2 rounds of an acu_wave_grid launch at any
occupancy, checked on periodic columns (test_gpu_decimal_edges)."""
import ctypes as C

import numpy as np
import pytest

import acu
import oracle_decimal as od
from acu import _abi as abi
from acu import ArrowError, DecimalArray, bitmap_bytes
from test_gpu_decimal_edges import P, Exp, Periodic, check_out, exp_from, gpu_aggregate, raw_of, run_out
from test_gpu_elementwise_rounds import SG, sized
from test_oracle_decimal import CMP_OPS, OPS, golden

pytestmark = pytest.mark.gpu

STATUS = {"InvalidArgument": abi.ERR_INVALID_ARGUMENT, "ArithmeticOverflow": abi.ERR_ARITHMETIC_OVERFLOW,
          "DivideByZero": abi.ERR_DIVIDE_BY_ZERO, "Compute": abi.ERR_COMPUTE}
ARITH_OPS = [abi.ADD_WRAPPING, abi.ADD, abi.SUB_WRAPPING, abi.SUB, abi.MUL_WRAPPING, abi.MUL, abi.DIV, abi.REM]
WIDTHS = [4, 8, 16]


def to_operand(d):
    validity = None if d.validity is None else [bool(x) for x in d.valid_mask()]
    return od.Operand(d.byte_width, d.precision, d.scale, d.raw_ints(), validity, d.is_scalar)


def same(got, exp):
    assert (got.precision, got.scale) == (exp.precision, exp.scale)
    assert got.raw_ints() == exp.values
    assert (got.validity is not None) == (exp.validity is not None)
    if exp.validity is not None:
        assert [bool(x) for x in got.valid_mask()] == exp.validity and got.null_count == exp.null_count


def run_both(fn_gpu, fn_oracle):
    try:
        exp = fn_oracle()
    except od.DecimalError as e:
        with pytest.raises(ArrowError) as g:
            fn_gpu()
        assert (g.value.status, g.value.message, g.value.index) == (STATUS[e.status], e.message, e.index)
        return None
    got = fn_gpu()
    same(got, exp)
    return got


def rand_ints(rng, w, n, big):
    """Small values, or a mix of small, 64-bit-sized and full-width magnitudes (the i128 fast and slow paths)."""
    if not big:
        return [int(x) for x in rng.integers(-10 ** 6, 10 ** 6, n)]
    kinds = rng.integers(0, 4, n)
    raw = rng.bytes(w * n)
    out = []
    for i, k in enumerate(kinds):
        full = int.from_bytes(raw[i * w:(i + 1) * w], "little", signed=True)
        if k == 0:
            out.append(full % 200 - 100)
        elif k == 1:
            out.append(full >> max(8 * w - 63, 0))
        elif k == 2:
            out.append(full)
        else:
            out.append(full >> int(rng.integers(0, 8 * w)))
    return out


def rand_dec(rng, w, p, s, n, null_p, big):
    vals = rand_ints(rng, w, n, big)
    items = [None if null_p and rng.random() < null_p else v for v in vals]
    return DecimalArray.from_ints(w, p, s, items)


# ---- the reference's literal vectors ---------------------------------------------------------------------------------
@pytest.mark.parametrize("i", range(len(golden()["arith"])))
def test_numeric_rs_test_decimal(gpu, i):
    c = golden()["arith"][i]
    a, b = (DecimalArray.from_ints(x["width"], x["precision"], x["scale"], x["values"]) for x in (c["a"], c["b"]))
    if "error" in c:
        with pytest.raises(ArrowError) as e:
            gpu.decimal_arith(OPS[c["op"]], a, b)
        assert e.value.status == STATUS[c["error"]] and e.value.message == c["message"]
    else:
        r = gpu.decimal_arith(OPS[c["op"]], a, b)
        assert [r.precision, r.scale] == c["type"] and r.to_list() == c["values"]


def test_test_neg(gpu):
    for c in golden()["neg"]:
        x = c["a"]
        r = gpu.decimal_neg(DecimalArray.from_ints(x["width"], x["precision"], x["scale"], x["values"]))
        assert r.to_list() == c["values"] and r.data_type() == f"Decimal{8 * x['width']}(9, 6)"


def test_comparison_rs(gpu):
    for c in golden()["cmp"]:
        a = DecimalArray.from_ints(c["width"], 10, 0, c["a"])
        b = DecimalArray.from_ints(c["width"], 10, 0, c["b"], scalar=c["b_scalar"])
        assert gpu.cmp(CMP_OPS[c["op"]], a, b).to_list() == c["expected"], c


def test_take_rs_decimal128(gpu):
    for c in golden()["take"]:
        v = DecimalArray.from_ints(16, c["precision"], c["scale"], c["values"])
        idx = acu.HostArray.from_list(abi.U32, c["indices"])
        r = gpu.take(v, idx)
        assert r.to_list() == c["expected"] and r.data_type() == "Decimal128(10, 5)"


def test_aggregate_edge_cases(gpu):
    for c in golden()["aggregate"]:
        a = DecimalArray.from_ints(16, 38, 0, c["values"], force_validity=True)
        assert (gpu.sum(a), gpu.min(a), gpu.max(a)) == (c["sum"], c["min"], c["max"]), c["name"]


# ---- every op x width x operand form against the oracle -----------------------------------------------------------------
TYPES = {4: [(9, 2), (9, 2), (7, 0), (5, -1)], 8: [(18, 4), (18, 4), (15, 1), (12, -2)], 16: [(38, 6), (38, 6), (30, 2), (20, -3)]}


@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("form", ["array-array", "array-scalar", "scalar-array", "null-scalar"])
@pytest.mark.parametrize("n", [0, 1, 37, 2048, 6000])
def test_ops_against_oracle(gpu, w, form, n):
    rng = np.random.default_rng(w * 1000 + n + len(form))
    for op in ARITH_OPS:
        for (p1, s1), (p2, s2) in ((TYPES[w][0], TYPES[w][1]), (TYPES[w][2], TYPES[w][3]), (TYPES[w][3], TYPES[w][0])):
            big = rng.random() < 0.5
            a = rand_dec(rng, w, p1, s1, n, 0.1, big)
            b = rand_dec(rng, w, p2, s2, n, 0.1, big)
            if form != "array-array":
                sv = rand_ints(rng, w, 1, big) if form != "null-scalar" else [None]
                s = DecimalArray.from_ints(w, p2, s2, sv, scalar=True)
                a, b = (s, b) if form == "scalar-array" else (a, s)
            if op in (abi.DIV, abi.REM) and form != "null-scalar":  # some zero divisors, not everywhere
                b = DecimalArray.from_ints(w, b.precision, b.scale, [v if (v is None or rng.random() > 0.001) else 0 for v in b.to_list()],
                                           scalar=b.is_scalar)
            run_both(lambda: gpu.decimal_arith(op, a, b), lambda: od.decimal_op(op, to_operand(a), to_operand(b)))


@pytest.mark.parametrize("w", WIDTHS)
def test_neg_against_oracle(gpu, w):
    rng = np.random.default_rng(w)
    lo, _ = od.lo_hi(w)
    for n in (0, 5, 3000):
        a = rand_dec(rng, w, TYPES[w][0][0], TYPES[w][0][1], n, 0.2, True)
        run_both(lambda: gpu.decimal_neg(a), lambda: od.neg(to_operand(a)))
    a = DecimalArray.from_ints(w, 9, 0, [1, None, 2, lo, lo])  # the first MIN is the error row
    with pytest.raises(ArrowError) as e:
        gpu.decimal_neg(a)
    assert e.value.index == 3 and e.value.message == f"Arithmetic overflow: Overflow happened on: - {lo}"


# ---- evaluation order, MIN % -1, the scalar's rescale ---------------------------------------------------------------------
@pytest.mark.parametrize("w", WIDTHS)
def test_min_rem_minus_one_is_an_overflow(gpu, w):
    lo, _ = od.lo_hi(w)
    mp = od.MAX_PRECISION[w]
    a = DecimalArray.from_ints(w, mp, 0, [7, lo, lo])
    b = DecimalArray.from_ints(w, mp, 0, [-1, 3, -1])
    with pytest.raises(ArrowError) as e:
        gpu.decimal_rem(a, b)
    assert e.value.status == abi.ERR_ARITHMETIC_OVERFLOW and e.value.index == 2
    assert e.value.message == f"Arithmetic overflow: Overflow happened on: {lo} % -1"
    # div at the maximum scale: result scale min(s1 + 4, MAX_SCALE) = s1, so no rescale and MIN / -1 itself overflows
    a = DecimalArray.from_ints(w, mp, mp, [7, lo, lo])
    with pytest.raises(ArrowError) as e:
        gpu.decimal_div(a, b)
    assert e.value.index == 2 and e.value.message == f"Arithmetic overflow: Overflow happened on: {lo} / -1"


@pytest.mark.parametrize("w", WIDTHS)
def test_wrapping_ops_are_checked(gpu, w):
    _, hi = od.lo_hi(w)
    mp = od.MAX_PRECISION[w]
    a, b = DecimalArray.from_ints(w, mp, 0, [1, hi]), DecimalArray.from_ints(w, mp, 0, [1, 1])
    for op in (abi.ADD_WRAPPING, abi.ADD):
        with pytest.raises(ArrowError) as e:
            gpu.decimal_arith(op, a, b)
        assert e.value.message == f"Arithmetic overflow: Overflow happened on: {hi} + 1" and e.value.index == 1


@pytest.mark.parametrize("w", WIDTHS)
def test_receiver_rescale_fails_before_zero_divisor(gpu, w):
    _, hi = od.lo_hi(w)
    mp = od.MAX_PRECISION[w]
    big = hi // 100
    a = DecimalArray.from_ints(w, mp, 0, [5, big])
    b = DecimalArray.from_ints(w, mp, 0, [1, 0])
    with pytest.raises(ArrowError) as e:  # div: l * 10^4 overflows before r == 0 is seen
        gpu.decimal_div(a, b)
    assert e.value.status == abi.ERR_ARITHMETIC_OVERFLOW and e.value.message == f"Arithmetic overflow: Overflow happened on: {big} * 10000"
    # rem with unequal scales: the argument's rescale overflows before its zero check
    a = DecimalArray.from_ints(w, mp, 2, [5, 0])
    b = DecimalArray.from_ints(w, mp, 0, [1, hi // 10])
    with pytest.raises(ArrowError) as e:
        gpu.decimal_rem(a, b)
    assert e.value.message == f"Arithmetic overflow: Overflow happened on: {hi // 10} * 100" and e.value.index == 1


def test_rem_multiplier_wraps_to_zero(gpu):
    """rem computes its multipliers with pow_wrapping: Decimal32 scales 9 and -23 give r_mul = 10^32 mod 2^32 = 0, so every
    valid row divides by zero although no divisor is 0."""
    a = DecimalArray.from_ints(4, 9, 9, [None, 5, 6])
    b = DecimalArray.from_ints(4, 1, -23, [3, 3, 3])
    run_both(lambda: gpu.decimal_rem(a, b), lambda: od.decimal_op(od.REM, to_operand(a), to_operand(b)))
    with pytest.raises(ArrowError) as e:
        gpu.decimal_rem(a, b)
    assert e.value.status == abi.ERR_DIVIDE_BY_ZERO and e.value.index == 1


@pytest.mark.parametrize("w", WIDTHS)
def test_scalar_rescale_is_per_row(gpu, w):
    mp = od.MAX_PRECISION[w]
    s = DecimalArray.from_ints(w, 3, -1, [10], scalar=True)  # rescaled by 10^(mp - 1 + 1) = 10^mp: always overflows
    b = DecimalArray.from_ints(w, mp, mp - 1, [None, None, 4, 5])
    with pytest.raises(ArrowError) as e:
        gpu.decimal_add(s, b)
    assert e.value.index == 2 and e.value.message == f"Arithmetic overflow: Overflow happened on: 10 * {10 ** mp}"
    r = gpu.decimal_add(s, DecimalArray.from_ints(w, mp, mp - 1, [None, None]))  # no valid row: no error
    assert r.to_list() == [None, None] and r.null_count == 2
    r = gpu.decimal_add(s, DecimalArray.from_ints(w, mp, mp - 1, []))
    assert r.length == 0


def test_pre_loop_errors_on_empty_arrays(gpu):
    e3 = DecimalArray.from_ints(16, 3, 3, [])
    e37 = DecimalArray.from_ints(16, 37, 37, [])
    with pytest.raises(ArrowError) as e:
        gpu.decimal_mul(e3, e37)
    assert e.value.message == "Invalid argument error: Output scale of Decimal128(3, 3) * Decimal128(37, 37) would exceed max scale of 38"
    with pytest.raises(ArrowError) as e:
        gpu.decimal_add(DecimalArray.from_ints(16, 3, -2, []), e37)
    assert e.value.message == "Arithmetic overflow: Overflow happened on: 10 ^ 39"
    # result-type validation after the rows: div precision (mul_pow + p1) = 0
    a, b = DecimalArray.from_ints(8, 1, 0, [5]), DecimalArray.from_ints(8, 1, -5, [1])
    run_both(lambda: gpu.decimal_div(a, b), lambda: od.decimal_op(od.DIV, to_operand(a), to_operand(b)))


def test_invalid_types_and_dtypes_are_rejected(gpu):
    with pytest.raises(ArrowError) as e:
        gpu.decimal_add(DecimalArray.from_ints(4, 10, 0, [1]), DecimalArray.from_ints(4, 9, 0, [1]))
    assert e.value.status == abi.ERR_INVALID_ARGUMENT and e.value.message == "Invalid argument error: precision 10 is greater than max 9"
    with pytest.raises(ArrowError) as e:
        gpu.decimal_add(DecimalArray.from_ints(16, 5, 6, [1]), DecimalArray.from_ints(16, 9, 0, [1]))
    assert e.value.message == "Invalid argument error: scale 6 is greater than precision 5"
    a = DecimalArray.from_ints(16, 9, 0, [1, 2])
    with pytest.raises(ArrowError) as e:
        gpu.cmp(abi.LT, a, DecimalArray.from_ints(16, 10, 0, [1, 2]))
    assert e.value.message == "Invalid argument error: Invalid comparison operation: Decimal128(9, 0) < Decimal128(10, 0)"
    # ACU_I128 stays out of the primitive entry points
    da = gpu.upload(a)
    try:
        d = da.descriptor()
        out = gpu.alloc_out(64, 2)
        assert gpu.lib.acu_arith(gpu.h, abi.I128, abi.ADD, C.byref(d), C.byref(d), C.byref(out)) == abi.ERR_INVALID_ARGUMENT
        assert gpu.lib.acu_cast_numeric(gpu.h, abi.I128, abi.I64, 1, C.byref(d), C.byref(out)) == abi.ERR_NOT_YET_IMPLEMENTED
        bits, cnt = C.c_uint64(0), C.c_int64(0)
        assert gpu.lib.acu_aggregate(gpu.h, abi.I128, abi.SUM, C.byref(d), C.byref(bits), C.byref(cnt)) == abi.ERR_INVALID_ARGUMENT
        d.values += 8  # misaligned Int128 values are refused before any launch
        assert gpu.lib.acu_cmp(gpu.h, abi.I128, abi.EQ, C.byref(d), C.byref(d), C.byref(out)) == abi.ERR_INVALID_ARGUMENT
        gpu._free_out(out)
    finally:
        da.free()


# ---- multi-round sizes ---------------------------------------------------------------------------------------------------
def test_multi_round_add_sum_cmp(gpu):
    """add (the right operand rescaled by 100), sum / min / max and a comparison with a scalar over more than one
    grid-stride round, on the periodic columns of test_gpu_decimal_edges (which also places failing rows for every
    occupancy)."""
    n = sized(gpu, SG)
    rng = np.random.default_rng(7)
    x = [int(v) for v in rng.integers(-2 ** 39, 2 ** 39, P)]
    y = [int(v) for v in rng.integers(-2 ** 39, 2 ** 39, P)]
    mask = rng.integers(0, 100, P) >= 3
    a = Periodic(gpu, abi.I128, raw_of(DecimalArray.from_ints(16, 38, 4, x)), mask, n)
    b = Periodic(gpu, abi.I128, raw_of(DecimalArray.from_ints(16, 38, 2, y)), None, n)
    t = DecimalArray.from_ints(16, 38, 4, [int(np.median(x))], scalar=True)
    dt = gpu.upload(t)
    try:
        ad, bd, td = a.descriptor(), b.descriptor(), dt.descriptor()
        ox = od.Operand(16, 38, 4, x, mask.tolist())
        exp = od.decimal_op(abi.ADD, ox, od.Operand(16, 38, 2, y))
        lt, rt, ot = abi.DecimalType(16, 38, 4), abi.DecimalType(16, 38, 2), abi.DecimalType()
        st, out = run_out(gpu, n, n * 16, lambda o: gpu.lib.acu_decimal_arith(gpu.h, abi.ADD, C.byref(lt), C.byref(ad), C.byref(rt),
                                                                              C.byref(bd), C.byref(ot), C.byref(o)))
        try:
            assert st == abi.OK and (ot.precision, ot.scale) == (38, 4)
            check_out(gpu, out, n, abi.I128, exp_from(exp, abi.I128), "add")
        finally:
            gpu._free_out(out)
        valid = [v for v, m in zip(x, mask) if m]
        total = (n // P) * sum(valid) + sum(v for v, m in zip(x[: n % P], mask[: n % P]) if m)
        assert gpu_aggregate(gpu, a) == (total, min(valid), max(valid))
        vals, validity = od.cmp(od.LT, ox, od.Operand(16, 38, 4, t.raw_ints(), None, True))
        st, out = run_out(gpu, n, bitmap_bytes(n), lambda o: gpu.lib.acu_cmp(gpu.h, abi.I128, abi.LT, C.byref(ad), C.byref(td), C.byref(o)))
        try:
            assert st == abi.OK
            check_out(gpu, out, n, acu.BOOL, Exp(np.array(vals), np.array(validity)), "cmp LT scalar")
        finally:
            gpu._free_out(out)
    finally:
        a.free()
        b.free()
        dt.free()


# ---- bit offsets and zero-copy unaligned slices ---------------------------------------------------------------------------
@pytest.mark.parametrize("shift", [1, 5, 63])
def test_decimal128_bit_offsets(gpu, shift):
    """Decimal128 rows [shift, shift + n) of an uploaded column: the values stay 16-byte aligned, the validity bit offset
    moves. Arithmetic, comparison with a scalar and the aggregates against the oracle on the same logical slice."""
    rng = np.random.default_rng(100 + shift)
    n = 4500
    a = rand_dec(rng, 16, 30, 2, n + shift, 0.1, True)
    b = rand_dec(rng, 16, 20, -3, n + shift, 0.1, False)
    ha, hb = a.slice(shift, n), b.slice(shift, n)
    for op in (abi.ADD, abi.SUB, abi.MUL, abi.DIV, abi.REM):
        da, ad = sliced_descriptor(gpu, a, shift, n)
        db, bd = sliced_descriptor(gpu, b, shift, n)
        out = gpu.alloc_out(n * 16, n)
        try:
            assert ad.values % 16 == 0 and ad.validity_offset == shift
            lt, rt, ot = abi.DecimalType(16, 30, 2), abi.DecimalType(16, 20, -3), abi.DecimalType()
            st = gpu.lib.acu_decimal_arith(gpu.h, op, C.byref(lt), C.byref(ad), C.byref(rt), C.byref(bd), C.byref(ot), C.byref(out))
            try:
                exp = od.decimal_op(op, to_operand(ha), to_operand(hb))
            except od.DecimalError as e:
                d = gpu.lib.acu_last_error(gpu.h).contents
                assert (st, d.message.decode(), d.index) == (STATUS[e.status], e.message, e.index)
                continue
            assert st == abi.OK
            got = a.like(gpu.download_out(out, a.dtype), ot.precision, ot.scale)
            out = None
            same(got, exp)
        finally:
            if out is not None:
                gpu._free_out(out)
            da.free()
            db.free()
    # comparison against a scalar, and sum / min / max, on the same slice
    da, ad = sliced_descriptor(gpu, a, shift, n)
    t = DecimalArray.from_ints(16, 30, 2, [int(np.median([v for v in ha.to_list() if v is not None]))], scalar=True)
    dt = gpu.upload(t)
    out = gpu.alloc_out(bitmap_bytes(n), n)
    try:
        td = dt.descriptor()
        gpu.check(gpu.lib.acu_cmp(gpu.h, abi.I128, abi.LT, C.byref(ad), C.byref(td), C.byref(out)))
        got = gpu.download_out(out, acu.BOOL)
        out = None
        vals, validity = od.cmp(od.LT, to_operand(ha), to_operand(t))
        assert [bool(x) for x in got.value_array()] == vals and [bool(x) for x in got.valid_mask()] == validity
        for op, kind in ((abi.SUM, "sum"), (abi.MIN, "min"), (abi.MAX, "max")):
            bits, cnt = (C.c_uint64 * 2)(), C.c_int64(0)
            gpu.check(gpu.lib.acu_aggregate_i128(gpu.h, op, C.byref(ad), bits, C.byref(cnt)))
            assert acu.halves_to_i128(np.array([[bits[0], bits[1]]], dtype=np.uint64))[0] == od.aggregate(kind, to_operand(ha))
    finally:
        if out is not None:
            gpu._free_out(out)
        da.free()
        dt.free()
    # the Python mirror's own bit offset (the validity bitmap starts at bit 3 of its first byte)
    items = ha.to_list()[:100]
    c = DecimalArray.from_ints(16, 30, 2, items, bit_offset=3)
    assert c.validity_offset == 3 and gpu.sum(c) == od.aggregate("sum", to_operand(DecimalArray.from_ints(16, 30, 2, items)))
    r = gpu.decimal_neg(c)
    assert r.to_list() == [None if v is None else -v for v in items]



def sliced_descriptor(gpu, d, shift, n):
    """Rows [shift, shift + n) of an uploaded DecimalArray as an acu_array: values pointer moved by shift elements (not
    16-byte aligned for Decimal32 / 64), validity bit offset moved by shift."""
    da = gpu.upload(d)
    desc = da.descriptor()
    desc.values += shift * d.byte_width
    desc.validity_offset += shift
    desc.len = n
    desc.null_count = -1 if d.validity is not None else 0
    return da, desc


@pytest.mark.parametrize("w", [4, 8])
@pytest.mark.parametrize("shift", [1, 3])
def test_unaligned_slices(gpu, w, shift):
    rng = np.random.default_rng(shift + w)
    n = 5000
    (p1, s1), (p2, s2) = TYPES[w][2], TYPES[w][3]
    a = rand_dec(rng, w, p1, s1, n + shift, 0.1, False)
    b = rand_dec(rng, w, p2, s2, n + shift, 0.1, False)
    for op in (abi.ADD, abi.SUB, abi.MUL, abi.DIV, abi.REM):
        da, ad = sliced_descriptor(gpu, a, shift, n)
        db, bd = sliced_descriptor(gpu, b, shift, n)
        out = gpu.alloc_out(n * w, n)
        try:
            assert ad.values % 16 != 0
            lt, rt, ot = abi.DecimalType(w, p1, s1), abi.DecimalType(w, p2, s2), abi.DecimalType()
            st = gpu.lib.acu_decimal_arith(gpu.h, op, C.byref(lt), C.byref(ad), C.byref(rt), C.byref(bd), C.byref(ot), C.byref(out))
            try:
                exp = od.decimal_op(op, to_operand(a.slice(shift, n)), to_operand(b.slice(shift, n)))
            except od.DecimalError as e:
                assert st == STATUS[e.status] and gpu.lib.acu_last_error(gpu.h).contents.index == e.index
                continue
            assert st == abi.OK
            got = a.like(gpu.download_out(out, a.dtype), ot.precision, ot.scale)
            out = None
            same(got, exp)
        finally:
            if out is not None:
                gpu._free_out(out)
            da.free()
            db.free()


# ---- fused compare -> filter plan and one stream-ordered section -------------------------------------------------------
def test_filter_plan_create_cmp_i128(gpu):
    rng = np.random.default_rng(3)
    n = 10000
    price = rand_dec(rng, 16, 38, 2, n, 0.05, True)
    qty = rand_dec(rng, 16, 38, 0, n, 0.05, False)
    t = DecimalArray.from_ints(16, 38, 2, [0], scalar=True)
    res, (count, _) = gpu.filter_cmp(qty, abi.GT_EQ, price, t)
    keep = [p is not None and p >= 0 for p in price.to_list()]
    assert res.to_list() == [q for q, k in zip(qty.to_list(), keep) if k] and count == sum(keep)
    assert res.data_type() == "Decimal128(38, 0)"


def test_section_cmp_filter_mul_sum(gpu):
    """cmp(price, scalar) -> plan -> filter(price), filter(discount) in one section, then decimal mul ->
    acu_aggregate_i128 in a second one (the product needs the filtered length), equals the synchronous calls."""
    rng = np.random.default_rng(11)
    n = 50000
    price = DecimalArray.from_int64(16, 15, 2, rng.integers(1, 10 ** 7, n), rng.integers(0, 100, n) >= 2)
    disc = DecimalArray.from_int64(16, 15, 2, rng.integers(0, 11, n))
    lo = DecimalArray.from_ints(16, 15, 2, [500000], scalar=True)
    # synchronous
    fp, _ = gpu.filter_cmp(price, abi.LT, price, lo)
    fd, _ = gpu.filter_cmp(disc, abi.LT, price, lo)
    prod = gpu.decimal_mul(fp, fd)
    want = gpu.sum(prod)
    # one section
    ups = [gpu.upload(x) for x in (price, disc, lo)]
    pd, dd, ld = (u.descriptor() for u in ups)
    plan = C.c_void_p()
    o_p, o_d, o_m = gpu.alloc_out(n * 16, n), gpu.alloc_out(n * 16, n), gpu.alloc_out(n * 16, n)
    try:
        bits, cnt = (C.c_uint64 * 2)(), C.c_int64(0)
        t15 = abi.DecimalType(16, 15, 2)
        ot = abi.DecimalType()
        gpu.async_begin()
        gpu.check(gpu.lib.acu_filter_plan_create_cmp(gpu.h, abi.I128, abi.LT, C.byref(pd), C.byref(ld), C.byref(plan)))
        gpu.check(gpu.lib.acu_filter_primitive(gpu.h, plan, 16, C.byref(pd), C.byref(o_p)))
        gpu.check(gpu.lib.acu_filter_primitive(gpu.h, plan, 16, C.byref(dd), C.byref(o_d)))
        # the filtered columns' lengths are still on the device: the product is sized for n rows, null counts unknown
        fa, fb = abi.Array(), abi.Array()
        for f, o in ((fa, o_p), (fb, o_d)):
            f.values, f.validity, f.len, f.null_count = o.values, None, 0, 0
        gpu.results_fetch()
        # filters finalised: len known, queue the product and the sum in a second section
        fa.len, fb.len = o_p.len, o_d.len
        fa.validity, fa.null_count = (o_p.validity, o_p.null_count) if o_p.has_validity else (None, 0)
        gpu.async_begin()
        gpu.check(gpu.lib.acu_decimal_arith(gpu.h, abi.MUL, C.byref(t15), C.byref(fa), C.byref(t15), C.byref(fb), C.byref(ot), C.byref(o_m)))
        m = abi.Array()
        m.values, m.validity, m.len, m.null_count = o_m.values, (o_m.validity if o_p.has_validity else None), o_p.len, -1
        gpu.check(gpu.lib.acu_aggregate_i128(gpu.h, abi.SUM, C.byref(m), bits, C.byref(cnt)))
        gpu.results_fetch()
        got = acu.halves_to_i128(np.array([[bits[0], bits[1]]], dtype=np.uint64))[0] if cnt.value else None
        assert (ot.precision, ot.scale) == (31, 4)
        assert got == want
        # acu_neg(ACU_I128) is stream-ordered too: two negations of the product queued in one section, one fetch
        o_n1, o_n2 = gpu.alloc_out(n * 16, n), gpu.alloc_out(n * 16, n)
        try:
            m.null_count = o_m.null_count if o_p.has_validity else 0
            gpu.async_begin()
            gpu.check(gpu.lib.acu_neg(gpu.h, abi.I128, 0, C.byref(m), C.byref(o_n1)))
            gpu.check(gpu.lib.acu_neg(gpu.h, abi.I128, 1, C.byref(m), C.byref(o_n2)))
            gpu.results_fetch()
            negs = [acu.halves_to_i128(gpu.d2h(o.values, o.len * 16, np.uint64).reshape(-1, 2)) for o in (o_n1, o_n2)]
            prod_vals = acu.halves_to_i128(gpu.d2h(o_m.values, o_m.len * 16, np.uint64).reshape(-1, 2))
            assert o_n1.len == o_m.len and negs[0] == negs[1] == [-v for v in prod_vals]
        finally:
            gpu._free_out(o_n1)
            gpu._free_out(o_n2)
    finally:
        for o in (o_p, o_d, o_m):
            gpu._free_out(o)
        if plan:
            gpu.lib.acu_filter_plan_destroy(gpu.h, plan)
        for u in ups:
            u.free()
