"""Decimal casts on the device (acu_cast_decimal / acu_cast_to_decimal / acu_cast_from_decimal) against
tests/oracle_decimal_cast.py, bit for bit: values at every slot (the unary casts compute under nulls too; the others write
0 there), validity, null_count, NullBuffer presence, status, message and error row.

The multi-round size is sized() of test_gpu_elementwise_rounds: at least 1.2 rounds of an acu_wave_grid launch at any
occupancy, with the first failing row placed for every occupancy (test_gpu_decimal_edges)."""
import ctypes as C
import math

import numpy as np
import pytest

import acu
import oracle_decimal as od
import oracle_decimal_cast as oc
from acu import _abi as abi
from acu import ArrowError, DecimalArray, HostArray
from test_gpu_decimal_edges import P, Call, Periodic, check_out, check_placements, exp_from, raw_of, raw_value
from test_gpu_elementwise_rounds import SG, sized
from test_oracle_decimal_cast import golden_cases

pytestmark = pytest.mark.gpu

STATUS = {"InvalidArgument": abi.ERR_INVALID_ARGUMENT, "ArithmeticOverflow": abi.ERR_ARITHMETIC_OVERFLOW, "Cast": abi.ERR_CAST,
          "Panic": abi.ERR_PANIC_OUT_OF_BOUNDS}
WIDTHS = [4, 8, 16]
INTS = [abi.I8, abi.I16, abi.I32, abi.I64, abi.U8, abi.U16, abi.U32, abi.U64]
NP_BITS = {abi.F32: np.uint32, abi.F64: np.uint64}


def to_operand(d):
    validity = None if d.validity is None else [bool(x) for x in d.valid_mask()]
    return od.Operand(d.byte_width, d.precision, d.scale, d.raw_ints(), validity)


def to_prim(h):
    vals = h.value_array()
    vals = [float(x) for x in vals] if h.dtype in (abi.F32, abi.F64) else [int(x) for x in vals]
    return oc.Prim(h.dtype, vals, None if h.validity is None else [bool(x) for x in h.valid_mask()])


def same(got, exp, dtype=None):
    if dtype in (abi.F32, abi.F64):
        g = np.asarray(got.value_array()).view(NP_BITS[dtype])
        e = np.array(exp.values, dtype=np.float32 if dtype == abi.F32 else np.float64).view(NP_BITS[dtype])
        assert np.array_equal(g, e)
    elif isinstance(got, DecimalArray):
        assert got.raw_ints() == exp.values
    else:
        assert [int(x) for x in got.value_array()] == exp.values
    assert (got.validity is not None) == (exp.validity is not None)
    if exp.validity is not None:
        assert [bool(x) for x in got.valid_mask()] == exp.validity
    assert got.null_count == exp.null_count


def run_both(fn_gpu, fn_oracle, dtype=None):
    try:
        exp = fn_oracle()
    except oc.CastError as e:
        with pytest.raises(ArrowError) as g:
            fn_gpu()
        assert (g.value.status, g.value.message, g.value.index) == (STATUS[e.status], e.message, e.index)
        return e
    got = fn_gpu()
    same(got, exp, dtype)
    return got


def dec_cast(gpu, a, w, p, s, safe):
    return run_both(lambda: gpu.cast_decimal(a, w, p, s, safe), lambda: oc.cast_decimal(to_operand(a), w, p, s, safe))


def to_dec(gpu, h, w, p, s, safe):
    return run_both(lambda: gpu.cast_to_decimal(h, w, p, s, safe), lambda: oc.cast_to_decimal(to_prim(h), w, p, s, safe))


def from_dec(gpu, a, to, safe):
    return run_both(lambda: gpu.cast_from_decimal(a, to, safe), lambda: oc.cast_from_decimal(to_operand(a), to, safe), to)


# ---- the reference's literal vectors -----------------------------------------------------------------------------------
def host_input(c):
    src = c["in"]
    if "width" in src:
        return DecimalArray.from_ints(src["width"], src["precision"], src["scale"], src["values"])
    return HostArray.from_list(src["dtype"], src["values"])


@pytest.mark.parametrize("c", golden_cases(), ids=lambda c: c["name"])
def test_reference_vectors(gpu, c):
    a, t = host_input(c), c["to"]
    if c["kind"] == "dec":
        call = lambda: gpu.cast_decimal(a, t["width"], t["precision"], t["scale"], c["safe"])  # noqa: E731
    elif c["kind"] == "to_dec":
        call = lambda: gpu.cast_to_decimal(a, t["width"], t["precision"], t["scale"], c["safe"])  # noqa: E731
    else:
        call = lambda: gpu.cast_from_decimal(a, t["dtype"], c["safe"])  # noqa: E731
    if "error" in c or "error_contains" in c:
        with pytest.raises(ArrowError) as e:
            call()
        assert e.value.message == c["error"] if c.get("error", "*") != "*" else c.get("error_contains", "") in e.value.message
    elif c["expected"] is None:  # the reference asserts only that the cast succeeds
        call()
    else:
        assert call().to_list() == c["expected"]


# ---- decimal -> decimal: every width pair x up / down / same scale x infallible / fallible x safe / unsafe ----------------
def rand_in_precision(rng, w, p, n, null_p=0.1, breakers=0):
    """Values within precision p (a few `breakers` at 10^p - 1 and -(10^p - 1)), nulls with 0 underneath."""
    hi = 10 ** p - 1
    vals = [int(x) for x in rng.integers(-min(hi, 2 ** 62), min(hi, 2 ** 62) + 1, n)]
    if p > 18:
        vals = [v * 10 ** (p - 18) + int(rng.integers(0, 2 ** 62)) % 10 ** (p - 18) for v in vals]
        vals = [max(-hi, min(hi, v)) for v in vals]
    for i in rng.integers(0, n, breakers):
        vals[int(i)] = hi if rng.random() < 0.5 else -hi
    return DecimalArray.from_ints(w, p, 0, [None if rng.random() < null_p else v for v in vals])


PAIR_TYPES = [  # (p_in, s_in, p_out, s_out) relative to each width's max precision: up / same / down, infallible / fallible
    lambda mi, mo: (min(mi, mo) - 3, 2, mo, 3),           # upscale, infallible
    lambda mi, mo: (mi, 2, mo, 4),                         # upscale, fallible
    lambda mi, mo: (min(mi, mo), 2, min(mi, mo), 2),       # same scale (clone when same width)
    lambda mi, mo: (mi, 2, max(min(mi, mo) - 1, 1), 2),   # same scale, narrower precision: fallible
    lambda mi, mo: (min(mi, mo), 5, min(mi, mo), 1),       # downscale, infallible
    lambda mi, mo: (mi, 4, max(mo - 5, 1), 1),            # downscale, fallible
]


@pytest.mark.parametrize("wi", WIDTHS)
@pytest.mark.parametrize("wo", WIDTHS)
@pytest.mark.parametrize("safe", [True, False])
def test_decimal_pairs(gpu, wi, wo, safe):
    rng = np.random.default_rng(wi * 100 + wo * 10 + safe)
    mi, mo = od.MAX_PRECISION[wi], od.MAX_PRECISION[wo]
    for k, f in enumerate(PAIR_TYPES):
        p_in, s_in, p_out, s_out = f(mi, mo)
        for n in (0, 1, 70, 5000):
            base = rand_in_precision(rng, wi, p_in, n, breakers=(2 if n > 10 and k in (1, 3, 5) and rng.random() < 0.5 else 0))
            a = DecimalArray(wi, p_in, s_in, base.values, base.length, base.validity, base.validity_offset, base.null_count)
            dec_cast(gpu, a, wo, p_out, s_out, safe)


@pytest.mark.parametrize("safe", [True, False])
def test_decimal_type_level_errors_and_zero_paths(gpu, safe):
    for n in (0, 3):
        a = DecimalArray.from_ints(4, 9, -128, [1, None, 2][:n])
        dec_cast(gpu, a, 16, 38, 10, safe)      # delta 138 wraps to -118: "Value overflows for output scale"
        dec_cast(gpu, DecimalArray.from_ints(16, 38, 0, [5, None, -7][:n]), 4, 9, 10, safe)   # delta 10 past Decimal32's table
        dec_cast(gpu, DecimalArray.from_ints(16, 38, 38, [5, None, -7][:n]), 8, 18, -100, safe)  # delta 138 wraps: all zero
        dec_cast(gpu, DecimalArray.from_ints(16, 38, 0, [5, None, -7][:n]), 16, 0, 0, safe)    # closing type check: precision 0
    # p_out above 127 is negative as i8: the "infallible" test fails, so rows see the precision error first (a scale change
    # or a width change: the same type with the same scale is the clone, decided in u8 before the i8 test)
    dec_cast(gpu, DecimalArray.from_ints(16, 38, 0, [5, 6]), 16, 200, 1, safe)
    dec_cast(gpu, DecimalArray.from_ints(8, 18, 0, [5, 6]), 16, 200, 0, safe)
    dec_cast(gpu, DecimalArray.from_ints(16, 38, 0, [5, 6]), 16, 38, 0, safe)
    e = dec_cast(gpu, DecimalArray.from_ints(16, 38, 0, [5, 6]), 16, 200, 0, safe)  # clone, then the type check
    assert isinstance(e, oc.CastError) and e.index == -1 and e.message.endswith("precision 200 is greater than max 38")
    a = DecimalArray.from_ints(16, 38, 0, [5, None, 7])
    a.values[1] = acu.i128_to_halves([2 ** 126])[0]
    r = dec_cast(gpu, a, 16, 38, 0, safe)  # the clone keeps the bytes under the null
    assert r.raw_ints() == [5, 2 ** 126, 7]


def test_garbage_under_nulls(gpu):
    """unary computes at null slots: a wrapping upscale writes the wrapped product there, and a narrowing that cannot
    convert a null slot's bytes is the unwrap panic at that slot."""
    big = 2 ** 120 + 12345
    a = DecimalArray.from_ints(16, 10, 0, [1, 2, 3, 4])
    a.values[2] = acu.i128_to_halves([big])[0]  # slot 2 valid-looking bytes, but null
    a.validity = acu.pack_bits([True, True, False, True])
    a.null_count = 1
    r = dec_cast(gpu, a, 16, 38, 20, True)      # p_in + 20 <= 38: infallible, wrapping
    assert r.raw_ints()[2] == od.wrap(16, big * 10 ** 20) and r.to_list() == [10 ** 20, 2 * 10 ** 20, None, 4 * 10 ** 20]
    b = DecimalArray.from_ints(16, 5, 0, [1, 2, 3, 4])
    b.values[2] = acu.i128_to_halves([big])[0]
    b.validity, b.null_count = a.validity, 1
    e = dec_cast(gpu, b, 4, 9, 2, False)        # 5 + 2 <= 9: unary; slot 2 does not fit i32
    assert isinstance(e, oc.CastError) and e.status == "Panic" and e.index == 2
    dec_cast(gpu, b, 4, 9, 2, True)             # the panic does not depend on `safe`
    dec_cast(gpu, b, 8, 5, -3, True)            # infallible downscale: i128 -> i64 after rounding fails at slot 2


# ---- integers -> decimal ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", INTS)
@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("safe", [True, False])
def test_integers_to_decimal(gpu, dt, w, safe):
    rng = np.random.default_rng(dt * 10 + w + safe)
    lo, hi = oc.INT_RANGE[dt]
    mp = od.MAX_PRECISION[w]
    for scale in (-3, -1, 0, 2, mp - 2):
        for n in (0, 5, 3000):
            vals = [int(x) for x in rng.integers(lo, hi, n, endpoint=True, dtype=acu.NP_DTYPES[dt])] if n else []
            if n:
                vals[:3] = [lo, hi, 0][:n]
            h = HostArray.from_list(dt, [None if rng.random() < 0.1 else v for v in vals])
            to_dec(gpu, h, w, mp, scale, safe)
            to_dec(gpu, h, w, min(mp, 5), min(scale, 5), safe)  # tight precision: precision errors / nulls
    to_dec(gpu, HostArray.from_list(dt, [1, None, 3]), w, mp, mp + 1, safe)  # 10^(mp+1) overflows the output native (or the type check)


def test_int8_factor_overflow_is_all_zero(gpu):
    h = HostArray.from_list(abi.I8, [127, None, -128])
    for safe in (True, False):
        r = to_dec(gpu, h, 16, 38, -3, safe)   # 10^3 overflows i8: unary(|_| 0), nulls kept
        assert r.to_list() == [0, None, 0] and r.raw_ints() == [0, 0, 0]


# ---- floats -> decimal ------------------------------------------------------------------------------------------------
SPECIAL = [0.0, -0.0, math.nan, math.inf, -math.inf, 5e-324, 2.2250738585072014e-308, 0.5, -0.5, 1.5, 2.5, -2.5,
           0.49999999999999994, 4503599627370495.5, -4503599627370495.5, 1.0e-5, 123.456, -9.99, 1e16, 1.7e38, -1.7e38, 3.4e38,
           9.2e18, -9.3e18, 2.147483647e9]


@pytest.mark.parametrize("dt", [abi.F32, abi.F64])
@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("safe", [True, False])
def test_floats_to_decimal(gpu, dt, w, safe):
    mp = od.MAX_PRECISION[w]
    for s in (0, 2, -2, mp):
        for i in range(len(SPECIAL)):  # each special value as the first failing row of its own array
            h = HostArray.from_list(dt, [1.25, None] + SPECIAL[i:])
            to_dec(gpu, h, w, mp, s, safe)
    rng = np.random.default_rng(w + dt)
    h = HostArray.from_numpy(dt, rng.standard_normal(4000) * 10.0 ** rng.integers(-3, 8, 4000), rng.random(4000) > 0.1)
    to_dec(gpu, h, w, mp, 3, safe)


def test_powi_scales(gpu):
    """Scales where 10_f64.powi(s) is not the correctly rounded 10^s (33, 37, -23): inputs whose result moves with it."""
    for s in (33, 37):
        mul_powi, mul_exact = oc.powi10(s), float(10 ** s)
        assert mul_powi != mul_exact
        vs = [x / 1000.0 for x in range(1, 1000)]
        moved = [v for v in vs if oc.round_half_away(mul_powi * v) != oc.round_half_away(mul_exact * v)]
        assert moved
        to_dec(gpu, HostArray.from_list(abi.F64, moved[:50]), 16, 38, s, True)
        ints = [10 ** (s - 30) * k + 7 for k in range(1, 300)]
        d = DecimalArray.from_ints(16, 38, s, ints)
        r = from_dec(gpu, d, abi.F64, True)
        assert any(float(x) / mul_powi != float(x) / mul_exact for x in ints)
    # -23: powi gives 1.0000000000000001e-23. 5e22 * powi(-23) is exactly 0.5 and rounds to 1, where the correctly rounded
    # 1e-23 gives 0.49999999999999994 and 0
    mul_powi, mul_exact = oc.powi10(-23), 1e-23
    ties = [5e22, -5e22, 1.5e23, 6.5e23, 1e23, 3e25, -7.5e24, 1.2345e30]
    assert oc.round_half_away(mul_powi * 5e22) == 1.0 and oc.round_half_away(mul_exact * 5e22) == 0.0
    r = to_dec(gpu, HostArray.from_list(abi.F64, ties), 16, 38, -23, False)
    assert r.raw_ints()[:2] == [1, -1]
    ints = [1, 7, 12345, -3, 10 ** 30]
    assert all(float(x) / mul_powi != float(x) / mul_exact for x in ints[:4])
    d = DecimalArray.from_ints(16, 38, -23, ints)
    r = from_dec(gpu, d, abi.F64, True)
    assert [float(v) for v in r.value_array()][:4] == [float(x) / mul_powi for x in ints[:4]]
    from_dec(gpu, d, abi.F32, True)


def test_i128_to_f64_ties_and_f32_double_rounding(gpu):
    ties = [2 ** 60 + 2 ** 7, 2 ** 60 + 3 * 2 ** 7, 2 ** 100 + 2 ** 47, 2 ** 100 + 3 * 2 ** 47, 2 ** 100 + 2 ** 47 + 1,
            -(2 ** 100 + 2 ** 47), 2 ** 127 - 1, -(2 ** 127), 2 ** 64, 2 ** 64 - 1, 2 ** 63]
    d = DecimalArray.from_ints(16, 38, 0, ties)
    r = from_dec(gpu, d, abi.F64, True)
    assert [float(x) for x in r.value_array()] == [float(v) for v in ties]  # Python's int -> float rounds to nearest even
    # f64 rounding then f32 rounding: 1 + 2^-24 + 2^-53 rounds to 1 + 2^-24 in f64 (a tie in f32) -> 1.0, whereas one
    # rounding to f32 would give 1 + 2^-23
    x = 2 ** 53 + 2 ** 29 + 1
    d = DecimalArray.from_ints(16, 38, 0, [x, None])
    r = from_dec(gpu, d, abi.F32, True)
    assert float(r.value_array()[0]) == 2.0 ** 53


# ---- decimal -> integers / floats ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("w", WIDTHS)
@pytest.mark.parametrize("to", INTS + [abi.F32, abi.F64])
@pytest.mark.parametrize("safe", [True, False])
def test_decimal_to_numeric(gpu, w, to, safe):
    rng = np.random.default_rng(w * 100 + to + safe)
    mp = od.MAX_PRECISION[w]
    lo, hi = od.lo_hi(w)
    for s in (0, 2, -1, -3, mp):
        for n in (0, 7, 3000):
            vals = [int(x) for x in rng.integers(-10 ** 6, 10 ** 6, n)]
            if n:
                vals[0] = hi // 10 ** (n % 3)
                vals[-1] = lo + 1
            a = DecimalArray.from_ints(w, mp, s, [None if rng.random() < 0.1 else v for v in vals])
            from_dec(gpu, a, to, safe)
            a = DecimalArray.from_ints(w, mp, s, vals)  # no nulls: the builder leaves out the NullBuffer unless a row fails
            from_dec(gpu, a, to, safe)
    from_dec(gpu, DecimalArray.from_ints(w, mp, -(mp + 1), [1]), to, safe)  # 10^(mp+1) overflows the decimal native


# ---- zero-copy slices, misaligned Decimal128, empty arrays --------------------------------------------------------------
def sliced_descriptor(gpu, d, shift, n):
    da = gpu.upload(d)
    desc = da.descriptor()
    desc.values += shift * d.width()
    desc.validity_offset += shift
    desc.len = n
    desc.null_count = -1 if d.validity is not None else 0
    return da, desc


@pytest.mark.parametrize("shift", [1, 5, 63])
def test_sliced_inputs(gpu, shift):
    rng = np.random.default_rng(shift)
    n = 4500
    for wi, wo, (p_in, s_in, p_out, s_out) in ((16, 8, (38, 6, 18, 2)), (4, 16, (9, 2, 38, 10)), (8, 4, (18, 3, 9, 1))):
        base = rand_in_precision(rng, wi, p_in, n + shift, breakers=3)
        a = DecimalArray(wi, p_in, s_in, base.values, base.length, base.validity, base.validity_offset, base.null_count)
        for safe in (True, False):
            da, ad = sliced_descriptor(gpu, a, shift, n)
            out = gpu.alloc_out(n * wo, n)
            try:
                ft, tt = abi.DecimalType(wi, p_in, s_in), abi.DecimalType(wo, p_out, s_out)
                st = gpu.lib.acu_cast_decimal(gpu.h, C.byref(ft), C.byref(tt), int(safe), C.byref(ad), C.byref(out))
                try:
                    exp = oc.cast_decimal(to_operand(a.slice(shift, n)), wo, p_out, s_out, safe)
                except oc.CastError as e:
                    d = gpu.lib.acu_last_error(gpu.h).contents
                    assert (st, d.message.decode(), d.index) == (STATUS[e.status], e.message, e.index)
                    continue
                assert st == abi.OK
                h = gpu.download_out(out, {4: abi.I32, 8: abi.I64, 16: abi.I128}[wo])
                out = None
                same(DecimalArray(wo, p_out, s_out, h.values, h.length, h.validity, 0, h.null_count), exp)
            finally:
                if out is not None:
                    gpu._free_out(out)
                da.free()
    # integer and float sources at odd offsets
    h = HostArray.from_numpy(abi.I16, rng.integers(-30000, 30000, n + shift), rng.random(n + shift) > 0.2)
    da, ad = sliced_descriptor(gpu, h, shift, n)
    out = gpu.alloc_out(n * 16, n)
    try:
        tt = abi.DecimalType(16, 10, 3)
        gpu.check(gpu.lib.acu_cast_to_decimal(gpu.h, abi.I16, C.byref(tt), 1, C.byref(ad), C.byref(out)))
        got = gpu.download_out(out, abi.I128)
        out = None
        exp = oc.cast_to_decimal(to_prim(h.slice(shift, n)), 16, 10, 3, True)
        same(DecimalArray(16, 10, 3, got.values, got.length, got.validity, 0, got.null_count), exp)
    finally:
        if out is not None:
            gpu._free_out(out)
        da.free()


def test_misaligned_decimal128_is_refused(gpu):
    a = DecimalArray.from_ints(16, 38, 2, [1, 2, 3])
    da = gpu.upload(a)
    out = gpu.alloc_out(64, 3)
    try:
        d = da.descriptor()
        d.values += 8
        ft, tt = abi.DecimalType(16, 38, 2), abi.DecimalType(16, 38, 1)
        assert gpu.lib.acu_cast_decimal(gpu.h, C.byref(ft), C.byref(tt), 1, C.byref(d), C.byref(out)) == abi.ERR_INVALID_ARGUMENT
        assert gpu.lib.acu_cast_from_decimal(gpu.h, C.byref(ft), abi.I64, 1, C.byref(d), C.byref(out)) == abi.ERR_INVALID_ARGUMENT
        d.values -= 8
        o = abi.ArrayOut()
        o.values, o.validity = out.values + 8, out.validity
        assert gpu.lib.acu_cast_to_decimal(gpu.h, abi.I64, C.byref(tt), 1, C.byref(d), C.byref(o)) == abi.ERR_INVALID_ARGUMENT
        assert "16-byte aligned" in gpu.lib.acu_last_error(gpu.h).contents.message.decode()
    finally:
        gpu._free_out(out)
        da.free()


def test_empty_arrays_raise_type_level_errors(gpu):
    e = DecimalArray.from_ints(4, 9, 2, [])
    with pytest.raises(ArrowError) as x:
        gpu.cast_decimal(DecimalArray.from_ints(16, 38, -128, []), 16, 38, 10)
    assert x.value.message == "Cast error: Cannot cast to Decimal128(38, 10). Value overflows for output scale"
    with pytest.raises(ArrowError) as x:
        gpu.cast_from_decimal(DecimalArray.from_ints(4, 9, -10, []), abi.I64)
    assert x.value.message == "Cast error: Cannot cast to \"Decimal32\". The scale -10 causes overflow."
    with pytest.raises(ArrowError) as x:
        gpu.cast_to_decimal(HostArray.from_list(abi.I64, []), 4, 9, 10)
    assert x.value.message == "Cast error: Cannot cast to \"Decimal32\"(9, 10). The scale causes overflow."
    r = gpu.cast_from_decimal(e, abi.I32)
    assert r.length == 0 and r.validity is None
    r = gpu.cast_decimal(e, 8, 5, 2, safe=True)  # fallible (9 > 5): unary_opt always carries a NullBuffer
    assert r.length == 0 and r.validity is not None
    r = gpu.cast_decimal(e, 8, 18, 2, safe=True)  # infallible: unary keeps the input's (absent) nulls
    assert r.length == 0 and r.validity is None


# ---- multi-round sizes: a rescale over more than one grid-stride round, and its first failing row at every placement -------
@pytest.mark.parametrize("wi,wo", [(16, 16), (8, 4)])
def test_multi_round_first_error_row(gpu, wi, wo):
    """Decimal(18, 4) -> (9 or 38, 1) on a periodic column (test_gpu_decimal_edges) with safe = True against the oracle
    on one period; then -> (9, 1) with safe = False and 10^17 at every placement of test_gpu_elementwise_rounds."""
    n = sized(gpu, SG)
    rng = np.random.default_rng(wi + wo)
    x = [int(v) for v in rng.integers(-2 * 10 ** 12, 2 * 10 ** 12, P)]
    mask = rng.integers(0, 100, P) >= 3
    src, dst = {8: abi.I64, 16: abi.I128}[wi], {4: abi.I32, 16: abi.I128}[wo]
    p_out = 9 if wo == 4 else 38
    col = Periodic(gpu, src, raw_of(DecimalArray.from_ints(wi, 18, 4, x)), mask, n)
    try:
        d = col.descriptor()
        ft, tt, t9 = abi.DecimalType(wi, 18, 4), abi.DecimalType(wo, p_out, 1), abi.DecimalType(wo, 9, 1)
        exp = oc.cast_decimal(od.Operand(wi, 18, 4, x, mask.tolist()), wo, p_out, 1, True)
        assert (exp.null_count > int((~mask).sum())) == (wo == 4)  # quotients past 9 digits become nulls
        st, out = Call(gpu, n, n * wo, lambda o: gpu.lib.acu_cast_decimal(gpu.h, C.byref(ft), C.byref(tt), 1, C.byref(d), C.byref(o)))()
        try:
            assert st == abi.OK
            check_out(gpu, out, n, dst, exp_from(exp, dst), f"{wi}->{wo} safe")
        finally:
            gpu._free_out(out)
        # values whose quotients all fit 9 digits, then 10^17 / 10^3 = 10^14: past Decimal32's i32 (the rescale itself
        # fails) and past 9 digits of Decimal128(9, 1)
        small = [v % 10 ** 11 - 5 * 10 ** 10 for v in x]
        col.base = (raw_of(DecimalArray.from_ints(wi, 18, 4, small)), mask)
        col.restore()
        if wo == 4:
            err = (abi.ERR_CAST, f"Cast error: Cannot cast to Decimal32(9, 1). Overflowing on {10 ** 17}")
        else:
            err = (abi.ERR_INVALID_ARGUMENT, f"Invalid argument error: {10 ** 13}.0 is too large to store in a Decimal128 of precision 9. "
                                             "Max is 99999999.9")
        call = Call(gpu, n, n * wo, lambda o: gpu.lib.acu_cast_decimal(gpu.h, C.byref(ft), C.byref(t9), 0, C.byref(d), C.byref(o)))
        st, out = call()
        gpu._free_out(out)
        assert st == abi.OK
        check_placements(gpu, n, [(col, raw_value(src, 10 ** 17))], call, lambda: err, f"{wi}->{wo}")
    finally:
        col.free()
