"""Python restatement of the reference's decimal casts, in Python integers and floats.

cast_decimal_to_decimal(_same_type) with make_upscaler / make_downscaler / apply_decimal_cast
(arrow-cast/src/cast/decimal.rs:161-529), cast_integer_to_decimal (mod.rs:366-444), cast_floating_point_to_decimal
(decimal.rs:836-885), cast_decimal_to_integer (:887-987) and cast_decimal_to_float (:994-1004, mod.rs:86-92), with
validate_decimal{32,64,}_precision and format_decimal_str_internal (arrow-data/src/decimal.rs:1030-1167).

Integer steps are exact and range-checked, so "checked" / "wrapping" are restated literally. Floats: Python floats are
IEEE binary64 and `*`, `/` are single correctly rounded operations. Python's round() is half-to-even and is not used;
round half away from zero is math.floor / math.ceil on the exact value. 10_f64.powi(e) is restated as the repeated
squaring loop of compiler-builtins' `pow`.

Arrays are od.Operand (width = 4 / 8 / 16 for decimals) or `Prim(dtype, values, validity)` for integer and float columns.
A result is `Out(values, validity, null_count)`: values at every slot (what the reference writes under nulls too).
"""
import math
from dataclasses import dataclass
from typing import List, Optional

import numpy as np

import oracle_decimal as od

I8, I16, I32, I64, U8, U16, U32, U64, F32, F64 = range(10)
DTYPE_NAME = ["Int8", "Int16", "Int32", "Int64", "UInt8", "UInt16", "UInt32", "UInt64", "Float32", "Float64"]
INT_RANGE = {I8: (-2 ** 7, 2 ** 7 - 1), I16: (-2 ** 15, 2 ** 15 - 1), I32: (-2 ** 31, 2 ** 31 - 1), I64: (-2 ** 63, 2 ** 63 - 1),
             U8: (0, 2 ** 8 - 1), U16: (0, 2 ** 16 - 1), U32: (0, 2 ** 32 - 1), U64: (0, 2 ** 64 - 1)}
PREFIX = {"InvalidArgument": "Invalid argument error: ", "ArithmeticOverflow": "Arithmetic overflow: ", "Cast": "Cast error: ",
          "Panic": ""}
UNWRAP_NONE = "called `Option::unwrap()` on a `None` value"


class CastError(Exception):
    """status: 'InvalidArgument' | 'ArithmeticOverflow' | 'Cast' | 'Panic'; message: Display text; index: row or -1."""

    def __init__(self, status, text, index=-1):
        message = PREFIX[status] + text
        super().__init__(message)
        self.status, self.message, self.index = status, message, index


@dataclass
class Prim:
    dtype: int
    values: list
    validity: Optional[List[bool]] = None

    def valid(self, i):
        return self.validity is None or self.validity[i]


@dataclass
class Out:
    values: list
    validity: Optional[List[bool]]
    null_count: int


def prefix(width):
    return f"Decimal{8 * width}"


def i8(v):
    return od.i8_wrap(v)


def max_for(width, p):
    """MAX_FOR_EACH_PRECISION[p], or None past the table."""
    return 10 ** p - 1 if 0 <= p <= od.MAX_PRECISION[width] else None


def is_valid_precision(width, v, p):
    return p <= od.MAX_PRECISION[width] and -(10 ** p - 1) <= v <= 10 ** p - 1


def format_decimal_str_internal(value_str, precision, scale, safe):
    sign, rest = ("-", value_str[1:]) if value_str.startswith("-") else ("", value_str)
    bound = min(precision, len(rest)) + len(sign) if safe else len(value_str)
    value_str = value_str[:bound]
    if scale == 0:
        return value_str
    if scale < 0:
        return value_str + "0" * (-scale)
    if len(rest) > scale:
        return f"{value_str[:len(value_str) - scale]}.{value_str[len(value_str) - scale:]}"
    return f"{sign}0.{rest.rjust(scale, '0')}"


def precision_error(width, v, p, s):
    name, mp = prefix(width), od.MAX_PRECISION[width]
    if p > mp:
        return CastError("InvalidArgument", f"Max precision of a {name} is {mp}, but got {p}")
    hi = 10 ** p - 1
    a = format_decimal_str_internal(str(v), p, s, False)
    if v > hi:
        return CastError("InvalidArgument", f"{a} is too large to store in a {name} of precision {p}. "
                                            f"Max is {format_decimal_str_internal(str(hi), p, s, True)}")
    return CastError("InvalidArgument", f"{a} is too small to store in a {name} of precision {p}. "
                                        f"Min is {format_decimal_str_internal(str(-hi), p, s, True)}")


def powi10(e):
    """10_f64.powi(e): compiler-builtins' pow (repeated squaring, 1 / r for e < 0)."""
    a, r, k = 10.0, 1.0, abs(e)
    while True:
        if k & 1:
            r *= a
        k >>= 1
        if not k:
            break
        a *= a
    return 1.0 / r if e < 0 else r


def round_half_away(x):
    """f64::round: half away from zero (x integral or not; NaN / inf pass through)."""
    if math.isnan(x) or math.isinf(x):
        return x
    f = math.floor(abs(x))
    r = f + 1 if abs(x) - f >= 0.5 else f
    return math.copysign(float(r), x)


def float_to_int(x, lo, hi):
    """num_traits to_iN of an f64: NaN / inf / out of range -> None, else truncation."""
    if math.isnan(x) or math.isinf(x):
        return None
    t = int(x)
    return t if lo <= t <= hi else None


def f32(v):
    """`as f32` of an f64: round to nearest even, inf beyond the f32 range."""
    with np.errstate(over="ignore"):
        return float(np.float32(v))


def float_debug(v, is_f32):
    """Rust's `{:?}` of an f32 / f64."""
    if math.isnan(v):
        return "NaN"
    if math.isinf(v):
        return "-inf" if v < 0 else "inf"
    if v == 0:
        return "-0.0" if math.copysign(1.0, v) < 0 else "0.0"
    for prec in range(18):
        t = f"{v:.{prec}e}"
        if (np.float32(t) == np.float32(v)) if is_f32 else (float(t) == v):
            break
    mant, e = t.lstrip("-").split("e")
    e = int(e)
    digits = mant.replace(".", "").rstrip("0") or "0"
    a = abs(v)
    lo, hi = (float(np.float32(1e-4)), float(np.float32(1e16))) if is_f32 else (1e-4, 1e16)
    sign = "-" if v < 0 else ""
    if a < lo or a >= hi:
        return f"{sign}{digits[0]}{'.' + digits[1:] if len(digits) > 1 else ''}e{e}"
    if e >= 0:
        whole = digits[:e + 1].ljust(e + 1, "0")
        return f"{sign}{whole}.{digits[e + 1:] or '0'}"
    return f"{sign}0.{'0' * (-e - 1)}{digits}"


def fits(width_or_dtype, v, decimal=True):
    if decimal:
        return od.fits(width_or_dtype, v)
    lo, hi = INT_RANGE[width_or_dtype]
    return lo <= v <= hi


def trunc_div(a, b):
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def _run(n, valid, kind, row, what):
    """Apply `row` (returns (value) or raises a _RowFail) under one of the reference's combinators."""
    out = [0] * n
    if kind == "unary":  # every slot; a failure is the unwrap panic at the lowest slot
        for i in range(n):
            try:
                out[i] = row(i)
            except _RowFail:
                raise CastError("Panic", UNWRAP_NONE, i)
        validity = None if valid is None else list(valid)
        return Out(out, validity, 0 if valid is None else valid.count(False))
    if kind == "opt":  # unary_opt: 0 + null on failure, always a NullBuffer
        validity = [True] * n if valid is None else list(valid)
        for i in range(n):
            if not validity[i]:
                continue
            try:
                out[i] = row(i)
            except _RowFail:
                validity[i] = False
        return Out(out, validity, validity.count(False))
    # try_unary
    for i in range(n):
        if valid is not None and not valid[i]:
            continue
        try:
            out[i] = row(i)
        except _RowFail as f:
            e = what(i, f)
            e.index = i
            raise e
    return Out(out, None if valid is None else list(valid), 0 if valid is None else valid.count(False))


class _RowFail(Exception):
    def __init__(self, step, mid=None):
        super().__init__(step)
        self.step, self.mid = step, mid


def _finish(out, width, p, s):
    msg = od.validate_type(width, p, s)
    if msg:
        raise CastError("InvalidArgument", msg)
    return out


def _validity(a):
    return None if a.validity is None else [bool(x) for x in a.validity]


def cast_decimal(a: od.Operand, width, p_out, s_out, safe) -> Out:
    """Decimal -> Decimal (all nine width pairs)."""
    wi, p_in, s_in, n = a.width, a.precision, a.scale, len(a.values)
    valid = _validity(a)
    name = f"{prefix(width)}({p_out}, {s_out})"

    def overflowing(i, f):
        if f.step == "precision":
            return precision_error(width, f.mid, p_out, s_out)
        return CastError("Cast", f"Cannot cast to {name}. Overflowing on {a.values[i]}")

    if wi == width and s_in == s_out and p_in <= p_out:  # array.clone(): compared as u8, before any i8 arithmetic
        return _finish(Out(list(a.values), valid, 0 if valid is None else valid.count(False)), width, p_out, s_out)
    if s_in <= s_out:
        delta = i8(s_out - s_in)
        mx = max_for(width, delta)
        if mx is None:
            raise CastError("Cast", f"Cannot cast to {name}. Value overflows for output scale")
        mul = mx + 1
        infallible = i8(i8(p_in) + delta) <= i8(p_out)
        if infallible:
            def row(i):
                x = a.values[i]
                if not fits(width, x):
                    raise _RowFail("none")
                return od.wrap(width, x * mul)
            return _finish(_run(n, valid, "unary", row, None), width, p_out, s_out)

        def row(i):
            x = a.values[i]
            if not fits(width, x) or not fits(width, x * mul):
                raise _RowFail("none")
            v = x * mul
            if not is_valid_precision(width, v, p_out):
                raise _RowFail("precision", v)
            return v
    else:
        delta = i8(s_in - s_out)
        mx = max_for(wi, delta)
        if mx is None:  # every value rounds to zero
            return _finish(Out([0] * n, valid, 0 if valid is None else valid.count(False)), width, p_out, s_out)
        div = mx + 1
        half = div // 2
        infallible = i8(i8(p_in) - delta) < i8(p_out)

        def down(x):
            d, r = trunc_div(x, div), x - trunc_div(x, div) * div
            if x >= 0 and r >= half:
                d += 1
            elif x < 0 and r <= -half:
                d -= 1
            if not fits(width, d):
                raise _RowFail("none")
            return d

        if infallible:
            return _finish(_run(n, valid, "unary", lambda i: down(a.values[i]), None), width, p_out, s_out)

        def row(i):
            v = down(a.values[i])
            if not is_valid_precision(width, v, p_out):
                raise _RowFail("precision", v)
            return v
    return _finish(_run(n, valid, "opt" if safe else "try", row, overflowing), width, p_out, s_out)


def cast_to_decimal(a: Prim, width, p, s, safe) -> Out:
    """Int8..UInt64 / Float32 / Float64 -> Decimal."""
    n, valid = len(a.values), a.validity
    name = f"{prefix(width)}({p}, {s})"
    if a.dtype in (F32, F64):
        mul = powi10(s)
        lo, hi = od.lo_hi(width)

        def row(i):
            x = round_half_away(mul * float(a.values[i]))
            v = float_to_int(x, lo, hi)
            if v is None:
                raise _RowFail("none")
            if not is_valid_precision(width, v, p):
                raise _RowFail("precision", v)
            return v

        def what(i, f):
            if f.step == "precision":
                return precision_error(width, f.mid, p, s)
            return CastError("Cast", f"Cannot cast to {name}. Overflowing on {float_debug(a.values[i], a.dtype == F32)}")
        return _finish(_run(n, valid, "opt" if safe else "try", row, what), width, p, s)

    if s < 0:
        factor = 10 ** (-s)
        if not fits(a.dtype, factor, decimal=False):  # beyond the source type: unary(|_| 0)
            return _finish(Out([0] * n, valid, 0 if valid is None else valid.count(False)), width, p, s)

        def row(i):
            v = trunc_div(a.values[i], factor)
            if not fits(width, v):
                raise _RowFail("none")
            if not is_valid_precision(width, v, p):
                raise _RowFail("precision", v)
            return v
    else:
        if not fits(width, 10 ** s):
            raise CastError("Cast", f"Cannot cast to \"{prefix(width)}\"({p}, {s}). The scale causes overflow.")
        factor = 10 ** s

        def row(i):
            x = a.values[i]
            if not fits(width, x):
                raise _RowFail("none")
            if not fits(width, x * factor):
                raise _RowFail("mul", x)
            v = x * factor
            if not is_valid_precision(width, v, p):
                raise _RowFail("precision", v)
            return v

    def what(i, f):
        if f.step == "precision":
            return precision_error(width, f.mid, p, s)
        if f.step == "mul":
            return CastError("ArithmeticOverflow", f"Overflow happened on: {f.mid} * {factor}")
        return CastError("Cast", f"Cannot cast to {name}. Overflowing on {a.values[i]}")
    return _finish(_run(n, valid, "opt" if safe else "try", row, what), width, p, s)


def cast_from_decimal(a: od.Operand, to, safe) -> Out:
    """Decimal -> Int8..UInt64 / Float32 / Float64."""
    n, valid, w, s = len(a.values), _validity(a), a.width, a.scale
    if to in (F32, F64):
        d = powi10(s)

        def row(i):
            x = float(a.values[i]) / d  # int -> float rounds to nearest, ties to even, then one IEEE division
            return f32(x) if to == F32 else x
        return _run(n, valid, "unary", row, None)
    k = 10 ** abs(s)
    if not fits(w, k):
        raise CastError("Cast", f"Cannot cast to \"{prefix(w)}\". The scale {s} causes overflow.")
    out, validity = [0] * n, [True] * n if valid is None else list(valid)
    for i in range(n):
        if not validity[i]:
            continue
        x = a.values[i]
        if s >= 0:
            v = trunc_div(x, k)
        else:
            v = x * k
            if not fits(w, v):
                if safe:
                    validity[i] = False
                    continue
                raise CastError("ArithmeticOverflow", f"Overflow happened on: {x} * {k}", i)
        if not fits(to, v, decimal=False):
            if safe:
                validity[i] = False
                continue
            raise CastError("Cast", f"value of {v} is out of range {DTYPE_NAME[to]}", i)
        out[i] = v
    nc = validity.count(False)
    return Out(out, validity if nc else None, nc)
