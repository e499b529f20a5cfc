"""Python restatement of the reference's decimal arithmetic, comparison and aggregates, in Python integers.

decimal_op (arrow-arith/src/numeric.rs:970-1107) with try_op! (:303-317), neg_checked (:116-136), compare_op on decimals
(arrow-ord/src/cmp.rs:220-382) and sum / min / max (arrow-arith/src/aggregate.rs:943,1012,1027). "Checked" is a range
check of the exact integer result, so this is exact by construction. The result type follows Rust's i8 / u8 arithmetic;
where the reference's i8 subtractions overflow (a panic in debug builds) it wraps, as a release build does, which is what
the library documents.

An operand is an `Operand`: width (4 / 8 / 16), precision, scale, raw values (Python ints at every slot, nulls included),
validity (list of bool, or None = no NullBuffer), null count, is_scalar.
"""
from dataclasses import dataclass
from typing import List, Optional

MAX_PRECISION = {4: 9, 8: 18, 16: 38}  # = MAX_SCALE
ADD_WRAPPING, ADD, SUB_WRAPPING, SUB, MUL_WRAPPING, MUL, DIV, REM = range(8)
OP_SYMBOL = {ADD_WRAPPING: "+", ADD: "+", SUB_WRAPPING: "-", SUB: "-", MUL_WRAPPING: "*", MUL: "*", DIV: "/", REM: "%"}
EQ, NEQ, LT, LT_EQ, GT, GT_EQ, DISTINCT, NOT_DISTINCT = range(8)


# Display of the ArrowError variants (arrow-schema/src/error.rs); DivideByZero displays as "Divide by zero error"
DISPLAY_PREFIX = {"InvalidArgument": "Invalid argument error: ", "ArithmeticOverflow": "Arithmetic overflow: ",
                  "DivideByZero": "", "Compute": "Compute error: "}


class DecimalError(Exception):
    """status: 'InvalidArgument' | 'ArithmeticOverflow' | 'DivideByZero' | 'Compute'; message: the error's Display text
    (what the reference's tests compare `to_string()` with); index: failing row or -1."""

    def __init__(self, status, text, index=-1):
        message = DISPLAY_PREFIX[status] + text
        super().__init__(message)
        self.status, self.message, self.index = status, message, index


@dataclass
class Operand:
    width: int
    precision: int
    scale: int
    values: List[int]
    validity: Optional[List[bool]] = None
    is_scalar: bool = False

    @property
    def null_count(self):
        return 0 if self.validity is None else sum(1 for v in self.validity if not v)

    def valid(self, i):
        return self.validity is None or self.validity[i]


# ---- Rust integer rules ------------------------------------------------------------------------------------------------
def i8_wrap(v):
    return ((v + 128) % 256) - 128


def i8_sat(v):
    return max(-128, min(127, v))


def u8_sat(v):
    return min(255, v)


def as_u8(v):  # i8 `as u8`
    return v % 256


def as_u32(v):  # i8 `as u32`, sign-extending
    return v % (1 << 32)


def lo_hi(width):
    b = 8 * width
    return -(1 << (b - 1)), (1 << (b - 1)) - 1


def fits(width, v):
    lo, hi = lo_hi(width)
    return lo <= v <= hi


def wrap(width, v):
    b = 8 * width
    return ((v + (1 << (b - 1))) % (1 << b)) - (1 << (b - 1))


def pow10_checked(width, exp):
    v = 10 ** exp if exp < 200 else None
    if v is None or not fits(width, v):
        raise DecimalError("ArithmeticOverflow", f"Overflow happened on: 10 ^ {exp}")
    return v


def pow10_wrapping(width, exp):
    return 0 if exp >= 8 * width else wrap(width, 10 ** exp)


def validate_type(width, p, s):
    """validate_decimal_precision_and_scale (arrow-array/src/types.rs:1442-1472): message or None."""
    mp = MAX_PRECISION[width]
    if p == 0:
        return f"precision cannot be 0, has to be between [1, {mp}]"
    if p > mp:
        return f"precision {p} is greater than max {mp}"
    if s > mp:
        return f"scale {s} is greater than max {mp}"
    if s > 0 and s > p:
        return f"scale {s} is greater than precision {p}"
    return None


def type_name(width, p, s):
    return f"Decimal{8 * width}({p}, {s})"


def result_type(op, width, p1, s1, p2, s2):
    """(precision, scale, l_mul, r_mul, checked_pows) before any row: raises the pre-loop errors."""
    mp = MAX_PRECISION[width]
    if op in (ADD, ADD_WRAPPING, SUB, SUB_WRAPPING, REM):
        rs = max(s1, s2)
        d1, d2 = i8_wrap(p1 - s1), i8_wrap(p2 - s2)
        le, re = as_u32(i8_wrap(rs - s1)), as_u32(i8_wrap(rs - s2))
        if op == REM:
            rp = min(as_u8(i8_sat(rs + min(d1, d2))), mp)
            return rp, rs, pow10_wrapping(width, le), pow10_wrapping(width, re)
        rp = min(u8_sat(as_u8(i8_sat(rs + max(d1, d2))) + 1), mp)
        return rp, rs, pow10_checked(width, le), pow10_checked(width, re)
    if op in (MUL, MUL_WRAPPING):
        rp = min(u8_sat(p1 + p2 + 1), mp)
        rs = i8_sat(s1 + s2)
        if rs > mp:
            raise DecimalError("InvalidArgument", f"Output scale of {type_name(width, p1, s1)} * {type_name(width, p2, s2)} "
                                                  f"would exceed max scale of {mp}")
        return rp, rs, 1, 1
    if op == DIV:
        rs = min(i8_sat(s1 + 4), mp)
        mul_pow = i8_wrap(i8_wrap(rs - s1) + s2)
        rp = min(as_u8(i8_sat(mul_pow + p1)), mp)
        if mul_pow > 0:
            return rp, rs, pow10_checked(width, mul_pow), 1
        if mul_pow < 0:
            return rp, rs, 1, pow10_checked(width, as_u32(i8_wrap(-mul_pow)))
        return rp, rs, 1, 1
    raise DecimalError("InvalidArgument", f"Invalid arithmetic operation: op {op}")


def _ovf(a, sym, b):
    return DecimalError("ArithmeticOverflow", f"Overflow happened on: {a} {sym} {b}")


def _mul(width, a, b):
    v = a * b
    if not fits(width, v):
        raise _ovf(a, "*", b)
    return v


def row(op, width, l, r, l_mul, r_mul):
    """One row in the reference's evaluation order: receiver, argument, then the op."""
    if op in (MUL, MUL_WRAPPING):
        return _mul(width, l, r)
    l = _mul(width, l, l_mul)
    r = _mul(width, r, r_mul)
    if op in (ADD, ADD_WRAPPING, SUB, SUB_WRAPPING):
        v = l + r if op in (ADD, ADD_WRAPPING) else l - r
        if not fits(width, v):
            raise _ovf(l, OP_SYMBOL[op], r)
        return v
    if r == 0:
        raise DecimalError("DivideByZero", "Divide by zero error")
    q = abs(l) // abs(r) * (1 if (l < 0) == (r < 0) else -1)  # truncated toward zero
    v = q if op == DIV else l - q * r
    if not fits(width, q):  # MIN / -1; checked_rem fails on the same pair
        raise _ovf(l, OP_SYMBOL[op], r)
    return v


@dataclass
class Result:
    width: int
    precision: int
    scale: int
    values: List[int]          # raw values, 0 under nulls
    validity: Optional[List[bool]]
    null_count: int


def decimal_op(op, a: Operand, b: Operand) -> Result:
    """decimal_op over try_op!: pre-loop errors, rows (lowest failing valid row), then with_precision_and_scale."""
    assert a.width == b.width
    w = a.width
    for t in (a, b):
        msg = validate_type(w, t.precision, t.scale)
        if msg:
            raise DecimalError("InvalidArgument", msg)
    rp, rs, l_mul, r_mul = result_type(op, w, a.precision, a.scale, b.precision, b.scale)

    def finish(values, validity, nc):
        msg = validate_type(w, rp, rs)
        if msg:
            raise DecimalError("InvalidArgument", msg)
        return Result(w, rp, rs, values, validity, nc)

    if a.is_scalar != b.is_scalar:  # try_unary over the array; a null scalar gives new_null
        s, arr = (a, b) if a.is_scalar else (b, a)
        n = len(arr.values)
        if s.null_count:
            return finish([0] * n, [False] * n, n)
        validity = arr.validity
        rows = [(s.values[0], arr.values[i]) if a.is_scalar else (arr.values[i], s.values[0]) for i in range(n)]
    else:  # try_binary
        if len(a.values) != len(b.values):
            raise DecimalError("Compute", "Cannot perform a binary operation on arrays of different length")
        n = len(a.values)
        if n == 0:
            return finish([], None, 0)
        an, bn = a.null_count, b.null_count
        if a.validity is not None and b.validity is not None and (an or bn):
            validity = [x and y for x, y in zip(a.validity, b.validity)]
        elif a.validity is not None and b.validity is None and an:
            validity = list(a.validity)
        elif b.validity is not None and a.validity is None and bn:
            validity = list(b.validity)
        else:
            validity = None
        rows = list(zip(a.values, b.values))
    out = []
    for i, (l, r) in enumerate(rows):
        if validity is not None and not validity[i]:
            out.append(0)
            continue
        try:
            out.append(row(op, w, l, r, l_mul, r_mul))
        except DecimalError as e:
            e.index = i
            raise
    nc = 0 if validity is None else sum(1 for v in validity if not v)
    return finish(out, None if validity is None else list(validity), nc)


def neg(a: Operand) -> Result:
    """neg_checked through try_unary, the input type kept."""
    out = []
    for i, v in enumerate(a.values):
        if not a.valid(i):
            out.append(0)
            continue
        if not fits(a.width, -v):
            raise DecimalError("ArithmeticOverflow", f"Overflow happened on: - {v}", i)
        out.append(-v)
    return Result(a.width, a.precision, a.scale, out, None if a.validity is None else list(a.validity), a.null_count)


def type_equal_or_error(op_text, a: Operand, b: Operand):
    """compare_op refuses decimal operands whose DataTypes differ (cmp.rs:260-263)."""
    lt, rt = type_name(a.width, a.precision, a.scale), type_name(b.width, b.precision, b.scale)
    if a.width != b.width or lt != rt:
        raise DecimalError("InvalidArgument", f"Invalid comparison operation: {lt} {op_text} {rt}")


def cmp(op, a: Operand, b: Operand):
    """(values, validity or None): values of every slot (predicate of the raw values), validity when the result has a
    NullBuffer. Both operands are decimals of one type (compare_op's type check is done by type_equal_or_error)."""
    ls, rs_ = a.is_scalar, b.is_scalar
    n = len(b.values) if ls and not rs_ else len(a.values)
    if not ls and not rs_ and len(a.values) != len(b.values):
        raise DecimalError("InvalidArgument", f"Cannot compare arrays of different lengths, got {len(a.values)} vs {len(b.values)}")
    if n == 0:
        return [], None
    ln, rn = a.null_count > 0, b.null_count > 0
    fold = op in (DISTINCT, NOT_DISTINCT)
    if not fold and ((ls and ln) or (rs_ and rn)) and not (ls and rs_):
        return [False] * n, [False] * n
    lv = [a.values[0 if ls and not rs_ else i] for i in range(n)]
    rv = [b.values[0 if rs_ and not ls else i] for i in range(n)]
    lm = [a.valid(0 if ls and not rs_ else i) for i in range(n)]
    rm = [b.valid(0 if rs_ and not ls else i) for i in range(n)]
    pred = {EQ: lambda x, y: x == y, NEQ: lambda x, y: x != y, LT: lambda x, y: x < y, LT_EQ: lambda x, y: x <= y,
            GT: lambda x, y: x > y, GT_EQ: lambda x, y: x >= y, DISTINCT: lambda x, y: x != y,
            NOT_DISTINCT: lambda x, y: x == y}[op]
    vals = [pred(x, y) for x, y in zip(lv, rv)]
    if op == DISTINCT:
        vals = [(p != q) or (p and q and v) for v, p, q in zip(vals, lm, rm)]
    elif op == NOT_DISTINCT:
        vals = [(not p and not q) or (p and q and v) for v, p, q in zip(vals, lm, rm)]
    if fold or not (ln or rn):
        return vals, None
    return vals, [p and q for p, q in zip(lm, rm)]


def aggregate(kind, a: Operand):
    """sum (add_wrapping in the native) / min / max; None iff no valid row."""
    vals = [v for i, v in enumerate(a.values) if a.valid(i)]
    if not vals:
        return None
    if kind == "sum":
        return wrap(a.width, sum(vals))
    return min(vals) if kind == "min" else max(vals)
