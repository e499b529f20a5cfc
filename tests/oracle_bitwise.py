"""CPU restatement of arrow-arith's bitwise kernels (bitwise.rs) and of product / product_checked / bit_and / bit_or /
bit_xor (aggregate.rs), in Python integers: exact by construction. The per-row functions work on Python ints; the array
functions apply them to every slot (the values under nulls included) and build the NullBuffer as `binary` / `unary` do.
product_checked is the reference's in-order fold, so it fails at the first valid row whose running product leaves the
native range, with the reference's message and that row."""
import numpy as np

DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64"]
OPS = ["and", "or", "xor", "and_not", "shift_left", "shift_right", "not"]


def bits_of(dtype):
    return np.dtype(dtype).itemsize * 8


def signed(dtype):
    return dtype.startswith("int")


def wrap(dtype, v):
    """v modulo 2^bits, as the dtype's value."""
    w = bits_of(dtype)
    v &= (1 << w) - 1
    return v - (1 << w) if signed(dtype) and v >> (w - 1) else v


def row(op, dtype, l, r):
    """One slot of bitwise_<op> (bitwise.rs:81-111, :176-207): shifts by r's two's-complement pattern modulo the width."""
    w = bits_of(dtype)
    if op == "and":
        return wrap(dtype, l & r)
    if op == "or":
        return wrap(dtype, l | r)
    if op == "xor":
        return wrap(dtype, l ^ r)
    if op == "and_not":
        return wrap(dtype, l & ~r)
    if op == "not":
        return wrap(dtype, ~l)
    amt = (r & ((1 << w) - 1)) % w  # wrapping_shl / wrapping_shr: the low log2(w) bits of r
    if op == "shift_left":
        return wrap(dtype, l << amt)
    return wrap(dtype, l >> amt)  # Python's >> is arithmetic on negative ints: signed shift_right; unsigned l >= 0


def array_op(op, dtype, left, lmask, right=None, rmask=None, scalar=None):
    """bitwise_<op>(left, right) / bitwise_<op>_scalar(left, scalar) / bitwise_not(left) -> (values, mask or None).
    left / right: lists of ints (every slot, nulls included); masks: lists of bools or None (no NullBuffer)."""
    if right is not None:  # binary: union of the NullBuffers (arity.rs:104-135); empty inputs give no NullBuffer
        vals = [row(op, dtype, l, r) for l, r in zip(left, right)]
        has_nulls = (lmask is not None and not all(lmask)) or (rmask is not None and not all(rmask))
        if not left or not has_nulls:
            return vals, None
        lm = lmask if lmask is not None else [True] * len(left)
        rm = rmask if rmask is not None else [True] * len(left)
        return vals, [x and y for x, y in zip(lm, rm)]
    r = scalar if scalar is not None else 0
    return [row(op, dtype, l, r) for l in left], (None if lmask is None else list(lmask))  # unary: nulls cloned


def valid_values(values, mask):
    return [v for v, ok in zip(values, mask if mask is not None else [True] * len(values)) if ok]


def aggregate(fn, dtype, values, mask=None):
    """product / bit_and / bit_or / bit_xor (aggregate.rs:82-106, :788-875): None iff no valid value. Integers only
    (float product is compared by tolerance)."""
    vs = valid_values(values, mask)
    if not vs:
        return None
    acc = {"product": 1, "bit_and": -1, "bit_or": 0, "bit_xor": 0}[fn]
    for v in vs:
        if fn == "product":
            acc = acc * v
        elif fn == "bit_and":
            acc &= v
        elif fn == "bit_or":
            acc |= v
        else:
            acc ^= v
        acc = wrap(dtype, acc)
    return acc


class ProductOverflow(Exception):
    def __init__(self, message, row):
        super().__init__(message)
        self.message, self.row = message, row


def product_checked(dtype, values, mask=None):
    """product_checked (aggregate.rs:963-1001): acc.mul_checked(v) in row order from 1; ProductOverflow with
    "Overflow happened on: {acc} * {value}" (arithmetic.rs:193-200) and the failing row."""
    if not valid_values(values, mask):
        return None
    w = bits_of(dtype)
    lo, hi = (-(1 << (w - 1)), (1 << (w - 1)) - 1) if signed(dtype) else (0, (1 << w) - 1)
    acc = 1
    for i, v in enumerate(values):
        if mask is not None and not mask[i]:
            continue
        p = acc * v
        if p < lo or p > hi:
            raise ProductOverflow(f"Overflow happened on: {acc} * {v}", i)
        acc = p
    return acc


def np_op(op, dtype, a, b=None):
    """array_op's values for numpy operands (b an array, a numpy scalar, or None for not): the same definitions,
    vectorised for columns too long for per-row Python ints. Pinned to `row` on the CPU."""
    w = bits_of(dtype)
    u = np.dtype(f"uint{w}")
    a = np.asarray(a, dtype=dtype)
    if op == "not":
        return ~a
    b = np.asarray(b, dtype=dtype)
    if op == "and":
        return a & b
    if op == "or":
        return a | b
    if op == "xor":
        return a ^ b
    if op == "and_not":
        return a & ~b
    amt = (b.view(u) & u.type(w - 1)) if b.ndim else u.type(int(b.view(u)) & (w - 1))
    if op == "shift_left":
        return (a.view(u) << amt).astype(u).view(dtype)
    return (a >> amt.astype(dtype)).astype(dtype)
