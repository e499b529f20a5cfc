"""The streaming primitive kernels over more than one grid-stride round, against the oracle at the usual bar (value bytes
including those under nulls, validity bits, null_count, NullBuffer presence, error status / text / index): k_arith (acu_arith
and acu_neg), k_cmp (acu_cmp and the fused compare -> filter plan), k_cast (acu_cast_numeric), and the out-of-bounds
detection of k_take and k_check_bounds.

k_arith, k_cmp, k_cast and k_take are launched with acu_wave_grid (common.cuh): 8 waves x SMs x p CTAs of 8 warps, where p
is the kernel's resident CTAs per SM, and a warp takes one unit per step (a 2048-row super-group, or a 256-index take tile).
p is cached inside the library, but a 256-thread CTA allows at most 8 resident CTAs per SM, so ROUND_MAX = 8 x SMs x 8 x 8
warps x unit bounds one round whatever p is. Every size here is at least 1.2 x ROUND_MAX and not a multiple of 64.
k_check_bounds runs acu_grid(.., 8) CTAs of 256 threads: a stride of exactly SMs x 8 x 256 indices.

Each kernel keeps its first failing row (and its valid count) in registers across rounds and merges it with atomicMin at
the end. Three placements of failing rows pin "the lowest failing valid row wins" without knowing p:
* two rows: for each p in 1..8, with W_p = 8 x SMs x p x 8 warps, rows unit x W_p - 1 (the last row of the highest warp's
  first round at that p) and unit x W_p (the first row of warp 0's second round). The lower one must be reported for every
  p; at the real p, a lowest-warp-wins rule or a row counted from the warp instead of the unit fails.
* one per unit: a failing row in every whole unit, at a position that varies with the unit's index mod 32. A round is a
  multiple of 32 units, so the thread that meets unit 0's row meets another one in every later round: a per-round reset or
  a last-failure-wins rule reports a later row.
* tail: a lower failing value under a null slot, which does not count, and failures in the ragged tail.
The operands are uploaded once; a placement patches its rows on the host and the device and puts them back afterwards.

Host memory and time: an operand of this length is 166 MB per byte of width on a 132-SM H100, so 8-byte operands appear in
two tests only, and values and validity masks come from the bit generator's raw output (`raw`) rather than from float draws
or bounded integer draws (sparse_mask's int16 draw costs about 1 s per 166M rows, and this file draws some 40 such arrays)."""
import ctypes as C

import numpy as np
import pytest

import acu
from acu import _abi as abi
from acu import BOOL, HostArray, bitmap_bytes
from test_gpu_device_slices import gpu_take
from test_gpu_elementwise_shapes import PAD, Column, call_out, gpu_filter_cmp, same, scalar

pytestmark = pytest.mark.gpu

CMP_OPS = [abi.EQ, abi.NEQ, abi.LT, abi.LT_EQ, abi.GT, abi.GT_EQ, abi.DISTINCT, abi.NOT_DISTINCT]
SG = 2048                     # rows per super-group of k_arith / k_cmp / k_cast: one per warp step
TILE = 256                    # indices per k_take warp tile
WAVES, WARPS_PER_CTA = 8, 8   # acu_wave_grid: 8 waves of 256-thread CTAs
MAX_CTAS_PER_SM = 8           # 2048 resident threads per SM on an H100
NULL_ROW = 1000               # the failing value under a null slot lies below every other placement
OVERFLOW = abi.ERR_ARITHMETIC_OVERFLOW
F32_SPECIALS = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1e-45, 1.0, -1.0], dtype=np.float32)


# ---- launch shapes ---------------------------------------------------------------------------------------------------------
def sms(gpu):
    return gpu.lib.acu_device_sm_count(gpu.h)


def wave_warps(gpu, p):
    """Warps of an acu_wave_grid launch whose kernel has p resident CTAs per SM (every launch here has more work than that)."""
    return WAVES * sms(gpu) * p * WARPS_PER_CTA


def check_bounds_stride(gpu):
    return sms(gpu) * 8 * 256


def sized(gpu, unit, tail=37):
    """At least 1.2 x ROUND_MAX rows of `unit`-row warp steps, the last 64-row word partial."""
    round_max = wave_warps(gpu, MAX_CTAS_PER_SM) * unit
    n = (int(1.2 * round_max) // 64 + 1) * 64 + tail
    assert_rounds(n, round_max)
    return n


def assert_rounds(n, per_round):
    assert n >= 1.2 * per_round, f"{n} rows are {n / per_round:.2f} rounds of {per_round}"
    assert n % 64 != 0


# ---- placements ------------------------------------------------------------------------------------------------------------
def one_per_unit(n, unit):
    """A row in each whole unit u at (u % 32) x (unit / 32) + ((u % 32) x 7 + 5) % (unit / 32)."""
    step = unit // 32
    k = np.arange(n // unit, dtype=np.int64) % 32
    return np.arange(n // unit, dtype=np.int64) * unit + k * step + (k * 7 + 5) % step


def placements(gpu, n, unit, nullable, stride=None):
    """(name, failing rows at valid slots, failing rows at null slots, expected first-error row). `stride` replaces the
    occupancy-dependent rounds of acu_wave_grid by the fixed stride of an acu_grid loop."""
    if stride is None:
        for p in range(1, MAX_CTAS_PER_SM + 1):
            hi = unit * wave_warps(gpu, p)
            assert hi < n
            yield f"two rows p={p}", [hi - 1, hi], [], hi - 1
        rows = one_per_unit(n, unit)
    else:
        yield "two rows", [stride - 1, stride], [], stride - 1
        rows = np.arange(7, n, stride, dtype=np.int64)
    yield "one per unit", rows, [], int(rows[0])
    tail = [n // unit * unit + 3, n - 1]
    assert tail[0] < tail[1]
    yield "tail", tail, [NULL_ROW] if nullable else [], tail[0]


class Patch:
    """`value` (and a validity bit) at some rows of an uploaded Column, on the host and the device; undo() restores them."""

    def __init__(self, gpu, col, shift, rows, value, valid):
        self.gpu, self.col = gpu, col
        h = col.host
        self.idx = np.asarray(rows, dtype=np.int64) + shift
        self.old = h.values[self.idx].copy()
        self.bytes = None
        if h.validity is not None:
            bits = self.idx + h.validity_offset
            self.bytes = np.unique(bits >> 3)
            self.old_bytes = h.validity[self.bytes].copy()
            mask = np.left_shift(1, bits & 7).astype(np.uint8)
            if valid:
                np.bitwise_or.at(h.validity, bits >> 3, mask)
            else:
                np.bitwise_and.at(h.validity, bits >> 3, ~mask)
        h.values[self.idx] = value
        self.upload()

    def upload(self):
        g, h, dev = self.gpu, self.col.host, self.col.dev
        if len(self.idx) > 64:
            g.h2d(dev.d_values, h.values)
            if self.bytes is not None:
                g.h2d(dev.d_validity, h.validity)
            return
        w = h.width()
        for i in self.idx:
            g.h2d(dev.d_values + int(i) * w, h.values[i: i + 1])
        for b in [] if self.bytes is None else self.bytes:
            g.h2d(dev.d_validity + int(b), h.validity[b: b + 1])

    def undo(self):
        h = self.col.host
        h.values[self.idx] = self.old
        if self.bytes is not None:
            h.validity[self.bytes] = self.old_bytes
        self.upload()


def patches(gpu, targets, rows, valid):
    """One Patch per (column, shift, value) of `targets`."""
    return [Patch(gpu, col, shift, rows, value, valid) for col, shift, value in targets] if len(rows) else []


def first_error(gpu_fn, oracle_fn, row, status, what, window_start=0):
    """The oracle fails at `row` with `status`, and the device with the same status, text and row. oracle_fn may run on a
    window of the operands that starts at row `window_start`."""
    with pytest.raises(acu.ArrowError) as oe:
        oracle_fn()
    exp = (oe.value.status, str(oe.value), window_start + oe.value.index)
    del oe  # the traceback holds the oracle's full-size output buffer
    assert (exp[0], exp[2]) == (status, row), f"{what}: the oracle reports {exp}, expected status {status} at row {row}"
    with pytest.raises(acu.ArrowError) as ge:
        gpu_fn()
    got = (ge.value.status, str(ge.value), ge.value.index)
    del ge
    assert got == exp, f"{what}: {got} != {exp}"


def check_placements(gpu, n, unit, targets, fns, status, what, nullable, stride=None, also=None):
    """Every placement on the operands `targets` ((column, shift, failing value) triples): both sides report the expected
    row. fns = (device call, oracle call, oracle call on the one row given or None). Where it is given, the two-row
    placements take the error text from the oracle on the lower row alone (which row fails first is fixed by construction
    there); the others run the oracle over the whole column. also(what), if given, runs while the one-per-unit and tail
    placements are in place."""
    gpu_fn, oracle_fn, oracle_at = fns
    for name, rows, null_rows, row in placements(gpu, n, unit, nullable, stride):
        applied = patches(gpu, targets, rows, True)
        applied += patches(gpu, targets, null_rows, False)
        try:
            if name.startswith("two rows") and oracle_at is not None:
                first_error(gpu_fn, lambda: oracle_at(row), row, status, f"{what}, {name}", window_start=row)
            else:
                first_error(gpu_fn, oracle_fn, row, status, f"{what}, {name}")
                if also is not None:
                    also(f"{what}, {name}")
        finally:
            for pt in reversed(applied):
                pt.undo()


def operand(col, shift, with_validity=True):
    """Rows [shift, shift + n) of an uploaded Column as (host, device descriptor), optionally without the validity bitmap."""
    h, d = col.at(shift)
    if shift:
        assert d.values % 16 != 0, f"a shift of {shift} elements left the values 16-byte aligned"
    if not with_validity:
        h = HostArray(h.dtype, h.values, h.length, None, 0, 0, 0)
        d.validity, d.validity_offset, d.null_count = None, 0, 0
    return h, d


def scalar_operand(sc):
    return sc[0], sc[1].descriptor()


def row_of(h, row):
    """Row `row` of a host operand as a one-row array; a scalar stays as it is."""
    return h if h.is_scalar else h.slice(row, 1)


def raw(rng, n, width=1):
    """n random unsigned integers of `width` bytes."""
    return rng.bit_generator.random_raw(-(-n * width // 8)).view(np.dtype(f"u{width}"))[:n]


def mask(rng, n, null_p):
    """A validity mask with about null_p of the slots null."""
    return raw(rng, n) >= int(null_p * 256)


def f32_values(rng, m, scale=0.37):
    v = raw(rng, m, 2).view(np.int16).astype(np.float32) * np.float32(scale)
    v[rng.integers(0, m, m // 16)] = F32_SPECIALS[rng.integers(0, len(F32_SPECIALS), m // 16, dtype=np.int8)]
    return v


# ---- 1. arithmetic -----------------------------------------------------------------------------------------------------------
def arith_fns(gpu, oracle, dtype, op, x, y, n):
    (xh, xd), (yh, yd) = x, y
    w = abi.DTYPE_SIZE[dtype]
    return (lambda: call_out(gpu, n * w, n, dtype, lambda out: gpu.lib.acu_arith(gpu.h, dtype, op, C.byref(xd), C.byref(yd), C.byref(out))),
            lambda: oracle.arith(op, xh, yh),
            lambda row: oracle.arith(op, row_of(xh, row), row_of(yh, row)))


FORMS = {"aa": "array/array", "as": "array/scalar", "sa": "scalar/array"}


def run_arith_cases(gpu, oracle, dtype, a, b, cases, nan_ok=False):
    """cases: (op, form, validity, (shift of a, shift of b), scalar, failing (a, b) values or None). `validity` names the
    array operands whose descriptor keeps its bitmap; the scalar stands for a in scalar/array and for b in array/scalar."""
    n = a.n
    for op, form, validity, (sa, sb), sv, fail in cases:
        sc = scalar(gpu, dtype, sv) if form != "aa" else None
        try:
            x = scalar_operand(sc) if form == "sa" else operand(a, sa, "a" in validity)
            y = scalar_operand(sc) if form == "as" else operand(b, sb, "b" in validity)
            what = f"arith dtype={dtype} op={op} {FORMS[form]} validity={validity or 'none'} shifts={sa}/{sb} n={n}"
            fns = arith_fns(gpu, oracle, dtype, op, x, y, n)
            same(fns[0](), fns[1](), what, nan_ok)
            if fail is None:
                continue
            fa, fb = fail
            divisor = sv if form == "as" else fb
            status = abi.ERR_DIVIDE_BY_ZERO if op in (abi.DIV, abi.REM) and divisor == 0 else OVERFLOW
            targets = ([(a, sa, fa)] if form != "sa" else []) + ([(b, sb, fb)] if form != "as" else [])
            check_placements(gpu, n, SG, targets, fns, status, what, nullable=validity != "")
        finally:
            if sc is not None:
                sc[1].free()


# Int8 operands: a in [-8, 7], b in [-8, 8] without 0 except under some of b's null slots, so that no product, sum or
# quotient of two valid slots fails; the scalars below keep the other side inside Int8 as well.
INT8_CASES = [
    (abi.ADD_WRAPPING, "aa", "ab", (0, 0), None, None),
    (abi.ADD, "aa", "ab", (0, 0), None, (100, 100)),
    (abi.ADD, "as", "a", (1, 0), 100, None),
    (abi.SUB, "sa", "", (0, 0), -100, (None, 100)),
    (abi.SUB, "aa", "b", (3, 1), None, None),
    (abi.MUL, "as", "a", (2, 0), 11, (100, None)),
    (abi.MUL, "aa", "", (0, 0), None, None),
    (abi.DIV, "aa", "ab", (1, 2), None, (-128, -1)),
    (abi.DIV, "as", "a", (0, 0), -1, None),
    (abi.REM, "sa", "b", (0, 3), 77, (None, 0)),
]


def test_arith_int8_multi_round(gpu, oracle):
    """Every Int8 class: wrapping, checked add / sub / mul and div / rem (EPL 16 aligned, EPL 1 shifted), with placements for
    add, sub, mul (checked), div (i8::MIN / -1) and rem (a zero divisor)."""
    n = sized(gpu, SG)
    rng = np.random.default_rng(31_000)
    m = PAD + n
    b_vals = (raw(rng, m) & 15).view(np.int8) - 8
    b_vals[b_vals == 0] = 8
    b_mask = mask(rng, m, 0.2)
    b_vals[~b_mask & (raw(rng, m) < 128)] = 0
    a = Column(gpu, abi.I8, (raw(rng, m) & 15).view(np.int8) - 8, mask(rng, m, 0.1))
    b = Column(gpu, abi.I8, b_vals, b_mask)
    del b_vals, b_mask
    try:
        run_arith_cases(gpu, oracle, abi.I8, a, b, INT8_CASES)
    finally:
        a.free()
        b.free()


U16_CASES = [  # values in [0, 255]: every valid product fits UInt16
    (abi.MUL, "aa", "ab", (0, 0), None, (256, 256)),
    (abi.MUL, "as", "a", (1, 0), 255, (300, None)),
    (abi.MUL, "sa", "", (0, 0), 255, None),
]

F32_CASES = [
    (abi.ADD, "aa", "a", (0, 0), None, None),
    (abi.ADD, "as", "", (1, 0), 0.5, None),
    (abi.DIV, "aa", "ab", (2, 1), None, None),
]


def test_arith_uint16_checked_mul_multi_round(gpu, oracle):
    n = sized(gpu, SG)
    rng = np.random.default_rng(31_100)
    m = PAD + n
    a = Column(gpu, abi.U16, raw(rng, m).astype(np.uint16), mask(rng, m, 0.1))
    b = Column(gpu, abi.U16, raw(rng, m).astype(np.uint16), mask(rng, m, 0.2))
    try:
        run_arith_cases(gpu, oracle, abi.U16, a, b, U16_CASES)
    finally:
        a.free()
        b.free()


def test_arith_float32_multi_round(gpu, oracle):
    n = sized(gpu, SG)
    rng = np.random.default_rng(31_200)
    m = PAD + n
    a = Column(gpu, abi.F32, f32_values(rng, m), mask(rng, m, 0.1))
    b = Column(gpu, abi.F32, f32_values(rng, m), mask(rng, m, 0.2))
    try:
        run_arith_cases(gpu, oracle, abi.F32, a, b, F32_CASES, nan_ok=True)
    finally:
        a.free()
        b.free()


def test_arith_int64_checked_multi_round(gpu, oracle):
    """Int64 checked mul, array/scalar (EPLV = 2). The placements run first; the host operand is dropped before the full
    comparison, so that it, the oracle's output and the device's output are not all held at once."""
    n = sized(gpu, SG)
    rng = np.random.default_rng(31_300)
    m = PAD + n
    a = Column(gpu, abi.I64, raw(rng, m, 2).view(np.int16).astype(np.int64), mask(rng, m, 0.1))
    sc = scalar(gpu, abi.I64, 3)
    try:
        what = f"arith Int64 mul array/scalar n={n}"
        fns = arith_fns(gpu, oracle, abi.I64, abi.MUL, operand(a, 0), scalar_operand(sc), n)
        check_placements(gpu, n, SG, [(a, 0, 1 << 62)], fns, OVERFLOW, what, nullable=True)
        gpu_fn, exp = fns[0], fns[1]()
        del fns
        a.host = None
        same(gpu_fn(), exp, what)
    finally:
        a.free()
        sc[1].free()


def neg_fns(gpu, oracle, dtype, x, n):
    xh, xd = x
    w = abi.DTYPE_SIZE[dtype]
    return (lambda: call_out(gpu, n * w, n, dtype, lambda out: gpu.lib.acu_neg(gpu.h, dtype, 1, C.byref(xd), C.byref(out))),
            lambda: oracle.neg(xh, True),
            lambda row: oracle.neg(row_of(xh, row), True))


def test_neg_multi_round(gpu, oracle):
    """neg_checked on Int8 (i8::MIN fails), aligned with validity and shifted without; Float32 neg."""
    n = sized(gpu, SG)
    rng = np.random.default_rng(31_400)
    m = PAD + n
    values = raw(rng, m).view(np.int8)
    values[values == -128] = 0
    a = Column(gpu, abi.I8, values, mask(rng, m, 0.1))
    f = Column(gpu, abi.F32, f32_values(rng, m), mask(rng, m, 0.1))
    try:
        for shift, with_validity in ((0, True), (1, False)):
            what = f"neg Int8 shift={shift} validity={with_validity} n={n}"
            fns = neg_fns(gpu, oracle, abi.I8, operand(a, shift, with_validity), n)
            same(fns[0](), fns[1](), what)
            check_placements(gpu, n, SG, [(a, shift, -128)], fns, OVERFLOW, what, nullable=with_validity)
        gpu_fn, oracle_fn, _ = neg_fns(gpu, oracle, abi.F32, operand(f, 0), n)
        same(gpu_fn(), oracle_fn(), f"neg Float32 n={n}", nan_ok=True)
    finally:
        a.free()
        f.free()


# ---- 2. comparison and the fused compare -> filter plan ----------------------------------------------------------------------
CMP_FORMS = ["array/array", "array/scalar", "scalar/array", "array/null scalar"]
CMP_DTYPES = [abi.I8, abi.I32, abi.F32]
CMP_SCALAR = {abi.I8: 1, abi.I32: -2, abi.F32: -0.0}


def cmp_values(rng, dtype, m):
    """Few distinct values, so that every comparison has both outcomes and ties; Float32 with its specials (both zeros, both
    NaN signs, infinities, a denormal)."""
    if dtype == abi.F32:
        return f32_values(rng, m, scale=0.5)
    v = (raw(rng, m) & 7).view(np.int8) - 4
    return v if dtype == abi.I8 else v.astype(np.int32) * 65537


@pytest.mark.parametrize("dtype", CMP_DTYPES)
def test_cmp_multi_round(gpu, oracle, dtype):
    """All 8 ops, each in one form aligned or shifted, rotating over dtypes so that every op meets both loads and every form
    (null scalar: DISTINCT / NOT_DISTINCT fold it, the others return all-null). Int32's right operand has no bitmap. Two ops
    per dtype also go through acu_filter_plan_create_cmp and filter an Int8 column."""
    j = CMP_DTYPES.index(dtype)
    n = sized(gpu, SG)
    rng = np.random.default_rng(32_000 + dtype)
    m = PAD + n
    a = Column(gpu, dtype, cmp_values(rng, dtype, m), mask(rng, m, 0.1))
    b = Column(gpu, dtype, cmp_values(rng, dtype, m), mask(rng, m, 0.2))
    v = Column(gpu, abi.I8, raw(rng, m).view(np.int8), mask(rng, m, 0.05))
    sc, nsc = scalar(gpu, dtype, CMP_SCALAR[dtype]), scalar(gpu, dtype, None)
    try:
        vh, vd = v.at(0)
        for k, op in enumerate(CMP_OPS):
            form = (k + j) % 4
            aligned = (k // 4 + j) % 2 == 0
            sa, sb = (0, 0) if aligned else (1 + k % 3, 1 + (k + 1) % 3)
            x = scalar_operand(sc) if form == 2 else operand(a, sa)
            y = scalar_operand(sc) if form == 1 else scalar_operand(nsc) if form == 3 else operand(b, sb, j != 1)
            (xh, xd), (yh, yd) = x, y
            what = f"cmp dtype={dtype} op={op} {CMP_FORMS[form]} shifts={sa}/{sb} n={n}"
            got = call_out(gpu, bitmap_bytes(n), n, BOOL, lambda out: gpu.lib.acu_cmp(gpu.h, dtype, op, C.byref(xd), C.byref(yd), C.byref(out)))
            same(got, oracle.cmp(op, xh, yh), what)
            del got
            if (k + 2 * j) % 4 == 0:
                (g, gplan), (e, eplan) = gpu_filter_cmp(gpu, dtype, op, xd, yd, vd, abi.I8), oracle.filter_cmp(vh, op, xh, yh)
                same(g, e, "filter " + what)
                assert gplan == eplan, f"filter {what}: (count, strategy) {gplan} != {eplan}"
    finally:
        for c in (a, b, v):
            c.free()
        sc[1].free()
        nsc[1].free()


# ---- 3. cast -----------------------------------------------------------------------------------------------------------------
def cast_fns(gpu, oracle, frm, to, safe, x, n):
    xh, xd = x
    return (lambda: call_out(gpu, n * abi.DTYPE_SIZE[to], n, to,
                             lambda out: gpu.lib.acu_cast_numeric(gpu.h, frm, to, int(safe), C.byref(xd), C.byref(out))),
            lambda: oracle.cast(xh, to, safe),
            lambda row: oracle.cast(row_of(xh, row), to, safe))


def test_cast_int8_to_int64_multi_round(gpu, oracle):
    """The infallible widening cast (EPL 16): safe=True gives every row's validity its own NullBuffer and null_count."""
    n = sized(gpu, SG)
    rng = np.random.default_rng(33_000)
    m = PAD + n
    a = Column(gpu, abi.I8, raw(rng, m).view(np.int8), mask(rng, m, 0.1))
    try:
        gpu_fn, oracle_fn, _ = cast_fns(gpu, oracle, abi.I8, abi.I64, True, operand(a, 0), n)
        same(gpu_fn(), oracle_fn(), f"cast Int8->Int64 safe=True n={n}")
    finally:
        a.free()


def cast_values(rng, frm, m):
    """Values that all fit the target type of CASTS."""
    if frm == abi.I16:
        return raw(rng, m).astype(np.int16)
    if frm == abi.I32:
        return raw(rng, m).view(np.int8).astype(np.int32)
    if frm == abi.F32:  # -32767.25 .. 32767.75: truncated toward zero, all fit Int16
        return raw(rng, m, 2).view(np.int16).astype(np.float32) + np.float32(0.75)
    return raw(rng, m, 2).astype(np.int64) * 65537


# (from, to, shift, input has validity, values that do not fit `to`): EPL 8 and 4 aligned, EPL 1 shifted, and an 8-byte
# input (always EPL 1) without validity, where safe=True builds the NullBuffer alone
CASTS = [
    (abi.I16, abi.U8, 0, True, [-1, 256, 32767]),
    (abi.I32, abi.I8, 3, True, [128, -129, 1 << 30]),
    (abi.F32, abi.I16, 0, True, [32768.0, np.nan, -32769.0, np.inf]),
    (abi.I64, abi.U32, 0, False, [-1, 1 << 32, -(1 << 40)]),
]


@pytest.mark.parametrize("frm,to,shift,with_validity,bad", CASTS, ids=["i16-u8", "i32-i8-shifted", "f32-i16", "i64-u32"])
def test_cast_fallible_multi_round(gpu, oracle, frm, to, shift, with_validity, bad):
    """safe=False reports the lowest failing valid row at every placement; with the one-per-unit and tail placements in
    place, safe=True turns the failing rows into nulls in every round."""
    n = sized(gpu, SG)
    rng = np.random.default_rng(33_100 + 10 * frm + to)
    m = PAD + n
    a = Column(gpu, frm, cast_values(rng, frm, m), mask(rng, m, 0.1) if with_validity else None)
    try:
        x = operand(a, shift)
        what = f"cast {frm}->{to} shift={shift} n={n}"
        fns = cast_fns(gpu, oracle, frm, to, False, x, n)
        same(fns[0](), fns[1](), what)
        safe_gpu, safe_oracle, _ = cast_fns(gpu, oracle, frm, to, True, x, n)
        input_nulls = n - int(x[0].valid_mask().sum())

        def safe_same(tag):
            exp = safe_oracle()
            assert exp.validity is not None and exp.null_count > input_nulls, f"{tag}: no failing row became null"
            same(safe_gpu(), exp, tag + " safe")

        # one failing value per placement family: every value of `bad` reaches the error text
        for k, value in enumerate(bad):
            if k == 0:
                check_placements(gpu, n, SG, [(a, shift, value)], fns, abi.ERR_CAST, what, with_validity, also=safe_same)
            else:
                p = k % MAX_CTAS_PER_SM + 1
                hi = SG * wave_warps(gpu, p)
                applied = patches(gpu, [(a, shift, value)], [hi - 1, hi], True)
                try:
                    first_error(fns[0], lambda: fns[2](hi - 1), hi - 1, abi.ERR_CAST, f"{what}, value {value} at p={p}",
                                window_start=hi - 1)
                finally:
                    for pt in reversed(applied):
                        pt.undo()
    finally:
        a.free()


# ---- 4. take out of bounds ---------------------------------------------------------------------------------------------------
def take_fns(gpu, oracle, v, idx, idx_dtype, check_bounds):
    """No one-row oracle call for indices with nulls: whether any index is null decides which bounds check runs."""
    (vh, vd), (ih, idd) = v, idx
    return (lambda: gpu_take(gpu, vh.dtype, vd, idd, idx_dtype, check_bounds), lambda: oracle.take(vh, ih, check_bounds),
            None if ih.validity is not None else lambda row: oracle.take(vh, row_of(ih, row), check_bounds))


def take_setup(gpu, rng, idx_dtype, nv, m):
    vals = Column(gpu, abi.I32, rng.integers(-1000, 1000, PAD + nv, dtype=np.int32), mask(rng, PAD + nv, 0.1))
    idx = Column(gpu, idx_dtype, rng.integers(0, nv, PAD + m, dtype=acu.NP_DTYPES[idx_dtype]), mask(rng, PAD + m, 0.05))
    return vals, idx


def test_take_out_of_bounds_multi_round(gpu, oracle):
    """UInt32 indices staged by cp.async.bulk: k_take's panic (256-index tiles) and check_bounds' error (k_check_bounds,
    fixed stride), with and without index nulls; out-of-bounds indices under null index slots do not count."""
    m = sized(gpu, TILE)
    stride = check_bounds_stride(gpu)
    assert_rounds(m, stride)
    rng = np.random.default_rng(34_000)
    nv = 1000
    vals, idx = take_setup(gpu, rng, abi.U32, nv, m)
    try:
        v = vals.at(0)
        for with_nulls in (False, True):
            for check_bounds, status, s in ((False, abi.ERR_PANIC_OUT_OF_BOUNDS, None), (True, abi.ERR_COMPUTE, stride)):
                what = f"take UInt32 nulls={with_nulls} check_bounds={check_bounds} m={m}"
                fns = take_fns(gpu, oracle, v, operand(idx, 0, with_nulls), abi.U32, check_bounds)
                check_placements(gpu, m, TILE, [(idx, 0, nv + 5)], fns, status, what, with_nulls, stride=s)
    finally:
        vals.free()
        idx.free()


def test_take_negative_index_multi_round(gpu, oracle):
    """Int32 indices one element into their allocation (per-lane staging) with -1 placed: take panics on the index as u32;
    check_bounds reports it when the indices have no nulls, and lets it through to the take's panic when they do (the
    nullable check only tests index >= len)."""
    m = sized(gpu, TILE)
    stride = check_bounds_stride(gpu)
    rng = np.random.default_rng(34_100)
    nv = 1000
    vals, idx = take_setup(gpu, rng, abi.I32, nv, m)
    try:
        v = vals.at(0)
        for check_bounds, status, s in ((False, abi.ERR_PANIC_OUT_OF_BOUNDS, None), (True, abi.ERR_COMPUTE, stride)):
            what = f"take Int32 check_bounds={check_bounds} m={m}"
            fns = take_fns(gpu, oracle, v, operand(idx, 1, False), abi.I32, check_bounds)
            check_placements(gpu, m, TILE, [(idx, 1, -1)], fns, status, what, False, stride=s)
        # with index nulls, -1 passes check_bounds and take panics at the lowest valid one
        row = stride + 5
        gpu_fn, oracle_fn, _ = take_fns(gpu, oracle, v, operand(idx, 1), abi.I32, True)
        applied = patches(gpu, [(idx, 1, -1)], [row, m - 1], True) + patches(gpu, [(idx, 1, -1)], [NULL_ROW], False)
        try:
            first_error(gpu_fn, oracle_fn, row, abi.ERR_PANIC_OUT_OF_BOUNDS, f"take Int32 with nulls check_bounds=True m={m}")
        finally:
            for pt in reversed(applied):
                pt.undo()
    finally:
        vals.free()
        idx.free()
