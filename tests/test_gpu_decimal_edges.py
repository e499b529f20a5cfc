"""Decimal arithmetic, negation, comparison, casts and sum / min / max on the device at their boundaries, and with
full-width values over more than one grid-stride round, against tests/oracle_decimal.py and tests/oracle_decimal_cast.py
at the usual bar: every value slot (under nulls too), validity bits, null_count, NullBuffer presence, and the status,
message and row of any error.

1. Boundary families (tests/decimal_edges_util.py; tests/test_oracle_decimal_edges.py checks the oracles against their
   closed forms on the same rows). A family's ok rows go into one array, with some failing inputs under null slots where
   the operation skips nulls; each failing row gets its own call after a prefix of ok rows, with safe = False, and all of
   them go into one array with safe = True, where they become nulls (the unary casts fail whatever `safe` is).
2. Multi-round. k_arith<., CLS_DECIMAL>, k_cmp<__int128>, k_dcast (each kind) and k_reduce<__int128> run
   acu_wave_grid launches whose round depends on the kernel's occupancy; every size here is sized() of
   test_gpu_elementwise_rounds (at least 1.2 x ROUND_MAX rows of 2048-row units, not a multiple of 64), and the failing rows
   take its placements (two rows for every occupancy p in 1..8, one per unit, the tail with a lower failing value under a
   null slot). A column is periodic: one period of P = 64 x 67 rows is uploaded and doubled on the device, so a Decimal128
   operand of ~166M rows never exists on the host; the expectation is the oracle on one period, compared chunk by chunk.
   Because 67 is odd, successive periods start at every 64-row word of a 2048-row unit."""
import ctypes as C

import numpy as np
import pytest

import acu
import decimal_edges_util as du
import oracle_decimal as od
import oracle_decimal_cast as oc
from acu import _abi as abi
from acu import ArrowError, DecimalArray, HostArray, bitmap_bytes, pack_bits
from test_gpu_elementwise_rounds import NULL_ROW, SG, placements, sized, wave_warps

pytestmark = pytest.mark.gpu

STATUS = {"InvalidArgument": abi.ERR_INVALID_ARGUMENT, "ArithmeticOverflow": abi.ERR_ARITHMETIC_OVERFLOW,
          "DivideByZero": abi.ERR_DIVIDE_BY_ZERO, "Compute": abi.ERR_COMPUTE, "Cast": abi.ERR_CAST,
          "Panic": abi.ERR_PANIC_OUT_OF_BOUNDS}
NATIVE = {4: abi.I32, 8: abi.I64, 16: abi.I128}
NP_BITS = {abi.F32: np.uint32, abi.F64: np.uint64}
FAMILIES = du.all_families()


# ---- host arrays, oracle operands, one call against the oracle ---------------------------------------------------------------
def with_nulls(h, null_rows):
    """h with the slots `null_rows` null (their values kept)."""
    if null_rows:
        mask = np.ones(h.length, dtype=bool)
        mask[list(null_rows)] = False
        h.validity, h.validity_offset, h.null_count = pack_bits(mask), 0, len(set(null_rows))
    return h


def dec(w, p, s, vals, null_rows=()):
    return with_nulls(DecimalArray.from_ints(w, p, s, vals), null_rows)


def prim(dtype, vals, null_rows=()):
    return with_nulls(HostArray.from_list(dtype, vals), null_rows)


def operand(d):
    validity = None if d.validity is None else [bool(x) for x in d.valid_mask()]
    return od.Operand(d.byte_width, d.precision, d.scale, d.raw_ints(), validity)


def prim_operand(h):
    vals = h.value_array()
    vals = [float(x) for x in vals] if h.dtype in (abi.F32, abi.F64) else [int(x) for x in vals]
    return oc.Prim(h.dtype, vals, None if h.validity is None else [bool(x) for x in h.valid_mask()])


def same(got, exp, what):
    dtype = got.dtype
    if dtype in (abi.F32, abi.F64):
        g = np.asarray(got.value_array()).view(NP_BITS[dtype])
        e = np.array(exp.values, dtype=np.float32 if dtype == abi.F32 else np.float64).view(NP_BITS[dtype])
        assert np.array_equal(g, e), what
    elif isinstance(got, DecimalArray):
        assert got.raw_ints() == exp.values, what
    else:
        assert [int(x) for x in got.value_array()] == exp.values, what
    assert (got.validity is not None) == (exp.validity is not None), what
    if exp.validity is not None:
        assert [bool(x) for x in got.valid_mask()] == exp.validity, what
    assert got.null_count == exp.null_count, what


def run_both(gpu_fn, oracle_fn, what):
    """The device call equals the oracle: the same result, or the same status, message and row."""
    try:
        exp = oracle_fn()
    except (od.DecimalError, oc.CastError) as e:
        with pytest.raises(ArrowError) as g:
            gpu_fn()
        assert (g.value.status, g.value.message, g.value.index) == (STATUS[e.status], e.message, e.index), what
        return None
    got = gpu_fn()
    same(got, exp, what)
    return exp


def family_calls(gpu, fam, rows, null_rows, safe):
    """(device call, oracle call) of family `fam` on input rows `rows` with `null_rows` null."""
    k, a = fam.kind, fam.args
    if k == "arith":
        op, w, p1, s1, p2, s2 = a
        x, y = dec(w, p1, s1, [r[0] for r in rows], null_rows), dec(w, p2, s2, [r[1] for r in rows])
        return (lambda: gpu.decimal_arith(op, x, y),
                lambda: od.decimal_op(op, operand(x), operand(y)))
    if k == "neg":
        x = dec(*a, rows, null_rows)
        return lambda: gpu.decimal_neg(x), lambda: od.neg(operand(x))
    if k == "dec":
        wi, p_in, s_in, wo, p_out, s_out = a
        x = dec(wi, p_in, s_in, rows, null_rows)
        return (lambda: gpu.cast_decimal(x, wo, p_out, s_out, safe),
                lambda: oc.cast_decimal(operand(x), wo, p_out, s_out, safe))
    if k == "to_dec":
        dt, w, p, s = a
        x = prim(dt, rows, null_rows)
        return lambda: gpu.cast_to_decimal(x, w, p, s, safe), lambda: oc.cast_to_decimal(prim_operand(x), w, p, s, safe)
    w, p, s, to = a
    x = dec(w, p, s, rows, null_rows)
    return lambda: gpu.cast_from_decimal(x, to, safe), lambda: oc.cast_from_decimal(operand(x), to, safe)


def check_family(gpu, fam, safe):
    """Returns the number of boundary rows checked."""
    what = f"{fam.name} safe={safe}"
    # ok rows, then two null slots: over failing inputs where nulls are skipped, over ok inputs where the cast runs at
    # every slot
    under = (fam.fail if fam.fail and not fam.unary else fam.ok)[:2]
    rows = fam.ok + under
    nulls = range(len(fam.ok), len(rows))
    if fam.ok:
        exp = run_both(*family_calls(gpu, fam, rows, nulls, safe), what)
        assert exp is not None, f"{what}: the ok rows fail"
    if safe and not fam.unary and fam.kind != "arith" and fam.fail:
        rows = fam.prefix() + fam.fail  # every failing row becomes a null
        exp = run_both(*family_calls(gpu, fam, rows, (), safe), what + " failing rows")
        assert exp is not None and exp.null_count == len(fam.fail), what
    else:
        for x in fam.fail:
            rows = fam.prefix() + [x]
            e = run_both(*family_calls(gpu, fam, rows, (), safe), f"{what} row {x!r}")
            assert e is None, f"{what}: {x!r} does not fail"
    return len(fam.ok) + len(fam.fail)


@pytest.mark.parametrize("group", list(FAMILIES))
def test_boundary_families(gpu, group):
    checked = 0
    for fam in FAMILIES[group]:
        for safe in (False, True) if fam.kind in ("dec", "to_dec", "from_dec") else (False,):
            checked += check_family(gpu, fam, safe)
    print(f"{group}: {len(FAMILIES[group])} families, {checked} boundary rows")


@pytest.mark.parametrize("values", du.aggregate_sets(), ids=lambda v: f"n{len(v)}")
def test_boundary_aggregates(gpu, values):
    a = DecimalArray.from_ints(16, 38, 0, values, force_validity=True)
    assert (gpu.sum(a), gpu.min(a), gpu.max(a)) == du.aggregate_closed(values)


# ---- periodic device columns ------------------------------------------------------------------------------------------------
P = 64 * 67                   # rows per period
SUPER = 67 * 32 * SG          # lcm(P, 32 units): the one-per-unit placement repeats with this period
CHUNK = P * 256               # rows per comparison chunk


def raw_of(h):
    """The P-row numpy value array of a host array (Decimal128: (P, 2) uint64 halves)."""
    return np.ascontiguousarray(np.asarray(h.values)[: h.length])


def raw_value(width_or_dtype, v):
    if width_or_dtype == abi.I128:
        return acu.i128_to_halves([v])
    return np.array([v], dtype=acu.NP_DTYPES[width_or_dtype])


class Periodic:
    """A device column of n rows whose row i holds row i % L of a pattern of L rows (L a multiple of 64), starting `shift`
    elements into its allocation. fill() uploads a pattern and doubles it on the device; patch() changes single rows;
    restore() brings back the base pattern."""

    def __init__(self, gpu, dtype, vals, valid, n, shift=0):
        self.gpu, self.dtype, self.n, self.shift = gpu, dtype, n, shift
        self.w = 16 if dtype == abi.I128 else abi.DTYPE_SIZE[dtype]
        self.base = (vals, valid)
        self.rows = -(-(shift + n) // 64) * 64
        self.d_values = gpu.malloc(self.rows * self.w + 16)
        self.d_valid = gpu.malloc(self.rows // 8 + 8) if valid is not None else None
        self.fill(vals, valid)

    def _double(self, dptr, unit, total):
        done = unit
        while done < total:
            c = min(done, total - done)
            self.gpu.check(self.gpu.lib.acu_memcpy_d2d(self.gpu.h, dptr + done, dptr, c))
            done += c

    def fill(self, vals, valid):
        L = len(vals)
        assert L % 64 == 0 and L <= self.rows
        self.gpu.h2d(self.d_values, np.roll(vals, self.shift, axis=0))  # allocation row j = pattern[(j - shift) % L]
        self._double(self.d_values, L * self.w, self.rows * self.w)
        self.mod = {}
        if valid is not None:
            self.packed = np.packbits(np.roll(valid, self.shift), bitorder="little")
            self.gpu.h2d(self.d_valid, self.packed)
            self._double(self.d_valid, L // 8, self.rows // 8)

    def restore(self):
        self.fill(*self.base)

    def patch(self, rows, value, valid=True):
        """`value` (a raw one-row array) at the logical rows `rows`, valid or null."""
        for r in rows:
            j = int(r) + self.shift
            self.gpu.h2d(self.d_values + j * self.w, value)
            if self.d_valid is None:
                assert valid
                continue
            b = j >> 3
            cur = self.mod.get(b, int(self.packed[b % len(self.packed)]))
            cur = cur | (1 << (j & 7)) if valid else cur & ~(1 << (j & 7))
            self.mod[b] = cur
            self.gpu.h2d(self.d_valid + b, np.array([cur], dtype=np.uint8))

    def fill_units(self, value):
        """The base pattern with `value` (valid) at the one-per-unit rows: a failing row in every whole 2048-row unit, at
        a position that varies with the unit's index mod 32. Returns the pattern's rows (period SUPER)."""
        vals, valid = self.base
        reps = SUPER // len(vals)
        v = np.tile(vals, (reps, 1) if vals.ndim == 2 else reps)
        m = None if valid is None else np.tile(valid, reps)
        unit = np.arange(SUPER // SG, dtype=np.int64)
        k = unit % 32
        rows = unit * SG + k * (SG // 32) + (k * 7 + 5) % (SG // 32)
        v[rows] = value
        if m is not None:
            m[rows] = True
        self.fill(v, m)
        return rows

    def descriptor(self):
        d = abi.Array()
        d.values = self.d_values + self.shift * self.w
        d.values_offset = 0
        d.validity = self.d_valid
        d.validity_offset = self.shift if self.d_valid else 0
        d.len = self.n
        d.null_count = -1 if self.d_valid else 0
        d.is_scalar = 0
        return d

    def free(self):
        self.gpu.free(self.d_values)
        self.gpu.free(self.d_valid)


def unit_rows(n, rows_in_super):
    """Every logical row below n that the one-per-unit pattern patches."""
    r = (np.arange(-(-n // SUPER), dtype=np.int64)[:, None] * SUPER + rows_in_super[None, :]).ravel()
    return r[r < n]


class Exp:
    """The expected output on one period: `vals` (raw numpy, P rows; a bool array for a Boolean output) and `valid` (bool
    array, or None without a NullBuffer)."""

    def __init__(self, vals, valid):
        self.vals, self.valid = vals, valid


def exp_from(res, dtype):
    """An oracle result of P rows as an Exp in the output native."""
    vals = raw_of(DecimalArray.from_ints(16, 38, 0, res.values)) if dtype == abi.I128 else \
        np.array(res.values, dtype=acu.NP_DTYPES[dtype])
    return Exp(vals, None if res.validity is None else np.array(res.validity, dtype=bool))


def run_out(gpu, n, nbytes, fn):
    """fn(out) into a fresh output; returns (status, out). The caller frees out."""
    out = gpu.alloc_out(nbytes, n)
    return fn(out), out


def tiled_bits(bits, n):
    """The packed bitmap of n rows whose row i is bits[i % P]."""
    reps = -(-n // P)
    return np.tile(np.packbits(bits, bitorder="little"), reps)[: (n + 7) // 8]


def check_out(gpu, out, n, out_dtype, exp, what, nulled=None):
    """The device output `out` of n rows against the period expectation `exp`, with the rows `nulled` (sorted) null and
    0 on top of it (failing rows of unary_opt, and slots made null)."""
    assert out.len == n, what
    assert bool(out.has_validity) == (exp.valid is not None or nulled is not None), f"{what}: NullBuffer presence"
    nb = (n + 7) // 8  # bitmap_bytes() pads to whole 64-bit words; the bytes past row n are not the result's
    last = np.uint8((1 << (n % 8)) - 1 if n % 8 else 0xFF)
    if out_dtype == acu.BOOL:
        got = gpu.d2h(out.values, nb)
        want = tiled_bits(exp.vals, n)
        got[-1] &= last
        want[-1] &= last
        assert np.array_equal(got, want), f"{what}: value bits differ"
    else:
        w = 16 if out_dtype == abi.I128 else abi.DTYPE_SIZE[out_dtype]
        npdt = np.uint64 if out_dtype == abi.I128 else NP_BITS.get(out_dtype, acu.NP_DTYPES[out_dtype])
        period = exp.vals.view(np.uint64) if out_dtype == abi.I128 else exp.vals.view(npdt)
        tile = np.tile(period, (CHUNK // P, 1) if period.ndim == 2 else CHUNK // P)
        for start in range(0, n, CHUNK):
            m = min(CHUNK, n - start)
            got = gpu.d2h(out.values + start * w, m * w, npdt)
            got = got.reshape(-1, 2) if out_dtype == abi.I128 else got
            want = tile[:m]
            if nulled is not None:
                sel = nulled[(nulled >= start) & (nulled < start + m)] - start
                if len(sel):
                    want = want.copy()
                    want[sel] = 0
            if not np.array_equal(got, want):
                bad = np.nonzero((got != want).reshape(m, -1).any(axis=1))[0]
                raise AssertionError(f"{what}: values differ at rows {(bad[:8] + start).tolist()}")
    if out.has_validity:
        got = gpu.d2h(out.validity, nb)
        want = tiled_bits(exp.valid if exp.valid is not None else np.ones(P, dtype=bool), n)
        if nulled is not None and len(nulled):
            np.bitwise_and.at(want, nulled >> 3, ~np.left_shift(1, nulled & 7).astype(np.uint8))
        got[-1] &= last
        want[-1] &= last
        assert np.array_equal(got, want), f"{what}: validity bits differ at bytes {np.nonzero(got != want)[0][:8].tolist()}"
        valid = int(np.unpackbits(want, bitorder="little")[:n].sum())
        assert out.null_count == n - valid, f"{what}: null_count {out.null_count} != {n - valid}"


def first_error(call, exp_err, row, what):
    """call() fails with exp_err = (status, message) at `row`."""
    st, out = call()
    try:
        assert st != abi.OK, f"{what}: no error, expected one at row {row}"
        d = gpu_last_error(call)
        assert (st, d[0], d[1]) == (exp_err[0], exp_err[1], row), what
    finally:
        call.gpu._free_out(out)


def gpu_last_error(call):
    d = call.gpu.lib.acu_last_error(call.gpu.h).contents
    return d.message.decode(), d.index


class Call:
    """A device call over periodic operands: fn(out) -> status, into an output of n rows of `out_bytes` bytes."""

    def __init__(self, gpu, n, out_bytes, fn):
        self.gpu, self.n, self.out_bytes, self.fn = gpu, n, out_bytes, fn

    def __call__(self):
        return run_out(self.gpu, self.n, self.out_bytes, self.fn)


def check_placements(gpu, n, targets, call, oracle_err, what, unary=False):
    """Every placement of test_gpu_elementwise_rounds with failing values on the periodic columns `targets` ((column,
    raw failing value) pairs): the call fails at the expected row with oracle_err() = (status, message) of the failing row
    alone. A unary call counts the failing value under the tail's null slot."""
    nullable = any(c.d_valid is not None for c, _ in targets)
    err = oracle_err()
    for name, rows, null_rows, row in placements(gpu, n, SG, nullable):
        try:
            if name == "one per unit":
                for c, v in targets:
                    in_super = c.fill_units(v)
                row = int(unit_rows(n, in_super)[0])
            else:
                for c, v in targets:
                    c.patch(rows, v, True)
                    if c.d_valid is not None:  # a column without a bitmap: the row is null through another operand
                        c.patch(null_rows, v, False)
            if unary and null_rows:
                row = min(row, min(null_rows))
            first_error(call, err, row, f"{what}, {name}")
        finally:
            for c, _ in targets:
                c.restore()


def ok_period(rng, draw, row_ok, tries=3):
    """P rows from draw(rng, P) -> list, each re-drawn (then halved) until row_ok(value) holds."""
    vals = draw(rng, P)
    for i in range(P):
        t = 0
        while not row_ok(vals[i]):
            vals[i] = draw(rng, 1)[0] if t < tries else (tuple(x >> 1 for x in vals[i]) if isinstance(vals[i], tuple) else vals[i] >> 1)
            t += 1
    return vals


def period_mask(rng, null_p):
    return rng.random(P) >= null_p


# ---- 2a. k_arith<., CLS_DECIMAL> and acu_neg(ACU_I128) ------------------------------------------------------------------------
ARITH_TYPES = {  # op: ((p1, s1), (p2, s2)) relative to the width's max precision; the rescale each one runs
    du.ADD: lambda mp: ((mp, 2), (mp, 0)),         # r * 100
    du.SUB: lambda mp: ((mp, 0), (mp, 3)),         # l * 1000
    du.MUL: lambda mp: ((mp, 1), (mp, 2)),
    du.DIV: lambda mp: ((mp, 0), (mp, 0)),         # l * 10^4
    du.REM: lambda mp: ((mp, 1), (mp, 0)),         # r * 10
}
ARITH_FAIL = {du.ADD: "max", du.SUB: "min", du.MUL: "max", du.DIV: "zero", du.REM: "zero"}


def arith_period(rng, w, op):
    (p1, s1), (p2, s2) = ARITH_TYPES[op](du.MAXP[w])

    def draw(rng, m):
        return list(zip(du.full_width(rng, w, m), du.full_width(rng, w, m)))
    vals = ok_period(rng, draw, lambda x: x[1] != 0 and du.arith_row(op, w, s1, s2, *x) is not du.FAIL)
    return (p1, s1), (p2, s2), [x[0] for x in vals], [x[1] for x in vals]


def failing_pair(w, op):
    lo, hi = du.native(w)
    return {"max": (hi, hi), "min": (lo, hi), "zero": (5, 0)}[ARITH_FAIL[op]]


@pytest.mark.parametrize("w", du.WIDTHS)
def test_decimal_arith_multi_round(gpu, w):
    """All five ops on full-width operands that succeed, aligned (the vectorised variant) and for Decimal32 / 64 one to
    three elements into the allocation (EPL = 1), with every placement of a failing pair; Decimal128 negation too."""
    n = sized(gpu, SG)
    rng = np.random.default_rng(41_000 + w)
    for k, op in enumerate((du.ADD, du.SUB, du.MUL, du.DIV, du.REM)):
        (p1, s1), (p2, s2), lv, rv = arith_period(rng, w, op)
        av, bv = period_mask(rng, 0.1), (period_mask(rng, 0.2) if k % 2 else None)
        # failing inputs under some of a's null slots, where try_binary does not evaluate
        fl, fr = failing_pair(w, op)
        for i in np.nonzero(~av)[0][::3]:
            lv[i], rv[i] = fl, fr
        ha, hb = DecimalArray.from_ints(w, p1, s1, lv), DecimalArray.from_ints(w, p2, s2, rv)
        exp_res = od.decimal_op(op, od.Operand(w, p1, s1, lv, av.tolist()), od.Operand(w, p2, s2, rv, None if bv is None else bv.tolist()))
        shifts = [(0, 0)] if w == 16 else [(0, 0), (1 + k % 3, 1 + (k + 1) % 3)]
        for sa, sb in shifts:
            what = f"Decimal{8 * w} op={op} shifts={sa}/{sb} n={n}"
            a = Periodic(gpu, NATIVE[w], raw_of(ha), av, n, sa)
            b = Periodic(gpu, NATIVE[w], raw_of(hb), bv, n, sb)
            try:
                lt, rt = abi.DecimalType(w, p1, s1), abi.DecimalType(w, p2, s2)
                ot = abi.DecimalType()
                ad, bd = a.descriptor(), b.descriptor()
                call = Call(gpu, n, n * w, lambda out: gpu.lib.acu_decimal_arith(gpu.h, op, C.byref(lt), C.byref(ad), C.byref(rt),
                                                                                  C.byref(bd), C.byref(ot), C.byref(out)))
                st, out = call()
                try:
                    assert st == abi.OK, (what, gpu_last_error(call))
                    assert (ot.precision, ot.scale) == (exp_res.precision, exp_res.scale), what
                    check_out(gpu, out, n, NATIVE[w], exp_from(exp_res, NATIVE[w]), what)
                finally:
                    gpu._free_out(out)
                if (sa, sb) == shifts[-1]:
                    def oracle_err():
                        with pytest.raises(od.DecimalError) as e:
                            od.decimal_op(op, od.Operand(w, p1, s1, [fl]), od.Operand(w, p2, s2, [fr]))
                        return STATUS[e.value.status], e.value.message
                    check_placements(gpu, n, [(a, raw_value(NATIVE[w], fl)), (b, raw_value(NATIVE[w], fr))], call, oracle_err, what)
            finally:
                a.free()
                b.free()
    if w == 16:
        lo, _ = du.native(16)
        vals = ok_period(rng, lambda r, m: du.full_width(r, 16, m), lambda x: x != lo)
        valid = period_mask(rng, 0.1)
        ha = DecimalArray.from_ints(16, 38, 0, vals)
        exp_res = od.neg(od.Operand(16, 38, 0, vals, valid.tolist()))
        a = Periodic(gpu, abi.I128, raw_of(ha), valid, n)
        try:
            ad = a.descriptor()
            call = Call(gpu, n, n * 16, lambda out: gpu.lib.acu_neg(gpu.h, abi.I128, 1, C.byref(ad), C.byref(out)))
            st, out = call()
            try:
                assert st == abi.OK
                check_out(gpu, out, n, abi.I128, exp_from(exp_res, abi.I128), "neg Decimal128")
            finally:
                gpu._free_out(out)
            check_placements(gpu, n, [(a, raw_value(abi.I128, lo))], call,
                             lambda: (abi.ERR_ARITHMETIC_OVERFLOW, f"Arithmetic overflow: Overflow happened on: - {lo}"), "neg Decimal128")
        finally:
            a.free()


# ---- 2b. k_cmp<__int128> -----------------------------------------------------------------------------------------------------
def test_cmp_i128_multi_round(gpu):
    """All 8 ops, array against array, on pairs with equal high limbs whose low limbs straddle 2^63, equal pairs,
    neighbours, and unrelated full-width values."""
    n = sized(gpu, SG)
    rng = np.random.default_rng(42_000)
    a_vals = du.full_width(rng, 16, P)
    b_vals = []
    for i, x in enumerate(a_vals):
        kind = i % 4
        if kind == 0:
            b_vals.append(x)
        elif kind == 1:
            hi = x >> 64
            b_vals.append((hi << 64) | (2 ** 63 - 1 if (x & (2 ** 64 - 1)) >= 2 ** 63 else 2 ** 63))
        elif kind == 2:
            b_vals.append(x + (1 if i % 8 == 2 else -1) if du.in_native(16, x + 1) and du.in_native(16, x - 1) else x)
        else:
            b_vals.append(du.full_width(rng, 16, 1)[0])
    av, bv = period_mask(rng, 0.1), period_mask(rng, 0.05)
    ha, hb = DecimalArray.from_ints(16, 38, 2, a_vals), DecimalArray.from_ints(16, 38, 2, b_vals)
    a = Periodic(gpu, abi.I128, raw_of(ha), av, n)
    b = Periodic(gpu, abi.I128, raw_of(hb), bv, n)
    try:
        ad, bd = a.descriptor(), b.descriptor()
        for op in range(8):
            vals, validity = od.cmp(op, od.Operand(16, 38, 2, a_vals, av.tolist()), od.Operand(16, 38, 2, b_vals, bv.tolist()))
            st, out = run_out(gpu, n, bitmap_bytes(n), lambda o: gpu.lib.acu_cmp(gpu.h, abi.I128, op, C.byref(ad), C.byref(bd), C.byref(o)))
            try:
                assert st == abi.OK
                check_out(gpu, out, n, acu.BOOL, Exp(np.array(vals), None if validity is None else np.array(validity)), f"cmp op={op}")
            finally:
                gpu._free_out(out)
    finally:
        a.free()
        b.free()


# ---- 2c. k_dcast, one instantiation per kind ------------------------------------------------------------------------------
def draw_i128_below(limit):
    """Random magnitudes below 2^(bit length of `limit` - 1) <= limit (every bit length up to that), both signs."""
    bits = limit.bit_length()

    def draw(rng, m):
        out = []
        for v in du.full_width(rng, 16, m):
            out.append((abs(v) >> (128 - bits + int(rng.integers(0, bits)))) * (1 if v >= 0 else -1))
        return out
    return draw


def half_ties(rng, k, limit, m):
    """q * 10^k + half and + half - 1: exact ties and near-ties of the rounding, both signs, below `limit`."""
    out = []
    for q in rng.integers(0, max(1, limit // 10 ** k), m):
        v = int(q) * 10 ** k + 10 ** k // 2 - int(rng.integers(0, 2))
        out.append(v if rng.random() < 0.5 else -v)
    return out


# kind: (source dtype, source decimal type or None, call builder, target, ok draw, ok test, failing value, unary spec)
def dcast_cases():
    lo128, hi128 = du.native(16)
    down_ok = 999_999_999 * 10 ** 20 + 10 ** 20 // 2 - 1     # rounds to 10^9 - 1 at 20 digits down
    return {
        # DK_DEC upscale, Int64 natives into Decimal128: 10^12 times (checked: 18 + 12 digits exceed 29)
        "dec up": dict(src=(abi.I64, (8, 18, 0)), to=("dec", 16, 29, 12), fail=2 ** 62,
                       draw=lambda rng, m: [int(x) for x in rng.integers(-(10 ** 17) + 1, 10 ** 17, m)]),
        # DK_DEC downscale, full-width Decimal128 dividends by 10^20 (three chunks) into Decimal32
        "dec down": dict(src=(abi.I128, (16, 38, 20)), to=("dec", 4, 9, 0), fail=10 ** 30,
                         draw=lambda rng, m: [v if abs(v) <= down_ok else v % down_ok for v in
                                              du.full_width(rng, 16, m // 2) + half_ties(rng, 20, down_ok, m - m // 2)],
                         unary=((16, 28, 20), 2 ** 120)),
        # DK_INT, Int64 into Decimal128 at scale 20: 2^62 * 10^20 overflows the multiply
        "int": dict(src=(abi.I64, None), to=("to_dec", 16, 38, 20), fail=2 ** 62,
                    draw=lambda rng, m: [int(x) for x in rng.integers(-(10 ** 18) + 1, 10 ** 18, m)]),
        # DK_FLOAT, Float64 into Decimal128(38, 10): ties m / 2^11 (x * 10^10 = odd / 2), and 1e29 past 38 digits
        "float": dict(src=(abi.F64, None), to=("to_dec", 16, 38, 10), fail=1e29,
                      draw=lambda rng, m: [float(x) for x in rng.standard_normal(m // 2) * 10.0 ** rng.integers(-3, 27, m // 2)]
                      + [(2 * int(q) + 1) / 2 ** 11 * (1 if q % 3 else -1) for q in rng.integers(0, 2 ** 28, m - m // 2)]),
        # DK_TO_INT, Decimal128 at scale 5 into Int64: a full-width division by 10^5, values up to 2^79
        "to int": dict(src=(abi.I128, (16, 38, 5)), to=("from_dec", abi.I64), fail=2 ** 100,
                       draw=draw_i128_below((2 ** 63 - 1) * 10 ** 5)),
        # DK_TO_FLOAT, full-width Decimal128 at scale 3 into Float64 (unary, no failure)
        "to float": dict(src=(abi.I128, (16, 38, 3)), to=("from_dec", abi.F64), fail=None,
                         draw=lambda rng, m: du.full_width(rng, 16, m)),
    }


def host_source(src, vals, scale_type=None):
    dtype, dt = src
    if dt is not None:
        w, p, s = scale_type or dt
        return DecimalArray.from_ints(w, p, s, vals)
    return HostArray.from_list(dtype, vals)


def dcast_fns(gpu, src_type, to, safe, desc):
    """(device fn(out), oracle fn(host array), output dtype, output width)."""
    dtype, dt = src_type
    if to[0] == "dec":
        _, wo, p, s = to
        ft, tt = abi.DecimalType(*dt), abi.DecimalType(wo, p, s)
        return (lambda out: gpu.lib.acu_cast_decimal(gpu.h, C.byref(ft), C.byref(tt), int(safe), C.byref(desc), C.byref(out)),
                lambda h: oc.cast_decimal(operand(h), wo, p, s, safe), NATIVE[wo], wo)
    if to[0] == "to_dec":
        _, wo, p, s = to
        tt = abi.DecimalType(wo, p, s)
        return (lambda out: gpu.lib.acu_cast_to_decimal(gpu.h, dtype, C.byref(tt), int(safe), C.byref(desc), C.byref(out)),
                lambda h: oc.cast_to_decimal(prim_operand(h), wo, p, s, safe), NATIVE[wo], wo)
    ft = abi.DecimalType(*dt)
    return (lambda out: gpu.lib.acu_cast_from_decimal(gpu.h, C.byref(ft), to[1], int(safe), C.byref(desc), C.byref(out)),
            lambda h: oc.cast_from_decimal(operand(h), to[1], safe), to[1], abi.DTYPE_SIZE[to[1]])


def cast_exp(res, out_dtype):
    if out_dtype in (abi.F32, abi.F64):
        return Exp(np.array(res.values, dtype=acu.NP_DTYPES[out_dtype]), None if res.validity is None else np.array(res.validity))
    return exp_from(res, out_dtype)


@pytest.mark.parametrize("kind", list(dcast_cases()))
def test_dcast_multi_round(gpu, kind):
    """One k_dcast instantiation per kind. try_unary (safe = False): every placement of the failing value reports the
    lowest valid failing row. unary_opt (safe = True): with the one-per-unit and tail placements in place, the failing
    rows become nulls in every round. unary (the downscale at a precision that makes it infallible, and decimal -> float):
    computes at null slots, and a failing value under the tail's null slot is the reported row."""
    c = dcast_cases()[kind]
    n = sized(gpu, SG)
    rng = np.random.default_rng(43_000 + len(kind))
    vals = c["draw"](rng, P)
    valid = period_mask(rng, 0.1)
    h = host_source(c["src"], vals)
    src_native = c["src"][0]
    col = Periodic(gpu, src_native, raw_of(h), valid, n)
    masked = with_nulls(host_source(c["src"], vals), np.nonzero(~valid)[0].tolist())
    try:
        desc = col.descriptor()
        for safe in (False, True):
            fn, oracle, out_dtype, ow = dcast_fns(gpu, c["src"], c["to"], safe, desc)
            what = f"{kind} safe={safe} n={n}"
            exp = cast_exp(oracle(masked), out_dtype)
            call = Call(gpu, n, n * ow, fn)
            st, out = call()
            try:
                assert st == abi.OK, (what, gpu_last_error(call))
                check_out(gpu, out, n, out_dtype, exp, what)
            finally:
                gpu._free_out(out)
            if c["fail"] is None:
                continue
            fv = raw_value(src_native, c["fail"])
            one = host_source(c["src"], [c["fail"]])

            def oracle_err():
                with pytest.raises(oc.CastError) as e:
                    dcast_fns(gpu, c["src"], c["to"], False, desc)[1](one)
                return STATUS[e.value.status], e.value.message
            if not safe:
                check_placements(gpu, n, [(col, fv)], call, oracle_err, what)
            else:
                def patched(tag, nulled):
                    st, out = call()
                    try:
                        assert st == abi.OK, (tag, gpu_last_error(call))
                        check_out(gpu, out, n, out_dtype, exp, tag, nulled=nulled)
                    finally:
                        gpu._free_out(out)
                run_patched(gpu, n, col, fv, patched)
        if "unary" in c:  # the same instantiation at an input precision that makes it infallible
            (w, p, s), bad = c["unary"]
            ft, tt = abi.DecimalType(w, p, s), abi.DecimalType(*c["to"][1:])
            call = Call(gpu, n, n * c["to"][1], lambda out: gpu.lib.acu_cast_decimal(gpu.h, C.byref(ft), C.byref(tt), 0, C.byref(desc),
                                                                                      C.byref(out)))
            what = f"{kind} unary n={n}"
            exp = cast_exp(oc.cast_decimal(od.Operand(w, p, s, vals, valid.tolist()), *c["to"][1:], False), NATIVE[c["to"][1]])
            st, out = call()
            try:
                assert st == abi.OK, (what, gpu_last_error(call))
                check_out(gpu, out, n, NATIVE[c["to"][1]], exp, what)
            finally:
                gpu._free_out(out)
            check_placements(gpu, n, [(col, raw_value(src_native, bad))], call,
                             lambda: (abi.ERR_PANIC_OUT_OF_BOUNDS, oc.UNWRAP_NONE), what, unary=True)
    finally:
        col.free()


def run_patched(gpu, n, col, fv, check):
    """check(tag, nulled rows) with the failing value at the one-per-unit rows, then at the tail (and under a null slot)."""
    try:
        rows = unit_rows(n, col.fill_units(fv))
        check("one per unit", rows)
    finally:
        col.restore()
    tail = [n // SG * SG + 3, n - 1]
    try:
        col.patch(tail, fv, True)
        col.patch([NULL_ROW], fv, False)
        check("tail", np.array(sorted([NULL_ROW] + tail), dtype=np.int64))
    finally:
        col.restore()


# ---- 2d. k_reduce<__int128> ------------------------------------------------------------------------------------------------
def test_reduce_i128_multi_round(gpu):
    """sum (wrapping past 2^127) / min / max of a periodic full-width column with equal high limbs and low limbs around
    2^63 in every period, and a unique minimum and maximum planted in the second round at every occupancy."""
    n = sized(gpu, SG)
    rng = np.random.default_rng(44_000)
    lo, hi = du.native(16)
    vals = du.full_width(rng, 16, P)
    for i in range(0, P, 5):  # pairs with one high limb, low limbs 2^63 - 1 and 2^63
        h = vals[i] >> 64
        vals[i] = (h << 64) | (2 ** 63 - 1 + (i // 5) % 2)
    vals = [max(lo + 1, min(hi - 1, v)) for v in vals]
    valid = period_mask(rng, 0.1)
    ha = DecimalArray.from_ints(16, 38, 0, vals)
    col = Periodic(gpu, abi.I128, raw_of(ha), valid, n)
    try:
        period = [v for v, m in zip(vals, valid) if m]
        tail = [v for v, m in zip(vals[: n % P], valid[: n % P]) if m]
        base_sum = (n // P) * sum(period) + sum(tail)
        assert gpu_aggregate(gpu, col) == (od.wrap(16, base_sum), min(period), max(period))
        for p in (1, 2, 8):  # the planted rows lie in the second round at occupancy p
            r_min, r_max = SG * wave_warps(gpu, p) + 7, SG * wave_warps(gpu, p) + 1000
            if r_max >= n:
                continue
            old = [vals[r % P] if valid[r % P] else 0 for r in (r_min, r_max)]
            try:
                col.patch([r_min], raw_value(abi.I128, lo), True)
                col.patch([r_max], raw_value(abi.I128, hi), True)
                s = od.wrap(16, base_sum - sum(old) + lo + hi)
                assert gpu_aggregate(gpu, col) == (s, lo, hi), f"p={p}"
            finally:
                col.restore()
    finally:
        col.free()


def gpu_aggregate(gpu, col):
    out = []
    d = col.descriptor()
    for op in (abi.SUM, abi.MIN, abi.MAX):
        bits, cnt = (C.c_uint64 * 2)(), C.c_int64(0)
        gpu.check(gpu.lib.acu_aggregate_i128(gpu.h, op, C.byref(d), bits, C.byref(cnt)))
        out.append(acu.halves_to_i128(np.array([[bits[0], bits[1]]], dtype=np.uint64))[0] if cnt.value else None)
    return tuple(out)
