"""acu_cmp, the fused compare -> filter plan, acu_cast_numeric and acu_arith at every shape of their single launch against
the oracle, bit for bit: columns shorter than one 2048-row super-group, whole super-groups, ragged tails, and value
pointers that are not 16-byte aligned. An unaligned operand is an uploaded column whose descriptor starts 1-3 elements
in (the zero-copy slice `Array::slice` makes), with the validity offset moved to match."""
import ctypes as C

import numpy as np
import pytest

import acu
from acu import _abi as abi
from acu import BOOL, HostArray, bitmap_bytes
from test_gpu_parity import rand_values

pytestmark = pytest.mark.gpu

LENGTHS = [1, 63, 64, 2047, 2048, 2049, 4095, 4097, 70001, 1_000_037]
CMP_OPS = [abi.EQ, abi.NEQ, abi.LT, abi.LT_EQ, abi.GT, abi.GT_EQ, abi.DISTINCT, abi.NOT_DISTINCT]
PAD = 3  # extra elements uploaded with every operand, so that a view shifted by 1-3 elements stays inside the allocation


class Column:
    """A host column of PAD + n rows uploaded once; `at(shift)` views rows [shift, shift + n) on both sides."""

    def __init__(self, gpu, dtype, values, mask):
        self.n = len(values) - PAD
        self.host = HostArray.from_numpy(dtype, values, mask, bit_offset=5 if mask is not None else 0)
        self.dev = gpu.upload(self.host)

    def at(self, shift):
        d = self.dev.descriptor()
        d.values = self.dev.d_values + shift * self.host.width()
        d.len = self.n
        if d.validity:
            d.validity_offset += shift
            d.null_count = -1
        return self.host.slice(shift, self.n), d

    def free(self):
        self.dev.free()


def scalar(gpu, dtype, value):
    h = HostArray.from_list(dtype, [value]).scalar()
    dev = gpu.upload(h)
    return h, dev


def same(got, exp, what, nan_ok=False):
    assert got.length == exp.length, f"{what}: length {got.length} != {exp.length}"
    assert (got.validity is None) == (exp.validity is None), f"{what}: NullBuffer presence differs"
    n = exp.length
    if exp.validity is not None:
        assert got.null_count == exp.null_count, f"{what}: null_count {got.null_count} != {exp.null_count}"
        assert np.array_equal(got.valid_mask(), exp.valid_mask()), f"{what}: validity bits differ"
    if exp.dtype == BOOL:  # rows [0, n): the oracle's not_distinct leaves ones in the padding bits of its last word
        gv, ev = got.value_array(), exp.value_array()
    elif nan_ok:  # float arithmetic: any NaN matches any NaN, every other value bit for bit
        gv, ev = got.value_array(), exp.value_array()
        assert np.array_equal(np.isnan(gv), np.isnan(ev)), f"{what}: NaN positions differ"
        gv, ev = gv[~np.isnan(gv)].view(np.uint8), ev[~np.isnan(ev)].view(np.uint8)
    else:  # values under nulls included
        gv, ev = np.ascontiguousarray(got.values).view(np.uint8)[: n * exp.width()], np.ascontiguousarray(exp.values).view(np.uint8)[: n * exp.width()]
    if not np.array_equal(gv, ev):
        bad = np.nonzero(gv != ev)[0]
        raise AssertionError(f"{what}: value bytes differ at {bad[:8]}")


def call_out(gpu, nbytes, rows, dtype, fn, shift_out=0):
    """Run fn(out) into a fresh output whose values start `shift_out` elements into their allocation; download it."""
    width = 1 if dtype == BOOL else abi.DTYPE_SIZE[dtype]
    out = gpu.alloc_out(nbytes + shift_out * width, rows)
    base = out.values
    try:
        out.values = base + shift_out * width
        gpu.check(fn(out))
        n = out.len
        vals = gpu.d2h(out.values, bitmap_bytes(n)) if dtype == BOOL else gpu.d2h(out.values, n * width, acu.NP_DTYPES[dtype])
        validity = gpu.d2h(out.validity, bitmap_bytes(n)) if out.has_validity else None
        return HostArray(dtype, vals, n, validity, 0, 0, out.null_count if out.has_validity else 0)
    finally:
        gpu.free(base)
        gpu.free(out.validity)


def same_or_same_error(gpu_fn, oracle_fn, what, nan_ok=False):
    try:
        exp = oracle_fn()
    except acu.ArrowError as e:
        with pytest.raises(acu.ArrowError) as gi:
            gpu_fn()
        assert (gi.value.status, str(gi.value), gi.value.index) == (e.status, str(e), e.index), what
        return
    same(gpu_fn(), exp, what, nan_ok)


def shapes():
    """(n, shift of the left operand, shift of the right operand): both aligned, then both unaligned by different amounts."""
    for k, n in enumerate(LENGTHS):
        yield n, 0, 0
        yield n, 1 + k % 3, 1 + (k + 1) % 3


# ---- acu_cmp and acu_filter_plan_create_cmp ------------------------------------------------------------------------------
def gpu_filter_cmp(gpu, dtype, op, ad, bd, vd, vdtype=abi.I64):
    plan = C.c_void_p()
    gpu.check(gpu.lib.acu_filter_plan_create_cmp(gpu.h, dtype, op, C.byref(ad), C.byref(bd), C.byref(plan)))
    try:
        count = gpu.lib.acu_filter_plan_count(plan)
        w = abi.DTYPE_SIZE[vdtype]
        res = call_out(gpu, count * w, count, vdtype,
                       lambda out: gpu.lib.acu_filter_primitive(gpu.h, plan, w, C.byref(vd), C.byref(out)))
        return res, (count, gpu.lib.acu_filter_plan_strategy(plan))
    finally:
        gpu.lib.acu_filter_plan_destroy(gpu.h, plan)


@pytest.mark.parametrize("dtype", [abi.I8, abi.I32, abi.I64, abi.F32, abi.F64])
def test_cmp_shapes(gpu, oracle, dtype):
    rng = np.random.default_rng(9100 + dtype)
    sc_host, sc_dev = scalar(gpu, dtype, rand_values(rng, dtype, 1, small=True)[0].item())
    nsc_host, nsc_dev = scalar(gpu, dtype, None)
    try:
        for k, (n, sa, sb) in enumerate(shapes()):
            m = PAD + n
            a = Column(gpu, dtype, rand_values(rng, dtype, m, small=True), rng.random(m) >= 0.1)
            b = Column(gpu, dtype, rand_values(rng, dtype, m, small=True), rng.random(m) >= 0.2 if k % 4 < 2 else None)
            vals = Column(gpu, abi.I64, rng.integers(-1000, 1000, m), rng.random(m) >= 0.05)
            try:
                (ah, ad), (bh, bd), (vh, vd) = a.at(sa), b.at(sb), vals.at(0)
                scd, nscd = sc_dev.descriptor(), nsc_dev.descriptor()
                for op in CMP_OPS:
                    for what, (x, xd), (y, yd) in (("array/array", (ah, ad), (bh, bd)), ("array/scalar", (ah, ad), (sc_host, scd)),
                                                   ("scalar/array", (sc_host, scd), (ah, ad)), ("array/null scalar", (ah, ad), (nsc_host, nscd))):
                        tag = f"dtype={dtype} op={op} {what} n={n} shifts={sa}/{sb}"
                        got = call_out(gpu, bitmap_bytes(n), n, BOOL,
                                       lambda out: gpu.lib.acu_cmp(gpu.h, dtype, op, C.byref(xd), C.byref(yd), C.byref(out)))
                        same(got, oracle.cmp(op, x, y), tag)
                        (g, gplan), (e, eplan) = gpu_filter_cmp(gpu, dtype, op, xd, yd, vd), oracle.filter_cmp(vh, op, x, y)
                        same(g, e, "filter " + tag)
                        assert gplan == eplan, tag
            finally:
                for c in (a, b, vals):
                    c.free()
    finally:
        sc_dev.free()
        nsc_dev.free()


# ---- acu_cast_numeric ----------------------------------------------------------------------------------------------------
FAILING = {  # values that do not fit the target type
    (abi.F64, abi.I32): [1e12, np.nan, -3e9, np.inf],
    (abi.I64, abi.U8): [-1, 256, 1 << 40],
    (abi.U64, abi.I64): [1 << 63, (1 << 64) - 1],
}


def cast_values(rng, frm, to, m):
    if frm == abi.F64:
        return rng.integers(-1_000_000, 1_000_000, m) + rng.random(m)
    if to == abi.U8:
        return rng.integers(0, 256, m)
    return rand_values(rng, frm, m, small=True)


@pytest.mark.parametrize("frm,to", [(abi.I64, abi.F64), (abi.I8, abi.I64), (abi.F64, abi.I32), (abi.I64, abi.U8), (abi.U64, abi.I64)])
def test_cast_shapes(gpu, oracle, frm, to):
    rng = np.random.default_rng(9200 + frm * 10 + to)
    for k, (n, shift, _) in enumerate(shapes()):
        m = PAD + n
        vals = np.asarray(cast_values(rng, frm, to, m)).astype(acu.NP_DTYPES[frm])
        mask = rng.random(m) >= 0.1 if k % 4 < 2 else None
        bad = FAILING.get((frm, to), [])
        runs = [(vals, True), (vals, False)]
        if bad:
            # failures in the head (the lowest under a null, where it must not count) and in the tail
            failing = vals.copy()
            rows = sorted({shift + r for r in (n // 3, n // 2, n - 1)})
            for j, r in enumerate(rows):
                failing[r] = bad[j % len(bad)]
            if mask is not None and n >= 3:
                mask[rows[0]] = False
            runs = [(failing, True), (failing, False), (vals, False)]
        for v, safe in runs:
            col = Column(gpu, frm, v, mask)
            try:
                h, d = col.at(shift)
                for shift_out in (0, 1):  # the output starts on a 16-byte boundary, or one element past it
                    tag = f"cast {frm}->{to} safe={safe} failures={v is not vals} n={n} shift={shift}/{shift_out}"
                    same_or_same_error(
                        lambda: call_out(gpu, n * abi.DTYPE_SIZE[to], n, to,
                                         lambda out: gpu.lib.acu_cast_numeric(gpu.h, frm, to, int(safe), C.byref(d), C.byref(out)),
                                         shift_out=shift_out),
                        lambda: oracle.cast(h, to, safe), tag)
            finally:
                col.free()


# ---- acu_arith: the kernel that already had this shape --------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [abi.I32, abi.I64, abi.F64])
def test_arith_shapes(gpu, oracle, dtype):
    rng = np.random.default_rng(9300 + dtype)
    for k, (n, sa, sb) in enumerate(shapes()):
        m = PAD + n
        a = Column(gpu, dtype, rand_values(rng, dtype, m), rng.random(m) >= 0.1)
        b = Column(gpu, dtype, rand_values(rng, dtype, m), rng.random(m) >= 0.2 if k % 4 < 2 else None)
        try:
            (ah, ad), (bh, bd) = a.at(sa), b.at(sb)
            for op in (abi.ADD_WRAPPING, abi.ADD):
                tag = f"arith dtype={dtype} op={op} n={n} shifts={sa}/{sb}"
                same_or_same_error(
                    lambda: call_out(gpu, n * abi.DTYPE_SIZE[dtype], n, dtype,
                                     lambda out: gpu.lib.acu_arith(gpu.h, dtype, op, C.byref(ad), C.byref(bd), C.byref(out))),
                    lambda: oracle.arith(op, ah, bh), tag, nan_ok=dtype == abi.F64)
        finally:
            a.free()
            b.free()


# ---- one launch per call --------------------------------------------------------------------------------------------------
def test_one_launch_per_call(gpu):
    """An aligned comparison or cast of 2049 rows (one super-group and a one-row tail) issues as many launches as one of 64
    rows, which is a single kernel plus the result bookkeeping."""
    rng = np.random.default_rng(9400)
    cols = {n: Column(gpu, abi.I64, rng.integers(-5, 5, PAD + n), None) for n in (64, 2049)}
    try:
        def launches(fn):
            fn()  # warm: leaves the result block clean, as every call in steady state finds it
            before = gpu.launch_count()
            fn()
            return gpu.launch_count() - before

        def cmp(n):
            _, d = cols[n].at(0)
            return launches(lambda: call_out(gpu, bitmap_bytes(n), n, BOOL,
                                             lambda out: gpu.lib.acu_cmp(gpu.h, abi.I64, abi.LT, C.byref(d), C.byref(d), C.byref(out))))

        def cast(n):
            _, d = cols[n].at(0)
            return launches(lambda: call_out(gpu, 8 * n, n, abi.F64,
                                             lambda out: gpu.lib.acu_cast_numeric(gpu.h, abi.I64, abi.F64, 1, C.byref(d), C.byref(out))))

        assert cmp(2049) == cmp(64)
        assert cast(2049) == cast(64)
    finally:
        for c in cols.values():
            c.free()
