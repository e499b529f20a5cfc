"""Device bitwise ops (acu_bitwise) and the product / product_checked / bit_and / bit_or / bit_xor aggregates against
tests/oracle_bitwise.py, bit for bit (float product: exact where every association order is exact, else by a relative
tolerance of n ulps computed here)."""
import ctypes as C

import numpy as np
import pytest

import acu
import oracle_bitwise as ob
from acu import _abi as abi
from acu import HostArray
from test_gpu_elementwise_shapes import PAD, Column, call_out, same

pytestmark = pytest.mark.gpu

INT_DTYPES = [abi.I8, abi.I16, abi.I32, abi.I64, abi.U8, abi.U16, abi.U32, abi.U64]
NAME = {d: abi.DTYPE_NAMES[d] for d in INT_DTYPES}
OPS = {"and": abi.BITWISE_AND, "or": abi.BITWISE_OR, "xor": abi.BITWISE_XOR, "and_not": abi.BITWISE_AND_NOT,
       "shift_left": abi.BITWISE_SHIFT_LEFT, "shift_right": abi.BITWISE_SHIFT_RIGHT, "not": abi.BITWISE_NOT}
AGG = {"product": abi.PRODUCT, "bit_and": abi.BIT_AND, "bit_or": abi.BIT_OR, "bit_xor": abi.BIT_XOR}
SG, WAVES, WARPS_PER_CTA, MAX_CTAS_PER_SM = 2048, 8, 8, 8


def round_max(gpu):
    """k_arith and k_reduce both run acu_wave_grid launches of 8-warp CTAs, one 2048-row super-group per warp step: one
    grid-stride round covers at most 8 waves x SMs x 8 CTAs x 8 warps x 2048 rows."""
    return WAVES * gpu.lib.acu_device_sm_count(gpu.h) * MAX_CTAS_PER_SM * WARPS_PER_CTA * SG


def rand(rng, dtype, n):
    info = np.iinfo(acu.NP_DTYPES[dtype])
    return rng.integers(info.min, info.max, n, dtype=acu.NP_DTYPES[dtype], endpoint=True)


def expect(op, dtype, a, b):
    """The oracle's HostArray for HostArrays a, b (b a scalar HostArray, or None for not)."""
    av, am = a.value_array(), (None if a.validity is None else list(a.valid_mask()))
    if b is None or b.is_scalar:
        s = None if b is None else b.value_array()[0]
        vals = ob.np_op(op, NAME[dtype], av, s)
        mask = am
    else:
        bm = None if b.validity is None else list(b.valid_mask())
        vals = ob.np_op(op, NAME[dtype], av, b.value_array())
        mask = None
        if a.length and ((am is not None and not all(am)) or (bm is not None and not all(bm))):
            mask = np.ones(a.length, dtype=bool)
            if am is not None:
                mask &= np.array(am, dtype=bool)
            if bm is not None:
                mask &= np.array(bm, dtype=bool)
    if mask is None:
        return HostArray.from_numpy(dtype, vals)
    return HostArray.from_numpy(dtype, vals, np.asarray(mask, dtype=bool))


def validity_cases(rng, n):
    """no NullBuffer, a NullBuffer without nulls, one with nulls"""
    return [None, np.ones(n, dtype=bool), rng.random(n) >= 0.3]


@pytest.mark.parametrize("dtype", INT_DTYPES)
def test_every_op_and_form(gpu, dtype):
    rng = np.random.default_rng(100 + dtype)
    w = abi.DTYPE_SIZE[dtype] * 8
    for n in (0, 1, 37, 2049, 70001):
        a_vals, b_vals = rand(rng, dtype, n), rand(rng, dtype, n)
        if n > 8:  # shift amounts over the whole range, the boundary values of both operands
            b_vals[:4] = np.array([w - 1, w, -1 if dtype < abi.U8 else np.iinfo(b_vals.dtype).max, 0], dtype=b_vals.dtype)
        for am in validity_cases(rng, n):
            for bm in validity_cases(rng, n):
                a = HostArray.from_numpy(dtype, a_vals, am)
                b = HostArray.from_numpy(dtype, b_vals, bm)
                for op, code in OPS.items():
                    if op == "not":
                        if bm is None:
                            same(gpu.bitwise(code, a), expect(op, dtype, a, None), f"{op} {NAME[dtype]} n={n}")
                        continue
                    same(gpu.bitwise(code, a, b), expect(op, dtype, a, b), f"{op} {NAME[dtype]} n={n}")
                    if op != "and_not" and bm is None:
                        for sv in (b_vals[:1] if n else [], [w + 3], [-1 if dtype < abi.U8 else 1]):
                            s = HostArray.from_numpy(dtype, np.array(sv if len(sv) else [5])[:1].astype(b_vals.dtype)).scalar()
                            same(gpu.bitwise(code, a, s), expect(op, dtype, a, s), f"{op}_scalar {NAME[dtype]} n={n}")


def test_in_place_and_unaligned_views(gpu):
    """out->values = a->values (binary_mut / unary_mut), and value pointers shifted 1-3 elements with validity at a bit
    offset (the descriptors of test_gpu_elementwise_shapes.py)."""
    rng = np.random.default_rng(5)
    for dtype in (abi.I8, abi.U16, abi.I32, abi.I64):
        n = 70001
        m = PAD + n
        a = Column(gpu, dtype, rand(rng, dtype, m), rng.random(m) >= 0.1)
        b = Column(gpu, dtype, rand(rng, dtype, m), rng.random(m) >= 0.2)
        try:
            for sa, sb, so in ((0, 0, 0), (1, 3, 2), (3, 2, 1)):
                (ah, ad), (bh, bd) = a.at(sa), b.at(sb)
                for op in ("xor", "shift_right", "and_not"):
                    got = call_out(gpu, n * abi.DTYPE_SIZE[dtype], n, dtype,
                                   lambda out: gpu.lib.acu_bitwise(gpu.h, dtype, OPS[op], C.byref(ad), C.byref(bd), C.byref(out)), so)
                    same(got, expect(op, dtype, ah, bh), f"{op} {NAME[dtype]} shifts {sa}/{sb}/{so}")
        finally:
            a.free()
            b.free()
        # in place: the result overwrites a's values
        av = rand(rng, dtype, 5000)
        h = HostArray.from_numpy(dtype, av, rng.random(5000) >= 0.5)
        da = gpu.upload(h)
        try:
            ad = da.descriptor()
            out = abi.ArrayOut()
            out.values = da.d_values
            out.validity = gpu.malloc(acu.bitmap_bytes(5000) + 8)
            gpu.check(gpu.lib.acu_bitwise(gpu.h, dtype, abi.BITWISE_NOT, C.byref(ad), None, C.byref(out)))
            got = gpu.d2h(da.d_values, 5000 * abi.DTYPE_SIZE[dtype], acu.NP_DTYPES[dtype])
            assert np.array_equal(got, ~av)
            gpu.free(out.validity)
        finally:
            da.free()


def test_past_one_round(gpu):
    """k_arith and k_reduce over at least 1.2 grid-stride rounds, with the one differing value in a later round."""
    rm = round_max(gpu)
    n = int(1.2 * rm) + 37
    late = rm + 12345
    rng = np.random.default_rng(11)
    a_vals = rng.integers(-128, 127, n, dtype=np.int8, endpoint=True)
    b_vals = rng.integers(-128, 127, n, dtype=np.int8, endpoint=True)
    a = HostArray.from_numpy(abi.I8, a_vals)
    b = HostArray.from_numpy(abi.I8, b_vals)
    same(gpu.bitwise(abi.BITWISE_XOR, a, b), HostArray.from_numpy(abi.I8, a_vals ^ b_vals), "xor past one round")
    s = HostArray.from_numpy(abi.I8, np.array([3], dtype=np.int8)).scalar()
    same(gpu.bitwise(abi.BITWISE_SHIFT_LEFT, a, s), HostArray.from_numpy(abi.I8, ob.np_op("shift_left", "int8", a_vals, np.int8(3))),
         "shift_left_scalar past one round")
    del a_vals, b_vals, a, b
    ones = np.ones(n, dtype=np.int8)
    ones[late] = -3
    assert gpu.product(HostArray.from_numpy(abi.I8, ones)) == -3
    zeros = np.zeros(n, dtype=np.int8)
    zeros[late] = 0x10
    assert gpu.bit_xor(HostArray.from_numpy(abi.I8, zeros)) == 0x10
    assert gpu.bit_or(HostArray.from_numpy(abi.I8, zeros)) == 0x10
    allset = np.full(n, -1, dtype=np.int8)
    allset[late] = ~np.int8(0x20)
    assert gpu.bit_and(HostArray.from_numpy(abi.I8, allset)) == int(~np.int8(0x20))


@pytest.mark.parametrize("dtype", INT_DTYPES)
def test_integer_aggregates(gpu, dtype):
    rng = np.random.default_rng(200 + dtype)
    for n in (0, 1, 5, 63, 4097, 100003):
        vals = rand(rng, dtype, n)
        for mask in (None, rng.random(n) >= 0.5, np.zeros(n, dtype=bool)):
            h = HostArray.from_numpy(dtype, vals, mask)
            ml = None if mask is None else list(mask)
            for fn, op in AGG.items():
                exp = ob.aggregate(fn, NAME[dtype], [int(x) for x in vals], ml)
                assert gpu.aggregate(op, h) == exp, (fn, NAME[dtype], n)
            small = (vals % 3 + 1).astype(vals.dtype)  # factors 1..3 fit often enough to reach the success path
            hs = HostArray.from_numpy(dtype, small, mask)
            for arr in (h, hs):
                vl = [int(x) for x in arr.value_array()]
                try:
                    exp = ob.product_checked(NAME[dtype], vl, ml)
                except ob.ProductOverflow as e:
                    with pytest.raises(acu.ArrowError) as gi:
                        gpu.product_checked(arr)
                    assert (gi.value.status, str(gi.value), gi.value.index) == (abi.ERR_ARITHMETIC_OVERFLOW, "Arithmetic overflow: " + e.message, e.row)
                    continue
                assert gpu.product_checked(arr) == exp, (NAME[dtype], n)


def checked_case(gpu, dtype, vals, mask=None):
    h = HostArray.from_numpy(dtype, np.asarray(vals, dtype=acu.NP_DTYPES[dtype]), mask)
    vl = [int(x) for x in h.value_array()]
    try:
        exp = ob.product_checked(NAME[dtype], vl, None if mask is None else list(mask))
    except ob.ProductOverflow as e:
        with pytest.raises(acu.ArrowError) as gi:
            gpu.product_checked(h)
        assert (gi.value.status, str(gi.value), gi.value.index) == (abi.ERR_ARITHMETIC_OVERFLOW, "Arithmetic overflow: " + e.message, e.row)
        return "error", e.row
    assert gpu.product_checked(h) == exp
    return "ok", exp


def test_product_checked_placements(gpu):
    chunk = 4096
    # first row, the ragged tail, and a chunk after several thousand others (the scan kernel loops over its chunks)
    for n, row in ((10, 0), (chunk * 3 + 17, chunk * 3 + 9), (chunk * 5000 + 123, chunk * 4321 + 77)):
        v = np.ones(n, dtype=np.int64)
        v[row] = 2**62
        v[row + 1 if row + 1 < n else 0] = 4 if row + 1 < n else 1
        if row == 0:
            v[1] = 4
        assert checked_case(gpu, abi.I64, v) == ("error", row + 1 if row else 1)
    # a zero before the would-be overflow (no error, 0), a zero after it (error)
    v = np.ones(50000, dtype=np.int32)
    v[[100, 30000, 40000]] = [0, 2**30, 4]
    assert checked_case(gpu, abi.I32, v) == ("ok", 0)
    v[100], v[45000] = 1, 0
    assert checked_case(gpu, abi.I32, v) == ("error", 40000)
    # i64::MIN reached exactly, then x1 (no error) and x-1 (error), also across a chunk boundary
    v = np.ones(3 * chunk, dtype=np.int64)
    v[[10, chunk + 5]] = [-(2**62), 2]
    assert checked_case(gpu, abi.I64, v) == ("ok", -(2**63))
    v[2 * chunk + 1] = -1
    assert checked_case(gpu, abi.I64, v) == ("error", 2 * chunk + 1)
    # a lower overflowing value under a null
    v = np.ones(10000, dtype=np.int16)
    v[[5, 6, 9000, 9001]] = [100, 400, 200, 200]
    mask = np.ones(10000, dtype=bool)
    mask[6] = False
    assert checked_case(gpu, abi.I16, v, mask) == ("error", 9001)
    # unsigned types, at and past the limit
    assert checked_case(gpu, abi.U8, [15, 17, 1]) == ("ok", 255)
    assert checked_case(gpu, abi.U8, [15, 17, 2]) == ("error", 2)
    assert checked_case(gpu, abi.U64, [2**32 - 1, 2**32 + 1, 1]) == ("ok", 2**64 - 1)
    assert checked_case(gpu, abi.U64, [2**32, 2**32]) == ("error", 1)
    assert checked_case(gpu, abi.I8, [-128, 1, 1, -1]) == ("error", 3)
    assert checked_case(gpu, abi.I8, [-64, 2, 1, 1]) == ("ok", -128)
    assert checked_case(gpu, abi.I8, [64, 2]) == ("error", 1)


def test_float_product(gpu):
    rng = np.random.default_rng(3)
    for dtype, npdt, eps, n in ((abi.F64, np.float64, 2.0**-52, 20001), (abi.F32, np.float32, 2.0**-23, 1001)):
        # exact in every association order: +-1 and 60 factors 2^+-1, so no partial product leaves the exponent range
        e = np.zeros(n, dtype=np.int64)
        e[rng.choice(n, 60, replace=False)] = rng.choice([-1, 1], 60)
        vals = np.ldexp(np.where(rng.random(n) < 0.5, -1.0, 1.0), e).astype(npdt)
        exp = float(np.prod(vals.astype(np.float64)))
        assert gpu.product(HostArray.from_numpy(dtype, vals)) == exp
        for special, res in (([2.0, -0.0, 4.0], -0.0), ([np.inf, -2.0], -np.inf), ([1.0, np.nan, 3.0], np.nan), ([np.inf, 0.0], np.nan)):
            got = gpu.product(HostArray.from_numpy(dtype, np.array(special, dtype=npdt)))
            if np.isnan(res):
                assert np.isnan(got)
            else:
                assert got == res and np.signbit(got) == np.signbit(res)
        # elsewhere: values in [0.5, 2] (log-uniform, so that the product stays far from the exponent range), relative
        # tolerance n ulps
        vals = np.exp2(rng.uniform(-1.0, 1.0, n)).astype(npdt)
        mask = rng.random(n) >= 0.25
        ref = float(np.prod(vals[mask].astype(np.float64)))
        k = int(mask.sum())
        for fn in (gpu.product, gpu.product_checked):
            got = fn(HostArray.from_numpy(dtype, vals, mask))
            assert abs(got - ref) <= k * eps * abs(ref), (fn, got, ref)
        assert gpu.product(HostArray.from_numpy(dtype, vals[:0])) is None
        assert gpu.product(HostArray.from_numpy(dtype, vals[:5], np.zeros(5, dtype=bool))) is None


def test_aggregate_columns_mixes_old_and_new_ops(gpu, oracle):
    rng = np.random.default_rng(8)
    cols, ops, exps = [], [], []
    for dtype in (abi.I32, abi.U8, abi.I64):
        vals = rand(rng, dtype, 9001)
        mask = rng.random(9001) >= 0.3
        for fn, op in (("sum", abi.SUM), ("product", abi.PRODUCT), ("bit_xor", abi.BIT_XOR), ("max", abi.MAX), ("bit_and", abi.BIT_AND)):
            cols.append(HostArray.from_numpy(dtype, vals, mask))
            ops.append(op)
            exps.append(oracle.aggregate(op, cols[-1]) if fn in ("sum", "max") else ob.aggregate(fn, NAME[dtype], [int(x) for x in vals], list(mask)))
    assert gpu.aggregate_columns(ops, cols) == exps


def test_section_chains_bitwise_and_aggregates(gpu):
    """bitwise -> aggregate(BIT_XOR) -> aggregate(PRODUCT) queued in one stream-ordered section equal the synchronous calls."""
    rng = np.random.default_rng(9)
    n = 200003
    a = HostArray.from_numpy(abi.I64, rand(rng, abi.I64, n), rng.random(n) >= 0.1)
    b = HostArray.from_numpy(abi.I64, rand(rng, abi.I64, n), rng.random(n) >= 0.1)
    sync = gpu.bitwise(abi.BITWISE_AND_NOT, a, b)
    exp_xor, exp_prod = gpu.bit_xor(sync), gpu.product(sync)
    da, db = gpu.upload(a), gpu.upload(b)
    out = gpu.alloc_out(n * 8, n)
    try:
        ad, bd = da.descriptor(), db.descriptor()
        bits = [C.c_uint64(0), C.c_uint64(0)]
        cnt = [C.c_int64(0), C.c_int64(0)]
        gpu.async_begin()
        gpu.check(gpu.lib.acu_bitwise(gpu.h, abi.I64, abi.BITWISE_AND_NOT, C.byref(ad), C.byref(bd), C.byref(out)))
        r = abi.Array()
        r.values, r.validity, r.validity_offset, r.len, r.null_count = out.values, out.validity, 0, n, -1
        gpu.check(gpu.lib.acu_aggregate(gpu.h, abi.I64, abi.BIT_XOR, C.byref(r), C.byref(bits[0]), C.byref(cnt[0])))
        gpu.check(gpu.lib.acu_aggregate(gpu.h, abi.I64, abi.PRODUCT, C.byref(r), C.byref(bits[1]), C.byref(cnt[1])))
        gpu.results_fetch()
        got = [int(np.array([bits[i].value], dtype=np.uint64).view(np.int64)[0]) for i in range(2)]
        assert cnt[0].value == cnt[1].value == n - sync.null_count
        assert got == [exp_xor, exp_prod]
        assert out.null_count == sync.null_count
    finally:
        gpu._free_out(out)
        da.free()
        db.free()


def test_refusals(gpu):
    a = HostArray.from_numpy(abi.I32, np.arange(10, dtype=np.int32))
    f = HostArray.from_numpy(abi.F64, np.arange(10, dtype=np.float64))
    s = HostArray.from_numpy(abi.I32, np.array([1], dtype=np.int32)).scalar()
    null_s = HostArray.from_list(abi.I32, [None]).scalar()

    def refused(fn, status=abi.ERR_INVALID_ARGUMENT):
        with pytest.raises(acu.ArrowError) as e:
            fn()
        assert e.value.status == status, str(e.value)

    refused(lambda: gpu.bitwise(abi.BITWISE_AND, s, a))                # scalar a
    refused(lambda: gpu.bitwise(abi.BITWISE_AND, a, null_s))           # null scalar
    refused(lambda: gpu.bitwise(abi.BITWISE_AND_NOT, a, s))            # no scalar and_not
    refused(lambda: gpu.bitwise(abi.BITWISE_XOR, f, f))                # float
    refused(lambda: gpu.bitwise(99, a, a))                             # unknown op
    refused(lambda: gpu.bitwise(abi.BITWISE_OR, a))                    # missing right operand
    with pytest.raises(acu.ArrowError) as e:
        gpu.bitwise(abi.BITWISE_OR, a, HostArray.from_numpy(abi.I32, np.arange(9, dtype=np.int32)))
    assert (e.value.status, str(e.value)) == (abi.ERR_COMPUTE, "Compute error: Cannot perform binary operation on arrays of different length")
    i128 = acu.DecimalArray.from_ints(16, 38, 0, [1, 2])
    da = gpu.upload(i128)
    try:
        ad = da.descriptor()
        out = gpu.alloc_out(32, 2)
        st = gpu.lib.acu_bitwise(gpu.h, abi.I128, abi.BITWISE_AND, C.byref(ad), C.byref(ad), C.byref(out))
        gpu._free_out(out)
        assert st == abi.ERR_INVALID_ARGUMENT
    finally:
        da.free()
    for op in (abi.BIT_AND, abi.BIT_OR, abi.BIT_XOR):
        refused(lambda: gpu.aggregate(op, f))
        refused(lambda: gpu.aggregate_columns([abi.SUM, op], [a, f]))
    refused(lambda: gpu.aggregate(17, a))
    # the entry points of other column kinds keep rejecting every op but their own
    for op in (abi.PRODUCT, abi.BIT_AND, abi.BIT_OR, abi.BIT_XOR):
        refused(lambda: gpu.aggregate_i128(op, i128))
        bits, cnt, val = C.c_uint64(0), C.c_int64(0), C.c_int32(0)
        row = C.c_int64(0)
        dbool = gpu.upload(HostArray.from_list(acu.BOOL, [True, False]))
        try:
            bd = dbool.descriptor()
            assert gpu.lib.acu_aggregate_boolean(gpu.h, op, C.byref(bd), C.byref(val), C.byref(cnt)) == abi.ERR_INVALID_ARGUMENT
            assert gpu.lib.acu_aggregate_fixed_size_binary(gpu.h, 1, op, C.byref(bd), C.byref(row), C.byref(cnt)) == abi.ERR_INVALID_ARGUMENT
            ba = abi.BytesArray()
            ba.nulls = bd
            assert gpu.lib.acu_aggregate_bytes(gpu.h, 4, op, C.byref(ba), C.byref(row), C.byref(cnt)) == abi.ERR_INVALID_ARGUMENT
            va = abi.ViewArray()
            va.nulls = bd
            assert gpu.lib.acu_aggregate_byte_view(gpu.h, op, C.byref(va), C.byref(row), C.byref(cnt)) == abi.ERR_INVALID_ARGUMENT
        finally:
            dbool.free()
        # both all-reduce entry points, before any collective
        dA = gpu.upload(a)
        try:
            ad = dA.descriptor()
            assert gpu.lib.acu_aggregate_allreduce(gpu.h, abi.I32, op, C.byref(ad), C.byref(bits), C.byref(cnt)) == abi.ERR_NOT_YET_IMPLEMENTED
        finally:
            dA.free()
        pb, pc = (C.c_uint64 * 1)(5), (C.c_int64 * 1)(1)
        assert gpu.lib.acu_comm_allreduce_aggregates(gpu.h, abi.I32, op, pb, pc, 1) == abi.ERR_NOT_YET_IMPLEMENTED
    # product_checked is synchronous: refused inside a section whatever the input, floats and empty arrays included
    gpu.async_begin()
    try:
        refused(lambda: gpu.product_checked(a))
        refused(lambda: gpu.product_checked(f))
        refused(lambda: gpu.product_checked(HostArray.from_numpy(abi.I32, np.zeros(0, dtype=np.int32))))
    finally:
        gpu.results_fetch()
