"""concat_elements on the device vs the oracle (tests/oracle_concat_elements.py), bit for bit: offsets, value bytes, views,
data-buffer bytes and buffer count, validity bits, NullBuffer presence, null_count, and error status / text / row.
The i32 / view / FixedSizeBinary overflow cases are built on the device (device buffers and offsets) and never
materialised on the host. Reference: arrow-string/src/concat_elements.rs."""
import ctypes as C

import numpy as np
import pytest

import acu
from acu import FixedSizeBinaryColumn, Utf8Column, ViewColumn
from acu import _abi as abi

from concat_util import column, golden_cases, run_case
from oracle_concat_elements import ConcatElementsOracle, first_overflow_row
from substring_util import bytes_col, nulls_of, sliced
from test_gpu_parity import expect_same_error

pytestmark = pytest.mark.gpu

ORACLE = ConcatElementsOracle()
CASES = golden_cases()
SIZES = [0, 1, 3, 5, 2047, 2048, 2049, 3 * 2048 + 3, 20001]
SECTION = "not available between acu_async_begin"


def assert_nulls(g, e, what):
    assert (g.validity is None) == (e.validity is None), f"{what}: NullBuffer presence"
    if e.validity is not None:
        assert np.array_equal(g.valid_mask(), e.valid_mask()), f"{what}: validity bits"
        assert g.null_count == e.null_count, f"{what}: null_count {g.null_count} != {e.null_count}"


def assert_result(got, exp, what):
    if isinstance(exp, Utf8Column):
        assert got.offsets.dtype == exp.offsets.dtype and np.array_equal(got.offsets, exp.offsets), f"{what}: offsets"
        assert bytes(got.data) == bytes(exp.data), f"{what}: bytes"
    elif isinstance(exp, FixedSizeBinaryColumn):
        assert got.values.shape == exp.values.shape and np.array_equal(got.values, exp.values), f"{what}: values"
    else:
        assert np.array_equal(got.views, exp.views), f"{what}: views"
        assert len(got.buffers) == len(exp.buffers), f"{what}: buffer count"
        for g, e in zip(got.buffers, exp.buffers):
            assert bytes(g) == bytes(e), f"{what}: data buffer"
    assert_nulls(got.nulls, exp.nulls, what)


def same(gpu, fn, what):
    got, exp = expect_same_error(gpu, ORACLE, fn)
    if exp is not None:
        assert_result(got, exp, what)
    return exp


def rand_bytes_items(rng, n, max_len, null_p, long_p=0.0, long_len=0):
    out = []
    for _ in range(n):
        if null_p and rng.random() < null_p:
            out.append(None)
            continue
        ln = int(rng.integers(long_len // 2, long_len + 1)) if long_p and rng.random() < long_p else int(rng.integers(0, max_len + 1))
        out.append(rng.integers(0, 256, ln, dtype=np.uint8).tobytes())
    return out


def with_nulls(col, mask, off=0, force=False):
    """col with a validity of `mask` starting at bit `off` (garbage stays under the null slots)."""
    col.nulls = nulls_of(np.concatenate([np.ones(off, bool), np.asarray(mask, bool)]), force=force).slice(off, len(mask)) if off else \
        nulls_of(mask, force=force)
    return col


# ---- the reference's cases ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_golden(gpu, case):
    same(gpu, lambda b: run_case(b, case), case["id"])


# ---- byte arrays --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [np.int32, np.int64])
@pytest.mark.parametrize("nulls", ["none", "left", "right", "both", "empty_buffers"])
def test_bytes_fuzz(gpu, dt, nulls):
    rng = np.random.default_rng(7 + (dt == np.int64) * 100 + len(nulls))
    for n in SIZES:
        # left and right sliced differently (offsets mid-buffer, validity bit offsets 3 and 5)
        la, ra = rand_bytes_items(rng, n + 7, 40, 0.0), rand_bytes_items(rng, n + 9, 20, 0.0)
        l = sliced(bytes_col(la, dt), 3, n) if n else bytes_col([], dt)
        r = sliced(bytes_col(ra, dt), 5, n) if n else bytes_col([], dt)
        if nulls in ("left", "both"):
            with_nulls(l, rng.random(n) > 0.3, off=3)
        if nulls in ("right", "both"):
            with_nulls(r, rng.random(n) > 0.1, off=5)
        if nulls == "empty_buffers":  # NullBuffers without a null: the union is None
            with_nulls(l, np.ones(n, bool), off=3, force=True)
            with_nulls(r, np.ones(n, bool), force=True)
        for utf8 in (True, False):
            same(gpu, lambda b: b.concat_elements(l, r, is_utf8=utf8), f"n={n} {nulls} utf8={utf8}")


def test_bytes_under_nulls_copied(gpu):
    l = bytes_col([b"ab", None, b"c", None], np.int32, garbage=b"XYZ")
    r = bytes_col([None, b"2", None, None], np.int32, garbage=b"Q")
    exp = same(gpu, lambda b: b.concat_elements(l, r), "under nulls")
    assert bytes(exp.data) == b"abQXYZ2cQXYZQ"


@pytest.mark.parametrize("dt", [np.int32, np.int64])
def test_bytes_long_rows(gpu, dt):
    """Rows of 0 .. 1e5 bytes: CTAs whose output passes the 48 KiB staging buffer take the direct path."""
    rng = np.random.default_rng(11)
    for n, long_p in [(64, 0.5), (5000, 0.01), (4099, 0.002)]:
        la = rand_bytes_items(rng, n, 30, 0.05, long_p, 100_000)
        ra = rand_bytes_items(rng, n, 7, 0.05, long_p / 2, 60_000)
        same(gpu, lambda b: b.concat_elements(bytes_col(la, dt), bytes_col(ra, dt), is_utf8=False), f"n={n}")


def test_bytes_empty_rows(gpu):
    for n in (1, 4, 2049):
        e = bytes_col([b""] * n, np.int32)
        same(gpu, lambda b: b.concat_elements(e, e), f"empty n={n}")
        same(gpu, lambda b: b.concat_elements_utf8_many([e, e, e]), f"empty many n={n}")


@pytest.mark.parametrize("k", [1, 2, 3, 17])
@pytest.mark.parametrize("dt", [np.int32, np.int64])
def test_many(gpu, k, dt):
    rng = np.random.default_rng(k * 31 + (dt == np.int64))
    for n in (0, 5, 2049, 3 * 2048 + 3):
        cols = []
        for j in range(k):
            c = sliced(bytes_col(rand_bytes_items(rng, n + j, 12, 0.0), dt), j, n) if n else bytes_col([], dt)
            if j % 3 == 1:
                with_nulls(c, rng.random(n) > 0.2, off=j % 8)
            cols.append(c)
        if k > 1:
            cols[-1] = cols[0]  # the same array more than once
        same(gpu, lambda b: b.concat_elements_utf8_many(cols), f"k={k} n={n}")


def test_many_errors(gpu):
    a, b3 = bytes_col([b"a", b"b"], np.int32), bytes_col([b"a"], np.int32)
    same(gpu, lambda b: b.concat_elements_utf8_many([]), "no operand")
    same(gpu, lambda b: b.concat_elements_utf8_many([a, a, b3]), "length mismatch")


# ---- views ----------------------------------------------------------------------------------------------------------
def view_items(rng, n, lens, null_p):
    return [None if null_p and rng.random() < null_p else rng.integers(97, 123, int(rng.choice(lens)), dtype=np.uint8).tobytes()
            for _ in range(n)]


@pytest.mark.parametrize("block", [64, 1 << 20])
def test_views_fuzz(gpu, block):
    """Totals around the inline bound, left values of 0-3 bytes with long totals, multi-buffer (block=64) and large inputs."""
    rng = np.random.default_rng(block)
    for n in SIZES:
        for lens_l, lens_r in [([0, 1, 2, 3], [9, 10, 11, 12, 13, 40]), ([5, 6, 7, 12, 13, 30], [0, 6, 7, 1]), ([0, 3], [0, 1, 2])]:
            l = ViewColumn.from_values(view_items(rng, n, lens_l, 0.1), block_size=block)
            r = ViewColumn.from_values(view_items(rng, n, lens_r, 0.0), block_size=block)
            for utf8 in (True, False):
                same(gpu, lambda b: b.concat_elements(l, r, is_utf8=utf8), f"n={n} {lens_l}|{lens_r}")


def test_views_boundary_rows(gpu):
    l = ViewColumn.from_values([b"", b"a", b"ab", b"abc", b"abcdef", b"abcdefgh", b"x" * 13, b"", None])
    r = ViewColumn.from_values([b"y" * 13, b"y" * 12, b"y" * 11, b"y" * 10, b"y" * 6, b"y" * 5, b"", b"", b"z" * 20])
    exp = same(gpu, lambda b: b.concat_elements(l, r), "boundary")
    assert [int.from_bytes(bytes(v[:4]), "little") for v in exp.views] == [13, 13, 13, 13, 12, 13, 13, 0, 0]


def test_views_null_rows_not_read(gpu):
    """Null rows holding valid long-view patterns into a real buffer contribute no bytes and are never dereferenced."""
    long = b"L" * 40
    l = ViewColumn.from_values([long, b"abc", long, long], block_size=1 << 10)
    r = ViewColumn.from_values([long, long, b"q", long], block_size=1 << 10)
    with_nulls(l, [False, True, True, True], off=2)
    with_nulls(r, [True, True, False, True], off=7)
    exp = same(gpu, lambda b: b.concat_elements(l, r), "null long views")
    assert sum(len(x) for x in exp.buffers) == 43 + 80


def test_views_empty_and_inline(gpu):
    e = ViewColumn.from_values([])
    same(gpu, lambda b: b.concat_elements(e, e), "empty")
    a = ViewColumn.from_values([b"ab", None, b""] * 1000)
    exp = same(gpu, lambda b: b.concat_elements(a, a), "all inline")
    assert exp.buffers == []


# ---- FixedSizeBinary ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("wl,wr", [(0, 0), (1, 1), (7, 7), (16, 16), (0, 5), (7, 1), (16, 3), (1, 16)])
def test_fsb(gpu, wl, wr):
    rng = np.random.default_rng(wl * 17 + wr)
    for n in (0, 1, 5, 2049, 20001):
        lv, rv = rng.integers(0, 256, (n + 3, wl), dtype=np.uint8), rng.integers(0, 256, (n + 3, wr), dtype=np.uint8)
        for nl, nr in [(None, None), (0.3, None), (None, 0.2), (0.1, 0.1)]:
            l = FixedSizeBinaryColumn(lv[2:2 + n], nulls_of(np.ones(n, bool)))
            r = FixedSizeBinaryColumn(rv[1:1 + n], nulls_of(np.ones(n, bool)))
            if nl:
                with_nulls(l, rng.random(n) > nl, off=2)
            if nr:
                with_nulls(r, rng.random(n) > nr, off=1)
            same(gpu, lambda b: b.concat_elements(l, r), f"w={wl}+{wr} n={n} nulls={nl},{nr}")


def test_fsb_width_errors(gpu):
    def fsb(w):
        return FixedSizeBinaryColumn(np.zeros((0, w), np.uint8), nulls_of([]))
    same(gpu, lambda b: b.concat_elements(fsb(2**31 - 1), fsb(2)), "width panic, zero rows")
    same(gpu, lambda b: b.concat_elements(fsb(2**30), fsb(2**30)), "width panic at 2^31")
    same(gpu, lambda b: b.concat_elements(fsb(2**30), fsb(2**30 - 1)), "width i32::MAX")


# ---- argument errors ------------------------------------------------------------------------------------------------
def test_dyn_errors(gpu):
    u, v = bytes_col([b"a"], np.int32), ViewColumn.from_values([b"a"])
    same(gpu, lambda b: b.concat_elements(u, v), "types differ")
    same(gpu, lambda b: b.concat_elements(u, bytes_col([b"a"], np.int64), is_utf8=False), "Binary vs LargeBinary")
    i = acu.HostArray.from_list(abi.I64, [1])
    same(gpu, lambda b: b.concat_elements(i, i), "unsupported")


def test_scalar_refused(gpu):
    for mk in (lambda: bytes_col([b"a"], np.int32), lambda: ViewColumn.from_values([b"a"]), lambda: FixedSizeBinaryColumn.from_values([b"a"], 1)):
        s, a = mk(), mk()
        s.nulls.is_scalar = True
        calls = [lambda: gpu.concat_elements(s, a), lambda: gpu.concat_elements(a, s)]
        if isinstance(a, Utf8Column):
            calls.append(lambda: gpu.concat_elements_utf8_many([a, s]))
        for c in calls:
            with pytest.raises(acu.ArrowError) as e:
                c()
            assert e.value.status == abi.ERR_INVALID_ARGUMENT and "not scalars" in str(e.value)


def test_refused_inside_section(gpu):
    """Synchronous: inside a section every entry point refuses before any argument check and leaves its outputs untouched;
    after the fetch the same calls run."""
    lib, h, R = gpu.lib, gpu.h, C.byref
    owned, keep = [], []
    try:
        du = gpu._upload_bytes_col(bytes_col([b"ab", b"c"], np.int32), owned)
        dv = gpu._upload_view_col(ViewColumn.from_values([b"ab", b"c"]), owned, keep)
        df = gpu._upload_fsb(FixedSizeBinaryColumn.from_values([b"a", b"b"], 1), owned)
        arr = (abi.BytesArray * 3)(du, du, du)
        buf = gpu.malloc(256)
        owned.append(buf)
        total, width = C.c_int64(-7), C.c_int32(-7)
        calls = [lambda o: lib.acu_concat_elements_bytes(h, 4, R(du), R(du), buf, None, 0, R(total), R(o)),
                 lambda o: lib.acu_concat_elements_bytes_many(h, 4, 3, arr, buf, None, 0, R(total), R(o)),
                 lambda o: lib.acu_concat_elements_bytes_many(h, 4, 0, arr, buf, None, 0, R(total), R(o)),
                 lambda o: lib.acu_concat_elements_byte_view(h, R(dv), R(dv), None, None, 0, R(total), R(o)),
                 lambda o: lib.acu_concat_elements_fixed_size_binary(h, 1, R(df), 1, R(df), R(width), R(o))]
        out = abi.ArrayOut()
        out.len = -7
        gpu.async_begin()
        try:
            for c in calls:
                assert c(out) == abi.ERR_INVALID_ARGUMENT
                assert SECTION.encode() in lib.acu_last_error(h).contents.message
        finally:
            gpu.results_fetch()
        assert out.len == -7 and total.value == -7 and width.value == -7
        out = gpu.alloc_out(64, 2)
        owned += [out.values, out.validity]
        for k, c in enumerate(calls):
            assert c(out) == (abi.ERR_COMPUTE if k == 2 else abi.OK)
    finally:
        for p in owned:
            gpu.free(p)


# ---- capacity too small: nothing is written -------------------------------------------------------------------------
def test_capacity_too_small_writes_nothing(gpu):
    lib, h = gpu.lib, gpu.h
    owned, keep = [], []
    try:
        u = bytes_col([b"abcdefghij", b"klmnopqrstu"] * 3000, np.int32)
        du = gpu._upload_bytes_col(u, owned)
        n = u.length
        total = C.c_int64(0)
        out = gpu.alloc_out(0, n)
        owned += [out.values, out.validity]
        d_off = gpu.malloc((n + 1) * 4)
        owned.append(d_off)
        assert lib.acu_concat_elements_bytes(h, 4, C.byref(du), C.byref(du), d_off, None, 0, C.byref(total), C.byref(out)) == abi.OK
        assert total.value == 2 * int(u.offsets[-1])
        d_data = gpu.malloc(total.value)
        owned.append(d_data)
        gpu.check(lib.acu_memset(h, d_data, 0xAB, total.value))
        st = lib.acu_concat_elements_bytes(h, 4, C.byref(du), C.byref(du), d_off, d_data, total.value - 1, C.byref(total), C.byref(out))
        assert st == abi.ERR_INVALID_ARGUMENT
        assert (gpu.d2h(d_data, total.value) == 0xAB).all()

        long = b"x" * 20
        v = ViewColumn.from_values([long, b"a"] * 3000)
        dv = gpu._upload_view_col(v, owned, keep)
        assert lib.acu_concat_elements_byte_view(h, C.byref(dv), C.byref(dv), None, None, 0, C.byref(total), C.byref(out)) == abi.OK
        assert total.value == 40 * 3000
        d_views = gpu.malloc(16 * 6000)
        owned.append(d_views)
        gpu.check(lib.acu_memset(h, d_views, 0xCD, 16 * 6000))
        gpu.check(lib.acu_memset(h, d_data, 0xAB, min(total.value, 2 * int(u.offsets[-1]))))
        st = lib.acu_concat_elements_byte_view(h, C.byref(dv), C.byref(dv), d_views, d_data, total.value - 1, C.byref(total), C.byref(out))
        assert st == abi.ERR_INVALID_ARGUMENT
        assert (gpu.d2h(d_views, 16 * 6000) == 0xCD).all()
        assert (gpu.d2h(d_data, min(total.value, 2 * int(u.offsets[-1]))) == 0xAB).all()
    finally:
        for p in owned:
            gpu.free(p)


# ---- overflows built on the device ----------------------------------------------------------------------------------
def device_bytes(gpu, owned, offsets, d_data):
    """acu_bytes_array over device data `d_data` with host-built (small) offsets."""
    d = abi.BytesArray()
    d_off = gpu.malloc(offsets.nbytes + 16)
    owned.append(d_off)
    gpu.h2d(d_off, offsets)
    d.offsets, d.data = d_off, d_data
    d.nulls = abi.Array()
    d.nulls.len = len(offsets) - 1
    return d


def expect_unwrap(gpu, fn, row):
    out = gpu.alloc_out(0, 1)
    try:
        total = C.c_int64(0)
        st = fn(None, None, 0, C.byref(total), C.byref(out))
        assert st == abi.ERR_PANIC_OUT_OF_BOUNDS
        d = gpu.lib.acu_last_error(gpu.h).contents
        assert d.message.decode() == "called `Option::unwrap()` on a `None` value" and d.index == row
    finally:
        gpu._free_out(out)


def test_i32_unwrap_panic_many(gpu):
    """_many over one ~0.8 GiB array whose row 4321 is heavy, passed three times: the row whose running end passes
    i32::MAX is found from the prefix sums of the three operands' lengths."""
    owned = []
    try:
        n, heavy = 5000, 4321
        lens = np.full(n, 7, dtype=np.int64)
        lens[heavy] = 800 << 20
        offs = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
        d_data = gpu.malloc(int(offs[-1]) + 16)
        owned.append(d_data)
        a = device_bytes(gpu, owned, offs, d_data)
        arr = (abi.BytesArray * 3)(a, a, a)
        d_out = gpu.malloc((n + 1) * 4)
        owned.append(d_out)
        row = first_overflow_row(3 * lens)
        assert row == heavy
        expect_unwrap(gpu, lambda oo, od, cap, tot, out: gpu.lib.acu_concat_elements_bytes_many(gpu.h, 4, 3, arr, d_out, od, cap, tot, out), row)
        # i64 offsets over the same bytes: no overflow, the total is exact
        offs64 = offs.astype(np.int64)
        a64 = device_bytes(gpu, owned, offs64, d_data)
        arr64 = (abi.BytesArray * 3)(a64, a64, a64)
        d_out64 = gpu.malloc((n + 1) * 8)
        owned.append(d_out64)
        out = gpu.alloc_out(0, n)
        owned += [out.values, out.validity]
        total = C.c_int64(0)
        gpu.check(gpu.lib.acu_concat_elements_bytes_many(gpu.h, 8, 3, arr64, d_out64, None, 0, C.byref(total), C.byref(out)))
        assert total.value == 3 * int(lens.sum())
        assert np.array_equal(gpu.d2h(d_out64, (n + 1) * 8, np.int64), np.concatenate([[0], np.cumsum(3 * lens)]))
    finally:
        for p in owned:
            gpu.free(p)


def test_i32_unwrap_panic_two_columns(gpu):
    """Two ~1.1 GiB columns over one device buffer, rows of different lengths; the failing row lies past the first CTA."""
    owned = []
    try:
        n = 6000
        rng = np.random.default_rng(5)
        size = 1100 << 20
        ll = rng.integers(0, 2 * size // n, n).astype(np.int64)
        rl = rng.integers(0, 2 * size // n, n).astype(np.int64)
        lo = np.concatenate([[0], np.cumsum(ll)])
        ro = np.concatenate([[0], np.cumsum(rl)])
        d_data = gpu.malloc(int(max(lo[-1], ro[-1])) + 16)
        owned.append(d_data)
        l, r = device_bytes(gpu, owned, lo.astype(np.int32), d_data), device_bytes(gpu, owned, ro.astype(np.int32), d_data)
        row = first_overflow_row(ll + rl)
        assert row is not None and row >= 2048
        d_out = gpu.malloc((n + 1) * 4)
        owned.append(d_out)
        expect_unwrap(gpu, lambda oo, od, cap, tot, out: gpu.lib.acu_concat_elements_bytes(gpu.h, 4, C.byref(l), C.byref(r), d_out, od, cap, tot,
                                                                                           out), row)
    finally:
        for p in owned:
            gpu.free(p)


def test_view_offset_overflow(gpu):
    """Two long views over the same 1.1 GiB range: 2.2 GiB of data => "byte array offset overflow" before any row is
    written. Null rows with such views count nothing."""
    owned = []
    try:
        size = 1100 << 20
        d_buf = gpu.malloc(size + 16)
        owned.append(d_buf)
        views = np.zeros((3, 16), np.uint8)
        big = np.frombuffer(np.array([size, 0x64636261, 0, 0], np.uint32).tobytes(), np.uint8)
        views[0] = big
        views[1] = big
        views[2, :4] = np.frombuffer(np.uint32(1).tobytes(), np.uint8)
        views[2, 4] = 0x7A
        table = (C.c_void_p * 1)(d_buf)

        def varr(rows, validity_mask=None):
            d = abi.ViewArray()
            dv = gpu.malloc(16 * len(rows) + 16)
            owned.append(dv)
            gpu.h2d(dv, views[rows])
            d.views, d.buffers, d.n_buffers = dv, table, 1
            d.nulls = gpu._upload_nulls(nulls_of(validity_mask if validity_mask is not None else [True] * len(rows)), owned)
            return d

        out = gpu.alloc_out(0, 4)
        owned += [out.values, out.validity]
        total = C.c_int64(0)
        d_views = gpu.malloc(16 * 4)
        owned.append(d_views)
        gpu.check(gpu.lib.acu_memset(gpu.h, d_views, 0xCD, 64))
        l, r = varr([0]), varr([1])
        for vo in (None, d_views):
            st = gpu.lib.acu_concat_elements_byte_view(gpu.h, C.byref(l), C.byref(r), vo, None, 0, C.byref(total), C.byref(out))
            assert st == abi.ERR_ARITHMETIC_OVERFLOW
            assert gpu.lib.acu_last_error(gpu.h).contents.message.decode() == "Arithmetic overflow: byte array offset overflow"
        assert (gpu.d2h(d_views, 64) == 0xCD).all()
        # the same views under null rows: only the valid rows' results count
        l, r = varr([0, 2, 0, 2], [False, True, True, True]), varr([1, 1, 2, 2], [True, True, False, True])
        gpu.check(gpu.lib.acu_concat_elements_byte_view(gpu.h, C.byref(l), C.byref(r), None, None, 0, C.byref(total), C.byref(out)))
        assert total.value == 1 + size and out.null_count == 2
    finally:
        for p in owned:
            gpu.free(p)
