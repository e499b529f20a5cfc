"""zip of Utf8 / LargeUtf8 / Binary, view, Boolean and FixedSizeBinary columns on the device against tests/oracle_zip.py, bit
for bit: offsets, data bytes, views (buffer-index rewrites under nulls included), the referenced buffer lists, value bits
and bytes under nulls, validity, null count, NullBuffer presence, and error status / text / row. Every case uses a fixed
seed. The grid-round cases are sized from zip.cu's launch constants and the bytes engine's rows per CTA (checked against
the source by test_zip_launch_constants.py)."""
import ctypes as C

import numpy as np
import pytest

import acu
from acu import FixedSizeBinaryColumn, HostArray, Utf8Column, ViewColumn, slice_column
from acu import _abi as abi

import oracle_zip as oz
import zip_util as zu
from oracle_filter_take import OracleError

pytestmark = pytest.mark.gpu

ZIP_THREADS = 256
ZIP_PER_SM = 16
ZIP_FSB_CHUNKS = 2
BY_ROWS = 2048  # bytes_engine.cuh: rows per CTA of the engine's passes
TYPES = ["utf8", "large_utf8", "view", "boolean", "fsb5"]
SIDES = ["array", "scalar", "null"]
MASKS = ["all_true", "all_false", "alternating", "runs", "random"]


def run_both(gpu, m, t, f, data=True):
    try:
        exp, eerr = oz.zip(m, t, f, data), None
    except OracleError as e:
        exp, eerr = None, e
    try:
        got, gerr = gpu.zip(m, t, f), None
    except acu.ArrowError as e:
        got, gerr = None, e
    if eerr is not None:
        assert gerr is not None, f"expected {eerr.message}"
        assert (gerr.status, gerr.message, gerr.index) == (eerr.status, eerr.message, eerr.index)
        return None
    assert gerr is None, gerr.message
    zu.assert_same(got, exp, t, f)
    return got


# ---- inputs ----------------------------------------------------------------------------------------------------------
def make_mask(rng, n, kind, with_nulls, bit_offset):
    if kind == "all_true":
        v = np.ones(n, bool)
    elif kind == "all_false":
        v = np.zeros(n, bool)
    elif kind == "alternating":
        v = np.arange(n) % 2 == 0
    elif kind == "runs":
        v = (np.arange(n) // 100) % 2 == 0
    else:
        v = rng.random(n) < 0.5
    valid = rng.random(n) >= 0.2 if with_nulls else None
    return zu.mask_array(v, valid, bit_offset)


def bytes_col(rng, n, ob, null_p=0.2, skip=3, bit_offset=0, scalar=False):
    """n rows after `skip` leading rows (offsets[0] != 0); null rows keep bytes under them."""
    total = n + skip
    lens = rng.integers(0, 25, total)
    offs = np.zeros(total + 1, np.int32 if ob == 4 else np.int64)
    offs[1:] = np.cumsum(lens)
    data = rng.integers(0, 256, int(offs[-1]) + 3, dtype=np.uint8)
    valid = rng.random(n) >= null_p
    return Utf8Column(offs[skip:], data, zu.nulls(valid if null_p else None, scalar, bit_offset, n))


def view_col(rng, n, null_p=0.2, scalar=False, block_size=48):
    items = [None if rng.random() < null_p else rng.integers(0, 256, int(rng.integers(0, 30)), dtype=np.uint8).tobytes() for _ in range(n)]
    garbage = []
    for _ in range(7):  # views under nulls: inline and long ones with arbitrary buffer indexes
        g = rng.integers(0, 256, 16, dtype=np.uint8)
        g[:4] = np.frombuffer(np.uint32(rng.choice([3, 40, 0xFFFFFFFF])).tobytes(), np.uint8)
        garbage.append(g)
    col = ViewColumn.from_values(items, block_size=block_size, scalar=scalar, garbage_under_nulls=garbage)
    if null_p == 0:
        col.nulls.validity, col.nulls.null_count = None, 0
    return col


def bool_col(rng, n, null_p=0.2, bit_offset=0, scalar=False):
    h = HostArray.bool_from_numpy(rng.random(n) < 0.5, (rng.random(n) >= null_p) if null_p else None, bit_offset, bit_offset)
    h.is_scalar = scalar
    return h


def fsb_col(rng, n, w, null_p=0.2, bit_offset=0, scalar=False):
    valid = rng.random(n) >= null_p
    return FixedSizeBinaryColumn(rng.integers(0, 256, (n, w), dtype=np.uint8), zu.nulls(valid if null_p else None, scalar, bit_offset, n))


def make_side(rng, typ, kind, n, bit_offset=0):
    """kind: array (n rows with nulls), scalar (valid), null (a null scalar with bytes / bits under it)."""
    sc = kind != "array"
    rows = 1 if sc else n
    p = 0.2 if kind == "array" else 0.0
    if typ in ("utf8", "large_utf8"):
        col = bytes_col(rng, rows, 4 if typ == "utf8" else 8, p, bit_offset=bit_offset, scalar=sc)
    elif typ == "view":
        col = view_col(rng, rows, p, sc)
    elif typ == "boolean":
        col = bool_col(rng, rows, p, bit_offset, sc)
    else:
        col = fsb_col(rng, rows, int(typ[3:]), p, bit_offset, sc)
    if kind == "null":
        nb = col if isinstance(col, HostArray) else col.nulls
        nb.validity, nb.validity_offset, nb.null_count = acu.pack_bits([False]), 0, 1
    return col


# ---- tests ----------------------------------------------------------------------------------------------------------
CASES = zu.golden_cases()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_golden(gpu, case):
    m, t, f = zu.golden_mask(case), zu.golden_side(case, "truthy"), zu.golden_side(case, "falsy")
    got = run_both(gpu, m, t, f)
    exp = case["expect"]
    assert zu.logical_rows(got) == [None if v is None else bytes.fromhex(v) for v in exp["values"]]


@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 200])
@pytest.mark.parametrize("typ", TYPES)
def test_every_side_combination(gpu, typ, n):
    """Arrays, valid scalars and null scalars on both sides, every mask shape with and without nulls, masks and validity at
    bit offsets 0, 1, 7 and 63."""
    rng = np.random.default_rng(1000 + n + 7 * TYPES.index(typ))
    k = 0
    for mk in MASKS:
        for mnull in (False, True):
            for ts in SIDES:
                for fs in SIDES:
                    off = (0, 1, 7, 63)[k % 4]
                    k += 1
                    m = make_mask(rng, n, mk, mnull, off)
                    t = make_side(rng, typ, ts, n, (off * 3) % 64)
                    f = make_side(rng, typ, fs, n, (off * 5) % 64)
                    run_both(gpu, m, t, f)


def test_bytes_sliced_and_multi_cta(gpu):
    """Sliced operands (offsets[0] != 0, validity at odd bit offsets) over several of the engine's CTAs."""
    rng = np.random.default_rng(7)
    n = 3 * BY_ROWS + 5
    for ob in (4, 8):
        base_t, base_f = bytes_col(rng, n + 40, ob), bytes_col(rng, n + 40, ob)
        t, f = slice_column(base_t, 17, n), slice_column(base_f, 33, n)
        for mk in MASKS:
            run_both(gpu, make_mask(rng, n, mk, True, 7), t, f)
        run_both(gpu, make_mask(rng, n, "random", True, 1), t, make_side(rng, "utf8" if ob == 4 else "large_utf8", "null", n))


def grid_rows(gpu, per_thread_rows):
    return gpu.lib.acu_device_sm_count(gpu.h) * ZIP_PER_SM * ZIP_THREADS * per_thread_rows


def test_views_past_one_grid_round_with_several_buffers(gpu):
    rng = np.random.default_rng(11)
    n = grid_rows(gpu, 1) + 65
    items_t = [None if i % 7 == 0 else bytes([i % 251]) * (i % 29) for i in range(n)]
    t = ViewColumn.from_values(items_t, block_size=4096)
    f = view_col(rng, n, 0.3, block_size=4096)
    assert len(t.buffers) > 1 and len(f.buffers) > 1
    run_both(gpu, make_mask(rng, n, "random", True, 63), t, f)
    run_both(gpu, make_mask(rng, n, "runs", False, 0), make_side(rng, "view", "scalar", n), f)


def test_boolean_past_one_grid_round(gpu):
    rng = np.random.default_rng(12)
    n = grid_rows(gpu, 64) + 65
    run_both(gpu, make_mask(rng, n, "random", True, 7), bool_col(rng, n, 0.1, 1), bool_col(rng, n, 0.1, 63))


@pytest.mark.parametrize("w", [16, 5])
def test_fsb_past_one_grid_round(gpu, w):
    rng = np.random.default_rng(13 + w)
    n = grid_rows(gpu, ZIP_FSB_CHUNKS) * 16 // w + 65
    run_both(gpu, make_mask(rng, n, "random", True, 1), fsb_col(rng, n, w), fsb_col(rng, n, w, 0.0))
    run_both(gpu, make_mask(rng, n, "alternating", False, 0), make_side(rng, f"fsb{w}", "scalar", n), fsb_col(rng, n, w))


@pytest.mark.parametrize("w", list(range(66)) + [127, 4097])
def test_fsb_widths(gpu, w):
    rng = np.random.default_rng(100 + w)
    n = 37
    for ts, fs in (("array", "array"), ("array", "null"), ("scalar", "array"), ("null", "scalar")):
        run_both(gpu, make_mask(rng, n, "random", True, w % 64), make_side(rng, f"fsb{w}", ts, n, 7), make_side(rng, f"fsb{w}", fs, n, 1))


@pytest.mark.parametrize("ts,fs", [(a, b) for a in SIDES for b in SIDES])
def test_fsb_32_with_scalars(gpu, ts, fs):
    """Width 32 with scalars, which acu_zip refuses, goes through the any-width kernel."""
    rng = np.random.default_rng(32)
    n = 300
    for mk in ("all_true", "random"):
        run_both(gpu, make_mask(rng, n, mk, True, 0), make_side(rng, "fsb32", ts, n), make_side(rng, "fsb32", fs, n))


def test_fsb_raw_unaligned_pointers(gpu):
    """Operands and output at odd addresses inside sentinel-filled allocations: no byte outside the output is written."""
    rng = np.random.default_rng(5)
    for w in (1, 3, 16, 20, 33):
        n = 301
        t, f = rng.integers(0, 256, (n, w), dtype=np.uint8), rng.integers(0, 256, (n, w), dtype=np.uint8)
        sel = rng.random(n) < 0.5
        m = zu.mask_array(sel)
        with gpu._scope() as s:
            md = s.upload(m).descriptor()
            buf = s.malloc(3 * (n * w + 64))
            gpu.h2d(buf, np.full(3 * (n * w + 64), 0xA5, np.uint8))
            tp, fp, op = buf + 3, buf + n * w + 64 + 5, buf + 2 * (n * w + 64) + 7
            gpu.h2d(tp, t)
            gpu.h2d(fp, f)
            td, fd = abi.Array(), abi.Array()
            td.values, td.len, fd.values, fd.len = tp, n, fp, n
            out = abi.ArrayOut()
            out.values, out.validity = op, s.malloc(64 + n)
            gpu.check(gpu.lib.acu_zip_fixed_size_binary(gpu.h, w, C.byref(md), C.byref(td), C.byref(fd), C.byref(out)))
            assert out.has_validity == 0 and out.null_count == 0
            region = gpu.d2h(buf + 2 * (n * w + 64), n * w + 64)
            np.testing.assert_array_equal(region[7:7 + n * w].reshape(n, w), np.where(sel[:, None], t, f))
            assert (region[:7] == 0xA5).all() and (region[7 + n * w:] == 0xA5).all()


MIB = 1 << 20
N_OVF = 2049


@pytest.mark.parametrize("branch", ["zip_impl", "mixed", "all_true", "one_null"])
def test_i32_offset_overflow(gpu, branch):
    """A 1 MiB scalar repeated past 2^31 bytes, on each bytes branch: the error comes from the sizing call, before a data
    buffer of that size exists."""
    big = zu.bytes_column([bytes(range(256)) * (MIB // 256)], scalar=True)
    if branch == "zip_impl":
        m, f = zu.mask_array(np.ones(N_OVF, bool)), zu.bytes_column([b"x"] * N_OVF)
    elif branch == "mixed":
        m, f = zu.mask_array(np.arange(2 * N_OVF) % 2 == 0), zu.bytes_column([bytes(MIB)], scalar=True)
    elif branch == "all_true":
        m, f = zu.mask_array(np.ones(N_OVF, bool)), zu.bytes_column([b"abc"], scalar=True)
    else:
        m, f = zu.mask_array(np.ones(N_OVF, bool)), zu.bytes_column([None], scalar=True)
    run_both(gpu, m, big, f, data=False)
    with gpu._scope() as s:  # the sizing call (no data buffer) already fails
        md, dt, df = s.upload(m).descriptor(), gpu._upload_bytes_col(big, s), gpu._upload_bytes_col(f, s)
        d_off, out, tot = s.malloc((m.length + 1) * 4), s.out(0, m.length), C.c_int64(0)
        st = gpu.lib.acu_zip_bytes(gpu.h, 4, C.byref(md), C.byref(dt), C.byref(df), d_off, None, 0, C.byref(tot), C.byref(out))
        assert st == (abi.ERR_INVALID_ARGUMENT if branch == "zip_impl" else abi.ERR_PANIC_OUT_OF_BOUNDS)


def test_large_utf8_past_4_gib(gpu):
    """A LargeUtf8 result of more than 2^32 bytes: every offset, and the bytes around 2^32 and at the end."""
    pat = (np.arange(MIB, dtype=np.int64) * 7 % 251).astype(np.uint8).tobytes()
    n = 4200
    t = zu.bytes_column([pat], ob=8, scalar=True)
    f = zu.bytes_column([b"f%d" % i for i in range(n)], ob=8)
    sel = np.ones(n, bool)
    sel[::97] = False
    m = zu.mask_array(sel)
    exp = oz.zip(m, t, f, data=False)
    total = int(exp.offsets[-1])
    assert total > (1 << 32)
    with gpu._scope() as s:
        md = s.upload(m).descriptor()
        dt, df = gpu._upload_bytes_col(t, s), gpu._upload_bytes_col(f, s)
        d_off = s.malloc((n + 1) * 8)
        out = s.out(0, n)
        tot = C.c_int64(0)
        gpu.check(gpu.lib.acu_zip_bytes(gpu.h, 8, C.byref(md), C.byref(dt), C.byref(df), d_off, None, 0, C.byref(tot), C.byref(out)))
        assert tot.value == total
        d_data = s.malloc(total)
        gpu.check(gpu.lib.acu_zip_bytes(gpu.h, 8, C.byref(md), C.byref(dt), C.byref(df), d_off, d_data, total, C.byref(tot), C.byref(out)))
        np.testing.assert_array_equal(gpu.d2h(d_off, (n + 1) * 8, np.int64), exp.offsets)
        assert out.has_validity == 0
        for row in (int(np.searchsorted(exp.offsets, 1 << 32, "right")) - 1, n - 1, n - 2):
            b, e = int(exp.offsets[row]), int(exp.offsets[row + 1])
            got = gpu.d2h(d_data + b, e - b).tobytes()
            assert got == (pat if sel[row] else b"f%d" % row), row


def test_scalar_view_inline_falsy_rebased(gpu):
    """zip.rs:759-769 on the device: the inline falsy view's buffer-index word is raised by truthy's buffer count."""
    t = zu.view_column([b"a" * 20], scalar=True)
    t.buffers = t.buffers + [np.zeros(4, np.uint8)]
    f = zu.view_column([b"short"], scalar=True)
    f.buffers = [np.zeros(8, np.uint8)]
    got = run_both(gpu, zu.mask_array([True, False, False]), t, f)
    assert got.views.view(np.uint32).reshape(-1, 4)[1, 2] == int(f.views.view(np.uint32)[0, 2]) + 2


def test_errors(gpu):
    m = zu.mask_array([True, False])
    run_both(gpu, m, zu.bytes_column([b"a"]), zu.bytes_column([b"a", b"b"]))
    run_both(gpu, m, zu.bytes_column([b"a", b"b"]), zu.bytes_column([b"a", b"b"], ob=8))
    run_both(gpu, m, zu.fsb_column([b"ab", b"cd"], 2), zu.fsb_column([b"abc", b"def"], 3))
    run_both(gpu, m, zu.view_column([b"a", b"b"]), zu.view_column([b"a", b"b", b"c"]))
    t2 = zu.bool_column([b"\x01", b"\x00"])
    t2.is_scalar = True
    run_both(gpu, m, t2, zu.bool_column([b"\x01", b"\x00"]))


def test_refused_inside_a_section(gpu):
    """All four calls synchronise, so each is refused between acu_async_begin and acu_results_fetch."""
    m = zu.mask_array([True])
    with gpu._scope() as s:
        md = s.upload(m).descriptor()
        bd = s.upload(zu.bool_column([b"\x01"])).descriptor()
        fd = gpu._upload_fsb(zu.fsb_column([b"ab"], 2), s)
        by = gpu._upload_bytes_col(zu.bytes_column([b"ab"]), s)
        vw = gpu._upload_view_col(zu.view_column([b"ab"]), s, s.keep)
        out, offs, views, tot, which = s.out(64, 1), s.malloc(64), s.malloc(64), C.c_int64(0), C.c_int32(0)
        calls = {
            "boolean": lambda: gpu.lib.acu_zip_boolean(gpu.h, C.byref(md), C.byref(bd), C.byref(bd), C.byref(out)),
            "fixed_size_binary": lambda: gpu.lib.acu_zip_fixed_size_binary(gpu.h, 2, C.byref(md), C.byref(fd), C.byref(fd), C.byref(out)),
            "bytes": lambda: gpu.lib.acu_zip_bytes(gpu.h, 4, C.byref(md), C.byref(by), C.byref(by), offs, None, 0, C.byref(tot), C.byref(out)),
            "byte_view": lambda: gpu.lib.acu_zip_byte_view(gpu.h, C.byref(md), C.byref(vw), C.byref(vw), views, C.byref(out), C.byref(which)),
        }
        for name, call in calls.items():
            gpu.async_begin()
            st = call()
            gpu.results_fetch()
            assert st == abi.ERR_INVALID_ARGUMENT, name
            assert "not available between acu_async_begin and acu_results_fetch" in gpu.lib.acu_last_error(gpu.h).contents.message.decode()


def test_views_must_be_16_byte_aligned(gpu):
    """The one alignment acu_zip_byte_view requires: that of the u128 views buffer."""
    m = zu.mask_array([True, False])
    with gpu._scope() as s:
        md = s.upload(m).descriptor()
        t = gpu._upload_view_col(zu.view_column([b"ab", b"cd"]), s, s.keep)
        f = gpu._upload_view_col(zu.view_column([b"ef", b"gh"]), s, s.keep)
        out, views, which = s.out(0, 2), s.malloc(64), C.c_int32(0)
        for case in ("truthy", "falsy", "out"):
            t2, f2 = abi.ViewArray.from_buffer_copy(t), abi.ViewArray.from_buffer_copy(f)
            dst = views
            if case == "truthy":
                t2.views = t.views + 8
            elif case == "falsy":
                f2.views = f.views + 8
            else:
                dst = views + 8
            st = gpu.lib.acu_zip_byte_view(gpu.h, C.byref(md), C.byref(t2), C.byref(f2), dst, C.byref(out), C.byref(which))
            assert st == abi.ERR_INVALID_ARGUMENT, case
            assert gpu.lib.acu_last_error(gpu.h).contents.message.decode() == "Invalid argument error: views must be 16-byte aligned"


@pytest.mark.parametrize("falsy_kind", ["scalar", "null"])
@pytest.mark.parametrize("w", [3, 16, 20, 33])
def test_fsb_raw_unaligned_output_with_nulls_and_scalar(gpu, w, falsy_kind):
    """Output 7 bytes past a 16-byte boundary (the first chunk is partial), a truthy array with nulls at validity bit offset
    5, and a falsy scalar (valid or null) at an odd address: the scalar's phase and the validity-word ownership off an
    aligned output, against the oracle, with no byte outside the output written."""
    rng = np.random.default_rng(40 + w)
    n = 700
    t_vals = rng.integers(0, 256, (n, w), dtype=np.uint8)
    s_vals = rng.integers(0, 256, (1, w), dtype=np.uint8)
    valid = rng.random(n) >= 0.25
    sel, mvalid = rng.random(n) < 0.5, rng.random(n) >= 0.1
    m = zu.mask_array(sel, mvalid, 3)
    tcol = FixedSizeBinaryColumn(t_vals, zu.nulls(valid, False, 5, n))
    fcol = FixedSizeBinaryColumn(s_vals, zu.nulls([False] if falsy_kind == "null" else None, True, 0, 1))
    exp = oz.zip(m, tcol, fcol)
    span = n * w + 64
    with gpu._scope() as s:
        md = s.upload(m).descriptor()
        buf = s.malloc(3 * span)
        gpu.h2d(buf, np.full(3 * span, 0xA5, np.uint8))
        tp, sp, op = buf + 3, buf + span + 5, buf + 2 * span + 7
        gpu.h2d(tp, t_vals)
        gpu.h2d(sp, s_vals)
        td = gpu._upload_nulls(tcol.nulls, s)
        td.values = tp
        fd = gpu._upload_nulls(fcol.nulls, s)
        fd.values = sp
        out = abi.ArrayOut()
        out.values, out.validity = op, s.malloc(acu.bitmap_bytes(n) + 8)
        gpu.check(gpu.lib.acu_zip_fixed_size_binary(gpu.h, w, C.byref(md), C.byref(td), C.byref(fd), C.byref(out)))
        region = gpu.d2h(buf + 2 * span, span)
        np.testing.assert_array_equal(region[7:7 + n * w].reshape(n, w), exp.values)
        assert (region[:7] == 0xA5).all() and (region[7 + n * w:] == 0xA5).all()
        assert bool(out.has_validity) == (exp.valid is not None)
        if exp.valid is not None:
            np.testing.assert_array_equal(acu.unpack_bits(gpu.d2h(out.validity, acu.bitmap_bytes(n)), 0, n), exp.valid)
            assert out.null_count == int(n - exp.valid.sum())
