"""filter / take of FixedSizeBinary columns on the device against tests/oracle_fixed_size_binary.py, bit for bit: the value
bytes (under null rows included), validity, null count, NullBuffer presence, length, and error status / text / row. Every
case uses a fixed seed. The grid-round cases are sized from fixed_size_binary.cu's launch constants (checked against the
source by test_fixed_size_binary_launch_constants.py)."""
import ctypes as C

import numpy as np
import pytest

import acu
from acu import FixedSizeBinaryColumn, FixedSizeListColumn, HostArray, ListColumn, RunEndColumn, StructColumn, UnionColumn, Utf8Column
from acu import _abi as abi

import oracle_fixed_size_binary as of
import oracle_list as ol
import test_oracle_fixed_size_binary as tg

pytestmark = pytest.mark.gpu

FSB_THREADS = 256
FSB_PER_SM = 8
INDEX_DTYPES = [abi.I8, abi.U8, abi.I16, abi.U16, abi.I32, abi.U32, abi.I64, abi.U64]
NP = {abi.I8: np.int8, abi.U8: np.uint8, abi.I16: np.int16, abi.U16: np.uint16, abi.I32: np.int32, abi.U32: np.uint32,
      abi.I64: np.int64, abi.U64: np.uint64}
WIDTHS = list(range(66)) + [127, 128, 129, 511, 512, 513, 768, 4095, 4096, 4097, 65537]


def chunks_per_thread(w):
    r = 2 if w >= 16 else 3 if w >= 8 else 5 if w >= 4 else 9 if w >= 2 else 17
    return 4 if r <= 3 else 2 if r <= 5 else 1


def random_column(rng, n, w, null_p=0.2, bit_offset=0):
    vals = rng.integers(0, 256, (n, w), dtype=np.uint8)
    mask = rng.random(n) >= null_p
    nulls = HostArray.from_list(abi.U8, [0 if v else None for v in mask], bit_offset=bit_offset)
    nulls.values = np.zeros(0, np.uint8)
    return FixedSizeBinaryColumn(vals, nulls)


def same(got, exp):
    assert got.length == exp.length
    assert got.values.shape == exp.values.shape
    assert np.array_equal(got.values, exp.values)
    assert of.has_buffer(got) == of.has_buffer(exp)
    if of.has_buffer(exp):
        assert np.array_equal(of.valid_mask(got), of.valid_mask(exp))
        assert got.nulls.null_count == exp.nulls.null_count


def gpu_filter(gpu, col, pred):
    return gpu.filter(col, HostArray.bool_from_numpy(np.asarray(pred, bool)))


def oracle_filter(col, pred):
    return of.filter(col, np.asarray(pred, bool))


def run_both(gpu_fn, oracle_fn):
    """(result, None) or (None, error) for the device and the oracle; errors compared on status, text and row."""
    try:
        exp, eerr = oracle_fn(), None
    except ol.OracleError as e:
        exp, eerr = None, e
    try:
        got, gerr = gpu_fn(), None
    except acu.ArrowError as e:
        got, gerr = None, e
    if eerr is not None:
        assert gerr is not None, "the device did not fail"
        assert (gerr.status, gerr.message, gerr.index) == (eerr.status, eerr.message, eerr.index)
        return
    assert gerr is None, gerr.message
    same(got, exp)


@pytest.mark.parametrize("i", range(len(tg.CASES)), ids=[f"{c['name']}-{k}" for k, c in enumerate(tg.CASES)])
def test_golden(gpu, i):
    case = tg.CASES[i]
    tg.check(case, lambda: tg.run_case(case, lambda col, p: gpu_filter(gpu, col, p),
                                       lambda col, ix: gpu.take(col, ix[4])))


@pytest.mark.parametrize("w", WIDTHS)
def test_filter_every_width(gpu, w):
    rng = np.random.default_rng(1000 + w)
    n = 300 if w < 4096 else 40
    col = random_column(rng, n, w)
    for pred in (rng.random(n) < 0.1, rng.random(n) < 0.9, np.zeros(n, bool), np.ones(n, bool), rng.random(n - 7) < 0.5):
        run_both(lambda: gpu_filter(gpu, col, pred), lambda: oracle_filter(col, pred))


@pytest.mark.parametrize("w", [0, 3, 16, 20, 32, 100])
def test_filter_predicate_with_nulls(gpu, w):
    """A null predicate slot does not select its row (prep_null_mask_filter)."""
    rng = np.random.default_rng(1500 + w)
    n = 400
    col = random_column(rng, n, w)
    for sel in (0.3, 0.95):
        pred = HostArray.bool_from_numpy(rng.random(n - 3) < sel, rng.random(n - 3) >= 0.2)
        mask = ol.filter_mask(pred)
        run_both(lambda: gpu.filter(col, pred), lambda: of.filter(col, mask))


@pytest.mark.parametrize("w", WIDTHS)
def test_take_every_width(gpu, w):
    rng = np.random.default_rng(2000 + w)
    n = 200 if w < 4096 else 30
    col = random_column(rng, n, w)
    dt = INDEX_DTYPES[w % 8]
    m = 257
    idx = rng.integers(0, min(n, np.iinfo(NP[dt]).max), m).astype(NP[dt])
    iv = rng.random(m) >= 0.15
    ix = HostArray.from_numpy(dt, idx, iv)
    run_both(lambda: gpu.take(col, ix), lambda: of.take(col, idx, iv, True, dt))
    ixn = HostArray.from_numpy(dt, idx)
    run_both(lambda: gpu.take(col, ixn, True), lambda: of.take(col, idx, None, False, dt, True))


@pytest.mark.parametrize("dt", INDEX_DTYPES)
@pytest.mark.parametrize("w", [0, 2, 3, 16, 20, 32])
@pytest.mark.parametrize("check", [False, True])
def test_take_index_types_nulls_and_errors(gpu, dt, w, check):
    rng = np.random.default_rng(3000 + w * 16 + dt)
    n = 50
    col = random_column(rng, n, w)
    info = np.iinfo(NP[dt])
    m = 64
    # in-bounds, null out-of-bounds, and negative indices for the signed types
    idx = rng.integers(0, n, m).astype(np.int64)
    iv = rng.random(m) >= 0.3
    idx[~iv & (rng.random(m) < 0.5)] = min(info.max, 120)
    if info.min < 0:
        idx[rng.integers(0, m, 2)] = -1
    idx = idx.astype(NP[dt])
    for valid, buf in ((iv, True), (None, False)):
        ix = HostArray.from_numpy(dt, idx, valid)
        run_both(lambda: gpu.take(col, ix, check), lambda: of.take(col, idx, valid, buf, dt, check))
    # values without nulls: the take_bits panic cannot occur
    col2 = random_column(rng, n, w, null_p=0.0)
    ix = HostArray.from_numpy(dt, idx, iv)
    run_both(lambda: gpu.take(col2, ix, check), lambda: of.take(col2, idx, iv, True, dt, check))


@pytest.mark.parametrize("w", [3, 33, 20, 36])
def test_take_u64_indices_that_wrap_into_the_buffer(gpu, w):
    rng = np.random.default_rng(4000 + w)
    n = 64
    col = random_column(rng, n, w, null_p=0.0)
    if w % 2:  # idx = k / w (mod 2^64): the slice starts at byte k, any byte of the buffer
        inv = pow(w, -1, 1 << 64)
        idx = np.array([int(k) * inv % (1 << 64) for k in rng.integers(0, n * w - w + 1, 40)], np.uint64)
    else:  # idx = row + c * 2^64 / tz (tz = the largest power of two dividing w): idx * w wraps to row * w
        tz = w & -w
        idx = np.array([(int(r) + int(c) * ((1 << 64) // tz)) % (1 << 64) for r, c in zip(rng.integers(0, n, 40), rng.integers(1, tz, 40))],
                       np.uint64)
    ix = HostArray.from_numpy(abi.U64, idx)
    run_both(lambda: gpu.take(col, ix), lambda: of.take(col, idx, None, False, abi.U64))


@pytest.mark.parametrize("w", [5, 20, 33])
@pytest.mark.parametrize("bit_offset", [1, 7, 63])
def test_sliced_columns(gpu, w, bit_offset):
    """The validity reaches the device at bit offset 1 / 7 / 63 (the values are copied afresh here; the raw-buffer tests
    below place them at unaligned addresses)."""
    rng = np.random.default_rng(5000 + w + bit_offset)
    col = random_column(rng, 300 + bit_offset, w).slice(bit_offset, 300)
    assert col.nulls.validity_offset == bit_offset
    pred = rng.random(300) < 0.4
    run_both(lambda: gpu_filter(gpu, col, pred), lambda: oracle_filter(col, pred))
    idx = rng.integers(0, 300, 100).astype(np.uint32)
    iv = rng.random(100) >= 0.2
    ix = HostArray.from_numpy(abi.U32, idx, iv)
    run_both(lambda: gpu.take(col, ix), lambda: of.take(col, idx, iv, True, abi.U32))


# ---- the C ABI on raw device buffers: values at any alignment, outputs inside a sentinel-filled allocation --------------
def _raw(gpu, col, vshift, oshift, m, call):
    """Run call(values Array, out ArrayOut) with the values at byte `vshift` of an allocation and the output at byte
    `oshift` of one with capacity exactly m * W; returns (the output bytes, the ArrayOut); the bytes around must keep the
    sentinel."""
    w = col.width
    n = col.length
    vbuf = gpu.malloc(n * w + vshift + 64)
    obuf = gpu.malloc(m * w + oshift + 64)
    vbits = gpu.malloc(acu.bitmap_bytes(n) + 8) if col.nulls.validity is not None else None
    obits = gpu.malloc(acu.bitmap_bytes(m) + 8)
    try:
        gpu.h2d(vbuf, np.full(n * w + vshift + 64, 0xA5, np.uint8))
        gpu.h2d(vbuf + vshift, col.values.reshape(-1))
        gpu.h2d(obuf, np.full(m * w + oshift + 64, 0x5A, np.uint8))
        a = abi.Array()
        a.values, a.len = vbuf + vshift, n
        if vbits:
            gpu.h2d(vbits, col.nulls.validity)
            a.validity, a.validity_offset, a.null_count = vbits, col.nulls.validity_offset, col.nulls.null_count
        out = abi.ArrayOut()
        out.values, out.validity = obuf + oshift, obits
        call(a, out)
        full = gpu.d2h(obuf, m * w + oshift + 64)
        assert (full[:oshift] == 0x5A).all() and (full[oshift + m * w:] == 0x5A).all(), "a byte outside the output was written"
        nulls = HostArray(abi.U8, np.zeros(0, np.uint8), out.len, gpu.d2h(obits, acu.bitmap_bytes(out.len)) if out.has_validity else None,
                          0, 0, out.null_count if out.has_validity else 0)
        return FixedSizeBinaryColumn(full[oshift:oshift + out.len * w].reshape(out.len, w), nulls)
    finally:
        for p in (vbuf, obuf, vbits, obits):
            gpu.free(p)


@pytest.mark.parametrize("w", [1, 2, 4, 8, 16, 20, 32, 64])
@pytest.mark.parametrize("vshift,oshift", [(0, 0), (1, 1), (3, 15), (8, 0), (0, 8)])
def test_raw_alignment_and_sentinels(gpu, w, vshift, oshift):
    rng = np.random.default_rng(6000 + w * 100 + vshift * 10 + oshift)
    n = 500
    col = random_column(rng, n, w)
    pred = rng.random(n) < 0.5
    k = int(pred.sum())
    with gpu._scope() as s:
        plan = gpu._plan(s, HostArray.bool_from_numpy(pred))
        got = _raw(gpu, col, vshift, oshift, k, lambda a, o: gpu.check(gpu.lib.acu_filter_fixed_size_binary(gpu.h, plan, w, C.byref(a), C.byref(o))))
    same(got, oracle_filter(col, pred))
    m = 333
    idx = rng.integers(0, n, m).astype(np.uint32)
    idx[::17] = n + 5  # null and out of bounds: zeros
    iv = rng.random(m) >= 0.2
    iv[::17] = False
    ix = HostArray.from_numpy(abi.U32, idx, iv)
    with gpu._scope() as s:
        idd = s.upload(ix).descriptor()
        got = _raw(gpu, col, vshift, oshift, m, lambda a, o: gpu.check(gpu.lib.acu_take_fixed_size_binary(gpu.h, w, C.byref(a), C.byref(idd), abi.U32, 0,
                                                                                                         C.byref(o))))
    same(got, of.take(col, idx, iv, True, abi.U32))


@pytest.mark.parametrize("w", [2, 4, 8, 16])
def test_raw_unaligned_native_width_out_of_bounds(gpu, w):
    """Native widths at an unaligned address go through the row gather with take_fixed_size's semantics: a null index past
    the values gives zeros, a valid one is the lowest row's "Out-of-bounds index"."""
    rng = np.random.default_rng(6500 + w)
    n, m = 300, 200
    col = random_column(rng, n, w)
    idx = rng.integers(0, n, m).astype(np.uint32)
    iv = rng.random(m) >= 0.2
    idx[5], iv[5] = n + 3, False
    idx[[77, 150]], iv[[77, 150]] = [n + 9, n], True
    ix = HostArray.from_numpy(abi.U32, idx, iv)
    with gpu._scope() as s:
        idd = s.upload(ix).descriptor()
        with pytest.raises(acu.ArrowError) as e:
            _raw(gpu, col, 1, 3, m, lambda a, o: gpu.check(gpu.lib.acu_take_fixed_size_binary(gpu.h, w, C.byref(a), C.byref(idd), abi.U32, 0,
                                                                                               C.byref(o))))
    assert (e.value.status, e.value.message, e.value.index) == (abi.ERR_PANIC_OUT_OF_BOUNDS, f"Out-of-bounds index {n + 9}", 77)
    idx[[77, 150]] = [1, 2]
    ix = HostArray.from_numpy(abi.U32, idx, iv)
    with gpu._scope() as s:
        idd = s.upload(ix).descriptor()
        got = _raw(gpu, col, 1, 3, m, lambda a, o: gpu.check(gpu.lib.acu_take_fixed_size_binary(gpu.h, w, C.byref(a), C.byref(idd), abi.U32, 0,
                                                                                                 C.byref(o))))
    same(got, of.take(col, idx, iv, True, abi.U32))


# ---- byte positions past 2^32 ------------------------------------------------------------------------------------------
def test_take_past_2_pow_32_bytes(gpu):
    """A 4.5 GB source and a 4.5 GB output of W = 4097 (the row gather): source and output byte positions pass 2^32. The
    source is a 16 MiB pattern repeated on the device, so every output byte is known on the host; the output is compared in
    32 MiB pieces, and its row hashes against the expected rows', to keep host memory small."""
    w = 4097
    n = (4_500_000_000 // w) + 1
    m = n
    rng = np.random.default_rng(11)
    pat = np.frombuffer(rng.bytes(1 << 24), np.uint8)
    plen = len(pat)
    src = gpu.malloc(n * w + 64)
    out = gpu.malloc(m * w + 64)
    obits = gpu.malloc(acu.bitmap_bytes(m) + 8)
    try:
        for off in range(0, n * w, plen):
            gpu.h2d(src + off, pat[:min(plen, n * w - off)])
        idx = rng.integers(0, n, m).astype(np.uint32)
        idx[:64] = np.arange(n - 64, n, dtype=np.uint32)  # the last source rows first: output positions < 2^32 read positions > 2^32
        ix = HostArray.from_numpy(abi.U32, idx)
        with gpu._scope() as s:
            idd = s.upload(ix).descriptor()
            a = abi.Array()
            a.values, a.len = src, n
            o = abi.ArrayOut(out, obits, 0, 0, 0)
            gpu.check(gpu.lib.acu_take_fixed_size_binary(gpu.h, w, C.byref(a), C.byref(idd), abi.U32, 0, C.byref(o)))
        assert o.len == m and not o.has_validity and m * w > 1 << 32 and n * w > 1 << 32
        rows_per_piece = (32 << 20) // w
        col = np.arange(w, dtype=np.int64)
        h_got, h_exp = [], []
        for r0 in range(0, m, rows_per_piece):
            r1 = min(r0 + rows_per_piece, m)
            got = gpu.d2h(out + r0 * w, (r1 - r0) * w).reshape(-1, w)
            exp = pat[(idx[r0:r1].astype(np.int64)[:, None] * w + col[None, :]) % plen]
            assert np.array_equal(got, exp), f"rows {r0}..{r1}"
            h_got.append(got.astype(np.uint64).sum(axis=1) * 31 + got[:, ::97].astype(np.uint64).sum(axis=1))
            h_exp.append(exp.astype(np.uint64).sum(axis=1) * 31 + exp[:, ::97].astype(np.uint64).sum(axis=1))
        assert np.array_equal(np.concatenate(h_got), np.concatenate(h_exp))
    finally:
        for p in (src, out, obits):
            gpu.free(p)


# ---- grid rounds ------------------------------------------------------------------------------------------------------
def _round_chunks(gpu, w):
    return gpu.lib.acu_device_sm_count(gpu.h) * FSB_PER_SM * FSB_THREADS * chunks_per_thread(w)


@pytest.mark.parametrize("w", [3, 20, 36])
def test_take_past_one_grid_round_and_lowest_error_row(gpu, w):
    rng = np.random.default_rng(7000 + w)
    m = int(_round_chunks(gpu, w) * 16 * 1.3) // w + 11
    n = 5000
    vals = rng.integers(0, 256, (n, w), dtype=np.uint8)
    col = of.column(vals, None)
    idx = rng.integers(0, n, m).astype(np.uint32)
    got = gpu.take(col, HostArray.from_numpy(abi.U32, idx))
    assert got.length == m and not of.has_buffer(got)
    assert np.array_equal(got.values, vals[idx])
    # failing rows in two rounds: the lower one is reported
    one_round_rows = _round_chunks(gpu, w) * 16 // w
    lo, hi = one_round_rows // 3, one_round_rows + one_round_rows // 7
    bad = idx.copy()
    bad[[lo, hi]] = n + 1
    with pytest.raises(acu.ArrowError) as e:
        gpu.take(col, HostArray.from_numpy(abi.U32, bad))
    assert e.value.index == lo and e.value.message == f"range start index {(n + 1) * w} out of range for slice of length {n * w}"


@pytest.mark.parametrize("w", [3, 20, 36])
def test_filter_past_one_grid_round(gpu, w):
    rng = np.random.default_rng(8000 + w)
    k = int(_round_chunks(gpu, w) * 16 * 1.3) // w + 5
    n = int(k / 0.7)
    vals = rng.integers(0, 256, (n, w), dtype=np.uint8)
    mask = rng.random(n) >= 0.2
    col = of.column(vals, mask)
    pred = rng.random(n) < 0.7
    got = gpu_filter(gpu, col, pred)
    assert np.array_equal(got.values, vals[pred])
    assert np.array_equal(of.valid_mask(got), mask[pred])


# ---- nesting and the record-batch calls ------------------------------------------------------------------------------
def test_struct_field(gpu):
    rng = np.random.default_rng(9000)
    f = random_column(rng, 100, 20)
    st = StructColumn([f, HostArray.from_numpy(abi.I64, rng.integers(0, 9, 100))], tg_nulls(rng.random(100) >= 0.1))
    pred = rng.random(100) < 0.5
    r = gpu_filter(gpu, st, pred)
    same(r.fields[0], oracle_filter(f, pred))
    idx = rng.integers(0, 100, 50).astype(np.int32)
    r = gpu.take(st, HostArray.from_numpy(abi.I32, idx))
    same(r.fields[0], of.take(f, idx, None, False, abi.I32))


def tg_nulls(mask):
    h = HostArray.from_list(abi.U8, [0 if v else None for v in mask])
    h.values = np.zeros(0, np.uint8)
    return h


@pytest.mark.parametrize("w", [0, 7, 20])
def test_list_child_step(gpu, w):
    rng = np.random.default_rng(9100 + w)
    child = random_column(rng, 60, w, null_p=0.0)
    child.nulls = HostArray(abi.U8, np.zeros(0, np.uint8), 60, acu.pack_bits(np.ones(60, bool)), 0, 0, 0)  # a NullBuffer without nulls
    offs = np.arange(0, 61, 3, dtype=np.int32)
    lst = ListColumn(offs, child, tg_nulls(np.ones(20, bool)))
    pred = np.zeros(20, bool)
    pred[[1, 4, 5]] = True
    r = gpu_filter(gpu, lst, pred)
    rows = np.concatenate([np.arange(3 * i, 3 * i + 3) for i in (1, 4, 5)])
    assert r.child.length == 9 and not of.has_buffer(r.child)  # MutableArrayData: every row, an empty NullBuffer dropped
    assert np.array_equal(r.child.values, child.values[rows])


@pytest.mark.parametrize("w,zeros", [(20, True), (16, False)])
def test_fixed_size_list_null_index(gpu, w, zeros):
    rng = np.random.default_rng(9200 + w)
    child = random_column(rng, 20, w, null_p=0.0)
    fsl = FixedSizeListColumn(2, child, tg_nulls(np.ones(10, bool)))
    ix = HostArray.from_list(abi.U32, [3, None, 1])
    ix.values[1] = 4
    r = gpu.take(fsl, ix)
    vals = r.child.values
    assert np.array_equal(vals[0:2], child.values[6:8]) and np.array_equal(vals[4:6], child.values[2:4])
    # take_value_indices_from_fixed_size_list appends nulls (value 0) for a null index: W = 16 gathers child row 0 under them
    assert (vals[2:4] == 0).all() if zeros else np.array_equal(vals[2:4], child.values[[0, 0]])


def test_dense_union_child(gpu):
    rng = np.random.default_rng(9300)
    a = random_column(rng, 6, 20)
    b = HostArray.from_numpy(abi.I32, np.arange(4, dtype=np.int32))
    u = UnionColumn(abi.UNION_DENSE, [0, 1], [a, b], [0, 1, 0, 0, 1, 0], [0, 0, 1, 2, 1, 5])
    r = gpu.take(u, HostArray.from_list(abi.U32, [5, 0, 2]))
    same(r.children[0], of.take(a, np.array([5, 0, 1]), None, False, abi.U32))


def test_run_end_filter_and_take_refusal(gpu):
    rng = np.random.default_rng(9400)
    vals = random_column(rng, 4, 20)
    ree = RunEndColumn(np.array([3, 5, 9, 10], np.int32), vals)
    pred = np.array([True, False, False, True, False, True, True, False, False, True])
    r = gpu.filter_run_end(ree, HostArray.bool_from_numpy(pred))
    assert list(r.run_ends) == [1, 2, 4, 5]
    assert r.values.length == 4 and np.array_equal(r.values.values, vals.values)
    assert np.array_equal(of.valid_mask(r.values), of.valid_mask(vals))
    with pytest.raises(acu.ArrowError) as e:
        gpu.take_run_end(ree, HostArray.from_list(abi.U32, [0, 4]))
    assert e.value.status == abi.ERR_NOT_YET_IMPLEMENTED


def test_record_batches(gpu):
    rng = np.random.default_rng(9500)
    n = 1000
    f = random_column(rng, n, 20)
    g = random_column(rng, n, 16)
    p = HostArray.from_numpy(abi.I64, rng.integers(0, 100, n), rng.random(n) >= 0.1)
    offs = np.arange(n + 1, dtype=np.int32)
    u = Utf8Column(offs, rng.integers(97, 123, n).astype(np.uint8), tg_nulls(rng.random(n) >= 0.1))
    pred = rng.random(n) < 0.4
    out = gpu.filter_record_batch([p, f, u, g], HostArray.bool_from_numpy(pred))
    same(out[1], oracle_filter(f, pred))
    same(out[3], oracle_filter(g, pred))
    assert out[0].to_list() == gpu.filter(p, HostArray.bool_from_numpy(pred)).to_list()
    idx = rng.integers(0, n, 300).astype(np.uint32)
    iv = rng.random(300) >= 0.1
    ix = HostArray.from_numpy(abi.U32, idx, iv)
    out = gpu.take_record_batch([f, p, g, u], ix)
    same(out[0], of.take(f, idx, iv, True, abi.U32))
    same(out[2], of.take(g, idx, iv, True, abi.U32))
    with pytest.raises(acu.ArrowError) as e:
        gpu.concat([f, f])
    assert e.value.status == abi.ERR_INVALID_ARGUMENT
