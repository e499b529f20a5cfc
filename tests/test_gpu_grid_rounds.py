"""The grid-stride kernels of boolean, nullif, the byte and view comparisons, concat, the filter slices and the view coalescing
primitives, run over more than one grid-stride round and compared with the oracle at the usual bar (value bits including those
under nulls, validity bits, null_count, NullBuffer presence, error status / text / index).

Every one of these kernels is launched with acu_grid(ctx, work, per_sm), which caps the grid at SMs x per_sm CTAs
(csrc/common.cuh). Below that cap each thread runs its loop body once, so the loop step, whatever a thread carries from one
round to the next (valid counts, first-error minima) and the partial last round only run at sizes past one round. The
rows_per_round helpers restate each launch shape from the SM count, and every test asserts that its size is at least 1.2
rounds of the kernel it names and not a multiple of 64, so the last word is partial and lies in a later round.

Where the oracle has no counterpart (the raw acu_bitmap_copy / acu_offsets_append entry points) a numpy restatement is the
reference. Inputs are built from random bytes, int16 draws and numpy cumsums: the largest cases have tens of millions of rows."""
import ctypes as C

import numpy as np
import pytest

import acu
from acu import _abi as abi
from acu import BOOL, HostArray, Utf8Column, ViewColumn, bitmap_bytes
from acu.coalesce_views import DeviceViewBackend
from oracle import OracleViewBackend
from test_gpu_parity import assert_same
from test_gpu_device_slices import same_bytes, sparse_mask

pytestmark = pytest.mark.gpu

CMP_OPS = [abi.EQ, abi.NEQ, abi.LT, abi.LT_EQ, abi.GT, abi.GT_EQ, abi.DISTINCT, abi.NOT_DISTINCT]
ALPHA = np.frombuffer(b"ab", dtype=np.uint8)
SCAN_ELEMS = 4096  # elements per k_scan_block CTA (csrc/bytes.cu)


# ---- launch shapes ---------------------------------------------------------------------------------------------------------
def sms(gpu):
    return gpu.lib.acu_device_sm_count(gpu.h)


def word_rows_per_round(gpu):
    """k_boolean (boolean.cu:103-104) and k_nullif (select.cu:199): acu_grid(words / 256, 16) CTAs of 256 threads, one 64-row
    word per thread."""
    return sms(gpu) * 16 * 256 * 64


def cmp_rows_per_round(gpu, rows_per_lane):
    """k_cmp_rows (rows_per_lane 4) and k_view_eq_inline (8) through cmp_grid (strcmp.cu:159-162, :178, :207, :233):
    SMs x 16 CTAs of 8 warps, rows_per_lane groups of 32 rows per warp."""
    return sms(gpu) * 16 * 8 * rows_per_lane * 32


def copy_words_per_round(gpu):
    """k_bitmap_copy / k_bitmap_fill (concat.cu:93, :107), k_offsets_append (concat.cu:117) and k_plan_slice_counts /
    k_plan_slices_emit (bytes.cu:1216): acu_grid(items / 256, 8) CTAs of 256 threads, one destination word (bitmaps), one
    offset entry or one mask word per thread."""
    return sms(gpu) * 8 * 256


def view_rows_per_round(gpu):
    """k_view_long_lens, _bytes_used, _fit, _rebase (one view per thread) and k_view_copy (one warp per 32 views)
    (views.cu:119-189): acu_grid(n / 256, 16) CTAs of 256 threads."""
    return sms(gpu) * 16 * 256


def sized(per_round, rounds=1.25, tail=37):
    """A size of about `rounds` rounds whose last 64-row word is partial."""
    n = int(rounds * per_round) // 64 * 64 + tail
    assert_rounds(n, per_round)
    return n


def assert_rounds(n, per_round):
    assert n >= 1.2 * per_round, f"{n} rows are {n / per_round:.2f} rounds of {per_round}"
    assert n % 64 != 0


# ---- builders ---------------------------------------------------------------------------------------------------------------
def bool_array(rng, n, with_validity, voff, noff):
    """A BooleanArray of n rows whose values start at bit `voff` and validity at bit `noff` of their buffers, drawn as random
    bytes (a quarter of the slots null); the bits around the array are random too."""
    values = rng.integers(0, 256, bitmap_bytes(n + voff) + 8, dtype=np.uint8)
    if not with_validity:
        return HostArray(BOOL, values, n, None, 0, voff, 0)
    size = bitmap_bytes(n + noff) + 8
    validity = rng.integers(0, 256, size, dtype=np.uint8) | rng.integers(0, 256, size, dtype=np.uint8)
    nc = n - int(np.unpackbits(validity, bitorder="little")[noff: noff + n].sum())
    return HostArray(BOOL, values, n, validity, noff, voff, nc)


# (values offset, validity offset) of the two operands: every bitmap at 0; every bitmap on a 64-row word past 0 (the
# word-aligned kernel with its `off >> 6` advance); a word-aligned operand beside one at odd bit offsets (the unaligned kernel)
OFFSETS = {"zero": ((0, 0), (0, 0)), "aligned": ((64, 128), (128, 64)), "mixed": ((64, 128), (3, 5))}


def utf8_nulls(n, mask, bit_offset, scalar=False):
    nulls = HostArray(abi.U8, np.zeros(0, np.uint8), n, None if mask is None else acu.pack_bits(mask, bit_offset),
                      bit_offset if mask is not None else 0, 0, 0 if mask is None else int(n - mask.sum()))
    nulls.is_scalar = scalar
    return nulls


def offsets_of(lens, odt):
    o = np.zeros(len(lens) + 1, dtype=odt)
    np.cumsum(lens, out=o[1:])
    return o


def tied_values(rng, n, odt, max_len=24):
    """Two value sets of n rows over a two-letter alphabet, as (offsets, bytes, lengths): b repeats a's bytes with a length
    change of -1 / 0 / +1 (new letters past a's end) and a new last letter in a third of the rows, so that ties run deep
    into the values, past the first 8-byte compare."""
    la = rng.integers(0, max_len + 1, n)
    oa = offsets_of(la, odt)
    da = ALPHA[rng.integers(0, 2, int(oa[-1]), dtype=np.uint8)]
    lb = np.clip(la + rng.integers(-1, 2, n), 0, max_len)
    ob = offsets_of(lb, odt)
    total = int(ob[-1])
    src = np.arange(total, dtype=np.int64) + np.repeat(oa[:-1].astype(np.int64) - ob[:-1], lb)
    inside = src < np.repeat(oa[1:].astype(np.int64), lb)
    db = np.where(inside, da[np.minimum(src, max(len(da) - 1, 0))], ALPHA[rng.integers(0, 2, total, dtype=np.uint8)])
    del src, inside
    flip = (lb > 0) & (rng.integers(0, 3, n) == 0)
    db[ob[1:][flip].astype(np.int64) - 1] = ALPHA[rng.integers(0, 2, int(flip.sum()), dtype=np.uint8)]
    pad = np.zeros(16, np.uint8)
    return (oa, np.concatenate([da, pad]), la), (ob, np.concatenate([db, pad]), lb)


def utf8_scalar(value, odt, null=False):
    data = np.concatenate([np.frombuffer(value, dtype=np.uint8), np.zeros(16, np.uint8)])
    return Utf8Column(np.array([0, 0 if null else len(value)], dtype=odt), data,
                      utf8_nulls(1, np.array([not null]), 0, scalar=True))


def view_column(rng, offs, data, lens, mask):
    """The values (offs, data, lens) as a view column: inline up to 12 bytes, longer ones out of line, the first half of
    the rows in data buffer 0 (the bytes as they are) and the second half in buffer 1 (the same bytes behind 7 others).
    Null slots carry garbage views of inline length."""
    n = len(lens)
    starts = offs[:-1].astype(np.int64)
    views = np.zeros((n, 16), dtype=np.uint8)
    views[:, :4] = lens.astype(np.uint32).view(np.uint8).reshape(n, 4)
    inline = lens <= 12
    for k in range(12):
        sel = (lens > k) & (inline if k >= 4 else True)
        views[sel, 4 + k] = data[starts[sel] + k]
    long_ = ~inline
    second = np.arange(n) >= n // 2
    views[long_, 8:12] = second[long_].astype(np.uint32).view(np.uint8).reshape(-1, 4)
    views[long_, 12:16] = np.where(second, starts + 7, starts)[long_].astype(np.uint32).view(np.uint8).reshape(-1, 4)
    if mask is not None:
        nulls = np.nonzero(~mask)[0]
        g = rng.integers(0, 256, (len(nulls), 16), dtype=np.uint8)
        g[:, 1:4] = 0
        g[:, 0] = rng.integers(0, 13, len(nulls))
        views[nulls] = g
    buffers = [data, np.concatenate([rng.integers(0, 256, 7, dtype=np.uint8), data])]
    return ViewColumn(views, buffers, utf8_nulls(n, mask, 0))


# ---- 1. boolean --------------------------------------------------------------------------------------------------------------
BINARY = ["and_", "or_", "and_not", "and_kleene", "or_kleene"]
# (a has validity, b has validity, offset class): every validity branch of the Kleene formulas (boolean.cu:40-49), every
# offset class; the other ops take one validity union case per offset class
KLEENE_CASES = [(False, False, "mixed"), (True, False, "aligned"), (False, True, "mixed"), (True, True, "aligned"),
                (True, True, "zero")]
PLAIN_CASES = [(True, True, "aligned"), (False, True, "mixed"), (True, False, "zero")]


@pytest.mark.parametrize("op", BINARY)
def test_boolean_binary_multi_round(gpu, oracle, op):
    n = sized(word_rows_per_round(gpu))
    rng = np.random.default_rng(100 + BINARY.index(op))
    for an, bn, cls in KLEENE_CASES if "kleene" in op else PLAIN_CASES:
        (avo, ano), (bvo, bno) = OFFSETS[cls]
        a, b = bool_array(rng, n, an, avo, ano), bool_array(rng, n, bn, bvo, bno)
        assert_same(getattr(gpu, op)(a, b), getattr(oracle, op)(a, b), f"{op} n={n} validity=({an},{bn}) offsets={cls}")


def test_boolean_unary_multi_round(gpu, oracle):
    n = sized(word_rows_per_round(gpu))
    rng = np.random.default_rng(110)
    for with_validity, cls in [(False, "zero"), (True, "aligned"), (True, "mixed")]:
        vo, no = OFFSETS[cls][1]
        a = bool_array(rng, n, with_validity, vo, no)
        for op in ("not_", "is_null", "is_not_null"):
            assert_same(getattr(gpu, op)(a), getattr(oracle, op)(a), f"{op} n={n} validity={with_validity} offsets={cls}")


# ---- 2. nullif ---------------------------------------------------------------------------------------------------------------
def test_nullif_multi_round(gpu, oracle):
    n = sized(word_rows_per_round(gpu))
    rng = np.random.default_rng(120)
    cases = [(False, False, "zero"), (True, False, "mixed"), (False, True, "aligned"), (True, True, "mixed"),
             (True, True, "aligned")]
    for ln, rn, cls in cases:
        (lvo, lno), (rvo, rno) = OFFSETS[cls]
        left, right = bool_array(rng, n, ln, lvo, lno), bool_array(rng, n, rn, rvo, rno)
        assert_same(gpu.nullif(left, right), oracle.nullif(left, right), f"nullif n={n} validity=({ln},{rn}) offsets={cls}")
    # right never Some(true) and left without nulls: the result has no nulls and drops its NullBuffer
    left, right = bool_array(rng, n, False, 3, 0), bool_array(rng, n, True, 64, 5)
    right.values[:] = 0
    got, exp = gpu.nullif(left, right), oracle.nullif(left, right)
    assert exp.validity is None
    assert_same(got, exp, f"nullif without nulls n={n}")


# ---- 3. cmp_bytes ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("odt", [np.int32, np.int64], ids=["utf8", "large_utf8"])
def test_cmp_bytes_multi_round(gpu, oracle, odt):
    n = sized(cmp_rows_per_round(gpu, 4))
    rng = np.random.default_rng(130 + np.dtype(odt).itemsize)
    (oa, da, _), (ob, db, _) = tied_values(rng, n, odt)
    a = Utf8Column(oa, da, utf8_nulls(n, sparse_mask(rng, n, 0.1), 3))
    b = Utf8Column(ob, db, utf8_nulls(n, sparse_mask(rng, n, 0.2), 6))
    scalars = [utf8_scalar(b"abbaabab", odt), utf8_scalar(b"ababbbabaabab", odt), utf8_scalar(b"", odt), utf8_scalar(b"", odt, null=True)]
    for op in CMP_OPS:
        assert_same(gpu.cmp_bytes(op, a, b), oracle.cmp_bytes(op, a, b), f"cmp_bytes op={op} n={n}")
        sc = scalars[op % len(scalars)]
        assert_same(gpu.cmp_bytes(op, a, sc), oracle.cmp_bytes(op, a, sc), f"cmp_bytes array/scalar op={op} n={n}")
        assert_same(gpu.cmp_bytes(op, sc, b), oracle.cmp_bytes(op, sc, b), f"cmp_bytes scalar/array op={op} n={n}")


# ---- 4. cmp_view -------------------------------------------------------------------------------------------------------------
def test_cmp_view_multi_round(gpu, oracle):
    n = sized(cmp_rows_per_round(gpu, 4))
    rng = np.random.default_rng(140)
    (oa, da, la), (ob, db, lb) = tied_values(rng, n, np.int64)
    a = view_column(rng, oa, da, la, sparse_mask(rng, n, 0.1))
    b = view_column(rng, ob, db, lb, sparse_mask(rng, n, 0.2))
    scalars = [b"", b"abba", b"abababbbabab", b"abababbbababa", b"abbaabababbabbbaab"]  # 0, 4, 12, 13 and 18 bytes
    for op in CMP_OPS:
        assert_same(gpu.cmp_view(op, a, b), oracle.cmp_view(op, a, b), f"cmp_view op={op} n={n}")
        for item in scalars:
            sc = ViewColumn.from_values([item], scalar=True)
            assert_same(gpu.cmp_view(op, a, sc), oracle.cmp_view(op, a, sc), f"cmp_view array/scalar op={op} {item!r}")
        sc = ViewColumn.from_values([scalars[op % len(scalars)]], scalar=True)
        assert_same(gpu.cmp_view(op, sc, b), oracle.cmp_view(op, sc, b), f"cmp_view scalar/array op={op}")


def test_view_eq_inline_multi_round(gpu, oracle):
    """== / != against a non-null scalar of at most 4 bytes (the eq_inline_scalar kernel), without validity, with validity and a
    cached null_count, and with validity and null_count = -1."""
    n = sized(cmp_rows_per_round(gpu, 8))
    rng = np.random.default_rng(150)
    lens = rng.integers(0, 7, n)
    offs = offsets_of(lens, np.int64)
    data = np.concatenate([ALPHA[rng.integers(0, 2, int(offs[-1]), dtype=np.uint8)], np.zeros(16, np.uint8)])
    mask = sparse_mask(rng, n, 0.15)
    for validity in ("none", "cached", "unknown"):
        col = view_column(rng, offs, data, lens, None if validity == "none" else mask)
        if validity == "unknown":
            col.nulls.null_count = -1
        for item in (b"ab", b"abba", b""):
            sc = ViewColumn.from_values([item], scalar=True)
            for op in (abi.EQ, abi.NEQ):
                got, exp = gpu.cmp_view(op, col, sc), oracle.cmp_view(op, col, sc)
                assert_same(got, exp, f"eq_inline op={op} {item!r} validity={validity}")
                assert_same(gpu.cmp_view(op, sc, col), exp, f"eq_inline scalar/array op={op} {item!r} validity={validity}")


# ---- 5. concat ---------------------------------------------------------------------------------------------------------------
def test_concat_bitmaps_multi_round(gpu, oracle):
    """The second and third inputs are each more than one round of k_bitmap_copy / k_bitmap_fill, and start mid-word
    because the first input's length is not a multiple of 64."""
    big = sized(copy_words_per_round(gpu) * 64)
    rng = np.random.default_rng(160)
    bools = [bool_array(rng, 100_013, True, 3, 5), bool_array(rng, big, False, 5, 0), bool_array(rng, big, True, 64, 7),
             bool_array(rng, 1001, False, 0, 0)]
    assert_same(gpu.concat(bools), oracle.concat(bools), "concat boolean")
    prims = []
    for n, null_p in [(70_001, 0.1), (big, None), (big, 0.3), (999, None)]:
        vals = rng.integers(-128, 128, n, dtype=np.int8)
        prims.append(HostArray.from_numpy(abi.I8, vals, None if null_p is None else sparse_mask(rng, n, null_p), bit_offset=1))
    assert_same(gpu.concat(prims), oracle.concat(prims), "concat int8")


@pytest.mark.parametrize("odt", [np.int32, np.int64], ids=["utf8", "large_utf8"])
def test_concat_utf8_multi_round(gpu, oracle, odt):
    """Inputs of more than one round of k_offsets_append each, two of them slices with offsets[0] != 0."""
    n = sized(copy_words_per_round(gpu))
    rng = np.random.default_rng(170 + np.dtype(odt).itemsize)
    cols = []
    for k in (0, 1234, 77):
        total = n + k
        lens = rng.integers(0, 20, total)
        offs = offsets_of(lens, odt)
        data = np.concatenate([rng.integers(97, 123, int(offs[-1]), dtype=np.uint8), np.zeros(16, np.uint8)])
        full = utf8_nulls(total, sparse_mask(rng, total, 0.1), 5)
        col = Utf8Column(offs[k:], data, full.slice(k, n) if k else full)
        if k:
            assert int(col.offsets[0]) != 0
        cols.append(col)
    same_bytes(to_triple(gpu.concat(cols)), to_triple(oracle.concat(cols)), f"concat {np.dtype(odt).name} offsets")


def to_triple(col):
    return col.offsets, col.data[: int(col.offsets[-1])], col.nulls


def offsets_append(gpu, src, first, count, base, odt):
    """acu_offsets_append of src[first .. first + count] onto a fresh destination -> (status, message, index, dst, begin, end)."""
    ob = np.dtype(odt).itemsize
    d_src, d_dst = gpu.malloc(src.nbytes + 16), gpu.malloc((count + 1) * ob + 16)
    try:
        gpu.h2d(d_src, src)
        begin, end = C.c_int64(0), C.c_int64(0)
        st = gpu.lib.acu_offsets_append(gpu.h, ob, d_src, first, count, base, d_dst, 0, C.byref(begin), C.byref(end))
        err = gpu.lib.acu_last_error(gpu.h).contents
        msg, idx = (err.message.decode(), err.index) if st != abi.OK else ("", -1)
        return st, msg, idx, gpu.d2h(d_dst, (count + 1) * ob, odt), begin.value, end.value
    finally:
        gpu.free(d_src)
        gpu.free(d_dst)


def test_offsets_append_multi_round(gpu):
    stride = copy_words_per_round(gpu)
    count = sized(stride) - 1
    assert count + 1 >= 1.2 * stride
    # a plain rebase of a source that starts at first = 17, LargeUtf8 offsets
    rng = np.random.default_rng(180)
    src = offsets_of(rng.integers(0, 50, count + 40), np.int64)
    st, _, _, dst, begin, end = offsets_append(gpu, src, 17, count, 1 << 40, np.int64)
    assert st == abi.OK and (begin, end) == (int(src[17]), int(src[17 + count]))
    assert np.array_equal(dst, (1 << 40) + src[17: 17 + count + 1] - src[17])
    # Utf8 offsets that pass INT32_MAX at entry j0: src[j] = 3j, base = INT32_MAX + 1 - 3 j0
    src = (3 * np.arange(count + 1, dtype=np.int64)).astype(np.int32)
    j = np.arange(count + 1, dtype=np.int64)
    for j0 in (stride + 4321,  # the first overflowing entry lies in the second round
               1000):          # ... in the first round, in a thread that runs a second round, where the entries overflow too
        assert j0 + stride <= count or j0 >= stride
        base = 2**31 - 3 * j0
        st, msg, idx, dst, begin, end = offsets_append(gpu, src, 0, count, base, np.int32)
        total = base + 3 * count
        assert st == abi.ERR_OFFSET_OVERFLOW and idx == j0 and msg == f"Offset overflow error: {total}", (st, msg, idx, j0)
        assert np.array_equal(dst, (base + 3 * j).astype(np.int32)), "every entry is written, wrapped to 32 bits"


def test_bitmap_copy_multi_round(gpu):
    n = sized(copy_words_per_round(gpu) * 64)
    rng = np.random.default_rng(190)
    nbytes = bitmap_bytes(n + 400) + 8
    src_bytes = rng.integers(0, 256, nbytes, dtype=np.uint8)
    src_bits = np.unpackbits(src_bytes, bitorder="little").astype(bool)
    d_src, d_dst = gpu.malloc(nbytes), gpu.malloc(nbytes)
    try:
        gpu.h2d(d_src, src_bytes)
        for soff, doff in [(int(rng.integers(1, 200)), int(rng.integers(1, 200))), (37, 128), (64, 101)]:
            base = rng.integers(0, 256, nbytes, dtype=np.uint8)
            gpu.h2d(d_dst, base)
            cnt = C.c_int64(0)
            gpu.check(gpu.lib.acu_bitmap_copy(gpu.h, d_src, soff, d_dst, doff, n, C.byref(cnt)))
            got = np.unpackbits(gpu.d2h(d_dst, nbytes), bitorder="little").astype(bool)
            exp = np.unpackbits(base, bitorder="little").astype(bool)
            exp[doff: doff + n] = src_bits[soff: soff + n]
            bad = np.nonzero(got != exp)[0]
            assert len(bad) == 0, f"bitmap_copy soff={soff} doff={doff}: bits differ at {bad[:8]}"
            assert cnt.value == int(src_bits[soff: soff + n].sum())
    finally:
        gpu.free(d_src)
        gpu.free(d_dst)


# ---- 6. filter slices --------------------------------------------------------------------------------------------------------
def run_bools(rng, n, p, period=200):
    """Alternating clear / set runs of geometric lengths with mean (1 - p) x period and p x period: runs that cross words."""
    k = 2 * n // period + 64
    lens = np.empty(2 * k, dtype=np.int64)
    lens[0::2] = rng.geometric(1.0 / max((1 - p) * period, 1.0), k)
    lens[1::2] = rng.geometric(1.0 / max(p * period, 1.0), k)
    while lens.sum() < n:
        lens *= 2
    return np.repeat(np.tile(np.array([False, True]), k), lens)[:n]


def slice_pairs(gpu, oracle, pred):
    dp = gpu.upload(pred)
    plan, out = C.c_void_p(), None
    try:
        pd = dp.descriptor()
        gpu.check(gpu.lib.acu_filter_plan_create(gpu.h, C.byref(pd), C.byref(plan)))
        cnt = C.c_int64(0)
        gpu.check(gpu.lib.acu_filter_plan_slices(gpu.h, plan, None, 0, C.byref(cnt)))
        out = gpu.malloc(cnt.value * 16 + 16)
        gpu.check(gpu.lib.acu_filter_plan_slices(gpu.h, plan, out, cnt.value, C.byref(cnt)))
        got = gpu.d2h(out, cnt.value * 16, np.uint64).reshape(-1, 2)
    finally:
        gpu.free(out)
        if plan:
            gpu.lib.acu_filter_plan_destroy(gpu.h, plan)
        dp.free()
    lib = oracle.lib
    lib.orc_filter_slices.restype = C.c_int64
    lib.orc_filter_slices.argtypes = [C.POINTER(abi.Array), C.c_void_p, C.c_int64]
    hd = acu.host_descriptor(pred)
    cap = pred.length // 2 + 2
    pairs = np.zeros(2 * cap, dtype=np.uint64)
    k = lib.orc_filter_slices(C.byref(hd), pairs.ctypes.data, cap)
    return got, pairs[: 2 * k].reshape(-1, 2)


@pytest.mark.parametrize("p", [0.02, 0.5, 0.98])
def test_filter_slices_multi_round(gpu, oracle, p):
    per_round = copy_words_per_round(gpu) * 64
    n = sized(per_round)
    rng = np.random.default_rng(200 + int(p * 100))
    bools = run_bools(rng, n, p)
    bools[per_round - 100: per_round + 100] = True  # one run across the round boundary
    if p == 0.5:
        pred = HostArray.bool_from_numpy(bools)
    else:
        pred = HostArray.bool_from_numpy(bools, sparse_mask(rng, n, 0.02), bit_offset=3 if p < 0.5 else 64, mask_offset=7)
    got, exp = slice_pairs(gpu, oracle, pred)
    assert len(exp) > 1000
    assert got.shape == exp.shape, f"p={p}: {len(got)} slices vs {len(exp)}"
    bad = np.nonzero((got != exp).any(axis=1))[0]
    assert len(bad) == 0, f"p={p}: slices differ at {bad[:8]}: {got[bad[:4]]} vs {exp[bad[:4]]}"


# ---- 7. view coalescing primitives -------------------------------------------------------------------------------------------
def coalesce_source(rng, n, long_p, big_p, n_buffers=2):
    """n views, mostly inline; a fraction long_p out of line (13-99 bytes), big_p of 256-699 bytes. The long values lie in
    n_buffers data buffers, in row order, with 0-15 bytes of padding in front of each so their 16-byte phases vary."""
    lens = rng.integers(0, 13, n).astype(np.int64)
    draw = rng.integers(0, 100_000, n, dtype=np.int32)
    is_big = draw < int(big_p * 100_000)
    is_long = draw < int((big_p + long_p) * 100_000)
    lens[is_long] = rng.integers(13, 100, int(is_long.sum()))
    lens[is_big] = rng.integers(256, 700, int(is_big.sum()))
    views = rng.integers(0, 256, (n, 16), dtype=np.uint8)  # inline bytes (and the bytes past each length) are arbitrary
    views[:, :4] = lens.astype(np.uint32).view(np.uint8).reshape(n, 4)
    rows = np.nonzero(is_long)[0]
    buf_of = (np.arange(len(rows)) * n_buffers) // max(len(rows), 1)
    buffers = []
    for bi in range(n_buffers):
        r = rows[buf_of == bi]
        ln = lens[r]
        gap = rng.integers(0, 16, len(r))
        off = np.cumsum(gap + ln) - ln
        buf = rng.integers(97, 123, int(off[-1] + ln[-1]) if len(r) else 0, dtype=np.uint8)
        views[r, 4:8] = buf[off[:, None] + np.arange(4)]
        views[r, 8:12] = np.full(len(r), bi, dtype=np.uint32).view(np.uint8).reshape(-1, 4)
        views[r, 12:16] = off.astype(np.uint32).view(np.uint8).reshape(-1, 4)
        buffers.append(buf)
    return ViewColumn(views, buffers, utf8_nulls(n, None, 0)), lens, is_long


def view_fit_expected(lens, offset, remaining):
    """First view i >= offset with remaining - (long bytes of [offset, i)) < len(i) (coalesce/byte_view.rs:259-271)."""
    ln = lens[offset:]
    longs = np.where(ln > 12, ln, 0)
    before = np.cumsum(longs) - longs
    fail = np.nonzero(remaining - before < ln)[0]
    return (int(fail[0]), int(before[fail[0]])) if len(fail) else (len(ln), int(longs.sum()))


def copy_strings_both(gpu, be_g, be_o, dg, do, n, dst_len, cap):
    """copy_strings of views [0, n) into a destination of `cap` bytes holding dst_len, on both backends: a 0xEE-filled device
    destination (so bytes the kernel misses show) against the oracle's -> (out views, destination bytes) of each."""
    pattern = np.full(cap + 16, 0xEE, dtype=np.uint8)
    d_dst, d_out = gpu.malloc(cap + 16), gpu.malloc(16 * n + 16)
    try:
        gpu.h2d(d_dst, pattern)
        assert d_dst % 16 == 0 and all(p % 16 == 0 for p, _, _ in dg["buffers"])
        nb_g = be_g.copy_strings(dg, 0, n, 3, d_dst, dst_len, cap, d_out, 0)
        got = (gpu.d2h(d_out, 16 * n), gpu.d2h(d_dst, cap))
    finally:
        gpu.free(d_dst)
        gpu.free(d_out)
    o_dst, o_out = pattern.copy(), np.zeros(16 * n + 16, dtype=np.uint8)
    nb_o = be_o.copy_strings(do, 0, n, 3, o_dst, dst_len, cap, o_out, 0)
    assert nb_g == nb_o
    return got, (o_out[: 16 * n], o_dst[:cap]), nb_o


def assert_same_views(got, exp, what):
    (gv, gd), (ev, ed) = got, exp
    bad = np.nonzero((gv.reshape(-1, 16) != ev.reshape(-1, 16)).any(axis=1))[0]
    assert len(bad) == 0, f"{what}: views differ at {bad[:8]}"
    bad = np.nonzero(gd != ed)[0]
    assert len(bad) == 0, f"{what}: destination bytes differ at {bad[:8]}"


def test_view_primitives_multi_round(gpu, oracle):
    per_round = view_rows_per_round(gpu)
    n = sized(per_round)
    rng = np.random.default_rng(210)
    col, lens, is_long = coalesce_source(rng, n, 0.2, 0.01)
    be_g, be_o = DeviceViewBackend(gpu), OracleViewBackend(oracle)
    dg, do = be_g.upload(col), be_o.upload(col)
    try:
        longs = np.where(is_long, lens, 0)
        assert be_g.bytes_used(dg) == be_o.bytes_used(do) == int(longs.sum())
        incl = np.cumsum(longs)
        t = int(np.nonzero(is_long[per_round + 1000:])[0][0]) + per_round + 1000  # a long view in the second round
        for offset, remaining, first in [(0, int(incl[t]) - 1, t),      # view t is the first that does not fit
                                         (5, int(incl[t] - incl[4]) - 1, t - 5),
                                         (0, 10**12, n),                # every view fits
                                         (0, int(lens[0]) - 1, 0)]:     # view 0 does not fit
            got, exp = be_g.fit(dg, offset, n - offset, remaining), be_o.fit(do, offset, n - offset, remaining)
            assert got == exp == view_fit_expected(lens, offset, remaining), (offset, remaining, got, exp)
            assert got[0] == first
        # the 128-bit body path runs for values of >= 256 bytes whose source and destination share a 16-byte phase; the
        # destination position of view i is dst_len + (long bytes before i), its source the view's offset in its buffer
        off = np.frombuffer(col.views[:, 12:16].tobytes(), dtype=np.uint32).astype(np.int64)
        for dst_len in (0, 5, 16 * 1001 + 9):
            same_phase = ((off - (dst_len + incl - longs)) % 16 == 0) & (lens >= 256)
            assert same_phase.sum() > 50 and ((lens >= 256) & ~same_phase).sum() > 50
            cap = dst_len + int(incl[-1]) + 100
            got, exp, nb = copy_strings_both(gpu, be_g, be_o, dg, do, n, dst_len, cap)
            assert nb == int(incl[-1])
            assert_same_views(got, exp, f"copy_strings dst_len={dst_len}")
        # rebase
        d_out = gpu.malloc(16 * n + 16)
        try:
            be_g.rebase(dg, 0, n, 7, d_out, 0)
            got = gpu.d2h(d_out, 16 * n)
        finally:
            gpu.free(d_out)
        exp = np.zeros(16 * n + 16, dtype=np.uint8)
        be_o.rebase(do, 0, n, 7, exp, 0)
        assert np.array_equal(got, exp[: 16 * n]), "rebase"
    finally:
        be_g.release_source(dg)


def test_view_fit_and_copy_three_scan_levels(gpu, oracle):
    """More than 4096^2 views: the inclusive scan of the long lengths behind fit and copy_strings runs its third level."""
    n = SCAN_ELEMS * SCAN_ELEMS + 5 * SCAN_ELEMS + 1234
    assert -(-n // SCAN_ELEMS) > SCAN_ELEMS, "the second scan level has more than one block, so a third one runs"
    rng = np.random.default_rng(220)
    col, lens, is_long = coalesce_source(rng, n, 0.001, 0.0001, n_buffers=3)
    be_g, be_o = DeviceViewBackend(gpu), OracleViewBackend(oracle)
    dg, do = be_g.upload(col), be_o.upload(col)
    try:
        longs = np.where(is_long, lens, 0)
        incl = np.cumsum(longs)
        t = int(np.nonzero(is_long[SCAN_ELEMS * SCAN_ELEMS + 100:])[0][0]) + SCAN_ELEMS * SCAN_ELEMS + 100
        for remaining, first in [(int(incl[t]) - 1, t), (10**12, n)]:
            got, exp = be_g.fit(dg, 0, n, remaining), be_o.fit(do, 0, n, remaining)
            assert got == exp == (first, int(incl[first - 1])), (remaining, got, exp)
        got, exp, nb = copy_strings_both(gpu, be_g, be_o, dg, do, n, 3, int(incl[-1]) + 64)
        assert nb == int(incl[-1])
        assert_same_views(got, exp, "copy_strings past 4096^2 views")
    finally:
        be_g.release_source(dg)
