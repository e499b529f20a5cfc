"""filter / take of List, LargeList and FixedSizeList columns on the device against tests/oracle_filter_take.py, bit for bit:
offsets, child values (the bytes under null rows included) and NullBuffer presence at every level."""
import numpy as np
import pytest

import acu
from acu import BOOL, DecimalArray, FixedSizeListColumn, HostArray, ListColumn, Utf8Column, ViewColumn
from acu import _abi as abi

import oracle_filter_take as oft
from oracle_filter_take import nulls_of

pytestmark = pytest.mark.gpu

INDEX_DTYPES = [abi.I8, abi.U8, abi.I16, abi.U16, abi.I32, abi.U32, abi.I64, abi.U64]


def child_of(kind, n, rng, null_p=0.2):
    mask = rng.random(n) >= null_p
    if kind == "i8":
        return HostArray.from_numpy(abi.I8, rng.integers(-128, 128, n), mask)
    if kind == "i32":
        return HostArray.from_numpy(abi.I32, rng.integers(-2**31, 2**31, n), mask)
    if kind == "i64":
        return HostArray.from_numpy(abi.I64, rng.integers(-2**62, 2**62, n), mask)
    if kind == "f64":
        return HostArray.from_numpy(abi.F64, rng.random(n) * 2e6 - 1e6, mask)
    if kind == "bool":
        return HostArray.bool_from_numpy(rng.random(n) < 0.5, mask, bit_offset=3, mask_offset=5)
    if kind == "dec128":
        return DecimalArray.from_int64(16, 38, 2, rng.integers(-2**62, 2**62, n), mask)
    if kind == "view":
        items = [bytes(rng.integers(97, 123, rng.integers(0, 30)).astype(np.uint8)) if m else None for m in mask]
        return ViewColumn.from_values(items, garbage_under_nulls=[np.arange(16, dtype=np.uint8)])
    if kind in ("utf8", "lbin"):  # bytes under null rows too
        lens = rng.integers(0, 12, n)
        offs = np.zeros(n + 1, dtype=np.int32 if kind == "utf8" else np.int64)
        offs[1:] = np.cumsum(lens)
        data = rng.integers(0, 256, int(offs[-1]) + 1).astype(np.uint8)
        return Utf8Column(offs, data, nulls_of(mask))
    raise ValueError(kind)


def list_of(child, rng, large=False, rows=None, null_p=0.2, max_len=6, base=0, bit_offset=0, lens=None):
    """A list over `child` whose offsets start at `base` (a slice) and cover at most the child."""
    if lens is None:
        lens = []
        pos = base
        while len(lens) < (rows if rows is not None else 10**9):
            ln = int(rng.integers(0, max_len + 1))
            if pos + ln > child.length:
                if rows is None:
                    break
                ln = 0
            lens.append(ln)
            pos += ln
    offs = np.zeros(len(lens) + 1, dtype=np.int64 if large else np.int32)
    offs[0] = base
    offs[1:] = base + np.cumsum(lens)
    mask = rng.random(len(lens)) >= null_p
    return ListColumn(offs, child, nulls_of(mask, bit_offset))


def fsl_of(child, size, rng, null_p=0.2, bit_offset=0):
    rows = child.length // size if size else 7
    mask = rng.random(rows) >= null_p
    return FixedSizeListColumn(size, child, nulls_of(mask, bit_offset))


def rand_pred(rng, n, p=0.5, null_p=0.1):
    return HostArray.bool_from_numpy(rng.random(n) < p, rng.random(n) >= null_p)


def rand_idx(rng, n_src, m, dtype=abi.U32, null_p=0.1, oob_under_nulls=True):
    vals = rng.integers(0, max(n_src, 1), m)
    mask = rng.random(m) >= null_p
    if oob_under_nulls:
        vals = np.where(mask, vals, n_src + 5)
    if n_src == 0:
        mask[:] = False
    vals = np.minimum(vals, min(int(np.iinfo(acu.NP_DTYPES[dtype]).max), 2**62))
    return HostArray.from_numpy(dtype, vals, mask)


def check_filter(gpu, col, pred):
    got = gpu.filter_list(col, pred)
    exp = oft.filter(col, oft.filter_mask(pred))
    assert oft.describe(got) == oft.describe(exp)
    return got


def check_take(gpu, col, idx, check_bounds=False):
    got = gpu.take_list(col, idx, check_bounds)
    exp = oft.take_host(col, idx, check_bounds)
    assert oft.describe(got) == oft.describe(exp)
    return got


def check_error(fn, efn):
    with pytest.raises(acu.ArrowError) as g:
        fn()
    with pytest.raises(oft.OracleError) as e:
        efn()
    assert (g.value.status, g.value.message) == (e.value.status, e.value.message)
    assert g.value.index == e.value.index
    return g.value


CHILDREN = ["i8", "i64", "f64", "dec128", "view", "bool", "utf8", "lbin"]


@pytest.mark.parametrize("kind", ["list", "large", "fsl"])
@pytest.mark.parametrize("child", CHILDREN)
def test_flat_children(gpu, kind, child):
    rng = np.random.default_rng(10 * CHILDREN.index(child) + len(kind))
    c = child_of(child, 3000, rng)
    if kind == "fsl":
        col = fsl_of(c, 3, rng, bit_offset=5)
    else:
        col = list_of(c, rng, large=kind == "large", base=7, bit_offset=3)
    n = col.length
    for p in (0.0, 0.05, 0.5, 1.0):
        check_filter(gpu, col, rand_pred(rng, n, p, null_p=0.0 if p == 1.0 else 0.1))
    check_filter(gpu, col, rand_pred(rng, n // 2, 0.5))  # a predicate shorter than the list
    for dt in (abi.U32, abi.I64):
        check_take(gpu, col, rand_idx(rng, n, 700, dt))
    check_take(gpu, col, rand_idx(rng, n, 300, abi.U64, null_p=0.0))


@pytest.mark.parametrize("dt", INDEX_DTYPES)
def test_index_dtypes(gpu, dt):
    rng = np.random.default_rng(int(dt))
    col = list_of(child_of("i64", 500, rng), rng, base=3)
    check_take(gpu, col, rand_idx(rng, min(col.length, 100), 200, dt))


def nested_cases(rng):
    utf8 = child_of("utf8", 4000, rng)
    inner = list_of(utf8, rng, rows=None, max_len=4, base=2, bit_offset=1)
    yield "List<List<Utf8>>", list_of(inner, rng, max_len=4, base=1, bit_offset=6)
    fsl = fsl_of(child_of("i32", 3 * 1200, rng), 3, rng)
    yield "List<FixedSizeList<Int32,3>>", list_of(fsl, rng, large=True, max_len=5, base=4)
    li = list_of(child_of("i64", 5000, rng), rng, rows=600, max_len=4)
    yield "FixedSizeList<List<Int64>,2>", fsl_of(li, 2, rng, bit_offset=2)
    inner3 = list_of(list_of(child_of("lbin", 6000, rng), rng, large=True, max_len=3), rng, max_len=3)
    yield "List<List<List<LargeBinary>>>", list_of(inner3, rng, max_len=3)


def test_nested(gpu):
    rng = np.random.default_rng(7)
    for name, col in nested_cases(rng):
        n = col.length
        for p in (0.0, 0.3, 1.0):
            check_filter(gpu, col, rand_pred(rng, n, p, null_p=0.0 if p == 1.0 else 0.1))
        check_take(gpu, col, rand_idx(rng, n, 400, abi.U32))
        check_take(gpu, col, rand_idx(rng, n, 400, abi.I64, null_p=0.0))


def test_null_lists_over_ranges(gpu):
    """Null lists over non-empty ranges: filter keeps their ranges, take empties them; child nulls over non-empty bytes."""
    rng = np.random.default_rng(3)
    c = child_of("utf8", 200, rng, null_p=0.5)
    col = list_of(c, rng, null_p=0.5, lens=[3] * 60)
    got = check_filter(gpu, col, HostArray.bool_from_numpy(np.ones(60, bool) & (np.arange(60) % 3 != 0)))
    assert got.offsets[-1] == 40 * 3
    got = check_take(gpu, col, HostArray.from_numpy(abi.U32, np.arange(60)[::-1]))
    assert (np.diff(got.offsets)[~got.nulls.valid_mask()] == 0).all()


def test_empty_and_all_null(gpu):
    rng = np.random.default_rng(4)
    c = child_of("i64", 50, rng)
    empty = ListColumn(np.zeros(1, np.int32), c, nulls_of([]))
    check_filter(gpu, empty, HostArray.bool_from_numpy(np.zeros(0, bool)))
    check_take(gpu, empty, HostArray.from_numpy(abi.U32, np.zeros(0, np.uint32)))
    zero_len = list_of(c, rng, lens=[0] * 40)
    check_filter(gpu, zero_len, rand_pred(rng, 40))
    check_take(gpu, zero_len, rand_idx(rng, 40, 30))
    all_null = list_of(c, rng, null_p=1.0, lens=[1] * 40)
    check_filter(gpu, all_null, rand_pred(rng, 40))
    check_take(gpu, all_null, rand_idx(rng, 40, 30))
    check_take(gpu, all_null, HostArray.from_numpy(abi.U32, np.arange(40)))
    fsl0 = FixedSizeListColumn(0, c.slice(0, 0), nulls_of(rng.random(9) > 0.3))
    check_filter(gpu, fsl0, rand_pred(rng, 9))
    check_take(gpu, fsl0, rand_idx(rng, 9, 5))


def test_force_validity_all_strategy(gpu):
    """A NullBuffer without nulls: kept by the ALL strategy (a slice), dropped otherwise."""
    rng = np.random.default_rng(5)
    c = child_of("i64", 300, rng, null_p=0.0)
    col = ListColumn(np.arange(0, 301, 3, dtype=np.int32), c, nulls_of(np.ones(100, bool), force=True))
    got = check_filter(gpu, col, HostArray.bool_from_numpy(np.ones(100, bool)))
    assert got.nulls.validity is not None
    got = check_filter(gpu, col, HostArray.bool_from_numpy(np.arange(100) % 2 == 0))
    assert got.nulls.validity is None
    check_take(gpu, col, HostArray.from_numpy(abi.U32, np.arange(100), np.ones(100, bool)))


def test_errors(gpu):
    rng = np.random.default_rng(6)
    c = child_of("i32", 8, rng, null_p=0.0)
    col = ListColumn(np.array([0, 3, 6, 8], np.int32), c, nulls_of([True, True, True]))
    pred = HostArray.bool_from_numpy(np.ones(5, bool))
    check_error(lambda: gpu.filter_list(col, pred), lambda: oft.filter(col, oft.filter_mask(pred)))
    for bad in (1000, 3):
        idx = HostArray.from_numpy(abi.U32, [0, bad])
        e = check_error(lambda: gpu.take_list(col, idx), lambda: oft.take_host(col, idx))
        assert e.message == f"index out of bounds: the len is 4 but the index is {1000 if bad == 1000 else 4}"
        check_error(lambda: gpu.take_list(col, idx, True), lambda: oft.take_host(col, idx, True))
    with_nulls = ListColumn(col.offsets, c, nulls_of([True, False, True]))
    idx = HostArray.from_numpy(abi.I64, [2, 0, 7])
    e = check_error(lambda: gpu.take_list(with_nulls, idx), lambda: oft.take_host(with_nulls, idx))
    assert e.message == "assertion failed: idx < self.bit_len"
    # out-of-bounds values under null indices are never read
    idx = HostArray.from_numpy(abi.U32, [2, 99, 0], [True, False, True])
    check_take(gpu, with_nulls, idx)
    check_take(gpu, col, idx)


def test_skewed_row(gpu):
    """One row of 1e6 children among empty rows, and row counts past one grid-stride round."""
    rng = np.random.default_rng(8)
    n_child = 1_000_000
    c = HostArray.from_numpy(abi.I64, rng.integers(-2**62, 2**62, n_child + 5), rng.random(n_child + 5) >= 0.01)
    lens = np.zeros(200_001, np.int64)
    lens[123_457] = n_child
    col = list_of(c, rng, lens=list(lens), base=5, null_p=0.0)
    pred = HostArray.bool_from_numpy(rng.random(len(lens)) < 0.5)
    pred.values = acu.pack_bits(np.asarray(pred.value_array()) | (np.arange(len(lens)) == 123_457))
    got = gpu.filter_list(col, pred)
    exp = oft.filter(col, oft.filter_mask(pred))
    assert oft.describe(got) == oft.describe(exp)
    idx = HostArray.from_numpy(abi.U32, np.array([123_457, 0, 123_457, 17], np.uint32))
    check_take(gpu, col, idx)


def test_many_rows(gpu):
    rng = np.random.default_rng(9)
    c = HostArray.from_numpy(abi.I32, rng.integers(-2**31, 2**31, 3_000_000), rng.random(3_000_000) >= 0.1)
    col = list_of(c, rng, max_len=4, null_p=0.1)
    n = col.length
    pred = rand_pred(rng, n, 0.3)
    got = gpu.filter_list(col, pred)
    mask = oft.filter_mask(pred)
    rows = np.nonzero(mask)[0]
    lens = np.diff(col.offsets)[rows]
    assert np.array_equal(np.diff(got.offsets), lens)
    starts = col.offsets[rows]
    exp_child = np.concatenate([np.arange(s, s + ln) for s, ln in zip(starts[:2000], lens[:2000])])
    assert np.array_equal(got.child.value_array()[:len(exp_child)], c.value_array()[exp_child])
    idx = HostArray.from_numpy(abi.U64, rng.integers(0, n, 500_000))
    got = gpu.take_list(col, idx)
    iv = idx.value_array()
    lv = col.nulls.valid_mask()[iv]
    lens = np.where(lv, np.diff(col.offsets)[iv], 0)
    assert np.array_equal(np.diff(got.offsets), lens)
    exp_child = np.concatenate([np.arange(col.offsets[i], col.offsets[i + 1]) for i, v in zip(iv[:3000], lv[:3000]) if v])
    assert np.array_equal(got.child.value_array()[:len(exp_child)], c.value_array()[exp_child])


def test_list_offset_overflow(gpu):
    """One i32 list-offset overflow: the unwrap panic at the first output row past i32::MAX (raised by the offsets pass,
    before any child is allocated)."""
    c = HostArray.from_numpy(abi.I8, np.zeros(1 << 20, np.int8))
    col = ListColumn(np.array([0, 1 << 20], np.int32), c, nulls_of([True]))
    idx = HostArray.from_numpy(abi.U32, np.zeros(2049, np.uint32))
    with pytest.raises(acu.ArrowError) as e:
        gpu.take_list(col, idx)
    assert e.value.status == abi.ERR_PANIC_OUT_OF_BOUNDS and e.value.message == oft.UNWRAP_NONE
    assert e.value.index == 2047  # 2048 rows of 2^20 children end past i32::MAX


def test_child_byte_overflow(gpu):
    """One child byte overflow: try_extend_offsets' InvalidArgumentError, which comes before the list's own panic."""
    big = 1 << 21
    child = Utf8Column(np.array([0, big], np.int32), np.zeros(big, np.uint8), nulls_of([True]))
    col = ListColumn(np.array([0, 1], np.int32), child, nulls_of([True]))
    idx = HostArray.from_numpy(abi.U32, np.zeros(1025, np.uint32))
    with pytest.raises(acu.ArrowError) as e:
        gpu.take_list(col, idx)
    assert e.value.status == abi.ERR_INVALID_ARGUMENT and e.value.message == "Invalid argument error: " + oft.EXTEND_OVERFLOW
    assert e.value.index == 1023  # 1024 strings of 2^21 bytes end past i32::MAX


@pytest.mark.parametrize("case", __import__("list_util").golden_cases(), ids=lambda c: c["name"])
def test_golden(gpu, case):
    from list_util import check, run_case
    check(case, lambda: run_case(case, gpu.filter_list, gpu.take_list), acu.ArrowError)


def test_fixed_size_list_oob_child_first(gpu):
    """take_fixed_size_list takes the child before it reads the list's validity: a valid out-of-bounds index is the child
    take's panic, and take_bits' only when index * size wraps back into the child."""
    c = HostArray.from_numpy(abi.I32, np.arange(9))
    col = FixedSizeListColumn(3, c, nulls_of([True, False, True]))
    idx = HostArray.from_numpy(abi.U32, [0, 5])
    e = check_error(lambda: gpu.take_list(col, idx), lambda: oft.take_host(col, idx))
    assert e.message == "Out-of-bounds index 15"
    idx = HostArray.from_numpy(abi.U32, [0, 1431655766])  # * 3 = 2 (mod 2^32)
    e = check_error(lambda: gpu.take_list(col, idx), lambda: oft.take_host(col, idx))
    assert e.message == "assertion failed: idx < self.bit_len"


@pytest.mark.parametrize("wrapped", [False, True])
def test_list_and_child_overflow(gpu, wrapped):
    """Both the list's i32 offsets (at output row 2047) and its Utf8 child's (at child row 2^30 - 1, in output row 1023)
    overflow: the child is extended first, so its InvalidArgumentError wins, also for a List nested in a FixedSizeList."""
    n = 1 << 20
    child = Utf8Column(np.arange(0, 2 * n + 1, 2, dtype=np.int32), np.zeros(2 * n, np.uint8), nulls_of(np.ones(n, bool)))
    col = ListColumn(np.array([0, n], np.int32), child, nulls_of([True]))
    if wrapped:  # the FixedSizeList's row map (2048 zeros) is the List's indices
        col = FixedSizeListColumn(1, col, nulls_of([True]))
    idx = HostArray.from_numpy(abi.U32, np.zeros(2048, np.uint32))
    with pytest.raises(acu.ArrowError) as e:
        gpu.take_list(col, idx)
    assert e.value.status == abi.ERR_INVALID_ARGUMENT and e.value.message == "Invalid argument error: " + oft.EXTEND_OVERFLOW
    assert e.value.index == (1 << 30) - 1
