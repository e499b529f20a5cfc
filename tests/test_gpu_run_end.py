"""filter / take of RunEndEncoded columns on the device against tests/oracle_run_end.py, bit for bit: run ends and their
type, the values child (the bytes under nulls included), NullBuffer presence, and status plus exact message."""
import zlib

import numpy as np
import pytest

import acu
from acu import DecimalArray, HostArray, ListColumn, RunEndColumn, Utf8Column, ViewColumn
from acu import _abi as abi

import oracle_run_end as ore
from run_end_util import check, golden_cases, run_case

pytestmark = pytest.mark.gpu

INDEX_DTYPES = [abi.I8, abi.U8, abi.I16, abi.U16, abi.I32, abi.U32, abi.I64, abi.U64]
R_TYPES = [np.int16, np.int32, np.int64]
RE_THREADS, RE_PER_SM = 256, 8  # csrc/run_end.cu launch constants (pinned by test_run_end_launch_constants.py)


def nulls_of(mask):
    h = HostArray.from_list(abi.U8, [0 if v else None for v in mask])
    h.values = np.zeros(0, np.uint8)
    return h


def values_of(kind, n, rng, null_p=0.2, distinct=3):
    """n physical values drawn from a few distinct ones, so that taken neighbours often compare equal."""
    mask = rng.random(n) >= null_p
    pick = rng.integers(0, distinct, n)
    if kind in ("i8", "i32", "i64"):
        dt = {"i8": abi.I8, "i32": abi.I32, "i64": abi.I64}[kind]
        return HostArray.from_numpy(dt, (pick * 37 - 50) % (100 if kind == "i8" else 10**6), mask)
    if kind in ("f32", "f64"):
        npdt = np.float32 if kind == "f32" else np.float64
        choices = np.array([0.0, -0.0, 1.5, np.nan, np.nan], npdt)
        v = choices[rng.integers(0, 5, n)]
        bits = v.view(np.uint32 if kind == "f32" else np.uint64)
        nan2 = np.isnan(v) & (rng.random(n) < 0.5)  # a second NaN payload
        bits[nan2] |= 1
        return HostArray.from_numpy(abi.F32 if kind == "f32" else abi.F64, v, mask)
    if kind == "bool":
        return HostArray.bool_from_numpy(pick % 2 == 0, mask, bit_offset=3, mask_offset=5)
    if kind == "dec128":
        return DecimalArray.from_int64(16, 38, 2, pick * 10**17 - 7, mask)
    words = [b"", b"ab", b"a much longer value than twelve bytes"]
    if kind == "view":
        return ViewColumn.from_values([words[p] if m else None for p, m in zip(pick, mask)], garbage_under_nulls=[np.arange(16, dtype=np.uint8)])
    if kind in ("utf8", "lbin"):
        items = [words[p] if m else b"zz" for p, m in zip(pick, mask)]  # bytes under null rows too
        offs = np.zeros(n + 1, np.int32 if kind == "utf8" else np.int64)
        offs[1:] = np.cumsum([len(x) for x in items])
        return Utf8Column(offs, np.frombuffer(b"".join(items) + b"\0", np.uint8).copy(), nulls_of(mask))
    if kind == "list":
        lens = rng.integers(0, 4, n)
        offs = np.zeros(n + 1, np.int32)
        offs[1:] = np.cumsum(lens)
        child = HostArray.from_numpy(abi.I64, rng.integers(-2**62, 2**62, int(offs[-1])), rng.random(int(offs[-1])) >= 0.2)
        return ListColumn(offs, child, nulls_of(mask))
    raise ValueError(kind)


def ree_of(values, rng, r_dtype=np.int32, mean_run=8):
    n = values.length
    lens = np.ones(n, np.int64) if mean_run == 1 else rng.integers(1, 2 * mean_run, n)
    return RunEndColumn(np.cumsum(lens).astype(r_dtype), values)


def expect_same(run_dev, run_orc):
    try:
        exp = run_orc()
    except ore.OracleError as e:
        with pytest.raises(acu.ArrowError) as got:
            run_dev()
        assert (got.value.status, got.value.message) == (e.status, e.message)
        return
    got = run_dev()
    assert ore.describe(got) == ore.describe(exp)


def dev_filter(gpu, col, pred):
    return lambda: gpu.filter_run_end(col, pred)


def orc_filter(col, pred):
    return lambda: ore.filter(col, ore.ol.filter_mask(pred))


def rand_pred(rng, n, p=0.5, null_p=0.1):
    return HostArray.bool_from_numpy(rng.random(n) < p, rng.random(n) >= null_p)


@pytest.mark.parametrize("case", golden_cases(), ids=lambda c: c["name"])
def test_golden(gpu, case):
    check(case, run_case(case, gpu.filter_run_end, gpu.take_run_end))


KINDS = ["i8", "i32", "i64", "f32", "f64", "bool", "dec128", "utf8", "lbin", "view"]


@pytest.mark.parametrize("r_dtype", R_TYPES, ids=lambda t: t.__name__)
@pytest.mark.parametrize("kind", KINDS + ["list"])
def test_filter_types(gpu, kind, r_dtype):
    rng = np.random.default_rng(zlib.crc32(f"filter {kind} {r_dtype.__name__}".encode()))
    col = ree_of(values_of(kind, 300, rng), rng, r_dtype, mean_run=4 if r_dtype == np.int16 else 8)
    for pred in (rand_pred(rng, col.length), rand_pred(rng, col.length, p=0.03, null_p=0.0),
                 rand_pred(rng, col.length, p=0.97, null_p=0.0), rand_pred(rng, col.length - 17)):
        expect_same(dev_filter(gpu, col, pred), orc_filter(col, pred))


@pytest.mark.parametrize("r_dtype", R_TYPES, ids=lambda t: t.__name__)
@pytest.mark.parametrize("kind", KINDS)
def test_take_types(gpu, kind, r_dtype):
    rng = np.random.default_rng(zlib.crc32(f"take {kind} {r_dtype.__name__}".encode()))
    col = ree_of(values_of(kind, 200, rng), rng, r_dtype, mean_run=4)
    n = col.length
    for ix in (rng.integers(0, n, 500), np.sort(rng.integers(0, n, 500)), np.sort(rng.integers(0, n, 500))[::-1],
               np.repeat(rng.integers(0, n, 50), 7)):
        idx = HostArray.from_numpy(abi.I64, ix, rng.random(len(ix)) >= 0.1)
        expect_same(lambda: gpu.take_run_end(col, idx), lambda: ore.take(col, idx))


def test_slices(gpu):
    """Offsets inside a run, on a run end and at +-1 of it; lengths ending mid-run."""
    rng = np.random.default_rng(11)
    col = ree_of(values_of("i64", 60, rng), rng, np.int32, mean_run=6)
    ends = [int(x) for x in col.run_ends]
    e = ends[5]
    for off in (e - 1, e, e + 1, (ends[5] + ends[6]) // 2, 0):
        for ln in (1, ends[9] - off - 1, ends[9] - off, col.length - off):
            s = col.slice(off, ln)
            for pred in (rand_pred(rng, ln), rand_pred(rng, max(ln - 2, 0), p=0.9, null_p=0.0)):
                expect_same(dev_filter(gpu, s, pred), orc_filter(s, pred))
            idx = HostArray.from_numpy(abi.U32, rng.integers(0, ln, 40))
            expect_same(lambda: gpu.take_run_end(s, idx), lambda: ore.take(s, idx))


@pytest.mark.parametrize("mean_run", [1, 8, 10**6])
def test_run_lengths(gpu, mean_run):
    rng = np.random.default_rng(mean_run)
    n_runs = 1 if mean_run == 10**6 else 400
    col = ree_of(values_of("i32", n_runs, rng, null_p=0.3), rng, np.int64, mean_run=min(mean_run, 50))
    if mean_run == 10**6:
        col = RunEndColumn(np.array([5000], np.int64), col.values)
    for pred in (rand_pred(rng, col.length), HostArray.bool_from_numpy(np.zeros(col.length, bool)),
                 HostArray.bool_from_numpy(np.ones(col.length, bool))):
        expect_same(dev_filter(gpu, col, pred), orc_filter(col, pred))
    idx = HostArray.from_numpy(abi.U64, rng.integers(0, col.length, 1000))
    expect_same(lambda: gpu.take_run_end(col, idx), lambda: ore.take(col, idx))


def test_filter_predicate_longer_than_array(gpu):
    col = ree_of(values_of("i32", 10, np.random.default_rng(0)), np.random.default_rng(1))
    pred = HostArray.bool_from_numpy(np.ones(col.length + 1, bool))
    expect_same(dev_filter(gpu, col, pred), orc_filter(col, pred))


@pytest.mark.parametrize("dtype", INDEX_DTYPES)
def test_take_index_dtypes(gpu, dtype):
    rng = np.random.default_rng(dtype)
    col = ree_of(values_of("utf8", 20, rng), rng, np.int16, mean_run=3)
    hi = min(col.length, 127)
    raw = rng.integers(0, hi, 300)
    idx = HostArray.from_numpy(dtype, raw, rng.random(300) >= 0.2)
    expect_same(lambda: gpu.take_run_end(col, idx), lambda: ore.take(col, idx))
    for check_bounds in (False, True):
        bad = HostArray.from_numpy(dtype, raw, rng.random(300) >= 0.2)
        bad.values[7] = hi + 3 if hi + 3 <= 127 else 127  # valid out-of-bounds value
        if col.length > 127:
            bad.values[7] = 0
        expect_same(lambda: gpu.take_run_end(col, bad, check_bounds), lambda: ore.take(col, bad, check_bounds))


@pytest.mark.parametrize("check_bounds", [False, True])
def test_take_null_over_out_of_bounds(gpu, check_bounds):
    """get_physical_indices reads the values of null slots too: a null over an out-of-bounds value fails."""
    col = RunEndColumn(np.array([3, 5, 9], np.int32), HostArray.from_list(abi.I64, [1, None, 3]))
    ok = HostArray.from_list(abi.U32, [0, None, 8, 4])
    ok.values[1] = 2
    expect_same(lambda: gpu.take_run_end(col, ok, check_bounds), lambda: ore.take(col, ok, check_bounds))
    bad = HostArray.from_list(abi.U32, [0, None, 8, 4])
    bad.values[1] = 9
    expect_same(lambda: gpu.take_run_end(col, bad, check_bounds), lambda: ore.take(col, bad, check_bounds))


@pytest.mark.parametrize("dtype", [abi.I8, abi.I32])
@pytest.mark.parametrize("check_bounds", [False, True])
def test_take_negative_indices(gpu, dtype, check_bounds):
    col = RunEndColumn(np.array([3, 5, 9], np.int64), HostArray.from_list(abi.I64, [1, 2, 3]))
    idx = HostArray.from_list(dtype, [0, 4, -1, 2])
    expect_same(lambda: gpu.take_run_end(col, idx, check_bounds), lambda: ore.take(col, idx, check_bounds))


def test_take_merges(gpu):
    """Equal values from different runs merge; adjacent null runs merge; a null never merges with a valid value."""
    vals = HostArray.from_list(abi.I32, [5, 7, 5, None, 7, None, 0])
    vals.values[3] = 5  # a null over the bits of its neighbour
    col = RunEndColumn(np.array([2, 4, 6, 8, 10, 12, 14], np.int32), vals)
    for ix in ([0, 5, 1, 2, 6, 10, 11, 7, 8], [4, 1, 6, 7, 10], [13, 12, 0, 4]):
        idx = HostArray.from_list(abi.U16, ix)
        expect_same(lambda: gpu.take_run_end(col, idx), lambda: ore.take(col, idx))
    got = gpu.take_run_end(col, HostArray.from_list(abi.U16, [0, 5, 1, 2, 6, 10, 11, 7, 8]))
    assert [int(x) for x in got.run_ends] == [3, 4, 8, 9]  # 5 5 5 | 7 | null x4 | 7


def test_take_float_bits(gpu):
    """total_cmp: -0.0 != 0.0 and NaNs with different payloads differ, also in adjacent runs."""
    v = np.array([0.0, -0.0, np.nan, np.nan, 1.0], np.float64)
    v.view(np.uint64)[3] |= 1
    col = RunEndColumn(np.array([1, 2, 3, 4, 5], np.int64), HostArray.from_numpy(abi.F64, v))
    idx = HostArray.from_list(abi.U8, [0, 1, 2, 3, 3, 2, 0, 0])
    expect_same(lambda: gpu.take_run_end(col, idx), lambda: ore.take(col, idx))
    assert [int(x) for x in gpu.take_run_end(col, idx).run_ends] == [1, 2, 3, 5, 6, 8]


def test_take_int16_unwrap(gpu):
    col = RunEndColumn(np.array([2, 5], np.int16), HostArray.from_list(abi.I8, [1, 2]))
    for m in (32767, 32768, 40000):
        idx = HostArray.from_numpy(abi.U16, np.arange(m) % 5)
        expect_same(lambda: gpu.take_run_end(col, idx), lambda: ore.take(col, idx))


def test_empty(gpu):
    col = RunEndColumn(np.array([2, 5], np.int32), HostArray.from_list(abi.I8, [1, 2]))
    idx = HostArray.from_numpy(abi.I32, np.zeros(0, np.int32))
    expect_same(lambda: gpu.take_run_end(col, idx), lambda: ore.take(col, idx))
    empty = RunEndColumn(np.zeros(0, np.int32), HostArray.from_list(abi.I8, []))
    expect_same(lambda: gpu.take_run_end(empty, idx), lambda: ore.take(empty, idx))
    one = HostArray.from_numpy(abi.I32, np.zeros(1, np.int32))
    expect_same(lambda: gpu.take_run_end(empty, one), lambda: ore.take(empty, one))
    pred = HostArray.bool_from_numpy(np.zeros(0, bool))
    expect_same(dev_filter(gpu, empty, pred), orc_filter(empty, pred))


def test_take_nested_values_refused(gpu):
    rng = np.random.default_rng(2)
    col = ree_of(values_of("list", 10, rng), rng)
    # the refusal stands where take_run builds its comparator: empty indices and the bounds errors come first
    for idx, cb in ((HostArray.from_list(abi.U32, [0, 1]), False), (HostArray.from_numpy(abi.U32, np.zeros(0, np.uint32)), False),
                    (HostArray.from_list(abi.U32, [0, col.length]), False), (HostArray.from_list(abi.U32, [0, col.length]), True)):
        expect_same(lambda: gpu.take_run_end(col, idx, cb), lambda: ore.take(col, idx, cb))


def _round(gpu):
    return gpu.lib.acu_device_sm_count(gpu.h) * RE_PER_SM * RE_THREADS


def test_filter_grid_rounds(gpu):
    """k_ree_filter_runs at 1.3 grid rounds of runs, mean run 2, with runs kept and dropped in every round."""
    rng = np.random.default_rng(21)
    n_runs = int(1.3 * _round(gpu))
    vals = HostArray.from_numpy(abi.I64, rng.integers(-9, 9, n_runs), rng.random(n_runs) >= 0.1)
    col = ree_of(vals, rng, np.int32, mean_run=2)
    s = col.slice(3, col.length - 3)
    for pred in (rand_pred(rng, s.length, p=0.2), rand_pred(rng, s.length - 1000, p=0.9, null_p=0.0)):
        expect_same(dev_filter(gpu, s, pred), orc_filter(s, pred))


@pytest.mark.parametrize("kind", ["i64", "view"])
def test_take_grid_rounds(gpu, kind):
    """k_ree_take_map and k_ree_run_ends at 1.3 grid rounds of indices, with the largest index in the last round."""
    rng = np.random.default_rng(23)
    col = ree_of(values_of(kind, 5000, rng, distinct=2), rng, np.int64, mean_run=3)
    m = int(1.3 * _round(gpu))
    ix = np.sort(rng.integers(0, col.length - 1, m))
    ix[-5] = col.length - 1
    idx = HostArray.from_numpy(abi.U32, ix)
    expect_same(lambda: gpu.take_run_end(col, idx), lambda: ore.take(col, idx))
    ix[-2] = col.length  # out of bounds only in the last round
    expect_same(lambda: gpu.take_run_end(col, idx), lambda: ore.take(col, idx))
