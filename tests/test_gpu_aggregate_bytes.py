"""min / max of Utf8 / Binary, LargeUtf8 / LargeBinary, Utf8View / BinaryView and FixedSizeBinary columns, and
min_boolean / max_boolean / bool_and / bool_or, on the device: the reference's literal vectors, and the row and valid count
against the CPU restatement (tests/oracle_aggregate.py) over sizes, null densities, offsets, ties and adversarial bytes."""
import numpy as np
import pytest

import acu
from acu import MAX, MIN, SUM, ArrowError, FixedSizeBinaryColumn, HostArray, Utf8Column
from acu import _abi as abi
from aggregate_util import (bool_array, bytes_column, fixed_column, load_aggregate_cases, random_items, run_golden_case, slice_column,
                            view_column)
from oracle_aggregate import AggregateOracle

pytestmark = pytest.mark.gpu

CASES = load_aggregate_cases()
ORC = AggregateOracle()
OPS = [MIN, MAX]
SIZES = [0, 1, 31, 32, 33, 64, 127, 129, 1000, 4097, 20001]
FORMS = ["utf8", "large_utf8", "view"]


def _garbage_view(op):
    """An inline view that encodes a value beating every valid one (min: one 0x00 byte; max: twelve 0xff bytes)."""
    v = np.zeros(16, np.uint8)
    if op == MIN:
        v[0] = 1
    else:
        v[0] = 12
        v[4:16] = 0xff
    return v


def _column(form, items, op, bit_offset=0, block_size=64):
    """A column of `items` whose null slots hold a value that would win under `op` if it were read."""
    if form == "view":
        return view_column(items, bit_offset=bit_offset, garbage_views=[_garbage_view(op)], block_size=block_size)
    return bytes_column(items, large=form == "large_utf8", bit_offset=bit_offset, garbage=b"\0" if op == MIN else b"\xff" * 24)


def _same(gpu, op, col):
    got, want = gpu.min_max_row(op, col), ORC.min_max_row(op, col)
    assert got == want, (op, got, want)
    return got


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_gpu_matches_reference_vector(gpu, case):
    run_golden_case(gpu, case)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("null_p", [0.0, 0.2, 1.0])
@pytest.mark.parametrize("n", SIZES)
def test_sizes_and_nulls(gpu, n, null_p, form):
    rng = np.random.default_rng(n * 7 + int(null_p * 10))
    # valid values from b..e never start with 0x00 or 0xff, so the null slots' contents would win if they were read
    items = random_items(rng, n + 9, null_p, alphabet=b"bcde", max_len=20)
    for op in OPS:
        col = _column(form, items, op, bit_offset=n % 8)
        _same(gpu, op, slice_column(col, 9, n))  # sliced: offsets / views / validity bit offset start mid-array
        _same(gpu, op, col)


@pytest.mark.parametrize("form", FORMS)
def test_adversarial_bytes(gpu, form):
    """empty values, 0x00 and 0xff bytes, prefix pairs ("a" / "a\\0"), inline and long views across several buffers."""
    rng = np.random.default_rng(5)
    for trial in range(20):
        items = random_items(rng, int(rng.integers(1, 3000)), 0.15, alphabet=b"a\0\xff", max_len=[3, 14, 40][trial % 3])
        for op in OPS:
            col = view_column(items, block_size=96) if form == "view" else bytes_column(items, large=form == "large_utf8")
            _same(gpu, op, col)
    for items in ([b"a\0", b"a"], [b"a", b"a\0"], [b"", b"\0"], [b"\xff" * 13, b"\xff" * 12], [b""] * 3):
        for op in OPS:
            _same(gpu, op, view_column(items) if form == "view" else bytes_column(items))


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("prefix", [9, 13, 24])
def test_shared_prefix_full_compare(gpu, form, prefix):
    """Every value shares a prefix longer than the key (8 bytes; 4 for views, 12 inline): every key ties."""
    rng = np.random.default_rng(prefix)
    tails = random_items(rng, 50000, 0.1, alphabet=b"xyz", max_len=6)
    items = [None if t is None else b"Q" * prefix + t for t in tails]
    for op in OPS:
        _same(gpu, op, _column(form, items, op, bit_offset=3, block_size=4096))


@pytest.mark.parametrize("form", FORMS)
def test_heavy_duplicates(gpu, form):
    rng = np.random.default_rng(11)
    pool = random_items(rng, 4096, 0.0, alphabet=b"bcdefgh", max_len=12)
    idx = rng.integers(0, len(pool), 1_000_000)
    mask = rng.random(len(idx)) >= 0.05
    items = [pool[i] if m else None for i, m in zip(idx, mask)]
    for op in OPS:
        _same(gpu, op, _column(form, items, op, block_size=1 << 16))
    # all rows equal: the first valid row is the answer
    same = [None] * 77 + [b"same-value-xyz"] * 200_000
    for op in OPS:
        assert _same(gpu, op, _column(form, same, op, block_size=1 << 16)) == (77, 200_000)


@pytest.mark.parametrize("form", FORMS)
def test_extremum_at_first_and_last_valid_row(gpu, form):
    n = 70_000
    base = [b"m" + bytes([65 + (i % 20)]) for i in range(n)]
    for pos in ("first", "last"):
        items = list(base)
        items[0], items[-1] = None, None
        k = 1 if pos == "first" else n - 2
        for op in OPS:
            items[k] = b"a" if op == MIN else b"z"
            row, cnt = _same(gpu, op, _column(form, items, op))
            assert row == k and cnt == n - 2


@pytest.mark.parametrize("width", [0, 1, 3, 8, 16, 33])
@pytest.mark.parametrize("null_p", [0.0, 0.2, 1.0])
def test_fixed_size_binary(gpu, width, null_p):
    rng = np.random.default_rng(width)
    for n in (1, 129, 20001):
        items = [None if rng.random() < null_p else rng.choice([0, 1, 7, 255], width).astype(np.uint8).tobytes() for _ in range(n + 5)]
        for op in OPS:
            col = fixed_column(items, width, bit_offset=5, garbage=(b"\0" if op == MIN else b"\xff") * width)
            _same(gpu, op, col)
            _same(gpu, op, slice_column(col, 5, n))


def test_multi_round_grid(gpu):
    """Enough rows that every CTA of the grid loops several times, with the extrema planted late and once."""
    rng = np.random.default_rng(2024)
    n = 60_000_000
    data = rng.integers(ord("b"), ord("y") + 1, 2 * n, dtype=np.uint8)
    data[2 * (n - 3): 2 * (n - 3) + 2] = ord("a")       # the only minimum, near the end
    for r in (n // 2 + 12345, n - 100):                  # the maximum twice: the lower row wins
        data[2 * r: 2 * r + 2] = ord("z")
    mask = rng.random(n) >= 0.05
    mask[[n - 3, n // 2 + 12345, n - 100]] = True
    nulls = HostArray.from_numpy(acu.U8, np.zeros(n, np.uint8), mask, 3)
    nulls.values = np.zeros(0, np.uint8)
    cols = [Utf8Column(np.arange(n + 1, dtype=np.int32) * 2, data, nulls), FixedSizeBinaryColumn(data.reshape(n, 2), nulls)]
    for col in cols:
        assert gpu.min_max_row(MIN, col) == (n - 3, int(mask.sum()))
        assert gpu.min_max_row(MAX, col) == (n // 2 + 12345, int(mask.sum()))


@pytest.mark.parametrize("n", [1, 63, 64, 65, 127, 128, 129, 1000, 100_003])
@pytest.mark.parametrize("offsets", [(0, 0), (3, 5), (63, 1)])
@pytest.mark.parametrize("null_p", [0.0, 0.2, 1.0])
def test_boolean(gpu, n, offsets, null_p):
    rng = np.random.default_rng(n)
    for p_true in (0.0, 0.5, 1.0):
        items = [None if rng.random() < null_p else bool(rng.random() < p_true) for _ in range(n)]
        a = bool_array(items, *offsets)
        for op in OPS:
            assert gpu.aggregate_boolean(op, a) == ORC.aggregate_boolean(op, a)
        s = a.slice(1, n - 1)  # unknown null count, shifted bit offsets
        for op in OPS:
            assert gpu.aggregate_boolean(op, s) == ORC.aggregate_boolean(op, s)
    # one false / one true hidden among the other value, next to a word boundary
    for k in sorted({0, min(63, n - 1), n - 1}):
        for fill, op in ((True, MIN), (False, MAX)):
            items = [fill] * n
            items[k] = not fill
            assert gpu.aggregate_boolean(op, bool_array(items, *offsets)) == (int(not fill), n)


def _expect_invalid(fn):
    with pytest.raises(ArrowError) as e:
        fn()
    assert e.value.status == abi.ERR_INVALID_ARGUMENT


def test_errors(gpu):
    col = bytes_column([b"a", None, b"b"])
    _expect_invalid(lambda: gpu.min_max_row(SUM, col))
    _expect_invalid(lambda: gpu.min_max_row(SUM, view_column([b"a"])))
    _expect_invalid(lambda: gpu.aggregate_boolean(SUM, bool_array([True])))
    bad = Utf8Column(col.offsets.astype(np.int16), col.data, col.nulls)  # offset width 2
    _expect_invalid(lambda: gpu.min_max_row(MIN, bad))


def test_negative_width_scalar_and_async_section(gpu):
    import ctypes as C
    lib, h = gpu.lib, gpu.h
    buf = gpu.malloc(64)
    try:
        row, cnt, val = C.c_int64(0), C.c_int64(0), C.c_int32(0)
        d = abi.Array()
        d.values, d.len = buf, 1
        assert lib.acu_aggregate_fixed_size_binary(h, -1, MIN, C.byref(d), C.byref(row), C.byref(cnt)) == abi.ERR_INVALID_ARGUMENT
        d.is_scalar = 1
        assert lib.acu_aggregate_fixed_size_binary(h, 4, MIN, C.byref(d), C.byref(row), C.byref(cnt)) == abi.ERR_INVALID_ARGUMENT
        assert lib.acu_aggregate_boolean(h, MAX, C.byref(d), C.byref(val), C.byref(cnt)) == abi.ERR_INVALID_ARGUMENT
        scalar = bytes_column([b"x"])
        scalar.nulls.is_scalar = True
        _expect_invalid(lambda: gpu.min_max_row(MIN, scalar))
        d.is_scalar = 0
        gpu.async_begin()
        try:
            assert lib.acu_aggregate_fixed_size_binary(h, 4, MIN, C.byref(d), C.byref(row), C.byref(cnt)) == abi.ERR_INVALID_ARGUMENT
            assert lib.acu_aggregate_boolean(h, MAX, C.byref(d), C.byref(val), C.byref(cnt)) == abi.ERR_INVALID_ARGUMENT
            _expect_invalid(lambda: gpu.min_max_row(MIN, bytes_column([b"a", b"b"])))
            _expect_invalid(lambda: gpu.min_max_row(MAX, view_column([b"a", b"b"])))
        finally:
            gpu.results_fetch()
        # the context is usable after the section
        assert gpu.min_max_row(MAX, bytes_column([b"a", b"c", b"b"])) == (1, 3)
        assert gpu.min_max_row(MIN, fixed_column([b"ab", b"aa"], 2)) == (1, 2)
    finally:
        gpu.free(buf)
