"""Every device buffer and filter plan a Context call allocates is released when the call returns, on success and on an
ordinary error path. The suite runs on one Context for the whole session, so a buffer leaked by one call would hold HBM
until the run ends. acu_bytes_allocated counts every acu_malloc allocation still live, plan storage included."""
import io

import numpy as np
import pytest

import acu
from acu import _abi as abi
from acu import (BOOL, DecimalArray, FixedSizeBinaryColumn, FixedSizeListColumn, HostArray, ListColumn, RunEndColumn,
                 Utf8Column, ViewColumn)

pytestmark = pytest.mark.gpu


def nulls_of(mask):
    h = HostArray.from_list(abi.U8, [0 if m else None for m in mask])
    h.values = np.zeros(0, np.uint8)
    return h


def utf8(items, dtype=np.int32):
    bs = [b"" if it is None else it for it in items]
    offsets = np.concatenate([[0], np.cumsum([len(b) for b in bs])]).astype(dtype)
    data = np.frombuffer(b"".join(bs), np.uint8).copy()
    return Utf8Column(offsets, data, nulls_of([it is not None for it in items]))


def i64(items):
    return HostArray.from_list(abi.I64, items)


def bools(items):
    return HostArray.from_list(BOOL, items)


def u32(items):
    return HostArray.from_numpy(abi.U32, np.array(items, np.uint32))


def no_leak(gpu, call, error=False):
    """Run `call` (expected to raise ArrowError when `error`) and check no device allocation outlives it."""
    before = gpu.lib.acu_bytes_allocated(gpu.h)
    if error:
        with pytest.raises(acu.ArrowError):
            call()
    else:
        call()
    assert gpu.lib.acu_bytes_allocated(gpu.h) == before


VIEWS = ViewColumn.from_values([b"a", None, b"a much longer value than twelve", b"bc"])
FSB = FixedSizeBinaryColumn.from_values([b"ab", None, b"cd", b"ef"], 2)
WORDS = utf8([b"apple", None, b"banana", b"cherry"])


def test_filter_and_take(gpu):
    vals, pred = i64([1, None, 3, 4]), bools([True, False, True, None])
    no_leak(gpu, lambda: gpu.filter(vals, pred))
    no_leak(gpu, lambda: gpu.filter(vals, bools([True] * 5)), error=True)  # predicate longer than the values
    no_leak(gpu, lambda: gpu.filter_plan(pred))
    no_leak(gpu, lambda: gpu.filter_slices(pred))
    no_leak(gpu, lambda: gpu.filter_cmp(vals, abi.LT, vals, i64([2]).scalar()))
    no_leak(gpu, lambda: gpu.filter_cmp(vals, abi.LT, vals, i64([1, 2])), error=True)
    no_leak(gpu, lambda: gpu.take(vals, u32([3, 0])))
    no_leak(gpu, lambda: gpu.take(vals, u32([4]), check_bounds=True), error=True)


def test_byte_filter_and_take(gpu):
    pred = bools([True, False, True, True])
    no_leak(gpu, lambda: gpu.filter_bytes(WORDS.offsets, WORDS.data, WORDS.nulls, pred))
    no_leak(gpu, lambda: gpu.filter_bytes(WORDS.offsets, WORDS.data, WORDS.nulls, bools([True] * 5)), error=True)
    no_leak(gpu, lambda: gpu.take_bytes(WORDS.offsets, WORDS.data, WORDS.nulls, u32([2, 0])))
    no_leak(gpu, lambda: gpu.take_bytes(WORDS.offsets, WORDS.data, WORDS.nulls, u32([9]), check_bounds=True), error=True)


def test_record_batches(gpu):
    cols = [i64([1, None, 3, 4]), bools([True, None, False, True]), WORDS]
    no_leak(gpu, lambda: gpu.filter_record_batch(cols, bools([True, False, True, True])))
    no_leak(gpu, lambda: gpu.filter_record_batch(cols, bools([True] * 5)), error=True)
    no_leak(gpu, lambda: gpu.take_record_batch(cols, u32([3, 1])))
    no_leak(gpu, lambda: gpu.take_record_batch(cols, u32([7]), check_bounds=True), error=True)
    no_leak(gpu, lambda: gpu.concat([i64([1, None]), i64([3])]))
    no_leak(gpu, lambda: gpu.concat([WORDS, WORDS]))
    no_leak(gpu, lambda: gpu.concat_batches([cols, cols]))
    no_leak(gpu, lambda: gpu.aggregate_columns([abi.SUM, abi.MAX], [i64([1, 2]), i64([None, 5])]))


def test_chain(gpu):
    col, pred, idx = i64([1, None, 3, 4]), bools([True, False, True, True]), u32([3, 0])
    a, b = HostArray.from_list(abi.F64, [1.0, 2.0]), HostArray.from_list(abi.F64, [0.5, None])
    no_leak(gpu, lambda: gpu.chain(col, pred, idx, a, b))
    no_leak(gpu, lambda: gpu.chain(col, None, idx, a, b, cmp_with=(abi.LT, col, i64([2]).scalar())))
    no_leak(gpu, lambda: gpu.chain(col, pred, u32([9]), a, HostArray.from_list(abi.F64, [1.0])), error=True)


def test_elementwise(gpu):
    a, b = i64([1, None, 3]), i64([4, 5, None])
    no_leak(gpu, lambda: gpu.add(a, b))
    no_leak(gpu, lambda: gpu.add(a, i64([1])), error=True)
    no_leak(gpu, lambda: gpu.neg(a))
    no_leak(gpu, lambda: gpu.neg(i64([-(1 << 63)])), error=True)
    no_leak(gpu, lambda: gpu.bitwise_and(a, b))
    no_leak(gpu, lambda: gpu.bitwise_not(a))
    no_leak(gpu, lambda: gpu.cmp(abi.LT, a, b))
    no_leak(gpu, lambda: gpu.cmp(abi.LT, a, i64([1, 2])), error=True)
    no_leak(gpu, lambda: gpu.and_kleene(bools([True, None]), bools([False, True])))
    no_leak(gpu, lambda: gpu.not_(bools([True, None])))
    no_leak(gpu, lambda: gpu.nullif(a, bools([True, False, None])))
    no_leak(gpu, lambda: gpu.zip(bools([True, False, True]), a, b))
    no_leak(gpu, lambda: gpu.cast(a, abi.I8))
    no_leak(gpu, lambda: gpu.cast(i64([300]), abi.I8, safe=False), error=True)  # cast overflow


def test_decimal(gpu):
    a = DecimalArray.from_ints(4, 9, 2, [123, None, -5])
    big = DecimalArray.from_ints(4, 9, 0, [(1 << 31) - 1])
    no_leak(gpu, lambda: gpu.decimal_add(a, a))
    no_leak(gpu, lambda: gpu.decimal_mul(big, big), error=True)  # decimal overflow
    no_leak(gpu, lambda: gpu.decimal_neg(a))
    no_leak(gpu, lambda: gpu.cast_decimal(a, 8, 18, 4))
    no_leak(gpu, lambda: gpu.cast_decimal(a, 4, 2, 2, safe=False), error=True)
    no_leak(gpu, lambda: gpu.cast_to_decimal(i64([1, None]), 16, 38, 2))
    no_leak(gpu, lambda: gpu.cast_from_decimal(a, abi.I64))
    no_leak(gpu, lambda: gpu.sum(DecimalArray.from_ints(16, 38, 0, [1, None, 2])))


def test_aggregates(gpu):
    no_leak(gpu, lambda: gpu.sum(i64([1, None, 3])))
    no_leak(gpu, lambda: gpu.sum_checked(i64([1, None, 3])))
    no_leak(gpu, lambda: gpu.sum_checked(i64([(1 << 63) - 1, 1])), error=True)
    no_leak(gpu, lambda: gpu.product_checked(i64([(1 << 62), 4])), error=True)
    no_leak(gpu, lambda: gpu.min_boolean(bools([True, None, False])))
    for col in (WORDS, VIEWS, FSB):
        no_leak(gpu, lambda: gpu.min_max_row(abi.MIN, col))


def test_byte_kernels(gpu):
    other = utf8([b"apple", b"b", None, b"cherry"])
    pat = utf8([b"%an%"])
    pat.nulls.is_scalar = True
    no_leak(gpu, lambda: gpu.cmp_bytes(abi.EQ, WORDS, other))
    no_leak(gpu, lambda: gpu.cmp_bytes(abi.EQ, WORDS, utf8([b"a", b"b"])), error=True)
    no_leak(gpu, lambda: gpu.cmp_view(abi.LT, VIEWS, VIEWS))
    no_leak(gpu, lambda: gpu.like_bytes(abi.LIKE, WORDS, pat))
    no_leak(gpu, lambda: gpu.like_view(abi.LIKE, VIEWS, ViewColumn.from_values([b"%a%"], scalar=True)))
    for col in (WORDS, VIEWS, FSB):
        no_leak(gpu, lambda: gpu.length(col))
        no_leak(gpu, lambda: gpu.substring(col, 1, 1))
        no_leak(gpu, lambda: gpu.concat_elements(col, col))
    no_leak(gpu, lambda: gpu.substring_by_char(WORDS, 1, 2))
    no_leak(gpu, lambda: gpu.concat_elements_utf8_many([WORDS, other, WORDS]))
    no_leak(gpu, lambda: gpu.concat_elements(WORDS, utf8([b"a"])), error=True)


def test_lists(gpu):
    inner = ListColumn(np.array([0, 2, 2, 3, 5], np.int32), i64([1, 2, None, 4, 5]), nulls_of([True, False, True, True]))
    nested = ListColumn(np.array([0, 1, 3, 4], np.int32), inner, nulls_of([True, True, False]))
    fixed = FixedSizeListColumn(2, WORDS, nulls_of([True, False]))
    for col in (inner, nested, fixed):
        no_leak(gpu, lambda: gpu.filter_list(col, bools([True, False] + [True] * (col.length - 2))))
        no_leak(gpu, lambda: gpu.filter_list(col, bools([True] * (col.length + 1))), error=True)
        no_leak(gpu, lambda: gpu.take_list(col, u32([1, 0, 1])))
        no_leak(gpu, lambda: gpu.take_list(col, u32([col.length]), check_bounds=True), error=True)


def test_nested_list_offset_overflow(gpu):
    """The unwrap panic of a List take whose i32 offsets pass i32::MAX at output row 2047, with a Utf8 child that is
    extended up to that row before the panic is raised."""
    child = Utf8Column(np.zeros((1 << 20) + 1, np.int32), np.zeros(0, np.uint8), nulls_of([True] * (1 << 20)))
    col = ListColumn(np.array([0, 1 << 20], np.int32), child, nulls_of([True]))
    no_leak(gpu, lambda: gpu.take_list(col, u32([0] * 2049)), error=True)


def test_run_end(gpu):
    prim = RunEndColumn(np.array([2, 5, 6], np.int32), i64([7, None, 9]))
    text = RunEndColumn(np.array([1, 3, 4], np.int16), utf8([b"apple", None, b"a string past twelve bytes"]))
    for col in (prim, text, prim.slice(1, 4)):
        no_leak(gpu, lambda: gpu.filter_run_end(col, bools([True, False] + [True] * (col.length - 2))))
        no_leak(gpu, lambda: gpu.filter_run_end(col, bools([True] * (col.length + 1))), error=True)
        no_leak(gpu, lambda: gpu.take_run_end(col, u32([col.length - 1, 0])))
        no_leak(gpu, lambda: gpu.take_run_end(col, u32([col.length])), error=True)  # Logical index ... is out of bounds


def test_ipc_read_stream(gpu):
    pa = pytest.importorskip("pyarrow")
    batch = pa.record_batch([pa.array([1, None, 3], pa.int64()), pa.array(["a", None, "ccc"])], names=["x", "s"])
    sink = io.BytesIO()
    with pa.ipc.new_stream(sink, batch.schema) as w:
        w.write_batch(batch)
    no_leak(gpu, lambda: gpu.ipc_read_stream(sink.getvalue()))
    no_leak(gpu, lambda: gpu.ipc_read_stream(sink.getvalue()[:-20]), error=True)
