"""Python oracle for filter / take of RunEndEncoded columns (filter_run_end_array arrow-select/src/filter.rs:628-677,
take_run take.rs:948-995, RunEndBuffer arrow-buffer/src/buffer/run.rs:232-378, RunArray::get_physical_indices
arrow-array/src/array/run_array.rs:343-356), restated over acu.RunEndColumn. The values child is filtered / taken by
tests/oracle_list.py, the oracle of every other column type."""
import bisect

import numpy as np

import acu
from acu import BOOL, DecimalArray, FixedSizeListColumn, HostArray, ListColumn, RunEndColumn, Utf8Column, ViewColumn
from acu import _abi as abi

import oracle_list as ol
from oracle_list import OracleError, UNWRAP_NONE

R_MAX = {2: 2**15 - 1, 4: 2**31 - 1, 8: 2**63 - 1}
INDEX_MAX = {abi.I8: 2**7 - 1, abi.U8: 2**8 - 1, abi.I16: 2**15 - 1, abi.U16: 2**16 - 1, abi.I32: 2**31 - 1, abi.U32: 2**32 - 1,
             abi.I64: 2**63 - 1, abi.U64: 2**64 - 1}
NESTED_TEXT = "take of a RunEndEncoded column with nested values is not yet implemented"


def empty(col):
    return RunEndColumn(np.zeros(0, col.run_ends.dtype), acu.empty_column(col.values), 0, 0)


# ---- RunEndBuffer (run.rs:232-267) -----------------------------------------------------------------------------------
def physical_index(col, i):
    """get_physical_index: binary_search of offset + i over the run ends, Ok(idx) -> idx + 1, Err(idx) -> idx."""
    return bisect.bisect_right([int(x) for x in col.run_ends], col.offset + i)


def start_physical(col):
    if col.offset == 0 or col.length == 0:
        return 0
    return physical_index(col, 0)


def end_physical(col):
    if col.length == 0:
        return 0
    if int(col.run_ends[-1]) == col.offset + col.length:
        return len(col.run_ends) - 1
    return physical_index(col, col.length - 1)


def values_slice(col):
    if col.length == 0:
        return acu.slice_column(col.values, 0, 0)
    s, e = start_physical(col), end_physical(col)
    return acu.slice_column(col.values, s, e - s + 1)


# ---- filter -----------------------------------------------------------------------------------------------------------
def filter(col, mask):
    """filter(col, predicate) with mask = oracle_list.filter_mask(predicate)."""
    mask = np.asarray(mask, dtype=bool)
    p = len(mask)
    if p > col.length:
        raise OracleError(abi.ERR_INVALID_ARGUMENT, f"Filter predicate of length {p} is larger than target array of length {col.length}")
    count = int(mask.sum())
    if count == 0:  # IterationStrategy::None: new_empty_array
        return empty(col)
    if count == p:  # IterationStrategy::All: values.slice(0, count)
        return col.slice(0, count)
    s, e = start_physical(col), end_physical(col)
    new_ends, keep = [], []
    start, running = 0, 0
    for i in range(s, e + 1):
        end = max(int(col.run_ends[i]) - col.offset, 0)  # saturating_sub
        end = min(end, p)
        sel = int(mask[start:end].sum()) if end > start else 0
        running += sel
        keep.append(sel > 0)
        if sel:
            new_ends.append(running)
        start = end
    values = ol.filter(values_slice(col), np.array(keep, dtype=bool))
    return RunEndColumn(np.array(new_ends, dtype=col.run_ends.dtype), values, 0, new_ends[-1])


# ---- take ---------------------------------------------------------------------------------------------------------------
def get_physical_indices(col, ix):
    """ix: ToIndices values (null slots included). The largest at or past the length is the error's index."""
    if not ix:
        return []
    mx = max(ix)
    if mx >= col.length:
        raise OracleError(abi.ERR_INVALID_ARGUMENT, f"Logical index {mx} is out of bounds for RunArray of length {col.length}")
    ends = [int(x) for x in col.run_ends]
    return [bisect.bisect_right(ends, col.offset + x) for x in ix]  # the first run whose end - offset > x


def check_bounds(n, idx, valid, dtype):
    """take.rs:167-209: skipped when the length does not fit the index type; null slots ignored."""
    if n > INDEX_MAX[dtype]:
        return
    all_valid = all(valid)
    for j, v in enumerate(idx):
        v = int(v)
        if not all_valid and not valid[j]:
            continue
        if v >= n or (v < 0 and all_valid):
            raise OracleError(abi.ERR_COMPUTE, f"Array index out of bounds, cannot get item at index {v} from {n} entries", j)


def comparator(v):
    """make_comparator(values, values, SortOptions::default()): (a, b) -> is_eq()."""
    vm = ol.valid_mask(v)
    if isinstance(v, (Utf8Column, ViewColumn)):
        same = lambda a, b: acu.column_value(v, a) == acu.column_value(v, b)  # noqa: E731
    elif v.dtype == BOOL:
        bits = v.value_array()
        same = lambda a, b: bool(bits[a]) == bool(bits[b])  # noqa: E731
    elif isinstance(v, DecimalArray):
        ints = v.raw_ints()
        same = lambda a, b: ints[a] == ints[b]  # noqa: E731
    else:  # integers, and floats under total_cmp: equal iff the bits are
        raw = np.asarray(v.values[:v.length]).view(np.dtype(f"u{v.width()}"))
        same = lambda a, b: raw[a] == raw[b]  # noqa: E731

    def eq(a, b):
        if not vm[a] or not vm[b]:  # two nulls are equal, a null never equals a value
            return bool(vm[a]) == bool(vm[b])
        return bool(same(a, b))
    return eq


def take(col, indices, check=False):
    """take(col, indices, TakeOptions{check_bounds: check}) for a HostArray of integer indices."""
    idx, valid = list(indices.value_array()), list(indices.valid_mask())
    if check:
        check_bounds(col.length, idx, valid, indices.dtype)
    if not idx:
        return empty(col)
    wide = indices.dtype in (abi.I64, abi.U64)
    phys = get_physical_indices(col, [ol._to_index(indices.dtype, v) for v in idx])
    if isinstance(col.values, (ListColumn, FixedSizeListColumn, RunEndColumn)):  # where take_run builds its comparator
        raise OracleError(abi.ERR_NOT_YET_IMPLEMENTED, "Not yet implemented: " + NESTED_TEXT)
    r_max, i_max = R_MAX[col.run_ends.itemsize], 2**64 - 1 if wide else 2**32 - 1
    new_ends, value_idx = [], []

    def push(ix, end):
        if ix > i_max or end > r_max:  # I::Native / T::Native::from_usize(..).unwrap()
            raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, UNWRAP_NONE)
        value_idx.append(ix)
        new_ends.append(end)

    eq = comparator(col.values)
    for q in range(1, len(phys)):
        if phys[q] != phys[q - 1] and not eq(phys[q], phys[q - 1]):
            push(phys[q - 1], q)
    push(phys[-1], len(phys))
    values = ol.take(col.values, value_idx, [True] * len(value_idx), False, abi.U64 if wide else abi.U32)
    return RunEndColumn(np.array(new_ends, dtype=col.run_ends.dtype), values, 0, len(phys))


# ---- comparison ---------------------------------------------------------------------------------------------------------
def describe(col):
    """The physical result: run-end type and values, logical window, and the values child as oracle_list describes it."""
    return ("ree", str(col.run_ends.dtype), [int(x) for x in col.run_ends], col.offset, col.length, ol.describe(col.values))


def logical(col):
    """The logical values of a RunEndColumn (None for nulls)."""
    vals = ol.to_pylist(col.values)
    ends = [int(x) for x in col.run_ends]
    return [vals[bisect.bisect_right(ends, col.offset + i)] for i in range(col.length)]
