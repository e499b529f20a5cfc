"""Python oracle for filter / take of Struct, sparse Union and dense Union columns (filter_struct / filter_sparse_union
filter.rs:1010-1054, the dense MutableArrayData fallback filter.rs:597-622 with arrow-data/src/transform/{structure,union}.rs,
take_impl's Struct and Union arms take.rs:270-298, :334-382, UnionArray::try_new union_array.rs:177-242), restated over
the host column classes of `acu`. Every other column type, and the list levels, go through tests/oracle_list.py: a list
whose child holds a struct or union runs its own level there over a row-id child, and the real child here."""
import numpy as np

import acu
from acu import BOOL, FixedSizeListColumn, HostArray, ListColumn, StructColumn, UnionColumn, ViewColumn, pack_bits
from acu import _abi as abi

import oracle_list as ol
from oracle_list import OracleError

UNION_TYPE_IDS = "Type Ids values must match one of the field type ids"
BIT_LEN = "assertion failed: idx < self.bit_len"


def _new(col):
    """col is, or holds below it, a struct or union."""
    if isinstance(col, (StructColumn, UnionColumn)):
        return True
    if isinstance(col, (ListColumn, FixedSizeListColumn)):
        return _new(col.child)
    return False


def _row_ids(col):
    """The list `col` over an Int64 child of row ids (0 .. child length)."""
    ids = HostArray.from_numpy(abi.I64, np.arange(col.child.length, dtype=np.int64))
    if isinstance(col, FixedSizeListColumn):
        return FixedSizeListColumn(col.size, ids, col.nulls)
    return ListColumn(col.offsets, ids, col.nulls)


def _with_child(r, child):
    if isinstance(r, FixedSizeListColumn):
        return FixedSizeListColumn(r.size, child, r.nulls)
    return ListColumn(r.offsets, child, r.nulls)


# ---- filter -------------------------------------------------------------------------------------------------------------
def filter(col, mask, child_step=None):
    """filter(col, predicate) with mask = ol.filter_mask(predicate); child_step as in oracle_list.filter."""
    n = len(mask)
    if not _new(col):
        return ol.filter(col, mask, child_step)
    if n > col.length:
        raise OracleError(abi.ERR_INVALID_ARGUMENT, f"Filter predicate of length {n} is larger than target array of length {col.length}")
    rows = [i for i in range(n) if mask[i]]
    count = len(rows)
    if isinstance(col, (ListColumn, FixedSizeListColumn)):
        r = ol.filter(_row_ids(col), mask, child_step)
        if isinstance(col, FixedSizeListColumn):
            clen = n * col.size
        else:
            clen = int(col.offsets[n]) if n else int(col.offsets[0])
        cmask = np.zeros(clen, dtype=bool)
        cmask[r.child.value_array().astype(np.int64)] = True
        step = child_step if child_step is not None else count != n
        return _with_child(r, filter(col.child, cmask, step))
    if isinstance(col, StructColumn):
        fields = [filter(f, mask, child_step) for f in col.fields]
        vm = col.nulls.valid_mask()
        out_mask = [bool(vm[r]) for r in rows]
        if count == 0:
            present = False
        elif count == n and not child_step:  # IterationStrategy::All: values.slice(0, count) keeps the NullBuffer
            present = col.nulls.validity is not None
        else:  # filter_nulls, or MutableArrayData's freeze: a NullBuffer only with a null
            present = not all(out_mask)
        return StructColumn(fields, ol._nulls(out_mask, present))
    # union
    if not col.dense:
        children = [filter(c, mask, child_step) for c in col.children]
        return UnionColumn(col.mode, col.field_type_ids, children, col.type_ids[rows])
    if not child_step and count == 0:
        return acu.empty_column(col)
    if not child_step and count == n:
        return col.slice(0, count)  # a dense slice keeps its children whole
    # build_extend_dense: per row the type id, the child's current length as offset, the child extended by one row
    tids = [int(col.type_ids[r]) for r in rows]
    lens = {t: 0 for t in col.field_type_ids}
    offs, child_rows = [], {t: [] for t in col.field_type_ids}
    for r, t in zip(rows, tids):
        offs.append(lens[t])
        lens[t] += 1
        child_rows[t].append(int(col.offsets[r]))
    children = [take(c, child_rows[t], [True] * len(child_rows[t]), False, abi.I32, False, True)
                for t, c in zip(col.field_type_ids, col.children)]
    return UnionColumn(col.mode, col.field_type_ids, children, np.array(tids, np.int8), np.array(offs, np.int32))


# ---- take ---------------------------------------------------------------------------------------------------------------
def _check_bounds(n, idx, idx_valid):
    """TakeOptions{check_bounds: true} (take.rs:167-209), as oracle_list.take states it."""
    for j in range(len(idx)):
        if not idx_valid[j] and not all(idx_valid):
            continue
        v = int(idx[j])
        if v >= n or (v < 0 and all(idx_valid)):
            raise OracleError(abi.ERR_COMPUTE, f"Array index out of bounds, cannot get item at index {v} from {n} entries", j)


def _flat_take(col, idx, idx_valid, idx_has_buffer, index_dtype, check_bounds, keep):
    """oracle_list.take of a column without struct or union levels, where a struct field or union child reaches cases the
    list children do not: take_primitive runs take_native before take_nulls (take.rs:405-416), so a valid index past a
    fixed-width column with nulls is take_native's panic; take_bits sets only the valid indices' bits, so a Boolean column's
    value under a null index is false."""
    if check_bounds:
        _check_bounds(col.length, idx, idx_valid)
    if isinstance(col, ViewColumn) or (isinstance(col, HostArray) and col.dtype != BOOL):
        for j, v in enumerate(idx):
            x = ol._to_index(index_dtype, v)
            if idx_valid[j] and x >= col.length:
                raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"Out-of-bounds index {x}", j)
    r = ol.take(col, idx, idx_valid, idx_has_buffer, index_dtype, False, keep)
    if isinstance(r, HostArray) and r.dtype == BOOL and not all(idx_valid):
        bits = r.value_array() & np.asarray(idx_valid, dtype=bool)
        r = HostArray(BOOL, pack_bits(bits), r.length, r.validity, r.validity_offset, 0, r.null_count)
    return r


def take(col, idx, idx_valid, idx_has_buffer, index_dtype=abi.U64, check_bounds=False, keep=False):
    """take(col, indices) as oracle_list.take; keep = the child step of a List take (MutableArrayData::extend)."""
    if not _new(col):
        return _flat_take(col, idx, idx_valid, idx_has_buffer, index_dtype, check_bounds, keep)
    n, m = col.length, len(idx)
    if check_bounds:
        _check_bounds(n, idx, idx_valid)
    ix = [ol._to_index(index_dtype, v) for v in idx]
    if isinstance(col, (ListColumn, FixedSizeListColumn)):
        r = ol.take(_row_ids(col), idx, idx_valid, idx_has_buffer, index_dtype, False, keep)
        ids = [int(x) for x in r.child.value_array()]
        cvalid = [bool(v) for v in r.child.valid_mask()]
        child = take(col.child, ids, cvalid, r.child.validity is not None, abi.U64, False,
                     keep or isinstance(col, ListColumn))
        return _with_child(r, child)
    if isinstance(col, StructColumn):
        fields = [take(f, idx, idx_valid, idx_has_buffer, index_dtype, False, keep) for f in col.fields]
        vm = col.nulls.valid_mask()
        if keep:
            mask = [bool(vm[ix[j]]) for j in range(m)]
            return StructColumn(fields, ol._nulls(mask, not all(mask)))
        has_buf = col.nulls.validity is not None
        mask = []
        for j in range(m):
            if not idx_valid[j]:
                mask.append(False)
            elif has_buf:  # array.is_valid(index): BooleanBuffer::value asserts idx < len
                if ix[j] >= n:
                    raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, BIT_LEN, j)
                mask.append(bool(vm[ix[j]]))
            else:
                mask.append(True)
        # StructArray::try_new drops a NullBuffer without nulls; new_empty_fields keeps it
        return StructColumn(fields, ol._nulls(mask, not all(mask) or not col.fields))
    # union: take_native of the type ids (and offsets): a null index gathers in bounds and gives 0 out of bounds
    tids, offs = [], []
    for j in range(m):
        if ix[j] < n:
            tids.append(int(col.type_ids[ix[j]]))
            offs.append(int(col.offsets[ix[j]]) if col.dense else 0)
        elif idx_valid[j]:
            raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"Out-of-bounds index {ix[j]}", j)
        else:
            tids.append(0)
            offs.append(0)
    if col.dense:
        children = []
        for t, c in zip(col.field_type_ids, col.children):
            sel = [o for o, tt in zip(offs, tids) if tt == t]
            children.append(take(c, sel, [True] * len(sel), False, abi.I32, False, keep))
        counts = [0] * 256
        new_offs = []
        for t in tids:
            new_offs.append(counts[t & 0xFF])
            counts[t & 0xFF] += 1
    else:
        children = [take(c, idx, idx_valid, idx_has_buffer, index_dtype, False, keep) for c in col.children]
    if any(t not in col.field_type_ids for t in tids):
        raise OracleError(abi.ERR_INVALID_ARGUMENT, UNION_TYPE_IDS)
    return UnionColumn(col.mode, col.field_type_ids, children, np.array(tids, np.int8),
                       np.array(new_offs, np.int32) if col.dense else None)


def take_host(col, indices, check_bounds=False):
    """take(col, indices) for a HostArray of indices."""
    vals = indices.value_array()
    return take(col, list(vals), list(indices.valid_mask()), indices.validity is not None, indices.dtype, check_bounds)


# ---- comparison ---------------------------------------------------------------------------------------------------------
def describe(col):
    """oracle_list.describe extended to struct and union levels at any depth."""
    if isinstance(col, StructColumn):
        nulls = None if col.nulls.validity is None else [bool(b) for b in col.nulls.valid_mask()]
        return ("struct", col.length, [describe(f) for f in col.fields], nulls)
    if isinstance(col, UnionColumn):
        return ("union", col.mode, list(col.field_type_ids), [int(x) for x in col.type_ids],
                None if col.offsets is None else [int(x) for x in col.offsets], [describe(c) for c in col.children])
    if isinstance(col, (ListColumn, FixedSizeListColumn)) and _new(col):
        nulls = None if col.nulls.validity is None else [bool(b) for b in col.nulls.valid_mask()]
        if isinstance(col, FixedSizeListColumn):
            return ("fsl", col.size, describe(col.child), nulls)
        return ("list", str(col.offsets.dtype), [int(x) for x in col.offsets], describe(col.child), nulls)
    return ol.describe(col)


def to_pylist(col):
    """Logical values: a struct row is the list of its field values, a union row is [type id, child value]."""
    if isinstance(col, StructColumn):
        vm = col.nulls.valid_mask()
        fields = [to_pylist(f) for f in col.fields]
        return [[f[i] for f in fields] if vm[i] else None for i in range(col.length)]
    if isinstance(col, UnionColumn):
        children = {t: to_pylist(c) for t, c in zip(col.field_type_ids, col.children)}
        out = []
        for i, t in enumerate(col.type_ids):
            t = int(t)
            out.append([t, children[t][int(col.offsets[i]) if col.dense else i]])
        return out
    if isinstance(col, (ListColumn, FixedSizeListColumn)) and _new(col):
        vm = col.nulls.valid_mask()
        child = to_pylist(col.child)
        if isinstance(col, FixedSizeListColumn):
            return [child[i * col.size:(i + 1) * col.size] if vm[i] else None for i in range(col.length)]
        o = [int(x) for x in col.offsets]
        return [child[o[i]:o[i + 1]] if vm[i] else None for i in range(col.length)]
    return ol.to_pylist(col)
