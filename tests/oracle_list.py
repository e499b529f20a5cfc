"""Python oracle for filter / take of List, LargeList and FixedSizeList columns (arrow-select/src/filter.rs:535-625,
take.rs:646-795, arrow-data/src/transform/{list,fixed_size_list,variable_size,utils}.rs), restated over the host column
classes of `acu`. It reproduces the physical result the device returns: offsets rebased to 0, the bytes under null rows,
and which levels carry a NullBuffer.

Columns: HostArray / DecimalArray (primitive, boolean), Utf8Column, ViewColumn, ListColumn, FixedSizeListColumn."""
import numpy as np

import acu
from acu import BOOL, DecimalArray, FixedSizeListColumn, HostArray, ListColumn, Utf8Column, ViewColumn, pack_bits
from acu import _abi as abi

EXTEND_OVERFLOW = ("offset overflow: data exceeds the capacity of the offset type. Try splitting into smaller batches or using "
                   "a larger type (e.g. LargeStringArray / LargeBinaryArray instead of StringArray / BinaryArray)")
UNWRAP_NONE = "called `Option::unwrap()` on a `None` value"
I32_MAX = 2**31 - 1


# Display of the ArrowError variants the list calls raise (arrow-schema/src/error.rs); a panic has no prefix
_PREFIX = {abi.ERR_INVALID_ARGUMENT: "Invalid argument error: ", abi.ERR_COMPUTE: "Compute error: "}


class OracleError(Exception):
    def __init__(self, status, message, index=-1):
        message = _PREFIX.get(status, "") + message
        super().__init__(message)
        self.status, self.message, self.index = status, message, index


def length(col):
    return col.length


def valid_mask(col):
    nulls = col if isinstance(col, HostArray) else col.nulls
    return nulls.valid_mask()


def _has_nulls(col):
    nulls = col if isinstance(col, HostArray) else col.nulls
    return nulls.validity is not None and not valid_mask(col).all()


def _nulls(mask, present):
    """A validity-only HostArray of `mask`, with a bitmap iff `present`."""
    mask = np.asarray(mask, dtype=bool)
    n = len(mask)
    h = HostArray(abi.U8, np.zeros(0, np.uint8), n, pack_bits(mask) if present else None, 0, 0, int(n - mask.sum()) if present else 0)
    return h


def _rebuild(col, rows, mask, present, fill_zero=None):
    """`col` gathered at logical `rows` (a list of source rows, -1 for a zero slot) for the flat types."""
    if isinstance(col, HostArray):
        n = len(rows)
        if col.dtype == BOOL:
            src = col.value_array()
            vals = [bool(src[r]) if r >= 0 else False for r in rows]
            out = HostArray(BOOL, pack_bits(vals), n, None, 0, 0, 0)
        elif isinstance(col, DecimalArray) and col.byte_width == 16:
            src = np.asarray(col.values[:col.length]).reshape(-1, 2)
            vals = np.zeros((n, 2), np.uint64)
            for k, r in enumerate(rows):
                if r >= 0:
                    vals[k] = src[r]
            out = HostArray(col.dtype, vals, n, None, 0, 0, 0)
        else:
            src = np.asarray(col.values[:col.length])
            vals = np.zeros(n, src.dtype)
            for k, r in enumerate(rows):
                if r >= 0:
                    vals[k] = src[r]
            out = HostArray(col.dtype, vals, n, None, 0, 0, 0)
        nb = _nulls(mask, present)
        out.validity, out.validity_offset, out.null_count = nb.validity, 0, nb.null_count
        return col.like(out) if isinstance(col, DecimalArray) else out
    if isinstance(col, ViewColumn):
        views = np.zeros((len(rows), 16), np.uint8)
        for k, r in enumerate(rows):
            if r >= 0:
                views[k] = col.views[r]
        return ViewColumn(views, col.buffers, _nulls(mask, present))
    raise TypeError(type(col))


def _bytes(col, rows, lens_zero, mask, present, overflow):
    """Utf8Column gathered at `rows`; rows in lens_zero get no bytes. overflow(row) raises for i32 overflow."""
    ob = col.offsets.dtype
    offs, data, pos = [0], [], 0
    for k, r in enumerate(rows):
        if r >= 0 and k not in lens_zero:
            s, e = int(col.offsets[r]), int(col.offsets[r + 1])
            pos += e - s
            if ob == np.int32 and pos > I32_MAX:
                overflow(k)
            data.append(bytes(col.data[s:e]))
        offs.append(pos)
    return Utf8Column(np.array(offs, dtype=ob), np.frombuffer(b"".join(data), dtype=np.uint8).copy(), _nulls(mask, present))


# ---- filter -----------------------------------------------------------------------------------------------------------
def filter_mask(predicate):
    """prep_null_mask_filter: selected = value & valid."""
    return predicate.value_array() & predicate.valid_mask()


def filter(col, mask, child_step=None):
    """filter(col, predicate) with mask = filter_mask(predicate) (len <= col length). child_step: `col` is a child of a
    list whose top level was filtered with a plan other than All (None at the top level). The reference builds that list
    with MutableArrayData (filter.rs:600), whose freeze keeps a level's NullBuffer only if it has a null
    (arrow-data/src/transform/mod.rs:936), also where this level's own plan selects every row; under a top-level All the
    reference slices every level as it is."""
    n = len(mask)
    if n > length(col):
        raise OracleError(abi.ERR_INVALID_ARGUMENT, f"Filter predicate of length {n} is larger than target array of length {length(col)}")
    rows = [i for i in range(n) if mask[i]]
    count = len(rows)
    vm = valid_mask(col)
    out_mask = [bool(vm[r]) for r in rows]
    nulls_as_is = col.validity is not None if isinstance(col, HostArray) else col.nulls.validity is not None
    if count == 0:
        present = False
    elif count == n and not child_step:  # IterationStrategy::All: the slice keeps its NullBuffer
        present = nulls_as_is
    else:
        present = _has_nulls(col) and not all(out_mask)
    step = child_step if child_step is not None else count != n
    if isinstance(col, (HostArray, ViewColumn)):
        return _rebuild(col, rows, out_mask, present)
    if isinstance(col, Utf8Column):
        return _bytes(col, rows, set(), out_mask, present, lambda k: None)
    if isinstance(col, FixedSizeListColumn):
        cmask = np.zeros(n * col.size, dtype=bool)
        for r in rows:
            cmask[r * col.size:(r + 1) * col.size] = True
        return FixedSizeListColumn(col.size, filter(col.child, cmask, step), _nulls(out_mask, present))
    offs = [int(x) for x in col.offsets]
    cmask = np.zeros(offs[n] if n else offs[0], dtype=bool)
    new = [0]
    for r in rows:
        cmask[offs[r]:offs[r + 1]] = True
        new.append(new[-1] + offs[r + 1] - offs[r])
    return ListColumn(np.array(new, dtype=col.offsets.dtype), filter(col.child, cmask, step), _nulls(out_mask, present))


# ---- take ---------------------------------------------------------------------------------------------------------------
def _to_index(dtype, v):
    """ToIndices: i8 / i16 sign-extend to u32, i32 / i64 reinterpret."""
    v = int(v)
    if dtype in (abi.I8, abi.I16, abi.I32):
        return v & 0xFFFFFFFF
    return v & 0xFFFFFFFFFFFFFFFF


def take(col, idx, idx_valid, idx_has_buffer, index_dtype=abi.U64, check_bounds=False, keep=False):
    """take(col, indices): idx = raw index values, idx_valid = their validity, idx_has_buffer = the indices carry a
    NullBuffer. keep = the child step of a List take (MutableArrayData::extend)."""
    n, m = length(col), len(idx)
    ix = [_to_index(index_dtype, v) for v in idx]
    if check_bounds:
        for j in range(m):
            if not idx_valid[j] and not all(idx_valid):
                continue
            v = int(idx[j])
            if v >= n or (v < 0 and all(idx_valid)):  # the nullable path only tests index >= len (take.rs:183)
                raise OracleError(abi.ERR_COMPUTE, f"Array index out of bounds, cannot get item at index {v} from {n} entries", j)
    vm = valid_mask(col)
    col_nulls = _has_nulls(col)
    idx_nulls = not all(idx_valid)

    def take_nulls_mask():
        if col_nulls:
            for j in range(m):
                if idx_valid[j] and ix[j] >= n:
                    raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, "assertion failed: idx < self.bit_len", j)
            mask = [bool(idx_valid[j] and vm[ix[j]]) for j in range(m)]
            return mask, not all(mask)
        return [bool(v) for v in idx_valid], idx_has_buffer

    if isinstance(col, FixedSizeListColumn):
        mask = [bool(idx_valid[j] and (ix[j] >= n or vm[ix[j]])) for j in range(m)]
        cidx, cvalid = [], []
        for j in range(m):
            for k in range(col.size):
                if idx_valid[j]:
                    cidx.append(((ix[j] * col.size) + k) & 0xFFFFFFFF)
                    cvalid.append(True)
                else:
                    cidx.append(0)
                    cvalid.append(False)
        # take_fixed_size_list takes the child before it reads the list's validity (take.rs:770-785)
        child = take(col.child, cidx, cvalid, idx_nulls and col.size > 0, abi.U32, False, keep)
        take_nulls_mask()
        return FixedSizeListColumn(col.size, child, _nulls(mask, not all(mask)))
    if isinstance(col, ListColumn):
        offs = [int(x) for x in col.offsets]
        if keep:
            mask, present = [bool(vm[ix[j]]) for j in range(m)], col_nulls
            present = present and not all(mask)
        else:
            mask, present = take_nulls_mask()
        new, cidx, pos = [0], [], 0
        for j in range(m):
            live = idx_valid[j] and (keep or mask[j])
            if live:
                if ix[j] >= n:
                    raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS,
                                      f"index out of bounds: the len is {n + 1} but the index is {ix[j] + 1 if ix[j] == n else ix[j]}", j)
                s, e = offs[ix[j]], offs[ix[j] + 1]
                cidx.extend(range(s, e))
                pos += e - s
                if col.offsets.dtype == np.int32 and pos > I32_MAX:
                    # the child of this row is extended first: its own overflow wins
                    take(col.child, cidx, [True] * len(cidx), False, abi.U64, False, True)
                    if keep:
                        raise OracleError(abi.ERR_INVALID_ARGUMENT, EXTEND_OVERFLOW, j)
                    raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, UNWRAP_NONE, j)
            new.append(pos)
        child = take(col.child, cidx, [True] * len(cidx), False, abi.U64, False, True)
        return ListColumn(np.array(new, dtype=col.offsets.dtype), child, _nulls(mask, present))
    if isinstance(col, Utf8Column):
        if keep:
            mask = [bool(vm[ix[j]]) for j in range(m)]

            def ovf(k):
                raise OracleError(abi.ERR_INVALID_ARGUMENT, EXTEND_OVERFLOW, k)
            return _bytes(col, ix, set(), mask, col_nulls and not all(mask), ovf)
        mask, present = take_nulls_mask()

        def ovf2(k):
            raise OracleError(abi.ERR_OFFSET_OVERFLOW, "offset overflow", k)
        rows = [ix[j] if idx_valid[j] else -1 for j in range(m)]
        for j in range(m):
            if idx_valid[j] and ix[j] >= n:
                raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"Out-of-bounds index {ix[j]}", j)
        return _bytes(col, rows, {j for j in range(m) if not mask[j]}, mask, present, ovf2)
    # primitive / boolean / decimal / view: take_native + take_nulls
    mask, present = take_nulls_mask()
    rows = []
    for j in range(m):
        if ix[j] < n:
            rows.append(ix[j])
        elif idx_valid[j]:
            raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"Out-of-bounds index {ix[j]}", j)
        else:
            rows.append(-1)
    return _rebuild(col, rows, mask, present)


def take_host(col, indices, check_bounds=False):
    """take(col, indices) for a HostArray of indices."""
    vals = indices.value_array()
    return take(col, list(vals), list(indices.valid_mask()), indices.validity is not None, indices.dtype, check_bounds)


# ---- comparison ---------------------------------------------------------------------------------------------------------
def describe(col):
    """Every physical fact the device must reproduce, as plain Python data: offsets, values (bytes under nulls
    included), validity bits and NullBuffer presence at every level."""
    if isinstance(col, HostArray):
        nulls = None if col.validity is None else [bool(b) for b in col.valid_mask()]
        if col.dtype == BOOL:
            vals = [bool(v) for v in col.value_array()]
        elif isinstance(col, DecimalArray):
            vals = col.raw_ints()
        else:
            vals = np.asarray(col.values[:col.length]).view(np.uint8).tolist()
        return ("flat", col.length, vals, nulls)
    nulls = None if col.nulls.validity is None else [bool(b) for b in col.nulls.valid_mask()]
    if isinstance(col, Utf8Column):
        s, e = int(col.offsets[0]), int(col.offsets[-1])
        return ("bytes", [int(x) - s for x in col.offsets], bytes(col.data[s:e]), nulls)
    if isinstance(col, ViewColumn):
        vm = col.nulls.valid_mask()
        return ("view", [bytes(col.views[i]) for i in range(col.length)], [acu.column_value(col, i) if vm[i] else None
                                                                          for i in range(col.length)], nulls)
    if isinstance(col, FixedSizeListColumn):
        return ("fsl", col.size, describe(col.child), nulls)
    return ("list", str(col.offsets.dtype), [int(x) for x in col.offsets], describe(col.child), nulls)


def to_pylist(col):
    """Logical values (None for nulls) of a column, for the reference's literal cases."""
    if isinstance(col, HostArray):
        return col.to_list()
    vm = col.nulls.valid_mask()
    if isinstance(col, (Utf8Column, ViewColumn)):
        return [acu.column_value(col, i) if vm[i] else None for i in range(col.length)]
    child = to_pylist(col.child)
    if isinstance(col, FixedSizeListColumn):
        return [child[i * col.size:(i + 1) * col.size] if vm[i] else None for i in range(col.length)]
    o = [int(x) for x in col.offsets]
    return [child[o[i]:o[i + 1]] if vm[i] else None for i in range(col.length)]
