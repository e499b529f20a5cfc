"""Python oracle for filter / take of every column type the device filters and takes, restated over the host column
classes of `acu`: primitive / Boolean / decimal, Utf8, view, FixedSizeBinary, List / LargeList / FixedSizeList, Struct,
sparse / dense Union and RunEndEncoded. It reproduces the physical result the device returns: offsets rebased to 0, the
bytes under null rows, and which levels carry a NullBuffer.

One `filter` and one `take`, one arm per column type; a nested level recurses into its real child whatever its type.
Reference sources: filter.rs:535-677, :946-1054; take.rs:167-209, :270-416, :646-995; arrow-data/src/transform
(MutableArrayData, the List child step); UnionArray::try_new union_array.rs:177-242; FixedSizeBinaryArray::try_new
fixed_size_binary_array.rs:178-201; RunEndBuffer run.rs:232-378.

The FixedSizeBinary arms are numpy, so that they also run at the widths the device tests use. Core's slice-index panics of
the dynamic-length FixedSizeBinary take are pinned as Rust 1.97's `Range<usize>::index` reports them through
`slice_index_fail(start, end, len)`: the start against the length first, then the end, then the order of the range. They
follow core's source for that release; no run of the reference checked them."""
import bisect

import numpy as np

import acu
from acu import (BOOL, DecimalArray, FixedSizeBinaryColumn, FixedSizeListColumn, HostArray, ListColumn, RunEndColumn,
                 StructColumn, UnionColumn, Utf8Column, ViewColumn, pack_bits)
from acu import _abi as abi

EXTEND_OVERFLOW = ("offset overflow: data exceeds the capacity of the offset type. Try splitting into smaller batches or using "
                   "a larger type (e.g. LargeStringArray / LargeBinaryArray instead of StringArray / BinaryArray)")
UNWRAP_NONE = "called `Option::unwrap()` on a `None` value"
BIT_LEN = "assertion failed: idx < self.bit_len"
UNION_TYPE_IDS = "Type Ids values must match one of the field type ids"
NESTED_TEXT = "take of a RunEndEncoded column with nested values is not yet implemented"
R_MAX = {2: 2**15 - 1, 4: 2**31 - 1, 8: 2**63 - 1}
INDEX_MAX = {abi.I8: 2**7 - 1, abi.U8: 2**8 - 1, abi.I16: 2**15 - 1, abi.U16: 2**16 - 1, abi.I32: 2**31 - 1, abi.U32: 2**32 - 1,
             abi.I64: 2**63 - 1, abi.U64: 2**64 - 1}
I32_MAX = 2**31 - 1
U64 = 2**64 - 1
NATIVE_WIDTHS = (1, 2, 4, 8, 16)

# Display of the ArrowError variants filter / take raise (arrow-schema/src/error.rs); a panic has no prefix
_PREFIX = {abi.ERR_INVALID_ARGUMENT: "Invalid argument error: ", abi.ERR_COMPUTE: "Compute error: "}


class OracleError(Exception):
    def __init__(self, status, message, index=-1):
        message = _PREFIX.get(status, "") + message
        super().__init__(message)
        self.status, self.message, self.index = status, message, index


def _below_a_level(col):
    """Context has a RunEndEncoded arm only at the top (filter_run_end / take_run_end): below a struct, union or list level a
    RunEndColumn reaches the flat arm, whose upload fails on it."""
    return AttributeError(f"'{type(col).__name__}' object has no attribute 'dtype'")


# ---- validity -----------------------------------------------------------------------------------------------------------
def nulls_of(mask, bit_offset=0, force=False):
    """A validity-only HostArray of `mask`: a NullBuffer (at `bit_offset`) iff a row is null or `force`."""
    mask = np.asarray(mask, dtype=bool)
    n = len(mask)
    if not force and mask.all():
        return HostArray(abi.U8, np.zeros(0, np.uint8), n, None, 0, 0, 0)
    return HostArray(abi.U8, np.zeros(0, np.uint8), n, pack_bits(mask, bit_offset), bit_offset, 0, int(n - mask.sum()))


def _nulls(col):
    return col if isinstance(col, HostArray) else col.nulls


def valid_mask(col):
    return _nulls(col).valid_mask()


def _has_nulls(col):
    return _nulls(col).validity is not None and not valid_mask(col).all()


# ---- rebuilding the flat types --------------------------------------------------------------------------------------------
def _rebuild(col, rows, mask, present):
    """`col` gathered at logical `rows` (a list of source rows, -1 for a zero slot) for HostArray / DecimalArray / view."""
    nb = nulls_of(mask, force=present)
    if isinstance(col, ViewColumn):
        views = np.zeros((len(rows), 16), np.uint8)
        for k, r in enumerate(rows):
            if r >= 0:
                views[k] = col.views[r]
        return ViewColumn(views, col.buffers, nb)
    n = len(rows)
    if col.dtype == BOOL:
        src = col.value_array()
        out = HostArray(BOOL, pack_bits([bool(src[r]) if r >= 0 else False for r in rows]), n, None, 0, 0, 0)
    else:
        src = np.asarray(col.values[:col.length])
        if isinstance(col, DecimalArray) and col.byte_width == 16:
            src = src.reshape(-1, 2)
        vals = np.zeros((n,) + src.shape[1:], src.dtype)
        for k, r in enumerate(rows):
            if r >= 0:
                vals[k] = src[r]
        out = HostArray(col.dtype, vals, n, None, 0, 0, 0)
    out.validity, out.validity_offset, out.null_count = nb.validity, 0, nb.null_count
    return col.like(out) if isinstance(col, DecimalArray) else out


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
    return Utf8Column(np.array(offs, dtype=ob), np.frombuffer(b"".join(data), dtype=np.uint8).copy(), nulls_of(mask, force=present))


def _fsb(values, valid, n=None):
    """A FixedSizeBinaryColumn of `values` ((rows, W) uint8) with the validity `valid` (None: no NullBuffer); n rows (the
    width-0 length rule can leave n != len(values) only for width 0)."""
    n = len(values) if n is None else n
    return FixedSizeBinaryColumn(np.ascontiguousarray(values, np.uint8).reshape(n, values.shape[1]),
                                 nulls_of(np.ones(n, bool) if valid is None else valid, force=valid is not None))


# ---- filter -------------------------------------------------------------------------------------------------------------
def filter_mask(predicate):
    """prep_null_mask_filter: selected = value & valid."""
    return predicate.value_array() & predicate.valid_mask()


def filter(col, mask, child_step=None):
    """filter(col, predicate) with mask = filter_mask(predicate) (len <= col length). child_step: `col` is a child of a
    list whose top level was filtered with a plan other than All (None at the top level). The reference builds that list
    with MutableArrayData (filter.rs:600), whose freeze keeps a level's NullBuffer only if it has a null
    (arrow-data/src/transform/mod.rs:936), also where this level's own plan selects every row; under a top-level All the
    reference slices every level as it is."""
    if isinstance(col, RunEndColumn):
        return _filter_run_end(col, mask)
    return _filter(col, mask, child_step)


def _filter(col, mask, child_step):
    if isinstance(col, RunEndColumn):
        raise _below_a_level(col)
    n = len(mask)
    if n > col.length:
        raise OracleError(abi.ERR_INVALID_ARGUMENT, f"Filter predicate of length {n} is larger than target array of length {col.length}")
    if isinstance(col, FixedSizeBinaryColumn):
        return _filter_fsb(col, np.asarray(mask, bool), child_step)
    rows = [i for i in range(n) if mask[i]]
    count = len(rows)
    if isinstance(col, UnionColumn):
        return _filter_union(col, mask, rows, child_step)
    vm = valid_mask(col)
    out_mask = [bool(vm[r]) for r in rows]
    if count == 0:
        present = False
    elif count == n and not child_step:  # IterationStrategy::All: values.slice(0, count) keeps the NullBuffer
        present = _nulls(col).validity is not None
    else:  # filter_nulls, or MutableArrayData's freeze: a NullBuffer only with a null
        present = _has_nulls(col) and not all(out_mask)
    step = child_step if child_step is not None else count != n
    if isinstance(col, (HostArray, ViewColumn)):
        return _rebuild(col, rows, out_mask, present)
    if isinstance(col, Utf8Column):
        return _bytes(col, rows, set(), out_mask, present, lambda k: None)
    if isinstance(col, StructColumn):  # filter_struct: the fields with the same plan, then filter_nulls
        return StructColumn([_filter(f, mask, child_step) for f in col.fields], nulls_of(out_mask, force=present))
    if isinstance(col, FixedSizeListColumn):
        cmask = np.zeros(n * col.size, dtype=bool)
        for r in rows:
            cmask[r * col.size:(r + 1) * col.size] = True
        return FixedSizeListColumn(col.size, _filter(col.child, cmask, step), nulls_of(out_mask, force=present))
    offs = [int(x) for x in col.offsets]
    cmask = np.zeros(offs[n] if n else offs[0], dtype=bool)
    new = [0]
    for r in rows:
        cmask[offs[r]:offs[r + 1]] = True
        new.append(new[-1] + offs[r + 1] - offs[r])
    return ListColumn(np.array(new, dtype=col.offsets.dtype), _filter(col.child, cmask, step), nulls_of(out_mask, force=present))


def _filter_union(col, mask, rows, child_step):
    """filter_sparse_union (filter.rs:1033-1054) / the dense MutableArrayData fallback (filter.rs:597-622,
    build_extend_dense)."""
    n, count = len(mask), len(rows)
    if not col.dense:
        children = [_filter(c, mask, child_step) for c in col.children]
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
    children = [_take(c, child_rows[t], [True] * len(child_rows[t]), False, abi.I32, False, True)
                for t, c in zip(col.field_type_ids, col.children)]
    return UnionColumn(col.mode, col.field_type_ids, children, np.array(tids, np.int8), np.array(offs, np.int32))


def _filter_fsb(col, mask, child_step):
    """filter_fixed_size_binary (filter.rs:946-996). child_step: MutableArrayData keeps every row, also of width 0, and
    drops a NullBuffer without nulls."""
    w, plen = col.width, len(mask)
    count = int(mask.sum())
    if count == 0:  # IterationStrategy::None: new_empty_array
        return _fsb(np.zeros((0, w), np.uint8), None)
    v = valid_mask(col)
    has_buffer = col.nulls.validity is not None
    if count == plen:  # IterationStrategy::All: values.slice(0, count) keeps the NullBuffer
        valid = v[:count] if has_buffer else None
        if child_step and valid is not None and valid.all():
            valid = None
        return _fsb(col.values[:count], valid)
    valid = None
    if _has_nulls(col):  # FilterPredicate::filter_nulls
        valid = v[:plen][mask]
        if valid.all():
            valid = None
    length = count if (w > 0 or valid is not None or child_step) else 0  # try_new of width 0
    return _fsb(col.values[:plen][mask][:length], valid, length)


# ---- take ---------------------------------------------------------------------------------------------------------------
def _to_index(dtype, v):
    """ToIndices (take.rs:1030-1084): i8 / i16 sign-extend to u32, i32 is reinterpreted as u32, i64 as u64."""
    v = int(v)
    if dtype in (abi.I8, abi.I16, abi.I32):
        return v & 0xFFFFFFFF
    return v & U64


def _check_bounds(n, idx, idx_valid, dtype):
    """TakeOptions{check_bounds: true} (take.rs:167-209): skipped when the length does not fit the index type
    (from_usize fails); null slots ignored when the indices have a null; a negative index fails only without one."""
    if n > INDEX_MAX[dtype]:
        return
    all_valid = all(idx_valid)
    for j, v in enumerate(idx):
        if not all_valid and not idx_valid[j]:
            continue
        v = int(v)
        if v >= n or (v < 0 and all_valid):  # the nullable path only tests index >= len (take.rs:183)
            raise OracleError(abi.ERR_COMPUTE, f"Array index out of bounds, cannot get item at index {v} from {n} entries", j)


def take(col, idx, idx_valid, idx_has_buffer, index_dtype=abi.U64, check_bounds=False, keep=False):
    """take(col, indices): idx = raw index values, idx_valid = their validity, idx_has_buffer = the indices carry a
    NullBuffer. keep = the child step of a List take (MutableArrayData::extend)."""
    if isinstance(col, RunEndColumn):
        return _take_run_end(col, idx, idx_valid, index_dtype, check_bounds)
    return _take(col, idx, idx_valid, idx_has_buffer, index_dtype, check_bounds, keep)


def take_host(col, indices, check_bounds=False):
    """take(col, indices) for a HostArray of indices."""
    return take(col, list(indices.value_array()), list(indices.valid_mask()), indices.validity is not None, indices.dtype,
                check_bounds)


def _take(col, idx, idx_valid, idx_has_buffer, index_dtype, check_bounds, keep):
    if isinstance(col, RunEndColumn):
        raise _below_a_level(col)
    n, m = col.length, len(idx)
    if check_bounds:
        _check_bounds(n, idx, idx_valid, index_dtype)
    ix = [_to_index(index_dtype, v) for v in idx]
    if isinstance(col, FixedSizeBinaryColumn):
        return _take_fsb(col, ix, idx_valid, idx_has_buffer, keep)
    if isinstance(col, UnionColumn):
        return _take_union(col, idx, ix, idx_valid, idx_has_buffer, index_dtype, keep)
    vm = valid_mask(col)
    col_nulls = _has_nulls(col)
    idx_nulls = not all(idx_valid)

    def take_nulls_mask():
        if col_nulls:
            for j in range(m):
                if idx_valid[j] and ix[j] >= n:
                    raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, BIT_LEN, j)
            mask = [bool(idx_valid[j] and vm[ix[j]]) for j in range(m)]
            return mask, not all(mask)
        return [bool(v) for v in idx_valid], idx_has_buffer

    if isinstance(col, StructColumn):
        # take_impl's Struct arm (take.rs:270-298): the fields first, then the validity
        fields = [_take(f, idx, idx_valid, idx_has_buffer, index_dtype, False, keep) for f in col.fields]
        if keep:
            mask = [bool(vm[ix[j]]) for j in range(m)]
            return StructColumn(fields, nulls_of(mask, force=not all(mask)))
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
        return StructColumn(fields, nulls_of(mask, force=not all(mask) or not col.fields))
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
        child = _take(col.child, cidx, cvalid, idx_nulls and col.size > 0, abi.U32, False, keep)
        take_nulls_mask()
        return FixedSizeListColumn(col.size, child, nulls_of(mask, force=not all(mask)))
    if isinstance(col, ListColumn):
        offs = [int(x) for x in col.offsets]
        if keep:
            mask = [bool(vm[ix[j]]) for j in range(m)]
            present = col_nulls and not all(mask)
        else:
            mask, present = take_nulls_mask()
        new, cidx, pos = [0], [], 0
        for j in range(m):
            if idx_valid[j] and (keep or mask[j]):
                if ix[j] >= n:
                    raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS,
                                      f"index out of bounds: the len is {n + 1} but the index is {ix[j] + 1 if ix[j] == n else ix[j]}", j)
                s, e = offs[ix[j]], offs[ix[j] + 1]
                cidx.extend(range(s, e))
                pos += e - s
                if col.offsets.dtype == np.int32 and pos > I32_MAX:
                    # the child of this row is extended first: its own overflow wins
                    _take(col.child, cidx, [True] * len(cidx), False, abi.U64, False, True)
                    if keep:
                        raise OracleError(abi.ERR_INVALID_ARGUMENT, EXTEND_OVERFLOW, j)
                    raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, UNWRAP_NONE, j)
            new.append(pos)
        child = _take(col.child, cidx, [True] * len(cidx), False, abi.U64, False, True)
        return ListColumn(np.array(new, dtype=col.offsets.dtype), child, nulls_of(mask, force=present))
    if isinstance(col, Utf8Column):
        if keep:
            mask = [bool(vm[ix[j]]) for j in range(m)]

            def ovf(k):
                raise OracleError(abi.ERR_INVALID_ARGUMENT, EXTEND_OVERFLOW, k)
            return _bytes(col, ix, set(), mask, col_nulls and not all(mask), ovf)
        mask, present = take_nulls_mask()

        def ovf2(k):
            raise OracleError(abi.ERR_OFFSET_OVERFLOW, "offset overflow", k)
        for j in range(m):
            if idx_valid[j] and ix[j] >= n:
                raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"Out-of-bounds index {ix[j]}", j)
        rows = [ix[j] if idx_valid[j] else -1 for j in range(m)]
        return _bytes(col, rows, {j for j in range(m) if not mask[j]}, mask, present, ovf2)
    # primitive / decimal / view: take_native, then take_nulls (take.rs:405-416); Boolean: take_nulls, then take_bits,
    # which sets only the valid indices' bits
    boolean = isinstance(col, HostArray) and col.dtype == BOOL
    bad = next((j for j in range(m) if idx_valid[j] and ix[j] >= n), None)
    if bad is not None and not boolean:
        raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"Out-of-bounds index {ix[bad]}", bad)
    mask, present = take_nulls_mask()
    if bad is not None:
        raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"Out-of-bounds index {ix[bad]}", bad)
    rows = [ix[j] if ix[j] < n and (idx_valid[j] or not boolean) else -1 for j in range(m)]
    return _rebuild(col, rows, mask, present)


def _take_union(col, idx, ix, idx_valid, idx_has_buffer, index_dtype, keep):
    """take_impl's Union arm (take.rs:334-382): take_native of the type ids (and offsets): a null index gathers in bounds
    and gives 0 out of bounds; UnionArray::try_new validates after the children are taken."""
    n, m = col.length, len(ix)
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
    new_offs = None
    if col.dense:
        children = []
        for t, c in zip(col.field_type_ids, col.children):
            sel = [o for o, tt in zip(offs, tids) if tt == t]
            children.append(_take(c, sel, [True] * len(sel), False, abi.I32, False, keep))
        counts = [0] * 256
        new_offs = []
        for t in tids:
            new_offs.append(counts[t & 0xFF])
            counts[t & 0xFF] += 1
        new_offs = np.array(new_offs, np.int32)
    else:
        children = [_take(c, idx, idx_valid, idx_has_buffer, index_dtype, False, keep) for c in col.children]
    if any(t not in col.field_type_ids for t in tids):
        raise OracleError(abi.ERR_INVALID_ARGUMENT, UNION_TYPE_IDS)
    return UnionColumn(col.mode, col.field_type_ids, children, np.array(tids, np.int8), new_offs)


def _take_fsb(col, x, idx_valid, idx_buffer, keep):
    """take_fixed_size_binary (take.rs:802-862) at the ToIndices values x. keep: MutableArrayData keeps every row, also of
    width 0."""
    idx_valid = np.asarray(idx_valid, bool)
    m, n, w = len(x), col.length, col.width
    idx_nulls = idx_buffer and not idx_valid.all()
    flat = col.values.reshape(-1)
    out = np.zeros((m, w), np.uint8)
    nbytes = n * w
    for j in range(m):
        if w in NATIVE_WIDTHS:  # take_fixed_size: take_native byte for byte
            if x[j] < n:
                out[j] = col.values[x[j]]
            elif idx_valid[j] or not idx_nulls:
                raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"Out-of-bounds index {x[j]}", j)
        else:  # take_fixed_size_binary_buffer_dynamic_length: usize arithmetic wraps
            if idx_nulls and not idx_valid[j]:
                continue
            s = (x[j] * w) & U64
            e = (s + w) & U64
            if s > nbytes:
                raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"range start index {s} out of range for slice of length {nbytes}", j)
            if e > nbytes:
                raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"range end index {e} out of range for slice of length {nbytes}", j)
            if s > e:
                raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"slice index starts at {s} but ends at {e}", j)
            out[j] = flat[s:e]
    # NullBuffer::union(take_nulls(values.nulls(), indices), indices.nulls())
    valid = idx_valid.copy() if idx_nulls else np.ones(m, bool)
    if _has_nulls(col):
        v = valid_mask(col)
        for j in range(m):
            if idx_nulls and not idx_valid[j]:
                continue
            if x[j] >= n:  # take_bits: BooleanBuffer::value
                raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, BIT_LEN, j)
            valid[j] = valid[j] and v[x[j]]
    has = not valid.all()
    length = m if (w > 0 or has or keep) else 0
    return _fsb(out[:length], valid[:length] if has else None, length)


# ---- RunEndEncoded (filter_run_end_array filter.rs:628-677, take_run take.rs:948-995) ----------------------------------
# Only at the top level: the values child is filtered / taken through the same arms as any column.
def empty_run_end(col):
    return RunEndColumn(np.zeros(0, col.run_ends.dtype), acu.empty_column(col.values), 0, 0)


def physical_index(col, i):
    """RunEndBuffer::get_physical_index: binary_search of offset + i over the run ends, Ok(idx) -> idx + 1, Err(idx) -> idx."""
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


def _filter_run_end(col, mask):
    mask = np.asarray(mask, dtype=bool)
    p = len(mask)
    if p > col.length:
        raise OracleError(abi.ERR_INVALID_ARGUMENT, f"Filter predicate of length {p} is larger than target array of length {col.length}")
    count = int(mask.sum())
    if count == 0:  # IterationStrategy::None: new_empty_array
        return empty_run_end(col)
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
    values = _filter(values_slice(col), np.array(keep, dtype=bool), None)
    return RunEndColumn(np.array(new_ends, dtype=col.run_ends.dtype), values, 0, new_ends[-1])


def get_physical_indices(col, ix):
    """ix: ToIndices values (null slots included). The largest at or past the length is the error's index."""
    if not ix:
        return []
    mx = max(ix)
    if mx >= col.length:
        raise OracleError(abi.ERR_INVALID_ARGUMENT, f"Logical index {mx} is out of bounds for RunArray of length {col.length}")
    ends = [int(x) for x in col.run_ends]
    return [bisect.bisect_right(ends, col.offset + x) for x in ix]  # the first run whose end - offset > x


def _comparator(v):
    """make_comparator(values, values, SortOptions::default()): (a, b) -> is_eq()."""
    vm = valid_mask(v)
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


# The value types whose runs the device does not merge (Context._run_values marks them RUN_VALUES_NESTED). The reference's
# make_comparator handles Struct and FixedSizeBinary values; refusing them is a limit of this device.
_RUN_VALUES_NESTED = (ListColumn, FixedSizeListColumn, RunEndColumn, StructColumn, UnionColumn, FixedSizeBinaryColumn)


def _take_run_end(col, idx, idx_valid, index_dtype, check_bounds):
    if check_bounds:
        _check_bounds(col.length, idx, idx_valid, index_dtype)
    if not len(idx):
        return empty_run_end(col)
    wide = index_dtype in (abi.I64, abi.U64)
    phys = get_physical_indices(col, [_to_index(index_dtype, v) for v in idx])
    if isinstance(col.values, _RUN_VALUES_NESTED):  # where take_run builds its comparator
        raise OracleError(abi.ERR_NOT_YET_IMPLEMENTED, "Not yet implemented: " + NESTED_TEXT)
    r_max, i_max = R_MAX[col.run_ends.itemsize], 2**64 - 1 if wide else 2**32 - 1
    new_ends, value_idx = [], []

    def push(ix, end):
        if ix > i_max or end > r_max:  # I::Native / T::Native::from_usize(..).unwrap()
            raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, UNWRAP_NONE)
        value_idx.append(ix)
        new_ends.append(end)

    eq = _comparator(col.values)
    for q in range(1, len(phys)):
        if phys[q] != phys[q - 1] and not eq(phys[q], phys[q - 1]):
            push(phys[q - 1], q)
    push(phys[-1], len(phys))
    values = _take(col.values, value_idx, [True] * len(value_idx), False, abi.U64 if wide else abi.U32, False, False)
    return RunEndColumn(np.array(new_ends, dtype=col.run_ends.dtype), values, 0, len(phys))


# ---- comparison ---------------------------------------------------------------------------------------------------------
def describe(col):
    """Every physical fact the device must reproduce, as plain Python data: offsets, values (bytes under nulls
    included), validity bits and NullBuffer presence at every level."""
    if isinstance(col, RunEndColumn):
        return ("ree", str(col.run_ends.dtype), [int(x) for x in col.run_ends], col.offset, col.length, describe(col.values))
    if isinstance(col, UnionColumn):
        return ("union", col.mode, list(col.field_type_ids), [int(x) for x in col.type_ids],
                None if col.offsets is None else [int(x) for x in col.offsets], [describe(c) for c in col.children])
    nulls = None if _nulls(col).validity is None else [bool(b) for b in valid_mask(col)]
    if isinstance(col, HostArray):
        if col.dtype == BOOL:
            vals = [bool(v) for v in col.value_array()]
        elif isinstance(col, DecimalArray):
            vals = col.raw_ints()
        else:
            vals = np.asarray(col.values[:col.length]).view(np.uint8).tolist()
        return ("flat", col.length, vals, nulls)
    if isinstance(col, FixedSizeBinaryColumn):
        return ("fsb", col.width, col.length, col.values.tobytes(), nulls, col.nulls.null_count if nulls is not None else 0)
    if isinstance(col, Utf8Column):
        s, e = int(col.offsets[0]), int(col.offsets[-1])
        return ("bytes", [int(x) - s for x in col.offsets], bytes(col.data[s:e]), nulls)
    if isinstance(col, ViewColumn):
        vm = valid_mask(col)
        return ("view", [bytes(col.views[i]) for i in range(col.length)], [acu.column_value(col, i) if vm[i] else None
                                                                          for i in range(col.length)], nulls)
    if isinstance(col, StructColumn):
        return ("struct", col.length, [describe(f) for f in col.fields], nulls)
    if isinstance(col, FixedSizeListColumn):
        return ("fsl", col.size, describe(col.child), nulls)
    return ("list", str(col.offsets.dtype), [int(x) for x in col.offsets], describe(col.child), nulls)


def to_pylist(col):
    """Logical values (None for nulls): a struct row is the list of its field values, a union row is [type id, child
    value], a FixedSizeBinary row its bytes."""
    if isinstance(col, RunEndColumn):
        return logical(col)
    if isinstance(col, UnionColumn):
        children = {t: to_pylist(c) for t, c in zip(col.field_type_ids, col.children)}
        return [[int(t), children[int(t)][int(col.offsets[i]) if col.dense else i]] for i, t in enumerate(col.type_ids)]
    if isinstance(col, HostArray):
        return col.to_list()
    vm = valid_mask(col)
    if isinstance(col, (Utf8Column, ViewColumn)):
        return [acu.column_value(col, i) if vm[i] else None for i in range(col.length)]
    if isinstance(col, FixedSizeBinaryColumn):
        return [bytes(col.values[i]) if vm[i] else None for i in range(col.length)]
    if isinstance(col, StructColumn):
        fields = [to_pylist(f) for f in col.fields]
        return [[f[i] for f in fields] if vm[i] else None for i in range(col.length)]
    child = to_pylist(col.child)
    if isinstance(col, FixedSizeListColumn):
        return [child[i * col.size:(i + 1) * col.size] if vm[i] else None for i in range(col.length)]
    o = [int(x) for x in col.offsets]
    return [child[o[i]:o[i + 1]] if vm[i] else None for i in range(col.length)]


def logical(col):
    """The logical values of a RunEndColumn (None for nulls)."""
    vals = to_pylist(col.values)
    ends = [int(x) for x in col.run_ends]
    return [vals[bisect.bisect_right(ends, col.offset + i)] for i in range(col.length)]
