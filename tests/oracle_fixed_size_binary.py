"""Python oracle for filter / take of FixedSizeBinary columns (filter_fixed_size_binary filter.rs:946-996,
take_fixed_size_binary take.rs:802-862, FixedSizeBinaryArray::try_new fixed_size_binary_array.rs:178-201), restated with
numpy over acu.FixedSizeBinaryColumn so that it also runs at the sizes the device tests use.

Core's slice-index panics of the dynamic-length take are pinned as Rust 1.97's `Range<usize>::index` reports them through
`slice_index_fail(start, end, len)`: the start against the length first ("range start index {s} out of range for slice of
length {len}"), then the end ("range end index {e} out of range for slice of length {len}"), then the order of the range
("slice index starts at {s} but ends at {e}"). They follow core's source for that release; no run of the reference checked
them."""
import numpy as np

from acu import FixedSizeBinaryColumn, HostArray, pack_bits
from acu import _abi as abi

from oracle_list import OracleError

BIT_LEN = "assertion failed: idx < self.bit_len"
NATIVE_WIDTHS = (1, 2, 4, 8, 16)
U64 = (1 << 64) - 1


def valid_mask(col):
    return col.nulls.valid_mask() if col.nulls.validity is not None else np.ones(col.length, bool)


def has_buffer(col):
    return col.nulls.validity is not None


def null_count(col):
    return int(col.length - valid_mask(col).sum()) if has_buffer(col) else 0


def column(values, valid, n=None):
    """A FixedSizeBinaryColumn of `values` ((rows, W) uint8) with the validity `valid` (None: no NullBuffer); n rows (the
    width-0 length rule can leave n != len(values) only for width 0)."""
    n = len(values) if n is None else n
    if valid is None:
        nulls = HostArray(abi.U8, np.zeros(0, np.uint8), n, None, 0, 0, 0)
    else:
        valid = np.asarray(valid, bool)
        nulls = HostArray(abi.U8, np.zeros(0, np.uint8), n, pack_bits(valid), 0, 0, int(n - valid.sum()))
    return FixedSizeBinaryColumn(np.ascontiguousarray(values, np.uint8).reshape(n, values.shape[1]), nulls)


def _empty(w):
    return column(np.zeros((0, w), np.uint8), None)


def filter(col, mask, child_step=False):
    """filter(col, predicate) with mask = oracle_list.filter_mask(predicate). child_step: the child of a list filtered with
    a plan that is not All (MutableArrayData: every row kept, a NullBuffer without nulls dropped)."""
    mask = np.asarray(mask, bool)
    n, w, plen = col.length, col.width, len(mask)
    if plen > n:
        raise OracleError(abi.ERR_INVALID_ARGUMENT, f"Filter predicate of length {plen} is larger than target array of length {n}")
    count = int(mask.sum())
    if count == 0:  # IterationStrategy::None: new_empty_array
        return _empty(w)
    v = valid_mask(col)
    if count == plen:  # IterationStrategy::All: values.slice(0, count) keeps the NullBuffer
        valid = v[:count] if has_buffer(col) else None
        if child_step and valid is not None and valid.all():
            valid = None
        return column(col.values[:count], valid)
    valid = None
    if has_buffer(col) and null_count(col) > 0:  # FilterPredicate::filter_nulls
        valid = v[:plen][mask]
        if valid.all():
            valid = None
    length = count if (w > 0 or valid is not None or child_step) else 0  # try_new of width 0
    return column(col.values[:plen][mask][:length], valid, length)


def to_indices(dtype, raw):
    """ToIndices (take.rs:1030-1084) as Python ints: i8 / i16 `as u32` sign-extend, i32 is reinterpreted as u32."""
    x = int(raw)
    if dtype in (abi.I8, abi.I16, abi.I32):
        return x & 0xFFFFFFFF
    return x & U64


def take(col, idx, idx_valid, idx_buffer, index_dtype, check_bounds=False):
    """take(col, indices): idx the raw index values, idx_valid their validity, idx_buffer whether the indices carry a
    NullBuffer."""
    idx = np.asarray(idx)
    m, n, w = len(idx), col.length, col.width
    idx_valid = np.ones(m, bool) if idx_valid is None else np.asarray(idx_valid, bool)
    idx_nulls = idx_buffer and not idx_valid.all()
    raw = [int(x) for x in idx]
    if check_bounds:  # check_bounds (take.rs:167-209)
        for j in range(m):
            if idx_nulls and not idx_valid[j]:
                continue
            v = raw[j]
            if v >= n or (v < 0 and not idx_nulls):
                raise OracleError(abi.ERR_COMPUTE, f"Array index out of bounds, cannot get item at index {v} from {n} entries", j)
    x = [to_indices(index_dtype, v) for v in raw]
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
    if null_count(col) > 0:
        v = valid_mask(col)
        for j in range(m):
            if idx_nulls and not idx_valid[j]:
                continue
            if x[j] >= n:  # take_bits: BooleanBuffer::value
                raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, BIT_LEN, j)
            valid[j] = valid[j] and v[x[j]]
    has = not valid.all()
    length = m if (w > 0 or has) else 0
    return column(out[:length], valid if has else None, length)
