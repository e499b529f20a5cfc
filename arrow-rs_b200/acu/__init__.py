"""acu — Python host-side mirror of the arrow-rs compute API over the arrow_cuda C ABI.

This is plumbing for tests and bench.py: arrays live in numpy on the host (``HostArray``,
mirroring PrimitiveArray / BooleanArray: values buffer + LSB-first validity bitmap + bit
offset + cached null_count) or in HBM (``DeviceArray``). ``Context`` exposes the reference's
function names (filter, take, add, lt, cast, sum ...) and raises ``ArrowError`` with the
reference's message text. The compute always happens in libarrow_cuda.so; nothing here
falls back to the CPU.

Reference API being mirrored: arrow/src/compute/mod.rs:20-40, arrow/src/compute/kernels.rs:20-34.
"""
import ctypes as C

import numpy as np

from . import _abi as abi
from ._abi import (ADD, ADD_WRAPPING, DISTINCT, DIV, EQ, F32, F64, GT, GT_EQ, I8, I16, I32, I64, LT, LT_EQ, MAX,
                   MIN, MUL, MUL_WRAPPING, NEQ, NOT_DISTINCT, REM, SUB, SUB_WRAPPING, SUM, U8, U16, U32, U64,
                   bitmap_bytes)

BOOL = "bool"
NP_DTYPES = [np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64, np.float32, np.float64]


class ArrowError(Exception):
    """Mirrors arrow_schema::ArrowError; str(e) == the reference's Display text."""

    def __init__(self, status, message, index=-1, detail=None):
        super().__init__(message)
        self.status = status
        self.message = message
        self.index = index
        self.detail = detail


def pack_bits(bools, offset=0):
    """LSB-first bitmap of `bools` starting at bit `offset`; padded to whole u64 words (+8 B)."""
    bools = np.asarray(bools, dtype=bool)
    n = len(bools) + offset
    buf = np.zeros(bitmap_bytes(n) + 8, dtype=np.uint8)
    if len(bools):
        padded = np.zeros(n, dtype=bool)
        padded[offset:] = bools
        packed = np.packbits(padded, bitorder="little")
        buf[: len(packed)] = packed
    return buf


def unpack_bits(buf, offset, n):
    if n == 0:
        return np.zeros(0, dtype=bool)
    bits = np.unpackbits(np.asarray(buf, dtype=np.uint8), bitorder="little")
    return bits[offset: offset + n].astype(bool)


class HostArray:
    """Primitive or boolean Arrow array in host memory (numpy)."""

    def __init__(self, dtype, values, length, validity=None, validity_offset=0, values_offset=0, null_count=-1,
                 is_scalar=False):
        self.dtype = dtype
        self.values = values            # np array of natives, or uint8 bitmap when dtype == BOOL
        self.values_offset = values_offset
        self.validity = validity        # uint8 bitmap or None
        self.validity_offset = validity_offset
        self.length = length
        self.null_count = null_count
        self.is_scalar = is_scalar

    # -- constructors ------------------------------------------------------------------
    @staticmethod
    def from_list(dtype, items, force_validity=False, bit_offset=0, scalar=False):
        """Build from a python list; None = null (like `Int32Array::from(vec![Some(1), None])`)."""
        n = len(items)
        mask = np.array([x is not None for x in items], dtype=bool)
        if dtype == BOOL:
            vals = pack_bits([bool(x) if x is not None else False for x in items], bit_offset)
            voff = bit_offset
        else:
            npdt = NP_DTYPES[dtype]
            vals = np.zeros(n, dtype=npdt)
            for i, x in enumerate(items):
                if x is not None:
                    vals[i] = x
            voff = 0
        validity = None
        nc = 0
        if force_validity or not mask.all():
            validity = pack_bits(mask, bit_offset)
            nc = int(n - mask.sum())
        return HostArray(dtype, vals, n, validity, bit_offset if validity is not None else 0, voff, nc, scalar)

    @staticmethod
    def from_numpy(dtype, values, mask=None, bit_offset=0):
        values = np.ascontiguousarray(values, dtype=NP_DTYPES[dtype])
        validity, nc = None, 0
        if mask is not None:
            mask = np.asarray(mask, dtype=bool)
            validity = pack_bits(mask, bit_offset)
            nc = int(len(mask) - mask.sum())
        return HostArray(dtype, values, len(values), validity, bit_offset if validity is not None else 0, 0, nc)

    @staticmethod
    def bool_from_numpy(bools, mask=None, bit_offset=0, mask_offset=0):
        bools = np.asarray(bools, dtype=bool)
        validity, nc = None, 0
        if mask is not None:
            mask = np.asarray(mask, dtype=bool)
            validity = pack_bits(mask, mask_offset)
            nc = int(len(mask) - mask.sum())
        return HostArray(BOOL, pack_bits(bools, bit_offset), len(bools), validity, mask_offset, bit_offset, nc)

    def scalar(self):
        """Wrap a 1-element array as a Datum scalar (arrow-array/src/scalar.rs:128-152)."""
        assert self.length == 1
        return HostArray(self.dtype, self.values, 1, self.validity, self.validity_offset, self.values_offset,
                         self.null_count, True)

    # -- views ------------------------------------------------------------------------
    def valid_mask(self):
        if self.validity is None:
            return np.ones(self.length, dtype=bool)
        return unpack_bits(self.validity, self.validity_offset, self.length)

    def value_array(self):
        if self.dtype == BOOL:
            return unpack_bits(self.values, self.values_offset, self.length)
        return np.asarray(self.values[: self.length])

    def to_list(self):
        vals, mask = self.value_array(), self.valid_mask()
        return [(v.item() if m else None) for v, m in zip(vals, mask)]

    def slice(self, offset, length):
        """Array::slice — zero-copy: pointer/bit-offset arithmetic only."""
        if self.dtype == BOOL:
            vals, voff = self.values, self.values_offset + offset
        else:
            vals, voff = self.values[offset:], 0
        nc = -1 if self.validity is not None else 0
        return HostArray(self.dtype, vals, length, self.validity, self.validity_offset + offset if self.validity is not None else 0,
                         voff, nc, False)

    def width(self):
        return 1 if self.dtype == BOOL else abi.DTYPE_SIZE[self.dtype]


DECIMAL_MAX_PRECISION = {4: 9, 8: 18, 16: 38}  # = MAX_SCALE
_DECIMAL_NATIVE = {4: abi.I32, 8: abi.I64, 16: abi.I128}
CMP_OP_TEXT = ["==", "!=", "<", "<=", ">", ">=", "IS DISTINCT FROM", "IS NOT DISTINCT FROM"]  # arrow-ord/src/cmp.rs:51-63


def i128_to_halves(ints):
    """Python ints (two's complement in 128 bits) -> an (n, 2) uint64 array of (low, high) halves."""
    out = np.zeros((len(ints), 2), dtype=np.uint64)
    for i, v in enumerate(ints):
        v &= (1 << 128) - 1
        out[i, 0], out[i, 1] = v & 0xFFFFFFFFFFFFFFFF, v >> 64
    return out


def halves_to_i128(halves):
    """(n, 2) uint64 (low, high) -> list of Python ints."""
    lo, hi = halves[:, 0].tolist(), halves[:, 1].view(np.int64).tolist()
    return [(h << 64) | l for l, h in zip(lo, hi)]


class DecimalArray(HostArray):
    """Decimal32 / Decimal64 / Decimal128(precision, scale) in host memory (PrimitiveArray<Decimal*Type>): `values` is an
    int32 / int64 array, or for Decimal128 an (n, 2) uint64 array of (low, high) halves; validity, bit offset, null_count and
    scalar-ness as HostArray. `dtype` is the native the C ABI sees (ACU_I32 / ACU_I64 / ACU_I128)."""

    def __init__(self, byte_width, precision, scale, values, length, validity=None, validity_offset=0, null_count=0,
                 is_scalar=False):
        super().__init__(_DECIMAL_NATIVE[byte_width], values, length, validity, validity_offset, 0, null_count, is_scalar)
        self.byte_width, self.precision, self.scale = byte_width, precision, scale

    @staticmethod
    def from_ints(byte_width, precision, scale, items, force_validity=False, bit_offset=0, scalar=False):
        """items: Python ints / None (None = null, value 0 under it)."""
        ints = [0 if x is None else int(x) for x in items]
        if byte_width == 16:
            vals = i128_to_halves(ints)
        else:
            bits = 8 * byte_width
            vals = np.array([((v + (1 << (bits - 1))) % (1 << bits)) - (1 << (bits - 1)) for v in ints],
                            dtype=np.int32 if byte_width == 4 else np.int64)
        mask = np.array([x is not None for x in items], dtype=bool)
        validity, nc = None, 0
        if force_validity or not mask.all():
            validity, nc = pack_bits(mask, bit_offset), int(len(items) - mask.sum())
        return DecimalArray(byte_width, precision, scale, vals, len(items), validity, bit_offset if validity is not None else 0,
                            nc, scalar)

    @staticmethod
    def from_int64(byte_width, precision, scale, ints, mask=None, bit_offset=0):
        """Vectorised constructor from an int64 numpy array (sign-extended for Decimal128)."""
        ints = np.asarray(ints, dtype=np.int64)
        if byte_width == 16:
            vals = np.empty((len(ints), 2), dtype=np.uint64)
            vals[:, 0] = ints.view(np.uint64)
            vals[:, 1] = (ints >> 63).view(np.uint64)
        else:
            vals = ints.astype(np.int32 if byte_width == 4 else np.int64)
        validity, nc = None, 0
        if mask is not None:
            mask = np.asarray(mask, dtype=bool)
            validity, nc = pack_bits(mask, bit_offset), int(len(mask) - mask.sum())
        return DecimalArray(byte_width, precision, scale, vals, len(ints), validity, bit_offset if validity is not None else 0, nc)

    def data_type(self):
        """Display of DataType::Decimal*(p, s)."""
        return f"Decimal{8 * self.byte_width}({self.precision}, {self.scale})"

    def like(self, h, precision=None, scale=None):
        """The HostArray `h` (a result with this array's native) as a DecimalArray of this / the given type."""
        return DecimalArray(self.byte_width, self.precision if precision is None else precision, self.scale if scale is None else scale,
                            h.values, h.length, h.validity, h.validity_offset, h.null_count, h.is_scalar)

    def width(self):
        return self.byte_width

    def raw_ints(self):
        """Python ints of every slot, nulls included."""
        if self.byte_width == 16:
            return halves_to_i128(np.asarray(self.values[: self.length]).reshape(-1, 2))
        return [int(v) for v in np.asarray(self.values[: self.length])]

    def value_array(self):
        return self.raw_ints()

    def to_list(self):
        return [v if m else None for v, m in zip(self.raw_ints(), self.valid_mask())]

    def scalar(self):
        assert self.length == 1
        d = self.like(self)
        d.is_scalar = True
        return d

    def slice(self, offset, length):
        nc = -1 if self.validity is not None else 0
        return DecimalArray(self.byte_width, self.precision, self.scale, self.values[offset:], length, self.validity,
                            self.validity_offset + offset if self.validity is not None else 0, nc, False)


def _np_ptr(a):
    return a.ctypes.data if a is not None else None


def host_descriptor(h):
    """acu_array pointing at numpy memory (used by the oracle wrapper in tests/)."""
    d = abi.Array()
    d.values = _np_ptr(h.values)
    d.values_offset = h.values_offset
    d.validity = _np_ptr(h.validity)
    d.validity_offset = h.validity_offset
    d.len = h.length
    d.null_count = h.null_count if h.validity is not None else 0
    d.is_scalar = 1 if h.is_scalar else 0
    return d


class Utf8Column:
    """A Utf8 / Binary column on the host: offsets (np.int32 | np.int64, rows + 1), value bytes (np.uint8) and a
    HostArray carrying only the validity / length (GenericByteArray, arrow-array/src/array/byte_array.rs)."""

    def __init__(self, offsets, data, nulls):
        self.offsets, self.data, self.nulls = offsets, data, nulls

    @property
    def length(self):
        return len(self.offsets) - 1


class ViewColumn:
    """A Utf8View / BinaryView column on the host (GenericByteViewArray, arrow-array/src/array/byte_view_array.rs): `views` is an
    (n, 16) uint8 array — length u32 | 12 inline bytes, or length | 4-byte prefix | buffer index u32 | offset u32
    (arrow-data/src/byte_view.rs) — `buffers` the data buffers (uint8 arrays), `nulls` a HostArray carrying validity / length /
    scalar-ness."""

    def __init__(self, views, buffers, nulls):
        self.views, self.buffers, self.nulls = views, buffers, nulls

    @property
    def length(self):
        return self.nulls.length

    @staticmethod
    def from_values(items, block_size=64, scalar=False, garbage_under_nulls=None):
        """items: list of bytes / str / None. Long values (> 12 bytes) are appended to data buffers of `block_size` bytes
        (a new buffer is started when one is full, like GenericByteViewBuilder)."""
        n = len(items)
        views = np.zeros((n, 16), dtype=np.uint8)
        buffers, cur = [], bytearray()
        for i, it in enumerate(items):
            if it is None:
                if garbage_under_nulls is not None:
                    views[i] = garbage_under_nulls[i % len(garbage_under_nulls)]
                continue
            b = it.encode() if isinstance(it, str) else bytes(it)
            views[i, :4] = np.frombuffer(np.uint32(len(b)).tobytes(), dtype=np.uint8)
            if len(b) <= 12:
                views[i, 4:4 + len(b)] = np.frombuffer(b, dtype=np.uint8)
            else:
                if len(cur) + len(b) > block_size and len(cur):
                    buffers.append(np.frombuffer(bytes(cur), dtype=np.uint8).copy())
                    cur = bytearray()
                views[i, 4:8] = np.frombuffer(b[:4], dtype=np.uint8)
                views[i, 8:12] = np.frombuffer(np.uint32(len(buffers)).tobytes(), dtype=np.uint8)
                views[i, 12:16] = np.frombuffer(np.uint32(len(cur)).tobytes(), dtype=np.uint8)
                cur += b
        if len(cur):
            buffers.append(np.frombuffer(bytes(cur), dtype=np.uint8).copy())
        mask = np.array([it is not None for it in items], dtype=bool)
        nulls = HostArray.from_list(U8, [0 if m else None for m in mask])
        nulls.values = np.zeros(0, np.uint8)
        if scalar:
            nulls.is_scalar = True
        return ViewColumn(views, buffers, nulls)

    def values(self):
        out, mask = [], self.nulls.valid_mask()
        for i in range(self.length):
            if not mask[i]:
                out.append(None)
                continue
            ln = int(np.frombuffer(self.views[i, :4].tobytes(), dtype=np.uint32)[0])
            if ln <= 12:
                out.append(bytes(self.views[i, 4:4 + ln]))
            else:
                bi, off = (int(x) for x in np.frombuffer(self.views[i, 8:16].tobytes(), dtype=np.uint32))
                out.append(bytes(self.buffers[bi][off:off + ln]))
        return out


class FixedSizeBinaryColumn:
    """A FixedSizeBinary column on the host (FixedSizeBinaryArray, arrow-array/src/array/fixed_size_binary_array.rs): `values`
    is an (n, width) uint8 array, `nulls` a HostArray carrying validity / length."""

    def __init__(self, values, nulls):
        self.values, self.nulls = np.ascontiguousarray(values, dtype=np.uint8), nulls

    @property
    def width(self):
        return self.values.shape[1]

    @property
    def length(self):
        return self.nulls.length

    @staticmethod
    def from_values(items, width):
        """items: list of bytes (each exactly `width` long) / None."""
        vals = np.zeros((len(items), width), dtype=np.uint8)
        for i, it in enumerate(items):
            if it is not None:
                assert len(it) == width
                vals[i] = np.frombuffer(bytes(it), dtype=np.uint8)
        nulls = HostArray.from_list(U8, [0 if it is not None else None for it in items])
        nulls.values = np.zeros(0, np.uint8)
        return FixedSizeBinaryColumn(vals, nulls)

    def slice(self, offset, length):
        """FixedSizeBinaryArray::slice: the rows and the validity move together."""
        nulls = self.nulls.slice(offset, length)
        nulls.values = np.zeros(0, np.uint8)
        return FixedSizeBinaryColumn(self.values[offset:offset + length], nulls)


class ListColumn:
    """A List (np.int32 offsets) / LargeList (np.int64) column on the host (GenericListArray,
    arrow-array/src/array/list_array.rs): `offsets` has rows + 1 entries from logical row 0 and holds ABSOLUTE child rows
    (a sliced list has offsets[0] != 0), `child` is a HostArray, Utf8Column, ViewColumn or list column, `nulls` a HostArray
    carrying validity / length."""

    def __init__(self, offsets, child, nulls):
        self.offsets, self.child, self.nulls = offsets, child, nulls

    @property
    def length(self):
        return len(self.offsets) - 1


class FixedSizeListColumn:
    """A FixedSizeList(size) column on the host (FixedSizeListArray): row i is child rows [i * size, (i + 1) * size); the
    child starts at the list's logical row 0."""

    def __init__(self, size, child, nulls):
        self.size, self.child, self.nulls = size, child, nulls

    @property
    def length(self):
        return self.nulls.length


class RunEndColumn:
    """A RunEndEncoded column on the host (RunArray, arrow-array/src/array/run_array.rs): `run_ends` (np.int16 | np.int32 |
    np.int64) are the physical run ends from physical entry 0, `values` the values child (one row per physical run: a
    HostArray, DecimalArray, Utf8Column, ViewColumn or list column), `offset` / `length` the logical slice."""

    def __init__(self, run_ends, values, offset=0, length=None):
        self.run_ends, self.values, self.offset = np.ascontiguousarray(run_ends), values, offset
        self.length = (int(self.run_ends[-1]) - offset if len(self.run_ends) else 0) if length is None else length

    def slice(self, offset, length):
        """RunArray::slice: only the logical window moves (run_array.rs, RunEndBuffer::slice run.rs:269-285)."""
        assert offset + length <= self.length, "the length + offset of the sliced RunEndBuffer cannot exceed the existing length"
        return RunEndColumn(self.run_ends, self.values, self.offset + offset, length)


class StructColumn:
    """A Struct column on the host (StructArray, arrow-array/src/array/struct_array.rs): `fields` are columns of the
    struct's length starting at its logical row 0 (any column this package filters / takes; an empty list is a struct
    without fields), `nulls` a HostArray carrying validity / length. Every field is treated as nullable."""

    def __init__(self, fields, nulls):
        self.fields, self.nulls = list(fields), nulls

    @property
    def length(self):
        return self.nulls.length

    def slice(self, offset, length):
        """StructArray::slice: every field and the validity move together."""
        nulls = self.nulls.slice(offset, length)
        nulls.values = np.zeros(0, np.uint8)
        return StructColumn([slice_column(f, offset, length) for f in self.fields], nulls)


class UnionColumn:
    """A sparse or dense Union column on the host (UnionArray, arrow-array/src/array/union_array.rs): `mode` is
    abi.UNION_SPARSE or abi.UNION_DENSE, `field_type_ids` the fields' distinct type ids in [0, 127] in field order,
    `children` one column per field, `type_ids` (np.int8) one per row and, for a dense union, `offsets` (np.int32) the
    row's position in its child. A sparse union's children have the union's length; a union has no NullBuffer."""

    def __init__(self, mode, field_type_ids, children, type_ids, offsets=None):
        self.mode, self.field_type_ids, self.children = mode, [int(x) for x in field_type_ids], list(children)
        self.type_ids = np.ascontiguousarray(type_ids, dtype=np.int8)
        self.offsets = None if offsets is None else np.ascontiguousarray(offsets, dtype=np.int32)

    @property
    def dense(self):
        return self.mode == abi.UNION_DENSE

    @property
    def length(self):
        return len(self.type_ids)

    def slice(self, offset, length):
        """UnionArray::slice: the type ids (and offsets) move; a dense union keeps its children whole, a sparse one slices
        them."""
        tids = self.type_ids[offset:offset + length]
        if self.dense:
            return UnionColumn(self.mode, self.field_type_ids, self.children, tids, self.offsets[offset:offset + length])
        return UnionColumn(self.mode, self.field_type_ids, [slice_column(c, offset, length) for c in self.children], tids)


def slice_column(col, offset, length):
    """Array::slice of any host column: the same buffers, a new logical window."""
    if isinstance(col, HostArray):  # DecimalArray included
        return col.slice(offset, length)
    if isinstance(col, (StructColumn, UnionColumn, FixedSizeBinaryColumn)):
        return col.slice(offset, length)
    nulls = col.nulls.slice(offset, length)
    if isinstance(col, Utf8Column):
        return Utf8Column(col.offsets[offset:offset + length + 1], col.data, nulls)
    if isinstance(col, ViewColumn):
        return ViewColumn(col.views[offset:offset + length], col.buffers, nulls)
    if isinstance(col, ListColumn):
        return ListColumn(col.offsets[offset:offset + length + 1], col.child, nulls)
    if isinstance(col, FixedSizeListColumn):
        return FixedSizeListColumn(col.size, slice_column(col.child, offset * col.size, length * col.size), nulls)
    if isinstance(col, RunEndColumn):
        return col.slice(offset, length)
    raise TypeError(f"cannot slice {type(col).__name__}")


def empty_column(col):
    """new_empty_array of col's type: no rows and no NullBuffer."""
    if isinstance(col, StructColumn):
        return StructColumn([empty_column(f) for f in col.fields], HostArray(abi.U8, np.zeros(0, np.uint8), 0, None, 0, 0, 0))
    if isinstance(col, UnionColumn):
        return UnionColumn(col.mode, col.field_type_ids, [empty_column(c) for c in col.children], np.zeros(0, np.int8),
                           np.zeros(0, np.int32) if col.dense else None)
    e = slice_column(col, 0, 0)
    tgt = e if isinstance(e, HostArray) else (None if isinstance(e, RunEndColumn) else e.nulls)
    if tgt is not None:
        tgt.validity, tgt.validity_offset, tgt.null_count = None, 0, 0
    if isinstance(e, (ListColumn, FixedSizeListColumn)):
        e.child = empty_column(e.child)
    return e


def column_value(col, row):
    """The bytes of logical row `row` of a Utf8Column / ViewColumn / FixedSizeBinaryColumn (`array.value(row)`)."""
    if isinstance(col, Utf8Column):
        return bytes(col.data[int(col.offsets[row]): int(col.offsets[row + 1])])
    if isinstance(col, FixedSizeBinaryColumn):
        return bytes(col.values[row])
    v = col.views[row]
    ln = int(np.frombuffer(v[:4].tobytes(), dtype=np.uint32)[0])
    if ln <= 12:
        return bytes(v[4:4 + ln])
    bi, off = (int(x) for x in np.frombuffer(v[8:16].tobytes(), dtype=np.uint32))
    return bytes(col.buffers[bi][off:off + ln])


class DeviceArray:
    """A HostArray's buffers uploaded to HBM (DeviceBuffer pair) with the same offsets."""

    def __init__(self, ctx, dtype, length, d_values, values_offset, d_validity, validity_offset, null_count, is_scalar,
                 owned):
        self.ctx, self.dtype, self.length = ctx, dtype, length
        self.d_values, self.values_offset = d_values, values_offset
        self.d_validity, self.validity_offset = d_validity, validity_offset
        self.null_count, self.is_scalar = null_count, is_scalar
        self._owned = owned

    def descriptor(self):
        d = abi.Array()
        d.values = self.d_values
        d.values_offset = self.values_offset
        d.validity = self.d_validity
        d.validity_offset = self.validity_offset
        d.len = self.length
        d.null_count = self.null_count if self.d_validity else 0
        d.is_scalar = 1 if self.is_scalar else 0
        return d

    def free(self):
        for p in self._owned:
            self.ctx.free(p)
        self._owned = []


class _Scope:
    """The owner of everything one Context call allocates: device pointers, uploaded DeviceArrays, ArrayOuts, filter plans
    (also those an entry point fills in as out-parameters) and host objects the device reads during the call, such as
    view pointer tables. On exit it releases them in reverse order and always attempts every release. A release error
    never replaces an exception already propagating; without one, the first release error is raised after the other
    releases have run. It allocates through ctx.malloc and releases through ctx.free and ctx.lib.acu_filter_plan_destroy,
    so a fake context can stand in for a Context.

    The upload helpers take an `owned` list that device pointers are appended to and a `keep` list for host objects; a
    scope stands in for the first (append) and its `keep` list for the second."""

    def __init__(self, ctx):
        self.ctx, self._held = ctx, []
        self.keep = []  # host objects the device reads during the call, dropped on exit

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc, tb):
        first = None
        while self._held:
            release, x = self._held.pop()
            try:
                release(x)
            except Exception as e:
                first = e if first is None else first
        self.keep.clear()
        if first is not None and exc_type is None:
            raise first
        return False

    def _hold(self, release, x):
        self._held.append((release, x))
        return x

    def append(self, p):
        """Own the device pointer p (a scope stands wherever a list of owned pointers is expected)."""
        return self._hold(self.ctx.free, p)

    def malloc(self, nbytes):
        return self.append(self.ctx.malloc(nbytes))

    def upload(self, h):
        """Context.upload(h), freed on exit."""
        return self._hold(DeviceArray.free, self.ctx.upload(h))

    def out(self, nbytes_values, n_rows):
        """An ArrayOut as Context.alloc_out allocates it."""
        out = abi.ArrayOut()
        out.values = self.malloc(nbytes_values + 16)
        out.validity = self.malloc(bitmap_bytes(n_rows) + 8)
        return out

    def plan(self):
        """A filter-plan handle for an entry point to fill in; destroyed on exit only if it was set."""
        return self._hold(self._destroy_plan, C.c_void_p())

    def _destroy_plan(self, plan):
        if plan:
            self.ctx.lib.acu_filter_plan_destroy(self.ctx.h, plan)


class Context:
    """acu_ctx wrapper: one device, one stream."""

    def __init__(self, device=0):
        self.lib = abi.load_library()
        h = C.c_void_p()
        st = self.lib.acu_ctx_create(device, C.byref(h))
        if st != abi.OK:
            raise RuntimeError(f"acu_ctx_create(device={device}) failed with status {st}: no usable CUDA device "
                               "(arrow-cuda has no CPU fallback)")
        self.h = h
        self.device = device

    def close(self):
        if self.h:
            self.lib.acu_ctx_destroy(self.h)
            self.h = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _scope(self):
        """`with self._scope() as s:` owns what one call allocates (see _Scope)."""
        return _Scope(self)

    # -- errors / memory -----------------------------------------------------------------
    def check(self, st):
        if st != abi.OK:
            d = self.lib.acu_last_error(self.h).contents
            raise ArrowError(st, d.message.decode(), d.index, d)

    def malloc(self, nbytes):
        p = C.c_void_p()
        self.check(self.lib.acu_malloc(self.h, max(int(nbytes), 1), C.byref(p)))
        return p.value

    def free(self, p):
        if p:
            self.check(self.lib.acu_free(self.h, p))

    def h2d(self, dptr, arr):
        arr = np.ascontiguousarray(arr)
        self.check(self.lib.acu_memcpy_h2d(self.h, dptr, arr.ctypes.data, arr.nbytes))

    def d2h(self, dptr, nbytes, dtype=np.uint8):
        out = np.empty(max(int(nbytes), 0) // np.dtype(dtype).itemsize, dtype=dtype)
        if out.nbytes:
            self.check(self.lib.acu_memcpy_d2h(self.h, out.ctypes.data, dptr, out.nbytes))
        return out

    def sync(self):
        self.check(self.lib.acu_ctx_sync(self.h))

    def async_begin(self):
        """Open a stream-ordered section (include/arrow_cuda.h): the supported entry points only enqueue."""
        self.check(self.lib.acu_async_begin(self.h))

    def results_fetch(self):
        """ONE D2H + ONE synchronisation; finalises the queued calls in order, raises the first error."""
        self.check(self.lib.acu_results_fetch(self.h))

    def launch_count(self):
        return self.lib.acu_launch_count(self.h)

    def upload(self, h):
        owned = []
        if h.dtype == BOOL:
            buf = np.asarray(h.values, dtype=np.uint8)
            dv = self.malloc(buf.nbytes + 8)
            self.h2d(dv, buf)
        else:
            vals = np.ascontiguousarray(h.values[: max(h.length, 1 if h.is_scalar else 0)])
            dv = self.malloc(vals.nbytes + 16)
            if vals.nbytes:
                self.h2d(dv, vals)
        owned.append(dv)
        dn = None
        if h.validity is not None:
            dn = self.malloc(h.validity.nbytes + 8)
            self.h2d(dn, h.validity)
            owned.append(dn)
        return DeviceArray(self, h.dtype, h.length, dv, h.values_offset, dn, h.validity_offset,
                           h.null_count if h.validity is not None else 0, h.is_scalar, owned)

    def _copy_in(self, arr, owned, pad=16):
        """A device copy of the numpy array `arr` in a buffer `pad` bytes longer; the pointer is appended to `owned`."""
        arr = np.ascontiguousarray(arr)
        p = self.malloc(arr.nbytes + pad)
        owned.append(p)
        if arr.nbytes:
            self.h2d(p, arr)
        return p

    def alloc_out(self, nbytes_values, n_rows):
        out = abi.ArrayOut()
        out.values = self.malloc(nbytes_values + 16)
        out.validity = self.malloc(bitmap_bytes(n_rows) + 8)
        return out

    def _nulls_out(self, out, n):
        """The NullBuffer of the n-row result `out` (an ArrayOut) as a HostArray without values."""
        validity = self.d2h(out.validity, bitmap_bytes(n)) if out.has_validity else None
        return HostArray(U8, np.zeros(0, np.uint8), n, validity, 0, 0, out.null_count if out.has_validity else 0)

    def _read_out(self, out, dtype):
        """The result ArrayOut `out` read back as a HostArray of `dtype`; its buffers stay allocated."""
        n = out.len
        if dtype == BOOL:
            vals = self.d2h(out.values, bitmap_bytes(n))
        elif dtype == abi.I128:
            vals = self.d2h(out.values, n * 16, np.uint64).reshape(-1, 2)
        else:
            vals = self.d2h(out.values, n * abi.DTYPE_SIZE[dtype], NP_DTYPES[dtype])
        nulls = self._nulls_out(out, n)
        return HostArray(dtype, vals, n, nulls.validity, 0, 0, nulls.null_count)

    def download_out(self, out, dtype):
        """_read_out, then the buffers of `out` are freed."""
        res = self._read_out(out, dtype)
        self._free_out(out)
        return res

    def _free_out(self, out):
        self.free(out.values)
        self.free(out.validity)

    def _call_out(self, inputs, nbytes_values, n_rows, call, dtype):
        """Upload the HostArrays `inputs` (None passes as a null descriptor), allocate an ArrayOut, run
        call(*input descriptors, out) and read the result back as `dtype`."""
        with self._scope() as s:
            descs = [None if x is None else s.upload(x).descriptor() for x in inputs]
            out = s.out(nbytes_values, n_rows)
            self.check(call(*[None if d is None else C.byref(d) for d in descs], C.byref(out)))
            return self._read_out(out, dtype)

    def _bytes_out(self, s, fn, n, ob, data_capacity=None, child_step=None):
        """A Utf8Column of n rows (ob-byte offsets) produced in two phases: the sizing call without a data buffer, then the
        copy into `data_capacity` bytes (default: exactly the size). fn(d_out_off, d_out_data, capacity, total_ref, out)
        calls the entry point; the buffers belong to the scope s. child_step as for _filter_with_plan."""
        d_off = s.malloc((n + 1) * ob + 16)
        out = s.out(0, n)
        total = C.c_int64(0)
        self.check(fn(d_off, None, 0, C.byref(total), C.byref(out)))
        cap = total.value if data_capacity is None else data_capacity
        d_data = s.malloc(cap + 16)
        self.check(fn(d_off, d_data, cap, C.byref(total), C.byref(out)))
        self._drop_empty_nulls(out, child_step)
        return Utf8Column(self.d2h(d_off, (n + 1) * ob, np.int32 if ob == 4 else np.int64), self.d2h(d_data, total.value),
                          self._nulls_out(out, n))

    # -- filter (arrow-select/src/filter.rs) ----------------------------------------------
    def _plan(self, s, predicate):
        """The filter plan of `predicate` (acu_filter_plan_create), owned by the scope s."""
        pd = s.upload(predicate).descriptor()
        plan = s.plan()
        self.check(self.lib.acu_filter_plan_create(self.h, C.byref(pd), C.byref(plan)))
        return plan

    def filter(self, values, predicate):
        """arrow::compute::filter(values, predicate) for primitive and boolean arrays."""
        with self._scope() as s:
            return self._filter_with_plan(values, self._plan(s, predicate))

    def filter_plan(self, predicate):
        """FilterBuilder::new(predicate).optimize().build() -> (count, strategy)."""
        with self._scope() as s:
            plan = self._plan(s, predicate)
            return self.lib.acu_filter_plan_count(plan), self.lib.acu_filter_plan_strategy(plan)

    def filter_slices(self, predicate):
        """SlicesIterator::new(&prep_null_mask_filter(predicate)).collect() -> [(start, end)] (filter.rs:44-77)."""
        with self._scope() as s:
            plan = self._plan(s, predicate)
            n = C.c_int64(0)
            self.check(self.lib.acu_filter_plan_slices(self.h, plan, None, 0, C.byref(n)))
            if n.value == 0:
                return []
            out = s.malloc(n.value * 16 + 16)
            self.check(self.lib.acu_filter_plan_slices(self.h, plan, out, n.value, C.byref(n)))
            pairs = self.d2h(out, n.value * 16, np.uint64).reshape(-1, 2)
            return [(int(a), int(b)) for a, b in pairs]

    def chain(self, col, pred, idx, a, b, arith_op=ADD, agg_op=SUM, cmp_with=None):
        """filter(col, pred) -> take(col, idx) -> arith(a, b) -> aggregate(taken) queued in ONE stream-ordered section
        (acu_async_begin ... acu_results_fetch): one synchronisation for the five calls. With cmp_with = (op, x, y) the
        predicate is cmp(op, x, y) computed inside the section too (`pred` is ignored). Returns
        (filtered, taken, arith result, aggregate or None); raises the first error in call order at the fetch."""
        n_pred = (cmp_with[2].length if cmp_with[1].is_scalar else cmp_with[1].length) if cmp_with else pred.length
        with self._scope() as s:
            dcol, didx, da, db = (s.upload(x) for x in (col, idx, a, b))
            plan = s.plan()
            if cmp_with:
                cx, cy = s.upload(cmp_with[1]), s.upload(cmp_with[2])
                o_pred = s.out(bitmap_bytes(n_pred), n_pred)
            else:
                dpred = s.upload(pred)
            # outputs of a filter whose plan is pending are sized for the predicate length
            o_f = s.out(max(n_pred, 1) * col.width(), n_pred)
            o_t = s.out(idx.length * col.width(), idx.length)
            n_ar = b.length if a.is_scalar and not b.is_scalar else a.length
            o_a = s.out(n_ar * a.width(), n_ar)
            bits, cnt = C.c_uint64(0), C.c_int64(0)
            cd, idd, ad, bd = dcol.descriptor(), didx.descriptor(), da.descriptor(), db.descriptor()
            self.async_begin()
            try:
                if cmp_with:
                    xd, yd = cx.descriptor(), cy.descriptor()
                    self.check(self.lib.acu_cmp(self.h, cmp_with[1].dtype, cmp_with[0], C.byref(xd), C.byref(yd), C.byref(o_pred)))
                    # the comparison's null count is still on the device: hand the plan a predicate without cached count is not
                    # allowed inside a section, so the fused entry point is the stream-ordered way to build a plan from a cmp
                    self.check(self.lib.acu_filter_plan_create_cmp(self.h, cmp_with[1].dtype, cmp_with[0], C.byref(xd), C.byref(yd), C.byref(plan)))
                else:
                    pd = dpred.descriptor()
                    self.check(self.lib.acu_filter_plan_create(self.h, C.byref(pd), C.byref(plan)))
                if col.dtype == BOOL:
                    self.check(self.lib.acu_filter_boolean(self.h, plan, C.byref(cd), C.byref(o_f)))
                    self.check(self.lib.acu_take_boolean(self.h, C.byref(cd), C.byref(idd), idx.dtype, 0, C.byref(o_t)))
                else:
                    self.check(self.lib.acu_filter_primitive(self.h, plan, col.width(), C.byref(cd), C.byref(o_f)))
                    self.check(self.lib.acu_take_primitive(self.h, col.width(), C.byref(cd), C.byref(idd), idx.dtype, 0, C.byref(o_t)))
                self.check(self.lib.acu_arith(self.h, a.dtype, arith_op, C.byref(ad), C.byref(bd), C.byref(o_a)))
                has_v = (col.validity is not None and col.null_count != 0) or idx.validity is not None
                taken = abi.Array()
                taken.values, taken.values_offset = o_t.values, 0
                taken.validity, taken.validity_offset = (o_t.validity if has_v else None), 0
                taken.len, taken.null_count, taken.is_scalar = idx.length, (-1 if has_v else 0), 0
                do_agg = col.dtype != BOOL
                if do_agg:
                    self.check(self.lib.acu_aggregate(self.h, col.dtype, agg_op, C.byref(taken), C.byref(bits), C.byref(cnt)))
            except BaseException:
                try:
                    self.results_fetch()
                except ArrowError:
                    pass
                raise
            self.results_fetch()
            pred_out = self._read_out(o_pred, BOOL) if cmp_with else None
            filtered = self._read_out(o_f, col.dtype)
            taken_h = self._read_out(o_t, col.dtype)
            added = self._read_out(o_a, a.dtype)
            agg = None
            if do_agg and cnt.value != 0:
                agg = np.array([bits.value], dtype=np.uint64).view(NP_DTYPES[col.dtype])[0].item()
            res = (filtered, taken_h, added, agg)
            return res + (pred_out,) if cmp_with else res

    # -- take (arrow-select/src/take.rs) ----------------------------------------------------
    def take(self, values, indices, check_bounds=False):
        with self._scope() as s:
            return self._take_level(values, s.upload(indices).descriptor(), indices.dtype, check_bounds, False)

    # -- variable width (Utf8) ---------------------------------------------------------------
    def take_bytes(self, offsets, data, nulls_of, indices, check_bounds=False):
        """take on a Utf8/Binary array given as (offsets np.int32/int64, data np.uint8, nulls_of HostArray
        carrying validity/len). Returns (offsets, data, nulls HostArray)."""
        r = self.take(Utf8Column(offsets, data, nulls_of), indices, check_bounds)
        return r.offsets, r.data, r.nulls

    def filter_bytes(self, offsets, data, nulls_of, predicate):
        r = self.filter(Utf8Column(offsets, data, nulls_of), predicate)
        return r.offsets, r.data, r.nulls

    # -- RecordBatch level (filter.rs:225-244, take.rs:1123-1133) ----------------------------
    # A batch is a list of columns; a column is a HostArray (primitive / boolean) or a
    # Utf8Column(offsets, data, nulls). Results keep the column order and kinds.
    @staticmethod
    def _column_kind(col):
        """(acu_column kind, width) of a host column: a Utf8Column's width is its offset width."""
        if isinstance(col, Utf8Column):
            return abi.COL_BYTES, col.offsets.dtype.itemsize
        if isinstance(col, FixedSizeBinaryColumn):
            return abi.COL_FIXED_SIZE_BINARY, col.width
        return (abi.COL_BOOLEAN, 0) if col.dtype == BOOL else (abi.COL_PRIMITIVE, col.width())

    def _upload_columns(self, columns, s):
        cols = (abi.Column * len(columns))()
        for c, col in enumerate(columns):
            cols[c].kind, cols[c].width = self._column_kind(col)
            if isinstance(col, Utf8Column):
                bd = self._upload_bytes_col(col, s)
                cols[c].array = bd.nulls
                cols[c].array.values = bd.offsets
                cols[c].data = bd.data
            elif isinstance(col, FixedSizeBinaryColumn):
                cols[c].array = self._upload_fsb(col, s)
            else:
                cols[c].array = s.upload(col).descriptor()
        return cols

    def _alloc_column_outs(self, columns, rows, data_caps, owned=None):
        """ColumnOuts for `columns`; the device pointers are appended to `owned` (None: _free_columns releases them)."""
        owned = [] if owned is None else owned

        def malloc(nbytes):
            p = self.malloc(nbytes)
            owned.append(p)
            return p
        outs = (abi.ColumnOut * len(columns))()
        for c, col in enumerate(columns):
            if isinstance(col, Utf8Column):
                outs[c].array.values = malloc((rows + 1) * col.offsets.dtype.itemsize + 16)
                outs[c].array.validity = malloc(bitmap_bytes(rows) + 8)
                outs[c].data = malloc(data_caps[c] + 16)
                outs[c].data_capacity = data_caps[c]
            elif isinstance(col, FixedSizeBinaryColumn):
                outs[c].array.values = malloc(rows * col.width + 16)
                outs[c].array.validity = malloc(bitmap_bytes(rows) + 8)
            else:
                outs[c].array.values = malloc((bitmap_bytes(rows) if col.dtype == BOOL else rows * col.width()) + 16)
                outs[c].array.validity = malloc(bitmap_bytes(rows) + 8)
        return outs

    def _free_columns(self, owned, outs):
        """Release the device pointers `owned` and the buffers of the ColumnOuts `outs` (None: none), as _free_out releases
        an ArrayOut, for callers that hold them without a scope."""
        with self._scope() as s:
            for p in list(owned) + [q for o in outs or () for q in (o.array.values, o.array.validity, o.data)]:
                s.append(p)

    def _read_column(self, kind, width, dtype, arr, data, data_len=None):
        """A column read back from the device buffers of an acu_column / acu_column_out: `arr` is an ArrayOut of its values
        (the offsets of a COL_BYTES column, `width` bytes each), validity and rows; `data` the bytes of a COL_BYTES column,
        data_len of them (None: up to the last offset). Returns a Utf8Column, a FixedSizeBinaryColumn of byte width `width`
        (COL_FIXED_SIZE_BINARY), or a HostArray of `dtype`."""
        if kind == abi.COL_FIXED_SIZE_BINARY:
            return self._fsb_out(arr, arr.len, width)
        if kind != abi.COL_BYTES:
            return self._read_out(arr, BOOL if kind == abi.COL_BOOLEAN else dtype)
        n = arr.len
        nulls = self._nulls_out(arr, n)
        offs = self.d2h(arr.values, (n + 1) * width, np.int32 if width == 4 else np.int64)
        return Utf8Column(offs, self.d2h(data, (int(offs[-1]) if n else 0) if data_len is None else data_len), nulls)

    def _download_columns(self, columns, outs):
        return [self._read_column(*self._column_kind(col), col.dtype if isinstance(col, HostArray) else None, o.array, o.data,
                                  o.data_len) for col, o in zip(columns, outs)]

    # -- Arrow IPC stream -> HBM (arrow-ipc/src/reader.rs StreamReader) ---------------------------
    def ipc_read_stream(self, stream_bytes, on_batch=None):
        """StreamReader over an in-memory IPC stream: every RecordBatch body is ONE host->device copy and its columns are
        views into that device buffer. Returns (schema, batches): schema = [(name, kind, width, dtype, nullable)], batches =
        lists of downloaded columns (HostArray / Utf8Column) — or whatever `on_batch(columns_descriptor_array, rows)` returns
        when given (the descriptors are only valid inside the callback)."""
        buf = np.frombuffer(bytes(stream_bytes), dtype=np.uint8).copy()
        h = C.c_void_p()
        n = C.c_int32(0)
        self.check(self.lib.acu_ipc_stream_open(self.h, buf.ctypes.data, len(buf), C.byref(h), C.byref(n)))
        try:
            schema = []
            for i in range(n.value):
                kind, width, dtype, nullable, name = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32(), C.c_char_p()
                self.lib.acu_ipc_stream_field(h, i, C.byref(kind), C.byref(width), C.byref(dtype), C.byref(nullable), C.byref(name))
                schema.append((name.value.decode(), kind.value, width.value, dtype.value, bool(nullable.value)))
            batches = []
            cols = (abi.Column * max(n.value, 1))()
            while True:
                rows = C.c_int64(0)
                self.check(self.lib.acu_ipc_stream_next(self.h, h, cols, C.byref(rows)))
                if rows.value < 0:
                    break
                if on_batch is not None:
                    batches.append(on_batch(cols, rows.value))
                    continue
                out = []
                for i, (name, kind, width, dtype, _) in enumerate(schema):
                    a = cols[i].array
                    arr = abi.ArrayOut(a.values, a.validity, rows.value, a.null_count, 1 if a.validity else 0)
                    out.append(self._read_column(kind, width, dtype, arr, cols[i].data))
                batches.append(out)
            return schema, batches
        finally:
            self.lib.acu_ipc_stream_close(self.h, h)

    # -- concat / concat_batches (arrow-select/src/concat.rs:495-640) ---------------------------
    def concat(self, columns):
        """arrow::compute::concat(&[..]): columns = HostArrays or Utf8Columns of one type."""
        with self._scope() as s:
            cols = self._upload_columns(columns, s) if columns else (abi.Column * 1)()
            rows = sum(c.length for c in columns)
            proto = columns[:1] if columns else [HostArray(U8, np.zeros(0, np.uint8), 0)]
            caps = [sum(int(c.data.nbytes) for c in columns)] if columns and isinstance(columns[0], Utf8Column) else [0]
            outs = self._alloc_column_outs(proto, max(rows, 1), caps, s)
            self.check(self.lib.acu_concat(self.h, len(columns), cols, outs))
            return self._download_columns(proto, outs)[0]

    def concat_batches(self, batches):
        """arrow::compute::concat_batches(schema, batches): batches = lists of columns (same schema)."""
        ncols = len(batches[0]) if batches else 0
        flat = [c for b in batches for c in b]
        with self._scope() as s:
            cols = self._upload_columns(flat, s) if flat else (abi.Column * 1)()
            rows = sum(b[0].length for b in batches) if ncols else 0
            proto = list(batches[0]) if batches else []
            caps = [sum(int(b[c].data.nbytes) for b in batches) if isinstance(proto[c], Utf8Column) else 0 for c in range(ncols)]
            outs = self._alloc_column_outs(proto, max(rows, 1), caps, s) if ncols else (abi.ColumnOut * 1)()
            n = C.c_int64(0)
            self.check(self.lib.acu_concat_batches(self.h, len(batches), ncols, cols, outs, C.byref(n)))
            return self._download_columns(proto, outs) if ncols else []

    def filter_record_batch(self, columns, predicate):
        """arrow::compute::filter_record_batch: one plan, every column, one synchronisation."""
        with self._scope() as s:
            cols = self._upload_columns(columns, s)
            plan = self._plan(s, predicate)
            count = self.lib.acu_filter_plan_count(plan)
            caps = [int(col.data.nbytes) if isinstance(col, Utf8Column) else 0 for col in columns]
            outs = self._alloc_column_outs(columns, count, caps, s)
            self.check(self.lib.acu_filter_record_batch(self.h, plan, len(columns), cols, outs))
            return self._download_columns(columns, outs)

    def take_record_batch(self, columns, indices, check_bounds=False, data_capacity=None):
        """arrow::compute::take_record_batch / take_arrays."""
        with self._scope() as s:
            cols = self._upload_columns(columns, s)
            idd = s.upload(indices).descriptor()
            m = indices.length
            caps = []
            for col in columns:
                if isinstance(col, Utf8Column):
                    lens = np.diff(col.offsets.astype(np.int64)) if len(col.offsets) > 1 else np.zeros(0, np.int64)
                    caps.append(int(data_capacity) if data_capacity is not None else int((lens.max() if lens.size else 0) * m))
                else:
                    caps.append(0)
            outs = self._alloc_column_outs(columns, m, caps, s)
            self.check(self.lib.acu_take_record_batch(self.h, len(columns), cols, C.byref(idd), indices.dtype, int(check_bounds), outs))
            return self._download_columns(columns, outs)

    def aggregate_columns(self, ops, columns):
        """[sum|min|max|product|bit_and|bit_or|bit_xor](column) for several primitive columns with one synchronisation ->
        [(value|None)]."""
        n = len(columns)
        with self._scope() as s:
            arrs = (abi.Array * n)(*[s.upload(c).descriptor() for c in columns])
            dts = (C.c_int32 * n)(*[c.dtype for c in columns])
            opv = (C.c_int32 * n)(*ops)
            bits, cnts = (C.c_uint64 * n)(), (C.c_int64 * n)()
            self.check(self.lib.acu_aggregate_columns(self.h, n, dts, opv, arrs, bits, cnts))
        out = []
        for i, c in enumerate(columns):
            if cnts[i] == 0:
                out.append(None)
            else:
                raw = np.array([bits[i]], dtype=np.uint64).view(np.uint8)[: abi.DTYPE_SIZE[c.dtype]]
                out.append(raw.view(NP_DTYPES[c.dtype])[0].item())
        return out

    # -- numeric (arrow-arith/src/numeric.rs) -----------------------------------------------
    def arith(self, op, a, b):
        assert a.dtype == b.dtype
        n = b.length if a.is_scalar and not b.is_scalar else a.length
        return self._call_out((a, b), n * a.width(), n, lambda ad, bd, out: self.lib.acu_arith(self.h, a.dtype, op, ad, bd, out), a.dtype)

    def add(self, a, b): return self.arith(ADD, a, b)
    def add_wrapping(self, a, b): return self.arith(ADD_WRAPPING, a, b)
    def sub(self, a, b): return self.arith(SUB, a, b)
    def sub_wrapping(self, a, b): return self.arith(SUB_WRAPPING, a, b)
    def mul(self, a, b): return self.arith(MUL, a, b)
    def mul_wrapping(self, a, b): return self.arith(MUL_WRAPPING, a, b)
    def div(self, a, b): return self.arith(DIV, a, b)
    def rem(self, a, b): return self.arith(REM, a, b)

    def neg(self, a, checked=True):
        return self._call_out((a,), a.length * a.width(), a.length,
                              lambda ad, out: self.lib.acu_neg(self.h, a.dtype, int(checked), ad, out), a.dtype)

    def neg_wrapping(self, a): return self.neg(a, checked=False)

    # -- bitwise (arrow-arith/src/bitwise.rs) ------------------------------------------------------
    def bitwise(self, op, a, b=None):
        """bitwise_and / or / xor / and_not / shift_left / shift_right (acu_bitwise_op) of two integer HostArrays, their
        _scalar forms (b a scalar HostArray) and bitwise_not (op = BITWISE_NOT, b None)."""
        assert b is None or a.dtype == b.dtype
        return self._call_out((a, b), a.length * a.width(), a.length,
                              lambda ad, bd, out: self.lib.acu_bitwise(self.h, a.dtype, op, ad, bd, out), a.dtype)

    def bitwise_and(self, a, b): return self.bitwise(abi.BITWISE_AND, a, b)
    def bitwise_or(self, a, b): return self.bitwise(abi.BITWISE_OR, a, b)
    def bitwise_xor(self, a, b): return self.bitwise(abi.BITWISE_XOR, a, b)
    def bitwise_and_not(self, a, b): return self.bitwise(abi.BITWISE_AND_NOT, a, b)
    def bitwise_shift_left(self, a, b): return self.bitwise(abi.BITWISE_SHIFT_LEFT, a, b)
    def bitwise_shift_right(self, a, b): return self.bitwise(abi.BITWISE_SHIFT_RIGHT, a, b)
    def bitwise_not(self, a): return self.bitwise(abi.BITWISE_NOT, a)

    # -- decimal arithmetic (decimal_op, arrow-arith/src/numeric.rs:970-1107) -----------------------------
    def decimal_arith(self, op, a, b):
        """add / sub / mul / div / rem (acu_arith_op) of two DecimalArrays (either may be a scalar): a DecimalArray of the
        reference's result type; raises ArrowError with the reference's text."""
        n = b.length if a.is_scalar and not b.is_scalar else a.length
        lt, rt, ot = (abi.DecimalType(x.byte_width, x.precision, x.scale) for x in (a, b, a))
        res = self._call_out((a, b), n * a.byte_width, n, lambda ad, bd, out: self.lib.acu_decimal_arith(
            self.h, op, C.byref(lt), ad, C.byref(rt), bd, C.byref(ot), out), a.dtype)
        return a.like(res, ot.precision, ot.scale)

    def decimal_add(self, a, b): return self.decimal_arith(ADD, a, b)
    def decimal_sub(self, a, b): return self.decimal_arith(SUB, a, b)
    def decimal_mul(self, a, b): return self.decimal_arith(MUL, a, b)
    def decimal_div(self, a, b): return self.decimal_arith(DIV, a, b)
    def decimal_rem(self, a, b): return self.decimal_arith(REM, a, b)

    def decimal_neg(self, a):
        """neg / neg_wrapping of a DecimalArray: neg_checked at every width (numeric.rs:116-136, :181-186)."""
        return a.like(self.neg(a, checked=True))

    @staticmethod
    def check_decimal_cmp(op, a, b):
        """compare_op's type check (arrow-ord/src/cmp.rs:228-263): after the length check, decimal operands must have equal
        DataTypes, precision included. The C ABI carries natives only, so the check lives here."""
        if not (isinstance(a, DecimalArray) and isinstance(b, DecimalArray)):
            return
        if a.data_type() == b.data_type():
            return
        if not a.is_scalar and not b.is_scalar and a.length != b.length:
            raise ArrowError(abi.ERR_INVALID_ARGUMENT,
                             f"Invalid argument error: Cannot compare arrays of different lengths, got {a.length} vs {b.length}")
        raise ArrowError(abi.ERR_INVALID_ARGUMENT,
                         f"Invalid argument error: Invalid comparison operation: {a.data_type()} {CMP_OP_TEXT[op]} {b.data_type()}")

    # -- cmp (arrow-ord/src/cmp.rs) -----------------------------------------------------------
    def cmp(self, op, a, b):
        self.check_decimal_cmp(op, a, b)
        assert a.dtype == b.dtype
        n = b.length if a.is_scalar else a.length
        return self._call_out((a, b), bitmap_bytes(n), n, lambda ad, bd, out: self.lib.acu_cmp(self.h, a.dtype, op, ad, bd, out), BOOL)

    # -- cmp on Utf8 / Binary and Utf8View / BinaryView operands (cmp.rs:783-898) -----------------
    def _upload_nulls(self, nulls, owned):
        d = abi.Array()
        d.len, d.is_scalar = nulls.length, 1 if nulls.is_scalar else 0
        d.validity_offset = nulls.validity_offset
        d.null_count = nulls.null_count if nulls.validity is not None else 0
        if nulls.validity is not None:
            d.validity = self._copy_in(nulls.validity, owned, 8)
        return d

    def _upload_bytes_col(self, col, owned):
        """acu_bytes_array of a Utf8Column uploaded to HBM (device pointers appended to `owned`)."""
        d = abi.BytesArray()
        d.offsets, d.data = self._copy_in(col.offsets, owned), self._copy_in(col.data, owned)
        d.nulls = self._upload_nulls(col.nulls, owned)
        return d

    def _upload_view_col(self, col, owned, keep):
        """acu_view_array of a ViewColumn uploaded to HBM; the host pointer table is appended to `keep`."""
        d = abi.ViewArray()
        d.views = self._copy_in(col.views, owned)
        ptrs = [self._copy_in(buf, owned) for buf in col.buffers]
        table = (C.c_void_p * max(len(ptrs), 1))(*ptrs)
        keep.append(table)
        d.buffers, d.n_buffers = table, len(ptrs)
        d.nulls = self._upload_nulls(col.nulls, owned)
        return d

    def _upload_fsb(self, col, owned):
        d = self._upload_nulls(col.nulls, owned)
        d.values = self._copy_in(col.values, owned)
        return d

    def _fsb_out(self, out, n, width):
        """The n-row FixedSizeBinary result `out` (an ArrayOut) read back; its buffers stay allocated."""
        return FixedSizeBinaryColumn(self.d2h(out.values, n * width).reshape(n, width), self._nulls_out(out, n))

    def _bytes_predicate(self, a, b, call):
        """A boolean result of two Utf8Column or two ViewColumn operands (nulls.is_scalar marks a Datum scalar):
        call(a descriptor, b descriptor, out) calls the entry point."""
        n = max(a.nulls.length if not a.nulls.is_scalar else 0, b.nulls.length if not b.nulls.is_scalar else 0, 1)
        with self._scope() as s:
            out = s.out(bitmap_bytes(n), n)
            if isinstance(a, Utf8Column):
                da, db = self._upload_bytes_col(a, s), self._upload_bytes_col(b, s)
            else:
                da, db = self._upload_view_col(a, s, s.keep), self._upload_view_col(b, s, s.keep)
            self.check(call(C.byref(da), C.byref(db), C.byref(out)))
            return self._read_out(out, BOOL)

    def cmp_bytes(self, op, a, b):
        """a, b: Utf8Column (offsets, data, nulls); nulls.is_scalar marks a Datum scalar."""
        assert a.offsets.dtype == b.offsets.dtype
        return self._bytes_predicate(a, b, lambda da, db, out: self.lib.acu_cmp_bytes(self.h, a.offsets.dtype.itemsize, op, da, db, out))

    def cmp_view(self, op, a, b):
        """a, b: ViewColumn."""
        return self._bytes_predicate(a, b, lambda da, db, out: self.lib.acu_cmp_byte_view(self.h, op, da, db, out))

    # -- like / ilike / contains / starts_with / ends_with / eq_ignore_ascii_case (arrow-string/src/like.rs) -------
    def like_bytes(self, op, a, b, is_utf8=True):
        """a (haystack), b (pattern / needle): Utf8Column; is_utf8=False for Binary / LargeBinary."""
        assert a.offsets.dtype == b.offsets.dtype
        return self._bytes_predicate(a, b, lambda da, db, out: self.lib.acu_like_bytes(self.h, a.offsets.dtype.itemsize, int(is_utf8),
                                                                                          op, da, db, out))

    def like_view(self, op, a, b, is_utf8=True):
        """a (haystack), b (pattern / needle): ViewColumn; is_utf8=False for BinaryView."""
        return self._bytes_predicate(a, b, lambda da, db, out: self.lib.acu_like_byte_view(self.h, int(is_utf8), op, da, db, out))

    # -- length / bit_length / substring / substring_by_char (arrow-string/src/length.rs, substring.rs) ------
    def _length(self, op, col):
        n = col.length
        wide = isinstance(col, Utf8Column) and col.offsets.dtype == np.int64
        with self._scope() as s:
            out = s.out(n * (8 if wide else 4), n)
            if isinstance(col, Utf8Column):
                d = self._upload_bytes_col(col, s)
                self.check(self.lib.acu_length_bytes(self.h, col.offsets.dtype.itemsize, op, C.byref(d), C.byref(out)))
            elif isinstance(col, ViewColumn):
                d = self._upload_view_col(col, s, s.keep)
                self.check(self.lib.acu_length_byte_view(self.h, op, C.byref(d), C.byref(out)))
            else:
                d = self._upload_fsb(col, s)
                self.check(self.lib.acu_length_fixed_size_binary(self.h, col.width, op, C.byref(d), C.byref(out)))
            return self._read_out(out, I64 if wide else I32)

    def length(self, col):
        """arrow_string::length::length of a Utf8Column, ViewColumn or FixedSizeBinaryColumn: an Int32 (Int64 for i64 offsets)
        HostArray carrying the input's NullBuffer."""
        return self._length(abi.LENGTH, col)

    def bit_length(self, col):
        return self._length(abi.BIT_LENGTH, col)

    def substring(self, col, start, length=None, is_utf8=True, data_capacity=None):
        """arrow_string::substring::substring(col, start, length) of a Utf8Column (is_utf8=False: Binary / LargeBinary),
        ViewColumn (is_utf8=False: BinaryView) or FixedSizeBinaryColumn. A view result shares the input's data buffers."""
        has_len, ln = (0, 0) if length is None else (1, int(length))
        n = col.length
        with self._scope() as s:
            if isinstance(col, Utf8Column):
                d = self._upload_bytes_col(col, s)
                ob = col.offsets.dtype.itemsize
                return self._bytes_out(s, lambda oo, od, cap, tot, out: self.lib.acu_substring_bytes(
                    self.h, ob, int(is_utf8), int(start), has_len, ln, C.byref(d), col.data.nbytes, oo, od, cap, tot, out), n, ob, data_capacity)
            if isinstance(col, ViewColumn):
                d = self._upload_view_col(col, s, s.keep)
                d_views = s.malloc(n * 16 + 16)
                out = s.out(0, n)
                self.check(self.lib.acu_substring_byte_view(self.h, int(is_utf8), int(start), has_len, ln, C.byref(d), d_views, C.byref(out)))
                views = self.d2h(d_views, n * 16).reshape(n, 16)
                return ViewColumn(views, col.buffers, self._nulls_out(out, n))
            d = self._upload_fsb(col, s)
            out = s.out(n * col.width, n)
            w = C.c_int32(0)
            self.check(self.lib.acu_substring_fixed_size_binary(self.h, col.width, int(start), has_len, ln, C.byref(d), C.byref(w), C.byref(out)))
            vals = self.d2h(out.values, n * w.value).reshape(n, w.value)
            return FixedSizeBinaryColumn(vals, self._nulls_out(out, n))

    def substring_by_char(self, col, start, length=None, data_capacity=None):
        """arrow_string::substring::substring_by_char of a Utf8Column (Utf8 / LargeUtf8)."""
        has_len, ln = (0, 0) if length is None else (1, int(length))
        with self._scope() as s:
            d = self._upload_bytes_col(col, s)
            ob = col.offsets.dtype.itemsize
            return self._bytes_out(s, lambda oo, od, cap, tot, out: self.lib.acu_substring_by_char(
                self.h, ob, int(start), has_len, ln, C.byref(d), oo, od, cap, tot, out), col.length, ob, data_capacity)

    # -- concat_elements (arrow-string/src/concat_elements.rs) ------------------------------------------------------
    @staticmethod
    def _concat_type(col, is_utf8):
        """Display of the DataType concat_elements_dyn matches on."""
        if isinstance(col, Utf8Column):
            large = "Large" if col.offsets.dtype == np.int64 else ""
            return large + ("Utf8" if is_utf8 else "Binary")
        if isinstance(col, ViewColumn):
            return "Utf8View" if is_utf8 else "BinaryView"
        if isinstance(col, FixedSizeBinaryColumn):
            return f"FixedSizeBinary({col.width})"
        if isinstance(col, DecimalArray):
            return col.data_type()
        if col.dtype == BOOL:
            return "Boolean"
        return abi.DTYPE_NAMES[col.dtype].capitalize().replace("Uint", "UInt")

    def concat_elements(self, l, r, is_utf8=True, data_capacity=None):
        """arrow_string::concat_elements::concat_elements_dyn(l, r) of two Utf8Column (is_utf8=False: Binary / LargeBinary),
        ViewColumn (is_utf8=False: BinaryView) or FixedSizeBinaryColumn operands of one type. A view result has one new data
        buffer (none when no result is longer than 12 bytes). `data_capacity` as for substring."""
        lt, rt = self._concat_type(l, is_utf8), self._concat_type(r, is_utf8)
        both_fsb = isinstance(l, FixedSizeBinaryColumn) and isinstance(r, FixedSizeBinaryColumn)
        if lt != rt and not both_fsb:
            raise ArrowError(abi.ERR_COMPUTE, f"Compute error: Cannot concat arrays of different types: {lt} != {rt}")
        if not isinstance(l, (Utf8Column, ViewColumn, FixedSizeBinaryColumn)):
            raise ArrowError(abi.ERR_NOT_YET_IMPLEMENTED, f"Not yet implemented: concat not supported for {lt}")
        n = l.length
        with self._scope() as s:
            if isinstance(l, Utf8Column):
                dl, dr = self._upload_bytes_col(l, s), self._upload_bytes_col(r, s)
                ob = l.offsets.dtype.itemsize
                return self._bytes_out(s, lambda oo, od, cap, tot, out: self.lib.acu_concat_elements_bytes(
                    self.h, ob, C.byref(dl), C.byref(dr), oo, od, cap, tot, out), n, ob, data_capacity)
            if isinstance(l, ViewColumn):
                dl, dr = self._upload_view_col(l, s, s.keep), self._upload_view_col(r, s, s.keep)
                d_views = s.malloc(n * 16 + 16)
                out = s.out(0, n)
                total = C.c_int64(0)
                self.check(self.lib.acu_concat_elements_byte_view(self.h, C.byref(dl), C.byref(dr), None, None, 0, C.byref(total), C.byref(out)))
                cap = total.value if data_capacity is None else data_capacity
                d_data = s.malloc(cap + 16)
                self.check(self.lib.acu_concat_elements_byte_view(self.h, C.byref(dl), C.byref(dr), d_views, d_data, cap, C.byref(total),
                                                                  C.byref(out)))
                views = self.d2h(d_views, n * 16).reshape(n, 16)
                buffers = [self.d2h(d_data, total.value)] if total.value else []
                return ViewColumn(views, buffers, self._nulls_out(out, n))
            dl, dr = self._upload_fsb(l, s), self._upload_fsb(r, s)
            out = s.out(n * (l.width + r.width), n)
            w = C.c_int32(0)
            self.check(self.lib.acu_concat_elements_fixed_size_binary(self.h, l.width, C.byref(dl), r.width, C.byref(dr), C.byref(w),
                                                                      C.byref(out)))
            vals = self.d2h(out.values, n * w.value).reshape(n, w.value)
            return FixedSizeBinaryColumn(vals, self._nulls_out(out, n))

    def concat_elements_utf8_many(self, cols, data_capacity=None):
        """arrow_string::concat_elements::concat_elements_utf8_many of Utf8Column operands with one offset width (the device
        path is the same for Binary / LargeBinary operands)."""
        with self._scope() as s:
            descs = (abi.BytesArray * max(len(cols), 1))(*[self._upload_bytes_col(c, s) for c in cols])
            ob = cols[0].offsets.dtype.itemsize if cols else 4
            n = cols[0].length if cols else 0
            return self._bytes_out(s, lambda oo, od, cap, tot, out: self.lib.acu_concat_elements_bytes_many(
                self.h, ob, len(cols), descs, oo, od, cap, tot, out), n, ob, data_capacity)

    # -- fused compare -> filter (cmp.rs:220-382 feeding filter.rs:254-273) -------------------
    def filter_cmp(self, values, op, a, b):
        """filter(values, &cmp::op(a, b)?) with the predicate never materialised: the comparison writes the filter plan."""
        self.check_decimal_cmp(op, a, b)
        assert a.dtype == b.dtype
        with self._scope() as s:
            ad, bd = s.upload(a).descriptor(), s.upload(b).descriptor()
            plan = s.plan()
            self.check(self.lib.acu_filter_plan_create_cmp(self.h, a.dtype, op, C.byref(ad), C.byref(bd), C.byref(plan)))
            res = self._filter_with_plan(values, plan)
            return res, (self.lib.acu_filter_plan_count(plan), self.lib.acu_filter_plan_strategy(plan))

    # -- nullif / zip (arrow-select/src/nullif.rs, zip.rs) ------------------------------------
    def nullif(self, left, right):
        """arrow::compute::nullif(left, right): same values, validity &= !(right is Some(true))."""
        with self._scope() as s:
            ld, rd = s.upload(left).descriptor(), s.upload(right).descriptor()
            out = s.out(0, max(left.length, 1))
            self.check(self.lib.acu_nullif(self.h, C.byref(ld), C.byref(rd), C.byref(out)))
            n = out.len
            nulls = self._nulls_out(out, n)
        if n == 0:  # the array is returned as it is
            return left
        # the result shares left's value buffer (logical slice starting at row 0)
        vals = left.values if left.dtype == BOOL else left.values[:n]
        return HostArray(left.dtype, vals, n, nulls.validity, 0, left.values_offset if left.dtype == BOOL else 0, nulls.null_count)

    @staticmethod
    def _zip_type(col):
        """What zip compares for "the same data type": the column class plus its offset width / byte width / dtype."""
        if isinstance(col, Utf8Column):
            return ("bytes", col.offsets.dtype.itemsize)
        if isinstance(col, ViewColumn):
            return ("view",)
        if isinstance(col, FixedSizeBinaryColumn):
            return ("fsb", col.width)
        return ("array", col.dtype)

    def zip(self, mask, truthy, falsy):
        """arrow::compute::zip(mask, truthy, falsy) for primitive, Boolean (HostArray), Utf8 / Binary (Utf8Column), view
        (ViewColumn) and FixedSizeBinary (FixedSizeBinaryColumn) operands; a scalar is a one-row operand marked is_scalar
        (nulls.is_scalar for the column classes). A view result references truthy's data buffers, falsy's, both (truthy's
        first) or none, as the reference decides."""
        typed = (Utf8Column, ViewColumn, FixedSizeBinaryColumn)
        if isinstance(truthy, typed) or isinstance(falsy, typed) or truthy.dtype == BOOL or falsy.dtype == BOOL:
            return self._zip_columns(mask, truthy, falsy)
        assert truthy.dtype == falsy.dtype and truthy.dtype != BOOL
        n = mask.length
        return self._call_out((mask, truthy, falsy), n * truthy.width(), max(n, 1),
                              lambda md, td, fd, out: self.lib.acu_zip(self.h, truthy.width(), md, td, fd, out), truthy.dtype)

    def _zip_columns(self, mask, truthy, falsy):
        if self._zip_type(truthy) != self._zip_type(falsy):  # zip.rs:117-121 / ScalarZipper::try_new
            raise ArrowError(abi.ERR_INVALID_ARGUMENT, "Invalid argument error: arguments need to have the same data type")
        n = mask.length
        with self._scope() as s:
            md = s.upload(mask).descriptor()
            if isinstance(truthy, Utf8Column):
                dt, df = self._upload_bytes_col(truthy, s), self._upload_bytes_col(falsy, s)
                ob = truthy.offsets.dtype.itemsize
                return self._bytes_out(s, lambda oo, od, cap, tot, out: self.lib.acu_zip_bytes(
                    self.h, ob, C.byref(md), C.byref(dt), C.byref(df), oo, od, cap, tot, out), n, ob)
            if isinstance(truthy, ViewColumn):
                dt, df = self._upload_view_col(truthy, s, s.keep), self._upload_view_col(falsy, s, s.keep)
                d_views = s.malloc(n * 16 + 16)
                out = s.out(0, n)
                which = C.c_int32(-1)
                self.check(self.lib.acu_zip_byte_view(self.h, C.byref(md), C.byref(dt), C.byref(df), d_views, C.byref(out), C.byref(which)))
                buffers = {abi.ZIP_BUFFERS_NONE: [], abi.ZIP_BUFFERS_TRUTHY: list(truthy.buffers), abi.ZIP_BUFFERS_FALSY: list(falsy.buffers),
                           abi.ZIP_BUFFERS_BOTH: list(truthy.buffers) + list(falsy.buffers)}[which.value]
                return ViewColumn(self.d2h(d_views, n * 16).reshape(n, 16), buffers, self._nulls_out(out, n))
            if isinstance(truthy, FixedSizeBinaryColumn):
                dt, df = self._upload_fsb(truthy, s), self._upload_fsb(falsy, s)
                out = s.out(n * truthy.width, n)
                self.check(self.lib.acu_zip_fixed_size_binary(self.h, truthy.width, C.byref(md), C.byref(dt), C.byref(df), C.byref(out)))
                return self._fsb_out(out, n, truthy.width)
            dt, df = s.upload(truthy).descriptor(), s.upload(falsy).descriptor()
            out = s.out(bitmap_bytes(n), n)
            self.check(self.lib.acu_zip_boolean(self.h, C.byref(md), C.byref(dt), C.byref(df), C.byref(out)))
            return self._read_out(out, BOOL)

    # -- boolean (arrow-arith/src/boolean.rs) -------------------------------------------------
    def boolean(self, op, a, b=None):
        n = max(a.length, 1)
        return self._call_out((a, b), bitmap_bytes(n), n, lambda ad, bd, out: self.lib.acu_boolean(self.h, op, ad, bd, out), BOOL)

    def and_(self, a, b): return self.boolean(abi.BOOL_AND, a, b)
    def or_(self, a, b): return self.boolean(abi.BOOL_OR, a, b)
    def and_not(self, a, b): return self.boolean(abi.BOOL_AND_NOT, a, b)
    def and_kleene(self, a, b): return self.boolean(abi.BOOL_AND_KLEENE, a, b)
    def or_kleene(self, a, b): return self.boolean(abi.BOOL_OR_KLEENE, a, b)
    def not_(self, a): return self.boolean(abi.BOOL_NOT, a)
    def is_null(self, a): return self.boolean(abi.BOOL_IS_NULL, a)
    def is_not_null(self, a): return self.boolean(abi.BOOL_IS_NOT_NULL, a)

    def eq(self, a, b): return self.cmp(EQ, a, b)
    def neq(self, a, b): return self.cmp(NEQ, a, b)
    def lt(self, a, b): return self.cmp(LT, a, b)
    def lt_eq(self, a, b): return self.cmp(LT_EQ, a, b)
    def gt(self, a, b): return self.cmp(GT, a, b)
    def gt_eq(self, a, b): return self.cmp(GT_EQ, a, b)
    def distinct(self, a, b): return self.cmp(DISTINCT, a, b)
    def not_distinct(self, a, b): return self.cmp(NOT_DISTINCT, a, b)

    # -- cast (arrow-cast/src/cast/mod.rs) -----------------------------------------------------
    def cast(self, a, to_dtype, safe=True):
        return self._call_out((a,), a.length * abi.DTYPE_SIZE[to_dtype], a.length,
                              lambda ad, out: self.lib.acu_cast_numeric(self.h, a.dtype, to_dtype, int(safe), ad, out), to_dtype)

    # -- decimal casts (arrow-cast/src/cast/decimal.rs) -------------------------------------------
    def cast_decimal(self, a, byte_width, precision, scale, safe=True):
        """cast(DecimalArray, Decimal{32,64,128}(precision, scale)) -> DecimalArray."""
        ft, tt = abi.DecimalType(a.byte_width, a.precision, a.scale), abi.DecimalType(byte_width, precision, scale)
        res = self._call_out((a,), a.length * byte_width, a.length, lambda ad, out: self.lib.acu_cast_decimal(
            self.h, C.byref(ft), C.byref(tt), int(safe), ad, out), _DECIMAL_NATIVE[byte_width])
        return DecimalArray(byte_width, precision, scale, res.values, res.length, res.validity, res.validity_offset, res.null_count)

    def cast_to_decimal(self, a, byte_width, precision, scale, safe=True):
        """cast(Int8..UInt64 / Float32 / Float64 HostArray, Decimal{32,64,128}(precision, scale)) -> DecimalArray."""
        tt = abi.DecimalType(byte_width, precision, scale)
        res = self._call_out((a,), a.length * byte_width, a.length, lambda ad, out: self.lib.acu_cast_to_decimal(
            self.h, a.dtype, C.byref(tt), int(safe), ad, out), _DECIMAL_NATIVE[byte_width])
        return DecimalArray(byte_width, precision, scale, res.values, res.length, res.validity, res.validity_offset, res.null_count)

    def cast_from_decimal(self, a, to_dtype, safe=True):
        """cast(DecimalArray, Int8..UInt64 / Float32 / Float64) -> HostArray."""
        ft = abi.DecimalType(a.byte_width, a.precision, a.scale)
        return self._call_out((a,), a.length * abi.DTYPE_SIZE[to_dtype], a.length, lambda ad, out: self.lib.acu_cast_from_decimal(
            self.h, C.byref(ft), to_dtype, int(safe), ad, out), to_dtype)

    # -- aggregate (arrow-arith/src/aggregate.rs) ----------------------------------------------
    def aggregate(self, op, a):
        if a.dtype == abi.I128:
            return self.aggregate_i128(op, a)
        bits, cnt = C.c_uint64(0), C.c_int64(0)
        with self._scope() as s:
            ad = s.upload(a).descriptor()
            self.check(self.lib.acu_aggregate(self.h, a.dtype, op, C.byref(ad), C.byref(bits), C.byref(cnt)))
        if cnt.value == 0:
            return None
        return np.array([bits.value], dtype=np.uint64).view(NP_DTYPES[a.dtype])[0].item() if abi.DTYPE_SIZE[a.dtype] == 8 \
            else np.array([bits.value], dtype=np.uint64).view(np.uint8)[: abi.DTYPE_SIZE[a.dtype]].view(NP_DTYPES[a.dtype])[0].item()

    def aggregate_i128(self, op, a):
        """sum (wrapping) / min / max of a Decimal128 column as a Python int, None without valid rows."""
        bits, cnt = (C.c_uint64 * 2)(), C.c_int64(0)
        with self._scope() as s:
            ad = s.upload(a).descriptor()
            self.check(self.lib.acu_aggregate_i128(self.h, op, C.byref(ad), bits, C.byref(cnt)))
        if cnt.value == 0:
            return None
        return halves_to_i128(np.array([[bits[0], bits[1]]], dtype=np.uint64))[0]

    def sum_checked(self, a):
        """arrow::compute::sum_checked (aggregate.rs:897): the in-order checked fold; raises ArrowError on overflow."""
        return self._checked_fold(self.lib.acu_sum_checked, a)

    def product_checked(self, a):
        """arrow::compute::product_checked (aggregate.rs:963): the in-order checked fold of mul_checked; raises ArrowError
        on the first overflowing valid row."""
        return self._checked_fold(self.lib.acu_product_checked, a)

    def _checked_fold(self, fn, a):
        bits, cnt = C.c_uint64(0), C.c_int64(0)
        with self._scope() as s:
            ad = s.upload(a).descriptor()
            self.check(fn(self.h, a.dtype, C.byref(ad), C.byref(bits), C.byref(cnt)))
        if cnt.value == 0:
            return None
        raw = np.array([bits.value], dtype=np.uint64).view(np.uint8)[: abi.DTYPE_SIZE[a.dtype]]
        return raw.view(NP_DTYPES[a.dtype])[0].item()

    def sum(self, a): return self.aggregate(SUM, a)
    def min(self, a): return self.aggregate(MIN, a)
    def max(self, a): return self.aggregate(MAX, a)
    def product(self, a): return self.aggregate(abi.PRODUCT, a)
    def bit_and(self, a): return self.aggregate(abi.BIT_AND, a)
    def bit_or(self, a): return self.aggregate(abi.BIT_OR, a)
    def bit_xor(self, a): return self.aggregate(abi.BIT_XOR, a)

    # -- min / max of byte columns, boolean min / max (aggregate.rs:372-568, :880-889) ----------
    def min_max_row(self, op, col):
        """(row, valid_count): the lowest logical row holding the minimum (op = MIN) / maximum (MAX) of a Utf8Column,
        ViewColumn or FixedSizeBinaryColumn, -1 when there is none."""
        row, cnt = C.c_int64(0), C.c_int64(0)
        with self._scope() as s:
            if isinstance(col, Utf8Column):
                d = self._upload_bytes_col(col, s)
                self.check(self.lib.acu_aggregate_bytes(self.h, col.offsets.dtype.itemsize, op, C.byref(d), C.byref(row), C.byref(cnt)))
            elif isinstance(col, ViewColumn):
                d = self._upload_view_col(col, s, s.keep)
                self.check(self.lib.acu_aggregate_byte_view(self.h, op, C.byref(d), C.byref(row), C.byref(cnt)))
            else:
                d = self._upload_fsb(col, s)
                self.check(self.lib.acu_aggregate_fixed_size_binary(self.h, col.width, op, C.byref(d), C.byref(row), C.byref(cnt)))
        return row.value, cnt.value

    def _min_max_value(self, op, col, as_str):
        row, _ = self.min_max_row(op, col)
        if row < 0:
            return None
        b = column_value(col, row)
        return b.decode() if as_str else b

    def min_string(self, col): return self._min_max_value(MIN, col, True)
    def max_string(self, col): return self._min_max_value(MAX, col, True)
    def min_binary(self, col): return self._min_max_value(MIN, col, False)
    def max_binary(self, col): return self._min_max_value(MAX, col, False)
    def min_string_view(self, col): return self._min_max_value(MIN, col, True)
    def max_string_view(self, col): return self._min_max_value(MAX, col, True)
    def min_binary_view(self, col): return self._min_max_value(MIN, col, False)
    def max_binary_view(self, col): return self._min_max_value(MAX, col, False)
    def min_fixed_size_binary(self, col): return self._min_max_value(MIN, col, False)
    def max_fixed_size_binary(self, col): return self._min_max_value(MAX, col, False)

    def aggregate_boolean(self, op, a):
        """(value, valid_count) of min_boolean (op = MIN) / max_boolean (MAX): value 0 | 1, -1 = None."""
        val, cnt = C.c_int32(0), C.c_int64(0)
        with self._scope() as s:
            ad = s.upload(a).descriptor()
            self.check(self.lib.acu_aggregate_boolean(self.h, op, C.byref(ad), C.byref(val), C.byref(cnt)))
        return val.value, cnt.value

    def _boolean_value(self, op, a):
        v, _ = self.aggregate_boolean(op, a)
        return None if v < 0 else bool(v)

    def min_boolean(self, a): return self._boolean_value(MIN, a)
    def max_boolean(self, a): return self._boolean_value(MAX, a)
    def bool_and(self, a): return self._boolean_value(MIN, a)
    def bool_or(self, a): return self._boolean_value(MAX, a)


    # -- List / LargeList / FixedSizeList (filter.rs:535-625, take.rs:646-795) -----------------
    # One C call per level: the list call returns the child's plan / row map, and the child is filtered / taken with it
    # through the entry point of its own type (the list calls again for a nested list).
    def _list_descriptor(self, col, s):
        d = abi.ListArray()
        if isinstance(col, FixedSizeListColumn):
            d.kind, d.list_size = abi.FIXED_SIZE_LIST, col.size
        else:
            d.kind = abi.LARGE_LIST if col.offsets.dtype == np.int64 else abi.LIST
            d.offsets = self._copy_in(col.offsets, s)
        d.nulls = self._upload_nulls(col.nulls, s)
        d.child_len = col.child.length
        return d

    def filter_list(self, col, predicate):
        """arrow::compute::filter of a ListColumn / FixedSizeListColumn (any nesting of the supported children)."""
        return self.filter(col, predicate)

    def _filter_with_plan(self, col, plan, child_step=None):
        """Filter any column this package filters with `plan`, one scope per nesting level.

        child_step: this level is the child of a list filtered with a plan that is not IterationStrategy::All (None at
        the top). The reference then builds every level below it with MutableArrayData, whose freeze drops a NullBuffer
        without nulls (arrow-data/src/transform/mod.rs:936), also where the child's own plan selects every row."""
        count = self.lib.acu_filter_plan_count(plan)
        with self._scope() as s:
            if isinstance(col, StructColumn):  # filter_struct (filter.rs:1010-1030): the fields, then filter_nulls
                fields = [self._filter_with_plan(f, plan, child_step) for f in col.fields]
                nd = self._upload_nulls(col.nulls, s)
                out = s.out(0, count)
                self.check(self.lib.acu_filter_nulls(self.h, plan, C.byref(nd), C.byref(out)))
                self._drop_empty_nulls(out, child_step)
                return StructColumn(fields, self._nulls_out(out, count))
            if isinstance(col, UnionColumn):
                return self._filter_union(col, plan, count, child_step, s)
            if isinstance(col, (ListColumn, FixedSizeListColumn)):
                d = self._list_descriptor(col, s)
                fixed = isinstance(col, FixedSizeListColumn)
                d_off = None if fixed else s.malloc((count + 1) * col.offsets.itemsize + 16)
                out = s.out(0, count)
                with self._scope() as cs:
                    child_plan = cs.plan()
                    self.check(self.lib.acu_filter_list(self.h, plan, C.byref(d), d_off, C.byref(out), C.byref(child_plan)))
                    # only the top level decides: under a top-level All the reference slices every level as it is
                    step = child_step if child_step is not None else count != self.lib.acu_filter_plan_len(plan)
                    child = self._filter_with_plan(col.child, child_plan, step)
                self._drop_empty_nulls(out, child_step)
                nulls = self._nulls_out(out, count)
                if fixed:
                    return FixedSizeListColumn(col.size, child, nulls)
                return ListColumn(self.d2h(d_off, (count + 1) * col.offsets.itemsize, col.offsets.dtype), child, nulls)
            if isinstance(col, FixedSizeBinaryColumn):
                d, w = self._upload_fsb(col, s), col.width
                out = s.out(count * w, count)
                self.check(self.lib.acu_filter_fixed_size_binary(self.h, plan, w, C.byref(d), C.byref(out)))
                self._drop_empty_nulls(out, child_step)
                # MutableArrayData keeps every extended row, also of width 0 (try_new's length rule is the top level's)
                return self._fsb_out(out, count if child_step else out.len, w)
            if isinstance(col, Utf8Column):
                bd = self._upload_bytes_col(col, s)
                ob = col.offsets.dtype.itemsize
                return self._bytes_out(s, lambda oo, od, cap, tot, out: self.lib.acu_filter_bytes(
                    self.h, plan, ob, bd.offsets, bd.data, C.byref(bd.nulls), oo, od, cap, tot, out), count, ob, child_step=child_step)
            if isinstance(col, ViewColumn):  # the views filter as 16-byte values; the data buffers are shared
                vd = self._upload_view_col(col, s, s.keep)
                arr = vd.nulls
                arr.values = vd.views
                out = s.out(count * 16, count)
                self.check(self.lib.acu_filter_primitive(self.h, plan, 16, C.byref(arr), C.byref(out)))
                self._drop_empty_nulls(out, child_step)
                views = self.d2h(out.values, count * 16).reshape(-1, 16)
                return ViewColumn(views, col.buffers, self._nulls_out(out, count))
            vd = s.upload(col).descriptor()
            out = s.out(count * col.width(), count)
            if col.dtype == BOOL:
                self.check(self.lib.acu_filter_boolean(self.h, plan, C.byref(vd), C.byref(out)))
            else:
                self.check(self.lib.acu_filter_primitive(self.h, plan, col.width(), C.byref(vd), C.byref(out)))
            self._drop_empty_nulls(out, child_step)
            res = self._read_out(out, col.dtype)
            return col.like(res) if isinstance(col, DecimalArray) else res

    def _union_descriptor(self, col, s):
        d = abi.UnionArray()
        d.mode, d.n_fields, d.len = col.mode, len(col.field_type_ids), col.length
        ids = (C.c_int8 * max(len(col.field_type_ids), 1))(*col.field_type_ids)
        s.keep.append(ids)
        d.field_type_ids = C.cast(ids, C.c_void_p)
        d.type_ids = self._copy_in(col.type_ids, s)
        if col.dense:
            d.offsets = self._copy_in(col.offsets, s)
        return d

    def _union_out(self, col, m, s):
        """Device buffers for acu_filter_union / acu_take_union of m output rows, and the host field starts."""
        tids = s.malloc(m + 16)
        offs = s.malloc(4 * m + 16) if col.dense else None
        rows = s.malloc(4 * m + 16) if col.dense else None
        return tids, offs, rows, (C.c_int64 * (len(col.children) + 1))()

    def _union_children(self, col, rows, starts, keep):
        """A dense union's children, child f taken / extended (keep) with rows [starts[f], starts[f + 1]) of the map."""
        children = []
        for f, child in enumerate(col.children):
            cd = abi.Array()
            cd.values, cd.len = rows + 4 * starts[f], starts[f + 1] - starts[f]
            children.append(self._take_level(child, cd, abi.I32, False, keep))
        return children

    def _filter_union(self, col, plan, count, child_step, s):
        """filter_sparse_union (filter.rs:1033-1054) / the dense MutableArrayData fallback (filter.rs:597-622,
        build_extend_dense): a dense union's children are extended row by row, so every level below it is frozen."""
        strategy = self.lib.acu_filter_plan_strategy(plan)
        if col.dense and child_step and strategy == abi.FILTER_ALL:
            # a list's child step extends every row even when its plan selects them all: the same rows as a take of 0..n
            idx = HostArray.from_numpy(U64, np.arange(count, dtype=np.uint64))
            return self._take_level(col, s.upload(idx).descriptor(), U64, False, True)
        d = self._union_descriptor(col, s)
        tids, offs, rows, starts = self._union_out(col, count, s)
        self.check(self.lib.acu_filter_union(self.h, plan, C.byref(d), tids, offs, rows, starts))
        if col.dense:
            if strategy == abi.FILTER_NONE:
                return empty_column(col)
            if strategy == abi.FILTER_ALL:
                return col.slice(0, count)  # values.slice(0, count): the children stay whole
            return UnionColumn(col.mode, col.field_type_ids, self._union_children(col, rows, starts, True),
                               self.d2h(tids, count, np.int8), self.d2h(offs, 4 * count, np.int32))
        children = [self._filter_with_plan(c, plan, child_step) for c in col.children]
        if strategy in (abi.FILTER_NONE, abi.FILTER_ALL):
            tids_h = col.type_ids[:count].copy()
        else:
            tids_h = self.d2h(tids, count, np.int8)
        return UnionColumn(col.mode, col.field_type_ids, children, tids_h)

    @staticmethod
    def _drop_empty_nulls(out, child_step):
        if child_step and out.has_validity and out.null_count == 0:
            out.has_validity = 0

    def take_list(self, col, indices, check_bounds=False):
        """arrow::compute::take of a ListColumn / FixedSizeListColumn by a HostArray of integer indices."""
        return self.take(col, indices, check_bounds)

    def _child_error_first(self, col, d, idd, index_dtype, row, s):
        """The List `col` (descriptor d) passes i32::MAX at output row `row`. The reference extends the child of rows
        0 ..= row before it unwraps that row's offset, so the child's own offset overflow comes first: raise it if there is
        one (the caller then raises the panic)."""
        if isinstance(col.child, (HostArray, ViewColumn)):
            return
        head = abi.Array.from_buffer_copy(idd)
        head.len = row
        rmap, _, _, _, cdt, _, _ = self._row_map(d, head, index_dtype, False, False, row, s)
        n0 = self._last_rows
        raw = self.d2h(idd.values + row * abi.DTYPE_SIZE[index_dtype], abi.DTYPE_SIZE[index_dtype], NP_DTYPES[index_dtype])
        ix = int(raw[0]) & (0xFFFFFFFF if index_dtype in (abi.I8, abi.I16, abi.I32) else 0xFFFFFFFFFFFFFFFF)
        w = abi.DTYPE_SIZE[cdt]
        extra = np.arange(int(col.offsets[ix]), int(col.offsets[ix + 1]), dtype=NP_DTYPES[cdt])
        full = s.malloc((n0 + len(extra)) * w + 16)
        if n0:
            self.check(self.lib.acu_memcpy_d2d(self.h, full, rmap, n0 * w))
        if len(extra):
            self.h2d(full + n0 * w, extra)
        cd = abi.Array()
        cd.values, cd.len = full, n0 + len(extra)
        self._take_level(col.child, cd, cdt, False, True)

    def _row_map(self, d, idd, index_dtype, check_bounds, keep, m, s):
        """acu_take_list both phases: (device row map, out ArrayOut of the list nulls, device offsets or None, child-index
        ArrayOut, row map dtype, offset width, a FixedSizeList's take_bits panic deferred behind its child)."""
        fixed = d.kind == abi.FIXED_SIZE_LIST
        ob = 0 if fixed else (8 if d.kind == abi.LARGE_LIST else 4)
        d_off = s.malloc((m + 1) * max(ob, 1) + 16)
        out = s.out(0, m)
        cdt = abi.U32 if fixed or d.child_len <= 0xFFFFFFFF else abi.U64
        rows = C.c_int64(0)
        cn = abi.ArrayOut()
        self.check(self.lib.acu_take_list(self.h, C.byref(d), C.byref(idd), index_dtype, int(check_bounds), int(keep), d_off, C.byref(out),
                                          cdt, None, 0, C.byref(rows), C.byref(cn)))
        n = rows.value
        rmap = s.malloc(n * abi.DTYPE_SIZE[cdt] + 16)
        cn.validity = s.malloc(bitmap_bytes(n) + 8)
        deferred = None
        try:
            self.check(self.lib.acu_take_list(self.h, C.byref(d), C.byref(idd), index_dtype, int(check_bounds), int(keep), d_off,
                                              C.byref(out), cdt, rmap, n, C.byref(rows), C.byref(cn)))
        except ArrowError as e:
            if not fixed or e.status != abi.ERR_PANIC_OUT_OF_BOUNDS:
                raise
            deferred = e
        self._last_rows = n
        return rmap, out, (d_off if ob else None), cn, cdt, ob, deferred

    def _take_level(self, col, idd, index_dtype, check_bounds, keep):
        """Take any column this package takes by the device indices `idd`, one scope per nesting level. keep: this level is
        a child step of a List / LargeList take (MutableArrayData::extend: every row keeps its range or bytes)."""
        m = idd.len
        with self._scope() as s:
            if isinstance(col, StructColumn):
                # take_impl's Struct arm (take.rs:270-298): the fields first, then the validity; check_bounds comes before
                # both, BooleanBuffer::value's panic after the fields' own errors
                nd = self._upload_nulls(col.nulls, s)
                out = s.out(0, m)
                deferred = None
                try:
                    self.check(self.lib.acu_take_nulls(self.h, C.byref(nd), C.byref(idd), index_dtype, int(check_bounds), C.byref(out)))
                except ArrowError as e:
                    if e.status != abi.ERR_PANIC_OUT_OF_BOUNDS:
                        raise
                    deferred = e
                fields = [self._take_level(f, idd, index_dtype, False, keep) for f in col.fields]
                if deferred is not None:
                    raise deferred
                nulls = self._nulls_out(out, m)
                if not col.fields and not keep and nulls.validity is None:  # new_empty_fields keeps its NullBuffer
                    nulls = HostArray(U8, np.zeros(0, np.uint8), m, pack_bits(np.ones(m, bool)), 0, 0, 0)
                return StructColumn(fields, nulls)
            if isinstance(col, UnionColumn):
                d = self._union_descriptor(col, s)
                tids, offs, rows, starts = self._union_out(col, m, s)
                deferred = None
                try:
                    self.check(self.lib.acu_take_union(self.h, C.byref(d), C.byref(idd), index_dtype, int(check_bounds), tids, offs, rows,
                                                       starts))
                except ArrowError as e:  # UnionArray::try_new validates after the children are taken
                    if not e.message.endswith(("Type Ids values must match one of the field type ids",
                                               "Offsets must be non-negative and within the length of the Array")):
                        raise
                    deferred = e
                if col.dense:
                    children = self._union_children(col, rows, starts, keep)
                else:
                    children = [self._take_level(c, idd, index_dtype, False, keep) for c in col.children]
                if deferred is not None:
                    raise deferred
                return UnionColumn(col.mode, col.field_type_ids, children, self.d2h(tids, m, np.int8),
                                   self.d2h(offs, 4 * m, np.int32) if col.dense else None)
            if isinstance(col, (ListColumn, FixedSizeListColumn)):
                d = self._list_descriptor(col, s)
                try:
                    rmap, out, d_off, cn, cdt, ob, deferred = self._row_map(d, idd, index_dtype, check_bounds, keep, m, s)
                except ArrowError as e:
                    if e.status == abi.ERR_PANIC_OUT_OF_BOUNDS and e.message.startswith("called `Option::unwrap()`"):
                        self._child_error_first(col, d, idd, index_dtype, e.index, s)
                    raise
                n = self._last_rows
                cd = abi.Array()
                cd.values, cd.len = rmap, n
                if cn.has_validity:
                    cd.validity, cd.null_count = cn.validity, cn.null_count
                # a List's child is extended (MutableArrayData); a FixedSizeList's child is taken (take_impl)
                child = self._take_level(col.child, cd, cdt, False, keep or ob != 0)
                if deferred is not None:  # take_fixed_size_list: the child's take ran first and did not fail
                    raise deferred
                nulls = self._nulls_out(out, m)
                if not ob:
                    return FixedSizeListColumn(col.size, child, nulls)
                return ListColumn(self.d2h(d_off, (m + 1) * ob, np.int32 if ob == 4 else np.int64), child, nulls)
            if isinstance(col, FixedSizeBinaryColumn):
                d, w = self._upload_fsb(col, s), col.width
                out = s.out(m * w, m)
                self.check(self.lib.acu_take_fixed_size_binary(self.h, w, C.byref(d), C.byref(idd), index_dtype, int(check_bounds),
                                                               C.byref(out)))
                return self._fsb_out(out, m if keep else out.len, w)
            if isinstance(col, Utf8Column):
                bd = self._upload_bytes_col(col, s)
                ob = col.offsets.dtype.itemsize

                def call(oo, od, cap, tot, out):
                    if keep:
                        return self.lib.acu_take_bytes_extend(self.h, ob, bd.offsets, bd.data, C.byref(bd.nulls), C.byref(idd), index_dtype,
                                                              oo, od, cap, tot, out)
                    return self.lib.acu_take_bytes(self.h, ob, bd.offsets, bd.data, C.byref(bd.nulls), C.byref(idd), index_dtype,
                                                   int(check_bounds), oo, od, cap, tot, out)
                return self._bytes_out(s, call, m, ob)
            if isinstance(col, ViewColumn):  # the views take as 16-byte values; the data buffers are shared
                vd = self._upload_view_col(col, s, s.keep)
                arr = vd.nulls
                arr.values = vd.views
                out = s.out(m * 16, m)
                self.check(self.lib.acu_take_primitive(self.h, 16, C.byref(arr), C.byref(idd), index_dtype, int(check_bounds), C.byref(out)))
                return ViewColumn(self.d2h(out.values, m * 16).reshape(-1, 16), col.buffers, self._nulls_out(out, m))
            vd = s.upload(col).descriptor()
            out = s.out(m * col.width(), m)
            if col.dtype == BOOL:
                self.check(self.lib.acu_take_boolean(self.h, C.byref(vd), C.byref(idd), index_dtype, int(check_bounds), C.byref(out)))
            else:
                self.check(self.lib.acu_take_primitive(self.h, col.width(), C.byref(vd), C.byref(idd), index_dtype, int(check_bounds),
                                                       C.byref(out)))
            res = self._read_out(out, col.dtype)
            return col.like(res) if isinstance(col, DecimalArray) else res

    # -- RunEndEncoded (filter_run_end_array filter.rs:628-677, take_run take.rs:948-995) ---------------------------
    # The run-end calls work on the run ends; the values child is filtered / taken with the plan / value indices they
    # return through the path of its own type, as a list hands its child plan / row map on.
    def _run_descriptor(self, col, owned):
        d = abi.RunArray()
        d.run_end_dtype = {2: abi.I16, 4: abi.I32, 8: abi.I64}[col.run_ends.dtype.itemsize]
        d.run_ends = self._copy_in(col.run_ends, owned)
        d.n_runs, d.offset, d.len = len(col.run_ends), col.offset, col.length
        return d

    def filter_run_end(self, col, predicate):
        """arrow::compute::filter of a RunEndColumn: the run ends keep their type, the values child is any column this
        package filters."""
        with self._scope() as s:
            plan = self._plan(s, predicate)
            d = self._run_descriptor(col, s)
            count = self.lib.acu_filter_plan_count(plan)
            w = col.run_ends.itemsize
            d_ends = s.malloc(max(min(count, len(col.run_ends)), 1) * w + 16)
            runs, vstart, vplan = C.c_int64(0), C.c_int64(0), s.plan()
            self.check(self.lib.acu_filter_run_end(self.h, plan, C.byref(d), d_ends, C.byref(runs), C.byref(vstart), C.byref(vplan)))
            if not vplan:
                if self.lib.acu_filter_plan_strategy(plan) == abi.FILTER_ALL:
                    return col.slice(0, count)  # values.slice(0, count) (filter.rs:546)
                return RunEndColumn(np.zeros(0, col.run_ends.dtype), empty_column(col.values), 0, 0)
            values = self._filter_with_plan(slice_column(col.values, vstart.value, self.lib.acu_filter_plan_len(vplan)), vplan)
            ends = self.d2h(d_ends, runs.value * w, col.run_ends.dtype)
            return RunEndColumn(ends, values, 0, int(ends[-1]))

    def _run_values(self, col, s):
        """acu_run_values of a values child for take's run merge (the uploads belong to the scope s)."""
        v = abi.RunValues()
        if isinstance(col, (ListColumn, FixedSizeListColumn, RunEndColumn, StructColumn, UnionColumn, FixedSizeBinaryColumn)):
            v.kind = abi.RUN_VALUES_NESTED
        elif isinstance(col, Utf8Column):
            v.kind, v.width, v.bytes = abi.RUN_VALUES_BYTES, col.offsets.itemsize, self._upload_bytes_col(col, s)
        elif isinstance(col, ViewColumn):
            v.kind, v.view = abi.RUN_VALUES_VIEW, self._upload_view_col(col, s, s.keep)
        else:
            v.array = s.upload(col).descriptor()
            v.kind, v.width = (abi.RUN_VALUES_BOOLEAN, 0) if col.dtype == BOOL else (abi.RUN_VALUES_FIXED, col.width())
        return v

    def take_run_end(self, col, indices, check_bounds=False):
        """arrow::compute::take of a RunEndColumn by a HostArray of integer indices (values: primitive, decimal, Boolean,
        Utf8 / Binary and view columns)."""
        with self._scope() as s:
            idd = s.upload(indices).descriptor()
            d = self._run_descriptor(col, s)
            vd = self._run_values(col.values, s)
            m = indices.length
            wide = indices.dtype in (abi.I64, abi.U64)
            d_ends = s.malloc(max(m, 1) * col.run_ends.itemsize + 16)
            d_vi = s.malloc(max(m, 1) * (8 if wide else 4) + 16)
            runs = C.c_int64(0)
            self.check(self.lib.acu_take_run_end(self.h, C.byref(d), C.byref(vd), C.byref(idd), indices.dtype, int(check_bounds), d_ends,
                                                 d_vi, C.byref(runs)))
            if m == 0:
                return RunEndColumn(np.zeros(0, col.run_ends.dtype), empty_column(col.values), 0, 0)
            cd = abi.Array()
            cd.values, cd.len = d_vi, runs.value
            values = self._take_level(col.values, cd, abi.U64 if wide else abi.U32, False, False)
            return RunEndColumn(self.d2h(d_ends, runs.value * col.run_ends.itemsize, col.run_ends.dtype), values, 0, m)
