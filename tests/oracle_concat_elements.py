"""CPU oracle of arrow-string/src/concat_elements.rs, restated in Python bytes and integers: every row concatenated (the
bytes under null slots included), NullBuffer::union (None unless some row is null), the i32 `from_usize(..).unwrap()` panic
row, FixedSizeBinary null rows as zero bytes, and the view builder's exact layout (inline views, one new data buffer in row
order). Errors are raised as acu.ArrowError with the status, message (the ArrowError Display, or the panic text) and
row the device reports. Same method names and outputs as acu.Context: concat_elements / concat_elements_utf8_many."""
import numpy as np

import acu
from acu import FixedSizeBinaryColumn, HostArray, Utf8Column, ViewColumn, column_value, pack_bits
from acu import _abi as abi

I32_MAX = 2**31 - 1
UNWRAP_NONE = "called `Option::unwrap()` on a `None` value"


def wrap32(v):
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >> 31 else v


def union_nulls(cols):
    """NullBuffer::union folded over the operands: the AND of the present validity masks, None without a null."""
    n = cols[0].length
    mask = np.ones(n, dtype=bool)
    for c in cols:
        if c.nulls.validity is not None:
            mask &= c.nulls.valid_mask()
    nc = int(n - mask.sum())
    return (pack_bits(mask), nc, mask) if nc else (None, 0, mask)


def nulls_host(n, validity, nc):
    return HostArray(abi.U8, np.zeros(0, np.uint8), n, validity, 0, 0, nc)


def first_overflow_row(row_lengths):
    """The first row whose running end passes i32::MAX, or None: the row `from_usize(..).unwrap()` panics at."""
    ends = np.cumsum(np.asarray(row_lengths, dtype=np.int64))
    over = np.nonzero(ends > I32_MAX)[0]
    return int(over[0]) if over.size else None


def raw_value(col, i):
    """The bytes of slot i of a Utf8Column, null or not (offsets[i]..offsets[i+1] of the value data)."""
    return bytes(col.data[int(col.offsets[i]): int(col.offsets[i + 1])])


def make_view(b, offset):
    """make_view(b, 0, offset) of the reference's builder: 16 bytes."""
    v = np.zeros(16, dtype=np.uint8)
    v[:4] = np.frombuffer(np.uint32(len(b)).tobytes(), dtype=np.uint8)
    if len(b) <= 12:
        v[4:4 + len(b)] = np.frombuffer(b, dtype=np.uint8)
    else:
        v[4:8] = np.frombuffer(b[:4], dtype=np.uint8)
        v[12:16] = np.frombuffer(np.uint32(offset).tobytes(), dtype=np.uint8)
    return v


class ConcatElementsOracle:
    @staticmethod
    def type_name(col, is_utf8):
        return acu.Context._concat_type(col, is_utf8)

    def _bytes(self, cols):
        n, ob = cols[0].length, cols[0].offsets.dtype.itemsize
        offs, data = [0], bytearray()
        for i in range(n):
            for c in cols:
                data += raw_value(c, i)
            if ob == 4 and len(data) > I32_MAX:
                raise acu.ArrowError(abi.ERR_PANIC_OUT_OF_BOUNDS, UNWRAP_NONE, i)
            offs.append(len(data))
        validity, nc, _ = union_nulls(cols)
        return Utf8Column(np.array(offs, dtype=cols[0].offsets.dtype), np.frombuffer(bytes(data), dtype=np.uint8).copy(),
                          nulls_host(n, validity, nc))

    def _views(self, l, r):
        n = l.length
        validity, nc, mask = union_nulls([l, r])
        vals = [column_value(l, i) + column_value(r, i) if mask[i] else None for i in range(n)]
        if sum(len(v) for v in vals if v is not None and len(v) > 12) > I32_MAX:
            raise acu.ArrowError(abi.ERR_ARITHMETIC_OVERFLOW, "Arithmetic overflow: byte array offset overflow")
        views, data = np.zeros((n, 16), dtype=np.uint8), bytearray()
        for i, v in enumerate(vals):
            if v is None:
                continue  # append_empty_view
            views[i] = make_view(v, len(data))
            if len(v) > 12:
                data += v
        buffers = [np.frombuffer(bytes(data), dtype=np.uint8).copy()] if data else []
        return ViewColumn(views, buffers, nulls_host(n, validity, nc))

    def _fsb(self, l, r):
        for w in (l.width, r.width):
            if w < 0:
                raise acu.ArrowError(abi.ERR_INVALID_ARGUMENT, f"Invalid argument error: Invalid size of FixedSizeBinaryArray({w})")
        w = l.width + r.width
        if wrap32(w) < 0:
            raise acu.ArrowError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"value length ({wrap32(w)}) of the array must >= 0")
        validity, nc, mask = union_nulls([l, r])
        vals = np.zeros((l.length, w), dtype=np.uint8)
        for i in range(l.length):
            if mask[i]:
                vals[i] = np.frombuffer(bytes(l.values[i]) + bytes(r.values[i]), dtype=np.uint8)
        return FixedSizeBinaryColumn(vals, nulls_host(l.length, validity, nc))

    def concat_elements(self, l, r, is_utf8=True, data_capacity=None):
        """concat_elements_dyn (concat_elements.rs:419-476)."""
        lt, rt = self.type_name(l, is_utf8), self.type_name(r, is_utf8)
        both_fsb = isinstance(l, FixedSizeBinaryColumn) and isinstance(r, FixedSizeBinaryColumn)
        if lt != rt and not both_fsb:
            raise acu.ArrowError(abi.ERR_COMPUTE, f"Compute error: Cannot concat arrays of different types: {lt} != {rt}")
        if not isinstance(l, (Utf8Column, ViewColumn, FixedSizeBinaryColumn)):
            raise acu.ArrowError(abi.ERR_NOT_YET_IMPLEMENTED, f"Not yet implemented: concat not supported for {lt}")
        if l.length != r.length:
            raise acu.ArrowError(abi.ERR_COMPUTE, f"Compute error: Arrays must have the same length: {l.length} != {r.length}")
        if isinstance(l, Utf8Column):
            out = self._bytes([l, r])
        elif isinstance(l, ViewColumn):
            out = self._views(l, r)
        else:
            return self._fsb(l, r)
        self._check_capacity(out, data_capacity)
        return out

    def concat_elements_utf8_many(self, cols, data_capacity=None):
        """concat_elements_utf8_many (concat_elements.rs:113-173)."""
        if not cols:
            raise acu.ArrowError(abi.ERR_COMPUTE, "Compute error: concat requires input of at least one array")
        size = cols[0].length
        if any(c.length != size for c in cols):
            raise acu.ArrowError(abi.ERR_COMPUTE, f"Compute error: Arrays must have the same length of {size}")
        out = self._bytes(cols)
        self._check_capacity(out, data_capacity)
        return out

    @staticmethod
    def _check_capacity(out, cap):
        need = len(out.data) if isinstance(out, Utf8Column) else sum(len(b) for b in out.buffers)
        if cap is not None and need > cap:
            raise acu.ArrowError(abi.ERR_INVALID_ARGUMENT, f"Invalid argument error: output data capacity {cap} < required {need}")
