"""CPU oracle of arrow-string/src/length.rs and substring.rs, restated literally in Python integers (wrapping offsets,
as_usize of negative offsets, is_char_boundary against the whole value-data buffer, the slice panics). Errors are raised
as acu.ArrowError with the status, message and row the device reports. Same method names and outputs as acu.Context:
length / bit_length / substring / substring_by_char over Utf8Column, ViewColumn and FixedSizeBinaryColumn."""
import numpy as np

import acu
from acu import FixedSizeBinaryColumn, HostArray, Utf8Column, ViewColumn, column_value, pack_bits
from acu import _abi as abi

ERR_COMPUTE, ERR_PANIC = 2, 8
U64 = (1 << 64) - 1


def wrap(v, bits):
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def as_usize(v):
    return v & U64


def is_cont(b):
    return 0x80 <= b <= 0xBF


def is_char_boundary(buf, pos):
    """str::is_char_boundary at usize `pos`."""
    return pos == 0 or pos == len(buf) or (pos < len(buf) and not is_cont(buf[pos]))


def boundary_error(off, row):
    return acu.ArrowError(ERR_COMPUTE, f"Compute error: The offset {off} is at an invalid utf-8 boundary.", row)


def slice_panic(s, e, n, row):
    if s > e:
        return acu.ArrowError(ERR_PANIC, f"slice index starts at {s} but ends at {e}", row)
    return acu.ArrowError(ERR_PANIC, f"range end index {e} out of range for slice of length {n}", row)


def valid_mask(col):
    return col.nulls.valid_mask()


def nulls_cloned(col):
    """nulls.cloned(): the input's NullBuffer as it is (present iff it has a validity buffer)."""
    n, m = col.length, valid_mask(col)
    if col.nulls.validity is None:
        return None, 0
    return pack_bits(m), int(n - m.sum())


def nulls_unsliced(col):
    """NullBuffer::from_unsliced_buffer: None without a null."""
    validity, nc = nulls_cloned(col)
    return (validity, nc) if nc > 0 else (None, 0)


def null_host(n, validity, nc):
    return HostArray(abi.U8, np.zeros(0, np.uint8), n, validity, 0, 0, nc)


def bytes_column(values, offsets_dtype, validity, nc):
    offs, data = [0], bytearray()
    for v in values:
        data += v
        offs.append(len(data))
    return Utf8Column(np.array(offs, dtype=offsets_dtype), np.frombuffer(bytes(data), dtype=np.uint8).copy(),
                      null_host(len(values), validity, nc))


def view_range(L, start, length):
    """view_substring_range (substring.rs:254-271)."""
    s = min(start, L) if start > 0 else 0 if start == 0 else max(L + start, 0)
    if length is None:
        return s, L
    x = min(s + wrap(length, 64), (1 << 63) - 1)  # saturating_add of `length as i64`
    return s, min(x, L)


def char_bounds(val, start, length):
    """utf8_bounds (substring.rs:219-251) on a valid UTF-8 value."""
    L = len(val)
    starts = [k for k, b in enumerate(val) if not is_cont(b)]
    if start >= 0:
        s = starts[start] if start < len(starts) else L
    else:
        back = -start
        s = starts[len(starts) - back] if back <= len(starts) else 0
    if length is None or length >= L - s:
        return s, L
    rel = [k for k in starts if k >= s]
    return s, (rel[length] if length < len(rel) else L)


class SubstringOracle:
    def _length(self, col, shift):
        n = col.length
        if isinstance(col, Utf8Column):
            bits = 8 * col.offsets.dtype.itemsize
            o = [int(x) for x in col.offsets[: n + 1]]
            vals = [wrap((o[i + 1] - o[i]) << shift, bits) for i in range(n)]
            dtype = abi.I32 if bits == 32 else abi.I64
        elif isinstance(col, ViewColumn):
            lens = np.frombuffer(np.ascontiguousarray(col.views[:n, :4]).tobytes(), dtype=np.uint32) if n else np.zeros(0, np.uint32)
            vals = [wrap(int(x) << shift, 32) for x in lens]
            dtype = abi.I32
        else:
            vals = [wrap(col.width << shift, 32)] * n
            dtype = abi.I32
        validity, nc = nulls_cloned(col)
        return HostArray(dtype, np.array(vals, dtype=acu.NP_DTYPES[dtype]), n, validity, 0, 0, nc)

    def length(self, col):
        return self._length(col, 0)

    def bit_length(self, col):
        return self._length(col, 3)

    def substring(self, col, start, length=None, is_utf8=True, data_capacity=None):
        if isinstance(col, Utf8Column):
            return self._byte_substring(col, start, length, is_utf8, data_capacity)
        if isinstance(col, ViewColumn):
            return self._view_substring(col, start, length, is_utf8)
        return self._fsb_substring(col, start, length)

    def _byte_substring(self, col, start, length, is_utf8, data_capacity):
        n, bits = col.length, 8 * col.offsets.dtype.itemsize
        st, ln = wrap(start, bits), None if length is None else wrap(length, bits)  # `start as i32`, `length as i32`
        o = [int(x) for x in col.offsets[: n + 1]]
        data = bytes(col.data)
        ranges = []
        for i in range(n):
            p0, p1 = o[i], o[i + 1]
            s = min(wrap(p0 + st, bits), p1) if st > 0 else p0 if st == 0 else max(wrap(p1 + st, bits), p0)
            if is_utf8 and st != 0 and not is_char_boundary(data, as_usize(s)):
                raise boundary_error(as_usize(s), i)
            e = p1 if ln is None else min(wrap(ln + s, bits), p1)
            if is_utf8 and ln is not None and not is_char_boundary(data, as_usize(e)):
                raise boundary_error(as_usize(e), i)
            ranges.append((as_usize(s), as_usize(e)))
        for i, (s, e) in enumerate(ranges):
            if s > e or e > len(data):
                raise slice_panic(s, e, len(data), i)
        out = [data[s:e] for s, e in ranges]
        if data_capacity is not None and data_capacity < sum(map(len, out)):
            raise acu.ArrowError(1, f"Invalid argument error: output data capacity {data_capacity} < required {sum(map(len, out))}", -1)
        return bytes_column(out, col.offsets.dtype, *nulls_unsliced(col))

    def _view_substring(self, col, start, length, is_utf8):
        m, out = valid_mask(col), []
        for i in range(col.length):
            if not m[i]:
                out.append(None)
                continue
            val = column_value(col, i)
            s, e = view_range(len(val), start, length)
            if is_utf8:
                for off in (s, e):
                    if not is_char_boundary(val, as_usize(off)):
                        raise boundary_error(as_usize(off), i)
            us, ue = as_usize(s), as_usize(e)
            if us > ue or ue > len(val):
                raise slice_panic(us, ue, len(val), i)
            out.append(val[s:e])
        return ViewColumn.from_values(out)

    def _fsb_substring(self, col, start, length):
        w, n = col.width, col.length
        new_start = min(start, w) if start > 0 else 0 if start == 0 else max(w - (-start), 0)
        new_len = w - new_start if length is None else min(length, w - new_start)
        vals = np.ascontiguousarray(col.values[:n, new_start:new_start + new_len]).reshape(n, new_len)
        validity, nc = nulls_unsliced(col)
        if new_len == 0 and validity is None:  # substring.rs:444-450
            validity, nc = pack_bits(np.ones(n, dtype=bool)), 0
        return FixedSizeBinaryColumn(vals, null_host(n, validity, nc))

    def substring_by_char(self, col, start, length=None, data_capacity=None):
        m, out = valid_mask(col), []
        for i in range(col.length):
            if not m[i]:
                out.append(b"")  # null slots become empty
                continue
            val = column_value(col, i)
            s, e = char_bounds(val, start, length)
            out.append(val[s:e])
        if data_capacity is not None and data_capacity < sum(map(len, out)):
            raise acu.ArrowError(1, f"Invalid argument error: output data capacity {data_capacity} < required {sum(map(len, out))}", -1)
        return bytes_column(out, col.offsets.dtype, *nulls_unsliced(col))
