"""Shared helpers of the zip tests: columns from the golden file's description, and the comparison of a device result with
an oracle_zip.ZipResult, bit for bit."""
import json
import os

import numpy as np

from acu import BOOL, FixedSizeBinaryColumn, HostArray, Utf8Column, ViewColumn, pack_bits, unpack_bits
from acu import _abi as abi

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "zip_vectors.json")


def golden_cases():
    with open(GOLDEN) as f:
        return json.load(f)


def nulls(valid, scalar=False, bit_offset=0, n=None):
    """The validity-only HostArray of an n-row column: `valid` (bools) or None for no NullBuffer."""
    if valid is None:
        return HostArray(abi.U8, np.zeros(0, np.uint8), (1 if scalar else 0) if n is None else n, None, 0, 0, 0, scalar)
    valid = np.asarray(valid, bool)
    return HostArray(abi.U8, np.zeros(0, np.uint8), len(valid), pack_bits(valid, bit_offset), bit_offset, 0,
                     int(len(valid) - valid.sum()), scalar)


def mask_array(values, valid=None, bit_offset=0):
    return HostArray.bool_from_numpy(np.asarray(values, bool), None if valid is None else np.asarray(valid, bool), bit_offset, bit_offset)


def bytes_column(items, ob=4, scalar=False, force_validity=False):
    """Utf8Column of bytes / None items (a null row is empty)."""
    items = [None if x is None else (x.encode() if isinstance(x, str) else bytes(x)) for x in items]
    lens = [0 if x is None else len(x) for x in items]
    offs = np.zeros(len(items) + 1, np.int32 if ob == 4 else np.int64)
    offs[1:] = np.cumsum(lens)
    data = np.frombuffer(b"".join(x for x in items if x is not None), np.uint8).copy()
    valid = [x is not None for x in items]
    nb = nulls(valid if (force_validity or not all(valid)) else None, scalar)
    nb.length = len(items)
    return Utf8Column(offs, data, nb)


def view_column(items, scalar=False, block_size=64):
    col = ViewColumn.from_values(items, block_size=block_size, scalar=scalar)
    return col


def bool_column(items, raw=None, scalar=False):
    vals = [bool(x[0]) if x is not None else False for x in items] if raw is None else [bool(x[0]) for x in raw]
    valid = [x is not None for x in items]
    h = HostArray.bool_from_numpy(np.array(vals, bool), None if all(valid) else np.array(valid))
    h.is_scalar = scalar
    return h


def fsb_column(items, w, raw=None, scalar=False):
    src = raw if raw is not None else [bytes(w) if x is None else x for x in items]
    vals = np.frombuffer(b"".join(bytes(x) for x in src), np.uint8).reshape(len(src), w) if src else np.zeros((0, w), np.uint8)
    valid = [x is not None for x in items]
    nb = nulls(None if all(valid) else valid, scalar)
    nb.length = len(items)
    return FixedSizeBinaryColumn(vals.copy(), nb)


def golden_side(case, key):
    d, typ = case[key], case["type"]
    items = [None if v is None else bytes.fromhex(v) for v in d["values"]]
    raw = None if "raw" not in d else [bytes.fromhex(v) for v in d["raw"]]
    sc = d["scalar"]
    if typ in ("utf8", "binary", "large_utf8", "large_binary"):
        return bytes_column(items, 8 if typ.startswith("large") else 4, sc)
    if typ in ("utf8view", "binaryview"):
        return view_column(items, sc)
    if typ == "boolean":
        return bool_column(items, raw, sc)
    return fsb_column(items, case["width"], raw, sc)


def golden_mask(case):
    m = case["mask"]
    return mask_array(m["values"], m["valid"])


def logical_rows(col):
    """Every row's value as bytes, None for a null row, of a host column or a device result."""
    if isinstance(col, Utf8Column):
        valid = col.nulls.valid_mask()
        return [bytes(col.data[int(col.offsets[i]) - int(col.offsets[0]):int(col.offsets[i + 1]) - int(col.offsets[0])])
                if valid[i] else None for i in range(col.length)]
    if isinstance(col, ViewColumn):
        return col.values()
    if isinstance(col, FixedSizeBinaryColumn):
        valid = col.nulls.valid_mask()
        return [bytes(col.values[i]) if valid[i] else None for i in range(col.length)]
    return [bytes([int(v)]) if m else None for v, m in zip(col.value_array(), col.valid_mask())]


def raw_rows(col):
    if isinstance(col, FixedSizeBinaryColumn):
        return [bytes(r) for r in col.values]
    return [bytes([int(v)]) for v in col.value_array()]


def oracle_as_column(r, t, f):
    """An oracle ZipResult as the host column the device call returns (views reference t's / f's buffers)."""
    nb = nulls(r.valid)
    nb.length = r.n
    if r.kind == "bytes":
        return Utf8Column(r.offsets, r.data, nb)
    if r.kind == "view":
        bufs = {abi.ZIP_BUFFERS_NONE: [], abi.ZIP_BUFFERS_TRUTHY: list(t.buffers), abi.ZIP_BUFFERS_FALSY: list(f.buffers),
                abi.ZIP_BUFFERS_BOTH: list(t.buffers) + list(f.buffers)}[r.buffers]
        return ViewColumn(r.views, bufs, nb)
    if r.kind == "fsb":
        return FixedSizeBinaryColumn(r.values, nb)
    return HostArray(BOOL, pack_bits(r.values), r.n, nb.validity, 0, 0, nb.null_count)


def assert_same(got, r, t, f):
    """The device result `got` equals the oracle result `r` bit for bit: offsets, data, views, the buffer list, value bits and
    bytes under nulls, NullBuffer presence, its bits and its null count."""
    n = r.n
    g_nulls = got if isinstance(got, HostArray) else got.nulls
    assert g_nulls.length == n if not isinstance(got, Utf8Column) else got.length == n
    assert (g_nulls.validity is not None) == (r.valid is not None), "NullBuffer presence"
    if r.valid is not None:
        np.testing.assert_array_equal(unpack_bits(g_nulls.validity, g_nulls.validity_offset, n), r.valid)
        assert g_nulls.null_count == int(n - r.valid.sum())
    if r.kind == "bytes":
        np.testing.assert_array_equal(np.asarray(got.offsets), r.offsets)
        assert got.offsets.dtype == r.offsets.dtype
        if r.data is not None:
            np.testing.assert_array_equal(np.asarray(got.data), r.data)
    elif r.kind == "view":
        np.testing.assert_array_equal(np.asarray(got.views).reshape(n, 16), r.views)
        exp = oracle_as_column(r, t, f).buffers
        assert [id(b) for b in got.buffers] == [id(b) for b in exp], "data-buffer list"
    elif r.kind == "fsb":
        np.testing.assert_array_equal(np.asarray(got.values).reshape(r.values.shape), r.values)
    else:
        np.testing.assert_array_equal(unpack_bits(got.values, got.values_offset, n), r.values)
