"""Column builders and the golden-vector runner shared by the byte / boolean min-max tests (CPU oracle and GPU)."""
import json
import os

import numpy as np

from acu import MIN, U8, FixedSizeBinaryColumn, HostArray, Utf8Column, ViewColumn

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "aggregate_vectors.json")


def load_aggregate_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def _nulls(mask, bit_offset=0):
    mask = np.asarray(mask, dtype=bool)
    nulls = HostArray.from_numpy(U8, np.zeros(len(mask), np.uint8), mask if (bit_offset or not mask.all()) else None, bit_offset)
    nulls.values = np.zeros(0, np.uint8)
    return nulls


def _as_bytes(x):
    return x.encode() if isinstance(x, str) else bytes(x)


def bytes_column(items, large=False, bit_offset=0, garbage=b""):
    """Utf8Column of `items` (bytes / str / None); `garbage` = the bytes stored under every null slot."""
    vals = [garbage if x is None else _as_bytes(x) for x in items]
    lens = np.array([len(v) for v in vals], dtype=np.int64)
    offsets = np.zeros(len(vals) + 1, dtype=np.int64 if large else np.int32)
    offsets[1:] = np.cumsum(lens)
    data = np.frombuffer(b"".join(vals), dtype=np.uint8).copy()
    return Utf8Column(offsets, data, _nulls([x is not None for x in items], bit_offset))


def view_column(items, bit_offset=0, garbage_views=None, block_size=64):
    """ViewColumn of `items`; `garbage_views` = 16-byte views stored under the null slots (cycled)."""
    col = ViewColumn.from_values(items, block_size=block_size, garbage_under_nulls=garbage_views)
    col.nulls = _nulls([x is not None for x in items], bit_offset)
    return col


def fixed_column(items, width, bit_offset=0, garbage=None):
    """FixedSizeBinaryColumn of `items` (each exactly `width` bytes, or None); `garbage` fills the null slots."""
    vals = np.zeros((len(items), width), dtype=np.uint8)
    for i, x in enumerate(items):
        b = garbage if x is None else _as_bytes(x)
        if b is not None:
            vals[i] = np.frombuffer(b[:width].ljust(width, b"\0"), dtype=np.uint8)
    return FixedSizeBinaryColumn(vals, _nulls([x is not None for x in items], bit_offset))


def slice_column(col, offset, length):
    """Array::slice of a byte / view / fixed-size-binary column: offsets (views, rows) and the validity bit offset move."""
    nulls = col.nulls.slice(offset, length)
    nulls.values = np.zeros(0, np.uint8)
    if isinstance(col, Utf8Column):
        return Utf8Column(col.offsets[offset: offset + length + 1], col.data, nulls)
    if isinstance(col, ViewColumn):
        return ViewColumn(col.views[offset: offset + length], col.buffers, nulls)
    return FixedSizeBinaryColumn(col.values[offset: offset + length], nulls)


def bool_array(items, bit_offset=0, mask_offset=0):
    """BooleanArray of `items` (bool / None) with the given value / validity bit offsets."""
    mask = np.array([x is not None for x in items], dtype=bool)
    vals = np.array([bool(x) for x in items], dtype=bool)
    return HostArray.bool_from_numpy(vals, mask if (mask_offset or not mask.all()) else None, bit_offset, mask_offset)


def golden_columns(case):
    """[(form, column)] of one byte-column case, in every array type its reference test runs it on."""
    dec = (lambda x: None if x is None else bytes.fromhex(x)) if case["kind"] == "binary" else (lambda x: x)
    items = [dec(x) for x in case["data"]]
    out = []
    for form in case["forms"]:
        if form in ("binary", "utf8", "large_binary", "large_utf8"):
            col = bytes_column(items, large=form.startswith("large"))
        elif form in ("binary_view", "utf8_view"):
            col = view_column(items)
        else:  # pad_inputs_and_test_fixed_size_binary: zero-pad every value to the longest one
            width = max([len(x) for x in items if x is not None], default=0)
            col = fixed_column([None if x is None else x.ljust(width, b"\0") for x in items], width)
        if "slice" in case:
            col = slice_column(col, *case["slice"])
        out.append((form, col))
    return out


def run_golden_case(backend, case):
    """Runs one golden case through the reference-named methods of `backend` (acu.Context or the CPU oracle)."""
    if case["kind"] == "boolean":
        a = bool_array(case["data"])
        if "slice" in case:
            a = a.slice(*case["slice"])
        assert backend.min_boolean(a) == case["min"] and backend.bool_and(a) == case["min"]
        assert backend.max_boolean(a) == case["max"] and backend.bool_or(a) == case["max"]
        return
    for form, col in golden_columns(case):
        if case["kind"] == "string":
            suffix = "_view" if form.endswith("view") else ""
            got = (getattr(backend, "min_string" + suffix)(col), getattr(backend, "max_string" + suffix)(col))
            assert got == (case["min"], case["max"]), form
        else:
            suffix = {"binary": "", "large_binary": "", "binary_view": "_view", "fixed_size_binary": "_fixed_size_binary"}[form]
            fn = (lambda m: "%s_binary%s" % (m, suffix)) if suffix != "_fixed_size_binary" else (lambda m: "%s_fixed_size_binary" % m)
            got = (getattr(backend, fn("min"))(col), getattr(backend, fn("max"))(col))
            width = col.width if form == "fixed_size_binary" else None
            want = tuple(None if x is None else (bytes.fromhex(x).ljust(width, b"\0") if width is not None else bytes.fromhex(x))
                         for x in (case["min"], case["max"]))
            assert got == want, form


def literal_fold(op, items):
    """The reference's fold over a python list (bytes / None): the lowest row holding min / max(bytes)."""
    best = -1
    for i, x in enumerate(items):
        if x is None:
            continue
        if best < 0 or (x < items[best] if op == MIN else x > items[best]):
            best = i
    return best


def random_items(rng, n, null_p, alphabet=b"ab\0\xff", max_len=20, distinct=None):
    """n random byte values (None with probability null_p) from a small alphabet, so that prefixes and ties are common."""
    pool = None
    if distinct:
        pool = [rng.choice(list(alphabet), int(rng.integers(0, max_len + 1))).astype(np.uint8).tobytes() for _ in range(distinct)]
    out = []
    for _ in range(n):
        if rng.random() < null_p:
            out.append(None)
        elif pool is not None:
            out.append(pool[int(rng.integers(0, len(pool)))])
        else:
            out.append(rng.choice(list(alphabet), int(rng.integers(0, max_len + 1))).astype(np.uint8).tobytes())
    return out

