"""Columns for the length / substring tests: the golden cases of tests/golden/substring_vectors.json expanded into the
array types they name, and random columns for the fuzz tests."""
import json
import os

import numpy as np

from acu import FixedSizeBinaryColumn, HostArray, Utf8Column, ViewColumn, column_value
from acu import _abi as abi

from oracle_filter_take import nulls_of

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "substring_vectors.json")
OFFSET_DTYPE = {"utf8": np.int32, "binary": np.int32, "large_utf8": np.int64, "large_binary": np.int64}


def golden_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def decode(items):
    return [None if x is None else bytes.fromhex(x) for x in items]


def bytes_col(items, dtype, garbage=b""):
    """A Utf8Column of `items` (bytes / None); `garbage` bytes are left under every null slot."""
    offs, data = [0], bytearray()
    for it in items:
        data += garbage if it is None else it
        offs.append(len(data))
    return Utf8Column(np.array(offs, dtype=dtype), np.frombuffer(bytes(data), dtype=np.uint8).copy(),
                      nulls_of([it is not None for it in items]))


def fsb_col(items, width):
    return FixedSizeBinaryColumn.from_values([None if it is None else it for it in items], width)


def column(typ, items):
    if typ in OFFSET_DTYPE:
        return bytes_col(items, OFFSET_DTYPE[typ])
    if typ in ("utf8_view", "binary_view"):
        return ViewColumn.from_values(items)
    width = max([len(x) for x in items if x is not None] + [0])
    return fsb_col(items, width)


def values(col):
    m = col.nulls.valid_mask()
    return [column_value(col, i) if m[i] else None for i in range(col.length)]


def sliced(col, off, n):
    """Array::slice of a Utf8Column: offsets start mid-buffer, the validity keeps a bit offset."""
    return Utf8Column(col.offsets[off:off + n + 1], col.data, col.nulls.slice(off, n))


def golden_inputs(case):
    """(array type, is_utf8, column) for every type the case names."""
    out = []
    for typ in case["types"]:
        utf8 = typ in ("utf8", "large_utf8", "utf8_view")
        k = case["kind"]
        if k == "sliced":
            dt = OFFSET_DTYPE[typ]
            full = Utf8Column(np.array(case["offsets"], dtype=dt), np.frombuffer(bytes.fromhex(case["data"]), dtype=np.uint8).copy(),
                              nulls_of(case["valid"]))
            col = sliced(full, *case["slice"])
        elif k == "fsb_sliced":
            w = case["width"]
            vals = np.frombuffer(bytes.fromhex(case["data"]), dtype=np.uint8).reshape(-1, w)
            off, n = case["slice"]
            full_nulls = nulls_of(case["valid"])
            col = FixedSizeBinaryColumn(vals[off:off + n], full_nulls.slice(off, n))
        elif k == "length_sliced":
            off, n = case["slice"]
            col = sliced(column(typ, decode(case["input"])), off, n)
        elif k == "view_matches":
            col = None
            out.append((typ, utf8, column(typ, decode(case["input"]))))
            out.append((typ + "_view", utf8, ViewColumn.from_values(decode(case["input"]))))
            continue
        else:
            col = column(typ, decode(case["input"]))
        out.append((typ, utf8, col))
    return out


def run_case(be, case, col, utf8):
    fn = case["fn"]
    if fn in ("length", "bit_length"):
        return getattr(be, fn)(col)
    if fn == "substring_by_char":
        return be.substring_by_char(col, case["start"], case["length"])
    return be.substring(col, case["start"], case["length"], is_utf8=utf8)


# continuation bytes 0x80..0xBF at both ends: ¿ (C2 BF), ÿ (C3 BF), U+FFFF (EF BF BF), U+10000 (F0 90 80 80)
UTF8_SCALARS = ["a", "b", "Z", "é", "ß", "Γ", "€", "⊢", "日", "😈", "🎉", " ", "¿", "ÿ", "\uffff", "\U00010000"]


def rand_str(rng, max_chars):
    k = int(rng.integers(0, max_chars + 1))
    return "".join(UTF8_SCALARS[int(x)] for x in rng.integers(0, len(UTF8_SCALARS), k)).encode()


def rand_items(rng, n, max_chars, null_p):
    return [None if (null_p and rng.random() < null_p) else rand_str(rng, max_chars) for _ in range(n)]
