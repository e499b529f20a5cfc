"""Columns for the concat_elements tests: the golden cases of tests/golden/concat_elements_vectors.json expanded into the
array types they name."""
import json
import os

from acu import ViewColumn

from substring_util import OFFSET_DTYPE, bytes_col, decode, fsb_col, sliced

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "concat_elements_vectors.json")


def golden_cases():
    with open(GOLDEN) as f:
        return json.load(f)["cases"]


def column(typ, items, width=None):
    if typ in OFFSET_DTYPE:
        return bytes_col(items, OFFSET_DTYPE[typ])
    if typ in ("utf8_view", "binary_view"):
        return ViewColumn.from_values(items)
    return fsb_col(items, width)


def is_utf8(typ):
    return typ in ("utf8", "large_utf8", "utf8_view")


def run_case(backend, case):
    """The case's call on `backend` (acu.Context or the oracle)."""
    if case["fn"] == "many":
        return backend.concat_elements_utf8_many([column("utf8", decode(a)) for a in case["arrays"]])
    widths = case.get("widths", [None, None])
    cols = [column(t, decode(case[side]), w) for t, side, w in zip(case["types"], ("left", "right"), widths)]
    if "slices" in case:
        cols = [sliced(c, off, n) for c, (off, n) in zip(cols, case["slices"])]
    return backend.concat_elements(cols[0], cols[1], is_utf8=is_utf8(case["types"][0]))
