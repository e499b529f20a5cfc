"""Pins the CPU restatement of min / max over byte, view, fixed-size-binary and boolean columns (tests/oracle_aggregate.py):
against the reference's literal test vectors (tests/golden/aggregate_vectors.json), against the reference's fold written
out over Python bytes, and across the array types that hold the same values."""
import numpy as np
import pytest

from acu import MAX, MIN
from aggregate_util import (bool_array, bytes_column, fixed_column, literal_fold, load_aggregate_cases, random_items, run_golden_case,
                            slice_column, view_column)
from oracle_aggregate import AggregateOracle

CASES = load_aggregate_cases()


@pytest.fixture(scope="module")
def orc():
    return AggregateOracle()


@pytest.mark.parametrize("case", CASES, ids=[c["id"] for c in CASES])
def test_oracle_matches_reference_vector(orc, case):
    run_golden_case(orc, case)


def test_golden_covers_every_form():
    forms = {f for c in CASES for f in c.get("forms", [])}
    assert forms == {"binary", "large_binary", "binary_view", "fixed_size_binary", "utf8", "large_utf8", "utf8_view"}
    assert any(c["kind"] == "boolean" for c in CASES) and any("slice" in c for c in CASES)


@pytest.mark.parametrize("seed", range(12))
@pytest.mark.parametrize("op", [MIN, MAX])
def test_oracle_matches_literal_fold(orc, seed, op):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(0, 300))
    items = random_items(rng, n, [0.0, 0.2, 1.0][seed % 3], distinct=[None, 5][seed % 2])
    want = literal_fold(op, items)
    n_valid = sum(x is not None for x in items)
    assert orc.min_max_row(op, bytes_column(items, large=seed % 2 == 1, bit_offset=seed % 8)) == (want, n_valid)
    assert orc.min_max_row(op, view_column(items, bit_offset=seed % 5)) == (want, n_valid)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("op", [MIN, MAX])
def test_view_and_byte_array_forms_agree(orc, seed, op):
    rng = np.random.default_rng(100 + seed)
    items = random_items(rng, 500, 0.1, alphabet=b"xy", max_len=30)
    # a shared 16-byte prefix: views hold it out of line, every key ties
    items = [None if x is None else b"P" * 16 + x for x in items]
    off = int(rng.integers(0, 40))
    cols = [bytes_column(items), bytes_column(items, large=True), view_column(items, block_size=100)]
    rows = {orc.min_max_row(op, slice_column(c, off, 400)) for c in cols}
    assert len(rows) == 1
    assert rows.pop()[0] == literal_fold(op, items[off: off + 400])


@pytest.mark.parametrize("width", [0, 1, 3, 8, 16, 33])
def test_fixed_size_binary_matches_literal_fold(orc, width):
    rng = np.random.default_rng(width)
    items = [None if rng.random() < 0.2 else rng.choice([0, 1, 255], width).astype(np.uint8).tobytes() for _ in range(200)]
    col = fixed_column(items, width, bit_offset=3, garbage=b"\0" * width)
    for op in (MIN, MAX):
        assert orc.min_max_row(op, col) == (literal_fold(op, items), sum(x is not None for x in items))


def test_nulls_are_never_read(orc):
    # bytes under null slots that would win if they were read: an empty value / 0x00 (min), 0xff... (max)
    items = [b"m", None, b"k", None, b"z", b"k"]
    for garbage, op, want in ((b"\0\0", MIN, 2), (b"\xff" * 20, MAX, 4)):
        assert orc.min_max_row(op, bytes_column(items, garbage=garbage)) == (want, 4)
    gview = np.zeros(16, np.uint8)
    gview[0] = 1  # an inline one-byte value 0x00
    assert orc.min_max_row(MIN, view_column(items, garbage_views=[gview])) == (2, 4)


def test_prefix_pairs_and_extreme_bytes(orc):
    items = [b"a\0", b"a", b"", b"\xff", b"\0", b"a"]
    assert orc.min_max_row(MIN, bytes_column(items)) == (2, 6)
    assert orc.min_max_row(MAX, bytes_column(items)) == (3, 6)
    assert orc.min_max_row(MIN, bytes_column(items[:2])) == (1, 2)  # "a" < "a\0"


@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 127, 128, 129])
@pytest.mark.parametrize("offsets", [(0, 0), (3, 5), (17, 63)])
def test_boolean_matches_literal_fold(orc, n, offsets):
    rng = np.random.default_rng(n)
    for p_true in (0.0, 0.5, 1.0):
        items = [None if rng.random() < 0.3 else bool(rng.random() < p_true) for _ in range(n)]
        a = bool_array(items, *offsets)
        valid = [x for x in items if x is not None]
        assert orc.min_boolean(a) == (min(valid) if valid else None)
        assert orc.max_boolean(a) == (max(valid) if valid else None)
