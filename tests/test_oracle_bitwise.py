"""The bitwise / product / bit-aggregate oracle (tests/oracle_bitwise.py) pinned to the reference's own test cases
(tests/golden/bitwise_vectors.json) and to boundary cases restated from the reference's definitions."""
import json
import os

import numpy as np
import pytest

import oracle_bitwise as ob

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bitwise_vectors.json")))


def slots(items):
    """logical values (None = null) -> (every slot with 0 under nulls, mask or None)"""
    mask = [x is not None for x in items]
    return [0 if x is None else x for x in items], (None if all(mask) else mask)


def logical(vals, mask):
    return [v if mask is None or m else None for v, m in zip(vals, mask if mask is not None else vals)]


@pytest.mark.parametrize("case", GOLDEN["bitwise"], ids=lambda c: c["src"])
def test_bitwise_golden(case):
    left, lmask = slots(case["left"])
    if case["right"] is not None:
        right, rmask = slots(case["right"])
        vals, mask = ob.array_op(case["fn"], case["dtype"], left, lmask, right, rmask)
    else:
        vals, mask = ob.array_op(case["fn"], case["dtype"], left, lmask, scalar=case["scalar"])
    assert logical(vals, mask) == case["expected"]


@pytest.mark.parametrize("case", GOLDEN["aggregate"], ids=lambda c: c["src"])
def test_aggregate_golden(case):
    vals, mask = slots(case["values"])
    if case["fn"] == "product_checked":
        if case["error"]:
            with pytest.raises(ob.ProductOverflow):
                ob.product_checked(case["dtype"], vals, mask)
        else:
            assert ob.product_checked(case["dtype"], vals, mask) == case["expected"]
    elif case["dtype"].startswith("float"):
        got = None if not ob.valid_values(vals, mask) else float(np.prod(ob.valid_values(vals, mask)))
        assert got == case["expected"]
    else:
        assert ob.aggregate(case["fn"], case["dtype"], vals, mask) == case["expected"]


@pytest.mark.parametrize("dtype", ob.DTYPES)
def test_shift_amounts_over_the_full_range_of_b(dtype):
    """The amount is b's two's-complement pattern modulo the width, for signed and unsigned b: numpy's shift of the
    unsigned view by (b & (w - 1)) is the independent restatement."""
    w = ob.bits_of(dtype)
    info = np.iinfo(dtype)
    u = np.dtype(f"uint{w}")
    bs = sorted(b for b in {info.min, info.min + 1, -w - 1, -w, -1, 0, 1, w - 1, w, w + 1, 2 * w - 1, info.max - 1, info.max}
                if info.min <= b <= info.max)
    for a in (info.min, -1 if info.min else 1, 1, 0x5A & info.max, info.max):
        for b in bs:
            amt = int(np.array(b, dtype=dtype).view(u)) & (w - 1)
            au = np.array(a, dtype=dtype).view(u)
            shl = int(np.array(au << u.type(amt), dtype=u).view(dtype))
            shr = int((np.array(a, dtype=dtype) >> np.dtype(dtype).type(amt)))
            assert ob.row("shift_left", dtype, a, b) == shl, (a, b)
            assert ob.row("shift_right", dtype, a, b) == shr, (a, b)
    assert ob.row("shift_left", "uint64", 8, 2**64 - 1) == 0  # bitwise.rs:230: shifts by 63


def test_product_checked_exact_boundaries():
    mn = -(2**63)
    assert ob.product_checked("int64", [-(2**62), 2]) == mn
    assert ob.product_checked("int64", [-(2**62), 2, 1, 1]) == mn
    with pytest.raises(ob.ProductOverflow) as e:
        ob.product_checked("int64", [-(2**62), 2, 1, -1])
    assert (e.value.message, e.value.row) == (f"Overflow happened on: {mn} * -1", 3)
    with pytest.raises(ob.ProductOverflow) as e:
        ob.product_checked("int64", [2**62, 2])
    assert e.value.row == 1
    assert ob.product_checked("int8", [-128, 1, 1]) == -128
    assert ob.product_checked("int8", [0, 127, 127]) == 0          # a zero before the would-be overflow
    with pytest.raises(ob.ProductOverflow) as e:
        ob.product_checked("int8", [16, 16, 0])                    # ... and after it
    assert (e.value.message, e.value.row) == ("Overflow happened on: 16 * 16", 1)
    assert ob.product_checked("uint8", [15, 17]) == 255
    with pytest.raises(ob.ProductOverflow):
        ob.product_checked("uint8", [16, 16])
    assert ob.product_checked("int8", [100, 100], [False, True]) == 100  # the overflowing value under a null


@pytest.mark.parametrize("fn", ["product", "bit_and", "bit_or", "bit_xor"])
def test_none_for_empty_or_all_null(fn):
    assert ob.aggregate(fn, "int32", [], None) is None
    assert ob.aggregate(fn, "int32", [1, 2], [False, False]) is None
    assert ob.product_checked("int32", [], None) is None
    assert ob.product_checked("int32", [7, 9], [False, False]) is None


def _fold_summary(dtype, xs):
    """The chunk summary of the product_checked kernel (csrc/sumchecked.cu), restated per row."""
    mag, neg, zero, pos_at, neg_at = 1, False, False, False, False
    for x in xs:
        if zero:
            break
        if x == 0:
            zero = True
            continue
        neg ^= x < 0
        if abs(x) > 1:
            mag, pos_at, neg_at = min(mag * abs(x), 2**64), False, False
        pos_at |= not neg
        neg_at |= neg
    return mag, neg, zero, pos_at, neg_at


def test_chunk_summary_decides_the_failing_chunk():
    """The composition rule the product_checked kernel scans with, against the in-order fold on random Int8 / UInt8 chunks
    of values that exercise the exact boundary (zeros, +-1, powers of two, -128, 127)."""
    rng = np.random.default_rng(42)
    for dtype, pool in (("int8", [0, 1, -1, 2, -2, 4, -4, 8, -8, 16, -16, 64, -64, -128, 127, 3, -3]),
                        ("uint8", [0, 1, 2, 3, 4, 16, 15, 17, 255, 128])):
        w = ob.bits_of(dtype)
        limit = (1 << (w - 1)) if ob.signed(dtype) else (1 << w) - 1
        for _ in range(3000):
            chunks = [list(rng.choice(pool, size=rng.integers(0, 4))) for _ in range(rng.integers(1, 5))]
            flat = [int(x) for c in chunks for x in c]
            try:
                ob.product_checked(dtype, flat)
                expect = None
            except ob.ProductOverflow as e:
                expect, acc = e.row, 0
                for k, c in enumerate(chunks):
                    acc += len(c)
                    if e.row < acc:
                        expect = k
                        break
            m, s, z, got = 1, False, False, None
            for k, c in enumerate(chunks):
                if z:
                    break
                mag, neg, zero, pos_at, neg_at = _fold_summary(dtype, [int(x) for x in c])
                p = min(m * mag, 2**64)
                if p > limit or (ob.signed(dtype) and p == limit and (neg_at if s else pos_at)):
                    got = k
                    break
                m, s, z = p, s ^ neg, zero
            assert got == expect, (dtype, chunks)


@pytest.mark.parametrize("dtype", ob.DTYPES)
def test_vectorised_oracle_matches_rows(dtype):
    info = np.iinfo(dtype)
    rng = np.random.default_rng(7)
    a = rng.integers(info.min, info.max, 300, dtype=dtype, endpoint=True)
    b = rng.integers(info.min, info.max, 300, dtype=dtype, endpoint=True)
    a[:4] = [info.min, info.max, 0, 1]
    b[:4] = [info.max, info.min, ob.bits_of(dtype), ob.bits_of(dtype) - 1]
    for op in ob.OPS:
        got = ob.np_op(op, dtype, a, b)
        assert got.dtype == np.dtype(dtype)
        assert [int(x) for x in got] == [ob.row(op, dtype, int(x), int(y)) for x, y in zip(a, b)], op
        if op != "not":
            s = np.array(b[1], dtype=dtype)[()]
            assert [int(x) for x in ob.np_op(op, dtype, a, s)] == [ob.row(op, dtype, int(x), int(s)) for x in a], op
