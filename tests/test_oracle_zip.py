"""tests/oracle_zip.py against the reference's byte and view zip tests and the hand-derived Boolean and FixedSizeBinary
cases (tests/golden/zip_vectors.json), plus the oracle's own rules that those cases do not reach, on the CPU. The device
tests run the same cases."""
import numpy as np
import pytest

from acu import _abi as abi

import oracle_zip as oz
import zip_util as zu
from oracle_filter_take import EXTEND_OVERFLOW, OracleError

CASES = zu.golden_cases()


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_oracle_matches_golden(case):
    m, t, f = zu.golden_mask(case), zu.golden_side(case, "truthy"), zu.golden_side(case, "falsy")
    r = oz.zip(m, t, f)
    col = zu.oracle_as_column(r, t, f)
    exp = case["expect"]
    assert zu.logical_rows(col) == [None if v is None else bytes.fromhex(v) for v in exp["values"]]
    assert (r.valid is not None) == exp["nulls"]
    if "raw" in exp:
        assert zu.raw_rows(col) == [bytes.fromhex(v) for v in exp["raw"]]


def test_golden_file_is_current():
    import runpy
    import os
    mod = runpy.run_path(os.path.join(os.path.dirname(zu.GOLDEN), "make_golden_zip.py"), run_name="golden")
    assert mod["cases"] == CASES


def test_fallback_differs_from_primitive_scalar_policy():
    """Two FixedSizeBinary scalars with a null falsy over a mixed mask: the unselected row holds the null scalar's bytes
    (PrimitiveScalarImpl would repeat the valid value), and an all-true mask leaves no NullBuffer."""
    t, f = zu.fsb_column([b"abc"], 3, scalar=True), zu.fsb_column([None], 3, raw=[b"xyz"], scalar=True)
    r = oz.zip(zu.mask_array([True, False]), t, f)
    assert [bytes(x) for x in r.values] == [b"abc", b"xyz"] and list(r.valid) == [True, False]
    assert oz.zip(zu.mask_array([True, True]), t, f).valid is None


def test_array_view_rebase_includes_nulls_and_wraps():
    t = zu.view_column([b"x" * 20, b"y" * 20], block_size=20)
    f = zu.view_column([b"z" * 30, None], block_size=64)
    fv = f.views.copy().view(np.uint32).reshape(-1, 4)
    fv[1] = [40, 0, 0xFFFFFFFF, 0]  # a long view under a null, buffer index at the u32 edge
    f.views = fv.view(np.uint8).reshape(-1, 16)
    r = oz.zip(zu.mask_array([False, False]), t, f)
    out = r.views.view(np.uint32).reshape(-1, 4)
    assert out[0, 2] == 2 and out[1, 2] == 1  # + len(t.buffers) == 2, wrapping
    assert r.buffers == abi.ZIP_BUFFERS_BOTH


def test_scalar_views_inline_falsy_rebased_when_it_has_buffers():
    """zip.rs:759-769: a mixed mask over two valid view scalars raises the falsy view's buffer index by truthy's buffer
    count whenever falsy has buffers, even when the falsy view is inline (the raised word is inline data)."""
    t = zu.view_column([b"a" * 20], scalar=True)
    f = zu.view_column([b"short"], scalar=True)
    f.buffers = [np.zeros(8, np.uint8)]
    r = oz.zip(zu.mask_array([True, False]), t, f)
    inline_word = int(f.views.view(np.uint32)[0, 2])
    assert r.views.view(np.uint32).reshape(-1, 4)[1, 2] == inline_word + len(t.buffers)
    assert r.buffers == abi.ZIP_BUFFERS_BOTH


MIB = b"q" * (1 << 20)
N_OVF = 2049  # 2048 rows of 1 MiB end at 2^31 > i32::MAX: row 2047 is the first past it


@pytest.mark.parametrize("fs_valid,mask,err", [
    (None, [True] * N_OVF, (abi.ERR_INVALID_ARGUMENT, EXTEND_OVERFLOW, N_OVF - 2)),
    (True, [i % 2 == 0 for i in range(2 * N_OVF)], (abi.ERR_PANIC_OUT_OF_BOUNDS, "overflow", -1)),
    (True, [True] * N_OVF, (abi.ERR_PANIC_OUT_OF_BOUNDS, "offset overflow", -1)),
    (False, [True] * N_OVF, (abi.ERR_PANIC_OUT_OF_BOUNDS, "offset overflow", -1)),
])
def test_i32_overflow_branches(fs_valid, mask, err):
    """A 1 MiB scalar repeated past 2^31 bytes: zip_impl's InvalidArgumentError at the first row past i32::MAX, or the
    scalar zipper's panic text of the branch that panics."""
    t = zu.bytes_column([MIB], scalar=True)
    if fs_valid is None:
        f = zu.bytes_column([b""] * len(mask))
    else:
        f = zu.bytes_column([MIB if fs_valid else None], scalar=True)
    with pytest.raises(OracleError) as e:
        oz.zip(zu.mask_array(mask), t, f, data=False)
    assert e.value.status == err[0] and e.value.message.endswith(err[1]) and e.value.index == err[2]


def test_length_and_type_errors():
    m = zu.mask_array([True, False])
    with pytest.raises(OracleError, match="all arrays should have the same length"):
        oz.zip(m, zu.bytes_column([b"a"]), zu.bytes_column([b"a", b"b"]))
    with pytest.raises(OracleError, match="arguments need to have the same data type"):
        oz.zip(m, zu.bytes_column([b"a", b"b"]), zu.bytes_column([b"a", b"b"], ob=8))
    with pytest.raises(OracleError, match="arguments need to have the same data type"):
        oz.zip(m, zu.fsb_column([b"ab", b"cd"], 2), zu.fsb_column([b"abc", b"def"], 3))
