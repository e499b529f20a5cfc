"""The RunEndEncoded kernels of csrc/run_end.cu where their code paths switch, past one grid-stride round and past 2^32
logical rows, against a vectorised numpy restatement of filter_run_end_array (filter.rs:628-677) and take_run
(take.rs:948-995), itself checked against tests/oracle_filter_take.py on small cases:

  k_ree_take_map    one thread per index, grid-stride: the largest index (warp butterfly, then atomicMax from each
                    warp's lane 0) with a single out-of-bounds value at every lane 0-31 of an even and an odd warp, in
                    block 1, in the last partial warp and in the second grid round, also under a null index; several
                    out-of-bounds values spread over blocks and rounds; UInt64 values >= 2^63 and Int64 -1. The 64-bit
                    `x + offset`: Int64 run ends up to 2^40 and 2^62 at slice offsets >= 2^32 with UInt8 / UInt16 /
                    UInt32 / UInt64 indices, Int8 / Int16 / Int32 -1 as row 2^32 - 1 of a longer column, Int32 run ends
                    ending at INT32_MAX.
  k_ree_run_ends    one bit per output position q in [0, M], ballot words of 32: M = 1 ... 1025 and one grid round of
                    bits - 1 / + 0 / + 1, with merges and breaks placed at q = 32k - 1 / 32k / 32k + 1. The comparator
                    (NullsThen<...>): values differing only where a narrower compare misses them (the high byte of
                    16-bit values, the top byte of 32-bit ones, the high word of 64-bit ones, the high half of
                    Decimal128), equal-length bytes differing at byte 0 / 7 / 8 / 15 / 16 / 31 / 32 or at the last byte
                    of 64 / 65 / 1000-byte values, equal bytes at different data alignments, views inline / prefix /
                    out-of-line / split over buffers / without buffers, Boolean at bit offsets 0 / 3 / 7, and every kind
                    with a sliced values child (validity offset 3). Int16 run ends at M = 32767 (k_ree_narrow16).
  k_ree_bounds,     one thread per physical run, a warp ranks 32 runs and lane 0 ranks its predecessor itself:
  k_ree_filter_runs clipped ends at x = 0 / 1 / 63 (mod 64) and 1023 / 1024 / 1025 (mod 1024) with a run's only selected
  and plan_rank     row on either side, predicate lengths 64k and 1024k - 1 / 1024k / 1024k + 1 (x == plen reads the
                    padded tile offset), runs longer than a tile, runs 31 / 32 / 33 / 32k whose keep rests on lane 0's
                    predecessor (also clipped to a short predicate), one round of runs - 1 / + 0 / + 1 and 2.5 rounds,
                    slices at offsets >= 2^32, Int16 run ends with a 32767-row predicate, and a predicate of more than
                    2^32 rows whose ranks pass 2^32.
  host strategy     All with a predicate shorter than the column, a zero-length predicate, a Slices predicate, a values
                    plan that keeps every run, and a plan from acu_filter_plan_create_cmp driven through ctypes.

The Python descriptor of a RunEndEncoded column allocates nothing in proportion to its logical length, so columns of
2^62 rows cost a few bytes; the values child of every case stays small. Every test asserts that its rows sit where it says
they do."""
import ctypes as C
import os
import re
import zlib

import numpy as np
import pytest

import acu
from acu import BOOL, DecimalArray, HostArray, ListColumn, RunEndColumn, Utf8Column, ViewColumn
from acu import _abi as abi

import oracle_filter_take as oft
from oracle_filter_take import OracleError, nulls_of
from test_gpu_list_boundaries import SIGNED, ref_strategy, to_index
from test_gpu_run_end import RE_PER_SM, RE_THREADS, values_of

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "arrow-rs_b200", "csrc")

TILE_ROWS = 1024       # compact.cu: a filter plan tile, plan_rank's tile_off[x >> 10]
TILE_WORDS = TILE_ROWS // 64
INDEX_DTYPES = [abi.I8, abi.U8, abi.I16, abi.U16, abi.I32, abi.U32, abi.I64, abi.U64]
R_TYPES = [np.int16, np.int32, np.int64]
NAMES = {abi.I8: "i8", abi.U8: "u8", abi.I16: "i16", abi.U16: "u16", abi.I32: "i32", abi.U32: "u32", abi.I64: "i64", abi.U64: "u64"}
SMALL = 4096           # values children up to this many rows are built by the oracle, larger ones by a numpy gather


# ---- 1. the vectorised reference ------------------------------------------------------------------------------------
def physical_range(ends, offset, length):
    """get_start_physical_index / get_end_physical_index (run.rs:243-267)."""
    e64 = np.asarray(ends).astype(np.int64)
    if length == 0:
        return 0, 0
    s = 0 if offset == 0 else int(np.searchsorted(e64, offset, "right"))
    e = len(e64) - 1 if int(e64[-1]) == offset + length else int(np.searchsorted(e64, offset + length - 1, "right"))
    return s, e


def ref_filter_runs(ends, offset, length, plen, count, rank):
    """filter_run_end_array over the run ends. rank(x) = selected predicate rows in [0, x) for an int64 array x. Returns
    ("none" | "all", None, None) or ("runs", new ends, kept physical rows); raises the length error."""
    if plen > length:
        raise OracleError(abi.ERR_INVALID_ARGUMENT, f"Filter predicate of length {plen} is larger than target array of length {length}")
    if count == 0:
        return "none", None, None
    if count == plen:
        return "all", None, None
    s, e = physical_range(ends, offset, length)
    clipped = np.clip(np.asarray(ends[s:e + 1]).astype(np.int64) - offset, 0, plen)  # saturating_sub, then min(p)
    rk = np.asarray(rank(clipped), np.int64)
    keep = np.diff(np.concatenate([[0], rk])) > 0
    return "runs", rk[keep].astype(np.asarray(ends).dtype), s + np.flatnonzero(keep)


def mask_rank(mask):
    cum = np.concatenate([[0], np.cumsum(np.asarray(mask, bool), dtype=np.int64)])
    return lambda x: cum[x]


def plain(v):
    return type(v) is HostArray and v.dtype != BOOL


def gather(v, rows, keep_nulls=False):
    """A primitive child gathered at `rows`, with a NullBuffer iff a gathered row is null (or keep_nulls and v has one)."""
    rows = np.asarray(rows, np.int64)
    vm = v.valid_mask()[rows]
    present = v.validity is not None if keep_nulls else not vm.all()
    return HostArray(v.dtype, np.asarray(v.values[:v.length])[rows], len(rows), acu.pack_bits(vm) if present else None, 0, 0,
                     int((~vm).sum()) if present else 0)


def ref_filter(col, mask):
    """filter(col, predicate) with mask = oracle_filter_take.filter_mask(predicate), as a RunEndColumn."""
    mask = np.asarray(mask, bool)
    how, ends, rows = ref_filter_runs(col.run_ends, col.offset, col.length, len(mask), int(mask.sum()), mask_rank(mask))
    if how == "none":
        return oft.empty_run_end(col)
    if how == "all":
        return col.slice(0, len(mask))
    s, e = physical_range(col.run_ends, col.offset, col.length)
    if e - s + 1 <= SMALL or not plain(col.values):
        keep = np.zeros(e - s + 1, bool)
        keep[rows - s] = True
        values = oft.filter(acu.slice_column(col.values, s, e - s + 1), keep)
    else:
        values = gather(col.values, rows, keep_nulls=len(rows) == e - s + 1)
    return RunEndColumn(ends, values, 0, int(ends[-1]))


def keys_of(v):
    """make_comparator classes of the physical values: equal keys iff is_eq (nulls one class, -1); None for nested."""
    if isinstance(v, (ListColumn, acu.FixedSizeListColumn, RunEndColumn)):
        return None
    vm = oft.valid_mask(v)
    if isinstance(v, (Utf8Column, ViewColumn)):
        items = [acu.column_value(v, i) if vm[i] else b"" for i in range(v.length)]  # views under nulls may be garbage
        ids = {}
        key = np.array([ids.setdefault(bytes(x), len(ids)) for x in items], np.int64)
    elif v.dtype == BOOL:
        key = v.value_array().astype(np.int64)
    elif isinstance(v, DecimalArray) and v.byte_width == 16:
        key = np.unique(np.asarray(v.values[:v.length]).reshape(-1, 2), axis=0, return_inverse=True)[1].reshape(-1)
    else:  # integers, decimals and floats under total_cmp: the bits
        key = np.unique(np.asarray(v.values[:v.length]).view(np.dtype(f"u{v.width()}")), return_inverse=True)[1].reshape(-1)
    return np.where(vm, np.asarray(key, np.int64), -1)


def ref_bounds(n, vals, valid, dtype):
    """take's check_bounds (take.rs:167-209): skipped where the length exceeds the index type; the first bad row."""
    if n > oft.INDEX_MAX[dtype]:
        return
    allv = valid is None or bool(np.all(valid))
    raw = np.asarray(vals).astype(np.int64 if dtype in SIGNED else np.uint64)
    bad = (raw >= n) | ((raw < 0) & allv) if dtype in SIGNED else raw >= np.uint64(n)
    if not allv:
        bad &= np.asarray(valid, bool)
    if bad.any():
        j = int(np.flatnonzero(bad)[0])
        raise OracleError(abi.ERR_COMPUTE, f"Array index out of bounds, cannot get item at index {int(vals[j])} from {n} entries", j)


def ref_take_runs(ends, offset, length, vals, valid, dtype, check_bounds, key):
    """take_run over the run ends: (new ends, value rows), (None, None) for empty indices; raises the reference's errors in
    its order (check_bounds, the largest logical index with null slots included, nested values, the run-end unwrap)."""
    if check_bounds:
        ref_bounds(length, vals, valid, dtype)
    m = len(vals)
    if m == 0:
        return None, None
    ix = to_index(vals, dtype)
    mx = int(ix.max())
    if mx >= length:
        raise OracleError(abi.ERR_INVALID_ARGUMENT, f"Logical index {mx} is out of bounds for RunArray of length {length}")
    phys = np.searchsorted(np.asarray(ends).astype(np.int64), ix.astype(np.int64) + offset, "right")
    if key is None:
        raise OracleError(abi.ERR_NOT_YET_IMPLEMENTED, "Not yet implemented: " + oft.NESTED_TEXT)
    if m > oft.R_MAX[np.asarray(ends).itemsize]:
        raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, oft.UNWRAP_NONE)
    k = key[phys]
    new = np.append(np.flatnonzero((phys[1:] != phys[:-1]) & (k[1:] != k[:-1])) + 1, m)
    return new.astype(np.asarray(ends).dtype), phys[new - 1]


def ref_take(col, idx, check_bounds=False):
    """take(col, indices, check_bounds) for a HostArray of integer indices, as a RunEndColumn."""
    valid = idx.valid_mask() if idx.validity is not None else None
    ends, rows = ref_take_runs(col.run_ends, col.offset, col.length, idx.value_array(), valid, idx.dtype, check_bounds, keys_of(col.values))
    if ends is None:
        return oft.empty_run_end(col)
    wide = idx.dtype in (abi.I64, abi.U64)
    if len(rows) <= SMALL or not plain(col.values):
        values = oft.take(col.values, [int(r) for r in rows], [True] * len(rows), False, abi.U64 if wide else abi.U32)
    else:
        values = gather(col.values, rows)
    return RunEndColumn(ends, values, 0, idx.length)


def assert_same(got, exp, what=""):
    assert got.run_ends.dtype == exp.run_ends.dtype, what
    assert np.array_equal(got.run_ends, exp.run_ends), what
    assert (got.offset, got.length) == (exp.offset, exp.length), what
    g, e = got.values, exp.values
    if plain(g) and plain(e) and e.length > SMALL:
        assert (g.dtype, g.length, g.validity is None) == (e.dtype, e.length, e.validity is None), what
        assert np.array_equal(np.asarray(g.values[:g.length]).view(np.uint8), np.asarray(e.values[:e.length]).view(np.uint8)), what
        assert np.array_equal(g.valid_mask(), e.valid_mask()), what
    else:
        assert oft.describe(g) == oft.describe(e), what


def expect(run_dev, run_ref, what=""):
    """The device result (or error status and message) equals the reference's; returns the reference result."""
    try:
        exp = run_ref()
    except OracleError as e:
        with pytest.raises(acu.ArrowError) as got:
            run_dev()
        assert (got.value.status, got.value.message) == (e.status, e.message), what
        return e
    assert_same(run_dev(), exp, what)
    return exp


def check_filter(gpu, col, pred, what=""):
    return expect(lambda: gpu.filter_run_end(col, pred), lambda: ref_filter(col, oft.filter_mask(pred)), what)


def check_take(gpu, col, idx, check_bounds=False, what=""):
    return expect(lambda: gpu.take_run_end(col, idx, check_bounds), lambda: ref_take(col, idx, check_bounds), what)


def _rand_ree(rng, kind, r_dtype):
    n_phys = int(rng.integers(1, 40))
    col = RunEndColumn(np.cumsum(rng.integers(1, 6, n_phys)).astype(r_dtype), values_of(kind, n_phys, rng, distinct=3))
    off = int(rng.integers(0, col.length)) if rng.random() < 0.6 else 0
    return col.slice(off, int(rng.integers(0, col.length - off + 1)))


def _rand_indices(rng, dtype, n, m):
    info = np.iinfo(acu.NP_DTYPES[dtype])
    vals = rng.integers(0, max(n, 1), m).astype(np.int64)
    pick = rng.random(m)
    vals = np.where(pick < 0.03, n + rng.integers(0, 3, m), vals)
    if dtype in SIGNED:
        vals = np.where((pick >= 0.03) & (pick < 0.05), -1, vals)
    vals = np.clip(vals, int(info.min), int(info.max)).astype(acu.NP_DTYPES[dtype])
    return HostArray.from_numpy(dtype, vals, rng.random(m) >= 0.15 if rng.random() < 0.5 else None)


def test_reference_matches_oracle():
    """The reference against tests/oracle_filter_take.py on 400 small random cases: every run-end type and value kind, slices,
    short and null predicates, all eight index dtypes with nulls, negative and out-of-bounds values, check_bounds."""
    rng = np.random.default_rng(4242)
    kinds = ["i8", "i32", "i64", "f32", "f64", "bool", "dec128", "utf8", "lbin", "view", "list"]
    seen = set()
    for case in range(400):
        kind, r_dtype = kinds[case % len(kinds)], R_TYPES[(case // len(kinds)) % 3]
        col = _rand_ree(rng, kind, r_dtype)
        plen = col.length if rng.random() < 0.5 else int(rng.integers(0, col.length + 2))
        p = float(rng.choice([0.0, 0.05, 0.5, 0.95, 1.0]))
        pred = HostArray.bool_from_numpy(rng.random(plen) < p, rng.random(plen) >= 0.1 if rng.random() < 0.5 else None)
        mask = oft.filter_mask(pred)
        err = _same_as_oracle(lambda: ref_filter(col, mask), lambda: oft.filter(col, mask), case)
        seen.add(("filter error",) if err else ("filter", col.offset > 0, 0 < plen < col.length))
        dtype = INDEX_DTYPES[case % 8]
        idx = _rand_indices(rng, dtype, col.length, int(rng.integers(0, 30)))
        cb = case % 3 == 0
        err = _same_as_oracle(lambda: ref_take(col, idx, cb), lambda: oft.take_host(col, idx, cb), case)
        seen.add(("take error", err.message.split(" ")[0]) if err else ("take", kind))
    for fact in [("filter error",), ("filter", True, True), ("filter", False, False), ("take error", "Compute"),
                 ("take error", "Invalid"), ("take error", "Not")] + [("take", k) for k in kinds[:-1]]:
        assert fact in seen, fact


def _same_as_oracle(run_ref, run_orc, case):
    """The reference's result (or error status and message) equals the oracle's; returns the oracle's error or None."""
    try:
        exp = run_orc()
    except OracleError as e:
        with pytest.raises(OracleError) as g:
            run_ref()
        assert (g.value.status, g.value.message) == (e.status, e.message), case
        return e
    assert oft.describe(run_ref()) == oft.describe(exp), case
    return None


# ---- 5. the constants the placements depend on ------------------------------------------------------------------------
def test_constants_pinned():
    """A retune of any of these moves the boundaries away from the rows placed on them: update the mirrors above (and the
    placements) together with the kernels. RE_THREADS / RE_PER_SM are pinned by test_run_end_launch_constants.py."""
    with open(os.path.join(CSRC, "run_end.cu"), encoding="utf-8") as f:
        src = f.read()
    with open(os.path.join(CSRC, "compact.cu"), encoding="utf-8") as f:
        compact = f.read()
    assert re.search(r"#define TILE_ROWS (\d+)\s", compact).group(1) == str(TILE_ROWS)
    assert "#define TILE_WORDS (TILE_ROWS / 64)" in compact
    assert "int64_t r = (int64_t)__ldg(tile_off + (x >> 10));" in src
    assert "for (int64_t k = (x >> 10) << 4; k < w; ++k)" in src
    assert TILE_ROWS == 1 << 10 and TILE_WORDS == 1 << 4
    # a warp ranks 32 runs / marks 32 output positions per ballot word; lane 0 ranks its predecessor itself
    assert "for (int64_t j0 = warp * 32; j0 < pl; j0 += nwarps * 32)" in src
    assert "if (lane == 0) prev = j0 == 0 ? 0 : clipped_rank(start + j0 - 1);" in src
    assert "for (int64_t q0 = warp * 32; q0 <= m; q0 += nwarps * 32)" in src
    assert "const int bgrid = re_grid(ctx, (m + 1 + 31) / 32 * 32);" in src
    assert "re_grid(ctx, (pl + 31) / 32 * 32)" in src and "const int grid = re_grid(ctx, m);" in src


def sms(gpu):
    return gpu.lib.acu_device_sm_count(gpu.h)


def grid_round(gpu):
    """Threads of one round of every run_end.cu kernel: indices of k_ree_take_map, runs of k_ree_filter_runs, output
    positions of k_ree_run_ends."""
    return sms(gpu) * RE_PER_SM * RE_THREADS


def i64_values(rng, n, null_p=0.1, distinct=None):
    v = rng.integers(-2**62, 2**62, n) if distinct is None else rng.integers(0, distinct, n) * 2**40 - 3
    return HostArray.from_numpy(abi.I64, v, rng.random(n) >= null_p)


# ---- 2. k_ree_take_map --------------------------------------------------------------------------------------------------
def oob_column(rng):
    return RunEndColumn(np.cumsum(rng.integers(1, 9, 700)).astype(np.int32), i64_values(rng, 700))


@pytest.mark.gpu
@pytest.mark.parametrize("null", [False, True], ids=["valid", "null"])
def test_take_one_out_of_bounds_lane(gpu, null):
    """A single out-of-bounds value at every lane of warp 2 (even) and warp 3 (odd), in block 1, in the last partial warp
    and in the second grid round: the butterfly and the per-warp atomicMax must carry it, also under a null index."""
    rng = np.random.default_rng(31 + null)
    col = oob_column(rng)
    R = grid_round(gpu)
    m = R + 300
    assert m % 32 == 300 % 32 and (m - 1) // 32 * 32 > m - 32  # the last warp is partial
    base = rng.integers(0, col.length, m).astype(np.uint32)
    valid = rng.random(m) >= 0.05
    check_take(gpu, col, HostArray.from_numpy(abi.U32, base, valid), what="no out-of-bounds index")
    places = [2 * 32 + lane for lane in range(32)] + [3 * 32 + lane for lane in range(32)] + [256 + 75, m - 1, m - 12, R + 5, R + 200]
    for pos in places:
        vals, vm = base.copy(), valid.copy()
        vals[pos] = col.length + pos
        vm[pos] = not null
        idx = HostArray.from_numpy(abi.U32, vals, vm)
        e = check_take(gpu, col, idx, what=f"position {pos}")
        assert isinstance(e, OracleError) and str(col.length + pos) in e.message, pos


@pytest.mark.gpu
def test_take_largest_of_many_out_of_bounds(gpu):
    """Several out-of-bounds values in different blocks, warps, lanes and rounds (some under null indices): the message
    names the largest, wherever it sits."""
    rng = np.random.default_rng(37)
    col = oob_column(rng)
    R = grid_round(gpu)
    m = int(2.5 * R)
    vals = rng.integers(0, col.length, m).astype(np.uint64)
    valid = rng.random(m) >= 0.1
    spots = [5, 256 + 17, 3 * 32 + 30, R - 1, R, R + 33, 2 * R + 19, m - 1]
    for largest in range(len(spots)):
        v = vals.copy()
        for k, pos in enumerate(spots):
            v[pos] = col.length + (10**6 if k == largest else 1 + k)
        idx = HostArray.from_numpy(abi.U64, v, valid)
        e = check_take(gpu, col, idx, what=f"largest at {spots[largest]}")
        assert f"Logical index {col.length + 10**6} is out" in e.message


@pytest.mark.gpu
@pytest.mark.parametrize("check_bounds", [False, True])
def test_take_wide_out_of_bounds_values(gpu, check_bounds):
    """UInt64 values >= 2^63 and Int64 -1 (= 18446744073709551615 as ToIndices reads it) name the full 64-bit value."""
    rng = np.random.default_rng(41)
    col = oob_column(rng)
    for dtype, bad in ((abi.U64, 2**63), (abi.U64, 2**64 - 1), (abi.U64, 2**63 + 12345), (abi.I64, -1), (abi.I64, -2**63)):
        v = rng.integers(0, col.length, 5000).astype(acu.NP_DTYPES[dtype])
        v[4000 + 17] = np.array(bad).astype(acu.NP_DTYPES[dtype]) if bad >= 0 else bad
        e = check_take(gpu, col, HostArray.from_numpy(dtype, v), check_bounds, what=f"{dtype} {bad}")
        assert isinstance(e, OracleError)
        if not check_bounds:
            assert f"Logical index {bad % 2**64} is out" in e.message


def huge_column(rng, top):
    """Int64 run ends from small ones through 2^32 to `top`: distinct values, but for the runs ending at 2^32 + 70000 and
    2^33 + 5 (merged by take), and two nulls."""
    ends = np.array([3, 2**32 - 2, 2**32 - 1, 2**32, 2**32 + 1, 2**32 + 3, 2**32 + 200, 2**32 + 70000, 2**33 + 5, 2**40,
                     2**40 + 7, top], np.int64)
    ends = np.unique(ends[ends <= top])
    v = np.arange(len(ends)) * 2**33 + 1
    v[8] = v[7]
    mask = np.ones(len(ends), bool)
    mask[[1, 4]] = False
    return RunEndColumn(ends, HostArray.from_numpy(abi.I64, v, mask))


@pytest.mark.gpu
@pytest.mark.parametrize("top", [2**40 + 100, 2**62], ids=["2^40", "2^62"])
@pytest.mark.parametrize("dtype", [abi.U8, abi.U16, abi.U32, abi.U64], ids=NAMES.get)
def test_take_offsets_past_2_32(gpu, top, dtype):
    """Slices at offsets >= 2^32: x + offset is 64-bit also for the narrow index kinds. Indices land on the last and first
    rows of every run in reach of the index type."""
    rng = np.random.default_rng(zlib.crc32(f"offsets {top} {dtype}".encode()))
    col = huge_column(rng, top)
    imax = oft.INDEX_MAX[dtype]
    for off in (2**32, 2**32 + 1, 2**32 + 150, 2**40 + 3):
        if off >= top:
            continue
        s = col.slice(off, top - off)
        rel = np.asarray(col.run_ends, np.int64) - off
        edges = np.concatenate([rel - 1, rel])
        edges = edges[(edges >= 0) & (edges < min(s.length, imax + 1))]
        assert len(edges) >= 2 and off >= 2**32
        ix = np.concatenate([edges, rng.integers(0, min(s.length, imax + 1), 200, dtype=np.uint64).astype(np.int64), edges[::-1]])
        idx = HostArray.from_numpy(dtype, ix.astype(np.uint64).astype(acu.NP_DTYPES[dtype]), rng.random(len(ix)) >= 0.1)
        exp = check_take(gpu, s, idx, what=f"offset {off}")
        # the edges fall in different physical runs: more than one output run
        assert len(exp.run_ends) > 1
        check_take(gpu, s, idx, check_bounds=True, what=f"offset {off} check_bounds")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [abi.I8, abi.I16, abi.I32], ids=NAMES.get)
@pytest.mark.parametrize("check_bounds", [False, True])
def test_take_negative_index_on_a_long_column(gpu, dtype, check_bounds):
    """ToIndices reads Int8 / Int16 / Int32 -1 as 2^32 - 1: a valid row of a column longer than 2^32 (check_bounds is
    skipped there, as the length exceeds the index type), out of bounds on a short one."""
    rng = np.random.default_rng(43)
    long_col = RunEndColumn(np.array([2**32 - 1, 2**32, 2**32 + 9, 2**33], np.int64), HostArray.from_list(abi.I64, [10, 20, 20, None]))
    assert to_index(np.array([-1]), dtype)[0] == 2**32 - 1
    for col in (long_col, long_col.slice(7, 2**33 - 7), RunEndColumn(np.array([100, 200], np.int32), HostArray.from_list(abi.I64, [1, 2]))):
        vals = np.array([0, -1, 5, -1, -1, 0, 1], acu.NP_DTYPES[dtype])
        exp = check_take(gpu, col, HostArray.from_numpy(dtype, vals), check_bounds, what=f"length {col.length}")
        if col.length > 2**32:
            assert not isinstance(exp, OracleError)
            phys = np.searchsorted(col.run_ends, col.offset + 2**32 - 1, "right")
            assert phys == (1 if col.offset == 0 else 2)


@pytest.mark.gpu
def test_take_int32_run_ends_at_int32_max(gpu):
    """An Int32 column ending at exactly INT32_MAX: its last rows, and INT32_MAX itself out of bounds."""
    ends = np.array([5, 2**30, 2**31 - 3, 2**31 - 2, 2**31 - 1], np.int32)
    col = RunEndColumn(ends, HostArray.from_list(abi.I32, [1, 1, 2, None, 2]))
    assert int(col.run_ends[-1]) == 2**31 - 1 == col.length
    ix = [2**31 - 2, 2**31 - 3, 2**31 - 4, 0, 4, 2**30, 2**30 - 1, 2**31 - 2]
    for dtype in (abi.U32, abi.I32, abi.I64):
        check_take(gpu, col, HostArray.from_list(dtype, ix), what=str(dtype))
        check_take(gpu, col, HostArray.from_list(dtype, ix), True)
        check_take(gpu, col, HostArray.from_list(dtype, ix + [2**31 - 1]), what=f"{dtype} INT32_MAX")
    check_take(gpu, col.slice(2**31 - 4, 3), HostArray.from_list(abi.U8, [0, 1, 2, 2, 1]))


# ---- 3. k_ree_run_ends and the comparator -------------------------------------------------------------------------------
def placed_indices(rng, key, m, targets):
    """m random physical rows (one row per run), then at each target q a merge (same key as row q - 1) for even k and a
    break (another key) for odd k of q = 32k +- 1 / 32k. Returns the indices and {q: ends a run}."""
    by_key = {}
    for p, k in enumerate(key):
        by_key.setdefault(int(k), []).append(p)
    ix = rng.integers(0, len(key), m)
    want = {}
    for n, q in enumerate(targets):
        prev = int(key[ix[q - 1]])
        brk = n % 2 == 1
        pool = [p for k, ps in by_key.items() if (k != prev) == brk for p in ps]
        ix[q] = pool[int(rng.integers(0, len(pool)))]
        want[q] = brk
    return ix, want


def boundary_targets(m):
    qs = {q for k in range(1, m // 32 + 2) for q in (32 * k - 1, 32 * k, 32 * k + 1)}
    return sorted(q for q in qs | {m - 1} if 1 <= q < m)


@pytest.mark.gpu
@pytest.mark.parametrize("m", [1, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025, "round-1", "round", "round+1"])
def test_run_end_bits(gpu, m):
    """Output positions q = 32k - 1 / 32k / 32k + 1 of the ballot words end a run or merge as placed, for M + 1 bits
    from 2 to one grid round + 1 (narrow and wide maps)."""
    R = grid_round(gpu)
    m = {"round-1": R - 2, "round": R - 1, "round+1": R}.get(m, m)  # M + 1 bits: R - 1 / R / R + 1
    rng = np.random.default_rng(m)
    n_phys = 64
    vals = HostArray.from_numpy(abi.I32, rng.integers(0, 3, n_phys) << 24, rng.random(n_phys) >= 0.15)
    col = RunEndColumn(np.arange(1, n_phys + 1, dtype=np.int32), vals)
    key = keys_of(vals)
    targets = boundary_targets(m)
    ix, want = placed_indices(rng, key, m, targets)
    for dtype in (abi.U32, abi.U64):
        exp = check_take(gpu, col, HostArray.from_numpy(dtype, ix.astype(acu.NP_DTYPES[dtype])), what=f"m {m}")
        ends = set(int(x) for x in exp.run_ends)
        assert m in ends
        for q, brk in want.items():
            assert (q in ends) == brk, q  # the run end of output row q - 1 is bit q


def fixed_cases():
    """(name, column of physical values): value pairs that differ only where a narrower compare misses them."""
    f32 = lambda *b: np.array(b, np.uint32).view(np.float32)  # noqa: E731
    f64 = lambda *b: np.array(b, np.uint64).view(np.float64)  # noqa: E731
    return {
        "i8": (abi.I8, np.array([1, -127, 0], np.int8)),
        "u8": (abi.U8, np.array([0x01, 0x81, 0xFF], np.uint8)),
        "i16": (abi.I16, np.array([0x0105, 0x7F05, -0x7EFB], np.int16)),
        "u16": (abi.U16, np.array([0x0105, 0xFF05, 0x8005], np.uint16)),
        "i32": (abi.I32, np.array([0x01020304, 0x7F020304, -0x7EFDFCFC], np.int32)),
        "f32": (abi.F32, f32(0x3F800001, 0xBF800001, 0x7F800001)),
        "i64": (abi.I64, np.array([5, 5 + 2**40, 5 - 2**62], np.int64)),
        "f64": (abi.F64, f64(0x3FF0000000000001, 0xBFF0000000000001, 0x7FF0000000000001)),
        "dec32": (4, [7, 7 + 2**24, 7 - 2**28]),
        "dec64": (8, [7, 7 + 2**40, 7 - 2**60]),
        "dec128": (16, [1, 1 + 2**64, -1, 2**64 - 1]),
    }


def fixed_values(name, rng, n):
    dt, choices = fixed_cases()[name]
    pick = rng.integers(0, len(choices), n)
    mask = rng.random(n) >= 0.15
    if name.startswith("dec"):
        return DecimalArray.from_ints(dt, acu.DECIMAL_MAX_PRECISION[dt], 0, [choices[p] if v else None for p, v in zip(pick, mask)])
    return HostArray.from_numpy(dt, np.asarray(choices)[pick], mask)


def bytes_items(rng, case):
    """Equal-length byte strings differing at one byte, equal ones, and a value with its own prefix."""
    if case.startswith("at"):
        d = int(case[2:])
        base = bytes(rng.integers(97, 123, max(d + 9, 40), dtype=np.uint8))
    else:
        ln = int(case[4:])
        base, d = bytes(rng.integers(97, 123, ln, dtype=np.uint8)), ln - 1
    alt = base[:d] + bytes([base[d] ^ 1]) + base[d + 1:]
    return [base, alt, base[:d] if d else b"", base[:d + 1]]


BYTES_CASES = ["at0", "at7", "at8", "at15", "at16", "at31", "at32", "last64", "last65", "last1000"]


def bytes_column(rng, items, n, off_dtype):
    """n physical rows of `items` with one-to-three-byte fillers between them, so that equal values sit at data offsets
    of every alignment mod 8."""
    rows, data, offs = [], bytearray(), [0]
    vals = []
    for i in range(n):
        it = items[int(rng.integers(0, len(items)))]
        if i % 2:
            it = b"xyz"[: 1 + i % 3]
        vals.append(it)
        data += it
        offs.append(len(data))
    mask = rng.random(n) >= 0.15
    col = Utf8Column(np.array(offs, off_dtype), np.frombuffer(bytes(data) + b"\0", np.uint8).copy(), nulls_of(mask))
    starts = {int(offs[i]) % 8 for i in range(n) if vals[i] == items[0]}
    assert len(starts) > 1  # the same value at different alignments
    return col


def take_many(gpu, col, rng, what, n_idx=3000):
    """Random indices over every pair of physical rows, plus every pair (p, p + 2) and (p + 2, p) in turn."""
    n = col.length
    ix = np.concatenate([rng.integers(0, n, n_idx), np.stack([np.arange(n - 2), np.arange(2, n)], 1).reshape(-1),
                         np.stack([np.arange(2, n), np.arange(n - 2)], 1).reshape(-1)])
    idx = HostArray.from_numpy(abi.U32, ix.astype(np.uint32), rng.random(len(ix)) >= 0.05)
    return check_take(gpu, col, idx, what=what)


def as_runs(values, rng, r_dtype=np.int32):
    return RunEndColumn(np.cumsum(rng.integers(1, 4, values.length)).astype(r_dtype), values)


def both_slices(gpu, values, rng, what, filter_too=True):
    """take (and filter) of the run column over `values` and over acu.slice_column(values, 3, n - 3)."""
    for sv in (values, acu.slice_column(values, 3, values.length - 3)):
        col = as_runs(sv, rng)
        exp = take_many(gpu, col, rng, what)
        assert len(exp.run_ends) > 1
        if filter_too:
            check_filter(gpu, col, HostArray.bool_from_numpy(rng.random(col.length) < 0.4), what)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(fixed_cases()))
def test_merge_fixed_width(gpu, name):
    """Neighbouring values that differ only in the high byte / top byte / high word / high 64 bits never merge; equal ones
    in different runs do; over a values child at validity offset 0 and 3."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    vals = fixed_values(name, rng, 160)
    key = keys_of(vals)
    assert len(set(key.tolist()) - {-1}) == len(fixed_cases()[name][1])  # every pair of choices differs
    both_slices(gpu, vals, rng, name)


@pytest.mark.gpu
@pytest.mark.parametrize("off_dtype", [np.int32, np.int64], ids=["utf8", "large"])
@pytest.mark.parametrize("case", BYTES_CASES)
def test_merge_bytes(gpu, case, off_dtype):
    """Utf8 / Binary and LargeUtf8 / LargeBinary values of equal length differing at one byte, equal values at different
    alignments (merged), a value against its own prefix."""
    rng = np.random.default_rng(zlib.crc32(f"{case} {off_dtype.__name__}".encode()))
    items = bytes_items(rng, case)
    assert len(items[0]) == len(items[1]) and items[0] != items[1]
    both_slices(gpu, bytes_column(rng, items, 120, off_dtype), rng, case)


def view_cases(rng):
    long40 = bytes(rng.integers(97, 123, 40, dtype=np.uint8))
    inline12 = b"abcdefghijkl"
    thirteen = b"wxyz" + bytes(rng.integers(97, 123, 9, dtype=np.uint8))
    return {
        "inline at byte 11": [inline12, inline12[:11] + b"m", b"", b"abcd", long40],
        "13 bytes at byte 12": [thirteen, thirteen[:12] + bytes([thirteen[12] ^ 1]), thirteen[:12], long40],
        "40 bytes at the last byte": [long40, long40[:39] + bytes([long40[39] ^ 1]), long40[:4] + b"\0" * 36, b""],
        "long value in two buffers": [long40, b"", long40[:12], thirteen],
    }


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["inline at byte 11", "13 bytes at byte 12", "40 bytes at the last byte", "long value in two buffers",
                                  "no data buffers"])
def test_merge_views(gpu, case):
    """Views: inline values differing at byte 11, out-of-line values sharing length and prefix, one long value stored in
    several buffers (merged), empty values beside data buffers, and an all-inline column without data buffers."""
    rng = np.random.default_rng(zlib.crc32(case.encode()))
    if case == "no data buffers":
        items = [b"abcdefghijkl", b"abcdefghijkm", b"", b"abcd", b"abcd\0"]
    else:
        items = view_cases(rng)[case]
    rows = [items[int(p)] if m else None for p, m in zip(rng.integers(0, len(items), 150), rng.random(150) >= 0.15)]
    vals = ViewColumn.from_values(rows, block_size=48, garbage_under_nulls=[np.arange(16, dtype=np.uint8)])
    if case == "no data buffers":
        assert len(vals.buffers) == 0
    else:
        assert len(vals.buffers) > 1
        if case == "long value in two buffers":
            where = {int(vals.views[i, 8:12].view(np.uint32)[0]) for i in range(150) if rows[i] == items[0]}
            assert len(where) > 1
    both_slices(gpu, vals, rng, case)


@pytest.mark.gpu
@pytest.mark.parametrize("bit_offset", [0, 3, 7])
def test_merge_boolean(gpu, bit_offset):
    rng = np.random.default_rng(bit_offset)
    vals = HostArray.bool_from_numpy(rng.random(150) < 0.5, rng.random(150) >= 0.15, bit_offset=bit_offset, mask_offset=5)
    assert vals.values_offset == bit_offset
    both_slices(gpu, vals, rng, f"bool at {bit_offset}")


@pytest.mark.gpu
def test_int16_run_ends_at_32767_wide(gpu):
    """Int16 run ends with M = 32767 UInt64 indices: the wide map, then the run ends narrowed by k_ree_narrow16."""
    rng = np.random.default_rng(47)
    vals = HostArray.from_numpy(abi.I16, rng.integers(0, 3, 300) << 8, rng.random(300) >= 0.1)
    col = RunEndColumn(np.cumsum(rng.integers(1, 4, 300)).astype(np.int16), vals)
    ix = rng.integers(0, col.length, 32767).astype(np.uint64)
    exp = check_take(gpu, col, HostArray.from_numpy(abi.U64, ix))
    assert int(exp.run_ends[-1]) == 32767 and exp.run_ends.dtype == np.int16 and len(exp.run_ends) > 1000


# ---- 4. k_ree_bounds, k_ree_filter_runs and plan_rank ---------------------------------------------------------------------
def boundary_column(rng, plen, extra=100, offset=0, r_dtype=np.int32):
    """Run ends (relative to `offset`) at x = 0 / 1 / 63 (mod 64) and 1023 / 1024 / 1025 (mod 1024) up to plen + extra;
    a predicate selecting exactly one row of most runs, alternately its first and its last row, none of every fifth."""
    rel = {x for k in range(1, plen // 64 + 2) for x in (64 * k, 64 * k + 1, 64 * k + 63)}
    rel |= {x for k in range(1, plen // 1024 + 2) for x in (1024 * k - 1, 1024 * k, 1024 * k + 1)}
    rel |= {plen, plen - 1, plen + 1, plen + extra}
    rel = np.array(sorted(x for x in rel if 0 < x <= plen + extra), np.int64)
    ends = (rel + offset).astype(r_dtype)
    col = RunEndColumn(ends, i64_values(rng, len(ends))).slice(offset, plen + extra) if offset else RunEndColumn(ends, i64_values(rng, len(ends)))
    mask = np.zeros(plen, bool)
    starts = np.concatenate([[0], rel[:-1]])
    for k, (a, b) in enumerate(zip(starts, rel)):
        if k % 5 != 4 and a < plen:
            mask[min(a if k % 2 else b - 1, plen - 1)] = True
    return col, mask


@pytest.mark.gpu
@pytest.mark.parametrize("plen", [64 * 37, 1024 * 5 - 1, 1024 * 5, 1024 * 5 + 1])
def test_filter_word_and_tile_edges(gpu, plen):
    """Clipped ends on and beside 64-row words and 1024-row tiles, the only selected row of a run on either side of the
    boundary, and predicate lengths 64k / 1024k - 1 / 1024k / 1024k + 1 (a run end at x == plen reads tile_off[plen >> 10])."""
    rng = np.random.default_rng(plen)
    col, mask = boundary_column(rng, plen)
    rel = np.asarray(col.run_ends, np.int64)
    assert {0, 1, 63} <= set((rel % 64).tolist()) and {1023, 0, 1} <= set((rel % 1024).tolist()) and plen in rel
    pred = HostArray.bool_from_numpy(mask, rng.random(plen) >= 0.02)
    check_filter(gpu, col, pred, "one selected row per run")
    check_filter(gpu, col, HostArray.bool_from_numpy(~mask), "all but one row per run")
    check_filter(gpu, col.slice(0, plen), pred, "column ends with the predicate")
    # the slice moves every clipped end by one row: now they sit on 63 / 0 / 62 and 1022 / 1023 / 0
    check_filter(gpu, col.slice(1, plen), HostArray.bool_from_numpy(mask), "offset 1")


@pytest.mark.gpu
def test_filter_runs_longer_than_a_tile(gpu):
    rng = np.random.default_rng(53)
    lens = rng.choice([1, 1023, 1024, 1025, 3000, 5000], 60)
    col = RunEndColumn(np.cumsum(lens).astype(np.int32), i64_values(rng, 60))
    ends = np.asarray(col.run_ends, np.int64)
    mask = np.zeros(col.length, bool)
    for k, e in enumerate(ends):
        if k % 3:
            mask[e - 1 - (k % 7) * 97 % lens[k]] = True
    check_filter(gpu, col, HostArray.bool_from_numpy(mask))
    check_filter(gpu, col.slice(700, col.length - 2000), HostArray.bool_from_numpy(mask[700:col.length - 2500]))


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [0, 5])
def test_filter_lane0_predecessor(gpu, offset):
    """Runs j = 31 / 32 / 33 and every 32k of the physical range: a selected row in run 32k - 1 but none in run 32k (the
    rank of lane 0's own predecessor decides), and runs past a short predicate, clipped to it."""
    rng = np.random.default_rng(59 + offset)
    n = 32 * 40 + 7
    lens = rng.integers(1, 5, n)
    col = RunEndColumn(np.cumsum(lens).astype(np.int32), i64_values(rng, n))
    s = col.slice(offset, col.length - offset)
    start, _ = physical_range(col.run_ends, offset, s.length)
    ends = np.asarray(col.run_ends, np.int64) - offset
    begins = np.maximum(np.concatenate([[0], ends[:-1]]), 0)
    mask = np.zeros(s.length, bool)
    for j in range(n - start):
        p = start + j
        lane = j % 32
        if (j % 64 == 32) if lane == 0 else (lane in (1, 31) or rng.random() < 0.3):
            mask[begins[p]:ends[p]][-1] = True
    for plen in (s.length, int(ends[start + 32 * 20]) - 1, int(ends[start + 32 * 20 + 1])):
        pred = HostArray.bool_from_numpy(mask[:plen])
        exp = check_filter(gpu, s, pred, f"plen {plen}")
        how, _, rows = ref_filter_runs(s.run_ends, s.offset, s.length, plen, int(mask[:plen].sum()), mask_rank(mask[:plen]))
        j_kept = set((rows - start).tolist())
        for k in range(1, 20):
            assert (32 * k - 1) in j_kept and (32 * k in j_kept) == (k % 2 == 1) and (32 * k + 1) in j_kept, k
        assert exp.length == int(mask[:plen].sum())


@pytest.mark.gpu
@pytest.mark.parametrize("runs", ["round-1", "round", "round+1", "2.5 rounds"])
def test_filter_run_rounds(gpu, runs):
    """Physical ranges of one grid round of runs - 1 / + 0 / + 1 and 2.5 rounds; runs round - 1 / round / round + 1 kept,
    dropped, kept (and the opposite), so the second round's lane 0 ranks its predecessor across the round."""
    R = grid_round(gpu)
    n = {"round-1": R - 1, "round": R, "round+1": R + 1, "2.5 rounds": int(2.5 * R)}[runs]
    rng = np.random.default_rng(n)
    lens = rng.integers(1, 4, n)
    col = RunEndColumn(np.cumsum(lens).astype(np.int32), i64_values(rng, n))
    ends = np.asarray(col.run_ends, np.int64)
    begins = np.concatenate([[0], ends[:-1]])
    for pattern in ((True, False, True), (False, True, False)):
        mask = rng.random(col.length) < 0.3
        for p, keep in zip((R - 1, R, R + 1, 2 * R - 1, 2 * R, 2 * R + 1), pattern * 2):
            if p < n:
                mask[begins[p]:ends[p]] = False
                mask[begins[p] + (p % 2) * (lens[p] - 1)] = keep
        _, _, rows = ref_filter_runs(col.run_ends, 0, col.length, col.length, int(mask.sum()), mask_rank(mask))
        for p, keep in zip((R - 1, R, R + 1), pattern):
            if p < n:
                assert (p in set(rows.tolist())) == keep
        check_filter(gpu, col, HostArray.bool_from_numpy(mask), str(pattern))
    check_filter(gpu, col.slice(1, col.length - 3), HostArray.bool_from_numpy(rng.random(col.length - 1000) < 0.5), "slice")


@pytest.mark.gpu
@pytest.mark.parametrize("offset", [2**32, 2**32 + 1, 2**32 + 1000, 2**40 + 7])
def test_filter_offsets_past_2_32(gpu, offset):
    """Int64 run ends at a slice offset >= 2^32; the runs of the slice end at word / tile edges, and its last run ends
    2^33 rows past the offset (clipped to the predicate)."""
    rng = np.random.default_rng(offset % 1000)
    plen = 1024 * 3 + 1
    col, mask = boundary_column(rng, plen, extra=100, offset=offset, r_dtype=np.int64)
    ends = np.append(np.asarray(col.run_ends), offset + 2**33 + 7)
    col = RunEndColumn(np.concatenate([[offset - 2**31], ends]), i64_values(rng, len(ends) + 1)).slice(offset, 2**33 + 7)
    assert int(col.run_ends[-1]) - col.offset > 2**32
    check_filter(gpu, col, HostArray.bool_from_numpy(mask), "short predicate")
    full = np.concatenate([mask, rng.random(2000) < 0.5])
    check_filter(gpu, col, HostArray.bool_from_numpy(full), "predicate into the last run")


@pytest.mark.gpu
def test_filter_int16_predicate_32767(gpu):
    rng = np.random.default_rng(61)
    col, mask = boundary_column(rng, 32767, extra=0, r_dtype=np.int16)
    assert int(col.run_ends[-1]) == 32767 == col.length
    check_filter(gpu, col, HostArray.bool_from_numpy(mask, rng.random(32767) >= 0.05))
    check_filter(gpu, col.slice(100, 32667), HostArray.bool_from_numpy(mask[100:]))


@pytest.mark.gpu
def test_filter_predicate_past_2_32(gpu):
    """A predicate of 2^32 + 4096 rows selecting every row but six, so that the kept runs' ranks pass 2^32. The packed
    predicate and the plan's mask are 0.5 GB each: about 0.55 GB of host memory and 1.1 GB of device memory."""
    plen = 2**32 + 4096
    zeros = np.array([5, 2**32 - 1, 2**32, 2**32 + 1, 2**32 + 1500, plen - 1], np.int64)
    packed = np.full(acu.bitmap_bytes(plen) + 8, 0xFF, np.uint8)
    packed[plen // 8 + 1:] = 0
    packed[plen // 8] = (1 << (plen % 8)) - 1
    for z in zeros:
        packed[z // 8] &= ~np.uint8(1 << (z % 8))
    pred = HostArray(BOOL, packed, plen, None, 0, 0, 0)
    ends = np.array([1000, 2**31, 2**32 - 1, 2**32, 2**32 + 1, 2**32 + 2, 2**32 + 64, 2**32 + 1024, 2**32 + 1025, plen - 1,
                     plen, plen + 50], np.int64)
    col = RunEndColumn(ends, HostArray.from_numpy(abi.I64, np.arange(len(ends)) * 11))
    rank = lambda x: x - np.searchsorted(zeros, x, "left")  # noqa: E731  selected rows below x, in closed form
    how, new, rows = ref_filter_runs(ends, 0, col.length, plen, plen - len(zeros), rank)
    assert how == "runs" and int(new[-1]) == plen - len(zeros) > 2**32
    assert rows.tolist() == [0, 1, 2, 6, 7, 8, 9]  # the runs of rows 2^32 - 1, 2^32, 2^32 + 1 and [plen - 1, plen + 50) drop
    exp = RunEndColumn(new, gather(col.values, rows, keep_nulls=False), 0, int(new[-1]))
    got = gpu.filter_run_end(col, pred)
    assert_same(got, exp)
    assert [int(x) for x in got.run_ends] == [999, 2**31 - 1, 2**32 - 2, 2**32 + 60, 2**32 + 1020, 2**32 + 1021, plen - 6]


# ---- the host strategy branches and the comparison plan ---------------------------------------------------------------------
@pytest.mark.gpu
def test_filter_strategies(gpu):
    """All with a predicate shorter than the column (a slice of its first rows), a zero-length predicate on a non-empty
    column, a Slices predicate, and a values plan that keeps every run."""
    rng = np.random.default_rng(67)
    col = RunEndColumn(np.cumsum(rng.integers(1, 6, 400)).astype(np.int32), i64_values(rng, 400)).slice(9, 1000)
    for what, mask, strategy in (("all, short", np.ones(700, bool), abi.FILTER_ALL), ("all", np.ones(1000, bool), abi.FILTER_ALL),
                                 ("zero-length", np.zeros(0, bool), abi.FILTER_NONE), ("none", np.zeros(1000, bool), abi.FILTER_NONE),
                                 ("slices", rng.random(1000) < 0.9, abi.FILTER_SLICES)):
        count = int(mask.sum())
        assert ref_strategy(count, len(mask)) == strategy, what
        exp = check_filter(gpu, col, HostArray.bool_from_numpy(mask), what)
        if strategy == abi.FILTER_ALL:
            assert (exp.offset, exp.length) == (9, count)
    # one selected row in every run of the slice: every run kept, through an All values plan
    s, e = physical_range(col.run_ends, col.offset, col.length)
    ends = np.asarray(col.run_ends, np.int64) - col.offset
    mask = np.zeros(col.length, bool)
    mask[np.clip(ends[s:e + 1], 1, col.length) - 1] = True
    _, new, rows = ref_filter_runs(col.run_ends, col.offset, col.length, col.length, int(mask.sum()), mask_rank(mask))
    assert len(rows) == e - s + 1 and 0 < mask.sum() < col.length
    check_filter(gpu, col, HostArray.bool_from_numpy(mask), "every run kept")


def abi_filter_run_end(gpu, col, plan):
    """acu_filter_run_end through ctypes with a given plan: (new run ends, kept physical rows, values plan strategy)."""
    lib, h = gpu.lib, gpu.h
    owned, vplan = [], C.c_void_p()
    try:
        d = gpu._run_descriptor(col, owned)
        w = col.run_ends.itemsize
        d_ends = gpu.malloc(len(col.run_ends) * w + 16)
        owned.append(d_ends)
        runs, vstart = C.c_int64(0), C.c_int64(0)
        gpu.check(lib.acu_filter_run_end(h, plan, C.byref(d), d_ends, C.byref(runs), C.byref(vstart), C.byref(vplan)))
        assert vplan
        pcount = lib.acu_filter_plan_count(vplan)
        buf = gpu.malloc(pcount * 4 + 16)
        owned.append(buf)
        gpu.check(lib.acu_filter_plan_indices(h, vplan, abi.U32, buf))
        return (gpu.d2h(d_ends, runs.value * w, col.run_ends.dtype), vstart.value + gpu.d2h(buf, pcount * 4, np.uint32).astype(np.int64),
                lib.acu_filter_plan_strategy(vplan))
    finally:
        if vplan:
            lib.acu_filter_plan_destroy(h, vplan)
        for p in owned:
            gpu.free(p)


@pytest.mark.gpu
def test_filter_with_comparison_plan(gpu):
    """A plan from acu_filter_plan_create_cmp (Int32 column < scalar, nulls unselected) gives the run ends and values plan
    of the equivalent boolean predicate."""
    rng = np.random.default_rng(71)
    col = RunEndColumn(np.cumsum(rng.integers(1, 5, 3000)).astype(np.int64), i64_values(rng, 3000)).slice(2, 6000)
    data = rng.integers(-100, 100, 5000).astype(np.int32)
    valid = rng.random(5000) >= 0.1
    a, b = HostArray.from_numpy(abi.I32, data, valid), HostArray.from_list(abi.I32, [17]).scalar()
    mask = (data < 17) & valid
    _, exp_ends, exp_rows = ref_filter_runs(col.run_ends, col.offset, col.length, 5000, int(mask.sum()), mask_rank(mask))
    da, db, bp = gpu.upload(a), gpu.upload(b), gpu.upload(HostArray.bool_from_numpy(data < 17, valid))
    plans = []
    try:
        for make in (lambda p: gpu.lib.acu_filter_plan_create_cmp(gpu.h, abi.I32, abi.LT, C.byref(da.descriptor()), C.byref(db.descriptor()), p),
                     lambda p: gpu.lib.acu_filter_plan_create(gpu.h, C.byref(bp.descriptor()), p)):
            plan = C.c_void_p()
            gpu.check(make(C.byref(plan)))
            plans.append(plan)
            assert gpu.lib.acu_filter_plan_count(plan) == int(mask.sum())
            ends, rows, strat = abi_filter_run_end(gpu, col, plan)
            assert ends.dtype == np.int64 and np.array_equal(ends, exp_ends) and np.array_equal(rows, exp_rows)
            s, e = physical_range(col.run_ends, col.offset, col.length)
            assert strat == ref_strategy(len(rows), e - s + 1)
    finally:
        for p in plans:
            gpu.lib.acu_filter_plan_destroy(gpu.h, p)
        for d in (da, db, bp):
            d.free()
    check_filter(gpu, col, HostArray.bool_from_numpy(data < 17, valid), "boolean predicate")
