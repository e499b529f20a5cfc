"""filter / take of Struct, sparse Union and dense Union columns on the device against tests/oracle_union.py, bit for bit:
type ids, offsets, every child buffer (the bytes under null rows included), NullBuffer presence and error status / text /
index. Every case uses a fixed seed. The partition's tile, warp and grid-round boundaries are sized from union.cu's
launch constants (checked against the source by test_union_launch_constants.py) and compared with a vectorised numpy
statement of the dense take."""
import numpy as np
import pytest

import acu
from acu import BOOL, DecimalArray, HostArray, ListColumn, StructColumn, UnionColumn, Utf8Column, ViewColumn
from acu import _abi as abi

import oracle_list as ol
import oracle_union as ou
import union_util as uu

pytestmark = pytest.mark.gpu

UN_THREADS = 256
UN_TILE_ROWS = 4096
UN_PER_SM = 8
INDEX_DTYPES = [abi.I8, abi.U8, abi.I16, abi.U16, abi.I32, abi.U32, abi.I64, abi.U64]
DENSE, SPARSE = abi.UNION_DENSE, abi.UNION_SPARSE


def nulls_of(mask, bit_offset=0, force=False):
    h = HostArray.from_list(abi.U8, [0 if v else None for v in mask], force_validity=force, bit_offset=bit_offset)
    h.values = np.zeros(0, np.uint8)
    return h


def child_of(kind, n, rng, null_p=0.2):
    mask = rng.random(n) >= null_p
    if kind == "i8":
        return HostArray.from_numpy(abi.I8, rng.integers(-128, 128, n), mask)
    if kind == "i64":
        return HostArray.from_numpy(abi.I64, rng.integers(-2**62, 2**62, n), mask)
    if kind == "i64nn":
        return HostArray.from_numpy(abi.I64, rng.integers(-2**62, 2**62, n))
    if kind == "bool":
        return HostArray.bool_from_numpy(rng.random(n) < 0.5, mask, bit_offset=3, mask_offset=5)
    if kind == "dec128":
        return DecimalArray.from_int64(16, 38, 2, rng.integers(-2**62, 2**62, n), mask)
    if kind == "view":
        items = [bytes(rng.integers(97, 123, rng.integers(0, 30)).astype(np.uint8)) if m else None for m in mask]
        return ViewColumn.from_values(items, garbage_under_nulls=[np.arange(16, dtype=np.uint8)])
    if kind == "utf8":  # bytes under null rows too: extend keeps them, take drops them
        lens = rng.integers(0, 9, n)
        offs = np.zeros(n + 1, dtype=np.int32)
        offs[1:] = np.cumsum(lens)
        return Utf8Column(offs, rng.integers(0, 256, int(offs[-1]) + 1).astype(np.uint8), nulls_of(mask))
    if kind == "list":
        inner = child_of("i64", 4 * n + 4, rng)
        lens = rng.integers(0, 5, n)
        offs = np.zeros(n + 1, np.int32)
        offs[1:] = np.cumsum(lens)
        return ListColumn(offs, inner, nulls_of(mask))
    if kind == "struct":
        return StructColumn([child_of("i64", n, rng), child_of("utf8", n, rng)], nulls_of(mask))
    raise ValueError(kind)


def dense_union(rng, ids, rows, kinds, p=None, extra=3):
    """A dense union of `rows` rows over fields `ids`; child f holds its rows plus `extra` unreferenced ones, its offsets
    point at a shuffled subset."""
    nf = len(ids)
    pick = rng.choice(nf, rows, p=p)
    tids = np.array(ids, np.int8)[pick]
    offs = np.zeros(rows, np.int32)
    children = []
    for f in range(nf):
        sel = np.nonzero(pick == f)[0]
        clen = len(sel) + extra
        offs[sel] = rng.permutation(clen)[:len(sel)]
        children.append(child_of(kinds[f % len(kinds)], clen, rng))
    return UnionColumn(DENSE, ids, children, tids, offs)


def sparse_union(rng, ids, rows, kinds):
    tids = np.array(ids, np.int8)[rng.integers(0, len(ids), rows)]
    return UnionColumn(SPARSE, ids, [child_of(kinds[f % len(kinds)], rows, rng) for f in range(len(ids))], tids)


def rand_pred(rng, n, p=0.5, null_p=0.1):
    return HostArray.bool_from_numpy(rng.random(n) < p, rng.random(n) >= null_p)


def rand_idx(rng, n_src, m, dtype=abi.U32, null_p=0.1):
    vals = rng.integers(0, max(n_src, 1), m)
    mask = rng.random(m) >= null_p
    return HostArray.from_numpy(dtype, vals, mask if null_p else None)


def _run(fn):
    try:
        return fn(), None
    except (acu.ArrowError, ou.OracleError) as e:
        return None, (e.status, e.message, e.index)


def check_filter(gpu, col, pred):
    exp, eerr = _run(lambda: ou.filter(col, ol.filter_mask(pred)))
    got, gerr = _run(lambda: gpu.filter(col, pred))
    assert gerr == eerr
    if eerr is None:
        assert ou.describe(got) == ou.describe(exp)
    return got


def check_take(gpu, col, idx, check_bounds=False):
    exp, eerr = _run(lambda: ou.take_host(col, idx, check_bounds))
    got, gerr = _run(lambda: gpu.take(col, idx, check_bounds))
    assert gerr == eerr
    if eerr is None:
        assert ou.describe(got) == ou.describe(exp)
    return got, gerr


# ---- the reference's cases ---------------------------------------------------------------------------------------------
CASES = uu.golden_cases()


@pytest.mark.parametrize("i", range(len(CASES)), ids=[f"{c['name']}-{k}" for k, c in enumerate(CASES)])
def test_golden(gpu, i):
    case = CASES[i]
    got = uu.run_case(case, gpu.filter, gpu.take)
    uu.check(case, got)
    exp = uu.run_case(case, lambda c, p: ou.filter(c, ol.filter_mask(p)), ou.take_host)
    assert ou.describe(got) == ou.describe(exp)


# ---- dense partition: field counts, ids, distributions -------------------------------------------------------------------
@pytest.mark.parametrize("nf,dist", [(1, "uniform"), (2, "uniform"), (5, "uniform"), (5, "skewed"), (5, "one"), (128, "uniform"),
                                     (128, "skewed")])
def test_dense_fields_and_distributions(gpu, nf, dist):
    rng = np.random.default_rng(100 + nf + len(dist))
    ids = [3, 7, 42, 127, 0][:nf] if nf <= 5 else list(rng.permutation(128))
    p = None
    if dist == "skewed":
        p = np.full(nf, 0.02 / max(nf - 1, 1))
        p[0] = 0.98 if nf > 1 else 1.0
        p /= p.sum()
    elif dist == "one":
        p = np.zeros(nf)
        p[nf - 1] = 1.0
    col = dense_union(rng, ids, 3000, ["i64", "i8", "utf8"], p)
    check_filter(gpu, col, rand_pred(rng, col.length))
    check_take(gpu, col, rand_idx(rng, col.length, 2500))


@pytest.mark.parametrize("kind", ["i8", "i64", "dec128", "bool", "utf8", "view", "list", "struct"])
@pytest.mark.parametrize("mode", [DENSE, SPARSE])
def test_child_types(gpu, kind, mode):
    rng = np.random.default_rng(7 + len(kind) + mode)
    col = (dense_union if mode == DENSE else sparse_union)(rng, [5, 1], 300, [kind, "i64"])
    check_filter(gpu, col, rand_pred(rng, col.length))
    check_take(gpu, col, rand_idx(rng, col.length, 250))
    check_take(gpu, col, rand_idx(rng, col.length, 250, null_p=0))


def test_union_inside_struct_inside_list(gpu):
    rng = np.random.default_rng(11)
    u = dense_union(rng, [2, 9], 200, ["utf8", "i64"])
    s = StructColumn([u, child_of("i64", 200, rng)], nulls_of(rng.random(200) >= 0.2))
    offs = np.zeros(61, np.int32)
    offs[1:] = np.cumsum(rng.integers(0, 4, 60))
    assert offs[-1] <= 200
    lst = ListColumn(offs, s, nulls_of(rng.random(60) >= 0.2))
    check_filter(gpu, lst, rand_pred(rng, 60))
    check_filter(gpu, lst, HostArray.bool_from_numpy(np.ones(60, bool)))
    check_take(gpu, lst, rand_idx(rng, 60, 80, null_p=0.1))
    su = sparse_union(rng, [4, 0], 200, ["struct", "utf8"])
    lst2 = ListColumn(offs, su, nulls_of(rng.random(60) >= 0.2))
    check_filter(gpu, lst2, rand_pred(rng, 60))
    check_take(gpu, lst2, rand_idx(rng, 60, 80, null_p=0.1))


def test_dense_union_in_list_with_an_all_plan_extends_every_row(gpu):
    rng = np.random.default_rng(12)
    u = dense_union(rng, [1, 6], 100, ["utf8", "i64"], extra=20)
    offs = np.array([0, 40, 40, 100], np.int32)
    lst = ListColumn(offs, u, nulls_of([True, False, True]))
    check_filter(gpu, lst, HostArray.bool_from_numpy(np.array([True, False, True])))


# ---- slices ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", [DENSE, SPARSE])
def test_sliced_unions(gpu, mode):
    rng = np.random.default_rng(20 + mode)
    col = (dense_union if mode == DENSE else sparse_union)(rng, [3, 4, 8], 500, ["utf8", "i64", "struct"])
    for off, ln in ((0, 500), (1, 498), (37, 300), (499, 1), (250, 0)):
        sl = col.slice(off, ln)
        check_filter(gpu, sl, rand_pred(rng, ln))
        check_take(gpu, sl, rand_idx(rng, ln, 200))


def test_sliced_structs(gpu):
    rng = np.random.default_rng(30)
    s = StructColumn([child_of("i64", 300, rng), child_of("utf8", 300, rng), child_of("bool", 300, rng)],
                     nulls_of(rng.random(300) >= 0.3, bit_offset=5))
    for off, ln in ((0, 300), (3, 200), (65, 130), (299, 1)):
        sl = s.slice(off, ln)
        check_filter(gpu, sl, rand_pred(rng, ln))
        check_take(gpu, sl, rand_idx(rng, ln, 150))


# ---- filter strategies and predicate lengths ---------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["dense", "sparse", "struct", "empty_struct"])
def test_filter_strategies_and_lengths(gpu, which):
    rng = np.random.default_rng(40 + len(which))
    n = 200
    if which == "dense":
        col = dense_union(rng, [0, 100], n, ["utf8", "i64"])
    elif which == "sparse":
        col = sparse_union(rng, [0, 100], n, ["utf8", "i64"])
    elif which == "struct":
        col = StructColumn([child_of("i64", n, rng), child_of("utf8", n, rng)], nulls_of(rng.random(n) >= 0.2))
    else:
        col = StructColumn([], nulls_of(rng.random(n) >= 0.2))
    for pred in (HostArray.bool_from_numpy(np.zeros(n, bool)), HostArray.bool_from_numpy(np.ones(n, bool)),
                 rand_pred(rng, n, null_p=0.3), rand_pred(rng, n - 17), HostArray.bool_from_numpy(np.ones(n - 17, bool)),
                 rand_pred(rng, n + 1)):
        check_filter(gpu, col, pred)


# ---- take: index types, nulls, bounds, duplicates, errors ----------------------------------------------------------------
@pytest.mark.parametrize("dtype", INDEX_DTYPES)
@pytest.mark.parametrize("which", ["dense", "sparse", "struct"])
def test_take_index_dtypes(gpu, dtype, which):
    rng = np.random.default_rng(50 + dtype + len(which))
    n = 100
    if which == "dense":
        col = dense_union(rng, [3, 7, 42], n, ["utf8", "i64", "struct"])
    elif which == "sparse":
        col = sparse_union(rng, [3, 7, 42], n, ["utf8", "i64", "struct"])
    else:
        col = StructColumn([child_of("i64", n, rng), child_of("view", n, rng)], nulls_of(rng.random(n) >= 0.2))
    check_take(gpu, col, rand_idx(rng, n, 120, dtype))  # duplicates
    check_take(gpu, col, rand_idx(rng, n, 0, dtype))
    bad = rand_idx(rng, n, 60, dtype)
    bad.values[17] = 101  # out of bounds
    for cb in (False, True):
        check_take(gpu, col, bad, cb)
    bad.validity = acu.pack_bits(np.arange(60) != 17)  # ... under a null: the gather reads 0 / type id 0
    bad.null_count = 1
    for cb in (False, True):
        check_take(gpu, col, bad, cb)


def test_null_out_of_bounds_index_fails_union_validation(gpu):
    rng = np.random.default_rng(60)
    for mode in (DENSE, SPARSE):
        col = (dense_union if mode == DENSE else sparse_union)(rng, [3, 7], 50, ["i64", "utf8"])
        idx = HostArray.from_list(abi.U32, [1, None, 2])
        idx.values[1] = 1000
        _, err = check_take(gpu, col, idx)
        assert err[0] == abi.ERR_INVALID_ARGUMENT and err[1].endswith(ou.UNION_TYPE_IDS)
        col0 = (dense_union if mode == DENSE else sparse_union)(rng, [0, 7], 50, ["i64", "utf8"])
        check_take(gpu, col0, idx)  # type id 0 is a field: no error


def test_child_error_is_reported_ahead_of_the_validation(gpu):
    # type id 0 names a field whose child is empty: a null out-of-bounds index's offset 0 panics in the child first
    col = UnionColumn(DENSE, [0, 5], [HostArray.from_list(abi.I64, []), HostArray.from_list(abi.I64, [1, 2])], [5, 5], [0, 1])
    idx = HostArray.from_list(abi.U32, [0, None])
    idx.values[1] = 9
    _, err = check_take(gpu, col, idx)
    assert err[0] == abi.ERR_PANIC_OUT_OF_BOUNDS
    # a union whose ids do not include 0: the validation error
    col2 = UnionColumn(DENSE, [5], [HostArray.from_list(abi.I64, [1, 2])], [5, 5], [0, 1])
    _, err = check_take(gpu, col2, idx)
    assert err[1].endswith(ou.UNION_TYPE_IDS)


def test_struct_validity_reads(gpu):
    rng = np.random.default_rng(70)
    n = 40
    for fields in ([], [child_of("i64", n, rng)], [child_of("utf8", n, rng), child_of("bool", n, rng)]):
        for nulls in (nulls_of(rng.random(n) >= 0.3), nulls_of(np.ones(n, bool), force=True), nulls_of(np.ones(n, bool))):
            s = StructColumn(fields, nulls)
            check_take(gpu, s, rand_idx(rng, n, 30))
            check_take(gpu, s, rand_idx(rng, n, 30, null_p=0))
            bad = HostArray.from_list(abi.U32, [0, 3, n + 5, 1])
            check_take(gpu, s, bad, True)
            if len(fields) < 2:  # a valid index past an Int64 field: the field's panic comes before the validity's
                check_take(gpu, s, bad)
            bad_null = HostArray.from_list(abi.U32, [0, None, 1])
            bad_null.values[1] = n + 5
            check_take(gpu, s, bad_null)
            check_filter(gpu, s, rand_pred(rng, n))


def test_empty_field_structs(gpu):
    rng = np.random.default_rng(80)
    s = StructColumn([], nulls_of([False, True, False, True, False, True], force=True))
    for idx in (HostArray.from_list(abi.U32, [0, 2, 1, 4]), HostArray.from_list(abi.U32, [1, 3]), HostArray.from_list(abi.U32, [])):
        check_take(gpu, s, idx)
    check_filter(gpu, s, HostArray.bool_from_numpy(np.array([True, True, False, True, False, False])))
    inner = StructColumn([child_of("i64", 30, rng), StructColumn([], nulls_of(np.ones(30, bool), force=True))],
                         nulls_of(rng.random(30) >= 0.2))
    check_take(gpu, inner, rand_idx(rng, 30, 25))
    check_filter(gpu, inner, rand_pred(rng, 30))


def test_run_end_take_refuses_struct_and_union_values(gpu):
    rng = np.random.default_rng(90)
    for values in (StructColumn([child_of("i64", 3, rng)], nulls_of([True] * 3)), sparse_union(rng, [1], 3, ["i64"])):
        col = acu.RunEndColumn(np.array([2, 5, 9], np.int32), values)
        with pytest.raises(acu.ArrowError) as e:
            gpu.take_run_end(col, HostArray.from_list(abi.U32, [0, 4]))
        assert e.value.status == abi.ERR_NOT_YET_IMPLEMENTED
        got = gpu.filter_run_end(col, HostArray.bool_from_numpy(np.array([True, False, True, True, False, False, True, False, True])))
        assert got.length == 5


# ---- partition boundaries ------------------------------------------------------------------------------------------------
def np_dense_take(col, idx):
    """take of a dense union of Int64 children without nulls by in-bounds indices without nulls, vectorised."""
    tids = col.type_ids[idx]
    src = col.offsets[idx]
    new = np.zeros(len(idx), np.int32)
    children = []
    for t, c in zip(col.field_type_ids, col.children):
        sel = np.nonzero(tids == t)[0]
        new[sel] = np.arange(len(sel), dtype=np.int32)
        children.append(np.asarray(c.values)[src[sel]])
    return tids, new, children


def _boundary_sizes(gpu):
    round_rows = gpu.lib.acu_device_sm_count(gpu.h) * UN_PER_SM * UN_TILE_ROWS
    return [1, 31, 32, 33, UN_THREADS - 1, UN_THREADS + 1, UN_TILE_ROWS - 1, UN_TILE_ROWS, UN_TILE_ROWS + 1,
            round_rows - 1, round_rows + 1, round_rows * 2 + UN_TILE_ROWS // 2 + 7]


BOUNDARY_CASES = [(k, 4) for k in range(12)] + [(k, 128) for k in (2, 8, 9, 10, 11)]


@pytest.mark.parametrize("k,nf", BOUNDARY_CASES)
def test_partition_boundaries(gpu, k, nf):
    """Take and filter of m rows at a warp, a tile and a grid round +- 1 and past two rounds, with 4 skewed fields and with
    128 fields (one k_union_scan block per field over many tiles, and 128 per-field tile bases in k_union_scatter)."""
    m = _boundary_sizes(gpu)[k]
    rng = np.random.default_rng(1000 + k + nf)
    if nf == 4:
        ids, p = [3, 7, 42, 127], [0.7, 0.2, 0.05, 0.05]
    else:
        ids, p = [int(x) for x in rng.permutation(128)], None
    n = m + 100
    pick = rng.choice(nf, n, p=p)
    tids = np.array(ids, np.int8)[pick]
    offs = np.zeros(n, np.int32)
    children = []
    for f in range(nf):
        sel = np.nonzero(pick == f)[0]
        offs[sel] = rng.permutation(len(sel)).astype(np.int32)
        children.append(HostArray.from_numpy(abi.I64, rng.integers(-2**62, 2**62, max(len(sel), 1))))
    col = UnionColumn(DENSE, ids, children, tids, offs)
    idx = rng.integers(0, n, m).astype(np.uint32)
    got = gpu.take(col, HostArray.from_numpy(abi.U32, idx))
    et, eo, ec = np_dense_take(col, idx)
    assert np.array_equal(got.type_ids, et) and np.array_equal(got.offsets, eo)
    for g, e in zip(got.children, ec):
        assert g.validity is None and np.array_equal(np.asarray(g.values[:g.length]), e)
    # filter of the first m rows: the take of the selected rows, or the empty union / the slice for NONE / ALL
    for mask in (rng.random(m) < 0.6, np.zeros(m, bool), np.ones(m, bool)):
        got = gpu.filter(col, HostArray.bool_from_numpy(mask))
        sel = np.nonzero(mask)[0].astype(np.uint32)
        assert got.length == len(sel)
        if len(sel) == m:  # values.slice(0, count): the children stay whole
            assert np.array_equal(got.type_ids, tids[:m]) and np.array_equal(got.offsets, offs[:m])
            assert all(g.length == c.length for g, c in zip(got.children, children))
            continue
        et, eo, ec = np_dense_take(col, sel)
        assert np.array_equal(got.type_ids, et) and np.array_equal(got.offsets, eo)
        for g, e in zip(got.children, ec):
            assert g.length == len(e) and np.array_equal(np.asarray(g.values[:g.length]), e)
