"""The List / LargeList / FixedSizeList kernels of csrc/list.cu where their code paths switch and past one grid-stride
round, against a vectorised numpy restatement of one list level (checked against tests/oracle_filter_take.py on small cases):

  k_list_expand    one thread per 64-bit child word: `base` and `child_end` mid-word and on word boundaries, rows that
                   start and end on words, a word of 64 one-row hops, words crossed by runs of empty rows (the binary
                   search), FixedSizeList rows spanning many words, 2.5 grid rounds of words.
  k_list_row_map   a warp owns 32 x RM_ROWS output child rows, lane rows c0 + lane + 32 i: output rows ending at lane
                   positions 31 / 32 / 33 and at 511 / 512 / 513 of a span, rows longer than a span, leading empty rows,
                   runs of empty rows (null index, null list, zero-length row), repeated and descending indices, both map
                   types, LargeList rows straddling 2^32 and near 2^40, the UInt32 map up to child row UINT32_MAX, and
                   2.5 rounds with row boundaries on the round boundaries.
  k_fsl_row_map    (u32)(index * size) + k, 0 and null under a null index; the validity walk of one word per thread at
                   index validity offsets 0 / 1 / 7 / 63, and both loops past one round.
  offsets engine   the i32 List take at exactly INT32_MAX and one past it, out-of-bounds and overflow rows in different
                   engine blocks in both orders; k_narrow_offsets past 2.5 rounds.

The ABI tests drive acu_filter_list / acu_take_list through ctypes and read their outputs (the child plan, the row map,
its validity) directly. acu_list_array carries no child pointer and neither call reads the child, so a descriptor may
declare a child far larger than any allocation: such a plan or row map is only copied back and compared, never handed
to a child gather. Every test asserts that its rows sit where it says they do."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import acu
from acu import FixedSizeListColumn, HostArray, ListColumn, Utf8Column, bitmap_bytes, pack_bits
from acu import _abi as abi

import oracle_filter_take as oft
from oracle_filter_take import nulls_of

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "arrow-rs_b200", "csrc")

# Mirrors of list.cu's launch geometry (pinned by test_constants_pinned).
RM_ROWS = 16           # child rows per lane of k_list_row_map: a warp owns a span of 32 x RM_ROWS rows
SPAN = 32 * RM_ROWS
THREADS = 256          # every list kernel runs 256-thread blocks
BLOCKS_PER_SM = 8      # acu_grid(ctx, ..., 8): at most SMs x 8 blocks
BY_ROWS = 2048         # bytes_engine.cuh: index rows per engine block

INDEX_DTYPES = [abi.I8, abi.U8, abi.I16, abi.U16, abi.I32, abi.U32, abi.I64, abi.U64]
SIGNED = (abi.I8, abi.I16, abi.I32, abi.I64)
I32_MAX, U32_MAX = 2**31 - 1, 2**32 - 1
FSL_SIZES = [1, 3, 63, 64, 65, 768, 4097]
OB = {abi.LIST: 4, abi.LARGE_LIST: 8, abi.FIXED_SIZE_LIST: 0}


# ---- 1. the vectorised one-level reference -----------------------------------------------------------------------------
def to_index(vals, dtype):
    """ToIndices as u64: i8 / i16 / i32 sign-extend and keep the low 32 bits, i64 reinterprets, unsigned as is."""
    v = np.asarray(vals)
    if dtype in (abi.I8, abi.I16, abi.I32):
        return (v.astype(np.int64) & 0xFFFFFFFF).astype(np.uint64)
    if dtype == abi.I64:
        return v.astype(np.int64).view(np.uint64)
    return v.astype(np.uint64)


def ref_filter(offsets, size, sel):
    """(child predicate over [0, child_end), new offsets or None) of one level; offsets are absolute (None: FSL)."""
    sel = np.asarray(sel, bool)
    if offsets is None:
        return np.repeat(sel, size), None
    offs = np.asarray(offsets, np.int64)
    n = len(sel)
    lens = np.diff(offs[:n + 1])
    pred = np.concatenate([np.zeros(int(offs[0]), bool), np.repeat(sel, lens)])
    new = np.concatenate([[0], np.cumsum(lens[sel])]).astype(np.asarray(offsets).dtype)
    return pred, new


def ref_strategy(count, n):
    """IterationStrategy::default_strategy (filter.rs:346-364) as the plan reports it."""
    if count == 0:
        return abi.FILTER_NONE
    if count == n:
        return abi.FILTER_ALL
    return abi.FILTER_SLICES if count / n > 0.8 else abi.FILTER_INDEX


def _bounds_error(vals, valid, dtype, n):
    """take's check_bounds (take.rs:183-208): the first index >= len (or < 0 without index nulls)."""
    allv = valid is None or bool(np.all(valid))
    if dtype in SIGNED:
        raw = np.asarray(vals).astype(np.int64)
        bad = (raw >= n) | ((raw < 0) & allv)
    else:
        raw = np.asarray(vals).astype(np.uint64)
        bad = raw >= np.uint64(n)
    if not allv:
        bad &= np.asarray(valid, bool)
    rows = np.flatnonzero(bad)
    if len(rows) == 0:
        return None
    j = int(rows[0])
    return oft.OracleError(abi.ERR_COMPUTE, f"Array index out of bounds, cannot get item at index {int(vals[j])} from {n} entries", j)


def ref_take_list(offsets, list_valid, vals, valid, dtype, check_bounds=False):
    """One List / LargeList take level: (new offsets, row lengths, source starts, error). The reference's loop visits the
    rows in order: the first out-of-bounds row panics in list_offsets[ix], the first row whose end passes i32::MAX
    panics in from_usize(..).unwrap(), whichever comes first; with list nulls take_nulls panics first."""
    offs = np.asarray(offsets, np.int64)
    n, m = len(offs) - 1, len(vals)
    if check_bounds and (err := _bounds_error(vals, valid, dtype, n)) is not None:
        return None, None, None, err
    ix = to_index(vals, dtype)
    v = np.ones(m, bool) if valid is None else np.asarray(valid, bool)
    lv = np.ones(n, bool) if list_valid is None else np.asarray(list_valid, bool)
    inb = ix < np.uint64(n)
    oob_rows = np.flatnonzero(v & ~inb)
    if len(oob_rows) and not lv.all():
        return None, None, None, oft.OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, "assertion failed: idx < self.bit_len", int(oob_rows[0]))
    ixs = np.where(inb, ix, 0).astype(np.int64)
    if n == 0:
        lv, offs = np.ones(1, bool), np.append(offs, offs[-1])  # every row is out of bounds or null
    live = v & inb & lv[ixs]
    lens = np.where(live, offs[ixs + 1] - offs[ixs], 0)
    ends = np.cumsum(lens)
    ovf_rows = np.flatnonzero(ends > I32_MAX) if np.asarray(offsets).dtype == np.int32 else []
    oob = int(oob_rows[0]) if len(oob_rows) else None
    ovf = int(ovf_rows[0]) if len(ovf_rows) else None
    if oob is not None and (ovf is None or oob < ovf):
        bad = int(ix[oob])
        return None, None, None, oft.OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS,
                                                f"index out of bounds: the len is {n + 1} but the index is {bad + 1 if bad == n else bad}", oob)
    if ovf is not None:
        return None, None, None, oft.OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, oft.UNWRAP_NONE, ovf)
    return np.concatenate([[0], ends]), lens, offs[ixs], None


def ref_list_map(new, lens, src, map_dtype):
    """The child row map: np.repeat(src_start - new_start, new_len) + arange(total), exact in i64."""
    total = int(new[-1])
    return (np.repeat(src - new[:-1], lens) + np.arange(total, dtype=np.int64)).astype(map_dtype)


def ref_fsl_map(vals, valid, dtype, size):
    """take_value_indices_from_fixed_size_list: (u32(index) * u32(size) + k) mod 2^32, 0 under a null index; the map's
    validity (None without index nulls) and null_count = null indices x size."""
    ix = to_index(vals, dtype) & np.uint64(U32_MAX)
    m = len(ix)
    mp = ((np.repeat((ix * np.uint64(size)) & np.uint64(U32_MAX), size) + np.tile(np.arange(size, dtype=np.uint64), m))
          & np.uint64(U32_MAX)).astype(np.uint32)
    if valid is None or np.all(valid):
        return mp, None, 0
    vm = np.repeat(np.asarray(valid, bool), size)
    mp[~vm] = 0
    return mp, vm, int((~np.asarray(valid, bool)).sum()) * size


def ref_take_fsl(n, list_valid, child_len, vals, valid, dtype, size, check_bounds=False):
    """A FixedSizeList take level's map, and its error: the child take's (the first valid map entry past the child),
    then take_bits' (a valid index past the list with list nulls)."""
    if check_bounds and (err := _bounds_error(vals, valid, dtype, n)) is not None:
        return None, None, err
    mp, vm, _ = ref_fsl_map(vals, valid, dtype, size)
    bad = np.flatnonzero((mp >= child_len) & (True if vm is None else vm))
    if len(bad):
        return None, None, oft.OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, f"Out-of-bounds index {int(mp[bad[0]])}", int(bad[0]))
    v = np.ones(len(vals), bool) if valid is None else np.asarray(valid, bool)
    if list_valid is not None and not np.all(list_valid) and (v & (to_index(vals, dtype) >= np.uint64(n))).any():
        j = int(np.flatnonzero(v & (to_index(vals, dtype) >= np.uint64(n)))[0])
        return None, None, oft.OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, "assertion failed: idx < self.bit_len", j)
    return mp, vm, None


def _rand_index_values(rng, dtype, n, m):
    """Index values of `dtype`: mostly in bounds, some out of bounds, negative ones for the signed types."""
    info = np.iinfo(acu.NP_DTYPES[dtype])
    vals = rng.integers(0, max(n, 1), m).astype(np.int64)
    pick = rng.random(m)
    vals = np.where(pick < 0.04, n, vals)
    vals = np.where((pick >= 0.04) & (pick < 0.07), min(int(info.max), 2**62), vals)
    if dtype in SIGNED:
        vals = np.where((pick >= 0.07) & (pick < 0.1), rng.integers(max(int(info.min), -2**40), 0, m), vals)
    return np.clip(vals, max(int(info.min), -2**62), min(int(info.max), 2**62)).astype(acu.NP_DTYPES[dtype])


def test_reference_matches_oracle():
    """The vectorised reference against tests/oracle_filter_take.py on 360 small cases: all three kinds, the eight index dtypes
    (negative i8 / i16 / i32 / i64 included), null indices, null lists, sliced lists, short predicates, check_bounds."""
    rng = np.random.default_rng(2024)
    seen = set()
    for case in range(360):
        kind = (abi.LIST, abi.LARGE_LIST, abi.FIXED_SIZE_LIST)[case % 3]
        dtype = INDEX_DTYPES[(case // 3) % 8]
        child_n = int(rng.integers(0, 80))
        child = HostArray.from_numpy(abi.I64, np.arange(child_n))  # child values are child rows
        lnull = float(rng.choice([0.0, 0.0, 0.3]))
        if kind == abi.FIXED_SIZE_LIST:
            size = int(rng.choice([0, 1, 2, 3, 5, 64]))
            rows = child_n // size if size else int(rng.integers(0, 9))
            lmask = rng.random(rows) >= lnull
            col = FixedSizeListColumn(size, child, nulls_of(lmask, int(rng.integers(0, 8))))
            offsets = None
        else:
            base = int(rng.integers(0, 4)) if child_n >= 4 else 0
            lens, pos = [], base
            while True:
                ln = int(rng.choice([0, 0, 1, 2, 3, 5]))
                if pos + ln > child_n:
                    break
                lens.append(ln)
                pos += ln
            offsets = np.concatenate([[base], base + np.cumsum(lens, dtype=np.int64)]).astype(np.int64 if kind == abi.LARGE_LIST else np.int32)
            lmask = rng.random(len(lens)) >= lnull
            col = ListColumn(offsets, child, nulls_of(lmask, int(rng.integers(0, 8))))
            rows = col.length
        seen.add(("sliced", kind != abi.FIXED_SIZE_LIST and int(offsets[0]) > 0))
        seen.add(("list nulls", not lmask.all()))
        # filter
        plen = int(rng.integers(0, rows + 1))
        pred = HostArray.bool_from_numpy(rng.random(plen) < rng.random(), rng.random(plen) >= 0.1)
        mask = oft.filter_mask(pred)
        exp = oft.filter(col, mask)
        cpred, new = ref_filter(offsets, col.size if offsets is None else 0, mask)
        assert np.array_equal(exp.child.value_array(), np.flatnonzero(cpred)), case
        if offsets is not None:
            assert exp.offsets.dtype == new.dtype and np.array_equal(exp.offsets, new), case
        # take
        m = int(rng.integers(0, 40))
        vals = _rand_index_values(rng, dtype, rows, m)
        if kind == abi.FIXED_SIZE_LIST and case % 2:  # indices whose index * size wraps back into the child
            vals = np.where(rng.random(m) < 0.5, vals, np.array(2**32 // max(col.size, 1) + 1, np.int64).astype(vals.dtype))
        valid = None if case % 4 == 0 else rng.random(m) >= 0.2
        cb = case % 5 == 0
        seen.add(("negative", dtype in SIGNED and bool((vals < 0).any())))
        seen.add(("index nulls", valid is not None and not valid.all()))
        idx_valid = [True] * m if valid is None else list(valid)
        try:
            got = oft.take(col, list(vals), idx_valid, valid is not None, dtype, cb)
            err = None
        except oft.OracleError as e:
            got, err = None, e
        if kind == abi.FIXED_SIZE_LIST:
            mp, vm, rerr = ref_take_fsl(rows, lmask, child_n, vals, valid, dtype, col.size, cb)
        else:
            new, lens, src, rerr = ref_take_list(offsets, lmask, vals, valid, dtype, cb)
        if err is not None or rerr is not None:
            assert err is not None and rerr is not None, (case, err, rerr)
            assert (err.status, err.message, err.index) == (rerr.status, rerr.message, rerr.index), case
            seen.add(("error", err.message.split(" ")[0]))
            continue
        if kind == abi.FIXED_SIZE_LIST:
            cvm = got.child.valid_mask()
            assert np.array_equal(cvm, np.ones(len(mp), bool) if vm is None else vm), case
            assert np.array_equal(got.child.value_array()[cvm], mp[cvm].astype(np.int64)), case
        else:
            assert np.array_equal(got.offsets.astype(np.int64), new), case
            assert np.array_equal(got.child.value_array(), ref_list_map(new, lens, src, np.int64)), case
    for fact in [("sliced", True), ("list nulls", True), ("negative", True), ("index nulls", True), ("error", "index"),
                 ("error", "assertion"), ("error", "Out-of-bounds"), ("error", "Compute")]:
        assert fact in seen, fact


# ---- 5. the constants the placements depend on -------------------------------------------------------------------------
def test_constants_pinned():
    """A retune of any of these moves the boundaries away from the rows placed on them: update the mirrors above (and the
    placements) together with the kernels."""
    with open(os.path.join(CSRC, "list.cu"), encoding="utf-8") as f:
        src = f.read()
    with open(os.path.join(CSRC, "bytes_engine.cuh"), encoding="utf-8") as f:
        eng = f.read()
    assert re.search(r"#define RM_ROWS (\d+)\s", src).group(1) == str(RM_ROWS)
    assert "for (int64_t c0 = warp * (32 * RM_ROWS); c0 < total; c0 += nwarps * (32 * RM_ROWS))" in src
    assert "const int64_t c = c0 + lane + 32 * i;" in src
    for k in ("k_list_expand", "k_list_row_map", "k_fsl_row_map"):
        assert re.search(r"__launch_bounds__\((\d+)\) " + k, src).group(1) == str(THREADS), k
    grids = re.findall(r"acu_grid\(ctx, ([^;]*?), (\d+)\)[,;]", src)
    assert len(grids) == 4, grids
    for work, per_sm in grids:
        assert int(per_sm) == BLOCKS_PER_SM, work
    assert re.findall(r"acu_grid\(ctx, [^;]*?, \d+\), (\d+), 0", src) == [str(THREADS)] * 3
    assert re.findall(r"k_list_row_map<uint(?:32|64)_t>, grid, (\d+), 0", src) == [str(THREADS)] * 2
    works = sorted(w for w, _ in grids)
    assert works == sorted(["(n_words + 255) / 256", "(m + 1 + 255) / 256", "(total + 32 * RM_ROWS * 8 - 1) / (32 * RM_ROWS * 8)",
                            "(total + 255) / 256"]), works
    assert re.search(r"#define BY_THREADS (\d+)\s", eng).group(1) == str(BY_ROWS // 4)
    assert re.search(r"#define BY_ROWS \(BY_THREADS \* (\d+)\)", eng).group(1) == "4"


def round_words(sms):
    """64-bit child words of one k_list_expand round (one word per thread); also the rows of one round of
    k_narrow_offsets and of k_fsl_row_map's map loop, and the words of its validity loop."""
    return sms * BLOCKS_PER_SM * THREADS


def round_rows(sms):
    """Output child rows of one k_list_row_map round."""
    return sms * BLOCKS_PER_SM * (THREADS // 32) * SPAN


# ---- ctypes drivers ----------------------------------------------------------------------------------------------------
def bits_of(buf, n, off=0):
    return np.unpackbits(np.asarray(buf, np.uint8), bitorder="little")[off:off + n].astype(bool)


def list_desc(gpu, owned, kind, offsets=None, size=0, n_rows=0, valid=None, valid_off=0, child_len=0):
    """An acu_list_array without a child: the list calls read only the offsets and the validity."""
    d = abi.ListArray()
    d.kind, d.list_size = kind, size
    if offsets is not None:
        off = np.ascontiguousarray(offsets)
        d.offsets = gpu.malloc(off.nbytes + 16)
        owned.append(d.offsets)
        gpu.h2d(d.offsets, off)
        n_rows = len(off) - 1
    nl = abi.Array()
    nl.len = n_rows
    if valid is not None:
        bits = pack_bits(valid, valid_off)
        nl.validity = gpu.malloc(bits.nbytes + 8)
        owned.append(nl.validity)
        gpu.h2d(nl.validity, bits)
        nl.validity_offset, nl.null_count = valid_off, int((~np.asarray(valid, bool)).sum())
    d.nulls = nl
    d.child_len = child_len
    return d


def abi_filter(gpu, desc, pred):
    """acu_filter_list: (new offsets, validity mask or None, child plan (len, count, strategy), selected child rows)."""
    lib, h = gpu.lib, gpu.h
    ob = OB[desc.kind]
    dp = gpu.upload(pred)
    plan, cp, owned = C.c_void_p(), C.c_void_p(), []
    try:
        pd = dp.descriptor()
        gpu.check(lib.acu_filter_plan_create(h, C.byref(pd), C.byref(plan)))
        count = lib.acu_filter_plan_count(plan)
        d_off = gpu.malloc((count + 1) * max(ob, 1) + 16)
        owned.append(d_off)
        out = gpu.alloc_out(0, count)
        owned += [out.values, out.validity]
        gpu.check(lib.acu_filter_list(h, plan, C.byref(desc), d_off, C.byref(out), C.byref(cp)))
        offs = gpu.d2h(d_off, (count + 1) * ob, np.int32 if ob == 4 else np.int64) if ob else None
        nulls = bits_of(gpu.d2h(out.validity, bitmap_bytes(count)), count) if out.has_validity else None
        plen, pcount, strat = lib.acu_filter_plan_len(cp), lib.acu_filter_plan_count(cp), lib.acu_filter_plan_strategy(cp)
        wide = plen > U32_MAX
        buf = gpu.malloc(pcount * (8 if wide else 4) + 16)
        owned.append(buf)
        gpu.check(lib.acu_filter_plan_indices(h, cp, abi.U64 if wide else abi.U32, buf))
        sel = gpu.d2h(buf, pcount * (8 if wide else 4), np.uint64 if wide else np.uint32)
        return offs, nulls, (plen, pcount, strat), sel
    finally:
        if cp:
            lib.acu_filter_plan_destroy(h, cp)
        if plan:
            lib.acu_filter_plan_destroy(h, plan)
        dp.free()
        for p in owned:
            gpu.free(p)


def abi_take(gpu, desc, idx, cdt, check_bounds=False, write_map=True):
    """acu_take_list, the sizing call and (write_map) the call that writes the row map: dict of rows, offsets, the list
    validity mask (None without a NullBuffer), map, map validity (None without one) and its null_count."""
    lib, h = gpu.lib, gpu.h
    ob, m = OB[desc.kind], idx.length
    di = gpu.upload(idx)
    owned = []
    try:
        idd = di.descriptor()
        d_off = gpu.malloc((m + 1) * max(ob, 1) + 16)
        owned.append(d_off)
        out = gpu.alloc_out(0, m)
        owned += [out.values, out.validity]
        cn, rows = abi.ArrayOut(), C.c_int64(-1)
        args = lambda mp, cap: (h, C.byref(desc), C.byref(idd), idx.dtype, int(check_bounds), 0, d_off, C.byref(out), cdt, mp, cap,
                                C.byref(rows), C.byref(cn))
        gpu.check(lib.acu_take_list(*args(None, 0)))
        res = {"rows": rows.value}
        if write_map:
            n, w = rows.value, (4 if cdt == abi.U32 else 8)
            rmap = gpu.malloc(n * w + 16)
            owned.append(rmap)
            cn.validity = gpu.malloc(bitmap_bytes(n) + 8)
            owned.append(cn.validity)
            gpu.check(lib.acu_take_list(*args(rmap, n)))
            assert rows.value == n
            res["map"] = gpu.d2h(rmap, n * w, np.uint32 if w == 4 else np.uint64)
            res["map_valid"] = bits_of(gpu.d2h(cn.validity, bitmap_bytes(n)), n) if cn.has_validity else None
            res["map_nulls"] = cn.null_count if cn.has_validity else 0
        res["offsets"] = gpu.d2h(d_off, (m + 1) * ob, np.int32 if ob == 4 else np.int64) if ob else None
        res["nulls"] = bits_of(gpu.d2h(out.validity, bitmap_bytes(m)), m) if out.has_validity else None
        return res
    finally:
        di.free()
        for p in owned:
            gpu.free(p)


def expect_error(fn, err):
    with pytest.raises(acu.ArrowError) as g:
        fn()
    assert (g.value.status, g.value.message, g.value.index) == (err.status, err.message, err.index)


def check_filter_abi(gpu, kind, offsets, pred, size=0, n_rows=0, valid=None, what=""):
    """The list's new offsets and validity, and the child plan row for row, against the reference."""
    owned = []
    try:
        child_end = int(offsets[-1]) if offsets is not None else n_rows * size
        desc = list_desc(gpu, owned, kind, offsets, size, n_rows, valid, 3, child_len=child_end)
        offs, nulls, (plen, pcount, strat), sel = abi_filter(gpu, desc, pred)
    finally:
        for p in owned:
            gpu.free(p)
    mask = oft.filter_mask(pred)
    cpred, new = ref_filter(offsets, size, mask)
    exp_sel = np.flatnonzero(cpred)
    exp_len = int(offsets[len(mask)]) if offsets is not None else len(mask) * size
    assert len(cpred) == exp_len
    assert (plen, pcount, strat) == (exp_len, len(exp_sel), ref_strategy(len(exp_sel), exp_len)), what
    assert np.array_equal(sel.astype(np.int64), exp_sel), what
    if offsets is not None:
        assert offs.dtype == new.dtype and np.array_equal(offs, new), what
    lv = np.ones(len(mask), bool) if valid is None else np.asarray(valid, bool)[:len(mask)]
    assert np.array_equal(lv[mask], np.ones(int(mask.sum()), bool) if nulls is None else nulls), what
    return cpred


def check_take_abi(gpu, kind, offsets, idx, cdt, valid=None, child_len=None, check_bounds=False, what=""):
    """A List / LargeList take's offsets, validity and row map against the reference; returns the reference offsets."""
    owned = []
    vals, iv = idx.value_array(), (idx.valid_mask() if idx.validity is not None else None)
    new, lens, src, err = ref_take_list(offsets, valid, vals, iv, idx.dtype, check_bounds)
    try:
        desc = list_desc(gpu, owned, kind, offsets, valid=valid, valid_off=5,
                         child_len=int(offsets[-1]) if child_len is None else child_len)
        if err is not None:
            expect_error(lambda: abi_take(gpu, desc, idx, cdt, check_bounds), err)
            return None
        res = abi_take(gpu, desc, idx, cdt, check_bounds)
    finally:
        for p in owned:
            gpu.free(p)
    assert res["rows"] == int(new[-1]), what
    assert np.array_equal(res["offsets"].astype(np.int64), new), what
    exp_map = ref_list_map(new, lens, src, np.uint32 if cdt == abi.U32 else np.uint64)
    assert res["map"].dtype == exp_map.dtype and np.array_equal(res["map"], exp_map), what
    assert res["map_valid"] is None
    lv = np.ones(len(offsets) - 1, bool) if valid is None else np.asarray(valid, bool)
    ix = to_index(vals, idx.dtype).astype(np.int64)
    exp_nulls = (np.ones(len(vals), bool) if iv is None else iv) & lv[np.where(ix < len(lv), ix, 0)]
    assert np.array_equal(exp_nulls, np.ones(len(vals), bool) if res["nulls"] is None else res["nulls"]), what
    return new


# ---- 2a. k_list_expand ---------------------------------------------------------------------------------------------------
def offsets_from(lens, base, dtype):
    return np.concatenate([[base], base + np.cumsum(np.asarray(lens, np.int64))]).astype(dtype)


def expand_layout(rng, base):
    """Row lengths from `base`: rows of 63 / 64 / 65 / 127 / 128 / 1000 starting and ending on words, a word of 64
    one-row hops, runs of 1 / 2 / 1000 empty rows inside words and on word boundaries, then random short rows."""
    lens, pos = [], base

    def add(ln):
        nonlocal pos
        lens.append(ln)
        pos += ln

    def to_word():
        if pos % 64:
            add(64 - pos % 64)

    to_word()
    for ln in (63, 1, 64, 65, 63, 127, 1, 128, 1000, 24):  # 63 / 65 / 127 end mid-word, 64 / 128 start and end on words
        add(ln)
    to_word()
    for _ in range(64):  # one word of 64 hops
        add(1)
    for run in (1, 2, 1000):
        add(17)
        for _ in range(run):  # a run of empty rows at child row 64 w + 17 (mid-word) ...
            add(0)
        add(47)
        for _ in range(run):  # ... and on a word boundary
            add(0)
        add(30)
        to_word()
    for ln in rng.integers(0, 9, 3000):
        add(int(ln))
    return lens


def end_on(lens, base, child_end_mod, rng):
    """Trailing rows so that child_end = 64 k + child_end_mod (child_end_mod in -1, 0, 1)."""
    lens = list(lens)
    pos = base + sum(lens)
    target = (pos // 64 + 2) * 64 + child_end_mod
    lens += [int(x) for x in rng.multinomial(target - pos, np.ones(5) / 5)]
    return lens


def expand_placements(offsets):
    """The facts the layout promises, from the offsets themselves."""
    o = np.asarray(offsets, np.int64)
    lens = np.diff(o)
    starts = o[:-1]
    for ln in (63, 64, 65, 127, 128, 1000):
        assert ((lens == ln) & (starts % 64 == 0)).any() or ((lens == ln) & ((starts + lens) % 64 == 0)).any(), ln
    one = np.flatnonzero((lens == 1) & (starts % 64 == 0))
    assert any((lens[k:k + 64] == 1).all() for k in one)  # a whole word of one-row hops
    empty = lens == 0
    for run, mid in ((1, True), (2, True), (1000, True), (1000, False)):
        ok = False
        for k in np.flatnonzero(empty[:-run] if run < len(empty) else empty):
            if empty[k:k + run].all() and (starts[k] % 64 != 0) == mid and (k == 0 or not empty[k - 1]):
                ok = True
                break
        assert ok, (run, mid)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [abi.LIST, abi.LARGE_LIST])
@pytest.mark.parametrize("base", [0, 1, 63, 64, 65])
def test_expand_placements(gpu, kind, base):
    """Rows on, across and inside 64-bit child words, `base` at 0 / 1 / 63 / 64 / 65, child_end on a word boundary and
    one off it either way; alternating, all-selected, random (with null slots) and short predicates."""
    rng = np.random.default_rng(100 + base + kind)
    dtype = np.int64 if kind == abi.LARGE_LIST else np.int32
    layout = expand_layout(rng, base)
    for d in (-1, 0, 1):
        lens = end_on(layout, base, d, rng)
        offs = offsets_from(lens, base, dtype)
        expand_placements(offs)
        assert int(offs[0]) == base and int(offs[-1]) % 64 == d % 64
        n = len(lens)
        valid = rng.random(n) >= 0.1
        preds = [HostArray.bool_from_numpy(np.arange(n) % 2 == 0), HostArray.bool_from_numpy(np.ones(n, bool)),
                 HostArray.bool_from_numpy(rng.random(n) < 0.5, rng.random(n) >= 0.1),
                 HostArray.bool_from_numpy(rng.random(n - 7) < 0.9)]
        for k, pred in enumerate(preds):
            check_filter_abi(gpu, kind, offs, pred, valid=valid if k % 2 else None, what=f"base={base} end{d:+d} pred {k}")


@pytest.mark.gpu
@pytest.mark.parametrize("size", FSL_SIZES)
def test_expand_fixed_size(gpu, size):
    """FixedSizeList rows of 1 .. 4097 children: a row spanning many words, rows ending mid-word and on words."""
    rng = np.random.default_rng(size)
    n = max(2000 // size, 40)
    ends = np.arange(1, n + 1) * size
    if size % 64:
        assert (ends % 64 != 0).any()
    for pred in (HostArray.bool_from_numpy(np.arange(n) % 2 == 1), HostArray.bool_from_numpy(np.ones(n, bool)),
                 HostArray.bool_from_numpy(rng.random(n) < 0.5, rng.random(n) >= 0.2), HostArray.bool_from_numpy(rng.random(n - 3) < 0.5)):
        check_filter_abi(gpu, abi.FIXED_SIZE_LIST, None, pred, size=size, n_rows=n, valid=rng.random(n) >= 0.2, what=f"size={size}")


@pytest.mark.gpu
@pytest.mark.parametrize("kind", [abi.LIST, abi.LARGE_LIST, abi.FIXED_SIZE_LIST])
def test_expand_rounds(gpu, kind):
    """2.5 grid rounds of child words, a random and an all-selected plan, every child row compared."""
    sms = gpu.lib.acu_device_sm_count(gpu.h)
    words = int(2.5 * round_words(sms)) + 77
    rng = np.random.default_rng(7 + kind)
    if kind == abi.FIXED_SIZE_LIST:
        size = 768
        n = words * 64 // size + 1
        offs = None
    else:
        size = 0
        lens = rng.integers(0, 120, words * 64 // 35)
        lens[rng.random(len(lens)) < 0.3] = 0
        offs = offsets_from(lens, 33, np.int64 if kind == abi.LARGE_LIST else np.int32)
        n = len(lens)
    child_end = int(offs[-1]) if offs is not None else n * size
    assert (child_end + 63) // 64 >= 2.5 * round_words(sms)
    for pred in (HostArray.bool_from_numpy(rng.random(n) < 0.5), HostArray.bool_from_numpy(np.ones(n, bool))):
        check_filter_abi(gpu, kind, offs, pred, size=size, n_rows=n, what="rounds")


# ---- 2b. k_list_row_map --------------------------------------------------------------------------------------------------
def row_map_case(rng, leading=5):
    """Output rows (as source row lengths in output order) whose ends fall on lane 31 / 32 / 33 and span 511 / 512 / 513
    positions, rows longer than a span, leading empty rows and runs of empty rows of three kinds.
    Returns (source lens, source validity, index values, index validity)."""
    out = []  # (length, kind) in output order; kind: "row", "null_index", "null_list", "zero"
    pos = 0
    for _ in range(leading):
        out.append((0, ["null_index", "null_list", "zero"][_ % 3]))
    for rep in range(3):
        for t in (31, 32, 33, 511, 512, 513):
            ln = (t - pos) % SPAN or SPAN
            ln += SPAN * int(rng.integers(0, 3)) if rep else 0
            out.append((ln, "row"))
            pos += ln
            for k in range(int(rng.integers(0, 4))):
                out.append((0, ["null_index", "null_list", "zero"][k % 3]))
        ln = 3 * SPAN + int(rng.integers(1, SPAN))  # longer than a span
        out.append((ln, "row"))
        pos += ln
        for _ in range(40):
            ln = int(rng.integers(1, 40))
            out.append((ln, "row"))
            pos += ln
    # source rows: one per distinct length (so indices repeat), created in reverse (so indices descend), plus a null
    # list row over a non-empty range and a zero-length row
    lengths = sorted({ln for ln, k in out if k == "row"}, reverse=True)
    src_lens = lengths + [9, 0]
    row_of = {ln: k for k, ln in enumerate(lengths)}
    null_row, zero_row = len(lengths), len(lengths) + 1
    src_valid = np.ones(len(src_lens), bool)
    src_valid[null_row] = False
    vals, ivalid = [], []
    for ln, k in out:
        vals.append(row_of[ln] if k == "row" else null_row if k == "null_list" else zero_row if k == "zero" else 1 << 30)
        ivalid.append(k != "null_index")
    return src_lens, src_valid, np.array(vals, np.int64), np.array(ivalid)


def row_map_placements(new, vals, ivalid, src_valid, src_lens):
    new = np.asarray(new, np.int64)
    lens = np.diff(new)
    ends = new[1:][lens > 0]
    assert {31, 32, 33, SPAN - 1, 0, 1} <= set((ends % SPAN).tolist())
    assert (lens > SPAN).any() and (lens[:3] == 0).all()
    iv = np.asarray(ivalid)
    srcl = np.asarray(src_lens)
    kinds = set()
    for j in np.flatnonzero(lens == 0):
        kinds.add("null_index" if not iv[j] else "null_list" if not src_valid[vals[j]] else "zero" if srcl[vals[j]] == 0 else "?")
    assert kinds == {"null_index", "null_list", "zero"}
    v = vals[iv]
    assert (np.diff(v) < 0).any() and len(np.unique(v)) < len(v)  # descending and repeated


ROW_MAP_CASES = [  # (kind, map dtype, base: the first source row's child row, or "umax": the last row ends at UINT32_MAX)
    (abi.LIST, abi.U32, 5), (abi.LIST, abi.U64, 5), (abi.LARGE_LIST, abi.U32, 0), (abi.LARGE_LIST, abi.U32, "umax"),
    (abi.LARGE_LIST, abi.U64, 2**32 - 2000), (abi.LARGE_LIST, abi.U64, 2**40 - 3), (abi.LARGE_LIST, abi.U64, 2**40 + 2**33 + 7),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kind,cdt,base", ROW_MAP_CASES, ids=lambda v: str(v))
def test_row_map_placements(gpu, kind, cdt, base):
    """Lane and span boundaries, long rows, empty rows from three sources, repeated and descending indices; LargeList
    rows straddling 2^32 and near 2^40 through the UInt64 map, and the UInt32 map up to child row UINT32_MAX."""
    rng = np.random.default_rng(ROW_MAP_CASES.index((kind, cdt, base)))
    src_lens, src_valid, vals, ivalid = row_map_case(rng)
    umax = base == "umax"
    if umax:
        base = U32_MAX - int(np.sum(src_lens))
    offs = offsets_from(src_lens, base, np.int64 if kind == abi.LARGE_LIST else np.int32)
    if umax:
        assert int(offs[-1]) == U32_MAX
    if cdt == abi.U64 and base > 2**32:
        assert int(offs[0]) > 2**32
    elif cdt == abi.U64 and kind == abi.LARGE_LIST:
        assert int(offs[0]) < 2**32 < int(offs[-1])
    for dtype in (abi.U32, abi.I64, abi.I16):
        idx = HostArray.from_numpy(dtype, vals.astype(acu.NP_DTYPES[dtype]) if dtype != abi.I16 else np.where(ivalid, vals, -3), ivalid, 3)
        new = check_take_abi(gpu, kind, offs, idx, cdt, valid=src_valid, child_len=int(offs[-1]) + 100 * (cdt == abi.U64),
                             what=f"dtype={dtype}")
        row_map_placements(new, vals, ivalid, src_valid, src_lens)


@pytest.mark.gpu
def test_row_map_u32_limit(gpu):
    """child_len = UINT32_MAX is accepted for the UInt32 map; UINT32_MAX + 1 is refused with its message."""
    offs = np.array([U32_MAX - 70, U32_MAX - 3, U32_MAX], np.int64)
    idx = HostArray.from_numpy(abi.U32, np.array([1, 0, 1], np.uint32))
    check_take_abi(gpu, abi.LARGE_LIST, offs, idx, abi.U32, child_len=U32_MAX)
    err = oft.OracleError(abi.ERR_INVALID_ARGUMENT, f"child of {U32_MAX + 1} rows needs a UInt64 row map")
    for kind, o in ((abi.LARGE_LIST, offs), (abi.LIST, np.array([0, 5, 9], np.int32))):
        owned = []
        try:
            desc = list_desc(gpu, owned, kind, o, child_len=U32_MAX + 1)
            expect_error(lambda: abi_take(gpu, desc, idx, abi.U32), err)
            assert abi_take(gpu, desc, idx, abi.U64)["rows"] > 0
        finally:
            for p in owned:
                gpu.free(p)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,cdt", [(abi.LIST, abi.U32), (abi.LARGE_LIST, abi.U64)])
def test_row_map_rounds(gpu, kind, cdt):
    """2.5 rounds of k_list_row_map with output rows ending exactly on the round boundaries, and (List) more than 2.5
    rounds of k_narrow_offsets over the m + 1 offsets."""
    sms = gpu.lib.acu_device_sm_count(gpu.h)
    rnd = round_rows(sms)
    rng = np.random.default_rng(11 + kind)
    m_min = int(2.5 * round_words(sms)) + 5
    mean = int(3 * rnd) // m_min + 1
    src_lens = rng.integers(0, 2 * mean, 4000)
    src_lens[:3] = [rnd, 0, 1]
    src_valid = rng.random(4000) >= 0.05
    src_valid[:3] = True
    vals = rng.integers(3, 4000, m_min + 1000)
    ivalid = rng.random(len(vals)) >= 0.02
    # the output row ending at round 1 / round 2: pad with single-child rows up to the boundary
    lens = np.where(ivalid & src_valid[vals], src_lens[vals], 0)
    ends = np.cumsum(lens)
    for r in (1, 2):
        j = int(np.searchsorted(ends, r * rnd - 1000))
        short = r * rnd - int(ends[j])
        assert short > 0
        vals = np.concatenate([vals[:j + 1], np.full(short, 2), vals[j + 1:]])
        ivalid = np.concatenate([ivalid[:j + 1], np.ones(short, bool), ivalid[j + 1:]])
        lens = np.where(ivalid & src_valid[vals], src_lens[vals], 0)
        ends = np.cumsum(lens)
    vals[-7] = 0  # one row of a whole round
    offs = offsets_from(src_lens, 11, np.int64 if kind == abi.LARGE_LIST else np.int32)
    idx = HostArray.from_numpy(abi.U32, vals, ivalid, 1)
    new = check_take_abi(gpu, kind, offs, idx, cdt, valid=src_valid, what="rounds")
    assert new[-1] >= 2.5 * rnd and {rnd, 2 * rnd} <= set(new.tolist())
    assert len(new) >= 2.5 * round_words(sms)


# ---- 2c. k_fsl_row_map ----------------------------------------------------------------------------------------------------
def fsl_nulls(size, m, rng):
    """Index validity with nulls at the rows holding the first and the last child row of some 64-bit words, and inside
    a row that covers a whole word."""
    valid = rng.random(m) >= 0.1
    for w in (1, 3, (m * size) // 64 - 1):
        if w * 64 + 63 < m * size:
            valid[(w * 64) // size] = False
            valid[(w * 64 + 63) // size] = False
    return valid


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", INDEX_DTYPES)
def test_fsl_row_map(gpu, dtype):
    """Sizes 1 .. 4097 at index validity offsets 0 / 1 / 7 / 63, index * size wrapping past 2^32, a last partial word."""
    rng = np.random.default_rng(int(dtype) + 50)
    info = np.iinfo(acu.NP_DTYPES[dtype])
    wrapped, partial = 0, 0
    for size in FSL_SIZES:
        m = max(3000 // size, 9) + 3
        for voff in (0, 1, 7, 63):
            vals = rng.integers(max(int(info.min), -2**40), min(int(info.max), 2**40) + 1, m).astype(acu.NP_DTYPES[dtype])
            valid = fsl_nulls(size, m, rng)
            total = m * size
            if size >= 64:
                full = [i for i in range(m) if (-(i * size) % 64) + 64 <= size]  # a row covering a whole word
                valid[full[len(full) // 2]] = False
            partial += total % 64 != 0
            idx = HostArray.from_numpy(dtype, vals, valid, voff)
            exp, vm, nc = ref_fsl_map(vals, valid, dtype, size)
            wrapped += int((((to_index(vals, dtype) & np.uint64(U32_MAX)) * np.uint64(size)) >> np.uint64(32) > 0).sum())
            owned = []
            try:
                desc = list_desc(gpu, owned, abi.FIXED_SIZE_LIST, size=size, n_rows=5000)
                res = abi_take(gpu, desc, idx, abi.U32)
            finally:
                for p in owned:
                    gpu.free(p)
            what = f"size={size} voff={voff}"
            assert res["rows"] == total and res["offsets"] is None, what
            assert np.array_equal(res["map"], exp), what
            assert np.array_equal(res["map_valid"], vm) and res["map_nulls"] == nc, what
            assert np.array_equal(res["nulls"], valid), what
    assert partial > 0
    if dtype not in (abi.U8, abi.U16):
        assert wrapped > 100


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 768])
def test_fsl_rounds(gpu, size):
    """More than one round of the map loop (one child row per thread) and of the validity loop (one word per thread)."""
    sms = gpu.lib.acu_device_sm_count(gpu.h)
    total_min = int(1.3 * round_words(sms) * 64) if size == 768 else int(2.5 * round_words(sms))
    m = total_min // size + 5
    rng = np.random.default_rng(size)
    vals = rng.integers(0, 2**32, m, dtype=np.uint64).astype(np.uint32)
    valid = rng.random(m) >= 0.1
    idx = HostArray.from_numpy(abi.U32, vals, valid, 1)
    exp, vm, nc = ref_fsl_map(vals, valid, abi.U32, size)
    assert m * size > total_min >= round_words(sms)
    owned = []
    try:
        desc = list_desc(gpu, owned, abi.FIXED_SIZE_LIST, size=size, n_rows=10)
        res = abi_take(gpu, desc, idx, abi.U32)
    finally:
        for p in owned:
            gpu.free(p)
    assert np.array_equal(res["map"], exp)
    assert np.array_equal(res["map_valid"], vm) and res["map_nulls"] == nc


# ---- 2d. the offsets engine: INT32_MAX, error rows across blocks ------------------------------------------------------------
BIG = 1 << 20
ENGINE_SRC = np.array([0, BIG, 2 * BIG - 1, 2 * BIG], np.int32)  # rows of 2^20, 2^20 - 1 and 1 child rows (no child)


def spread(m, picks):
    """m index rows over ENGINE_SRC: the rows in `picks` (row -> source row), every other row a null index."""
    vals = np.full(m, 2, np.int64)
    valid = np.zeros(m, bool)
    for j, r in picks.items():
        vals[j], valid[j] = r, True
    return vals, valid


@pytest.mark.gpu
def test_engine_int32_max(gpu):
    """2047 rows of 2^20 and one of 2^20 - 1 children spread over 20 engine blocks end at exactly INT32_MAX: accepted,
    last offset INT32_MAX. One child row more fails at the row that passes it. Sizing calls only (no map)."""
    rng = np.random.default_rng(31)
    m = 20 * BY_ROWS + 17
    rows = np.sort(rng.choice(m - 100, 2048, replace=False))
    picks = {int(j): 0 for j in rows}
    picks[int(rows[1000])] = 1
    vals, valid = spread(m, picks)
    assert len({j // BY_ROWS for j in rows}) >= 15
    for dtype in (abi.U32, abi.I64):
        idx = HostArray.from_numpy(dtype, vals, valid)
        new, _, _, err = ref_take_list(ENGINE_SRC, None, vals, valid, dtype)
        assert err is None and int(new[-1]) == I32_MAX
        owned = []
        try:
            desc = list_desc(gpu, owned, abi.LIST, ENGINE_SRC, child_len=2 * BIG)
            res = abi_take(gpu, desc, idx, abi.U32, write_map=False)
            assert res["rows"] == I32_MAX and int(res["offsets"][-1]) == I32_MAX
            assert np.array_equal(res["offsets"].astype(np.int64), new)
            # one more child row: row 2 (one child) after the last big row
            extra = int(rows[-1]) + 1 + int(rng.integers(0, m - int(rows[-1]) - 1))
            v2, ok2 = vals.copy(), valid.copy()
            v2[extra], ok2[extra] = 2, True
            _, _, _, err = ref_take_list(ENGINE_SRC, None, v2, ok2, dtype)
            assert err.message == oft.UNWRAP_NONE and err.index == extra
            expect_error(lambda: abi_take(gpu, desc, HostArray.from_numpy(dtype, v2, ok2), abi.U32, write_map=False), err)
        finally:
            for p in owned:
                gpu.free(p)


@pytest.mark.gpu
@pytest.mark.parametrize("check_bounds", [False, True])
def test_engine_error_rows(gpu, check_bounds):
    """Out-of-bounds and i32-overflow rows in different engine blocks, far apart (past 4096 blocks) and close, in both
    orders; several out-of-bounds rows (the lowest is reported); out-of-bounds values under null indices (ignored)."""
    rng = np.random.default_rng(41 + check_bounds)
    far = 4100 * BY_ROWS
    m = far + 3 * BY_ROWS
    owned = []
    try:
        desc = list_desc(gpu, owned, abi.LIST, ENGINE_SRC, child_len=2 * BIG)
        cases = []
        for oob_at, ovf_at in ((5 * BY_ROWS + 3, far + 100), (far + 100, 5 * BY_ROWS + 3), (BY_ROWS - 1, BY_ROWS), (BY_ROWS, BY_ROWS - 1)):
            cases.append((oob_at, ovf_at))
        for oob_at, ovf_at in cases:
            # 2048 rows of 2^20 end at 2^31 > INT32_MAX: place the 2048th at ovf_at, the rest before it
            before = np.sort(rng.choice(min(ovf_at, m), 2047, replace=False))
            picks = {int(j): 0 for j in before if j != oob_at}
            while len(picks) < 2047:
                j = int(rng.integers(0, ovf_at))
                if j != oob_at:
                    picks[j] = 0
            picks[ovf_at] = 0
            vals, valid = spread(m, picks)
            vals[oob_at], valid[oob_at] = 3 + 7 * (oob_at % 2), True  # 3 is the list length (an index of len)
            later = oob_at + BY_ROWS * 3 + 1
            if later < m and later not in picks:
                vals[later], valid[later] = 1 << 30, True  # a second, later out-of-bounds row
            nul = np.flatnonzero(~valid)[:50]
            vals[nul] = 1 << 31  # out of bounds under null indices
            for dtype in (abi.U32, abi.U64):
                idx = HostArray.from_numpy(dtype, vals, valid)
                _, _, _, err = ref_take_list(ENGINE_SRC, None, vals, valid, dtype, check_bounds)
                first = oob_at if check_bounds else min(oob_at, ovf_at)
                assert err is not None and err.index == first
                assert (err.message == oft.UNWRAP_NONE) == (ovf_at < oob_at and not check_bounds)
                expect_error(lambda: abi_take(gpu, desc, idx, abi.U32, check_bounds, write_map=False), err)
    finally:
        for p in owned:
            gpu.free(p)


# ---- 3. end to end through Context.filter_list / take_list ----------------------------------------------------------------
def assert_flat(got, values, valid, what):
    assert got.length == len(values), what
    gv = got.valid_mask()
    assert np.array_equal(gv, valid), what
    assert np.array_equal(np.asarray(got.value_array())[valid].view(np.uint8), np.asarray(values)[valid].view(np.uint8)), what


@pytest.mark.gpu
def test_e2e_fsl_float32_768(gpu):
    """FixedSizeList<Float32, 768>: a take past one round of the map's validity walk and a filter, whole child."""
    sms = gpu.lib.acu_device_sm_count(gpu.h)
    size, n = 768, 3000
    rng = np.random.default_rng(768)
    cvals = rng.standard_normal(n * size).astype(np.float32)
    cvalid = rng.random(n * size) >= 0.01
    col = FixedSizeListColumn(size, HostArray.from_numpy(abi.F32, cvals, cvalid), nulls_of(rng.random(n) >= 0.1, 2))
    m = int(1.2 * round_words(sms) * 64) // size + 11
    vals = rng.integers(0, n, m)
    ivalid = rng.random(m) >= 0.1
    got = gpu.take_list(col, HostArray.from_numpy(abi.U32, vals, ivalid, 3))
    mp, vm, _ = ref_fsl_map(vals, ivalid, abi.U32, size)
    assert len(mp) > round_words(sms) * 64
    assert_flat(got.child, cvals[mp], vm & cvalid[mp], "take child")
    assert np.array_equal(got.nulls.valid_mask(), ivalid & col.nulls.valid_mask()[vals])
    pred = HostArray.bool_from_numpy(rng.random(n) < 0.6)
    got = gpu.filter_list(col, pred)
    cpred, _ = ref_filter(None, size, oft.filter_mask(pred))
    assert_flat(got.child, cvals[cpred], cvalid[cpred], "filter child")


@pytest.mark.gpu
def test_e2e_list_int64_take(gpu):
    """List<Int64>: a take of 2.5 row-map rounds of child rows, every child row compared."""
    sms = gpu.lib.acu_device_sm_count(gpu.h)
    rng = np.random.default_rng(64)
    n_src = 20000
    lens = rng.integers(0, 40, n_src)
    offs = offsets_from(lens, 3, np.int32)
    cn = int(offs[-1]) + 2
    cvals = rng.integers(-2**62, 2**62, cn)
    cvalid = rng.random(cn) >= 0.02
    col = ListColumn(offs, HostArray.from_numpy(abi.I64, cvals, cvalid), nulls_of(rng.random(n_src) >= 0.05, 1))
    m = 3 * round_rows(sms) // 17
    vals = rng.integers(0, n_src, m)
    ivalid = rng.random(m) >= 0.05
    got = gpu.take_list(col, HostArray.from_numpy(abi.I64, vals, ivalid))
    new, ln, src, err = ref_take_list(offs, col.nulls.valid_mask(), vals, ivalid, abi.I64)
    assert err is None and new[-1] >= 2.5 * round_rows(sms)
    assert np.array_equal(got.offsets.astype(np.int64), new)
    mp = ref_list_map(new, ln, src, np.int64)
    assert_flat(got.child, cvals[mp], cvalid[mp], "child")


@pytest.mark.gpu
def test_e2e_large_list_utf8_filter(gpu):
    """LargeList<Utf8>: a filter past 2 rounds of k_list_expand's child words, the whole Utf8 child compared."""
    sms = gpu.lib.acu_device_sm_count(gpu.h)
    rng = np.random.default_rng(8)
    n_child = int(2.4 * round_words(sms) * 64) + 333
    slens = rng.integers(0, 4, n_child)
    soffs = np.concatenate([[0], np.cumsum(slens)]).astype(np.int32)
    data = rng.integers(97, 123, int(soffs[-1]) + 1).astype(np.uint8)
    svalid = rng.random(n_child) >= 0.05
    child = Utf8Column(soffs, data, nulls_of(svalid))
    lens = rng.integers(0, 46, n_child // 25)
    offs = offsets_from(lens, 5, np.int64)
    assert offs[-1] <= n_child and (int(offs[-1]) + 63) // 64 > 2 * round_words(sms)
    col = ListColumn(offs, child, nulls_of(rng.random(len(lens)) >= 0.1))
    pred = HostArray.bool_from_numpy(rng.random(len(lens)) < 0.5, rng.random(len(lens)) >= 0.05)
    got = gpu.filter_list(col, pred)
    cpred, new = ref_filter(offs, 0, oft.filter_mask(pred))
    assert np.array_equal(got.offsets, new)
    rows = np.flatnonzero(cpred)
    rl = slens[rows]
    exp_off = np.concatenate([[0], np.cumsum(rl)])
    assert np.array_equal(got.child.offsets.astype(np.int64), exp_off)
    pos = np.repeat(soffs[rows].astype(np.int64) - exp_off[:-1], rl) + np.arange(int(exp_off[-1]))
    assert np.array_equal(got.child.data[:int(exp_off[-1])], data[pos])
    assert np.array_equal(got.child.nulls.valid_mask(), svalid[rows])


# ---- 4. NullBuffer presence where the child plan is All and the parent's is not ----------------------------------------------
def presence_cases():
    """(name, list, predicate): the unselected rows are empty and offsets[0] == 0, so the child plan selects all of
    [0, child_end) while the parent plan does not. Children: a NullBuffer without nulls, and nulls only past child_end."""
    forced = HostArray.from_list(abi.I32, list(range(12)), force_validity=True)
    tail = HostArray.from_list(abi.I32, list(range(12)) + [None, 5, None])
    lens = [2, 0, 3, 0, 0, 4, 1, 0, 2]
    sel = np.array([1, 0, 1, 1, 0, 1, 1, 0, 1], bool)
    pred = HostArray.bool_from_numpy(sel)
    for name, child in (("forced", forced), ("nulls past child_end", tail)):
        yield f"List<Int32> {name}", ListColumn(offsets_from(lens, 0, np.int32), child, nulls_of(np.ones(len(lens), bool))), pred
        # nested: the inner list's plan is All too, and so is its child's
        inner = ListColumn(offsets_from([3, 0, 4, 5], 0, np.int64), child, nulls_of(np.ones(4, bool), force=True))
        yield f"List<LargeList<Int32>> {name}", ListColumn(offsets_from([1, 0, 2, 0, 1], 0, np.int32), inner,
                                                            nulls_of(np.ones(5, bool))), HostArray.bool_from_numpy(np.array([1, 0, 1, 0, 1], bool))
        fsl = FixedSizeListColumn(2, child, nulls_of(np.ones(6, bool), force=True))
        yield f"List<FixedSizeList<Int32, 2>> {name}", ListColumn(offsets_from([2, 0, 4], 0, np.int32), fsl,
                                                                   nulls_of(np.ones(3, bool))), HostArray.bool_from_numpy(np.array([1, 0, 1], bool))


def levels_present(col):
    """NullBuffer presence of every level below the top."""
    out = []
    while isinstance(col, (ListColumn, FixedSizeListColumn)):
        col = col.child
        out.append((col if isinstance(col, HostArray) else col.nulls).validity is not None)
    return out


def test_presence_oracle():
    """The reference's rule (arrow-select/src/filter.rs:600: a filter that is not All goes through MutableArrayData;
    arrow-data/src/transform/mod.rs:936: freeze keeps a NullBuffer only if it has a null): no level below a list
    filtered that way keeps a NullBuffer without nulls, even where its own plan selects every row. A top-level All
    slices, and every level keeps its NullBuffer."""
    for name, col, pred in presence_cases():
        mask = oft.filter_mask(pred)
        cpred, _ = ref_filter(col.offsets, 0, mask)
        assert cpred.all() and not mask.all(), name
        assert levels_present(oft.filter(col, mask)) == [False] * len(levels_present(col)), name
        all_pred = np.ones(col.length, bool)
        assert levels_present(oft.filter(col, all_pred)) == levels_present(col) == [True] * len(levels_present(col)), name


@pytest.mark.gpu
def test_presence_filter(gpu):
    """The device follows the same rule at every level (and keeps every NullBuffer under a top-level All)."""
    for name, col, pred in presence_cases():
        got = gpu.filter_list(col, pred)
        assert oft.describe(got) == oft.describe(oft.filter(col, oft.filter_mask(pred))), name
        assert levels_present(got) == [False] * len(levels_present(col)), name
        got = gpu.filter_list(col, HostArray.bool_from_numpy(np.ones(col.length, bool)))
        assert levels_present(got) == [True] * len(levels_present(col)), name


@pytest.mark.gpu
def test_presence_take(gpu):
    """take_list's child step (take.rs:663: MutableArrayData with use_nulls = child null_count > 0, then freeze): a child
    without nulls in the taken ranges gets no NullBuffer, for both kinds of child, one level down and two."""
    for name, col, _ in presence_cases():
        idx = HostArray.from_numpy(abi.U32, np.arange(col.length)[::-1].copy())
        got = gpu.take_list(col, idx)
        assert oft.describe(got) == oft.describe(oft.take_host(col, idx)), name
        assert levels_present(got) == [False] * len(levels_present(col)), name
