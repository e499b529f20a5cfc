"""filter, take, zip, the byte gathers and the reductions on zero-copy device slices, against the oracle on the same logical
slice, bit for bit (values including the bytes under null slots, validity bits, null_count, NullBuffer presence, error
status / text / index).

`Array::slice` moves the values pointer by offset * width, and every producer of device columns passes such pointers on
(acu_import_column, the IPC reader's views into one body, the C++ mirror's slices). Several launchers pick another kernel
or another staging path when a buffer is not 16-byte aligned: filter (8-, 4- or 1-byte loads instead of cp.async in
k_filter_fused, also below 4 % selectivity, where aligned values take k_filter_values_async), take (per-lane index staging instead of cp.async.bulk), the Utf8 gathers with
32-bit indices (the generic kernels instead of FAST / k_dict_*) and zip (k_zip_elem instead of k_zip). `Context.upload`
re-aligns every column, so the tests here build the shifted descriptors themselves, and every helper asserts that the
pointer it produces is not 16-byte aligned. Shifts are whole elements at the element's natural alignment.

The multi-round sizes are derived from the SM count: no launch here has more than 8 waves x SMs x 64 resident warps, so
a size above that many work units (1024-row filter tiles, 256-index take tiles, 2048-row reduce super-groups; for zip
32 x SMs CTAs of 256 threads) runs every kernel through at least two grid-stride rounds.

Float sums are compared exactly: integer-valued inputs with sum |x| < 2^24 (Float32) or 2^53 (Float64) make every partial
sum exactly representable, so any association order gives Python's exact integer sum."""
import ctypes as C
import types

import numpy as np
import pytest

import acu
from acu import _abi as abi
from acu import BOOL, HostArray, Utf8Column, bitmap_bytes
from test_gpu_elementwise_shapes import PAD, Column, call_out, same, same_or_same_error
from test_gpu_parity import SIZES, rand_bool, rand_values
from test_gpu_recordbatch import check_columns, oracle_filter, oracle_take

pytestmark = pytest.mark.gpu

NP = acu.NP_DTYPES
INDEX_DTYPES = [abi.U8, abi.I8, abi.U16, abi.I16, abi.U32, abi.I32, abi.U64, abi.I64]
ALL_DTYPES = [abi.I8, abi.I16, abi.I32, abi.I64, abi.U8, abi.U16, abi.U32, abi.U64, abi.F32, abi.F64]


def unaligned_shifts(width):
    """Every whole-element shift that leaves a 16-byte aligned base unaligned: 1 .. 16 / width - 1."""
    return list(range(1, 16 // width))


def multi_round(gpu, unit):
    """About 1.2x the rows one launch of 8 waves x SMs x 64 warps covers in a single grid-stride round, one `unit` per warp."""
    return int(1.2 * 8 * gpu.lib.acu_device_sm_count(gpu.h) * 64 * unit)


def sparse_mask(rng, n, null_p):
    """A validity mask without a float temporary per row (the multi-round sizes reach 1e8 rows)."""
    return rng.integers(0, 1000, n, dtype=np.int16) >= int(null_p * 1000)


def at(col, shift, n, exact_count=False):
    """Rows [shift, shift + n) of an uploaded Column as (host slice, device descriptor); the descriptor's values pointer is
    `shift` elements into the allocation. exact_count gives both sides the cached null_count instead of -1."""
    _, d = col.at(shift)
    h = col.host.slice(shift, n)
    d.len = n
    if shift:
        assert d.values % 16 != 0, f"a shift of {shift} x {col.host.width()} bytes left the values 16-byte aligned"
    if exact_count and d.validity:
        d.null_count = h.null_count = int((~h.valid_mask()).sum())
    return h, d


def column(gpu, dtype, values, mask, shift, n, exact_count=False):
    """Upload `values` (>= shift + n + PAD rows) once and view rows [shift, shift + n)."""
    assert len(values) >= shift + n + PAD
    col = Column(gpu, dtype, values[: shift + n + PAD], None if mask is None else mask[: shift + n + PAD])
    return (col,) + at(col, shift, n, exact_count)


def index_column(gpu, rng, idx_dtype, m, n_values, shift, null_p, exact_count=True):
    raw = rng.integers(0, max(n_values, 1), shift + m + PAD).astype(NP[idx_dtype])
    mask = None if null_p is None else sparse_mask(rng, shift + m + PAD, null_p)
    return column(gpu, idx_dtype, raw, mask, shift, m, exact_count)


class SlicedUtf8:
    """A zero-copy Utf8 / LargeUtf8 slice: rows [k, k + n) of an uploaded column. The offsets pointer is moved by k entries
    (so offsets[0] != 0), the value bytes are shared and the validity offset is moved; `host` is the same slice."""

    def __init__(self, gpu, rng, n, k, odt, null_p, max_len=12):
        self.gpu, self.ob = gpu, np.dtype(odt).itemsize
        total = n + k
        lens = rng.integers(1 if k else 0, max_len + 1, total)
        offsets = np.zeros(total + 1, dtype=odt)
        offsets[1:] = np.cumsum(lens)
        data = rng.integers(97, 123, int(offsets[-1]) + 16).astype(np.uint8)
        mask = None if null_p is None else rng.random(total) >= null_p
        validity = None if mask is None else acu.pack_bits(mask, 3)
        full = HostArray(abi.U8, np.zeros(0, np.uint8), total, validity, 3 if mask is not None else 0, 0,
                         0 if mask is None else int(total - mask.sum()))
        nulls = full.slice(k, n) if k else full
        self.host = Utf8Column(offsets[k:], data, nulls)
        self.d_off_base, self.d_data = gpu.malloc(offsets.nbytes + 16), gpu.malloc(data.nbytes + 16)
        gpu.h2d(self.d_off_base, offsets)
        gpu.h2d(self.d_data, data)
        self.d_valid = None
        if validity is not None:
            self.d_valid = gpu.malloc(validity.nbytes + 8)
            gpu.h2d(self.d_valid, validity)
        self.d_off = self.d_off_base + k * self.ob
        if k:
            assert self.d_off % 16 != 0 and int(self.host.offsets[0]) != 0
        self.nulls = abi.Array()
        self.nulls.validity, self.nulls.validity_offset, self.nulls.len = self.d_valid, nulls.validity_offset, n
        self.nulls.null_count = int((~nulls.valid_mask()).sum()) if validity is not None else 0

    def column(self):
        c = abi.Column()
        c.kind, c.width, c.array, c.data = abi.COL_BYTES, self.ob, self.nulls, self.d_data
        c.array.values = self.d_off
        return c

    def free(self):
        for p in (self.d_off_base, self.d_data, self.d_valid):
            self.gpu.free(p)


def call_bytes(gpu, ob, rows, odt, fn):
    """Two-phase byte output of fn(out_offsets, out_data, capacity, total, out_nulls): size, then copy."""
    d_out_off = gpu.malloc((rows + 1) * ob + 16)
    out = gpu.alloc_out(0, rows)
    d_out_data = None
    try:
        total = C.c_int64(0)
        gpu.check(fn(d_out_off, None, 0, C.byref(total), C.byref(out)))
        d_out_data = gpu.malloc(total.value + 16)
        gpu.check(fn(d_out_off, d_out_data, total.value, C.byref(total), C.byref(out)))
        n = out.len
        validity = gpu.d2h(out.validity, bitmap_bytes(n)) if out.has_validity else None
        return (gpu.d2h(d_out_off, (n + 1) * ob, odt), gpu.d2h(d_out_data, total.value),
                HostArray(abi.U8, np.zeros(0, np.uint8), n, validity, 0, 0, out.null_count if out.has_validity else 0))
    finally:
        gpu._free_out(out)
        gpu.free(d_out_off)
        gpu.free(d_out_data)


def same_bytes(got, exp, what):
    (go, gd, gn), (eo, ed, en) = got, exp
    assert np.array_equal(go, eo), f"{what}: offsets differ"
    assert np.array_equal(gd, ed), f"{what}: bytes differ"
    assert (gn.validity is None) == (en.validity is None), f"{what}: NullBuffer presence differs"
    if en.validity is not None:
        assert gn.null_count == en.null_count, f"{what}: null_count {gn.null_count} != {en.null_count}"
        assert np.array_equal(gn.valid_mask(), en.valid_mask()), f"{what}: validity bits differ"


class Plan:
    def __init__(self, gpu, pred):
        self.gpu, self.dp = gpu, gpu.upload(pred)
        self.h = C.c_void_p()
        pd = self.dp.descriptor()
        gpu.check(gpu.lib.acu_filter_plan_create(gpu.h, C.byref(pd), C.byref(self.h)))
        self.count = gpu.lib.acu_filter_plan_count(self.h)

    def filter(self, dtype, vd):
        w = abi.DTYPE_SIZE[dtype]
        return call_out(self.gpu, self.count * w, self.count, dtype,
                        lambda out: self.gpu.lib.acu_filter_primitive(self.gpu.h, self.h, w, C.byref(vd), C.byref(out)))

    def filter_bytes(self, src):
        g = self.gpu
        return call_bytes(g, src.ob, self.count, src.host.offsets.dtype,
                          lambda oo, od, cap, tot, out: g.lib.acu_filter_bytes(g.h, self.h, src.ob, src.d_off, src.d_data, C.byref(src.nulls),
                                                                               oo, od, cap, tot, out))

    def free(self):
        self.gpu.lib.acu_filter_plan_destroy(self.gpu.h, self.h)
        self.dp.free()


def gpu_take(gpu, dtype, vd, idd, idx_dtype, check_bounds):
    m = idd.len
    w = abi.DTYPE_SIZE[dtype]
    return call_out(gpu, m * w, m, dtype,
                    lambda out: gpu.lib.acu_take_primitive(gpu.h, w, C.byref(vd), C.byref(idd), idx_dtype, int(check_bounds), C.byref(out)))


def gpu_take_bytes(gpu, src, idd, idx_dtype, check_bounds=False):
    return call_bytes(gpu, src.ob, idd.len, src.host.offsets.dtype,
                      lambda oo, od, cap, tot, out: gpu.lib.acu_take_bytes(gpu.h, src.ob, src.d_off, src.d_data, C.byref(src.nulls), C.byref(idd),
                                                                           idx_dtype, int(check_bounds), oo, od, cap, tot, out))


def bits_value(dtype, bits, cnt):
    if cnt == 0:
        return None
    return np.array([bits], dtype=np.uint64).view(np.uint8)[: abi.DTYPE_SIZE[dtype]].view(NP[dtype])[0].item()


def gpu_aggregate(gpu, dtype, op, d):
    bits, cnt = C.c_uint64(0), C.c_int64(0)
    gpu.check(gpu.lib.acu_aggregate(gpu.h, dtype, op, C.byref(d), C.byref(bits), C.byref(cnt)))
    return bits_value(dtype, bits.value, cnt.value)


def gpu_sum_checked(gpu, dtype, d):
    bits, cnt = C.c_uint64(0), C.c_int64(0)
    gpu.check(gpu.lib.acu_sum_checked(gpu.h, dtype, C.byref(d), C.byref(bits), C.byref(cnt)))
    return bits_value(dtype, bits.value, cnt.value)


def same_scalar(got, exp, what, nan_sign=False):
    """nan_sign: min / max order NaNs by totalOrder, so the sign of a NaN result is part of it (a sum's NaN sign is not)."""
    if isinstance(exp, float) and np.isnan(exp):
        assert isinstance(got, float) and np.isnan(got), f"{what}: {got} != NaN"
        assert not nan_sign or np.signbit(got) == np.signbit(exp), f"{what}: NaN sign differs"
    else:
        assert got == exp, f"{what}: {got} != {exp}"
        if isinstance(exp, float):
            assert np.signbit(got) == np.signbit(exp), f"{what}: sign of {got} != sign of {exp}"


def same_sum_checked(gpu, dtype, d, h, oracle, what):
    """The same value, or the same error status, text and failing row."""
    try:
        exp = oracle.sum_checked(h)
    except acu.ArrowError as e:
        with pytest.raises(acu.ArrowError) as gi:
            gpu_sum_checked(gpu, dtype, d)
        assert (gi.value.status, str(gi.value), gi.value.index) == (e.status, str(e), e.index), what
        return
    same_scalar(gpu_sum_checked(gpu, dtype, d), exp, what)


def launches(gpu, fn):
    fn()  # warm: first-use occupancy queries and a clean result block
    before = gpu.launch_count()
    fn()
    return gpu.launch_count() - before


# ---- 1. filter ----------------------------------------------------------------------------------------------------------
FILTER_LENGTHS = [1, 63, 64, 65, 1023, 1024, 1025, 4097, 70001]
SELECTIVITIES = [0.0, 0.01, 0.03, 0.1, 0.5, 0.9, 1.0]
VALIDITY = ["none", "5% nulls", "no nulls, cached 0", "5% nulls, count unknown"]


def validity_column(gpu, rng, dtype, n, shift, validity):
    m = shift + n + PAD
    values = rand_values(rng, dtype, m)
    mask = None if validity == "none" else (np.ones(m, dtype=bool) if validity.startswith("no nulls") else rng.random(m) >= 0.05)
    col, h, d = column(gpu, dtype, values, mask, shift, n, exact_count=validity != "5% nulls, count unknown")
    return col, h, d


@pytest.mark.parametrize("dtype", [abi.I8, abi.I16, abi.I32, abi.I64, abi.F64])
@pytest.mark.parametrize("true_p", SELECTIVITIES)
def test_filter_shifted_column(gpu, oracle, dtype, true_p):
    """k_filter_fused<W, false> with its 8-byte / 4-byte / byte loads, the validity compacted in the same pass or, below
    4 % selectivity, through k_compress_bits."""
    rng = np.random.default_rng(20_000 + dtype * 100 + int(true_p * 100))
    shifts = unaligned_shifts(abi.DTYPE_SIZE[dtype])
    k = 0
    for n in FILTER_LENGTHS:
        for validity in VALIDITY:
            for pred_null_p in (None, 0.1):
                shift = shifts[k % len(shifts)]
                k += 1
                pred = rand_bool(rng, n, true_p, pred_null_p)
                col, h, d = validity_column(gpu, rng, dtype, n, shift, validity)
                plan = Plan(gpu, pred)
                try:
                    assert (plan.count, gpu.lib.acu_filter_plan_strategy(plan.h)) == oracle.filter_plan(pred)
                    same(plan.filter(dtype, d), oracle.filter(h, pred),
                         f"filter dtype={dtype} n={n} p={true_p} shift={shift} validity={validity} pred_nulls={pred_null_p}")
                finally:
                    plan.free()
                    col.free()


@pytest.mark.parametrize("dtype,shift", [(abi.I8, 7), (abi.I64, 1)])
def test_filter_shifted_column_multi_round(gpu, oracle, dtype, shift):
    rng = np.random.default_rng(20_500 + dtype)
    n = multi_round(gpu, 1024)
    m = shift + n + PAD
    info = np.iinfo(NP[dtype])
    values = rng.integers(info.min, info.max, m, dtype=NP[dtype], endpoint=True)
    col, h, d = column(gpu, dtype, values, sparse_mask(rng, m, 0.05), shift, n, exact_count=True)
    pred = HostArray.bool_from_numpy(rng.integers(0, 2, n, dtype=np.uint8).astype(bool), sparse_mask(rng, n, 0.02))
    plan = Plan(gpu, pred)
    try:
        same(plan.filter(dtype, d), oracle.filter(h, pred), f"filter dtype={dtype} n={n} shift={shift}")
    finally:
        plan.free()
        col.free()


def filter_launches(gpu, fn):
    """(all launches, launches of the filter's value and bit-compaction kernels) of fn, after a warm call."""
    fn()
    gpu.check(gpu.lib.acu_kernel_stats_reset(gpu.h))
    before = gpu.launch_count()
    fn()
    gpu.check(gpu.lib.acu_ctx_sync(gpu.h))
    ms, n = C.c_double(0), C.c_int64(0)
    gpu.check(gpu.lib.acu_kernel_stats(gpu.h, abi.K_FILTER, C.byref(ms), C.byref(n)))
    return gpu.launch_count() - before, n.value


def test_shifted_filter_takes_the_aligned_launches(gpu):
    """A column with nulls is filtered by as many launches whether its values base is 16-byte aligned or not: at 50 %
    selectivity one value launch that also compacts the validity (no k_compress_bits), and below 4 % the value launch
    plus k_zero_outputs + k_compress_bits for the validity."""
    rng = np.random.default_rng(20_600)
    n = 70001
    col, _, aligned = column(gpu, abi.I64, rng.integers(-9, 9, n + 1 + PAD), rng.random(n + 1 + PAD) >= 0.05, 0, n, exact_count=True)
    _, shifted = at(col, 1, n, exact_count=True)
    assert aligned.values % 16 == 0 and aligned.null_count > 0 and shifted.null_count > 0
    dense, sparse = Plan(gpu, rand_bool(rng, n, 0.5, 0.05)), Plan(gpu, rand_bool(rng, n, 0.02, 0.05))
    try:
        assert dense.count * 25 >= n and sparse.count * 25 < n
        d_al, d_sh = (filter_launches(gpu, lambda: dense.filter(abi.I64, d)) for d in (aligned, shifted))
        s_al, s_sh = (filter_launches(gpu, lambda: sparse.filter(abi.I64, d)) for d in (aligned, shifted))
        assert d_al == d_sh and s_al == s_sh
        assert d_al[1] == 1 and s_al[1] == 2  # timed filter kernels: the value kernel, + k_compress_bits when sparse
        assert s_al[0] == d_al[0] + 2  # + k_zero_outputs and k_compress_bits
    finally:
        dense.free()
        sparse.free()
        col.free()


# ---- 2. filter_record_batch ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [4097, 70001])
def test_filter_record_batch_shifted_columns(gpu, oracle, n):
    """Equal-width columns of both alignment classes (one launch each), nine shifted Int32 columns (more than the 8 columns
    one launch takes), a boolean column and a shifted Utf8 column, under sparse (< 4 %), half and full (All) plans."""
    rng = np.random.default_rng(21_000 + n)
    specs = ([(abi.I32, 0), (abi.I32, 0)] + [(abi.I32, 1 + j % 3) for j in range(9)]
             + [(abi.I64, 0), (abi.I64, 1), (abi.I16, 3), (abi.I8, 5), (abi.F64, 1), (abi.U16, 0)])
    owned, hosts, descs = [], [], []
    try:
        for j, (dtype, shift) in enumerate(specs):
            col, h, d = validity_column(gpu, rng, dtype, n, shift, VALIDITY[j % 4])
            owned.append(col)
            hosts.append(h)
            c = abi.Column()
            c.kind, c.width, c.array = abi.COL_PRIMITIVE, abi.DTYPE_SIZE[dtype], d
            descs.append(c)
        b = rand_bool(rng, n, 0.5, 0.1)
        db = gpu.upload(b)
        owned.append(db)
        hosts.append(b)
        c = abi.Column()
        c.kind, c.width, c.array = abi.COL_BOOLEAN, 0, db.descriptor()
        descs.append(c)
        s = SlicedUtf8(gpu, rng, n, 5, np.int32, 0.1)
        owned.append(s)
        hosts.append(s.host)
        descs.append(s.column())
        cols = (abi.Column * len(descs))(*descs)
        for true_p, pred_null_p in [(0.02, 0.05), (0.5, 0.05), (1.0, None)]:
            pred = rand_bool(rng, n, true_p, pred_null_p)
            plan = Plan(gpu, pred)
            outs = None
            try:
                caps = [int(x.data.nbytes) if isinstance(x, Utf8Column) else 0 for x in hosts]
                outs = gpu._alloc_column_outs(hosts, plan.count, caps)
                gpu.check(gpu.lib.acu_filter_record_batch(gpu.h, plan.h, len(descs), cols, outs))
                check_columns(gpu._download_columns(hosts, outs), hosts, lambda col: oracle_filter(oracle, col, pred),
                              f"filter_record_batch n={n} p={true_p}")
            finally:
                gpu._free_columns([], outs)
                plan.free()
    finally:
        for o in owned:
            o.free()


# ---- 3. stream-ordered section --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("true_p", [0.0, 0.5, 1.0])
def test_section_on_shifted_inputs(gpu, oracle, true_p):
    """plan -> filter of a shifted column with nulls (mode 3: k_compress_bits reads the pending count) -> take with a shifted
    index array -> sum of the taken column, queued in one section, against the synchronous calls and the oracle. Inside a
    section every input carries its exact null_count."""
    rng = np.random.default_rng(22_000 + int(true_p * 10))
    n, m = 70001, 5000
    col, h, d = column(gpu, abi.I64, rng.integers(-1000, 1000, n + 1 + PAD), rng.random(n + 1 + PAD) >= 0.1, 1, n, exact_count=True)
    icol, ih, idd = index_column(gpu, rng, abi.U32, m, n, 3, 0.1)
    pred = rand_bool(rng, n, true_p, 0.05 if 0 < true_p < 1 else None)
    dp = gpu.upload(pred)
    plan = C.c_void_p()
    o_f, o_t = gpu.alloc_out(n * 8, n), gpu.alloc_out(m * 8, m)
    bits, cnt = C.c_uint64(0), C.c_int64(0)
    try:
        pd = dp.descriptor()
        gpu.async_begin()
        try:
            gpu.check(gpu.lib.acu_filter_plan_create(gpu.h, C.byref(pd), C.byref(plan)))
            gpu.check(gpu.lib.acu_filter_primitive(gpu.h, plan, 8, C.byref(d), C.byref(o_f)))
            gpu.check(gpu.lib.acu_take_primitive(gpu.h, 8, C.byref(d), C.byref(idd), abi.U32, 0, C.byref(o_t)))
            taken = abi.Array()
            taken.values, taken.validity, taken.len, taken.null_count = o_t.values, o_t.validity, m, -1
            gpu.check(gpu.lib.acu_aggregate(gpu.h, abi.I64, abi.SUM, C.byref(taken), C.byref(bits), C.byref(cnt)))
        except BaseException:
            try:
                gpu.results_fetch()
            except acu.ArrowError:
                pass
            raise
        gpu.results_fetch()
        filtered, taken_h = gpu.download_out(o_f, abi.I64), gpu.download_out(o_t, abi.I64)
        o_f = o_t = None
        exp_f, exp_t = oracle.filter(h, pred), oracle.take(h, ih)
        tag = f"section p={true_p}"
        same(filtered, exp_f, "filter in " + tag)
        same(taken_h, exp_t, "take in " + tag)
        assert bits_value(abi.I64, bits.value, cnt.value) == oracle.sum(exp_t), "sum in " + tag
        sync_plan = Plan(gpu, pred)
        try:
            same(sync_plan.filter(abi.I64, d), filtered, "synchronous filter vs " + tag)
        finally:
            sync_plan.free()
        same(gpu_take(gpu, abi.I64, d, idd, abi.U32, False), taken_h, "synchronous take vs " + tag)
    finally:
        for o in (o_f, o_t):
            if o is not None:
                gpu._free_out(o)
        if plan:
            gpu.lib.acu_filter_plan_destroy(gpu.h, plan)
        dp.free()
        col.free()
        icol.free()


# ---- 4. take ------------------------------------------------------------------------------------------------------------
TAKE_COUNTS = [255, 256, 257, 2047, 2048, 2049, 70001]
TAKE_VARIANTS = [  # (value dtype, value shift, value nulls, index nulls, check_bounds)
    (abi.I64, 0, None, None, False), (abi.I32, 3, 0.1, None, True), (abi.I8, 5, None, 0.2, False),
    (abi.I16, 1, 0.3, 0.3, True), (abi.F64, 1, 0.1, 0.1, False)]


@pytest.mark.parametrize("idx_dtype", INDEX_DTYPES)
def test_take_shifted_indices(gpu, oracle, idx_dtype):
    """Index arrays whose base is not 16-byte aligned: every index tile, full ones included, is staged by per-lane loads."""
    rng = np.random.default_rng(23_000 + idx_dtype)
    shifts = unaligned_shifts(abi.DTYPE_SIZE[idx_dtype])
    idx_max = min(int(np.iinfo(NP[idx_dtype]).max), 100_000)
    nv = min(5000, idx_max)
    k = 0
    for m in TAKE_COUNTS:
        for vdtype, vshift, vnull, inull, cb in TAKE_VARIANTS:
            ishift = shifts[k % len(shifts)]
            k += 1
            vals = rand_values(rng, vdtype, vshift + nv + PAD)
            vcol, vh, vd = column(gpu, vdtype, vals, None if vnull is None else rng.random(len(vals)) >= vnull, vshift, nv)
            raw = rng.integers(0, nv, ishift + m + PAD).astype(NP[idx_dtype])
            imask = None
            if inull is not None:
                imask = rng.random(len(raw)) >= inull
                hidden = np.nonzero(~imask)[0]
                raw[hidden[: len(hidden) // 2]] = idx_max  # out of bounds under null slots: 0, never a panic
            icol, ih, idd = column(gpu, idx_dtype, raw, imask, ishift, m)
            try:
                tag = f"take idx={idx_dtype}+{ishift} values={vdtype}+{vshift} m={m} nulls={vnull}/{inull} check_bounds={cb}"
                same_or_same_error(lambda: gpu_take(gpu, vdtype, vd, idd, idx_dtype, cb), lambda: oracle.take(vh, ih, cb), tag)
            finally:
                vcol.free()
                icol.free()


@pytest.mark.parametrize("idx_dtype", [abi.U8, abi.I16, abi.I32, abi.U64])
def test_take_shifted_indices_out_of_bounds(gpu, oracle, idx_dtype):
    """An out-of-bounds index at a valid slot inside a full tile: the same panic (or check_bounds error) text and row."""
    rng = np.random.default_rng(23_500 + idx_dtype)
    shift = unaligned_shifts(abi.DTYPE_SIZE[idx_dtype])[-1]
    nv, m = 100, 2049
    vcol, vh, vd = column(gpu, abi.I64, rng.integers(-50, 50, nv + 1 + PAD), None, 1, nv)
    raw = rng.integers(0, nv, shift + m + PAD).astype(NP[idx_dtype])
    mask = rng.random(len(raw)) >= 0.1
    for row in (1000, 1500):
        raw[shift + row], mask[shift + row] = 120, True
    try:
        for imask in (None, mask):
            icol, ih, idd = column(gpu, idx_dtype, raw, imask, shift, m)
            try:
                for cb in (False, True):
                    tag = f"take out of bounds idx={idx_dtype}+{shift} nulls={imask is not None} check_bounds={cb}"
                    with pytest.raises(acu.ArrowError):
                        oracle.take(vh, ih, cb)
                    same_or_same_error(lambda: gpu_take(gpu, abi.I64, vd, idd, idx_dtype, cb), lambda: oracle.take(vh, ih, cb), tag)
            finally:
                icol.free()
    finally:
        vcol.free()


def test_take_shifted_indices_multi_round(gpu, oracle):
    rng = np.random.default_rng(23_700)
    m, nv = multi_round(gpu, 256), 1_000_003
    vcol, vh, vd = column(gpu, abi.I64, rng.integers(-2**62, 2**62, nv + 1 + PAD), sparse_mask(rng, nv + 1 + PAD, 0.1), 1, nv, exact_count=True)
    icol, ih, idd = index_column(gpu, rng, abi.U32, m, nv, 1, 0.05)
    try:
        same(gpu_take(gpu, abi.I64, vd, idd, abi.U32, False), oracle.take(vh, ih), f"take m={m}")
    finally:
        vcol.free()
        icol.free()


def test_take_boolean_shifted_indices(gpu, oracle):
    rng = np.random.default_rng(23_800)
    nv = 5000
    values = rand_bool(rng, nv, 0.5, 0.2, offset=3)
    dv = gpu.upload(values)
    try:
        for idx_dtype, shift in [(abi.U16, 3), (abi.U32, 1), (abi.I64, 1), (abi.U8, 13)]:
            for m in (257, 2048, 70001):
                icol, ih, idd = index_column(gpu, rng, idx_dtype, m, min(nv, 255 if idx_dtype == abi.U8 else nv), shift, 0.1)
                try:
                    vd = dv.descriptor()
                    for cb in (False, True):
                        got = call_out(gpu, bitmap_bytes(m), m, BOOL,
                                       lambda out: gpu.lib.acu_take_boolean(gpu.h, C.byref(vd), C.byref(idd), idx_dtype, int(cb), C.byref(out)))
                        same(got, oracle.take(values, ih, cb), f"take_boolean idx={idx_dtype}+{shift} m={m} check_bounds={cb}")
                finally:
                    icol.free()
    finally:
        dv.free()


@pytest.mark.parametrize("m", [2049, 70001])
def test_take_record_batch_shifted(gpu, oracle, m):
    rng = np.random.default_rng(23_900 + m)
    nv = 9000
    specs = [(abi.I8, 5), (abi.I8, 0), (abi.I16, 0), (abi.I16, 7), (abi.I32, 1), (abi.I64, 1), (abi.I64, 0), (abi.F64, 1)]
    owned, hosts, descs = [], [], []
    try:
        for j, (dtype, shift) in enumerate(specs):
            col, h, d = validity_column(gpu, rng, dtype, nv, shift, VALIDITY[j % 4])
            owned.append(col)
            hosts.append(h)
            c = abi.Column()
            c.kind, c.width, c.array = abi.COL_PRIMITIVE, abi.DTYPE_SIZE[dtype], d
            descs.append(c)
        cols = (abi.Column * len(descs))(*descs)
        for idx_dtype, shift, null_p in [(abi.U32, 2, 0.1), (abi.I64, 1, None), (abi.U16, 5, 0.05)]:
            icol, ih, idd = index_column(gpu, rng, idx_dtype, m, nv, shift, null_p)
            owned.append(icol)
            outs = gpu._alloc_column_outs(hosts, m, [0] * len(hosts))
            try:
                gpu.check(gpu.lib.acu_take_record_batch(gpu.h, len(descs), cols, C.byref(idd), idx_dtype, 0, outs))
                check_columns(gpu._download_columns(hosts, outs), hosts, lambda col: oracle_take(oracle, col, ih),
                              f"take_record_batch idx={idx_dtype}+{shift} m={m}")
            finally:
                gpu._free_columns([], outs)
    finally:
        for o in owned:
            o.free()


# ---- 5. byte gathers -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("odt", [np.int32, np.int64])
def test_byte_gathers_on_sliced_sources(gpu, oracle, odt):
    """take_bytes with aligned 32-bit indices (the FAST kernels for i32 offsets) and with shifted ones (the generic kernels),
    and filter_bytes, all on a zero-copy slice whose first offset is not 0."""
    rng = np.random.default_rng(24_000 + np.dtype(odt).itemsize)
    for n, k, max_len in [(5000, 3, 12), (70001, 1, 40)]:
        src = SlicedUtf8(gpu, rng, n, k, odt, 0.1, max_len)
        try:
            for idx_dtype in (abi.U32, abi.I32):
                for shift in (0, 1, 3):
                    for m, null_p in [(20_000, 0.1), (2049, None)]:
                        icol, ih, idd = index_column(gpu, rng, idx_dtype, m, n, shift, null_p)
                        try:
                            if shift == 0:
                                assert idd.values % 16 == 0
                            for cb in (False, True):
                                tag = f"take_bytes offsets={np.dtype(odt).name} n={n} idx={idx_dtype}+{shift} m={m} check_bounds={cb}"
                                same_bytes(gpu_take_bytes(gpu, src, idd, idx_dtype, cb),
                                           oracle.take_bytes(src.host.offsets, src.host.data, src.host.nulls, ih, cb), tag)
                        finally:
                            icol.free()
            for true_p in (0.0, 0.1, 0.5, 1.0):
                pred = rand_bool(rng, n, true_p, 0.05 if true_p < 1 else None)
                plan = Plan(gpu, pred)
                try:
                    same_bytes(plan.filter_bytes(src), oracle.filter_bytes(src.host.offsets, src.host.data, src.host.nulls, pred),
                               f"filter_bytes offsets={np.dtype(odt).name} n={n} p={true_p}")
                finally:
                    plan.free()
        finally:
            src.free()


def test_dictionary_gather_on_sliced_dictionary(gpu, oracle):
    """At least 65,536 aligned 32-bit keys into a sliced dictionary of at most 8,192 short entries: the k_dict_* kernels."""
    rng = np.random.default_rng(24_100)
    for n, k in [(3000, 5), (8192, 1)]:
        src = SlicedUtf8(gpu, rng, n, k, np.int32, 0.1)
        try:
            for idx_dtype, null_p in [(abi.U32, 0.1), (abi.I32, None)]:
                icol, ih, idd = index_column(gpu, rng, idx_dtype, 100_003, n, 0, null_p)
                try:
                    assert idd.values % 16 == 0
                    same_bytes(gpu_take_bytes(gpu, src, idd, idx_dtype), oracle.take_bytes(src.host.offsets, src.host.data, src.host.nulls, ih),
                               f"dictionary take n={n} k={k} idx={idx_dtype}")
                finally:
                    icol.free()
        finally:
            src.free()


def test_take_bytes_offset_overflow_on_sliced_source(gpu, oracle):
    """take.rs test_take_bytes_offset_overflow on a slice: one 1 MB value selected i32::MAX / 1e6 + 1 times, through aligned
    (FAST) and shifted (generic) indices, with and without index nulls: the reference's error and capacity."""
    value_len = 1_000_000
    n = (2**31 - 1) // value_len + 1
    offsets = np.array([0, 7, 7 + value_len, 7 + value_len + 3], dtype=np.int32)
    data = np.full(int(offsets[-1]) + 16, ord("a"), dtype=np.uint8)
    d_off, d_data = gpu.malloc(offsets.nbytes + 16), gpu.malloc(data.nbytes)
    gpu.h2d(d_off, offsets)
    gpu.h2d(d_data, data)
    nulls = abi.Array()
    nulls.len = 2
    src = types.SimpleNamespace(ob=4, d_off=d_off + 4, d_data=d_data, nulls=nulls,  # rows [1, 3): offsets[0] = 7
                                host=Utf8Column(offsets[1:], data, HostArray(abi.U8, np.zeros(0, np.uint8), 2, None, 0, 0, 0)))
    assert src.d_off % 16 != 0
    try:
        for m, mask in [(n, None), (n + 1, np.arange(n + 1 + 3 + PAD) != 3)]:
            for shift in (0, 3):
                icol, ih, idd = column(gpu, abi.I32, np.zeros(m + 3 + PAD, dtype=np.int32), mask, shift, m, exact_count=True)
                try:
                    with pytest.raises(acu.ArrowError) as e:
                        oracle.take_bytes(src.host.offsets, src.host.data, src.host.nulls, ih)
                    assert e.value.status == abi.ERR_OFFSET_OVERFLOW and str(e.value) == f"Offset overflow error: {n * value_len}"
                    same_or_same_error(lambda: gpu_take_bytes(gpu, src, idd, abi.I32),
                                       lambda: oracle.take_bytes(src.host.offsets, src.host.data, src.host.nulls, ih),
                                       f"offset overflow m={m} shift={shift}")
                finally:
                    icol.free()
    finally:
        gpu.free(d_off)
        gpu.free(d_data)


# ---- 6. zip -----------------------------------------------------------------------------------------------------------------
def zip_call(gpu, dtype, md, td, fd, n, shift_out):
    w = abi.DTYPE_SIZE[dtype]

    def fn(out):
        assert (out.values % 16 != 0) == bool(shift_out)
        assert out.values % 16 or (td.values or 0) % 16 or (fd.values or 0) % 16, "every operand is 16-byte aligned"
        return gpu.lib.acu_zip(gpu.h, w, C.byref(md), C.byref(td), C.byref(fd), C.byref(out))
    return call_out(gpu, n * w, n, dtype, fn, shift_out=shift_out)


def same_zip(got, exp, n, what):
    same(got, exp, what)
    if got.validity is not None:  # the null count is the popcount of whole words: bits past the last row stay clear
        assert not np.unpackbits(got.validity, bitorder="little")[n:].any(), f"{what}: padding bits set"


@pytest.mark.parametrize("dtype", [abi.I8, abi.I16, abi.I32, abi.I64])
def test_zip_shifted(gpu, oracle, dtype):
    """k_zip_elem<W>: truthy, falsy or the output (or all three) not 16-byte aligned; one side with nulls beside one without a
    validity buffer; scalars; masks with nulls; the lengths of SIZES and one multi-round size."""
    rng = np.random.default_rng(25_000 + dtype)
    w = abi.DTYPE_SIZE[dtype]
    shifts = unaligned_shifts(w)
    lengths = [n for n in SIZES if n] + [int(1.2 * 32 * gpu.lib.acu_device_sm_count(gpu.h) * 256)]  # 32 x SMs CTAs of 256
    scalars = [(HostArray.from_list(dtype, [7]).scalar(), "scalar"), (HostArray.from_list(dtype, [None]).scalar(), "null scalar")]
    dscal = [(h, gpu.upload(h), what) for h, what in scalars]
    try:
        for k, n in enumerate(lengths):
            s, s2 = shifts[k % len(shifts)], shifts[(k + 1) % len(shifts)]
            m = s + s2 + n + PAD
            mask = rand_bool(rng, n, 0.5, 0.1 if k % 2 else None)
            dm = gpu.upload(mask)
            tcol = Column(gpu, dtype, rand_values(rng, dtype, m), rng.random(m) >= 0.1)
            fcol = Column(gpu, dtype, rand_values(rng, dtype, m), None)
            try:
                md = dm.descriptor()
                for ts, fs, so in [(s, 0, 0), (0, s, 0), (0, 0, 1), (s, s2, 1)]:
                    (th, td), (fh, fd) = at(tcol, ts, n), at(fcol, fs, n)
                    tag = f"zip dtype={dtype} n={n} shifts={ts}/{fs}/{so}"
                    same_zip(zip_call(gpu, dtype, md, td, fd, n, so), oracle.zip(mask, th, fh), n, tag)
                    same_zip(zip_call(gpu, dtype, md, fd, td, n, so), oracle.zip(mask, fh, th), n, tag + " swapped")
                for sh, sdev, what in dscal:
                    sd = sdev.descriptor()
                    (th, td) = at(tcol, s, n)
                    same_zip(zip_call(gpu, dtype, md, sd, td, n, 0), oracle.zip(mask, sh, th), n, f"zip {what}/shifted n={n}")
                    same_zip(zip_call(gpu, dtype, md, td, sd, n, 1), oracle.zip(mask, th, sh), n, f"zip shifted/{what} n={n}")
            finally:
                tcol.free()
                fcol.free()
                dm.free()
    finally:
        for _, sdev, _ in dscal:
            sdev.free()


# ---- 7. reductions ------------------------------------------------------------------------------------------------------------
def exact_floats(rng, dtype, n):
    """Integer-valued floats whose absolute sum stays below 2^24 (Float32) / 2^53 (Float64)."""
    lim = min(1000, (2**24 - 1) // max(n, 1)) if dtype == abi.F32 else 1_000_000
    return rng.integers(-lim, lim + 1, n).astype(NP[dtype])


def exact_sum(h):
    vals, valid = h.value_array(), h.valid_mask()
    return float(sum(int(v) for v in vals[valid])) if valid.any() else None


@pytest.mark.parametrize("dtype", ALL_DTYPES)
def test_aggregate_shifted(gpu, oracle, dtype):
    rng = np.random.default_rng(26_000 + dtype)
    shifts = unaligned_shifts(abi.DTYPE_SIZE[dtype])
    is_float = dtype in (abi.F32, abi.F64)
    for k, n in enumerate(n for n in SIZES if n):
        shift = shifts[k % len(shifts)]
        for null_p in (None, 0.1, 1.0):
            m = shift + n + PAD
            mask = None if null_p is None else rng.random(m) >= null_p
            col, h, d = column(gpu, dtype, rand_values(rng, dtype, m), mask, shift, n)
            try:
                for op in (abi.MIN, abi.MAX) + (() if is_float else (abi.SUM,)):
                    same_scalar(gpu_aggregate(gpu, dtype, op, d), oracle.aggregate(op, h), f"op={op} dtype={dtype} n={n} shift={shift}", nan_sign=True)
                if not is_float:
                    same_sum_checked(gpu, dtype, d, h, oracle, f"sum_checked dtype={dtype} n={n} shift={shift}")
            finally:
                col.free()
            if is_float:
                for s in (0, shift):  # the exact check on aligned columns too
                    col, h, d = column(gpu, dtype, exact_floats(rng, dtype, m), mask, s, n)
                    try:
                        exp = exact_sum(h)
                        assert oracle.sum(h) == exp
                        for got in (gpu_aggregate(gpu, dtype, abi.SUM, d), gpu_sum_checked(gpu, dtype, d)):
                            same_scalar(got, exp, f"exact sum dtype={dtype} n={n} shift={s} nulls={null_p}")
                    finally:
                        col.free()


@pytest.mark.parametrize("dtype", [abi.F32, abi.F64])
def test_float_sum_special_values(gpu, oracle, dtype):
    """Order-independent results: any NaN gives NaN, +inf with -inf gives NaN, +inf alone gives +inf, and a column of -0.0
    gives +0.0 (the accumulator starts at +0.0). NaN / -inf under a null slot are never summed."""
    rng = np.random.default_rng(26_500 + dtype)
    for n, shift in [(1000, 1), (70001, unaligned_shifts(abi.DTYPE_SIZE[dtype])[-1]), (4097, 0)]:
        m = shift + n + PAD
        rows = shift + rng.choice(n, 4, replace=False)
        mask = np.ones(m, dtype=bool)
        mask[rows[3]] = False
        cases = []
        for specials, exp in [({rows[0]: np.nan}, np.nan), ({rows[0]: np.inf, rows[1]: -np.inf}, np.nan),
                              ({rows[0]: np.inf, rows[3]: np.nan}, np.inf), ({rows[0]: np.inf, rows[3]: -np.inf}, np.inf)]:
            v = exact_floats(rng, dtype, m)
            for r, x in specials.items():
                v[r] = x
            cases.append((v, mask, exp))
        cases.append((np.full(m, -0.0, dtype=NP[dtype]), None, 0.0))
        for v, msk, exp in cases:
            col, h, d = column(gpu, dtype, v, msk, shift, n)
            try:
                tag = f"sum dtype={dtype} n={n} shift={shift} expect={exp}"
                same_scalar(oracle.sum(h), exp, "oracle " + tag)
                same_scalar(gpu_aggregate(gpu, dtype, abi.SUM, d), exp, tag)
                same_scalar(gpu_sum_checked(gpu, dtype, d), exp, "sum_checked " + tag)
            finally:
                col.free()


def test_aggregate_columns_shifted(gpu, oracle):
    """acu_aggregate_columns over columns of different shifts, lengths, types and ops in one call."""
    rng = np.random.default_rng(26_700)
    specs = [(abi.I8, 5, 70001, abi.MIN), (abi.I8, 0, 4097, abi.SUM), (abi.I32, 1, 65, abi.MAX), (abi.I64, 1, 12345, abi.SUM),
             (abi.F64, 1, 1000, abi.MIN), (abi.F32, 3, 70001, abi.SUM), (abi.U16, 7, 33, abi.MAX), (abi.I64, 0, 1, abi.SUM),
             (abi.F64, 1, 4095, abi.SUM), (abi.U8, 15, 8191, abi.SUM), (abi.U32, 2, 129, abi.MIN), (abi.F32, 1, 31, abi.MAX)]
    owned, hosts, descs = [], [], []
    try:
        for j, (dtype, shift, n, op) in enumerate(specs):
            m = shift + n + PAD
            vals = exact_floats(rng, dtype, m) if dtype in (abi.F32, abi.F64) and op == abi.SUM else rand_values(rng, dtype, m)
            col, h, d = column(gpu, dtype, vals, rng.random(m) >= 0.1 if j % 3 else None, shift, n)
            owned.append(col)
            hosts.append(h)
            descs.append(d)
        k = len(specs)
        arrs = (abi.Array * k)(*descs)
        dts, ops = (C.c_int32 * k)(*[s[0] for s in specs]), (C.c_int32 * k)(*[s[3] for s in specs])
        bits, cnts = (C.c_uint64 * k)(), (C.c_int64 * k)()
        gpu.check(gpu.lib.acu_aggregate_columns(gpu.h, k, dts, ops, arrs, bits, cnts))
        for j, (dtype, shift, n, op) in enumerate(specs):
            same_scalar(bits_value(dtype, bits[j], cnts[j]), oracle.aggregate(op, hosts[j]), f"column {j} dtype={dtype} op={op} shift={shift} n={n}",
                    nan_sign=True)
    finally:
        for col in owned:
            col.free()


@pytest.mark.parametrize("dtype", [abi.I8, abi.U8])
def test_reduce_shifted_multi_round(gpu, oracle, dtype):
    """sum / min / max / sum_checked past one grid-stride round of k_reduce and of the checked fold."""
    rng = np.random.default_rng(26_900 + dtype)
    n, shift = multi_round(gpu, 2048), 7
    m = shift + n + PAD
    info = np.iinfo(NP[dtype])
    mask = sparse_mask(rng, m, 0.05)
    col, h, d = column(gpu, dtype, rng.integers(info.min, info.max, m, dtype=NP[dtype], endpoint=True), mask, shift, n, exact_count=True)
    try:
        for op in (abi.SUM, abi.MIN, abi.MAX):
            same_scalar(gpu_aggregate(gpu, dtype, op, d), oracle.aggregate(op, h), f"op={op} dtype={dtype} n={n}")
    finally:
        col.free()
    # 400 valid sparse rows whose running sum stays in range (I8: +100, -100, ...; U8: 1, 0, ...), then the same with one
    # overflow at the last of them
    vals = np.zeros(m, dtype=NP[dtype])
    rows = np.sort(rng.choice(np.arange(shift, shift + n), 400, replace=False))
    vals[rows] = np.where(np.arange(400) % 2 == 0, 100, -100) if dtype == abi.I8 else np.arange(400) % 2 == 0
    mask[rows] = True
    for overflow in (False, True):
        v = vals.copy()
        if overflow:  # I8: 100 + 100 at the last two rows, U8: 199 + 200
            v[rows[-2:] if dtype == abi.I8 else rows[-1:]] = 100 if dtype == abi.I8 else 200
        col, h, d = column(gpu, dtype, v, mask, shift, n, exact_count=True)
        if overflow:
            with pytest.raises(acu.ArrowError):
                oracle.sum_checked(h)
        try:
            same_sum_checked(gpu, dtype, d, h, oracle, f"sum_checked dtype={dtype} n={n} overflow={overflow}")
        finally:
            col.free()


# ---- 8. import path ----------------------------------------------------------------------------------------------------------
_NOOP_ARRAY_RELEASE = C.CFUNCTYPE(None, C.POINTER(abi.ArrowArray))(lambda a: None)
_NOOP_SCHEMA_RELEASE = C.CFUNCTYPE(None, C.POINTER(abi.ArrowSchema))(lambda s: None)


@pytest.mark.parametrize("dtype,fmt,k", [(abi.I64, b"l", 1), (abi.I32, b"i", 3), (abi.I16, b"s", 5), (abi.U8, b"C", 9), (abi.F64, b"g", 1)])
def test_imported_device_slice(gpu, oracle, dtype, fmt, k):
    """A sliced array at the C Device Data Interface (offset = k over whole device buffers), exactly as a sliced Rust array
    arrives: acu_import_column moves the values pointer, and filter, take and sum run on it."""
    rng = np.random.default_rng(27_000 + dtype)
    n = 70001
    vals = exact_floats(rng, dtype, n + k) if dtype == abi.F64 else rand_values(rng, dtype, n + k, small=True)
    full = HostArray.from_numpy(dtype, vals, rng.random(n + k) >= 0.1)
    dev = gpu.upload(full)
    try:
        bufs = (C.c_void_p * 2)(dev.d_validity, dev.d_values)
        arr, sch = abi.ArrowDeviceArray(), abi.ArrowSchema()
        arr.array.length, arr.array.null_count, arr.array.offset = n, -1, k
        arr.array.n_buffers, arr.array.buffers = 2, C.cast(bufs, C.POINTER(C.c_void_p))
        arr.array.release = _NOOP_ARRAY_RELEASE
        arr.device_id, arr.device_type = gpu.device, abi.DEVICE_CUDA
        sch.format, sch.release = fmt, _NOOP_SCHEMA_RELEASE
        col, got_dtype = abi.Column(), C.c_int32(-1)
        gpu.check(gpu.lib.acu_import_column(gpu.h, C.byref(arr), C.byref(sch), C.byref(col), C.byref(got_dtype)))
        d = col.array
        assert got_dtype.value == dtype and d.values == dev.d_values + k * abi.DTYPE_SIZE[dtype] and d.values % 16 != 0
        assert d.validity == dev.d_validity and d.validity_offset == k
        h = full.slice(k, n)
        pred = rand_bool(rng, n, 0.5, 0.05)
        plan = Plan(gpu, pred)
        try:
            same(plan.filter(dtype, d), oracle.filter(h, pred), "filter of an imported slice")
        finally:
            plan.free()
        icol, ih, idd = index_column(gpu, rng, abi.U32, 20_000, n, 0, 0.1)
        try:
            same(gpu_take(gpu, dtype, d, idd, abi.U32, True), oracle.take(h, ih, True), "take of an imported slice")
        finally:
            icol.free()
        same_scalar(gpu_aggregate(gpu, dtype, abi.SUM, d), oracle.sum(h), "sum of an imported slice")
    finally:
        dev.free()


# ---- 6. offset alignment -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("odt", [np.int32, np.int64])
def test_byte_gathers_refuse_misaligned_offsets(gpu, odt):
    """Every byte kernel reads and writes offsets as whole 4- or 8-byte words: take_bytes, filter_bytes and a Utf8 column of
    take_record_batch / filter_record_batch refuse a source or output offset buffer half a word off, before anything writes
    the output offsets. 70,000 aligned 32-bit keys into 100 rows would take the dictionary kernels with i32 offsets."""
    ob = np.dtype(odt).itemsize
    half = ob // 2
    rng = np.random.default_rng(24_200 + ob)
    n, m = 100, 70_000
    src = SlicedUtf8(gpu, rng, n, 0, odt, 0.1)
    icol, _, idd = index_column(gpu, rng, abi.U32, m, n, 0, 0.1)
    plan = Plan(gpu, rand_bool(rng, n, 0.5, None))
    d_src, d_out, d_data = gpu.malloc((n + 1) * ob + 16), gpu.malloc((m + 1) * ob + 16), gpu.malloc(16 * m + 16)
    gpu.h2d(d_src + half, src.host.offsets)
    out = gpu.alloc_out(0, m)
    total = C.c_int64(0)

    def record_batch(take, off, out_off):
        col = src.column()
        col.array.values = off
        cols = (abi.Column * 1)(col)
        outs = (abi.ColumnOut * 1)()
        outs[0].array.values, outs[0].array.validity = out_off, out.validity
        outs[0].data, outs[0].data_capacity = d_data, 16 * m
        if take:
            return gpu.lib.acu_take_record_batch(gpu.h, 1, cols, C.byref(idd), abi.U32, 0, outs)
        return gpu.lib.acu_filter_record_batch(gpu.h, plan.h, 1, cols, outs)

    calls = {
        "take_bytes": lambda off, oo: gpu.lib.acu_take_bytes(gpu.h, ob, off, src.d_data, C.byref(src.nulls), C.byref(idd), abi.U32, 0, oo,
                                                             d_data, 16 * m, C.byref(total), C.byref(out)),
        "filter_bytes": lambda off, oo: gpu.lib.acu_filter_bytes(gpu.h, plan.h, ob, off, src.d_data, C.byref(src.nulls), oo, d_data, 16 * m,
                                                                 C.byref(total), C.byref(out)),
        "take_record_batch": lambda off, oo: record_batch(True, off, oo),
        "filter_record_batch": lambda off, oo: record_batch(False, off, oo),
    }
    sentinel = np.full((m + 1) * ob + 16, 0xA5, dtype=np.uint8)
    try:
        for name, call in calls.items():
            for off, out_off, which in [(src.d_off, d_out + half, "out_offsets"), (d_src + half, d_out, "offsets")]:
                gpu.h2d(d_out, sentinel)
                with pytest.raises(acu.ArrowError) as e:
                    gpu.check(call(off, out_off))
                assert e.value.status == abi.ERR_INVALID_ARGUMENT and str(e.value) == f"Invalid argument error: offsets must be {ob}-byte aligned", \
                    f"{name}, {which} at +{half}: {e.value.status} {e.value}"
                assert np.array_equal(gpu.d2h(d_out, sentinel.nbytes), sentinel), f"{name}, {which} at +{half}: out_offsets written"
            gpu.check(call(src.d_off, d_out))  # the same call on aligned buffers runs
    finally:
        gpu._free_out(out)
        for p in (d_src, d_out, d_data):
            gpu.free(p)
        plan.free()
        icol.free()
        src.free()
