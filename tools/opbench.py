#!/usr/bin/env python
"""tools/opbench.py — per-op device-time table for every config of BASELINE.json (SURVEY.md §8(d)).

For each op: algorithmic bytes (each input read once, each output written once, bitmaps
ceil(rows/8)) / kernel-only CUDA-event time (acu_kernel_stats) vs the measured HBM peak.
Writes one JSON object per line and a markdown table to stdout; used to fill profiles/.
"""
import argparse
import ctypes as C
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "arrow-rs_b200"))
import numpy as np  # noqa: E402

import acu  # noqa: E402
from acu import _abi as abi  # noqa: E402


def peak():
    try:
        return float(json.load(open(os.path.join(REPO, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 3350.0  # H100 SXM data sheet HBM3 bandwidth


class Bench:
    def __init__(self, ctx, reps):
        self.ctx, self.lib, self.h, self.reps, self.rows = ctx, ctx.lib, ctx.h, reps, []
        self.peak = peak()
        self.only = None
        self.quiet = False

    def arr(self, values, validity, n, nc, voff=0, scalar=0):
        a = abi.Array()
        a.values, a.values_offset, a.validity, a.validity_offset, a.len, a.null_count, a.is_scalar = values, voff, validity, 0, n, nc, scalar
        return a

    def out(self, vbytes, rows):
        o = abi.ArrayOut()
        o.values, o.validity = self.ctx.malloc(vbytes + 64), self.ctx.malloc(abi.bitmap_bytes(rows) + 64)
        return o

    def gen(self, kind, seed, n, width, param=0):
        d = self.ctx.malloc(n * width + 64)
        self.ctx.check(self.lib.acu_generate_values(self.h, kind, seed, 0, param, d, n))
        return d

    def bits(self, seed, p, n):
        d = self.ctx.malloc(abi.bitmap_bytes(n) + 64)
        self.ctx.check(self.lib.acu_generate_bits(self.h, seed, 0, p, d, n))
        c = C.c_int64(0)
        self.ctx.check(self.lib.acu_bitmap_count(self.h, d, 0, None, 0, n, C.byref(c)))
        return d, c.value

    def nulls(self, validity, offset, n):
        c = C.c_int64(0)
        self.ctx.check(self.lib.acu_bitmap_count(self.h, validity, offset, None, 0, n, C.byref(c)))
        return n - c.value

    def timed(self, name, classes, alg_bytes, rows, fn, note=""):
        if self.only and not any(t in name for t in self.only.split("|")):
            return
        for _ in range(2):
            fn()
        self.ctx.check(self.lib.acu_kernel_stats_reset(self.h))
        ms = C.c_float(0)
        self.ctx.check(self.lib.acu_timer_start_slot(self.h, 3))
        for _ in range(self.reps):
            fn()
        self.ctx.check(self.lib.acu_timer_stop_slot(self.h, 3, C.byref(ms)))
        k_ms = 0.0
        for cls in classes:
            tot, cnt = C.c_double(0), C.c_int64(0)
            self.ctx.check(self.lib.acu_kernel_stats(self.h, cls, C.byref(tot), C.byref(cnt)))
            k_ms += tot.value
        k_ms /= self.reps
        gbs = alg_bytes / (k_ms * 1e-3) / 1e9
        row = {"op": name, "rows": rows, "kernel_ms": round(k_ms, 4), "call_ms": round(ms.value / self.reps, 4),
               "algorithmic_bytes": alg_bytes, "achieved_gbs": round(gbs, 1), "frac_of_measured_peak": round(gbs / self.peak, 4),
               "mrows_s": round(rows / (k_ms * 1e-3) / 1e6, 1), "note": note}
        self.rows.append(row)
        if not self.quiet:
            print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--small-rows", type=int, default=100_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default=None, help="substring of the op names to run (alternatives separated by |)")
    ap.add_argument("--decimal-rows", type=int, default=250_000_000, help="rows of the decimal columns (4 GB per Decimal128 column)")
    args = ap.parse_args()
    n, ns = args.rows, args.small_rows
    with acu.Context(0) as ctx:
        b = Bench(ctx, args.reps)
        b.only = args.only
        if b.only and all("decimal" in t for t in b.only.split("|")):  # the decimal rows need none of the configs' columns
            decimal_rows(b, ctx, args.decimal_rows)
            return
        lib, h = ctx.lib, ctx.h
        bb = abi.bitmap_bytes(n)
        # ---------------- config 3: binary add/mul + cmp Float64 1e9, 5 % nulls ----------------
        da, dbv = b.gen(2, 42, n, 8), b.gen(2, 43, n, 8)
        va, nva = b.bits(44, 0.95, n)
        vb, nvb = b.bits(45, 0.95, n)
        A, Bv = b.arr(da, va, n, n - nva), b.arr(dbv, vb, n, n - nvb)
        o = b.out(n * 8, n)
        for name, op in [("add f64", abi.ADD), ("mul f64", abi.MUL), ("div f64", abi.DIV)]:
            b.timed(name, [abi.K_ARITH], 24 * n + 3 * n / 8, n, lambda op=op: ctx.check(lib.acu_arith(h, abi.F64, op, C.byref(A), C.byref(Bv), C.byref(o))))
        for name, op in [("lt f64", abi.LT), ("eq f64", abi.EQ)]:
            b.timed(name, [abi.K_CMP], 16 * n + 4 * n / 8, n, lambda op=op: ctx.check(lib.acu_cmp(h, abi.F64, op, C.byref(A), C.byref(Bv), C.byref(o))))
        # the same columns one element in: value pointers 8 bytes past a 16-byte boundary run the one-element-per-lane kernel
        Au, Bu = b.arr(da + 8, va, n - 1, b.nulls(va, 1, n - 1)), b.arr(dbv + 8, vb, n - 1, b.nulls(vb, 1, n - 1))
        Au.validity_offset = Bu.validity_offset = 1
        b.timed("lt f64 unaligned", [abi.K_CMP], 16 * (n - 1) + 4 * (n - 1) / 8, n - 1,
                lambda: ctx.check(lib.acu_cmp(h, abi.F64, abi.LT, C.byref(Au), C.byref(Bu), C.byref(o))))
        sc = b.arr(dbv, None, 1, 0, scalar=1)
        b.timed("add f64 array+scalar", [abi.K_ARITH], 16 * n + 2 * n / 8, n, lambda: ctx.check(lib.acu_arith(h, abi.F64, abi.ADD, C.byref(A), C.byref(sc), C.byref(o))))
        # Int64 checked add on the same buffers reinterpreted (values in [-2^61, 2^61) -> no overflow)
        di, dj = b.gen(1, 42, n, 8), None
        ctx.free(dbv)
        dj = b.gen(1, 43, n, 8)
        I, J = b.arr(di, va, n, n - nva), b.arr(dj, vb, n, n - nvb)
        b.timed("add i64 checked", [abi.K_ARITH], 24 * n + 3 * n / 8, n, lambda: ctx.check(lib.acu_arith(h, abi.I64, abi.ADD, C.byref(I), C.byref(J), C.byref(o))))
        b.timed("add_wrapping i64", [abi.K_ARITH], 24 * n + 3 * n / 8, n, lambda: ctx.check(lib.acu_arith(h, abi.I64, abi.ADD_WRAPPING, C.byref(I), C.byref(J), C.byref(o))))
        # bitwise (arrow-arith/src/bitwise.rs) on the same inputs: the k_arith skeleton and bytes of add_wrapping above
        b.timed("bitwise_and i64", [abi.K_ARITH], 24 * n + 3 * n / 8, n, lambda: ctx.check(lib.acu_bitwise(h, abi.I64, abi.BITWISE_AND, C.byref(I), C.byref(J), C.byref(o))))
        I32, s32 = b.arr(di, va, n, n - nva), b.arr(dj, None, 1, 0, scalar=1)
        b.timed("shift_left i32 array<<scalar", [abi.K_ARITH], 8 * n + 2 * n / 8, n,
                lambda: ctx.check(lib.acu_bitwise(h, abi.I32, abi.BITWISE_SHIFT_LEFT, C.byref(I32), C.byref(s32), C.byref(o))))
        # predicate construction (arrow-arith/src/boolean.rs): bitmaps only, 1e9 rows
        bl, nbl = b.bits(50, 0.5, n)
        br, nbr = b.bits(51, 0.5, n)
        BL, BR = b.arr(bl, va, n, n - nva), b.arr(br, vb, n, n - nvb)
        b.timed("and_kleene bool (nulls both sides)", [abi.K_CMP], 6 * n / 8, n,
                lambda: ctx.check(lib.acu_boolean(h, abi.BOOL_AND_KLEENE, C.byref(BL), C.byref(BR), C.byref(o))))
        b.timed("is_not_null", [abi.K_CMP], 2 * n / 8, n, lambda: ctx.check(lib.acu_boolean(h, abi.BOOL_IS_NOT_NULL, C.byref(A), None, C.byref(o))))
        ctx.free(bl)
        ctx.free(br)
        # aggregates over a full column
        bits_, cnt_ = C.c_uint64(0), C.c_int64(0)
        for name, dt, arr_, op in [("sum i64", abi.I64, I, abi.SUM), ("min f64", abi.F64, A, abi.MIN), ("sum f64", abi.F64, A, abi.SUM),
                                   ("bit_xor i64", abi.I64, I, abi.BIT_XOR), ("product i64", abi.I64, I, abi.PRODUCT),
                                   ("product f64", abi.F64, A, abi.PRODUCT)]:
            b.timed(name, [abi.K_REDUCE], 8 * n + n / 8, n, lambda dt=dt, arr_=arr_, op=op: ctx.check(lib.acu_aggregate(h, dt, op, C.byref(arr_), C.byref(bits_), C.byref(cnt_))))
        # the checked folds on the same validity with values whose running sum / product fit (all -1; a zero would end
        # product_checked's reads of its chunk): no error, so the timed work is the chunk-summary pass and the one-CTA scan
        dones = ctx.malloc(n * 8 + 64)
        ctx.check(lib.acu_memset(h, dones, 0xFF, n * 8))
        ones = b.arr(dones, va, n, n - nva)
        for name, fn in [("sum_checked i64", lib.acu_sum_checked), ("product_checked i64", lib.acu_product_checked)]:
            b.timed(name, [abi.K_REDUCE], 8 * n + n / 8, n, lambda fn=fn: ctx.check(fn(h, abi.I64, C.byref(ones), C.byref(bits_), C.byref(cnt_))),
                    note="all values -1")
        ctx.free(dones)
        # the same folds on the random Int64 column: both fail within the first rows, so the time is all three passes (the
        # chunk summaries still read every row, the error walk reads one chunk)
        def overflowing(fn):
            st = fn(h, abi.I64, C.byref(I), C.byref(bits_), C.byref(cnt_))
            if st != abi.ERR_ARITHMETIC_OVERFLOW:
                raise RuntimeError(f"expected an overflow, got status {st}")

        for name, fn in [("sum_checked i64 overflowing", lib.acu_sum_checked), ("product_checked i64 overflowing", lib.acu_product_checked)]:
            b.timed(name, [abi.K_REDUCE], 8 * n + n / 8, n, lambda fn=fn: overflowing(fn), note="random values: ArithmeticOverflow near the first row")
        ctx.free(dj)
        # ---------------- config 2: filter + take Int64 1e9 ----------------
        # the same Int64 column one element in (values 8 bytes past a 16-byte boundary, validity offset 1), and its first n
        # bytes as an Int8 column: the workloads on each side of the kernel's alignment and < 4 % validity choices
        Iu = b.arr(di + 8, va, n - 1, b.nulls(va, 1, n - 1))
        Iu.validity_offset = 1
        I8 = b.arr(di, va, n, n - nva)
        for sel in (0.001, 0.01, 0.1, 0.5, 0.9):
            dp, m = b.bits(46, sel, n)
            pred = b.arr(dp, None, n, 0)
            pred_u = b.arr(dp, None, n - 1, 0)
            of = b.out(m * 8, m)
            plan = C.c_void_p()

            def run_filter(pred=pred, width=8, col=I):
                p = C.c_void_p()
                ctx.check(lib.acu_filter_plan_create(h, C.byref(pred), C.byref(p)))
                ctx.check(lib.acu_filter_primitive(h, p, width, C.byref(col), C.byref(of)))
                lib.acu_filter_plan_destroy(h, p)

            note = f"selected {m}; plan + values + validity kernels"
            b.timed(f"filter i64 s={sel}", [abi.K_FILTER, abi.K_FILTER_PLAN], 8 * n + 2 * n / 8 + 8 * m + m / 8, n, run_filter, note=note)
            if sel in (0.01, 0.5):
                b.timed(f"filter i64 s={sel} unaligned", [abi.K_FILTER, abi.K_FILTER_PLAN], 8 * n + 2 * n / 8 + 8 * m + m / 8, n - 1,
                        lambda: run_filter(pred=pred_u, col=Iu), note=note + "; values one element in")
            if sel == 0.01:
                b.timed(f"filter i8 s={sel}", [abi.K_FILTER, abi.K_FILTER_PLAN], n + 2 * n / 8 + m + m / 8, n,
                        lambda: run_filter(width=1, col=I8), note=note)
            if sel in (0.1, 0.5):
                didx = ctx.malloc(m * 4 + 64)
                ctx.check(lib.acu_filter_plan_create(h, C.byref(pred), C.byref(plan)))
                ctx.check(lib.acu_filter_plan_indices(h, plan, abi.U32, didx))
                lib.acu_filter_plan_destroy(h, plan)
                ix = b.arr(didx, None, m, 0)
                b.timed(f"take i64 monotone M/N={sel}", [abi.K_TAKE], 20.25 * m, m, lambda: ctx.check(lib.acu_take_primitive(h, 8, C.byref(I), C.byref(ix), abi.U32, 0, C.byref(of))),
                        note="index distribution A (selected rows)")
                ctx.free(didx)
            ctx.free(dp)
            ctx._free_out(of)
        m = ns
        drand = b.gen(3, 47, m, 4, param=n)
        ix = b.arr(drand, None, m, 0)
        ot = b.out(m * 8, m)
        b.timed("take i64 uniform random M=1e8", [abi.K_TAKE], 20.25 * m, m, lambda: ctx.check(lib.acu_take_primitive(h, 8, C.byref(I), C.byref(ix), abi.U32, 0, C.byref(ot))),
                note="index distribution B")
        ctx.free(drand)
        ctx._free_out(ot)
        # ---------------- config 4: cast Int64 -> Float64 (1e8) and Dictionary<Int32,Utf8> -> Utf8 (1e8) ----------------
        Is = b.arr(di, va, ns, -1)
        oc = b.out(ns * 8, ns)
        b.timed("cast i64->f64", [abi.K_CAST], 16 * ns + 2 * ns / 8, ns, lambda: ctx.check(lib.acu_cast_numeric(h, abi.I64, abi.F64, 1, C.byref(Is), C.byref(oc))))
        Iu = b.arr(di + 8, va, ns, -1)
        Iu.validity_offset = 1
        b.timed("cast i64->f64 unaligned", [abi.K_CAST], 16 * ns + 2 * ns / 8, ns,
                lambda: ctx.check(lib.acu_cast_numeric(h, abi.I64, abi.F64, 1, C.byref(Iu), C.byref(oc))), note="input one element in")
        Fs = b.arr(da, va, ns, -1)
        b.timed("cast f64->i32 safe", [abi.K_CAST], 12 * ns + 2 * ns / 8, ns,
                lambda: ctx.check(lib.acu_cast_numeric(h, abi.F64, abi.I32, 1, C.byref(Fs), C.byref(oc))), note="narrowing: out-of-range values become null")
        D = 4096
        rng = np.random.default_rng(1)
        lens = rng.integers(4, 13, D)
        offs = np.zeros(D + 1, dtype=np.int32)
        offs[1:] = np.cumsum(lens)
        data = rng.integers(97, 123, int(offs[-1]) + 16).astype(np.uint8)
        d_off, d_data = ctx.malloc(offs.nbytes + 64), ctx.malloc(data.nbytes + 64)
        ctx.h2d(d_off, offs)
        ctx.h2d(d_data, data)
        dkeys = b.gen(4, 48, ns, 4, param=D)
        kv, nkv = b.bits(49, 0.95, ns)
        keys = b.arr(dkeys, kv, ns, ns - nkv)
        dict_nulls = b.arr(None, None, D, 0)
        d_out_off = ctx.malloc((ns + 1) * 4 + 64)
        d_out_data = ctx.malloc(ns * 13 + 64)
        on = abi.ArrayOut()
        on.validity = ctx.malloc(abi.bitmap_bytes(ns) + 64)
        total = C.c_int64(0)
        b.timed("cast dict<i32,utf8>->utf8", [abi.K_TAKE, abi.K_BYTES], 4 * ns + ns / 8 + 4 * (ns + 1) + 0.95 * ns * 8 + ns / 8, ns,
                lambda: ctx.check(lib.acu_take_bytes(h, 4, d_off, d_data, C.byref(dict_nulls), C.byref(keys), abi.I32, 0, d_out_off, d_out_data, ns * 13, C.byref(total), C.byref(on))),
                note="kernel_ms = validity + table + lengths + copy kernels (the three tiny scan kernels only show in call_ms)")
        # ---------------- min / max of byte columns (arrow-arith/src/aggregate.rs:460-568), bool_and ----------------
        if not b.only or any(t in "min_string max_string cmp_bytes bool_and" for t in b.only.split("|")):
            agg_bytes_rows(b, ctx, ns, d_off, d_data, dkeys, keys, dict_nulls, d_out_off, d_out_data, on, offs, data, D, va, nva, n)
        # ---------------- like family (arrow-string/src/like.rs) ----------------
        if not b.only or any(t in "like starts_with ends_with contains cmp_bytes cmp_byte_view" for t in b.only.split("|")):
            like_rows(b, ctx, ns, d_off, d_data, keys, dict_nulls, d_out_off, d_out_data, on, offs, data, D)
        # ---------------- length / substring (arrow-string/src/length.rs, substring.rs) ----------------
        if not b.only or any(t in "substring length" for t in b.only.split("|")):
            substring_rows(b, ctx, ns, d_off, d_data, keys, dict_nulls, d_out_off, d_out_data, on, offs, data, D)
        # ---------------- concat_elements (arrow-string/src/concat_elements.rs) ----------------
        if not b.only or any(t in "concat_elements" for t in b.only.split("|")):
            concat_elements_rows(b, ctx, ns, d_off, d_data, keys, dict_nulls, d_out_off, d_out_data, on, offs, data, D)
    print("\n| op | rows | kernel ms | GB/s (algorithmic) | % of measured HBM peak | Mrows/s |")
    print("|---|---|---|---|---|---|")
    for r in b.rows:
        print(f"| {r['op']} | {r['rows']:.3g} | {r['kernel_ms']} | {r['achieved_gbs']} | {100 * r['frac_of_measured_peak']:.1f} | {r['mrows_s']} |")


def decimal_rows(b, ctx, n):
    """Decimal128 add (equal / unequal scales), mul, div, lt against a scalar and sum, and Decimal64 add with unequal scales,
    on n-row columns with 5 % nulls. |values| < 2^40 (divisors odd): no row fails and every i128 row takes the 64-bit fast
    paths of the checked multiply and the division. Algorithmic bytes: 48.375 / row for the i128 binary ops, 24.375 for
    Decimal64, 16.375 for lt vs a scalar, 16.125 for sum."""
    lib, h = ctx.lib, ctx.h
    rng = np.random.default_rng(5)
    x = rng.integers(-2 ** 40, 2 ** 40, n)
    y = rng.integers(-2 ** 40, 2 ** 40, n) | 1

    def upload(ints, width):
        if width == 16:
            vals = np.empty((n, 2), dtype=np.uint64)
            vals[:, 0] = ints.view(np.uint64)
            vals[:, 1] = (ints >> 63).view(np.uint64)
        else:
            vals = ints
        d = ctx.malloc(n * width + 64)
        ctx.h2d(d, vals)
        return d

    va, nva = b.bits(60, 0.95, n)
    vb, nvb = b.bits(61, 0.95, n)
    dx, dy = upload(x, 16), upload(y, 16)
    A, B = b.arr(dx, va, n, n - nva), b.arr(dy, vb, n, n - nvb)
    o = b.out(n * 16, n)
    ot = abi.DecimalType()
    for name, op, (p1, s1), (p2, s2) in [("decimal128 add equal scales", abi.ADD, (38, 2), (38, 2)),
                                         ("decimal128 add unequal scales", abi.ADD, (38, 2), (38, 4)),
                                         ("decimal128 mul", abi.MUL, (38, 2), (38, 2)),
                                         ("decimal128 div", abi.DIV, (38, 2), (38, 2))]:
        L, R = abi.DecimalType(16, p1, s1), abi.DecimalType(16, p2, s2)
        b.timed(name, [abi.K_ARITH], 48 * n + 3 * n / 8, n,
                lambda op=op, L=L, R=R: ctx.check(lib.acu_decimal_arith(h, op, C.byref(L), C.byref(A), C.byref(R), C.byref(B), C.byref(ot), C.byref(o))))
    ds = ctx.malloc(64)
    ctx.h2d(ds, np.array([0, 0], dtype=np.uint64))
    S = b.arr(ds, None, 1, 0, scalar=1)
    b.timed("decimal128 lt scalar", [abi.K_CMP], 16 * n + 3 * n / 8, n,
            lambda: ctx.check(lib.acu_cmp(h, abi.I128, abi.LT, C.byref(A), C.byref(S), C.byref(o))))
    bits, cnt = (C.c_uint64 * 2)(), C.c_int64(0)
    b.timed("decimal128 sum", [abi.K_REDUCE], 16 * n + n / 8, n, lambda: ctx.check(lib.acu_aggregate_i128(h, abi.SUM, C.byref(A), bits, C.byref(cnt))))
    for d in (dx, dy):
        ctx.free(d)
    dx, dy = upload(x, 8), upload(y, 8)
    A64, B64 = b.arr(dx, va, n, n - nva), b.arr(dy, vb, n, n - nvb)
    L, R = abi.DecimalType(8, 18, 2), abi.DecimalType(8, 18, 4)
    b.timed("decimal64 add unequal scales", [abi.K_ARITH], 24 * n + 3 * n / 8, n,
            lambda: ctx.check(lib.acu_decimal_arith(h, abi.ADD, C.byref(L), C.byref(A64), C.byref(R), C.byref(B64), C.byref(ot), C.byref(o))))
    for d in (dx, dy, ds, va, vb, o.values, o.validity):
        ctx.free(d)
    decimal_cast_rows(b, ctx, n, x)


def decimal_cast_rows(b, ctx, n, x):
    """The decimal casts (CastOptions{safe: true}) on n-row columns with 5 % nulls, from the 64-bit-sized values x
    (|x| < 2^40), and for the Decimal128 sources also from full-width values (|v| ~ 2^100: the i128 division and conversion
    slow paths). Algorithmic bytes: input + output values, input + output validity (n / 4)."""
    lib, h = ctx.lib, ctx.h
    rng = np.random.default_rng(6)
    va, nva = b.bits(62, 0.95, n)
    o = b.out(n * 16, n)

    def col(vals):
        d = ctx.malloc(vals.nbytes + 64)
        ctx.h2d(d, vals)
        return d

    halves = np.empty((n, 2), dtype=np.uint64)
    halves[:, 0] = x.view(np.uint64)
    halves[:, 1] = (x >> 63).view(np.uint64)
    wide = np.empty((n, 2), dtype=np.uint64)
    wide[:, 0] = rng.integers(0, 2 ** 63, n).view(np.uint64) * np.uint64(2)
    wide[:, 1] = rng.integers(-2 ** 36, 2 ** 36, n).view(np.uint64)
    d128, d128w, d64, df = col(halves), col(wide), col(x), col(x.astype(np.float64) / 1000.0)
    D = {k: abi.DecimalType(*t) for k, t in (("38,10", (16, 38, 10)), ("38,2", (16, 38, 2)), ("18,2", (8, 18, 2)), ("38,6", (16, 38, 6)))}
    for label, d in (("64-bit values", d128), ("full-width values", d128w)):
        A = b.arr(d, va, n, n - nva)
        b.timed(f"decimal128 cast (38,10)->(38,2) {label}", [abi.K_CAST], 32 * n + n / 4, n,
                lambda A=A: ctx.check(lib.acu_cast_decimal(h, C.byref(D["38,10"]), C.byref(D["38,2"]), 1, C.byref(A), C.byref(o))),
                note="infallible downscale (38 - 8 < 38): unary, rounded half away from zero")
        b.timed(f"decimal128 cast (38,10)->float64 {label}", [abi.K_CAST], 24 * n + n / 4, n,
                lambda A=A: ctx.check(lib.acu_cast_from_decimal(h, C.byref(D["38,10"]), abi.F64, 1, C.byref(A), C.byref(o))))
        b.timed(f"decimal128 cast (38,2)->int64 {label}", [abi.K_CAST], 24 * n + n / 4, n,
                lambda A=A: ctx.check(lib.acu_cast_from_decimal(h, C.byref(D["38,2"]), abi.I64, 1, C.byref(A), C.byref(o))))
    A64 = b.arr(d64, va, n, n - nva)
    b.timed("decimal64 cast (18,2)->decimal128(38,6)", [abi.K_CAST], 24 * n + n / 4, n,
            lambda: ctx.check(lib.acu_cast_decimal(h, C.byref(D["18,2"]), C.byref(D["38,6"]), 1, C.byref(A64), C.byref(o))),
            note="infallible widening upscale")
    b.timed("decimal cast int64->decimal128(38,2)", [abi.K_CAST], 24 * n + n / 4, n,
            lambda: ctx.check(lib.acu_cast_to_decimal(h, abi.I64, C.byref(D["38,2"]), 1, C.byref(A64), C.byref(o))))
    AF = b.arr(df, va, n, n - nva)
    b.timed("decimal cast float64->decimal128(38,10)", [abi.K_CAST], 24 * n + n / 4, n,
            lambda: ctx.check(lib.acu_cast_to_decimal(h, abi.F64, C.byref(D["38,10"]), 1, C.byref(AF), C.byref(o))))
    for d in (d128, d128w, d64, df, va, o.values, o.validity):
        ctx.free(d)


def dict_view_column(b, ctx, keys, offs, data, D, ns):
    """The dictionary-decoded column as all-inline views: take(dictionary views, keys) with 16-byte elements."""
    dict_views = np.zeros((D, 16), dtype=np.uint8)
    for k in range(D):
        ln = int(offs[k + 1] - offs[k])
        dict_views[k, :4] = np.frombuffer(np.uint32(ln).tobytes(), np.uint8)
        dict_views[k, 4:4 + ln] = data[offs[k]: offs[k + 1]]
    d_dv = ctx.malloc(dict_views.nbytes + 64)
    ctx.h2d(d_dv, dict_views)
    ovw = b.out(ns * 16, ns)
    ctx.check(ctx.lib.acu_take_primitive(ctx.h, 16, C.byref(b.arr(d_dv, None, D, 0)), C.byref(keys), abi.I32, 0, C.byref(ovw)))
    ctx.free(d_dv)
    V = abi.ViewArray()
    V.views, V.buffers, V.n_buffers = ovw.values, (C.c_void_p * 1)(), 0
    V.nulls = b.arr(None, ovw.validity, ns, ovw.null_count if ovw.has_validity else 0)
    return V, ovw


def agg_bytes_rows(b, ctx, ns, d_off, d_data, dkeys, keys, dict_nulls, d_out_off, d_out_data, on, offs, data, D, va, nva, n):
    """min_string / max_string on the dictionary-decoded Utf8 column (D = 4096 values of 4..12 bytes, 5 % nulls) and on the
    same values as an all-inline view column; an adversarial Utf8 / view pair whose values share a 24-byte prefix; bool_and on
    a 1e9-row bitmap with validity. acu_cmp_bytes lt on the same Utf8 column (it reads the same bytes twice) is the bar."""
    lib, h = ctx.lib, ctx.h
    total = C.c_int64(0)
    ctx.check(lib.acu_take_bytes(h, 4, d_off, d_data, C.byref(dict_nulls), C.byref(keys), abi.I32, 0, d_out_off, d_out_data, ns * 13,
                                 C.byref(total), C.byref(on)))
    row, cnt = C.c_int64(0), C.c_int64(0)
    U = abi.BytesArray()
    U.offsets, U.data = d_out_off, d_out_data
    U.nulls = b.arr(None, on.validity, ns, on.null_count)
    ub = 4 * (ns + 1) + total.value + ns / 8  # offsets + value bytes + validity
    for name, op in (("min_string utf8 dict-decoded", abi.MIN), ("max_string utf8 dict-decoded", abi.MAX)):
        b.timed(name, [abi.K_REDUCE], ub, ns, lambda op=op: ctx.check(lib.acu_aggregate_bytes(h, 4, op, C.byref(U), C.byref(row), C.byref(cnt))),
                note=f"D={D}, lengths 4..12, 5% nulls; {total.value} value bytes")
    ob = ctx.malloc(abi.bitmap_bytes(ns) + 64)
    ov = abi.ArrayOut()
    ov.values, ov.validity = ob, ctx.malloc(abi.bitmap_bytes(ns) + 64)
    b.timed("min_max bar: cmp_bytes lt utf8 dict-decoded", [abi.K_CMP], 2 * ub + ns / 8, ns,
            lambda: ctx.check(lib.acu_cmp_bytes(h, 4, abi.LT, C.byref(U), C.byref(U), C.byref(ov))), note="reads the column twice")
    ctx._free_out(ov)
    # the same values as an all-inline view column
    V, ovw = dict_view_column(b, ctx, keys, offs, data, D, ns)
    vb = 16 * ns + ns / 8
    for name, op in (("min_string_view inline dict-decoded", abi.MIN), ("max_string_view inline dict-decoded", abi.MAX)):
        b.timed(name, [abi.K_REDUCE], vb, ns, lambda op=op: ctx.check(lib.acu_aggregate_byte_view(h, op, C.byref(V), C.byref(row), C.byref(cnt))),
                note="views only (all values inline)")
    ctx._free_out(ovw)
    # adversarial: every value = the same 24-byte prefix + an 8-byte tail (4096 distinct tails): every key ties
    na = 10_000_000
    rng = np.random.default_rng(3)
    tails = rng.integers(97, 123, (D, 8)).astype(np.uint8)
    vals = np.empty((na, 32), dtype=np.uint8)
    vals[:, :24] = np.frombuffer(b"shared-prefix-of-24-byte", np.uint8)
    vals[:, 24:] = tails[rng.integers(0, D, na)]
    mask = rng.random(na) >= 0.05
    nulls = acu.HostArray.from_numpy(abi.U8, np.zeros(na, np.uint8), mask)
    d_vals, d_aoff, d_valid = ctx.malloc(vals.nbytes + 64), ctx.malloc(4 * (na + 1) + 64), ctx.malloc(nulls.validity.nbytes + 64)
    ctx.h2d(d_vals, vals)
    ctx.h2d(d_aoff, np.arange(na + 1, dtype=np.int32) * 32)
    ctx.h2d(d_valid, nulls.validity)
    views = np.zeros((na, 4), dtype=np.uint32)
    views[:, 0] = 32
    views[:, 1] = np.frombuffer(b"shar", np.uint32)[0]
    views[:, 3] = np.arange(na, dtype=np.uint32) * 32  # buffer 0 = the Utf8 value bytes
    d_views = ctx.malloc(views.nbytes + 64)
    ctx.h2d(d_views, views)
    UA = abi.BytesArray()
    UA.offsets, UA.data, UA.nulls = d_aoff, d_vals, b.arr(None, d_valid, na, na - int(mask.sum()))
    VA = abi.ViewArray()
    VA.views, VA.buffers, VA.n_buffers = d_views, (C.c_void_p * 1)(d_vals), 1
    VA.nulls = UA.nulls
    for name, op in (("min_string utf8 24-byte shared prefix", abi.MIN), ("max_string utf8 24-byte shared prefix", abi.MAX)):
        b.timed(name, [abi.K_REDUCE], 4 * (na + 1) + 32 * na + na / 8, na,
                lambda op=op: ctx.check(lib.acu_aggregate_bytes(h, 4, op, C.byref(UA), C.byref(row), C.byref(cnt))), note="every key ties")
    ov2 = b.out(abi.bitmap_bytes(na), na)
    b.timed("min_max bar: cmp_bytes lt utf8 24-byte shared prefix", [abi.K_CMP], 2 * (4 * (na + 1) + 32 * na + na / 8) + na / 8, na,
            lambda: ctx.check(lib.acu_cmp_bytes(h, 4, abi.LT, C.byref(UA), C.byref(UA), C.byref(ov2))), note="reads the column twice")
    ctx._free_out(ov2)
    for name, op in (("min_string_view 24-byte shared prefix", abi.MIN), ("max_string_view 24-byte shared prefix", abi.MAX)):
        b.timed(name, [abi.K_REDUCE], 16 * na + 32 * na + na / 8, na,
                lambda op=op: ctx.check(lib.acu_aggregate_byte_view(h, op, C.byref(VA), C.byref(row), C.byref(cnt))),
                note="every key ties: algorithmic bytes count the value bytes as read once")
    for p in (d_vals, d_aoff, d_valid, d_views):
        ctx.free(p)
    # bool_and on a 1e9-row bitmap with validity (values almost all true: the answer needs the whole pass)
    bv, _ = b.bits(52, 0.999, n)
    BA = b.arr(bv, va, n, n - nva)
    val = C.c_int32(0)
    b.timed("bool_and 1e9", [abi.K_REDUCE], 2 * n / 8, n, lambda: ctx.check(lib.acu_aggregate_boolean(h, abi.MIN, C.byref(BA), C.byref(val), C.byref(cnt))))
    ctx.free(bv)


def substring_rows(b, ctx, ns, d_off, d_data, keys, dict_nulls, d_out_off, d_out_data, on, offs, data, D):
    """length, substring(s, 1, 3), substring(s, -4, None), substring_by_char(s, 1, 3) on the dictionary-decoded Utf8 column of
    config 4 (D = 4096 values of 4..12 bytes, 5 % nulls) and the view forms on the same values as all-inline views.
    Algorithmic bytes (DESIGN.md §3): length = 4(N+1) + 4N + 2N/8; byte substring = 4(N+1) + 4(N+1) + 2S + 2N/8 with S the
    selected bytes (the Utf8 boundary bytes are not counted); view substring = 16N + 16N + 2N/8 (every value is inline).
    A byte substring is timed as the two calls a caller makes: the sizing call, then the copy."""
    lib, h = ctx.lib, ctx.h
    total = C.c_int64(0)
    ctx.check(lib.acu_take_bytes(h, 4, d_off, d_data, C.byref(dict_nulls), C.byref(keys), abi.I32, 0, d_out_off, d_out_data, ns * 13,
                                 C.byref(total), C.byref(on)))
    U = abi.BytesArray()
    U.offsets, U.data = d_out_off, d_out_data
    U.nulls = b.arr(None, on.validity, ns, on.null_count)
    data_len = total.value
    V, ovw = dict_view_column(b, ctx, keys, offs, data, D, ns)
    ol = b.out(ns * 4, ns)
    b.timed("substring: length utf8 dict-decoded", [abi.K_BYTES], 4 * (ns + 1) + 4 * ns + 2 * ns / 8, ns,
            lambda: ctx.check(lib.acu_length_bytes(h, 4, abi.LENGTH, C.byref(U), C.byref(ol))), note=f"D={D}, lengths 4..12, 5% nulls")
    b.timed("substring: length view inline dict-decoded", [abi.K_BYTES], 16 * ns + 4 * ns + 2 * ns / 8, ns,
            lambda: ctx.check(lib.acu_length_byte_view(h, abi.LENGTH, C.byref(V), C.byref(ol))), note="reads the length word of each view")
    so_off, so_data = ctx.malloc((ns + 1) * 4 + 64), ctx.malloc(data_len + 64)
    onn = abi.ArrayOut()
    onn.validity = ctx.malloc(abi.bitmap_bytes(ns) + 64)
    sel = C.c_int64(0)
    for name, by_char, start, has_len, ln in [("substring(s, 1, 3)", False, 1, 1, 3), ("substring(s, -4, None)", False, -4, 0, 0),
                                              ("substring_by_char(s, 1, 3)", True, 1, 1, 3)]:
        def call(cap, out, by_char=by_char, start=start, has_len=has_len, ln=ln):
            if by_char:
                ctx.check(lib.acu_substring_by_char(h, 4, start, has_len, ln, C.byref(U), so_off, out, cap, C.byref(sel), C.byref(onn)))
            else:
                ctx.check(lib.acu_substring_bytes(h, 4, 1, start, has_len, ln, C.byref(U), data_len, so_off, out, cap, C.byref(sel), C.byref(onn)))
        call(0, None)
        s_bytes = sel.value
        b.timed(f"substring: {name} utf8 dict-decoded", [abi.K_BYTES], 8 * (ns + 1) + 2 * s_bytes + 2 * ns / 8, ns,
                lambda call=call: (call(0, None), call(data_len, so_data)), note=f"sizing + copy call; S = {s_bytes} selected bytes")
    ovs = b.out(ns * 16, ns)
    for name, start, has_len, ln in [("substring(s, 1, 3)", 1, 1, 3), ("substring(s, -4, None)", -4, 0, 0)]:
        b.timed(f"substring: {name} view inline dict-decoded", [abi.K_BYTES], 32 * ns + 2 * ns / 8, ns,
                lambda start=start, has_len=has_len, ln=ln: ctx.check(lib.acu_substring_byte_view(h, 1, start, has_len, ln, C.byref(V), ovs.values, C.byref(ovs))),
                note="views only (all values inline)")
    for p in (so_off, so_data, onn.validity):
        ctx.free(p)
    ctx._free_out(ol)
    ctx._free_out(ovs)
    ctx._free_out(ovw)


def concat_elements_rows(b, ctx, ns, d_off, d_data, keys, dict_nulls, d_out_off, d_out_data, on, offs, data, D):
    """concat_elements(s, s), concat_elements_utf8_many(s, s, s), the view form on the same values and FixedSizeBinary 8 + 8, on
    the dictionary-decoded Utf8 column of config 4 (D = 4096 values of 4..12 bytes, 5 % nulls). The yardstick is the same
    bytes engine's copy, substring(s, 0, None), timed in the same run. A byte concat is timed as the sizing call plus the copy.
    The three-operand row runs on the first half of the rows, since 3S passes i32::MAX.
    Algorithmic bytes (DESIGN.md §3), S = the column's value bytes, K operands: K(4(N+1) + S) read + 4(N+1) + KS written +
    (K + 1)N/8 validity; views: 2 x 16N read + 16N + L written (L = the bytes of the results longer than 12) + 3N/8;
    FixedSizeBinary 8 + 8: 16N read + 16N written + 3N/8."""
    lib, h = ctx.lib, ctx.h
    total = C.c_int64(0)
    ctx.check(lib.acu_take_bytes(h, 4, d_off, d_data, C.byref(dict_nulls), C.byref(keys), abi.I32, 0, d_out_off, d_out_data, ns * 13,
                                 C.byref(total), C.byref(on)))
    U = abi.BytesArray()
    U.offsets, U.data = d_out_off, d_out_data
    U.nulls = b.arr(None, on.validity, ns, on.null_count)
    S = total.value
    note = f"D={D}, lengths 4..12, 5% nulls, S = {S} bytes"
    o_off, o_data = ctx.malloc((ns + 1) * 4 + 64), ctx.malloc(3 * S + 64)
    onn = abi.ArrayOut()
    onn.validity = ctx.malloc(abi.bitmap_bytes(ns) + 64)
    out_len = C.c_int64(0)

    def substring(cap, out):
        ctx.check(lib.acu_substring_bytes(h, 4, 1, 0, 0, 0, C.byref(U), S, o_off, out, cap, C.byref(out_len), C.byref(onn)))
    b.timed("concat_elements: yardstick substring(s, 0, None) utf8 dict-decoded", [abi.K_BYTES], 8 * (ns + 1) + 2 * S + 2 * ns / 8, ns,
            lambda: (substring(0, None), substring(S, o_data)), note="the bytes engine's copy rate: sizing + copy call; " + note)

    def pair(cap, out):
        ctx.check(lib.acu_concat_elements_bytes(h, 4, C.byref(U), C.byref(U), o_off, out, cap, C.byref(out_len), C.byref(onn)))
    b.timed("concat_elements: concat_elements(s, s) utf8 dict-decoded", [abi.K_BYTES], 3 * 4 * (ns + 1) + 4 * S + 3 * ns / 8, ns,
            lambda: (pair(0, None), pair(2 * S, o_data)), note="sizing + copy call; " + note)
    # three operands over the whole column would pass i32::MAX (3S > 2^31): the first half of the rows
    nh = ns // 2
    Uh = abi.BytesArray()
    Uh.offsets, Uh.data = d_out_off, d_out_data
    Uh.nulls = b.arr(None, on.validity, nh, -1)
    three = (abi.BytesArray * 3)(Uh, Uh, Uh)

    def many(cap, out):
        ctx.check(lib.acu_concat_elements_bytes_many(h, 4, 3, three, o_off, out, cap, C.byref(out_len), C.byref(onn)))
    many(0, None)
    Sh = out_len.value // 3
    b.timed("concat_elements: concat_elements_utf8_many(s, s, s) utf8 dict-decoded", [abi.K_BYTES], 4 * 4 * (nh + 1) + 6 * Sh + 4 * nh / 8, nh,
            lambda: (many(0, None), many(3 * Sh, o_data)), note=f"sizing + copy call; the first {nh} rows, S = {Sh} bytes")
    ctx.free(o_off)
    V, ovw = dict_view_column(b, ctx, keys, offs, data, D, ns)
    ovs = b.out(ns * 16, ns)
    ctx.check(lib.acu_concat_elements_byte_view(h, C.byref(V), C.byref(V), None, None, 0, C.byref(out_len), C.byref(ovs)))
    L = out_len.value

    def views(cap, vo, out):
        ctx.check(lib.acu_concat_elements_byte_view(h, C.byref(V), C.byref(V), vo, out, cap, C.byref(out_len), C.byref(ovs)))
    b.timed("concat_elements: concat_elements(v, v) view dict-decoded", [abi.K_BYTES], 48 * ns + L + 3 * ns / 8, ns,
            lambda: (views(0, None, None), views(L, ovs.values, o_data)), note=f"sizing + copy call; L = {L} bytes of long results")
    ctx._free_out(ovs)
    ctx._free_out(ovw)
    ctx.free(o_data)
    fl, fr = b.gen(1, 50, ns, 8), b.gen(1, 51, ns, 8)
    vr, nvr = b.bits(52, 0.95, ns)
    FL, FR = b.arr(fl, on.validity, ns, on.null_count), b.arr(fr, vr, ns, ns - nvr)
    of = b.out(ns * 16, ns)
    w = C.c_int32(0)
    b.timed("concat_elements: fixed_size_binary 8 + 8", [abi.K_BYTES], 32 * ns + 3 * ns / 8, ns,
            lambda: ctx.check(lib.acu_concat_elements_fixed_size_binary(h, 8, C.byref(FL), 8, C.byref(FR), C.byref(w), C.byref(of))),
            note="5% nulls on each side")
    for p in (fl, fr, vr, onn.validity):
        ctx.free(p)
    ctx._free_out(of)


def like_rows(b, ctx, ns, d_off, d_data, keys, dict_nulls, d_out_off, d_out_data, on, offs, data, D):
    """like / starts_with / ends_with / contains / ilike against a scalar on the dictionary-decoded Utf8 column of config 4
    (D = 4096 values of 4..12 bytes, mean 8, 5 % nulls) and on the same values as all-inline views, with acu_cmp_bytes /
    acu_cmp_byte_view EQ against the same scalar as the same-traffic yardstick. Algorithmic bytes (DESIGN.md §3): Utf8 =
    offsets + validity + result bits + the value bytes the op must read (eq: rows whose length equals the needle's, prefix /
    suffix: the needle's length in rows at least that long, substring / glob: every value byte); views = 16 B per view +
    validity + result bits (every value is inline)."""
    lib, h = ctx.lib, ctx.h
    total = C.c_int64(0)
    ctx.check(lib.acu_take_bytes(h, 4, d_off, d_data, C.byref(dict_nulls), C.byref(keys), abi.I32, 0, d_out_off, d_out_data, ns * 13,
                                 C.byref(total), C.byref(on)))
    lens = np.diff(ctx.d2h(d_out_off, 4 * (ns + 1), np.int32))
    U = abi.BytesArray()
    U.offsets, U.data = d_out_off, d_out_data
    U.nulls = b.arr(None, on.validity, ns, on.null_count)
    base = 4 * (ns + 1) + ns / 8 + ns / 8
    V, ovw = dict_view_column(b, ctx, keys, offs, data, D, ns)
    vbytes = 16 * ns + ns / 8 + ns / 8
    ov = b.out(abi.bitmap_bytes(ns), ns)
    keep = []

    def scalars(pat):
        """A one-row Utf8 scalar and view scalar holding `pat` (<= 12 bytes)."""
        raw = pat.encode()
        so, sd, sv = ctx.malloc(64), ctx.malloc(64), ctx.malloc(64)
        ctx.h2d(so, np.array([0, len(raw)], np.int32))
        ctx.h2d(sd, np.frombuffer(raw + b"\0" * 8, np.uint8))
        v = np.zeros(16, np.uint8)
        v[:4] = np.frombuffer(np.uint32(len(raw)).tobytes(), np.uint8)
        v[4:4 + len(raw)] = np.frombuffer(raw, np.uint8)
        ctx.h2d(sv, v)
        keep.extend([so, sd, sv])
        S = abi.BytesArray()
        S.offsets, S.data, S.nulls = so, sd, b.arr(None, None, 1, 0, scalar=1)
        SV = abi.ViewArray()
        SV.views, SV.buffers, SV.n_buffers, SV.nulls = sv, (C.c_void_p * 1)(), 0, b.arr(None, None, 1, 0, scalar=1)
        return S, SV

    rows = [("like 'abc'", abi.LIKE, "abc", int((lens == 3).sum()) * 3),
            ("starts_with 'ab'", abi.STARTS_WITH, "ab", int((lens >= 2).sum()) * 2),
            ("ends_with 'ab'", abi.ENDS_WITH, "ab", int((lens >= 2).sum()) * 2),
            ("contains 'abc'", abi.CONTAINS, "abc", total.value),
            ("like '%a_c%'", abi.LIKE, "%a_c%", total.value),
            ("ilike '%abc%'", abi.ILIKE, "%abc%", total.value)]
    note = f"D={D}, lengths 4..12, 5% nulls; {total.value} value bytes"
    for name, op, pat, value_bytes in rows:
        S, SV = scalars(pat)
        b.timed(f"like: {name} utf8 dict-decoded", [abi.K_CMP], base + value_bytes, ns,
                lambda op=op, S=S: ctx.check(lib.acu_like_bytes(h, 4, 1, op, C.byref(U), C.byref(S), C.byref(ov))), note=note)
        b.timed(f"like: {name} view inline dict-decoded", [abi.K_CMP], vbytes, ns,
                lambda op=op, SV=SV: ctx.check(lib.acu_like_byte_view(h, 1, op, C.byref(V), C.byref(SV), C.byref(ov))), note="views only (all values inline)")
    S, SV = scalars("abc")
    b.timed("like bar: cmp_bytes eq 'abc' utf8 dict-decoded", [abi.K_CMP], base + int((lens == 3).sum()) * 3, ns,
            lambda: ctx.check(lib.acu_cmp_bytes(h, 4, abi.EQ, C.byref(U), C.byref(S), C.byref(ov))), note=note)
    b.timed("like bar: cmp_byte_view eq 'abc' view inline dict-decoded", [abi.K_CMP], 8 * ns + ns / 8 + ns / 8, ns,
            lambda: ctx.check(lib.acu_cmp_byte_view(h, abi.EQ, C.byref(V), C.byref(SV), C.byref(ov))),
            note="eq_inline_scalar: reads the low 8 bytes of each view")
    for p in keep:
        ctx.free(p)
    ctx._free_out(ov)
    ctx._free_out(ovw)


if __name__ == "__main__":
    main()
