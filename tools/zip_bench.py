"""Kernel time of zip on Utf8, Utf8View, Boolean and FixedSizeBinary columns (acu_kernel_stats: the CUDA-event time of every
kernel the call launches, host transfers excluded), printed as algorithmic bytes over that time and as a fraction of the
H100 SXM data sheet's 3.35 TB/s, with the card's name and power limit read in the same run. No target is asserted.

Columns: Utf8 and Utf8View with --rows rows (1e8 by default), value lengths uniform in 0..16 (mean 8), 5 % nulls; Boolean
with --bool-rows rows (1e9) without nulls; FixedSizeBinary(16) and (20) with --rows rows without nulls. Masks: p = 0.5
random bits, and runs of 1024 rows. Operands: array / array, array / scalar and scalar / scalar. A Utf8 zip is both calls of
the two-phase API (sizing, then copy), as a caller makes them.

Algorithmic bytes: each byte the operation must read or write once. n rows; A the rows whose value comes from an array
side (n for array / array, the selected rows of the array side for array / scalar, 0 for scalar / scalar); D the result's
value bytes, Da those of them taken from array rows; a scalar's value is read once.
  Utf8:      n / 8 mask + 4 A offsets + Da bytes + A / 8 validity bits read, + each scalar's bytes;
             4 n offsets + D bytes written, + n / 8 validity when the result has a NullBuffer;
  Utf8View:  n / 8 mask + 16 A views + A / 8 validity bits read, + 16 per scalar; 16 n views written, + n / 8 validity;
  Boolean:   n / 8 mask + n / 8 value bits of the chosen sides read; n / 8 written;
  FSB(W):    n / 8 mask + n W chosen bytes read; n W written.
Yardsticks in the same run: acu_filter_bytes at s = 0.5 on the same Utf8 column (two-phase; n / 8 predicate + 4 k offsets +
D bytes + k / 8 validity bits of the k selected rows read, 4 k offsets + D bytes + k / 8 validity written), and acu_zip with
elem_bytes = 16 against FixedSizeBinary(16) on the same buffers (the two 1.6 GB outputs compared in full, byte for byte).

  python3 tools/zip_bench.py [--rows 100000000] [--bool-rows 1000000000] [--reps 3]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "arrow-rs_b200"))
import acu  # noqa: E402
from acu import BOOL, HostArray  # noqa: E402
from acu import _abi as abi  # noqa: E402

PEAK_GBS = 3350.0


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def kernel_ms(ctx):
    total = 0.0
    for cls in range(8):
        t, n = C.c_double(0), C.c_int64(0)
        ctx.check(ctx.lib.acu_kernel_stats(ctx.h, cls, C.byref(t), C.byref(n)))
        total += t.value
    return total


def best_of(ctx, reps, call):
    call()  # warm-up
    times = []
    for _ in range(reps):
        ctx.check(ctx.lib.acu_kernel_stats_reset(ctx.h))
        call()
        times.append(kernel_ms(ctx))
    return min(times)


def bits(rng, n, kind, chunk=1 << 26):
    """p = 0.5 random bits, runs of 1024, or (kind = float p) Bernoulli(p) bits, LSB first."""
    out = np.empty((n + 7) // 8 + 8, np.uint8)
    for s in range(0, n, chunk):
        e = min(s + chunk, n)
        if kind == "runs1024":
            b = (np.arange(s, e) // 1024) % 2 == 0
        else:
            b = rng.random(e - s) < (0.5 if kind == "random" else kind)
        out[s // 8:(e + 7) // 8] = np.packbits(b, bitorder="little")
    return out


def row(name, ms, nbytes):
    gbs = nbytes / ms / 1e6
    return {"case": name, "kernel_ms": round(ms, 4), "algorithmic_GB": round(nbytes / 1e9, 4), "GB_s": round(gbs, 1),
            "frac_of_3.35TBs": round(gbs / PEAK_GBS, 4)}


class Dev:
    """Device buffers of one run, freed at the end."""

    def __init__(self, ctx):
        self.ctx, self.ptrs = ctx, []

    def put(self, arr, pad=64):
        arr = np.ascontiguousarray(arr)
        p = self.ctx.malloc(arr.nbytes + pad)
        self.ptrs.append(p)
        step = 1 << 28
        raw = arr.reshape(-1).view(np.uint8)
        for off in range(0, raw.nbytes, step):
            self.ctx.h2d(p + off, raw[off:off + step])
        return p

    def alloc(self, nbytes):
        p = self.ctx.malloc(nbytes + 64)
        self.ptrs.append(p)
        return p

    def free(self):
        for p in self.ptrs:
            self.ctx.free(p)
        self.ptrs = []


def arr_desc(values, n, validity=None, nc=0, scalar=False, voff=0):
    d = abi.Array()
    d.values, d.values_offset, d.validity, d.len, d.null_count, d.is_scalar = values, voff, validity, n, nc, int(scalar)
    return d


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--bool-rows", type=int, default=1_000_000_000)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    n = args.rows
    out_rows = []
    with acu.Context(0) as ctx:
        lib, h = ctx.lib, ctx.h
        dev = Dev(ctx)
        try:
            host_masks = {k: bits(rng, n, k) for k in ("random", "runs1024")}
            masks = {k: dev.put(v) for k, v in host_masks.items()}
            sels = {k: np.unpackbits(v[:(n + 7) // 8], bitorder="little")[:n].astype(bool) for k, v in host_masks.items()}
            # ---- Utf8: two columns, lengths 0..16, 5 % nulls ----
            cols, col_lens = [], []
            for _ in range(2):
                lens = rng.integers(0, 17, n).astype(np.int32)
                offs = np.zeros(n + 1, np.int32)
                np.cumsum(lens, out=offs[1:])
                data = dev.put(np.frombuffer(rng.bytes(int(offs[-1])), np.uint8))
                valid = bits(rng, n, 0.95)
                nc = n - int(np.unpackbits(valid[:(n + 7) // 8], bitorder="little")[:n].sum())
                cols.append((dev.put(offs), data, dev.put(valid), nc, int(offs[-1])))
                col_lens.append(lens)
            sc_offs = dev.put(np.array([0, 8], np.int32))
            sc_data = dev.put(np.frombuffer(b"scalar!!", np.uint8))
            sc2_data = dev.put(np.frombuffer(b"falsy!!!", np.uint8))

            def bytes_side(c, scalar=False, other=False):
                b = abi.BytesArray()
                if scalar:
                    b.offsets, b.data, b.nulls = sc_offs, sc2_data if other else sc_data, arr_desc(None, 1, scalar=True)
                else:
                    b.offsets, b.data, b.nulls = c[0], c[1], arr_desc(None, n, c[2], c[3])
                return b

            out_offs, out_data, out_valid = dev.alloc(4 * (n + 1)), dev.alloc(16 * n + 64), dev.alloc(n // 8 + 64)
            for mk, mp in masks.items():
                md = arr_desc(mp, n)
                for combo in ("array/array", "array/scalar", "scalar/scalar"):
                    t = bytes_side(cols[0], combo == "scalar/scalar")
                    f = bytes_side(cols[1], combo != "array/array", True)
                    o = abi.ArrayOut(None, out_valid, 0, 0, 0)
                    tot = C.c_int64(0)

                    def z():
                        ctx.check(lib.acu_zip_bytes(h, 4, C.byref(md), C.byref(t), C.byref(f), out_offs, None, 0, C.byref(tot), C.byref(o)))
                        ctx.check(lib.acu_zip_bytes(h, 4, C.byref(md), C.byref(t), C.byref(f), out_offs, out_data, 16 * n, C.byref(tot), C.byref(o)))
                    ms = best_of(ctx, args.reps, z)
                    sel = sels[mk]
                    if combo == "array/array":
                        a_rows, d_arr, scalar_bytes = n, tot.value, 0
                    elif combo == "array/scalar":
                        a_rows, d_arr, scalar_bytes = int(sel.sum()), int(col_lens[0][sel].sum()), 8
                    else:
                        a_rows, d_arr, scalar_bytes = 0, 0, 16
                    nulls_out = n / 8 if combo != "scalar/scalar" else 0
                    nbytes = n / 8 + 4 * a_rows + d_arr + a_rows / 8 + scalar_bytes + 4 * n + tot.value + nulls_out
                    out_rows.append(row(f"utf8 zip {combo} mask={mk}", ms, nbytes))
            # yardstick: filter_bytes at s = 0.5 on the first Utf8 column
            pred = HostArray(BOOL, bits(rng, n, "random"), n, None, 0, 0, 0)
            with ctx._scope() as sc:
                plan = ctx._plan(sc, pred)
                k = lib.acu_filter_plan_count(plan)
                nulls = arr_desc(None, n, cols[0][2], cols[0][3])
                o = abi.ArrayOut(None, out_valid, 0, 0, 0)
                tot = C.c_int64(0)

                def fb():
                    ctx.check(lib.acu_filter_bytes(h, plan, 4, cols[0][0], cols[0][1], C.byref(nulls), out_offs, None, 0, C.byref(tot), C.byref(o)))
                    ctx.check(lib.acu_filter_bytes(h, plan, 4, cols[0][0], cols[0][1], C.byref(nulls), out_offs, out_data, 16 * n, C.byref(tot),
                                                   C.byref(o)))
                ms = best_of(ctx, args.reps, fb)
                out_rows.append(row("yardstick acu_filter_bytes s=0.5", ms, n / 8 + 8 * k + 2 * tot.value + 2 * k / 8))
            # ---- Utf8View: views of the same length distribution, long ones pointing into one buffer ----
            vbuf = dev.put(np.frombuffer(rng.bytes(1 << 20), np.uint8))
            table = (C.c_void_p * 1)(vbuf)
            views = []
            for c in range(2):
                v = np.frombuffer(rng.bytes(16 * n), np.uint32).reshape(n, 4).copy()
                ln = rng.integers(0, 17, n).astype(np.uint32)
                v[:, 0] = ln
                v[ln > 12, 2] = 0
                v[ln > 12, 3] = rng.integers(0, (1 << 20) - 16, int((ln > 12).sum())).astype(np.uint32)
                views.append(dev.put(v))
                del v

            def view_side(c, scalar=False):
                d = abi.ViewArray()
                d.views, d.buffers, d.n_buffers = views[c], table, 1
                d.nulls = arr_desc(None, 1, scalar=True) if scalar else arr_desc(None, n, cols[c][2], cols[c][3])
                return d
            out_views = dev.alloc(16 * n)
            for mk, mp in masks.items():
                md = arr_desc(mp, n)
                for combo in ("array/array", "array/scalar", "scalar/scalar"):
                    t, f = view_side(0, combo == "scalar/scalar"), view_side(1, combo != "array/array")
                    o = abi.ArrayOut(None, out_valid, 0, 0, 0)
                    which = C.c_int32(0)

                    def zv():
                        ctx.check(lib.acu_zip_byte_view(h, C.byref(md), C.byref(t), C.byref(f), out_views, C.byref(o), C.byref(which)))
                    ms = best_of(ctx, args.reps, zv)
                    a_rows = {"array/array": n, "array/scalar": int(sels[mk].sum()), "scalar/scalar": 0}[combo]
                    scalars = {"array/array": 0, "array/scalar": 1, "scalar/scalar": 2}[combo]
                    nulls_out = n / 8 if combo != "scalar/scalar" else 0
                    nbytes = n / 8 + 16 * a_rows + a_rows / 8 + 16 * scalars + 16 * n + nulls_out
                    out_rows.append(row(f"utf8view zip {combo} mask={mk}", ms, nbytes))
            dev.free()
            # ---- Boolean ----
            nb = args.bool_rows
            bm = dev.put(bits(rng, nb, "random"))
            bt, bf = dev.put(bits(rng, nb, "random")), dev.put(bits(rng, nb, "random"))
            bo = dev.alloc(nb // 8 + 64)
            md, td, fd = arr_desc(bm, nb), arr_desc(bt, nb), arr_desc(bf, nb)
            o = abi.ArrayOut(bo, dev.alloc(64), 0, 0, 0)

            def zb():
                ctx.check(lib.acu_zip_boolean(h, C.byref(md), C.byref(td), C.byref(fd), C.byref(o)))
            ms = best_of(ctx, args.reps, zb)
            out_rows.append(row("boolean zip array/array mask=random", ms, 3 * nb / 8))
            dev.free()
            # ---- FixedSizeBinary(16), (20), and acu_zip<16> on the same buffers ----
            mp = dev.put(bits(rng, n, "random"))
            md = arr_desc(mp, n)
            for w in (16, 20):
                tv = dev.put(np.frombuffer(rng.bytes(n * w), np.uint8))
                fv = dev.put(np.frombuffer(rng.bytes(n * w), np.uint8))
                ov = dev.alloc(n * w)
                td, fd = arr_desc(tv, n), arr_desc(fv, n)
                o = abi.ArrayOut(ov, dev.alloc(n // 8 + 64), 0, 0, 0)

                def zf():
                    ctx.check(lib.acu_zip_fixed_size_binary(h, w, C.byref(md), C.byref(td), C.byref(fd), C.byref(o)))
                ms = best_of(ctx, args.reps, zf)
                out_rows.append(row(f"fsb({w}) zip array/array mask=random", ms, n / 8 + 2 * n * w))
                ov2 = None
                if w == 16:
                    ov2 = dev.alloc(n * w)
                    o2 = abi.ArrayOut(ov2, dev.alloc(n // 8 + 64), 0, 0, 0)

                    def zp():
                        ctx.check(lib.acu_zip(h, 16, C.byref(md), C.byref(td), C.byref(fd), C.byref(o2)))
                    ms2 = best_of(ctx, args.reps, zp)
                    piece = 1 << 26
                    for off in range(0, n * w, piece):
                        ln = min(piece, n * w - off)
                        assert np.array_equal(ctx.d2h(ov + off, ln), ctx.d2h(ov2 + off, ln)), "acu_zip<16> and the FixedSizeBinary zip differ"
                    out_rows.append(row("yardstick acu_zip elem_bytes=16 mask=random", ms2, n / 8 + 2 * n * w))
                for p in (tv, fv, ov) + ((ov2,) if ov2 else ()):
                    ctx.free(p)
                    dev.ptrs.remove(p)
        finally:
            dev.free()
    print(json.dumps({"card": card(), "rows": out_rows}, indent=1))


if __name__ == "__main__":
    main()
