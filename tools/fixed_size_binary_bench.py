"""Kernel time of filter / take on FixedSizeBinary(W) columns (acu_kernel_stats: the CUDA-event time of every kernel the call
launches, host transfers excluded), printed as algorithmic bytes over that time and as a fraction of the H100 SXM data
sheet's 3.35 TB/s, with the card's name and power limit read in the same run. No target is asserted. The source columns
have no NullBuffer, so no validity moves.

Algorithmic bytes (each byte the operation must read or write once; n = source rows, s = selected fraction, M = indices):
  filter: n / 8 predicate bits read, s * n * W selected bytes read and written;
  take:   M * 4 index bytes (UInt32) read, M * W bytes read and written.

Widths 3, 20, 32, 36, 64, 768 and 4096 over sources of --source-gb GB (2 by default, far past the 50 MB L2); filter at
s = 0.1 and 0.9, take with uniform random and with monotone (sorted) indices. A / B at W = 32 on the same data: the new row gather against k_take<32> (take
without null indices, where both give the same bytes) and against k_filter_fused<32> (filter: the output pointer is
placed one byte past a 16-byte boundary, which sends W = 32 through the row gather); the outputs are compared byte for
byte before the times are printed.

  python3 tools/fixed_size_binary_bench.py [--source-gb 2] [--take-gb 0.5] [--reps 3]"""
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
WIDTHS = [3, 20, 32, 36, 64, 768, 4096]


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
    times = []
    for _ in range(reps):
        ctx.check(ctx.lib.acu_kernel_stats_reset(ctx.h))
        call()
        times.append(kernel_ms(ctx))
    return min(times)


def bernoulli_bits(rng, n, p, chunk=1 << 26):
    out = np.empty((n + 7) // 8, np.uint8)
    for s in range(0, n, chunk):
        e = min(s + chunk, n)
        out[s // 8:(e + 7) // 8] = np.packbits(rng.random(e - s) < p, bitorder="little")
    return HostArray(BOOL, out, n, None, 0, 0, 0)


def row(name, w, ms, nbytes):
    gbs = nbytes / ms / 1e6
    return {"case": name, "W": w, "kernel_ms": round(ms, 4), "algorithmic_GB": round(nbytes / 1e9, 4), "GB_s": round(gbs, 1),
            "frac_of_3.35TBs": round(gbs / PEAK_GBS, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--source-gb", type=float, default=2.0)
    ap.add_argument("--take-gb", type=float, default=0.5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--widths", default=",".join(map(str, WIDTHS)))
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    rows = []
    with acu.Context(0) as ctx:
        lib, h = ctx.lib, ctx.h
        for w in [int(x) for x in args.widths.split(",")]:
            n = int(args.source_gb * 1e9) // w
            m = int(args.take_gb * 1e9) // w
            src = ctx.malloc(n * w + 64)
            chunk = np.frombuffer(rng.bytes(1 << 24), np.uint8)
            for off in range(0, n * w, len(chunk)):
                ctx.h2d(src + off, chunk[:min(len(chunk), n * w - off)])
            vals = abi.Array()
            vals.values, vals.len = src, n
            out = ctx.malloc(max(n, m) * w + 64)
            obits = ctx.malloc(acu.bitmap_bytes(max(n, m)) + 8)
            try:
                for s in (0.1, 0.9):
                    pred = bernoulli_bits(rng, n, s)
                    with ctx._scope() as sc:
                        plan = ctx._plan(sc, pred)
                        k = lib.acu_filter_plan_count(plan)
                        o = abi.ArrayOut(out + (1 if w == 32 else 0), obits, 0, 0, 0)

                        def f():
                            ctx.check(lib.acu_filter_fixed_size_binary(h, plan, w, C.byref(vals), C.byref(o)))
                        ms = best_of(ctx, args.reps, f)
                        rows.append(row(f"filter s={s}", w, ms, n / 8 + 2 * k * w))
                        if w == 32:  # A / B: k_filter_fused<32> on the same data and plan, output aligned
                            got = ctx.d2h(out + 1, k * w)
                            oa = abi.ArrayOut(out, obits, 0, 0, 0)

                            def g():
                                ctx.check(lib.acu_filter_primitive(h, plan, 32, C.byref(vals), C.byref(oa)))
                            ms2 = best_of(ctx, args.reps, g)
                            assert np.array_equal(got, ctx.d2h(out, k * w)), "filter A / B outputs differ"
                            rows.append(row(f"filter s={s} k_filter_fused<32>", w, ms2, n / 8 + 2 * k * w))
                for kind in ("random", "monotone"):
                    idx = rng.integers(0, n, m, dtype=np.uint32)
                    if kind == "monotone":
                        idx.sort()
                    ix = HostArray.from_numpy(abi.U32, idx)
                    with ctx._scope() as sc:
                        idd = sc.upload(ix).descriptor()
                        o = abi.ArrayOut(out, obits, 0, 0, 0)

                        def t():
                            ctx.check(lib.acu_take_fixed_size_binary(h, w, C.byref(vals), C.byref(idd), abi.U32, 0, C.byref(o)))
                        ms = best_of(ctx, args.reps, t)
                        rows.append(row(f"take {kind}", w, ms, m * 4 + 2 * m * w))
                        if w == 32:  # A / B: k_take<32> (no null indices: the same bytes)
                            got = ctx.d2h(out, m * w)

                            def t2():
                                ctx.check(lib.acu_take_primitive(h, 32, C.byref(vals), C.byref(idd), abi.U32, 0, C.byref(o)))
                            ms2 = best_of(ctx, args.reps, t2)
                            assert np.array_equal(got, ctx.d2h(out, m * w)), "take A / B outputs differ"
                            rows.append(row(f"take {kind} k_take<32>", w, ms2, m * 4 + 2 * m * w))
            finally:
                ctx.free(src)
                ctx.free(out)
                ctx.free(obits)
    print(json.dumps({"card": card(), "rows": rows}, indent=1))


if __name__ == "__main__":
    main()
