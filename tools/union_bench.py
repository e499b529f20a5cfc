"""Kernel time of filter / take on dense Union columns of K Int64 children (acu_kernel_stats: the CUDA-event time of every
kernel the calls launch, host transfers excluded), for the union call alone (acu_filter_union / acu_take_union: the type-id
and offset compaction or gather plus the partition) and for the whole column (the children's takes included), printed as
algorithmic bytes over that time, with the card's name and power limit read in the same run. No target is asserted.

Algorithmic bytes (each byte the operation must read or write once; n = union rows, c = output rows):
  union call, filter: the predicate bits, the type ids (1 B) and offsets (4 B) read, then per output row its type id,
                      new offset and row-map entry (1 + 4 + 4 B) written;
  union call, take:   the indices (4 B) and, per output row, its type id and offset read and its type id, new offset and
                      row-map entry written;
  whole column:       the union call, plus per output row its row-map entry read and its Int64 child value read and written.

  python3 tools/union_bench.py [--rows 1000000000] [--take 100000000] [--fields 2,8,128]"""
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
from acu import BOOL, HostArray, UnionColumn  # noqa: E402
from acu import _abi as abi  # noqa: E402


def kernel_ms(ctx):
    total = 0.0
    for cls in range(8):
        t, n = C.c_double(0), C.c_int64(0)
        ctx.check(ctx.lib.acu_kernel_stats(ctx.h, cls, C.byref(t), C.byref(n)))
        total += t.value
    return total


def timed(ctx, fn):
    ctx.check(ctx.lib.acu_kernel_stats_reset(ctx.h))
    out = fn()
    return out, kernel_ms(ctx)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def bernoulli_bits(rng, n, p, chunk=1 << 26):
    out = np.empty((n + 7) // 8, np.uint8)
    for s in range(0, n, chunk):
        e = min(s + chunk, n)
        out[s // 8:(e + 7) // 8] = np.packbits(rng.random(e - s) < p, bitorder="little")
    return HostArray(BOOL, out, n, None, 0, 0, 0)


def dense_union(rng, rows, k):
    """K Int64 children of rows / K rows each; type ids uniform over K distinct ids, offsets uniform within the child."""
    ids = list(range(0, 128, 128 // k))[:k]
    clen = (rows + k - 1) // k
    tids = np.array(ids, np.int8)[rng.integers(0, k, rows, dtype=np.int64)]
    offs = rng.integers(0, clen, rows, dtype=np.int32)
    children = [HostArray.from_numpy(abi.I64, rng.integers(-2**62, 2**62, clen)) for _ in range(k)]
    return UnionColumn(abi.UNION_DENSE, ids, children, tids, offs)


def union_call(ctx, col, pred=None, idx=None):
    """acu_filter_union / acu_take_union alone; returns the output rows."""
    with ctx._scope() as s:
        d = ctx._union_descriptor(col, s)
        if pred is not None:
            plan = ctx._plan(s, pred)
            m = ctx.lib.acu_filter_plan_count(plan)
            tids, offs, rows, starts = ctx._union_out(col, m, s)
            ctx.check(ctx.lib.acu_kernel_stats_reset(ctx.h))
            ctx.check(ctx.lib.acu_filter_union(ctx.h, plan, C.byref(d), tids, offs, rows, starts))
        else:
            idd = s.upload(idx).descriptor()
            m = idx.length
            tids, offs, rows, starts = ctx._union_out(col, m, s)
            ctx.check(ctx.lib.acu_kernel_stats_reset(ctx.h))
            ctx.check(ctx.lib.acu_take_union(ctx.h, C.byref(d), C.byref(idd), idx.dtype, 0, tids, offs, rows, starts))
        return m, kernel_ms(ctx)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--take", type=int, default=100_000_000)
    ap.add_argument("--fields", default="2,8,128")
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    results = []
    n = args.rows
    with acu.Context(0) as ctx:
        for k in (int(x) for x in args.fields.split(",")):
            col = dense_union(rng, n, k)
            pred = bernoulli_bits(rng, n, 0.1)
            c, ms_union = union_call(ctx, col, pred=pred)
            _, ms_col = timed(ctx, lambda: ctx.filter(col, pred))
            alg_union = n / 8 + 5 * n + 9 * c
            alg_col = alg_union + c * (4 + 16)
            results.append({"op": "filter 10%", "fields": k, "rows": n, "out_rows": c, "union_kernel_ms": ms_union,
                            "union_GB/s": alg_union / ms_union / 1e6, "column_kernel_ms": ms_col, "column_GB/s": alg_col / ms_col / 1e6})
            del pred
            for order in ("random", "monotone"):
                ix = rng.integers(0, n, args.take).astype(np.uint32)
                if order == "monotone":
                    ix.sort()
                idx = HostArray.from_numpy(abi.U32, ix)
                m, ms_union = union_call(ctx, col, idx=idx)
                _, ms_col = timed(ctx, lambda: ctx.take(col, idx))
                alg_union = 4 * m + 5 * m + 9 * m
                alg_col = alg_union + m * (4 + 16)
                results.append({"op": f"take {order}", "fields": k, "rows": m, "union_kernel_ms": ms_union,
                                "union_GB/s": alg_union / ms_union / 1e6, "column_kernel_ms": ms_col, "column_GB/s": alg_col / ms_col / 1e6})
                del idx, ix
            del col
    print(json.dumps({"card": card(), "results": results}, indent=1))


if __name__ == "__main__":
    main()
