"""Kernel time of filter / take on List<Int64>, List<Utf8> and FixedSizeList<Float32, 768> columns (acu_kernel_stats:
the CUDA-event time of every kernel the calls launch, host transfers excluded), printed as algorithmic bytes over that
time, with the card's name and power limit read in the same run. No target is asserted.

Algorithmic bytes (each byte the operation must read or write once):
  filter: the predicate bits, the list's offsets and validity, the selected rows' offsets and child values out, and the
          child values read (the whole selected child range);
  take:   the indices, two offsets and a validity bit per taken row, the new offsets, the taken child values read and
          written. The child row map (4 B per child row, written by the list call and read by the child's take) is NOT
          counted: it is the known extra cost of taking a list one level at a time, reported beside the result.

  python3 tools/list_bench.py [--rows 100000000] [--utf8-rows 10000000] [--fsl-rows 1000000]"""
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
from acu import FixedSizeListColumn, HostArray, ListColumn, Utf8Column  # noqa: E402
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


def nulls(n, rng):
    h = HostArray.from_numpy(abi.U8, np.zeros(n, np.uint8), rng.random(n) >= 0.05)
    h.values = np.zeros(0, np.uint8)
    return h


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--utf8-rows", type=int, default=10_000_000)
    ap.add_argument("--fsl-rows", type=int, default=1_000_000)
    ap.add_argument("--take", type=int, default=10_000_000)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    results = []
    with acu.Context(0) as ctx:
        cases = []
        lens = rng.integers(0, 17, args.rows)  # 8 children per row on average
        offs = np.zeros(args.rows + 1, np.int64)
        np.cumsum(lens, out=offs[1:])
        child = HostArray.from_numpy(abi.I64, rng.integers(-2**62, 2**62, int(offs[-1])))
        cases.append(("List<Int64>", ListColumn(offs.astype(np.int32) if offs[-1] < 2**31 else offs, child, nulls(args.rows, rng)), 8))
        ulens = rng.integers(0, 17, args.utf8_rows)
        uoffs = np.zeros(args.utf8_rows + 1, np.int32)
        np.cumsum(ulens, out=uoffs[1:])
        slen = rng.integers(0, 17, int(uoffs[-1]))
        soffs = np.zeros(len(slen) + 1, np.int64)
        np.cumsum(slen, out=soffs[1:])
        strings = Utf8Column(soffs, rng.integers(0, 256, int(soffs[-1])).astype(np.uint8), nulls(len(slen), rng))
        cases.append(("List<LargeUtf8>", ListColumn(uoffs, strings, nulls(args.utf8_rows, rng)), None))
        fsl_child = HostArray.from_numpy(abi.F32, rng.random(args.fsl_rows * 768).astype(np.float32))
        cases.append(("FixedSizeList<Float32,768>", FixedSizeListColumn(768, fsl_child, nulls(args.fsl_rows, rng)), 4))
        for name, col, w in cases:
            n = col.length
            pred = HostArray.bool_from_numpy(rng.random(n) < 0.1)
            got, ms = timed(ctx, lambda: ctx.filter_list(col, pred))
            sel_children = got.child.length
            child_bytes = sel_children * w if w else int(got.child.offsets[-1]) + 8 * (sel_children + 1)
            off_w = 0 if isinstance(col, FixedSizeListColumn) else col.offsets.itemsize
            alg = n / 8 * 2 + n * off_w + got.length * off_w + 2 * child_bytes
            results.append({"op": "filter 10%", "column": name, "rows": n, "kernel_ms": ms, "GB/s": alg / ms / 1e6})
            idx = HostArray.from_numpy(abi.U32, rng.integers(0, n, min(args.take, n)).astype(np.uint32))
            got, ms = timed(ctx, lambda: ctx.take_list(col, idx))
            taken_children = got.child.length
            child_bytes = taken_children * w if w else int(got.child.offsets[-1]) + 8 * (taken_children + 1)
            alg = idx.length * (4 + 2 * off_w + off_w) + idx.length / 8 + 2 * child_bytes
            results.append({"op": "take uniform", "column": name, "rows": idx.length, "kernel_ms": ms, "GB/s": alg / ms / 1e6,
                            "row_map_bytes_not_counted": 2 * 4 * taken_children})
    print(json.dumps({"card": card(), "results": results}, indent=1))


if __name__ == "__main__":
    main()
