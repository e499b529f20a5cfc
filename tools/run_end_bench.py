"""Kernel time of filter / take on RunEndEncoded<Int32, Int64> and RunEndEncoded<Int32, Utf8> columns (acu_kernel_stats: the
CUDA-event time of every kernel the calls launch, the values child's filter / take included, host transfers excluded),
printed as algorithmic bytes over that time, with the card's name and power limit read in the same run. No target is
asserted.

Algorithmic bytes (each byte the operation must read or write once; R = 4-byte run ends, V = a value's bytes: 8 for Int64,
its offset and its data bytes for Utf8):
  filter: the predicate bits, the run ends of the slice read, then per kept run its new run end written and its value read
          and written;
  take:   the indices, one run end per index, then per output run its run end and value index written and its value read
          and written. The binary search's other run-end reads are not counted: they are the cost of a random lookup.

  python3 tools/run_end_bench.py [--rows 1000000000] [--mean-run 8] [--take 100000000] [--utf8-rows 1000000000]"""
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
from acu import BOOL, HostArray, RunEndColumn, Utf8Column  # noqa: E402
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
    """A predicate of n rows selecting each with probability p, packed LSB first, without an n-element float array."""
    out = np.empty((n + 7) // 8, np.uint8)
    for s in range(0, n, chunk):
        e = min(s + chunk, n)
        out[s // 8:(e + 7) // 8] = np.packbits(rng.random(e - s) < p, bitorder="little")
    return HostArray(BOOL, out, n, None, 0, 0, 0)


def run_ends(rng, n_rows, mean_run):
    n_runs = n_rows // mean_run
    lens = rng.integers(1, 2 * mean_run, n_runs).astype(np.int64)
    ends = np.cumsum(lens)
    ends = ends[ends < n_rows]
    return np.append(ends, n_rows).astype(np.int32)


def value_bytes(col, rows):
    if isinstance(col, Utf8Column):
        return rows * col.offsets.itemsize + int(col.offsets[-1] - col.offsets[0])
    return rows * col.width()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1_000_000_000)
    ap.add_argument("--utf8-rows", type=int, default=1_000_000_000)
    ap.add_argument("--mean-run", type=int, default=8)
    ap.add_argument("--take", type=int, default=100_000_000)
    args = ap.parse_args()
    rng = np.random.default_rng(0)
    results = []
    with acu.Context(0) as ctx:
        for name, rows in (("RunEndEncoded<Int32, Int64>", args.rows), ("RunEndEncoded<Int32, Utf8>", args.utf8_rows)):
            ends = run_ends(rng, rows, args.mean_run)
            n_runs = len(ends)
            if name.endswith("Int64>"):
                values = HostArray.from_numpy(abi.I64, rng.integers(-2**62, 2**62, n_runs))
            else:
                lens = rng.integers(0, 17, n_runs)
                offs = np.zeros(n_runs + 1, np.int32)
                np.cumsum(lens, out=offs[1:])
                nulls = HostArray(abi.U8, np.zeros(0, np.uint8), n_runs, None, 0, 0, 0)
                values = Utf8Column(offs, rng.integers(97, 123, int(offs[-1]) + 1).astype(np.uint8), nulls)
            col = RunEndColumn(ends, values)
            pred = bernoulli_bits(rng, rows, 0.1)
            got, ms = timed(ctx, lambda: ctx.filter_run_end(col, pred))
            kept = len(got.run_ends)
            alg = rows / 8 + 4 * n_runs + kept * 4 + 2 * value_bytes(got.values, kept)
            results.append({"op": "filter 10%", "column": name, "rows": rows, "runs": n_runs, "kept_runs": kept, "kernel_ms": ms,
                            "GB/s": alg / ms / 1e6})
            del got, pred
            for order in ("uniform", "monotone"):
                ix = rng.integers(0, rows, args.take).astype(np.uint32)
                if order == "monotone":
                    ix.sort()
                idx = HostArray.from_numpy(abi.U32, ix)
                got, ms = timed(ctx, lambda: ctx.take_run_end(col, idx))
                out_runs = len(got.run_ends)
                alg = args.take * (4 + 4) + out_runs * (4 + 4) + 2 * value_bytes(got.values, out_runs)
                results.append({"op": f"take {order}", "column": name, "rows": args.take, "runs_out": out_runs, "kernel_ms": ms,
                                "GB/s": alg / ms / 1e6})
                del got, idx, ix
    print(json.dumps({"card": card(), "results": results}, indent=1))


if __name__ == "__main__":
    main()
