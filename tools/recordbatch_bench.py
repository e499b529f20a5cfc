#!/usr/bin/env python
"""tools/recordbatch_bench.py — BASELINE.json configs[4] (SURVEY.md §8(d) config #5):

RecordBatch {i0,i1,i2: Int64, f0,f1,f2: Float64, s0,s1: Utf8}, 6 batches of 2^26 rows per GPU
(4.03e8 rows per GPU, weak scaling), every batch resident in HBM, per batch:

    filter_record_batch(batch, predicate 10 % set)            arrow-select/src/filter.rs:225-244
      -> take_record_batch(filtered, monotone half-sample)    arrow-select/src/take.rs:1123-1133
      -> sum of the 6 numeric columns                         arrow-arith/src/aggregate.rs:943
and ONE NCCL all-reduce of the 6 {partial, valid_count} pairs after the last batch.

The predicate is scanned once per batch (one acu_filter_plan shared by the 8 columns, as
FilterPredicate does, filter.rs:459-478). Run under torchrun for N > 1 (one rank per GPU).
Prints one JSON line (rank 0): Mrows/s over all ranks, per-kernel-class device time,
algorithmic bytes and the fraction of the measured HBM peak.
"""
import argparse
import ctypes as C
import json
import os
import sys

# The contract is ONE JSON line on stdout. Libraries loaded later (NCCL prints "NCCL version ..." when NCCL_DEBUG is set)
# write to file descriptor 1 directly, so the real stdout is set aside and fd 1 is pointed at stderr for everything else.
_REAL_STDOUT = None


def isolate_stdout():
    """Called by main() only (importing this module must not touch the importer's stdout)."""
    global _REAL_STDOUT
    if _REAL_STDOUT is None:
        sys.stdout.flush()
        _REAL_STDOUT = os.dup(1)
        os.dup2(2, 1)


def emit_line(text):
    if _REAL_STDOUT is None:
        print(text, flush=True)
    else:
        os.write(_REAL_STDOUT, (text + "\n").encode())


REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "arrow-rs_b200"))
import numpy as np  # noqa: E402

DICT_ENTRIES = 4096
BATCHES = 6  # about 5 GB of HBM per 2^26-row batch: six leave room on an 80 GB H100 for bench.py's resident headline table
NUMERIC = [("i0", 0), ("i1", 0), ("i2", 0), ("f0", 2), ("f1", 2), ("f2", 2)]  # (name, generator kind)


def peak():
    try:
        return float(json.load(open(os.path.join(REPO, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        return 3350.0  # H100 SXM data sheet HBM3 bandwidth


class Table:
    def __init__(self, ctx, abi, rank, n_batches, batch_rows, selectivity, nulls):
        self.ctx, self.abi, self.rows = ctx, abi, batch_rows
        lib, h = ctx.lib, ctx.h
        n = batch_rows
        bb = abi.bitmap_bytes(n)
        rng = np.random.default_rng(7)
        lens = rng.integers(4, 13, DICT_ENTRIES)
        offs = np.zeros(DICT_ENTRIES + 1, dtype=np.int32)
        offs[1:] = np.cumsum(lens)
        data = rng.integers(97, 123, int(offs[-1]) + 16).astype(np.uint8)
        d_doff, d_ddata = ctx.malloc(offs.nbytes + 64), ctx.malloc(data.nbytes + 64)
        ctx.h2d(d_doff, offs)
        ctx.h2d(d_ddata, data)
        dict_nulls = self.arr(None, None, DICT_ENTRIES, 0)
        d_keys = ctx.malloc(n * 4 + 64)
        self.batches = []
        self.input_bytes = 0
        for b in range(n_batches):
            first_row = (rank * n_batches + b) * n
            cols = []
            for ci, (name, kind) in enumerate(NUMERIC):
                dv, dn = ctx.malloc(n * 8), ctx.malloc(bb)
                ctx.check(lib.acu_generate_values(h, kind, 100 + ci, first_row, 0, dv, n))
                ctx.check(lib.acu_generate_bits(h, 200 + ci, first_row, 1.0 - nulls, dn, n))
                cols.append(("prim", self.arr(dv, dn, n, n - self.count(dn, n))))
            for si in range(2):
                kv = ctx.malloc(bb)
                ctx.check(lib.acu_generate_values(h, 4, 300 + si, first_row, DICT_ENTRIES, d_keys, n))
                ctx.check(lib.acu_generate_bits(h, 400 + si, first_row, 1.0 - nulls, kv, n))
                keys = self.arr(d_keys, kv, n, n - self.count(kv, n))
                d_off, d_data = ctx.malloc((n + 1) * 4 + 64), ctx.malloc(n * 9 + 64)
                on = abi.ArrayOut()
                on.validity = ctx.malloc(bb)
                total = C.c_int64(0)
                ctx.check(lib.acu_take_bytes(h, 4, d_doff, d_ddata, C.byref(dict_nulls), C.byref(keys), abi.I32, 0, d_off, d_data,
                                             n * 9, C.byref(total), C.byref(on)))
                ctx.free(kv)
                cols.append(("utf8", d_off, d_data, self.arr(None, on.validity, n, on.null_count), total.value))
                self.input_bytes += 0
            dp = ctx.malloc(bb)
            ctx.check(lib.acu_generate_bits(h, 46, first_row, selectivity, dp, n))
            count = self.count(dp, n)
            # take indices: the set bits of a p = 0.5 bitmap over the filtered rows (monotone half-sample)
            dh = ctx.malloc(abi.bitmap_bytes(count) + 64)
            ctx.check(lib.acu_generate_bits(h, 47, first_row, 0.5, dh, count))
            half = self.arr(dh, None, count, 0)
            plan = C.c_void_p()
            ctx.check(lib.acu_filter_plan_create(h, C.byref(half), C.byref(plan)))
            m = lib.acu_filter_plan_count(plan)
            d_idx = ctx.malloc(m * 4 + 64)
            ctx.check(lib.acu_filter_plan_indices(h, plan, abi.U32, d_idx))
            lib.acu_filter_plan_destroy(h, plan)
            ctx.free(dh)
            self.batches.append({"cols": cols, "pred": self.arr(dp, None, n, 0), "count": count, "idx": self.arr(d_idx, None, m, 0), "m": m})
        ctx.free(d_keys)
        self.cmax = max(b["count"] for b in self.batches)
        self.mmax = max(b["m"] for b in self.batches)
        self.lanes = [self.make_lane(ctx)]
        self.f_out, self.t_out, self.f_str, self.t_str = self.lanes[0]["f_out"], self.lanes[0]["t_out"], self.lanes[0]["f_str"], self.lanes[0]["t_str"]

    def make_lane(self, ctx):
        """Output buffers of one stream (ctx): batches handled by different lanes are independent (like RecordBatches handed
        to different executor threads), each lane has its own outputs, result blocks and scratch."""
        cmax, mmax = self.cmax, self.mmax
        out = lambda vbytes, rows: self.out(vbytes, rows, ctx)  # noqa: E731
        return {"ctx": ctx,
                "f_out": [out(cmax * 8, cmax) for _ in NUMERIC], "t_out": [out(mmax * 8, mmax) for _ in NUMERIC],
                "f_str": [(ctx.malloc((cmax + 1) * 4 + 64), ctx.malloc(cmax * 13 + 64), out(0, cmax), cmax * 13) for _ in range(2)],
                "t_str": [(ctx.malloc((mmax + 1) * 4 + 64), ctx.malloc(mmax * 13 + 64), out(0, mmax), mmax * 13) for _ in range(2)]}

    def add_lane(self, ctx):
        self.lanes.append(self.make_lane(ctx))

    def arr(self, values, validity, n, nc):
        a = self.abi.Array()
        a.values, a.values_offset, a.validity, a.validity_offset, a.len, a.null_count, a.is_scalar = values, 0, validity, 0, n, nc, 0
        return a

    def out(self, vbytes, rows, ctx=None):
        ctx = ctx or self.ctx
        o = self.abi.ArrayOut()
        o.values = ctx.malloc(vbytes + 64) if vbytes else None
        o.validity = ctx.malloc(self.abi.bitmap_bytes(rows) + 64)
        return o

    def count(self, d_bits, n):
        c = C.c_int64(0)
        self.ctx.check(self.ctx.lib.acu_bitmap_count(self.ctx.h, d_bits, 0, None, 0, n, C.byref(c)))
        return c.value

    def as_in(self, o):
        return self.arr(o.values, o.validity if o.has_validity else None, o.len, o.null_count if o.has_validity else 0)

    def columns_of(self, cols):
        """(acu_column array) for [('prim', Array) | ('utf8', d_off, d_data, nulls Array, nbytes)]."""
        abi = self.abi
        arr = (abi.Column * len(cols))()
        for c, col in enumerate(cols):
            if col[0] == "prim":
                arr[c].kind, arr[c].width, arr[c].array = abi.COL_PRIMITIVE, 8, col[1]
            else:
                arr[c].kind, arr[c].width = abi.COL_BYTES, 4
                arr[c].array = col[3]
                arr[c].array.values = col[1]
                arr[c].data = col[2]
        return arr

    def outs_of(self, prim_outs, str_outs):
        abi = self.abi
        arr = (abi.ColumnOut * 8)()
        for c in range(6):
            arr[c].array = prim_outs[c]
        for si in range(2):
            o_off, o_data, o_n, cap = str_outs[si]
            arr[6 + si].array = o_n
            arr[6 + si].array.values = o_off
            arr[6 + si].data, arr[6 + si].data_capacity = o_data, cap
        return arr

    def alg_bytes(self, n, cnt, m, f_bytes, t_bytes):
        alg = n / 8
        alg += 6 * (8 * n + n / 8 + 8 * cnt + cnt / 8)
        alg += sum(4 * (n + 1) + n / 8 + 4 * (cnt + 1) + 2 * fb + cnt / 8 for fb in f_bytes)
        alg += 6 * 20.25 * m
        alg += sum(4 * m + 8 * m + m / 8 + 4 * (m + 1) + 2 * tb + m / 8 for tb in t_bytes)
        alg += 6 * (8 * m + m / 8)
        return alg

    def run_batches(self, lane, batches, acc):
        """filter_record_batch -> take_record_batch -> 6 sums for `batches` on one lane (ctx / stream); partials into acc."""
        ctx, abi = lane["ctx"], self.abi
        lib, h = ctx.lib, ctx.h
        f_outs, t_outs = self.outs_of(lane["f_out"], lane["f_str"]), self.outs_of(lane["t_out"], lane["t_str"])
        dts = (C.c_int32 * 6)(abi.I64, abi.I64, abi.I64, abi.F64, abi.F64, abi.F64)
        ops = (C.c_int32 * 6)(*[abi.SUM] * 6)
        bits, vc = (C.c_uint64 * 6)(), (C.c_int64 * 6)()
        isum, fsum, cnts = acc["isum"], acc["fsum"], acc["cnts"]
        for bt in batches:
            n, cnt, m = self.rows, bt["count"], bt["m"]
            if "columns" not in bt:
                bt["columns"] = self.columns_of(bt["cols"])
            plan = C.c_void_p()
            ctx.check(lib.acu_filter_plan_create(h, C.byref(bt["pred"]), C.byref(plan)))
            ctx.check(lib.acu_filter_record_batch(h, plan, 8, bt["columns"], f_outs))
            lib.acu_filter_plan_destroy(h, plan)
            fcols = []
            for c in range(6):
                fcols.append(("prim", self.as_in(f_outs[c].array)))
            for si in range(2):
                o = f_outs[6 + si]
                fcols.append(("utf8", o.array.values, o.data, self.as_in(o.array), o.data_len))
            ctx.check(lib.acu_take_record_batch(h, 8, self.columns_of(fcols), C.byref(bt["idx"]), abi.U32, 0, t_outs))
            tin = (abi.Array * 6)(*[self.as_in(t_outs[c].array) for c in range(6)])
            ctx.check(lib.acu_aggregate_columns(h, 6, dts, ops, tin, bits, vc))
            acc["alg"] += self.alg_bytes(n, cnt, m, [f_outs[6].data_len, f_outs[7].data_len], [t_outs[6].data_len, t_outs[7].data_len])
            for ci in range(6):
                if vc[ci]:
                    if ci < 3:
                        isum[ci] = (isum[ci] + bits[ci]) & ((1 << 64) - 1)
                    else:
                        fsum[ci - 3] += np.frombuffer(np.uint64(bits[ci]).tobytes(), dtype=np.float64)[0]
                    cnts[ci] += vc[ci]

    def step(self):
        """One pass over every batch through the RecordBatch-level entry points (one synchronisation per call);
        returns ([6 partial bit patterns], [6 valid counts], algorithmic bytes). With more than one lane (add_lane) the
        batches are dealt round-robin to one host thread per lane: the host gaps of one lane (result fetch, descriptor
        set-up) overlap the kernels of the other. Float64 partials are then summed per lane and across lanes (a different
        association order than the serial loop: inside the documented Float64-sum tolerance)."""
        accs = [{"isum": [0, 0, 0], "fsum": [0.0, 0.0, 0.0], "cnts": [0] * 6, "alg": 0} for _ in self.lanes]
        if len(self.lanes) == 1:
            self.run_batches(self.lanes[0], self.batches, accs[0])
        else:
            import threading
            errs = []

            def work(k):
                try:
                    self.run_batches(self.lanes[k], self.batches[k::len(self.lanes)], accs[k])
                except BaseException as e:  # noqa: BLE001
                    errs.append(e)
            ths = [threading.Thread(target=work, args=(k,)) for k in range(len(self.lanes))]
            for t in ths:
                t.start()
            for t in ths:
                t.join()
            if errs:
                raise errs[0]
        isum = [sum(a["isum"][i] for a in accs) & ((1 << 64) - 1) for i in range(3)]
        fsum = [sum(a["fsum"][i] for a in accs) for i in range(3)]
        cnts = [sum(a["cnts"][i] for a in accs) for i in range(6)]
        return self.final_reduce(isum, fsum, cnts, sum(a["alg"] for a in accs))

    def final_reduce(self, isum, fsum, cnts, alg):
        # one NCCL all-reduce per dtype group (3 Int64 sums, 3 Float64 sums) after the last batch
        ctx, abi = self.ctx, self.abi
        lib, h = ctx.lib, ctx.h
        ib, ic = (C.c_uint64 * 3)(*isum), (C.c_int64 * 3)(*cnts[:3])
        ctx.check(lib.acu_comm_allreduce_aggregates(h, abi.I64, abi.SUM, ib, ic, 3))
        fbits = [int(np.frombuffer(np.float64(x).tobytes(), dtype=np.uint64)[0]) for x in fsum]
        fb, fc = (C.c_uint64 * 3)(*fbits), (C.c_int64 * 3)(*cnts[3:])
        ctx.check(lib.acu_comm_allreduce_aggregates(h, abi.F64, abi.SUM, fb, fc, 3))
        return list(ib) + list(fb), list(ic) + list(fc), alg

    def step_per_column(self):
        """The same pass through the single-array entry points (one or two synchronisations per column and op)."""
        ctx, abi = self.ctx, self.abi
        lib, h = ctx.lib, ctx.h
        isum, fsum, cnts, alg = [0, 0, 0], [0.0, 0.0, 0.0], [0] * 6, 0
        for bt in self.batches:
            n, cnt, m = self.rows, bt["count"], bt["m"]
            plan = C.c_void_p()
            ctx.check(lib.acu_filter_plan_create(h, C.byref(bt["pred"]), C.byref(plan)))
            si = 0
            fstr = []
            for ci, col in enumerate(bt["cols"]):
                if col[0] == "prim":
                    ctx.check(lib.acu_filter_primitive(h, plan, 8, C.byref(col[1]), C.byref(self.f_out[ci])))
                else:
                    _, d_off, d_data, nulls, nbytes = col
                    o_off, o_data, o_n, cap = self.f_str[si]
                    total = C.c_int64(0)
                    ctx.check(lib.acu_filter_bytes(h, plan, 4, d_off, d_data, C.byref(nulls), o_off, o_data, cap, C.byref(total), C.byref(o_n)))
                    fstr.append((o_off, o_data, self.as_in(o_n), total.value))
                    si += 1
            lib.acu_filter_plan_destroy(h, plan)
            for ci in range(6):
                fin = self.as_in(self.f_out[ci])
                ctx.check(lib.acu_take_primitive(h, 8, C.byref(fin), C.byref(bt["idx"]), abi.U32, 0, C.byref(self.t_out[ci])))
            tb = []
            for si in range(2):
                o_off, o_data, nulls, _ = fstr[si]
                t_off, t_data, t_n, cap = self.t_str[si]
                total = C.c_int64(0)
                ctx.check(lib.acu_take_bytes(h, 4, o_off, o_data, C.byref(nulls), C.byref(bt["idx"]), abi.U32, 0, t_off, t_data, cap, C.byref(total), C.byref(t_n)))
                tb.append(total.value)
            alg += self.alg_bytes(n, cnt, m, [f[3] for f in fstr], tb)
            for ci in range(6):
                tin = self.as_in(self.t_out[ci])
                bits, c = C.c_uint64(0), C.c_int64(0)
                dt = abi.I64 if ci < 3 else abi.F64
                ctx.check(lib.acu_aggregate(h, dt, abi.SUM, C.byref(tin), C.byref(bits), C.byref(c)))
                if c.value:
                    if ci < 3:
                        isum[ci] = (isum[ci] + bits.value) & ((1 << 64) - 1)
                    else:
                        fsum[ci - 3] += np.frombuffer(np.uint64(bits.value).tobytes(), dtype=np.float64)[0]
                    cnts[ci] += c.value
        return self.final_reduce(isum, fsum, cnts, alg)


def main():
    isolate_stdout()
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--batches", type=int, default=BATCHES)
    ap.add_argument("--batch-rows", type=int, default=1 << 26)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--selectivity", type=float, default=0.10)
    ap.add_argument("--nulls", type=float, default=0.05)
    ap.add_argument("--streams", type=int, default=int(os.environ.get("ACU_RB_STREAMS", "3")),
                    help="lanes (ctx + stream + host thread) the batches are dealt to; 1 = the serial loop")
    ap.add_argument("--per-column", action="store_true", help="use the single-array entry points (a synchronisation per column)")
    args = ap.parse_args()
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if os.environ.get("ACU_BENCH_NUMA", "1") != "0":  # host threads (one per lane) next to the GPU, like bench.py's ranks
        sys.path.insert(0, REPO)
        try:
            from bench import numa_bind
            numa_bind(local_rank)
        except Exception:
            pass
    import acu
    from acu import _abi as abi
    from acu.rendezvous import Group
    ctx = acu.Context(local_rank)
    lib, h = ctx.lib, ctx.h
    group = Group(ctx, rank, local_rank, world)
    barrier = group.barrier

    tb = Table(ctx, abi, rank, args.batches, args.batch_rows, args.selectivity, args.nulls)
    extra = [acu.Context(local_rank) for _ in range(max(args.streams, 1) - 1)] if not args.per_column else []
    for c in extra:
        tb.add_lane(c)
    ctxs = [ctx] + extra
    step = tb.step_per_column if args.per_column else tb.step
    for _ in range(args.warmup):
        step()
    barrier()
    for c in ctxs:
        c.sync()
        c.check(lib.acu_kernel_stats_reset(c.h))
    launches0 = sum(c.launch_count() for c in ctxs)
    ms = C.c_float(0)
    import time
    t0 = time.perf_counter()
    ctx.check(lib.acu_timer_start_slot(h, 1))
    for _ in range(args.steps):
        sums, cnts, alg = step()
    ctx.check(lib.acu_timer_stop_slot(h, 1, C.byref(ms)))
    for c in ctxs:
        c.sync()
    wall_ms = (time.perf_counter() - t0) * 1e3
    barrier()
    # one lane: CUDA events on its stream; several lanes: host clock around steps that start and end with every stream idle
    # (each step ends with a synchronising all-reduce on lane 0 after all worker threads have joined)
    step_ms = (ms.value if len(ctxs) == 1 else wall_ms) / args.steps
    step_ms = group.max_over_ranks(step_ms)
    names = ["arith", "cmp", "cast", "filter", "filter_plan", "take", "reduce", "bytes"]
    kern = {}
    for cls, nm in enumerate(names):
        tot_ms, tot_n = 0.0, 0
        for c in ctxs:
            tot, cnt = C.c_double(0), C.c_int64(0)
            c.check(lib.acu_kernel_stats(c.h, cls, C.byref(tot), C.byref(cnt)))
            tot_ms += tot.value
            tot_n += cnt.value
        if tot_n:
            kern[nm] = {"ms_per_step": round(tot_ms / args.steps, 4), "launches_per_step": tot_n / args.steps}
    if rank == 0:
        rows = args.batches * args.batch_rows
        ksum = sum(v["ms_per_step"] for v in kern.values())
        emit_line(json.dumps({
            "metric": "Mrows/sec filter_record_batch -> take_record_batch -> sum, 8-column RecordBatch", "value": rows * world / (step_ms * 1e-3) / 1e6,
            "unit": "Mrows/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": step_ms, "scaling": "weak",
            "config": {"workload": "RecordBatch{3xInt64,3xFloat64,2xUtf8(D=4096, len 4..12)}", "batches_per_gpu": args.batches, "batch_rows": args.batch_rows,
                       "rows_per_gpu": rows, "selectivity": args.selectivity, "null_density": args.nulls, "take": "monotone half-sample of the filtered rows (UInt32)",
                       "entry_points": "per-column" if args.per_column else "record-batch (one synchronisation per call)",
                       "streams": len(ctxs), "timer": "CUDA events on the ctx stream" if len(ctxs) == 1 else "host clock around steps bracketed by a synchronisation of every stream",
                       "collective": "2 NCCL all-reduces (3 Int64 + 3 Float64 sums with valid counts) after the last batch"},
            "algorithmic_bytes_per_step": alg, "achieved_gbs": alg / (step_ms * 1e-3) / 1e9, "frac_of_measured_peak": alg / (step_ms * 1e-3) / 1e9 / peak(),
            "kernel_ms_per_step": round(ksum, 3), "kernels": kern, "gpu_launches": sum(c.launch_count() for c in ctxs) - launches0,
            "check": {"sums_bits": [int(x) for x in sums], "valid_counts": [int(x) for x in cnts]}}))
    group.close()
    for c in extra:
        c.close()


if __name__ == "__main__":
    main()
