"""BatchCoalescer (arrow-select/src/coalesce.rs:148-590) over device-resident in-progress columns.

Output batches hold exactly ``target_batch_size`` rows in input order (the last one is produced
by ``finish_buffered_batch``). Every in-progress column lives in HBM at its final capacity and rows
are appended in place (``InProgressArray::copy_rows``, coalesce.rs:492-520):

  * fixed-width values      -> acu_memcpy_d2d at ``buffered_rows * width``
  * validity / boolean bits -> acu_bitmap_copy at bit ``buffered_rows`` (acu_bitmap_fill for all-valid pieces)
  * Utf8 offsets / bytes    -> acu_offsets_append (rebased on the running byte total) + acu_memcpy_d2d

``push_batch_with_filter`` = filter_record_batch (one plan, one synchronisation) followed by
``push_batch`` of the device-resident result, which is what the reference documents it to be
equivalent to (coalesce.rs:236-237); ``push_batch_with_indices`` likewise with take_record_batch.

This module is the Python host mirror used by the tests; arrays cross it as HostArray / Utf8Column
(uploaded on push, downloaded when a completed batch is popped).
"""
import ctypes as C
from collections import deque

import numpy as np

from . import _abi as abi
from . import BOOL, NP_DTYPES, U8, HostArray, Utf8Column, bitmap_bytes


class _Column:
    """One in-progress column (device buffers at capacity ``target`` rows)."""

    def __init__(self, ctx, kind, target):
        self.ctx, self.kind, self.target = ctx, kind, target
        self.width = 0 if kind in (BOOL, "utf8", "large_utf8") else abi.DTYPE_SIZE[kind]
        self.ob = 4 if kind == "utf8" else 8 if kind == "large_utf8" else 0
        self._fresh()

    def _fresh(self):
        ctx, t = self.ctx, self.target
        self.d_valid = ctx.malloc(bitmap_bytes(t) + 8)
        self.valid_materialised = False  # all rows so far are valid and d_valid holds nothing yet
        self.null_count = 0
        if self.ob:
            self.d_values = ctx.malloc((t + 1) * self.ob + 16)  # offsets
            self.data_cap = 1 << 16
            self.d_data = ctx.malloc(self.data_cap)
            self.data_len = 0
            ctx.h2d(self.d_values, np.zeros(1, dtype=np.int32 if self.ob == 4 else np.int64))
        elif self.kind == BOOL:
            self.d_values = ctx.malloc(bitmap_bytes(t) + 8)
        else:
            self.d_values = ctx.malloc(t * self.width + 16)

    def _reserve_data(self, need):
        if need <= self.data_cap:
            return
        cap = self.data_cap
        while cap < need:
            cap *= 2
        ctx = self.ctx
        d_new = ctx.malloc(cap)
        if self.data_len:
            ctx.check(ctx.lib.acu_memcpy_d2d(ctx.h, d_new, self.d_data, self.data_len))
        ctx.free(self.d_data)
        self.d_data, self.data_cap = d_new, cap

    def copy_rows(self, src, offset, n, at):
        """Append rows [offset, offset + n) of the device source column ``src`` at row ``at``."""
        ctx = self.ctx
        lib, h = ctx.lib, ctx.h
        # ---- validity (NullBufferBuilder semantics: nothing is materialised until the first null arrives)
        src_valid = src["validity"]
        nulls_here = 0
        if src_valid is not None and src["null_count"] != 0:
            c = C.c_int64(0)
            ctx.check(lib.acu_bitmap_count(h, src_valid, src["validity_offset"] + offset, None, 0, n, C.byref(c)))
            nulls_here = n - c.value
        if nulls_here:
            if not self.valid_materialised:
                ctx.check(lib.acu_bitmap_fill(h, self.d_valid, 0, at, 1))
                self.valid_materialised = True
            ctx.check(lib.acu_bitmap_copy(h, src_valid, src["validity_offset"] + offset, self.d_valid, at, n, None))
            self.null_count += nulls_here
        elif self.valid_materialised:
            ctx.check(lib.acu_bitmap_fill(h, self.d_valid, at, n, 1))
        # ---- values
        if self.ob:
            s0, s1 = C.c_int64(0), C.c_int64(0)
            ctx.check(lib.acu_offsets_append(h, self.ob, src["values"], offset, n, self.data_len, self.d_values, at, C.byref(s0), C.byref(s1)))
            nbytes = s1.value - s0.value
            self._reserve_data(self.data_len + nbytes)
            if nbytes:
                ctx.check(lib.acu_memcpy_d2d(h, self.d_data + self.data_len, src["data"] + s0.value, nbytes))
            self.data_len += nbytes
        elif self.kind == BOOL:
            ctx.check(lib.acu_bitmap_copy(h, src["values"], src["values_offset"] + offset, self.d_values, at, n, None))
        else:
            ctx.check(lib.acu_memcpy_d2d(h, self.d_values + at * self.width, src["values"] + offset * self.width, n * self.width))

    def finish(self, rows):
        """Download the finished column (HostArray / Utf8Column) and start a fresh in-progress one."""
        ctx = self.ctx
        validity = ctx.d2h(self.d_valid, bitmap_bytes(rows)) if self.valid_materialised and self.null_count else None
        if self.ob:
            odt = np.int32 if self.ob == 4 else np.int64
            offs = ctx.d2h(self.d_values, (rows + 1) * self.ob, odt)
            data = ctx.d2h(self.d_data, self.data_len)
            out = Utf8Column(offs, data, HostArray(U8, np.zeros(0, np.uint8), rows, validity, 0, 0, self.null_count if validity is not None else 0))
            ctx.free(self.d_data)
        elif self.kind == BOOL:
            out = HostArray(BOOL, ctx.d2h(self.d_values, bitmap_bytes(rows)), rows, validity, 0, 0, self.null_count if validity is not None else 0)
        else:
            out = HostArray(self.kind, ctx.d2h(self.d_values, rows * self.width, NP_DTYPES[self.kind]), rows, validity, 0, 0,
                            self.null_count if validity is not None else 0)
        ctx.free(self.d_values)
        ctx.free(self.d_valid)
        self._fresh()
        return out

    def release(self):
        for p in (self.d_values, self.d_valid, getattr(self, "d_data", None)):
            if p:
                self.ctx.free(p)


class BatchCoalescer:
    """``BatchCoalescer::new(schema, target_batch_size)``; schema = one kind per column: an acu dtype code, acu.BOOL,
    "utf8" or "large_utf8"."""

    def __init__(self, ctx, schema, target_batch_size):
        assert target_batch_size > 0
        self.ctx, self.schema, self.target = ctx, list(schema), target_batch_size
        self.cols = [_Column(ctx, k, target_batch_size) for k in self.schema]
        self.buffered_rows = 0
        self.completed = deque()

    # -- device views of pushed columns -----------------------------------------------------------
    def _upload(self, columns, s):
        views = []
        for c in self.ctx._upload_columns(columns, s):
            views.append({"values": c.array.values, "values_offset": c.array.values_offset, "validity": c.array.validity,
                          "validity_offset": c.array.validity_offset, "null_count": c.array.null_count, "data": c.data})
        return views

    def _views_of_outs(self, columns, outs):
        views = []
        for col, o in zip(columns, outs):
            views.append({"values": o.array.values, "values_offset": 0, "validity": o.array.validity if o.array.has_validity else None,
                          "validity_offset": 0, "null_count": o.array.null_count if o.array.has_validity else 0, "data": o.data})
        return views

    def _check_columns(self, columns):
        if len(columns) != len(self.cols):  # coalesce.rs:475-481
            raise abi_error(f"Batch has {len(columns)} columns but BatchCoalescer expects {len(self.cols)}")

    # -- push ---------------------------------------------------------------------------------------
    def push_batch(self, columns):
        self._check_columns(columns)
        num_rows = columns[0].length if columns else 0
        with self.ctx._scope() as s:
            try:
                self._push_device(self._upload(columns, s), num_rows)
            finally:
                self.ctx.sync()

    def push_batch_with_filter(self, columns, predicate):
        self._check_columns(columns)
        ctx = self.ctx
        with ctx._scope() as s:
            try:
                cols = ctx._upload_columns(columns, s)
                plan = ctx._plan(s, predicate)
                count = ctx.lib.acu_filter_plan_count(plan)
                caps = [int(c.data.nbytes) if isinstance(c, Utf8Column) else 0 for c in columns]
                outs = ctx._alloc_column_outs(columns, count, caps, s)
                ctx.check(ctx.lib.acu_filter_record_batch(ctx.h, plan, len(columns), cols, outs))
                self._push_device(self._views_of_outs(columns, outs), count)
            finally:
                ctx.sync()

    def push_batch_with_indices(self, columns, indices):
        self._check_columns(columns)
        ctx = self.ctx
        with ctx._scope() as s:
            try:
                cols = ctx._upload_columns(columns, s)
                idd = s.upload(indices).descriptor()
                m = indices.length
                caps = []
                for c in columns:
                    if isinstance(c, Utf8Column):
                        lens = np.diff(c.offsets.astype(np.int64)) if len(c.offsets) > 1 else np.zeros(0, np.int64)
                        caps.append(int((lens.max() if lens.size else 0) * m))
                    else:
                        caps.append(0)
                outs = ctx._alloc_column_outs(columns, m, caps, s)
                ctx.check(ctx.lib.acu_take_record_batch(ctx.h, len(columns), cols, C.byref(idd), indices.dtype, 0, outs))
                self._push_device(self._views_of_outs(columns, outs), m)
            finally:
                ctx.sync()

    def _push_device(self, views, num_rows):
        """BatchCoalescer::push_batch (coalesce.rs:488-529) on device-resident columns."""
        offset = 0
        while num_rows > self.target - self.buffered_rows:
            remaining = self.target - self.buffered_rows
            for col, v in zip(self.cols, views):
                col.copy_rows(v, offset, remaining, self.buffered_rows)
            self.buffered_rows += remaining
            offset += remaining
            num_rows -= remaining
            self.finish_buffered_batch()
        if num_rows > 0:
            for col, v in zip(self.cols, views):
                col.copy_rows(v, offset, num_rows, self.buffered_rows)
        self.buffered_rows += num_rows
        if self.buffered_rows >= self.target:
            self.finish_buffered_batch()

    # -- output ---------------------------------------------------------------------------------------
    def get_buffered_rows(self):
        return self.buffered_rows

    def finish_buffered_batch(self):
        if self.buffered_rows == 0:
            return
        self.completed.append([c.finish(self.buffered_rows) for c in self.cols])
        self.buffered_rows = 0

    def is_empty(self):
        return self.buffered_rows == 0 and not self.completed

    def has_completed_batch(self):
        return bool(self.completed)

    def next_completed_batch(self):
        return self.completed.popleft() if self.completed else None

    def close(self):
        for c in self.cols:
            c.release()
        self.cols = []


def abi_error(message):
    from . import ArrowError
    return ArrowError(abi.ERR_INVALID_ARGUMENT, message)
