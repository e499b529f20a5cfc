"""CPU restatement of the reference's min / max of byte, view and fixed-size-binary columns and of boolean columns
(arrow-arith/src/aggregate.rs: min_max_helper :460-485, min_max_view_helper :491-518, min_boolean / max_boolean :372-457,
bool_and / bool_or :880-889), with the method names of acu.Context so that one test body runs on both backends.

TEST INFRASTRUCTURE: the checker, never the thing measured or shipped.

The reference folds the valid rows in ascending order and replaces its accumulator only on a strict < / >, so it returns
the LOWEST logical row holding the extremal value; values order like Rust's `&[u8]` (lexicographic on unsigned bytes, a
proper prefix first). The restatement below finds that row column-at-a-time with numpy: it keeps the valid rows whose
bytes are extremal at positions 0..p-1 and narrows them on byte p, where a value that has ended sorts before every byte.
When one row is left, or every remaining value has ended (they are then equal), the first remaining row is the answer.
Null slots are never read. tests/test_oracle_aggregate_bytes.py pins it against the literal fold and the golden vectors.
"""
import numpy as np

from acu import MAX, MIN, FixedSizeBinaryColumn, Utf8Column, column_value


def _valid_items(col):
    """(rows, flat, starts, lens) of the valid rows: the value of rows[k] is flat[starts[k] : starts[k] + lens[k]]."""
    rows = np.nonzero(col.nulls.valid_mask())[0]
    if isinstance(col, Utf8Column):
        offs = col.offsets.astype(np.int64)
        return rows, col.data, offs[rows], offs[rows + 1] - offs[rows]
    if isinstance(col, FixedSizeBinaryColumn):
        w = col.width
        return rows, col.values.reshape(-1), rows.astype(np.int64) * w, np.full(len(rows), w, dtype=np.int64)
    # views: the view slots followed by the data buffers, as one flat byte array
    views = np.ascontiguousarray(col.views).reshape(-1, 16)
    flat = np.concatenate([views.reshape(-1)] + list(col.buffers)) if len(col.buffers) else views.reshape(-1)
    base = np.cumsum([views.size] + [b.size for b in col.buffers])[:-1].astype(np.int64) if len(col.buffers) else np.zeros(0, np.int64)
    words = views[rows].copy().view(np.uint32)  # (len(rows), 4): length, prefix, buffer index, offset
    lens = words[:, 0].astype(np.int64)
    inline = lens <= 12
    starts = np.where(inline, rows.astype(np.int64) * 16 + 4, 0)
    if (~inline).any():
        starts[~inline] = base[words[~inline, 2].astype(np.int64)] + words[~inline, 3].astype(np.int64)
    return rows, flat, starts, lens


def arg_extreme(op, col):
    """(row, valid_count) of min (op = MIN) / max (MAX): the lowest row holding the extremal value, -1 = None."""
    rows, flat, starts, lens = _valid_items(col)
    if len(rows) == 0:
        return -1, 0
    flat = np.concatenate([np.asarray(flat, dtype=np.uint8).reshape(-1), np.zeros(1, np.uint8)])
    cand = np.arange(len(rows))
    p = 0
    while len(cand) > 1:
        ended = lens[cand] <= p
        b = np.where(ended, -1, flat[np.where(ended, 0, starts[cand] + p)].astype(np.int32))
        target = b.min() if op == MIN else b.max()
        cand = cand[b == target]
        if target == -1:  # every remaining value ended here: they are equal
            break
        p += 1
    return int(rows[cand[0]]), len(rows)


class AggregateOracle:
    """The CPU backend of the byte / boolean min and max (same method names as acu.Context)."""

    def min_max_row(self, op, col):
        return arg_extreme(op, col)

    def _min_max_value(self, op, col, as_str):
        row, _ = self.min_max_row(op, col)
        if row < 0:
            return None
        b = column_value(col, row)
        return b.decode() if as_str else b

    def min_string(self, col): return self._min_max_value(MIN, col, True)
    def max_string(self, col): return self._min_max_value(MAX, col, True)
    def min_binary(self, col): return self._min_max_value(MIN, col, False)
    def max_binary(self, col): return self._min_max_value(MAX, col, False)
    def min_string_view(self, col): return self._min_max_value(MIN, col, True)
    def max_string_view(self, col): return self._min_max_value(MAX, col, True)
    def min_binary_view(self, col): return self._min_max_value(MIN, col, False)
    def max_binary_view(self, col): return self._min_max_value(MAX, col, False)
    def min_fixed_size_binary(self, col): return self._min_max_value(MIN, col, False)
    def max_fixed_size_binary(self, col): return self._min_max_value(MAX, col, False)

    def aggregate_boolean(self, op, a):
        """(value, valid_count): min_boolean is false iff a valid slot is false, max_boolean true iff a valid slot is true."""
        valid = a.valid_mask()
        n_valid = int(valid.sum())
        if n_valid == 0:
            return -1, 0
        vals = a.value_array()[valid]
        return (int(vals.all()) if op == MIN else int(vals.any())), n_valid

    def _boolean_value(self, op, a):
        v, _ = self.aggregate_boolean(op, a)
        return None if v < 0 else bool(v)

    def min_boolean(self, a): return self._boolean_value(MIN, a)
    def max_boolean(self, a): return self._boolean_value(MAX, a)
    def bool_and(self, a): return self._boolean_value(MIN, a)
    def bool_or(self, a): return self._boolean_value(MAX, a)

