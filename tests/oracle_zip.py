"""Python oracle for zip(mask, truthy, falsy) (arrow-select/src/zip.rs) of Utf8 / Binary / LargeUtf8 / LargeBinary
(acu.Utf8Column), Utf8View / BinaryView (acu.ViewColumn), Boolean (acu.HostArray) and FixedSizeBinary
(acu.FixedSizeBinaryColumn) operands, restated with numpy so that it also runs at the sizes the device tests use.

Three paths, as the reference:
  zip_impl            MutableArrayData (arrow-data/src/transform): row i is row i of the chosen side (row 0 of a scalar), its
                      bytes and bits under nulls included; a NullBuffer iff some input has a null, dropped when the result has
                      none. Byte offsets are rebased (try_extend_offsets: an i32 end past i32::MAX is an InvalidArgumentError at
                      that row); a falsy view longer than 12 bytes gets its buffer index raised by truthy's buffer count.
  BytesScalarImpl     two Utf8 / Binary scalars.
  ByteViewScalarImpl  two view scalars.
Boolean and FixedSizeBinary with two scalars take FallbackImpl, which is zip_impl.

A result is a ZipResult: `valid` is the NullBuffer as a bool array, or None when there is none."""
import numpy as np

from acu import FixedSizeBinaryColumn, HostArray, Utf8Column, ViewColumn
from acu import _abi as abi

from oracle_filter_take import EXTEND_OVERFLOW, OracleError

I32_MAX = (1 << 31) - 1


class ZipResult:
    def __init__(self, kind, n, valid, **kw):
        self.kind, self.n, self.valid = kind, n, valid
        self.offsets = kw.get("offsets")   # bytes: np.int32 / np.int64, n + 1
        self.data = kw.get("data")         # bytes: np.uint8 (None when not built)
        self.views = kw.get("views")       # view: (n, 16) uint8
        self.buffers = kw.get("buffers")   # view: abi.ZIP_BUFFERS_*
        self.values = kw.get("values")     # Boolean: bool (n); FixedSizeBinary: (n, W) uint8


def _nulls(col):
    return col if isinstance(col, HostArray) else col.nulls


def is_scalar(col):
    return bool(_nulls(col).is_scalar)


def _valid(col):
    return _nulls(col).valid_mask()


def _has_null(col):
    return not _valid(col).all()


def selection(mask):
    """maybe_prep_null_mask_filter (zip.rs:662-671): a null mask slot counts as false."""
    return mask.value_array() & mask.valid_mask()


def _spread(x, scalar, n):
    """Row i of a side: x[i], or x[0] for a scalar."""
    return np.repeat(x[:1], n, axis=0) if scalar else x[:n]


def _check(mask, t, f):
    n = mask.length
    for side in (t, f):  # zip.rs:123-145; ScalarZipper::try_new (zip.rs:288-297) uses the same text
        if is_scalar(side) and _nulls(side).length != 1:
            raise OracleError(abi.ERR_INVALID_ARGUMENT, "scalar arrays must have 1 element")
        if not is_scalar(side) and _nulls(side).length != n:
            raise OracleError(abi.ERR_INVALID_ARGUMENT, "all arrays should have the same length")


def _impl_valid(sel, t, f, n):
    """zip_impl's NullBuffer: built iff some input has a null, dropped when the result has none."""
    if not (_has_null(t) or _has_null(f)):
        return None
    v = np.where(sel, _spread(_valid(t), is_scalar(t), n), _spread(_valid(f), is_scalar(f), n))
    return None if v.all() else v


def _build_bytes(ob, sel_t, t_start, t_len, f_start, f_len, t_data, f_data, data):
    lens = np.where(sel_t, t_len, f_len).astype(np.int64)
    offs = np.zeros(len(lens) + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    out = None
    if data:
        buf = np.concatenate([np.asarray(t_data, np.uint8), np.asarray(f_data, np.uint8)])
        starts = np.where(sel_t, t_start, f_start + len(t_data)).astype(np.int64)
        idx = np.repeat(starts - offs[:-1], lens) + np.arange(int(offs[-1]), dtype=np.int64)
        out = buf[idx]
    return offs.astype(np.int32 if ob == 4 else np.int64), out


def _rows(col, n):
    o = np.asarray(col.offsets, np.int64)
    return _spread(o[:-1], is_scalar(col), n), _spread(np.diff(o), is_scalar(col), n)


def zip_bytes(mask, t, f, data=True):
    """data=False: the offsets, validity and errors alone (result.data None)."""
    _check(mask, t, f)
    ob, n, sel = t.offsets.dtype.itemsize, mask.length, selection(mask)
    ts_, tl = _rows(t, n)
    fs_, fl = _rows(f, n)
    if not (is_scalar(t) and is_scalar(f)):
        lens = np.where(sel, tl, fl)
        ends = np.cumsum(lens)
        if ob == 4 and n and ends[-1] > I32_MAX:
            raise OracleError(abi.ERR_INVALID_ARGUMENT, EXTEND_OVERFLOW, int(np.argmax(ends > I32_MAX)))
        offs, d = _build_bytes(ob, sel, ts_, tl, fs_, fl, t.data, f.data, data)
        return ZipResult("bytes", n, _impl_valid(sel, t, f, n), offsets=offs, data=d)
    # BytesScalarImpl::create_output (zip.rs:622-660)
    t_ok, f_ok = not _has_null(t), not _has_null(f)
    cnt = int(sel.sum())
    if t_ok and f_ok:
        valid, pick = None, sel
    elif t_ok:  # the value where the predicate holds, empty null rows elsewhere
        valid, pick = sel.copy(), sel
        fl = np.zeros(n, np.int64)
    elif f_ok:
        valid, pick = ~sel, sel
        tl = np.zeros(n, np.int64)
    else:
        valid, pick = np.zeros(n, bool), sel
        tl, fl = np.zeros(n, np.int64), np.zeros(n, np.int64)
    total = int(np.where(pick, tl, fl).sum())
    if ob == 4 and total > I32_MAX:
        mixed = t_ok and f_ok and 0 < cnt < n  # OffsetBufferBuilder::finish, else from_repeated_length / from_lengths
        raise OracleError(abi.ERR_PANIC_OUT_OF_BOUNDS, "overflow" if mixed else "offset overflow")
    offs, d = _build_bytes(ob, pick, ts_, tl, fs_, fl, t.data, f.data, data)
    return ZipResult("bytes", n, valid, offsets=offs, data=d)


def _u32(views):
    return np.ascontiguousarray(views, np.uint8).reshape(-1, 16).view(np.uint32)


def _rebase(views, add, inline_too=False):
    """views with buffer_index += add (wrapping u32) on every view longer than 12 bytes (every view when inline_too)."""
    v = _u32(views).copy()
    long_ = np.ones(len(v), bool) if inline_too else v[:, 0] > 12
    v[long_, 2] = (v[long_, 2].astype(np.uint64) + add) & 0xFFFFFFFF
    return v.view(np.uint8).reshape(-1, 16)


def zip_view(mask, t, f):
    _check(mask, t, f)
    n, sel = mask.length, selection(mask)
    nt, nf = len(t.buffers), len(f.buffers)
    tv = _spread(np.asarray(t.views, np.uint8).reshape(-1, 16), is_scalar(t), n)
    fv = _spread(np.asarray(f.views, np.uint8).reshape(-1, 16), is_scalar(f), n)
    if not (is_scalar(t) and is_scalar(f)):  # build_extend_view (transform/mod.rs:222-239), nulls included
        views = np.where(sel[:, None], tv, _rebase(fv, nt))
        return ZipResult("view", n, _impl_valid(sel, t, f, n), views=views, buffers=abi.ZIP_BUFFERS_BOTH)
    # ByteViewScalarImpl::create_output (zip.rs:820-860)
    t_ok, f_ok = not _has_null(t), not _has_null(f)
    cnt = int(sel.sum())
    zeros = np.zeros((n, 16), np.uint8)
    if t_ok and f_ok:
        if cnt == 0:
            return ZipResult("view", n, None, views=fv, buffers=abi.ZIP_BUFFERS_FALSY)
        if cnt == n:
            return ZipResult("view", n, None, views=tv, buffers=abi.ZIP_BUFFERS_TRUTHY)
        if nf:  # the falsy view is re-based even when it is inline (zip.rs:759-769)
            return ZipResult("view", n, None, views=np.where(sel[:, None], tv, _rebase(fv, nt, True)), buffers=abi.ZIP_BUFFERS_BOTH)
        return ZipResult("view", n, None, views=np.where(sel[:, None], tv, fv), buffers=abi.ZIP_BUFFERS_TRUTHY)
    if t_ok:
        return (ZipResult("view", n, sel.copy(), views=tv, buffers=abi.ZIP_BUFFERS_TRUTHY) if cnt
                else ZipResult("view", n, np.zeros(n, bool), views=zeros, buffers=abi.ZIP_BUFFERS_NONE))
    if f_ok:
        return (ZipResult("view", n, ~sel, views=fv, buffers=abi.ZIP_BUFFERS_FALSY) if n - cnt
                else ZipResult("view", n, np.zeros(n, bool), views=zeros, buffers=abi.ZIP_BUFFERS_NONE))
    return ZipResult("view", n, np.zeros(n, bool), views=zeros, buffers=abi.ZIP_BUFFERS_NONE)


def zip_boolean(mask, t, f):
    _check(mask, t, f)
    n, sel = mask.length, selection(mask)
    vals = np.where(sel, _spread(t.value_array(), t.is_scalar, n), _spread(f.value_array(), f.is_scalar, n))
    return ZipResult("boolean", n, _impl_valid(sel, t, f, n), values=vals)


def zip_fixed_size_binary(mask, t, f):
    _check(mask, t, f)
    n, sel = mask.length, selection(mask)
    vals = np.where(sel[:, None], _spread(t.values, is_scalar(t), n), _spread(f.values, is_scalar(f), n))
    return ZipResult("fsb", n, _impl_valid(sel, t, f, n), values=vals.reshape(n, t.width))


def data_type(col):
    if isinstance(col, Utf8Column):
        return ("bytes", col.offsets.dtype.itemsize)
    if isinstance(col, ViewColumn):
        return ("view",)
    if isinstance(col, FixedSizeBinaryColumn):
        return ("fsb", col.width)
    return ("array", col.dtype)


def zip(mask, t, f, data=True):
    if data_type(t) != data_type(f):
        raise OracleError(abi.ERR_INVALID_ARGUMENT, "arguments need to have the same data type")
    if isinstance(t, Utf8Column):
        return zip_bytes(mask, t, f, data)
    if isinstance(t, ViewColumn):
        return zip_view(mask, t, f)
    if isinstance(t, FixedSizeBinaryColumn):
        return zip_fixed_size_binary(mask, t, f)
    return zip_boolean(mask, t, f)
