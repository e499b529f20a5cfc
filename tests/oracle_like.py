"""CPU restatement of arrow-string/src/like.rs (like_op / op_scalar / op_binary), predicate.rs (Predicate, regex_like) and
binary_like.rs, with the method names of acu.Context (like_bytes / like_view). TEST INFRASTRUCTURE: the checker.

regex_like is restated as a glob over Unicode scalars (bit-parallel NFA): `\\x` literal x, trailing `\\` a backslash, `%`
any run, `_` one scalar. Case-insensitive literals use simple case folding: an ASCII letter matches both cases, plus
U+212A (k) and U+017F (s); U+0131 folds with status T only and does not match i (so no str.upper / str.lower). op_scalar
runs the predicate at every slot and keeps the haystack's NullBuffer; ilike's fast paths need is_ascii, over
[offsets[0], offsets[len]) for Utf8 and over the valid slots for views. op_binary: a row with a null side is None (value
bit 0), NullBuffer iff some row is None. A non-ASCII ilike pattern is NotYetImplemented where the reference compiles it.
"""
import numpy as np

from acu import BOOL, ArrowError, HostArray, Utf8Column, column_value, pack_bits
from acu import _abi as abi

OP_NAMES = ["LIKE", "NLIKE", "ILIKE", "NILIKE", "CONTAINS", "STARTS_WITH", "ENDS_WITH", "EQ_IGNORE_ASCII_CASE"]
OPS = {"like": abi.LIKE, "nlike": abi.NLIKE, "ilike": abi.ILIKE, "nilike": abi.NILIKE, "contains": abi.CONTAINS,
       "starts_with": abi.STARTS_WITH, "ends_with": abi.ENDS_WITH, "eq_ignore_ascii_case": abi.EQ_IGNORE_ASCII_CASE}
ERR_INVALID_ARGUMENT, ERR_NOT_YET_IMPLEMENTED = 1, 7
FOLD_EXTRA = {"k": "K", "s": "ſ"}


# ---- regex_like as a glob ---------------------------------------------------------------------------------------------
def like_tokens(pattern):
    """regex_like's reading of a pattern (a str): ('lit', ch) / '%' / '_'."""
    out, i = [], 0
    while i < len(pattern):
        c = pattern[i]
        i += 1
        if c == "\\":
            if i < len(pattern):
                out.append(("lit", pattern[i]))
                i += 1
            else:
                out.append(("lit", "\\"))
        elif c in "%_":
            out.append(c)
        else:
            out.append(("lit", c))
    return out


def fold_class(c):
    """The scalars a case-insensitive literal c matches (simple case folding, ASCII pattern characters)."""
    if "a" <= c.lower() <= "z" and c.isascii():
        lo = c.lower()
        return {lo, lo.upper()} | ({FOLD_EXTRA[lo]} if lo in FOLD_EXTRA else set())
    return {c}


def glob_match(pattern, haystack, icase):
    """regex_like(pattern, icase).is_match(haystack), both str: a bit-parallel NFA walk over the haystack's scalars. State
    k (bit k) = the first k tokens are matched; a `%` state keeps itself on any scalar and passes to k + 1 unconsumed."""
    toks = []
    for t in like_tokens(pattern):
        if not (t == "%" and toks and toks[-1] == "%"):  # %% = %
            toks.append(t)
    pct = any_ = 0
    lit = {}
    for k, t in enumerate(toks):
        if t == "%":
            pct |= 1 << k
        elif t == "_":
            any_ |= 1 << k
        else:
            for c in (fold_class(t[1]) if icase else {t[1]}):
                lit[c] = lit.get(c, 0) | (1 << k)
    d = 1
    d |= (d & pct) << 1
    for ch in haystack:
        d = (((d & (any_ | lit.get(ch, 0))) << 1) | (d & pct))
        d |= (d & pct) << 1
        if not d:
            return False
    return bool(d >> len(toks) & 1)


def regex_like(pattern, end_anchor="$"):
    """regex_like's translation (predicate.rs:247-303) as a regex string; end_anchor=r"\\Z" gives the same regex for
    Python's `re`, whose `$` also matches before a final newline."""
    meta = set("\\.+*?()|[]{}^$#&-~")
    out, i = [], 0
    if pattern.startswith("%"):
        i = 1
    else:
        out.append("^")
    while i < len(pattern):
        c = pattern[i]
        i += 1
        if c == "\\":
            if i < len(pattern):
                n = pattern[i]
                i += 1
                out.append(("\\" if n in meta else "") + n)
            else:
                out.append("\\\\")
        elif c == "%":
            out.append(".*")
        elif c == "_":
            out.append(".")
        else:
            out.append(("\\" if c in meta else "") + c)
    s = "".join(out)
    return s[:-2] if s.endswith(".*") else s + end_anchor


# ---- predicate.rs -----------------------------------------------------------------------------------------------------
def has_wildcard(p):
    return any(c in p for c in "%_\\")


def predicate_like(p):
    if not has_wildcard(p):
        return ("eq", p)
    if p.endswith("%") and not has_wildcard(p[:-1]):
        return ("starts_with", p[:-1])
    if p.startswith("%") and not has_wildcard(p[1:]):
        return ("ends_with", p[1:])
    if p.startswith("%") and p.endswith("%") and not has_wildcard(p[1:-1]):
        return ("contains", p[1:-1])
    return ("regex", p)


def predicate_ilike(p, is_ascii):
    if is_ascii and p.isascii():
        if not has_wildcard(p):
            return ("ieq_ascii", p)
        if p.endswith("%") and not p.endswith("\\%") and not has_wildcard(p[:-1]):
            return ("istarts_with_ascii", p[:-1])
        if p.startswith("%") and not has_wildcard(p[1:]):
            return ("iends_with_ascii", p[1:])
    return ("iregex", p)


def evaluate(pred, hay):
    """Predicate::evaluate on haystack bytes (UTF-8 for the string predicates)."""
    kind, v = pred
    if kind == "regex" or kind == "iregex":
        return glob_match(v, hay.decode("utf-8"), kind == "iregex")
    nb = v.encode() if isinstance(v, str) else v
    if kind == "eq":
        return hay == nb
    if kind == "contains":
        return nb in hay
    if kind == "starts_with":
        return hay.startswith(nb)
    if kind == "ends_with":
        return hay.endswith(nb)
    if kind == "ieq_ascii":
        return len(hay) == len(nb) and hay.lower() == nb.lower()  # bytes.lower(): ASCII letters only
    if kind == "istarts_with_ascii":
        return len(hay) >= len(nb) and hay[:len(nb)].lower() == nb.lower()
    if kind == "iends_with_ascii":
        return len(hay) >= len(nb) and hay[len(hay) - len(nb):].lower() == nb.lower()
    raise ValueError(kind)


# ---- like_op ----------------------------------------------------------------------------------------------------------
def _slots(col):
    """(bytes at every slot, valid mask) of a Utf8Column / ViewColumn."""
    n = col.length
    return [column_value(col, i) for i in range(n)], col.nulls.valid_mask()


def _result(vals, valid, has_nulls, n):
    vals = np.asarray(vals, dtype=bool) if n else np.zeros(0, dtype=bool)
    if not has_nulls:
        return HostArray(BOOL, pack_bits(vals), n, None, 0, 0, 0)
    valid = np.asarray(valid, dtype=bool)
    return HostArray(BOOL, pack_bits(vals), n, pack_bits(valid), 0, 0, int(n - valid.sum()))


def _new_null(n):
    return _result([False] * n, [False] * n, True, n) if n else _result([], [], False, 0)


def like_op(op, l, r, is_utf8, is_view):
    ls, rs = bool(l.nulls.is_scalar), bool(r.nulls.is_scalar)
    if l.length != r.length and not ls and not rs:
        raise ArrowError(ERR_INVALID_ARGUMENT, f"Invalid argument error: Cannot compare arrays of different lengths, got {l.length} vs {r.length}")
    n = r.length if ls else l.length
    if not is_utf8 and op not in (abi.CONTAINS, abi.STARTS_WITH, abi.ENDS_WITH):
        raise ArrowError(ERR_INVALID_ARGUMENT, f"Invalid argument error: Invalid binary operation: {OP_NAMES[op]}")
    neg = op in (abi.NLIKE, abi.NILIKE)
    ilike = op in (abi.ILIKE, abi.NILIKE)
    nyi = f"Not yet implemented: {OP_NAMES[op]} with a non-ASCII pattern (full Unicode case folding)"
    lvals, lvalid = _slots(l)
    rvals, rvalid = _slots(r)
    if rs:  # op_scalar
        if not rvalid[0]:
            return _new_null(n)
        pat = rvals[0]
        if ilike and not pat.isascii():
            raise ArrowError(ERR_NOT_YET_IMPLEMENTED, nyi, -1)
        if n == 0:
            return _result([], [], False, 0)
        if op in (abi.LIKE, abi.NLIKE):
            pred = predicate_like(pat.decode())
        elif ilike:
            if is_view:  # GenericByteViewArray::is_ascii: the valid slots
                is_ascii = all(v.isascii() for v, ok in zip(lvals, lvalid) if ok)
            elif isinstance(l, Utf8Column):  # GenericByteArray::is_ascii: the whole [offsets[0], offsets[len]) range
                o = l.offsets
                is_ascii = bytes(l.data[int(o[0]):int(o[n])]).isascii()
            pred = predicate_ilike(pat.decode(), is_ascii)
        else:
            pred = ({abi.CONTAINS: "contains", abi.STARTS_WITH: "starts_with", abi.ENDS_WITH: "ends_with",
                     abi.EQ_IGNORE_ASCII_CASE: "ieq_ascii"}[op], pat)
        vals = [evaluate(pred, h) != neg for h in lvals]
        return _result(vals, lvalid, l.nulls.validity is not None, n)
    # op_binary
    if n == 0:
        return _result([], [], False, 0)
    vals, valid = [], []
    for i in range(n):
        li = 0 if ls else i
        ok = bool(lvalid[li]) and bool(rvalid[i])
        valid.append(ok)
        if not ok:
            vals.append(False)
            continue
        h, p = lvals[li], rvals[i]
        if op in (abi.LIKE, abi.NLIKE):
            m = evaluate(predicate_like(p.decode()), h)
        elif ilike:
            if not p.isascii():
                raise ArrowError(ERR_NOT_YET_IMPLEMENTED, nyi, i)
            m = evaluate(("iregex", p.decode()), h)
        else:
            m = evaluate(({abi.CONTAINS: "contains", abi.STARTS_WITH: "starts_with", abi.ENDS_WITH: "ends_with",
                           abi.EQ_IGNORE_ASCII_CASE: "ieq_ascii"}[op], p), h)
        vals.append(m != neg)
    return _result(vals, valid, not all(valid), n)


class LikeOracle:
    """The CPU backend of the LIKE family (same method names as acu.Context)."""

    def like_bytes(self, op, a, b, is_utf8=True):
        return like_op(op, a, b, is_utf8, False)

    def like_view(self, op, a, b, is_utf8=True):
        return like_op(op, a, b, is_utf8, True)
