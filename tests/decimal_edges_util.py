"""Boundary inputs for the decimal arithmetic and cast kernels, with a closed form of every row in exact Python arithmetic.

Each family is one operation at one type (an op and its operand types, a cast and its source / target types). Its inputs
sit where the kernels switch between code paths: native MIN / MAX and one beyond, the rescale products at
floor(MAX / 10^k), the 64-bit limb boundaries of the i128 multiply and divide (2^63, 2^64, 2^127), the chunk counts of the
full-width division by 10^k, exact rounding ties, and the bit lengths of the i128 -> f64 conversion. A family's rows are
split into `ok` (the closed form gives a value) and `fail` (the closed form gives FAIL), so that one call can check every
`ok` row and each `fail` row can be placed on its own after a prefix of `ok` rows.

The closed forms here restate the operations from their definitions (range checks on Python ints, `fractions.Fraction`
for rounding half away from zero, `float(int)` for the correctly rounded int -> f64) rather than from tests/oracle_decimal*.py,
so a misreading shared by the oracle and the kernels shows up as a disagreement with them."""
import math
from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

ADD, SUB, MUL, DIV, REM = 1, 3, 5, 6, 7          # acu_arith_op values (ADD_WRAPPING .. REM = 0 .. 7)
I8, I16, I32, I64, U8, U16, U32, U64, F32, F64 = range(10)
INTS = [I8, I16, I32, I64, U8, U16, U32, U64]
INT_BOUNDS = {I8: (-2 ** 7, 2 ** 7 - 1), I16: (-2 ** 15, 2 ** 15 - 1), I32: (-2 ** 31, 2 ** 31 - 1),
              I64: (-2 ** 63, 2 ** 63 - 1), U8: (0, 2 ** 8 - 1), U16: (0, 2 ** 16 - 1), U32: (0, 2 ** 32 - 1),
              U64: (0, 2 ** 64 - 1)}
WIDTHS = [4, 8, 16]
MAXP = {4: 9, 8: 18, 16: 38}
FAIL = object()
PREFIX = 5  # ok rows ahead of each failing row


def native(w):
    """(MIN, MAX) of the w-byte two's complement native."""
    return -(1 << (8 * w - 1)), (1 << (8 * w - 1)) - 1


def in_native(w, v):
    lo, hi = native(w)
    return lo <= v <= hi


def trunc_q(a, b):
    """a / b truncated toward zero."""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def round_half_away(f: Fraction):
    q = math.floor(abs(f) + Fraction(1, 2))
    return q if f >= 0 else -q


@dataclass
class Family:
    kind: str                  # "arith" | "neg" | "dec" | "to_dec" | "from_dec"
    args: tuple                # the operation's parameters (see the builders)
    ok: list = field(default_factory=list)
    exp: list = field(default_factory=list)   # closed-form result of each ok row
    fail: list = field(default_factory=list)
    unary: bool = False        # a failing row fails whatever `safe` is (the reference's `unary(..).unwrap()`)

    @property
    def name(self):
        return f"{self.kind}{self.args}"

    def prefix(self):
        return self.ok[:PREFIX]


# ---- closed forms ----------------------------------------------------------------------------------------------------------
def arith_row(op, w, s1, s2, l, r):
    """decimal add / sub / mul / div / rem of Decimal(w)(_, s1) l and (_, s2) r: both operands brought to the result's
    scale by exact multiplication (each product range-checked), then the exact op, range-checked; div truncates."""
    mp = MAXP[w]
    if op == MUL:
        v = l * r
        return v if in_native(w, v) else FAIL
    if op == DIV:
        e = min(s1 + 4, mp) - s1 + s2
        lm, rm = (10 ** e, 1) if e >= 0 else (1, 10 ** -e)
    else:
        rs = max(s1, s2)
        lm, rm = 10 ** (rs - s1), 10 ** (rs - s2)
    L, R = l * lm, r * rm
    if not (in_native(w, L) and in_native(w, R)):
        return FAIL
    if op in (ADD, SUB):
        v = L + R if op == ADD else L - R
        return v if in_native(w, v) else FAIL
    if R == 0:
        return FAIL
    q = trunc_q(L, R)
    if not in_native(w, q):
        return FAIL
    return q if op == DIV else L - q * R


def dec_mode(wi, p_in, s_in, wo, p_out, s_out):
    """'clone' | 'zero' | 'unary' | 'checked': which combinator cast_decimal_to_decimal applies (for the plain types used
    here: 0 <= scales, precisions within the widths' tables)."""
    if wi == wo and s_in == s_out and p_in <= p_out:
        return "clone"
    if s_out >= s_in:
        return "unary" if p_in + (s_out - s_in) <= p_out else "checked"
    if s_in - s_out > MAXP[wi]:
        return "zero"
    return "unary" if p_in - (s_in - s_out) < p_out else "checked"


def dec_row(wi, p_in, s_in, wo, p_out, s_out, x):
    """Decimal -> decimal of one value x (a wi-byte native): upscale = x * 10^k (wrapping when unary), downscale = x / 10^k
    rounded half away from zero; the result must fit the wo-byte native and, when checked, p_out digits."""
    mode = dec_mode(wi, p_in, s_in, wo, p_out, s_out)
    if mode == "clone":
        return x
    if mode == "zero":
        return 0
    if s_out >= s_in:
        if not in_native(wo, x):
            return FAIL
        v = x * 10 ** (s_out - s_in)
        if mode == "unary":
            lo, _ = native(wo)
            return (v - lo) % (1 << (8 * wo)) + lo
        if not in_native(wo, v):
            return FAIL
    else:
        v = round_half_away(Fraction(x, 10 ** (s_in - s_out)))
        if not in_native(wo, v):
            return FAIL
    if mode == "checked" and abs(v) > 10 ** p_out - 1:
        return FAIL
    return v


def f64_scale(s):
    """10^s as the f64 the casts multiply / divide by, for |s| <= 22 (there it is the correctly rounded 10^s)."""
    assert abs(s) <= 22
    return float(Fraction(10) ** s)


def to_dec_row(dtype, w, p, s, x):
    """Integer / float x -> Decimal(w)(p, s). Integers: x * 10^s (x first narrowed to the native, the product
    range-checked), or x / 10^-s truncated; floats: one IEEE multiply by 10^s, rounded half away from zero, then the
    native's range. The result must have at most p digits."""
    if dtype in (F32, F64):
        m = x * f64_scale(s)
        if math.isnan(m) or math.isinf(m):
            return FAIL
        v = round_half_away(Fraction(m))
        lo, hi = native(w)
        if not lo <= v <= hi:
            return FAIL
    elif s < 0:
        f = 10 ** -s
        lo, hi = INT_BOUNDS[dtype]
        if f > hi:
            return 0
        v = trunc_q(x, f)
        if not in_native(w, v):
            return FAIL
    else:
        if not in_native(w, x) or not in_native(w, x * 10 ** s):
            return FAIL
        v = x * 10 ** s
    return v if abs(v) <= 10 ** p - 1 else FAIL


def from_dec_row(w, s, to, x):
    """Decimal(w)(_, s) x -> integer type `to` (x / 10^s truncated, or x * 10^-s range-checked in the native, then the
    type's range) or float: float(x) / 10^s, with Float32 the f64 rounded again."""
    if to == F64:
        return float(x) / f64_scale(s)
    if to == F32:
        return float(np.float32(float(x) / f64_scale(s)))
    v = trunc_q(x, 10 ** s) if s >= 0 else x * 10 ** -s
    if not in_native(w, v):
        return FAIL
    lo, hi = INT_BOUNDS[to]
    return v if lo <= v <= hi else FAIL


def neg_row(w, v):
    return -v if in_native(w, -v) else FAIL


# ---- inputs ----------------------------------------------------------------------------------------------------------------
def full_width(rng, w, n):
    """n random w-byte natives: full bit patterns, and each shifted right by a random amount (every magnitude)."""
    raw = rng.bytes(w * n)
    out = []
    for i in range(n):
        v = int.from_bytes(raw[i * w:(i + 1) * w], "little", signed=True)
        out.append(v if i % 2 == 0 else v >> int(rng.integers(0, 8 * w)))
    return out


def around(*centres, d=1):
    """Every c - d .. c + d."""
    return [c + k for c in centres for k in range(-d, d + 1)]


def limb_edges():
    """±(2^63 - 1), ±2^63, ±2^64 and their neighbours: the i64 fast paths and the 64-bit limb boundaries."""
    return sorted({s * v for v in around(2 ** 63, 2 ** 64) for s in (1, -1)})


def split(fam: Family, inputs, row_fn, max_fail=None):
    """Append each input to ok (with its closed form) or fail; the fail list keeps at most max_fail rows, evenly spread."""
    seen_ok, fails = set(fam.ok), []
    for x in inputs:
        v = row_fn(x)
        if v is FAIL:
            fails.append(x)
        elif x not in seen_ok:
            seen_ok.add(x)
            fam.ok.append(x)
            fam.exp.append(v)
    fails = list(dict.fromkeys(fails))
    if max_fail is not None and len(fails) > max_fail:
        fails = [fails[int(i)] for i in np.linspace(0, len(fails) - 1, max_fail)]
    fam.fail += fails
    return fam


# ---- arithmetic ------------------------------------------------------------------------------------------------------------
def add_sub_families():
    """Results at MAX, MIN, MAX + 1, MIN - 1; and for every rescale exponent d the scale range allows, the rescaled
    operand at floor(MAX / 10^d) / ceil(MIN / 10^d) and one beyond, on the left and on the right."""
    fams = []
    for w in WIDTHS:
        lo, hi = native(w)
        mp = MAXP[w]
        for op in (ADD, SUB):
            sg = 1 if op == ADD else -1
            pairs = []
            for t in (hi, lo, hi + 1, lo - 1, hi - 1, lo + 1):
                for a in (0, 1, -1, 2, 7, hi // 3, lo // 2, t // 2, t - hi, t - lo):
                    b = sg * (t - a)
                    if in_native(w, a) and in_native(w, b):
                        pairs += [(a, b), (b, a) if op == ADD else (a, b)]
            pairs += [(hi, hi), (lo, lo), (hi, lo), (lo, hi), (0, lo), (-1, lo), (-1, hi), (0, hi)]
            fams.append(split(Family("arith", (op, w, mp, 0, mp, 0)), pairs, lambda x, op=op, w=w: arith_row(op, w, 0, 0, *x)))
            for d in range(1, mp + 1):
                if 10 ** d > hi:
                    break
                q_hi, q_lo = hi // 10 ** d, -((-lo) // 10 ** d)
                edge = around(q_hi, q_lo)
                for left in (True, False):  # the rescaled operand on the left (s1 = 0 < s2 = d) or on the right
                    s1, s2 = (0, d) if left else (d, 0)
                    pairs = [(v, 0) if left else (0, v) for v in edge]
                    pairs += [(q_hi, 5), (q_lo, -5)] if left else [(5, q_hi), (-5, q_lo)]
                    fams.append(split(Family("arith", (op, w, mp, s1, mp, s2)), pairs,
                                      lambda x, op=op, w=w, s1=s1, s2=s2: arith_row(op, w, s1, s2, *x)))
    return fams


def mul_families():
    """Decimal128: a pair on each side of every branch of the i128 multiply (both in i64; both with a high limb; the
    cross term's overflow; the carry into the high limb; the final range test, 2^127 legal only for a negative result),
    with operands at ±2^63 and ±2^64; Decimal32 / 64: products at the native MIN / MAX and one beyond."""
    fams = []
    for w in WIDTHS:
        lo, hi = native(w)
        mp = MAXP[w]
        pairs = []
        mults = [1, 2, 3, 7, 10, 11, 127, 1 << 16, (1 << 16) + 1, 46341, 3037000499, 3037000500]
        if w == 16:
            mults += [2 ** 31, 2 ** 32 - 1, 2 ** 32, 2 ** 63 - 1, 2 ** 63, 2 ** 63 + 1, 2 ** 64 - 1, 2 ** 64, 2 ** 64 + 1,
                      13043817825332782212, 2 ** 96, 2 ** 97]
        for a in mults:
            if not in_native(w, a):
                continue
            for t in (hi, lo):
                q = t // a
                for b in around(q, -q):
                    pairs += [(a, b), (b, a), (-a, b)]
        if w == 16:
            e = limb_edges()
            pairs += [(a, b) for a in e for b in e]
            m = 2 ** 127 - 1
            pairs += [(m, 1), (m, -1), (-m, 1), (-m, -1), (1, m), (lo, 1), (lo, -1), (1, lo), (-1, lo)]
            pairs += [(s * 2 ** 64, t * 2 ** 63) for s in (1, -1) for t in (1, -1)]          # |product| = 2^127
            pairs += [(s * 2 ** 63, t * 2 ** 64) for s in (1, -1) for t in (1, -1)]
            pairs += [(s * 2 ** 96, t * 2 ** 31) for s in (1, -1) for t in (1, -1)]          # 2^127 via the cross term
            pairs += [(2 ** 96, 2 ** 32), (2 ** 97, 2 ** 32 - 1), (2 ** 96, 2 ** 31 - 1)]   # cross term over 64 bits
            pairs += [(2 ** 65 - 1, 2 ** 64 - 1), (2 ** 64 + 2 ** 63, 2 ** 63 - 1), (2 ** 64 + 1, 2 ** 63 - 1),
                      (2 ** 64 + 1, 2 ** 63), (-(2 ** 64 + 1), 2 ** 63)]                    # the carry into the high limb
            pairs += [(s * (2 ** 64 + k), t * (2 ** 64 + j)) for s in (1, -1) for t in (1, -1) for k in (0, 1) for j in (0, 5)]
        pairs = [p for p in pairs if in_native(w, p[0]) and in_native(w, p[1])]
        fams.append(split(Family("arith", (MUL, w, mp, 0, mp, 0)), pairs, lambda x, w=w: arith_row(MUL, w, 0, 0, *x)))
    return fams


def div_rem_families(rng):
    """l, r at ±(2^63 - 1), ±2^63, ±2^64 (the i64 fast path against the software division), r = ±1, MIN / -1 and
    MIN % -1 (one row each), zero divisors, and a rescaled l (div's l * 10^4) at floor(MAX / 10^4) and one beyond."""
    fams = []
    for w in WIDTHS:
        lo, hi = native(w)
        mp = MAXP[w]
        vals = [1, -1, 2, -2, 3, -7, 10, hi, lo + 1, -hi, hi // 2, lo // 3] + full_width(rng, w, 8)
        if w == 16:
            vals += limb_edges() + [10 ** 19, -(10 ** 19), 2 ** 100 + 12345, -(2 ** 90)]
        else:
            vals += around(hi // 2, lo // 2, 2 ** (4 * w - 1))
        vals = [v for v in dict.fromkeys(vals) if in_native(w, v)]
        for op in (DIV, REM):
            # DIV at scale (mp, mp) / (mp, 0) keeps its operands (result scale mp, no rescale); REM at equal scales too
            s1 = mp if op == DIV else 0
            pairs = [(a, b) for a in vals for b in vals] + [(7, 0), (lo, 0)]
            pairs = [p for p in pairs if p != (lo, -1)] + [(lo, -1)]
            fam = split(Family("arith", (op, w, mp, s1, mp, 0)), pairs, lambda x, op=op, w=w, s1=s1: arith_row(op, w, s1, 0, *x))
            fams.append(fam)
        q = hi // 10 ** 4
        edge = around(q, -q, -((-lo) // 10 ** 4))
        pairs = [(v, r) for v in edge for r in (1, -1, 3, 10 ** 4, hi)]
        fams.append(split(Family("arith", (DIV, w, mp, 0, mp, 0)), pairs, lambda x, w=w: arith_row(DIV, w, 0, 0, *x)))
    return fams


def neg_families(rng):
    fams = []
    for w in WIDTHS:
        lo, hi = native(w)
        vals = [hi, lo + 1, 0, 1, -1] + full_width(rng, w, 16) + [lo]
        fams.append(split(Family("neg", (w, MAXP[w], 0)), vals, lambda x, w=w: neg_row(w, x)))
    return fams


# ---- decimal -> decimal ----------------------------------------------------------------------------------------------------
def dec_inputs(rng, wi, wo, k, down, p_out):
    """Dividends / multiplicands for a scale change by k digits."""
    lo, hi = native(wi)
    olo, ohi = native(wo)
    vals = full_width(rng, wi, 12) + [hi, lo, -hi, 0, 1, -1]
    if down:
        K = 10 ** k
        half = K // 2
        vals += [hi - half, -(hi - half), lo + half]
        for q in [0, 1, 2, 7, hi // K, hi // K - 1, (10 ** p_out - 1), ohi, olo] + [int(x) for x in rng.integers(0, 2 ** 62, 3)]:
            for s in (1, -1):
                vals += [s * (q * K + half), s * (q * K + half - 1), s * (q * K + half + 1)]
        # a rounded result at exactly the output native's MIN / MAX and one beyond
        vals += [ohi * K + half - 1, ohi * K + half, olo * K - half + 1, olo * K - half, (10 ** p_out - 1) * K + half - 1,
                 (10 ** p_out - 1) * K + half]
    else:
        K = 10 ** k
        for m in (ohi, olo, 10 ** p_out - 1):
            q = m // K if m > 0 else -((-m) // K)
            vals += around(q, d=1) + [-q, -q - 1]
        vals += around(ohi, olo)
    return [v for v in dict.fromkeys(vals) if lo <= v <= hi]


def dec_families(rng):
    """Every width pair, every scale change from -38 to +38 digits the pair allows (downscale by k: input scale k, output
    scale 0; upscale by k: input scale 0, output scale k), at full input and output precision; plus, per pair, small
    changes at the smallest input precision the input scale allows, where the unary (unchecked) path runs on values beyond that precision and only the
    output native's range is checked."""
    fams = []
    for wi in WIDTHS:
        for wo in WIDTHS:
            mi, mo = MAXP[wi], MAXP[wo]
            for k in range(-mo, mi + 1):  # k > 0: downscale by k; k < 0: upscale by -k
                down = k > 0
                s_in, s_out = (k, 0) if down else (0, -k)
                args = (wi, mi, s_in, wo, mo, s_out)
                fam = Family("dec", args, unary=dec_mode(*args) == "unary")
                fams.append(split(fam, dec_inputs(rng, wi, wo, abs(k), down, mo), lambda x, a=args: dec_row(*a, x), max_fail=6))
            for k in (-1, 0, 1, 2):
                down = k > 0
                s_in, s_out = (k, 0) if down else (0, -k)
                args = (wi, max(1, s_in), s_in, wo, mo, s_out)
                if dec_mode(*args) != "unary":
                    continue
                fam = Family("dec", args, unary=True)
                fams.append(split(fam, dec_inputs(rng, wi, wo, abs(k), down, mo), lambda x, a=args: dec_row(*a, x), max_fail=6))
    return fams


# ---- integer / float -> decimal ----------------------------------------------------------------------------------------------
def int_to_dec_families():
    """Each integer type into each width, scales -(mp + 1) .. mp + 1 at full precision: the type's MIN / MAX, the
    multiplicands at floor(MAX_out / 10^s) and floor((10^mp - 1) / 10^s) and one beyond, and for negative scales values
    around multiples of 10^-s."""
    fams = []
    for dt in INTS:
        tlo, thi = INT_BOUNDS[dt]
        for w in WIDTHS:
            mp = MAXP[w]
            olo, ohi = native(w)
            for s in range(-(mp + 1), mp + 2):
                if s >= 0 and 10 ** s > ohi:
                    continue  # a type-level error ("the scale causes overflow"), no rows
                vals = [tlo, thi, tlo + 1, thi - 1, 0, 1]
                if s >= 0:
                    for m in (ohi, olo, 10 ** mp - 1, -(10 ** mp - 1)):
                        q = abs(m) // 10 ** s
                        vals += around(q if m > 0 else -q)
                    vals += around(ohi, olo)
                else:
                    f = 10 ** -s
                    vals += around(f, -f, thi // f * f, tlo // f * f, (10 ** mp) * f, -(10 ** mp) * f)
                vals = [v for v in dict.fromkeys(vals) if tlo <= v <= thi]
                args = (dt, w, mp, s)
                fams.append(split(Family("to_dec", args), vals, lambda x, a=args: to_dec_row(*a, x), max_fail=4))
    return fams


def nexts(x, n=2, f32=False):
    """x and its n neighbouring floats on each side (in Float32 when f32)."""
    t = np.float32 if f32 else np.float64
    with np.errstate(over="ignore"):
        out, up, dn = [t(x)], t(x), t(x)
        for _ in range(n):
            up, dn = np.nextafter(up, t(np.inf)), np.nextafter(dn, t(-np.inf))
            out += [up, dn]
    return [float(v) for v in out]


def float_to_dec_families(rng):
    """Float64 / Float32 into each width at scales 0, 1, 2, 3, 7 and -1, -3: values on both sides of 2^31, 2^63 and
    2^127 (scaled back by 10^s), of 10^p - 1 at the output precision, and ties: inputs whose product with 10^s is exactly
    k + 0.5, with the neighbouring floats."""
    fams = []
    for dt in (F64, F32):
        f32 = dt == F32
        for w in WIDTHS:
            mp = MAXP[w]
            for s in (0, 1, 2, 3, 7, -1, -3):
                fk = f64_scale(s)
                centres = []
                for e in (31, 63, 127):
                    centres += [2.0 ** e / fk, -(2.0 ** e) / fk, (2.0 ** e - 1) / fk]
                centres += [(10.0 ** mp - 1) / fk, -(10.0 ** mp - 1) / fk, 10.0 ** mp / fk]
                if s >= 0:  # x = m / 2^(s+1), m odd: x * 10^s = m * 5^s / 2 is exactly an odd multiple of 1/2
                    ms = [1, 3, 5, 2 ** 20 + 1] + [int(v) | 1 for v in rng.integers(1, 2 ** 40 // 5 ** s, 6)]
                    centres += [sg * m / 2 ** (s + 1) for m in ms for sg in (1, -1)]
                vals = []
                for c in centres:
                    vals += nexts(c, 2, f32)
                vals += [float(np.float32(v)) if f32 else float(v) for v in rng.standard_normal(8) * 10.0 ** rng.integers(-2, mp // 2 + 1, 8)]
                vals += [math.inf, -math.inf, math.nan, 0.0, -0.0]
                args = (dt, w, mp, s)
                fam = Family("to_dec", args)
                # the input rows are floats: nan never equals itself, so rows are kept by position, not deduplicated
                fails = []
                for x in vals:
                    v = to_dec_row(dt, w, mp, s, x)
                    if v is FAIL:
                        fails.append(x)
                    else:
                        fam.ok.append(x)
                        fam.exp.append(v)
                fam.fail = [fails[int(i)] for i in np.linspace(0, len(fails) - 1, min(len(fails), 24))]
                fams.append(fam)
    return fams


# ---- decimal -> integer / float ----------------------------------------------------------------------------------------------
def dec_to_int_families(rng):
    """Each width into each integer type: scales 0 .. mp (the truncating division at every chunk count), scaled values at
    the type's MIN / MAX and one beyond; negative scales with x * 10^-s at the native's range and one beyond."""
    fams = []
    for w in WIDTHS:
        lo, hi = native(w)
        mp = MAXP[w]
        for to in INTS:
            tlo, thi = INT_BOUNDS[to]
            for s in list(range(0, mp + 1)) + [-1, -2, -(mp // 2), -(mp - 1)]:
                vals = [hi, lo, 0, 1, -1] + full_width(rng, w, 6)
                if s >= 0:
                    K = 10 ** s
                    for t in (thi, tlo, thi + 1, tlo - 1):
                        vals += [t * K, t * K + (K - 1 if t >= 0 else -(K - 1)), t * K - 1 if t > 0 else t * K + 1]
                else:
                    f = 10 ** -s
                    vals += around(hi // f, -(hi // f), -((-lo) // f), thi // f, tlo // f if tlo < 0 else 0)
                vals = [v for v in dict.fromkeys(vals) if lo <= v <= hi]
                args = (w, mp, s, to)
                fams.append(split(Family("from_dec", args), vals, lambda x, w=w, s=s, to=to: from_dec_row(w, s, to, x), max_fail=4))
    return fams


def dec_to_float_families(rng):
    """Decimal128 at scale 0 into Float64 and Float32: a value of every bit length 63 .. 127 of each sign, values exactly
    halfway between two doubles with an even and with an odd mantissa, the same ± 1 (the sticky bit), ±2^63, -2^127."""
    vals = [2 ** 63, -(2 ** 63), -(2 ** 127), 2 ** 127 - 1, 2 ** 63 - 1, 2 ** 64, 2 ** 64 - 1]
    for bits in range(63, 128):
        for _ in range(2):
            v = (1 << (bits - 1)) | int.from_bytes(rng.bytes(16), "little") % (1 << (bits - 1))
            vals += [v, -v]
        if bits >= 55:
            sh = bits - 54
            for mant in ((1 << 52) | 2, (1 << 52) | 3, (1 << 53) - 1):  # 53-bit mantissas: even, odd, all ones
                t = ((mant << 1) | 1) << (sh - 1)  # exactly halfway above `mant`
                if t.bit_length() <= 127:
                    vals += [t, t + 1, t - 1, -t, -t + 1, -t - 1]
    vals = [v for v in dict.fromkeys(vals) if in_native(16, v)]
    fams = []
    for to in (F64, F32):
        fam = Family("from_dec", (16, 38, 0, to))
        fams.append(split(fam, vals, lambda x, to=to: from_dec_row(16, 0, to, x)))
    return fams


# ---- sum / min / max ---------------------------------------------------------------------------------------------------------
def aggregate_sets():
    """Decimal128 value lists (None = null): equal high limbs with low limbs straddling 2^63, where a signed compare of the
    low limb inverts min and max; and sums that wrap past 2^127 (sum is add_wrapping)."""
    sets = []
    for h in (0, -1, 1, 5, -7, 2 ** 62, -(2 ** 62)):
        base = h << 64
        lows = [2 ** 63 - 1, 2 ** 63, 2 ** 63 + 1, 0, 2 ** 64 - 1, 1]
        sets.append([base + x for x in lows])
        sets.append([base + 2 ** 63, None, base + 2 ** 63 - 1])
        sets.append([base + 2 ** 63 - 1] * 40 + [base + 2 ** 63] + [base + 2 ** 63 - 1] * 30)
        sets.append([base + 2 ** 63] * 50 + [base + 2 ** 63 - 1] + [None] * 3 + [base + 2 ** 63] * 20)
    lo, hi = native(16)
    sets += [[hi, 1], [lo, -1], [hi] * 3, [lo] * 5, [hi, hi, lo, 7], [hi, None, 1, 2 ** 126, 2 ** 126],
             [lo + 1, -2, None], [2 ** 126] * 64 + [2 ** 126] * 3]
    return sets


def aggregate_closed(vals):
    v = [x for x in vals if x is not None]
    if not v:
        return None, None, None
    lo, _ = native(16)
    return (sum(v) - lo) % (1 << 128) + lo, min(v), max(v)


def all_families(seed=20261017):
    rng = np.random.default_rng(seed)
    return {"add/sub": add_sub_families(), "mul": mul_families(), "div/rem": div_rem_families(rng), "neg": neg_families(rng),
            "decimal -> decimal": dec_families(rng), "integer -> decimal": int_to_dec_families(),
            "float -> decimal": float_to_dec_families(rng), "decimal -> integer": dec_to_int_families(rng),
            "decimal -> float": dec_to_float_families(rng)}
