"""Correctly rounded reference for the float function library, and the inputs that test it (CPU only).

The oracle (oracle/oracle.c) calls glibc, so a bar stated as "within k ulp of the oracle" says nothing about the true
value.  This module computes the true value with mpmath at 160 bits and rounds it once, to nearest even, into
Float64 or Float32:

* subnormal results round to a multiple of 2^-1074 (2^-149);
* |v| >= MAX + 1/2 ulp rounds to +-inf;
* the exponent comes from ``mp.frexp`` (exact), never from a logarithm;
* cbrt(x) is sign(x) * cbrt(|x|) (mpmath's cbrt of a negative number is the principal complex root).

``degrees``, ``radians`` and ``round`` are not mathematical functions here but Rust's formulas (one product with
Rust's constant, rounded to nearest; halves away from zero).  They are restated in numpy with the constants of
oracle.c.  ``log(x, base)`` is ``ln x / ln b`` rounded twice; its reference is that formula over correctly rounded
logarithms for the IEEE-defined cases and the once-rounded true quotient otherwise.

Every reference carries two masks next to the values:

* ``ieee``: the result is fixed by IEEE 754 / C99 Annex F -- a NaN, +-inf or +-0 operand, a domain error, or an
  overflow / underflow so far past the threshold that no rounding can reach a finite non-zero value;
* ``representable``: the true value is a float of the width (checked at 160 and again at 400 bits), for example
  log2(2^k), cbrt(27), exp(0) or ceil(x).

The point sets are the edge set of each function and width (specials, subnormals, domain bounds, overflow and
underflow points, poles, rounding ties, exact cases), strips of +-64 ulp around each threshold, a sweep of 2^14
uniformly random bit patterns (every exponent and both signs) and uniform values from each function's usual range.
Everything is seeded and computed once per process (``functools.lru_cache``).
"""
from __future__ import annotations

import functools
import math
from dataclasses import dataclass
from fractions import Fraction

import mpmath
import numpy as np
from mpmath import mp

PREC = 160          # working precision of the reference
PREC_CHECK = 400    # a result that looks representable at PREC is confirmed at this precision
STRIP = 64          # ulps on each side of a threshold
SWEEP = 1 << 14     # random bit patterns per width
UNIFORM = 2048      # uniform values from each function's usual range

UNARIES = ["abs", "sin", "cos", "tan", "acos", "asin", "atan", "cbrt", "ceil", "cosh", "degrees", "exp", "expm1",
           "floor", "log10", "log2", "radians", "round", "sinh", "sqrt", "tanh"]
BINARIES = ["atan2", "hypot", "log"]
RUST_FORMULAS = {"degrees", "radians", "round"}


@dataclass(frozen=True)
class Fmt:
    name: str
    np: type
    bits: type      # unsigned integer of the same width
    p: int          # significand bits
    qmin: int       # exponent of the smallest subnormal
    emax: int       # 2^emax is the first power of two that overflows


FMTS = {"F64": Fmt("F64", np.float64, np.uint64, 53, -1074, 1024),
        "F32": Fmt("F32", np.float32, np.uint32, 24, -149, 128)}


@dataclass
class Ref:
    x: tuple                 # the operand arrays (one for a unary, two for a binary)
    values: np.ndarray       # correctly rounded result
    ieee: np.ndarray         # result fixed by IEEE 754 / Annex F
    representable: np.ndarray


# ---- rounding -----------------------------------------------------------------------------------------------------

def round_mpf(v, fmt: Fmt):
    """Round a non-zero finite mpf to the nearest float of ``fmt`` (ties to even).  Returns (float, exact, far): exact
    when v is that float, far when v lies beyond the overflow or underflow threshold by at least a factor 2."""
    neg = v < 0
    _, e = mp.frexp(v)                      # |v| = m 2^e, 1/2 <= m < 1
    if e > fmt.emax:
        return (-math.inf if neg else math.inf), False, e > fmt.emax + 1
    if e < fmt.qmin - 1:                    # |v| < 2^(qmin-2): a quarter of the smallest subnormal
        return (-0.0 if neg else 0.0), False, True
    q = max(e - fmt.p, fmt.qmin)
    s = abs(mp.ldexp(v, -q))                # exact
    n = int(mp.floor(s))
    r = s - n                               # exact: s carries at most PREC bits
    if r > 0.5 or (r == 0.5 and n & 1):
        n += 1
    if n == 0:
        return (-0.0 if neg else 0.0), False, False
    if n.bit_length() + q > fmt.emax:
        return (-math.inf if neg else math.inf), False, False
    out = math.ldexp(n, q)
    return (-out if neg else out), r == 0, False


def round_fraction(fr: Fraction, fmt: Fmt) -> float:
    """Round an exact rational to the nearest float of ``fmt`` (ties to even), with subnormals and overflow."""
    if fr == 0:
        return 0.0
    neg, a = fr < 0, abs(fr)
    e = a.numerator.bit_length() - a.denominator.bit_length()
    if a >= Fraction(2) ** e:
        e += 1                              # now 2^(e-1) <= a < 2^e
    q = max(e - fmt.p, fmt.qmin)
    s = a / Fraction(2) ** q
    n = s.numerator // s.denominator
    r = s - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n & 1):
        n += 1
    if n.bit_length() + q > fmt.emax:
        out = math.inf
    else:
        out = math.ldexp(n, q)
    return -out if neg else out


def _pi_fraction() -> Fraction:
    with mp.workprec(256):
        m, e = mp.frexp(mp.pi)
        return Fraction(int(mp.ldexp(m, 256))) / Fraction(2) ** (256 - e)


# ---- the unary functions ------------------------------------------------------------------------------------------

def _special_unary(name, x):
    """The IEEE / Annex F result of ``name`` at x, or None when x is an ordinary point of the function."""
    if math.isnan(x):
        return math.nan
    inf, zero = math.isinf(x), x == 0.0
    pos = x > 0 or (zero and math.copysign(1.0, x) > 0)
    if name in ("sin", "tan"):
        return math.nan if inf else (x if zero else None)
    if name == "cos":
        return math.nan if inf else (1.0 if zero else None)
    if name in ("acos", "asin"):
        if inf or abs(x) > 1:
            return math.nan
        if name == "asin" and zero:
            return x
        return None
    if name == "atan":
        return x if zero else None
    if name in ("cbrt", "sinh"):
        return x if (inf or zero) else None
    if name == "cosh":
        return math.inf if inf else (1.0 if zero else None)
    if name == "tanh":
        return math.copysign(1.0, x) if inf else (x if zero else None)
    if name == "exp":
        return (math.inf if pos else 0.0) if inf else (1.0 if zero else None)
    if name == "expm1":
        return (math.inf if pos else -1.0) if inf else (x if zero else None)
    if name in ("log10", "log2", "log"):
        if zero:
            return -math.inf
        if x < 0:
            return math.nan
        return math.inf if inf else None
    if name == "sqrt":
        if zero:
            return x
        if x < 0:
            return math.nan
        return math.inf if inf else None
    raise KeyError(name)


def _mp_unary(name, v):
    if name == "cbrt":
        r = mp.cbrt(abs(v))
        return -r if v < 0 else r
    return {"sin": mp.sin, "cos": mp.cos, "tan": mp.tan, "acos": mp.acos, "asin": mp.asin, "atan": mp.atan,
            "cosh": mp.cosh, "exp": mp.exp, "expm1": mp.expm1, "log10": mp.log10, "log2": lambda t: mp.log(t, 2),
            "log": mp.log, "sinh": mp.sinh, "sqrt": mp.sqrt, "tanh": mp.tanh}[name](v)


def _true_value(fn, args, fmt: Fmt):
    """Correctly rounded fn(*args) for finite float args, with the two masks (ieee, representable)."""
    with mp.workprec(PREC):
        v = fn(*[mp.mpf(a) for a in args])
        if v == 0:
            return 0.0, False, True
        out, exact, far = round_mpf(v, fmt)
    if exact:                               # confirm at a higher precision before calling it representable
        with mp.workprec(PREC_CHECK):
            exact = fn(*[mp.mpf(a) for a in args]) == mp.mpf(out)
    return out, far, exact


def rust_round(x: np.ndarray) -> np.ndarray:
    """f64::round / f32::round: to the nearest integer, halfway cases away from zero (exact in numpy)."""
    with np.errstate(invalid="ignore"):
        t = np.trunc(x)
        up = np.abs(x - t) >= x.dtype.type(0.5)           # x - t is exact: the fraction of a float
        r = np.where(up, t + np.copysign(x.dtype.type(1), x), t)
    return np.copysign(r, x)                              # -0.4 -> -0.0, like trunc


def rust_degrees(x: np.ndarray) -> np.ndarray:
    """f64::to_degrees = x * (180.0 / PI); f32::to_degrees = x * 57.2957795130823208767981548141051703_f32."""
    if x.dtype == np.float64:
        c = np.float64(180.0) / np.float64(round_fraction(_pi_fraction(), FMTS["F64"]))
    else:
        c = np.float32(round_fraction(Fraction("57.2957795130823208767981548141051703"), FMTS["F32"]))
    with np.errstate(over="ignore", invalid="ignore"):
        return x * c


def rust_radians(x: np.ndarray) -> np.ndarray:
    """f64::to_radians = x * (PI / 180.0); f32::to_radians = x * (PI_f32 / 180.0_f32)."""
    fmt = FMTS["F64"] if x.dtype == np.float64 else FMTS["F32"]
    c = fmt.np(round_fraction(_pi_fraction(), fmt)) / fmt.np(180.0)
    with np.errstate(over="ignore", invalid="ignore"):
        return x * c


def unary_reference(name: str, x: np.ndarray) -> Ref:
    """Correctly rounded name(x) for every element of a Float64 or Float32 array."""
    fmt = FMTS["F64" if x.dtype == np.float64 else "F32"]
    n = len(x)
    special = ~np.isfinite(x) | (x == 0)
    if name in RUST_FORMULAS or name in ("abs", "ceil", "floor"):
        fn = {"degrees": rust_degrees, "radians": rust_radians, "round": rust_round, "abs": np.abs,
              "ceil": np.ceil, "floor": np.floor}[name]
        with np.errstate(invalid="ignore"):
            vals = fn(x).astype(fmt.np)
        return Ref((x,), vals, special.copy(), np.ones(n, bool))
    vals = np.empty(n, fmt.np)
    ieee = np.zeros(n, bool)
    rep = np.zeros(n, bool)
    for i, xi in enumerate(x.tolist()):
        s = _special_unary(name, xi)
        if s is not None:
            vals[i], ieee[i], rep[i] = s, True, True
        else:
            vals[i], ieee[i], rep[i] = _true_value(functools.partial(_mp_unary, name), (xi,), fmt)
    return Ref((x,), vals, ieee, rep)


# ---- the math binaries --------------------------------------------------------------------------------------------

def _special_atan2(y, x):
    """C99 Annex F.9.1.4 atan2(y, x), or None for two finite non-zero operands."""
    if math.isnan(y) or math.isnan(x):
        return math.nan
    sy = math.copysign(1.0, y)
    if y == 0.0:
        if x > 0 or (x == 0 and math.copysign(1.0, x) > 0):
            return y                                        # atan2(+-0, +x) = +-0, atan2(+-0, +0) = +-0
        return sy * math.pi                                 # atan2(+-0, -x) = +-pi, atan2(+-0, -0) = +-pi
    if math.isinf(y):
        if math.isinf(x):
            return sy * (math.pi / 4 if x > 0 else 3 * math.pi / 4)
        return sy * math.pi / 2
    if x == 0.0:
        return sy * math.pi / 2
    if math.isinf(x):
        return y * 0.0 if x > 0 else sy * math.pi          # +-0 or +-pi
    return None


def _special_hypot(x, y):
    """C99 Annex F.9.4.3: hypot(+-inf, y) = +inf even for a NaN y; hypot(x, +-0) = |x|."""
    if math.isinf(x) or math.isinf(y):
        return math.inf
    if math.isnan(x) or math.isnan(y):
        return math.nan
    if x == 0.0:
        return abs(y)
    if y == 0.0:
        return abs(x)
    return None


def _ieee_constant(v: float, fmt: Fmt) -> float:
    """An Annex F result of atan2 (+-0, +-pi/4, +-pi/2, +-3pi/4, +-pi, held as a Float64) rounded correctly into fmt."""
    if not math.isfinite(v) or v == 0.0:
        return v
    with mp.workprec(PREC):
        k = round(v / math.pi * 4)                          # v is k pi / 4
        return round_mpf(mp.pi * k / 4, fmt)[0]


def ln_reference(x: np.ndarray) -> Ref:
    """Correctly rounded natural logarithm (the building block of log(x, base))."""
    fmt = FMTS["F64" if x.dtype == np.float64 else "F32"]
    vals = np.empty(len(x), fmt.np)
    ieee = np.zeros(len(x), bool)
    rep = np.zeros(len(x), bool)
    for i, xi in enumerate(x.tolist()):
        s = _special_unary("log", xi)
        if s is not None:
            vals[i], ieee[i], rep[i] = s, True, True
        else:
            vals[i], ieee[i], rep[i] = _true_value(mp.log, (xi,), fmt)
    return Ref((x,), vals, ieee, rep)


def binary_reference(name: str, a: np.ndarray, b: np.ndarray) -> Ref:
    """Correctly rounded atan2(a, b) / hypot(a, b); for log(a, base=b) the formula ln a / ln b in the column's width
    where either logarithm is +-0, +-inf or NaN (ieee), and the once-rounded true quotient elsewhere."""
    fmt = FMTS["F64" if a.dtype == np.float64 else "F32"]
    n = len(a)
    vals = np.empty(n, fmt.np)
    ieee = np.zeros(n, bool)
    rep = np.zeros(n, bool)
    if name == "log":
        la, lb = ln_reference(a).values, ln_reference(b).values
        with np.errstate(all="ignore"):
            formula = la / lb
        fixed = ~np.isfinite(la) | ~np.isfinite(lb) | (la == 0) | (lb == 0)
        for i in range(n):
            if fixed[i]:
                vals[i], ieee[i], rep[i] = formula[i], True, True
            else:
                vals[i], ieee[i], rep[i] = _true_value(lambda u, v: mp.log(u) / mp.log(v), (float(a[i]), float(b[i])), fmt)
        return Ref((a, b), vals, ieee, rep)
    special = _special_atan2 if name == "atan2" else _special_hypot
    fn = mp.atan2 if name == "atan2" else mp.hypot
    for i, (ai, bi) in enumerate(zip(a.tolist(), b.tolist())):
        s = special(ai, bi)
        if s is not None:
            vals[i], ieee[i], rep[i] = (_ieee_constant(s, fmt) if name == "atan2" else s), True, True
        else:
            vals[i], ieee[i], rep[i] = _true_value(fn, (ai, bi), fmt)
    return Ref((a, b), vals, ieee, rep)


# ---- distances ----------------------------------------------------------------------------------------------------

def to_ordinal(x: np.ndarray) -> np.ndarray:
    """Floats -> integers in the same order, one apart per ulp (+0 and -0 both 0)."""
    it = np.int64 if x.dtype == np.float64 else np.int32
    i = x.view(it).astype(np.int64)
    return np.where(i < 0, np.int64(np.iinfo(it).min) - i, i)


def from_ordinal(o: np.ndarray, fmt: Fmt) -> np.ndarray:
    it = np.int64 if fmt.np is np.float64 else np.int32
    o = np.asarray(o, np.int64)
    i = np.where(o < 0, np.int64(np.iinfo(it).min) - o, o).astype(it)
    return i.view(fmt.np)


def ulps(got: np.ndarray, want: np.ndarray) -> np.ndarray:
    """ulp distance; 0 for NaN vs NaN, a huge number for NaN vs a number."""
    d = np.abs(to_ordinal(got) - to_ordinal(want))
    gn, wn = np.isnan(got), np.isnan(want)
    d = np.where(gn & wn, 0, d)
    return np.where(gn ^ wn, np.iinfo(np.int64).max, d)


def same_bits(got: np.ndarray, want: np.ndarray) -> np.ndarray:
    """Bit-identical, with every NaN equal to every other NaN (IEEE 754 leaves a produced NaN's payload open)."""
    u = np.dtype(f"u{got.dtype.itemsize}")
    return (got.view(u) == want.view(u)) | (np.isnan(got) & np.isnan(want))


# ---- point sets ---------------------------------------------------------------------------------------------------

def strip(t: float, fmt: Fmt, k: int = STRIP) -> np.ndarray:
    """The 2k+1 floats of fmt centred on fmt(t)."""
    c = to_ordinal(np.array([t], fmt.np))[0]
    return from_ordinal(np.arange(c - k, c + k + 1), fmt)


def _cr(value_mp, fmt: Fmt) -> float:
    return round_mpf(value_mp, fmt)[0]


def _common_edges(fmt: Fmt) -> list:
    tiny = [math.ldexp(1.0, fmt.qmin), math.ldexp(2.0, fmt.qmin), math.ldexp(3.0, fmt.qmin),
            math.ldexp(1.0, fmt.qmin + fmt.p - 1) - math.ldexp(1.0, fmt.qmin),       # largest subnormal
            math.ldexp(1.0, fmt.qmin + fmt.p - 1)]                                   # smallest normal
    big = float(np.finfo(fmt.np).max)
    one_side = [0.0, 1.0, 0.5, 2.0, 3.0, 0.1, 10.0, 100.0, big, math.inf,
                float(np.nextafter(fmt.np(1), fmt.np(0))), float(np.nextafter(fmt.np(1), fmt.np(2))),
                math.pi, math.pi / 2, math.pi / 4] + tiny
    one_side += [math.ldexp(1.0, k) for k in (-10, -20, -27, -30, -53, -60, -100, -126, -500, -1000, 20, 60, 100, 127,
                                              500, 1000, 1023) if fmt.qmin <= k < fmt.emax]
    return one_side + [-v for v in one_side] + [math.nan]


def edge_set(name: str, tname: str) -> np.ndarray:
    """The inputs at the edges of ``name``'s domain in width tname (strips of +-64 ulp around each threshold)."""
    fmt = FMTS[tname]
    pts = _common_edges(fmt)
    strips = []
    big = float(np.finfo(fmt.np).max)
    min_sub = math.ldexp(1.0, fmt.qmin)
    with mp.workprec(PREC):
        if name in ("exp", "expm1", "cosh", "sinh"):
            strips.append(_cr(mp.log(big), fmt))                                     # exp overflow
            strips.append(_cr(mp.log(2 * mp.mpf(big)), fmt))                         # cosh / sinh overflow
            strips.append(-_cr(mp.log(2 * mp.mpf(big)), fmt))
        if name == "exp":
            strips.append(_cr(mp.log(mp.ldexp(1, fmt.qmin + fmt.p - 1)), fmt))      # result leaves the normals
            strips.append(_cr(mp.log(min_sub), fmt))
            strips.append(_cr(mp.log(mp.mpf(min_sub) / 2), fmt))                   # underflow to 0
        if name == "expm1":
            strips.append(_cr(mp.log(mp.ldexp(1, -fmt.p - 1)), fmt))                # rounds to -1 below this
            pts += [math.ldexp(s, -k) for k in range(1, 80) for s in (1, -1) if -k >= fmt.qmin]
        if name == "tanh":
            strips.append(_cr(mp.atanh(1 - mp.ldexp(1, -fmt.p - 1)), fmt))          # saturates to 1
            strips.append(-_cr(mp.atanh(1 - mp.ldexp(1, -fmt.p - 1)), fmt))
            pts += [0.55, -0.55, 22.0, 9.0]
        if name in ("acos", "asin"):
            strips += [1.0, -1.0, 0.5, -0.5]
        if name == "atan":
            strips += [1.0, -1.0]
        if name in ("sin", "cos", "tan"):
            for k in (1, 2, 3, 4, 5, 7, 100, 10 ** 6):                            # zeros of sin / cos, poles of tan
                strips.append(_cr(mp.pi * k / 2, fmt))
            pts += [1e22, 1.7e308, 1e15, 6381956970095103 * 2.0 ** 797]             # huge arguments
        if name in ("log10", "log2"):
            strips.append(1.0)
            strips.append(min_sub)
            pts += [math.ldexp(1.0, k) for k in range(fmt.qmin, fmt.emax)]          # log2(2^k) = k
            pts += [float(fmt.np(10.0 ** k)) for k in range(0, 23)]                 # log10(10^k) = k when exact
        if name == "sqrt":
            pts += [float(m * m) for m in range(1, 200)] + [math.ldexp(1.0, 2 * k) for k in range(fmt.qmin // 2, fmt.emax // 2)]
            strips.append(min_sub)
        if name == "cbrt":
            pts += [float(m ** 3) for m in range(1, 200)] + [-float(m ** 3) for m in range(1, 200)]
            pts += [math.ldexp(1.0, 3 * k) for k in range(-(-fmt.qmin // 3), fmt.emax // 3)]
            strips.append(min_sub)
        if name in ("round", "ceil", "floor"):
            for k in list(range(0, 21)) + [2 ** (fmt.p - 3) + 1, 2 ** (fmt.p - 2) - 1, 2 ** (fmt.p - 2) + 1]:
                strips.append(k + 0.5)
            pts += [float(2 ** (fmt.p - 1) + 1), float(2 ** fmt.p), float(2 ** fmt.p + 2), float(2 ** (fmt.p - 1)) + 0.5]
        if name in ("degrees", "radians"):
            strips.append(big / 57.29577951308232 if name == "degrees" else big)
            strips.append(min_sub)
    for t in strips:
        pts += strip(t, fmt).tolist() + (-strip(t, fmt)).tolist()
    with np.errstate(over="ignore"):
        out = np.array(pts, np.float64).astype(fmt.np)
    return out


def sweep(tname: str, seed: int = 2026) -> np.ndarray:
    """SWEEP uniformly random bit patterns: every exponent, both signs, NaNs with payloads."""
    fmt = FMTS[tname]
    rng = np.random.default_rng(seed + fmt.p)
    return rng.integers(0, np.iinfo(fmt.bits).max, SWEEP, dtype=fmt.bits, endpoint=True).view(fmt.np)


def uniform(name: str, tname: str, seed: int = 7) -> np.ndarray:
    """UNIFORM values from the range a user passes most often (the ranges of the random parity test)."""
    rng = np.random.default_rng(seed + UNARIES.index(name))
    if name in ("acos", "asin"):
        v = rng.uniform(-1, 1, UNIFORM)
    elif name in ("log10", "log2", "sqrt"):
        v = rng.uniform(1e-3, 1e6, UNIFORM)
    elif name in ("exp", "expm1", "cosh", "sinh"):
        v = rng.uniform(-20, 20, UNIFORM)
    else:
        v = np.concatenate([rng.uniform(-2e6, 2e6, UNIFORM // 2), rng.uniform(-10, 10, UNIFORM // 2)])
    return v.astype(FMTS[tname].np)


def binary_specials(tname: str) -> np.ndarray:
    fmt = FMTS[tname]
    one_side = [0.0, math.ldexp(1.0, fmt.qmin), 1.0, math.inf, 0.5, 2.0, 3.0, 4.0, 1e30, float(np.finfo(fmt.np).max)]
    return np.array(one_side + [-v for v in one_side] + [math.nan], fmt.np)


# ---- cached references --------------------------------------------------------------------------------------------

@functools.lru_cache(maxsize=None)
def unary_points(name: str, tname: str):
    """(edges, uniform, sweep) inputs of one function and width."""
    return edge_set(name, tname), uniform(name, tname), sweep(tname)


@functools.lru_cache(maxsize=None)
def unary_case(name: str, tname: str) -> Ref:
    """The reference over every point of one function and width, in the order edges + uniform + sweep."""
    return unary_reference(name, np.concatenate(unary_points(name, tname)))


@functools.lru_cache(maxsize=None)
def binary_case(name: str, tname: str) -> Ref:
    """The full cross product of the specials, then SWEEP pairs of random bit patterns."""
    sp = binary_specials(tname)
    sw_a, sw_b = sweep(tname, 11), sweep(tname, 12)
    a = np.concatenate([np.repeat(sp, len(sp)), sw_a])
    b = np.concatenate([np.tile(sp, len(sp)), sw_b])
    return binary_reference(name, a, b)


# ---- exact references of cast -------------------------------------------------------------------------------------

INT_RANGE = {"I8": (-2 ** 7, 2 ** 7 - 1), "I16": (-2 ** 15, 2 ** 15 - 1), "I32": (-2 ** 31, 2 ** 31 - 1),
             "I64": (-2 ** 63, 2 ** 63 - 1), "U8": (0, 2 ** 8 - 1), "U16": (0, 2 ** 16 - 1), "U32": (0, 2 ** 32 - 1),
             "U64": (0, 2 ** 64 - 1)}


def int_to_float_ties(iname: str, tname: str) -> list:
    """Integers of type iname exactly halfway between two floats of tname (both tie directions), +-1 around them,
    and the extremes of the type.  Empty when every value of iname is a float of tname."""
    lo, hi = INT_RANGE[iname]
    p = FMTS[tname].p
    out = set()
    for e in range(p, hi.bit_length()):                    # binade [2^e, 2^(e+1)): ulp 2^(e-p+1), halves are integers
        ulp = 1 << (e - p + 1)
        for k in (0, 1, 2, 3, (1 << (p - 1)) - 2, (1 << (p - 1)) - 1):
            mid = (1 << e) + k * ulp + ulp // 2
            for v in (mid - 1, mid, mid + 1, -mid - 1, -mid, -mid + 1):
                if lo <= v <= hi:
                    out.add(v)
    if out:
        out |= {lo, hi, lo + 1, hi - 1}
    return sorted(out)


def float_to_float_ties() -> np.ndarray:
    """Float64 values at and next to the midpoints between consecutive Float32 values: normal binades, the subnormal
    band, the smallest subnormal, and both sides of the overflow threshold 3.4028235677973366e38."""
    f32, f64 = FMTS["F32"], FMTS["F64"]
    lows = []
    for e in list(range(-149, 128, 7)) + [-149, -127, -126, -125, 126, 127]:
        for m in (1, 2, 3, (1 << 23) - 1, 1 << 23, (1 << 23) + 1, (1 << 24) - 2, (1 << 24) - 1):
            v = math.ldexp(m, e - 23) if e >= -126 else math.ldexp(m % (1 << 23), -149)
            if 0 < v < 3.4028234663852886e38:
                lows.append(v)
    pts = [0.0, math.ldexp(1.0, -150), math.ldexp(3.0, -151), 3.4028235677973366e38, 3.4028234663852886e38]
    for a in lows:
        b = float(np.nextafter(np.float32(a), np.float32(np.inf)))
        mid = (a + b) / 2                                    # exact in Float64
        pts += [mid, a]
    arr = np.array(pts, np.float64)
    out = np.concatenate([strip(v, f64, 2) for v in arr])
    return np.concatenate([out, -out, np.array([np.inf, -np.inf, np.nan])])


def float_to_int_bounds(fname: str, iname: str) -> np.ndarray:
    """Floats of fname at, and 1..3 ulp on either side of, every bound of the window of a float -> iname cast."""
    lo, hi = INT_RANGE[iname]
    fmt = FMTS[fname]
    bounds = [lo - 1, lo, lo + 1, hi, hi + 1, hi + 2, 0, -1, 1]
    pts = []
    for c in bounds:
        t = round_fraction(Fraction(c), fmt)
        if math.isfinite(t):
            pts += strip(t, fmt, 3).tolist()
    pts += [0.5, -0.5, 0.999, -0.999, math.inf, -math.inf, math.nan, -0.0]
    with np.errstate(over="ignore"):
        return np.array(pts, np.float64).astype(fmt.np)


def exact_f64_to_f32(x: float) -> float:
    """`x as f32`: NaN, +-inf and +-0 carry over, every other value rounds once to nearest even."""
    if not math.isfinite(x) or x == 0.0:
        return x
    return round_fraction(Fraction(x), FMTS["F32"])


def exact_int_to_float(v: int, tname: str) -> float:
    return round_fraction(Fraction(v), FMTS[tname])


def exact_float_to_int(x: float, iname: str):
    """num::cast::<float, iname>: the truncated value when it is representable, else None (NaN and +-inf too)."""
    if not math.isfinite(x):
        return None
    t = int(x)                                               # truncation toward zero, exact
    lo, hi = INT_RANGE[iname]
    return t if lo <= t <= hi else None
