"""Exact references for the readers' and writer's number conversions (csrc/csv_parse.cuh, csrc/csv_format.cuh), and a seeded corpus
of the inputs where those conversions are hardest.  Standard library and numpy only; no GPU.

Reading: a string of Rust's f32 / f64 FromStr grammar is rounded to nearest-even from its exact value, the same integer rule for
both widths (Float32 never through Float64, and nothing taken from the platform's libc).  `undecidable` says which strings the
parser's fast path may hand to its exact fallback: those whose first 19 significant digits w (times 10^q) and w + 1 round apart, and
the rare products whose 128-bit truncation ends in 64 one bits.

Writing: the shortest digits that read back, the closest among several, are what numpy prints with unique=True (csv_write_oracle);
`shortest_closest_ok` checks that claim exactly for one value and its text."""
from __future__ import annotations

import importlib.util
import os
import re
import struct
from dataclasses import dataclass
from fractions import Fraction
from typing import List, Optional, Tuple

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.environ.get("BDF_CONVERSION_CSRC", os.path.join(os.path.dirname(HERE), "rust-dataframe_b200", "csrc"))


@dataclass(frozen=True)
class Fmt:
    width: int       # 32 or 64
    mbits: int       # explicit mantissa bits
    bias: int
    min_p10: int     # eisel_lemire's shortcut edges: below min_p10 a 19-digit w * 10^q is zero, above max_p10 infinite
    max_p10: int
    min_rte: int     # the powers of ten where w * 10^q can be exactly halfway between two floats
    max_rte: int

    @property
    def emax(self) -> int:
        return 2 * self.bias + 1   # the biased exponent of inf / NaN


F32 = Fmt(32, 23, 127, -65, 38, -17, 10)
F64 = Fmt(64, 52, 1023, -342, 308, -4, 23)
FMTS = {32: F32, 64: F64}

_FLOAT_RE = re.compile(r"([+-]?)([0-9]+\.?[0-9]*|\.[0-9]+)(?:[eE]([+-]?[0-9]+))?")
_SPECIAL_RE = re.compile(r"([+-]?)(inf|infinity|nan)", re.IGNORECASE)


def lex(s: str) -> Optional[Tuple[bool, int, int]]:
    """(negative, N, E) with the value N * 10^E for a finite string of the grammar; None for a syntax error or a special."""
    m = _FLOAT_RE.fullmatch(s)
    if not m:
        return None
    ip, _, fp = m.group(2).partition(".")
    n = int(ip + fp) if ip + fp else 0
    return m.group(1) == "-", n, (int(m.group(3)) if m.group(3) else 0) - len(fp)


def round_exact(neg: bool, n: int, e: int, f: Fmt) -> int:
    """The bits of N * 10^E (with the sign) rounded to nearest-even in format f: subnormals, overflow to inf, signed zero."""
    sign = (1 << (f.width - 1)) if neg else 0
    if n == 0 or e + len(str(n)) < -400:   # below 10^-400: under half the smallest subnormal of either width
        return sign
    if e + len(str(n)) > 400:
        return sign | (f.emax << f.mbits)
    num, den = (n * 10 ** e, 1) if e >= 0 else (n, 10 ** -e)
    e2 = num.bit_length() - den.bit_length()            # 2^e2 <= num / den < 2^(e2 + 2)
    if (num << max(0, -e2)) < (den << max(0, e2)):
        e2 -= 1
    u = max(e2, 1 - f.bias) - f.mbits                   # the weight of the last mantissa bit
    a, b = (num, den << u) if u >= 0 else (num << -u, den)
    m, r = divmod(a, b)
    if 2 * r > b or (2 * r == b and m & 1):
        m += 1
    if m == 1 << (f.mbits + 1):
        m >>= 1
        u += 1
    if m < 1 << f.mbits:                                # subnormal (or zero)
        return sign | m
    be = u + f.mbits + f.bias
    if be >= f.emax:
        return sign | (f.emax << f.mbits)
    return sign | (be << f.mbits) | (m - (1 << f.mbits))


def parse_bits(s: str, f: Fmt) -> Optional[int]:
    """Rust's FromStr of s in format f as a bit pattern (NaN is the quiet NaN with the sign given), or None for a syntax error."""
    m = _SPECIAL_RE.fullmatch(s)
    if m:
        sign = (1 << (f.width - 1)) if m.group(1) == "-" else 0
        nan = (1 << (f.mbits - 1)) if m.group(2).lower() == "nan" else 0
        return sign | (f.emax << f.mbits) | nan
    x = lex(s)
    return None if x is None else round_exact(*x, f)


# ---- which strings the fast path may leave undecided ----------------------------------------------------------------------------
def _pow5_128():
    spec = importlib.util.spec_from_file_location("_gen_csv_pow5", os.path.join(CSRC, "gen_csv_pow5.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.pow5_128


_M64 = (1 << 64) - 1


def product_ambiguous(w: int, q: int, f: Fmt) -> bool:
    """True where the 128-bit truncated product w * 5^q of Eisel-Lemire (with the table of gen_csv_pow5.py) ends in 64 one bits
    outside the range where it is exact, so that the product alone cannot decide the rounding."""
    if w == 0 or q < f.min_p10 or q > f.max_p10:
        return False
    t = _pow5_128()(q)
    wn = w << (64 - w.bit_length())
    p = wn * (t >> 64)
    hi, lo = p >> 64, p & _M64
    mask = _M64 >> (f.mbits + 3)
    if hi & mask == mask:
        lo += (wn * (t & _M64)) >> 64
        if lo > _M64:
            lo &= _M64
    return lo == _M64 and (q < -27 or q > 55)


def leading19(n: int, e: int) -> Tuple[int, int, bool]:
    """(w, q, dropped): w the first 19 significant digits of N, value = w * 10^q plus a nonzero rest when dropped."""
    s = str(n)
    if len(s) <= 19:
        return n, e, False
    rest = s[19:]
    return int(s[:19]), e + len(rest), rest.strip("0") != ""


def undecidable(s: str, f: Fmt) -> bool:
    """Whether the parser may report s as needing exact rounding (kFloatSlow)."""
    x = lex(s)
    if x is None:
        return False
    neg, n, e = x
    w, q, dropped = leading19(n, e)
    if w and dropped and round_exact(False, w, q, f) != round_exact(False, w + 1, q, f):
        return True
    return product_ambiguous(w, q, f) or (dropped and product_ambiguous(w + 1, q, f))


# ---- formatting -------------------------------------------------------------------------------------------------------------------
def bits_to_float(b: int, f: Fmt):
    if f.width == 32:
        return np.array([b], np.uint32).view(np.float32)[0]
    return np.array([b], np.uint64).view(np.float64)[0]


def exact_value(b: int, f: Fmt) -> Fraction:
    """The exact value of a finite pattern."""
    be, frac = (b >> f.mbits) & f.emax, b & ((1 << f.mbits) - 1)
    c, q = (frac | (1 << f.mbits), be - f.bias - f.mbits) if be else (frac, 1 - f.bias - f.mbits)
    v = Fraction(c) * Fraction(2) ** q
    return -v if b >> (f.width - 1) else v


def shortest_closest_ok(text: str, b: int, f: Fmt) -> bool:
    """For a finite nonzero pattern: text reads back to b, no decimal with fewer significant digits does, and neither neighbour
    with the same number of digits that also reads back is closer to the exact value."""
    x = lex(text)
    if x is None or round_exact(*x, f) != b:
        return False
    _, d, e = x
    while d % 10 == 0:
        d //= 10
        e += 1
    mag = b & ((1 << (f.width - 1)) - 1)
    v = abs(exact_value(b, f))

    def reads_back(dd: int, ee: int) -> bool:
        return dd > 0 and round_exact(False, dd, ee, f) == mag

    if reads_back(d // 10, e + 1) or reads_back(d // 10 + 1, e + 1):
        return False
    dist = abs(Fraction(d) * Fraction(10) ** e - v)
    return all(not reads_back(dd, e) or abs(Fraction(dd) * Fraction(10) ** e - v) >= dist for dd in (d - 1, d + 1))


# ---- the corpus -------------------------------------------------------------------------------------------------------------------
def _dyadic_decimal(m: int, p: int) -> Tuple[str, int]:
    """m * 2^p (m > 0) exactly as (digits, E): the value is int(digits) * 10^E, digits without trailing zeros."""
    if p >= 0:
        d, e = str(m << p), 0
    else:
        d, e = str(m * 5 ** -p), p
    t = d.rstrip("0")
    return t, e + len(d) - len(t)


def _sci(d: str, e: int, neg: bool = False) -> str:
    """digits * 10^e written as d.ddd e<x>."""
    x = e + len(d) - 1
    return ("-" if neg else "") + d[0] + ("." + d[1:] if len(d) > 1 else "") + f"e{x}"


def _midpoint_strings(c: int, q: int) -> List[str]:
    """The midpoint (2c + 1) 2^(q-1) between c 2^q and its upper neighbour: all of its digits, nudged above and below by a tail, cut
    to 17..25 significant digits, and each cut plus one in its last digit (the w / w + 1 pair of the parser)."""
    d, e = _dyadic_decimal(2 * c + 1, q - 1)
    out = [_sci(d, e), _sci(d + "0001", e - 4)]
    below = str(int(d) - 1) + "9999" if len(str(int(d) - 1)) == len(d) else None
    if below:
        out.append(_sci(below, e - 4))
    for k in (17, 18, 19, 20, 21, 25):
        if len(d) > k:
            cut = d[:k]
            out.append(_sci(cut, e + len(d) - k))
            out.append(_sci(str(int(cut) + 1), e + len(d) - k))
    return out


def _spellings(rng, s: str) -> List[str]:
    """The same number written other ways: leading zeros, a positional fraction, trailing zeros on the integer part, a padded or
    upper-case exponent, signs."""
    neg, n, e = lex(s)
    d = str(n)
    sg = "-" if neg else ""
    out = [sg + "000" + d + f"e{e}", ("+" if not neg else "-") + d + f"E{e:+05d}", sg + d + "000" + f"e{e - 3}"]
    if -400 < e < 0:
        if len(d) > -e:
            out.append(sg + d[:e] + "." + d[e:])
        else:
            out.append(sg + "0." + "0" * (-e - len(d)) + d)
    elif 0 <= e < 40:
        out.append(sg + d + "0" * e + ("." if rng.random() < 0.5 else ""))
    return out


def parse_corpus(seed: int = 20261018, mantissas: int = 3, spell_every: int = 23) -> List[str]:
    """The hard strings for both widths, deterministic in seed."""
    rng = np.random.default_rng(seed)
    out: List[str] = []
    for f in (F64, F32):
        top = (1 << f.mbits) - 1
        for be in range(0, f.emax):
            fracs = {0, 1, top} | {int(x) for x in rng.integers(0, top + 1, mantissas)}
            for frac in sorted(fracs):
                if be == 0 and frac == 0:
                    continue
                c = frac | (1 << f.mbits) if be else frac
                q = be - f.bias - f.mbits if be else 1 - f.bias - f.mbits
                out += _midpoint_strings(c, q)
        out.append(_sci(*_dyadic_decimal(1, 1 - f.bias - f.mbits - 1)))   # half the smallest subnormal
        # the shortcut edges of eisel_lemire: 19-digit mantissas with q just inside and just outside [min_p10, max_p10]
        for q in (f.min_p10 - 1, f.min_p10, f.max_p10, f.max_p10 + 1):
            for w in [10 ** 18, 10 ** 19 - 1] + [int(x) for x in rng.integers(10 ** 18, 10 ** 19, 6, dtype=np.uint64)]:
                out += [f"{w}e{q}", f"{w}e{q}".replace("e", "9e" if q > 0 else "1e")]
        # exact ties inside [min_rte, max_rte]: (2c + 1) 2^p = w 10^q with w of at most 19 digits, and w +- 1 beside them
        lo, hi = 1 << (f.mbits + 1), 1 << (f.mbits + 2)
        for q in range(f.min_rte, f.max_rte + 1):
            for _ in range(4):
                if q >= 0:
                    t_lo, t_hi = -(-lo // 5 ** q), hi // 5 ** q
                    if t_lo >= t_hi:
                        continue
                    t = int(rng.integers(t_lo, t_hi)) | 1
                    if t >= t_hi:
                        t -= 2
                    if t < t_lo:
                        continue
                    w = t << int(rng.integers(0, 3))   # p = q .. q + 2
                else:
                    s_odd = int(rng.integers(lo, hi)) | 1
                    w = s_odd * 5 ** -q << int(rng.integers(0, 3))
                if w >= 10 ** 19:
                    continue
                out += [f"{w}e{q}", f"{w + 1}e{q}", f"{w - 1}e{q}"]
    # the textbook ties and near-ties
    out += ["9007199254740993", "9007199254740995", "9007199254740993e1", "9007199254740993e-1", "90071992547409930e-1",
            "9007199254740993.0000000000000000001", "9007199254740992.9999999999999999999", "16777217", "16777219", "16777217e3",
            "33554434", "33554438e1", "1677721700000000000e-11", "16777217.000000000000000000001", "16777216.999999999999999999999"]
    # extremes, by name
    out += ["1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308", "179769313486231580793728971405301e276",
            "4.9406564584124654e-324", "5e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "2.2250738585072011e-308",
            "2.2250738585072014e-308", "3.4028235e38", "3.40282356779733661637539395458142568448e38", "3.4028236e38", "1.4e-45",
            "1.401298464324817e-45", "7.006492321624085e-46", "7.006492321624086e-46", "1.1754943e-38", "1.17549435e-38"]
    # mantissa carries at 19 and 20 digits
    for q in (-300, -40, -20, -1, 0, 1, 20, 30, 290):
        out += [f"{'9' * 19}e{q}", f"{'9' * 20}e{q}", f"{'9' * 19}5e{q}", f"{'9' * 18}8{'9' * 2}e{q}", f"1{'0' * 18}e{q}",
                f"1{'0' * 19}1e{q}"]
    # other spellings of a sample, and the grammar's corners
    out += [x for i, s in enumerate(list(out)) if i % spell_every == 0 for x in _spellings(rng, s)]
    out += [".5", "+.5", "-.5", "1.", "-1.", "0.", "00", "-0", "+0", "0e0", "1e99999999999", "-1e99999999999", "0e999999999999",
            "1e-99999999999", "1e+99999999999", "0.000000000000000000000000000000000000000000001", "1E-5", "1e+0008", "1e0008",
            "inf", "-inf", "+Infinity", "INFINITY", "NaN", "-nan", "+NAN",
            # syntax errors: the grammar, not the value, decides
            "", "+", "-", ".", "e5", ".e5", "1e", "1e+", "1e-", "1.5.", "1..5", "--1", "+-1", "1 ", " 1", "1_0", "0x10", "1e5.5", "infinit",
            "infinityy", "nana", "in", "1,5", "1d5", "1f", "١"]
    return out


def random_shortest(seed: int, n: int, f: Fmt) -> List[str]:
    """n shortest round-trip strings of random finite patterns of format f (repr for Float64, numpy's unique digits for Float32)."""
    rng = np.random.default_rng(seed)
    if f.width == 64:
        v = rng.integers(0, 1 << 64, n, dtype=np.uint64).view(np.float64)
        return [repr(x) for x in v[np.isfinite(v)].tolist()]
    v = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32).view(np.float32)
    return [np.format_float_scientific(x, unique=True) for x in v[np.isfinite(v)]]


def format_patterns(seed: int, f: Fmt, n_random: int = 20000) -> np.ndarray:
    """The patterns to format in format f, both signs: every power of two with its neighbours, every subnormal power of two, the
    nearest values to the powers of ten with their neighbours, the extremes, and seeded random patterns."""
    rng = np.random.default_rng(seed)
    top = (1 << (f.mbits)) - 1
    pats = set()
    for be in range(1, f.emax):
        p = be << f.mbits
        pats |= {p - 1, p, p + 1, p + top}
    pats |= {1 << k for k in range(f.mbits)} | {(1 << k) + 1 for k in range(f.mbits)} | {(1 << k) - 1 for k in range(1, f.mbits + 1)}
    pats |= {1, 2, top, top + 1, (f.emax << f.mbits) - 1, f.emax << f.mbits, 0}
    for k in range(-330 if f.width == 64 else -46, 310 if f.width == 64 else 40):
        b = round_exact(False, 1, k, f)
        if b < f.emax << f.mbits:
            pats |= {b - 1, b, b + 1} if b else {b}
    mag_hi = f.emax << f.mbits
    dt = np.uint64 if f.width == 64 else np.uint32
    rnd = rng.integers(0, mag_hi, n_random, dtype=np.uint64)
    pats |= {int(x) for x in rnd}
    pats = sorted(x for x in pats if 0 <= x <= mag_hi)
    mags = np.array(pats, dtype=dt)
    sign = dt(1 << (f.width - 1))
    return np.concatenate([mags, mags | sign])
