"""The checker of the float function library, pinned against the correctly rounded reference (no GPU).

The GPU parity tests hold the kernels to "within k ulp of the oracle", and the oracle is glibc.  These tests record
how far glibc itself is from the true value on the edge sets, the bit-pattern sweeps and the uniform values of
tests/math_reference.py, so that a change of glibc, of oracle.c or of the reference shows up here first:

* results fixed by IEEE 754 / C99 Annex F (specials, sign of zero, +-inf, NaN) are bit-exact;
* the largest distance of every function from the true value is the number in GLIBC_ULP, no more and no less;
* degrees, radians and round are Rust's formulas, bit for bit;
* cast rounds ties and truncates at the window bounds exactly like int / Fraction arithmetic.
"""
import math
from fractions import Fraction

import numpy as np
import pytest

import math_reference as R

# Largest ulp distance of the oracle (glibc 2.39, x86-64) from the correctly rounded value over every point of
# math_reference.unary_case / binary_case.  Where it is not 0 or 1, the worst point is named.
GLIBC_ULP = {
    "F64": {"abs": 0, "sin": 1, "cos": 8, "tan": 14, "acos": 1, "asin": 1, "atan": 0, "cbrt": 3, "ceil": 0, "cosh": 2,
            "degrees": 0, "exp": 1, "expm1": 1, "floor": 0, "log10": 1, "log2": 0, "radians": 0, "round": 0, "sinh": 2,
            "sqrt": 0, "tanh": 2, "atan2": 0, "hypot": 1, "log": 2},
    "F32": {"abs": 0, "sin": 1, "cos": 1, "tan": 1, "acos": 1, "asin": 1, "atan": 1, "cbrt": 1, "ceil": 0, "cosh": 2,
            "degrees": 0, "exp": 1, "expm1": 1, "floor": 0, "log10": 1, "log2": 1, "radians": 0, "round": 0, "sinh": 2,
            "sqrt": 0, "tanh": 2, "atan2": 1, "hypot": 0, "log": 2},
}
# cos / tan (F64): 8 and 14 ulp only at 6381956970095103 * 2^797, the hardest argument reduction of the format
# (cos there is -4.687e-19); at most 1 ulp everywhere else.  cosh / sinh (F64): 2 ulp just below the overflow point
# ln(2 MAX).  log(x, base) is ln x / ln b rounded twice, hence 2.
HARD_TRIG = 6381956970095103 * 2.0 ** 797
# glibc's cbrt (F64) misses the exact result of some exact cubes (cbrt(2^-1074) = 2^-358, cbrt(2^-27) = 2^-9, ...).
MISSES_REPRESENTABLE = {("cbrt", "F64")}


class Chunk:
    def __init__(self, values, dtype):
        self.values, self.dtype, self.offset, self.length = np.ascontiguousarray(values), dtype, 0, len(values)
        self.validity, self.null_count = None, 0


def oracle_unary(oracle, name, tname, x):
    dt = getattr(oracle, tname)
    st, out = oracle.col_unary(getattr(oracle, name.upper()), dt, [Chunk(x, dt)])
    assert st == oracle.OK
    return out[0].values


def oracle_binary(oracle, name, tname, a, b):
    dt = getattr(oracle, tname)
    st, out = oracle.col_binary(getattr(oracle, name.upper()), dt, [Chunk(a, dt)], [Chunk(b, dt)])
    assert st == oracle.OK
    return out[0].values


def bits(x):
    return x.view(np.dtype(f"u{x.dtype.itemsize}"))


# ---- the reference itself -------------------------------------------------------------------------------------------

def test_rounding_handles_subnormals_overflow_and_ties():
    f64, f32 = R.FMTS["F64"], R.FMTS["F32"]
    F = Fraction
    assert R.round_fraction(F(2) ** -1075, f64) == 0.0                        # half the smallest subnormal: tie to even
    assert R.round_fraction(F(3) * F(2) ** -1076, f64) == 5e-324               # above the tie
    assert R.round_fraction(F(3) * F(2) ** -1075, f64) == 2 * 5e-324           # 1.5 quanta: tie to even (2)
    assert R.round_fraction(F(2) ** -150, f32) == 0.0
    assert R.round_fraction(F(2) ** -150 + F(2) ** -200, f32) == 2.0 ** -149
    mx = F(2) ** 1024 - F(2) ** 971                                           # Float64 MAX
    assert R.round_fraction(mx + F(2) ** 970, f64) == math.inf                 # MAX + 1/2 ulp -> inf
    assert R.round_fraction(mx + F(2) ** 970 - 1, f64) == 1.7976931348623157e308
    assert R.round_fraction(F(3.4028235677973366e38), f32) == math.inf        # Float32 MAX + 1/2 ulp
    assert R.round_fraction(F(np.nextafter(3.4028235677973366e38, 0)), f32) == float(np.finfo(np.float32).max)
    assert R.round_fraction(F(2 ** 53 + 1), f64) == 2.0 ** 53                 # tie to even
    assert R.round_fraction(F(2 ** 53 + 3), f64) == 2.0 ** 53 + 4
    assert R.round_fraction(F(-(2 ** 24 + 1)), f32) == -(2.0 ** 24)


def test_reference_values_at_known_points():
    ref = lambda name, xs, t="F64": R.unary_reference(name, np.array(xs, R.FMTS[t].np)).values.tolist()
    assert ref("exp", [1.2e291, -1.2e291, 709.782712893384, 709.7827128933841]) == [math.inf, 0.0, 1.7976931348622732e308, math.inf]
    assert ref("cbrt", [-27.0, 27.0, 5e-324, -0.0]) == [-3.0, 3.0, 2.0 ** -358, -0.0]
    assert ref("log2", [2.0 ** -1074, 1024.0, 0.0, -1.0])[:3] == [-1074.0, 10.0, -math.inf]
    assert ref("log10", [1e22, 1000.0, 1.0]) == [22.0, 3.0, 0.0]
    assert ref("expm1", [1e-300, -1e-300, -40.0]) == [1e-300, -1e-300, -1.0]
    assert ref("sin", [HARD_TRIG]) == [math.sin(HARD_TRIG)]
    assert ref("cos", [HARD_TRIG]) == [-4.687165924254628e-19]
    below = float(np.float32(88.72283))                                      # the last Float32 whose exp is finite
    assert ref("exp", [88.72284, below], "F32") == [math.inf, float(np.float32(math.exp(below)))]
    assert ref("acos", [1.0, -1.0]) == [0.0, math.pi] and math.isnan(ref("acos", [1.0000000000000002])[0])
    at = R.binary_reference("atan2", np.array([0.0, -0.0, 0.0, -0.0, -1.0, np.inf]), np.array([-0.0, -0.0, 0.0, 0.0, 0.0, -np.inf]))
    assert at.values.tolist() == [math.pi, -math.pi, 0.0, -0.0, -math.pi / 2, 3 * math.pi / 4]
    assert np.signbit(at.values[3]) and at.ieee.all()
    hy = R.binary_reference("hypot", np.array([np.inf, np.nan, 3.0, -0.0]), np.array([np.nan, -np.inf, 4.0, -2.0]))
    assert hy.values.tolist() == [math.inf, math.inf, 5.0, 2.0] and hy.representable.all()
    lg = R.binary_reference("log", np.array([8.0, 2.0, 1.0, 0.0, -1.0]), np.array([1.0, 0.0, 1.0, 2.0, 2.0]))
    assert lg.values[:2].tolist() == [math.inf, -0.0] and np.isnan(lg.values[2]) and lg.values[3] == -math.inf
    assert np.signbit(lg.values[1]) and np.isnan(lg.values[4]) and lg.ieee.all()


# ---- the oracle against the reference ------------------------------------------------------------------------------

@pytest.mark.parametrize("tname", ["F64", "F32"])
@pytest.mark.parametrize("name", R.UNARIES)
def test_oracle_unary_against_true_value(oracle, name, tname):
    ref = R.unary_case(name, tname)
    got = oracle_unary(oracle, name, tname, ref.x[0])
    ieee_bad = np.nonzero(~R.same_bits(got, ref.values) & ref.ieee)[0]
    assert ieee_bad.size == 0, f"{name}<{tname}> IEEE results differ at x={ref.x[0][ieee_bad[:5]]}: {got[ieee_bad[:5]]} vs {ref.values[ieee_bad[:5]]}"
    d = R.ulps(got, ref.values)
    worst = int(d.max())
    assert worst == GLIBC_ULP[tname][name], f"{name}<{tname}>: glibc is {worst} ulp from the true value at x={ref.x[0][d.argmax()]!r}"
    if name in ("cos", "tan") and tname == "F64":
        assert int(d[ref.x[0] != HARD_TRIG].max()) <= 1
    missed = np.nonzero(ref.representable & ~R.same_bits(got, ref.values))[0]
    assert (missed.size > 0) == ((name, tname) in MISSES_REPRESENTABLE), f"{name}<{tname}> exact results missed at {ref.x[0][missed[:5]]}"


@pytest.mark.parametrize("tname", ["F64", "F32"])
@pytest.mark.parametrize("name", R.BINARIES)
def test_oracle_binary_against_true_value(oracle, name, tname):
    ref = R.binary_case(name, tname)
    a, b = ref.x
    got = oracle_binary(oracle, name, tname, a, b)
    bad = np.nonzero(~R.same_bits(got, ref.values) & (ref.ieee | ref.representable))[0]
    assert bad.size == 0, f"{name}<{tname}> differs at {list(zip(a[bad[:4]], b[bad[:4]]))}: {got[bad[:4]]} vs {ref.values[bad[:4]]}"
    d = R.ulps(got, ref.values)
    assert int(d.max()) == GLIBC_ULP[tname][name], f"{name}<{tname}>: {int(d.max())} ulp at {a[d.argmax()]!r}, {b[d.argmax()]!r}"


@pytest.mark.parametrize("tname", ["F64", "F32"])
def test_rust_formulas_bit_exact(oracle, tname):
    """degrees / radians / round are the oracle's formulas (oracle.c unary_f64 / unary_f32), restated in numpy."""
    for name, fn in (("degrees", R.rust_degrees), ("radians", R.rust_radians), ("round", R.rust_round)):
        x = np.concatenate(R.unary_points(name, tname))
        got = oracle_unary(oracle, name, tname, x)
        assert R.same_bits(got, fn(x)).all(), name
    npdt = R.FMTS[tname].np
    below_half = float(np.nextafter(npdt(0.5), npdt(0)))                    # 0.49999999999999994 in Float64
    odd = float(2 ** (R.FMTS[tname].p - 1) + 1)                              # 2^52 + 1: no fraction, odd
    x = np.array([0.5, -0.5, 1.5, 2.5, -2.5, below_half, -below_half, -0.4, odd], npdt)
    want = np.array([1.0, -1.0, 2.0, 3.0, -3.0, 0.0, -0.0, -0.0, odd], npdt)
    assert np.array_equal(bits(R.rust_round(x)), bits(want))
    assert np.array_equal(bits(oracle_unary(oracle, "round", tname, x)), bits(want))


# ---- cast: ties and window bounds ---------------------------------------------------------------------------------

INT_NAMES = ["I8", "I16", "I32", "I64", "U8", "U16", "U32", "U64"]


@pytest.mark.parametrize("iname", INT_NAMES)
def test_oracle_cast_rounding_is_exact(oracle, iname):
    """int -> float ties, float -> int window bounds and f64 -> f32 ties against int / Fraction arithmetic."""
    idt = oracle.NP_DTYPES[getattr(oracle, iname)]
    for tname in ("F32", "F64"):
        vals = R.int_to_float_ties(iname, tname)
        if not vals:
            continue
        st, out = oracle.col_cast(getattr(oracle, iname), getattr(oracle, tname), [Chunk(np.array(vals, idt), getattr(oracle, iname))])
        want = np.array([R.exact_int_to_float(v, tname) for v in vals], R.FMTS[tname].np)
        assert np.array_equal(bits(out[0].values), bits(want)), f"{iname}->{tname}"
    for fname in ("F32", "F64"):
        x = R.float_to_int_bounds(fname, iname)
        st, out = oracle.col_cast(getattr(oracle, fname), getattr(oracle, iname), [Chunk(x, getattr(oracle, fname))])
        want = [R.exact_float_to_int(float(v), iname) for v in x]
        assert out[0].valid_mask().tolist() == [w is not None for w in want], f"{fname}->{iname}"
        assert out[0].values.tolist() == [0 if w is None else w for w in want], f"{fname}->{iname}"


def test_oracle_f64_to_f32_ties_are_exact(oracle):
    x = R.float_to_float_ties()
    st, out = oracle.col_cast(oracle.F64, oracle.F32, [Chunk(x, oracle.F64)])
    want = np.array([R.exact_f64_to_f32(v) for v in x.tolist()], np.float32)
    assert R.same_bits(out[0].values, want).all()
    assert np.isinf(want).sum() >= 4 and (want[np.abs(x) <= 2.0 ** -150] == 0).all()   # up to the tie with 0
