"""The distribution rules without a GPU: the numpy restatements of tests/distribution_oracle.py against exact arithmetic, numpy and
pandas; bdf_hist_density (a pure function) against numpy; the appended header enums and kernel names."""
import os
import re
from fractions import Fraction

import numpy as np
import pytest

import distribution_oracle as do

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200df.h")


def _bits(x):
    return np.float64(x).view(np.uint64)


def _exact_percentile(s, p):
    """The stated sequence with every operation rounded once: Fractions, rounded to f64 after each step."""
    n = len(s)
    pos = float(Fraction(n - 1) * Fraction(p))
    lo, hi = np.floor(pos), np.ceil(pos)
    a, b = float(s[int(lo)]), float(s[int(hi)])
    if lo == hi or a == b:
        return a
    t1 = float(Fraction(float(Fraction(hi) - Fraction(pos))) * Fraction(a))
    t2 = float(Fraction(float(Fraction(pos) - Fraction(lo))) * Fraction(b))
    return float(Fraction(t1) + Fraction(t2))


@pytest.mark.parametrize("seed", range(20))
def test_percentile_restatement_is_the_rounded_exact_sequence(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 300))
    v = rng.normal(0, 1e3, n) * (10.0 ** rng.integers(-5, 5, n))
    for p in list(rng.random(8)) + [0.0, 1.0, 0.5, 0.25, 0.75]:
        got = do.percentile(v, p)
        want = _exact_percentile(np.sort(v), p)
        assert _bits(got) == _bits(want), (p, got, want)


@pytest.mark.parametrize("seed", range(10))
def test_percentile_restatement_matches_numpy_linear_within_one_ulp(seed):
    rng = np.random.default_rng(100 + seed)
    v = rng.uniform(-1e6, 1e6, int(rng.integers(2, 5000)))
    s = np.sort(v)
    for p in rng.random(16):
        got, ref = do.percentile(v, p), float(np.quantile(v, p, method="linear"))
        # numpy interpolates as a + (b - a) * t, a different operation order: within one ulp of the larger operand
        pos = (len(v) - 1) * p
        scale = max(abs(s[int(np.floor(pos))]), abs(s[int(np.ceil(pos))]))
        assert abs(got - ref) <= np.spacing(scale), (p, got, ref)


def test_percentile_exact_at_the_ends_at_one_value_and_at_ties():
    v = np.array([3.0, -1.0, 7.5, 2.0])
    assert do.percentile(v, 0.0) == -1.0 and do.percentile(v, 1.0) == 7.5
    assert do.percentile(np.array([4.25]), 0.37) == 4.25
    t = np.array([2.0, 2.0, 2.0, 9.0])
    assert do.percentile(t, 0.4) == 2.0   # a == b: no interpolation, even where it would round
    assert do.percentile(np.array([0.1] * 7), 0.33) == 0.1
    assert do.percentile(np.array([], dtype=np.float64), 0.5) is None


def test_percentile_special_values():
    assert _bits(do.percentile(np.array([-0.0, -0.0]), 0.5)) == _bits(0.0)
    assert _bits(do.percentile(np.array([-np.inf, np.inf]), 0.5)) == 0x7FF8000000000000
    assert do.percentile(np.array([-np.inf, np.inf]), 0.0) == -np.inf
    assert _bits(do.percentile(np.array([1.0, np.nan, np.nan]), 0.5)) == 0x7FF8000000000000
    big = np.array([2**62 + 1, 2**62 + 3], dtype=np.int64)
    assert do.percentile(big, 0.0) == float(2**62)   # read as f64 after the integer order


def test_percentile_p_times_n_minus_one():
    """A percentile formed with p * n instead of p * (n - 1) differs here."""
    v = np.arange(10, dtype=np.float64)
    assert do.percentile(v, 0.5) == 4.5
    assert do.percentile(v, 1.0) == 9.0


def _numpy_hist(x, nbins, rng=None):
    f = x.astype(np.float64)
    f = f[~np.isnan(f)]
    return np.histogram(f, nbins, range=rng)


@pytest.mark.parametrize("seed", range(12))
def test_edge_and_bin_rules_are_numpys(seed):
    rng = np.random.default_rng(200 + seed)
    nbins = int(rng.choice([1, 2, 3, 7, 10, 64, 1000, 2047, 2048, 2049]))
    lo, hi = sorted(rng.normal(0, 10.0 ** rng.integers(-3, 6), 2))
    edges = do.edges_restated(lo, hi, nbins)
    x = np.concatenate([rng.uniform(lo, hi, 5000), edges, np.nextafter(edges, -np.inf), np.nextafter(edges, np.inf)])
    x = x[(x >= lo) & (x <= hi)]
    try:
        counts, ref_edges = np.histogram(x, nbins, range=(lo, hi))
    except ValueError:   # numpy refuses bins narrower than the spacing of the doubles there
        pytest.skip("numpy refuses this range")
    assert (edges.view(np.uint64) == ref_edges.view(np.uint64)).all()
    assert (do.bins_restated(x, edges) == counts).all()


def test_edge_rule_degenerate_ranges():
    for lo in (0.0, 3.0, -7.25, 1e15):
        counts, ref = np.histogram(np.array([lo]), 4)
        assert (do.edges_restated(lo, lo, 4).view(np.uint64) == ref.view(np.uint64)).all()
    tiny = 5e-324   # the step rounds to 0: numpy's linspace takes i / nbins * delta (its histogram refuses such a range)
    ref = np.linspace(0.0, tiny, 4)
    assert (do.edges_restated(0.0, tiny, 3).view(np.uint64) == ref.view(np.uint64)).all()


def test_numpys_edge_correction_is_needed():
    """Values that the formula alone puts in the wrong bin: the one-step correction moves them, so dropping it changes counts."""
    rng = np.random.default_rng(7)
    found = False
    for _ in range(200):
        lo, hi = sorted(rng.normal(0, 1e3, 2))
        nb = int(rng.integers(3, 50))
        e = do.edges_restated(lo, hi, nb)
        x = e[1:-1]
        raw = np.minimum(((x - lo) / (hi - lo) * nb).astype(np.int64), nb - 1)
        if (np.bincount(raw, minlength=nb) != do.bins_restated(x, e)).any():
            found = True
            break
    assert found


def test_oracle_histogram_drops_nan_and_keeps_explicit_range():
    x = np.array([np.nan, 1.0, 2.0, 3.0, np.nan, 10.0])
    e, c = do.histogram(x, 3)
    ref_c, ref_e = np.histogram(np.array([1.0, 2.0, 3.0, 10.0]), 3)
    assert (c == ref_c).all() and (e == ref_e).all()
    e, c = do.histogram(x, 2, (0.0, 2.5))
    assert c.tolist() == [1, 1]   # 3 and 10 outside, NaN never counted
    e, c = do.histogram(np.array([], dtype=np.float64), 4)
    assert e[0] == 0.0 and e[-1] == 1.0 and c.sum() == 0


@pytest.mark.parametrize("nbins", [1, 3, 10, 100])
def test_hist_density_is_numpys(rdf, nbins):
    rng = np.random.default_rng(nbins)
    x = rng.normal(0, 1, 1000)
    dens, edges = np.histogram(x, nbins, density=True)
    counts, _ = np.histogram(x, nbins)
    got = rdf.hist_density(edges, counts)
    assert (got.view(np.uint64) == dens.view(np.uint64)).all()


def test_hist_density_errors(rdf):
    N = rdf.native
    import ctypes as C

    e = (C.c_double * 2)(0.0, 1.0)
    c = (C.c_int64 * 1)(1)
    o = (C.c_double * 1)()
    assert N.lib().bdf_hist_density(0, e, c, o) == N.INVALID
    assert N.lib().bdf_hist_density(1, None, c, o) == N.INVALID
    assert N.lib().bdf_hist_density(1, e, c, None) == N.INVALID
    assert N.lib().bdf_hist_density((1 << 24) + 1, e, c, o) == N.INVALID


def test_mode_and_uniques_oracles_against_pandas():
    pd = pytest.importorskip("pandas")
    rng = np.random.default_rng(3)
    for dt in ("int8", "int64", "uint16", "float64"):
        v = rng.integers(0, 20, 500).astype(dt)
        vals, counts = do.uniques(v)
        vc = pd.Series(v).value_counts().sort_index()
        assert (vals == vc.index.to_numpy()).all() and (counts == vc.to_numpy()).all()
        m, f = do.mode(v)
        top = vc[vc == vc.max()]
        assert m == top.index.min() and f == vc.max()   # ties to the smallest value


def test_mode_and_uniques_oracles_nan_and_signed_zero():
    v = np.array([np.nan, -0.0, 0.0, 1.0, np.nan, 1.0, -np.nan])
    vals, counts = do.uniques(v)
    assert vals.tolist()[:2] == [0.0, 1.0] and np.isnan(vals[2]) and counts.tolist() == [2, 2, 3]
    assert np.signbit(vals[0])   # the class's first row in row order is -0.0
    m, f = do.mode(v)
    assert np.isnan(m) and f == 3
    m, f = do.mode(np.array([5, 2, 5, 2, 9], dtype=np.int32))
    assert m == 2 and f == 2   # a tie goes to the smallest value, not the largest
    assert do.mode(np.array([], dtype=np.int32)) == (None, 0)


def _enum(text, name):
    m = re.search(r"typedef enum \{([^}]*)\} " + name + ";", text, re.S)
    return [t.strip().split("=")[0].strip() for t in m.group(1).split(",") if t.strip()]


def test_header_appends_the_enums_and_kernel_names(rdf):
    text = open(HEADER).read()
    fns = _enum(text, "bdf_group_fn")
    assert fns[-2:] == ["BDF_GROUP_MEDIAN", "BDF_GROUP_MODE"] and fns.index("BDF_GROUP_VAR_POP") == 14
    assert "BDF_GROUP_MEDIAN = 32" in text   # 15..31 stay unknown ids
    ks = _enum(text, "bdf_kernel_id")
    assert ks[-2:] == ["BDF_K_SELECT", "BDF_K_HIST"] and ks.index("BDF_K_PARQUET_WRITE") == 21
    N = rdf.native
    assert N.KERNEL_NAMES[-2:] == ["select", "hist"] and len(N.KERNEL_NAMES) == len(ks)
    assert (N.GROUP_MEDIAN, N.GROUP_MODE, N.K_SELECT, N.K_HIST) == (32, 33, 22, 23)
    assert N.GROUP_FNS["exact_median"] == 32 and N.GROUP_FNS["mode"] == 33 and "median" not in N.GROUP_FNS
    assert "#define BDF_ABI_VERSION 3" in text
