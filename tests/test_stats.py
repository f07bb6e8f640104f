"""The statistical aggregates without a GPU: the exact oracle against scipy / numpy, the context-free bdf_moments_stat /
bdf_moments_merge against their numpy restatement bit for bit, and the header's structs and enums against ctypes."""
import os
import subprocess

import numpy as np
import pytest
import scipy.stats

import stats_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(v):
    return None if v is None else np.float64(v).view(np.uint64)


def test_exact_oracle_agrees_with_scipy_and_numpy():
    rng = np.random.default_rng(3)
    for x in (rng.normal(2.0, 3.0, 5000), rng.exponential(1.5, 3001), rng.integers(-1000, 1000, 777).astype(np.float64)):
        r = so.exact_moments(x)
        n = x.shape[0]
        assert np.isclose(r["mean"], x.mean(), rtol=1e-13)
        assert np.isclose(r["m2"] / (n - 1), np.var(x, ddof=1), rtol=1e-12)
        assert np.isclose(r["m2"] / n, np.var(x, ddof=0), rtol=1e-12)
        assert np.isclose(so.stat_np(r, "skewness"), scipy.stats.skew(x, bias=True), rtol=1e-10, atol=1e-13)
        assert np.isclose(so.stat_np(r, "kurtosis"), scipy.stats.kurtosis(x, bias=True, fisher=True), rtol=1e-10, atol=1e-13)
        assert np.isclose(so.stat_np(r, "stddev"), np.std(x, ddof=1), rtol=1e-12)


def test_exact_oracle_special_columns():
    r = so.exact_moments(np.array([0.1, 0.1, 0.1]))
    assert (r["mean"], r["m2"], r["m3"], r["m4"]) == (0.1, 0.0, 0.0, 0.0)
    r = so.exact_moments(np.array([1.0, np.inf]))
    assert np.isnan(r["mean"]) and np.isnan(r["m4"])
    # the naive power sums fail the bars on an ill-conditioned column; the exact record passes them
    rng = np.random.default_rng(5)
    x = 1e6 + rng.uniform(-1, 1, 1 << 14)
    ref = so.exact_moments(x)
    assert so.within_bars(ref, ref) is None
    assert so.within_bars(so.naive_moments(x), ref) is not None


def test_distinct_oracle_rules():
    assert so.count_sum_distinct(np.array([1.5, -0.0, 0.0, 1.5, np.nan, np.nan]))[0] == 3
    c, s = so.count_sum_distinct(np.array([-0.0, -0.0]))
    assert c == 1 and s == 0.0 and not np.signbit(s)
    c, s = so.count_sum_distinct(np.array([2 ** 31 - 1, 1, 1], dtype=np.int32))
    assert c == 2 and s == np.int32(-2 ** 31)


def _records(rng):
    recs = [{"count": 0, "mean": 0.0, "m2": 0.0, "m3": 0.0, "m4": 0.0},
            {"count": 1, "mean": 3.25, "m2": 0.0, "m3": 0.0, "m4": 0.0},
            {"count": 7, "mean": 0.1, "m2": 0.0, "m3": 0.0, "m4": 0.0},
            {"count": 5, "mean": float("nan"), "m2": float("nan"), "m3": float("nan"), "m4": float("nan")},
            {"count": 2, "mean": 1e300, "m2": 1e300, "m3": -1e300, "m4": 1e308}]
    for _ in range(300):
        n = int(rng.integers(1, 1 << 40))
        m2 = float(abs(rng.normal()) * 10.0 ** rng.integers(-5, 8))
        recs.append({"count": n, "mean": float(rng.normal() * 10.0 ** rng.integers(-3, 9)), "m2": m2,
                     "m3": float(rng.normal() * m2 ** 1.5), "m4": float(abs(rng.normal()) * m2 * m2)})
    return recs


def test_moments_stat_matches_the_numpy_restatement(rdf):
    rng = np.random.default_rng(11)
    for rec in _records(rng):
        for stat in so.STATS:
            got, want = rdf.moments_stat(rec, stat), so.stat_np(rec, stat)
            assert (got is None) == (want is None), (rec, stat)
            if want is not None:
                assert _bits(got) == _bits(want) or (np.isnan(got) and np.isnan(want)), (rec, stat, got, want)


def test_moments_merge_matches_the_numpy_restatement(rdf):
    rng = np.random.default_rng(12)
    recs = _records(rng)
    for i in range(400):
        a, b = recs[int(rng.integers(len(recs)))], recs[int(rng.integers(len(recs)))]
        got, want = rdf.moments_merge(a, b), so.merge_np(a, b)
        assert got["count"] == want["count"]
        for k in ("mean", "m2", "m3", "m4"):
            assert _bits(got[k]) == _bits(want[k]) or (np.isnan(got[k]) and np.isnan(want[k])), (a, b, k, got[k], want[k])


def test_moments_merge_of_split_columns_is_accurate(rdf):
    rng = np.random.default_rng(13)
    x = 1e6 + rng.uniform(-1, 1, 4096)
    ref = so.exact_moments(x)
    rec = {"count": 0, "mean": 0.0, "m2": 0.0, "m3": 0.0, "m4": 0.0}
    for part in np.array_split(x, 17):
        r = so.exact_moments(part)
        rec = rdf.moments_merge(rec, {k: r[k] for k in ("count", "mean", "m2", "m3", "m4")})
    assert so.within_bars(rec, ref) is None


def test_stat_errors(rdf):
    import ctypes as C

    N = rdf.native
    r, out, some = N.MomentRec(3, 1.0, 2.0, 0.0, 1.0), C.c_double(), C.c_int32()
    assert N.lib().bdf_moments_stat(C.byref(r), 6, C.byref(out), C.byref(some)) == N.INVALID
    assert N.lib().bdf_moments_stat(C.byref(r), -1, C.byref(out), C.byref(some)) == N.INVALID
    assert N.lib().bdf_moments_stat(None, 0, C.byref(out), C.byref(some)) == N.INVALID
    assert N.lib().bdf_moments_merge(C.byref(r), None, C.byref(r)) == N.INVALID
    with pytest.raises(rdf.ComputeError):
        rdf.moments_stat({"count": 1, "mean": 0.0, "m2": 0.0, "m3": 0.0, "m4": 0.0}, "median")


def test_header_structs_and_enums_match_ctypes(rdf, tmp_path):
    import ctypes as C

    N = rdf.native
    src = tmp_path / "layout.c"
    src.write_text(r'''
#include <stddef.h>
#include <stdio.h>
#include "b200df.h"
int main(void) {
    printf("%zu %zu %zu %zu %zu %zu\n", sizeof(bdf_moment_rec), offsetof(bdf_moment_rec, mean), offsetof(bdf_moment_rec, m4),
           sizeof(bdf_distinct_rec), offsetof(bdf_distinct_rec, sum), sizeof(bdf_stat));
    printf("%d %d %d %d %d %d\n", BDF_STAT_VARIANCE, BDF_STAT_VAR_POP, BDF_STAT_STDDEV, BDF_STAT_STDDEV_POP, BDF_STAT_SKEWNESS,
           BDF_STAT_KURTOSIS);
    printf("%d %d %d %d %d %d %d %d\n", BDF_GROUP_LAST, BDF_GROUP_KURTOSIS, BDF_GROUP_SKEWNESS, BDF_GROUP_STDDEV,
           BDF_GROUP_SUM_DISTINCT, BDF_GROUP_VARIANCE, BDF_GROUP_STDDEV_POP, BDF_GROUP_VAR_POP);
    printf("%d %d\n", BDF_K_WINDOW, BDF_K_MOMENTS);
    return 0;
}
''')
    exe = tmp_path / "layout"
    subprocess.check_call(["cc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    lines = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split("\n")
    assert [int(v) for v in lines[0].split()] == [C.sizeof(N.MomentRec), N.MomentRec.mean.offset, N.MomentRec.m4.offset,
                                                  C.sizeof(N.DistinctRec), N.DistinctRec.sum.offset, 4]
    assert [int(v) for v in lines[1].split()] == [N.STATS[s] for s in ("variance", "var_pop", "stddev", "stddev_pop", "skewness", "kurtosis")]
    assert [int(v) for v in lines[2].split()] == [N.GROUP_LAST] + [N.GROUP_FNS[f] for f in (
        "kurtosis", "skewness", "stddev", "sum_distinct", "variance", "stddev_pop", "var_pop")]
    assert [int(v) for v in lines[3].split()] == [N.K_WINDOW, N.K_MOMENTS] and N.KERNEL_NAMES[N.K_MOMENTS] == "moments"
