"""Exact reference for the statistical aggregates (include/b200df.h "statistical aggregates").

Every f64 value is a dyadic rational, so the moments of a column can be computed exactly: scale the values to integers
X = x * 2^E, take n, S = sum X and sum (n X - S)^k for k = 2, 3, 4 with Python integers; the mean and m2..m4 are then exact
Fractions, rounded once to f64.  Also: a numpy restatement of bdf_moments_stat / bdf_moments_merge with the header's operation
order, and count / sum of the distinct values with the key rules (all NaNs are one value, -0.0 == 0.0)."""
from __future__ import annotations

from fractions import Fraction
from typing import Dict, Iterable, Optional

import numpy as np

STATS = ("variance", "var_pop", "stddev", "stddev_pop", "skewness", "kurtosis")


def valid_values(chunks) -> np.ndarray:
    """The valid values of a list of PrimitiveArrays, read `as f64`, in row order."""
    parts = []
    for c in chunks:
        v = np.asarray(c.values)[c.offset:c.offset + c.length]
        parts.append(v[c.valid_mask()])
    return np.concatenate(parts).astype(np.float64) if parts else np.zeros(0)


def exact_moments(x: np.ndarray) -> Dict[str, object]:
    """The moment record of the f64 values x, each field the exact value rounded once, plus the exact references of the accuracy
    bars: sum |x - mean|^3 ("abs3"), sum (x - mean)^4 and mean |x| ("mean_abs"), and the exact Fractions ("exact")."""
    x = np.asarray(x, dtype=np.float64)
    n = int(x.shape[0])
    if n == 0:
        return {"count": 0, "mean": 0.0, "m2": 0.0, "m3": 0.0, "m4": 0.0, "abs3": 0.0, "mean_abs": 0.0, "sigma": 0.0}
    if not np.isfinite(x).all():
        nan = float("nan")
        return {"count": n, "mean": nan, "m2": nan, "m3": nan, "m4": nan, "abs3": nan, "mean_abs": nan, "sigma": nan}
    ratios = [float(v).as_integer_ratio() for v in x]
    e = max(q.bit_length() - 1 for _, q in ratios)
    xs = [p << (e - (q.bit_length() - 1)) for p, q in ratios]
    s = sum(xs)
    s2 = s3 = s4 = a3 = 0
    for xi in xs:
        d = n * xi - s
        d2 = d * d
        s2 += d2
        s3 += d2 * d
        s4 += d2 * d2
        a3 += d2 * abs(d)
    scale = 1 << e
    mean = Fraction(s, n * scale)
    m2 = Fraction(s2, n ** 2 * scale ** 2)
    m3 = Fraction(s3, n ** 3 * scale ** 3)
    m4 = Fraction(s4, n ** 4 * scale ** 4)
    abs3 = Fraction(a3, n ** 3 * scale ** 3)
    mean_abs = Fraction(sum(abs(v) for v in xs), n * scale)
    return {"count": n, "mean": float(mean), "m2": float(m2), "m3": float(m3), "m4": float(m4), "abs3": float(abs3),
            "mean_abs": float(mean_abs), "sigma": float(m2 / n) ** 0.5, "exact": (mean, m2, m3, m4)}


def naive_moments(x: np.ndarray) -> Dict[str, float]:
    """The power-sum formulas (sum x^k, then the central sums) in f64: what the bars must reject."""
    x = np.asarray(x, dtype=np.float64)
    n = float(x.shape[0])
    s1, s2, s3, s4 = x.sum(), (x * x).sum(), (x ** 3).sum(), (x ** 4).sum()
    mean = s1 / n
    m2 = s2 - n * mean * mean
    m3 = s3 - 3 * mean * s2 + 3 * mean * mean * s1 - n * mean ** 3
    m4 = s4 - 4 * mean * s3 + 6 * mean * mean * s2 - 4 * mean ** 3 * s1 + n * mean ** 4
    return {"count": int(n), "mean": mean, "m2": m2, "m3": m3, "m4": m4}


def within_bars(got: Dict[str, float], ref: Dict[str, object]) -> Optional[str]:
    """None when the record `got` meets the accuracy bars against the exact `ref`, else what failed:
    |m2 - exact| <= 2^-40 max(1, |mean| / sigma) m2, the same form for m3 against sum |x - mean|^3 and m4 against sum (x - mean)^4,
    and |mean - exact| <= 2^-44 mean |x|."""
    if got["count"] != ref["count"]:
        return f"count {got['count']} != {ref['count']}"
    if ref["count"] == 0:
        return None
    if np.isnan(ref["mean"]):
        bad = [k for k in ("mean", "m2", "m3", "m4") if not np.isnan(got[k])]
        return f"{bad} not NaN" if bad else None
    cond = max(1.0, abs(ref["mean"]) / ref["sigma"]) if ref["sigma"] > 0 else 1.0
    checks = (("m2", ref["m2"]), ("m3", ref["abs3"]), ("m4", ref["m4"]))
    for k, scale in checks:
        if abs(got[k] - ref[k]) > 2.0 ** -40 * cond * scale:
            return f"{k}: got {got[k]!r}, exact {ref[k]!r} (bar {2.0 ** -40 * cond * scale:.3g})"
    if abs(got["mean"] - ref["mean"]) > 2.0 ** -44 * ref["mean_abs"]:
        return f"mean: got {got['mean']!r}, exact {ref['mean']!r}"
    return None


# ---- numpy restatement of bdf_moments_stat / bdf_moments_merge (the header's operation order; numpy rounds every operation) ----

def stat_np(rec: Dict[str, float], stat: str) -> Optional[float]:
    f = np.float64
    c = int(rec["count"])
    if c == 0:
        return None
    n, m2, m3, m4 = f(c), f(rec["m2"]), f(rec["m3"]), f(rec["m4"])
    with np.errstate(all="ignore"):
        if stat == "variance":
            return None if c == 1 else float(m2 / (n - f(1)))
        if stat == "var_pop":
            return float(m2 / n)
        if stat == "stddev":
            return None if c == 1 else float(np.sqrt(m2 / (n - f(1))))
        if stat == "stddev_pop":
            return float(np.sqrt(m2 / n))
        if stat == "skewness":
            return None if m2 == 0 else float((np.sqrt(n) * m3) / (m2 * np.sqrt(m2)))
        if stat == "kurtosis":
            return None if m2 == 0 else float((n * m4) / (m2 * m2) - f(3))
    raise ValueError(stat)


def merge_np(a: Dict[str, float], b: Dict[str, float]) -> Dict[str, float]:
    if b["count"] == 0:
        return dict(a)
    if a["count"] == 0:
        return dict(b)
    f = np.float64
    cnt = int(a["count"]) + int(b["count"])
    n, na, nb = f(cnt), f(a["count"]), f(b["count"])
    with np.errstate(all="ignore"):
        delta = f(b["mean"]) - f(a["mean"])
        fr = delta / n
        mean = f(a["mean"]) + fr * nb
        t = (delta * fr) * (na * nb)
        m2 = (f(a["m2"]) + f(b["m2"])) + t
        m3 = ((f(a["m3"]) + f(b["m3"])) + (t * fr) * (na - nb)) + (f(3) * fr) * (na * f(b["m2"]) - nb * f(a["m2"]))
        f2 = fr * fr
        poly = (na * na - na * nb) + nb * nb
        m4 = (((f(a["m4"]) + f(b["m4"])) + (t * f2) * poly) + (f(6) * f2) * ((na * na) * f(b["m2"]) + (nb * nb) * f(a["m2"]))) + \
            (f(4) * fr) * (na * f(b["m3"]) - nb * f(a["m3"]))
    return {"count": cnt, "mean": float(mean), "m2": float(m2), "m3": float(m3), "m4": float(m4)}


# ---- distinct values ----

def distinct_values(x: np.ndarray) -> np.ndarray:
    """The distinct values of x (valid values only) in ascending order, with the key rules: all NaNs are one value (last),
    -0.0 == 0.0 (kept as +0.0)."""
    x = np.asarray(x)
    if x.dtype.kind == "f":
        nan = np.isnan(x)
        u = np.unique(x[~nan] + x.dtype.type(0))   # -0.0 + 0.0 = +0.0
        return np.concatenate([u, x[nan][:1]]) if nan.any() else u
    return np.unique(x)


def count_sum_distinct(x: np.ndarray):
    """(count, sum): the sum in the dtype of x -- integers wrap, floats accumulate in double from +0.0 in ascending order."""
    u = distinct_values(x)
    if u.dtype.kind == "f":
        s = 0.0
        for v in u.astype(np.float64):
            s += v
        return int(u.shape[0]), u.dtype.type(s)
    with np.errstate(over="ignore"):
        return int(u.shape[0]), u.sum(dtype=u.dtype)


def group_values(keys: Iterable[np.ndarray], x: np.ndarray):
    """{key tuple: valid values of x in row order} for whole-valid key columns (numpy arrays)."""
    out: Dict[tuple, list] = {}
    for i, k in enumerate(zip(*keys)):
        out.setdefault(tuple(k), []).append(i)
    return {k: np.asarray(v) for k, v in out.items()}
