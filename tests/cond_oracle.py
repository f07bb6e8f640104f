"""A numpy restatement of the null-handling and conditional functions (include/b200df.h "null handling and conditional
selection"), checked against pyarrow, SQLite and hand-written Spark cases in test_cond.py and used as the reference of
test_cond_gpu.py.

An argument is ``(values, valid)``: two numpy arrays of one length (a scalar is broadcast by ``scalar``).  Results are
``(values, valid)`` too; values under a NULL are 0.  Every selection moves bits: values are copied through unsigned views, so
NaN payloads and the sign of zero survive exactly as the kernels keep them."""
from __future__ import annotations

import numpy as np


def _bits(v: np.ndarray) -> np.ndarray:
    return v.view(np.dtype(f"u{v.dtype.itemsize}")) if v.dtype != np.bool_ else v


def scalar(value, n: int, dtype) -> tuple:
    """A scalar argument of n rows: None is a NULL literal."""
    if value is None:
        return np.zeros(n, dtype=dtype), np.zeros(n, dtype=bool)
    return np.full(n, value, dtype=dtype), np.ones(n, dtype=bool)


def _empty(args):
    v0 = args[0][0]
    return np.zeros_like(v0), np.zeros(v0.shape[0], dtype=bool)


def coalesce(args):
    out, ov = _empty(args)
    ob = _bits(out)
    pending = np.ones(out.shape[0], dtype=bool)
    for v, m in args:
        take = pending & m
        ob[take] = _bits(v)[take]
        ov |= take
        pending &= ~take
    return out, ov


def _greater(x: np.ndarray, y: np.ndarray) -> np.ndarray:
    """x > y in DataFrame::sort's order: every NaN equal and above +inf, -0.0 == 0.0."""
    if x.dtype.kind == "f":
        nx, ny = np.isnan(x), np.isnan(y)
        with np.errstate(invalid="ignore"):
            return (nx & ~ny) | (~nx & ~ny & (x > y))
    return x > y


def extreme(args, greatest: bool):
    out, ov = _empty(args)
    ob = _bits(out)
    for v, m in args:
        better = _greater(v, out) if greatest else _greater(out, v)
        take = m & (~ov | better)
        ob[take] = _bits(v)[take]
        ov |= m
    return out, ov


def greatest(args):
    return extreme(args, True)


def least(args):
    return extreme(args, False)


def nanvl(a, b):
    (av, am), (bv, bm) = a, b
    nan = am & np.isnan(av)
    out, ov = _empty([a])
    ob = _bits(out)
    keep = am & ~nan
    ob[keep] = _bits(av)[keep]
    fromb = nan & bm
    ob[fromb] = _bits(bv)[fromb]
    return out, keep | fromb


def case_when(conds, values):
    """conds: n (values, valid) Boolean arguments; values: n + 1 arguments, the last the else (scalar(None, ..) when missing)."""
    out, ov = _empty(values)
    ob = _bits(out)
    pending = np.ones(out.shape[0], dtype=bool)
    for k, (v, m) in enumerate(values):
        hit = pending & (conds[k][0] & conds[k][1] if k < len(conds) else True)
        sel = hit & m
        ob[sel] = _bits(v)[sel]
        ov |= sel
        pending &= ~hit
    return out, ov


def is_null(a):
    return ~a[1], np.ones(a[1].shape[0], dtype=bool)


def is_not_null(a):
    return a[1].copy(), np.ones(a[1].shape[0], dtype=bool)


def is_nan(a):
    v, m = a
    nan = m & np.isnan(v) if v.dtype.kind == "f" else np.zeros(v.shape[0], dtype=bool)
    return nan, np.ones(v.shape[0], dtype=bool)


def same(got, want) -> bool:
    """Equal validity, and equal bits in every valid slot."""
    gv, gm = got
    wv, wm = want
    if not np.array_equal(gm, wm):
        return False
    return bool(np.array_equal(_bits(np.asarray(gv))[wm], _bits(np.asarray(wv))[wm]))
