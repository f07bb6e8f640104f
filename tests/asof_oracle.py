"""The as-of join of bdf_join_asof_dev and the existence joins of bdf_join_indices_dev restated in numpy: the checker of
tests/test_join_asof_gpu.py and tests/test_join_semi_gpu.py, itself checked against pandas.merge_asof and an inner join in
tests/test_join_asof.py.

A key is a pair (values, valid mask) of numpy arrays over a side's rows (chunks concatenated); `by` is a list of them.
Candidates of a left row: the right rows whose `by` tuple equals its own (join_oracle.key_codes: every key valid, NaN == NaN,
-0.0 == 0.0) and whose `on` key is valid and not NaN.  A left row whose `on` is null or NaN gets no partner.  Among the candidates,
"searchsorted inside the `by` group" gives the picks: BACKWARD the last row of the greatest key <= l (< l without exact matches),
FORWARD the first row of the least key >= l (> l), NEAREST the nearer of the two, ties backward.  A pick farther than the tolerance is
dropped.  Integer distances are exact; float distances are the float64 difference, equal keys at distance 0.  Results are int64 right
row numbers, -1 for NULL.
"""
from __future__ import annotations

import numpy as np

from join_oracle import key_codes

DIRECTIONS = ("backward", "forward", "nearest")


def _order(v: np.ndarray) -> np.ndarray:
    """uint64 keys in the sort's order (floats: -0.0 == 0.0; NaNs are removed before this is used)."""
    if v.dtype.kind == "f":
        x = v.astype(np.float64)
        x = np.where(x == 0, 0.0, x)
        b = x.view(np.uint64)
        return np.where(b >> np.uint64(63), ~b, b | np.uint64(1 << 63))
    if v.dtype.kind == "i":
        return v.astype(np.int64).view(np.uint64) ^ np.uint64(1 << 63)
    return v.astype(np.uint64)


def _number(on) -> np.ndarray:
    v, m = on
    ok = np.asarray(m, bool).copy()
    if v.dtype.kind == "f":
        ok &= ~np.isnan(v)
    return ok


def _distance(v: np.ndarray, hi: np.ndarray, lo: np.ndarray):
    """Distance from lo to hi (hi >= lo in key order), element-wise: uint64 for integer keys, float64 for float keys."""
    if v.dtype.kind == "f":
        a, b = v[hi].astype(np.float64), v[lo].astype(np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            d = a - b
        return np.where(_order(v[hi]) == _order(v[lo]), 0.0, d)
    return _order(v[hi]) - _order(v[lo])


def join_asof(left_on, right_on, left_by=(), right_by=(), direction="backward", allow_exact_matches=True, tolerance=None) -> np.ndarray:
    assert direction in DIRECTIONS
    lv, rv = left_on[0], right_on[0]
    nl, nr = len(lv), len(rv)
    if left_by:
        lc, rc = key_codes(list(left_by), list(right_by))
    else:
        lc, rc = np.zeros(nl, np.int64), np.zeros(nr, np.int64)
    lok = _number(left_on) & (lc >= 0)
    rok = _number(right_on) & (rc >= 0)
    out = np.full(nl, -1, np.int64)
    if not lok.any() or not rok.any():
        return out
    # dense ranks of the on keys over both sides, so (group, rank) is one int64 that sorts like (group, on)
    keys = np.concatenate([_order(lv[lok]), _order(rv[rok])])
    _, rank = np.unique(keys, return_inverse=True)
    rank = rank.reshape(-1).astype(np.int64)
    span = int(rank.max()) + 1
    lrows, rrows = np.nonzero(lok)[0], np.nonzero(rok)[0]
    lcomp = lc[lrows] * span + rank[:lrows.size]
    rcomp = rc[rrows] * span + rank[lrows.size:]
    order = np.argsort(rcomp, kind="stable")                      # inside a (group, key) run: right row order
    rs, rcs, rgs = rrows[order], rcomp[order], rc[rrows][order]
    ge = np.searchsorted(rcs, lcomp, "left")
    gt = np.searchsorted(rcs, lcomp, "right")
    b = (gt if allow_exact_matches else ge) - 1
    f = ge if allow_exact_matches else gt
    g = lc[lrows]
    hb = (b >= 0) & (rgs[np.clip(b, 0, len(rs) - 1)] == g) & (direction != "forward")
    hf = (f < len(rs)) & (rgs[np.clip(f, 0, len(rs) - 1)] == g) & (direction != "backward")
    rb, rf = rs[np.clip(b, 0, len(rs) - 1)], rs[np.clip(f, 0, len(rs) - 1)]
    # distances: left minus backward pick, forward pick minus left; both indices into concatenated values
    both = np.concatenate([lv, rv])
    li = lrows
    db = _distance(both, li, nl + rb)
    df = _distance(both, nl + rf, li)
    back = hb & (~hf | (db <= df))
    pick = np.where(back, rb, rf)
    has = hb | hf
    if tolerance is not None:
        d = np.where(back, db, df)
        if lv.dtype.kind == "f":
            has &= d <= float(tolerance)
        else:
            has &= d <= np.uint64(int(tolerance))
    out[li[has]] = pick[has]
    return out


def join_exists(left, right, anti: bool) -> np.ndarray:
    """LEFT SEMI (anti=False) / LEFT ANTI: the left rows with (without) a partner, ascending, as int64."""
    lc, rc = key_codes(left, right)
    has = (lc >= 0) & np.isin(lc, rc[rc >= 0])
    return np.nonzero(~has if anti else has)[0].astype(np.int64)
