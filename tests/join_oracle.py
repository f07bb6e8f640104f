"""The equi-join of bdf_join_indices_dev restated in numpy (the checker of tests/test_join_gpu.py; itself checked against pyarrow
and pandas in tests/test_join.py).

A side is a list of criteria, each a pair (values, valid mask) of numpy arrays over the side's rows (chunks concatenated).
Match: every criterion valid on both rows and equal, with all NaNs equal and -0.0 == 0.0.  Order: left rows in row order, each
left row's partners in ascending right row order; LEFT keeps a left row without a partner once with a NULL right index; RIGHT is
LEFT with the sides swapped and the outputs swapped back; FULL is the LEFT output followed by every right row no left row matched,
in right row order, with a NULL left index.  Indices come back as int64 arrays with -1 for NULL.
"""
from __future__ import annotations

import numpy as np

HOWS = ("left", "right", "inner", "full")


def _bits(v: np.ndarray) -> np.ndarray:
    """A uint64 per value such that two values are equal as keys exactly when their codes are."""
    if v.dtype.kind == "f":
        x = v.astype(np.float64)
        x = np.where(x == 0, 0.0, x)              # -0.0 == 0.0
        x = np.where(np.isnan(x), np.nan, x)      # every NaN is one value
        return x.view(np.uint64)
    if v.dtype.kind == "i":
        return v.astype(np.int64).view(np.uint64)
    return v.astype(np.uint64)


def key_codes(left, right):
    """Integer codes of the key tuples of both sides (equal tuples, equal codes); -1 where a criterion is null."""
    nl, nr = len(left[0][0]), len(right[0][0])
    cols = np.stack([np.concatenate([_bits(lv), _bits(rv)]) for (lv, _), (rv, _) in zip(left, right)], axis=1)
    valid = np.ones(nl + nr, bool)
    for (_, lm), (_, rm) in zip(left, right):
        valid &= np.concatenate([np.asarray(lm, bool), np.asarray(rm, bool)])
    codes = np.full(nl + nr, -1, np.int64)
    if valid.any():
        _, inv = np.unique(cols[valid], axis=0, return_inverse=True)
        codes[valid] = inv.reshape(-1)
    return codes[:nl], codes[nl:]


def plan(left, right, how):
    """Per left row: its partners' first position in `rs` (right rows sorted by code, stable), its partner count and its output
    count; with `rs`, that is the whole LEFT / INNER output without writing it."""
    lc, rc = key_codes(left, right)
    order = np.argsort(rc, kind="stable")
    rs = order[rc[order] >= 0]
    rcs = rc[rs]
    lo = np.searchsorted(rcs, lc, "left")
    cnt = np.where(lc >= 0, np.searchsorted(rcs, lc, "right") - lo, 0)
    out_cnt = np.maximum(cnt, 1) if how in ("left", "full") else cnt
    return {"lc": lc, "rc": rc, "rs": rs, "lo": lo, "cnt": cnt, "out_cnt": out_cnt}


def pairs_at(p, pos: np.ndarray):
    """(left, right) of the LEFT / INNER output at the given positions (-1 = NULL)."""
    offs = np.cumsum(p["out_cnt"]) - p["out_cnt"]
    i = np.searchsorted(offs, pos, "right") - 1   # the last row starting at or before pos: rows without output share offsets
    j = pos - offs[i]
    r = np.full(i.shape, -1, np.int64)
    m = p["cnt"][i] > 0
    r[m] = p["rs"][p["lo"][i[m]] + j[m]]
    return i.astype(np.int64), r


def join_indices(left, right, how):
    """(left_idx, right_idx): int64 arrays, -1 = NULL."""
    assert how in HOWS
    if how == "right":
        r, l = join_indices(right, left, "left")
        return l, r
    p = plan(left, right, how)
    total = int(p["out_cnt"].sum())
    li, ri = pairs_at(p, np.arange(total, dtype=np.int64)) if total else (np.zeros(0, np.int64), np.zeros(0, np.int64))
    if how == "full":
        hit = np.isin(p["rc"], p["lc"][p["lc"] >= 0]) & (p["rc"] >= 0)
        extra = np.nonzero(~hit)[0]
        li = np.concatenate([li, np.full(extra.size, -1, np.int64)])
        ri = np.concatenate([ri, extra.astype(np.int64)])
    return li, ri
