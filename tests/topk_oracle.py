"""A numpy restatement of bdf_top_k_indices_dev's rounds (include/b200df.h "top-k"), checked against the C oracle's lexsort in
test_topk.py.  A criterion is (values, valid, descending) over the concatenated rows.

Round j works on a tie set (row ids, ascending) and `need`, the rows still to choose.  With v valid keys in the tie set: need > v
chooses every valid row and makes the nulls the next ties; otherwise the threshold t is the key of rank need - 1 (ascending) or
v - need (descending) among the valid keys, BEFORE rows (key < t ascending, key > t descending) are chosen and the rows equal to t
tie.  When the ties hold exactly the rows still needed, or on the last criterion, the first `need` ties in row order are chosen.
The chosen rows, ascending, are then ordered by a stable sort of their criteria."""
from __future__ import annotations

from typing import List, Sequence, Tuple

import numpy as np

Criterion = Tuple[np.ndarray, np.ndarray, bool]


def sort_key(values: np.ndarray) -> np.ndarray:
    """The order-preserving uint64 key of DataFrame::sort: every NaN one value above +inf, -0.0 == 0.0."""
    v = np.asarray(values)
    if v.dtype.kind == "f":
        x = v.astype(np.float64)
        x = np.where(x == 0, 0.0, x)
        b = x.view(np.uint64)
        key = np.where(b >> np.uint64(63) != 0, ~b, b | np.uint64(1 << 63))
        return np.where(np.isnan(x), np.uint64(0xFFFFFFFFFFFFFFFF), key)
    if v.dtype.kind == "i":
        return (v.astype(np.int64).view(np.uint64) ^ np.uint64(1 << 63))
    return v.astype(np.uint64)


def _stable_order(keys: List[np.ndarray], valid: List[np.ndarray], desc: Sequence[bool]) -> np.ndarray:
    """Stable lexicographic order: per criterion nulls last, then the key ascending or descending."""
    cols = []
    for key, ok, d in zip(keys, valid, desc):
        cols.append(~ok)                                                  # nulls last in both directions
        cols.append(np.where(ok, ~key if d else key, np.uint64(0)))
    return np.lexsort(cols[::-1], axis=0) if cols else np.zeros(0, np.int64)


def chosen_rows(criteria: Sequence[Criterion], k: int) -> np.ndarray:
    """The rows the rounds choose, ascending."""
    n = len(criteria[0][0])
    need = min(max(k, 0), n)
    chosen = np.zeros(n, bool)
    tie = np.arange(n)
    for j, (values, valid, desc) in enumerate(criteria):
        if need == 0:
            break
        key, ok = sort_key(values)[tie], np.asarray(valid, bool)[tie]
        v = int(ok.sum())
        if need > v:
            before, equal = ok, ~ok
        else:
            ranked = np.sort(key[ok])
            t = ranked[v - need] if desc else ranked[need - 1]
            before = ok & ((key > t) if desc else (key < t))
            equal = ok & (key == t)
        chosen[tie[before]] = True
        need -= int(before.sum())
        if need == 0:
            break
        tie = tie[equal]
        if len(tie) == need or j + 1 == len(criteria):
            chosen[tie[:need]] = True
            break
    return np.flatnonzero(chosen)


def top_k(criteria: Sequence[Criterion], k: int) -> np.ndarray:
    """The first min(k, n) rows of the stable sort, as uint32 row numbers."""
    rows = chosen_rows(criteria, k)
    order = _stable_order([sort_key(v)[rows] for v, _, _ in criteria], [np.asarray(m, bool)[rows] for _, m, _ in criteria],
                          [d for _, _, d in criteria])
    return rows[order].astype(np.uint32)
