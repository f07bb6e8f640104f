"""Numpy restatement of bdf_duplicated_dev and bdf_set_op_dev (include/b200df.h "distinct rows and set operations"): the checker of the
set-operation tests, never the thing under test.

A side is a list of key columns, each ``(values, valid)`` as numpy arrays of one length.  Key equality is group-by's, taken from
tests/group_by_oracle._canon: nulls equal each other, all NaNs are one value and -0.0 == 0.0.  The restatement is cross-checked
against pandas' duplicated, SQLite's INTERSECT / EXCEPT and collections.Counter arithmetic in tests/test_setops.py."""
from __future__ import annotations

import numpy as np

from group_by_oracle import _canon

KEEPS = ("first", "last", False)
OPS = ("intersect", "intersect_all", "except", "except_all")


def _bits(v: np.ndarray) -> np.ndarray:
    """The canonical values as uint64 bit patterns (one equality class per pattern)."""
    if v.dtype == bool:
        return v.astype(np.uint64)
    return v.view(f"u{v.dtype.itemsize}").astype(np.uint64)


def row_ids(sides):
    """One id per row of every side (the sides concatenated in order): equal rows get equal ids."""
    cols = []
    for k in range(len(sides[0])):
        v = np.concatenate([np.asarray(s[k][0]) for s in sides])
        m = np.concatenate([np.asarray(s[k][1], bool) for s in sides])
        c, nan = _canon(v, m)
        cols += [m.astype(np.uint64), nan.astype(np.uint64), _bits(c)]
    if not cols or cols[0].shape[0] == 0:
        return np.zeros(0, np.int64)
    _, inv = np.unique(np.stack(cols, axis=1), axis=0, return_inverse=True)
    return inv.reshape(-1).astype(np.int64)


def _ranks(g: np.ndarray):
    """(rank of every row among the earlier rows with its id, rows with its id)."""
    order = np.argsort(g, kind="stable")
    sg = g[order]
    start = np.r_[True, sg[1:] != sg[:-1]] if g.shape[0] else np.zeros(0, bool)
    run = np.cumsum(start) - 1
    first = np.flatnonzero(start)
    rank = np.empty(g.shape[0], np.int64)
    rank[order] = np.arange(g.shape[0]) - first[run]
    size = np.bincount(g, minlength=int(g.max()) + 1 if g.shape[0] else 0)
    return rank, size[g]


def duplicated(keys, keep="first") -> np.ndarray:
    """pandas' duplicated(keep=...) over the rows of `keys`."""
    g = row_ids([keys])
    rank, size = _ranks(g)
    if keep == "first":
        return rank > 0
    if keep == "last":
        return rank < size - 1
    if keep is False:
        return size > 1
    raise ValueError(keep)


def q_of(op: str, cl, cr):
    """The number of left rows a run with cl left and cr right rows keeps."""
    cl, cr = np.asarray(cl), np.asarray(cr)
    if op == "intersect":
        return ((cl > 0) & (cr > 0)).astype(np.int64)
    if op == "intersect_all":
        return np.minimum(cl, cr)
    if op == "except":
        return (cr == 0).astype(np.int64)
    if op == "except_all":
        return np.maximum(cl - cr, 0)
    raise ValueError(op)


def set_op(left, right, op: str) -> np.ndarray:
    """The keep-mask over the left rows: every run keeps its first q_of(op, cl, cr) left rows in row order."""
    nl = len(left[0][0])
    g = row_ids([left, right])
    gl, gr = g[:nl], g[nl:]
    n_ids = int(g.max()) + 1 if g.shape[0] else 0
    cl, cr = np.bincount(gl, minlength=n_ids), np.bincount(gr, minlength=n_ids)
    rank, _ = _ranks(gl)
    return rank < q_of(op, cl[gl], cr[gl])
