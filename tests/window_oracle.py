"""Numpy restatement of bdf_window_dev (include/b200df.h): the checker of the window tests, never the thing under test.

Chunks are duck-typed like the rest of the oracle: ``values`` (np.ndarray), ``offset``, ``length`` and ``valid_mask()``.  The reference
declares the window functions without bodies (src/functions/window.rs:1-11), so the operator is defined by the header; this restatement
is cross-checked against SQLite's window functions in tests/test_window.py."""
from __future__ import annotations

import numpy as np

RANKING = ("row_number", "rank", "dense_rank", "percent_rank", "cume_dist")
AGGREGATES = ("sum", "count", "min", "max", "avg")


def concat(chunks):
    if not chunks:
        return np.zeros(0), np.zeros(0, bool)
    v = np.concatenate([np.asarray(c.values)[c.offset:c.offset + c.length] for c in chunks])
    m = np.concatenate([np.asarray(c.valid_mask(), bool) for c in chunks])
    return v, m


def _key_parts(v, m, descending):
    """(null flag, NaN flag, value rank) of one criterion: nulls last in both directions, every NaN one value above every number,
    -0.0 == 0.0; descending reverses the valid values only."""
    if v.dtype.kind == "f":
        nan = np.isnan(v) & m
        c = np.where(np.isnan(v), 0.0, v) + 0.0
    else:
        nan = np.zeros(v.shape[0], bool)
        c = v
    c = np.where(m & ~nan, c, 0).astype(v.dtype)
    rank = np.unique(c, return_inverse=True)[1].astype(np.int64).reshape(-1)
    if descending:
        return ~m, np.where(m, ~nan, False), np.where(m & ~nan, -rank, 0)
    return ~m, nan, np.where(m & ~nan, rank, 0)


def _heads(parts, order, n):
    head = np.zeros(n, bool)
    if n:
        head[0] = True
    if n > 1:
        for p in parts:
            s = p[order]
            head[1:] |= s[1:] != s[:-1]
    return head


def _bounds(head, n):
    """first / last sorted position of the run of every position, and its run index."""
    rid = np.cumsum(head) - 1
    starts = np.nonzero(head)[0]
    ends = np.append(starts[1:], n) - 1
    return starts[rid], ends[rid], rid


def _seg_scan(a, first, op):
    """Inclusive scan of a within runs that start at first[i] (Hillis-Steele doubling: a fixed tree, no cancellation across runs)."""
    a = a.copy()
    n = a.shape[0]
    idx = np.arange(n)
    d = 1
    while d < n:
        ok = idx - d >= first
        b = a.copy()
        b[d:][ok[d:]] = op(a[d:][ok[d:]], a[:-d][ok[d:]])
        a = b
        d *= 2
    return a


def total_order_key(v):
    u = np.dtype(f"u{v.dtype.itemsize}")
    bits = np.where(np.isnan(v), np.array(np.nan, v.dtype), v).view(u)
    sign = u.type(1) << u.type(8 * v.dtype.itemsize - 1)
    return np.where(bits & sign, ~bits, bits | sign).astype(u)


def from_total_order_key(k, dtype):
    u = np.dtype(f"u{np.dtype(dtype).itemsize}")
    k = k.astype(u)
    sign = u.type(1) << u.type(8 * np.dtype(dtype).itemsize - 1)
    return np.where(k & sign, k ^ sign, ~k).astype(u).view(dtype)


def window(partition, order, calls, n=None):
    """partition: [chunks]; order: [(chunks, descending)]; calls: [(function, chunks or None, arg)] with arg the (offset, default)
    of lag / lead (default None: NULL) and the frame ("rows" | "range" | "partition") of an aggregate.  Returns one dict per call
    in row order: values, valid, and for float sum and for avg ``exact`` = (long-double sum of the frame's valid values,
    long-double sum of their magnitudes, frame rows), and for every aggregate ``count`` = the valid values of the frame."""
    keys = [(concat(ch), False) for ch in partition] + [(concat(ch), d) for ch, d in order]
    if n is None:
        n = keys[0][0][0].shape[0] if keys else concat(next(c[1] for c in calls if c[1] is not None))[0].shape[0]
    lex, pparts, oparts = [], [], []
    for k, ((v, m), d) in enumerate(keys):
        parts = _key_parts(v, m, d)
        (pparts if k < len(partition) else oparts).extend(parts)
    for (v, m), d in reversed(keys):
        nul, nan, rank = _key_parts(v, m, d)
        lex += [rank, nan, nul]
    order_idx = np.lexsort(lex) if lex and n else np.arange(n)   # stable: ties keep row order
    phead = _heads(pparts, order_idx, n)
    qhead = phead | _heads(oparts, order_idx, n)
    ps, pe, _ = _bounds(phead, n)
    qs, qe, qid = _bounds(qhead, n)
    pos = np.arange(n)
    rows = pe - ps + 1
    res = []
    for fn, chunks, arg in calls:
        sorted_out = None
        cnt = None
        if fn == "row_number":
            sorted_out = ((pos - ps + 1).astype(np.uint32), np.ones(n, bool), None)
        elif fn == "rank":
            sorted_out = ((qs - ps + 1).astype(np.uint32), np.ones(n, bool), None)
        elif fn == "dense_rank":
            sorted_out = ((qid - qid[ps] + 1).astype(np.uint32) if n else np.zeros(0, np.uint32), np.ones(n, bool), None)
        elif fn == "percent_rank":
            v = np.where(rows == 1, 0.0, (qs - ps).astype(np.float64) / np.maximum(rows - 1, 1).astype(np.float64))
            sorted_out = (v, np.ones(n, bool), None)
        elif fn == "cume_dist":
            sorted_out = ((qe - ps + 1).astype(np.float64) / rows.astype(np.float64), np.ones(n, bool), None)
        else:
            xv, xm = concat(chunks)
            sv, sm = xv[order_idx], xm[order_idx]
            if fn in ("lag", "lead"):
                k, default = arg
                j = pos - k if fn == "lag" else pos + k
                inside = (j >= ps) if fn == "lag" else (j <= pe)
                jj = np.clip(j, 0, max(n - 1, 0))
                vals = np.where(inside, np.where(sm[jj], sv[jj], 0), 0 if default is None else default).astype(xv.dtype)
                valid = np.where(inside, sm[jj], default is not None)
                sorted_out = (vals, valid, None)
            else:
                end = {"rows": pos, "range": qe, "partition": pe}[arg]
                cnt = _seg_scan(sm.astype(np.int64), ps, np.add)[end] if n else np.zeros(0, np.int64)
                has = cnt > 0
                exact = None
                if fn in ("sum", "avg") and (xv.dtype.kind == "f" or fn == "avg"):
                    ld = np.where(sm, sv, 0).astype(np.longdouble)
                    exact = (_seg_scan(ld, ps, np.add)[end], _seg_scan(np.abs(ld), ps, np.add)[end], end - ps + 1)
                if fn == "count":
                    sorted_out = (cnt, np.ones(n, bool), None)
                elif fn == "sum":
                    if xv.dtype.kind == "f":
                        vals = exact[0].astype(np.float64).astype(xv.dtype)
                    else:
                        u = np.where(sm, sv, 0).astype(xv.dtype).astype(np.int64 if xv.dtype.kind == "i" else np.uint64).view(np.uint64)
                        vals = _seg_scan(u, ps, np.add)[end].astype(xv.dtype)   # wrapping
                    sorted_out = (vals, np.ones(n, bool), exact)
                elif fn == "avg":
                    vals = np.where(has, (exact[0] / np.maximum(cnt, 1)).astype(np.float64), 0.0)
                    sorted_out = (vals, has, exact)
                else:
                    red = np.minimum if fn == "min" else np.maximum
                    if xv.dtype.kind == "f":
                        key = total_order_key(sv)
                        fill = np.iinfo(key.dtype).max if fn == "min" else 0
                        kk = _seg_scan(np.where(sm, key, fill).astype(key.dtype), ps, red)[end]
                        vals = from_total_order_key(kk, xv.dtype)
                    else:
                        info = np.iinfo(xv.dtype)
                        vals = _seg_scan(np.where(sm, sv, info.max if fn == "min" else info.min).astype(xv.dtype), ps, red)[end]
                    sorted_out = (np.where(has, vals, 0).astype(xv.dtype), has, None)
        v, m, ex = sorted_out
        out_cnt = None
        if cnt is not None:
            out_cnt = np.empty_like(cnt)
            out_cnt[order_idx] = cnt
        out_v = np.empty_like(v)
        out_m = np.empty_like(m)
        out_v[order_idx] = v
        out_m[order_idx] = m
        out_ex = None
        if ex is not None:
            out_ex = tuple(np.empty_like(e) for e in ex)
            for o, e in zip(out_ex, ex):
                o[order_idx] = e
        res.append(dict(values=out_v, valid=out_m, exact=out_ex, count=out_cnt))
    return res
