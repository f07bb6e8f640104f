"""Numpy restatement of bdf_window_dev's bounded frames and value functions (include/b200df.h, "Bounded frames"): the checker of the
frame tests, never the thing under test.  Frames are resolved row by row from the header's rules and aggregated over the resolved
positions directly; this restatement is cross-checked against SQLite's frames in tests/test_window_frames.py.

A frame is "rows" | "range" | "partition" (the existing frames) or ("rows" | "range", start, end) with signed offsets, None meaning
UNBOUNDED.  Calls are (function, chunks, arg): arg is the frame of an aggregate, and (frame, n, ignore_nulls) of first_value,
last_value and nth_value.  Results are dicts as window_oracle.window returns them."""
from __future__ import annotations

import bisect

import numpy as np

from window_oracle import _bounds, _heads, _key_parts, concat, from_total_order_key, total_order_key

VALUES = ("first_value", "last_value", "nth_value")


def _sorted_space(partition, order, n):
    keys = [(concat(ch), False) for ch in partition] + [(concat(ch), d) for ch, d in order]
    lex, pparts, oparts = [], [], []
    for k, ((v, m), d) in enumerate(keys):
        (pparts if k < len(partition) else oparts).extend(_key_parts(v, m, d))
    for (v, m), d in reversed(keys):
        nul, nan, rank = _key_parts(v, m, d)
        lex += [rank, nan, nul]
    idx = np.lexsort(lex) if lex and n else np.arange(n)   # stable: ties keep row order
    phead = _heads(pparts, idx, n)
    qhead = phead | _heads(oparts, idx, n)
    ps, pe, _ = _bounds(phead, n)
    _, qe, _ = _bounds(qhead, n)
    return idx, ps, pe, qe


def _range_bounds(key, desc, lo_hi, idx, ps, pe):
    """RANGE BETWEEN over one order key (chunks): [s, e] of every sorted position."""
    v, m = concat(key)
    v, m = v[idx], m[idx]
    is_f = v.dtype.kind == "f"
    nan = np.isnan(v) & m if is_f else np.zeros(v.shape[0], bool)
    cls = np.where(~m, 2, np.where(nan, 0 if desc else 1, 1 if desc else 0))
    num = 1 if desc else 0
    start, end = lo_hi
    n = v.shape[0]
    s, e = ps.copy(), pe.copy()
    conv = float if is_f else int
    part_start = np.unique(ps)
    for p0 in part_start:
        p1 = pe[p0]
        c = cls[p0:p1 + 1]
        a = p0 + int(np.searchsorted(c, num, "left"))
        b = p0 + int(np.searchsorted(c, num, "right"))   # numbers: [a, b)
        keys = [conv(x) for x in v[a:b]]
        neg = [-x for x in keys] if desc else keys       # ascending either way
        for i in range(p0, p1 + 1):
            if cls[i] != num:
                run = (p0 + int(np.searchsorted(c, cls[i], "left")), p0 + int(np.searchsorted(c, cls[i], "right")) - 1)
                if start is not None:
                    s[i] = run[0]
                if end is not None:
                    e[i] = run[1]
                continue
            x = conv(v[i])
            if start is not None:
                t = x - start if desc else x + start
                s[i] = a + (bisect.bisect_left(neg, -t) if desc else bisect.bisect_left(neg, t))
            if end is not None:
                t = x - end if desc else x + end
                e[i] = a + (bisect.bisect_right(neg, -t) if desc else bisect.bisect_right(neg, t)) - 1
    return s, e


def frame_bounds(partition, order, frame, n):
    """(sorted order, s, e) of every sorted position for one frame."""
    idx, ps, pe, qe = _sorted_space(partition, order, n)
    pos = np.arange(n)
    if frame == "rows":
        return idx, ps, pos
    if frame == "range":
        return idx, ps, qe
    if frame == "partition":
        return idx, ps, pe.copy()
    kind, start, end = frame
    if kind == "rows":
        s = ps if start is None else np.maximum(ps, pos + start)
        e = pe if end is None else np.minimum(pe, pos + end)
        return idx, s, e
    assert len(order) == 1, "RANGE BETWEEN needs exactly one order column"
    s, e = _range_bounds(order[0][0], order[0][1], (start, end), idx, ps, pe)
    return idx, s, e


def _sparse_table(a, red):
    t = [a]
    k = 1
    while 2 * k <= a.shape[0]:
        t.append(red(t[-1][:-k], t[-1][k:]))
        k *= 2
    return t


def _range_reduce(a, s, e, red, fill):
    """red over a[s..e] for every row (fill where s > e), with a sparse table: O(n log n)."""
    out = np.full(s.shape[0], fill, a.dtype)
    ok = s <= e
    if not ok.any():
        return out
    t = _sparse_table(a, red)
    ln = e[ok] - s[ok] + 1
    lv = np.floor(np.log2(ln)).astype(np.int64)
    res = np.empty(int(ok.sum()), a.dtype)
    for k in np.unique(lv):
        sel = lv == k
        ss, ee = s[ok][sel], e[ok][sel]
        res[sel] = red(t[k][ss], t[k][ee - (1 << k) + 1])
    out[ok] = res
    return out


def _prefix(a):
    return np.concatenate([np.zeros(1, a.dtype), np.cumsum(a)])


def _frame_sums(sv, sm, s, e):
    """(exact sum, sum of magnitudes) over [s, e] as long doubles, NaN / inf by IEEE rules.  Finite values that are multiples of 2^-20
    below 2^40 are summed exactly through integer prefixes; other inputs frame by frame."""
    n = s.shape[0]
    ok = s <= e
    ss, ee = np.where(ok, s, 0), np.where(ok, e + 1, 0)
    x = np.where(sm, sv, 0).astype(np.float64)
    fin = np.isfinite(x)
    cnt = lambda b: np.where(ok, _prefix(b.astype(np.int64))[ee] - _prefix(b.astype(np.int64))[ss], 0)
    n_nan, n_pinf, n_ninf = cnt(np.isnan(x)), cnt(x == np.inf), cnt(x == -np.inf)
    xf = np.where(fin, x, 0.0)
    scaled = xf * 2.0 ** 20
    if np.all(scaled == np.round(scaled)) and np.all(np.abs(scaled) < 2.0 ** 40):
        q = scaled.astype(np.int64)
        P, A = _prefix(q), _prefix(np.abs(q))
        exact = np.where(ok, (P[ee] - P[ss]), 0).astype(np.longdouble) / np.longdouble(2.0 ** 20)
        mag = np.where(ok, (A[ee] - A[ss]), 0).astype(np.longdouble) / np.longdouble(2.0 ** 20)
    else:
        ld = xf.astype(np.longdouble)
        exact = np.zeros(n, np.longdouble)
        mag = np.zeros(n, np.longdouble)
        for i in np.nonzero(ok)[0]:
            w = ld[s[i]:e[i] + 1]
            exact[i] = w.sum()
            mag[i] = np.abs(w).sum()
    exact = np.where(n_pinf > 0, np.inf, exact)
    exact = np.where(n_ninf > 0, -np.inf, exact)
    exact = np.where((n_nan > 0) | ((n_pinf > 0) & (n_ninf > 0)), np.nan, exact).astype(np.longdouble)
    return exact, mag


def _aggregate(fn, xv, sv, sm, s, e):
    ok = s <= e
    ss, ee = np.where(ok, s, 0), np.where(ok, e + 1, 0)
    C = _prefix(sm.astype(np.int64))
    cnt = np.where(ok, C[ee] - C[ss], 0)
    has = cnt > 0
    k = np.maximum(e - s + 1, 0)
    exact = None
    if fn in ("sum", "avg") and (xv.dtype.kind == "f" or fn == "avg"):
        ex, mag = _frame_sums(sv, sm, s, e)
        exact = (ex, mag, k)
    if fn == "count":
        return cnt, np.ones(s.shape[0], bool), None, cnt
    if fn == "sum":
        if xv.dtype.kind == "f":
            vals = exact[0].astype(np.float64).astype(xv.dtype)
        else:
            u = np.where(sm, sv, 0).astype(xv.dtype).astype(np.int64 if xv.dtype.kind == "i" else np.uint64).view(np.uint64)
            P = _prefix(u)   # wrapping
            vals = np.where(ok, P[ee] - P[ss], 0).astype(np.uint64).astype(xv.dtype)
        return vals, np.ones(s.shape[0], bool), exact, cnt
    if fn == "avg":
        vals = np.where(has, (exact[0] / np.maximum(cnt, 1)).astype(np.float64), 0.0)
        return vals, has, exact, cnt
    red = np.minimum if fn == "min" else np.maximum
    if xv.dtype.kind == "f":
        key = total_order_key(sv)
        fill = np.iinfo(key.dtype).max if fn == "min" else 0
        kk = _range_reduce(np.where(sm, key, fill).astype(key.dtype), s, e, red, fill)
        vals = from_total_order_key(kk, xv.dtype)
    else:
        info = np.iinfo(xv.dtype)
        fill = info.max if fn == "min" else info.min
        vals = _range_reduce(np.where(sm, sv, fill).astype(xv.dtype), s, e, red, fill)
    return np.where(has, vals, 0).astype(xv.dtype), has, None, cnt


def _value(fn, xv, sv, sm, s, e, nth, ignore_nulls):
    n = s.shape[0]
    ok = s <= e
    want = 1 if fn == "first_value" else nth
    if not ignore_nulls:
        j = s if fn == "first_value" else e if fn == "last_value" else s + nth - 1
        found = ok & (j <= e)
    else:
        C = _prefix(sm.astype(np.int64))
        ss, ee = np.where(ok, s, 0), np.where(ok, e + 1, 0)
        before, have = C[ss], np.where(ok, C[ee] - C[ss], 0)
        rank = have if fn == "last_value" else np.full(n, want, np.int64)   # the rank-th valid slot of the frame
        found = ok & (rank >= 1) & (rank <= have)
        valid_pos = np.nonzero(sm)[0]
        j = np.where(found, valid_pos[np.clip(before + rank - 1, 0, max(valid_pos.shape[0] - 1, 0))] if valid_pos.shape[0] else 0, 0)
    jj = np.clip(np.where(found, j, 0), 0, max(n - 1, 0))
    valid = found & sm[jj] if n else np.zeros(0, bool)
    vals = np.where(valid, sv[jj], 0).astype(xv.dtype) if n else np.zeros(0, xv.dtype)
    return vals, valid, None, None


def window(partition, order, calls, n=None):
    """partition: [chunks]; order: [(chunks, descending)]; calls: [(function, chunks, arg)] of aggregates (arg = frame) and value
    functions (arg = (frame, n, ignore_nulls)).  Returns one dict per call in row order: values, valid, and as window_oracle.window
    ``exact`` = (exact sum, sum of magnitudes, frame rows) for float sum and avg, and ``count`` for aggregates."""
    if n is None:
        first = partition[0] if partition else order[0][0] if order else next(c[1] for c in calls)
        n = concat(first)[0].shape[0]
    res = []
    for fn, chunks, arg in calls:
        frame, nth, ign = (arg, None, False) if fn not in VALUES else arg
        if frame is None:
            frame = "range" if order else "partition"
        idx, s, e = frame_bounds(partition, order, frame, n)
        xv, xm = concat(chunks)
        sv, sm = xv[idx], xm[idx]
        if fn in VALUES:
            v, m, ex, cnt = _value(fn, xv, sv, sm, s, e, nth, ign)
        else:
            v, m, ex, cnt = _aggregate(fn, xv, sv, sm, s, e)
        back = lambda a: None if a is None else _unsort(a, idx)
        res.append(dict(values=back(v), valid=back(m), exact=None if ex is None else tuple(back(a) for a in ex), count=back(cnt),
                        bounds=(back(s), back(e))))
    return res


def _unsort(a, idx):
    out = np.empty_like(a)
    out[idx] = a
    return out
