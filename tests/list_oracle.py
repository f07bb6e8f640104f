"""The list functions (include/b200df.h "list columns") restated in plain Python over lists of lists: None is a null list or a
null element.  Equality is the key equality of sort / group-by / join: integers exact, every NaN one value, -0.0 == 0.0."""
from __future__ import annotations

import math

import numpy as np

NULL = ("null",)


class Panic(Exception):
    """The reference panics (array_max / array_min of an empty list: .max().unwrap())."""


def key(x):
    if x is None:
        return NULL
    if isinstance(x, (float, np.floating)):
        if math.isnan(x):
            return ("nan",)
        return (float(x) + 0.0,)   # -0.0 + 0.0 == +0.0
    return (int(x),)


def _sort_key(x):
    if x is None:
        return (2, 0.0)
    if isinstance(x, (float, np.floating)) and math.isnan(x):
        return (1, 0.0)
    return (0, x)


def _total_order(x):   # group-by's float min / max: -0.0 < +0.0, NaN greatest
    if isinstance(x, (float, np.floating)):
        if math.isnan(x):
            return (2, 0.0, 0)
        return (1, float(x), 0 if math.copysign(1.0, x) < 0 else 1)
    return (1, int(x), 0)


def _canonical(x):   # NaN comes back as the positive quiet NaN
    if isinstance(x, (float, np.floating)) and math.isnan(x):
        return type(x)(np.nan) if isinstance(x, np.floating) else float("nan")
    return x


def array_contains(l, v):
    return None if l is None else any(x is not None and key(x) == key(v) for x in l)


def array_position(l, v):
    if l is None:
        return 0
    for i, x in enumerate(l):
        if x is not None and key(x) == key(v):
            return i + 1
    return 0


def _extreme(l, pick):
    if l is None:
        return None
    if not l:
        raise Panic("empty list")
    valid = [x for x in l if x is not None]
    return _canonical(pick(valid, key=_total_order)) if valid else None


def array_max(l):
    return _extreme(l, max)


def array_min(l):
    return _extreme(l, min)


def size(l):
    return -1 if l is None else len(l)


def array_remove(l, v):
    return [] if l is None else [x for x in l if x is None or key(x) != key(v)]


def array_sort(l):
    return [] if l is None else sorted(l, key=_sort_key)


def _distinct(xs):
    seen, out = set(), []
    for x in xs:
        k = key(x)
        if k not in seen:
            seen.add(k)
            out.append(x)
    return out


def array_distinct(l):
    return [] if l is None else _distinct(l)


def array_except(a, b):
    if a is None:
        return []
    kb = {key(x) for x in (b or [])}
    return [x for x in _distinct(a) if key(x) not in kb]


def array_intersect(a, b):
    if a is None:
        return []
    kb = {key(x) for x in (b or [])}
    return [x for x in _distinct(a) if key(x) in kb]


def array_union(a, b):
    return [] if a is None else _distinct(list(a) + list(b or []))


def array_repeat(l, count):
    if count < 0:
        raise ValueError("count < 0")
    return [] if l is None else list(l) * count


def explode(lists):
    rows, values = [], []
    for r, l in enumerate(lists):
        for x in (l or []):
            rows.append(r)
            values.append(x)
    return rows, values
