"""Whole lists moved between rows, and lists built per group (include/b200df.h bdf_list_take_dev, bdf_list_filter_dev and
bdf_group_by_lists_dev), restated in plain Python over lists of lists: None is a null list, a null element, a null index or a null
key.  Equality and order are those of sort / group-by: integers exact, every NaN one value and greatest, -0.0 == 0.0."""
from __future__ import annotations

import math

import numpy as np

from list_oracle import key


def take(lists, indices):
    """Column::take of whole lists: a null index gives a null list; an index past the end is an error."""
    out = []
    for i in indices:
        if i is None:
            out.append(None)
            continue
        if not 0 <= i < len(lists):
            raise IndexError(i)
        out.append(lists[i])
    return out


def filter_(lists, mask):
    """The lists where the mask is valid and true."""
    return [l for l, m in zip(lists, mask) if m is True]


def _order(x):
    """Ascending sort order of one key value: numbers, then NaN, then null."""
    if x is None:
        return (2, 0)
    if isinstance(x, (float, np.floating)):
        if math.isnan(x):
            return (1, 0)
        return (0, float(x) + 0.0)
    return (0, int(x))


def groups(keys):
    """The groups of the key tuples (keys: one list per key column) in DataFrame::sort order: [(key tuple, [rows in row order])]."""
    n = len(keys[0]) if keys else 0
    by = {}
    for r in range(n):
        k = tuple(key(col[r]) for col in keys)
        by.setdefault(k, (tuple(col[r] for col in keys), []))[1].append(r)
    return sorted(by.values(), key=lambda g: tuple(_order(v) for v in g[0]))


def collect_list(keys, x):
    """[(key tuple, list)]: the valid values of every group in row order; a group without one gives []."""
    return [(k, [x[r] for r in rows if x[r] is not None]) for k, rows in groups(keys)]


def collect_set(keys, x):
    """[(key tuple, list)]: the distinct valid values of every group, ascending (NaN greatest), each with the bits of its first
    occurrence in row order."""
    out = []
    for k, rows in groups(keys):
        first = {}
        for r in rows:
            if x[r] is not None and key(x[r]) not in first:
                first[key(x[r])] = x[r]
        out.append((k, sorted(first.values(), key=_order)))
    return out
