"""numpy restatements of the distribution rules of include/b200df.h ("distributions"): the exact percentile, mode and uniques under the
sort's key equality, and numpy.histogram with the stated range rules.  Every GPU result is compared bit for bit with these."""
import numpy as np

QNAN = np.frombuffer(np.uint64(0x7FF8000000000000).tobytes(), dtype=np.float64)[0]


def canonical(x: float) -> float:
    """What a key stands for: +0.0 for a zero, the positive quiet NaN for NaN."""
    x = float(x)
    if x != x:
        return float(QNAN)
    return 0.0 if x == 0.0 else x


def quiet(x: float) -> float:
    return float(QNAN) if x != x else x


def key_sorted(v: np.ndarray) -> np.ndarray:
    """The valid values in the sort's key order, read as f64 (NaN last; -0.0 and 0.0 equal)."""
    f = v.astype(np.float64)
    if v.dtype.kind in "iu":
        return np.sort(v, kind="stable").astype(np.float64)
    return np.sort(f, kind="stable")   # numpy puts NaN last, and sorts -0.0 == 0.0 stably


def interp(a: float, b: float, pos: float, lo: float, hi: float) -> float:
    """The stated sequence: a when lo == hi or a == b, else (hi - pos) * a + (pos - lo) * b, one rounding per operation."""
    a, b = canonical(a), canonical(b)
    if lo == hi or a == b:
        return quiet(a)
    with np.errstate(invalid="ignore", over="ignore"):
        r = float(np.float64(np.float64(hi - pos) * np.float64(a)) + np.float64(np.float64(pos - lo) * np.float64(b)))
    return quiet(r)


def percentile(valid: np.ndarray, p: float):
    """Spark's exact percentile of the valid values (any numeric dtype); None without a value."""
    n = len(valid)
    if n == 0:
        return None
    s = key_sorted(valid)
    if valid.dtype.kind in "iu":   # order by the integers, then read as f64 (Int64 beyond 2^53 rounds)
        s = np.sort(valid, kind="stable")
    pos = float(np.float64(n - 1) * np.float64(p))
    lo, hi = np.floor(pos), np.ceil(pos)
    return interp(float(s[int(lo)]), float(s[int(hi)]), pos, lo, hi)


def _key_classes(valid: np.ndarray):
    """(representative, count) per class in ascending key order; the representative is the class's first element in row order."""
    if valid.dtype.kind == "f":
        k = valid.astype(np.float64)
        k = np.where(k == 0, 0.0, k)
        isnan = np.isnan(k)
        keyed = [(2, 0.0) if isnan[i] else (1, k[i]) for i in range(len(k))]
    else:
        keyed = [(1, int(x)) for x in valid]
    order = sorted(range(len(valid)), key=lambda i: keyed[i])   # Python's sort is stable: first row of a class first
    out = []
    for i in order:
        if out and keyed[out[-1][2]] == keyed[i]:
            out[-1][1] += 1
        else:
            out.append([valid[i], 1, i])
    return [(rep, cnt) for rep, cnt, _ in out]


def uniques(valid: np.ndarray):
    """(values, counts): the distinct valid values ascending, each the first of its class in row order."""
    cl = _key_classes(valid)
    return np.array([c[0] for c in cl], dtype=valid.dtype), np.array([c[1] for c in cl], dtype=np.int64)


def mode(valid: np.ndarray):
    """(value, frequency) of the most frequent class, ties to the smallest key; (None, 0) without a value."""
    cl = _key_classes(valid)
    if not cl:
        return None, 0
    best = max(range(len(cl)), key=lambda i: (cl[i][1], -i))
    return cl[best][0], cl[best][1]


def hist_range(valid: np.ndarray, rng=None):
    """The (lo, hi) the histogram uses before numpy's lo == hi widening: the explicit range, else [min, max] of the non-NaN values
    (a -0.0 bound is +0.0), else [0, 1]."""
    if rng is not None:
        return float(rng[0]), float(rng[1])
    f = valid.astype(np.float64)
    f = f[~np.isnan(f)]
    if len(f) == 0:
        return 0.0, 1.0
    return float(f.min()) + 0.0, float(f.max()) + 0.0


def histogram(valid: np.ndarray, nbins: int, rng=None):
    """numpy.histogram over the valid values read as f64, NaN dropped, with the stated range."""
    f = valid.astype(np.float64)
    f = f[~np.isnan(f)]
    lo, hi = hist_range(valid, rng)
    counts, edges = np.histogram(f, nbins, range=(lo, hi))
    return edges, counts.astype(np.int64)


def edges_restated(lo: float, hi: float, nbins: int) -> np.ndarray:
    """The header's edge rule: edges[i] = i * ((hi - lo) / nbins) + lo in two roundings (i / nbins * (hi - lo) + lo when the step is 0),
    edges[nbins] = hi; lo == hi widened by 0.5 first."""
    if lo == hi:
        lo, hi = lo - 0.5, hi + 0.5
    delta = np.float64(hi) - np.float64(lo)
    step = delta / np.float64(nbins)
    i = np.arange(nbins + 1, dtype=np.float64)
    e = (i / nbins * delta + lo) if step == 0 else (i * step + np.float64(lo))
    e[-1] = hi
    return e


def bins_restated(x: np.ndarray, edges: np.ndarray) -> np.ndarray:
    """The header's bin rule with numpy's one-step correction; x already restricted to [edges[0], edges[-1]]."""
    nb = len(edges) - 1
    lo, hi = edges[0], edges[-1]
    i = ((x - lo) / (hi - lo) * nb).astype(np.int64)
    i = np.minimum(i, nb - 1)
    dec = x < edges[i]
    i[dec] -= 1
    inc = (x >= edges[i + 1]) & (i != nb - 1)
    i[inc] += 1
    return np.bincount(i, minlength=nb).astype(np.int64)
