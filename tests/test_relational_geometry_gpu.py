"""The sort-based operators where their geometry changes, against the CPU references bit for bit.

Sort, group-by, join, window, lists and distributions all sit on the stable radix sort, and every one of their kernels switches
path at constants of its own.  The tests here put lengths, group sizes, list lengths and candidate counts exactly on those
switch points instead of leaving them to random sizes:

  * radix sort (k_sort.cu): SORT_TILE-key tiles, and the first lengths where a CTA of the capped grid (SORT_CTAS_PER_SM x SMs)
    walks two tiles and carries its digit bases; 32- and 64-bit keys; key sets built for the skipped-digit rule, whose pass
    count is read back from the sort's launch record;
  * the one-CTA scans of 1024 threads (k_scan_one, k_window_carry): 1023, 1024, 1025 and 2049 totals;
  * the group fold (k_group.cu): each lane count, groups of LANE_ROWS x LANES (+1) rows and of one and two BIG_GROUP segments (+1),
    extremes planted on segment and group ends, an all-null long group, a cancelling float column held to the stated sum bar;
  * list find (k_list.cu): each lane count, lists on the long-path threshold and on LONG_LIST segment ends, first matches
    planted on both sides of a segment boundary;
  * the select histogram (k_dist.cu): exactly SEL_SMEM_BINS / 256 candidate prefixes at a level (shared memory), then one more
    (global atomics).

A non-GPU test re-reads every constant from csrc/, so a retuned kernel fails loudly here instead of silently testing the wrong
edges.  The 2^31..2^32-1 row range that UInt32 sort indices allow is not covered: a sort there needs ~45 GB of device memory.
"""
import math
import os
import re
from fractions import Fraction

import numpy as np
import pytest

import distribution_oracle as do
import group_by_oracle as gbo
import join_oracle as jo
import list_oracle as lo
import window_frame_oracle as WF
import window_oracle as W
from helpers import assert_same_array

gpu = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "rust-dataframe_b200", "csrc")

# ---------------------------------------------------------------------------------------------------------
# the constants; test_switch_points_match_csrc re-reads every one of them from the sources

THREADS = 256                  # common.cuh kThreads
SORT_TILE = 512 * 8            # k_sort.cu kSortTile = kSortThreads * kSortItems: keys per scatter tile
SORT_CTAS_PER_SM = 4           # k_sort.cu sort_pass_ctas: the grid of a pass is at most 4 x SMs CTAs
SCAN_THREADS = 1024            # k_scan_one / k_window_carry: one CTA, each thread owns ceil(count / 1024) totals
JOIN_TILE = THREADS * 8        # k_join.cu kJoinTile = scan.cuh kScanTile: probe rows per CTA total
WIN_TILE = THREADS * 8         # k_window.cu kWinTile: rows per scan tile
LANE_RULE = (64, 4)            # k_group.cu / k_list.cu: lanes = avg > 64 ? 32 : avg > 4 ? 8 : 1
LANE_ROWS = 512                # k_group.cu kLaneRows: a 1- or 8-lane group longer than LANE_ROWS x LANES goes to k_group_medium
BIG_GROUP = 65536              # k_group.cu kBigGroup: longer groups go to k_group_big, in segments of this many rows
LANE_ROUNDS = 64               # k_list.cu kLaneRounds: a list longer than LANE_ROUNDS x LANES goes to k_list_find_long
LONG_LIST = 16384              # k_list.cu kLongList: elements per segment of k_list_find_long
SEL_SMEM_BINS = 8192           # k_dist.cu kSelSmemBins: select bins (prefixes x 256 digits) counted in shared memory
SEL_SMEM_PREFIXES = SEL_SMEM_BINS // 256


def lanes_for(avg):
    return 32 if avg > LANE_RULE[0] else 8 if avg > LANE_RULE[1] else 1


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_switch_points_match_csrc():
    """Every switch point above, read back from the kernel sources (the SM count comes from the device at run time)."""
    common, srt, runtime = _read("common.cuh"), _read("k_sort.cu"), _read("runtime.cu")
    scan_h, scan, csvw = _read("scan.cuh"), _read("k_scan.cu"), _read("k_csv_write.cu")
    join, win, grp, lst, dist = _read("k_join.cu"), _read("k_window.cu"), _read("k_group.cu"), _read("k_list.cu"), _read("k_dist.cu")

    def num(src, pat):
        m = re.search(pat, src)
        assert m, f"pattern {pat!r} not found"
        return int(m.group(1))

    assert num(common, r"constexpr int kThreads = (\d+);") == THREADS
    # radix sort: tile, grid cap, key widths, the skipped digit and the launch record's bytes
    items, sthreads = num(srt, r"constexpr int kSortItems = (\d+);"), num(srt, r"constexpr int kSortThreads = (\d+);")
    assert re.search(r"constexpr int kSortTile = kSortThreads \* kSortItems;", srt) and items * sthreads == SORT_TILE
    assert num(srt, r"std::min<int64_t>\(tiles, \(int64_t\)sm_count \* (\d+)\)") == SORT_CTAS_PER_SM
    assert re.search(r"int sort_key_bytes\(int dtype\) \{ return dtype_width\(dtype\) <= 4 \? 4 : 8; \}", srt)
    for t in ("int8_t", "int16_t", "int32_t", "uint8_t", "uint16_t", "uint32_t", "float"):
        assert re.search(r"template <> struct KeyOf<%s> \{ using type = uint32_t; \};" % t, srt), t
    assert re.search(r"sizeof\(K\) == 4 \? digit_peers\(d\) : __match_any_sync", srt)
    assert re.search(r"if \(descending\) k = ~k & MASK;", srt)
    assert re.search(r"for \(int mode = 0; mode < \(nullable \? 2 : 1\)", runtime)
    assert re.search(r"if \(\(\(differ >> \(8 \* d\)\) & 0xff\) == 0\) continue;", runtime)
    assert re.search(r"pass_bytes \+= \(int64_t\)\(3 \* kb \+ 8\) \* n;", runtime)
    assert re.search(r"rec\.bytes = 8 \* n \+ pass_bytes \+ 4 \* n;", runtime)
    # the 1024-thread scans
    for src, pat in ((srt, r"launch_scan_one<unsigned int>\(block_hist, "), (scan, r"__launch_bounds__\(1024\) k_scan_one\("),
                     (scan, r"k_scan_one<T><<<1, 1024, 0, s>>>"), (scan, r"k_scan_one<unsigned long long><<<1, 1024, 0, s>>>\(sums, tiles, data \+ n\)"),
                     (win, r"constexpr int kWinCarryThreads = (\d+);")):
        assert re.search(pat, src), pat
    assert num(win, r"constexpr int kWinCarryThreads = (\d+);") == SCAN_THREADS
    assert re.search(r"per = \(count \+ 1023\) / 1024;", scan) and re.search(r"per = \(n_tiles \+ kWinCarryThreads - 1\) / kWinCarryThreads;", win)
    assert re.search(r"constexpr int kScanTile = kThreads \* kScanItems;", scan_h) and THREADS * num(scan_h, r"constexpr int kScanItems = (\d+);") == JOIN_TILE
    assert re.search(r"constexpr int kJoinTile = kScanTile;", join) and re.search(r"constexpr int kCsvwTile = kScanTile;", csvw)
    assert re.search(r"constexpr int kWinTile = kThreads \* kWinItems;", win) and THREADS * num(win, r"constexpr int kWinItems = (\d+);") == WIN_TILE
    # group fold and list find: the lane rule in both, the thresholds of the second paths
    for src in (grp, lst):
        m = re.search(r"const int lanes = avg > (\d+) \? 32 : avg > (\d+) \? 8 : 1;", src)
        assert m and (int(m.group(1)), int(m.group(2))) == LANE_RULE
    assert num(grp, r"constexpr long long kBigGroup = (\d+);") == BIG_GROUP
    assert num(grp, r"constexpr long long kLaneRows = (\d+);") == LANE_ROWS
    assert re.search(r"if \(mine && big && e - b > kBigGroup\)", grp) and re.search(r"LANES < 32 && mine && big && e - b > kLaneRows \* LANES", grp)
    assert re.search(r"if \(LANES == 1\) out\.nonempty\[g0 >> 5\] = word;", grp)
    assert num(lst, r"constexpr long long kLongList = (\d+);") == LONG_LIST
    assert num(lst, r"constexpr long long kLaneRounds = (\d+);") == LANE_ROUNDS
    assert re.search(r"if \(e - b > kLaneRounds \* LANES\)", lst)
    # select
    assert num(dist, r"constexpr int kSelSmemBins = (\d+);") == SEL_SMEM_BINS
    assert re.search(r"unsigned int\* sh = n_bins <= kSelSmemBins \? s_bins : nullptr;", dist)
    assert SORT_TILE == 4096 and JOIN_TILE == WIN_TILE == 2048 and SEL_SMEM_PREFIXES == 32


# ---------------------------------------------------------------------------------------------------------
# helpers

def sm_count(ctx):
    return ctx.device_info()["sm_count"]


def chunked(rdf, v, m, n_chunks, rng, sliced=True):
    """v (and mask m or None) as n_chunks ragged chunks, each a slice at offset 1..7 of a padded array when sliced."""
    n = v.shape[0]
    cuts = np.sort(rng.choice(np.arange(1, n), size=min(n_chunks - 1, max(n - 1, 0)), replace=False)) if n > 1 else np.zeros(0, int)
    bounds = [0] + [int(c) for c in cuts] + [n]
    out = []
    for k, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        off = (k * 3 + 1) % 8 if sliced else 0
        pv = np.concatenate([np.zeros(off, v.dtype), v[a:b]])
        pm = None if m is None else np.concatenate([np.zeros(off, bool), m[a:b]])
        arr = rdf.PrimitiveArray.from_numpy(pv, pm)
        arr.null_count = 0 if pm is None else -1
        out.append(arr.slice(off, b - a))
    return out


def one(col):
    arrs = col.download()
    assert len(arrs) == 1
    return arrs[0].value_slice(), arrs[0].valid_mask()


def assert_bits(got, gm, want, wm, what):
    """Same validity, and the same bits under it (NaNs compared as a class)."""
    assert np.array_equal(gm, wm), f"{what}: validity differs at {np.nonzero(gm != wm)[0][:5]}"
    g, w = got[gm], np.ascontiguousarray(np.asarray(want)[wm], dtype=got.dtype)
    if g.dtype.kind == "f":
        nan = np.isnan(g)
        assert np.array_equal(nan, np.isnan(w)), what
        g, w = g[~nan], w[~nan]
    u = np.dtype(f"u{g.dtype.itemsize}")
    bad = np.nonzero(g.view(u) != w.view(u))[0]
    assert bad.size == 0, f"{what}: {bad.size} values differ, first at {bad[:5]}: got {g[bad[:5]]}, want {w[bad[:5]]}"


# ---------------------------------------------------------------------------------------------------------
# radix sort

SORT_TYPES = ["I32", "U32", "F32", "I64", "U64", "F64"]   # one 32-bit-key and one 64-bit-key type of each kind


def np_dtype(tname):
    return np.dtype({"I32": np.int32, "U32": np.uint32, "F32": np.float32, "I64": np.int64, "U64": np.uint64, "F64": np.float64}[tname])


def sort_keys(v, valid, descending):
    """The kernel's keys (k_sort_keys): order-preserving unsigned keys of the type's width, -0.0 == 0.0, every NaN the largest key,
    ~k for descending, 0 for a null slot."""
    w = v.dtype.itemsize
    u = np.dtype(f"u{w}")
    sign = u.type(1) << u.type(8 * w - 1)
    if v.dtype.kind == "i":
        k = v.view(u) ^ sign
    elif v.dtype.kind == "u":
        k = v.copy()
    else:
        x = np.where(v == 0, v.dtype.type(0), v)
        b = x.view(u)
        k = np.where(b & sign, ~b, b | sign).astype(u)
        k[np.isnan(v)] = ~u.type(0)
    if descending:
        k = ~k
    k = np.where(valid, k, u.type(0)).astype(u)
    return k


def expected_passes(v, valid, descending):
    """Radix passes the digit skip leaves: one per byte on which the keys are not all equal, plus the null-flag pass when some
    rows are null and some are not."""
    k = sort_keys(v, valid, descending).astype(np.uint64)
    differ = int(np.bitwise_or.reduce(k)) ^ int(np.bitwise_and.reduce(k))
    passes = sum(1 for d in range(v.dtype.itemsize) if (differ >> (8 * d)) & 0xff)
    return passes + (1 if valid.any() and not valid.all() else 0)


def from_keys(k, dtype):
    """Values whose ascending keys are k (k avoids the keys of NaN and -0.0 for floats)."""
    w = dtype.itemsize
    u = np.dtype(f"u{w}")
    k = k.astype(u)
    sign = u.type(1) << u.type(8 * w - 1)
    if dtype.kind == "i":
        return (k ^ sign).view(dtype)
    if dtype.kind == "u":
        return k
    return np.where(k & sign, k ^ sign, ~k).astype(u).view(dtype)


def float_specials(dtype):
    if dtype == np.float32:
        bits = np.array([0x7FC00000, 0x7FC00001, 0x7F800001, 0x7FA00000, 0xFFC00000, 0xFF800001, 0xFFFFFFFF,   # NaNs
                         0x80000000, 0x00000000, 0x00000001, 0x007FFFFF, 0x80000001, 0x807FFFFF,             # +-0, subnormals
                         0x7F800000, 0xFF800000, 0x7F7FFFFF, 0xFF7FFFFF], np.uint32)                        # +-inf, +-max
        return bits.view(np.float32)
    bits = np.array([0x7FF8000000000000, 0x7FF8000000000001, 0x7FF0000000000001, 0x7FF4000000000000, 0xFFF8000000000000,
                     0xFFF0000000000001, 0xFFFFFFFFFFFFFFFF, 0x8000000000000000, 0, 1, 0x000FFFFFFFFFFFFF, 0x8000000000000001,
                     0x800FFFFFFFFFFFFF, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF], np.uint64)
    return bits.view(np.float64)


def random_values(rng, dtype, n):
    """Random keys over the whole type, with the float specials (every NaN class, +-0, subnormals, +-inf, +-max) or MIN / MAX
    sprinkled in, and runs of ties."""
    if dtype.kind == "f":
        u = np.dtype(f"u{dtype.itemsize}")
        v = rng.integers(0, np.iinfo(u).max, n, dtype=u, endpoint=True).view(dtype).copy()
        v[np.isnan(v)] = 1.5
        sp = float_specials(dtype)
    else:
        info = np.iinfo(dtype)
        v = rng.integers(info.min, info.max, n, dtype=dtype, endpoint=True)
        sp = np.array([info.min, info.max, info.min + 1, info.max - 1, 0], dtype)
    if n:
        at = rng.integers(0, n, max(1, n // 50))
        v[at] = sp[rng.integers(0, sp.size, at.size)]
        ties = rng.integers(0, n, max(1, n // 20))
        v[ties] = v[ties[0]]
    return v


def run_sort(rdf, ctx, oracle, chunks, v, valid, descending, what):
    """Sort one criterion on the device; indices and the taken column against the oracle, the pass count against the key set."""
    n = v.shape[0]
    col = rdf.Column.upload(chunks, ctx=ctx)
    ctx.synchronize()
    ctx.profile_read()
    ctx.profile_enable(True)
    try:
        idx = rdf.sort_indices([(col, descending)])
        recs = [r for r in ctx.profile_read() if r["kernel"] == "sort"]
    finally:
        ctx.profile_enable(False)
    got = idx.download()[0].value_slice()
    st, want = oracle.lexsort_indices([(chunks, descending)])
    assert st == oracle.OK
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, f"{what}: indices differ at {bad[:5]} of {n}: got {got[bad[:5]]}, want {want[bad[:5]]}"
    taken = col.take(idx).download()[0]
    _, wt = oracle.take(chunks, want)
    assert_same_array(taken, wt, what=f"{what}: take")
    assert len(recs) == 1 and recs[0]["rows"] == n, recs
    kb = 4 if v.dtype.itemsize <= 4 else 8
    passes, rest = divmod(recs[0]["bytes"] - 12 * n, (3 * kb + 8) * n)
    assert rest == 0 and passes == expected_passes(v, valid, descending), (what, recs[0]["bytes"], passes)
    col.free()
    idx.free()
    return passes


@gpu
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("tname", SORT_TYPES)
def test_sort_tile_and_grid_edges(rdf, ctx, oracle, tname, descending):
    """Lengths around one and two tiles, and around G tiles for G = SORT_CTAS_PER_SM x SMs: the first lengths at which a CTA
    scatters two tiles and carries its digit bases from one to the next.  A few sliced chunks with ~10 % nulls."""
    dt = np_dtype(tname)
    T, G = SORT_TILE, SORT_CTAS_PER_SM * sm_count(ctx)
    rng = np.random.default_rng(SORT_TYPES.index(tname) * 2 + descending)
    big = [G * T - 1, G * T, G * T + 1] if not descending else [G * T + 1]
    for n in [T - 1, T, T + 1, 2 * T + 1] + big:
        v = random_values(rng, dt, n)
        m = rng.random(n) >= 0.1
        run_sort(rdf, ctx, oracle, chunked(rdf, v, m, 5, rng), v, m, descending, f"{tname} n={n}")


def _digit_key_sets(rng, dt, n):
    """(name, values, mask) key sets for the digit skip, built in key space so every byte is where the test wants it."""
    w = dt.itemsize
    u64 = np.uint64
    base = sum(0x5A << (8 * d) for d in range(w))     # a key with no NaN / -0.0 value behind it in either width
    out = [("all equal", from_keys(np.full(n, base, u64), dt), np.ones(n, bool))]
    for d in range(w):
        top = d == w - 1
        hi = 254 if (top and dt.kind == "f") else 255
        digit = rng.integers(1 if (top and dt.kind == "f") else 0, hi, n, endpoint=True).astype(u64)
        k = (np.full(n, base, u64) & ~u64(0xff << (8 * d))) | (digit << u64(8 * d))
        out.append((f"byte {d} only", from_keys(k, dt), np.ones(n, bool)))
    for p in (1, 40, SORT_TILE + 5, n - 1):   # one row whose top byte differs: the OR / AND must see every row
        k = np.full(n, base, u64)
        k[p] = (k[p] & ~u64(0xff << (8 * w - 8))) | u64(0x10 << (8 * w - 8))
        out.append((f"outlier at {p}", from_keys(k, dt), np.ones(n, bool)))
    top_bit = np.full(n, base, u64) ^ np.where(rng.random(n) < 0.5, u64(1 << (8 * w - 1)), u64(0))
    out.append(("top bit only", from_keys(top_bit, dt), np.ones(n, bool)))
    if dt.kind != "u":   # the same magnitude with either sign
        mag = from_keys(np.full(n, base, u64), dt)
        out.append(("sign only", np.where(rng.random(n) < 0.5, mag, -mag).astype(dt), np.ones(n, bool)))
    # tile 1 (rows T..2T) shares the lowest digit, so in the first pass one peer group holds every lane of its warps
    k = rng.integers(0, 1 << 62, n, dtype=np.int64).astype(u64) & u64((1 << (8 * w)) - 1)
    k[SORT_TILE:2 * SORT_TILE] = (k[SORT_TILE:2 * SORT_TILE] & ~u64(0xff)) | u64(0x37)
    if dt.kind == "f":   # keep the top byte away from the NaN and -0.0 keys
        k = (k & ~u64(0xff << (8 * w - 8))) | (rng.integers(1, 254, n, endpoint=True).astype(u64) << u64(8 * w - 8))
    out.append(("one digit in a tile", from_keys(k, dt), np.ones(n, bool)))
    rnd = random_values(rng, dt, n)
    out.append(("nullable, no null", rnd, np.ones(n, bool)))
    out.append(("all null", rnd, np.zeros(n, bool)))
    return out


@gpu
@pytest.mark.parametrize("tname", SORT_TYPES)
def test_sort_digit_skip(rdf, ctx, oracle, tname):
    """Key sets on which the digit skip decides: no pass, exactly one pass for a byte, the top bit or the sign, a tile on one digit,
    a nullable column without a null and an all-null column.  The pass count comes from the sort's launch record."""
    dt = np_dtype(tname)
    rng = np.random.default_rng(40 + SORT_TYPES.index(tname))
    T = SORT_TILE
    for n in (3 * T + 1,):
        for name, v, m in _digit_key_sets(rng, dt, n):
            for descending in (False, True):
                mask = m if name in ("nullable, no null", "all null") else None
                chunks = chunked(rdf, v, mask, 3, rng)
                passes = run_sort(rdf, ctx, oracle, chunks, v, m, descending, f"{tname} {name} desc={descending}")
                if name in ("all equal", "all null"):
                    assert passes == 0
                elif name.startswith(("byte", "outlier")) or name == "top bit only":
                    assert passes == 1


# ---------------------------------------------------------------------------------------------------------
# the one-CTA scans of 1024 threads

SCAN_COUNTS = [SCAN_THREADS - 1, SCAN_THREADS, SCAN_THREADS + 1, 2 * SCAN_THREADS + 1]


@gpu
@pytest.mark.parametrize("count", SCAN_COUNTS)
def test_join_scan_block_counts(rdf, ctx, count):
    """count CTA totals in k_scan_one: probe rows (the left side of inner and left joins) filling count - 1 tiles and part
    of one more.  Partner counts run 0..3 from key to key, so output offsets grow unevenly."""
    rng = np.random.default_rng(count)
    n_probe = (count - 1) * JOIN_TILE + 1 + (count * 37) % (JOIN_TILE - 1)
    assert -(-n_probe // JOIN_TILE) == count
    card = 1000
    rkeys = np.repeat(np.arange(card, dtype=np.int32), np.arange(card) % 4)   # key k has k % 4 partners
    rkeys = rkeys[rng.permutation(rkeys.size)]
    lkeys = rng.integers(0, card + 50, n_probe).astype(np.int32)               # some keys have no partner at all
    lm = rng.random(n_probe) >= 0.05
    left, right = [(lkeys, lm)], [(rkeys, np.ones(rkeys.size, bool))]
    lc = rdf.Column.upload(chunked(rdf, lkeys, lm, 4, rng), ctx=ctx)
    rc = rdf.Column.upload(chunked(rdf, rkeys, None, 2, rng), ctx=ctx)
    for how in ("inner", "left"):
        li, ri = rdf.join_indices([lc], [rc], how)
        got = []
        for c in (li, ri):
            v, m = one(c)
            got.append(np.where(m, v.astype(np.int64), -1))
        wl, wr = jo.join_indices(left, right, how)
        assert got[0].shape == wl.shape, (how, got[0].shape, wl.shape)
        assert np.array_equal(got[0], wl) and np.array_equal(got[1], wr), how


@gpu
@pytest.mark.parametrize("count", SCAN_COUNTS)
def test_window_carry_tile_counts(rdf, ctx, count):
    """count scan tiles in k_window_carry.  Partitions start exactly on a tile boundary, one row before and one row after one, and
    one partition spans the tiles of several carry threads.  Running sum / min / max and first_value against the oracles."""
    rng = np.random.default_rng(100 + count)
    n = count * WIN_TILE - 7
    per = -(-count // SCAN_THREADS)
    starts = {0, 5 * WIN_TILE, 9 * WIN_TILE - 1, 13 * WIN_TILE + 1, (count // 2) * WIN_TILE}
    span_start = max(0, count - 1 - 3 * per - 2) * WIN_TILE + 100   # the last partition spans > 3 carry threads' tiles
    starts.add(span_start)
    starts = sorted(s for s in starts if s < n)
    head = np.zeros(n, bool)
    head[starts] = True
    part = (np.cumsum(head) - 1).astype(np.int32)          # partition keys ascending in row order: the sorted space is row order
    order = np.arange(n, dtype=np.int64)
    xi = rng.integers(-2 ** 40, 2 ** 40, n).astype(np.int64)
    xf = rng.integers(-2 ** 20, 2 ** 20, n).astype(np.float64)
    xm = rng.random(n) >= 0.1
    pc, oc = chunked(rdf, part, None, 3, rng, sliced=False), chunked(rdf, order, None, 3, rng, sliced=False)
    ic, fc = chunked(rdf, xi, xm, 3, rng), chunked(rdf, xf, xm, 3, rng)
    cp, co, ci, cf = (rdf.Column.upload(c, ctx=ctx) for c in (pc, oc, ic, fc))
    calls = [("sum", ci, "range"), ("min", ci, "range"), ("max", cf, "range")]
    got = rdf.window([cp], [(co, False)], calls + [("first_value", cf, "range", True)])
    want = W.window([pc], [(oc, False)], [(fn, {id(ci): ic, id(cf): fc}[id(c)], fr) for fn, c, fr in calls], n=n)
    want.append(WF.window([pc], [(oc, False)], [("first_value", fc, ("range", None, True))], n=n)[0])
    for g, w, call in zip(got, want, calls + [("first_value", cf)]):
        gv, gm = one(g)
        assert_bits(gv, gm, w["values"], w["valid"], f"{call[0]} over {count} tiles")


# ---------------------------------------------------------------------------------------------------------
# group-by fold paths

GROUP_DTYPES = ["int64", "int16", "float32", "float64"]
FILLER = {1: 1, 8: 16, 32: 100}   # filler group lengths whose average picks the lane count


def long_group_lengths(lanes):
    return [LANE_ROWS * lanes, LANE_ROWS * lanes + 1, BIG_GROUP, BIG_GROUP + 1, 2 * BIG_GROUP, 2 * BIG_GROUP + 1]


def _group_case(rng, lanes, dtype):
    """(keys, values, mask, cancel, glen, starts) in row order, and the per-group lengths / sorted-space starts in key order."""
    longs = long_group_lengths(lanes)
    f = FILLER[lanes]
    total_long = sum(longs)
    n_fill = {1: total_long // 2, 8: total_long // 16, 32: total_long // 100}[lanes]
    n_groups = n_fill + len(longs)
    glen = np.full(n_groups, f, np.int64)
    long_ids = [40 * j + 3 for j in range(len(longs))]   # a long group shares its 32-group bitmap word with short ones
    glen[long_ids] = longs
    n = int(glen.sum())
    assert lanes_for(n // n_groups) == lanes
    sstart = np.concatenate([[0], np.cumsum(glen)[:-1]])   # sorted space: groups by key, rows in row order
    gid = np.repeat(np.arange(n_groups), glen)
    within = np.arange(n) - sstart[gid]
    dt = np.dtype(dtype)
    if dt.kind == "f":
        lo, hi = -2.0 ** 20, 2.0 ** 20
        v = rng.integers(-2 ** 20 + 1, 2 ** 20, n).astype(dt)
    else:
        info = np.iinfo(dt)
        lo, hi = info.min, info.max
        v = rng.integers(info.min + 1, info.max, n, dtype=dt)
    m = rng.random(n) >= 0.1
    for j, (g, L) in enumerate(zip(long_ids, longs)):
        b = sstart[g]
        if L == BIG_GROUP + 1:   # all null
            m[b:b + L] = False
            continue
        if L == 2 * BIG_GROUP:         # the first row of the second segment and the last of the first
            at_min, at_max = BIG_GROUP, BIG_GROUP - 1
        elif L == 2 * BIG_GROUP + 1:   # the lone row of the third segment, the group's first row
            at_min, at_max = 2 * BIG_GROUP, 0
        else:                          # the group's first and last row
            at_min, at_max = 0, L - 1
        v[b + at_min], v[b + at_max] = lo, hi
        m[b + at_min] = m[b + at_max] = True
    # the cancelling column: small values, and in the long groups large +- pairs around them
    cancel = rng.uniform(-1, 1, n)
    in_long = np.isin(gid, long_ids) & (within % 2 == 0) & (within + 1 < glen[gid])
    big = rng.uniform(1e12, 1e13, int(in_long.sum()))
    idx = np.nonzero(in_long)[0]
    cancel[idx] += big
    cancel[idx + 1] -= big
    # row order: whole groups in a random order of their keys
    layout = rng.permutation(n_groups)
    lstart = np.empty(n_groups, np.int64)
    lstart[layout] = np.concatenate([[0], np.cumsum(glen[layout])[:-1]])
    pos = lstart[gid] + within
    keys, vals, mask, canc = (np.empty(n, np.int32), np.empty(n, dt), np.empty(n, bool), np.empty(n))
    keys[pos], vals[pos], mask[pos], canc[pos] = gid.astype(np.int32), v, m, cancel
    return keys, vals, mask, canc, (v, m, cancel, glen, sstart)


def _exact_variance(v, m, glen, sstart):
    """Per group: the sample variance of the valid values read as f64, exact (Fractions), and its condition max(1, |mean| / sigma);
    None for fewer than two values."""
    x = np.where(m, v.astype(np.float64), 0.0)
    ints = np.array([int(t) for t in x], dtype=object)   # every value here is an integer
    cnt = np.add.reduceat(m.astype(np.int64), sstart)
    s1 = np.add.reduceat(ints, sstart)
    s2 = np.add.reduceat(ints * ints, sstart)
    out = []
    for c, a, b in zip(cnt.tolist(), s1, s2):
        if c < 2:
            out.append(None)
            continue
        m2 = Fraction(c * b - a * a, c)
        var = m2 / (c - 1)
        mean = Fraction(a, c)
        sigma = math.sqrt(float(m2 / c))
        out.append((var, max(1.0, abs(float(mean)) / sigma) if sigma > 0 else 1.0))
    return out


@gpu
@pytest.mark.parametrize("dtype", GROUP_DTYPES)
@pytest.mark.parametrize("lanes", [1, 8, 32])
def test_group_fold_paths(rdf, ctx, lanes, dtype):
    """Groups of LANE_ROWS x LANES (+1) rows and of one and two BIG_GROUP segments (+1) among filler groups whose average length
    picks the lane count.  sum / count / min / max / first / last bit for bit (integers wrap), avg exact from the exact double sum,
    variance against Fractions."""
    rng = np.random.default_rng(lanes * 10 + GROUP_DTYPES.index(dtype))
    keys, vals, mask, canc, (sv, sm, scanc, glen, sstart) = _group_case(rng, lanes, dtype)
    kch = chunked(rdf, keys, None, 3, rng, sliced=False)
    vch = chunked(rdf, vals, mask, 3, rng)
    ck, cv = rdf.Column.upload(kch, ctx=ctx), rdf.Column.upload(vch, ctx=ctx)
    fns = ["sum", "count", "min", "max", "first", "last"]
    with_avg = dtype != "int64"   # an Int64 avg is a double sum of values up to 2^63: not exact
    gk, res = rdf.group_by([ck], [(cv, f) for f in fns] + ([(cv, "avg")] if with_avg else []) + [(cv, "variance")])
    okeys, ores = gbo.group_by([kch], [(vch, f) for f in fns])
    kv, km = one(gk[0])
    assert_bits(kv, km, okeys[0][0], okeys[0][1], "keys")
    assert np.array_equal(kv, np.arange(glen.size, dtype=np.int32))
    for fn, r, o in zip(fns, res, ores):
        gv, gm = one(r)
        assert_bits(gv, gm, o["values"], o["valid"], f"{fn} ({lanes} lanes, {dtype})")
    cnt = ores[1]["values"]
    if with_avg:
        s = np.add.reduceat(np.where(sm, sv, 0).astype(np.float64), sstart)   # exact: integers far below 2^53
        gv, gm = one(res[len(fns)])
        assert_bits(gv, gm, s / np.maximum(cnt, 1), cnt > 0, "avg")
    gv, gm = one(res[-1])
    want = _exact_variance(sv, sm, glen, sstart)
    assert np.array_equal(gm, np.array([w is not None for w in want])), "variance validity"
    for g in np.nonzero(gm)[0]:
        var, cond = want[g]
        assert abs(Fraction(float(gv[g])) - var) <= Fraction(2.0 ** -40 * cond) * var + Fraction(2.0 ** -1000), (g, gv[g], float(var))
    if dtype == "float64":   # the cancelling column, held to the stated bar 16 log2(n) eps sum|x| against math.fsum
        cc = rdf.Column.upload(chunked(rdf, canc, None, 3, rng), ctx=ctx)
        _, (rs,) = rdf.group_by([ck], [(cc, "sum")])
        gs, _ = one(rs)
        for g in range(glen.size):
            x = scanc[sstart[g]:sstart[g] + glen[g]]
            exact = math.fsum(x)
            if glen[g] == 1:
                assert gs[g] == x[0]
                continue
            bar = 16 * math.log2(glen[g]) * 2.0 ** -53 * float(np.abs(x).sum()) + abs(exact) * 2.0 ** -53
            assert abs(gs[g] - exact) <= bar, (g, glen[g], gs[g], exact, bar)


# ---------------------------------------------------------------------------------------------------------
# list find

LIST_FILLER = {1: 1, 8: 16, 32: 100}
NEEDLE = 7


def _list_case(rng, lanes, dtype):
    """One list chunk: filler lists whose average picks the lane count, lists on the long-path threshold, and long lists of
    LONG_LIST x k - 1, x k and x k + 1 elements whose first match sits on a segment's last element, the next segment's first
    element, twice (the earlier must win) or nowhere; a null element holding the needle ahead of each first match."""
    specials = [LANE_ROUNDS * lanes, LANE_ROUNDS * lanes + 1] + [LONG_LIST * k + d for k in (1, 2, 3) for d in (-1, 0, 1)]
    total_special = sum(specials)
    f = LIST_FILLER[lanes]
    n_fill = {1: total_special // 2, 8: total_special // 16, 32: total_special // 100}[lanes]
    lens = np.full(n_fill + len(specials), f, np.int64)
    where = rng.choice(lens.size, len(specials), replace=False)
    lens[where] = specials
    lvalid = rng.random(lens.size) >= 0.02
    lvalid[where] = True
    lens[~lvalid] = 0
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    n_elem = int(off[-1])
    assert lanes_for(n_elem // lens.size) == lanes
    vals = rng.integers(0, 20, n_elem).astype(dtype)
    vals[vals == NEEDLE] = NEEDLE + 1
    vm = rng.random(n_elem) >= 0.05
    fill = np.ones(lens.size, bool)
    fill[where] = False
    hits = np.nonzero(np.repeat(fill, lens) & (rng.random(n_elem) < 0.2))[0]
    vals[hits] = NEEDLE                                   # filler lists: matches anywhere, some of them null
    for j, (li, L) in enumerate(zip(where, specials)):
        b = int(off[li])
        vm[b:b + L] = True
        pattern = j % 4
        if pattern == 0:
            at = [min(LONG_LIST - 1, L - 1)]              # the last element of the first segment
        elif pattern == 1:
            at = [min(LONG_LIST, L - 1)]                  # the first element of the second segment
        elif pattern == 2:
            at = [min(LONG_LIST - 1, L - 2), L - 1]       # twice: the earlier wins
        else:
            at = []                                       # nowhere
        for a in at:
            vals[b + a] = NEEDLE
        if at and at[0] > 0:
            vals[b + at[0] - 1] = NEEDLE
            vm[b + at[0] - 1] = False                      # a null element holding the needle does not match
    return off, lvalid, vals, vm, where


@gpu
@pytest.mark.parametrize("dtype", ["int32", "float64"])
@pytest.mark.parametrize("lanes", [1, 8, 32])
def test_list_find_paths(rdf, ctx, lanes, dtype):
    rng = np.random.default_rng(lanes + (7 if dtype == "float64" else 0))
    off, lvalid, vals, vm, where = _list_case(rng, lanes, np.dtype(dtype))
    n_lists = lvalid.size
    child = rdf.PrimitiveArray.from_numpy(vals, vm)
    child.null_count = -1
    arr = rdf.ListArray(getattr(rdf, "I32" if dtype == "int32" else "F64"), off, np.packbits(lvalid, bitorder="little"), 0, n_lists,
                        int((~lvalid).sum()), child)
    col = rdf.ListColumn.upload([arr], ctx)
    py = vals.tolist()
    lists = [None if not lvalid[j] else [py[i] if vm[i] else None for i in range(off[j], off[j + 1])] for j in range(n_lists)]
    needle = np.dtype(dtype).type(NEEDLE)
    want_pos = np.array([lo.array_position(l, needle) for l in lists], np.int64)
    want_con = [lo.array_contains(l, needle) for l in lists]
    assert set(want_pos[where].tolist()) >= {0, LONG_LIST, LONG_LIST + 1}   # the planted patterns are there
    gp = col.array_position(needle).download()
    assert len(gp) == 1
    bad = np.nonzero(gp[0].value_slice().astype(np.int64) != want_pos)[0]
    assert bad.size == 0, (lanes, dtype, bad[:5], gp[0].value_slice()[bad[:5]], want_pos[bad[:5]])
    gc = col.array_contains(needle).download()[0]
    got_con = [bool(b) if ok else None for b, ok in zip(gc.value_bits()[:n_lists], gc.valid_mask())]
    assert got_con == want_con


# ---------------------------------------------------------------------------------------------------------
# select levels

@gpu
@pytest.mark.parametrize("dtype", ["int32", "int64", "float64"])
@pytest.mark.parametrize("n_prefixes", [SEL_SMEM_PREFIXES, SEL_SMEM_PREFIXES + 1])
def test_select_prefix_bins(rdf, ctx, n_prefixes, dtype):
    """Percentiles at n_prefixes ranks that lie in distinct high bytes: every level after the first histograms n_prefixes x 256
    bins, in shared memory up to SEL_SMEM_BINS and in global atomics one prefix beyond.  Ties and nulls included; every result
    against the exact order statistic."""
    dt = np.dtype(dtype)
    w = dt.itemsize
    rng = np.random.default_rng(n_prefixes * 3 + w)
    n_valid = 2 ** 17 + 1                      # (n - 1) * p is exact for p = r / 2^17
    buckets = np.arange(8, 248, 6)             # 40 high bytes, away from the NaN and -0.0 keys of a float
    hb = rng.choice(buckets, n_valid)
    low = rng.integers(0, 1 << 62, n_valid, dtype=np.int64).astype(np.uint64) & np.uint64((1 << (8 * w - 8)) - 1)
    low[rng.random(n_valid) < 0.3] = np.uint64(0x1234)                # ties
    k = (hb.astype(np.uint64) << np.uint64(8 * w - 8)) | low
    v = from_keys(k, dt)
    srt = np.sort(k)
    first = {}
    for i, b in enumerate((srt >> np.uint64(8 * w - 8)).tolist()):
        first.setdefault(b, []).append(i)
    chosen = sorted(rng.choice(sorted(first), n_prefixes, replace=False).tolist())
    ranks = [first[b][len(first[b]) // 2] for b in chosen]
    ps = [r / 2 ** 17 for r in ranks]
    n = n_valid + n_valid // 9
    vals = np.zeros(n, dt)
    mask = np.zeros(n, bool)
    at = np.sort(rng.choice(n, n_valid, replace=False))
    vals[at], mask[at] = v, True
    vals[~mask] = v[0]
    col = rdf.Column.upload(chunked(rdf, vals, mask, 3, rng), ctx=ctx)
    ctx.synchronize()
    ctx.profile_read()
    ctx.profile_enable(True)
    try:
        got = col.percentile(ps)
        recs = [r for r in ctx.profile_read() if r["kernel"] == "select"]
    finally:
        ctx.profile_enable(False)
    assert recs[0]["rows"] == n and len(recs) >= 3, recs   # level 0, a compaction, and a level over n_prefixes prefixes
    for p, g in zip(ps, got):
        want = do.percentile(v, p)
        assert np.float64(g).view(np.uint64) == np.float64(want).view(np.uint64), (p, g, want)
