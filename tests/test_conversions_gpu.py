"""The device's number conversions on the hard corpus of tests/conversion_reference.py: from_csv and from_json (scalars and
List<Float> cells) bit for bit against exact rounding, with as many fields sent to the host's exact fallback as the host build of
csv_parse.cuh sends there; the fallback's capacity at its edge in all three readers; and to_csv against numpy's shortest digits and
the host build of csv_format.cuh."""
import os
import re
from collections import OrderedDict

import numpy as np
import pytest

import conversion_reference as cr
import csv_oracle as co
import csv_write_oracle as wo
import json_oracle as jo
from helpers import pool_used
from test_conversions import SLOW, build_harness

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
RUNTIME = os.path.join(os.path.dirname(HERE), "rust-dataframe_b200", "csrc", "runtime.cu")
_JSON_NUMBER = re.compile(r"-?(0|[1-9][0-9]*)(\.[0-9]+)?([eE][+-]?[0-9]+)?")
PART_SLOW = 60_000   # exact-fallback fields per file, under the fallback's 65 536


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return build_harness(tmp_path_factory.mktemp("conversion_harness"))


@pytest.fixture(scope="module")
def corpus(harness):
    """The valid corpus strings with their exact bits and the host harness's slow flags, per width."""
    strings = [s for s in cr.parse_corpus() if cr.parse_bits(s, cr.F64) is not None]
    ref = {w: np.array([cr.parse_bits(s, cr.FMTS[w]) for s in strings], np.uint64) for w in (64, 32)}
    slow = {w: harness.parse_float(strings, w)[1] == SLOW for w in (64, 32)}
    return strings, ref, slow


def _parts(slow_per_row, limit=PART_SLOW):
    """[start, end) row ranges, in order, each with at most `limit` slow fields."""
    parts, s, acc = [], 0, 0
    for i, k in enumerate(slow_per_row.tolist()):
        if acc + k > limit:
            parts.append((s, i))
            s, acc = i, 0
        acc += k
    parts.append((s, len(slow_per_row)))
    return parts


def _bits(col):
    out = []
    for a in col.download():
        v = np.asarray(a.value_slice())
        out.append(v.view(np.uint64 if v.dtype == np.float64 else np.uint32))
        assert np.asarray(a.valid_mask(), dtype=bool).all()
    return np.concatenate(out)


def _list_bits(lc):
    rows, vals = [], []
    for ch in lc.download():
        v = np.asarray(ch.values.value_slice())
        vals.append(v.view(f"u{v.dtype.itemsize}"))
        rows.append(np.diff(np.asarray(ch.offsets[:ch.length + 1])))
    return np.concatenate(rows), np.concatenate(vals)


@pytest.mark.parametrize("quoted", [False, True])
@pytest.mark.parametrize("batch", [7, 1000, 4096])
def test_csv_corpus_both_widths(rdf, ctx, tmp_path, harness, corpus, batch, quoted):
    """Every corpus string as a Float64 and a Float32 field of one record; every field the host harness leaves undecided
    written quoted in the second copy.  The device's bits are the exact rounding and its exact-fallback count is the harness's."""
    strings, ref, slow = corpus
    per_row = slow[64].astype(int) + slow[32].astype(int)
    for s0, s1 in _parts(per_row):
        rows = []
        for i in range(s0, s1):
            s = strings[i]
            rows.append(",".join(f'"{s}"' if quoted and slow[w][i] else s for w in (64, 32)))
        p = tmp_path / "c.csv"
        p.write_bytes(("a,b\n" + "\n".join(rows) + "\n").encode())
        with rdf.CsvFile(str(p), schema=[co.F64, co.F32], batch_size=batch, ctx=ctx) as f:
            cols = f.read()
            exact = f.stats()["exact_fields"]
        assert np.array_equal(_bits(cols["a"]), ref[64][s0:s1])
        assert np.array_equal(_bits(cols["b"]), ref[32][s0:s1].astype(np.uint32))
        want = int(per_row[s0:s1].sum())
        print(f"CSV rows {s0}..{s1} batch {batch} quoted {quoted}: exact_fields {exact}, host harness {want}")
        assert exact == want


def _json_strings(corpus):
    strings, ref, slow = corpus
    keep = [i for i, s in enumerate(strings) if _JSON_NUMBER.fullmatch(s)]
    return keep


@pytest.mark.parametrize("batch", [7, 1000])
def test_json_scalars(rdf, ctx, tmp_path, corpus, batch):
    """The corpus strings that are JSON numbers, as a Float64 and a Float32 member of each record."""
    strings, ref, slow = corpus
    keep = np.array(_json_strings(corpus))
    assert len(keep) > 100_000
    per_row = slow[64][keep].astype(int) + slow[32][keep].astype(int)
    for s0, s1 in _parts(per_row):
        idx = keep[s0:s1]
        p = tmp_path / "s.json"
        p.write_bytes("".join('{"f": %s, "g": %s}\n' % (strings[i], strings[i]) for i in idx).encode())
        with rdf.JsonFile(str(p), schema=[("f", co.F64), ("g", co.F32)], batch_size=batch, ctx=ctx) as f:
            cols = f.read()
            exact = f.stats()["exact_fields"]
        assert np.array_equal(_bits(cols["f"]), ref[64][idx])
        assert np.array_equal(_bits(cols["g"]), ref[32][idx].astype(np.uint32))
        print(f"JSON scalars {s0}..{s1} batch {batch}: exact_fields {exact}, host harness {int(per_row[s0:s1].sum())}")
        assert exact == int(per_row[s0:s1].sum())


@pytest.mark.parametrize("width", [64, 32])
def test_json_lists(rdf, ctx, tmp_path, corpus, width):
    """The same numbers as elements of List<Float64> / List<Float32> cells of 0 to 6 elements, read in batches of 97 rows so that
    the exact fallback's patches land in many list chunks of the child column."""
    strings, ref, slow = corpus
    keep = np.array(_json_strings(corpus))
    rng = np.random.default_rng(width)
    dt = co.F64 if width == 64 else co.F32
    for s0, s1 in _parts(slow[width][keep].astype(int)):
        idx = keep[s0:s1]
        lens, lines, k = [], [], 0
        while k < len(idx):
            n = int(rng.integers(0, 7))
            lines.append('{"l": [%s]}\n' % ", ".join(strings[i] for i in idx[k:k + n]))
            lens.append(min(n, len(idx) - k))
            k += n
        p = tmp_path / "l.json"
        p.write_bytes("".join(lines).encode())
        with rdf.JsonFile(str(p), schema=[("l", jo.LIST_BASE + dt)], batch_size=97, ctx=ctx) as f:
            got_lens, vals = _list_bits(f.read_list("l"))
            exact = f.stats()["exact_fields"]
        assert got_lens.tolist() == lens
        assert np.array_equal(vals, ref[width][idx].astype(vals.dtype))
        want = int(slow[width][idx].sum())
        print(f"JSON List<F{width}> {s0}..{s1}: exact_fields {exact}, host harness {want}")
        assert exact == want


# ---- the exact fallback's capacity --------------------------------------------------------------------------------------------
def _capacities():
    """(minimum, divisor) of the fallback list in each reader, read from runtime.cu."""
    src = open(RUNTIME).read()
    found = re.findall(r"slow_cap = std::max<long long>\((\d+), (float_fields|total) / (\d+)\)", src)
    assert len(found) == 3, found
    return [(int(a), int(c)) for a, _, c in found]


def test_capacity_constants_match_csrc():
    assert _capacities() == [(65536, 64)] * 3


def _hard_strings(harness, n):
    """n distinct Float64 strings near 1.0 that must go to the exact fallback: the midpoint after 1 + k 2^-52 cut to 25 digits."""
    out = []
    for k in range(n):
        d, e = cr._dyadic_decimal(2 * ((1 << 52) + k) + 1, -53)
        out.append(d[0] + "." + d[1:25])
    _, st = harness.parse_float(out, 64)
    assert (st == SLOW).all() and len(set(out)) == n
    return out


@pytest.mark.parametrize("reader", ["csv", "json", "json_list"])
def test_fallback_capacity_edge(rdf, ctx, tmp_path, harness, reader):
    """Exactly `cap` fallback fields read correctly; one more is UnsupportedType with the documented message, and leaks nothing."""
    minimum, div = _capacities()[0]
    cap = minimum   # the files hold fewer than minimum * div floats, so the minimum is the capacity
    strings = _hard_strings(harness, cap + 1)
    ref = np.array([cr.parse_bits(s, cr.F64) for s in strings], np.uint64)

    def read(n):
        p = tmp_path / f"cap_{n}"
        if reader == "csv":
            p.write_bytes(("x\n" + "\n".join(strings[:n]) + "\n").encode())
            f = rdf.CsvFile(str(p), schema=[co.F64], ctx=ctx)
            return f, lambda: _bits(f.read()["x"])
        if reader == "json":
            p.write_bytes("".join('{"x": %s}\n' % s for s in strings[:n]).encode())
            f = rdf.JsonFile(str(p), schema=[("x", co.F64)], ctx=ctx)
            return f, lambda: _bits(f.read()["x"])
        p.write_bytes("".join('{"x": [%s]}\n' % ", ".join(strings[k:min(k + 4, n)]) for k in range(0, n, 4)).encode())
        f = rdf.JsonFile(str(p), schema=[("x", jo.LIST_BASE + co.F64)], ctx=ctx)
        return f, lambda: _list_bits(f.read_list("x"))[1]

    f, go = read(cap)
    with f:
        assert np.array_equal(go(), ref[:cap])
        assert f.stats()["exact_fields"] == cap
    f, go = read(cap + 1)
    with f:
        ctx.synchronize()
        before = pool_used(ctx)
        what = "fields" if reader == "csv" else "values"
        with pytest.raises(rdf.UnsupportedType, match=f"{cap + 1} float {what} need exact rounding, more than the {cap} one read resolves"):
            go()
        ctx.synchronize()
        assert pool_used(ctx) == before


# ---- the writer ---------------------------------------------------------------------------------------------------------------
def _column(rdf, ctx, vals, dt):
    return rdf.Column.upload([rdf.PrimitiveArray.from_numpy(vals)], ctx=ctx, dtype=dt)


@pytest.mark.parametrize("width", [64, 32])
def test_to_csv_format_corpus(rdf, ctx, tmp_path, harness, width):
    """to_csv of the format corpus, byte for byte against numpy's digits and the host build of the formatter; read back by
    from_csv to the same bits, every field decided on the device."""
    f = cr.FMTS[width]
    pats = cr.format_patterns(3, f)
    vals = pats.view(np.float64 if width == 64 else np.float32)
    dt = co.F64 if width == 64 else co.F32
    p = tmp_path / "w.csv"
    rdf.write_csv(str(p), OrderedDict([("x", _column(rdf, ctx, vals, dt))]))
    got = p.read_bytes()
    assert got == wo.write([("x", dt, vals, None)])
    assert got == b"x\n" + harness.format_lines(pats, width)
    with rdf.CsvFile(str(p), schema=[dt], batch_size=4096, ctx=ctx) as rf:
        back = _bits(rf.read()["x"])
        assert rf.stats()["exact_fields"] == 0
    assert np.array_equal(back, pats)


def test_to_csv_large_float32(rdf, ctx, tmp_path, harness):
    """Every 257th Float32 pattern (about 2^24) and the first and last 64 patterns of every exponent of both signs, NaNs left out:
    the device's file against the host formatter's text, and read back to the same bits."""
    strided = np.arange(0, 1 << 32, 257, dtype=np.uint64)
    j = np.concatenate([np.arange(64), np.arange((1 << 23) - 64, 1 << 23)]).astype(np.uint64)
    edges = ((np.arange(512, dtype=np.uint64) << np.uint64(23))[:, None] | j[None, :]).ravel()
    pats = np.concatenate([strided, edges])
    pats = pats[(pats & np.uint64(0x7FFFFFFF)) <= np.uint64(0x7F800000)].astype(np.uint32)
    p = tmp_path / "big.csv"
    rdf.write_csv(str(p), OrderedDict([("x", _column(rdf, ctx, pats.view(np.float32), co.F32))]))
    got = p.read_bytes()
    assert got == b"x\n" + harness.format_lines(pats.astype(np.uint64), 32)
    del got
    with rdf.CsvFile(str(p), schema=[co.F32], batch_size=1 << 20, ctx=ctx) as rf:
        back = _bits(rf.read()["x"])
        assert rf.stats()["exact_fields"] == 0
    assert np.array_equal(back, pats)
