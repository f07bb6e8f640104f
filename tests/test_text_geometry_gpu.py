"""The CSV and JSON readers and writers where their geometry changes, against the restatements (csv_oracle, json_oracle,
csv_write_oracle, json_write_oracle) bit for bit and byte for byte.

Readers: every (DFA state, byte class) pair on the first byte of a tokenizer thread (16 B), warp (512 B) and CTA (4096 B), and on the
CTA-state scan's per-thread run edges in files of 1023..3073 tiles; headers wider than one and three CTAs; the first of two
failures; RecordBatch sizes around the 32-row validity words and the 256-row parse tiles; the JSON key table at its 2^16 cap.
Writers: 256-row CTAs around the 24576-byte shared window and at every 16-byte alignment; every dtype at its longest text (the
table that sizes CSV blocks); blocks of a wide Float64 frame across the 8 MiB staging slots; JSON blocks cut at exactly 64 MiB,
windows at the 2^21-row and 2^23-element caps.  Each case asserts the shape it names (planted offsets and DFA states, CTA text
sizes, block and window rows from the launch records), so a case that stops reaching its edge fails.

The two cases marked "Large" write 134 and 220 MB of text and skip without 2 GB of free disk; the JSON cut cases write 64 MB."""
import os
import re
import shutil
from collections import OrderedDict

import numpy as np
import pytest

import csv_oracle as co
import csv_write_oracle as cwo
import json_oracle as jo
import json_write_oracle as jwo
import text_geometry_helpers as h
from helpers import pool_used

MiB = 1 << 20
BATCHES = [1, 31, 32, 33, 255, 256, 257, 511, 513]
CAP = 64 * MiB          # kCsvwText / kJsonwText
STAGE = 8 * MiB         # kStageBytes
STAGE_SLOTS = 6         # kStageSlots: kStageSlots - 1 in flight
JSONW_ROWS, JSONW_ELEMS = 1 << 21, 1 << 23

# the longest text of each dtype (I8 .. F64, Boolean): the most negative integers, the largest unsigned, the negative smallest
# subnormals (positional: 0.000...) and false
EXTREMES = [np.int8(-128), np.int16(-32768), np.int32(-2 ** 31), np.int64(-2 ** 63), np.uint8(255), np.uint16(65535), np.uint32(2 ** 32 - 1),
            np.uint64(2 ** 64 - 1), np.array([0x80000001], np.uint32).view(np.float32)[0], np.array([0x8000000000000001], np.uint64).view(np.float64)[0],
            False]


def max_field_lengths():
    return [len(cwo.format_values(dt, np.array([v]))[0]) for dt, v in enumerate(EXTREMES)]


def big_disk(tmp_path):
    if shutil.disk_usage(str(tmp_path)).free < 2 << 30:
        pytest.skip("needs 2 GB of free disk")


# ---- the constants every case assumes ---------------------------------------------------------------------------------

def test_constants_match_csrc():
    common, scan = h.source("common.cuh"), h.source("scan.cuh")
    kcsv, kjson, kcw, kjw, rt = (h.source(n) for n in ("k_csv.cu", "k_json.cu", "k_csv_write.cu", "k_json_write.cu", "runtime.cu"))
    env = {"kThreads": h.constant(common, "kThreads", {})}
    assert env["kThreads"] == 256
    env["kScanItems"] = h.constant(scan, "kScanItems", env)
    assert h.constant(scan, "kScanTile", env) == 2048
    env["kCsvBytes"] = h.constant(kcsv, "kCsvBytes", env)
    assert (env["kCsvBytes"], h.constant(kcsv, "kCsvTile", env), h.constant(kcsv, "kCsvRows", env)) == (h.THREAD, h.CTA, 256)
    assert h.THREAD * 32 == h.WARP
    # the CTA-state scan: one CTA of 1024 threads, each over ceil(tiles / 1024) consecutive tiles
    assert "__launch_bounds__(1024) k_csv_dfa_scan" in kcsv and "k_csv_dfa_scan<<<1, 1024" in kcsv and "(count + 1023) / 1024" in kcsv
    env["kJsonBytes"] = h.constant(kjson, "kJsonBytes", env)
    assert (env["kJsonBytes"], h.constant(kjson, "kJsonTile", env), h.constant(kjson, "kJsonRows", env)) == (h.THREAD, h.CTA, 256)
    assert h.constant(rt, "kJsonKeyCap", env) == 1 << 16
    assert 'if (n_cols > 65535) return fail(BDF_UNSUPPORTED, "more than 65535 columns")' in rt
    assert h.constant(kcw, "kCsvwWindow", env) == 24576 and h.constant(kjw, "kJsonwWindow", env) == 24576
    assert h.constant(rt, "kCsvwText", env) == CAP and h.constant(rt, "kCsvwMaxRows", env) == 1 << 21
    table = [int(x) for x in re.search(r"kCsvwMaxField\[11\] = \{([^}]*)\}", rt).group(1).split(",")]
    assert table == max_field_lengths() == [4, 6, 11, 20, 3, 5, 10, 20, 48, 327, 5]
    assert (h.constant(rt, "kJsonwText", env), h.constant(rt, "kJsonwMaxRows", env), h.constant(rt, "kJsonwElems", env)) == (CAP, JSONW_ROWS, JSONW_ELEMS)
    assert (h.constant(rt, "kStageBytes", env), h.constant(rt, "kStageSlots", env)) == (STAGE, STAGE_SLOTS)


# ---- CSV reader -------------------------------------------------------------------------------------------------------

def csv_check(rdf, ctx, tmp_path, data: bytes, batch_size=1024, name="t.csv", **kw):
    """The whole file against csv_oracle.read: schema, row count, field count, every non-Utf8 column, chunk lengths and bitmaps."""
    p = tmp_path / name
    p.write_bytes(data)
    ref = co.read(data, batch_size=batch_size, **kw)
    with rdf.CsvFile(str(p), batch_size=batch_size, ctx=ctx, **kw) as f:
        assert [n for n, _, _ in f.schema] == ref.names
        assert [dt if dt >= 0 else co.UTF8 for _, dt, _ in f.schema] == ref.dtypes
        if kw.get("schema") is None:
            assert [nl for _, _, nl in f.schema] == ref.nullable
        assert f.num_rows == ref.num_rows
        assert f.stats()["fields"] == len(co.records(data)) * len(ref.names)
        idx = [i for i, dt in enumerate(ref.dtypes) if dt != co.UTF8]
        cols = f.read(idx)
        n = ref.num_rows
        for i in idx:
            v, m, lens, hv = h.host(cols[ref.names[i]])
            rv, rm = ref.column(i)
            assert np.array_equal(m, rm), ref.names[i]
            assert np.array_equal(v[m], rv[rm].astype(v.dtype)), ref.names[i]
            assert lens == [min(batch_size, n - s) for s in range(0, n, batch_size)]
            assert hv == [bool((~rm[s:s + batch_size]).any()) for s in range(0, n, batch_size)]
    return ref


def csv_check_plan(rdf, ctx, tmp_path, plan: h.CsvPlan, name="big.csv"):
    """A file too large for csv_oracle.read: the planted records checked with the oracle (CsvPlan.check_plants), the columns
    against the ids and checks the plan wrote."""
    plan.check_plants()
    p = tmp_path / name
    p.write_bytes(bytes(plan.buf))
    with rdf.CsvFile(str(p), ctx=ctx) as f:
        assert [(n, dt) for n, dt, _ in f.schema] == [("id", co.I64), ("p", -1), ("check", co.I64)]
        assert f.num_rows == plan.rows and f.stats()["fields"] == plan.fields()
        cols = f.read(["id", "check"])
    for name, want in (("id", plan.ids), ("check", plan.checks)):
        v, m, _, _ = h.host(cols[name])
        wm = np.array([x is not None for x in want])
        wv = np.array([0 if x is None else x for x in want], np.int64)
        assert np.array_equal(m, wm), name
        bad = np.nonzero(v[m] != wv[wm])[0]
        assert bad.size == 0, (name, bad[:5])


@pytest.mark.gpu
def test_csv_every_state_and_class_at_thread_warp_and_cta_edges(rdf, ctx, tmp_path):
    rng = np.random.default_rng(1)
    plan = h.CsvPlan()
    for kind in ("thread", "warp", "cta"):
        for state, cls in h.PAIRS:
            e = plan.next_edge(kind, rng)
            plan.plant_at(e, state, cls)
            assert h.edge_kind(e) == kind
    plan.fill_to(len(plan.buf) + 100)
    plan.check_plants()
    assert len(plan.plants) == 3 * 27 and {(s, k) for _, s, k, *_ in plan.plants} == set(h.PAIRS)
    ref = csv_check(rdf, ctx, tmp_path, bytes(plan.buf))
    assert ref.num_rows == plan.rows and ref.dtypes == [co.I64, co.UTF8, co.I64]


@pytest.mark.gpu
@pytest.mark.parametrize("tiles", [1023, 1024, 1025, 2049, 3073])
def test_csv_pairs_on_the_state_scan_run_edges(rdf, ctx, tmp_path, tiles):
    """per = ceil(tiles / 1024) tiles per thread of k_csv_dfa_scan: the pairs planted on the first byte of run-edge tiles (k * per)
    and of tiles inside a run (k * per + 1, k * per + per - 1)."""
    per = -(-tiles // 1024)
    runs = (tiles - 2) // per
    ks = np.unique(np.linspace(1, runs - 1, 40).astype(int))
    targets = sorted({int(k) * per for k in ks} | ({int(k) * per + d for k in ks for d in {1, per - 1}} if per > 1 else set()))
    assert len(targets) >= 27 and max(targets) < tiles - 1
    plan = h.CsvPlan()
    for j, t in enumerate(targets):
        plan.plant_at(t * h.CTA, *h.PAIRS[j % len(h.PAIRS)])
    # end: a multiple of 4096 for 1023 / 3073 tiles, one byte before and after one for 1024 / 1025, a multiple of 16 for 2049
    end = {1023: tiles * h.CTA, 1024: tiles * h.CTA - 1, 1025: (tiles - 1) * h.CTA + 1, 2049: tiles * h.CTA - 48, 3073: tiles * h.CTA}[tiles]
    plan.fill_to(end)
    assert -(-len(plan.buf) // h.CTA) == tiles
    inside = [t for t in targets if t % per]
    assert per == 1 or len(inside) >= 27
    csv_check_plan(rdf, ctx, tmp_path, plan)


@pytest.mark.gpu
@pytest.mark.parametrize("terminated", [True, False])
def test_csv_file_lengths_around_16_and_4096(rdf, ctx, tmp_path, terminated):
    for end in (3 * h.CTA - 1, 3 * h.CTA, 3 * h.CTA + 1, 16 * 601 - 1, 16 * 601, 16 * 601 + 1):
        for last in (b"7,z,9", b'7,z,"9"'):   # the file ends in InField or QuoteInQuoted
            plan = h.CsvPlan()
            rng = np.random.default_rng(end)
            for state, cls in h.PAIRS[:10]:
                plan.plant_at(plan.next_edge("thread", rng), state, cls)
            tail = last + (b"\n" if terminated else b"")
            plan.fill_to(end - len(tail))
            plan.buf += tail
            assert len(plan.buf) == end
            ref = csv_check(rdf, ctx, tmp_path, bytes(plan.buf))
            assert ref.num_rows == plan.rows + 1


@pytest.mark.gpu
def test_csv_first_record_past_the_first_ctas(rdf, ctx, tmp_path):
    for width in (h.CTA + 200, 3 * h.CTA + 200):
        k = width // 6
        head = ",".join("c%04d" % j for j in range(k)).encode()
        rows = [",".join(str(-100000 - (r * 31 + j) % 99991) for j in range(k)).encode() for r in range(5)]
        data = head + b"\n" + b"\n".join(rows) + b"\n"
        assert data.index(b"\n") > width - 200
        csv_check(rdf, ctx, tmp_path, data, batch_size=2)
        body = b"\n".join(rows) + b"\n"
        assert body.index(b"\n") > h.CTA
        csv_check(rdf, ctx, tmp_path, body, has_header=False)
        csv_check(rdf, ctx, tmp_path, rows[0], has_header=False)            # one record, ended by the end of the file
        one = b"h" * width + b"\n" + b"".join(b"%d\n" % (r * 7 - 3) for r in range(40))
        csv_check(rdf, ctx, tmp_path, one, batch_size=7)                   # a single-field first record


@pytest.mark.gpu
def test_csv_first_of_two_unequal_records(rdf, ctx, tmp_path):
    """k_csv_check runs min(fields / 256, 16 * SMs) CTAs over the fields: the two bad records lie in later grid-stride rounds, the
    second in a lower CTA of its round than the first; the message names the first, its record, line and byte."""
    n = 900_000                                   # 1.8 M fields: four rounds of 132 * 16 CTAs
    for a, b in (((350_000, b"5\n"), (600_000, b"5,6,7\n")), ((350_000, b"5,6,7\n"), (600_000, b"5\n"))):
        recs = [b"1,2\n"] * n
        recs[a[0]], recs[b[0]] = a[1], b[1]
        data = b"a,b\n" + b"".join(recs)
        fields = 2 * (a[0] + 1)
        assert fields > 132 * 16 * 256 and (2 * (b[0] + 1)) % (132 * 16 * 256) // 256 < fields % (132 * 16 * 256) // 256
        with pytest.raises(co.CsvError) as ei:
            co.read(data)
        r = a[0] + 1
        assert f"(record {r})" in str(ei.value)
        byte = 4 + 4 * a[0]
        line = data[:byte].count(b"\n") + 1
        found = a[1].count(b",") + 1
        p = tmp_path / "u.csv"
        p.write_bytes(data)
        with pytest.raises(rdf.ComputeError, match=rf"CSV error: record {r} \(line: {line}, byte: {byte}\): found record with {found} fields, "
                                                     rf"but the previous record has 2 fields"):
            rdf.CsvFile(str(p), ctx=ctx)


def first_parse_error(recs, proj, batch, dtype):
    """The failure the reference reaches first: batch by batch, the projected columns in the projection's order, rows in order."""
    n = len(recs)
    for s in range(0, n, batch):
        for c in proj:
            for r in range(s, min(n, s + batch)):
                v = recs[r][c]
                if v != b"" and co.parse_int(v, dtype) is None:
                    return v.decode(), c, r
    return None


@pytest.mark.gpu
def test_csv_first_parse_error_by_batch_then_projected_column(rdf, ctx, tmp_path):
    rows, k, batch = 1000, 5, 100
    cells = [[str(r * k + c) for c in range(k)] for r in range(rows)]
    for r, c in [(250, 1), (305, 0), (390, 3), (310, 4), (360, 1), (520, 0), (610, 4), (611, 3)]:
        cells[r][c] = f"x{r}c{c}"
    data = ("a,b,c,d,e\n" + "".join(",".join(row) + "\n" for row in cells)).encode()
    recs = co.records(data)[1:]
    p = tmp_path / "e.csv"
    p.write_bytes(data)
    with rdf.CsvFile(str(p), schema=[co.I64] * k, batch_size=batch, ctx=ctx) as f:
        for proj in ([3, 0, 4], [4, 0], [1, 4], [0, 3], [2], [4, 3, 1, 0]):
            want = first_parse_error(recs, proj, batch, co.I64)
            if proj in ([3, 0, 4], [4, 0]):   # a key ordered by row before column would name another field
                by_row = min((r // batch, r, proj.index(c)) for r in range(rows) for c in proj if not cells[r][c].isdigit())
                assert (by_row[1], proj[by_row[2]]) != (want[2], want[1])
            if want is None:
                got = f.read(proj)
                assert len(got) == len(proj)
                continue
            v, c, r = want
            with pytest.raises(rdf.ParseError, match=rf"^Error while parsing value {v} for column {c} at line {r + 1}$"):
                f.read(proj)


def null_rows(n, batch):
    """Rows null on validity-word and parse-tile edges of every batch (of one row in seven for batches of one row), and all of
    batch 1."""
    r = np.arange(n)
    edge = np.isin(r % batch, [0, 30, 31, 32, 33, 63, 64, 254, 255, 256, 257, 511, 512, batch - 1]) if batch > 1 else r % 7 == 3
    return edge | (r // batch == 1)


@pytest.mark.gpu
@pytest.mark.parametrize("batch", BATCHES)
def test_csv_batch_sizes_with_nulls_on_word_and_tile_edges(rdf, ctx, tmp_path, batch):
    n = 3 * 513 + 50
    null = null_rows(n, batch)
    rng = np.random.default_rng(batch)
    lines = ["i,f,b"]
    for r in range(n):
        if null[r]:
            lines.append(",,")
        else:
            lines.append(f"{int(rng.integers(-2 ** 62, 2 ** 62))},{rng.normal() * 1e3:.6f},{'true' if r % 3 else 'false'}")
    ref = csv_check(rdf, ctx, tmp_path, ("\n".join(lines) + "\n").encode(), batch_size=batch)
    assert ref.dtypes == [co.I64, co.F64, co.BOOL] and all(ref.nullable)
    assert not ref.column(0)[1][batch:2 * batch].any()   # one batch all null


# ---- JSON reader ------------------------------------------------------------------------------------------------------

def json_check(rdf, ctx, tmp_path, data: bytes, batch_size=1024, schema=None, columns=None):
    p = tmp_path / "t.json"
    p.write_bytes(data)
    ref = jo.read(data, schema=schema, batch_size=batch_size)
    with rdf.JsonFile(str(p), schema=schema, batch_size=batch_size, ctx=ctx) as f:
        assert [n for n, _, _ in f.schema] == ref.names
        assert [dt for _, dt, _ in f.schema] == ref.dtypes
        assert [nl for _, _, nl in f.schema] == ref.nullable
        assert f.num_rows == ref.num_rows
        n = ref.num_rows
        want_lens = [min(batch_size, n - s) for s in range(0, n, batch_size)]
        idx = [i for i, dt in enumerate(ref.dtypes) if 0 <= dt <= co.BOOL] if columns is None else columns
        cols = f.read(idx)
        for i in idx:
            v, m, lens, hv = h.host(cols[ref.names[i]])
            rv, rm = ref.column(i)
            assert np.array_equal(m, rm), ref.names[i]
            assert np.array_equal(v, rv.astype(v.dtype)), ref.names[i]
            assert lens == want_lens
            assert hv == [bool((~rm[s:s + batch_size]).any()) for s in range(0, n, batch_size)]
        if columns is None:
            for i in [i for i, dt in enumerate(ref.dtypes) if dt >= jo.LIST_BASE]:
                rows, lens, hv = h.list_host(f.read_list(i))
                want = ref.list_column(i)
                assert rows == want, ref.names[i]
                assert lens == want_lens
                assert hv == [any(x is None for x in want[s:s + batch_size]) for s in range(0, n, batch_size)]
    return ref


class JsonPlan:
    """Records {"id":I,"p":"x...","v":V} of chosen lengths, so that a line end lands on an exact offset."""

    def __init__(self):
        self.buf = bytearray()
        self.n = 0

    def rec(self, k):
        self.n += 1
        return b'{"id":%d,"p":"%s","v":%d.5}' % (self.n, b"x" * k, self.n * 3)

    def fill_to(self, target, eol=b"\n"):
        while target - len(self.buf) > 300:
            self.buf += self.rec(100) + eol
        base = len(b'{"id":%d,"p":"","v":%d.5}' % (self.n + 1, (self.n + 1) * 3)) + len(eol)
        assert target - len(self.buf) >= base
        self.buf += self.rec(target - len(self.buf) - base) + eol


@pytest.mark.gpu
def test_json_line_ends_at_thread_warp_and_cta_edges(rdf, ctx, tmp_path):
    plan = JsonPlan()
    seen = []
    for unit in (h.THREAD, h.WARP, h.CTA):
        for what in ("lf first", "lf last", "crlf split", "blank line", "crlf blank"):
            kind = {h.THREAD: "thread", h.WARP: "warp", h.CTA: "cta"}[unit]
            e = (len(plan.buf) + 80 + unit - 1) // unit * unit
            while h.edge_kind(e) != kind:
                e += unit
            if what == "lf first":
                plan.fill_to(e + 1)                      # the record's '\n' is the unit's first byte
                at = e
            elif what == "lf last":
                plan.fill_to(e)                          # ... the previous unit's last byte
                at = e - 1
            elif what == "crlf split":
                plan.fill_to(e + 1, b"\r\n")
                at = e
                assert plan.buf[e - 1:e + 1] == b"\r\n"
            elif what == "blank line":
                plan.fill_to(e)
                plan.buf += b"\n"
                at = e
            else:
                plan.fill_to(e)
                plan.buf += b"\r\n"
                at = e + 1
            assert plan.buf[at] == 10 and h.edge_kind(e) == kind
            seen.append(what)
    plan.buf += plan.rec(3 * h.CTA + 100) + b"\n"            # a record longer than three CTAs
    plan.fill_to(len(plan.buf) + 500)
    json_check(rdf, ctx, tmp_path, bytes(plan.buf))
    assert len(seen) == 15
    for end in (3 * h.CTA - 1, 3 * h.CTA, 3 * h.CTA + 1):    # no final newline
        plan = JsonPlan()
        plan.fill_to(end - 200)
        plan.fill_to(end, b"")
        assert len(plan.buf) == end and plan.buf[-1:] == b"}"
        ref = json_check(rdf, ctx, tmp_path, bytes(plan.buf))
        assert ref.num_rows == plan.n


@pytest.mark.gpu
def test_json_duplicate_keys_across_tiles_and_escaped_spellings(rdf, ctx, tmp_path):
    pad = "x" * (h.CTA + 300)
    lines = ['{"x":1,"\\u0079":2,"p":"%s","x":3}' % pad,       # x twice, a tile apart: the last wins; y first seen escaped
             '{"y":4,"p":"%s","\\u0079":5,"x":6}' % pad,        # y twice in two spellings
             '{"z":7,"y":8}',
             '{"\\u0078":9,"p":"%s","z":10,"x":11,"z":12}' % pad]
    data = ("\n".join(lines) + "\n").encode()
    ref = json_check(rdf, ctx, tmp_path, data)
    assert ref.names == ["x", "y", "p", "z"]
    assert ref.column(0)[0].tolist() == [3, 6, 0, 11] and ref.column(1)[0].tolist() == [2, 5, 8, 0]
    assert data.index(b'"x":3') // h.CTA > data.index(b'"x":1') // h.CTA


def wide_record(keys):
    return ("{" + ",".join('"k%d":%d' % (j, j) for j in range(keys)) + "}\n").encode()


@pytest.mark.gpu
def test_json_key_table_at_its_cap(rdf, ctx, tmp_path):
    data = wide_record(1 << 16) + b'{"k0":5,"k65535":6}\n'
    json_check(rdf, ctx, tmp_path, data, schema=[("k0", co.I64), ("k65535", co.I64)])       # 2^16 raw keys: accepted
    p = tmp_path / "over.json"
    p.write_bytes(wide_record((1 << 16) + 1))
    ctx.synchronize()
    before = pool_used(ctx)
    with pytest.raises(rdf.UnsupportedType):
        rdf.JsonFile(str(p), schema=[("k0", co.I64)], ctx=ctx)
    ctx.synchronize()
    assert pool_used(ctx) == before
    ref = json_check(rdf, ctx, tmp_path, wide_record(65535), columns=[0, 7, 65534])          # 65535 inferred columns
    assert len(ref.names) == 65535
    p.write_bytes(wide_record(65536))
    with pytest.raises(rdf.UnsupportedType, match="more than 65535 columns"):
        rdf.JsonFile(str(p), ctx=ctx)
    ctx.synchronize()
    assert pool_used(ctx) == before


@pytest.mark.gpu
@pytest.mark.parametrize("batch", BATCHES)
def test_json_scalars_and_lists_at_batch_sizes(rdf, ctx, tmp_path, batch):
    n = 3 * 513 + 50
    null = null_rows(n, batch)
    loc = np.arange(n) % batch
    lines = []
    for r in range(n):
        i = "null" if null[r] else str(r * 1000003 - 7)
        b = "null" if null[r] else ("true" if r % 3 else "false")
        if null[r]:
            l = "null"
        elif loc[r] in (1, 34, 65, 258) or r % 11 == 0:
            l = "[]"
        elif loc[r] in (2, 35, 66, 259) or r % 13 == 0:
            l = str(r)                                   # a bare number: a list of one
        else:
            l = "[" + ",".join(str(r + j) for j in range(r % 4 + 1)) + "]"
        lines.append('{"i":%s,"l":%s,"b":%s}' % (i, l, b))
    ref = json_check(rdf, ctx, tmp_path, ("\n".join(lines) + "\n").encode(), batch_size=batch)
    assert ref.dtypes == [co.I64, jo.LIST_BASE + co.I64, co.BOOL]


# ---- CSV writer -------------------------------------------------------------------------------------------------------

def upload(rdf, ctx, dt, vals, valid=None, lens=None):
    lens = [len(vals)] if lens is None else lens
    chunks, s = [], 0
    for n in lens:
        v = vals[s:s + n]
        m = None if valid is None else valid[s:s + n]
        if dt == cwo.BOOL:
            a = rdf.BooleanArray.from_numpy(v, m)
        else:
            a = rdf.PrimitiveArray.from_numpy(v, m)
        if m is not None:
            a.null_count = int((~m).sum())
        chunks.append(a)
        s += n
    return rdf.Column.upload(chunks, ctx=ctx, dtype=dt)


def cta_frame(base, ncols):
    """Int64 columns whose 256-row CTAs of text are 24575, 24576 and 24577 bytes, then 17 CTAs at successive 16-byte offsets, then
    one all-null row (a CTA of fewer than 16 bytes)."""
    extras = h.cta_extras(base)
    cols = h.int_columns(extras + [0], ncols)
    valid = np.ones(len(extras) + 1, bool)
    valid[-1] = False
    return cols, valid


def assert_cta_shapes(text):
    sizes = h.cta_texts(text)
    assert sizes[:3] == [24575, 24576, 24577]
    starts = np.cumsum([0] + sizes)[:-1]
    assert sorted(int(s) % 16 for s in starts[3:19]) == list(range(16))
    assert sizes[-1] < 16 and starts[-1] % 16 != 0


@pytest.mark.gpu
def test_csv_write_ctas_around_the_shared_window(rdf, ctx, tmp_path):
    cols, valid = cta_frame(95, 5)
    host = [(f"c{j}", 3, v, valid) for j, v in enumerate(cols)]
    dev = OrderedDict((nm, upload(rdf, ctx, dt, v, m)) for nm, dt, v, m in host)
    p = tmp_path / "w.csv"
    recs = h.recorded(ctx, "csv_write", lambda: rdf.write_csv(str(p), dev))
    want = cwo.write(host)
    got = p.read_bytes()
    assert got == want
    head = len(cwo.header([c[0] for c in host]))
    assert_cta_shapes(want[head:])
    assert h.csv_write_blocks(recs) == [(len(valid), len(want) - head)]
    back = rdf.DeviceFrame.from_csv(str(p), schema=[co.I64] * 5, batch_size=777, ctx=ctx)   # round trip
    for nm, _, v, m in host:
        gv, gm, _, _ = h.host(back.column(nm))
        assert np.array_equal(gm, m) and np.array_equal(gv[gm], v[m]), nm


def csv_blocks_expected(max_row, rows):
    block = min(1 << 21, CAP // max_row)
    return block, [min(block, rows - s) for s in range(0, rows, block)]


@pytest.mark.gpu
def test_csv_write_every_dtype_at_its_longest_text(rdf, ctx, tmp_path):
    """Large (134 MB).  25 copies of the 11 dtypes, every value at its longest text (the negative subnormal extremes, Float64's also
    near 2^-1022), so each block's text lies within one row of block_rows * max_row: the kCsvwMaxField table is a true bound."""
    big_disk(tmp_path)
    lens = max_field_lengths()
    f64_long = [v for v in (EXTREMES[9], -2.2250738585072014e-308, -2.2250738585072009e-308, -4.4501477170144023e-308)
                if len(cwo.format_float(np.float64(v))) == lens[9]]
    assert len(f64_long) >= 2
    reps = 25
    names, dts, vals = [], [], []
    for r in range(reps):
        for dt, v in enumerate(EXTREMES):
            if dt == 9:
                v = np.float64(f64_long[r % len(f64_long)])
            names.append(f"d{dt}_{r}")
            dts.append(dt)
            vals.append(v)
    ncols = len(names)
    max_row = ncols + 2 + reps * sum(lens)
    block, want_rows = csv_blocks_expected(max_row, 2 * (CAP // max_row) + 7)
    n = sum(want_rows)
    assert len(want_rows) == 3 and 2 * block <= max_row   # within one row: 2 bytes of slack a row, block rows <= max_row / 2
    host1 = [(nm, dt, np.array([v] * 1, dtype=bool if dt == cwo.BOOL else type(v)), None) for nm, dt, v in zip(names, dts, vals)]
    one = cwo.write(host1)
    head = cwo.header(names).encode()
    row = one[len(head):]
    assert [len(x) for x in row[:-1].split(b",")] == [lens[dt] for dt in dts]
    assert len(row) == max_row - 2
    dev = OrderedDict()
    for nm, dt, v in zip(names, dts, vals):
        dev[nm] = upload(rdf, ctx, dt, np.full(n, v, dtype=bool if dt == cwo.BOOL else type(v)))
    p = tmp_path / "long.csv"
    recs = h.recorded(ctx, "csv_write", lambda: rdf.write_csv(str(p), dev))
    blocks = h.csv_write_blocks(recs)
    assert [r for r, _ in blocks] == want_rows
    for r, b in blocks:
        assert b == r * len(row)
    assert blocks[0][1] + max_row >= block * max_row and block * max_row <= CAP
    assert p.stat().st_size == len(head) + n * len(row)
    assert p.read_bytes() == head + row * n
    os.unlink(p)


@pytest.mark.gpu
def test_csv_write_wide_float64_blocks_across_staging_slots(rdf, ctx, tmp_path):
    """Large (220 MB).  2000 Float64 columns: max_row = 2002 + 2000 * 327, so 102 rows a block; values of ~270 characters put
    more than 40 MiB of text in a block, over five 8 MiB staging slots.  Chunk edges at a block edge and one row either side,
    with empty chunks at block edges."""
    big_disk(tmp_path)
    ncols, n = 2000, 400
    lens = max_field_lengths()
    block, want_rows = csv_blocks_expected(ncols + 2 + ncols * lens[9], n)
    assert block == 102 and want_rows == [102, 102, 102, 94]
    chunk_lens = [101, 1, 0, 1, 101, 0, 101, 95]
    assert sum(chunk_lens) == n and set(np.cumsum(chunk_lens).tolist()) >= {101, 102, 103, 204, 305}
    rng = np.random.default_rng(5)
    pool = (rng.uniform(1, 10, 4096) * 10.0 ** -rng.integers(230, 300, 4096)) * np.where(rng.random(4096) < 0.5, -1, 1)
    strs = [s.encode() for s in cwo.format_values(9, pool)]
    idx = rng.integers(0, 4096, (n, ncols))
    names = [f"f{j}" for j in range(ncols)]
    dev = OrderedDict((names[j], upload(rdf, ctx, 9, pool[idx[:, j]], None, chunk_lens)) for j in range(ncols))
    p = tmp_path / "wide.csv"
    recs = h.recorded(ctx, "csv_write", lambda: rdf.write_csv(str(p), dev))
    rows = [b",".join(strs[i] for i in idx[r]) + b"\n" for r in range(n)]
    head = cwo.header(names).encode()
    sample = [(names[j], 9, pool[idx[:3, j]], None) for j in range(ncols)]
    assert cwo.write(sample) == head + b"".join(rows[:3])
    blocks = h.csv_write_blocks(recs)
    assert [r for r, _ in blocks] == want_rows
    s = 0
    for r, b in blocks:
        assert b == sum(len(x) for x in rows[s:s + r])
        s += r
    assert all(b > (STAGE_SLOTS - 1) * STAGE for _, b in blocks[:3])
    assert p.read_bytes() == head + b"".join(rows)
    os.unlink(p)


# ---- JSON writer ------------------------------------------------------------------------------------------------------

def upload_list(rdf, ctx, dt, offsets, values, valid=None):
    v = None if valid is None else rdf.arrays.pack_validity(valid)
    nulls = 0 if valid is None else int((~valid).sum())
    arr = rdf.ListArray(dt, offsets.astype(np.int32), v, 0, len(offsets) - 1, nulls, rdf.PrimitiveArray.from_numpy(values))
    return rdf.ListColumn.upload([arr], ctx=ctx, dtype=dt)


@pytest.mark.gpu
def test_json_write_ctas_around_the_shared_window(rdf, ctx, tmp_path):
    cols, valid = cta_frame(94, 4)
    host = [{"name": "abcd"[j], "dtype": 3, "values": v, "valid": valid} for j, v in enumerate(cols)]
    dev = OrderedDict((c["name"], upload(rdf, ctx, 3, c["values"], c["valid"])) for c in host)
    p = tmp_path / "w.json"
    recs = h.recorded(ctx, "json_write", lambda: rdf.write_json(str(p), dev))
    want = jwo.write(host)
    assert p.read_bytes() == want
    assert_cta_shapes(want)
    assert h.json_write_blocks(recs) == [(len(valid), len(want))] and h.json_write_windows(recs) == [len(valid)]
    with rdf.JsonFile(str(p), schema=[(c, co.I64) for c in "abcd"], batch_size=300, ctx=ctx) as f:   # round trip
        back = f.read(list("abcd"))
    for c in host:
        gv, gm, _, _ = h.host(back[c["name"]])
        assert np.array_equal(gm, c["valid"]) and np.array_equal(gv[gm], c["values"][gm])


@pytest.mark.gpu
@pytest.mark.parametrize("longer", [False, True])
def test_json_write_block_cut_at_exactly_64_mib(rdf, ctx, tmp_path, longer):
    """64-byte rows: the first 2^20 fill a text buffer exactly and make one block; with one of them a byte longer the cut moves
    back one row."""
    n = (1 << 20) + 300
    name = "c" * 39
    v = 10 ** 18 + np.arange(n, dtype=np.int64)
    if longer:
        v[5] = -v[5]
    dev = OrderedDict([(name, upload(rdf, ctx, 3, v))])
    p = tmp_path / "cut.json"
    recs = h.recorded(ctx, "json_write", lambda: rdf.write_json(str(p), dev))
    pre = b'{"' + name.encode() + b'":'
    want = b"".join(pre + b"%d}\n" % x for x in v.tolist())
    assert len(pre + b"%d}\n" % v[0]) == 64
    assert jwo.write([{"name": name, "dtype": 3, "values": v[:64]}]) == want[:64 * 64 + (1 if longer else 0)]
    first = (1 << 20) - (1 if longer else 0)
    assert h.json_write_blocks(recs) == [(first, CAP - (63 if longer else 0)), (n - first, len(want) - CAP + (63 if longer else 0))]
    assert h.json_write_windows(recs) == [n]
    assert p.read_bytes() == want


@pytest.mark.gpu
@pytest.mark.parametrize("extra", [0, 1])
def test_json_write_window_row_cap(rdf, ctx, tmp_path, extra):
    n = JSONW_ROWS + extra
    v = (np.arange(n) % 10).astype(np.int8)
    dev = OrderedDict([("a", upload(rdf, ctx, 0, v))])
    p = tmp_path / "rows.json"
    recs = h.recorded(ctx, "json_write", lambda: rdf.write_json(str(p), dev))
    want = np.tile(np.frombuffer(b'{"a":0}\n', np.uint8), (n, 1))
    want[:, 5] += v.astype(np.uint8)
    want = want.tobytes()
    assert jwo.write([{"name": "a", "dtype": 0, "values": v[:20]}]) == want[:160]
    assert h.json_write_windows(recs) == [JSONW_ROWS] + [1] * extra
    assert [r for r, _ in h.json_write_blocks(recs)] == [JSONW_ROWS] + [1] * extra
    assert p.read_bytes() == want


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["exact-empty", "exact-null", "exact-long", "over-long"])
def test_json_write_window_element_cap(rdf, ctx, tmp_path, case):
    """2^20 lists of 8 elements hold exactly 2^23 elements (or 2^23 + 1, the first list one longer); then an empty, a null or a
    long list, then 10 more lists.  A window takes every row up to the cap: empty and null lists ride along."""
    m = 1 << 20
    kind = case.split("-")[1]
    lens = np.full(m + 11, 8, np.int64)
    if case.startswith("over"):
        lens[0] = 9
    lens[m] = {"empty": 0, "null": 0, "long": 5}[kind]
    valid = np.ones(m + 11, bool)
    valid[m] = kind != "null"
    offs = np.concatenate([[0], np.cumsum(lens)])
    row_of = np.repeat(np.arange(m + 11), lens)
    vals = ((row_of + np.arange(offs[-1]) - offs[:-1][row_of]) % 10).astype(np.int8)
    dev = OrderedDict([("l", upload_list(rdf, ctx, 0, offs, vals, None if valid.all() else valid))])
    p = tmp_path / "elems.json"
    recs = h.recorded(ctx, "json_write", lambda: rdf.write_json(str(p), dev))
    lines = []
    for r in range(m + 11):
        if not valid[r]:
            lines.append(b"{}\n")
        else:
            lines.append(b'{"l":[' + b",".join(b"%d" % x for x in vals[offs[r]:offs[r + 1]].tolist()) + b"]}\n")
    want = b"".join(lines)
    rows_py = [None if not valid[r] else vals[offs[r]:offs[r + 1]].tolist() for r in range(m - 5, m + 11)]
    assert jwo.write([{"name": "l", "dtype": 0, "lists": rows_py}]) == b"".join(lines[m - 5:])
    if case.startswith("exact"):
        assert offs[m] == JSONW_ELEMS
        first = m + (1 if kind != "long" else 0)
    else:
        assert offs[m - 1] < JSONW_ELEMS < offs[m]
        first = m - 1
    assert h.json_write_windows(recs) == [first, m + 11 - first]
    elem_recs = [r["rows"] for i, r in enumerate(recs) if r["dtype"] == h.U64 and i > 0 and recs[i - 1]["dtype"] == -1 and recs[i - 1]["bytes"] == 0
                 and i + 2 < len(recs) and recs[i + 1]["dtype"] == h.U32 and recs[i + 2]["dtype"] == h.U64]
    assert elem_recs == [int(offs[first]), int(offs[-1] - offs[first])]
    assert p.read_bytes() == want


@pytest.mark.gpu
def test_json_write_list_chunks_inside_a_block_and_round_trip(rdf, ctx, tmp_path):
    rng = np.random.default_rng(9)
    chunk_lens = [300, 0, 1, 255, 257, 0, 31, 33, 4000]
    n = sum(chunk_lens)
    rows = [None if rng.random() < 0.1 else [None if rng.random() < 0.1 else int(x) for x in rng.integers(-10 ** 9, 10 ** 9, rng.integers(0, 6))]
            for _ in range(n)]
    ids = np.arange(n, dtype=np.int64) * 7 - 3
    cols = [{"name": "l", "dtype": 3, "lists": rows}, {"name": "i", "dtype": 3, "values": ids}]
    chunks, s = [], 0
    for k in chunk_lens:
        chunks.append(rdf.ListArray.from_pylist(3, rows[s:s + k]))
        s += k
    dev = OrderedDict([("l", rdf.ListColumn.upload(chunks, ctx=ctx, dtype=3)), ("i", upload(rdf, ctx, 3, ids, None, chunk_lens))])
    p = tmp_path / "lc.json"
    recs = h.recorded(ctx, "json_write", lambda: rdf.write_json(str(p), dev))
    want = jwo.write(cols)
    assert p.read_bytes() == want
    assert h.json_write_blocks(recs) == [(n, len(want))]
    with rdf.JsonFile(str(p), schema=[("l", jo.LIST_BASE + co.I64), ("i", co.I64)], batch_size=257, ctx=ctx) as f:   # round trip
        got, _, _ = h.list_host(f.read_list("l"))
        gi, gm, _, _ = h.host(f.read(["i"])["i"])
    assert got == rows
    assert gm.all() and np.array_equal(gi, ids)
