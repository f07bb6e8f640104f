"""The Parquet reader and writer where their geometry changes, each file checked against pyarrow, which is independent of this library.

Reader (k_parquet.cu over parquet_decode.cuh): each data page is cut into tiles of TILE rows, one CTA each.  k_pq_levels ORs validity
bits into the output chunk (row r of a file -> chunk r / batch) with atomicOr, so a 32-row word can be shared by two pages, two tiles
or two output chunks; k_pq_values finds each valid row's value index from the valid counts of the page's earlier tiles and a binary
search of the run table, and BYTE_STREAM_SPLIT needs the page's whole count; k_pq_snappy copies overlapping snappy copies with one
warp.  The cases below put page lengths, output chunk boundaries, definition-level runs, dictionary id runs and bit widths, snappy
elements and BYTE_STREAM_SPLIT nulls on those edges.  Every file's page headers are read back and asserted to have the shape its
case names (tests/parquet_helpers.py chunk_pages); the fixtures that pyarrow cannot write are built by hand.  The device result must
equal pyarrow.parquet.read_table bit for bit: the same null slots, 0 in a null slot, the same chunk lengths and bitmap presence.

Writer (k_parquet_write.cu over parquet_encode.cuh, planned by runtime.cu's parquet_write): data pages of PAGE_ROWS rows, tiles of
WTILE rows that also end at source chunk edges, level bits and dictionary ids ORed into the page body a word at a time (an id at bit
offset sh of a word with sh + bw > 32 carries into the next word), a dictionary per chunk unless its entries exceed DICT_LIMIT
bytes, and snappy page bodies cut into fragments of FRAGMENT bytes.  Every written file is read back by pyarrow and by this library's
reader, equal to the source bit for bit, and its page headers and bodies are asserted to have the layout the case targets.

test_constants_match_csrc re-reads every constant from csrc/, so a retuned kernel fails here instead of testing the wrong edges.
"""
import os
import re

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import parquet_helpers as H

gpu = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "rust-dataframe_b200", "csrc")

# the constants; test_constants_match_csrc re-reads every one of them from the sources
THREADS = 256           # common.cuh kThreads
TILE = 2048             # parquet_decode.cuh pq::kTileRows: rows per CTA of k_pq_levels / k_pq_values
WTILE = 2048            # parquet_encode.cuh pq::kWTileRows: rows per CTA of k_pqw_count / k_pqw_encode
FRAGMENT = 65536        # parquet_encode.cuh pq::kFragment: bytes per independently compressed snappy fragment
PAGE_ROWS = 1 << 17     # runtime.cu kPqwPageRows: rows per written data page
DICT_LIMIT = 1 << 20    # runtime.cu kPqwDictLimit: bytes of dictionary entries a written chunk may keep


def id_bit_width(entries: int) -> int:
    """parquet_encode.cuh id_bit_width: max(1, ceil(log2 entries))."""
    return max(1, (entries - 1).bit_length())


def _read(*parts):
    with open(os.path.join(*parts)) as f:
        return f.read()


def test_constants_match_csrc():
    common, dec, enc = _read(CSRC, "common.cuh"), _read(CSRC, "parquet_decode.cuh"), _read(CSRC, "parquet_encode.cuh")
    rd, wr, runtime = _read(CSRC, "k_parquet.cu"), _read(CSRC, "k_parquet_write.cu"), _read(CSRC, "runtime.cu")
    header = _read(ROOT, "include", "b200df.h")

    def num(src, pat):
        m = re.search(pat, src)
        assert m, f"pattern {pat!r} not found"
        return int(m.group(1))

    assert num(common, r"constexpr int kThreads = (\d+);") == THREADS
    assert num(dec, r"constexpr int kTileRows = (\d+);") == TILE
    assert num(enc, r"constexpr int kWTileRows = (\d+);") == WTILE
    assert num(enc, r"constexpr uint32_t kFragment = (\d+);") == FRAGMENT
    assert 1 << num(runtime, r"static constexpr int64_t kPqwPageRows = \(int64_t\)1 << (\d+);") == PAGE_ROWS
    assert 1 << num(runtime, r"static constexpr int64_t kPqwDictLimit = \(int64_t\)1 << (\d+);") == DICT_LIMIT
    # the limit counts entries x physical bytes, and a chunk at exactly the limit keeps its dictionary
    assert re.search(r"if \(cnt == 0 \|\| cnt \* pc->width > kPqwDictLimit\) continue;", runtime)
    assert re.search(r"int bw = 1;\s+while \(bw < 32 && \(\(uint64_t\)1 << bw\) < n\) bw\+\+;", enc)
    assert [id_bit_width(n) for n in (1, 2, 3, 4, 5, 1 << 17, (1 << 17) + 1)] == [1, 1, 2, 2, 3, 17, 18]
    # the tiles: kThreads threads of 8 consecutive rows, in both directions; a page and a tile never cross a row group
    assert re.search(r"kPqRowsPerThread = pq::kTileRows / kThreads;", rd) and re.search(r"kRowsPerThread = pq::kWTileRows / kThreads;", wr)
    assert TILE == WTILE == THREADS * 8
    assert re.search(r"std::min\(\{r1, starts\[b \+ 1\], r \+ \(int64_t\)pq::kWTileRows\}\)", runtime)   # a written tile ends at a chunk edge
    # the documented rules these cases assert
    assert "2^17 rows per data page" in header and "max(1, ceil(log2 entries))" in header and "would exceed 1 MiB" in header
    assert "64 KiB" in header and "fragments" in header


# ----------------------------------------------------------------------------------------------------------------------------------
# reader fixtures: each builds its file(s) and asserts, from the page headers and bodies, the shape its case names.  The non-GPU test
# test_reader_fixture_shapes runs them all; the GPU tests read them.

PAGE_ROW_COUNTS = [1, 31, 32, 33, 2047, 2048, 2049, 4095, 4096, 4097, 6145]
TYPES = {"i32": pa.int32(), "i64": pa.int64(), "f64": pa.float64(), "b": pa.bool_()}


def _values(name, n, rng, dictionary):
    if name == "b":
        return rng.random(n) < 0.5
    if dictionary:
        v = rng.integers(-40, 40, n)
        return (v * 0.25) if name == "f64" else v.astype(np.int32 if name == "i32" else np.int64)
    if name == "f64":
        return rng.standard_normal(n) * 1e6
    t = np.int32 if name == "i32" else np.int64
    info = np.iinfo(t)
    return rng.integers(info.min, info.max, n, dtype=t, endpoint=True)


def _typed_table(n, rng, encodings=("plain", "dict", "bss"), valid_every=None):
    """Columns {type}_{encoding}_{o|r}: optional ones with about 10 % nulls (none at the multiples of valid_every: pyarrow cuts a page
    after a batch of rows only when the batch has a value), required ones without.  Returns the table and the use_dictionary /
    use_byte_stream_split lists."""
    cols, fields, dict_cols, bss_cols = [], [], [], []
    for t, pt in TYPES.items():
        for e in encodings:
            if e != "plain" and t == "b":
                continue
            for opt in (True, False):
                name = f"{t}_{e}_{'o' if opt else 'r'}"
                m = rng.random(n) < 0.1 if opt else None
                if opt and valid_every:
                    m[::valid_every] = False
                cols.append(pa.array(_values(t, n, rng, e == "dict"), pt, mask=m))
                fields.append(pa.field(name, pt, nullable=opt))
                (dict_cols if e == "dict" else bss_cols if e == "bss" else []).append(name)
    return pa.Table.from_arrays(cols, schema=pa.schema(fields)), dict_cols, bss_cols


def _expected_pages(rows, per_page):
    return [per_page] * (rows // per_page) + ([rows % per_page] if rows % per_page else [])


def _assert_encodings(path, t, dict_cols, bss_cols):
    for i, name in enumerate(t.column_names):
        encs = {H.page_info(h)[2] for h, _ in H.chunk_pages(path, i) if h[1] != 2}
        if name in dict_cols:
            assert encs <= {H.ENC_PLAIN_DICTIONARY, H.ENC_RLE_DICTIONARY} and encs, (name, encs)
        elif name in bss_cols:
            assert encs == {H.ENC_BSS}, (name, encs)
        elif name.startswith("b_"):
            assert encs <= {H.ENC_PLAIN, H.ENC_RLE} and encs, (name, encs)
        else:
            assert encs == {H.ENC_PLAIN}, (name, encs)


def page_rows_file(d, n, version):
    """Pages of n rows, n rows and 7 rows (n = 1: nine pages of one row): the later pages start at rows n and 2n, which for most n are
    not multiples of 32, so two pages OR into the same validity word (and for Boolean into the same value word)."""
    rng = np.random.default_rng(n * 2 + (version == "2.0"))
    rows = 2 * n + 7
    t, dict_cols, bss_cols = _typed_table(rows, rng, valid_every=n)
    p = str(d / f"rows{n}-v{version}.parquet")
    pq.write_table(t, p, write_batch_size=n, data_page_size=1, data_page_version=version, use_dictionary=dict_cols,
                   use_byte_stream_split=bss_cols, compression="snappy" if version == "1.0" else "none", dictionary_pagesize_limit=1 << 20)
    for i in range(t.num_columns):
        pages = H.chunk_pages(p, i)
        assert H.data_page_rows(pages) == _expected_pages(rows, n), (n, t.column_names[i])
        assert {H.page_info(h)[0] for h, _ in pages if h[1] != 2} == {"v1" if version == "1.0" else "v2"}
    _assert_encodings(p, t, dict_cols, bss_cols)
    return [p]


OUT_BATCHES = [1, 31, 33, 2047, 2049, 3000]
DIR_FILES = [(4097, 2047, 3000, "1.0"), (2050, 2049, None, "2.0"), (6145, 2049, 4100, "1.0")]   # rows, rows per page, per row group, version


def output_chunks_dir(d):
    """Three files in one directory, several row groups, pages of 2048 +- 1 rows: an output chunk boundary of any batch size above
    falls inside a tile, inside a validity word and inside a page, and the first output chunk of each file (out0) moves."""
    rng = np.random.default_rng(77)
    d = d / "dir"
    d.mkdir()
    paths = []
    for k, (rows, per_page, per_rg, version) in enumerate(DIR_FILES):
        t, dict_cols, bss_cols = _typed_table(rows, rng, encodings=("plain", "dict"), valid_every=per_page)
        p = str(d / f"part-{k}.parquet")
        pq.write_table(t, p, write_batch_size=per_page, data_page_size=1, data_page_version=version, use_dictionary=dict_cols,
                       row_group_size=per_rg or rows)
        md = pq.ParquetFile(p).metadata
        rg = [md.row_group(g).num_rows for g in range(md.num_row_groups)]
        assert rg == _expected_pages(rows, per_rg or rows)
        for g in range(len(rg)):
            assert H.data_page_rows(H.chunk_pages(p, 0, g)) == _expected_pages(rg[g], per_page)
        paths.append(p)
    return paths


def _level_stream(runs):
    """(levels, stream) of runs ("rle", level, count) and ("bp", levels): a bit-packed run whose last group of 8 may be partial (its
    padding is zero), only at the end of a page."""
    lv, out = [], bytearray()
    for r in runs:
        if r[0] == "rle":
            lv += [r[1]] * r[2]
            out += H.rle_levels([(r[1], r[2])])
        else:
            x = list(r[1])
            lv += x
            out += H.hybrid_encode(np.array(x), 1, [("bp", (len(x) + 7) // 8)])
    return np.array(lv, dtype=np.int64), bytes(out)


def level_pages(rng):
    """Pages of definition-level run shapes pyarrow does not emit, in one chunk (so the later pages start at rows that are not
    multiples of 32)."""
    bp = lambda n: ("bp", (rng.random(n) < 0.5).astype(int))
    return [
        # nulls covering tiles 0 and 1 whole, then a valid run from tile 3 to tile 5
        [("rle", 0, 2 * TILE), ("rle", 1, 2000), bp(48), ("rle", 1, 4500), bp(13)],
        # runs ending one row before a tile edge, one after, exactly at one, one before the next, and a one-row run exactly at it
        [("rle", 1, TILE - 1), ("rle", 0, 2), ("rle", 1, TILE - 1), ("rle", 0, TILE - 1), ("rle", 1, 1), ("rle", 0, 1), ("rle", 1, 2000)],
        # alternating single-row runs across a tile edge
        [("rle", k % 2 == 0, 1) for k in range(TILE + 52)],
        # a page of nulls only: its before / all counts are 0
        [("rle", 0, TILE + 52)],
        # one valid row, the page's last
        [("rle", 0, 2 * TILE), ("rle", 1, 1)],
        # one bit-packed run of 2051 levels: its last group of 8 holds 3
        [bp(TILE + 3)],
        # one row, null; one row, valid
        [("rle", 0, 1)],
        [("rle", 1, 1)],
        # no nulls
        [("rle", 1, 33)],
    ]


def levels_file(d):
    rng = np.random.default_rng(31)
    pages, want_v, want_m = [], [], []
    for runs in level_pages(rng):
        runs = [(r[0], int(r[1]), r[2]) if r[0] == "rle" else r for r in runs]
        lv, stream = _level_stream(runs)
        vals = rng.integers(-2 ** 63, 2 ** 63 - 1, int(lv.sum()), dtype=np.int64)
        body = H.struct_pack_u32(len(stream)) + stream + vals.tobytes()
        pages.append((len(lv), H.ENC_PLAIN, body, None))
        full = np.zeros(len(lv), dtype=np.int64)
        full[lv == 1] = vals
        want_v.append(full); want_m.append(lv == 1)
    p = str(d / "levels.parquet")
    H.hand_file(p, 2, pages)
    # the file holds the runs as built, and pyarrow reads the values and nulls the levels say
    got = H.chunk_pages(p)
    assert H.data_page_rows(got) == [pg[0] for pg in pages]
    for (h, body), runs in zip(got, level_pages(np.random.default_rng(31))):
        levels, _ = H.page_sections(h, body, True, False)
        kinds = [r[0] for r in H.hybrid_runs(levels, 1, H.page_info(h)[1])]
        assert kinds == [r[0] for r in runs]
    col = pq.read_table(p).column("x").combine_chunks()
    m = np.concatenate(want_m)
    assert np.array_equal(np.asarray(col.is_valid()), m)
    assert np.array_equal(np.asarray(col.fill_null(0)), np.where(m, np.concatenate(want_v), 0))
    return [p]


ID_KS = list(range(21))


def dict_width_file(d, k, plus):
    """A dictionary of exactly 2^k (+ 1) Int32 and Int64 entries, so the ids need every bit width from 1 to 21.  Rows: runs of 2047,
    2048 and 2049 equal ids (RLE runs across tile edges), every entry once in shuffled order (bit-packed runs), then short runs and
    single ids mixed, in the same first page.  i64n is i64 with nulls inside the runs, so value and row indices differ across tiles."""
    rng = np.random.default_rng(1000 + 2 * k + plus)
    m = (1 << k) + plus
    ids = [np.repeat(np.arange(3) % m, [TILE - 1, TILE, TILE + 1]), rng.permutation(m)]
    mix = []
    while sum(len(x) for x in mix) < 3000:
        mix.append(np.repeat(rng.integers(0, m), rng.choice([1, 3, 9, 40, 300])))
        mix.append(rng.integers(0, m, 21))
    ids = np.concatenate(ids + mix)
    n = len(ids)
    nulls = np.zeros(n, dtype=bool)
    nulls[: 3 * TILE][rng.random(3 * TILE) < 0.2] = True      # inside the long runs: every entry still occurs
    i32 = (np.arange(m, dtype=np.int64) * 1021 - (1 << 30)).astype(np.int32)
    i64 = np.arange(m, dtype=np.int64) * 1_000_003 - (1 << 40)
    t = pa.table({"i32": pa.array(i32[ids]), "i64": pa.array(i64[ids]), "i64n": pa.array(i64[ids], mask=nulls)})
    p = str(d / f"ids-{k}-{plus}.parquet")
    pq.write_table(t, p, compression="none", dictionary_pagesize_limit=1 << 30, data_page_size=1 << 22, row_group_size=n)
    bw = id_bit_width(m)
    for i in range(3):
        pages = H.chunk_pages(p, i)
        assert H.page_info(pages[0][0]) == ("dict", m, H.ENC_PLAIN)
        widths = []
        for h, body in pages[1:]:
            assert H.page_info(h)[2] in (H.ENC_PLAIN_DICTIONARY, H.ENC_RLE_DICTIONARY)
            widths.append(H.page_sections(h, body, True, False)[1][0])
        # pyarrow sizes each page's ids for the entries seen so far: the last page has the dictionary's width
        assert widths == sorted(widths) and widths[-1] == bw, (k, plus, widths)
        if i == 1:   # the first page: an RLE run crossing a tile edge, and bit-packed runs
            h, body = pages[1]
            vals = H.page_sections(h, body, True, False)[1]
            runs = H.hybrid_runs(vals[1:], vals[0], H.page_info(h)[1])
            at, crossing, packed = 0, False, False
            for r in runs:
                crossing |= r[0] == "rle" and r[1] >= TILE - 8 and at // TILE != (at + r[1] - 1) // TILE
                packed |= r[0] == "bp"
                at += r[1]
            assert crossing and (packed or m == 1), (k, plus)
    return [p]


def dict_fallback_file(d):
    """A dictionary chunk that falls back to PLAIN part-way: the first PLAIN page starts at a row inside a tile and a validity word."""
    rng = np.random.default_rng(5)
    n = 40000
    v = np.where(np.arange(n) < 10000, rng.integers(0, 50, n), np.arange(n) * 3)
    t = pa.table({"x": pa.array(v, mask=rng.random(n) < 0.1), "y": pa.array(v.astype(np.float64) * 0.5)})
    p = str(d / "fallback.parquet")
    pq.write_table(t, p, dictionary_pagesize_limit=1 << 16, write_batch_size=777, compression="snappy")
    for i in range(2):
        pages = [H.page_info(h) for h, _ in H.chunk_pages(p, i)]
        assert pages[0][0] == "dict"
        encs = [e for _, _, e in pages[1:]]
        first_plain = encs.index(H.ENC_PLAIN)
        assert first_plain > 0 and set(encs[:first_plain]) <= {H.ENC_PLAIN_DICTIONARY, H.ENC_RLE_DICTIONARY}
        assert set(encs[first_plain:]) == {H.ENC_PLAIN}
        row = sum(r for _, r, _ in pages[1:1 + first_plain])
        assert row % TILE and row % 32, row
    return [p]


SNAPPY_OFFSETS = list(range(1, 41)) + [63, 64, 65]
LITERAL_LENGTHS = [1, 2, 31, 32, 33, 59, 60, 61, 63, 64, 65, 255, 256, 257, 4095, 65536, 65537]


def _copy_tag(off, ln, j):
    """Copy tags in turn: the 1-byte offset form where it fits, else the 2- and 4-byte forms."""
    if 4 <= ln <= 11 and off < 2048 and j % 3 == 0:
        return 1
    return 4 if j % 3 == 1 else 2


def _rle_len(c):
    return len(H.rle_levels([(1, c)]))


def _snappy_page(rng, value_elements, total=None):
    """(rows, raw body, snappy stream) of an optional Int32 V1 page without nulls: the 4-byte level length and levels as the first
    literal, then value_elements, then a literal up to a whole value (or up to `total` decompressed bytes, the level runs sized to
    make that exact)."""
    vbytes = sum(len(e[1]) if e[0] == "lit" else e[2] for e in value_elements)
    if total is None:
        rows = vbytes // 4 + 1
        runs = [(1, rows)]
    else:
        found = None
        for rows in range((total - 6) // 4, (total - 6) // 4 - 16, -1):
            for a in (0, 1):
                for b in range(4):
                    r = rows - 64 * a - b
                    if found is None and r > 0 and 4 + _rle_len(r) + 3 * a + 2 * b + 4 * rows == total and 4 * rows > vbytes:
                        found = rows, [(1, r)] + [(1, 64)] * a + [(1, 1)] * b
        rows, runs = found
    levels = H.rle_levels(runs)
    pad = 4 * rows - vbytes
    els = [("lit", H.struct_pack_u32(len(levels)) + levels)] + value_elements + [("lit", rng.bytes(pad))]
    raw, stream = H.snappy_encode(els)
    assert total is None or len(raw) == total
    return rows, raw, stream


def snappy_file(d):
    """Hand-built snappy pages: copies at offsets 1..40, 63, 64, 65 with every length 1..64 in all three tag forms and a 64 KiB run of
    overlapping copies; literals of every length class around the warp's 32-byte step and the tag's extra length bytes; and pages whose
    decompressed size is 65 536 bytes and one byte either side."""
    rng = np.random.default_rng(9)
    copies = [("lit", rng.bytes(100))]
    j = 0
    for off in SNAPPY_OFFSETS:
        for ln in range(1, 65):
            copies.append(("copy", off, ln, _copy_tag(off, ln, j)))
            j += 1
        copies.append(("lit", rng.bytes(off % 7 + 1)))
    copies += [("copy", 1, 64, 2)] * (FRAGMENT // 64)
    lits = []
    for k, ln in enumerate(LITERAL_LENGTHS):
        lits += [("lit", rng.bytes(ln)), ("copy", 1 + k % 5, 9, 1)]
    sized = lambda: [("lit", rng.bytes(200))] + [("copy", off, 33, 2) for off in (3, 17, 64)] * 300
    pages = [_snappy_page(rng, copies), _snappy_page(rng, lits)] + [_snappy_page(rng, sized(), FRAGMENT + dt) for dt in (-1, 0, 1)]
    p = str(d / "snappy.parquet")
    H.hand_file(p, 1, [(rows, H.ENC_PLAIN, raw, stream) for rows, raw, stream in pages], codec=1)
    got = H.chunk_pages(p)
    assert [h[2] for h, _ in got][2:] == [FRAGMENT - 1, FRAGMENT, FRAGMENT + 1]
    seen_copies, seen_lits = set(), set()
    for (h, body), (rows, raw, stream) in zip(got, pages):
        assert body == stream and pa.decompress(body, h[2], codec="snappy").to_pybytes() == raw
        n, els = H.snappy_elements(body)
        assert n == len(raw) == h[2]
        seen_copies |= {(kind, off, ln) for kind, ln, off, _ in els if kind != "lit"}
        seen_lits |= {ln for kind, ln, _, _ in els if kind == "lit"}
    for off in SNAPPY_OFFSETS:
        assert {ln for kind, o, ln in seen_copies if o == off} == set(range(1, 65)), off
    assert {kind for kind, _, _ in seen_copies} == {"copy1", "copy2", "copy4"}
    assert set(LITERAL_LENGTHS) <= seen_lits
    want = np.concatenate([np.frombuffer(raw[4 + int.from_bytes(raw[:4], "little"):], dtype=np.int32) for _, raw, _ in pages])
    assert np.array_equal(pq.read_table(p).column("x").to_numpy(), want)
    return [p]


BSS_ROWS = [TILE + 1, TILE + 33, 2 * TILE + 1, 2 * TILE + 33]


def bss_file(d, n, where, version):
    """BYTE_STREAM_SPLIT pages of n rows (two of them) whose nulls are only in the page's first tile, or only in its last: the page's
    count of encoded values differs from its rows, and only some tiles know.  Every page has a null at the tile's last row and
    random ones in the rest of the tile."""
    rng = np.random.default_rng(n + (where == "last"))
    r = np.arange(2 * n) % n
    lo, hi = (0, TILE) if where == "first" else ((n - 1) // TILE * TILE, n)
    in_tile = (r >= lo) & (r < hi)
    m = (in_tile & (rng.random(2 * n) < 0.3)) | (r == hi - 1)
    t = pa.table({"f64": pa.array(rng.standard_normal(2 * n), mask=m), "f32": pa.array(rng.standard_normal(2 * n).astype(np.float32), mask=m),
                  "i32": pa.array(rng.integers(-2 ** 31, 2 ** 31, 2 * n).astype(np.int32), mask=m),
                  "i64": pa.array(rng.integers(-2 ** 63, 2 ** 63 - 1, 2 * n, dtype=np.int64), mask=m)})
    p = str(d / f"bss-{n}-{where}-{version}.parquet")
    pq.write_table(t, p, use_dictionary=False, use_byte_stream_split=True, write_batch_size=n, data_page_size=1, data_page_version=version,
                   compression="snappy" if version == "1.0" else "none")
    for i in range(4):
        pages = H.chunk_pages(p, i)
        assert H.data_page_rows(pages) == [n, n] and {H.page_info(h)[2] for h, _ in pages} == {H.ENC_BSS}
        for h, body in pages:   # each page has nulls, all of them inside the named tile
            levels, _ = H.page_sections(h, body, True, version == "1.0")
            null_rows = np.flatnonzero(H.hybrid_decode(levels, 1, n) == 0)
            assert len(null_rows) and lo <= null_rows.min() and null_rows.max() < hi, (n, where, null_rows)
            if version == "2.0":
                assert h[8][2] == len(null_rows)
    return [p]


READER_FIXTURES = (
    [(f"rows{n}-v{v}", lambda d, n=n, v=v: page_rows_file(d, n, v)) for n in PAGE_ROW_COUNTS for v in ("1.0", "2.0")]
    + [("dir", output_chunks_dir), ("levels", levels_file), ("fallback", dict_fallback_file), ("snappy", snappy_file)]
    + [(f"ids-{k}-{p}", lambda d, k=k, p=p: dict_width_file(d, k, p)) for k in (0, 1, 2, 3, 7, 8, 16) for p in (0, 1)]
    + [(f"bss-{n}-{w}-{v}", lambda d, n=n, w=w, v=v: bss_file(d, n, w, v)) for n in BSS_ROWS for w in ("first", "last") for v in ("1.0", "2.0")]
)


@pytest.mark.parametrize("make", [f for _, f in READER_FIXTURES], ids=[i for i, _ in READER_FIXTURES])
def test_reader_fixture_shapes(tmp_path, make):
    """Every reader fixture has the page rows, encodings, run kinds, bit widths and snappy elements its case claims (no GPU)."""
    make(tmp_path)


# ----------------------------------------------------------------------------------------------------------------------------------
# reader cases (GPU)

@gpu
@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("n", PAGE_ROW_COUNTS)
def test_page_rows_on_tile_edges(rdf, ctx, tmp_path, n, version):
    (p,) = page_rows_file(tmp_path, n, version)
    H.check_read(rdf, ctx, [p], p, 1 << 20)
    H.check_read(rdf, ctx, [p], p, 1000)


@gpu
@pytest.mark.parametrize("batch", OUT_BATCHES)
def test_output_chunks_across_pages_and_tiles(rdf, ctx, tmp_path, batch):
    paths = output_chunks_dir(tmp_path)
    names = ["i32_plain_o", "i64_dict_o", "f64_plain_r", "b_plain_o"] if batch < 64 else None   # one output chunk per row or two
    H.check_read(rdf, ctx, paths, os.path.dirname(paths[0]), batch, names)


@gpu
@pytest.mark.parametrize("batch", [1 << 20, 1000, 33])
def test_definition_level_runs(rdf, ctx, tmp_path, batch):
    (p,) = levels_file(tmp_path)
    H.check_read(rdf, ctx, [p], p, batch)


@gpu
@pytest.mark.parametrize("plus", [0, 1])
@pytest.mark.parametrize("k", ID_KS)
def test_every_dictionary_id_bit_width(rdf, ctx, tmp_path, k, plus):
    (p,) = dict_width_file(tmp_path, k, plus)
    H.check_read(rdf, ctx, [p], p, 1 << 20)


@gpu
def test_dictionary_falls_back_inside_a_tile(rdf, ctx, tmp_path):
    (p,) = dict_fallback_file(tmp_path)
    H.check_read(rdf, ctx, [p], p, 1 << 20)
    H.check_read(rdf, ctx, [p], p, 1000)


@gpu
def test_snappy_copies_on_one_warp(rdf, ctx, tmp_path):
    (p,) = snappy_file(tmp_path)
    H.check_read(rdf, ctx, [p], p, 1 << 20)


@gpu
@pytest.mark.parametrize("version", ["1.0", "2.0"])
@pytest.mark.parametrize("where", ["first", "last"])
@pytest.mark.parametrize("n", BSS_ROWS)
def test_byte_stream_split_nulls_across_tiles(rdf, ctx, tmp_path, n, where, version):
    (p,) = bss_file(tmp_path, n, where, version)
    H.check_read(rdf, ctx, [p], p, 1 << 20)


# ----------------------------------------------------------------------------------------------------------------------------------
# writer cases (GPU): the device writes, pyarrow and this library's reader read back

def _upload(rdf, ctx, arr: pa.Array, cuts):
    """A device column of arr cut into chunks of the given lengths."""
    chunks, s = [], 0
    for ln in cuts:
        a = arr.slice(s, ln)
        s += ln
        if pa.types.is_boolean(a.type):
            vbuf, dbuf = a.buffers()
            chunks.append(rdf.BooleanArray(np.frombuffer(dbuf, dtype=np.uint8), np.frombuffer(vbuf, dtype=np.uint8) if vbuf is not None else None,
                                           a.offset, len(a), a.null_count if vbuf is not None else 0, keepalive=a))
        else:
            chunks.append(rdf.PrimitiveArray.from_arrow(a))
    assert s == len(arr)
    return rdf.Column.upload(chunks, ctx=ctx, dtype=10 if pa.types.is_boolean(arr.type) else None)


def _odd_cuts(n):
    cuts, s, k = [], 0, 0
    while s < n:
        ln = min([7, 1999, 1, 3333, 2049][k % 5], n - s)
        cuts.append(ln)
        s += ln
        k += 1
    return cuts


def _write_and_read_back(rdf, ctx, path, arrays, cuts, **opt):
    cols = {k: _upload(rdf, ctx, a, cuts) for k, a in arrays.items()}
    rdf.write_parquet(path, cols, **opt)
    got = pq.read_table(path)
    assert got.column_names == list(arrays)
    with rdf.ParquetFile(path, batch_size=1 << 20) as f:
        dev = f.read(list(arrays), ctx=ctx)
    for name, a in arrays.items():
        gv, gm = H.expected_bits(got.column(name))
        ev, em = H.expected_bits(a)
        assert np.array_equal(gm, em) and np.array_equal(gv, ev), name
        dv, dm, _, _ = H.device_bits(dev[name])
        assert np.array_equal(dm, em) and np.array_equal(np.where(dm, dv, 0), ev), name
    return pq.ParquetFile(path).metadata


def _page_starts(rg_rows):
    return [s for s in range(0, rg_rows, PAGE_ROWS)]


WRITE_EDGES = ([(f"one-{n}", n, "one", 0) for n in (PAGE_ROWS - 1, PAGE_ROWS, PAGE_ROWS + 1, 2 * PAGE_ROWS + 2049)]
               + [("rg1", 100, "odd", 1), ("rg31", 5000, "odd", 31), ("rg2047", 20000, "odd", 2047), ("rg2049", 20000, "odd", 2049),
                  ("rg-page+1", 2 * PAGE_ROWS + 2049, "odd", PAGE_ROWS + 1)])


@gpu
@pytest.mark.parametrize("n,layout,rg", [w[1:] for w in WRITE_EDGES], ids=[w[0] for w in WRITE_EDGES])
def test_writer_page_and_tile_edges(rdf, ctx, tmp_path, n, layout, rg):
    """Data pages of PAGE_ROWS rows and their remainders, row groups cut across odd chunks; columns without nulls, with only nulls,
    and with one null at each page's first, last and 32 k-th row (one RLE level run, or one bit-packed run).  Each chunk keeps a
    dictionary exactly when its distinct values fit DICT_LIMIT bytes."""
    rng = np.random.default_rng(n + rg)
    rg_sizes = _expected_pages(n, rg or n)
    rows_in_page = np.concatenate([np.concatenate([np.arange(min(PAGE_ROWS, g - s)) for s in _page_starts(g)]) for g in rg_sizes])
    page_len = np.concatenate([np.concatenate([np.full(min(PAGE_ROWS, g - s), min(PAGE_ROWS, g - s)) for s in _page_starts(g)])
                               for g in rg_sizes])
    first, last = rows_in_page == 0, rows_in_page == page_len - 1
    k32 = rows_in_page == np.minimum(32 * 37, (page_len - 1) // 32 * 32)
    arrays = {
        "none": pa.array(rng.integers(0, 1000, n)),
        "all": pa.array(np.zeros(n, dtype=np.float64), mask=np.ones(n, dtype=bool)),
        "first": pa.array(rng.integers(-100, 100, n).astype(np.int32), mask=first),
        "last": pa.array(rng.standard_normal(n), mask=last),
        "k32": pa.array(rng.integers(0, 2 ** 40, n), mask=k32),
        "b": pa.array(rng.random(n) < 0.5, mask=first | k32),
        # every value distinct: a dictionary for a row group of at most 262 144 valid rows, PLAIN above
        "plain": pa.array((rng.permutation(n) * 0.5 - 1000).astype(np.float32), mask=last),
    }
    width = {"none": 8, "all": 8, "first": 4, "last": 8, "k32": 8, "b": None, "plain": 4}
    md = _write_and_read_back(rdf, ctx, str(tmp_path / "w.parquet"), arrays, [n] if layout == "one" else _odd_cuts(n), row_group_rows=rg)
    p = str(tmp_path / "w.parquet")
    assert [md.row_group(g).num_rows for g in range(md.num_row_groups)] == rg_sizes
    for g in sorted({0, len(rg_sizes) // 2, len(rg_sizes) - 1}):
        want_pages = _expected_pages(rg_sizes[g], PAGE_ROWS)
        g0 = sum(rg_sizes[:g])
        for i, name in enumerate(arrays):
            pages = H.chunk_pages(p, i, g)
            assert H.data_page_rows(pages) == want_pages, (name, g)
            valid = np.asarray(arrays[name].slice(g0, rg_sizes[g]).drop_null())
            entries = len(np.unique(valid.view(f"u{valid.dtype.itemsize}"))) if width[name] else 0
            if width[name] and 0 < entries * width[name] <= DICT_LIMIT:   # Boolean: never a dictionary
                assert H.page_info(pages[0][0]) == ("dict", entries, H.ENC_PLAIN_DICTIONARY), (name, g)
                assert {H.page_info(h)[2] for h, _ in pages[1:]} == {H.ENC_PLAIN_DICTIONARY}, (name, g)
            else:
                assert {H.page_info(h)[:3:2] for h, _ in pages} == {("v1", H.ENC_PLAIN)}, (name, g, entries)
            if name == "plain" and rg_sizes[g] > 2 * PAGE_ROWS:
                assert entries * 4 > DICT_LIMIT   # the PLAIN side of the limit is reached
            for h, body in pages:
                if h[1] == 2:
                    continue
                kind, rows, _ = H.page_info(h)
                levels, _ = H.page_sections(h, body, True, False)
                runs = H.hybrid_runs(levels, 1, rows)
                if name in ("none", "all"):
                    assert runs == [("rle", rows, int(name == "none"))], (name, g)
                else:
                    assert len(runs) == 1 and runs[0][0] == "bp" or rows == 1, (name, g, runs)


def _valid_rows(levels, rows):
    return int(H.hybrid_decode(levels, 1, rows).sum())


def _ids_straddle(body, valid, bw):
    """Whether any id of a data page's one bit-packed run has sh + bw > 32 in its 32-bit word of the page body."""
    lev_len = int.from_bytes(body[:4], "little")
    at = 4 + lev_len
    assert body[at] == bw
    _, at = H._varint(body, at + 1)
    bits = at * 8 + np.arange(valid, dtype=np.int64) * bw
    return bool(((bits % 32) + bw > 32).any())


@gpu
@pytest.mark.parametrize("plus", [0, 1])
@pytest.mark.parametrize("k", ID_KS)
def test_writer_every_id_bit_width(rdf, ctx, tmp_path, k, plus):
    """Chunks of exactly 2^k (+ 1) distinct Int32 and Int64 values: the bit width byte is max(1, ceil(log2 entries)) while the
    dictionary fits DICT_LIMIT bytes, else the chunk is PLAIN.  Odd source chunks start tiles at odd rows of a page, and a nullable
    column moves the ids' start in the body, so ids straddle 32-bit words (sh + bw > 32) at every width where that can happen."""
    rng = np.random.default_rng(2000 + 2 * k + plus)
    m = (1 << k) + plus
    n = m + 3 * TILE
    # widths 1, 2, 4 and 8 never straddle; 16 straddles when the ids start at an odd byte: choose n so the mixed column's first page does
    for extra in range(64):
        rows = min(n + extra, PAGE_ROWS)
        at = 4 + len(H._varint_encode(((rows + 7) // 8) << 1 | 1, None)) + (rows + 7) // 8 + 1
        at += len(H._varint_encode(((rows - 1 + 7) // 8) << 1 | 1, None))
        if at % 2:
            n += extra
            break
    ids = np.concatenate([rng.permutation(m), rng.integers(0, m, n - m)])
    nulls = np.zeros(n, dtype=bool)
    nulls[m + 5] = True   # a repeat: every entry still occurs
    i32 = (np.arange(m, dtype=np.int64) * 1021 - (1 << 30)).astype(np.int32)
    i64 = np.arange(m, dtype=np.int64) * 1_000_003 - (1 << 40)
    arrays = {"i32": pa.array(i32[ids]), "i64": pa.array(i64[ids]), "i64n": pa.array(i64[ids], mask=nulls)}
    p = str(tmp_path / "ids.parquet")
    _write_and_read_back(rdf, ctx, p, arrays, _odd_cuts(n), row_group_rows=n)
    bw = id_bit_width(m)
    straddle = False
    for i, (name, width) in enumerate((("i32", 4), ("i64", 8), ("i64n", 8))):
        pages = H.chunk_pages(p, i)
        if m * width > DICT_LIMIT:
            assert {H.page_info(h)[0] for h, _ in pages} == {"v1"} and {H.page_info(h)[2] for h, _ in pages} == {H.ENC_PLAIN}, name
            continue
        assert H.page_info(pages[0][0]) == ("dict", m, H.ENC_PLAIN_DICTIONARY), name
        assert H.data_page_rows(pages) == _expected_pages(n, PAGE_ROWS)
        for h, body in pages[1:]:
            kind, rows, enc = H.page_info(h)
            assert enc == H.ENC_PLAIN_DICTIONARY
            levels, vals = H.page_sections(h, body, True, False)
            assert vals[0] == bw, (name, vals[0], bw)
            straddle |= _ids_straddle(body, _valid_rows(levels, rows), bw)
    if m * 4 <= DICT_LIMIT and bw not in (1, 2, 4, 8):
        assert straddle, (k, plus, bw)


@gpu
@pytest.mark.parametrize("plus", [0, 1])
@pytest.mark.parametrize("dtype", ["f64", "f32", "i64", "i32"])
def test_writer_dictionary_limit(rdf, ctx, tmp_path, dtype, plus):
    """DICT_LIMIT bytes of entries keep the dictionary; one entry more writes the chunk PLAIN.  Floats include -0.0 and 0.0 and NaNs
    of different payloads: separate entries by bit pattern, round-tripped bit for bit."""
    width = 8 if dtype in ("f64", "i64") else 4
    m = DICT_LIMIT // width + plus
    rng = np.random.default_rng(m + width)
    ut = np.uint64 if width == 8 else np.uint32
    if dtype.startswith("f"):
        ft = np.float64 if width == 8 else np.float32
        special = (np.array([0, 1 << 63, 0x7FF8000000000001, 0xFFF8000000000002, 0x7FF0000000000005], dtype=np.uint64) if width == 8 else
                   np.array([0, 1 << 31, 0x7FC00001, 0xFFC00002, 0x7F800005], dtype=np.uint32))
        finite = ((np.arange(m - 5) + 1) * 1.5).astype(ft).view(ut)
        entries = np.concatenate([special, finite]).view(ft)
        assert len(np.unique(entries.view(ut))) == m
        pt = pa.float64() if width == 8 else pa.float32()
    else:
        it = np.int64 if width == 8 else np.int32
        entries = (np.arange(m, dtype=np.int64) * 7 - m).astype(it)
        pt = pa.int64() if width == 8 else pa.int32()
    ids = np.concatenate([rng.permutation(m), rng.integers(0, m, 5000)])
    p = str(tmp_path / "lim.parquet")
    _write_and_read_back(rdf, ctx, p, {"x": pa.array(entries[ids], pt)}, _odd_cuts(len(ids)), row_group_rows=len(ids))
    cm = pq.ParquetFile(p).metadata.row_group(0).column(0)
    pages = H.chunk_pages(p, 0)
    if plus == 0:
        assert cm.has_dictionary_page and H.page_info(pages[0][0]) == ("dict", m, H.ENC_PLAIN_DICTIONARY)
        assert pages[0][0][2] == DICT_LIMIT   # exactly 1 MiB of entries
    else:
        assert not cm.has_dictionary_page and {H.page_info(h)[2] for h, _ in pages} == {H.ENC_PLAIN}


def _body_shape(total):
    """(value width, rows, valid rows) of an Int64 / Int32 PLAIN page whose uncompressed body is `total` bytes: the 4-byte level
    length, one RLE level run (no nulls) or one bit-packed run (nulls), then the values."""
    for w in (8, 4):
        for rows in range(total // w, total // (w + 1), -1):
            if 4 + _rle_len(rows) + w * rows == total:
                return w, rows, rows
            groups = (rows + 7) // 8
            rest = total - 4 - len(H._varint_encode(groups << 1 | 1, None)) - groups
            if rest % w == 0 and 0 < rest // w < rows:
                return w, rows, rest // w
    raise AssertionError(total)


@gpu
@pytest.mark.parametrize("data", ["random", "repeat", "edge"])
@pytest.mark.parametrize("total", [FRAGMENT - 1, FRAGMENT, FRAGMENT + 1, 3 * FRAGMENT + 1])
def test_writer_snappy_fragments(rdf, ctx, tmp_path, total, data):
    """A page body of `total` bytes, incompressible, highly repetitive, or a repeat that crosses each fragment edge: one snappy stream
    that pyarrow decodes, made of independently compressed fragments of FRAGMENT bytes (an element boundary at every fragment edge,
    no copy reaching before its fragment), the values round-tripped."""
    w, rows, valid = _body_shape(total)
    rng = np.random.default_rng(total + len(data))
    it = np.int64 if w == 8 else np.int32
    if data == "random":
        v = rng.integers(np.iinfo(it).min, np.iinfo(it).max, rows, dtype=it, endpoint=True)
    elif data == "repeat":
        v = np.full(rows, 1234567, dtype=it)
    else:   # a block of 1000 values repeated: every fragment edge falls inside a repeat
        v = np.tile(rng.integers(np.iinfo(it).min, np.iinfo(it).max, 1000, dtype=it, endpoint=True), rows // 1000 + 1)[:rows]
    mask = np.zeros(rows, dtype=bool)
    mask[rng.choice(rows, rows - valid, replace=False)] = True
    p = str(tmp_path / "s.parquet")
    _write_and_read_back(rdf, ctx, p, {"x": pa.array(v, mask=mask)}, [rows], compression="snappy", dictionary=False)
    assert pq.ParquetFile(p).metadata.row_group(0).column(0).compression == "SNAPPY"
    (h, body), = H.chunk_pages(p, 0)
    assert h[2] == total
    raw = pa.decompress(body, total, codec="snappy").to_pybytes()
    n, els = H.snappy_elements(body)
    assert n == total
    starts = {op for _, _, _, op in els}
    edges = list(range(FRAGMENT, total, FRAGMENT))
    assert set(edges) <= starts and len(edges) + 1 == -(-total // FRAGMENT)
    for kind, ln, off, op in els:
        assert kind == "lit" or op - off >= op // FRAGMENT * FRAGMENT, (op, off)
        assert (op + ln - 1) // FRAGMENT == op // FRAGMENT   # no element crosses a fragment edge
    if data == "random":   # the values stay literals
        assert sum(ln for kind, ln, _, _ in els if kind == "lit") >= w * valid
    else:
        assert len(body) < total // 4 and any(kind != "lit" for kind, _, _, _ in els)
    lev = int.from_bytes(raw[:4], "little")
    assert len(raw) == 4 + lev + w * valid
