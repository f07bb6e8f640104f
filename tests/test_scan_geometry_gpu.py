"""The shared prefix scan (k_scan.cu) on its edges, through the operators that had no scan-edge test of their own, against their oracles.

Every operator that turns per-row counts into offsets runs the same kernels: the one-CTA scan of 1024 threads (k_scan_one), and for
longer inputs the tile sums of kScanTile entries, their one-CTA scan and the per-tile rescan.  The join and the window put their
own scans on the edges in test_relational_geometry_gpu.py; here are the others:

  * the JSON reader: files of kScanTile x k - 1, x k and x k + 1 records whose line counts need 1023, 1024, 1025 and 2049 tile sums,
    and whose sizes need as many newline tiles (JSON_TILE bytes each, scanned by k_scan_one);
  * the CSV reader: files whose tokenizer needs 1023, 1024, 1025 and 2049 tiles (CSV_TILE bytes each);
  * list take: kScanTile x k - 1, x k and x k + 1 indices;
  * the CSV writer: exactly one block of CSVW_MAX_ROWS rows (1024 tile sums), and one row fewer and more, byte for byte.

A non-GPU test re-reads every constant from csrc/, so a retuned kernel fails here instead of testing the wrong edges.
"""
import os
import re

import numpy as np
import pyarrow as pa
import pytest

import csv_oracle as co
import csv_write_oracle as wo
import json_oracle as jo
import list_frame_oracle as lfo

gpu = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "rust-dataframe_b200", "csrc")

# the constants; test_constants_match_csrc re-reads every one of them from the sources
THREADS = 256                  # common.cuh kThreads
SCAN_TILE = THREADS * 8        # scan.cuh kScanTile: entries per tile sum
JSON_TILE = THREADS * 16       # k_json.cu kJsonTile: bytes per CTA of the newline count
CSV_TILE = THREADS * 16        # k_csv.cu kCsvTile: bytes per CTA of the tokenizer
CSVW_MAX_ROWS = 1 << 21        # runtime.cu kCsvwMaxRows: rows per block of the CSV writer
SCAN_COUNTS = [1023, 1024, 1025, 2049]


def _read(name):
    with open(os.path.join(CSRC, name)) as f:
        return f.read()


def test_constants_match_csrc():
    common, scan_h, scan = _read("common.cuh"), _read("scan.cuh"), _read("k_scan.cu")
    js, csv, runtime = _read("k_json.cu"), _read("k_csv.cu"), _read("runtime.cu")

    def num(src, pat):
        m = re.search(pat, src)
        assert m, f"pattern {pat!r} not found"
        return int(m.group(1))

    assert num(common, r"constexpr int kThreads = (\d+);") == THREADS
    assert re.search(r"constexpr int kScanTile = kThreads \* kScanItems;", scan_h)
    assert THREADS * num(scan_h, r"constexpr int kScanItems = (\d+);") == SCAN_TILE
    assert re.search(r"per = \(count \+ 1023\) / 1024;", scan) and re.search(r"k_scan_one<T><<<1, 1024, 0, s>>>", scan)
    assert re.search(r"constexpr int kJsonTile = kThreads \* kJsonBytes;", js) and THREADS * num(js, r"constexpr int kJsonBytes = (\d+);") == JSON_TILE
    assert re.search(r"constexpr int kCsvTile = kThreads \* kCsvBytes;", csv) and THREADS * num(csv, r"constexpr int kCsvBytes = (\d+);") == CSV_TILE
    assert re.search(r"static constexpr int64_t kCsvwMaxRows = \(int64_t\)1 << (\d+);", runtime).group(1) == "21"
    # the readers and list take run these scans
    assert re.search(r"launch_scan_one\(counts, tiles, counts \+ tiles, s\)", js)
    assert re.search(r"launch_scan_one\(block_counts, tiles, block_counts \+ tiles, s\)", csv)
    assert len(re.findall(r"= launch_scan\((members|is_rec|counts|sizes), ", runtime)) == 4
    assert SCAN_TILE == 2048 and CSVW_MAX_ROWS // SCAN_TILE == 1024


def _tiles(n, tile):
    return -(-n // tile)


# ---------------------------------------------------------------------------------------------------------
# JSON reader

LIST_VALUES = [b"[1,2]", b"null ", b"[]   ", b"[-3] ", b"[7,8]"]   # one width, so every record line has the same length


def _json_file(rng, count, d):
    """Lines, bytes and records for `count` tile sums of the line scans, `count` newline tiles and kScanTile x k + d records."""
    lines = (count - 1) * SCAN_TILE + 1 + (count * 37) % (SCAN_TILE - 1)   # lines = newlines + 1
    size = (count - 1) * JSON_TILE + 1 + (count * 53) % (JSON_TILE - 1)
    newlines = lines - 1
    rec_len = len(b'{"a":%7d,"l":%s}' % (0, LIST_VALUES[0]))
    k = (size - newlines) // rec_len // SCAN_TILE - 1
    records = SCAN_TILE * k + d
    pad = size - newlines - records * rec_len                            # spaces inside the first record
    assert k >= 1 and 0 <= pad and records <= newlines
    at = np.sort(rng.choice(newlines, records, replace=False))          # which lines hold a record; the others are blank
    a = rng.integers(-999999, 9999999, records)
    lv = rng.integers(0, len(LIST_VALUES), records)
    out = [b""] * newlines
    for j, (i, x, v) in enumerate(zip(at.tolist(), a.tolist(), lv.tolist())):
        out[i] = b'{%s"a":%7d,"l":%s}' % (b" " * (pad if j == 0 else 0), x, LIST_VALUES[v])
    data = b"\n".join(out) + b"\n"
    assert len(data) == size and data.count(b"\n") + 1 == lines
    return data, records


def _list_rows(lc):
    rows = []
    for ch in lc.download():
        vals = np.asarray(ch.values.value_slice()).tolist()
        vm = ch.values.valid_mask()
        for k in range(ch.length):
            valid = ch.validity is None or (ch.validity[k >> 3] >> (k & 7)) & 1
            s, e = int(ch.offsets[k]), int(ch.offsets[k + 1])
            rows.append([vals[j] if vm[j] else None for j in range(s, e)] if valid else None)
    return rows


@gpu
@pytest.mark.parametrize("count", SCAN_COUNTS)
def test_json_scan_tiles(rdf, ctx, tmp_path, count):
    """count tile sums in the line scans and count newline tiles; kScanTile x k - 1, x k or x k + 1 records in the list scan."""
    rng = np.random.default_rng(200 + count)
    d = (-1, 0, 1, -1)[SCAN_COUNTS.index(count)]
    data, records = _json_file(rng, count, d)
    assert _tiles(data.count(b"\n") + 1, SCAN_TILE) == count and _tiles(len(data), JSON_TILE) == count
    p = tmp_path / "t.json"
    p.write_bytes(data)
    ref = jo.read(data, batch_size=65536)
    assert ref.num_rows == records
    with rdf.JsonFile(str(p), batch_size=65536, ctx=ctx) as f:
        assert [n for n, _, _ in f.schema] == ref.names == ["a", "l"] and f.num_rows == records
        col = f.read([0])["a"]
        got = np.concatenate([a.value_slice() for a in col.download()])
        want, wm = ref.column(0)
        assert wm.all() and np.array_equal(got, want.astype(got.dtype))
        assert _list_rows(f.read_list(1)) == ref.list_column(1)


# ---------------------------------------------------------------------------------------------------------
# CSV reader

@gpu
@pytest.mark.parametrize("count", SCAN_COUNTS)
def test_csv_tokenizer_tiles(rdf, ctx, tmp_path, count):
    """A file of count tokenizer tiles: count CTA totals of field ends in k_scan_one, the file's field index from them."""
    rng = np.random.default_rng(300 + count)
    rows = ((count - 1) * CSV_TILE + 1 + (count * 61) % (CSV_TILE - 32) - 4 + 15) // 16   # 16-byte rows after the 4-byte header
    v = rng.integers(1000000, 9999999, (rows, 2))
    data = b"a,b\n" + "".join(f"{x},{y}\n" for x, y in v.tolist()).encode()
    assert _tiles(len(data), CSV_TILE) == count
    p = tmp_path / "t.csv"
    p.write_bytes(data)
    ref = co.read(data, batch_size=65536)
    assert ref.num_rows == rows
    with rdf.CsvFile(str(p), batch_size=65536, ctx=ctx) as f:
        assert f.num_rows == rows
        cols = f.read([0, 1])
        for i, name in enumerate(("a", "b")):
            got = np.concatenate([a.value_slice() for a in cols[name].download()])
            want, wm = ref.column(i)
            assert wm.all() and np.array_equal(got, want.astype(got.dtype)) and np.array_equal(got, v[:, i])


# ---------------------------------------------------------------------------------------------------------
# list take

@gpu
@pytest.mark.parametrize("k", [1, 2, 1024])
def test_list_take_scan_tiles(rdf, ctx, k):
    """kScanTile x k - 1, x k and x k + 1 taken lists: as many sizes scanned into element offsets."""
    rng = np.random.default_rng(400 + k)
    n_lists = 5000
    lens = rng.integers(0, 6, n_lists)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    vals = rng.integers(-100, 100, int(off[-1])).astype(np.int32)
    vm = rng.random(vals.size) >= 0.1
    lvalid = rng.random(n_lists) >= 0.05
    arr = pa.ListArray.from_arrays(pa.array(off), pa.array(vals, mask=~vm), mask=pa.array(~lvalid))
    lists = [None if x is None else list(x) for x in arr.to_pylist()]
    lc = rdf.ListColumn.upload([rdf.ListArray.from_arrow(arr)], ctx)
    for d in (-1, 0, 1):
        n = SCAN_TILE * k + d
        idx = rng.integers(0, n_lists, n)
        got = lc.take(rdf.Column.upload([rdf.PrimitiveArray.from_numpy(idx.astype(np.uint32))], ctx))
        assert got.n_chunks == 1
        assert got.download()[0].to_pylist() == lfo.take(lists, idx.tolist()), (k, d)


# ---------------------------------------------------------------------------------------------------------
# CSV writer

@gpu
@pytest.mark.parametrize("d", [-1, 0, 1])
def test_csv_write_block_edges(rdf, ctx, tmp_path, d):
    """One Int32 column of CSVW_MAX_ROWS + d rows: a block of exactly CSVW_MAX_ROWS rows is 1024 tile sums; one more row starts a
    second block of one row."""
    rng = np.random.default_rng(500 + d)
    n = CSVW_MAX_ROWS + d
    v = rng.integers(-2 ** 31, 2 ** 31, n, dtype=np.int64).astype(np.int32)
    m = rng.random(n) >= 0.1
    a = rdf.PrimitiveArray.from_numpy(v, m)
    a.null_count = int((~m).sum())
    p = tmp_path / "w.csv"
    rdf.write_csv(str(p), {"a": rdf.Column.upload([a], ctx=ctx, dtype=co.I32)})
    assert p.read_bytes() == wo.write([("a", co.I32, v, m)])
