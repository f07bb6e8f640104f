"""Parquet fixtures shared by tests/test_parquet.py (CPU), tests/test_parquet_gpu.py and tests/test_parquet_geometry_gpu.py: pyarrow-written
files, a small Thrift compact-protocol reader for page headers, byte patches that make the device-detected errors, hand-built files with
the page shapes pyarrow does not write, snappy streams of chosen elements, and the check of a device read against pyarrow.  The CPU
tests run the patched bytes through the sanitized host build of the decoders before the GPU tests read them on the device."""
from __future__ import annotations

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pyarrow.parquet as pq


def table(n: int, seed: int = 0, null_frac: float = 0.1) -> pa.Table:
    """Every type of the reader's table, optional columns with about null_frac nulls, plus a string and a struct column."""
    rng = np.random.default_rng(seed)

    def mask():
        return rng.random(n) < null_frac if null_frac else None

    return pa.table({
        "b": pa.array(rng.random(n) < 0.5, mask=mask()),
        "i8": pa.array(rng.integers(-128, 128, n), pa.int8(), mask=mask()),
        "i16": pa.array(rng.integers(-2 ** 15, 2 ** 15, n), pa.int16(), mask=mask()),
        "i32": pa.array(rng.integers(-2 ** 31, 2 ** 31, n), pa.int32(), mask=mask()),
        "i64": pa.array(rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64), pa.int64(), mask=mask()),
        "u8": pa.array(rng.integers(0, 256, n), pa.uint8(), mask=mask()),
        "u16": pa.array(rng.integers(0, 2 ** 16, n), pa.uint16(), mask=mask()),
        "u32": pa.array(rng.integers(0, 2 ** 32, n), pa.uint32(), mask=mask()),
        "u64": pa.array(rng.integers(0, 2 ** 64, n, dtype=np.uint64), pa.uint64(), mask=mask()),
        "f32": pa.array(rng.standard_normal(n).astype(np.float32), mask=mask()),
        "f64": pa.array(rng.integers(0, 50, n) * 0.5, mask=mask()),   # repetitive: dictionary pages
        "s": pa.array([str(i) for i in range(n)]),
        "d": pa.array(rng.integers(-20000, 20000, n).astype(np.int32), pa.date32(), mask=mask()),
        "t32": pa.array(rng.integers(0, 86_400_000, n).astype(np.int32), pa.time32("ms"), mask=mask()),
        "t64": pa.array(rng.integers(0, 86_400_000_000, n), pa.time64("us"), mask=mask()),
        "tsu": pa.array(rng.integers(-2 ** 50, 2 ** 50, n), pa.timestamp("us", tz="UTC"), mask=mask()),
        "tsn": pa.array(rng.integers(-2 ** 60, 2 ** 60, n), pa.timestamp("ns"), mask=mask()),
        "tsz": pa.array(rng.integers(-2 ** 40, 2 ** 40, n), pa.timestamp("ms", tz="+01:00"), mask=mask()),
        "st": pa.array([{"a": i} for i in range(n)]),
    })


def required(t: pa.Table) -> pa.Table:
    """The same columns (of a table without nulls) declared non-nullable: required Parquet columns."""
    return pa.Table.from_arrays(t.columns, schema=pa.schema([pa.field(f.name, f.type, nullable=False) for f in t.schema]))


EXPECT_DTYPE = {"b": 10, "i8": 0, "i16": 1, "i32": 2, "i64": 3, "u8": 4, "u16": 5, "u32": 6, "u64": 7, "f32": 8, "f64": 9, "s": -1, "d": 2,
                "t32": 2, "t64": 3, "tsu": 3, "tsn": 3, "tsz": 3, "st": -1}

# writer options of the test matrix: (id, kwargs of pq.write_table)
MATRIX = [
    ("v1-snappy", dict(data_page_version="1.0")),
    ("v2-snappy", dict(data_page_version="2.0")),
    ("v1-none-small-pages", dict(data_page_version="1.0", compression="none", data_page_size=2048)),
    ("v2-none-rg", dict(data_page_version="2.0", compression="none", row_group_size=1700)),
    ("v2-snappy-rg-small", dict(data_page_version="2.0", row_group_size=999, data_page_size=1024)),
    ("plain", dict(use_dictionary=False, data_page_version="2.0")),
    ("dict-fallback", dict(dictionary_pagesize_limit=256, data_page_size=512)),
    ("bss", dict(use_dictionary=False, use_byte_stream_split=["f32", "f64", "i32", "i64", "d", "tsu"], data_page_version="2.0")),
]


# ---- Thrift compact protocol: just enough to find the end of a page header and a field inside it -------------------------------------
def _varint(b: bytes, i: int):
    v, s = 0, 0
    while True:
        x = b[i]
        i += 1
        v |= (x & 0x7F) << s
        s += 7
        if not x & 0x80:
            return v, i


def _varint_encode(v: int, width):
    """ULEB128 of v; with `width`, padded to that many bytes (continuation bits on the padding)."""
    out = bytearray()
    while True:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
        if not v:
            break
    while width is not None and len(out) < width:
        out.append(0x80)
    out[-1] &= 0x7F
    return bytes(out)


def skip_struct(b: bytes, i: int) -> int:
    """Position after the compact-protocol struct starting at b[i]."""
    last = 0
    while True:
        h = b[i]
        i += 1
        if h == 0:
            return i
        t, d = h & 0x0F, h >> 4
        if d == 0:
            _, i = _varint(b, i)
        i = _skip(b, i, t)


def _skip(b: bytes, i: int, t: int) -> int:
    if t in (1, 2):
        return i
    if t == 3:
        return i + 1
    if t in (4, 5, 6):
        return _varint(b, i)[1]
    if t == 7:
        return i + 8
    if t == 8:
        n, i = _varint(b, i)
        return i + n
    if t in (9, 10):
        h = b[i]
        i += 1
        n, et = h >> 4, h & 0x0F
        if n == 15:
            n, i = _varint(b, i)
        for _ in range(n):
            i = _skip(b, i, 3 if et in (1, 2) else et)
        return i
    if t == 12:
        return skip_struct(b, i)
    raise ValueError(f"thrift type {t}")


def first_data_page(path: str, column: int = 0):
    """(file bytes, page header start, page data start) of the first data page of a column of row group 0."""
    md = pq.ParquetFile(path).metadata.row_group(0).column(column)
    b = bytearray(open(path, "rb").read())
    start = md.data_page_offset
    return b, start, skip_struct(bytes(b), start)


def dict_index_fixture(path: str) -> None:
    """An uncompressed, dictionary-encoded Int64 column of 100 distinct values whose dictionary page header is patched to say 70
    values: the data pages then hold ids 70..99, outside the dictionary (a device-detected error)."""
    vals = np.tile(np.arange(100, dtype=np.int64) * 3, 20)
    pq.write_table(pa.table({"x": pa.array(vals, pa.int64())}), path, compression="none", data_page_version="2.0")
    md = pq.ParquetFile(path).metadata.row_group(0).column(0)
    b = bytearray(open(path, "rb").read())
    d0 = md.dictionary_page_offset
    hdr_end = skip_struct(bytes(b), d0)
    k = bytes(b[d0:hdr_end]).find(b"\x15\xc8\x01")   # DictionaryPageHeader.num_values = 100 (zigzag varint c8 01)
    assert k > 0
    b[d0 + k + 1:d0 + k + 3] = b"\x8c\x01"           # 70, the same length
    open(path, "wb").write(bytes(b))


def snappy_fixture(path: str):
    """A snappy V2 Float64 column whose first data page declares a wrong uncompressed length in its snappy preamble.  Returns the
    corrupted compressed values section and the size the page header declares (for the sanitized CPU decoder)."""
    rng = np.random.default_rng(3)
    t = pa.Table.from_arrays([pa.array(rng.integers(0, 1000, 4000) * 0.25)], schema=pa.schema([pa.field("x", pa.float64(), nullable=False)]))
    pq.write_table(t, path, compression="snappy", data_page_version="2.0", use_dictionary=False)   # required: no level section
    b, start, data = first_data_page(path)
    # PageHeader: field 2 uncompressed_page_size, field 3 compressed_page_size (i32, zigzag), read from the header
    hdr = bytes(b[start:data])
    i, last, fields = 0, 0, {}
    while hdr[i] != 0:
        h = hdr[i]
        i += 1
        t, d = h & 0x0F, h >> 4
        fid = last + d
        last = fid
        if t == 5 and fid in (2, 3):
            v, i = _varint(hdr, i)
            fields[fid] = (v >> 1) ^ -(v & 1)
        else:
            i = _skip(hdr, i, t)
    raw, comp = fields[2], fields[3]
    assert b[data] != 0x05
    b[data] = 0x05   # the preamble's first byte: the stream now declares 5 bytes, not the page's 32000
    open(path, "wb").write(bytes(b))
    return bytes(b[data:data + comp]), raw


# ---- a Thrift compact-protocol writer and hand-built Parquet files: what pyarrow does not write ---------------------------------------
def _zz(v: int) -> int:
    return (v << 1) ^ (v >> 63)


class ThriftWriter:
    """Compact protocol, just the forms a Parquet footer and page header use."""

    def __init__(self):
        self.b = bytearray()
        self._last = [0]

    def _field(self, fid: int, t: int):
        d = fid - self._last[-1]
        if 0 < d <= 15:
            self.b.append(d << 4 | t)
        else:
            self.b.append(t)
            self.b += _varint_encode(_zz(fid), None)
        self._last[-1] = fid

    def i32(self, fid, v):
        self._field(fid, 5); self.b += _varint_encode(_zz(v), None); return self

    def i64(self, fid, v):
        self._field(fid, 6); self.b += _varint_encode(_zz(v), None); return self

    def binary(self, fid, v: bytes):
        self._field(fid, 8); self.b += _varint_encode(len(v), None) + v; return self

    def begin(self, fid=None):
        """A struct field (fid) or a struct element of a list (None)."""
        if fid is not None:
            self._field(fid, 12)
        self._last.append(0)
        return self

    def end(self):
        self.b.append(0)
        self._last.pop()
        return self

    def list(self, fid, etype: int, n: int):
        self._field(fid, 9)
        self.b += bytes([n << 4 | etype]) if n < 15 else bytes([0xF0 | etype]) + _varint_encode(n, None)
        return self


def hybrid_encode(values, bw: int, runs) -> bytes:
    """The RLE / bit-packed hybrid of `values` as the given runs: ("rle", count) or ("bp", groups of 8)."""
    out, i = bytearray(), 0
    for kind, n in runs:
        if kind == "rle":
            out += _varint_encode(n << 1, None)
            out += int(values[i]).to_bytes((bw + 7) // 8, "little")
            i += n
        else:
            out += _varint_encode((n << 1) | 1, None)
            bits = 0
            for j in range(n * 8):
                v = int(values[i + j]) if i + j < len(values) else 0
                bits |= v << (j * bw)
            out += bits.to_bytes(n * bw, "little")
            i += n * 8
    return bytes(out)


def _page_header(ptype: int, raw: int, comp: int, num_values: int, encoding: int) -> bytes:
    w = ThriftWriter().i32(1, ptype).i32(2, raw).i32(3, comp)
    if ptype == 2:
        w.begin(7).i32(1, num_values).i32(2, encoding).end()
    else:
        w.begin(5).i32(1, num_values).i32(2, encoding).i32(3, 3).i32(4, 3).end()
    w.b.append(0)
    return bytes(w.b)


# (physical type, converted type, numpy dtype of the physical values) of every legacy column written by legacy_file
LEGACY = [("c_u8", 1, 11, np.int32), ("c_u16", 1, 12, np.int32), ("c_u32", 1, 13, np.int32), ("c_u64", 2, 14, np.int64),
          ("c_i8", 1, 15, np.int32), ("c_i16", 1, 16, np.int32), ("c_i32", 1, 17, np.int32), ("c_i64", 2, 18, np.int64),
          ("c_date", 1, 6, np.int32), ("c_tms", 1, 7, np.int32), ("c_tus", 2, 8, np.int64), ("c_tsms", 2, 9, np.int64),
          ("c_tsus", 2, 10, np.int64), ("c_dict", 2, None, np.int64)]
LEGACY_DTYPE = {"c_u8": 4, "c_u16": 5, "c_u32": 6, "c_u64": 7, "c_i8": 0, "c_i16": 1, "c_i32": 2, "c_i64": 3, "c_date": 2, "c_tms": 2,
                "c_tus": 3, "c_tsms": 3, "c_tsus": 3, "c_dict": 3}
LEGACY_TAG = {"c_date": (1, 0, None), "c_tms": (4, 1, None), "c_tus": (5, 2, None), "c_tsms": (3, 1, "UTC"), "c_tsus": (3, 2, "UTC")}


def legacy_values(n: int, seed: int = 0):
    """Per LEGACY column: physical values (in range for the converted type) and a validity mask (about 10 % nulls)."""
    rng = np.random.default_rng(seed)
    lim = {11: (0, 256), 12: (0, 1 << 16), 13: (0, 1 << 32), 14: (0, 1 << 63), 15: (-128, 128), 16: (-(1 << 15), 1 << 15),
           17: (-(1 << 31), 1 << 31), 18: (-(1 << 62), 1 << 62), 6: (-20000, 20000), 7: (0, 86_400_000), 8: (0, 86_400_000_000),
           9: (-(1 << 40), 1 << 40), 10: (-(1 << 50), 1 << 50), None: (0, 40)}
    out = {}
    for name, phys, conv, npdt in LEGACY:
        lo, hi = lim[conv]
        v = rng.integers(lo, hi, n, dtype=np.int64)
        if npdt == np.int32:
            v = v.astype(np.uint32).view(np.int32) if conv == 13 else v.astype(np.int32)
        out[name] = (v, rng.random(n) >= 0.1)
    return out


def legacy_file(path: str, n: int = 3000, seed: int = 0, variant: str = "ok"):
    """A file with only legacy converted types (no logical types), written by hand: one row group, V1 pages, uncompressed, optional
    columns.  c_dict is dictionary-encoded with PLAIN_DICTIONARY ids.  `variant` makes one host-detected error in c_i32 (or c_dict):
    "outside" (its chunk runs past the file), "two_dicts", "no_dict" (ids without a dictionary page) or "file_path"."""
    vals = legacy_values(n, seed)
    body = bytearray(b"PAR1")
    chunks = []
    for name, phys, conv, npdt in LEGACY:
        v, m = vals[name]
        levels = hybrid_encode(m.astype(int), 1, [("bp", (n + 7) // 8)])
        start = len(body)
        dict_off = None
        if name == "c_dict":
            dvals = np.arange(40, dtype=np.int64) * 7 + 1
            ids = (v[m]).astype(int)
            dpage = dvals.tobytes()
            n_dicts = 2 if variant == "two_dicts" else 0 if variant == "no_dict" else 1
            for _ in range(n_dicts):
                if dict_off is None:
                    dict_off = len(body)
                body += _page_header(2, len(dpage), len(dpage), 40, 2) + dpage
            groups = (len(ids) + 7) // 8
            vsec = bytes([6]) + hybrid_encode(ids, 6, [("bp", groups)])
            enc = 2
            vals[name] = (np.where(m, dvals[np.clip(v, 0, 39)], 0), m)
        else:
            vsec = v[m].tobytes()
            enc = 0
        data = struct_pack_u32(len(levels)) + levels + vsec   # V1: the levels with their 4-byte length, then the values
        data_off = len(body)
        body += _page_header(0, len(data), len(data), n, enc) + data
        total = len(body) - start
        if variant == "outside" and name == "c_i32":
            total += 10 ** 6
        chunks.append((name, phys, conv, start, data_off, dict_off, total, enc))
    w = ThriftWriter().i32(1, 1)
    w.list(2, 12, len(LEGACY) + 1)
    w.begin().binary(4, b"schema").i32(5, len(LEGACY)).end()
    for name, phys, conv, npdt in LEGACY:
        w.begin().i32(1, phys).i32(3, 1).binary(4, name.encode())
        if conv is not None:
            w.i32(6, conv)
        w.end()
    w.i64(3, n)
    w.list(4, 12, 1).begin()
    w.list(1, 12, len(chunks))
    for name, phys, conv, start, data_off, dict_off, total, enc in chunks:
        w.begin()
        if variant == "file_path" and name == "c_i32":
            w.binary(1, b"other.parquet")
        w.i64(2, start).begin(3)
        w.i32(1, phys).list(2, 5, 2)
        w.b += _varint_encode(_zz(enc), None) + _varint_encode(_zz(3), None)
        w.list(3, 8, 1)
        w.b += _varint_encode(len(name), None) + name.encode()
        w.i32(4, 0).i64(5, n).i64(6, total).i64(7, total).i64(9, data_off)
        if dict_off is not None:
            w.i64(11, dict_off)
        w.end().end()
    w.i64(2, len(body)).i64(3, n).end()
    w.b.append(0)
    footer = bytes(w.b)
    body += footer + struct_pack_u32(len(footer)) + b"PAR1"
    open(path, "wb").write(bytes(body))
    return vals


def struct_pack_u32(v: int) -> bytes:
    return int(v).to_bytes(4, "little")


def read_struct(b: bytes, i: int):
    """A compact-protocol struct as {field id: value} (nested structs as dicts, lists as lists); returns (dict, end)."""
    out, last = {}, 0
    while True:
        h = b[i]
        i += 1
        if h == 0:
            return out, i
        t, d = h & 0x0F, h >> 4
        if d:
            fid = last + d
        else:
            z, i = _varint(b, i)
            fid = (z >> 1) ^ -(z & 1)
        last = fid
        out[fid], i = _read_value(b, i, t)


def _read_value(b, i, t):
    if t in (1, 2):
        return t == 1, i
    if t == 3:
        return b[i], i + 1
    if t in (4, 5, 6):
        z, i = _varint(b, i)
        return (z >> 1) ^ -(z & 1), i
    if t == 8:
        n, i = _varint(b, i)
        return bytes(b[i:i + n]), i + n
    if t == 12:
        return read_struct(b, i)
    if t in (9, 10):
        h = b[i]
        i += 1
        n, et = h >> 4, h & 0x0F
        if n == 15:
            n, i = _varint(b, i)
        vals = []
        for _ in range(n):
            v, i = _read_value(b, i, 3 if et in (1, 2) else et)
            vals.append(v)
        return vals, i
    return _skip(b, i, t) and None, _skip(b, i, t)


def chunk_pages(path: str, column: int = 0, row_group: int = 0):
    """[(page header as a dict, page bytes after the header)] of a column chunk."""
    md = pq.ParquetFile(path).metadata.row_group(row_group).column(column)
    b = open(path, "rb").read()
    pos = md.dictionary_page_offset if md.has_dictionary_page else md.data_page_offset
    end = pos + md.total_compressed_size
    pages = []
    while pos < end:
        h, data = read_struct(b, pos)
        pages.append((h, b[data:data + h[3]]))
        pos = data + h[3]
    return pages


# ---- what a page holds: its kind, rows and encoding, its level and value sections, the runs of a hybrid stream ----------------------
ENC_PLAIN, ENC_PLAIN_DICTIONARY, ENC_RLE, ENC_RLE_DICTIONARY, ENC_BSS = 0, 2, 3, 8, 9


def page_info(h: dict):
    """(kind, values, encoding) of a page header: kind "dict", "v1" or "v2"."""
    if h[1] == 2:
        return "dict", h[7][1], h[7][2]
    if h[1] == 0:
        return "v1", h[5][1], h[5][2]
    assert h[1] == 3, h[1]
    return "v2", h[8][1], h[8][4]


def data_page_rows(pages) -> list:
    return [page_info(h)[1] for h, _ in pages if h[1] != 2]


def page_sections(h: dict, body: bytes, optional: bool, snappy: bool):
    """(definition-level stream or None, values section) of a data page, decompressed."""
    kind = page_info(h)[0]
    if kind == "v2":
        rep, dl = h[8].get(6, 0), h[8].get(5, 0)
        levels = body[rep:rep + dl] if dl else None
        vals = body[rep + dl:]
        if snappy and h[8].get(7, True):
            vals = pa.decompress(vals, h[2] - rep - dl, codec="snappy").to_pybytes()
        return levels, vals
    if snappy:
        body = pa.decompress(body, h[2], codec="snappy").to_pybytes()
    if not optional:
        return None, body
    n = int.from_bytes(body[:4], "little")
    return body[4:4 + n], body[4 + n:]


def hybrid_runs(s: bytes, bw: int, need: int) -> list:
    """The runs of an RLE / bit-packed hybrid stream until `need` values are covered: ("rle", count, value) or ("bp", count)."""
    runs, p, cov = [], 0, 0
    while cov < need:
        h, p = _varint(s, p)
        if h & 1:
            count = (h >> 1) * 8
            runs.append(("bp", count))
            p += (h >> 1) * bw
        else:
            count = h >> 1
            vb = (bw + 7) // 8
            runs.append(("rle", count, int.from_bytes(s[p:p + vb], "little")))
            p += vb
        cov += count
    return runs


def hybrid_decode(s: bytes, bw: int, n: int) -> np.ndarray:
    """The first n values of an RLE / bit-packed hybrid stream."""
    out, p = [], 0
    while len(out) < n:
        h, p = _varint(s, p)
        if h & 1:
            groups = h >> 1
            bits = int.from_bytes(s[p:p + groups * bw], "little")
            out += [(bits >> (j * bw)) & ((1 << bw) - 1) for j in range(groups * 8)]
            p += groups * bw
        else:
            vb = (bw + 7) // 8
            out += [int.from_bytes(s[p:p + vb], "little")] * (h >> 1)
            p += vb
    return np.array(out[:n], dtype=np.int64)


# ---- snappy streams of chosen elements --------------------------------------------------------------------------------------------
def snappy_encode(elements) -> tuple:
    """(uncompressed bytes, snappy stream) of elements ("lit", bytes) and ("copy", offset, length, tag) with tag 1 (copy with a 1-byte
    offset, length 4..11, offset < 2048), 2 (2-byte offset, length 1..64) or 4 (4-byte offset, length 1..64)."""
    out, tags = bytearray(), bytearray()
    for e in elements:
        if e[0] == "lit":
            m = len(e[1]) - 1
            if m < 60:
                tags.append(m << 2)
            else:
                nb = (m.bit_length() + 7) // 8
                tags.append((59 + nb) << 2)
                tags += m.to_bytes(nb, "little")
            tags += e[1]
            out += e[1]
            continue
        _, off, ln, tag = e
        assert 0 < off <= len(out)
        if tag == 1:
            assert 4 <= ln <= 11 and off < 2048
            tags += bytes([1 | (ln - 4) << 2 | (off >> 8) << 5, off & 0xFF])
        else:
            assert 1 <= ln <= 64
            tags.append((2 if tag == 2 else 3) | (ln - 1) << 2)
            tags += off.to_bytes(2 if tag == 2 else 4, "little")
        for j in range(ln):
            out.append(out[len(out) - off])
    return bytes(out), _varint_encode(len(out), None) + bytes(tags)


def snappy_elements(stream: bytes) -> tuple:
    """(uncompressed length, [(kind, length, offset, output position)]) of a snappy stream; kind "lit", "copy1", "copy2" or "copy4"."""
    n, i = _varint(stream, 0)
    els, op = [], 0
    while i < len(stream):
        t = stream[i]
        i += 1
        if t & 3 == 0:
            ln = (t >> 2) + 1
            if ln > 60:
                nb = ln - 60
                ln = int.from_bytes(stream[i:i + nb], "little") + 1
                i += nb
            els.append(("lit", ln, 0, op))
            i += ln
        elif t & 3 == 1:
            ln, off = 4 + ((t >> 2) & 7), (t >> 5) << 8 | stream[i]
            i += 1
            els.append(("copy1", ln, off, op))
        else:
            nb = 2 if t & 3 == 2 else 4
            ln, off = (t >> 2) + 1, int.from_bytes(stream[i:i + nb], "little")
            i += nb
            els.append((f"copy{nb}", ln, off, op))
        op += ln
    assert op == n
    return n, els


# ---- a hand-built file of one column chunk ----------------------------------------------------------------------------------------
def rle_levels(runs) -> bytes:
    """A definition-level stream (bit width 1) of RLE runs (value, count)."""
    return b"".join(_varint_encode(c << 1, None) + bytes([v]) for v, c in runs)


def hand_file(path: str, phys: int, pages, codec: int = 0) -> None:
    """One optional column "x" (physical type phys, no logical type) in one row group, written by hand.  pages: (rows, encoding,
    raw body, compressed body or None) of V1 data pages, the body being the 4-byte level length, the levels and the values.  codec 1
    (SNAPPY): a page without its compressed body is compressed by pyarrow."""
    body = bytearray(b"PAR1")
    start = len(body)
    encs = {3}
    data_off = len(body)
    n = 0
    for rows, enc, raw, comp in pages:
        if comp is None:
            comp = pa.compress(raw, codec="snappy", asbytes=True) if codec else raw
        body += _page_header(0, len(raw), len(comp), rows, enc) + comp
        encs.add(enc)
        n += rows
    total = len(body) - start
    w = ThriftWriter().i32(1, 1)
    w.list(2, 12, 2)
    w.begin().binary(4, b"schema").i32(5, 1).end()
    w.begin().i32(1, phys).i32(3, 1).binary(4, b"x").end()
    w.i64(3, n)
    w.list(4, 12, 1).begin()
    w.list(1, 12, 1)
    w.begin().i64(2, start).begin(3)
    w.i32(1, phys).list(2, 5, len(encs))
    for e in sorted(encs):
        w.b += _varint_encode(_zz(e), None)
    w.list(3, 8, 1)
    w.b += _varint_encode(1, None) + b"x"
    w.i32(4, codec).i64(5, n).i64(6, total).i64(7, total).i64(9, data_off)
    w.end().end()
    w.i64(2, total).i64(3, n).end()
    w.b.append(0)
    footer = bytes(w.b)
    body += footer + struct_pack_u32(len(footer)) + b"PAR1"
    open(path, "wb").write(bytes(body))


# ---- a device read against pyarrow.parquet ------------------------------------------------------------------------------------------
def device_bits(col):
    """(values as unsigned bits, validity, chunk lengths, bitmap presence per chunk) of a device column."""
    vals, valid, lens, hv = [], [], [], []
    for a in col.download():
        m = np.asarray(a.valid_mask(), dtype=bool)
        if hasattr(a, "value_bits"):
            v = np.asarray(a.value_bits(), dtype=np.uint64)
        else:
            v = np.asarray(a.value_slice())
            v = v.view(f"u{v.dtype.itemsize}").astype(np.uint64)
        vals.append(v); valid.append(m); lens.append(a.length); hv.append(a.validity is not None)
    return np.concatenate(vals), np.concatenate(valid), lens, hv


def expected_bits(arr):
    """(values as unsigned bits, nulls as 0; validity) of an Arrow array or chunked array; temporal values as their integers."""
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    valid = np.asarray(arr.is_valid())
    t = arr.type
    if pa.types.is_boolean(t):
        v = np.asarray(pc.fill_null(arr, False)).astype(np.uint64)
    else:
        if pa.types.is_temporal(t):
            arr = arr.cast(pa.int32() if t.bit_width == 32 else pa.int64())
        v = np.asarray(pc.fill_null(arr, pa.scalar(0).cast(arr.type)) if arr.null_count else arr)
        v = v.view(f"u{v.dtype.itemsize}").astype(np.uint64)
    return v, valid


def check_read(rdf, ctx, paths, read_path, batch_size, names=None):
    """DataFrame::from_parquet of read_path (the files `paths`, in order) against pyarrow.parquet.read_table of each: every value bit for
    bit, the same null slots, 0 in a null slot, the output chunk lengths (every file cut into batches of batch_size), the bitmap
    presence of each chunk, and the temporal tags."""
    tables = [pq.read_table(p) for p in paths]
    with rdf.ParquetFile(read_path, batch_size=batch_size) as f:
        if names is None:
            names = [n for n, dt, _ in f.schema if dt >= 0]
        cols = f.read(names, ctx=ctx)
        assert f.num_rows == sum(t.num_rows for t in tables)
        for name in names:
            got, gvalid, lens, hv = device_bits(cols[name])
            want_lens, want_hv, wv, wvalid = [], [], [], []
            for t in tables:
                v, m = expected_bits(t.column(name))
                wv.append(v); wvalid.append(m)
                for s in range(0, t.num_rows, batch_size):
                    want_lens.append(min(batch_size, t.num_rows - s))
                    want_hv.append(not m[s:s + batch_size].all())
            wv, wvalid = np.concatenate(wv), np.concatenate(wvalid)
            assert lens == want_lens, name
            assert hv == want_hv, name
            assert np.array_equal(gvalid, wvalid), name
            assert np.array_equal(got[wvalid], wv[wvalid]), name
            assert not got[~wvalid].any(), name   # a null slot holds 0
            tag = f.temporal_columns.get(name)
            t = tables[0].schema.field(name).type
            if pa.types.is_temporal(t):
                assert tag is not None, name
                if pa.types.is_timestamp(t):
                    assert (tag.unit, tag.tz) == ({"ms": 1, "us": 2, "ns": 3}[t.unit], t.tz), name
            else:
                assert tag is None, name
