"""The Parquet reader without a GPU: the open, schema, types and row / batch counts against pyarrow over a matrix of files pyarrow writes
at test time; directories; the host-detected errors from bdf_parquet_check; and the decoders of csrc/parquet_decode.cuh compiled for
the host with g++ and the address and undefined-behaviour sanitizers (snappy against pyarrow's codec, hand-built and corrupt streams,
RLE / bit-packed hybrid streams and their truncations)."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pyarrow as pa
import pyarrow.parquet as pq
import pytest

import parquet_helpers as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "rust-dataframe_b200", "csrc")

UNIT = {"s": 0, "ms": 1, "us": 2, "ns": 3}


def _expected_tag(t: pa.DataType):
    """(kind, unit, tz) the reader gives a pyarrow type read back from Parquet (Timestamp(s) is stored, and read, as ms)."""
    if pa.types.is_date32(t):
        return (1, 0, None)
    if pa.types.is_time32(t):
        return (4, UNIT[t.unit], None)
    if pa.types.is_time64(t):
        return (5, UNIT[t.unit], None)
    if pa.types.is_timestamp(t):
        return (3, max(UNIT[t.unit], 1), t.tz)
    return None


@pytest.mark.parametrize("wid,kw", H.MATRIX, ids=[m[0] for m in H.MATRIX])
@pytest.mark.parametrize("shape", ["optional", "required"])
def test_schema_matrix(rdf, tmp_path, wid, kw, shape):
    t = H.table(3000, seed=1, null_frac=0.1 if shape == "optional" else 0.0)
    if shape == "required":
        t = H.required(t)
    p = str(tmp_path / "t.parquet")
    pq.write_table(t, p, **kw)
    arrow = pq.ParquetFile(p).schema_arrow
    with rdf.ParquetFile(p, batch_size=1000) as f:
        assert f.num_rows == 3000 and f.num_batches == 3
        assert [n for n, _, _ in f.schema] == arrow.names
        for (name, dt, nullable), fld in zip(f.schema, arrow):
            assert dt == H.EXPECT_DTYPE[name], name
            if dt >= 0:
                assert nullable == fld.nullable, name
                f.check(name)
            else:
                with pytest.raises(rdf.UnsupportedType, match="not on the device path"):
                    f.check(name)
            tag = f.temporal_columns.get(name)
            want = _expected_tag(fld.type)
            assert (None if tag is None else (tag.kind, tag.unit, tag.tz)) == want, name


def test_directory(rdf, tmp_path):
    d = tmp_path / "d"
    d.mkdir()
    for k, n in enumerate([1500, 2048, 1]):
        pq.write_table(H.table(n, seed=k), str(d / f"part-{k}.parquet"), row_group_size=700)
    (d / "_SUCCESS").write_bytes(b"")
    (d / ".crc").write_bytes(b"x")
    with rdf.ParquetFile(str(d), batch_size=1024) as f:
        assert f.num_rows == 1500 + 2048 + 1
        assert f.num_batches == 2 + 2 + 1   # each file starts a new batch
    # a file whose columns differ is named
    pq.write_table(pa.table({"other": [1, 2]}), str(d / "zz.parquet"))
    with pytest.raises(rdf.ComputeError, match="zz.parquet"):
        rdf.ParquetFile(str(d))
    # a file with zero row groups is skipped
    os.remove(str(d / "zz.parquet"))
    pq.ParquetWriter(str(d / "zz-empty.parquet"), H.table(1, seed=0).schema).close()
    assert pq.ParquetFile(str(d / "zz-empty.parquet")).metadata.num_row_groups == 0
    with rdf.ParquetFile(str(d), batch_size=1024) as f:
        assert (f.num_rows, f.num_batches) == (1500 + 2048 + 1, 5)
    # nothing left
    e = tmp_path / "empty"
    e.mkdir()
    (e / "_SUCCESS").write_bytes(b"")
    pq.ParquetWriter(str(e / "only-empty.parquet"), H.table(1, seed=0).schema).close()
    with pytest.raises(rdf.ReferencePanic):
        rdf.ParquetFile(str(e))


def test_legacy_converted_types(rdf, tmp_path):
    """A hand-written file with only converted types (no logical types), and PLAIN_DICTIONARY ids: read by pyarrow too, which checks
    the test's writer."""
    p = str(tmp_path / "legacy.parquet")
    H.legacy_file(p)
    arrow = pq.read_table(p).schema
    md = pq.ParquetFile(p).metadata.row_group(0)
    assert "PLAIN_DICTIONARY" in md.column(len(H.LEGACY) - 1).encodings
    with rdf.ParquetFile(p) as f:
        assert [n for n, _, _ in f.schema] == arrow.names
        for (name, dt, nullable), fld in zip(f.schema, arrow):
            assert dt == H.LEGACY_DTYPE[name], name
            assert nullable
            f.check(name)
            tag = f.temporal_columns.get(name)
            assert (None if tag is None else (tag.kind, tag.unit, tag.tz)) == H.LEGACY_TAG.get(name), name
            assert (None if tag is None else (tag.kind, tag.unit, tag.tz)) == _expected_tag(fld.type), name


@pytest.mark.parametrize("variant,column,status,message", [
    ("outside", "c_i32", "ComputeError", r"row group 0, column 6: the column chunk \[\d+, \+\d+\) lies outside the file"),
    ("two_dicts", "c_dict", "ComputeError", r"row group 0, column 13, page 1: more than one dictionary page"),
    ("no_dict", "c_dict", "ComputeError", r"row group 0, column 13, page 0: a dictionary-encoded page without a dictionary page"),
])
def test_hand_built_chunk_errors(rdf, tmp_path, variant, column, status, message):
    p = str(tmp_path / f"{variant}.parquet")
    H.legacy_file(p, variant=variant)
    with rdf.ParquetFile(p) as f:
        with pytest.raises(getattr(rdf, status), match=r"\[bdf status 8\] Parquet error in .*" + message):
            f.check(column)
        f.check("c_i64")   # the other columns still read


def test_column_chunk_in_another_file(rdf, tmp_path):
    p = str(tmp_path / "fp.parquet")
    H.legacy_file(p, variant="file_path")
    with pytest.raises(rdf.UnsupportedType, match=r"row group 0: a column chunk in another file \(other.parquet\) is not supported"):
        rdf.ParquetFile(p)


def test_nullable_is_or_over_files(rdf, tmp_path):
    d = tmp_path / "d"
    d.mkdir()
    pq.write_table(H.required(H.table(100, seed=1, null_frac=0.0)), str(d / "a.parquet"))
    pq.write_table(H.table(100, seed=2), str(d / "b.parquet"))
    with rdf.ParquetFile(str(d)) as f:
        assert all(nl for _, dt, nl in f.schema if dt >= 0)


def _patched(tmp_path, src: str, fn) -> str:
    b = bytearray(open(src, "rb").read())
    fn(b)
    p = str(tmp_path / "bad.parquet")
    open(p, "wb").write(bytes(b))
    return p


def test_host_detected_errors(rdf, tmp_path):
    src = str(tmp_path / "ok.parquet")
    pq.write_table(H.table(2000, seed=3), src, compression="none", data_page_version="1.0")

    def magic(b):
        b[0:4] = b"PAR2"
    with pytest.raises(rdf.ComputeError, match=r"Parquet error in .*bad.parquet: bad magic"):
        rdf.ParquetFile(_patched(tmp_path, src, magic))

    def encrypted(b):
        b[-4:] = b"PARE"
    with pytest.raises(rdf.UnsupportedType, match="encrypted"):
        rdf.ParquetFile(_patched(tmp_path, src, encrypted))

    def footer_len(b):
        b[-8:-4] = struct.pack("<I", len(b))
    with pytest.raises(rdf.ComputeError, match="footer .* outside the file"):
        rdf.ParquetFile(_patched(tmp_path, src, footer_len))

    # a page header that no longer parses inside its chunk: the column's check and read fail, the others still pass
    md = pq.ParquetFile(src).metadata.row_group(0).column(4)

    def header(b):
        b[md.data_page_offset:md.data_page_offset + 8] = b"\xff" * 8
    with rdf.ParquetFile(_patched(tmp_path, src, header)) as f:
        with pytest.raises(rdf.ComputeError, match=r"row group 0, column 4, page \d+: the page header runs past its column chunk"):
            f.check(4)
        f.check(3)

    # data-page num_values that do not add up to the row group's rows (the first data page's num_values, zigzag, one less)
    b0, start, data = H.first_data_page(src, 3)
    hdr = bytes(b0[start:data])
    k = hdr.find(b"\x15", hdr.find(b"\x2c") + 1)   # DataPageHeader (field 5, struct) then num_values (field 1, i32)
    v, end = H._varint(hdr, k + 1)

    def num_values(b):
        b[start + k + 1:start + end] = bytes(H._varint_encode(v - 2, end - k - 1))
    with rdf.ParquetFile(_patched(tmp_path, src, num_values)) as f:
        with pytest.raises(rdf.ComputeError, match="num_values add up to 1999, the row group has 2000 rows"):
            f.check(3)


@pytest.mark.parametrize("codec", ["gzip", "brotli", "lz4", "zstd"])
def test_unsupported_codec(rdf, tmp_path, codec):
    p = str(tmp_path / "t.parquet")
    t = H.table(500, seed=1)
    pq.write_table(t, p, compression={"i32": codec, "i64": "snappy"} | {n: "none" for n in t.column_names if n not in ("i32", "i64")})
    with rdf.ParquetFile(p) as f:
        with pytest.raises(rdf.UnsupportedType, match=f"codec {codec.upper().replace('LZ4', 'LZ4_RAW')} is not supported"):
            f.check("i32")
        f.check("i64")


def test_unsupported_encoding(rdf, tmp_path):
    p = str(tmp_path / "t.parquet")
    pq.write_table(pa.table({"x": np.arange(1000, dtype=np.int64), "y": np.arange(1000.0)}), p, use_dictionary=False,
                   column_encoding={"x": "DELTA_BINARY_PACKED", "y": "PLAIN"})
    with rdf.ParquetFile(p) as f:
        with pytest.raises(rdf.UnsupportedType, match="encoding DELTA_BINARY_PACKED"):
            f.check("x")
        f.check("y")


# ---- the decoders on the host, under the sanitizers -----------------------------------------------------------------------------------
DRIVER = r"""
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "parquet_decode.cuh"
static std::vector<uint8_t> slurp(const char* p) {
    FILE* f = fopen(p, "rb"); std::vector<uint8_t> v; int c;
    while ((c = fgetc(f)) != EOF) v.push_back((uint8_t)c);
    fclose(f); return v;
}
int main(int argc, char** argv) {
    // exact-size heap buffers, so that ASan sees any access past either end
    std::vector<uint8_t> in = slurp(argv[2]);
    uint8_t* ib = (uint8_t*)malloc(in.size() ? in.size() : 1);
    for (size_t i = 0; i < in.size(); i++) ib[i] = in[i];
    if (argv[1][0] == 's') {   // snappy <in> <out_n> <out file>
        const uint32_t on = (uint32_t)atol(argv[3]);
        uint8_t* ob = (uint8_t*)malloc(on ? on : 1);
        const int e = pq::snappy_decode(ib, (uint32_t)in.size(), ob, on);
        printf("%d\n", e);
        if (!e) { FILE* f = fopen(argv[4], "wb"); fwrite(ob, 1, on, f); fclose(f); }
        free(ob);
    } else if (argv[1][0] == 'p') {   // page <data page bytes> <dictionary page bytes> <kind> <max_def> <num_values> <encoding> <width> <dict count> <def_len>
        std::vector<uint8_t> dv = slurp(argv[3]);
        uint8_t* db = (uint8_t*)malloc(dv.size() ? dv.size() : 1);
        for (size_t i = 0; i < dv.size(); i++) db[i] = dv[i];
        pq::Page p{};
        p.src = 0; p.dst = -1; p.comp = (int)in.size(); p.kind = atoi(argv[4]); p.max_def = atoi(argv[5]); p.num_values = atoi(argv[6]);
        p.encoding = atoi(argv[7]); p.width = atoi(argv[8]); p.def_len = atoi(argv[10]);
        const uint32_t dict_count = (uint32_t)atol(argv[9]), nv = (uint32_t)p.num_values;
        pq::Run* dr = (pq::Run*)malloc(sizeof(pq::Run) * (nv + 1));
        pq::Run* ir = (pq::Run*)malloc(sizeof(pq::Run) * (nv + 1));
        pq::Layout L;
        uint32_t dn = 0, dc = 0, in_ = 0, ic = 0, vi = 0, nvalid = 0;
        const uint8_t* is = nullptr; uint32_t isn = 0; int bw = 0;
        int e = pq::page_layout(p, ib, nullptr, &L);
        if (!e && p.max_def) e = pq::hybrid_walk(L.def, L.def_n, 1, nv, dr, nv + 1, &dn, &dc, pq::E_LEVELS);
        if (!e && pq::uses_index(p.encoding)) e = pq::index_stream(p, L, &is, &isn, &bw);
        if (!e && pq::uses_index(p.encoding)) e = pq::hybrid_walk(is, isn, bw, nv, ir, nv + 1, &in_, &ic, pq::E_INDEX);
        for (uint32_t k = 0; !e && k < nv; k++) {
            uint32_t d = 1;
            if (p.max_def) e = pq::hybrid_get(L.def, L.def_n, 1, dr, dn, dc, k, &d, pq::E_LEVELS);
            if (e || !d) continue;
            nvalid++;
            uint64_t x = 0;
            if (p.encoding == pq::ENC_PLAIN) e = pq::plain_get(L.val, L.val_n, p.width, vi, &x);
            else {
                uint32_t id = 0;
                e = pq::hybrid_get(is, isn, bw, ir, in_, ic, vi, &id, pq::E_INDEX);
                if (!e && id >= dict_count) e = pq::E_DICT_RANGE;
                if (!e) e = pq::plain_get(db, (uint32_t)dv.size(), p.width, id, &x);
            }
            vi++;
        }
        printf("%d %u\n", e, nvalid);
        free(dr); free(ir); free(db);
    } else {                   // hybrid <in> <bw> <need>
        const int bw = atoi(argv[3]);
        const uint32_t need = (uint32_t)atol(argv[4]);
        pq::Run* runs = (pq::Run*)malloc(sizeof(pq::Run) * (need + 1));
        uint32_t nr = 0, cover = 0;
        int e = pq::hybrid_walk(ib, (uint32_t)in.size(), bw, need, runs, need + 1, &nr, &cover, pq::E_LEVELS);
        printf("%d %u", e, cover);
        for (uint32_t k = 0; !e && k < cover; k++) {
            uint32_t v = 0;
            const int g = pq::hybrid_get(ib, (uint32_t)in.size(), bw, runs, nr, cover, k, &v, pq::E_LEVELS);
            if (g) { printf(" E%d", g); break; }
            printf(" %u", v);
        }
        printf("\n");
        free(runs);
    }
    free(ib);
    return 0;
}
"""


@pytest.fixture(scope="module")
def dec(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ is not installed")
    d = tmp_path_factory.mktemp("pqdec")
    (d / "drv.cpp").write_text(DRIVER)
    exe = str(d / "pqdec")
    subprocess.check_call([gxx, "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-I", CSRC, str(d / "drv.cpp"), "-o", exe])
    n = [0]

    def run(mode, data: bytes, *args):
        n[0] += 1
        src = d / f"in{n[0]}"
        src.write_bytes(data)
        out = d / f"out{n[0]}"
        if args and isinstance(args[0], bytes):   # a second input file (the dictionary page of the page mode)
            (d / f"aux{n[0]}").write_bytes(args[0])
            args = (d / f"aux{n[0]}",) + args[1:]
        r = subprocess.run([exe, mode, str(src), *map(str, args), str(out)], capture_output=True, text=True)
        assert r.returncode == 0 and "Sanitizer" not in r.stderr and "runtime error" not in r.stderr, r.stderr
        return r.stdout.split(), (out.read_bytes() if out.exists() else None)
    return run


E_SNAPPY, E_SNAPPY_SIZE, E_LEVELS = 1, 2, 3


@pytest.mark.parametrize("kind", ["random", "repetitive", "runs", "empty", "large"])
def test_snappy_against_pyarrow(dec, kind):
    rng = np.random.default_rng(len(kind))
    data = {"random": rng.bytes(70000), "repetitive": bytes(rng.integers(0, 4, 100000, dtype=np.uint8)),
            "runs": b"abcd" * 30000 + bytes(range(256)) * 50, "empty": b"",
            "large": np.repeat(rng.bytes(5000), 200).tobytes()}[kind]
    comp = pa.Codec("snappy").compress(data, asbytes=True)
    st, out = dec("s", comp, len(data))
    assert st == ["0"] and (out or b"") == data


def _lit(b: bytes) -> bytes:
    n = len(b) - 1
    if n < 60:
        return bytes([n << 2]) + b
    nb = (n.bit_length() + 7) // 8
    return bytes([(59 + nb) << 2]) + n.to_bytes(nb, "little") + b


def _pre(n: int) -> bytes:
    return bytes(H._varint_encode(n, None))


def test_snappy_tag_forms(dec):
    cases = [
        (_pre(10) + _lit(b"ab") + bytes([((8 - 4) << 2) | 1 | (0 << 5), 2]), b"ab" * 5),            # copy1, overlapping (offset 2 < 8)
        (_pre(7) + _lit(b"xyz") + bytes([(3 << 2) | 2, 3, 0]), b"xyzxyzx"),                          # copy2, overlapping
        (_pre(6) + _lit(b"abc") + bytes([(2 << 2) | 3, 3, 0, 0, 0]), b"abcabc"),                     # copy4 (4-byte offset)
        (_pre(300) + _lit(bytes(range(200)) + bytes(100)), bytes(range(200)) + bytes(100)),          # a literal with a 2-byte length
        (_pre(65) + _lit(b"q") + bytes([(63 << 2) | 2, 1, 0]) + bytes([(0 << 2) | 2, 1, 0]), b"q" * 66),
    ]
    for stream, want in cases[:4]:
        st, out = dec("s", stream, len(want))
        assert st == ["0"] and out == want, stream
    st, _ = dec("s", cases[4][0], 65)   # the last copy runs past the declared size
    assert st == [str(E_SNAPPY_SIZE)]


def test_snappy_corrupt(dec, tmp_path):
    good = _pre(6) + _lit(b"abc") + bytes([(2 << 2) | 2, 3, 0])
    assert dec("s", good, 6)[0] == ["0"]
    cases = {
        "truncated literal": (_pre(10) + bytes([9 << 2]) + b"abc", 10, E_SNAPPY),
        "offset 0": (_pre(6) + _lit(b"abc") + bytes([(2 << 2) | 2, 0, 0]), 6, E_SNAPPY),
        "before the start": (_pre(6) + _lit(b"abc") + bytes([(2 << 2) | 2, 4, 0]), 6, E_SNAPPY),
        "output overrun": (_pre(4) + _lit(b"abcdef"), 4, E_SNAPPY_SIZE),
        "length mismatch": (_pre(5) + _lit(b"abc"), 5, E_SNAPPY_SIZE),
        "header mismatch": (good, 7, E_SNAPPY_SIZE),
        "truncated copy": (_pre(6) + _lit(b"abc") + bytes([(2 << 2) | 3, 3]), 6, E_SNAPPY),
        "truncated preamble": (b"\x80", 1, E_SNAPPY),
    }
    for name, (stream, n, code) in cases.items():
        st, _ = dec("s", stream, n)
        assert st == [str(code)], name
    # the corrupted page of the GPU test's fixture: the same bytes the device reads
    comp, raw = H.snappy_fixture(str(tmp_path / "sn.parquet"))
    assert dec("s", comp, raw)[0] == [str(E_SNAPPY_SIZE)]


@pytest.mark.parametrize("bw", [0, 1, 3, 8, 13, 32])
def test_hybrid_streams(dec, bw):
    rng = np.random.default_rng(bw)
    vals = list(rng.integers(0, 1 << bw, 300, dtype=np.uint64)) if bw else [0] * 300
    runs = [("bp", 3), ("rle", 40), ("bp", 1), ("rle", 1), ("bp", 20), ("rle", 59)]
    i = 0
    for kind, n in runs:
        cnt = n if kind == "rle" else 8 * n
        if kind == "rle":
            vals[i:i + cnt] = [vals[i]] * cnt
        i += cnt
    total = i
    vals = vals[:total]
    s = H.hybrid_encode(vals, bw, runs)
    st, _ = dec("h", s, bw, total)
    assert st[0] == "0" and int(st[1]) == total
    assert [int(x) for x in st[2:]] == [int(v) for v in vals]
    # every truncation: an error or fewer values, never an access outside the stream
    for cut in range(0, len(s), max(1, len(s) // 40)):
        st, _ = dec("h", s[:cut], bw, total)
        assert st[0] in ("0", str(E_LEVELS)), cut
        if st[0] == "0":
            assert int(st[1]) < total or bw == 0
            assert [int(x) for x in st[2:]] == [int(v) for v in vals[:int(st[1])]]


def test_dictionary_pages_under_the_sanitizers(dec, tmp_path):
    """The data pages of the GPU test's patched-dictionary fixture (ids past the 70-value dictionary) and of the hand-built
    PLAIN_DICTIONARY column, decoded as the kernels decode them."""
    p = str(tmp_path / "di.parquet")
    H.dict_index_fixture(p)
    pages = H.chunk_pages(p)
    dh, dpage = pages[0]
    assert dh[1] == 2 and dh[7][1] == 70
    for h, data in pages[1:]:
        v2 = h[8]
        st, _ = dec("p", data, dpage, 1, 1, v2[1], v2[4], 8, dh[7][1], v2[5])
        assert st[0] == "5"   # E_DICT_RANGE
    # the same pages with the dictionary's true size decode without an error
    for h, data in pages[1:]:
        v2 = h[8]
        st, _ = dec("p", data, dpage, 1, 1, v2[1], v2[4], 8, 100, v2[5])
        assert st[0] == "0" and int(st[1]) == v2[1]
    q = str(tmp_path / "legacy.parquet")
    vals = H.legacy_file(q)
    pages = H.chunk_pages(q, len(H.LEGACY) - 1)
    (dh, dpage), (h, data) = pages
    st, _ = dec("p", data, dpage, 0, 1, h[5][1], h[5][2], 8, dh[7][1], 0)
    assert st == ["0", str(int(vals["c_dict"][1].sum()))]


def test_hybrid_bad_bit_width(dec):
    st, _ = dec("h", b"\x02\x01", 33, 1)
    assert st[0] == "8"
