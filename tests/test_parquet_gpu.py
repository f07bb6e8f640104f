"""DataFrame::from_parquet on the device against pyarrow.parquet: every value bit for bit, the same null slots, chunk lengths and bitmap
presence, over a matrix of files pyarrow writes at test time; projection, launch counts, the reference's CSV data, a frame operation,
and the device-detected errors."""
import ctypes as C
import os

import numpy as np
import pyarrow.compute as pc
import pyarrow.csv as pacsv
import pyarrow.parquet as pq
import pytest

import parquet_helpers as H
from helpers import pool_used

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "uk_cities_with_headers.csv")


@pytest.mark.parametrize("wid,kw", H.MATRIX, ids=[m[0] for m in H.MATRIX])
@pytest.mark.parametrize("null_frac", [0.0, 0.1])
def test_matrix(rdf, ctx, tmp_path, wid, kw, null_frac):
    p = str(tmp_path / "t.parquet")
    pq.write_table(H.table(5000, seed=len(wid), null_frac=null_frac), p, **kw)
    H.check_read(rdf, ctx, [p], p, 1024)


def test_all_null_and_required(rdf, ctx, tmp_path):
    p1, p2 = str(tmp_path / "n.parquet"), str(tmp_path / "r.parquet")
    pq.write_table(H.table(3000, seed=5, null_frac=1.0), p1)
    pq.write_table(H.required(H.table(3000, seed=6, null_frac=0.0)), p2, data_page_version="2.0")
    H.check_read(rdf, ctx, [p1], p1, 1024)
    H.check_read(rdf, ctx, [p2], p2, 1024)


@pytest.mark.parametrize("batch_size", [7, 1024, 1 << 20])
def test_batch_sizes_and_directory(rdf, ctx, tmp_path, batch_size):
    d = tmp_path / "dir"
    d.mkdir()
    paths = []
    for k, kw in enumerate([dict(row_group_size=700), dict(data_page_version="2.0", compression="none"), dict(row_group_size=2000)]):
        p = str(d / f"part-{k}.parquet")
        pq.write_table(H.table(2500 + 311 * k, seed=10 + k), p, **kw)
        paths.append(p)
    (d / "_SUCCESS").write_bytes(b"")
    (d / ".hidden").write_bytes(b"junk")
    pq.ParquetWriter(str(d / "zz-empty.parquet"), H.table(1, seed=1).schema).close()   # no row groups: skipped
    assert pq.ParquetFile(str(d / "zz-empty.parquet")).metadata.num_row_groups == 0
    H.check_read(rdf, ctx, paths, str(d), batch_size)


def test_projection_uploads_only_its_chunks(rdf, ctx, tmp_path):
    p = str(tmp_path / "t.parquet")
    pq.write_table(H.table(20000, seed=2), p, row_group_size=6000)
    md = pq.ParquetFile(p).metadata
    with rdf.ParquetFile(p) as f:
        for proj in (["i64"], ["f64", "b", "tsu"]):
            f.read(proj, ctx=ctx)
            idx = [md.schema.names.index(n) for n in proj]
            want = sum(md.row_group(g).column(i).total_compressed_size for g in range(md.num_row_groups) for i in idx)
            assert f.stats()["uploaded_bytes"] == want


def test_launch_count_is_fixed(rdf, ctx, tmp_path):
    one = str(tmp_path / "one.parquet")
    pq.write_table(H.table(3000, seed=1), one)
    d = tmp_path / "many"
    d.mkdir()
    for k in range(3):
        pq.write_table(H.table(3000, seed=k), str(d / f"{k}.parquet"), row_group_size=1200 if k else 3000)
    counts = []
    for path in (one, str(d)):
        ctx.profile_enable(True)
        ctx.profile_read()
        with rdf.ParquetFile(path) as f:
            f.read(["i32", "f64", "b"], ctx=ctx)
        recs = ctx.profile_read()
        ctx.profile_enable(False)
        counts.append(sum(1 for r in recs if r["kernel"] == "parquet"))
    assert counts[0] == counts[1] == 4


def test_reference_csv_data(rdf, ctx, tmp_path):
    p = str(tmp_path / "uk.parquet")
    pq.write_table(pacsv.read_csv(GOLDEN), p)
    a = rdf.DeviceFrame.from_parquet(p, ctx=ctx)
    b = rdf.DeviceFrame.from_csv(GOLDEN, ctx=ctx)
    assert list(a.columns) == list(b.columns)
    for n in a.columns:
        ga, va, la, _ = H.device_bits(a.columns[n])
        gb, vb, lb, _ = H.device_bits(b.columns[n])
        assert la == lb and np.array_equal(va, vb) and np.array_equal(ga[va], gb[vb]), n


def test_legacy_converted_types(rdf, ctx, tmp_path):
    p = str(tmp_path / "legacy.parquet")
    H.legacy_file(p, n=5000, seed=4)
    H.check_read(rdf, ctx, [p], p, 1024)


def test_sort_on_parquet_frame(rdf, ctx, tmp_path):
    """A stable sort with nulls last on a Parquet frame against pyarrow's sort_indices (stable, nulls at the end)."""
    p = str(tmp_path / "t.parquet")
    t = H.table(4000, seed=8, null_frac=0.1)
    pq.write_table(t, p, row_group_size=1500)
    fr = rdf.DeviceFrame.from_parquet(p, columns=["i16", "f64"], ctx=ctx)
    for name in ("i16", "f64"):
        idx = rdf.sort_indices([(fr.columns[name], False)])
        got = np.concatenate([np.asarray(a.value_slice()) for a in idx.download()])
        want = np.asarray(pc.sort_indices(t, sort_keys=[(name, "ascending")], null_placement="at_end"))
        assert np.array_equal(got, want), name


def test_device_detected_errors(rdf, ctx, tmp_path):
    for make, what in ((H.dict_index_fixture, "dictionary index"), (H.snappy_fixture, "decompressed size")):
        p = str(tmp_path / f"{what[:4]}.parquet")
        make(p)
        with rdf.ParquetFile(p) as f:
            f.check(0)   # nothing the host can see
            ctx.synchronize()
            before = pool_used(ctx)
            with pytest.raises(rdf.ComputeError, match=f"Parquet error in .*row group 0, column 0, page .*{what}"):
                f.read([0], ctx=ctx)
            ctx.synchronize()
            assert pool_used(ctx) == before


def test_multi_gpu_context_refused(rdf, tmp_path):
    p = str(tmp_path / "t.parquet")
    pq.write_table(H.table(100, seed=1), p)
    m = rdf.Context.multi(0)
    try:
        with rdf.ParquetFile(p) as f:
            with pytest.raises(rdf.UnsupportedType, match="one GPU"):
                f.read(["i32"], ctx=m)
    finally:
        m.close()
