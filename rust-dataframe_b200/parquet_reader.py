"""Parquet files straight to the GPU: DataFrame::from_parquet (src/dataframe.rs).

The library maps the file (or every file of a directory), reads the footers and page headers on the host, uploads the projected
column chunks still compressed, and decompresses and decodes them on the device (csrc/parquet.cu, csrc/k_parquet.cu; the rules are in
include/b200df.h):

    with ParquetFile(path) as f:             # 1024 rows per batch; each file starts a new batch
        f.schema                             # [(name, dtype or -1, nullable)]; temporal columns report their physical dtype
        f.temporal_columns                   # {name: TemporalType}
        cols = f.read(["id", "ts"])          # -> {name: Column}, one chunk per RecordBatch; temporal columns come back tagged
    write_parquet("out.parquet", cols, compression="snappy")   # encoded and compressed on the device (csrc/k_parquet_write.cu)
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Mapping, Optional, Sequence, Union

from . import _native as N
from .arrays import TemporalType


class ParquetFile:
    def __init__(self, path: str, batch_size: int = 1024):
        """Opening needs no GPU: the footers and page headers are read on the host."""
        self.path = str(path)
        opts = N.ParquetOptions(int(batch_size))
        self.handle = C.c_void_p()
        N.raise_for_status(N.lib().bdf_parquet_open(self.path.encode(), C.byref(opts), C.byref(self.handle)))
        nc, nb, nr = C.c_int32(), C.c_int64(), C.c_int64()
        N.raise_for_status(N.lib().bdf_parquet_describe(self.handle, C.byref(nc), C.byref(nb), C.byref(nr)))
        self.num_columns, self.num_batches, self.num_rows = nc.value, nb.value, nr.value
        self.schema = []
        self.temporal_columns: Dict[str, TemporalType] = {}
        for i in range(self.num_columns):
            name, dt, nl = C.c_char_p(), C.c_int32(), C.c_int32()
            N.raise_for_status(N.lib().bdf_parquet_column(self.handle, i, C.byref(name), C.byref(dt), C.byref(nl)))
            n = name.value.decode("utf-8", "replace")
            self.schema.append((n, dt.value, bool(nl.value)))
            tt = N.TemporalTypeC()
            N.raise_for_status(N.lib().bdf_parquet_temporal_column(self.handle, i, C.byref(tt)))
            if tt.kind:
                self.temporal_columns[n] = TemporalType(tt.kind, tt.unit, tt.tz.decode() if tt.tz else None)

    # -- lifetime --
    def close(self) -> None:
        if self.handle:
            N.lib().bdf_parquet_close(self.handle)
            self.handle = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- metadata --
    def column_index(self, col: Union[int, str]) -> int:
        if isinstance(col, int):
            return col
        for i, (name, _, _) in enumerate(self.schema):
            if name == col:
                return i
        raise KeyError(col)

    def check(self, column: Union[int, str]) -> None:
        """Raise what a read of the column would raise for every cause the host can detect (no GPU)."""
        N.raise_for_status(N.lib().bdf_parquet_check(self.handle, self.column_index(column)))

    def stats(self) -> dict:
        """Of the last read: pages decoded, compressed bytes uploaded, host time of the upload."""
        np_, ub, ms = C.c_int64(), C.c_int64(), C.c_double()
        N.raise_for_status(N.lib().bdf_parquet_stats(self.handle, C.byref(np_), C.byref(ub), C.byref(ms)))
        return {"pages": np_.value, "uploaded_bytes": ub.value, "upload_ms": ms.value}

    # -- device --
    def read(self, columns: Optional[Sequence[Union[int, str]]] = None, ctx: Optional[N.Context] = None) -> Dict[str, "object"]:
        """The chosen columns (default: every column on the device path) as device Columns, one chunk per RecordBatch; temporal
        columns come back tagged with their TemporalType."""
        from .functions import Column

        ctx = ctx or N.default_context()
        if columns is None:
            idx = [i for i, (_, dt, _) in enumerate(self.schema) if dt >= 0]
        else:
            idx = [self.column_index(c) for c in columns]
        k = len(idx)
        arr = (C.c_int32 * max(k, 1))(*idx)
        outs = (C.c_void_p * max(k, 1))()
        N.raise_for_status(N.lib().bdf_parquet_read(ctx.handle, self.handle, k, arr, outs))
        res = {}
        for j, i in enumerate(idx):
            name = self.schema[i][0]
            res[name] = Column(ctx, C.c_void_p(outs[j]), self.temporal_columns.get(name))
        return res


_CODECS = {"none": 0, "uncompressed": 0, "snappy": 1}


def write_parquet(path: str, columns: Mapping[str, "object"], compression: str = "none", dictionary: bool = True,
                  row_group_rows: int = 0) -> None:
    """Device Columns (chunk b of every column has the same length) -> a Parquet file, encoded and compressed on the device
    (bdf_parquet_write; the rules are in include/b200df.h).  One row group per chunk (row_group_rows = 0) or row_group_rows rows per
    row group; Date / Time / Timestamp columns are written as such from ``Column.temporal``."""
    if compression not in _CODECS:
        raise ValueError(f"compression is one of {sorted(_CODECS)}, not {compression!r}")
    from .functions import Column

    names = list(columns)
    for s in names:
        if not isinstance(columns[s], Column):
            raise N.UnsupportedType(f"column {s!r} is a {type(columns[s]).__name__}: only numeric, Boolean and temporal columns are written to Parquet")
    k = len(names)
    ctx = columns[names[0]].ctx if k else N.default_context()
    cnames = (C.c_char_p * max(k, 1))(*[s.encode() for s in names])
    handles = (C.c_void_p * max(k, 1))(*[columns[s].handle for s in names])
    tags = [getattr(columns[s], "temporal", None) for s in names]
    types = (N.TemporalTypeC * max(k, 1))(*[N.TemporalTypeC(t.kind, t.unit, t.tz.encode() if t.tz is not None else None) if t is not None
                                             else N.TemporalTypeC(0, 0, None) for t in tags])
    opts = N.ParquetWriteOptions(_CODECS[compression], 1 if dictionary else 0, int(row_group_rows))
    N.raise_for_status(N.lib().bdf_parquet_write(ctx.handle, str(path).encode(), k, cnames, handles, types, C.byref(opts)))
