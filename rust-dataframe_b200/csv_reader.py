"""CSV files straight to and from the GPU: DataFrame::from_csv (src/dataframe.rs:349-389), LazyFrame::read(Csv) (src/evaluation.rs:328)
and DataFrame::to_csv (src/dataframe.rs:527-543).

The library maps the file, uploads its bytes, tokenizes them with csv-core's record DFA run as a scan, checks the field counts,
infers the schema and parses the requested columns on the device (csrc/k_csv.cu; the rules are in include/b200df.h):

    with CsvFile(path) as f:                 # arrow's defaults: header, ',', infer from every record, 1024 rows per batch
        f.schema                             # [(name, dtype or -1, nullable)]; Utf8 columns are -1 (not on the device path)
        cols = f.read(["lat", "lng"])        # -> {name: Column}, one chunk per RecordBatch
    write_csv("out.csv", cols)               # a header, ',', floats in their shortest round-trip digits (csrc/k_csv_write.cu)
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Mapping, Optional, Sequence, Union

from . import _native as N

UTF8 = N.UTF8


class CsvFile:
    def __init__(self, path: str, has_header: bool = True, delimiter: str = ",", max_records: Optional[int] = None, batch_size: int = 1024,
                 schema: Optional[Sequence[int]] = None, ctx: Optional[N.Context] = None):
        """``schema``: one dtype per column (0..9, BOOL, UTF8 or -1 to skip); None infers it from the first ``max_records`` data
        records (None: all of them)."""
        self.ctx = ctx or N.default_context()
        self.path = str(path)
        d = delimiter.encode() if isinstance(delimiter, str) else bytes(delimiter)
        if len(d) != 1:
            raise ValueError("the delimiter is one byte")
        opts = N.CsvOptions(1 if has_header else 0, d[0], -1 if max_records is None else int(max_records), int(batch_size))
        self.handle = C.c_void_p()
        if schema is None:
            st = N.lib().bdf_csv_open(self.ctx.handle, self.path.encode(), C.byref(opts), 0, None, C.byref(self.handle))
        else:
            arr = (C.c_int32 * max(len(schema), 1))(*[int(t) for t in schema])
            st = N.lib().bdf_csv_open(self.ctx.handle, self.path.encode(), C.byref(opts), len(schema), arr, C.byref(self.handle))
        N.raise_for_status(st)
        nc, nb, nr = C.c_int32(), C.c_int64(), C.c_int64()
        N.raise_for_status(N.lib().bdf_csv_describe(self.handle, C.byref(nc), C.byref(nb), C.byref(nr)))
        self.num_columns, self.num_batches, self.num_rows = nc.value, nb.value, nr.value
        self.schema = []
        for i in range(self.num_columns):
            name, dt, nl = C.c_char_p(), C.c_int32(), C.c_int32()
            N.raise_for_status(N.lib().bdf_csv_column(self.handle, i, C.byref(name), C.byref(dt), C.byref(nl)))
            self.schema.append((name.value.decode("utf-8", "replace"), dt.value, bool(nl.value)))

    # -- lifetime --
    def close(self) -> None:
        if self.handle:
            N.lib().bdf_csv_close(self.ctx.handle, self.handle)
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

    def stats(self) -> dict:
        """fields in the file, float fields the last read rounded exactly on the host, host time of the upload."""
        nf, ex, ms = C.c_int64(), C.c_int64(), C.c_double()
        N.raise_for_status(N.lib().bdf_csv_stats(self.handle, C.byref(nf), C.byref(ex), C.byref(ms)))
        return {"fields": nf.value, "exact_fields": ex.value, "upload_ms": ms.value}

    # -- device --
    def read(self, columns: Optional[Sequence[Union[int, str]]] = None) -> Dict[str, "object"]:
        """The chosen columns (default: every column of a type on the path) as device Columns, one chunk per RecordBatch."""
        from .functions import Column

        if columns is None:
            idx = [i for i, (_, dt, _) in enumerate(self.schema) if dt >= 0]
        else:
            idx = [self.column_index(c) for c in columns]
        k = len(idx)
        arr = (C.c_int32 * max(k, 1))(*idx)
        outs = (C.c_void_p * max(k, 1))()
        N.raise_for_status(N.lib().bdf_csv_read(self.ctx.handle, self.handle, k, arr, outs))
        return {self.schema[i][0]: Column(self.ctx, C.c_void_p(outs[j])) for j, i in enumerate(idx)}


def write_csv(path: str, columns: Mapping[str, "object"], has_header: bool = True, delimiter: str = ",") -> None:
    """Device Columns (chunk b of every column has the same length) -> a CSV file, formatted on the device (bdf_csv_write; the rules
    are in include/b200df.h).  ``delimiter`` may not be a byte that occurs in a value (a digit, '-', '.', quotes, line ends, letters
    of NaN / inf / true / false)."""
    d = delimiter.encode() if isinstance(delimiter, str) else bytes(delimiter)
    if len(d) != 1:
        raise ValueError("the delimiter is one byte")
    names = list(columns)
    k = len(names)
    ctx = columns[names[0]].ctx if k else N.default_context()
    cnames = (C.c_char_p * max(k, 1))(*[s.encode() for s in names])
    handles = (C.c_void_p * max(k, 1))(*[columns[s].handle for s in names])
    opts = N.CsvWriteOptions(1 if has_header else 0, d[0])
    N.raise_for_status(N.lib().bdf_csv_write(ctx.handle, str(path).encode(), k, cnames, handles, C.byref(opts)))
