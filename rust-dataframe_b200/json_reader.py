"""Line-delimited JSON files straight to the GPU: DataFrame::from_json (src/dataframe.rs) and LazyFrame::read(Json)
(src/evaluation.rs:329).

The library maps the file, uploads its bytes, finds and checks the records (one object per line), lists their members, resolves
the keys, infers the schema and converts the requested columns on the device (csrc/k_json.cu; the rules are in include/b200df.h):

    with JsonFile(path) as f:                # infer from every record, 1024 rows per batch
        f.schema                             # [(name, dtype or -1, nullable)]; List<T> columns are LIST_BASE + T
        cols = f.read(["id", "price"])       # -> {name: Column}, one chunk per RecordBatch
        tags = f.read_list("tags")           # -> ListColumn

and writes device columns back as line-delimited JSON, formatted on the device (csrc/k_json_write.cu):

    write_json(path, {"id": ids, "when": stamps, "tags": tags}, explicit_nulls=False)
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, Mapping, Optional, Sequence, Tuple, Union

from . import _native as N


class JsonFile:
    def __init__(self, path: str, schema: Optional[Sequence[Tuple[str, int]]] = None, max_records: Optional[int] = None,
                 batch_size: int = 1024, ctx: Optional[N.Context] = None):
        """``schema``: (name, dtype) pairs (0..9, BOOL, LIST_BASE + T, UTF8 or -1 to skip); None infers it from the first
        ``max_records`` records (None: all of them)."""
        self.ctx = ctx or N.default_context()
        self.path = str(path)
        opts = N.JsonOptions(-1 if max_records is None else int(max_records), int(batch_size))
        self.handle = C.c_void_p()
        if schema is None:
            st = N.lib().bdf_json_open(self.ctx.handle, self.path.encode(), C.byref(opts), 0, None, None, C.byref(self.handle))
        else:
            k = len(schema)
            names = (C.c_char_p * max(k, 1))(*[str(n).encode() for n, _ in schema])
            dts = (C.c_int32 * max(k, 1))(*[int(t) for _, t in schema])
            st = N.lib().bdf_json_open(self.ctx.handle, self.path.encode(), C.byref(opts), k, names, dts, C.byref(self.handle))
        N.raise_for_status(st)
        nc, nb, nr = C.c_int32(), C.c_int64(), C.c_int64()
        N.raise_for_status(N.lib().bdf_json_describe(self.handle, C.byref(nc), C.byref(nb), C.byref(nr)))
        self.num_columns, self.num_batches, self.num_rows = nc.value, nb.value, nr.value
        self.schema = []
        for i in range(self.num_columns):
            name, dt, nl = C.c_char_p(), C.c_int32(), C.c_int32()
            N.raise_for_status(N.lib().bdf_json_column(self.handle, i, C.byref(name), C.byref(dt), C.byref(nl)))
            self.schema.append((name.value.decode("utf-8", "replace"), dt.value, bool(nl.value)))

    # -- lifetime --
    def close(self) -> None:
        if self.handle:
            N.lib().bdf_json_close(self.ctx.handle, self.handle)
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
        """object members in the file, float values the last read rounded exactly on the host, host time of the upload."""
        nm, ex, ms = C.c_int64(), C.c_int64(), C.c_double()
        N.raise_for_status(N.lib().bdf_json_stats(self.handle, C.byref(nm), C.byref(ex), C.byref(ms)))
        return {"members": nm.value, "exact_fields": ex.value, "upload_ms": ms.value}

    # -- device --
    def read(self, columns: Optional[Sequence[Union[int, str]]] = None) -> Dict[str, "object"]:
        """The chosen numeric / Boolean columns (default: every one in the schema) as device Columns, one chunk per RecordBatch."""
        from .functions import Column

        if columns is None:
            idx = [i for i, (_, dt, _) in enumerate(self.schema) if 0 <= dt <= N.BOOL]
        else:
            idx = [self.column_index(c) for c in columns]
        k = len(idx)
        arr = (C.c_int32 * max(k, 1))(*idx)
        outs = (C.c_void_p * max(k, 1))()
        N.raise_for_status(N.lib().bdf_json_read(self.ctx.handle, self.handle, k, arr, outs))
        return {self.schema[i][0]: Column(self.ctx, C.c_void_p(outs[j])) for j, i in enumerate(idx)}

    def read_list(self, column: Union[int, str]) -> "object":
        """One List<T> column as a device ListColumn, one chunk per RecordBatch."""
        from .functions import ListColumn

        h = C.c_void_p()
        N.raise_for_status(N.lib().bdf_json_read_list(self.ctx.handle, self.handle, self.column_index(column), C.byref(h)))
        return ListColumn(self.ctx, h)


def write_json(path: str, columns: Mapping[str, "object"], explicit_nulls: bool = False) -> None:
    """Device Columns and ListColumns (chunk b of every column has the same row count) -> a line-delimited JSON file, one object per
    row, formatted on the device (bdf_json_write; the rules are in include/b200df.h).  Columns tagged with a TemporalType
    (``Column.temporal``) are written as date / time / timestamp strings.  A NULL member is left out unless ``explicit_nulls``; NaN and
    infinities are written as null."""
    from .functions import ListColumn

    names = list(columns)
    k = len(names)
    ctx = columns[names[0]].ctx if k else N.default_context()
    cnames = (C.c_char_p * max(k, 1))(*[s.encode() for s in names])
    is_list = [isinstance(columns[s], ListColumn) for s in names]
    handles = (C.c_void_p * max(k, 1))(*[None if l else columns[s].handle for s, l in zip(names, is_list)])
    lists = (C.c_void_p * max(k, 1))(*[columns[s].handle if l else None for s, l in zip(names, is_list)])
    tags = [None if l else getattr(columns[s], "temporal", None) for s, l in zip(names, is_list)]
    types = (N.TemporalTypeC * max(k, 1))(*[N.TemporalTypeC(t.kind, t.unit, t.tz.encode() if t.tz is not None else None) if t is not None
                                             else N.TemporalTypeC(0, 0, None) for t in tags])
    opts = N.JsonWriteOptions(1 if explicit_nulls else 0)
    N.raise_for_status(N.lib().bdf_json_write(ctx.handle, str(path).encode(), k, cnames, handles, types, lists, C.byref(opts)))
