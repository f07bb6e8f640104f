"""Arrow IPC files either side of the path (SURVEY 8(f) N4): DataFrame::from_arrow / to_arrow, src/dataframe.rs:391-407, 515-525.

The library maps the file and decodes the Arrow metadata itself (csrc/ipc.cu); this module is the ctypes face of it:

    f = IpcFile(path)                       # no GPU needed: schema, batches, zero-copy host views
    f.schema                                # [(name, dtype or -1, nullable)]
    cols = f.read(["a", "b"])               # -> {name: Column}, one chunk per RecordBatch, straight from the mapping
    write_ipc(path, {"c": col, "d": col2})  # device columns -> IPC file that any Arrow implementation reads
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Union

import numpy as np

from . import _native as N
from .arrays import NP_DTYPES, BooleanArray, PrimitiveArray, TemporalType

BOOL = 10


class IpcFile:
    def __init__(self, path: str):
        self.path = str(path)
        self.handle = C.c_void_p()
        N.raise_for_status(N.lib().bdf_ipc_open(self.path.encode(), C.byref(self.handle)))
        nc, nb, nr = C.c_int32(), C.c_int64(), C.c_int64()
        N.raise_for_status(N.lib().bdf_ipc_describe(self.handle, C.byref(nc), C.byref(nb), C.byref(nr)))
        self.num_columns, self.num_batches, self.num_rows = nc.value, nb.value, nr.value
        self.schema = []
        for i in range(self.num_columns):
            name, dt, nl = C.c_char_p(), C.c_int32(), C.c_int32()
            N.raise_for_status(N.lib().bdf_ipc_column(self.handle, i, C.byref(name), C.byref(dt), C.byref(nl)))
            self.schema.append((name.value.decode("utf-8", "replace"), dt.value, bool(nl.value)))
        # List<T> columns keep dtype -1 in `schema` (outside the column path); their BDF_LIST_BASE + T codes are here
        self.list_columns = {}
        for i in range(self.num_columns):
            ld = C.c_int32()
            N.raise_for_status(N.lib().bdf_ipc_list_column(self.handle, i, C.byref(ld)))
            if ld.value >= 0:
                self.list_columns[self.schema[i][0]] = ld.value
        # Date / Time / Timestamp columns also keep dtype -1 in `schema`; their types are here (read them by name)
        self.temporal_columns = {}
        for i in range(self.num_columns):
            tt = N.TemporalTypeC()
            N.raise_for_status(N.lib().bdf_ipc_temporal_column(self.handle, i, C.byref(tt)))
            if tt.kind:
                self.temporal_columns[self.schema[i][0]] = TemporalType(tt.kind, tt.unit, tt.tz.decode() if tt.tz else None)

    # -- lifetime --
    def close(self) -> None:
        if self.handle:
            N.lib().bdf_ipc_close(self.handle)
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

    def batch_rows(self, batch: int) -> int:
        r = C.c_int64()
        N.raise_for_status(N.lib().bdf_ipc_batch_rows(self.handle, batch, C.byref(r)))
        return r.value

    def view(self, batch: int, col: Union[int, str]):
        """Zero-copy host array over the mapping (valid until close()): PrimitiveArray or BooleanArray."""
        ci = self.column_index(col)
        v = N.View()
        N.raise_for_status(N.lib().bdf_ipc_view(self.handle, batch, ci, C.byref(v)))
        dtype = self.schema[ci][1]
        n = v.len
        nvb = (n + 7) // 8
        validity = None
        if v.validity:
            validity = np.ctypeslib.as_array(C.cast(v.validity, C.POINTER(C.c_uint8)), shape=(nvb,)) if nvb else np.zeros(0, np.uint8)
        if dtype == BOOL:
            vals = np.ctypeslib.as_array(C.cast(v.values, C.POINTER(C.c_uint8)), shape=(nvb,)) if nvb else np.zeros(0, np.uint8)
            return BooleanArray(vals, validity, 0, n, v.null_count, keepalive=self)
        npdt = np.dtype(NP_DTYPES[dtype])
        if n:
            raw = np.ctypeslib.as_array(C.cast(v.values, C.POINTER(C.c_uint8)), shape=(n * npdt.itemsize,))
            vals = raw.view(npdt)
        else:
            vals = np.zeros(0, npdt)
        return PrimitiveArray(dtype, vals, validity, 0, n, v.null_count, keepalive=self)

    # -- device --
    def read(self, columns: Optional[Sequence[Union[int, str]]] = None, ctx: Optional[N.Context] = None, asynchronous: bool = False,
             batches: Optional[Sequence[int]] = None) -> Dict[str, "object"]:
        """The chosen columns (default: every column of a type on the path) as device Columns, one chunk per RecordBatch.
        ``batches`` restricts the read to those RecordBatches (one rank's share: ``parallel.shard_indices``)."""
        from .functions import Column, ListColumn

        if columns is None:
            idx = [i for i, (_, dt, _) in enumerate(self.schema) if dt >= 0]
        else:
            idx = [self.column_index(c) for c in columns]
            temporal = [i for i in idx if self.schema[i][0] in self.temporal_columns]
            if temporal:   # Date / Time / Timestamp columns come back as tagged Columns of their physical dtype
                if batches is not None:
                    raise N.UnsupportedType("temporal columns are read whole (every RecordBatch)")
                ctx = ctx or N.default_context()
                rest = [i for i in idx if i not in temporal]
                res = self.read(rest, ctx, asynchronous) if rest else {}
                for i in temporal:
                    name = self.schema[i][0]
                    h = C.c_void_p()
                    N.raise_for_status(N.lib().bdf_ipc_read_temporal(ctx.handle, self.handle, i, N.ASYNC if asynchronous else 0, C.byref(h)))
                    col = Column(ctx, h, self.temporal_columns[name])
                    col._hold = self if asynchronous else None
                    res[name] = col
                return {self.schema[i][0]: res[self.schema[i][0]] for i in idx}
            lists = [i for i in idx if self.schema[i][0] in self.list_columns]
            if lists:   # List<T> columns come back as ListColumns, one chunk per RecordBatch
                if batches is not None:
                    raise N.UnsupportedType("list columns are read whole (every RecordBatch)")
                ctx = ctx or N.default_context()
                res = self.read([i for i in idx if i not in lists], ctx, asynchronous) if len(lists) < len(idx) else {}
                for i in lists:
                    h = C.c_void_p()
                    N.raise_for_status(N.lib().bdf_ipc_read_list(ctx.handle, self.handle, i, 0, C.byref(h)))
                    res[self.schema[i][0]] = ListColumn(ctx, h)
                return {self.schema[i][0]: res[self.schema[i][0]] for i in idx}
        if not idx:   # no column of a type on the path: an empty frame, not BDF_INVALID from the C side
            return {}
        ctx = ctx or N.default_context()
        arr = (C.c_int32 * len(idx))(*idx)
        outs = (C.c_void_p * len(idx))()
        flags = N.ASYNC if asynchronous else 0
        if batches is None:
            N.raise_for_status(N.lib().bdf_ipc_read(ctx.handle, self.handle, len(idx), arr, flags, outs))
        else:
            bl = list(batches)
            barr = (C.c_int64 * max(len(bl), 1))(*bl)
            N.raise_for_status(N.lib().bdf_ipc_read_batches(ctx.handle, self.handle, len(idx), arr, len(bl), barr, flags, outs))
        res = {}
        for i, h in zip(idx, outs):
            col = Column(ctx, C.c_void_p(h))
            col._hold = self if asynchronous else None   # the mapping must outlive the copies
            res[self.schema[i][0]] = col
        return res


def write_ipc_host(path: str, columns: Dict[str, List]) -> None:
    """Host chunks ([PrimitiveArray | BooleanArray] per column, chunk b of every column = RecordBatch b) -> IPC file."""
    names = list(columns)
    k = len(names)
    nb = len(columns[names[0]]) if k else 0
    cnames = (C.c_char_p * k)(*[s.encode() for s in names])
    dtypes = (C.c_int32 * k)(*[(columns[s][0].dtype if columns[s] else 9) for s in names])
    views = [N.make_views(columns[s]) for s in names]
    ptrs = (C.POINTER(N.View) * k)(*[C.cast(v, C.POINTER(N.View)) for v in views])
    for s in names:
        if len(columns[s]) != nb:
            raise N.ComputeError("columns have different numbers of chunks")
    N.raise_for_status(N.lib().bdf_ipc_write_host(str(path).encode(), k, cnames, dtypes, nb, ptrs))


def write_ipc(path: str, columns: Dict[str, "object"]) -> None:
    """Device Columns -> IPC file (DataFrame::to_arrow).  Columns tagged with a TemporalType are written as Date / Time / Timestamp
    fields (bdf_ipc_write_typed); ListColumns as List<item: T> fields (bdf_ipc_write_lists)."""
    from .functions import ListColumn

    names = list(columns)
    k = len(names)
    ctx = columns[names[0]].ctx
    cnames = (C.c_char_p * k)(*[s.encode() for s in names])
    is_list = [isinstance(columns[s], ListColumn) for s in names]
    handles = (C.c_void_p * k)(*[None if l else columns[s].handle for s, l in zip(names, is_list)])
    tags = [getattr(columns[s], "temporal", None) for s in names]
    if any(is_list):
        lists = (C.c_void_p * k)(*[columns[s].handle if l else None for s, l in zip(names, is_list)])
        types = (N.TemporalTypeC * k)(*[N.TemporalTypeC(t.kind, t.unit, t.tz.encode() if t.tz is not None else None) if t is not None
                                         else N.TemporalTypeC(0, 0, None) for t in tags])
        N.raise_for_status(N.lib().bdf_ipc_write_lists(ctx.handle, str(path).encode(), k, cnames, handles, types, lists))
        return
    if any(t is not None for t in tags):
        types = (N.TemporalTypeC * k)(*[N.TemporalTypeC(t.kind, t.unit, t.tz.encode() if t.tz is not None else None) if t is not None
                                         else N.TemporalTypeC(0, 0, None) for t in tags])
        N.raise_for_status(N.lib().bdf_ipc_write_typed(ctx.handle, str(path).encode(), k, cnames, handles, types))
        return
    N.raise_for_status(N.lib().bdf_ipc_write(ctx.handle, str(path).encode(), k, cnames, handles))
