"""Host-side Arrow ``PrimitiveArray<T>`` stand-in used by the Python mirror of the reference API.

The reference passes ``Vec<&PrimitiveArray<T>>`` (one array per RecordBatch chunk, src/table.rs:114-123)
into ``ScalarFunctions`` / ``AggregateFunctions``.  This class keeps the same memory contract the C ABI
consumes (include/b200df.h ``bdf_view``): a values buffer, an optional LSB-first validity bitmap
(1 = valid), a logical ``offset`` that applies to both, ``len`` and a cached ``null_count``.
pyarrow arrays convert in both directions without copying the buffers.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence

import numpy as np

I8, I16, I32, I64, U8, U16, U32, U64, F32, F64 = range(10)
NP_DTYPES = [np.dtype(t) for t in (np.int8, np.int16, np.int32, np.int64, np.uint8, np.uint16, np.uint32, np.uint64,
                                   np.float32, np.float64)]
DTYPE_NAMES = ["Int8", "Int16", "Int32", "Int64", "UInt8", "UInt16", "UInt32", "UInt64", "Float32", "Float64"]
_NP_TO_DTYPE = {dt: i for i, dt in enumerate(NP_DTYPES)}


def dtype_of(np_dtype) -> int:
    return _NP_TO_DTYPE[np.dtype(np_dtype)]


def width_of(dtype: int) -> int:
    return NP_DTYPES[dtype].itemsize


def is_float(dtype: int) -> bool:
    return dtype in (F32, F64)


def pack_validity(mask: np.ndarray) -> np.ndarray:
    """bool mask (True = valid) -> Arrow bitmap bytes (LSB first), padded to whole bytes."""
    return np.packbits(np.asarray(mask, dtype=bool), bitorder="little")


DATE32, DATE64, TIMESTAMP, TIME32, TIME64 = range(1, 6)   # bdf_temporal_kind
_UNITS = {"s": 0, "ms": 1, "us": 2, "ns": 3}
_UNIT_NAMES = ["s", "ms", "us", "ns"]
_KIND_NAMES = {DATE32: "date32", DATE64: "date64", TIMESTAMP: "timestamp", TIME32: "time32", TIME64: "time64"}


class TemporalType:
    """bdf_temporal_type: the Arrow temporal type a column of physical Int32 / Int64 values carries (include/b200df.h "dates and
    timestamps").  ``unit`` is an arrow TimeUnit (0 = s .. 3 = ns, or "s" / "ms" / "us" / "ns"); ``tz`` only for timestamps."""

    __slots__ = ("kind", "unit", "tz")

    def __init__(self, kind: int, unit=0, tz: Optional[str] = None):
        self.kind = int(kind)
        self.unit = _UNITS[unit] if isinstance(unit, str) else int(unit)
        self.tz = tz

    @classmethod
    def date32(cls): return cls(DATE32)

    @classmethod
    def date64(cls): return cls(DATE64, "ms")

    @classmethod
    def timestamp(cls, unit="us", tz: Optional[str] = None): return cls(TIMESTAMP, unit, tz)

    @classmethod
    def time32(cls, unit="s"): return cls(TIME32, unit)

    @classmethod
    def time64(cls, unit="us"): return cls(TIME64, unit)

    @property
    def dtype(self) -> int:
        """The physical dtype of the values (Int32 for Date32 / Time32, else Int64)."""
        return I32 if self.kind in (DATE32, TIME32) else I64

    def to_arrow(self):
        import pyarrow as pa

        u = _UNIT_NAMES[self.unit] if 0 <= self.unit < 4 else "s"
        if self.kind == DATE32:
            return pa.date32()
        if self.kind == DATE64:
            return pa.date64()
        if self.kind == TIMESTAMP:
            return pa.timestamp(u, tz=self.tz)
        if self.kind == TIME32:
            return pa.time32(u)
        return pa.time64(u)

    @classmethod
    def from_arrow(cls, typ) -> Optional["TemporalType"]:
        """The TemporalType of a pyarrow DataType, or None for a type that is not Date / Time / Timestamp."""
        import pyarrow as pa

        if pa.types.is_date32(typ):
            return cls(DATE32)
        if pa.types.is_date64(typ):
            return cls(DATE64, "ms")
        if pa.types.is_timestamp(typ):
            return cls(TIMESTAMP, typ.unit, typ.tz)
        if pa.types.is_time32(typ):
            return cls(TIME32, typ.unit)
        if pa.types.is_time64(typ):
            return cls(TIME64, typ.unit)
        return None

    def __eq__(self, other) -> bool:
        return isinstance(other, TemporalType) and (self.kind, self.unit, self.tz) == (other.kind, other.unit, other.tz)

    def __hash__(self) -> int:
        return hash((self.kind, self.unit, self.tz))

    def __repr__(self) -> str:
        name = _KIND_NAMES.get(self.kind, str(self.kind))
        if self.kind == DATE32:
            return "TemporalType(date32)"
        tz = f", tz={self.tz!r}" if self.tz is not None else ""
        return f"TemporalType({name}, {_UNIT_NAMES[self.unit] if 0 <= self.unit < 4 else self.unit}{tz})"


class PrimitiveArray:
    """One chunk of a column: Arrow layout over numpy buffers.  ``temporal`` (a TemporalType or None) says that the Int32 / Int64
    values are dates, times or timestamps."""

    __slots__ = ("dtype", "values", "validity", "offset", "length", "null_count", "_keepalive", "temporal")

    def __init__(self, dtype: int, values: np.ndarray, validity: Optional[np.ndarray] = None, offset: int = 0,
                 length: Optional[int] = None, null_count: int = -1, keepalive=None):
        values = np.asarray(values)
        if values.dtype != NP_DTYPES[dtype]:
            raise TypeError(f"values dtype {values.dtype} does not match {DTYPE_NAMES[dtype]}")
        if not values.flags.c_contiguous:
            values = np.ascontiguousarray(values)
        self.dtype = dtype
        self.values = values
        self.validity = None if validity is None else np.ascontiguousarray(validity, dtype=np.uint8)
        self.offset = int(offset)
        self.length = int(values.shape[0] - offset if length is None else length)
        if self.offset < 0 or self.length < 0 or self.offset + self.length > values.shape[0]:
            raise ValueError("offset/length outside the values buffer")
        if self.validity is not None and self.validity.shape[0] * 8 < self.offset + self.length:
            raise ValueError("validity bitmap too short")
        self.null_count = 0 if self.validity is None else int(null_count)
        self._keepalive = keepalive
        self.temporal = None

    # ---- constructors ------------------------------------------------------------------------------
    @classmethod
    def from_numpy(cls, values: np.ndarray, mask: Optional[np.ndarray] = None) -> "PrimitiveArray":
        """mask: True = valid.  No bitmap is attached when mask is None (like a Vec<T> -> array)."""
        values = np.ascontiguousarray(values)
        dtype = dtype_of(values.dtype)
        if mask is None:
            return cls(dtype, values)
        mask = np.asarray(mask, dtype=bool)
        return cls(dtype, values, pack_validity(mask), 0, values.shape[0], int((~mask).sum()))

    @classmethod
    def from_pylist(cls, dtype: int, items: Iterable) -> "PrimitiveArray":
        """None entries become nulls (payload 0), like Arrow's From<Vec<Option<T>>>."""
        items = list(items)
        mask = np.array([x is not None for x in items], dtype=bool)
        vals = np.array([0 if x is None else x for x in items], dtype=NP_DTYPES[dtype])
        if mask.all():
            return cls(dtype, vals)
        return cls(dtype, vals, pack_validity(mask), 0, len(items), int((~mask).sum()))

    @classmethod
    def from_arrow(cls, arr) -> "PrimitiveArray":
        """Zero-copy view of a pyarrow primitive array (offset and validity preserved)."""
        import pyarrow as pa

        temporal = TemporalType.from_arrow(arr.type)
        np_dt = NP_DTYPES[temporal.dtype] if temporal is not None else np.dtype(arr.type.to_pandas_dtype())
        dtype = dtype_of(np_dt)
        vbuf, dbuf = arr.buffers()
        n_total = arr.offset + len(arr)
        values = (np.frombuffer(dbuf, dtype=np_dt, count=n_total) if dbuf is not None and n_total
                  else np.zeros(n_total, dtype=np_dt))
        validity = np.frombuffer(vbuf, dtype=np.uint8) if vbuf is not None else None
        out = cls(dtype, values, validity, arr.offset, len(arr), arr.null_count if vbuf is not None else 0, keepalive=arr)
        out.temporal = temporal
        return out

    def to_arrow(self):
        import pyarrow as pa

        typ = self.temporal.to_arrow() if self.temporal is not None else pa.from_numpy_dtype(NP_DTYPES[self.dtype])
        vbuf = pa.py_buffer(self.validity) if self.validity is not None else None
        return pa.Array.from_buffers(typ, self.length, [vbuf, pa.py_buffer(self.values)],
                                     null_count=self.null_count if self.validity is not None else 0,
                                     offset=self.offset)

    # ---- accessors (names follow arrow-rs) -----------------------------------------------------------
    def __len__(self) -> int:
        return self.length

    def len(self) -> int:
        return self.length

    def valid_mask(self) -> np.ndarray:
        if self.validity is None:
            return np.ones(self.length, dtype=bool)
        bits = np.unpackbits(self.validity, bitorder="little")
        return bits[self.offset:self.offset + self.length].astype(bool)

    def is_valid(self, i: int) -> bool:
        if self.validity is None:
            return True
        j = self.offset + i
        return bool((self.validity[j >> 3] >> (j & 7)) & 1)

    def is_null(self, i: int) -> bool:
        return not self.is_valid(i)

    def value(self, i: int):
        return self.values[self.offset + i]

    def value_slice(self) -> np.ndarray:
        return self.values[self.offset:self.offset + self.length]

    def compute_null_count(self) -> int:
        if self.validity is None:
            return 0
        if self.null_count < 0:
            self.null_count = int(self.length - self.valid_mask().sum())
        return self.null_count

    def slice(self, offset: int, length: int) -> "PrimitiveArray":
        """Zero-copy slice (ArrayData::slice): shares buffers, moves the offset."""
        if offset < 0 or length < 0 or offset + length > self.length:
            raise ValueError("slice out of bounds")
        out = PrimitiveArray(self.dtype, self.values, self.validity, self.offset + offset, length, -1, keepalive=self._keepalive)
        out.temporal = self.temporal
        return out

    def to_pylist(self) -> List:
        m = self.valid_mask()
        v = self.value_slice()
        return [v[i].item() if m[i] else None for i in range(self.length)]

    def __repr__(self) -> str:
        return f"PrimitiveArray<{DTYPE_NAMES[self.dtype]}>(len={self.length}, offset={self.offset}, nulls={self.null_count})"


class BooleanArray:
    """Arrow BooleanArray chunk: bit-packed values (LSB first) + optional validity; `offset` counts bits."""

    dtype = 10  # BDF_BOOL
    __slots__ = ("values", "validity", "offset", "length", "null_count", "_keepalive")

    def __init__(self, values: np.ndarray, validity: Optional[np.ndarray] = None, offset: int = 0, length: int = 0,
                 null_count: int = -1, keepalive=None):
        self._keepalive = keepalive    # e.g. the mapped IPC file the buffers point into
        self.values = np.ascontiguousarray(values, dtype=np.uint8)
        self.validity = None if validity is None else np.ascontiguousarray(validity, dtype=np.uint8)
        self.offset, self.length = int(offset), int(length)
        self.null_count = 0 if self.validity is None else int(null_count)

    @classmethod
    def from_numpy(cls, bits: np.ndarray, mask: Optional[np.ndarray] = None) -> "BooleanArray":
        bits = np.asarray(bits, dtype=bool)
        validity = None if mask is None else pack_validity(mask)
        return cls(pack_validity(bits), validity, 0, bits.shape[0], 0 if mask is None else int((~np.asarray(mask, bool)).sum()))

    def slice(self, offset: int, length: int) -> "BooleanArray":
        return BooleanArray(self.values, self.validity, self.offset + offset, length, -1, keepalive=self._keepalive)

    def value_bits(self) -> np.ndarray:
        return np.unpackbits(self.values, bitorder="little")[self.offset:self.offset + self.length].astype(bool)

    def valid_mask(self) -> np.ndarray:
        if self.validity is None:
            return np.ones(self.length, dtype=bool)
        return np.unpackbits(self.validity, bitorder="little")[self.offset:self.offset + self.length].astype(bool)

    def to_pylist(self) -> List:
        v, m = self.value_bits(), self.valid_mask()
        return [bool(v[i]) if m[i] else None for i in range(self.length)]

    def __len__(self) -> int:
        return self.length


def chunk_lengths(chunks: Sequence[PrimitiveArray]) -> List[int]:
    return [c.length for c in chunks]


class ListArray:
    """One chunk of an Arrow ``List<T>`` column (32-bit offsets, T one of the ten numeric types): the memory contract of
    ``bdf_list_view`` -- Int32 offsets and an optional list validity bitmap, both starting at ``offset``, over a child
    ``PrimitiveArray`` that the offsets index (from the child's own offset)."""

    __slots__ = ("dtype", "offsets", "validity", "offset", "length", "null_count", "values", "_keepalive")

    def __init__(self, dtype: int, offsets: np.ndarray, validity: Optional[np.ndarray], offset: int, length: int, null_count: int,
                 values: PrimitiveArray, keepalive=None):
        self.dtype = dtype
        self.offsets = np.ascontiguousarray(offsets, dtype=np.int32)
        self.validity = None if validity is None else np.ascontiguousarray(validity, dtype=np.uint8)
        self.offset = int(offset)
        self.length = int(length)
        if self.offsets.shape[0] < self.offset + self.length + 1:
            raise ValueError("offsets buffer too short")
        self.null_count = 0 if self.validity is None else int(null_count)
        self.values = values
        self._keepalive = keepalive

    @classmethod
    def from_pylist(cls, dtype: int, items: Iterable) -> "ListArray":
        """[[1, 2], None, [], [None, 3]]: None lists are null (spanning no element), None elements are null elements."""
        items = list(items)
        offsets = [0]
        flat: list = []
        for x in items:
            if x is not None:
                flat.extend(x)
            offsets.append(len(flat))
        mask = np.array([x is not None for x in items], dtype=bool)
        validity = None if mask.all() else pack_validity(mask)
        return cls(dtype, np.array(offsets, dtype=np.int32), validity, 0, len(items), int((~mask).sum()),
                   PrimitiveArray.from_pylist(dtype, flat))

    @classmethod
    def from_arrow(cls, arr) -> "ListArray":
        """Zero-copy view of a pyarrow ListArray (list offset, child offset and both validities preserved)."""
        import pyarrow as pa

        if not pa.types.is_list(arr.type):
            raise TypeError(f"{arr.type} is not a List with 32-bit offsets")
        child = PrimitiveArray.from_arrow(arr.values)
        bufs = arr.buffers()
        n_off = arr.offset + len(arr) + 1
        offsets = np.frombuffer(bufs[1], dtype=np.int32, count=n_off) if bufs[1] is not None else np.zeros(n_off, np.int32)
        validity = np.frombuffer(bufs[0], dtype=np.uint8) if bufs[0] is not None else None
        return cls(child.dtype, offsets, validity, arr.offset, len(arr), arr.null_count, child, keepalive=arr)

    def __len__(self) -> int:
        return self.length

    def valid_mask(self) -> np.ndarray:
        if self.validity is None:
            return np.ones(self.length, dtype=bool)
        bits = np.unpackbits(self.validity, bitorder="little")
        return bits[self.offset:self.offset + self.length].astype(bool)

    def to_pylist(self) -> list:
        """None for a null list; elements as numpy scalars of the child type, None for a null element."""
        vm = self.valid_mask()
        cm = self.values.valid_mask()
        vals = self.values.values[self.values.offset:self.values.offset + self.values.length]
        out = []
        for k in range(self.length):
            if not vm[k]:
                out.append(None)
                continue
            b, e = int(self.offsets[self.offset + k]), int(self.offsets[self.offset + k + 1])
            out.append([vals[i] if cm[i] else None for i in range(b, e)])
        return out
