"""Shared comparison helpers for the parity tests."""
from __future__ import annotations

import ctypes as C

import numpy as np


def pool_used(ctx) -> int:
    """Bytes of the device's default memory pool (every stream-ordered allocation of the library) now in use."""
    cu = C.CDLL("libcuda.so.1")
    dev, pool, used = C.c_int(), C.c_void_p(), C.c_uint64()
    assert cu.cuInit(0) == 0 and cu.cuDeviceGet(C.byref(dev), ctx.device) == 0
    assert cu.cuDeviceGetDefaultMemPool(C.byref(pool), dev) == 0
    assert cu.cuMemPoolGetAttribute(pool, 7, C.byref(used)) == 0   # CU_MEMPOOL_ATTR_USED_MEM_CURRENT
    return used.value


def ulp_distance(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """Units-in-the-last-place distance between float arrays of the same dtype (NaN == NaN -> 0)."""
    assert a.dtype == b.dtype
    it = np.int64 if a.dtype == np.float64 else np.int32
    ia, ib = a.view(it).astype(np.int64), b.view(it).astype(np.int64)
    sign = np.int64(np.iinfo(it).min)
    ia = np.where(ia < 0, sign - ia, ia)  # map to a monotonic integer line
    ib = np.where(ib < 0, sign - ib, ib)
    d = np.abs(ia - ib)
    both_nan = np.isnan(a) & np.isnan(b)
    one_nan = np.isnan(a) ^ np.isnan(b)
    d = np.where(both_nan, 0, d)
    d = np.where(one_nan, np.iinfo(np.int64).max, d)
    return d


def valid_mask_of(arr) -> np.ndarray:
    return arr.valid_mask()


def values_of(arr) -> np.ndarray:
    return arr.values[arr.offset:arr.offset + arr.length]


def assert_same_array(got, want, *, what="", exact=True, max_ulp=0, check_payload=True):
    """got: PrimitiveArray from the CUDA path; want: OracleArray.  Validity compared logically
    (bitmap presence is not observable through the reference API), values bit-exact or within max_ulp."""
    assert got.length == want.length, f"{what}: length {got.length} != {want.length}"
    gm, wm = valid_mask_of(got), valid_mask_of(want)
    bad = np.nonzero(gm != wm)[0]
    assert bad.size == 0, f"{what}: validity differs at {bad[:8]} (got {gm[bad[:8]]}, want {wm[bad[:8]]})"
    want_nulls = int((~wm).sum())
    got_nulls = got.null_count if got.validity is not None else 0
    assert got_nulls == want_nulls, f"{what}: null_count {got_nulls} != {want_nulls}"
    if want.validity is not None and want.null_count >= 0:
        assert want.null_count == want_nulls
    gv, wv = values_of(got), values_of(want)
    assert gv.dtype == wv.dtype, f"{what}: dtype {gv.dtype} != {wv.dtype}"
    sel = np.ones(got.length, dtype=bool) if check_payload else gm
    if exact:
        gb = gv.view(np.dtype(f"u{gv.dtype.itemsize}"))
        wb = wv.view(np.dtype(f"u{wv.dtype.itemsize}"))
        differ = gb != wb
        if gv.dtype.kind == "f":  # IEEE 754 leaves the sign/payload of a produced NaN open: x86 makes 0xFFF8.., the GPU 0x7FFF..
            differ &= ~(np.isnan(gv) & np.isnan(wv))
        bad = np.nonzero(differ & sel)[0]
        assert bad.size == 0, f"{what}: {bad.size} values differ, first at {bad[:5]}: got {gv[bad[:5]]}, want {wv[bad[:5]]}"
    else:
        d = ulp_distance(gv[gm], wv[gm])
        worst = int(d.max()) if d.size else 0
        assert worst <= max_ulp, f"{what}: max ulp distance {worst} > {max_ulp}"
    if got.validity is not None:  # padding bits beyond len must be zero
        nbits = got.validity.shape[0] * 8
        if got.offset == 0 and nbits > got.length:
            bits = np.unpackbits(got.validity[: (got.length + 7) // 8], bitorder="little")
            assert not bits[got.length:].any(), f"{what}: non-zero padding bits in the validity bitmap"


def random_mask(rng, n, null_frac):
    return rng.random(n) >= null_frac
