"""The readers' and writer's number conversions on the host, against exact arithmetic: csrc/csv_parse.cuh (Eisel-Lemire and the
integer grammar, shared by from_csv and from_json) and csrc/csv_format.cuh (Schubfach, used by to_csv).

Both headers compile as plain C++ with __device__ defined empty; tests/conversion_harness.cpp wraps them for ctypes.  The float
references are tests/conversion_reference.py (exact rounding of the decimal value), numpy's shortest digits (csv_write_oracle),
glibc's strtof_l / strtod_l and exact integer comparisons inside the harness.  BDF_CONVERSION_CSRC points the build at another copy
of csrc/."""
import ctypes as C
import os
import shutil
import struct
import subprocess
import time
from fractions import Fraction

import numpy as np
import pytest

import conversion_reference as cr
import csv_oracle as co
import csv_write_oracle as wo

HERE = os.path.dirname(os.path.abspath(__file__))
OK, BAD, SLOW = 0, 1, 2
CHECKS = ["checked", "round trip", "digits", "shortest", "closest", "parse"]


class Harness:
    def __init__(self, path):
        self.lib = C.CDLL(path)
        i64p, u64p, i32p = C.POINTER(C.c_int64), C.POINTER(C.c_uint64), C.POINTER(C.c_int32)
        self.lib.h_parse_float.argtypes = [C.c_char_p, i64p, C.c_int64, C.c_int, u64p, i32p]
        self.lib.h_parse_int.argtypes = [C.c_char_p, i64p, C.c_int64, C.c_int, u64p, i32p]
        self.lib.h_format.argtypes = [u64p, C.c_int64, C.c_int, C.c_char_p, C.c_int64]
        self.lib.h_check_list.argtypes = [u64p, C.c_int64, C.c_int, C.c_int, i64p, u64p, C.c_int, C.POINTER(C.c_int)]
        self.lib.h_check_f32.argtypes = [C.c_uint32, C.c_int, i64p, u64p, C.c_int, C.POINTER(C.c_int)]
        self.lib.h_flog.argtypes = [C.c_int, C.c_int]
        self.lib.h_format_lines.argtypes = [u64p, C.c_int64, C.c_int, C.c_void_p, C.c_int64]
        self.lib.h_format_lines.restype = C.c_int64

    @staticmethod
    def _fields(strings):
        enc = [s.encode() if isinstance(s, str) else s for s in strings]
        off = np.zeros(len(enc) + 1, np.int64)
        off[1:] = np.cumsum([len(b) for b in enc])
        return b"".join(enc), off

    def parse_float(self, strings, width):
        """(bits, status) of every string."""
        buf, off = self._fields(strings)
        bits, st = np.zeros(len(strings), np.uint64), np.zeros(len(strings), np.int32)
        self.lib.h_parse_float(buf, off.ctypes.data_as(C.POINTER(C.c_int64)), len(strings), width,
                               bits.ctypes.data_as(C.POINTER(C.c_uint64)), st.ctypes.data_as(C.POINTER(C.c_int32)))
        return bits, st

    def parse_int(self, strings, dtype):
        buf, off = self._fields(strings)
        out, ok = np.zeros(len(strings), np.uint64), np.zeros(len(strings), np.int32)
        self.lib.h_parse_int(buf, off.ctypes.data_as(C.POINTER(C.c_int64)), len(strings), dtype,
                             out.ctypes.data_as(C.POINTER(C.c_uint64)), ok.ctypes.data_as(C.POINTER(C.c_int32)))
        return out, ok.astype(bool)

    def format(self, bits, width):
        bits = np.ascontiguousarray(bits, np.uint64)
        slot = 400
        buf = C.create_string_buffer(slot * len(bits))
        self.lib.h_format(bits.ctypes.data_as(C.POINTER(C.c_uint64)), len(bits), width, buf, slot)
        raw = buf.raw
        return [raw[i * slot:raw.index(b"\0", i * slot)].decode() for i in range(len(bits))]

    def format_lines(self, bits, width) -> bytes:
        """The writer's text of every pattern, one per line."""
        bits = np.ascontiguousarray(bits, np.uint64)
        cap = 400 * len(bits) + 400 if width == 64 else 64 * len(bits) + 400   # Float32 text is at most 47 bytes
        buf = np.empty(cap, np.uint8)
        n = self.lib.h_format_lines(bits.ctypes.data_as(C.POINTER(C.c_uint64)), len(bits), width, buf.ctypes.data, cap)
        assert n >= 0
        return buf[:n].tobytes()

    def _result(self, counts, bad, nb):
        c = dict(zip(CHECKS, counts.tolist()))
        c["first_bad"] = [(hex(int(bad[2 * i])), CHECKS[int(bad[2 * i + 1])]) for i in range(nb.value)]
        return c

    def check_list(self, bits, width):
        bits = np.ascontiguousarray(bits, np.uint64)
        counts, bad, nb = np.zeros(len(CHECKS), np.int64), np.zeros(16, np.uint64), C.c_int()
        self.lib.h_check_list(bits.ctypes.data_as(C.POINTER(C.c_uint64)), len(bits), width, os.cpu_count() or 1,
                              counts.ctypes.data_as(C.POINTER(C.c_int64)), bad.ctypes.data_as(C.POINTER(C.c_uint64)), 8, C.byref(nb))
        return self._result(counts, bad, nb)

    def check_f32(self, stride):
        counts, bad, nb = np.zeros(len(CHECKS), np.int64), np.zeros(16, np.uint64), C.c_int()
        self.lib.h_check_f32(stride, os.cpu_count() or 1, counts.ctypes.data_as(C.POINTER(C.c_int64)),
                             bad.ctypes.data_as(C.POINTER(C.c_uint64)), 8, C.byref(nb))
        return self._result(counts, bad, nb)


def build_harness(out_dir) -> Harness:
    """g++ over tests/conversion_harness.cpp and the headers of BDF_CONVERSION_CSRC (default: the package's csrc/)."""
    cxx = shutil.which("g++")
    if cxx is None:
        pytest.skip("g++ is not installed: the conversion headers cannot be compiled for the host")
    so = os.path.join(str(out_dir), "conversion_harness.so")
    subprocess.run([cxx, "-O2", "-std=c++17", "-D__device__=", "-I", cr.CSRC, "-shared", "-fPIC", "-pthread",
                    os.path.join(HERE, "conversion_harness.cpp"), "-o", so], check=True)
    return Harness(so)


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return build_harness(tmp_path_factory.mktemp("conversion_harness"))


@pytest.fixture(scope="module")
def corpus():
    return cr.parse_corpus()


def _f64_bits(s: str) -> int:
    return struct.unpack("<Q", struct.pack("<d", float(s)))[0]


def test_reference_agrees_with_python_float(corpus):
    """The exact Float64 rounding of the reference against Python's own correctly rounded float(), on every valid corpus string."""
    valid = [s for s in corpus if cr.lex(s) is not None]
    assert len(valid) > 100_000
    bad = [s for s in valid if cr.parse_bits(s, cr.F64) != _f64_bits(s)]
    assert bad == []
    # and Float32 against csv_oracle's independent Fraction rounding, on a sample
    bad32 = [s for s in valid[::37] if cr.parse_bits(s, cr.F32) != co.parse_float_bits(s.encode(), co.F32)]
    assert bad32 == []


@pytest.mark.parametrize("width", [64, 32])
def test_parse_corpus_exactly(harness, corpus, width):
    """Every corpus string in both widths: kFloatOk is the exact rounding bit for bit, kFloatBad is exactly the grammar's
    refusals, and kFloatSlow only where the reference says 19 digits (or the 128-bit product) cannot decide."""
    f = cr.FMTS[width]
    bits, st = harness.parse_float(corpus, width)
    wrong, bad_grammar, needless_slow, slow = [], [], [], 0
    for s, b, k in zip(corpus, bits.tolist(), st.tolist()):
        ref = cr.parse_bits(s, f)
        if (k == BAD) != (ref is None):
            bad_grammar.append((s, k))
        elif k == OK and b != ref:
            wrong.append((s, hex(b), hex(ref)))
        elif k == SLOW:
            slow += 1
            if not cr.undecidable(s, f):
                needless_slow.append(s)
    assert wrong == [], f"{len(wrong)} wrong: {wrong[:5]}"
    assert bad_grammar == [], bad_grammar[:5]
    assert needless_slow == [], f"{len(needless_slow)} slow without cause: {needless_slow[:5]}"
    assert slow > 1000   # the corpus does reach the exact fallback


@pytest.mark.parametrize("width", [64, 32])
def test_undecided_strings_are_reported_slow(harness, corpus, width):
    """The converse: a string whose first 19 digits and the next 19-digit value round apart is never decided by the fast path."""
    f = cr.FMTS[width]
    _, st = harness.parse_float(corpus, width)
    missed = []
    for s, k in zip(corpus, st.tolist()):
        x = cr.lex(s)
        if x is None:
            continue
        w, q, dropped = cr.leading19(x[1], x[2])
        if dropped and cr.round_exact(False, w, q, f) != cr.round_exact(False, w + 1, q, f) and k != SLOW:
            missed.append(s)
    assert missed == []


def test_shortest_round_trip_strings_never_go_slow(harness):
    """Strings of at most 17 significant digits lose nothing to w's 19 digits, so the fast path decides every one of them: a
    million of Python's Float64 reprs and 200 000 of numpy's Float32 shortest strings, read in both widths."""
    s64 = cr.random_shortest(1, 1_000_000, cr.F64)
    s32 = cr.random_shortest(2, 200_000, cr.F32)
    assert len(s64) > 990_000 and len(s32) > 190_000
    for strings in (s64, s32):
        for width in (64, 32):
            _, st = harness.parse_float(strings, width)
            assert int((st == SLOW).sum()) == 0, [s for s, k in zip(strings, st) if k == SLOW][:5]
            assert int((st == BAD).sum()) == 0
    bits, _ = harness.parse_float(s64, 64)
    assert np.array_equal(bits, np.array([float(s) for s in s64], np.float64).view(np.uint64))
    bits, _ = harness.parse_float(s32, 32)
    assert np.array_equal(bits.astype(np.uint32), np.array([np.float32(s) for s in s32], np.float32).view(np.uint32))
    sample = s64[:20_000]
    bits, _ = harness.parse_float(sample, 32)
    assert bits.tolist() == [cr.parse_bits(s, cr.F32) for s in sample]


def test_parse_int_at_every_limit(harness):
    """parse_int at each dtype's limits and one past them, signs, -0 for the unsigned types, and the grammar's refusals."""
    for dt in range(8):
        bits = 8 << (dt & 3)
        lo, hi = (0, (1 << bits) - 1) if dt >= co.U8 else (-(1 << (bits - 1)), (1 << (bits - 1)) - 1)
        cases = [str(x) for x in (lo - 1, lo, lo + 1, hi - 1, hi, hi + 1, 0, 2 ** 64 - 1, 2 ** 64, 2 ** 64 + 9, 10 ** 20)]
        cases += ["-0", "+0", "0", "+" + str(hi), "000" + str(hi), "-000" + str(abs(lo)), "", "+", "-", "1.0", " 1", "1 ", "0x1",
                  "1e2", "99999999999999999999999"]
        out, ok = harness.parse_int(cases, dt)
        for s, v, k in zip(cases, out.tolist(), ok.tolist()):
            want = co.parse_int(s.encode(), dt)
            assert k == (want is not None), (dt, s)
            if k:
                assert v == want % 2 ** 64, (dt, s)


def _floor_log(base: int, x: Fraction) -> int:
    """floor(log_base(x)) of a positive rational, exactly."""
    k = (x.numerator.bit_length() - x.denominator.bit_length()) * 1233 // 4096 if base == 10 else \
        x.numerator.bit_length() - x.denominator.bit_length()
    while Fraction(base) ** k > x:
        k -= 1
    while Fraction(base) ** (k + 1) <= x:
        k += 1
    return k


def test_formatter_logarithms_over_their_ranges(harness):
    """csvf_flog10pow2 / csvf_flog10tq over |q| <= 1200 and csvf_flog2pow10 over |e| <= 400, the ranges csv_format.cuh promises,
    against exact rational logarithms.  (The offset of csvf_flog10tq may move by about -9.6e8 .. +1.9e8 without changing one value
    in its range; a change that does is caught here and by the format tests.)"""
    for q in range(-1200, 1201):
        assert harness.lib.h_flog(0, q) == _floor_log(10, Fraction(2) ** q), q
        assert harness.lib.h_flog(1, q) == _floor_log(10, Fraction(3, 4) * Fraction(2) ** q), q
    for e in range(-400, 401):
        assert harness.lib.h_flog(2, e) == _floor_log(2, Fraction(10) ** e), e


@pytest.mark.parametrize("width", [64, 32])
def test_format_patterns_match_the_oracle(harness, width):
    """The writer's text of every power of two and its neighbours, every subnormal power of two, the powers of ten, the extremes
    and 20 000 random patterns, both signs, byte for byte against numpy's shortest digits; and that text checked exactly for
    shortest and closest on a sample."""
    f = cr.FMTS[width]
    pats = cr.format_patterns(3, f)
    got = harness.format(pats, width)
    np_t = np.float64 if width == 64 else np.float32
    vals = pats.view(np_t)
    want = [wo.format_float(v) for v in vals]
    diff = [(hex(int(b)), g, w) for b, g, w in zip(pats.tolist(), got, want) if g != w]
    assert diff == [], f"{len(diff)} differ: {diff[:5]}"
    step = 7 if width == 32 else 29
    bad = [(hex(int(b)), t) for b, t, v in zip(pats.tolist()[::step], got[::step], vals[::step])
           if np.isfinite(v) and v != 0 and not cr.shortest_closest_ok(t, int(b), f)]
    assert bad == []


@pytest.mark.parametrize("width", [64, 32])
def test_format_then_parse_is_identity_on_the_patterns(harness, width):
    """For the format corpus, the text reads back through glibc and through the library's own parser (never slow) to the
    same bits, and it is shortest and closest by exact integer comparison."""
    f = cr.FMTS[width]
    r = harness.check_list(cr.format_patterns(4, f), width)
    assert r["checked"] > 4000
    assert all(r[k] == 0 for k in CHECKS[1:]), r


def test_format_float64_random(harness):
    """Four million seeded Float64 patterns (NaNs dropped) through every check: glibc's strtod_l reads the text back to the bits,
    the digits are the shortest that do and the closest among those, and the library's parser reads them back without slowing."""
    rng = np.random.default_rng(5)
    pats = rng.integers(0, 1 << 64, 4_000_000, dtype=np.uint64)
    pats = pats[(pats & np.uint64(0x7FFFFFFFFFFFFFFF)) <= np.uint64(0x7FF0000000000000)]
    t0 = time.time()
    r = harness.check_list(pats, 64)
    print(f"Float64: {r['checked']} random patterns checked in {time.time() - t0:.1f} s")
    assert r["checked"] == len(pats)
    assert all(r[k] == 0 for k in CHECKS[1:]), r


def _f32_expected(stride: int) -> int:
    """Float32 patterns h_check_f32 visits: the non-NaN multiples of stride, and for stride > 1 the non-NaN boundary patterns of
    every exponent that are not multiples."""
    def multiples(lo, hi):   # multiples of stride in [lo, hi)
        return (hi - 1) // stride - (lo - 1) // stride if lo > 0 else (hi - 1) // stride + 1
    nan = [(0x7F800001, 0x80000000), (0xFF800001, 0x100000000)]
    n = multiples(0, 1 << 32) - sum(multiples(a, b) for a, b in nan)
    if stride > 1:
        j = np.concatenate([np.arange(4096), np.arange((1 << 23) - 4096, 1 << 23)]).astype(np.uint64)
        top = (np.arange(512, dtype=np.uint64) << np.uint64(23))[:, None]   # sign and exponent
        b = (top | j[None, :]).ravel()
        n += int(((b % np.uint64(stride) != 0) & ((b & np.uint64(0x7FFFFFFF)) <= np.uint64(0x7F800000))).sum())
    return n


def test_format_every_float32(harness):
    """Float32 formatting against exact checks: glibc's strtof_l reads the text back to the bits, no shorter decimal does, no
    neighbour with as many digits is closer, and the library's parser reads the text back without slowing.

    All 2^32 - 2 (2^23 - 1) patterns but the NaNs take about ten minutes on 8 cores (strtof_l on long positional text is the larger
    part), so by default the walk visits every 17th pattern plus the first and last 4096 patterns of every exponent of both signs:
    2.56e8 patterns in about 25 s on 8 cores.  BDF_CONVERSION_EXHAUSTIVE=1 walks all of them."""
    stride = 1 if os.environ.get("BDF_CONVERSION_EXHAUSTIVE") == "1" else 17
    t0 = time.time()
    r = harness.check_f32(stride)
    print(f"Float32 (stride {stride}): {r['checked']} patterns checked in {time.time() - t0:.1f} s")
    assert r["checked"] == _f32_expected(stride)
    if stride == 1:
        assert r["checked"] == 2 ** 32 - 2 * (2 ** 23 - 1)
    assert all(r[k] == 0 for k in CHECKS[1:]), r
