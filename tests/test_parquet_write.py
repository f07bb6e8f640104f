"""The Parquet writer's encoders (csrc/parquet_encode.cuh) compiled on the host with g++ and the address and undefined-behaviour
sanitizers, and checked against the reader's decoders (parquet_decode.cuh) and pyarrow's snappy codec: the fragment compressor on
random, repetitive, run-length, empty, 64 KiB and multi-fragment inputs; the bit-packed hybrid writer at several bit widths; the
statistics fold with its float rules; the Thrift footer's round trip through pyarrow is on the GPU side (test_parquet_write_gpu.py)."""
import os
import shutil
import struct
import subprocess

import numpy as np
import pyarrow as pa
import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "rust-dataframe_b200", "csrc")

DRIVER = r"""
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "parquet_encode.cuh"
static std::vector<uint8_t> slurp(const char* p) {
    FILE* f = fopen(p, "rb"); std::vector<uint8_t> v; int c;
    while ((c = fgetc(f)) != EOF) v.push_back((uint8_t)c);
    fclose(f); return v;
}
static uint8_t* exact(const std::vector<uint8_t>& v) {   // an exact-size heap copy, so that ASan sees any access past its end
    uint8_t* b = (uint8_t*)malloc(v.size() ? v.size() : 1);
    for (size_t i = 0; i < v.size(); i++) b[i] = v[i];
    return b;
}
int main(int argc, char** argv) {
    std::vector<uint8_t> in = slurp(argv[2]);
    uint8_t* ib = exact(in);
    const uint32_t n = (uint32_t)in.size();
    if (argv[1][0] == 'z') {   // snappy <in> <out>: one stream of fragments, then the reader's decoder over it
        uint32_t nf = (n + pq::kFragment - 1) / pq::kFragment, cap = 5;
        for (uint32_t f = 0; f < nf; f++) cap += pq::snappy_bound(n - f * pq::kFragment < pq::kFragment ? n - f * pq::kFragment : pq::kFragment);
        uint8_t* ob = (uint8_t*)malloc(cap);
        uint32_t* table = (uint32_t*)malloc(sizeof(uint32_t) * pq::kHashSize);
        uint32_t op = 0;
        if (!pq::put_uleb(ob, cap, &op, n)) return 2;
        for (uint32_t f = 0; f < nf; f++) {
            const uint32_t s = f * pq::kFragment, len = n - s < pq::kFragment ? n - s : pq::kFragment;
            uint32_t fl = 0;
            // the fragment's own worst-case slot, as on the device
            if (!pq::snappy_fragment(ib + s, len, ob + op, pq::snappy_bound(len), &fl, table)) return 3;
            op += fl;
        }
        uint8_t* cb = (uint8_t*)malloc(op ? op : 1);
        memcpy(cb, ob, op);
        uint8_t* db = (uint8_t*)malloc(n ? n : 1);
        const int e = pq::snappy_decode(cb, op, db, n);
        printf("%d %u %d\n", e, op, e == 0 && (n == 0 || memcmp(db, ib, n) == 0));
        FILE* o = fopen(argv[3], "wb"); fwrite(cb, 1, op, o); fclose(o);
        free(ob); free(cb); free(db); free(table);
    } else if (argv[1][0] == 'h') {   // hybrid <u32 values> <bw>: one bit-packed run, read back by the reader's run walk
        const int bw = atoi(argv[3]);
        const uint32_t cnt = n / 4;
        std::vector<uint32_t> v(cnt);
        memcpy(v.data(), ib, (size_t)cnt * 4);
        const uint32_t cap = pq::packed_header_len(cnt) + pq::packed_body_len(cnt, bw);
        std::vector<uint8_t> zero(cap, 0);
        uint8_t* ob = exact(zero);
        uint32_t op = 0;
        if (!pq::put_packed_run(v.data(), cnt, bw, ob, cap, &op) || op != cap) { printf("write failed\n"); return 0; }
        uint32_t small = 0;   // one byte short: refused
        uint8_t* sb = exact(std::vector<uint8_t>(cap - 1, 0));
        const bool refused = !pq::put_packed_run(v.data(), cnt, bw, sb, cap - 1, &small);
        pq::Run* runs = (pq::Run*)malloc(sizeof(pq::Run) * (cnt + 1));
        uint32_t nr = 0, cover = 0;
        int e = pq::hybrid_walk(ob, cap, bw, cnt, runs, cnt + 1, &nr, &cover, pq::E_LEVELS);
        uint32_t bad = 0;
        for (uint32_t k = 0; !e && k < cnt; k++) {
            uint32_t x = 0;
            e = pq::hybrid_get(ob, cap, bw, runs, nr, cover, k, &x, pq::E_LEVELS);
            if (x != v[k]) bad++;
        }
        // an RLE run of the first value, read back the same way
        std::vector<uint8_t> rz(pq::rle_run_len(cnt, bw), 0);
        uint8_t* rb = exact(rz);
        uint32_t rop = 0;
        const bool rok = pq::put_rle_run(rb, (uint32_t)rz.size(), &rop, cnt, cnt ? v[0] : 0, bw);
        uint32_t rnr = 0, rcover = 0, rbad = 0;
        int re = pq::hybrid_walk(rb, (uint32_t)rz.size(), bw, cnt, runs, cnt + 1, &rnr, &rcover, pq::E_LEVELS);
        for (uint32_t k = 0; !re && k < cnt; k++) {
            uint32_t x = 0;
            re = pq::hybrid_get(rb, (uint32_t)rz.size(), bw, runs, rnr, rcover, k, &x, pq::E_LEVELS);
            if (x != v[0]) rbad++;
        }
        printf("%d %u %u %d %d %d %u %d\n", e, cover, bad, refused ? 1 : 0, rok ? 1 : 0, re, rbad, pq::id_bit_width(cnt));
        free(ob); free(sb); free(rb); free(runs);
    } else {   // stats <u64 values> <ord> <width> <validity bytes, one per value>
        const int ord = atoi(argv[3]), width = atoi(argv[4]);
        std::vector<uint8_t> vm = slurp(argv[5]);
        const uint32_t cnt = n / 8;
        pq::Stats s = pq::stats_empty(), a = pq::stats_empty(), b = pq::stats_empty();
        for (uint32_t k = 0; k < cnt; k++) {
            uint64_t x;
            memcpy(&x, ib + 8 * k, 8);
            pq::stats_add(&s, ord, width, vm[k] != 0, x);
            pq::stats_add(k % 2 ? &a : &b, ord, width, vm[k] != 0, x);   // two halves merged give the same fold
        }
        pq::stats_merge(&a, b);
        const bool same = a.kmin == s.kmin && a.kmax == s.kmax && a.count == s.count && a.nulls == s.nulls;
        if (!s.count) printf("none %llu %d\n", s.nulls, same ? 1 : 0);
        else printf("%llu %llu %llu %d\n", (unsigned long long)pq::stat_value(ord, width, s.kmin, false),
                    (unsigned long long)pq::stat_value(ord, width, s.kmax, true), s.nulls, same ? 1 : 0);
    }
    free(ib);
    return 0;
}
"""

ORD_SIGNED, ORD_UNSIGNED, ORD_FLOAT, ORD_DOUBLE = range(4)


@pytest.fixture(scope="module")
def enc(tmp_path_factory):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("g++ is not installed")
    d = tmp_path_factory.mktemp("pqenc")
    (d / "drv.cpp").write_text(DRIVER)
    exe = str(d / "pqenc")
    subprocess.check_call([gxx, "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                           "-I", CSRC, str(d / "drv.cpp"), "-o", exe])
    n = [0]

    def run(mode, data: bytes, *args):
        n[0] += 1
        src, out = d / f"in{n[0]}", d / f"out{n[0]}"
        src.write_bytes(data)
        extra = []
        for a in args:
            if isinstance(a, bytes):
                p = d / f"aux{n[0]}"
                p.write_bytes(a)
                extra.append(str(p))
            else:
                extra.append(str(a))
        r = subprocess.run([exe, mode, str(src), *extra, str(out)], capture_output=True, text=True)
        assert r.returncode == 0 and "Sanitizer" not in r.stderr and "runtime error" not in r.stderr, r.stderr
        return r.stdout.split(), (out.read_bytes() if out.exists() else None)
    return run


def _inputs():
    rng = np.random.default_rng(7)
    K = 65536
    return {
        "empty": b"",
        "one": b"x",
        "random": rng.integers(0, 256, 100_000, dtype=np.uint8).tobytes(),
        "repetitive": (b"the quick brown fox jumps over the lazy dog " * 4000)[:150_000],
        "runs": np.repeat(rng.integers(0, 256, 300, dtype=np.uint8), 700).tobytes(),
        "zeros": bytes(200_000),
        "exact_64k": rng.integers(0, 4, K, dtype=np.uint8).tobytes(),
        "64k_minus_1": rng.integers(0, 4, K - 1, dtype=np.uint8).tobytes(),
        "64k_plus_1": rng.integers(0, 4, K + 1, dtype=np.uint8).tobytes(),
        "multi_fragment": np.arange(1_000_000, dtype=np.int64).tobytes()[: 5 * K + 123],
        "floats": np.round(rng.normal(size=50_000), 1).tobytes(),
    }


@pytest.mark.parametrize("name", list(_inputs()))
def test_snappy_round_trip(enc, name):
    data = _inputs()[name]
    out, comp = enc("z", data)
    assert out[0] == "0" and out[2] == "1", out   # the reader's own snappy_next loop gives the input back
    assert pa.Codec("snappy").decompress(comp, decompressed_size=len(data)).to_pybytes() == data
    frags = (len(data) + 65535) // 65536
    assert len(comp) <= 5 + sum(32 + f + f // 6 for f in [min(65536, len(data) - i * 65536) for i in range(frags)])
    if name in ("repetitive", "runs", "zeros"):
        assert len(comp) < len(data) / 10


def test_snappy_incompressible_within_bound(enc):
    data = np.random.default_rng(1).integers(0, 256, 3 * 65536 + 7, dtype=np.uint8).tobytes()
    out, comp = enc("z", data)
    assert out[0] == "0" and out[2] == "1"
    assert len(comp) <= 5 + 4 * 32 + len(data) + len(data) // 6


@pytest.mark.parametrize("bw", [1, 3, 8, 13, 32])
@pytest.mark.parametrize("count", [1, 7, 8, 9, 1000, 4099])
def test_hybrid_writer(enc, bw, count):
    rng = np.random.default_rng(bw * 1000 + count)
    hi = (1 << bw) if bw < 32 else (1 << 32)
    v = rng.integers(0, hi, count, dtype=np.uint64).astype(np.uint32)
    out, _ = enc("h", v.tobytes(), bw)
    e, cover, bad, refused, rok, re, rbad, idbw = map(int, out)
    assert (e, cover, bad) == (0, count, 0)
    assert refused == 1                      # one byte short of its size: the writer refuses
    assert (rok, re, rbad) == (1, 0, 0)
    assert idbw == max(1, int(np.ceil(np.log2(count)))) if count > 1 else idbw == 1


def _stats(enc, values: np.ndarray, valid, ord_, width):
    raw = values.view(f"u{values.dtype.itemsize}").astype(np.uint64)
    out, _ = enc("s", raw.tobytes(), ord_, width, bytes(np.asarray(valid, dtype=np.uint8)))
    assert out[-1] == "1"   # the fold of two halves merged equals the fold of the whole
    return out[:-1]


def test_stats_signed_and_unsigned(enc):
    v = np.array([5, -3, 7, -100, 2], dtype=np.int32)
    mn, mx, nulls = _stats(enc, v, [1, 1, 1, 0, 1], ORD_SIGNED, 4)
    assert (np.uint32(int(mn)).view(np.int32), np.uint32(int(mx)).view(np.int32), int(nulls)) == (-3, 7, 1)
    u = np.array([1, 0x80000001, 5], dtype=np.uint32)
    mn, mx, _ = _stats(enc, u, [1, 1, 1], ORD_UNSIGNED, 4)
    assert (int(mn), int(mx)) == (1, 0x80000001)
    mn, mx, _ = _stats(enc, u, [1, 1, 1], ORD_SIGNED, 4)   # the same bits in signed order
    assert (int(mn), int(mx)) == (0x80000001, 5)
    w = np.array([2 ** 63 + 5, 3], dtype=np.uint64)
    mn, mx, _ = _stats(enc, w, [1, 1], ORD_UNSIGNED, 8)
    assert (int(mn), int(mx)) == (3, 2 ** 63 + 5)
    b = np.array([1, 0, 1], dtype=np.uint8)
    mn, mx, _ = _stats(enc, b, [1, 1, 1], ORD_UNSIGNED, 1)
    assert (int(mn), int(mx)) == (0, 1)


def test_stats_floats(enc):
    d = np.array([np.nan, 1.5, -2.0, np.inf, np.nan], dtype=np.float64)
    mn, mx, _ = _stats(enc, d, [1] * 5, ORD_DOUBLE, 8)
    assert struct.unpack("<d", struct.pack("<Q", int(mn)))[0] == -2.0
    assert struct.unpack("<d", struct.pack("<Q", int(mx)))[0] == np.inf
    z = np.array([0.0, -0.0, 0.0], dtype=np.float64)   # a zero minimum is -0.0, a zero maximum +0.0
    mn, mx, _ = _stats(enc, z, [1] * 3, ORD_DOUBLE, 8)
    assert (int(mn), int(mx)) == (0x8000000000000000, 0)
    z = np.array([0.0], dtype=np.float64)
    mn, mx, _ = _stats(enc, z, [1], ORD_DOUBLE, 8)
    assert (int(mn), int(mx)) == (0x8000000000000000, 0)
    f = np.array([np.float32("nan"), -0.0, 3.0], dtype=np.float32)
    mn, mx, _ = _stats(enc, f, [1] * 3, ORD_FLOAT, 4)
    assert (int(mn), np.uint32(int(mx)).view(np.float32)) == (0x80000000, np.float32(3.0))
    f = np.array([-1.0, -0.0], dtype=np.float32)
    mn, mx, _ = _stats(enc, f, [1, 1], ORD_FLOAT, 4)
    assert (np.uint32(int(mn)).view(np.float32), int(mx)) == (np.float32(-1.0), 0)


def test_stats_without_min_max(enc):
    assert _stats(enc, np.array([1, 2, 3], dtype=np.int64), [0, 0, 0], ORD_SIGNED, 8) == ["none", "3"]
    assert _stats(enc, np.array([np.nan, np.nan], dtype=np.float64), [1, 1], ORD_DOUBLE, 8) == ["none", "0"]
    assert _stats(enc, np.array([np.nan], dtype=np.float32), [0], ORD_FLOAT, 4) == ["none", "1"]
