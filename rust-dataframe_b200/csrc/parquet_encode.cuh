// parquet_encode.cuh -- the encoders of the Parquet writer (k_parquet_write.cu), written as __host__ __device__ functions in the style
// of parquet_decode.cuh, so that the CPU tests compile and run exactly this code (tests/test_parquet_write.py builds it with g++ and
// the sanitizers, and decodes what it writes with the reader's decoders).
//
// Every write is checked against the end of its output before it happens: a writer that would run past `cap` returns false and
// leaves *op where the last whole element ended.
#pragma once

#include <stdint.h>

#include "parquet_decode.cuh"

namespace pq {

// ---- ULEB128 and the RLE / bit-packed hybrid -------------------------------------------------------------------------------------
PQ_HD uint32_t uleb_len(uint64_t v) {
    uint32_t n = 1;
    while (v >= 0x80) { v >>= 7; n++; }
    return n;
}

PQ_HD bool put_uleb(uint8_t* out, uint32_t cap, uint32_t* op, uint64_t v) {
    if (uleb_len(v) > cap - *op) return false;
    while (v >= 0x80) { out[(*op)++] = (uint8_t)(v | 0x80); v >>= 7; }
    out[(*op)++] = (uint8_t)v;
    return true;
}

// An RLE run: `count` copies of v in bit width bw (the value takes ceil(bw / 8) bytes, little-endian).
PQ_HD uint32_t rle_run_len(uint32_t count, int bw) { return uleb_len((uint64_t)count << 1) + (uint32_t)(bw + 7) / 8; }
PQ_HD bool put_rle_run(uint8_t* out, uint32_t cap, uint32_t* op, uint32_t count, uint32_t v, int bw) {
    if (rle_run_len(count, bw) > cap - *op) return false;
    put_uleb(out, cap, op, (uint64_t)count << 1);
    for (int i = 0; i < (bw + 7) / 8; i++) out[(*op)++] = (uint8_t)(v >> (8 * i));
    return true;
}

// One bit-packed run of `count` values: its header (groups of 8 values) and its body (whole groups, zero padded).
PQ_HD uint32_t packed_header_len(uint32_t count) { return uleb_len((uint64_t)((count + 7) / 8) << 1 | 1); }
PQ_HD uint32_t packed_body_len(uint32_t count, int bw) { return (count + 7) / 8 * (uint32_t)bw; }
PQ_HD bool put_packed_header(uint8_t* out, uint32_t cap, uint32_t* op, uint32_t count) {
    return put_uleb(out, cap, op, (uint64_t)((count + 7) / 8) << 1 | 1);
}
// OR value k of bit width bw into a zeroed bit-packed body (LSB first).  The kernels do the same with atomicOr on 32-bit words.
PQ_HD void pack_value(uint8_t* body, uint32_t k, int bw, uint32_t v) {
    const uint64_t bit = (uint64_t)k * (uint64_t)bw;
    for (int i = 0; i < bw; i++)
        if ((v >> i) & 1) body[(bit + i) / 8] |= (uint8_t)(1u << ((bit + i) % 8));
}

// The serial writer of a whole hybrid stream as one bit-packed run (what the writer's id and level sections are): the header and
// the values packed in bit width bw (<= 32).  The body must be zero on entry.
PQ_HD bool put_packed_run(const uint32_t* v, uint32_t n, int bw, uint8_t* out, uint32_t cap, uint32_t* op) {
    if (!put_packed_header(out, cap, op, n)) return false;
    if (packed_body_len(n, bw) > cap - *op) return false;
    for (uint32_t k = 0; k < n; k++) pack_value(out + *op, k, bw, v[k]);
    *op += packed_body_len(n, bw);
    return true;
}

// Bit width of dictionary ids for n entries: max(1, ceil(log2 n)).
PQ_HD int id_bit_width(uint32_t n) {
    int bw = 1;
    while (bw < 32 && ((uint64_t)1 << bw) < n) bw++;
    return bw;
}

// ---- snappy ------------------------------------------------------------------------------------------------------------------------
// A page body is one snappy stream: the preamble (its length as a varint), then the elements of independently compressed fragments of
// kFragment bytes.  No copy reaches before the start of its fragment, which the format allows, so the fragments compress in parallel.
constexpr uint32_t kFragment = 65536;
constexpr int kHashBits = 12;
constexpr uint32_t kHashSize = 1u << kHashBits;
constexpr uint32_t kEmpty = 0xffffffffu;
constexpr int kWindow = 32;   // positions hashed together (one per lane of a warp)

PQ_HD uint32_t snappy_bound(uint32_t n) { return 32 + n + n / 6; }
PQ_HD uint32_t load32(const uint8_t* p) { return (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
PQ_HD uint32_t snappy_hash(uint32_t x) { return (x * 0x1e35a7bdu) >> (32 - kHashBits); }

// The tag of a literal of len (>= 1) bytes; the bytes themselves follow it.  False when tag and bytes do not fit.
PQ_HD bool snappy_literal_tag(uint32_t len, uint8_t* out, uint32_t cap, uint32_t* op) {
    const uint32_t m = len - 1;
    const uint32_t extra = m < 60 ? 0 : m < (1u << 8) ? 1 : m < (1u << 16) ? 2 : m < (1u << 24) ? 3 : 4;
    if ((uint64_t)1 + extra + len > (uint64_t)(cap - *op)) return false;
    if (!extra) { out[(*op)++] = (uint8_t)(m << 2); return true; }
    out[(*op)++] = (uint8_t)((59 + extra) << 2);
    for (uint32_t i = 0; i < extra; i++) out[(*op)++] = (uint8_t)(m >> (8 * i));
    return true;
}

// A copy of len (>= 4) bytes from off (1 .. 65535) bytes back, as copies of at most 64 bytes.
PQ_HD bool snappy_copy(uint32_t off, uint32_t len, uint8_t* out, uint32_t cap, uint32_t* op) {
    auto copy2 = [&](uint32_t l) {
        if (cap - *op < 3) return false;
        out[(*op)++] = (uint8_t)(2 | ((l - 1) << 2));
        out[(*op)++] = (uint8_t)off;
        out[(*op)++] = (uint8_t)(off >> 8);
        return true;
    };
    while (len >= 68) { if (!copy2(64)) return false; len -= 64; }
    if (len > 64) { if (!copy2(60)) return false; len -= 60; }
    if (len < 12 && off < 2048) {
        if (cap - *op < 2) return false;
        out[(*op)++] = (uint8_t)(1 | ((len - 4) << 2) | ((off >> 8) << 5));
        out[(*op)++] = (uint8_t)off;
        return true;
    }
    return copy2(len);
}

// Compress in[0, n) (n <= kFragment) as snappy elements, without a preamble.  The search is the warp's (k_pqw_snappy), done serially:
// at cursor ip, the positions ip .. ip + 31 (those with 4 bytes left) are hashed; each reads its candidate from the table as it was
// before this window, then every position is stored (for a slot several positions hash to, the last one); the first position whose
// candidate lies before it and holds the same 4 bytes starts a match, extended byte by byte.  Without one the cursor moves on 32.
// table: kHashSize entries of scratch.  Returns false when the output does not fit cap.
PQ_HD bool snappy_fragment(const uint8_t* in, uint32_t n, uint8_t* out, uint32_t cap, uint32_t* out_len, uint32_t* table) {
    for (uint32_t i = 0; i < kHashSize; i++) table[i] = kEmpty;
    uint32_t ip = 0, lit = 0, op = 0;
    while (ip + 4 <= n) {
        uint32_t cand[kWindow], h[kWindow];
        int m = 0;
        for (; m < kWindow && ip + m + 4 <= n; m++) {
            h[m] = snappy_hash(load32(in + ip + m));
            cand[m] = table[h[m]];
        }
        for (int l = 0; l < m; l++) table[h[l]] = ip + l;
        int f = -1;
        for (int l = 0; l < m && f < 0; l++)
            if (cand[l] < ip + l && load32(in + cand[l]) == load32(in + ip + l)) f = l;
        if (f < 0) { ip += kWindow; continue; }
        const uint32_t p = ip + f, c = cand[f];
        uint32_t len = 4;
        while (p + len < n && in[c + len] == in[p + len]) len++;
        if (p > lit) {
            if (!snappy_literal_tag(p - lit, out, cap, &op)) return false;
            for (uint32_t j = lit; j < p; j++) out[op++] = in[j];
        }
        if (!snappy_copy(p - c, len, out, cap, &op)) return false;
        ip = lit = p + len;
    }
    if (n > lit) {
        if (!snappy_literal_tag(n - lit, out, cap, &op)) return false;
        for (uint32_t j = lit; j < n; j++) out[op++] = in[j];
    }
    *out_len = op;
    return true;
}

// ---- values and statistics ----------------------------------------------------------------------------------------------------------
// How a column's value becomes its stored physical value (the input's raw bits, zero-extended to 64).
enum : int { CONV_NONE = 0, CONV_SEXT, CONV_MUL1000, CONV_DAYS };   // copy / zero-extend, sign-extend, x 1000, floor(ms / 86 400 000)
// The order statistics use: the logical type's.
enum : int { ORD_SIGNED = 0, ORD_UNSIGNED, ORD_FLOAT, ORD_DOUBLE };

// in_width: bytes of the input value; the result is the physical value's bits (its low 4 bytes for INT32 / FLOAT).
PQ_HD uint64_t convert(int conv, int in_width, uint64_t v) {
    const int sh = 64 - 8 * in_width;
    const int64_t s = in_width == 8 ? (int64_t)v : (int64_t)(v << sh) >> sh;   // sign-extended input
    switch (conv) {
        case CONV_SEXT: return (uint64_t)s;
        case CONV_MUL1000: return (uint64_t)s * 1000u;
        case CONV_DAYS: {
            const int64_t d = s / 86400000 - (s % 86400000 < 0 ? 1 : 0);
            return (uint64_t)d;
        }
        default: return v;
    }
}

// The order-preserving unsigned key of a physical value of `width` bytes (false: a NaN, which statistics skip).  Floats: -0.0 sorts
// just below +0.0.
PQ_HD bool stat_key(int ord, int width, uint64_t v, uint64_t* key) {
    if (width == 4) v &= 0xffffffffull;
    switch (ord) {
        case ORD_SIGNED: *key = (width == 4 ? (uint64_t)(int64_t)(int32_t)(uint32_t)v : v) ^ 0x8000000000000000ull; return true;
        case ORD_FLOAT: {
            const uint32_t f = (uint32_t)v;
            if ((f & 0x7fffffffu) > 0x7f800000u) return false;
            *key = (f & 0x80000000u) ? (uint64_t)(~f) : (uint64_t)(f | 0x80000000u);
            return true;
        }
        case ORD_DOUBLE: {
            if ((v & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) return false;
            *key = (v & 0x8000000000000000ull) ? ~v : (v | 0x8000000000000000ull);
            return true;
        }
        default: *key = v; return true;
    }
}

// The physical value of a key; a zero minimum is written -0.0 and a zero maximum +0.0 (the format's rule for floats).
PQ_HD uint64_t stat_value(int ord, int width, uint64_t key, bool is_max) {
    switch (ord) {
        case ORD_SIGNED: {
            const uint64_t v = key ^ 0x8000000000000000ull;
            return width == 4 ? (v & 0xffffffffull) : v;
        }
        case ORD_FLOAT: {
            const uint32_t k = (uint32_t)key;
            uint32_t f = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
            if ((f & 0x7fffffffu) == 0) f = is_max ? 0u : 0x80000000u;
            return f;
        }
        case ORD_DOUBLE: {
            uint64_t f = (key & 0x8000000000000000ull) ? (key & 0x7fffffffffffffffull) : ~key;
            if ((f & 0x7fffffffffffffffull) == 0) f = is_max ? 0ull : 0x8000000000000000ull;
            return f;
        }
        default: return key;
    }
}

// Statistics of a page or column chunk: the null count, and the keys of the smallest and largest valid non-NaN values (count of them).
struct Stats { unsigned long long kmin, kmax, count, nulls; };
PQ_HD Stats stats_empty() { return Stats{~0ull, 0ull, 0ull, 0ull}; }
PQ_HD void stats_add(Stats* s, int ord, int width, bool valid, uint64_t v) {
    uint64_t k;
    if (!valid) { s->nulls++; return; }
    if (!stat_key(ord, width, v, &k)) return;
    s->count++;
    if (k < s->kmin) s->kmin = k;
    if (k > s->kmax) s->kmax = k;
}
PQ_HD void stats_merge(Stats* s, const Stats& o) {
    s->nulls += o.nulls;
    s->count += o.count;
    if (o.kmin < s->kmin) s->kmin = o.kmin;
    if (o.kmax > s->kmax) s->kmax = o.kmax;
}

// ---- the writer's page table ------------------------------------------------------------------------------------------------------------
// A page of one block, built on the host (runtime.cu) in file order.  Offsets are bytes into the block's buffers.
struct WPage {
    long long slot;      // its body's slot in the raw buffer; the compressed body is compacted back to the same place
    long long frag0;     // its first fragment slot (snappy); fragment j at (frag0 + j) * snappy_bound(kFragment) in the fragment buffer
    int rows;            // rows (data page) or dictionary entries (dictionary page)
    int kind;            // KIND_V1 or KIND_DICT
    int id_bw;           // data page of a dictionary chunk: the ids' bit width; 0: PLAIN values
    int width;           // physical value bytes (0: Boolean, bit-packed)
    int in_width;        // input value bytes
    int conv, ord;       // CONV_*, ORD_*
    int n_frags;         // fragment slots (snappy; 0 for an uncompressed page)
    int tile0, n_tiles;  // its tiles in the block's tile table
};
// A tile: rows [first, first + rows) of a page, all from one source chunk (a column chunk, or the chunk's distinct values).
struct WTile {
    const void* values;          // the source's values at row 0 of the tile's chunk
    const uint32_t* validity;    // null: no nulls
    const uint32_t* ids;         // dictionary ids of the tile's rows (at its first row), null for PLAIN
    long long src_row;           // row of the tile's first row in the source
    int bit_off, val_bit_off;    // validity / Boolean value bit offsets of the source
    int page, first, rows, pad;
};
// What the kernels give back per page: its sizes, null count and statistics.
struct WPageOut {
    Stats st;
    unsigned int raw_len;    // uncompressed body bytes
    unsigned int comp_len;   // body bytes as written (= raw_len for an uncompressed page)
    unsigned int err;        // 1: a fragment did not fit its slot (cannot happen within the bound)
    unsigned int pad;
};
constexpr int kWTileRows = 2048;   // rows per tile: 256 threads x 8 consecutive rows

}  // namespace pq

#ifdef PQ_HOST_WRITE
#include <string>
#include <vector>

namespace pq {

// Thrift compact-protocol writer and the footer structures of the Parquet writer (parquet.cu).
struct WChunkMeta {
    int phys = 0, codec = 0;
    std::vector<int> encodings;
    long long num_values = 0, total_uncompressed = 0, total_compressed = 0, data_page_offset = 0, dict_page_offset = -1;
    bool has_stats = false, has_minmax = false;
    long long null_count = 0;
    std::string min_value, max_value;
};
struct WColumn {
    std::string name;
    int phys = 0;
    int converted = -1;          // ConvertedType, -1 none
    int logical = 0;             // LogicalType union member, 0 none: 6 DATE, 7 TIME, 8 TIMESTAMP, 10 INTEGER
    int int_bits = 0, int_signed = 1;
    int time_unit = 0;           // 1 MILLIS, 2 MICROS, 3 NANOS
    bool utc = false;
};
// A DATA_PAGE (V1, RLE levels) or DICTIONARY_PAGE header.
std::string page_header(int kind, int raw_len, int comp_len, int num_values, int encoding);
// The FileMetaData: version 1, the schema, the row groups and their column chunks, created_by, ARROW:schema, column orders.
std::string file_metadata(const std::vector<WColumn>& cols, const std::vector<long long>& rg_rows, const std::vector<std::vector<WChunkMeta>>& chunks,
                          const std::string& arrow_schema_b64);
std::string base64(const std::string& s);

}  // namespace pq
#endif
