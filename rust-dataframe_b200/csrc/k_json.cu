// k_json.cu -- line-delimited JSON straight to device columns (DataFrame::from_json, src/dataframe.rs; LazyFrame::read(Json),
// src/evaluation.rs:329).  The host side is runtime.cu (json_open / json_read / json_read_list); the grammar and the value rules
// are json_parse.cuh.
//
// A raw '\n' cannot occur inside a valid JSON string, so every '\n' ends a record and the records are found without any lexer
// state: the newline positions are compacted (count / scan / scatter, as the CSV field index), and every record is then walked by
// one thread.  Records of event and log data are short (tens to hundreds of bytes), so a warp walks 32 neighbouring lines and
// their bytes come through L1 together.
//   k_json_nl_count / k_json_nl_index   the '\n' positions: per-CTA counts, their scan (k_scan_one of k_scan.cu), the positions
//   k_json_lex          per line: blank, a record, or malformed (the first bad line by atomicMin); the members of its object; the
//                       exclusive 64-bit scans of these per-line counts (launch_scan) give the first member and the record of every line
//   k_json_members      per line again: one 32-byte entry per member (record, key bytes, value bytes, value class)
//   k_json_keys         the distinct keys: an open-addressing table on (hash, length) with the first member of each (atomicMin)
//   k_json_resolve      every member's key checked byte for byte against its table entry (a hash collision is reported, never
//                       trusted); its column from the host's dictionary; the slot (record, column) keeps the LAST member
//                       (atomicMax on the member index + 1), which is serde_json's last-wins for a key repeated in one object
//   k_json_infer        per (inferred record, column): the class bits of the slot's value (or "missing"), OR-ed per column
//   k_json_parse        (column, tile of 256 rows of one RecordBatch): the slot's value converted, as k_csv_parse: validity and
//                       Boolean words by warp ballot, valid counts per warp, floats the fast path cannot round on the exact list
//   k_json_list_count / k_json_list_fill   List<T>: the element count and list validity per row, then (after the scan of the
//                       counts) the offsets of every chunk from 0 and the elements converted into the child column
#include "common.cuh"
#include "json_parse.cuh"
#include "scan.cuh"

#include <algorithm>

namespace bdf {

constexpr int kJsonBytes = 16;                     // bytes per thread of the newline pass
constexpr int kJsonTile = kThreads * kJsonBytes;   // bytes per CTA
constexpr int kJsonRows = kThreads;                // rows per CTA of the parser

struct JsonMember {
    unsigned long long kstart, vstart;   // key bytes (inside the quotes) and value bytes, from the start of the text
    uint32_t klen, vlen;
    uint32_t rec;                        // the record (non-blank line) it belongs to
    uint16_t cls;                        // json::k* class of the value
    uint16_t escaped;                    // the key holds a backslash escape
};
static_assert(sizeof(JsonMember) == 32, "JsonMember layout");

struct JsonKey {   // one distinct raw key
    unsigned long long hash;    // ~0: empty
    unsigned long long first;   // its first member
    unsigned long long kstart;  // the first member's key bytes
    uint32_t klen, rec;         // and its record
};
static_assert(sizeof(JsonKey) == 32, "JsonKey layout");

struct JsonColDesc {   // as CsvColDesc
    char* values;
    long long vstride;
    uint32_t* validity;
    long long bstride;
    uint32_t* warp_counts;
    int dtype;
    int file_col;
};

struct JsonSlow {   // as CsvSlow: a float the fast path could not round
    long long start, end;
    int col, pad;
    long long chunk, row;
};

struct JsonListChunk {   // where list chunk i goes
    int32_t* offsets;
    uint32_t* validity;
    char* values;
    uint32_t* value_validity;
};

__device__ __forceinline__ void line_span(const unsigned long long* __restrict__ nl, long long n_nl, long long n, long long i, long long* s, long long* e) {
    *s = i > 0 ? (long long)nl[i - 1] + 1 : 0;
    *e = i < n_nl ? (long long)nl[i] : n;
}

__device__ __forceinline__ uint32_t nl_mask(const uint8_t* __restrict__ text, long long n, long long g) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(text) + g);   // the buffer is padded to whole tiles
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
    const long long off = g * kJsonBytes;
    const int cnt = off >= n ? 0 : (int)(n - off < kJsonBytes ? n - off : kJsonBytes);
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < kJsonBytes; k++)
        if (k < cnt && (uint8_t)(w[k >> 2] >> (8 * (k & 3))) == '\n') m |= 1u << k;
    return m;
}

__global__ void __launch_bounds__(kThreads) k_json_nl_count(const uint8_t* __restrict__ text, long long n, unsigned long long* __restrict__ counts) {
    const int total = cta_sum(__popc(nl_mask(text, n, (long long)blockIdx.x * kThreads + threadIdx.x)));
    if (threadIdx.x == 0) counts[blockIdx.x] = (unsigned long long)total;
}

__global__ void __launch_bounds__(kThreads)
k_json_nl_index(const uint8_t* __restrict__ text, long long n, const unsigned long long* __restrict__ offsets, unsigned long long* __restrict__ nl) {
    const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
    uint32_t m = nl_mask(text, n, g);
    unsigned long long off = offsets[blockIdx.x] + (unsigned long long)cta_exclusive_sum(__popc(m));
    while (m) {
        const int k = __ffs(m) - 1;
        m &= m - 1;
        nl[off++] = (unsigned long long)(g * kJsonBytes + k);
    }
}

struct CountMembers {
    unsigned long long n = 0;
    __device__ void member(const uint8_t*, const uint8_t*, const uint8_t*, const uint8_t*, int, bool) { n++; }
};

__global__ void __launch_bounds__(kThreads)
k_json_lex(const uint8_t* __restrict__ text, long long n, const unsigned long long* __restrict__ nl, long long n_nl, unsigned long long* __restrict__ members,
           unsigned long long* __restrict__ is_rec, unsigned long long* __restrict__ bad) {
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i <= n_nl; i += (long long)gridDim.x * kThreads) {
        long long s, e;
        line_span(nl, n_nl, n, i, &s, &e);
        json::Cursor c{text + s, text + e, 0, nullptr};
        CountMembers v;
        const int r = json::record(c, v);
        if (r == json::kBad) atomicMin(bad, (unsigned long long)i);
        members[i] = v.n;
        is_rec[i] = r == json::kRecord ? 1ull : 0ull;
    }
}

struct EmitMembers {
    const uint8_t* text;
    JsonMember* out;
    uint32_t rec;
    __device__ void member(const uint8_t* k0, const uint8_t* k1, const uint8_t* v0, const uint8_t* v1, int cls, bool esc) {
        *out++ = JsonMember{(unsigned long long)(k0 - text), (unsigned long long)(v0 - text), (uint32_t)(k1 - k0), (uint32_t)(v1 - v0), rec,
                            (uint16_t)cls, (uint16_t)(esc ? 1 : 0)};
    }
};

__global__ void __launch_bounds__(kThreads)
k_json_members(const uint8_t* __restrict__ text, long long n, const unsigned long long* __restrict__ nl, long long n_nl,
               const unsigned long long* __restrict__ first_member, const unsigned long long* __restrict__ rec_of, JsonMember* __restrict__ out) {
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i <= n_nl; i += (long long)gridDim.x * kThreads) {
        long long s, e;
        line_span(nl, n_nl, n, i, &s, &e);
        json::Cursor c{text + s, text + e, 0, nullptr};
        EmitMembers v{text, out + first_member[i], (uint32_t)rec_of[i]};
        json::record(c, v);
    }
}

__device__ __forceinline__ unsigned key_home(unsigned long long h, unsigned cap) { return (unsigned)(h ^ (h >> 32)) & (cap - 1); }

__global__ void __launch_bounds__(kThreads)
k_json_keys(const uint8_t* __restrict__ text, const JsonMember* __restrict__ m, long long n_members, JsonKey* __restrict__ table, unsigned cap,
            unsigned int* __restrict__ full) {
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n_members; i += (long long)gridDim.x * kThreads) {
        const JsonMember x = m[i];
        const unsigned long long h = json::key_hash(text + x.kstart, text + x.kstart + x.klen);
        unsigned s = key_home(h, cap);
        bool done = false;
        for (unsigned probe = 0; probe < cap && !done; probe++, s = (s + 1) & (cap - 1)) {
            unsigned long long cur = *(volatile unsigned long long*)&table[s].hash;
            if (cur == ~0ull) cur = atomicCAS(&table[s].hash, ~0ull, h);
            if (cur == ~0ull || cur == h) {
                if (*(volatile unsigned long long*)&table[s].first > (unsigned long long)i) atomicMin(&table[s].first, (unsigned long long)i);
                done = true;
            }
        }
        if (!done) atomicOr(full, 1u);
    }
}

__global__ void __launch_bounds__(kThreads) k_json_key_gather(JsonKey* __restrict__ table, unsigned cap, const JsonMember* __restrict__ m) {
    const unsigned s = blockIdx.x * kThreads + threadIdx.x;
    if (s >= cap || table[s].hash == ~0ull) return;
    const JsonMember x = m[table[s].first];
    table[s].kstart = x.kstart;
    table[s].klen = x.klen;
    table[s].rec = x.rec;
}

__global__ void __launch_bounds__(kThreads)
k_json_resolve(const uint8_t* __restrict__ text, const JsonMember* __restrict__ m, long long n_members, const JsonKey* __restrict__ table, unsigned cap,
               const int* __restrict__ col_of, int n_cols, unsigned int* __restrict__ slots, unsigned int* __restrict__ collision) {
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n_members; i += (long long)gridDim.x * kThreads) {
        const JsonMember x = m[i];
        const uint8_t* k = text + x.kstart;
        const unsigned long long h = json::key_hash(k, k + x.klen);
        unsigned s = key_home(h, cap);
        for (unsigned probe = 0; probe < cap && table[s].hash != h; probe++) s = (s + 1) & (cap - 1);
        const JsonKey e = table[s];
        bool same = e.hash == h && e.klen == x.klen;
        for (uint32_t j = 0; same && j < x.klen; j++) same = k[j] == text[e.kstart + j];
        if (!same) { atomicOr(collision, 1u); continue; }
        const int col = col_of[s];
        if (col >= 0) atomicMax(&slots[(unsigned long long)x.rec * n_cols + col], (unsigned int)(i + 1));
    }
}

__global__ void __launch_bounds__(kThreads)
k_json_infer(const JsonMember* __restrict__ m, const unsigned int* __restrict__ slots, long long n_slots, int n_cols, unsigned int* __restrict__ col_bits) {
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n_slots; i += (long long)gridDim.x * kThreads) {
        const unsigned int s = slots[i];
        const unsigned int bit = s ? (unsigned int)m[s - 1].cls : (unsigned int)json::kMissing;
        unsigned int* slot = col_bits + (i % n_cols);
        if ((*(volatile unsigned int*)slot & bit) != bit) atomicOr(slot, bit);
    }
}

__device__ __forceinline__ void put(char* dst, long long i, int dtype, uint64_t v) {
    switch (dtype_width(dtype)) {
        case 1: reinterpret_cast<uint8_t*>(dst)[i] = (uint8_t)v; break;
        case 2: reinterpret_cast<uint16_t*>(dst)[i] = (uint16_t)v; break;
        case 4: reinterpret_cast<uint32_t*>(dst)[i] = (uint32_t)v; break;
        default: reinterpret_cast<uint64_t*>(dst)[i] = v; break;
    }
}

// __maxnreg__ rather than __launch_bounds__: under the latter ptxas keeps 32 registers and spills around the float path
__global__ void __maxnreg__(64)
k_json_parse(const uint8_t* __restrict__ text, const JsonMember* __restrict__ m, const unsigned int* __restrict__ slots, int n_file_cols,
             const JsonColDesc* __restrict__ cols, long long n_rows, long long batch, long long tiles_per_chunk, JsonSlow* __restrict__ slow,
             unsigned long long* __restrict__ n_slow, long long slow_cap) {
    const int p = blockIdx.y;
    const JsonColDesc d = cols[p];
    const long long chunk = blockIdx.x / (unsigned)tiles_per_chunk, tt = blockIdx.x % (unsigned)tiles_per_chunk;   // 32-bit: no division call
    const long long row = tt * kJsonRows + threadIdx.x;
    const long long clen = min(batch, n_rows - chunk * batch);
    bool valid = false, bval = false;
    if (row < clen) {
        const unsigned int s = slots[(unsigned long long)(chunk * batch + row) * n_file_cols + d.file_col];
        uint64_t bits = 0;
        int r = json::kConvNull;
        long long vs = 0, ve = 0;
        if (s) {
            const JsonMember x = m[s - 1];
            vs = (long long)x.vstart;
            ve = vs + x.vlen;
            r = json::convert(text + vs, text + ve, d.dtype, &bits);
        }
        char* dst = d.values + chunk * d.vstride;
        valid = r != json::kConvNull;
        if (r == json::kConvSlow) {
            const unsigned long long k = atomicAdd(n_slow, 1ull);
            if ((long long)k < slow_cap) slow[k] = JsonSlow{vs, ve, p, 0, chunk, row};
        } else if (d.dtype == 10) {
            bval = valid && bits;
        } else {
            put(dst, row, d.dtype, valid ? bits : 0);   // a NULL slot is zeroed, so a read is deterministic
        }
    }
    const unsigned vw = __ballot_sync(0xffffffffu, valid), bw = __ballot_sync(0xffffffffu, bval);
    const long long row0 = row - (threadIdx.x & 31);
    if ((threadIdx.x & 31) == 0 && row0 < clen) {
        d.validity[(chunk * d.bstride) / 4 + (row0 >> 5)] = vw;
        if (d.dtype == 10) reinterpret_cast<uint32_t*>(d.values + chunk * d.vstride)[row0 >> 5] = bw;
    }
    if ((threadIdx.x & 31) == 0 && tt * kJsonRows < clen)
        d.warp_counts[(chunk * tiles_per_chunk + tt) * kWarpsPerCta + (threadIdx.x >> 5)] = (uint32_t)__popc(vw);
}

// The value of a List<T> cell: an array (its elements), a bare number (one element), anything else a NULL list (-1).
struct CountElems {
    __device__ void operator()(int64_t, const uint8_t*, const uint8_t*) {}
};

__device__ __forceinline__ long long list_len(const uint8_t* __restrict__ text, const JsonMember* __restrict__ m, unsigned int s) {
    if (!s) return -1;
    const JsonMember x = m[s - 1];
    const uint8_t* v = text + x.vstart;
    if (*v == '[') {
        CountElems f;
        return (long long)json::elements(v, v + x.vlen, f);
    }
    return (*v == '-' || json::is_digit(*v)) ? 1 : -1;
}

__global__ void __launch_bounds__(kThreads)
k_json_list_count(const uint8_t* __restrict__ text, const JsonMember* __restrict__ m, const unsigned int* __restrict__ slots, int n_file_cols, int file_col,
                  long long n_rows, long long batch, long long tiles_per_chunk, unsigned long long* __restrict__ counts, uint32_t* __restrict__ valid_words,
                  unsigned long long* __restrict__ chunk_nulls) {
    const long long chunk = blockIdx.x / (unsigned)tiles_per_chunk, tt = blockIdx.x % (unsigned)tiles_per_chunk;   // 32-bit: no division call
    const long long row = tt * kJsonRows + threadIdx.x;
    const long long clen = min(batch, n_rows - chunk * batch);
    bool valid = false;
    if (row < clen) {
        const long long r = chunk * batch + row;
        const long long len = list_len(text, m, slots[(unsigned long long)r * n_file_cols + file_col]);
        valid = len >= 0;
        counts[r] = valid ? (unsigned long long)len : 0ull;
    }
    const unsigned vw = __ballot_sync(0xffffffffu, valid);
    const long long row0 = row - (threadIdx.x & 31);
    if ((threadIdx.x & 31) == 0 && row0 < clen) {
        valid_words[chunk * ((batch + 31) / 32) + (row0 >> 5)] = vw;
        const int in = (int)min(32LL, clen - row0);
        if (in - __popc(vw)) atomicAdd(&chunk_nulls[chunk], (unsigned long long)(in - __popc(vw)));
    }
}

struct FillElems {
    char* values;
    uint32_t* value_validity;
    int dtype;
    long long base;   // the row's first element in its chunk
    long long chunk;
    unsigned long long nulls;
    JsonSlow* slow;
    unsigned long long* n_slow;
    long long slow_cap;
    const uint8_t* text;
    __device__ void operator()(int64_t i, const uint8_t* s, const uint8_t* e) {
        const long long k = base + i;
        uint64_t bits = 0;
        const int r = json::convert(s, e, dtype, &bits);
        if (r == json::kConvSlow) {
            const unsigned long long j = atomicAdd(n_slow, 1ull);
            if ((long long)j < slow_cap) slow[j] = JsonSlow{(long long)(s - text), (long long)(e - text), 0, 0, chunk, k};
        } else {
            put(values, k, dtype, r == json::kConvOk ? bits : 0);
        }
        if (r != json::kConvNull) atomicOr(&value_validity[k >> 5], 1u << (k & 31));
        else nulls++;
    }
};

__global__ void __maxnreg__(80)   // as k_json_parse
k_json_list_fill(const uint8_t* __restrict__ text, const JsonMember* __restrict__ m, const unsigned int* __restrict__ slots, int n_file_cols, int file_col,
                 int dtype, long long n_rows, long long batch, long long tiles_per_chunk, const unsigned long long* __restrict__ offs,
                 const uint32_t* __restrict__ valid_words, const JsonListChunk* __restrict__ out, unsigned long long* __restrict__ elem_nulls,
                 JsonSlow* __restrict__ slow, unsigned long long* __restrict__ n_slow, long long slow_cap) {
    const long long chunk = blockIdx.x / (unsigned)tiles_per_chunk, tt = blockIdx.x % (unsigned)tiles_per_chunk;   // 32-bit: no division call
    const long long row = tt * kJsonRows + threadIdx.x;
    const long long clen = min(batch, n_rows - chunk * batch);
    const JsonListChunk o = out[chunk];
    if (row < clen) {
        const long long r = chunk * batch + row;
        const unsigned long long o0 = offs[chunk * batch];
        const long long base = (long long)(offs[r] - o0);
        o.offsets[row + 1] = (int32_t)(offs[r + 1] - o0);
        if (row == 0) o.offsets[0] = 0;
        if ((row & 31) == 0) o.validity[row >> 5] = valid_words[chunk * ((batch + 31) / 32) + (row >> 5)];
        const unsigned int s = slots[(unsigned long long)r * n_file_cols + file_col];
        if (offs[r + 1] > offs[r]) {   // a valid list with elements
            const JsonMember x = m[s - 1];
            const uint8_t* v = text + x.vstart;
            FillElems f{o.values, o.value_validity, dtype, base, chunk, 0, slow, n_slow, slow_cap, text};
            if (*v == '[') json::elements(v, v + x.vlen, f);
            else f(0, v, v + x.vlen);
            if (f.nulls) atomicAdd(&elem_nulls[chunk], f.nulls);
        }
    }
}

__global__ void __launch_bounds__(kThreads)
k_json_bounds(const unsigned long long* __restrict__ offs, long long n_rows, long long batch, long long n_chunks, unsigned long long* __restrict__ out) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i <= n_chunks) out[i] = offs[min(i * batch, n_rows)];
}

// ---- launchers ------------------------------------------------------------------------------------------------------
int json_tile_bytes() { return kJsonTile; }
int json_parse_rows() { return kJsonRows; }
size_t json_member_bytes() { return sizeof(JsonMember); }
size_t json_key_bytes() { return sizeof(JsonKey); }
size_t json_desc_bytes() { return sizeof(JsonColDesc); }
size_t json_slow_bytes() { return sizeof(JsonSlow); }
size_t json_list_chunk_bytes() { return sizeof(JsonListChunk); }

static unsigned grid_for(long long items, int sm_count) {
    return (unsigned)std::max<long long>(1, std::min<long long>((items + kThreads - 1) / kThreads, (long long)sm_count * 16));
}

// text: padded to whole tiles.  counts: n_tiles + 1 entries; *n_nl (counts[n_tiles]) = the number of '\n'.
cudaError_t launch_json_nl_count(const uint8_t* text, long long n, unsigned long long* counts, cudaStream_t s) {
    const long long tiles = std::max<long long>((n + kJsonTile - 1) / kJsonTile, 1);
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidValue;
    k_json_nl_count<<<(unsigned)tiles, kThreads, 0, s>>>(text, n, counts);
    return launch_scan_one(counts, tiles, counts + tiles, s);   // its error check covers the launch above
}

cudaError_t launch_json_nl_index(const uint8_t* text, long long n, const unsigned long long* offsets, unsigned long long* nl, cudaStream_t s) {
    const long long tiles = std::max<long long>((n + kJsonTile - 1) / kJsonTile, 1);
    k_json_nl_index<<<(unsigned)tiles, kThreads, 0, s>>>(text, n, offsets, nl);
    return cudaGetLastError();
}

cudaError_t launch_json_lex(const uint8_t* text, long long n, const unsigned long long* nl, long long n_nl, unsigned long long* members,
                            unsigned long long* is_rec, unsigned long long* bad, int sm_count, cudaStream_t s) {
    k_json_lex<<<grid_for(n_nl + 1, sm_count), kThreads, 0, s>>>(text, n, nl, n_nl, members, is_rec, bad);
    return cudaGetLastError();
}

cudaError_t launch_json_members(const uint8_t* text, long long n, const unsigned long long* nl, long long n_nl, const unsigned long long* first_member,
                                const unsigned long long* rec_of, void* members, int sm_count, cudaStream_t s) {
    k_json_members<<<grid_for(n_nl + 1, sm_count), kThreads, 0, s>>>(text, n, nl, n_nl, first_member, rec_of, (JsonMember*)members);
    return cudaGetLastError();
}

// table: cap entries (a power of two), filled with 0xff bytes beforehand.
cudaError_t launch_json_keys(const uint8_t* text, const void* members, long long n_members, void* table, unsigned cap, unsigned int* full, int sm_count,
                             cudaStream_t s) {
    if (n_members > 0) k_json_keys<<<grid_for(n_members, sm_count), kThreads, 0, s>>>(text, (const JsonMember*)members, n_members, (JsonKey*)table, cap, full);
    k_json_key_gather<<<(cap + kThreads - 1) / kThreads, kThreads, 0, s>>>((JsonKey*)table, cap, (const JsonMember*)members);
    return cudaGetLastError();
}

cudaError_t launch_json_resolve(const uint8_t* text, const void* members, long long n_members, const void* table, unsigned cap, const int* col_of, int n_cols,
                                unsigned int* slots, unsigned int* collision, int sm_count, cudaStream_t s) {
    if (n_members <= 0) return cudaSuccess;
    k_json_resolve<<<grid_for(n_members, sm_count), kThreads, 0, s>>>(text, (const JsonMember*)members, n_members, (const JsonKey*)table, cap, col_of, n_cols,
                                                                      slots, collision);
    return cudaGetLastError();
}

cudaError_t launch_json_infer(const void* members, const unsigned int* slots, long long n_slots, int n_cols, unsigned int* col_bits, int sm_count, cudaStream_t s) {
    if (n_slots <= 0) return cudaSuccess;
    k_json_infer<<<grid_for(n_slots, sm_count), kThreads, 0, s>>>((const JsonMember*)members, slots, n_slots, n_cols, col_bits);
    return cudaGetLastError();
}

cudaError_t launch_json_parse(const uint8_t* text, const void* members, const unsigned int* slots, int n_file_cols, const void* cols, int n_cols, long long n_rows,
                              long long batch, void* slow, unsigned long long* n_slow, long long slow_cap, cudaStream_t s) {
    if (n_rows <= 0 || n_cols <= 0) return cudaSuccess;
    const long long tpc = (batch + kJsonRows - 1) / kJsonRows;
    const long long tiles = (n_rows + batch - 1) / batch * tpc;
    if (tiles > 0x7fffffffLL || n_cols > 65535) return cudaErrorInvalidValue;
    k_json_parse<<<dim3((unsigned)tiles, (unsigned)n_cols), kThreads, 0, s>>>(text, (const JsonMember*)members, slots, n_file_cols, (const JsonColDesc*)cols,
                                                                              n_rows, batch, tpc, (JsonSlow*)slow, n_slow, slow_cap);
    return cudaGetLastError();
}

// counts: n_rows + 1 entries (the scan runs in place afterwards); valid_words: n_chunks * ceil(batch / 32); chunk_nulls: n_chunks, zeroed.
cudaError_t launch_json_list_count(const uint8_t* text, const void* members, const unsigned int* slots, int n_file_cols, int file_col, long long n_rows,
                                   long long batch, unsigned long long* counts, uint32_t* valid_words, unsigned long long* chunk_nulls, cudaStream_t s) {
    if (n_rows <= 0) return cudaSuccess;
    const long long tpc = (batch + kJsonRows - 1) / kJsonRows;
    const long long tiles = (n_rows + batch - 1) / batch * tpc;
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidValue;
    k_json_list_count<<<(unsigned)tiles, kThreads, 0, s>>>(text, (const JsonMember*)members, slots, n_file_cols, file_col, n_rows, batch, tpc, counts, valid_words,
                                                          chunk_nulls);
    return cudaGetLastError();
}

// bounds: n_chunks + 1 entries, the scanned count at the first row of every chunk and the total.
cudaError_t launch_json_bounds(const unsigned long long* offs, long long n_rows, long long batch, long long n_chunks, unsigned long long* bounds, cudaStream_t s) {
    k_json_bounds<<<(unsigned)((n_chunks + 1 + kThreads - 1) / kThreads), kThreads, 0, s>>>(offs, n_rows, batch, n_chunks, bounds);
    return cudaGetLastError();
}

cudaError_t launch_json_list_fill(const uint8_t* text, const void* members, const unsigned int* slots, int n_file_cols, int file_col, int dtype, long long n_rows,
                                  long long batch, const unsigned long long* offs, const uint32_t* valid_words, const void* out, unsigned long long* elem_nulls,
                                  void* slow, unsigned long long* n_slow, long long slow_cap, cudaStream_t s) {
    if (n_rows <= 0) return cudaSuccess;
    const long long tpc = (batch + kJsonRows - 1) / kJsonRows;
    const long long tiles = (n_rows + batch - 1) / batch * tpc;
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidValue;
    k_json_list_fill<<<(unsigned)tiles, kThreads, 0, s>>>(text, (const JsonMember*)members, slots, n_file_cols, file_col, dtype, n_rows, batch, tpc, offs,
                                                         valid_words, (const JsonListChunk*)out, elem_nulls, (JsonSlow*)slow, n_slow, slow_cap);
    return cudaGetLastError();
}

}  // namespace bdf
