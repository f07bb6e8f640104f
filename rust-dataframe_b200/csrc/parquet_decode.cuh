// parquet_decode.cuh -- the decoders of the Parquet reader (k_parquet.cu), written as __host__ __device__ functions so that the
// CPU tests compile and run exactly the code the kernels run (tests/test_parquet.py builds them with g++ and the sanitizers).
//
// Every decoder checks a read against the end of its input, and a write against the end of its output, before the access; a
// corrupt stream returns one of the E_* codes and touches nothing outside its buffers.
#pragma once

#include <stdint.h>

#ifdef __CUDACC__
#define PQ_HD __host__ __device__ __forceinline__
#else
#define PQ_HD inline
#endif

namespace pq {

// Per-page error codes (the device's error word; the host turns them into messages: error_text in parquet.cu).
enum : int {
    E_OK = 0,
    E_SNAPPY,          // corrupt snappy stream
    E_SNAPPY_SIZE,     // decompressed size differs from the page header
    E_LEVELS,          // definition-level stream malformed or shorter than the page
    E_INDEX,           // dictionary-index (or Boolean RLE) stream malformed or shorter than the values
    E_DICT_RANGE,      // dictionary index outside the dictionary
    E_VALUES,          // value stream shorter than the values
    E_LAYOUT,          // level or value section outside the page
    E_BIT_WIDTH,       // bit width above 32
    E_LEVEL_VALUE,     // definition level above the column's maximum
    E_RUNS,            // more runs than the run table holds
    E_NCODES
};

// Page kinds and the Thrift enum values the kernels switch on.
enum : int { KIND_V1 = 0, KIND_V2 = 1, KIND_DICT = 2 };
enum : int { ENC_PLAIN = 0, ENC_PLAIN_DICTIONARY = 2, ENC_RLE = 3, ENC_RLE_DICTIONARY = 8, ENC_BYTE_STREAM_SPLIT = 9 };
enum : int { PHYS_BOOLEAN = 0, PHYS_INT32 = 1, PHYS_INT64 = 2, PHYS_FLOAT = 4, PHYS_DOUBLE = 5 };

// One page of the page table, built on the host (parquet.cu) and read by every kernel.  Offsets are bytes into the upload buffer
// (the projected column chunks, still compressed) or into the decompression scratch.
struct Page {
    long long src;        // the page's bytes after its header, in the upload buffer
    long long dst;        // its decompressed bytes in the scratch; -1: decoded where it is
    long long row0;       // row of its first value within its file
    long long runs;       // first entry of its run tables: [runs, + cap_def) definition levels, [runs + cap_def, + cap_idx) indices
    long long tile0;      // first tile of the page (data pages)
    int comp;             // bytes after the header in the upload buffer
    int raw;              // uncompressed size of what the codec covers (V2: the values section only)
    int kind;             // KIND_*
    int snappy;           // 1: the codec covers its bytes and is SNAPPY
    int encoding;         // values encoding (ENC_*)
    int phys;             // physical type (PHYS_*)
    int width;            // bytes per physical value (1 bit for BOOLEAN: 0)
    int out_width;        // bytes per output value (0: bit-packed Boolean)
    int max_def;          // 0 required, 1 optional
    int num_values;       // values (= rows) in the page; the dictionary size for a dictionary page
    int def_len, rep_len; // V2: byte lengths of the level sections (uncompressed, before the values)
    int dict;             // the page table index of the chunk's dictionary page, -1 for none
    int cap_def, cap_idx; // entries of its two run tables: min(values, stream bytes) + 1 (every kept run has a value and a header
                          // byte), 0 for a stream the page does not have
    int n_tiles;
    int out0;             // first output chunk (Out index) of its column and file
};

struct Tile { int page; int first; };                    // rows [first, first + kTileRows) of a data page
struct Out { char* values; uint32_t* validity; };        // one output chunk; validity null for a required column
struct Run { uint32_t first; uint32_t pos; };            // a hybrid run: its first value and the byte it starts at (| kRle)
constexpr uint32_t kRle = 0x80000000u;
constexpr int kTileRows = 2048;                          // rows per tile: 256 threads x 8 consecutive rows

// ---- snappy ------------------------------------------------------------------------------------------------------------------
// One element of a snappy stream: a literal (src = its input position) or a copy (src = its offset back from the output cursor).
struct SnappyOp { int copy; uint32_t len; uint32_t src; };

// The preamble: the uncompressed length as a varint of at most 5 bytes.
PQ_HD int snappy_preamble(const uint8_t* in, uint32_t n, uint32_t* ip, uint32_t* out_len) {
    uint64_t v = 0;
    for (int s = 0; s < 35; s += 7) {
        if (*ip >= n) return E_SNAPPY;
        const uint8_t b = in[(*ip)++];
        v |= (uint64_t)(b & 0x7f) << s;
        if (!(b & 0x80)) {
            if (v > 0xffffffffull) return E_SNAPPY;
            *out_len = (uint32_t)v;
            return E_OK;
        }
    }
    return E_SNAPPY;
}

// Parse the element at *ip and check it against the input end and the output cursor `op` of `out_n` bytes before any byte moves.
PQ_HD int snappy_next(const uint8_t* in, uint32_t n, uint32_t* ip, uint32_t op, uint32_t out_n, SnappyOp* e) {
    if (*ip >= n) return E_SNAPPY;
    const uint32_t tag = in[(*ip)++];
    uint64_t len, off = 0;
    switch (tag & 3) {
        case 0: {
            len = (tag >> 2) + 1;
            if (len > 60) {
                const uint32_t nb = (uint32_t)len - 60;   // 1..4 bytes of length - 1
                if (n - *ip < nb) return E_SNAPPY;
                uint64_t l = 0;
                for (uint32_t i = 0; i < nb; i++) l |= (uint64_t)in[*ip + i] << (8 * i);
                *ip += nb;
                len = l + 1;
            }
            if (len > n - *ip) return E_SNAPPY;                // a truncated literal
            if (len > out_n - op) return E_SNAPPY_SIZE;        // more output than the header declares
            e->copy = 0; e->len = (uint32_t)len; e->src = *ip;
            *ip += (uint32_t)len;
            return E_OK;
        }
        case 1:
            if (n - *ip < 1) return E_SNAPPY;
            len = 4 + ((tag >> 2) & 7);
            off = ((uint64_t)(tag >> 5) << 8) | in[*ip];
            *ip += 1;
            break;
        case 2:
            if (n - *ip < 2) return E_SNAPPY;
            len = 1 + (tag >> 2);
            off = (uint64_t)in[*ip] | (uint64_t)in[*ip + 1] << 8;
            *ip += 2;
            break;
        default:
            if (n - *ip < 4) return E_SNAPPY;
            len = 1 + (tag >> 2);
            off = (uint64_t)in[*ip] | (uint64_t)in[*ip + 1] << 8 | (uint64_t)in[*ip + 2] << 16 | (uint64_t)in[*ip + 3] << 24;
            *ip += 4;
            break;
    }
    if (off == 0 || off > op) return E_SNAPPY;             // offset 0, or before the start of the output
    if (len > out_n - op) return E_SNAPPY_SIZE;
    e->copy = 1; e->len = (uint32_t)len; e->src = (uint32_t)off;
    return E_OK;
}

// Serial decode of a whole stream into out[0, out_n): the reference the warp decoder of k_pq_snappy follows element by element.
// A copy with offset < len repeats the last `offset` bytes: out[op + j] = out[op - off + j % off].
PQ_HD int snappy_decode(const uint8_t* in, uint32_t n, uint8_t* out, uint32_t out_n) {
    uint32_t ip = 0, op = 0, want = 0;
    int err = snappy_preamble(in, n, &ip, &want);
    if (err) return err;
    if (want != out_n) return E_SNAPPY_SIZE;
    while (ip < n) {
        SnappyOp e;
        if ((err = snappy_next(in, n, &ip, op, out_n, &e))) return err;
        if (e.copy) for (uint32_t j = 0; j < e.len; j++) out[op + j] = out[op - e.src + j % e.src];
        else for (uint32_t j = 0; j < e.len; j++) out[op + j] = in[e.src + j];
        op += e.len;
    }
    return op == out_n ? E_OK : E_SNAPPY_SIZE;
}

// ---- the RLE / bit-packed hybrid -----------------------------------------------------------------------------------------------
// Walk the run headers of stream s[0, n) of bit width bw (<= 32) until `need` values are covered or the stream ends, writing at
// most `cap` runs.  *cover: the values the runs hold (a final bit-packed run cut short by the stream end covers only its whole
// values).  Runs of zero values are not kept.
PQ_HD int hybrid_walk(const uint8_t* s, uint32_t n, int bw, uint32_t need, Run* runs, uint32_t cap, uint32_t* n_runs, uint32_t* cover,
                      int err_code) {
    if (bw < 0 || bw > 32) return E_BIT_WIDTH;
    uint64_t cov = 0;
    uint32_t p = 0, k = 0;
    while (cov < need && p < n) {
        uint64_t h = 0;
        int s_ = 0;
        for (;;) {
            if (p >= n || s_ > 28) return err_code;
            const uint8_t b = s[p++];
            h |= (uint64_t)(b & 0x7f) << s_;
            s_ += 7;
            if (!(b & 0x80)) break;
        }
        uint64_t count;
        if (h & 1) {
            count = (h >> 1) * 8;
            if (!count) continue;
            const uint64_t bytes = (h >> 1) * (uint64_t)bw;
            if (k >= cap) return E_RUNS;
            runs[k++] = Run{(uint32_t)cov, p};
            if (bytes > n - p) {   // cut short by the stream end: only its whole values count
                const uint64_t have = bw ? ((uint64_t)(n - p) * 8) / (uint64_t)bw : count;
                cov += have < count ? have : count;
                p = n;
                break;
            }
            p += (uint32_t)bytes;
        } else {
            count = h >> 1;
            const uint32_t vb = (uint32_t)(bw + 7) / 8;
            if (!count) { if (vb > n - p) return err_code; p += vb; continue; }
            if (vb > n - p) return err_code;
            if (k >= cap) return E_RUNS;
            runs[k++] = Run{(uint32_t)cov, p | kRle};
            p += vb;
        }
        cov += count;
    }
    *n_runs = k;
    *cover = (uint32_t)(cov < need ? cov : need);
    return E_OK;
}

// Value k of a walked stream.
PQ_HD int hybrid_get(const uint8_t* s, uint32_t n, int bw, const Run* runs, uint32_t n_runs, uint32_t cover, uint32_t k, uint32_t* v,
                     int err_code) {
    if (k >= cover || n_runs == 0) return err_code;
    uint32_t lo = 0, hi = n_runs - 1;   // the last run with first <= k
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) / 2;
        if (runs[mid].first <= k) lo = mid; else hi = mid - 1;
    }
    const Run r = runs[lo];
    const uint32_t pos = r.pos & ~kRle;
    if (r.pos & kRle) {
        const uint32_t vb = (uint32_t)(bw + 7) / 8;
        if (pos > n || vb > n - pos) return err_code;
        uint32_t x = 0;
        for (uint32_t i = 0; i < vb; i++) x |= (uint32_t)s[pos + i] << (8 * i);
        *v = bw >= 32 ? x : (x & ((1u << bw) - 1));
        return E_OK;
    }
    const uint64_t bit = (uint64_t)(k - r.first) * (uint64_t)bw;
    const uint64_t b0 = pos + bit / 8, b1 = pos + (bit + bw + 7) / 8;   // bytes [b0, b1) hold the value
    if (bw == 0) { *v = 0; return E_OK; }
    if (b1 > n) return err_code;
    uint64_t x = 0;
    for (uint64_t i = b0; i < b1; i++) x |= (uint64_t)s[i] << (8 * (i - b0));
    x >>= bit % 8;
    *v = (uint32_t)(bw >= 32 ? x : (x & ((1ull << bw) - 1)));
    return E_OK;
}

// ---- fixed-width values ----------------------------------------------------------------------------------------------------------
// PLAIN: value k of width w (4 or 8) at k * w.
PQ_HD int plain_get(const uint8_t* s, uint32_t n, int w, uint32_t k, uint64_t* v) {
    const uint64_t at = (uint64_t)k * (uint64_t)w;
    if (at + (uint64_t)w > n) return E_VALUES;
    uint64_t x = 0;
    for (int i = 0; i < w; i++) x |= (uint64_t)s[at + i] << (8 * i);
    *v = x;
    return E_OK;
}

// PLAIN Boolean: bit k, LSB first.
PQ_HD int bit_get(const uint8_t* s, uint32_t n, uint32_t k, uint64_t* v) {
    if (k / 8 >= n) return E_VALUES;
    *v = (s[k / 8] >> (k % 8)) & 1;
    return E_OK;
}

// BYTE_STREAM_SPLIT over nn values of width w: byte i of value k is at i * nn + k.
PQ_HD int bss_get(const uint8_t* s, uint32_t n, int w, uint32_t nn, uint32_t k, uint64_t* v) {
    if (k >= nn || (uint64_t)nn * (uint64_t)w > n) return E_VALUES;
    uint64_t x = 0;
    for (int i = 0; i < w; i++) x |= (uint64_t)s[(uint64_t)i * nn + k] << (8 * i);
    *v = x;
    return E_OK;
}

// ---- page layout ---------------------------------------------------------------------------------------------------------------------
// Where a data page's definition levels and values lie once its bytes are decompressed: `data` is the decompressed page (V1) or
// values section (V2), `raw_page` the page's bytes in the upload buffer.
struct Layout { const uint8_t* def; uint32_t def_n; const uint8_t* val; uint32_t val_n; };

PQ_HD int page_layout(const Page& p, const uint8_t* upload, const uint8_t* scratch, Layout* L) {
    const uint8_t* raw_page = upload + p.src;
    L->def = nullptr; L->def_n = 0;
    if (p.kind == KIND_V2) {
        if ((int64_t)p.rep_len + p.def_len > p.comp || p.rep_len < 0 || p.def_len < 0) return E_LAYOUT;
        L->def = raw_page + p.rep_len;
        L->def_n = (uint32_t)p.def_len;
        if (p.dst >= 0) { L->val = scratch + p.dst; L->val_n = (uint32_t)p.raw; }
        else { L->val = raw_page + p.rep_len + p.def_len; L->val_n = (uint32_t)(p.comp - p.rep_len - p.def_len); }
        return E_OK;
    }
    const uint8_t* d = p.dst >= 0 ? scratch + p.dst : raw_page;
    const uint32_t n = (uint32_t)(p.dst >= 0 ? p.raw : p.comp);
    uint32_t at = 0;
    if (p.max_def > 0) {   // V1: a 4-byte length, then the levels
        if (n < 4) return E_LAYOUT;
        const uint32_t len = (uint32_t)d[0] | (uint32_t)d[1] << 8 | (uint32_t)d[2] << 16 | (uint32_t)d[3] << 24;
        if (len > n - 4) return E_LAYOUT;
        L->def = d + 4;
        L->def_n = len;
        at = 4 + len;
    }
    L->val = d + at;
    L->val_n = n - at;
    return E_OK;
}

// The index stream inside a values section: dictionary ids start after a bit-width byte, Boolean RLE after a 4-byte length.
PQ_HD int index_stream(const Page& p, const Layout& L, const uint8_t** s, uint32_t* n, int* bw) {
    if (p.encoding == ENC_RLE) {
        if (L.val_n < 4) return E_INDEX;
        const uint32_t len = (uint32_t)L.val[0] | (uint32_t)L.val[1] << 8 | (uint32_t)L.val[2] << 16 | (uint32_t)L.val[3] << 24;
        if (len > L.val_n - 4) return E_INDEX;
        *s = L.val + 4; *n = len; *bw = 1;
        return E_OK;
    }
    if (L.val_n < 1) return E_INDEX;
    *bw = L.val[0];
    if (*bw > 32) return E_BIT_WIDTH;
    *s = L.val + 1; *n = L.val_n - 1;
    return E_OK;
}

PQ_HD bool uses_index(int encoding) {
    return encoding == ENC_PLAIN_DICTIONARY || encoding == ENC_RLE_DICTIONARY || encoding == ENC_RLE;
}

}  // namespace pq

#ifdef PQ_HOST_PLAN
#include <string>
#include <vector>

struct bdf_parquet;

namespace pq {

// What a read needs from the open file (parquet.cu): the byte ranges to upload, the page and tile tables, and the output chunking.
struct Plan {
    struct Seg { const uint8_t* src; long long len, dst; };
    std::vector<Seg> segs;               // projected column chunks, headers included, in upload order
    std::vector<Page> pages;             // dictionary and data pages of every projected chunk
    std::vector<Tile> tiles;
    std::vector<int> label;              // per page: file, row group, column, page within its chunk (4 ints)
    std::vector<long long> chunk_lens;   // output chunks of one column: every file's RecordBatches in order
    long long upload_bytes = 0, scratch_bytes = 0, run_entries = 0;
    long long batch = 1024;              // rows per output chunk
};

// The plan for columns cols[0, n) (each checked as bdf_parquet_check does); the output chunks of column i are the Outs
// [i * chunk_lens.size(), (i + 1) * chunk_lens.size()).  A failure sets the library's error and returns its status.
int plan(const bdf_parquet* f, int n, const int32_t* cols, Plan* out);
// The status and message of a device-detected error `code` on page `page` of the plan.
int page_error(const bdf_parquet* f, const Plan& plan, int page, int code);
// Record the last read's page count, uploaded bytes and upload time (bdf_parquet_stats).
void set_stats(const bdf_parquet* f, long long n_pages, long long uploaded, double upload_ms);

}  // namespace pq
#endif
