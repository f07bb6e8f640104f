// k_csv.cu -- CSV files straight to device columns (DataFrame::from_csv, src/dataframe.rs:349-389: arrow's csv::Reader over the
// csv / csv-core crates).  The host side is runtime.cu (csv_open / csv_read); the field rules are csv_parse.cuh.
//
// Tokenizing is csv-core's record DFA over bytes, five states (StartRecord, StartField, InField, InQuoted, QuoteInQuoted), run as
// a scan: every thread owns 16 bytes and computes the transition FUNCTION of its bytes from all five start states at once, packed
// into one word (5 x 3 bits).  Composition of such functions is associative, so
//   k_csv_dfa_reduce   the CTA's function (a warp scan, then the 8 warps in order);
//   k_csv_dfa_scan     one CTA: the true state at the first byte of every CTA, and the state at the end of the file;
//   k_csv_mark         the exclusive scan inside the CTA gives every thread its start state; it walks its 16 bytes and writes
//                      two 16-bit masks: the bytes that end a field (delimiter or terminator) and those that end a record, and
//                      the CTA's count of field ends, whose exclusive scan (k_scan_one of k_scan.cu) ends with the total;
//   k_csv_index        the masks -> the field index: one int64 per field, the byte where it ends, bit 63 set when the field
//                      ends its record; the first such field gives the first record's field count.
// A field starts one byte after the end of the previous one; after a record end, csv-core skips every '\r' / '\n' first (blank
// lines make no record), so the start needs no storage of its own.
//   k_csv_check        every record has as many fields as the first one (the reader is not flexible): the first field where
//                      the record-end bit disagrees with that count.
//   k_csv_infer        one thread per field of the inferred records: the class bits {empty, bool, int, decimal, other} of every
//                      column, OR-ed in global memory (the host applies the merge rule).
//   k_csv_parse        (column, tile of 256 rows of one RecordBatch): one thread per field, a NULL slot holds zero; validity and
//                      boolean values are assembled by warp ballot, so every chunk starts its own bitmap words; valid counts per
//                      warp.  The first failing field by (batch, column, row) is kept with an atomicMin; floats the fast path
//                      cannot round go on a list that the host resolves exactly;
//   k_csv_scatter      writes the host's exact values.
#include "common.cuh"
#include "csv_parse.cuh"
#include "scan.cuh"

#include <algorithm>

namespace bdf {

constexpr int kCsvBytes = 16;                    // bytes per thread of the tokenizer
constexpr int kCsvTile = kThreads * kCsvBytes;   // bytes per CTA
constexpr int kCsvRows = kThreads;               // rows per CTA of the parser
constexpr unsigned long long kCsvRecBit = 1ull << 63;
constexpr unsigned long long kCsvPosMask = kCsvRecBit - 1;

enum { kSR = 0, kSF, kIF, kIQ, kQQ };
constexpr uint32_t pack5(int a, int b, int c, int d, int e) { return (uint32_t)(a | b << 3 | c << 6 | d << 9 | e << 12); }
constexpr uint32_t kIdent = pack5(kSR, kSF, kIF, kIQ, kQQ);
// next state of (SR, SF, IF, IQ, QQ) for each byte class
constexpr uint32_t kOnDelim = pack5(kSF, kSF, kSF, kIQ, kSF);
constexpr uint32_t kOnQuote = pack5(kIQ, kIQ, kIF, kQQ, kIQ);
constexpr uint32_t kOnTerm = pack5(kSR, kSR, kSR, kIQ, kSR);
constexpr uint32_t kOnOther = pack5(kIF, kIF, kIF, kIQ, kIF);

__device__ __forceinline__ int apply(uint32_t f, int s) { return (int)((f >> (3 * s)) & 7u); }
// a, then b
__device__ __forceinline__ uint32_t compose(uint32_t a, uint32_t b) {
    uint32_t r = 0;
#pragma unroll
    for (int s = 0; s < 5; s++) r |= (uint32_t)apply(b, apply(a, s)) << (3 * s);
    return r;
}
__device__ __forceinline__ uint32_t on_byte(uint8_t b, uint8_t delim) {
    return b == delim ? kOnDelim : b == '"' ? kOnQuote : (b == '\r' || b == '\n') ? kOnTerm : kOnOther;
}

__device__ __forceinline__ void load16(const uint8_t* __restrict__ text, long long n, long long g, uint8_t (&b)[kCsvBytes], int* cnt) {
    const long long off = g * kCsvBytes;
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(text) + g);   // the buffer is padded to whole tiles
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int k = 0; k < kCsvBytes; k++) b[k] = (uint8_t)(w[k >> 2] >> (8 * (k & 3)));
    *cnt = off >= n ? 0 : (int)(n - off < kCsvBytes ? n - off : kCsvBytes);
}

__device__ __forceinline__ uint32_t thread_fn(const uint8_t (&b)[kCsvBytes], int cnt, uint8_t delim) {
    uint32_t f = kIdent;
#pragma unroll
    for (int k = 0; k < kCsvBytes; k++)
        if (k < cnt) f = compose(f, on_byte(b[k], delim));
    return f;
}

// inclusive warp scan of functions (lane i: lanes 0..i in order)
__device__ __forceinline__ uint32_t warp_scan_fn(uint32_t f) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, f, o);
        if (lane >= o) f = compose(y, f);
    }
    return f;
}

__global__ void __launch_bounds__(kThreads) k_csv_dfa_reduce(const uint8_t* __restrict__ text, long long n, uint8_t delim, uint32_t* __restrict__ agg) {
    __shared__ uint32_t s_warp[kWarpsPerCta];
    uint8_t b[kCsvBytes];
    int cnt;
    load16(text, n, (long long)blockIdx.x * kThreads + threadIdx.x, b, &cnt);
    const uint32_t f = warp_scan_fn(thread_fn(b, cnt, delim));
    if ((threadIdx.x & 31) == 31) s_warp[threadIdx.x >> 5] = f;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t t = kIdent;
#pragma unroll
        for (int w = 0; w < kWarpsPerCta; w++) t = compose(t, s_warp[w]);
        agg[blockIdx.x] = t;
    }
}

// One CTA of 1024 threads, each owning a contiguous run of CTAs: start[i] = state at the first byte of CTA i; *final = at the end.
__global__ void __launch_bounds__(1024) k_csv_dfa_scan(const uint32_t* __restrict__ agg, long long count, uint8_t* __restrict__ start, int* __restrict__ final_state) {
    __shared__ uint32_t s_warp[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long per = (count + 1023) / 1024;
    const long long begin = min(count, (long long)threadIdx.x * per), end = min(count, begin + per);
    uint32_t run = kIdent;
    for (long long i = begin; i < end; i++) run = compose(run, agg[i]);
    const uint32_t incl = warp_scan_fn(run);
    uint32_t excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = kIdent;
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t before = kIdent;
    for (int w = 0; w < warp; w++) before = compose(before, s_warp[w]);
    int s = apply(compose(before, excl), kSR);
    for (long long i = begin; i < end; i++) { start[i] = (uint8_t)s; s = apply(agg[i], s); }
    if (threadIdx.x == 1023) *final_state = s;
}

__global__ void __launch_bounds__(kThreads)
k_csv_mark(const uint8_t* __restrict__ text, long long n, uint8_t delim, const uint8_t* __restrict__ start, uint16_t* __restrict__ fe,
           uint16_t* __restrict__ re, unsigned long long* __restrict__ block_counts) {
    __shared__ uint32_t s_warp[kWarpsPerCta];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
    uint8_t b[kCsvBytes];
    int cnt;
    load16(text, n, g, b, &cnt);
    const uint32_t incl = warp_scan_fn(thread_fn(b, cnt, delim));
    uint32_t excl = __shfl_up_sync(0xffffffffu, incl, 1);
    if (lane == 0) excl = kIdent;
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    uint32_t before = kIdent;
    for (int w = 0; w < warp; w++) before = compose(before, s_warp[w]);
    int s = apply(compose(before, excl), start[blockIdx.x]);
    uint32_t fbits = 0, rbits = 0;
#pragma unroll
    for (int k = 0; k < kCsvBytes; k++) {
        if (k >= cnt) break;
        const uint8_t c = b[k];
        const bool d = c == delim, t = c == '\r' || c == '\n';
        if (s != kIQ && (d || (t && s != kSR))) fbits |= 1u << k;
        if (t && (s == kSF || s == kIF || s == kQQ)) rbits |= 1u << k;
        s = apply(on_byte(c, delim), s);
    }
    fe[g] = (uint16_t)fbits;
    re[g] = (uint16_t)rbits;
    const int c = cta_sum(__popc(fbits));
    if (threadIdx.x == 0) block_counts[blockIdx.x] = (unsigned long long)c;
}

__global__ void __launch_bounds__(kThreads)
k_csv_index(const uint16_t* __restrict__ fe, const uint16_t* __restrict__ re, long long n16, const unsigned long long* __restrict__ block_offsets,
            unsigned long long* __restrict__ ends, unsigned long long* __restrict__ first_rec) {
    const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
    const uint32_t fbits = g < n16 ? fe[g] : 0u, rbits = g < n16 ? re[g] : 0u;
    unsigned long long off = block_offsets[blockIdx.x] + (unsigned long long)cta_exclusive_sum(__popc(fbits));
    uint32_t m = fbits;
    while (m) {
        const int k = __ffs(m) - 1;
        m &= m - 1;
        const bool rec = (rbits >> k) & 1u;
        ends[off] = (unsigned long long)(g * kCsvBytes + k) | (rec ? kCsvRecBit : 0ull);
        if (rec) atomicMin(first_rec, off);
        off++;
    }
}

__global__ void __launch_bounds__(kThreads)
k_csv_check(const unsigned long long* __restrict__ ends, long long n_fields, long long k, unsigned long long* __restrict__ bad) {
    for (long long f = (long long)blockIdx.x * kThreads + threadIdx.x; f < n_fields; f += (long long)gridDim.x * kThreads) {
        const bool rec = (ends[f] & kCsvRecBit) != 0, want = (f + 1) % k == 0;
        if (rec != want) atomicMin(bad, (unsigned long long)f);
    }
}

// Raw bytes of field f: [start, end).
__device__ __forceinline__ void field_span(const uint8_t* __restrict__ text, const unsigned long long* __restrict__ ends, long long f,
                                           long long* start, long long* end) {
    const long long e = (long long)(ends[f] & kCsvPosMask);
    const unsigned long long p = f > 0 ? ends[f - 1] : ~0ull;   // the first field starts like one after a record end at byte -1
    long long s = (long long)((p + 1) & kCsvPosMask);
    if (p & kCsvRecBit)
        while (s < e && (text[s] == '\r' || text[s] == '\n')) s++;
    *start = s;
    *end = e;
}

__global__ void __launch_bounds__(kThreads)
k_csv_infer(const uint8_t* __restrict__ text, const unsigned long long* __restrict__ ends, long long f0, long long f1, long long k,
            unsigned int* __restrict__ col_bits) {
    for (long long f = f0 + (long long)blockIdx.x * kThreads + threadIdx.x; f < f1; f += (long long)gridDim.x * kThreads) {
        long long s, e;
        field_span(text, ends, f, &s, &e);
        const unsigned int bit = (unsigned int)csv::classify(csv::Unquote(text + s, text + e));
        unsigned int* slot = col_bits + (f % k);
        if ((*(volatile unsigned int*)slot & bit) == 0) atomicOr(slot, bit);
    }
}

struct CsvColDesc {
    char* values;            // chunk 0 of the output column
    long long vstride;       // bytes between chunks
    uint32_t* validity;      // chunk 0's bitmap
    long long bstride;
    uint32_t* warp_counts;   // [tile][warp] valid slots, tile = chunk * tiles_per_chunk + tile in chunk
    int dtype;               // 0..9, or 10 boolean
    int file_col;
};

struct CsvSlow {   // a float field the fast path could not round
    long long start, end;   // its raw bytes
    int col;                // index into the projection
    int pad;
    long long chunk, row;
};

__global__ void __launch_bounds__(kThreads)
k_csv_parse(const uint8_t* __restrict__ text, const unsigned long long* __restrict__ ends, const CsvColDesc* __restrict__ cols, int n_cols, long long f0,
            long long k, long long n_rows, long long batch, long long tiles_per_chunk, unsigned long long* __restrict__ err_key,
            CsvSlow* __restrict__ slow, unsigned long long* __restrict__ n_slow, long long slow_cap) {
    const int p = blockIdx.y;
    const CsvColDesc d = cols[p];
    const long long chunk = (long long)blockIdx.x / tiles_per_chunk, tt = (long long)blockIdx.x % tiles_per_chunk;
    const long long row = tt * kCsvRows + threadIdx.x;
    const long long clen = min(batch, n_rows - chunk * batch);
    const bool active = row < clen;
    bool valid = false, bval = false;
    if (active) {
        const long long f = f0 + (chunk * batch + row) * k + d.file_col;
        long long s, e;
        field_span(text, ends, f, &s, &e);
        const csv::Unquote u(text + s, text + e);
        csv::Unquote probe = u;
        bool ok = true;
        char* dst = d.values + chunk * d.vstride;
        if (probe.next() < 0) {   // an empty field (unquoted or "") is NULL; its slot is zeroed so a read is deterministic
            if (d.dtype != 10) switch (dtype_width(d.dtype)) {
                case 1: reinterpret_cast<uint8_t*>(dst)[row] = 0; break;
                case 2: reinterpret_cast<uint16_t*>(dst)[row] = 0; break;
                case 4: reinterpret_cast<uint32_t*>(dst)[row] = 0; break;
                default: reinterpret_cast<uint64_t*>(dst)[row] = 0; break;
            }
        } else {
            valid = true;
            if (d.dtype == 10) {
                ok = csv::parse_bool(u, &bval);
            } else if (d.dtype == T_F32 || d.dtype == T_F64) {
                uint64_t bits = 0;
                const int r = d.dtype == T_F64 ? csv::parse_float(u, CSV_F64, &bits) : csv::parse_float(u, CSV_F32, &bits);
                if (r == csv::kFloatBad) ok = false;
                else if (r == csv::kFloatSlow) {
                    const unsigned long long slot = atomicAdd(n_slow, 1ull);
                    if ((long long)slot < slow_cap) slow[slot] = CsvSlow{s, e, p, 0, chunk, row};
                } else if (d.dtype == T_F64) reinterpret_cast<uint64_t*>(dst)[row] = bits;
                else reinterpret_cast<uint32_t*>(dst)[row] = (uint32_t)bits;
            } else {
                uint64_t v = 0;
                ok = csv::parse_int(u, d.dtype, &v);
                if (ok) switch (dtype_width(d.dtype)) {
                    case 1: reinterpret_cast<uint8_t*>(dst)[row] = (uint8_t)v; break;
                    case 2: reinterpret_cast<uint16_t*>(dst)[row] = (uint16_t)v; break;
                    case 4: reinterpret_cast<uint32_t*>(dst)[row] = (uint32_t)v; break;
                    default: reinterpret_cast<uint64_t*>(dst)[row] = v; break;
                }
            }
        }
        if (!ok) atomicMin(err_key, (unsigned long long)((chunk * n_cols + p) * batch + row));
    }
    const unsigned vw = __ballot_sync(0xffffffffu, valid), bw = __ballot_sync(0xffffffffu, bval);
    const long long row0 = row - (threadIdx.x & 31);
    if ((threadIdx.x & 31) == 0 && row0 < clen) {
        d.validity[(chunk * d.bstride) / 4 + (row0 >> 5)] = vw;
        if (d.dtype == 10) reinterpret_cast<uint32_t*>(d.values + chunk * d.vstride)[row0 >> 5] = bw;
    }
    if ((threadIdx.x & 31) == 0 && tt * kCsvRows < clen) d.warp_counts[(chunk * tiles_per_chunk + tt) * kWarpsPerCta + (threadIdx.x >> 5)] = (uint32_t)__popc(vw);
}

struct CsvPatch { unsigned long long dst, bits; int width, pad; };

__global__ void __launch_bounds__(kThreads) k_csv_scatter(const CsvPatch* __restrict__ patches, long long n) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n) return;
    const CsvPatch pt = patches[i];
    if (pt.width == 8) *reinterpret_cast<unsigned long long*>(pt.dst) = pt.bits;
    else *reinterpret_cast<uint32_t*>(pt.dst) = (uint32_t)pt.bits;
}

// ---- launchers ------------------------------------------------------------------------------------------------------
int csv_tile_bytes() { return kCsvTile; }
int csv_parse_rows() { return kCsvRows; }
size_t csv_desc_bytes() { return sizeof(CsvColDesc); }
size_t csv_slow_bytes() { return sizeof(CsvSlow); }
size_t csv_patch_bytes() { return sizeof(CsvPatch); }

// text: padded to whole tiles.  agg / start: one entry per tile.  fe / re: n_tiles * kThreads entries.  block_counts: n_tiles + 1.
cudaError_t launch_csv_tokenize(const uint8_t* text, long long n, uint8_t delim, uint32_t* agg, uint8_t* start, int* final_state, uint16_t* fe,
                                uint16_t* re, unsigned long long* block_counts, cudaStream_t s) {
    const long long tiles = std::max<long long>((n + kCsvTile - 1) / kCsvTile, 1);
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidValue;
    k_csv_dfa_reduce<<<(unsigned)tiles, kThreads, 0, s>>>(text, n, delim, agg);
    k_csv_dfa_scan<<<1, 1024, 0, s>>>(agg, tiles, start, final_state);
    k_csv_mark<<<(unsigned)tiles, kThreads, 0, s>>>(text, n, delim, start, fe, re, block_counts);
    return launch_scan_one(block_counts, tiles, block_counts + tiles, s);   // its error check covers the launches above
}

cudaError_t launch_csv_index(const uint16_t* fe, const uint16_t* re, long long n, const unsigned long long* block_offsets, unsigned long long* ends,
                             unsigned long long* first_rec, cudaStream_t s) {
    const long long tiles = std::max<long long>((n + kCsvTile - 1) / kCsvTile, 1);
    k_csv_index<<<(unsigned)tiles, kThreads, 0, s>>>(fe, re, tiles * kThreads, block_offsets, ends, first_rec);
    return cudaGetLastError();
}

cudaError_t launch_csv_check(const unsigned long long* ends, long long n_fields, long long k, unsigned long long* bad, int sm_count, cudaStream_t s) {
    if (n_fields <= 0) return cudaSuccess;
    const long long want = (n_fields + kThreads - 1) / kThreads;
    k_csv_check<<<(unsigned)std::min<long long>(want, (long long)sm_count * 16), kThreads, 0, s>>>(ends, n_fields, k, bad);
    return cudaGetLastError();
}

cudaError_t launch_csv_infer(const uint8_t* text, const unsigned long long* ends, long long f0, long long f1, long long k, unsigned int* col_bits,
                             int sm_count, cudaStream_t s) {
    if (f1 <= f0) return cudaSuccess;
    const long long want = (f1 - f0 + kThreads - 1) / kThreads;
    k_csv_infer<<<(unsigned)std::min<long long>(want, (long long)sm_count * 16), kThreads, 0, s>>>(text, ends, f0, f1, k, col_bits);
    return cudaGetLastError();
}

cudaError_t launch_csv_parse(const uint8_t* text, const unsigned long long* ends, const void* cols, int n_cols, long long f0, long long k, long long n_rows,
                             long long batch, unsigned long long* err_key, void* slow, unsigned long long* n_slow, long long slow_cap, cudaStream_t s) {
    if (n_rows <= 0 || n_cols <= 0) return cudaSuccess;
    const long long tpc = (batch + kCsvRows - 1) / kCsvRows;
    const long long chunks = (n_rows + batch - 1) / batch;
    const long long tiles = chunks * tpc;
    if (tiles > 0x7fffffffLL || n_cols > 65535) return cudaErrorInvalidValue;
    k_csv_parse<<<dim3((unsigned)tiles, (unsigned)n_cols), kThreads, 0, s>>>(text, ends, (const CsvColDesc*)cols, n_cols, f0, k, n_rows, batch, tpc, err_key,
                                                                             (CsvSlow*)slow, n_slow, slow_cap);
    return cudaGetLastError();
}

cudaError_t launch_csv_scatter(const void* patches, long long n, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_csv_scatter<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, s>>>((const CsvPatch*)patches, n);
    return cudaGetLastError();
}

}  // namespace bdf
