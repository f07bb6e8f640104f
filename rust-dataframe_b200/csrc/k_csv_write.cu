// k_csv_write.cu -- device columns to CSV text (DataFrame::to_csv, src/dataframe.rs:527-543: arrow's csv::Writer).  The host side is
// runtime.cu (csv_write); the field rules are csv_format.cuh and include/b200df.h.
//
// The rows are written in blocks of at most a few million rows, so the text of one block fits a fixed device buffer; per block:
//   k_csvw_measure  one thread per row walks the column table and computes the row's byte length from every value, validity bit and
//                   dtype (floats: their shortest digits); the CTA's total goes to block_sums, the tile sums of launch_scan_sums
//                   (k_scan.cu), which then turns the lengths into byte offsets and puts the block's total behind its last row.
//   k_csvw_emit     one row per thread: formats it again (the digits are recomputed rather than stored: a few hundred integer
//                   instructions per float against the 8+ bytes per field a stored form would move) into a shared-memory window
//                   at its offset, then the CTA stores its contiguous byte range with aligned 16-byte stores, single bytes only at
//                   the unaligned head and tail.  A CTA whose text does not fit the window writes its rows straight to global
//                   memory (only rows averaging more than 96 bytes can do that).
// Rows are read through a per-(chunk, column) descriptor table in device memory, so there is no limit on the number of columns;
// the chunk of a row is found once per CTA by binary search and then by a forward walk.
#include "common.cuh"
#include "csv_format.cuh"
#include "scan.cuh"

namespace bdf {

constexpr int kCsvwTile = kScanTile;              // rows per measure CTA
constexpr int kCsvwWindow = 24576;                 // bytes of text a CTA of the emit step stages in shared memory

struct CsvwArgs {
    const CsvwDesc* cols;            // [chunk][column]
    const long long* chunk_start;    // n_chunks + 1 row starts
    int n_cols, n_chunks;
    long long row0, rows;            // the block: rows [row0, row0 + rows) of the frame
    int delim;
};

__device__ __forceinline__ bool csvw_bit(const uint32_t* __restrict__ w, long long i) { return (__ldg(w + (i >> 5)) >> (i & 31)) & 1u; }

// The last chunk whose first row is <= g (empty chunks share their start with the next one, so this is the chunk holding g).
__device__ __forceinline__ int csvw_chunk_of(const CsvwArgs& a, long long g) {
    int lo = 0, hi = a.n_chunks - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(a.chunk_start + mid) <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// One field; writes it when W.  Returns its length.
template <bool W>
__device__ __forceinline__ int csvw_field(const CsvwDesc& d, long long r, char* p) {
    const void* v = d.values;
    switch (d.dtype) {
        case T_I8: { const int64_t x = __ldg((const int8_t*)v + r); const uint64_t m = x < 0 ? 0 - (uint64_t)x : (uint64_t)x;
                     if (W) csvf_int_put(m, x < 0, p); return csvf_int_len(m, x < 0); }
        case T_I16: { const int64_t x = __ldg((const int16_t*)v + r); const uint64_t m = x < 0 ? 0 - (uint64_t)x : (uint64_t)x;
                      if (W) csvf_int_put(m, x < 0, p); return csvf_int_len(m, x < 0); }
        case T_I32: { const int64_t x = __ldg((const int32_t*)v + r); const uint64_t m = x < 0 ? 0 - (uint64_t)x : (uint64_t)x;
                      if (W) csvf_int_put(m, x < 0, p); return csvf_int_len(m, x < 0); }
        case T_I64: { const int64_t x = __ldg((const long long*)v + r); const uint64_t m = x < 0 ? 0 - (uint64_t)x : (uint64_t)x;
                      if (W) csvf_int_put(m, x < 0, p); return csvf_int_len(m, x < 0); }
        case T_U8: { const uint64_t m = __ldg((const uint8_t*)v + r); if (W) csvf_int_put(m, false, p); return csvf_int_len(m, false); }
        case T_U16: { const uint64_t m = __ldg((const uint16_t*)v + r); if (W) csvf_int_put(m, false, p); return csvf_int_len(m, false); }
        case T_U32: { const uint64_t m = __ldg((const uint32_t*)v + r); if (W) csvf_int_put(m, false, p); return csvf_int_len(m, false); }
        case T_U64: { const uint64_t m = __ldg((const unsigned long long*)v + r); if (W) csvf_int_put(m, false, p); return csvf_int_len(m, false); }
        case T_F32: { const CsvFloat x = csvf_f32(__ldg((const uint32_t*)v + r)); if (W) csvf_float_put(x, p); return csvf_float_len(x); }
        case T_F64: { const CsvFloat x = csvf_f64(__ldg((const unsigned long long*)v + r)); if (W) csvf_float_put(x, p); return csvf_float_len(x); }
        default: {   // Boolean
            const bool b = csvw_bit((const uint32_t*)v, d.val_bit_off + r);
            if (W) {
                if (b) { p[0] = 't'; p[1] = 'r'; p[2] = 'u'; p[3] = 'e'; }
                else { p[0] = 'f'; p[1] = 'a'; p[2] = 'l'; p[3] = 's'; p[4] = 'e'; }
            }
            return b ? 4 : 5;
        }
    }
}

// Row `local` of chunk `ch`: fields, delimiters, "\n"; a lone empty field is written "" (the reader skips blank lines).
template <bool W>
__device__ int csvw_row(const CsvwArgs& a, int ch, long long local, char* p) {
    const CsvwDesc* d = a.cols + (size_t)ch * a.n_cols;
    int len = 0;
    for (int j = 0; j < a.n_cols; j++) {
        const CsvwDesc c = d[j];
        if (j) { if (W) p[len] = (char)a.delim; len++; }
        if (!c.validity || csvw_bit(c.validity, c.bit_off + local)) len += csvw_field<W>(c, local, p + len);
        else if (a.n_cols == 1) { if (W) { p[0] = '"'; p[1] = '"'; } len += 2; }
    }
    if (W) p[len] = '\n';
    return len + 1;
}

__global__ void __launch_bounds__(kThreads) k_csvw_measure(const CsvwArgs a, unsigned long long* __restrict__ lens, unsigned long long* __restrict__ block_sums) {
    __shared__ int s_chunk;
    const long long base = (long long)blockIdx.x * kCsvwTile;
    if (threadIdx.x == 0) s_chunk = csvw_chunk_of(a, a.row0 + base);
    __syncthreads();
    int ch = s_chunk;
    unsigned long long sum = 0;
    for (int it = 0; it < kScanItems; it++) {
        const long long i = base + it * kThreads + threadIdx.x;
        if (i >= a.rows) break;
        const long long g = a.row0 + i;
        while (__ldg(a.chunk_start + ch + 1) <= g) ch++;
        const unsigned long long len = (unsigned long long)csvw_row<false>(a, ch, g - __ldg(a.chunk_start + ch), nullptr);
        lens[i] = len;
        sum += len;
    }
    sum = cta_sum(sum);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = sum;
}

__global__ void __launch_bounds__(kThreads) k_csvw_emit(const CsvwArgs a, const unsigned long long* __restrict__ offs, char* __restrict__ out) {
    __shared__ __align__(16) char s_text[kCsvwWindow + 16];
    __shared__ int s_chunk;
    const long long r0 = (long long)blockIdx.x * kThreads, r1 = min(a.rows, r0 + kThreads), i = r0 + threadIdx.x;
    if (threadIdx.x == 0) s_chunk = csvw_chunk_of(a, a.row0 + r0);
    __syncthreads();
    const unsigned long long o0 = __ldg(offs + r0), n = __ldg(offs + r1) - o0;
    const bool staged = n <= (unsigned long long)kCsvwWindow;
    if (i < r1) {
        const long long g = a.row0 + i;
        int ch = s_chunk;
        while (__ldg(a.chunk_start + ch + 1) <= g) ch++;
        const unsigned long long o = __ldg(offs + i);
        csvw_row<true>(a, ch, g - __ldg(a.chunk_start + ch), staged ? s_text + (o - o0) : out + o);
    }
    if (!staged) return;   // uniform over the CTA
    __syncthreads();
    char* dst = out + o0;
    const int m = (int)n;
    const int head = min(m, (int)((16 - ((uintptr_t)dst & 15)) & 15));
    const int vecs = (m - head) >> 4;
    for (int b = threadIdx.x; b < head; b += kThreads) dst[b] = s_text[b];
    const uint32_t* sw = (const uint32_t*)s_text;
    for (int v = threadIdx.x; v < vecs; v += kThreads) {
        const int src = head + (v << 4), w0 = src >> 2, sh = (src & 3) * 8;
        uint32_t w[5];
#pragma unroll
        for (int k = 0; k < 5; k++) w[k] = sw[w0 + k];   // up to 4 bytes past the text: inside the window's 16 spare bytes
        uint4 q;
        q.x = __funnelshift_r(w[0], w[1], sh);
        q.y = __funnelshift_r(w[1], w[2], sh);
        q.z = __funnelshift_r(w[2], w[3], sh);
        q.w = __funnelshift_r(w[3], w[4], sh);
        st_stream16(dst + src, q);
    }
    for (int b = head + (vecs << 4) + threadIdx.x; b < m; b += kThreads) dst[b] = s_text[b];
}

static CsvwArgs csvw_args(const CsvwDesc* cols, const long long* chunk_start, int n_cols, int n_chunks, long long row0, long long rows, int delim) {
    CsvwArgs a;
    a.cols = cols; a.chunk_start = chunk_start; a.n_cols = n_cols; a.n_chunks = n_chunks; a.row0 = row0; a.rows = rows; a.delim = delim;
    return a;
}

// lens: rows + 1 entries; block_sums: scan_tile_sums(rows) entries.
cudaError_t launch_csvw_measure(const CsvwDesc* cols, const long long* chunk_start, int n_cols, int n_chunks, long long row0, long long rows,
                                unsigned long long* lens, unsigned long long* block_sums, cudaStream_t s) {
    if (rows <= 0) return cudaSuccess;
    k_csvw_measure<<<(unsigned)((rows + kCsvwTile - 1) / kCsvwTile), kThreads, 0, s>>>(csvw_args(cols, chunk_start, n_cols, n_chunks, row0, rows, 0), lens,
                                                                                        block_sums);
    return cudaGetLastError();
}

cudaError_t launch_csvw_emit(const CsvwDesc* cols, const long long* chunk_start, int n_cols, int n_chunks, long long row0, long long rows, int delim,
                             const unsigned long long* offs, char* out, cudaStream_t s) {
    if (rows <= 0) return cudaSuccess;
    k_csvw_emit<<<(unsigned)((rows + kThreads - 1) / kThreads), kThreads, 0, s>>>(csvw_args(cols, chunk_start, n_cols, n_chunks, row0, rows, delim), offs, out);
    return cudaGetLastError();
}

}  // namespace bdf
