// k_json_write.cu -- device columns to line-delimited JSON text (include/b200df.h "line-delimited JSON files straight from the
// device"; the value rules are json_format.cuh).  The host side is runtime.cu (json_write).
//
// A list row has no longest possible text, so rows are taken in WINDOWS and the text blocks are cut from measured lengths:
//   k_jsonw_window     one thread: the window's end row -- at most max_rows rows and elem_cap list elements, at least one row --
//                      and where each list column's elements of the window start (the plan, JsonwArgs::plan).
//   k_jsonw_elem_len   one thread per list element of the window (every list column's, one after another): the element's text
//                      length plus its comma, with the tile sums of launch_scan_sums (k_scan.cu), which scans them.  A list's text
//                      is then a difference of two scan entries, so a hot list is spread over the whole GPU.
//   k_jsonw_measure    one thread per row walks the column table: "name": and the value of every member it writes, the commas,
//                      the braces and "\n"; the scan turns the lengths into the window's byte offsets.
//   k_jsonw_cut        one thread: cuts the window's text into blocks at row boundaries where it reaches the buffer's capacity
//                      (a row longer than that is a block of its own) and reports each block's rows, bytes and elements.
//   k_jsonw_emit       one thread per row of a block writes '{', the scalar members, each list member's "name":[ and ], the commas
//                      and "}\n" into a shared-memory window at its offset; the CTA then stores its byte range with aligned 16-byte
//                      stores, as k_csvw_emit does (a CTA whose text does not fit writes its rows straight to global memory).
//                      The bytes between a list's brackets are left to:
//   k_jsonw_elem_emit  one thread per element of one list column in the block: finds its row in the chunk's offsets and writes
//                      the element at the row's list position plus its scan position, then its comma.
// Every byte has one writer: the same frame always gives the same bytes.
#include "common.cuh"
#include "json_format.cuh"
#include "scan.cuh"

namespace bdf {

constexpr int kJsonwWindow = 24576;   // bytes of text a CTA of the emit step stages in shared memory

__device__ __forceinline__ bool jsonw_bit(const uint32_t* __restrict__ w, long long i) { return (__ldg(w + (i >> 5)) >> (i & 31)) & 1u; }

// The last chunk whose first row is <= g (empty chunks share their start with the next one, so this is the chunk holding g).
__device__ __forceinline__ int jsonw_chunk_of(const JsonwArgs& a, long long g) {
    int lo = 0, hi = a.n_chunks - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(a.chunk_start + mid) <= g) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// The last chunk of column j whose first element is <= e.
__device__ __forceinline__ int jsonw_elem_chunk_of(const JsonwArgs& a, int j, long long e) {
    int lo = 0, hi = a.n_chunks - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (a.desc[(size_t)mid * a.n_cols + j].estart <= e) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// The element of list column j that starts row g (g may be the frame's row count: then the column's element count).
__device__ long long jsonw_elem_at(const JsonwArgs& a, int j, long long g) {
    const int ch = jsonw_chunk_of(a, g);
    const JsonwDesc& d = a.desc[(size_t)ch * a.n_cols + j];
    const long long local = g - __ldg(a.chunk_start + ch);
    return d.estart + (local ? (long long)__ldg(d.loffs + local) : 0);
}

// False for a NaN or an infinity: JSON has no number for them, so they are written as null.
__device__ __forceinline__ bool jsonw_finite(int dtype, const void* v, long long r) {
    if (dtype == T_F32) return (__ldg((const uint32_t*)v + r) & 0x7f800000u) != 0x7f800000u;
    if (dtype == T_F64) return (__ldg((const unsigned long long*)v + r) & 0x7ff0000000000000ull) != 0x7ff0000000000000ull;
    return true;
}

// One finite value of dtype `dtype` (a temporal type when c.tkind); writes it when W.  Returns its length.
template <bool W>
__device__ __forceinline__ int jsonw_value(const JsonwCol& c, int dtype, const void* v, int val_bit_off, long long r, char* p) {
    if (c.tkind != JT_NONE) {
        const long long x = dtype == T_I32 ? (long long)__ldg((const int32_t*)v + r) : __ldg((const long long*)v + r);
        if (W) jsonf_time_put(x, c.tkind, c.upd, c.ups, c.off, c.frac, c.suffix_len, c.suffix, p);
        return jsonf_time_len(x, c.tkind, c.upd, c.off, c.frac, c.suffix_len);
    }
    switch (dtype) {
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
        case T_F32: { const CsvFloat x = csvf_f32(__ldg((const uint32_t*)v + r)); if (W) jsonf_float_put(x, true, p); return jsonf_float_len(x, true); }
        case T_F64: { const CsvFloat x = csvf_f64(__ldg((const unsigned long long*)v + r)); if (W) jsonf_float_put(x, false, p); return jsonf_float_len(x, false); }
        default: {   // Boolean
            const bool b = jsonw_bit((const uint32_t*)v, val_bit_off + r);
            if (W) {
                if (b) { p[0] = 't'; p[1] = 'r'; p[2] = 'u'; p[3] = 'e'; }
                else { p[0] = 'f'; p[1] = 'a'; p[2] = 'l'; p[3] = 's'; p[4] = 'e'; }
            }
            return b ? 4 : 5;
        }
    }
}

__device__ __forceinline__ void jsonw_null(char* p) { p[0] = 'n'; p[1] = 'u'; p[2] = 'l'; p[3] = 'l'; }

// The start of list element e of list L in the window's element scan.
__device__ __forceinline__ long long jsonw_scan_at(const JsonwArgs& a, int L, long long e) {
    return a.plan[2 + a.n_lists + L] + (e - a.plan[2 + L]);
}

// Row `local` of chunk `ch`, at byte `at` of the window's text: the object and "\n".  When W, writes it at p and records each
// written list's '[' (as a window byte) in lpos[L * lpos_stride + wi].
template <bool W>
__device__ __forceinline__ long long jsonw_row(const JsonwArgs& a, int ch, long long local, const unsigned long long* __restrict__ escan, long long* lpos,
                               long long lpos_stride, long long wi, long long at, char* p) {
    const JsonwDesc* d = a.desc + (size_t)ch * a.n_cols;
    long long len = 1;
    if (W) p[0] = '{';
    bool first = true;
    for (int j = 0; j < a.n_cols; j++) {
        const JsonwCol& c = a.cols[j];
        const JsonwDesc dj = d[j];
        const bool present = c.list >= 0 ? !dj.lvalid || jsonw_bit(dj.lvalid, local)
                                         : (!dj.validity || jsonw_bit(dj.validity, dj.bit_off + local)) && jsonw_finite(c.dtype, dj.values, local);
        if (!present && !a.explicit_nulls) continue;
        if (!first) { if (W) p[len] = ','; len++; }
        first = false;
        if (W) for (int k = 0; k < c.name_len; k++) p[len + k] = a.names[c.name_at + k];
        len += c.name_len;
        if (!present) { if (W) jsonw_null(p + len); len += 4; }
        else if (c.list >= 0) {
            const long long e0 = dj.estart + __ldg(dj.loffs + local), e1 = dj.estart + __ldg(dj.loffs + local + 1);
            const long long n = 2 + (long long)(escan[jsonw_scan_at(a, c.list, e1)] - escan[jsonw_scan_at(a, c.list, e0)]) - (e1 > e0 ? 1 : 0);
            if (W) {
                p[len] = '[';
                p[len + n - 1] = ']';
                lpos[c.list * lpos_stride + wi] = at + len;
            }
            len += n;
        } else {
            len += jsonw_value<W>(c, c.dtype, dj.values, dj.val_bit_off, local, p + len);
        }
    }
    if (W) { p[len] = '}'; p[len + 1] = '\n'; }
    return len + 2;
}

__global__ void k_jsonw_window(const JsonwArgs a, long long row0, long long rows, long long max_rows, long long elem_cap) {
    long long* plan = a.plan;
    auto elems = [&](long long g) {
        long long s = 0;
        for (int L = 0; L < a.n_lists; L++) s += jsonw_elem_at(a, __ldg(a.list_cols + L), g);
        return s;
    };
    const long long s0 = elems(row0);
    long long lo = row0 + 1, hi = min(rows, row0 + max_rows);   // the last end row within the cap (row0 + 1 at least)
    while (lo < hi) {
        const long long mid = lo + (hi - lo + 1) / 2;
        if (elems(mid) - s0 <= elem_cap) lo = mid; else hi = mid - 1;
    }
    plan[0] = lo;
    long long seg = 0;
    for (int L = 0; L < a.n_lists; L++) {
        const int j = __ldg(a.list_cols + L);
        const long long e0 = jsonw_elem_at(a, j, row0);
        plan[2 + L] = e0;
        plan[2 + a.n_lists + L] = seg;
        seg += jsonw_elem_at(a, j, lo) - e0;
    }
    plan[1] = seg;
}

__global__ void __launch_bounds__(kThreads) k_jsonw_elem_len(const JsonwArgs a, long long n, unsigned long long* __restrict__ lens,
                                                             unsigned long long* __restrict__ block_sums) {
    const long long base = (long long)blockIdx.x * kScanTile;
    unsigned long long sum = 0;
    for (int it = 0; it < kScanItems; it++) {
        const long long i = base + it * kThreads + threadIdx.x;
        if (i >= n) break;
        int L = 0;
        for (int k = 1; k < a.n_lists; k++) if (a.plan[2 + a.n_lists + k] <= i) L = k;
        const int j = __ldg(a.list_cols + L);
        const long long e = a.plan[2 + L] + (i - a.plan[2 + a.n_lists + L]);
        const int ch = jsonw_elem_chunk_of(a, j, e);
        const JsonwDesc& d = a.desc[(size_t)ch * a.n_cols + j];
        const long long le = e - d.estart;
        const int dt = a.cols[j].dtype;
        const bool present = (!d.validity || jsonw_bit(d.validity, d.bit_off + le)) && jsonw_finite(dt, d.values, le);
        const unsigned long long l = (unsigned long long)(present ? jsonw_value<false>(a.cols[j], dt, d.values, d.val_bit_off, le, nullptr) : 4) + 1;   // and the comma
        lens[i] = l;
        sum += l;
    }
    sum = cta_sum(sum);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = sum;
}

__global__ void __launch_bounds__(kThreads) k_jsonw_measure(const JsonwArgs a, long long row0, long long rows, const unsigned long long* __restrict__ escan,
                                                            unsigned long long* __restrict__ lens, unsigned long long* __restrict__ block_sums) {
    __shared__ int s_chunk;
    const long long base = (long long)blockIdx.x * kScanTile;
    if (threadIdx.x == 0) s_chunk = jsonw_chunk_of(a, row0 + base);
    __syncthreads();
    int ch = s_chunk;
    unsigned long long sum = 0;
    for (int it = 0; it < kScanItems; it++) {
        const long long i = base + it * kThreads + threadIdx.x;
        if (i >= rows) break;
        const long long g = row0 + i;
        while (__ldg(a.chunk_start + ch + 1) <= g) ch++;
        const unsigned long long len = (unsigned long long)jsonw_row<false>(a, ch, g - __ldg(a.chunk_start + ch), escan, nullptr, 0, 0, 0, nullptr);
        lens[i] = len;
        sum += len;
    }
    sum = cta_sum(sum);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = sum;
}

// cuts[0] = the number of blocks nb; then nb + 1 entries of 2 + n_lists: the block's first row (from the window's first), its first
// byte in the window's text, and the first element of each list column.  Stops after max_cuts blocks (the window then ends there).
__global__ void k_jsonw_cut(const JsonwArgs a, long long row0, long long rows, const unsigned long long* __restrict__ offs,
                            unsigned long long cap, int max_cuts, long long* cuts) {
    const int stride = 2 + a.n_lists;
    auto put = [&](int k, long long r) {
        long long* e = cuts + 1 + (size_t)k * stride;
        e[0] = r;
        e[1] = (long long)offs[r];
        for (int L = 0; L < a.n_lists; L++) e[2 + L] = jsonw_elem_at(a, __ldg(a.list_cols + L), row0 + r);
    };
    long long r = 0;
    int nb = 0;
    while (r < rows && nb < max_cuts) {
        put(nb, r);
        long long lo = r + 1, hi = rows;   // the last end whose text fits (one row at least)
        while (lo < hi) {
            const long long mid = lo + (hi - lo + 1) / 2;
            if (offs[mid] - offs[r] <= cap) lo = mid; else hi = mid - 1;
        }
        r = lo;
        nb++;
    }
    put(nb, r);
    cuts[0] = nb;
}

__global__ void __launch_bounds__(kThreads, 4) k_jsonw_emit(const JsonwArgs a, long long wrow0, long long r0, long long r1,
                                                         const unsigned long long* __restrict__ offs, unsigned long long base,
                                                         const unsigned long long* __restrict__ escan, long long* __restrict__ lpos,
                                                         long long lpos_stride, char* __restrict__ out) {
    __shared__ __align__(16) char s_text[kJsonwWindow + 16];
    __shared__ int s_chunk;
    const long long c0 = r0 + (long long)blockIdx.x * kThreads, c1 = min(r1, c0 + kThreads), g = c0 + threadIdx.x;
    if (threadIdx.x == 0) s_chunk = jsonw_chunk_of(a, c0);
    __syncthreads();
    const unsigned long long o0 = offs[c0 - wrow0], n = offs[c1 - wrow0] - o0;
    const bool staged = n <= (unsigned long long)kJsonwWindow;
    if (g < c1) {
        int ch = s_chunk;
        while (__ldg(a.chunk_start + ch + 1) <= g) ch++;
        const unsigned long long o = offs[g - wrow0];
        jsonw_row<true>(a, ch, g - __ldg(a.chunk_start + ch), escan, lpos, lpos_stride, g - wrow0, (long long)o,
                        staged ? s_text + (o - o0) : out + (o - base));
    }
    if (!staged) return;   // uniform over the CTA
    __syncthreads();
    char* dst = out + (o0 - base);
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

__global__ void __launch_bounds__(kThreads) k_jsonw_elem_emit(const JsonwArgs a, int L, long long e0, long long e1, long long wrow0,
                                                              const unsigned long long* __restrict__ escan, const long long* __restrict__ lpos,
                                                              long long lpos_stride, unsigned long long base, char* __restrict__ out) {
    const long long e = e0 + (long long)blockIdx.x * kThreads + threadIdx.x;
    if (e >= e1) return;
    const int j = __ldg(a.list_cols + L);
    const int ch = jsonw_elem_chunk_of(a, j, e);
    const JsonwDesc& d = a.desc[(size_t)ch * a.n_cols + j];
    const long long le = e - d.estart;
    long long lo = 0, hi = __ldg(a.chunk_start + ch + 1) - __ldg(a.chunk_start + ch) - 1;   // the last list starting at or before le
    while (lo < hi) {
        const long long mid = lo + (hi - lo + 1) / 2;
        if (__ldg(d.loffs + mid) <= le) lo = mid; else hi = mid - 1;
    }
    if (d.lvalid && !jsonw_bit(d.lvalid, lo)) return;   // the elements of a null list are not written
    const long long g = __ldg(a.chunk_start + ch) + lo;
    const long long first = d.estart + __ldg(d.loffs + lo), end = d.estart + __ldg(d.loffs + lo + 1);
    const unsigned long long at = (unsigned long long)lpos[L * lpos_stride + (g - wrow0)] + 1 + (escan[jsonw_scan_at(a, L, e)] - escan[jsonw_scan_at(a, L, first)]);
    char* p = out + (at - base);
    const JsonwCol& c = a.cols[j];
    int len = 4;
    if ((!d.validity || jsonw_bit(d.validity, d.bit_off + le)) && jsonw_finite(c.dtype, d.values, le)) len = jsonw_value<true>(c, c.dtype, d.values, d.val_bit_off, le, p);
    else jsonw_null(p);
    if (e + 1 < end) p[len] = ',';
}

cudaError_t launch_jsonw_window(const JsonwArgs& a, long long row0, long long rows, long long max_rows, long long elem_cap, cudaStream_t s) {
    k_jsonw_window<<<1, 1, 0, s>>>(a, row0, rows, max_rows, elem_cap);
    return cudaGetLastError();
}

// lens: n + 1 entries; block_sums: scan_tile_sums(n) entries.
cudaError_t launch_jsonw_elem_len(const JsonwArgs& a, long long n, unsigned long long* lens, unsigned long long* block_sums, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_jsonw_elem_len<<<(unsigned)((n + kScanTile - 1) / kScanTile), kThreads, 0, s>>>(a, n, lens, block_sums);
    return cudaGetLastError();
}

cudaError_t launch_jsonw_measure(const JsonwArgs& a, long long row0, long long rows, const unsigned long long* escan, unsigned long long* lens,
                                 unsigned long long* block_sums, cudaStream_t s) {
    if (rows <= 0) return cudaSuccess;
    k_jsonw_measure<<<(unsigned)((rows + kScanTile - 1) / kScanTile), kThreads, 0, s>>>(a, row0, rows, escan, lens, block_sums);
    return cudaGetLastError();
}

cudaError_t launch_jsonw_cut(const JsonwArgs& a, long long row0, long long rows, const unsigned long long* offs, unsigned long long cap, int max_cuts,
                             long long* cuts, cudaStream_t s) {
    k_jsonw_cut<<<1, 1, 0, s>>>(a, row0, rows, offs, cap, max_cuts, cuts);
    return cudaGetLastError();
}

cudaError_t launch_jsonw_emit(const JsonwArgs& a, long long wrow0, long long r0, long long r1, const unsigned long long* offs, unsigned long long base,
                              const unsigned long long* escan, long long* lpos, long long lpos_stride, char* out, cudaStream_t s) {
    if (r1 <= r0) return cudaSuccess;
    k_jsonw_emit<<<(unsigned)((r1 - r0 + kThreads - 1) / kThreads), kThreads, 0, s>>>(a, wrow0, r0, r1, offs, base, escan, lpos, lpos_stride, out);
    return cudaGetLastError();
}

cudaError_t launch_jsonw_elem_emit(const JsonwArgs& a, int list, long long e0, long long e1, long long wrow0, const unsigned long long* escan,
                                   const long long* lpos, long long lpos_stride, unsigned long long base, char* out, cudaStream_t s) {
    if (e1 <= e0) return cudaSuccess;
    k_jsonw_elem_emit<<<(unsigned)((e1 - e0 + kThreads - 1) / kThreads), kThreads, 0, s>>>(a, list, e0, e1, wrow0, escan, lpos, lpos_stride, base, out);
    return cudaGetLastError();
}

}  // namespace bdf
