// k_parquet.cu -- Parquet column chunks straight to device columns (DataFrame::from_parquet, src/dataframe.rs).  The footer and the
// page headers are read on the host (parquet.cu), which builds one page table over every projected column chunk of every file; the
// chunks are uploaded still compressed, and each step below is ONE launch over that table, whatever the number of files, row groups,
// columns or pages.  The decoders are parquet_decode.cuh.
//   k_pq_snappy   one warp per page: every SNAPPY page (V2: its values section) into the scratch at the offset the host chose.  The
//                 lanes parse each tag together (the same bytes, broadcast) and copy its bytes together; an overlapping copy reads
//                 out[op - off + j % off], which the warp can write in any order.  Uncompressed pages stay where they are.
//   k_pq_runs     one thread per (page, stream): the run headers of the definition levels (stream 0) and of the dictionary ids or
//                 Boolean RLE values (stream 1) into the page's run tables.  The walk is serial; the decode below is parallel.
//   k_pq_levels   one CTA per tile of 2048 rows of a page: each row's definition level (a binary search in the run table), its
//                 validity bit straight into the output chunk (row r of a file -> chunk r / batch), the chunk's null count, and the
//                 tile's valid count
//   k_pq_values   the same tiles: each valid row's value index in its page (the valid counts of the page's earlier tiles plus a CTA
//                 scan), the value decoded (PLAIN, dictionary gather with its bounds check, BYTE_STREAM_SPLIT, Boolean bit or RLE),
//                 narrowed to the column's dtype and written into the output chunk; a null row gets 0
// A failure sets the page's error word (first code wins); the host reads the words back once, after the last step.
#include "common.cuh"
#include "parquet_decode.cuh"

namespace bdf {

using pq::Page;
using pq::Tile;
using pq::Out;
using pq::Run;

constexpr int kPqRowsPerThread = pq::kTileRows / kThreads;
static_assert(kPqRowsPerThread * kThreads == pq::kTileRows, "tile geometry");

__device__ __forceinline__ void pq_fail(int* err, int page, int code) { atomicCAS(err + page, 0, code); }

__global__ void __launch_bounds__(kThreads) k_pq_snappy(const Page* pages, int n_pages, const uint8_t* upload, uint8_t* scratch, int* err) {
    const int lane = threadIdx.x & 31;
    const int warps = gridDim.x * (blockDim.x / 32);
    for (int pi = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32; pi < n_pages; pi += warps) {
        const Page p = pages[pi];
        if (p.dst < 0) continue;
        const int skip = p.kind == pq::KIND_V2 ? p.rep_len + p.def_len : 0;
        if (skip < 0 || skip > p.comp) { if (lane == 0) pq_fail(err, pi, pq::E_LAYOUT); continue; }
        const uint8_t* in = upload + p.src + skip;
        const uint32_t n = (uint32_t)(p.comp - skip), out_n = (uint32_t)p.raw;
        uint8_t* out = scratch + p.dst;
        uint32_t ip = 0, op = 0, want = 0;
        int e = pq::snappy_preamble(in, n, &ip, &want);
        if (!e && want != out_n) e = pq::E_SNAPPY_SIZE;
        while (!e && ip < n) {
            pq::SnappyOp s;
            e = pq::snappy_next(in, n, &ip, op, out_n, &s);
            if (e) break;
            if (s.copy) for (uint32_t j = lane; j < s.len; j += 32) out[op + j] = out[op - s.src + j % s.src];
            else for (uint32_t j = lane; j < s.len; j += 32) out[op + j] = in[s.src + j];
            op += s.len;
            __syncwarp();   // the next copy may read what this one wrote
        }
        if (!e && op != out_n) e = pq::E_SNAPPY_SIZE;
        if (e && lane == 0) pq_fail(err, pi, e);
    }
}

__global__ void __launch_bounds__(kThreads) k_pq_runs(const Page* pages, int n_pages, const uint8_t* upload, const uint8_t* scratch, Run* runs,
                                                      uint2* meta, int* err) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= 2ll * n_pages) return;
    const int pi = (int)(t / 2), stream = (int)(t % 2);
    const Page p = pages[pi];
    meta[t] = make_uint2(0, 0);
    if (p.kind == pq::KIND_DICT) return;
    if (stream == 0 && p.max_def == 0) return;
    if (stream == 1 && !pq::uses_index(p.encoding)) return;
    pq::Layout L;
    int e = pq::page_layout(p, upload, scratch, &L);
    uint32_t nr = 0, cover = 0;
    if (!e && stream == 0) {
        e = pq::hybrid_walk(L.def, L.def_n, 1, (uint32_t)p.num_values, runs + p.runs, (uint32_t)p.cap_def, &nr, &cover, pq::E_LEVELS);
        if (!e && cover < (uint32_t)p.num_values) e = pq::E_LEVELS;
    } else if (!e) {
        const uint8_t* s; uint32_t n; int bw;
        e = pq::index_stream(p, L, &s, &n, &bw);
        if (!e) e = pq::hybrid_walk(s, n, bw, (uint32_t)p.num_values, runs + p.runs + p.cap_def, (uint32_t)p.cap_idx, &nr, &cover, pq::E_INDEX);
    }
    if (e) { pq_fail(err, pi, e); return; }
    meta[t] = make_uint2(nr, cover);
}

// Definition level of row k of page p: 1 = valid.
__device__ __forceinline__ int pq_def(const Page& p, const pq::Layout& L, const Run* runs, uint2 m, uint32_t k, int* e) {
    if (p.max_def == 0) return 1;
    uint32_t v = 0;
    *e = pq::hybrid_get(L.def, L.def_n, 1, runs + p.runs, m.x, m.y, k, &v, pq::E_LEVELS);
    if (!*e && v > (uint32_t)p.max_def) *e = pq::E_LEVEL_VALUE;
    return (int)v == p.max_def;
}

__device__ __forceinline__ int pq_block_sum(int v, int* sm) {
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sm[threadIdx.x / 32] = v;
    __syncthreads();
    int s = 0;
    for (int w = 0; w < kWarpsPerCta; w++) s += sm[w];
    return s;
}

__global__ void __launch_bounds__(kThreads) k_pq_levels(const Page* pages, const Tile* tiles, int n_tiles, const uint8_t* upload,
                                                        const uint8_t* scratch, const Run* runs, const uint2* meta, const Out* outs,
                                                        long long batch, int* tile_valid, unsigned long long* nulls, int* err) {
    __shared__ int sm[kWarpsPerCta];
    if ((int)blockIdx.x >= n_tiles) return;
    const Tile tl = tiles[blockIdx.x];
    const Page p = pages[tl.page];
    pq::Layout L;
    int e = pq::page_layout(p, upload, scratch, &L);
    const uint2 m = meta[2 * tl.page];
    const uint32_t k0 = (uint32_t)tl.first + threadIdx.x * kPqRowsPerThread;
    int valid = 0;
    long long cur_chunk = -1, cur_word = -1;
    uint32_t bits = 0;
    unsigned long long cur_nulls = 0;
    for (int i = 0; i < kPqRowsPerThread && !e; i++) {
        const uint32_t k = k0 + i;
        if (k >= (uint32_t)p.num_values) break;
        const int v = pq_def(p, L, runs, m, k, &e);
        if (e) break;
        valid += v;
        const long long r = p.row0 + k, chunk = p.out0 + r / batch, pos = r % batch;
        if (!outs[chunk].validity) continue;   // a column required in every file has no bitmap; required in this file only: all valid
        if (chunk != cur_chunk) {
            if (cur_chunk >= 0 && cur_nulls) atomicAdd(nulls + cur_chunk, cur_nulls);
            cur_nulls = 0;
        }
        if (chunk != cur_chunk || pos / 32 != cur_word) {
            if (bits) atomicOr(outs[cur_chunk].validity + cur_word, bits);
            bits = 0;
            cur_chunk = chunk; cur_word = pos / 32;
        }
        if (v) bits |= 1u << (pos % 32); else cur_nulls++;
    }
    if (bits) atomicOr(outs[cur_chunk].validity + cur_word, bits);
    if (cur_nulls) atomicAdd(nulls + cur_chunk, cur_nulls);
    if (e) pq_fail(err, tl.page, e);
    const int total = pq_block_sum(valid, sm);
    if (threadIdx.x == 0) tile_valid[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads) k_pq_values(const Page* pages, const Tile* tiles, int n_tiles, const uint8_t* upload,
                                                        const uint8_t* scratch, const Run* runs, const uint2* meta, const Out* outs,
                                                        long long batch, const int* tile_valid, int* err) {
    __shared__ int sm[kWarpsPerCta];
    __shared__ int sm_scan[kWarpsPerCta];
    if ((int)blockIdx.x >= n_tiles) return;
    const Tile tl = tiles[blockIdx.x];
    const Page p = pages[tl.page];
    pq::Layout L;
    int e = pq::page_layout(p, upload, scratch, &L);
    const uint2 md = meta[2 * tl.page], mi = meta[2 * tl.page + 1];
    const uint32_t k0 = (uint32_t)tl.first + threadIdx.x * kPqRowsPerThread;
    int flags = 0, cnt = 0;
    for (int i = 0; i < kPqRowsPerThread && !e; i++) {
        const uint32_t k = k0 + i;
        if (k >= (uint32_t)p.num_values) break;
        const int v = pq_def(p, L, runs, md, k, &e);
        flags |= v << i;
        cnt += v;
    }
    // valid values of the page before this tile, and in the whole page (BYTE_STREAM_SPLIT needs the count of encoded values)
    int before = 0, all = 0;
    const int my_tile = (int)blockIdx.x - (int)p.tile0;
    for (int t = threadIdx.x; t < p.n_tiles; t += kThreads) {
        const int c = tile_valid[p.tile0 + t];
        all += c;
        if (t < my_tile) before += c;
    }
    before = pq_block_sum(before, sm);
    all = pq_block_sum(all, sm);
    // exclusive scan of the per-thread counts
    int incl = cnt;
    const int lane = threadIdx.x & 31, warp = threadIdx.x / 32;
    for (int o = 1; o < 32; o <<= 1) {
        const int x = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += x;
    }
    if (lane == 31) sm_scan[warp] = incl;
    __syncthreads();
    int woff = 0;
    for (int w = 0; w < warp; w++) woff += sm_scan[w];
    uint32_t vi = (uint32_t)(before + woff + incl - cnt);

    const uint8_t* is = nullptr; uint32_t in_n = 0; int bw = 0;
    if (!e && pq::uses_index(p.encoding)) e = pq::index_stream(p, L, &is, &in_n, &bw);
    const uint8_t* dict = nullptr; uint32_t dict_n = 0, dict_count = 0;
    if (p.dict >= 0) {
        const Page d = pages[p.dict];
        dict = d.dst >= 0 ? scratch + d.dst : upload + d.src;
        dict_n = (uint32_t)(d.dst >= 0 ? d.raw : d.comp);
        dict_count = (uint32_t)d.num_values;
    }
    long long cur_chunk = -1, cur_word = -1;
    uint32_t bits = 0;
    for (int i = 0; i < kPqRowsPerThread && !e; i++) {
        const uint32_t k = k0 + i;
        if (k >= (uint32_t)p.num_values) break;
        const long long r = p.row0 + k, chunk = p.out0 + r / batch, pos = r % batch;
        uint64_t x = 0;
        const bool valid = (flags >> i) & 1;
        if (valid) {
            switch (p.encoding) {
                case pq::ENC_PLAIN:
                    e = p.phys == pq::PHYS_BOOLEAN ? pq::bit_get(L.val, L.val_n, vi, &x) : pq::plain_get(L.val, L.val_n, p.width, vi, &x);
                    break;
                case pq::ENC_BYTE_STREAM_SPLIT: e = pq::bss_get(L.val, L.val_n, p.width, (uint32_t)all, vi, &x); break;
                case pq::ENC_RLE: {
                    uint32_t b = 0;
                    e = pq::hybrid_get(is, in_n, bw, runs + p.runs + p.cap_def, mi.x, mi.y, vi, &b, pq::E_INDEX);
                    x = b;
                    break;
                }
                default: {   // dictionary ids
                    uint32_t id = 0;
                    e = pq::hybrid_get(is, in_n, bw, runs + p.runs + p.cap_def, mi.x, mi.y, vi, &id, pq::E_INDEX);
                    if (!e && (dict == nullptr || id >= dict_count)) e = pq::E_DICT_RANGE;
                    if (!e) e = p.phys == pq::PHYS_BOOLEAN ? pq::bit_get(dict, dict_n, id, &x) : pq::plain_get(dict, dict_n, p.width, id, &x);
                    break;
                }
            }
            if (e) break;
            vi++;
        }
        char* dst = outs[chunk].values;
        switch (p.out_width) {
            case 0:
                if (chunk != cur_chunk || pos / 32 != cur_word) {
                    if (bits) atomicOr((uint32_t*)outs[cur_chunk].values + cur_word, bits);
                    bits = 0;
                    cur_chunk = chunk; cur_word = pos / 32;
                }
                if (x & 1) bits |= 1u << (pos % 32);
                break;
            case 1: ((uint8_t*)dst)[pos] = (uint8_t)x; break;     // narrowed to the low bits (documented in b200df.h)
            case 2: ((uint16_t*)dst)[pos] = (uint16_t)x; break;
            case 4: ((uint32_t*)dst)[pos] = (uint32_t)x; break;
            default: ((uint64_t*)dst)[pos] = x; break;
        }
    }
    if (bits) atomicOr((uint32_t*)outs[cur_chunk].values + cur_word, bits);
    if (e) pq_fail(err, tl.page, e);
}

size_t pq_page_bytes() { return sizeof(Page); }
size_t pq_tile_bytes() { return sizeof(Tile); }
size_t pq_out_bytes() { return sizeof(Out); }
size_t pq_run_bytes() { return sizeof(Run); }

cudaError_t launch_pq_snappy(const void* pages, int n_pages, const uint8_t* upload, uint8_t* scratch, int* err, int sm_count, cudaStream_t s) {
    const int per_cta = kThreads / 32;
    const int grid = std::max(1, std::min((n_pages + per_cta - 1) / per_cta, sm_count * 8));
    k_pq_snappy<<<grid, kThreads, 0, s>>>((const Page*)pages, n_pages, upload, scratch, err);
    return cudaGetLastError();
}

cudaError_t launch_pq_runs(const void* pages, int n_pages, const uint8_t* upload, const uint8_t* scratch, void* runs, void* meta, int* err,
                           cudaStream_t s) {
    const long long n = 2ll * n_pages;
    const int grid = (int)std::max<long long>(1, (n + kThreads - 1) / kThreads);
    k_pq_runs<<<grid, kThreads, 0, s>>>((const Page*)pages, n_pages, upload, scratch, (Run*)runs, (uint2*)meta, err);
    return cudaGetLastError();
}

cudaError_t launch_pq_levels(const void* pages, const void* tiles, int n_tiles, const uint8_t* upload, const uint8_t* scratch, const void* runs,
                             const void* meta, const void* outs, long long batch, int* tile_valid, unsigned long long* nulls, int* err,
                             cudaStream_t s) {
    k_pq_levels<<<std::max(n_tiles, 1), kThreads, 0, s>>>((const Page*)pages, (const Tile*)tiles, n_tiles, upload, scratch, (const Run*)runs,
                                                          (const uint2*)meta, (const Out*)outs, batch, tile_valid, nulls, err);
    return cudaGetLastError();
}

cudaError_t launch_pq_values(const void* pages, const void* tiles, int n_tiles, const uint8_t* upload, const uint8_t* scratch, const void* runs,
                             const void* meta, const void* outs, long long batch, const int* tile_valid, int* err, cudaStream_t s) {
    k_pq_values<<<std::max(n_tiles, 1), kThreads, 0, s>>>((const Page*)pages, (const Tile*)tiles, n_tiles, upload, scratch, (const Run*)runs,
                                                          (const uint2*)meta, (const Out*)outs, batch, tile_valid, err);
    return cudaGetLastError();
}

}  // namespace bdf
