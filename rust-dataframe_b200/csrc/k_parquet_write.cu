// k_parquet_write.cu -- device columns to Parquet pages (DataFrame::to_parquet, src/dataframe.rs).  runtime.cu's parquet_write cuts
// the file into blocks of consecutive pages (in file order) and builds their page and tile tables on the host; every step below is ONE
// launch over a block's tables, whatever its number of pages, column chunks or row groups.  The encoders are parquet_encode.cuh.
//   k_pqw_rgid, k_pqw_dict_runs, k_pqw_dict_ids   the dictionary of every chunk of one column: after sorted_runs over (row group,
//                 value bits), the valid runs of each row group are its dictionary (ascending bits); each row gets its run's index
//                 inside its row group, its run found from the prefix popcounts of the head bits
//   k_pqw_count   one CTA per tile: the tile's valid rows
//   k_pqw_layout  one thread per page: the valid rows before each tile, the page's null count, the definition-level section (one RLE
//                 run for a page without nulls or with only nulls, else the header of one bit-packed run) and the id section's header
//   k_pqw_encode  one CTA per tile, one read of the column: the level bits (copied from the validity), the values (widened or
//                 converted, PLAIN) or the ids (bit-packed with atomicOr into the zeroed body), and the page statistics
//   k_pqw_snappy  one warp per 64 KiB fragment of a page body, a shared-memory hash table per warp: snappy_fragment's search with
//                 the 32 positions of a window hashed by the 32 lanes and the match picked by a ballot; into its worst-case slot
//   k_pqw_compact one CTA per fragment: the preamble and the fragments of each page, concatenated back into the page's slot
#include <algorithm>

#include "common.cuh"
#include "parquet_encode.cuh"

namespace bdf {

using pq::WPage;
using pq::WTile;
using pq::WPageOut;

constexpr int kRowsPerThread = pq::kWTileRows / kThreads;
static_assert(kRowsPerThread * kThreads == pq::kWTileRows, "tile geometry");
constexpr int kSnappyWarps = 4;   // warps per CTA of k_pqw_snappy: 4 x 8 KiB of hash table

__global__ void k_pqw_rgid(const long long* __restrict__ rg_start, int n_rg, long long n, uint32_t* __restrict__ out) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        int lo = 0, hi = n_rg - 1;   // the last row group starting at or before i
        while (lo < hi) {
            const int mid = (lo + hi + 1) / 2;
            if (rg_start[mid] <= i) lo = mid; else hi = mid - 1;
        }
        out[i] = (uint32_t)lo;
    }
}

__global__ void k_pqw_dict_runs(const uint32_t* __restrict__ run_rg, const uint32_t* __restrict__ run_valid, long long n_runs,
                                unsigned int* __restrict__ count, unsigned int* __restrict__ first) {
    for (long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x; r < n_runs; r += (long long)gridDim.x * blockDim.x) {
        if (run_valid && !((run_valid[r >> 5] >> (r & 31)) & 1)) continue;   // the null run of its row group
        atomicAdd(count + run_rg[r], 1u);
        atomicMin(first + run_rg[r], (unsigned int)r);
    }
}

// head: bit i set when sorted row i starts a run; prefix[w]: the runs that start before row 32w (launch_scan_popcount), so
// the run of a row costs one word and one popcount.
__global__ void k_pqw_dict_ids(const uint32_t* __restrict__ head, const unsigned long long* __restrict__ prefix, const uint32_t* __restrict__ perm,
                               const uint32_t* __restrict__ run_rg, const unsigned int* __restrict__ first, long long n, uint32_t* __restrict__ ids) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i & 31);
        const uint32_t through = b == 31 ? 0xffffffffu : (2u << b) - 1u;   // bits 0 .. b
        const long long run = (long long)prefix[i >> 5] + __popc(head[i >> 5] & through) - 1;
        ids[perm[i]] = (uint32_t)run - first[run_rg[run]];   // a null row's id is never read
    }
}

__device__ __forceinline__ bool tile_valid_bit(const WTile& t, int i) {
    if (!t.validity) return true;
    const long long b = (long long)t.bit_off + t.src_row + i;
    return (t.validity[b >> 5] >> (b & 31)) & 1;
}

// Block-wide exclusive scan of one count per thread (kThreads threads).
__device__ __forceinline__ unsigned int cta_exclusive_scan(unsigned int x, unsigned int* total) {
    __shared__ unsigned int warp_sums[kWarpsPerCta];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned int inc = x;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned int y = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += y;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    unsigned int before = 0, all = 0;
    for (int w = 0; w < kWarpsPerCta; w++) {
        if (w < warp) before += warp_sums[w];
        all += warp_sums[w];
    }
    __syncthreads();
    *total = all;
    return before + inc - x;
}

__global__ void __launch_bounds__(kThreads) k_pqw_count(const WTile* __restrict__ tiles, unsigned int* __restrict__ tile_valid) {
    const WTile t = tiles[blockIdx.x];
    unsigned int v = 0;
    for (int k = 0; k < kRowsPerThread; k++) {
        const int i = threadIdx.x * kRowsPerThread + k;
        if (i < t.rows && tile_valid_bit(t, i)) v++;
    }
    unsigned int total;
    cta_exclusive_scan(v, &total);
    if (threadIdx.x == 0) tile_valid[blockIdx.x] = total;
}

// Per page: [0] byte offset of the level bits in the body (0: the levels are one RLE run), [1] byte offset of the values / ids.
__global__ void k_pqw_layout(const WPage* __restrict__ pages, int n_pages, const unsigned int* __restrict__ tile_valid, unsigned int* __restrict__ tile_base,
                             uint8_t* __restrict__ raw, uint2* __restrict__ lay, WPageOut* __restrict__ out) {
    const int pi = blockIdx.x * blockDim.x + threadIdx.x;
    if (pi >= n_pages) return;
    const WPage p = pages[pi];
    unsigned int valid = 0;
    for (int t = 0; t < p.n_tiles; t++) { tile_base[p.tile0 + t] = valid; valid += tile_valid[p.tile0 + t]; }
    uint8_t* body = raw + p.slot;
    WPageOut o{};
    o.st = pq::stats_empty();
    o.st.nulls = (unsigned long long)(p.rows - (int)valid);
    const uint32_t cap = 0xffffffffu;   // the host sized the slot for the worst case of every section
    uint32_t op = 0, lev_at = 0;
    if (p.kind == pq::KIND_DICT) {
        op = (uint32_t)p.rows * (uint32_t)p.width;
    } else {
        op = 4;
        if (valid == 0 || valid == (unsigned int)p.rows) pq::put_rle_run(body, cap, &op, (uint32_t)p.rows, valid ? 1u : 0u, 1);
        else {
            pq::put_packed_header(body, cap, &op, (uint32_t)p.rows);
            lev_at = op;
            op += pq::packed_body_len((uint32_t)p.rows, 1);
        }
        const uint32_t len = op - 4;
        body[0] = (uint8_t)len; body[1] = (uint8_t)(len >> 8); body[2] = (uint8_t)(len >> 16); body[3] = (uint8_t)(len >> 24);
    }
    uint32_t val_at = p.kind == pq::KIND_DICT ? 0 : op;
    if (p.kind != pq::KIND_DICT) {
        if (p.id_bw) {
            body[op++] = (uint8_t)p.id_bw;
            if (valid) pq::put_packed_header(body, cap, &op, valid);
            val_at = op;
            if (valid) op += pq::packed_body_len(valid, p.id_bw);
        } else {
            op += p.width ? valid * (uint32_t)p.width : (valid + 7) / 8;
        }
    }
    o.raw_len = op;
    o.comp_len = op;
    out[pi] = o;
    lay[pi] = make_uint2(lev_at, val_at);
}

// OR the low bw bits of v at bit `bit` of a 4-byte aligned body.
__device__ __forceinline__ void or_bits(uint8_t* body, unsigned long long bit, uint32_t v, int bw) {
    if (bw < 32) v &= (1u << bw) - 1u;
    if (!v) return;
    uint32_t* w = (uint32_t*)body + (bit >> 5);
    const int sh = (int)(bit & 31);
    atomicOr(w, v << sh);
    if (sh + bw > 32) atomicOr(w + 1, (uint32_t)((unsigned long long)v >> (32 - sh)));
}

__device__ __forceinline__ uint64_t load_value(const WTile& t, int in_width, int i) {
    const long long r = t.src_row + i;
    switch (in_width) {
        case 0: { const long long b = (long long)t.val_bit_off + r; return (((const uint32_t*)t.values)[b >> 5] >> (b & 31)) & 1; }
        case 1: return ((const uint8_t*)t.values)[r];
        case 2: return ((const uint16_t*)t.values)[r];
        case 4: return ((const uint32_t*)t.values)[r];
        default: return ((const unsigned long long*)t.values)[r];
    }
}

__global__ void __launch_bounds__(kThreads) k_pqw_encode(const WTile* __restrict__ tiles, const WPage* __restrict__ pages, const unsigned int* __restrict__ tile_base,
                                                         const uint2* __restrict__ lay, uint8_t* __restrict__ raw, WPageOut* __restrict__ out) {
    const WTile t = tiles[blockIdx.x];
    const WPage p = pages[t.page];
    const uint2 L = lay[t.page];
    uint8_t* body = raw + p.slot;
    const int i0 = threadIdx.x * kRowsPerThread;
    unsigned int vmask = 0, nv = 0;
    for (int k = 0; k < kRowsPerThread; k++)
        if (i0 + k < t.rows && tile_valid_bit(t, i0 + k)) { vmask |= 1u << k; nv++; }
    unsigned int total;
    unsigned int kv = tile_base[blockIdx.x] + cta_exclusive_scan(nv, &total);
    if (L.x && i0 < t.rows)   // mixed page: the level bits are the validity bits
        or_bits(body, (unsigned long long)L.x * 8 + (unsigned long long)(t.first + i0), vmask, kRowsPerThread);
    pq::Stats st = pq::stats_empty();
    const bool data = p.kind != pq::KIND_DICT;
    for (int k = 0; k < kRowsPerThread; k++) {
        if (!((vmask >> k) & 1)) continue;
        const int i = i0 + k;
        if (p.id_bw) {
            or_bits(body, (unsigned long long)L.y * 8 + (unsigned long long)kv * (unsigned)p.id_bw, t.ids[i], p.id_bw);
        } else if (!p.width) {
            or_bits(body, (unsigned long long)L.y * 8 + kv, (uint32_t)load_value(t, 0, i), 1);
        }
        const uint64_t v = p.width ? pq::convert(p.conv, p.in_width, load_value(t, p.in_width, i)) : load_value(t, 0, i);
        if (!p.id_bw && p.width) {
            uint8_t* d = body + L.y + (unsigned long long)kv * (unsigned)p.width;
            for (int b = 0; b < p.width; b++) d[b] = (uint8_t)(v >> (8 * b));
        }
        if (data) pq::stats_add(&st, p.ord, p.width ? p.width : 1, true, v);
        kv++;
    }
    if (!data) return;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long a = __shfl_xor_sync(0xffffffffu, st.kmin, o), b = __shfl_xor_sync(0xffffffffu, st.kmax, o),
                                 c = __shfl_xor_sync(0xffffffffu, st.count, o);
        st.kmin = a < st.kmin ? a : st.kmin;
        st.kmax = b > st.kmax ? b : st.kmax;
        st.count += c;
    }
    if ((threadIdx.x & 31) == 0 && st.count) {
        WPageOut* o = out + t.page;
        atomicMin(&o->st.kmin, st.kmin);
        atomicMax(&o->st.kmax, st.kmax);
        atomicAdd(&o->st.count, st.count);
    }
}

// One warp per fragment slot; frag_page[f]: the page the slot belongs to.
__global__ void __launch_bounds__(kSnappyWarps * 32) k_pqw_snappy(const WPage* __restrict__ pages, const int* __restrict__ frag_page, int n_frags,
                                                                  const uint8_t* __restrict__ raw, const WPageOut* __restrict__ out, uint8_t* __restrict__ frag,
                                                                  unsigned int* __restrict__ frag_len) {
    __shared__ uint16_t tables[kSnappyWarps][pq::kHashSize];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int f = blockIdx.x * kSnappyWarps + wib;
    if (f >= n_frags) return;
    uint16_t* table = tables[wib];
    const WPage p = pages[frag_page[f]];
    const uint32_t raw_len = out[frag_page[f]].raw_len;
    const uint32_t start = (uint32_t)(f - p.frag0) * pq::kFragment;
    const uint32_t n = start < raw_len ? min(pq::kFragment, raw_len - start) : 0u;
    const uint8_t* in = raw + p.slot + start;
    const uint32_t cap = pq::snappy_bound(pq::kFragment);
    uint8_t* o = frag + (long long)f * cap;
    for (uint32_t i = lane; i < pq::kHashSize; i += 32) table[i] = 0xffff;
    __syncwarp();
    uint32_t ip = 0, lit = 0, op = 0;
    bool ok = true;
    // a literal in[from, to): the tag by lane 0 (every lane computes the same op), the bytes by all lanes
    auto literal = [&](uint32_t from, uint32_t to) {
        uint32_t op2 = op;
        const bool fits = pq::snappy_literal_tag(to - from, o, cap, &op2);   // only the tag's bytes; each lane writes the same ones
        if (!fits) return false;
        __syncwarp();
        for (uint32_t j = lane; j < to - from; j += 32) o[op2 + j] = in[from + j];
        op = op2 + (to - from);
        return true;
    };
    while (ok && ip + 4 <= n) {
        const uint32_t pos = ip + lane;
        const bool act = pos + 4 <= n;
        const unsigned int act_mask = __ballot_sync(0xffffffffu, act);
        uint32_t h = 0, cand = pq::kEmpty;
        if (act) {
            h = pq::snappy_hash(pq::load32(in + pos));
            const uint16_t c = table[h];
            cand = c == 0xffff ? pq::kEmpty : c;
        }
        __syncwarp();
        if (act) {
            const unsigned int same = __match_any_sync(act_mask, h);
            if (lane == 31 - __clz(same)) table[h] = (uint16_t)pos;   // the last position of the window wins, as in snappy_fragment
        }
        __syncwarp();
        const bool hit = act && cand < pos && pq::load32(in + cand) == pq::load32(in + pos);
        const unsigned int hits = __ballot_sync(0xffffffffu, hit);
        if (!hits) { ip += pq::kWindow; continue; }
        const int fl = __ffs(hits) - 1;
        const uint32_t p0 = ip + fl, c0 = __shfl_sync(0xffffffffu, cand, fl);
        uint32_t len = 4;
        for (;;) {   // 32 bytes compared per step
            const uint32_t at = p0 + len + lane;
            const bool diff = at >= n || in[c0 + len + lane] != in[at];
            const unsigned int d = __ballot_sync(0xffffffffu, diff);
            if (d) { len += __ffs(d) - 1; break; }
            len += 32;
        }
        if (p0 > lit && !literal(lit, p0)) { ok = false; break; }
        ok = pq::snappy_copy(p0 - c0, len, o, cap, &op);   // every lane writes the same bytes
        __syncwarp();
        ip = lit = p0 + len;
    }
    if (ok && n > lit) ok = literal(lit, n);
    if (lane == 0) frag_len[f] = ok ? op : 0xffffffffu;
}

// One CTA per fragment slot: the page's preamble (fragment 0) and this fragment's bytes at their place in the compressed body.
__global__ void __launch_bounds__(kThreads) k_pqw_compact(const WPage* __restrict__ pages, const int* __restrict__ frag_page, const uint8_t* __restrict__ frag,
                                                          const unsigned int* __restrict__ frag_len, uint8_t* __restrict__ raw, WPageOut* __restrict__ out) {
    const int f = blockIdx.x;
    const int pi = frag_page[f];
    const WPage p = pages[pi];
    const uint32_t raw_len = out[pi].raw_len;
    const uint32_t pre = pq::uleb_len(raw_len);
    uint32_t at = pre, all = pre;
    bool bad = false;
    for (int j = 0; j < p.n_frags; j++) {
        const unsigned int l = frag_len[p.frag0 + j];
        if (l == 0xffffffffu) { bad = true; break; }
        if (p.frag0 + j < f) at += l;
        all += l;
    }
    if (bad) { if (threadIdx.x == 0) out[pi].err = 1; return; }
    uint8_t* body = raw + p.slot;
    const uint32_t cap = pq::snappy_bound(pq::kFragment);
    const unsigned int l = frag_len[f];
    for (uint32_t j = threadIdx.x; j < l; j += blockDim.x) body[at + j] = frag[(long long)f * cap + j];
    if (f == p.frag0 && threadIdx.x == 0) {
        uint32_t op = 0;
        pq::put_uleb(body, pre, &op, raw_len);
        out[pi].comp_len = all;
    }
}

cudaError_t launch_pqw_rgid(const long long* rg_start, int n_rg, long long n, uint32_t* out, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_pqw_rgid<<<(unsigned)std::min<long long>((n + kThreads - 1) / kThreads, 8LL * sm_count), kThreads, 0, s>>>(rg_start, n_rg, n, out);
    return cudaGetLastError();
}

cudaError_t launch_pqw_dict(const uint32_t* run_rg, const uint32_t* run_valid, long long n_runs, const uint32_t* head, const unsigned long long* prefix,
                            const uint32_t* perm, long long n, unsigned int* count, unsigned int* first, uint32_t* ids, int sm_count, cudaStream_t s) {
    if (n <= 0 || n_runs <= 0) return cudaSuccess;
    k_pqw_dict_runs<<<(unsigned)std::min<long long>((n_runs + kThreads - 1) / kThreads, 8LL * sm_count), kThreads, 0, s>>>(run_rg, run_valid, n_runs, count, first);
    k_pqw_dict_ids<<<(unsigned)std::min<long long>((n + kThreads - 1) / kThreads, 8LL * sm_count), kThreads, 0, s>>>(head, prefix, perm, run_rg, first, n, ids);
    return cudaGetLastError();
}

cudaError_t launch_pqw_encode(const void* pages, int n_pages, const void* tiles, int n_tiles, unsigned int* tile_valid, unsigned int* tile_base, void* lay,
                              uint8_t* raw, void* out, cudaStream_t s) {
    if (n_pages <= 0) return cudaSuccess;
    if (n_tiles) k_pqw_count<<<n_tiles, kThreads, 0, s>>>((const WTile*)tiles, tile_valid);
    k_pqw_layout<<<(n_pages + 127) / 128, 128, 0, s>>>((const WPage*)pages, n_pages, tile_valid, tile_base, raw, (uint2*)lay, (WPageOut*)out);
    if (n_tiles) k_pqw_encode<<<n_tiles, kThreads, 0, s>>>((const WTile*)tiles, (const WPage*)pages, tile_base, (const uint2*)lay, raw, (WPageOut*)out);
    return cudaGetLastError();
}

cudaError_t launch_pqw_snappy(const void* pages, const int* frag_page, int n_frags, uint8_t* raw, void* out, uint8_t* frag, unsigned int* frag_len,
                              cudaStream_t s) {
    if (n_frags <= 0) return cudaSuccess;
    k_pqw_snappy<<<(n_frags + kSnappyWarps - 1) / kSnappyWarps, kSnappyWarps * 32, 0, s>>>((const WPage*)pages, frag_page, n_frags, raw, (const WPageOut*)out,
                                                                                         frag, frag_len);
    k_pqw_compact<<<n_frags, kThreads, 0, s>>>((const WPage*)pages, frag_page, frag, frag_len, raw, (WPageOut*)out);
    return cudaGetLastError();
}

size_t pqw_page_bytes() { return sizeof(WPage); }
size_t pqw_tile_bytes() { return sizeof(WTile); }
size_t pqw_out_bytes() { return sizeof(WPageOut); }

}  // namespace bdf
