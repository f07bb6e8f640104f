// k_sort.cu -- DataFrame::sort (src/dataframe.rs:194-222): lexsort_to_indices over the criteria columns, then
// Column::take for every column (src/table.rs:218-241).  SURVEY 8(f) names sort right after the N4 row.
//
// arrow-rs lexsort_to_indices is a STABLE sort of row indices under a lexicographic comparator: per criterion, two
// valid slots compare by value (reversed when `descending`), a null slot is greater than any valid slot when
// nulls_first == false (the reference hard-codes false, :205-208) whatever `descending` says, two nulls are equal;
// floats compare with partial_cmp with NaN greater than everything and -0.0 == 0.0.  A stable LSD radix sort
// reproduces exactly that order: criteria are processed from the LAST to the FIRST; within a criterion the value is
// mapped to an order-preserving unsigned key (sign flip for ints; the usual float transform with -0.0 and NaN
// canonicalised; bitwise NOT for descending; 0 for null slots), sorted byte by byte, and a final 2-bucket pass on the
// null flag moves the nulls behind the valid rows without disturbing either group.
//
// Pass structure (per 8-bit digit): k_radix_hist (per-CTA digit counts over the CTA's contiguous range of tiles) ->
// k_scan_one (k_scan.cu: one CTA, exclusive scan in digit-major order) -> k_radix_scatter (per tile: warp-level peer masks from per-bit ballots -> ranks,
// reorder through shared memory, write each digit's run contiguously).  A digit on which every key agrees is skipped:
// k_sort_keys also folds the OR and the AND of the keys it builds.
// HBM traffic per executed pass: 8 (hist) + 12 + 12 B/row with 64-bit keys, 4 + 8 + 8 with 32-bit keys (criteria of at most
// 4 bytes); a Float64/Int64 criterion = 8 value passes (+1 if nullable), Int32/Float32 = 4 (+1).
#include "sort_keys.cuh"

#include <algorithm>

namespace bdf {

constexpr int kSortItems = 8;                          // keys per thread in the scatter kernel
constexpr int kSortThreads = 512;                      // scatter CTA: 16 warps
constexpr int kSortWarps = kSortThreads / 32;
constexpr int kSortTile = kSortThreads * kSortItems;   // 4096 keys per tile: a digit's run in a tile averages 16 keys (128 B of keys,
                                                       // 64 B of indices) on a uniformly distributed byte; 2048-key tiles were slower

// keys[i] = key of row idx[i] (idx == nullptr: row i) of the chunked column; mode 1: the null flag instead.
// Also folds the bitwise OR and AND of every key written into agree[0], agree[1]: a byte on which OR == AND is the
// same in all keys, so its radix pass would be the identity and is skipped.  (A first version accumulated the full
// 8 x 256 digit histogram with shared-memory atomics here; only "is the digit constant" was ever used.)
// Key width: 32-bit keys for criteria of at most 4 bytes (and their null flags), 64-bit otherwise -- a pass moves
// 4 + 8 + 8 B/row instead of 8 + 12 + 12.
template <typename T> struct KeyOf { using type = unsigned long long; };
template <> struct KeyOf<int8_t> { using type = uint32_t; };
template <> struct KeyOf<int16_t> { using type = uint32_t; };
template <> struct KeyOf<int32_t> { using type = uint32_t; };
template <> struct KeyOf<uint8_t> { using type = uint32_t; };
template <> struct KeyOf<uint16_t> { using type = uint32_t; };
template <> struct KeyOf<uint32_t> { using type = uint32_t; };
template <> struct KeyOf<float> { using type = uint32_t; };

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_sort_keys(const SortChunk* __restrict__ chunks, int n_chunks, const uint32_t* __restrict__ idx, int64_t n, int mode, int descending,
            typename KeyOf<T>::type* __restrict__ keys, unsigned long long* __restrict__ agree) {
    constexpr unsigned long long MASK = sizeof(T) == 8 ? ~0ull : ((1ull << (8 * (sizeof(T) & 7))) - 1ull);
    unsigned long long acc_or = 0ull, acc_and = ~0ull;
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) {
        const int64_t r = idx ? (int64_t)idx[i] : i;
        const int c = n_chunks == 1 ? 0 : chunk_of(chunks, n_chunks, r);
        const SortChunk ch = chunks[c];
        const int64_t local = r - ch.start;
        const bool valid = ch.validity ? chunk_bit(ch.validity, ch.bit_off + local) : true;
        unsigned long long k;
        if (mode) k = valid ? 0ull : 1ull;
        else {
            k = 0ull;
            if (valid) {
                k = SortKey<T>::of(((const T*)ch.values)[local]);
                if (descending) k = ~k & MASK;
            }
        }
        keys[i] = (typename KeyOf<T>::type)k;
        acc_or |= k;
        acc_and &= k;
    }
    const unsigned int or_lo = __reduce_or_sync(0xffffffffu, (unsigned int)acc_or), or_hi = __reduce_or_sync(0xffffffffu, (unsigned int)(acc_or >> 32));
    const unsigned int and_lo = __reduce_and_sync(0xffffffffu, (unsigned int)acc_and), and_hi = __reduce_and_sync(0xffffffffu, (unsigned int)(acc_and >> 32));
    if ((threadIdx.x & 31) == 0) {
        atomicOr(&agree[0], ((unsigned long long)or_hi << 32) | or_lo);
        atomicAnd(&agree[1], ((unsigned long long)and_hi << 32) | and_lo);
    }
}

__global__ void __launch_bounds__(kThreads) k_iota(uint32_t* __restrict__ out, int64_t n) {
    for (int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) out[i] = (uint32_t)i;
}

// ---- one radix pass -----------------------------------------------------------------------------------------------
// CTA b owns tiles [b * tiles_per_cta, ...): block_hist[d * G + b] = number of its keys with digit d.
template <typename K>
__global__ void __launch_bounds__(kThreads)
k_radix_hist(const K* __restrict__ keys, int64_t n, int shift, int64_t tiles_per_cta, unsigned int* __restrict__ block_hist) {
    __shared__ unsigned int s_hist[256];
    s_hist[threadIdx.x] = 0;
    __syncthreads();
    const int64_t begin = (int64_t)blockIdx.x * tiles_per_cta * kSortTile;
    const int64_t end = min(n, begin + tiles_per_cta * kSortTile);
    for (int64_t i = begin + threadIdx.x; i < end; i += kThreads) atomicAdd(&s_hist[(keys[i] >> shift) & 0xff], 1u);
    __syncthreads();
    block_hist[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] = s_hist[threadIdx.x];
}

// Lanes of the warp holding the same 9-bit value (digit, or 256 for "not a key"): one ballot per bit instead of MATCH.ANY.  A
// profile showed the scatter kernel bound by the pipe that executes MATCH (eight MATCH.ANY per thread and tile) while the ALU
// was mostly idle.  Nine VOTEs turned out to cost about what one MATCH costs: faster with 32-bit keys, slower with 64-bit
// keys -- so the ballots serve the 32-bit instantiation and MATCH.ANY stays in the 64-bit one.
__device__ __forceinline__ unsigned int digit_peers(unsigned int d) {
    unsigned int peers = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < 9; b++) {
        const bool bit = (d >> b) & 1u;
        const unsigned int m = __ballot_sync(0xffffffffu, bit);
        peers &= bit ? m : ~m;
    }
    return peers;
}

// Stable scatter of the CTA's tiles.  Within a tile, warp w owns elements [w*256, (w+1)*256) as 8 rows of 32 lanes, so
// (warp, row, lane) order is the input order; ranks come from match_any + per-warp digit counters.  Threads 0..255 own
// one digit each in the counting phases.
template <typename K> constexpr size_t scatter_smem() { return (size_t)kSortTile * (sizeof(K) + 4) + (size_t)kSortWarps * 256 * 4 + 2 * 256 * 4 + 8 * 4; }
template <typename K>
__global__ void __launch_bounds__(kSortThreads)
k_radix_scatter(const K* __restrict__ keys_in, const uint32_t* __restrict__ idx_in, int64_t n, int shift, int64_t tiles_per_cta,
                const unsigned int* __restrict__ block_offsets, K* __restrict__ keys_out, uint32_t* __restrict__ idx_out) {
    extern __shared__ __align__(16) unsigned char sort_smem[];
    K* s_key = reinterpret_cast<K*>(sort_smem);
    uint32_t* s_idx = reinterpret_cast<uint32_t*>(s_key + kSortTile);
    unsigned int (*s_cnt)[256] = reinterpret_cast<unsigned int (*)[256]>(s_idx + kSortTile);
    unsigned int* s_start = &s_cnt[kSortWarps][0];   // first slot of each digit's run in the sorted tile
    unsigned int* s_gbase = s_start + 256;           // global position of the next key of each digit written by this CTA
    unsigned int* s_wsum = s_gbase + 256;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned int lt_mask = (1u << lane) - 1u;
    if (tid < 256) s_gbase[tid] = block_offsets[(int64_t)tid * gridDim.x + blockIdx.x];
    const int64_t tile_begin = (int64_t)blockIdx.x * tiles_per_cta;
    for (int64_t t = tile_begin; t < tile_begin + tiles_per_cta; t++) {
        const int64_t base = t * kSortTile;
        if (base >= n) break;
        const int in_tile = (int)min((int64_t)kSortTile, n - base);
        for (int i = tid; i < kSortWarps * 256; i += kSortThreads) (&s_cnt[0][0])[i] = 0;
        __syncthreads();
        K key[kSortItems];
        uint32_t id[kSortItems];
        unsigned int rank[kSortItems];
#pragma unroll
        for (int it = 0; it < kSortItems; it++) {
            const int e = warp * (kSortItems * 32) + it * 32 + lane;
            const bool ok = e < in_tile;
            key[it] = ok ? keys_in[base + e] : (K)0;
            id[it] = ok ? idx_in[base + e] : 0u;
        }
#pragma unroll
        for (int it = 0; it < kSortItems; it++) {
            const int e = warp * (kSortItems * 32) + it * 32 + lane;
            const bool ok = e < in_tile;
            const unsigned int d = ok ? (unsigned int)((key[it] >> shift) & 0xff) : 256u;   // 256: not a key
            const unsigned int peers = sizeof(K) == 4 ? digit_peers(d) : __match_any_sync(0xffffffffu, d);
            const int leader = __ffs(peers) - 1;
            unsigned int old = 0;
            if (lane == leader && ok) { old = s_cnt[warp][d]; s_cnt[warp][d] = old + __popc(peers); }
            old = __shfl_sync(0xffffffffu, old, leader);
            rank[it] = old + __popc(peers & lt_mask);
            __syncwarp();
        }
        __syncthreads();
        // thread d < 256: exclusive prefix over the warps for digit d, then exclusive scan over the digits
        unsigned int run = 0, x = 0;
        if (tid < 256) {
#pragma unroll
            for (int w = 0; w < kSortWarps; w++) { const unsigned int c = s_cnt[w][tid]; s_cnt[w][tid] = run; run += c; }
            x = run;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const unsigned int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
            if (lane == 31) s_wsum[warp] = x;
        }
        __syncthreads();
        if (tid < 256) {
            unsigned int wbase = 0;
#pragma unroll
            for (int w = 0; w < 8; w++) wbase += (w < warp) ? s_wsum[w] : 0u;
            s_start[tid] = wbase + x - run;
        }
        __syncthreads();
#pragma unroll
        for (int it = 0; it < kSortItems; it++) {
            const int e = warp * (kSortItems * 32) + it * 32 + lane;
            if (e < in_tile) {
                const unsigned int d = (unsigned int)((key[it] >> shift) & 0xff);
                const unsigned int pos = s_start[d] + s_cnt[warp][d] + rank[it];
                s_key[pos] = key[it];
                s_idx[pos] = id[it];
            }
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kSortItems; k++) {
            const int sl = k * kSortThreads + tid;
            if (sl < in_tile) {
                const K kk = s_key[sl];
                const unsigned int d = (unsigned int)((kk >> shift) & 0xff);
                const unsigned int g = s_gbase[d] + ((unsigned int)sl - s_start[d]);
                keys_out[g] = kk;
                idx_out[g] = s_idx[sl];
            }
        }
        __syncthreads();
        if (tid < 256) s_gbase[tid] += run;   // thread d owns digit d
        __syncthreads();
    }
}

// ---- take -----------------------------------------------------------------------------------------------------------
// out[i] = values[indices[i]] over chunked values and chunked indices (concatenated row spaces); a null index or a null
// value gives a null slot with payload 0.  One row per thread: a warp assembles one validity word with a ballot.
// The gathered load asks L2 for 64 B around the address instead of the default 128 B, which about halves the DRAM bytes of a
// random gather of Float64 rows (benchmarks/gather_probe.cu).  The kernel is bound by the DRAM's random-access rate whatever
// the flavour of load, so the time hardly moves -- the halved traffic is for whoever shares the HBM with it.
template <typename T> __device__ __forceinline__ T gather_load(const T* p) {
    if constexpr (sizeof(T) == 8) { unsigned long long r; asm volatile("ld.global.L2::64B.u64 %0, [%1];" : "=l"(r) : "l"(p)); return bit_cast_to<T>(r); }
    else if constexpr (sizeof(T) == 4) { unsigned int r; asm volatile("ld.global.L2::64B.u32 %0, [%1];" : "=r"(r) : "l"(p)); return bit_cast_to<T>(r); }
    else if constexpr (sizeof(T) == 2) { unsigned short r; asm volatile("ld.global.L2::64B.u16 %0, [%1];" : "=h"(r) : "l"(p)); return bit_cast_to<T>(r); }
    else { unsigned int r; asm volatile("ld.global.L2::64B.u8 %0, [%1];" : "=r"(r) : "l"(p)); return bit_cast_to<T>((unsigned char)r); }
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_take(const SortChunk* __restrict__ vals, int n_vals, const SortChunk* __restrict__ idxs, int n_idxs, int64_t n, int64_t n_rows_values, T* __restrict__ out,
       uint32_t* __restrict__ vout, uint32_t* __restrict__ warp_counts, int* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    bool valid = false;
    T v = (T)0;
    if (i < n) {
        const int ic = n_idxs == 1 ? 0 : chunk_of(idxs, n_idxs, i);
        const SortChunk ich = idxs[ic];
        const int64_t il = i - ich.start;
        valid = ich.validity ? chunk_bit(ich.validity, ich.bit_off + il) : true;
        if (valid) {
            const int64_t r = (int64_t)((const uint32_t*)ich.values)[il];
            if (r >= n_rows_values) { atomicOr(flags, 1); valid = false; }   // arrow take: index out of bounds is an error
            else {
                const int c = n_vals == 1 ? 0 : chunk_of(vals, n_vals, r);
                const SortChunk ch = vals[c];
                const int64_t local = r - ch.start;
                valid = ch.validity ? chunk_bit(ch.validity, ch.bit_off + local) : true;
                if (valid) v = gather_load((const T*)ch.values + local);
            }
        }
        out[i] = v;
    }
    const unsigned int word = __ballot_sync(0xffffffffu, valid);
    if ((threadIdx.x & 31) == 0) {
        if (vout && (i < n)) vout[i >> 5] = word;
        if (vout) warp_counts[(int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5)] = __popc(word);
    }
}

// Boolean values: gather bits, one output word of values and one of validity per warp.
__global__ void __launch_bounds__(kThreads)
k_take_bool(const SortChunk* __restrict__ vals, int n_vals, const SortChunk* __restrict__ idxs, int n_idxs, int64_t n, int64_t n_rows_values,
            uint32_t* __restrict__ out, uint32_t* __restrict__ vout, uint32_t* __restrict__ warp_counts, int* __restrict__ flags) {
    const int64_t i = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    bool valid = false, bit = false;
    if (i < n) {
        const int ic = n_idxs == 1 ? 0 : chunk_of(idxs, n_idxs, i);
        const SortChunk ich = idxs[ic];
        const int64_t il = i - ich.start;
        valid = ich.validity ? chunk_bit(ich.validity, ich.bit_off + il) : true;
        if (valid) {
            const int64_t r = (int64_t)((const uint32_t*)ich.values)[il];
            if (r >= n_rows_values) { atomicOr(flags, 1); valid = false; }
            else {
                const int c = n_vals == 1 ? 0 : chunk_of(vals, n_vals, r);
                const SortChunk ch = vals[c];
                const int64_t local = r - ch.start;
                valid = ch.validity ? chunk_bit(ch.validity, ch.bit_off + local) : true;
                bit = valid && chunk_bit((const uint32_t*)ch.values, ch.val_bit_off + local);
            }
        }
    }
    const unsigned int vword = __ballot_sync(0xffffffffu, valid), bword = __ballot_sync(0xffffffffu, bit);
    if ((threadIdx.x & 31) == 0) {
        if (i < n) { out[i >> 5] = bword; if (vout) vout[i >> 5] = vword; }
        if (vout) warp_counts[(int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5)] = __popc(vword);
    }
}

// ---- launchers ------------------------------------------------------------------------------------------------------
size_t sort_chunk_size() { return sizeof(SortChunk); }
void fill_sort_chunk(void* base, int64_t i, const void* values, const uint32_t* validity, int64_t start, int32_t bit_off, int32_t val_bit_off) {
    SortChunk* c = (SortChunk*)base + i;
    c->values = values; c->validity = validity; c->start = start; c->bit_off = bit_off; c->val_bit_off = val_bit_off;
}
int sort_tile_elems() { return kSortTile; }
int take_tile_elems() { return kThreads; }

static int grid_for(int64_t n, int sm_count) {
    const int64_t want = (n + kThreads - 1) / kThreads;
    return (int)std::max<int64_t>(1, std::min<int64_t>(want, (int64_t)sm_count * 8));
}

cudaError_t launch_iota(uint32_t* out, int64_t n, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_iota<<<grid_for(n, sm_count), kThreads, 0, s>>>(out, n);
    return cudaGetLastError();
}

int sort_key_bytes(int dtype) { return dtype_width(dtype) <= 4 ? 4 : 8; }

cudaError_t launch_sort_keys(int dtype, const void* chunks, int n_chunks, const uint32_t* idx, int64_t n, int mode, int descending,
                             void* keys, unsigned long long* agree, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const SortChunk* ch = (const SortChunk*)chunks;
    const int g = grid_for(n, sm_count);
    switch (dtype) {
#define BDF_SORT_CASE(ID, T) case ID: k_sort_keys<T><<<g, kThreads, 0, s>>>(ch, n_chunks, idx, n, mode, descending, (typename KeyOf<T>::type*)keys, agree); break;
        BDF_SORT_CASE(0, int8_t) BDF_SORT_CASE(1, int16_t) BDF_SORT_CASE(2, int32_t) BDF_SORT_CASE(3, int64_t)
        BDF_SORT_CASE(4, uint8_t) BDF_SORT_CASE(5, uint16_t) BDF_SORT_CASE(6, uint32_t) BDF_SORT_CASE(7, uint64_t)
        BDF_SORT_CASE(8, float) BDF_SORT_CASE(9, double)
#undef BDF_SORT_CASE
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// One stable pass on bits [shift, shift+8).  block_hist: 256 * sort_pass_ctas(n, sm_count) counters.
int sort_pass_ctas(int64_t n, int sm_count) {
    const int64_t tiles = (n + kSortTile - 1) / kSortTile;
    return (int)std::max<int64_t>(1, std::min<int64_t>(tiles, (int64_t)sm_count * 4));
}
template <typename K>
static cudaError_t radix_pass(const K* keys_in, const uint32_t* idx_in, int64_t n, int shift, unsigned int* block_hist, K* keys_out, uint32_t* idx_out,
                              int sm_count, cudaStream_t s) {
    const int64_t tiles = (n + kSortTile - 1) / kSortTile;
    const int g = sort_pass_ctas(n, sm_count);
    const int64_t per = (tiles + g - 1) / g;
    static const cudaError_t attr = cudaFuncSetAttribute(k_radix_scatter<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)scatter_smem<K>());
    if (attr != cudaSuccess) return attr;
    k_radix_hist<K><<<g, kThreads, 0, s>>>(keys_in, n, shift, per, block_hist);
    const cudaError_t e = launch_scan_one<unsigned int>(block_hist, (long long)256 * g, nullptr, s);
    if (e != cudaSuccess) return e;
    k_radix_scatter<K><<<g, kSortThreads, scatter_smem<K>(), s>>>(keys_in, idx_in, n, shift, per, block_hist, keys_out, idx_out);
    return cudaGetLastError();
}
cudaError_t launch_radix_pass(int key_bytes, const void* keys_in, const uint32_t* idx_in, int64_t n, int shift, unsigned int* block_hist,
                              void* keys_out, uint32_t* idx_out, int sm_count, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    if (key_bytes == 4) return radix_pass<uint32_t>((const uint32_t*)keys_in, idx_in, n, shift, block_hist, (uint32_t*)keys_out, idx_out, sm_count, s);
    return radix_pass<unsigned long long>((const unsigned long long*)keys_in, idx_in, n, shift, block_hist, (unsigned long long*)keys_out, idx_out, sm_count, s);
}

cudaError_t launch_take(int dtype, const void* vals, int n_vals, const void* idxs, int n_idxs, int64_t n, int64_t n_rows_values, void* out,
                        uint32_t* vout, uint32_t* warp_counts, int* flags, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const int64_t g = (n + kThreads - 1) / kThreads;
    if (g > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    const SortChunk* v = (const SortChunk*)vals;
    const SortChunk* ix = (const SortChunk*)idxs;
    switch (dtype) {
#define BDF_TAKE_CASE(ID, T) case ID: k_take<T><<<(unsigned)g, kThreads, 0, s>>>(v, n_vals, ix, n_idxs, n, n_rows_values, (T*)out, vout, warp_counts, flags); break;
        BDF_TAKE_CASE(0, int8_t) BDF_TAKE_CASE(1, int16_t) BDF_TAKE_CASE(2, int32_t) BDF_TAKE_CASE(3, int64_t)
        BDF_TAKE_CASE(4, uint8_t) BDF_TAKE_CASE(5, uint16_t) BDF_TAKE_CASE(6, uint32_t) BDF_TAKE_CASE(7, uint64_t)
        BDF_TAKE_CASE(8, float) BDF_TAKE_CASE(9, double)
#undef BDF_TAKE_CASE
        case 10: k_take_bool<<<(unsigned)g, kThreads, 0, s>>>(v, n_vals, ix, n_idxs, n, n_rows_values, (uint32_t*)out, vout, warp_counts, flags); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

}  // namespace bdf
