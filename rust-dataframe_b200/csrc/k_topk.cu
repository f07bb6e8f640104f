// k_topk.cu -- the first k rows of DataFrame::sort without sorting every row (include/b200df.h "top-k").
//
// The host (runtime.cu top_k_indices_dev) works one criterion per round: the radix select of k_dist.cu finds the threshold key t of
// the rows still to choose, and k_topk_mark classifies every row of the round's tie set against it:
//   BEFORE  ascending key < t, descending key > t (or, when the tie set holds fewer valid values than rows still to choose, every
//           valid row); OR-ed into the "chosen" bitmap over all n rows;
//   TIE     key == t (or, in the second case, the null rows); written as a bitmap over the tie set's positions;
//   AFTER   everything else, nulls included (nulls sort last in both directions).
// Keys are SortKey<T> (sort_keys.cuh), so the classes follow the sort's order by construction: -0.0 == 0.0, every NaN one value
// above +inf.
//   Positional rounds (the tie set is every row: ids == null) write both bitmaps at the row's position.  A warp's 32 / E lanes that
//   share a bitmap word OR their bits together by shuffles, and the first of them stores the word: no atomics when the chunk's
//   first and last rows sit on word boundaries (the chunk owns its words); otherwise the word is OR-ed in with atomicOr across the
//   two words it straddles.  Plain stores are safe in the chosen bitmap because a tie set of every row means no row has been
//   chosen yet.
//   Gathered rounds (ids: the tie set's row numbers, ascending; the criterion was taken at them) write the TIE bitmap by position and
//   OR each BEFORE row into the chosen bitmap at its row number (atomicOr; OR commutes, so the bits do not depend on timing).
// The BEFORE and TIE counts are integer atomics, once per warp: exact.
//   k_topk_choose  OR the first `count` row numbers of a compacted TIE set into the chosen bitmap (the tie prefix in row order).
// The tile walk is k_dist's: kThreads x kUnroll vectors of 16 bytes per tile, grid strided, bounded (kThreads, 2).
#include <algorithm>

#include "common.cuh"
#include "sort_keys.cuh"

namespace bdf {

constexpr int kTopkCtasPerSm = 8;

struct TopkChunk {
    const void* values;
    const uint32_t* validity;
    int64_t len, tile0, row0;   // row0: the position of the chunk's first row in the bitmaps
    int32_t bit_off;
    int32_t owns_words;         // row0 and row0 + len are multiples of 32 (or the end of the column): plain word stores
};

struct TopkMark {
    unsigned long long t;       // the threshold key
    int all_valid;              // 1: BEFORE = every valid row, TIE = every null row
    int descending;
    const uint32_t* ids;        // gathered rounds: the row number of every tie-set position; null: positional
    uint32_t* chosen;           // bit per row
    uint32_t* tie;              // bit per tie-set position, zeroed by the caller
    unsigned long long* counts; // [0] BEFORE, [1] TIE
};

int topk_chunk_size() { return (int)sizeof(TopkChunk); }
int topk_tile_elems(int dtype) { return kThreads * kUnroll * (16 / dtype_width(dtype)); }

void fill_topk_chunk(void* descs, int64_t i, const void* values, const uint32_t* validity, int64_t len, int64_t tile0, int64_t row0, int bit_off,
                     bool owns_words) {
    ((TopkChunk*)descs)[i] = TopkChunk{values, validity, len, tile0, row0, bit_off, owns_words ? 1 : 0};
}

// A word of bits whose bit 0 is position p: stored when the chunk owns its words, else OR-ed into the one or two words it covers.
__device__ __forceinline__ void put_word(uint32_t* __restrict__ words, int64_t p, uint32_t bits, bool owns) {
    if (owns) { words[p >> 5] = bits; return; }
    if (!bits) return;
    const int sh = (int)(p & 31);
    atomicOr(words + (p >> 5), bits << sh);
    if (sh && (bits >> (32 - sh))) atomicOr(words + (p >> 5) + 1, bits >> (32 - sh));
}

template <typename T>
__global__ void __launch_bounds__(kThreads, 2)
k_topk_mark(const TopkChunk* __restrict__ chunks, int n_chunks, int64_t tiles, TopkMark mk) {
    constexpr int E = 16 / (int)sizeof(T);
    constexpr int TILE = kThreads * kUnroll * E;
    constexpr int G = 32 / E;   // lanes per bitmap word
    const int lane = threadIdx.x & 31;
    const unsigned long long t = mk.t;
    const bool all_valid = mk.all_valid != 0, desc = mk.descending != 0;
    const uint32_t* ids = mk.ids;
    unsigned long long n_before = 0, n_tie = 0;
#pragma unroll 1
    for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int c = n_chunks == 1 ? 0 : find_chunk(chunks, n_chunks, tile);
        const T* __restrict__ pi = (const T*)chunks[c].values;
        const uint32_t* __restrict__ vi = chunks[c].validity;
        const int64_t len = chunks[c].len, off = chunks[c].bit_off, row0 = chunks[c].row0;
        const bool owns = chunks[c].owns_words != 0;
        const int64_t base = (tile - chunks[c].tile0) * TILE;
        Vec<T, E> x[kUnroll];
        uint32_t m[kUnroll], in[kUnroll];
        if (base + TILE <= len) {
            const T* __restrict__ p = pi + base + (int64_t)threadIdx.x * E;
#pragma unroll
            for (int j = 0; j < kUnroll; j++) x[j].load(p + (int64_t)j * kThreads * E);
#pragma unroll
            for (int j = 0; j < kUnroll; j++) in[j] = (E == 32) ? 0xffffffffu : ((1u << E) - 1u);
            if (vi) {
                MaskRaw<E, kUnroll> rv;
                mask_issue<E, kUnroll>(rv, vi, off + base + (int64_t)threadIdx.x * E, kThreads * E);
#pragma unroll
                for (int j = 0; j < kUnroll; j++) m[j] = mask_get<E, kUnroll>(rv, j);
            } else {
#pragma unroll
                for (int j = 0; j < kUnroll; j++) m[j] = in[j];
            }
        } else {
#pragma unroll
            for (int j = 0; j < kUnroll; j++) {
                const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
                in[j] = tail_mask<E>(e0, len);
                m[j] = in[j];
                if (in[j] && vi) m[j] &= load_bits<E>(vi, off + e0);
#pragma unroll
                for (int e = 0; e < E; e++) x[j].e[e] = ((in[j] >> e) & 1u) ? pi[e0 + e] : (T)0;
            }
        }
#pragma unroll
        for (int j = 0; j < kUnroll; j++) {
            uint32_t before = 0, tie = 0;
            if (all_valid) {
                before = m[j];
                tie = in[j] & ~m[j];
            } else {
#pragma unroll
                for (int e = 0; e < E; e++) {
                    const unsigned long long k = SortKey<T>::of(x[j].e[e]);
                    const uint32_t valid = (m[j] >> e) & 1u;
                    before |= (valid & (desc ? k > t : k < t)) << e;
                    tie |= (valid & (k == t)) << e;
                }
            }
            n_before += __popc(before);
            n_tie += __popc(tie);
            const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
            if (ids && before) {
                uint32_t b = before;
                while (b) {
                    const int e = __ffs(b) - 1;
                    b &= b - 1;
                    const uint32_t row = __ldg(ids + e0 + e);
                    atomicOr(mk.chosen + (row >> 5), 1u << (row & 31));
                }
            }
            uint32_t wb = before << (E * (lane % G)), wt = tie << (E * (lane % G));
#pragma unroll
            for (int o = 1; o < G; o <<= 1) {
                wb |= __shfl_xor_sync(0xffffffffu, wb, o);
                wt |= __shfl_xor_sync(0xffffffffu, wt, o);
            }
            if ((lane % G) == 0 && e0 < len) {
                if (!ids) put_word(mk.chosen, row0 + e0, wb, owns);
                put_word(mk.tie, row0 + e0, wt, owns);
            }
        }
    }
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        n_before += __shfl_xor_sync(0xffffffffu, n_before, s);
        n_tie += __shfl_xor_sync(0xffffffffu, n_tie, s);
    }
    if (lane == 0) {
        if (n_before) atomicAdd(&mk.counts[0], n_before);
        if (n_tie) atomicAdd(&mk.counts[1], n_tie);
    }
}

__global__ void __launch_bounds__(kThreads)
k_topk_choose(const uint32_t* __restrict__ ids, long long count, uint32_t* __restrict__ chosen) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= count) return;
    const uint32_t row = __ldg(ids + i);
    atomicOr(chosen + (row >> 5), 1u << (row & 31));
}

template <typename T>
static cudaError_t mark_one(const void* chunks, int n_chunks, int64_t tiles, const TopkMark& mk, int sm_count, cudaStream_t s) {
    const unsigned grid = (unsigned)std::min<int64_t>(tiles, (int64_t)sm_count * kTopkCtasPerSm);
    k_topk_mark<T><<<grid, kThreads, 0, s>>>((const TopkChunk*)chunks, n_chunks, tiles, mk);
    return cudaGetLastError();
}

cudaError_t launch_topk_mark(int dtype, const void* chunks, int n_chunks, int64_t tiles, unsigned long long t, bool all_valid, bool descending,
                             const uint32_t* ids, uint32_t* chosen, uint32_t* tie, unsigned long long* counts, int sm_count, cudaStream_t s) {
    if (tiles <= 0) return cudaSuccess;
    const TopkMark mk{t, all_valid ? 1 : 0, descending ? 1 : 0, ids, chosen, tie, counts};
    switch (dtype) {
        case T_I8: return mark_one<int8_t>(chunks, n_chunks, tiles, mk, sm_count, s);
        case T_I16: return mark_one<int16_t>(chunks, n_chunks, tiles, mk, sm_count, s);
        case T_I32: return mark_one<int32_t>(chunks, n_chunks, tiles, mk, sm_count, s);
        case T_I64: return mark_one<int64_t>(chunks, n_chunks, tiles, mk, sm_count, s);
        case T_U8: return mark_one<uint8_t>(chunks, n_chunks, tiles, mk, sm_count, s);
        case T_U16: return mark_one<uint16_t>(chunks, n_chunks, tiles, mk, sm_count, s);
        case T_U32: return mark_one<uint32_t>(chunks, n_chunks, tiles, mk, sm_count, s);
        case T_U64: return mark_one<uint64_t>(chunks, n_chunks, tiles, mk, sm_count, s);
        case T_F32: return mark_one<float>(chunks, n_chunks, tiles, mk, sm_count, s);
        case T_F64: return mark_one<double>(chunks, n_chunks, tiles, mk, sm_count, s);
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_topk_choose(const uint32_t* ids, long long count, uint32_t* chosen, cudaStream_t s) {
    if (count <= 0) return cudaSuccess;
    const long long blocks = (count + kThreads - 1) / kThreads;
    if (blocks > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    k_topk_choose<<<(unsigned)blocks, kThreads, 0, s>>>(ids, count, chosen);
    return cudaGetLastError();
}

}  // namespace bdf
