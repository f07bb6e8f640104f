// k_dist.cu -- column distributions (include/b200df.h "distributions"): the MSD radix select behind the exact percentiles, the
// equal-width histogram, and the run kernels of mode, uniques and the per-group median.
//
// Streaming kernels (select histogram, select compaction, range, histogram) walk k_reduce's chunk descriptors tile by tile, grid
// strided: a tile is kThreads x kUnroll vectors of 16 bytes, read with the validity bits at the chunk's bit offset.  Every lane
// visits every element slot of its tile (invalid ones with a flag), so warp-collective steps inside the per-element body are safe.
//   k_sel_hist     the digit histogram of the candidate keys: a key is a candidate when its decided high bits equal one of the m
//                  sorted prefixes (binary search); bin = prefix index * 256 + digit.  Up to kSelSmemBins bins are counted per CTA in
//                  shared memory (u32) and merged into the global u64 histogram; more go straight to global atomics.  Increments are
//                  warp-aggregated with __match_any_sync, so a column of one value costs one atomic per warp step, not 32 on one bank.
//                  The AND and OR of the candidate keys come back too: bits where they agree need no digit pass.
//   k_sel_compact  the candidates whose bucket was chosen, appended to a scratch buffer through one warp-aggregated atomic cursor
//                  (selection does not depend on order).  Later digits read only that buffer, as RAW keys.
//   k_dist_range   the smallest and largest non-NaN valid value (order-preserving keys, atomicMin / atomicMax once per warp).
//   k_hist         numpy.histogram's uniform-bin rule with its one-step correction against the edges.  Up to kHistSmemBins bins the
//                  edges are staged in shared memory and the bins privatised per CTA; beyond, edges come from global memory and
//                  bins are global u64 atomics.  Warp-aggregated like k_sel_hist.
// Every count is an integer, so atomics leave the results exact and independent of scheduling.
// The streaming kernels are bounded (kThreads, 2): with (kThreads) alone ptxas spilled 4-8 bytes in the select kernels.
//   k_dist_groups  per group: its first distinct run (lower bound in the run heads) and the end of its valid prefix (nulls sort
//                  last inside a group in the second sort: a binary search over the sorted validity bits).
//   k_dist_runs    per distinct run: its row count (the next head in the group, else the valid end); optionally each group's
//                  atomicMax of (count << 32) | (0xffffffff - rank in group), whose maximum is the most frequent, smallest value.
//   k_dist_mode    per group: the sorted row of that run (a gather index, NULL without a valid value) and its count.
//   k_dist_median  per group: the two order statistics of the valid prefix, interpolated by dist_interp.
#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "dist.cuh"
#include "sort_keys.cuh"

namespace bdf {

constexpr int kSelSmemBins = 8192;    // 32 KiB of u32 bins: up to 32 prefixes of 256 digits per CTA in shared memory
constexpr int kHistSmemBins = 2048;   // edges (16 KiB) + u32 bins (8 KiB) in shared memory
constexpr int kDistCtasPerSm = 8;

template <typename T> struct KeyOf { using type = typename std::conditional<sizeof(T) <= 4, uint32_t, unsigned long long>::type; };

int dist_tile_elems(int dtype) { return kThreads * kUnroll * (16 / dtype_width(dtype)); }

// The grid-strided tile walk over the chunks of descs; f(value, valid) for every element slot of every tile of this CTA.
template <typename T, typename F>
__device__ __forceinline__ void dist_walk(const RedDesc* __restrict__ descs, int n_chunks, int64_t total_tiles, F& f) {
    constexpr int E = 16 / (int)sizeof(T);
    constexpr int TILE = kThreads * kUnroll * E;
#pragma unroll 1
    for (int64_t tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int c = n_chunks == 1 ? 0 : find_chunk(descs, n_chunks, tile);
        const T* __restrict__ pi = (const T*)descs[c].in;
        const uint32_t* __restrict__ vi = descs[c].vin;
        const int64_t len = descs[c].len, off = descs[c].off;
        const int64_t base = (tile - descs[c].tile0) * TILE;
        Vec<T, E> x[kUnroll];
        uint32_t m[kUnroll];
        if (base + TILE <= len) {
            const T* __restrict__ p = pi + base + (int64_t)threadIdx.x * E;
#pragma unroll
            for (int j = 0; j < kUnroll; j++) x[j].load(p + (int64_t)j * kThreads * E);
            if (vi) {
                MaskRaw<E, kUnroll> rv;
                mask_issue<E, kUnroll>(rv, vi, off + base + (int64_t)threadIdx.x * E, kThreads * E);
#pragma unroll
                for (int j = 0; j < kUnroll; j++) m[j] = mask_get<E, kUnroll>(rv, j);
            } else {
#pragma unroll
                for (int j = 0; j < kUnroll; j++) m[j] = (E == 32) ? 0xffffffffu : ((1u << E) - 1u);
            }
        } else {
#pragma unroll
            for (int j = 0; j < kUnroll; j++) {
                const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
                const uint32_t in_range = tail_mask<E>(e0, len);
                m[j] = in_range;
                if (in_range && vi) m[j] &= load_bits<E>(vi, off + e0);
#pragma unroll
                for (int e = 0; e < E; e++) x[j].e[e] = ((in_range >> e) & 1u) ? pi[e0 + e] : (T)0;
            }
        }
#pragma unroll
        for (int j = 0; j < kUnroll; j++)
#pragma unroll
            for (int e = 0; e < E; e++) f(x[j].e[e], (m[j] >> e) & 1u);
    }
}

// One warp-aggregated increment of bin (< 0: none); every lane of the warp calls it.
__device__ __forceinline__ void warp_count(int bin, unsigned int* __restrict__ sh, unsigned long long* __restrict__ gl) {
    const unsigned peers = __match_any_sync(0xffffffffu, bin);
    if (bin >= 0 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) {
        if (sh) atomicAdd(&sh[bin], (unsigned)__popc(peers));
        else atomicAdd(&gl[bin], (unsigned long long)__popc(peers));
    }
}

// The index of (key & pmask) among the m sorted prefixes, or -1.  step0: the largest power of two <= m - 1 (0 when m == 1): the
// search takes the same steps in every lane, so the warp stays converged for the collective that follows.
template <typename K>
__device__ __forceinline__ int prefix_index(K key, K pmask, const unsigned long long* __restrict__ prefixes, int m, int step0) {
    const unsigned long long k = (unsigned long long)(key & pmask);
    int lo = 0;
    for (int s = step0; s > 0; s >>= 1) lo = (lo + s < m && __ldg(&prefixes[lo + s]) <= k) ? lo + s : lo;
    return __ldg(&prefixes[lo]) == k ? lo : -1;
}

template <typename T, bool RAW>
__device__ __forceinline__ typename KeyOf<T>::type key_of(T v) {
    if constexpr (RAW) return v;
    else return (typename KeyOf<T>::type)SortKey<T>::of(v);
}

struct SelLevel {
    const unsigned long long* prefixes;   // m sorted prefixes (the decided high bits, lower bits zero)
    unsigned long long pmask;             // the decided bits
    int m;
    int shift;                            // the digit is bits [shift, shift + 8) of the key
};

// ---- select: digit histogram ------------------------------------------------------------------------------------------------
template <typename T, bool RAW>
__global__ void __launch_bounds__(kThreads, 2)
k_sel_hist(const RedDesc* __restrict__ descs, int n_chunks, int64_t tiles, SelLevel lv, unsigned long long* __restrict__ hist,
           unsigned long long* __restrict__ and_or) {
    using K = typename KeyOf<T>::type;
    extern __shared__ unsigned int s_bins[];
    const int n_bins = lv.m * 256;
    unsigned int* sh = n_bins <= kSelSmemBins ? s_bins : nullptr;
    if (sh) {
        for (int b = threadIdx.x; b < n_bins; b += kThreads) sh[b] = 0;
        __syncthreads();
    }
    K a = (K)~(K)0, o = 0;
    // kernel parameters are copied to locals: a lambda capturing a parameter by reference would take its address (a stack copy)
    const K pmask = (K)lv.pmask;
    const unsigned long long* prefixes = lv.prefixes;
    const int m = lv.m, shift = lv.shift, step0 = m > 1 ? 1 << (31 - __clz(m - 1)) : 0;
    unsigned long long* gl = hist;
    auto f = [&](T v, uint32_t valid) {
        const K key = key_of<T, RAW>(v);
        const int cls = valid ? prefix_index<K>(key, pmask, prefixes, m, step0) : -1;
        const bool in = cls >= 0;
        const int bin = in ? cls * 256 + (int)((key >> shift) & 255u) : -1;
        a &= in ? key : (K)~(K)0;
        o |= in ? key : (K)0;
        warp_count(bin, sh, gl);
    };
    dist_walk<T>(descs, n_chunks, tiles, f);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        a &= __shfl_xor_sync(0xffffffffu, a, s);
        o |= __shfl_xor_sync(0xffffffffu, o, s);
    }
    if ((threadIdx.x & 31) == 0) {
        atomicAnd(&and_or[0], (unsigned long long)a | (sizeof(K) == 4 ? 0xffffffff00000000ull : 0ull));
        atomicOr(&and_or[1], (unsigned long long)o);
    }
    if (sh) {
        __syncthreads();
        for (int b = threadIdx.x; b < n_bins; b += kThreads)
            if (sh[b]) atomicAdd(&hist[b], (unsigned long long)sh[b]);
    }
}

// ---- select: compaction of the chosen buckets -----------------------------------------------------------------------------
template <typename T, bool RAW>
__global__ void __launch_bounds__(kThreads, 2)
k_sel_compact(const RedDesc* __restrict__ descs, int n_chunks, int64_t tiles, SelLevel lv, const uint32_t* __restrict__ chosen,
              typename KeyOf<T>::type* __restrict__ out, unsigned long long* __restrict__ cursor) {
    using K = typename KeyOf<T>::type;
    const K pmask = (K)lv.pmask;
    const unsigned long long* prefixes = lv.prefixes;
    const int m = lv.m, shift = lv.shift, step0 = m > 1 ? 1 << (31 - __clz(m - 1)) : 0;
    const uint32_t* ch = chosen;
    K* dst = out;
    unsigned long long* cur = cursor;
    const unsigned lane = threadIdx.x & 31;
    auto f = [&](T v, uint32_t valid) {
        const K key = key_of<T, RAW>(v);
        const int cls = valid ? prefix_index<K>(key, pmask, prefixes, m, step0) : -1;
        const int bin = cls >= 0 ? cls * 256 + (int)((key >> shift) & 255u) : 0;
        const bool keep = cls >= 0 && ((__ldg(&ch[bin >> 5]) >> (bin & 31)) & 1u);
        const unsigned ballot = __ballot_sync(0xffffffffu, keep);
        if (!ballot) return;
        unsigned long long base = 0;
        if (lane == (unsigned)(__ffs(ballot) - 1)) base = atomicAdd(cur, (unsigned long long)__popc(ballot));
        base = __shfl_sync(0xffffffffu, base, __ffs(ballot) - 1);
        if (keep) dst[base + __popc(ballot & ((1u << lane) - 1u))] = key;
    };
    dist_walk<T>(descs, n_chunks, tiles, f);
}

// ---- histogram: range and counts ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(kThreads, 2)
k_dist_range(const RedDesc* __restrict__ descs, int n_chunks, int64_t tiles, unsigned long long* __restrict__ min_max) {
    unsigned long long kmin = ~0ull, kmax = 0;
    bool any = false;
    auto f = [&](T v, uint32_t valid) {
        if (valid && v == v) {   // NaN is never counted
            const unsigned long long k = SortKey<T>::of(v);
            kmin = k < kmin ? k : kmin;
            kmax = k > kmax ? k : kmax;
            any = true;
        }
    };
    dist_walk<T>(descs, n_chunks, tiles, f);
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
        const unsigned long long a = __shfl_xor_sync(0xffffffffu, kmin, s), b = __shfl_xor_sync(0xffffffffu, kmax, s);
        kmin = a < kmin ? a : kmin;
        kmax = b > kmax ? b : kmax;
    }
    const bool warp_any = __any_sync(0xffffffffu, any);
    if ((threadIdx.x & 31) == 0 && warp_any) {
        atomicMin(&min_max[0], kmin);
        atomicMax(&min_max[1], kmax);
    }
}

struct HistParams {
    const double* edges;   // nbins + 1
    double lo, hi;         // edges[0], edges[nbins]
    int nbins;
};

template <typename T>
__global__ void __launch_bounds__(kThreads, 2)
k_hist(const RedDesc* __restrict__ descs, int n_chunks, int64_t tiles, HistParams hp, unsigned long long* __restrict__ counts) {
    extern __shared__ double s_edges[];
    const int nb = hp.nbins;
    const bool priv = nb <= kHistSmemBins;
    unsigned int* sh = priv ? (unsigned int*)(s_edges + nb + 1) : nullptr;
    const double* edges = hp.edges;
    if (priv) {
        for (int b = threadIdx.x; b <= nb; b += kThreads) s_edges[b] = hp.edges[b];
        for (int b = threadIdx.x; b < nb; b += kThreads) sh[b] = 0;
        __syncthreads();
        edges = s_edges;
    }
    const double lo = hp.lo, hi = hp.hi, denom = __dsub_rn(hi, lo), fnb = (double)nb;
    unsigned long long* gl = counts;
    auto f = [&](T v, uint32_t valid) {
        int bin = -1;
        const double x = (double)v;
        if (valid && x >= lo && x <= hi) {   // false for NaN
            long long i = (long long)__dmul_rn(__ddiv_rn(__dsub_rn(x, lo), denom), fnb);
            if (i >= nb) i = nb - 1;
            if (i < 0) i = 0;
            if (x < edges[i]) i--;
            else if (i != nb - 1 && x >= edges[i + 1]) i++;
            bin = (int)i;
        }
        warp_count(bin, sh, gl);
    };
    dist_walk<T>(descs, n_chunks, tiles, f);
    if (priv) {
        __syncthreads();
        for (int b = threadIdx.x; b < nb; b += kThreads)
            if (sh[b]) atomicAdd(&counts[b], (unsigned long long)sh[b]);
    }
}

// ---- runs: mode, uniques, per-group median --------------------------------------------------------------------------------
__device__ __forceinline__ long long lower_bound_pos(const uint32_t* __restrict__ a, long long n, long long x) {
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if ((long long)a[mid] < x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__global__ void k_dist_groups(const uint32_t* __restrict__ starts, long long n_groups, long long n_rows, const uint32_t* __restrict__ pos,
                              long long n_pos, const uint32_t* __restrict__ valid, uint32_t* __restrict__ first_run, uint32_t* __restrict__ vend) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_groups) return;
    const long long s = starts[g], e = g + 1 < n_groups ? (long long)starts[g + 1] : n_rows;
    if (first_run) first_run[g] = (uint32_t)lower_bound_pos(pos, n_pos, s);
    long long lo = s, hi = e;   // the first null of the group (valid values first)
    if (valid)
        while (lo < hi) {
            const long long mid = (lo + hi) >> 1;
            if ((valid[mid >> 5] >> (mid & 31)) & 1u) lo = mid + 1; else hi = mid;
        }
    else lo = e;
    vend[g] = (uint32_t)lo;
}

__global__ void k_dist_runs(const uint32_t* __restrict__ pos, long long n_pos, const uint32_t* __restrict__ starts, long long n_groups,
                            long long n_rows, const uint32_t* __restrict__ first_run, const uint32_t* __restrict__ vend,
                            long long* __restrict__ counts, unsigned long long* __restrict__ best) {
    const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long g = -1;
    unsigned long long packed = 0;
    if (k < n_pos) {
        const long long p = pos[k];
        long long lo = 0, hi = n_groups - 1;   // the last group starting at or before p
        while (lo < hi) {
            const long long mid = (lo + hi + 1) >> 1;
            if ((long long)starts[mid] <= p) lo = mid; else hi = mid - 1;
        }
        g = lo;
        const long long ge = g + 1 < n_groups ? (long long)starts[g + 1] : n_rows;
        const long long nxt = (k + 1 < n_pos && (long long)pos[k + 1] < ge) ? (long long)pos[k + 1] : (long long)vend[g];
        const long long cnt = nxt - p;
        if (counts) counts[k] = cnt;
        packed = ((unsigned long long)cnt << 32) | (0xffffffffull - (unsigned long long)(k - first_run[g]));
    }
    if (!best) return;
    // few groups (the whole column is one): a warp, then a CTA, whose runs share a group makes one atomic instead of one per run
    __shared__ long long s_g[kWarpsPerCta];
    __shared__ unsigned long long s_p[kWarpsPerCta];
    const bool uniform = __match_any_sync(0xffffffffu, g) == 0xffffffffu && g >= 0;
    if (uniform) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            const unsigned long long q = __shfl_xor_sync(0xffffffffu, packed, o);
            packed = q > packed ? q : packed;
        }
    } else if (g >= 0) {
        atomicMax(&best[g], packed);
    }
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { s_g[w] = uniform ? g : -1; s_p[w] = packed; }
    __syncthreads();
    if (threadIdx.x == 0) {
        bool all = s_g[0] >= 0;
        unsigned long long m = s_p[0];
        for (int i = 1; i < kWarpsPerCta; i++) { all = all && s_g[i] == s_g[0]; m = s_p[i] > m ? s_p[i] : m; }
        if (all) atomicMax(&best[s_g[0]], m);
        else
            for (int i = 0; i < kWarpsPerCta; i++)
                if (s_g[i] >= 0) atomicMax(&best[s_g[i]], s_p[i]);
    }
}

__global__ void k_dist_mode(const unsigned long long* __restrict__ best, long long n_groups, const uint32_t* __restrict__ first_run,
                            const uint32_t* __restrict__ pos, uint32_t* __restrict__ row, uint32_t* __restrict__ row_valid,
                            long long* __restrict__ freq) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long b = g < n_groups ? best[g] : 0ull;
    const bool some = b != 0;
    const unsigned w = __ballot_sync(0xffffffffu, some);
    if (g >= n_groups) return;
    if ((threadIdx.x & 31) == 0) row_valid[g >> 5] = w;
    row[g] = some ? pos[first_run[g] + (0xffffffffull - (b & 0xffffffffull))] : 0u;
    if (freq) freq[g] = (long long)(b >> 32);
}

template <typename T>
__global__ void k_dist_median(const T* __restrict__ sval, const uint32_t* __restrict__ starts, long long n_groups, const uint32_t* __restrict__ vend,
                              double* __restrict__ out, uint32_t* __restrict__ out_valid) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    double r = 0.0;
    bool some = false;
    if (g < n_groups) {
        const long long s = starts[g], v = (long long)vend[g] - s;
        if (v > 0) {
            const double p = __dmul_rn((double)(v - 1), 0.5), lo = floor(p), hi = ceil(p);
            r = dist_interp((double)sval[s + (long long)lo], (double)sval[s + (long long)hi], p, lo, hi);
            some = true;
        }
    }
    const unsigned w = __ballot_sync(0xffffffffu, some);
    if (g >= n_groups) return;
    if ((threadIdx.x & 31) == 0) out_valid[g >> 5] = w;
    out[g] = r;
}

// ---- launchers --------------------------------------------------------------------------------------------------------------
static unsigned dist_grid(int64_t tiles, int sm_count) { return (unsigned)std::min<int64_t>(tiles, (int64_t)sm_count * kDistCtasPerSm); }

template <typename T, bool RAW>
static cudaError_t sel_one(bool compact, const RedDesc* d, int n, int64_t tiles, const SelLevel& lv, unsigned long long* hist,
                           unsigned long long* and_or, const uint32_t* chosen, void* out, unsigned long long* cursor, int sm_count, cudaStream_t s) {
    if (tiles <= 0) return cudaSuccess;
    const unsigned grid = dist_grid(tiles, sm_count);
    if (compact) {
        k_sel_compact<T, RAW><<<grid, kThreads, 0, s>>>(d, n, tiles, lv, chosen, (typename KeyOf<T>::type*)out, cursor);
    } else {
        const size_t smem = lv.m * 256 <= kSelSmemBins ? (size_t)lv.m * 256 * sizeof(unsigned) : 0;
        k_sel_hist<T, RAW><<<grid, kThreads, smem, s>>>(d, n, tiles, lv, hist, and_or);
    }
    return cudaGetLastError();
}

// One select pass over the chunks in d (key_bytes 0: a column of dtype, read through SortKey; 4 / 8: a scratch buffer of raw keys).
// compact = false: the digit histogram (lv.m x 256 u64 bins, zeroed by the caller) and the AND / OR of the candidate keys
// (initialised by the caller); true: the keys of the chosen buckets appended at *cursor.
cudaError_t launch_select_pass(int dtype, int key_bytes, bool compact, const RedDesc* d, int n, int64_t tiles, const unsigned long long* prefixes,
                               int m, unsigned long long pmask, int shift, unsigned long long* hist, unsigned long long* and_or,
                               const uint32_t* chosen, void* out, unsigned long long* cursor, int sm_count, cudaStream_t s) {
    if (m < 1 || shift < 0 || shift > 56) return cudaErrorInvalidValue;
    const SelLevel lv{prefixes, pmask, m, shift};
    if (key_bytes == 4) return sel_one<uint32_t, true>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
    if (key_bytes == 8) return sel_one<unsigned long long, true>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
    switch (dtype) {
        case T_I8: return sel_one<int8_t, false>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
        case T_I16: return sel_one<int16_t, false>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
        case T_I32: return sel_one<int32_t, false>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
        case T_I64: return sel_one<int64_t, false>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
        case T_U8: return sel_one<uint8_t, false>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
        case T_U16: return sel_one<uint16_t, false>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
        case T_U32: return sel_one<uint32_t, false>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
        case T_U64: return sel_one<uint64_t, false>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
        case T_F32: return sel_one<float, false>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
        case T_F64: return sel_one<double, false>(compact, d, n, tiles, lv, hist, and_or, chosen, out, cursor, sm_count, s);
        default: return cudaErrorInvalidValue;
    }
}

template <typename T>
static cudaError_t hist_one(bool range, const RedDesc* d, int n, int64_t tiles, const HistParams& hp, unsigned long long* out, int sm_count,
                            cudaStream_t s) {
    if (tiles <= 0) return cudaSuccess;
    const unsigned grid = dist_grid(tiles, sm_count);
    if (range) {
        k_dist_range<T><<<grid, kThreads, 0, s>>>(d, n, tiles, out);
    } else {
        const size_t smem = hp.nbins <= kHistSmemBins ? (size_t)(hp.nbins + 1) * sizeof(double) + (size_t)hp.nbins * sizeof(unsigned) : 0;
        k_hist<T><<<grid, kThreads, smem, s>>>(d, n, tiles, hp, out);
    }
    return cudaGetLastError();
}

// range = true: the order-preserving keys of the smallest and largest non-NaN valid value into out[0] / out[1] (initialised by the
// caller to ~0 / 0); false: the counts of the nbins bins into out (zeroed by the caller).
cudaError_t launch_hist(int dtype, bool range, const RedDesc* d, int n, int64_t tiles, const double* edges, double lo, double hi, int nbins,
                        unsigned long long* out, int sm_count, cudaStream_t s) {
    const HistParams hp{edges, lo, hi, nbins};
    switch (dtype) {
        case T_I8: return hist_one<int8_t>(range, d, n, tiles, hp, out, sm_count, s);
        case T_I16: return hist_one<int16_t>(range, d, n, tiles, hp, out, sm_count, s);
        case T_I32: return hist_one<int32_t>(range, d, n, tiles, hp, out, sm_count, s);
        case T_I64: return hist_one<int64_t>(range, d, n, tiles, hp, out, sm_count, s);
        case T_U8: return hist_one<uint8_t>(range, d, n, tiles, hp, out, sm_count, s);
        case T_U16: return hist_one<uint16_t>(range, d, n, tiles, hp, out, sm_count, s);
        case T_U32: return hist_one<uint32_t>(range, d, n, tiles, hp, out, sm_count, s);
        case T_U64: return hist_one<uint64_t>(range, d, n, tiles, hp, out, sm_count, s);
        case T_F32: return hist_one<float>(range, d, n, tiles, hp, out, sm_count, s);
        case T_F64: return hist_one<double>(range, d, n, tiles, hp, out, sm_count, s);
        default: return cudaErrorInvalidValue;
    }
}

static unsigned blocks_for(long long n) { return (unsigned)((n + kThreads - 1) / kThreads); }

// Per group: first_run (may be null when pos is) and vend, the end of the valid prefix (valid: the sorted validity, null = all valid).
cudaError_t launch_dist_groups(const uint32_t* starts, long long n_groups, long long n_rows, const uint32_t* pos, long long n_pos, const uint32_t* valid,
                               uint32_t* first_run, uint32_t* vend, cudaStream_t s) {
    if (n_groups <= 0) return cudaSuccess;
    k_dist_groups<<<blocks_for(n_groups), kThreads, 0, s>>>(starts, n_groups, n_rows, pos, n_pos, valid, first_run, vend);
    return cudaGetLastError();
}

// Per run: its count (counts may be null) and the per-group best (may be null; zeroed by the caller).
cudaError_t launch_dist_runs(const uint32_t* pos, long long n_pos, const uint32_t* starts, long long n_groups, long long n_rows, const uint32_t* first_run,
                             const uint32_t* vend, long long* counts, unsigned long long* best, cudaStream_t s) {
    if (n_pos <= 0) return cudaSuccess;
    k_dist_runs<<<blocks_for(n_pos), kThreads, 0, s>>>(pos, n_pos, starts, n_groups, n_rows, first_run, vend, counts, best);
    return cudaGetLastError();
}

cudaError_t launch_dist_mode(const unsigned long long* best, long long n_groups, const uint32_t* first_run, const uint32_t* pos, uint32_t* row,
                             uint32_t* row_valid, long long* freq, cudaStream_t s) {
    if (n_groups <= 0) return cudaSuccess;
    k_dist_mode<<<blocks_for(n_groups), kThreads, 0, s>>>(best, n_groups, first_run, pos, row, row_valid, freq);
    return cudaGetLastError();
}

cudaError_t launch_dist_median(int dtype, const void* sval, const uint32_t* starts, long long n_groups, const uint32_t* vend, double* out,
                               uint32_t* out_valid, cudaStream_t s) {
    if (n_groups <= 0) return cudaSuccess;
    const unsigned g = blocks_for(n_groups);
    switch (dtype) {
        case T_I8: k_dist_median<int8_t><<<g, kThreads, 0, s>>>((const int8_t*)sval, starts, n_groups, vend, out, out_valid); break;
        case T_I16: k_dist_median<int16_t><<<g, kThreads, 0, s>>>((const int16_t*)sval, starts, n_groups, vend, out, out_valid); break;
        case T_I32: k_dist_median<int32_t><<<g, kThreads, 0, s>>>((const int32_t*)sval, starts, n_groups, vend, out, out_valid); break;
        case T_I64: k_dist_median<int64_t><<<g, kThreads, 0, s>>>((const int64_t*)sval, starts, n_groups, vend, out, out_valid); break;
        case T_U8: k_dist_median<uint8_t><<<g, kThreads, 0, s>>>((const uint8_t*)sval, starts, n_groups, vend, out, out_valid); break;
        case T_U16: k_dist_median<uint16_t><<<g, kThreads, 0, s>>>((const uint16_t*)sval, starts, n_groups, vend, out, out_valid); break;
        case T_U32: k_dist_median<uint32_t><<<g, kThreads, 0, s>>>((const uint32_t*)sval, starts, n_groups, vend, out, out_valid); break;
        case T_U64: k_dist_median<uint64_t><<<g, kThreads, 0, s>>>((const uint64_t*)sval, starts, n_groups, vend, out, out_valid); break;
        case T_F32: k_dist_median<float><<<g, kThreads, 0, s>>>((const float*)sval, starts, n_groups, vend, out, out_valid); break;
        case T_F64: k_dist_median<double><<<g, kThreads, 0, s>>>((const double*)sval, starts, n_groups, vend, out, out_valid); break;
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

}  // namespace bdf
