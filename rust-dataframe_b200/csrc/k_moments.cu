// k_moments.cu -- the moment record (count, mean, m2, m3, m4; moments.cuh) of a whole column, all chunks, in ONE pass and ONE launch,
// then a finish with a fixed grid.  The statistics of bdf_moments* (variance, stddev, skewness, kurtosis and the population forms)
// are derived from it on the host.
//
// Numerics: as good as a two-pass algorithm, reading the data once.  A thread holds its 8 * k values of a tile in registers (f64:
// kUnroll vectors of 2; narrower types: more vectors, converted `as f64`); every batch of 8 values is reduced to its own record
// two-pass style -- the batch mean from the batch sum, then the central sums of the same registers -- and merged into the thread's
// running record (Chan / Pebay, moments.cuh).  Records then merge up a fixed tree: the xor-shuffle tree of the warp, the warps in
// warp order, one partial per CTA; k_moments_finish folds the partials with one CTA in a fixed assignment.  No atomics, so the same
// chunks give the same bits.  The naive power sums (sum x^2 - n mean^2) are never formed.
//   * a batch whose valid values are all equal (as f64) gets mean = that value and m2 = m3 = m4 = 0 exactly (the batch mean of three
//     0.1 is not 0.1); merging such records keeps the value and the zeros, so a constant column has variance 0, not 1e-17;
//   * a batch with a NaN or an infinity (its sum is not finite) gets NaN moments, and NaN sticks through every merge.
// Roofline: HBM, sizeof(T) + [nullable]/8 bytes per row -- 8 B/row for f64, as k_reduce.
#include "common.cuh"
#include "moments.cuh"

namespace bdf {

// Reduce one batch of up to 8 values (bit k of `bits`: v[k] is valid) to a record and merge it into `run`.
__device__ __forceinline__ void batch_moments(Moments& run, const double (&v)[8], uint32_t bits) {
    if (!bits) return;
    double ref = 0.0;
#pragma unroll
    for (int k = 7; k >= 0; k--)
        if ((bits >> k) & 1u) ref = v[k];   // the first valid value
    double s = 0.0;
    bool same = true;
#pragma unroll
    for (int k = 0; k < 8; k++)
        if ((bits >> k) & 1u) { s = __dadd_rn(s, v[k]); same = same && v[k] == ref; }
    Moments r;
    r.count = __popc(bits);
    if (!isfinite(s)) {
        r.mean = r.m2 = r.m3 = r.m4 = (double)NAN;
    } else if (same) {
        r.mean = ref; r.m2 = r.m3 = r.m4 = 0.0;
    } else {
        r.mean = r.count == 8 ? __dmul_rn(s, 0.125) : __ddiv_rn(s, (double)r.count);   // s / 8 exactly, without the division
        r.m2 = r.m3 = r.m4 = 0.0;
#pragma unroll
        for (int k = 0; k < 8; k++)
            if ((bits >> k) & 1u) {
                const double d = __dsub_rn(v[k], r.mean), d2 = __dmul_rn(d, d);
                r.m2 = __dadd_rn(r.m2, d2);
                r.m3 = __dadd_rn(r.m3, __dmul_rn(d2, d));
                r.m4 = __dadd_rn(r.m4, __dmul_rn(d2, d2));
            }
    }
    run = moments_merge(run, r);
}

// The thread's kUnroll vectors of E values of one tile (m[j]: the valid bits of vector j), 8 values per batch.
template <typename T, int E>
__device__ __forceinline__ void tile_moments(Moments& run, const Vec<T, E> (&x)[kUnroll], const uint32_t (&m)[kUnroll]) {
    constexpr int PER = kUnroll * E;
    static_assert(PER % 8 == 0, "batches of 8");
#pragma unroll
    for (int b = 0; b < PER / 8; b++) {
        double v[8];
        uint32_t bits = 0;
#pragma unroll
        for (int k = 0; k < 8; k++) {
            const int i = b * 8 + k;
            v[k] = (double)x[i / E].e[i % E];
            bits |= ((m[i / E] >> (i % E)) & 1u) << k;
        }
        batch_moments(run, v, bits);
    }
}

__device__ __forceinline__ Moments shfl_moments(const Moments& a, int o) {
    Moments b;
    b.count = __shfl_xor_sync(0xffffffffu, a.count, o);
    b.mean = __shfl_xor_sync(0xffffffffu, a.mean, o);
    b.m2 = __shfl_xor_sync(0xffffffffu, a.m2, o);
    b.m3 = __shfl_xor_sync(0xffffffffu, a.m3, o);
    b.m4 = __shfl_xor_sync(0xffffffffu, a.m4, o);
    return b;
}

// The CTA's record: the xor-shuffle tree of every warp, then thread 0 merges the warps in warp order.
__device__ __forceinline__ void cta_moments(Moments run, Moments* __restrict__ dst) {
    __shared__ Moments s_m[kWarpsPerCta];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) run = moments_merge(run, shfl_moments(run, o));
    if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = run;
    __syncthreads();
    if (threadIdx.x == 0) {
        Moments t = s_m[0];
#pragma unroll
        for (int w = 1; w < kWarpsPerCta; w++) t = moments_merge(t, s_m[w]);
        *dst = t;
    }
}

constexpr int kMomentTiles = 4;   // tiles per CTA: fewer partials for the finish, still many CTAs per SM

// The tile walk of k_reduce: this CTA's tiles chunk by chunk, full tiles as a pointer-bumping loop, then the partial last tile.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_moments(const RedDesc* __restrict__ descs, int n_chunks, int64_t total_tiles, Moments* __restrict__ cta_partials) {
    constexpr int E = 16 / (int)sizeof(T);
    constexpr int TILE = kThreads * kUnroll * E;
    Moments run{0, 0.0, 0.0, 0.0, 0.0};
    int64_t tile = (int64_t)blockIdx.x * kMomentTiles;
    const int64_t tile_end = min(tile + kMomentTiles, total_tiles);
#pragma unroll 1
    while (tile < tile_end) {
        const int c = (n_chunks == 1) ? 0 : find_chunk(descs, n_chunks, tile);
        const T* __restrict__ pi = (const T*)descs[c].in;
        const uint32_t* __restrict__ vi = descs[c].vin;
        const int64_t len = descs[c].len, off = descs[c].off, c_tile0 = descs[c].tile0;
        const int64_t chunk_end = c_tile0 + (len + TILE - 1) / TILE;
        if (tile >= chunk_end) break;
        const int64_t run_end = min(tile_end, chunk_end);
        const int n_full = (int)max((int64_t)0, min(run_end, c_tile0 + len / TILE) - tile);
        const int64_t base0 = (tile - c_tile0) * TILE;
        const T* __restrict__ p = pi + base0 + (int64_t)threadIdx.x * E;
        const int64_t bit0 = off + base0 + (int64_t)threadIdx.x * E;
        const uint32_t* __restrict__ vp = vi ? vi + (bit0 >> 5) : nullptr;
        const int sh = (int)(bit0 & 31);
#pragma unroll 1
        for (int t = 0; t < n_full; t++) {
            Vec<T, E> x[kUnroll];
#pragma unroll
            for (int j = 0; j < kUnroll; j++) x[j].load(p + (int64_t)j * kThreads * E);
            uint32_t m[kUnroll];
            if (vi) {
                MaskRaw<E, kUnroll> rv;
                mask_issue_at<E, kUnroll>(rv, vp, sh, kThreads * E / 32);
#pragma unroll
                for (int j = 0; j < kUnroll; j++) m[j] = mask_get<E, kUnroll>(rv, j);
                vp += TILE / 32;
            } else {
#pragma unroll
                for (int j = 0; j < kUnroll; j++) m[j] = (E == 32) ? 0xffffffffu : ((1u << E) - 1u);
            }
            tile_moments<T, E>(run, x, m);
            p += TILE;
        }
        tile += n_full;
        if (tile < run_end) {   // the partial last tile of the chunk
            const int64_t base = (tile - c_tile0) * TILE;
            Vec<T, E> x[kUnroll];
            uint32_t m[kUnroll];
#pragma unroll
            for (int j = 0; j < kUnroll; j++) {
                const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
                const uint32_t in_range = tail_mask<E>(e0, len);
                m[j] = in_range;
                if (in_range && vi) m[j] &= load_bits<E>(vi, off + e0);
#pragma unroll
                for (int e = 0; e < E; e++) x[j].e[e] = ((in_range >> e) & 1u) ? pi[e0 + e] : (T)0;
            }
            tile_moments<T, E>(run, x, m);
            tile++;
        }
    }
    cta_moments(run, &cta_partials[blockIdx.x]);
}

// One CTA: thread t merges the partials [t n / 256, (t + 1) n / 256) in order, then the CTA tree of k_moments.  n == 0 gives the
// empty record.
__global__ void __launch_bounds__(kThreads) k_moments_finish(const Moments* __restrict__ parts, long long n, Moments* __restrict__ result) {
    const long long b = n * threadIdx.x / kThreads, e = n * (threadIdx.x + 1) / kThreads;
    Moments run{0, 0.0, 0.0, 0.0, 0.0};
    for (long long i = b; i < e; i++) run = moments_merge(run, parts[i]);
    cta_moments(run, result);
}

int64_t moments_partials(int64_t tiles) { return (tiles + kMomentTiles - 1) / kMomentTiles; }

template <typename T>
static cudaError_t launch_one(const RedDesc* d, int n, int64_t tiles, Moments* partials, Moments* result, cudaStream_t s) {
    if (tiles > 0) k_moments<T><<<(unsigned)moments_partials(tiles), kThreads, 0, s>>>(d, n, tiles, partials);
    k_moments_finish<<<1, kThreads, 0, s>>>(partials, moments_partials(tiles), result);
    return cudaGetLastError();
}

// The record of the chunks described by d (tiles of elems_per_tile(dtype) elements) into *result; partials: moments_partials(tiles)
// records of device memory.
cudaError_t launch_moments(int dtype, const RedDesc* d, int n, int64_t tiles, Moments* partials, Moments* result, cudaStream_t s) {
    if (tiles < 0 || moments_partials(tiles) > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    switch (dtype) {
        case T_I8: return launch_one<int8_t>(d, n, tiles, partials, result, s);
        case T_I16: return launch_one<int16_t>(d, n, tiles, partials, result, s);
        case T_I32: return launch_one<int32_t>(d, n, tiles, partials, result, s);
        case T_I64: return launch_one<int64_t>(d, n, tiles, partials, result, s);
        case T_U8: return launch_one<uint8_t>(d, n, tiles, partials, result, s);
        case T_U16: return launch_one<uint16_t>(d, n, tiles, partials, result, s);
        case T_U32: return launch_one<uint32_t>(d, n, tiles, partials, result, s);
        case T_U64: return launch_one<uint64_t>(d, n, tiles, partials, result, s);
        case T_F32: return launch_one<float>(d, n, tiles, partials, result, s);
        case T_F64: return launch_one<double>(d, n, tiles, partials, result, s);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace bdf
