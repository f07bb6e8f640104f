// scan.cuh -- the warp- and CTA-wide sums that every prefix scan of the library is built from, and the one tile geometry of the
// multi-CTA 64-bit scan (k_scan.cu).  A producer that writes tile sums for launch_scan_sums / launch_scan_popcount sums exactly
// kScanTile entries per CTA: CTA b covers entries [b * kScanTile, (b + 1) * kScanTile).
#pragma once
#include "common.cuh"

namespace bdf {

constexpr int kScanItems = 8;                     // consecutive entries per thread of k_scan_apply
constexpr int kScanTile = kThreads * kScanItems;  // entries per tile sum

// Inclusive sum over lanes 0..lane of the warp.
template <typename T>
__device__ __forceinline__ T warp_inclusive_sum(T x) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    return x;
}

// CTA-wide exclusive sum of one value per thread over kWarps warps; *total = the CTA's sum when total is given.  Every thread of the
// CTA calls it, once per kernel: its shared scratch is not fenced for a second call.
template <typename T, int kWarps = kWarpsPerCta>
__device__ __forceinline__ T cta_exclusive_sum(T x, T* total = nullptr) {
    __shared__ T s_warp[kWarps];
    const int warp = threadIdx.x >> 5;
    const T inc = warp_inclusive_sum(x);
    if ((threadIdx.x & 31) == 31) s_warp[warp] = inc;
    __syncthreads();
    T before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < kWarps; w++) {
        if (w < warp) before += s_warp[w];
        all += s_warp[w];
    }
    if (total) *total = all;
    return before + inc - x;
}

// The CTA's sum of one value per thread, returned to every thread.  Every thread of the CTA calls it, once per kernel.
template <typename T>
__device__ __forceinline__ T cta_sum(T x) {
    __shared__ T s_warp[kWarpsPerCta];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = x;
    __syncthreads();
    T t = 0;
#pragma unroll
    for (int w = 0; w < kWarpsPerCta; w++) t += s_warp[w];
    return t;
}

}  // namespace bdf
