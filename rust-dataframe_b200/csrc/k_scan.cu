// k_scan.cu -- exclusive prefix scans: per-row counts into offsets, for every operator that first counts what each input produces
// (join, window runs, the CSV and JSON readers, list take, the radix sort and both writers).
//   k_scan_one        one CTA of 1024 threads, each owning a contiguous run of ceil(count / 1024) entries (its loads are independent
//                     of each other): one CTA-wide scan of the run totals, then the runs are rewritten in place; the total lands
//                     behind them when asked for.  (A first version walked the array 1024 entries at a time with a carried total:
//                     one dependent iteration per 1024 entries.)
//   k_scan_tile_sums  the sum of every tile of kScanTile entries (scan.cuh)
//   k_scan_apply      every tile rescanned in place from its scanned tile sum, kScanItems consecutive entries per thread
//   k_scan_popcount   the popcount of every bitmap word, and the tile sums of the popcounts
// The multi-CTA scan is tile sums -> k_scan_one over them -> k_scan_apply; producers that already know their counts write the tile
// sums themselves (cta_sum at kScanTile) and skip the first kernel.
#include "scan.cuh"

#include <algorithm>

namespace bdf {

template <typename T>
__global__ void __launch_bounds__(1024) k_scan_one(T* __restrict__ data, long long count, T* __restrict__ total) {
    const long long per = (count + 1023) / 1024;
    const long long begin = min(count, (long long)threadIdx.x * per), end = min(count, begin + per);
    T sum = 0;
    for (long long i = begin; i < end; i++) sum += data[i];
    T run = cta_exclusive_sum<T, 32>(sum);
    for (long long i = begin; i < end; i++) { const T v = data[i]; data[i] = run; run += v; }
    if (total && threadIdx.x == 1023) *total = run;
}

__global__ void __launch_bounds__(kThreads) k_scan_tile_sums(const unsigned long long* __restrict__ data, long long n, unsigned long long* __restrict__ sums) {
    const long long base = (long long)blockIdx.x * kScanTile + (long long)threadIdx.x * kScanItems;
    unsigned long long s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; k++)
        if (base + k < n) s += data[base + k];
    const unsigned long long t = cta_sum(s);
    if (threadIdx.x == 0) sums[blockIdx.x] = t;
}

__global__ void __launch_bounds__(kThreads) k_scan_apply(unsigned long long* __restrict__ data, long long n, const unsigned long long* __restrict__ offsets) {
    const long long base = (long long)blockIdx.x * kScanTile + (long long)threadIdx.x * kScanItems;
    unsigned long long v[kScanItems], s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; k++) {
        v[k] = base + k < n ? data[base + k] : 0ull;
        s += v[k];
    }
    unsigned long long run = offsets[blockIdx.x] + cta_exclusive_sum(s);
#pragma unroll
    for (int k = 0; k < kScanItems; k++)
        if (base + k < n) { data[base + k] = run; run += v[k]; }
}

__global__ void __launch_bounds__(kThreads)
k_scan_popcount(const uint32_t* __restrict__ words, long long n_words, unsigned long long* __restrict__ counts, unsigned long long* __restrict__ sums) {
    const long long base = (long long)blockIdx.x * kScanTile + (long long)threadIdx.x * kScanItems;
    unsigned s = 0;
#pragma unroll
    for (int k = 0; k < kScanItems; k++)
        if (base + k < n_words) { const unsigned c = __popc(words[base + k]); counts[base + k] = c; s += c; }
    const unsigned t = cta_sum(s);   // at most 32 x kScanTile
    if (threadIdx.x == 0) sums[blockIdx.x] = t;
}

// ---- launchers ------------------------------------------------------------------------------------------------------
template <typename T>
cudaError_t launch_scan_one(T* data, long long count, T* total, cudaStream_t s) {
    k_scan_one<T><<<1, 1024, 0, s>>>(data, count, total);
    return cudaGetLastError();
}
template cudaError_t launch_scan_one<unsigned int>(unsigned int*, long long, unsigned int*, cudaStream_t);
template cudaError_t launch_scan_one<unsigned long long>(unsigned long long*, long long, unsigned long long*, cudaStream_t);

long long scan_tile_sums(long long n) { return std::max<long long>((n + kScanTile - 1) / kScanTile, 1); }

cudaError_t launch_scan_sums(unsigned long long* data, long long n, unsigned long long* sums, cudaStream_t s) {
    if (n <= 0) return cudaMemsetAsync(data, 0, sizeof(unsigned long long), s);
    const long long tiles = scan_tile_sums(n);
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidValue;
    k_scan_one<unsigned long long><<<1, 1024, 0, s>>>(sums, tiles, data + n);
    k_scan_apply<<<(unsigned)tiles, kThreads, 0, s>>>(data, n, sums);
    return cudaGetLastError();
}

cudaError_t launch_scan(unsigned long long* data, long long n, unsigned long long* sums, cudaStream_t s) {
    const long long tiles = scan_tile_sums(n);
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidValue;
    if (n > 0) k_scan_tile_sums<<<(unsigned)tiles, kThreads, 0, s>>>(data, n, sums);
    return launch_scan_sums(data, n, sums, s);
}

cudaError_t launch_scan_popcount(const uint32_t* words, long long n_words, unsigned long long* counts, unsigned long long* sums, cudaStream_t s) {
    const long long tiles = scan_tile_sums(n_words);
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidValue;
    if (n_words > 0) k_scan_popcount<<<(unsigned)tiles, kThreads, 0, s>>>(words, n_words, counts, sums);
    return launch_scan_sums(counts, n_words, sums, s);
}

}  // namespace bdf
