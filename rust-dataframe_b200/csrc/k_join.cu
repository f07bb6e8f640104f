// k_join.cu -- equi-join indices (Transformation::Join -> DataFrame::join, src/dataframe.rs:626-719 -> calc_equijoin_indices,
// src/functions/join.rs:19-137), sort-based.
//
// The host (runtime.cu join_dev) sorts the build side's keys with the stable radix lexsort of k_sort.cu, gathers them, and
// compacts the distinct key tuples and the first sorted row of every run with the head kernel and stream compaction of the
// group-by.  The kernels here:
//   k_join_count        one thread per probe row, reading the probe side's chunks in place: a binary search of the distinct
//                       build tuples in the sort's total order (sort_keys.cuh: the very key transform the sort used, null last)
//                       gives the run of equal build rows; writes the run's first sorted row and the row's output count
//                       (outer joins: at least 1), marks the run as hit (full join), and the CTA's total: the tile sums of
//                       launch_scan_sums (k_scan.cu), which turns the counts into 64-bit output offsets and puts the total behind
//                       the last one.
//   k_join_emit         load-balanced by OUTPUT position: every CTA owns kJoinTile output rows, finds the probe rows that produce
//                       them with a binary search of the offsets, and writes (probe row, perm[run start + j]) and both validity
//                       bitmaps as whole words.  A hot key with 10^5 x 10^3 partners is spread over the whole GPU.  Rows past
//                       the probe part are the unmatched build rows a full join appends (null probe index).
//   k_join_unmatched    full join: every sorted build row of a run nobody hit sets its ORIGINAL row's bit in a mask; the mask
//                       then compacts an iota (k_filter.cu), which lists the unmatched rows in ascending row order.
//   k_join_exists       LEFT SEMI / ANTI: one thread per probe row writes "has a partner" (or its complement) as a bit, by ballot;
//                       the mask then compacts an iota of the probe rows.  No counts, no scan, no emit.
//   k_join_asof         one thread per probe row: the run of its `by` keys, then a binary search of the `on` key inside that run's
//                       valid, non-NaN prefix (the build side is sorted by (by..., on)); direction, exactness and tolerance pick
//                       one sorted row, whose original row number is written with the validity word by ballot.
// All three probe kernels find the build run through join_find_run, so they cannot disagree on key equality.
#include "scan.cuh"
#include "sort_keys.cuh"

#include <algorithm>

namespace bdf {

constexpr int kMaxJoinKeys = 16;
constexpr int kJoinTile = kScanTile;              // rows per CTA of the count and emit kernels
constexpr uint32_t kNoMatch = 0xffffffffu;         // match start of a probe row without partners (build rows are < 2^32 - 1)

struct JoinKey {
    const SortChunk* probe;        // chunk table of the probe column (the concatenated row space)
    const void* build;             // the distinct build keys of this criterion, in sort order (one chunk)
    const uint32_t* build_valid;   // its validity (bit offset 0), or null
    int n_chunks;
    int dtype;
};
struct JoinKeys { JoinKey k[kMaxJoinKeys]; int n; };

// Build run r against the probe tuple (every probe key valid): <0, 0, >0 as run r sorts before, equal to, after the probe.
__device__ __forceinline__ int join_cmp_run(const JoinKeys& keys, const unsigned long long (&pk)[kMaxJoinKeys], long long r) {
#pragma unroll
    for (int k = 0; k < kMaxJoinKeys; k++) {
        if (k >= keys.n) break;
        const JoinKey& K = keys.k[k];
        if (K.build_valid && !((__ldg(K.build_valid + (r >> 5)) >> (r & 31)) & 1u)) return 1;   // null sorts after every value
        const unsigned long long b = sort_key_at(K.dtype, K.build, r);
        if (b != pk[k]) return b < pk[k] ? -1 : 1;
    }
    return 0;
}

// The build run whose key tuple equals probe row i's, every criterion read through its chunk table, or -1 when there is none.  A
// null in any criterion matches nothing.  With no criteria (an as-of join without `by` keys) every row belongs to run 0.
__device__ __forceinline__ long long join_find_run(const JoinKeys& keys, long long i, long long n_runs) {
    unsigned long long pk[kMaxJoinKeys];
    bool valid = true;
#pragma unroll
    for (int k = 0; k < kMaxJoinKeys; k++) {
        pk[k] = 0;
        if (k < keys.n && valid) {
            const JoinKey& K = keys.k[k];
            const SortChunk ch = K.probe[K.n_chunks == 1 ? 0 : chunk_of(K.probe, K.n_chunks, i)];
            const long long local = i - ch.start;
            valid = ch.validity ? chunk_bit(ch.validity, ch.bit_off + local) : true;
            if (valid) pk[k] = sort_key_at(K.dtype, ch.values, local);
        }
    }
    if (!valid || n_runs <= 0) return -1;
    long long lo = 0, hi = n_runs;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if (join_cmp_run(keys, pk, mid) < 0) lo = mid + 1;
        else hi = mid;
    }
    return lo < n_runs && join_cmp_run(keys, pk, lo) == 0 ? lo : -1;
}

__global__ void __launch_bounds__(kThreads)
k_join_count(const __grid_constant__ JoinKeys keys, long long n_probe, const uint32_t* __restrict__ run_starts, long long n_runs, long long n_build,
             int outer, unsigned long long* __restrict__ counts, uint32_t* __restrict__ match_start, unsigned char* __restrict__ hit,
             unsigned long long* __restrict__ block_sums) {
    unsigned long long total = 0;
    for (int it = 0; it < kScanItems; it++) {
        const long long i = (long long)blockIdx.x * kJoinTile + it * kThreads + threadIdx.x;
        if (i >= n_probe) break;
        unsigned long long cnt = 0;
        uint32_t start = kNoMatch;
        const long long r = join_find_run(keys, i, n_runs);
        if (r >= 0) {
            start = run_starts[r];
            cnt = (unsigned long long)((r + 1 < n_runs ? (long long)run_starts[r + 1] : n_build) - (long long)start);
            if (hit) hit[r] = 1;
        }
        if (outer && cnt == 0) cnt = 1;
        counts[i] = cnt;
        match_start[i] = start;
        total += cnt;
    }
    total = cta_sum(total);
    if (threadIdx.x == 0) block_sums[blockIdx.x] = total;
}

// The last probe row i in [lo, hi] with offs[i] <= o (offs is non-decreasing; probe rows of an inner join may produce nothing).
__device__ __forceinline__ long long join_row_of(const unsigned long long* __restrict__ offs, long long lo, long long hi, unsigned long long o) {
    while (lo < hi) {
        const long long mid = (lo + hi + 1) >> 1;
        if (offs[mid] <= o) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__global__ void __launch_bounds__(kThreads)
k_join_emit(const unsigned long long* __restrict__ offs, long long n_probe, const uint32_t* __restrict__ match_start, const uint32_t* __restrict__ perm,
            unsigned long long probe_rows, const uint32_t* __restrict__ unmatched, unsigned long long n_out, uint32_t* __restrict__ probe_out,
            uint32_t* __restrict__ probe_valid, uint32_t* __restrict__ build_out, uint32_t* __restrict__ build_valid) {
    __shared__ long long s_range[2];
    const unsigned long long o0 = (unsigned long long)blockIdx.x * kJoinTile;
    if (threadIdx.x < 2) {   // the probe rows behind this CTA's first and last output row of the probe part
        long long r = 0;
        if (o0 < probe_rows) {
            const unsigned long long o = threadIdx.x == 0 ? o0 : min(o0 + kJoinTile, probe_rows) - 1;
            r = join_row_of(offs, 0, n_probe - 1, o);
        }
        s_range[threadIdx.x] = r;
    }
    __syncthreads();
    const long long lo = s_range[0], hi = s_range[1];
    for (int it = 0; it < kScanItems; it++) {
        const unsigned long long o = o0 + (unsigned long long)(it * kThreads + threadIdx.x);
        bool pv = false, bv = false;
        uint32_t p = 0, b = 0;
        if (o < probe_rows) {
            const long long i = join_row_of(offs, lo, hi, o);
            p = (uint32_t)i;
            pv = true;
            const uint32_t s = match_start[i];
            if (s != kNoMatch) { b = __ldg(perm + (unsigned long long)s + (o - offs[i])); bv = true; }
        } else if (o < n_out) {
            b = unmatched[o - probe_rows];
            bv = true;
        }
        if (o < n_out) { probe_out[o] = p; build_out[o] = b; }
        const unsigned pw = __ballot_sync(0xffffffffu, pv), bw = __ballot_sync(0xffffffffu, bv);
        if ((threadIdx.x & 31) == 0 && o < n_out) {
            if (probe_valid) probe_valid[o >> 5] = pw;
            if (build_valid) build_valid[o >> 5] = bw;
        }
    }
}

// Sorted build row s belongs to the last run whose start is <= s; an unhit run's rows are unmatched: bit perm[s] of the mask.
__global__ void __launch_bounds__(kThreads)
k_join_unmatched(const uint32_t* __restrict__ perm, long long n_build, const uint32_t* __restrict__ run_starts, long long n_runs,
                 const unsigned char* __restrict__ hit, uint32_t* __restrict__ mask) {
    for (long long s = (long long)blockIdx.x * kThreads + threadIdx.x; s < n_build; s += (long long)gridDim.x * kThreads) {
        long long lo = 0, hi = n_runs - 1;
        while (lo < hi) {
            const long long mid = (lo + hi + 1) >> 1;
            if ((long long)run_starts[mid] <= s) lo = mid; else hi = mid - 1;
        }
        if (!hit[lo]) {
            const uint32_t r = perm[s];
            atomicOr(mask + (r >> 5), 1u << (r & 31));
        }
    }
}

// LEFT SEMI (anti = 0) / LEFT ANTI (anti = 1): bit i of mask = probe row i has a partner (has none).  Rows past n_probe stay 0.
__global__ void __launch_bounds__(kThreads)
k_join_exists(const __grid_constant__ JoinKeys keys, long long n_probe, long long n_runs, int anti, uint32_t* __restrict__ mask) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool m = false;
    if (i < n_probe) m = (join_find_run(keys, i, n_runs) >= 0) != (anti != 0);
    const unsigned w = __ballot_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0 && i < n_probe) mask[i >> 5] = w;
}

enum : int { kAsofBackward = 0, kAsofForward, kAsofNearest };   // bdf_asof_direction

// The as-of join's `on` key: the probe side's chunk table, the build side gathered in sorted order (by..., on), and the rules.
struct AsofOn {
    const SortChunk* probe;
    int n_chunks;
    int dtype;
    const void* build;             // on, in sorted order (one chunk)
    const uint32_t* build_valid;   // its validity (bit offset 0), or null
    int direction;                 // bdf_asof_direction
    int exact;                     // allow_exact_matches
    int has_tol;
    unsigned long long tol;        // integer keys: the bound on the key distance
    double tol_f;                  // float keys
};

// The sort key of every NaN (sort_keys.cuh): the only key above every number.
__device__ __forceinline__ bool asof_is_nan_key(int dtype, unsigned long long k) {
    return (dtype == T_F32 && k == 0xffffffffull) || (dtype == T_F64 && k == ~0ull);
}
__device__ __forceinline__ double asof_as_double(int dtype, const void* values, long long i) {
    return dtype == T_F32 ? (double)((const float*)values)[i] : ((const double*)values)[i];
}
// Distances, from the smaller key (lo) to the larger (hi).  Integer keys: the sort keys are the values shifted by a constant, so their
// unsigned difference is the exact distance and cannot wrap (INT64_MIN to INT64_MAX is 2^64 - 1).  Float keys (below): the difference of
// the values widened to double, rounded once; equal keys (infinities included) are at distance 0.
__device__ __forceinline__ double asof_float_dist(unsigned long long klo, double lo, unsigned long long khi, double hi) {
    return klo == khi ? 0.0 : hi - lo;
}

__global__ void __launch_bounds__(kThreads)
k_join_asof(const __grid_constant__ JoinKeys by, const __grid_constant__ AsofOn on, long long n_probe, const uint32_t* __restrict__ run_starts,
            long long n_runs, long long n_build, const uint32_t* __restrict__ perm, uint32_t* __restrict__ out, uint32_t* __restrict__ out_valid) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool ok = false;
    uint32_t res = 0;
    if (i < n_probe) {
        const SortChunk ch = on.probe[on.n_chunks == 1 ? 0 : chunk_of(on.probe, on.n_chunks, i)];
        const long long local = i - ch.start;
        const bool lvalid = ch.validity ? chunk_bit(ch.validity, ch.bit_off + local) : true;
        const unsigned long long lk = lvalid ? sort_key_at(on.dtype, ch.values, local) : 0ull;
        const long long r = lvalid && !asof_is_nan_key(on.dtype, lk) ? join_find_run(by, i, n_runs) : -1;
        if (r >= 0) {
            const long long s = by.n ? (long long)run_starts[r] : 0;
            const long long e = r + 1 < n_runs ? (long long)run_starts[r + 1] : n_build;
            // the run's numbers come first: nulls sort last, NaN above every number
            long long lo = s, hi = e;
            while (lo < hi) {
                const long long mid = (lo + hi) >> 1;
                const bool num = (!on.build_valid || ((__ldg(on.build_valid + (mid >> 5)) >> (mid & 31)) & 1u)) &&
                                 !asof_is_nan_key(on.dtype, sort_key_at(on.dtype, on.build, mid));
                if (num) lo = mid + 1; else hi = mid;
            }
            const long long pe = lo;
            // ge: the first position with key >= lk; gt: the first with key > lk
            lo = s; hi = pe;
            while (lo < hi) {
                const long long mid = (lo + hi) >> 1;
                if (sort_key_at(on.dtype, on.build, mid) < lk) lo = mid + 1; else hi = mid;
            }
            const long long ge = lo;
            hi = pe;
            while (lo < hi) {
                const long long mid = (lo + hi) >> 1;
                if (sort_key_at(on.dtype, on.build, mid) <= lk) lo = mid + 1; else hi = mid;
            }
            const long long gt = lo;
            // backward: the last of the greatest keys <= (<) lk; forward: the first of the least keys >= (>) lk (the sort is stable)
            const long long b = (on.exact ? gt : ge) - 1, f = on.exact ? ge : gt;
            const bool hb = b >= s && on.direction != kAsofForward, hf = f < pe && on.direction != kAsofBackward;
            const unsigned long long kb = hb ? sort_key_at(on.dtype, on.build, b) : 0ull, kf = hf ? sort_key_at(on.dtype, on.build, f) : 0ull;
            const bool flt = dtype_is_float(on.dtype);
            const double l = flt ? asof_as_double(on.dtype, ch.values, local) : 0.0;
            const double vb = flt && hb ? asof_as_double(on.dtype, on.build, b) : 0.0, vf = flt && hf ? asof_as_double(on.dtype, on.build, f) : 0.0;
            bool back = hb;
            if (hb && hf) back = flt ? asof_float_dist(kb, vb, lk, l) <= asof_float_dist(lk, l, kf, vf) : lk - kb <= kf - lk;   // ties go backward
            if (hb || hf) {
                ok = true;
                if (on.has_tol) {
                    if (flt) ok = back ? asof_float_dist(kb, vb, lk, l) <= on.tol_f : asof_float_dist(lk, l, kf, vf) <= on.tol_f;
                    else ok = (back ? lk - kb : kf - lk) <= on.tol;
                }
                if (ok) res = __ldg(perm + (back ? b : f));
            }
        }
        out[i] = res;
    }
    const unsigned w = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0 && i < n_probe) out_valid[i >> 5] = w;
}

// ---- launchers ------------------------------------------------------------------------------------------------------
static JoinKeys join_keys(int n_keys, const int* dtypes, const void* const* probe_tables, const int* probe_chunks, const void* const* build_keys,
                          const uint32_t* const* build_valid) {
    JoinKeys jk{};
    for (int k = 0; k < n_keys; k++)
        jk.k[k] = JoinKey{(const SortChunk*)probe_tables[k], build_keys[k], build_valid[k], probe_chunks[k], dtypes[k]};
    jk.n = n_keys;
    return jk;
}

// Criterion k: dtype, the probe column's chunk table (sort_table) and chunk count, the distinct build keys and their validity.
cudaError_t launch_join_count(int n_keys, const int* dtypes, const void* const* probe_tables, const int* probe_chunks, const void* const* build_keys,
                              const uint32_t* const* build_valid, long long n_probe, const uint32_t* run_starts, long long n_runs, long long n_build,
                              int outer, unsigned long long* counts, uint32_t* match_start, unsigned char* hit, unsigned long long* block_sums,
                              cudaStream_t s) {
    if (n_probe <= 0) return cudaSuccess;
    if (n_keys < 1 || n_keys > kMaxJoinKeys) return cudaErrorInvalidValue;
    const JoinKeys jk = join_keys(n_keys, dtypes, probe_tables, probe_chunks, build_keys, build_valid);
    const long long blocks = (n_probe + kJoinTile - 1) / kJoinTile;
    k_join_count<<<(unsigned)blocks, kThreads, 0, s>>>(jk, n_probe, run_starts, n_runs, n_build, outer, counts, match_start, hit, block_sums);
    return cudaGetLastError();
}

cudaError_t launch_join_emit(const unsigned long long* offs, long long n_probe, const uint32_t* match_start, const uint32_t* perm, unsigned long long probe_rows,
                             const uint32_t* unmatched, unsigned long long n_out, uint32_t* probe_out, uint32_t* probe_valid, uint32_t* build_out,
                             uint32_t* build_valid, cudaStream_t s) {
    if (n_out == 0) return cudaSuccess;
    const unsigned long long blocks = (n_out + kJoinTile - 1) / kJoinTile;
    if (blocks > 0x7fffffffull) return cudaErrorInvalidConfiguration;
    k_join_emit<<<(unsigned)blocks, kThreads, 0, s>>>(offs, n_probe, match_start, perm, probe_rows, unmatched, n_out, probe_out, probe_valid, build_out,
                                                      build_valid);
    return cudaGetLastError();
}

// mask: ceil(n_build / 32) zeroed words.
cudaError_t launch_join_unmatched(const uint32_t* perm, long long n_build, const uint32_t* run_starts, long long n_runs, const unsigned char* hit,
                                  uint32_t* mask, int sm_count, cudaStream_t s) {
    if (n_build <= 0) return cudaSuccess;
    const long long want = (n_build + kThreads - 1) / kThreads;
    k_join_unmatched<<<(unsigned)std::min<long long>(want, (long long)sm_count * 8), kThreads, 0, s>>>(perm, n_build, run_starts, n_runs, hit, mask);
    return cudaGetLastError();
}

// mask: a boolean column of n_probe rows (whole words are written).
cudaError_t launch_join_exists(int n_keys, const int* dtypes, const void* const* probe_tables, const int* probe_chunks, const void* const* build_keys,
                               const uint32_t* const* build_valid, long long n_probe, long long n_runs, int anti, uint32_t* mask, cudaStream_t s) {
    if (n_probe <= 0) return cudaSuccess;
    if (n_keys < 1 || n_keys > kMaxJoinKeys) return cudaErrorInvalidValue;
    const long long blocks = (n_probe + kThreads - 1) / kThreads;
    if (blocks > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    k_join_exists<<<(unsigned)blocks, kThreads, 0, s>>>(join_keys(n_keys, dtypes, probe_tables, probe_chunks, build_keys, build_valid), n_probe, n_runs,
                                                        anti, mask);
    return cudaGetLastError();
}

// The `by` criteria as for launch_join_count (0..16 of them; none: the build side is one run and run_starts may be null), the `on`
// key's probe table and sorted build values, and the build side's sort permutation.  out / out_valid: n_probe UInt32 rows.
cudaError_t launch_join_asof(int n_by, const int* dtypes, const void* const* probe_tables, const int* probe_chunks, const void* const* build_keys,
                             const uint32_t* const* build_valid, int on_dtype, const void* on_table, int on_chunks, const void* on_build,
                             const uint32_t* on_build_valid, int direction, int exact, int has_tol, unsigned long long tol, double tol_f,
                             long long n_probe, const uint32_t* run_starts, long long n_runs, long long n_build, const uint32_t* perm, uint32_t* out,
                             uint32_t* out_valid, cudaStream_t s) {
    if (n_probe <= 0) return cudaSuccess;
    if (n_by < 0 || n_by > kMaxJoinKeys) return cudaErrorInvalidValue;
    const long long blocks = (n_probe + kThreads - 1) / kThreads;
    if (blocks > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    const AsofOn on{(const SortChunk*)on_table, on_chunks, on_dtype, on_build, on_build_valid, direction, exact, has_tol, tol, tol_f};
    k_join_asof<<<(unsigned)blocks, kThreads, 0, s>>>(join_keys(n_by, dtypes, probe_tables, probe_chunks, build_keys, build_valid), on, n_probe,
                                                      run_starts, n_runs, n_build, perm, out, out_valid);
    return cudaGetLastError();
}

}  // namespace bdf
