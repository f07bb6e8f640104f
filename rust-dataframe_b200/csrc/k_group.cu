// k_group.cu -- group-by on SORTED rows (SURVEY 8(f) tail: `GroupAggregate`, a `panic!` in the reference,
// src/evaluation.rs:73; the shape of the operator is src/expression.rs:114-221 `try_aggregate`).
//
// The host (runtime.cu group_by_dev) sorts the key columns with the stable radix lexsort of k_sort.cu and gathers the keys
// with k_take, so every group is one contiguous run of rows and the rows of a group keep their original order.  The kernels:
//   k_group_heads   bit i = 1 iff sorted row i starts a group: any of up to 16 keys differs from row i-1 (per key: nulls form
//                   ONE value, after all values -- the order of DataFrame::sort; NaN == NaN, -0.0 == 0.0 like the sort keys).
//                   The bitmap is a boolean column: `filter(sorted key, heads)` = the distinct keys, `filter(iota, heads)` = the
//                   first row of every group -- both through the existing stream compaction of k_filter.cu.  With "AND the
//                   last column's validity" the same kernel marks the first row of every distinct valid value inside a group
//                   (count_distinct: keys..., value sorted together).
//   k_group_reduce  one warp per group: lane l folds rows start + l, start + l + 32, ... in order, then a fixed xor-shuffle
//                   tree: deterministic (no atomics on values), integers wrap like AggregateFunctions::sum, floats are
//                   accumulated in double like K4.  sum / count always exist; min / max are NULL for a group without a
//                   valid value.  A group of more than kBigGroup rows is not folded by its warp: the warp registers it in a
//                   work list and k_group_big folds it one CTA per 64 Ki-row segment (thread-strided fold + fixed block
//                   tree), k_group_big_finish then folds a group's segment partials in segment order -- still deterministic,
//                   and a single hot key is spread over the whole GPU instead of one warp.  The accumulator is a template
//                   argument: ACC 0 folds what the single-key entry always folded (FusedAgg), ACC 1 what only bdf_group_by_dev
//                   asks for (GroupAggX, group_acc.cuh), ACC 2 the moment record of the statistics (GroupMoments) -- the three
//                   share every fold path, order and tree.
//                   In a 1- or 8-lane launch a group longer than kLaneRows rows per lane goes to a second list instead, and
//                   k_group_medium folds each of those with a warp (the 32-lane order and tree), so a few long groups among
//                   many one-row groups do not leave single threads walking tens of thousands of rows.
//   k_group_bounds  the original row number of every group's first and last row (first / last: a take of those rows).
//   k_group_distinct  one thread per group: the number of distinct-value heads inside the group's row range, by two
//                   binary searches over their compacted positions -- O(log n) per group, a hot key needs nothing special.
#include "group_acc.cuh"

namespace bdf {

// ---- (a) multi-key heads ----------------------------------------------------------------------------------------------
constexpr int kMaxGroupKeys = 17;   // 16 keys + the value column of count_distinct
struct HeadKey { const void* values; const uint32_t* valid; int width; int is_float; };
struct HeadKeys { HeadKey k[kMaxGroupKeys]; int n; int and_last_valid; };

template <typename T>
__device__ __forceinline__ bool group_same_key(T a, T b) {
    if constexpr (IsFloat<T>::value) return a == b || (a != a && b != b);
    else return a == b;
}

__device__ __forceinline__ bool head_key_differs(const HeadKey& k, long long i) {
    const bool vi = k.valid ? ((k.valid[i >> 5] >> (i & 31)) & 1u) : true;
    const bool vp = k.valid ? ((k.valid[(i - 1) >> 5] >> ((i - 1) & 31)) & 1u) : true;
    if (vi != vp) return true;
    if (!vi) return false;   // both null: one value
    switch (k.width) {       // equality is bitwise for integers: one comparison per width
        case 1: return ((const uint8_t*)k.values)[i] != ((const uint8_t*)k.values)[i - 1];
        case 2: return ((const uint16_t*)k.values)[i] != ((const uint16_t*)k.values)[i - 1];
        case 4: return k.is_float ? !group_same_key(((const float*)k.values)[i - 1], ((const float*)k.values)[i])
                                  : ((const uint32_t*)k.values)[i] != ((const uint32_t*)k.values)[i - 1];
        default: return k.is_float ? !group_same_key(((const double*)k.values)[i - 1], ((const double*)k.values)[i])
                                   : ((const uint64_t*)k.values)[i] != ((const uint64_t*)k.values)[i - 1];
    }
}

__global__ void __launch_bounds__(kThreads)
k_group_heads(const __grid_constant__ HeadKeys keys, long long n, uint32_t* __restrict__ head_words) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool h = false;
    if (i < n) {
        h = i == 0;
        for (int k = 0; k < keys.n && !h; k++) h = head_key_differs(keys.k[k], i);
        if (h && keys.and_last_valid) {
            const uint32_t* v = keys.k[keys.n - 1].valid;
            h = v ? ((v[i >> 5] >> (i & 31)) & 1u) : true;
        }
    }
    const unsigned w = __ballot_sync(0xffffffffu, h);
    if ((threadIdx.x & 31) == 0 && i < n) head_words[i >> 5] = w;
}

// ---- (b) per-group fold -------------------------------------------------------------------------------------------------
template <typename T, int ACC> struct GroupAcc { using type = FusedAgg<T>; };
template <typename T> struct GroupAcc<T, 1> { using type = GroupAggX<T>; };
template <typename T> struct GroupAcc<T, 2> { using type = GroupMoments<T>; };

// Where the results of one value column go.  min / max / avg (and nonempty, their shared validity) may be null; ACC 2 writes only
// the moment records `mom`.
template <typename T> struct GroupOuts { T *sum, *min, *max; long long* count; double* avg; uint32_t* nonempty; Moments* mom; };

// Hot keys.  The work list lives in device memory: {counters, list[]} then the segment partials.
constexpr long long kBigGroup = 65536;   // rows a single warp still folds itself; also the segment length of k_group_big
constexpr size_t kPartBytes = 40;        // the largest accumulator (GroupMoments)
struct BigGroup { unsigned long long g, begin, end; unsigned int seg0, n_seg; };
struct BigWork { unsigned int n_groups, n_segments, n_medium; BigGroup list[1]; };   // list[capacity] follows
// A group longer than kLaneRows rows per lane of a 1- or 8-lane launch is folded by a warp of its own (k_group_medium): one
// thread must not walk tens of thousands of rows while its neighbours are done after one.
constexpr long long kLaneRows = 512;
static_assert(sizeof(GroupAggX<long long>) <= kPartBytes && sizeof(GroupAggX<double>) <= kPartBytes && sizeof(FusedAgg<long long>) <= kPartBytes &&
              sizeof(GroupMoments<double>) <= kPartBytes, "partials");

template <typename T, int ACC>
__device__ __forceinline__ void group_write(const typename GroupAcc<T, ACC>::type& acc, unsigned long long cnt, long long g, const GroupOuts<T>& o,
                                            bool set_valid) {
    constexpr unsigned long long flip = GroupFlip<T>::value;
    if constexpr (ACC == 2) {
        o.mom[g] = acc.m;   // the statistics are derived in k_group_stats
    } else if constexpr (ACC == 0) {
        o.count[g] = (long long)cnt;
        const FusedAgg<T>& a = acc;
        if constexpr (IsFloat<T>::value) {
            o.sum[g] = (T)a.sum;
        } else {
            using U = typename UnsignedOf<T>::type;
            o.sum[g] = (T)(U)a.sum;   // wrapping
            if (o.min) {
                o.min[g] = cnt ? (T)(U)(a.kmin ^ flip) : (T)0;
                o.max[g] = cnt ? (T)(U)(a.kmax ^ flip) : (T)0;
                if (cnt && set_valid) atomicOr(&o.nonempty[g >> 5], 1u << (g & 31));
            }
        }
    } else {
        o.count[g] = (long long)cnt;
        double dsum;
        if constexpr (IsFloat<T>::value) {
            dsum = acc.sum;
            o.sum[g] = (T)acc.sum;
            if (o.min) o.min[g] = cnt ? FloatKey<T>::value(acc.kmin) : (T)0;
            if (o.max) o.max[g] = cnt ? FloatKey<T>::value(acc.kmax) : (T)0;
        } else {
            using U = typename UnsignedOf<T>::type;
            dsum = acc.dsum;
            o.sum[g] = (T)(U)acc.a.sum;
            if (o.min) o.min[g] = cnt ? (T)(U)(acc.a.kmin ^ flip) : (T)0;
            if (o.max) o.max[g] = cnt ? (T)(U)(acc.a.kmax ^ flip) : (T)0;
        }
        if (o.avg) o.avg[g] = dsum;   // divided by the count in k_group_avg (a double division is a call: it spills here)
        if (cnt && set_valid && o.nonempty) atomicOr(&o.nonempty[g >> 5], 1u << (g & 31));
    }
}

// One CTA per (hot group, segment): thread t folds rows begin + t, begin + t + 256, ... of the segment, then warp trees, then the
// warps in order -> partial[seg0 + segment].  The grid is fixed; CTAs walk the work items (the counters are only known on the device).
template <typename T, int ACC>
__global__ void __launch_bounds__(kThreads)
k_group_big(const T* __restrict__ val, const uint32_t* __restrict__ vvalid, const BigWork* __restrict__ big, typename GroupAcc<T, ACC>::type* __restrict__ part,
            unsigned long long* __restrict__ part_cnt) {
    using Acc = typename GroupAcc<T, ACC>::type;
    __shared__ Acc s_a[kWarpsPerCta];
    __shared__ unsigned long long s_c[kWarpsPerCta];
    const unsigned int n_big = big->n_groups, n_seg = big->n_segments;
    for (unsigned int w = blockIdx.x; w < n_seg; w += gridDim.x) {
        unsigned int gi = 0;
        while (gi < n_big && !(big->list[gi].seg0 <= w && w < big->list[gi].seg0 + big->list[gi].n_seg)) gi++;   // a handful of hot groups
        if (gi == n_big) continue;
        const BigGroup bg = big->list[gi];
        const long long b = (long long)bg.begin + (long long)(w - bg.seg0) * kBigGroup;
        const long long e = min((long long)bg.end, b + kBigGroup);
        Acc a;
        a.init();
        unsigned long long cnt = 0;
        for (long long i = b + threadIdx.x; i < e; i += kThreads) {
            const bool ok = vvalid ? ((vvalid[i >> 5] >> (i & 31)) & 1u) : true;
            a.add(val[i], ok, GroupFlip<T>::value);
            cnt += ok ? 1ull : 0ull;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { a.merge_shfl(o); cnt += __shfl_xor_sync(0xffffffffu, cnt, o); }
        __syncthreads();   // the previous work item's readers are done with the shared arrays
        if ((threadIdx.x & 31) == 0) { s_a[threadIdx.x >> 5] = a; s_c[threadIdx.x >> 5] = cnt; }
        __syncthreads();
        if (threadIdx.x == 0) {
            Acc t = s_a[0];
            unsigned long long total = s_c[0];
#pragma unroll
            for (int k = 1; k < kWarpsPerCta; k++) { t.merge(s_a[k]); total += s_c[k]; }
            part[w] = t;
            part_cnt[w] = total;
        }
    }
}

// One thread per hot group: its segment partials in segment order.
template <typename T, int ACC>
__global__ void k_group_big_finish(const BigWork* __restrict__ big, const typename GroupAcc<T, ACC>::type* __restrict__ part,
                                   const unsigned long long* __restrict__ part_cnt, const GroupOuts<T> out) {
    const unsigned int gi = blockIdx.x * blockDim.x + threadIdx.x;
    if (gi >= big->n_groups) return;
    const BigGroup bg = big->list[gi];
    typename GroupAcc<T, ACC>::type a = part[bg.seg0];
    unsigned long long cnt = part_cnt[bg.seg0];
    for (unsigned int k = 1; k < bg.n_seg; k++) { a.merge(part[bg.seg0 + k]); cnt += part_cnt[bg.seg0 + k]; }
    group_write<T, ACC>(a, cnt, (long long)bg.g, out, true);
}

// LANES lanes per group (32, 8 or 1 -- the launcher picks by the average group length, so ~1e8 one-row groups do not spend a
// warp each).  No lane leaves before the shuffles: a sub-group that is past the end, or defers its group, folds an empty range.
template <typename T, int LANES, int ACC>
__global__ void __launch_bounds__(kThreads)
k_group_reduce(const T* __restrict__ val, const uint32_t* __restrict__ vvalid, const uint32_t* __restrict__ starts, long long n_groups,
               long long n_rows, const GroupOuts<T> out, BigWork* __restrict__ big, unsigned long long* __restrict__ medium) {
    constexpr int kGroupsPerWarp = 32 / LANES;
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    const long long g = t / LANES;
    const int sub = threadIdx.x & (LANES - 1);
    bool mine = g < n_groups;
    long long b = 0, e = 0;
    if (mine) { b = starts[g]; e = g + 1 < n_groups ? (long long)starts[g + 1] : n_rows; }
    if (mine && big && e - b > kBigGroup) {   // a hot key: leave it to k_group_big (one CTA per segment)
        if (sub == 0) {
            const unsigned int nseg = (unsigned int)((e - b + kBigGroup - 1) / kBigGroup);
            const unsigned int slot = atomicAdd(&big->n_groups, 1u);
            const unsigned int base = atomicAdd(&big->n_segments, nseg);
            big->list[slot] = BigGroup{(unsigned long long)g, (unsigned long long)b, (unsigned long long)e, base, nseg};
        }
        mine = false;
        e = b;
    } else if (LANES < 32 && mine && big && e - b > kLaneRows * LANES) {   // long among short groups: k_group_medium folds it
        if (sub == 0) medium[atomicAdd(&big->n_medium, 1u)] = (unsigned long long)g;
        mine = false;
        e = b;
    }
    typename GroupAcc<T, ACC>::type a;
    a.init();
    unsigned long long cnt = 0;
    constexpr unsigned long long flip = GroupFlip<T>::value;
    for (long long i = b + sub; i < e; i += LANES) {
        const bool ok = vvalid ? ((vvalid[i >> 5] >> (i & 31)) & 1u) : true;
        a.add(val[i], ok, flip);
        cnt += ok ? 1ull : 0ull;
    }
#pragma unroll
    for (int o = LANES / 2; o > 0; o >>= 1) { a.merge_shfl(o); cnt += __shfl_xor_sync(0xffffffffu, cnt, o); }
    const bool writer = mine && sub == 0;
    if (writer) group_write<T, ACC>(a, cnt, g, out, false);
    if constexpr (!IsFloat<T>::value || ACC != 0) {
        if (out.nonempty) {   // min/max/avg validity: the warp's groups share one bitmap word -> one store (LANES == 1) or one atomic per warp
            const unsigned bal = __ballot_sync(0xffffffffu, writer && cnt != 0);
            if ((threadIdx.x & 31) == 0) {
                const long long g0 = (t >> 5) * kGroupsPerWarp;
                if (g0 < n_groups) {
                    unsigned word = 0;
#pragma unroll
                    for (int j = 0; j < kGroupsPerWarp; j++) word |= ((bal >> (j * LANES)) & 1u) << (((unsigned)g0 + j) & 31u);
                    if (LANES == 1) out.nonempty[g0 >> 5] = word;   // hot groups of this word are OR-ed in later by k_group_big_finish
                    else if (word) atomicOr(&out.nonempty[g0 >> 5], word);
                }
            }
        }
    }
}

// avg[g] holds the group's double sum: divide it by the count (NULL rows keep 0).
__global__ void k_group_avg(const long long* __restrict__ count, long long n_groups, double* __restrict__ avg) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g < n_groups) avg[g] = count[g] ? avg[g] / (double)count[g] : 0.0;
}

// A warp per group of the medium list, in the order and with the tree of the 32-lane k_group_reduce (grid-stride over the
// list, whose length is only known on the device).  The validity bit is OR-ed in: the 1-lane launch stores whole words.
template <typename T, int ACC>
__global__ void __launch_bounds__(kThreads)
k_group_medium(const T* __restrict__ val, const uint32_t* __restrict__ vvalid, const uint32_t* __restrict__ starts, long long n_groups,
               long long n_rows, const BigWork* __restrict__ big, const unsigned long long* __restrict__ medium, const GroupOuts<T> out) {
    const unsigned int n_med = big->n_medium;
    const int lane = threadIdx.x & 31;
    constexpr unsigned long long flip = GroupFlip<T>::value;
    for (unsigned int w = blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5); w < n_med; w += gridDim.x * kWarpsPerCta) {
        const long long g = (long long)medium[w];
        const long long b = starts[g], e = g + 1 < n_groups ? (long long)starts[g + 1] : n_rows;
        typename GroupAcc<T, ACC>::type a;
        a.init();
        unsigned long long cnt = 0;
        for (long long i = b + lane; i < e; i += 32) {
            const bool ok = vvalid ? ((vvalid[i >> 5] >> (i & 31)) & 1u) : true;
            a.add(val[i], ok, flip);
            cnt += ok ? 1ull : 0ull;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { a.merge_shfl(o); cnt += __shfl_xor_sync(0xffffffffu, cnt, o); }
        if (lane == 0) group_write<T, ACC>(a, cnt, g, out, true);
    }
}

// ---- (c) first / last rows and distinct counts ---------------------------------------------------------------------
__global__ void k_group_bounds(const uint32_t* __restrict__ idx, const uint32_t* __restrict__ starts, long long n_groups, long long n_rows,
                               uint32_t* __restrict__ first, uint32_t* __restrict__ last) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_groups) return;
    const long long e = g + 1 < n_groups ? (long long)starts[g + 1] : n_rows;
    if (first) first[g] = idx[starts[g]];
    if (last) last[g] = idx[e - 1];
}

__device__ __forceinline__ long long lower_bound_u32(const uint32_t* __restrict__ a, long long n, long long x) {
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if ((long long)a[mid] < x) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// out: the group's distinct-value count (may be null); first: the index of its first distinct value in the compacted list (may be
// null), i.e. the group starts of the distinct values themselves (sum_distinct folds them with launch_group_reduce).
__global__ void k_group_distinct(const uint32_t* __restrict__ pos, long long n_pos, const uint32_t* __restrict__ starts, long long n_groups,
                                 long long n_rows, long long* __restrict__ out, uint32_t* __restrict__ first) {
    const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= n_groups) return;
    const long long e = g + 1 < n_groups ? (long long)starts[g + 1] : n_rows;
    const long long b = lower_bound_u32(pos, n_pos, (long long)starts[g]);
    if (out) out[g] = lower_bound_u32(pos, n_pos, e) - b;
    if (first) first[g] = (uint32_t)b;
}

// ---- launchers ------------------------------------------------------------------------------------------------------
// Key k: values, validity (or null), width in bytes, float flag.  and_last_valid: a head also needs the last column valid.
cudaError_t launch_group_heads(int n_keys, const void* const* values, const uint32_t* const* valid, const int* widths, const int* is_float,
                               int and_last_valid, long long n, uint32_t* words, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    if (n_keys < 1 || n_keys > kMaxGroupKeys) return cudaErrorInvalidValue;
    HeadKeys hk{};
    for (int k = 0; k < n_keys; k++) hk.k[k] = HeadKey{values[k], valid[k], widths[k], is_float[k]};
    hk.n = n_keys;
    hk.and_last_valid = and_last_valid;
    const long long rows = (n + 31) / 32 * 32;
    k_group_heads<<<(unsigned)((rows + kThreads - 1) / kThreads), kThreads, 0, s>>>(hk, n, words);
    return cudaGetLastError();
}

size_t group_big_scratch_bytes(long long n_rows) {   // work list + segment partials for any distribution of n_rows rows
    const size_t max_groups = (size_t)(n_rows / kBigGroup) + 2, max_segs = 2 * max_groups + 2, max_medium = (size_t)(n_rows / kLaneRows) + 2;
    return 64 + max_groups * sizeof(BigGroup) + max_segs * (kPartBytes + 8) + max_medium * 8 + 256;
}

template <typename T, int ACC>
static cudaError_t reduce_one(const void* val, const uint32_t* vvalid, const uint32_t* starts, long long n_groups, long long n_rows, const GroupOuts<T>& out,
                              void* scratch, int sm_count, cudaStream_t s) {
    using Acc = typename GroupAcc<T, ACC>::type;
    BigWork* big = (BigWork*)scratch;
    cudaError_t e = cudaMemsetAsync(big, 0, 16, s);   // the three counters
    if (e != cudaSuccess) return e;
    const size_t max_groups = (size_t)(n_rows / kBigGroup) + 2, max_segs = 2 * max_groups + 2;
    char* p = (char*)scratch + 64 + max_groups * sizeof(BigGroup);
    p = (char*)(((uintptr_t)p + 15) & ~(uintptr_t)15);
    Acc* part = (Acc*)p;
    unsigned long long* part_cnt = (unsigned long long*)(p + max_segs * kPartBytes);
    unsigned long long* medium = part_cnt + max_segs;
    const long long avg = n_rows / n_groups;   // lanes per group by the average group length
    const int lanes = avg > 64 ? 32 : avg > 4 ? 8 : 1;
    const unsigned grid = (unsigned)((n_groups * lanes + kThreads - 1) / kThreads);
    if (lanes == 32) k_group_reduce<T, 32, ACC><<<grid, kThreads, 0, s>>>((const T*)val, vvalid, starts, n_groups, n_rows, out, big, medium);
    else if (lanes == 8) k_group_reduce<T, 8, ACC><<<grid, kThreads, 0, s>>>((const T*)val, vvalid, starts, n_groups, n_rows, out, big, medium);
    else k_group_reduce<T, 1, ACC><<<grid, kThreads, 0, s>>>((const T*)val, vvalid, starts, n_groups, n_rows, out, big, medium);
    if (lanes < 32 && n_rows > kLaneRows)   // finds nothing to do when no group is long
        k_group_medium<T, ACC><<<(unsigned)(sm_count * 4), kThreads, 0, s>>>((const T*)val, vvalid, starts, n_groups, n_rows, big, medium, out);
    if (n_rows > kBigGroup) {   // hot keys are possible: the two follow-up kernels find nothing to do when there are none
        k_group_big<T, ACC><<<(unsigned)(sm_count * 4), kThreads, 0, s>>>((const T*)val, vvalid, big, part, part_cnt);
        k_group_big_finish<T, ACC><<<(unsigned)((max_groups + 127) / 128), 128, 0, s>>>(big, part, part_cnt, out);
    }
    if (out.avg) k_group_avg<<<(unsigned)((n_groups + kThreads - 1) / kThreads), kThreads, 0, s>>>(out.count, n_groups, out.avg);
    return cudaGetLastError();
}

template <typename T>
static cudaError_t reduce_typed(bool extra, const void* val, const uint32_t* vvalid, const uint32_t* starts, long long n_groups, long long n_rows, void* sum,
                                long long* count, void* mn, void* mx, double* avg, uint32_t* nonempty, void* scratch, int sm_count, cudaStream_t s) {
    const GroupOuts<T> out{(T*)sum, (T*)mn, (T*)mx, count, avg, nonempty};
    return extra ? reduce_one<T, 1>(val, vvalid, starts, n_groups, n_rows, out, scratch, sm_count, s)
                 : reduce_one<T, 0>(val, vvalid, starts, n_groups, n_rows, out, scratch, sm_count, s);
}

template <typename T>
static cudaError_t moments_typed(const void* val, const uint32_t* vvalid, const uint32_t* starts, long long n_groups, long long n_rows, Moments* mom,
                                 void* scratch, int sm_count, cudaStream_t s) {
    GroupOuts<T> out{};
    out.mom = mom;
    return reduce_one<T, 2>(val, vvalid, starts, n_groups, n_rows, out, scratch, sm_count, s);
}

// The moment record of every group (the fold paths of launch_group_reduce with the GroupMoments accumulator).
cudaError_t launch_group_moments(int dtype, const void* val, const uint32_t* vvalid, const uint32_t* starts, long long n_groups, long long n_rows,
                                 Moments* mom, void* scratch, int sm_count, cudaStream_t s) {
    if (n_groups <= 0) return cudaSuccess;
    if (n_groups > 0x7fffffffLL * kWarpsPerCta) return cudaErrorInvalidConfiguration;
#define BDF_MOMENTS(T) moments_typed<T>(val, vvalid, starts, n_groups, n_rows, mom, scratch, sm_count, s)
    switch (dtype) {
        case T_I8: return BDF_MOMENTS(int8_t);
        case T_I16: return BDF_MOMENTS(int16_t);
        case T_I32: return BDF_MOMENTS(int32_t);
        case T_I64: return BDF_MOMENTS(int64_t);
        case T_U8: return BDF_MOMENTS(uint8_t);
        case T_U16: return BDF_MOMENTS(uint16_t);
        case T_U32: return BDF_MOMENTS(uint32_t);
        case T_U64: return BDF_MOMENTS(uint64_t);
        case T_F32: return BDF_MOMENTS(float);
        case T_F64: return BDF_MOMENTS(double);
        default: return cudaErrorInvalidValue;
    }
#undef BDF_MOMENTS
}

// One statistic of every group's record (moments_stat): the value and the validity bit (0 = None).  The divisions live here, out
// of the fold, as avg's do in k_group_avg; a warp's 32 groups share one bitmap word, which its first lane stores.
__global__ void __launch_bounds__(kThreads)
k_group_stats(const Moments* __restrict__ mom, long long n_groups, int stat, double* __restrict__ out, uint32_t* __restrict__ valid) {
    const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
    double v = 0.0;
    const bool some = g < n_groups && moments_stat(mom[g], stat, &v);
    if (g < n_groups) out[g] = some ? v : 0.0;
    const unsigned w = __ballot_sync(0xffffffffu, some);
    if ((threadIdx.x & 31) == 0 && g < n_groups) valid[g >> 5] = w;
}

cudaError_t launch_group_stats(const Moments* mom, long long n_groups, int stat, double* out, uint32_t* valid, cudaStream_t s) {
    if (n_groups <= 0) return cudaSuccess;
    k_group_stats<<<(unsigned)((n_groups + kThreads - 1) / kThreads), kThreads, 0, s>>>(mom, n_groups, stat, out, valid);
    return cudaGetLastError();
}

// scratch: group_big_scratch_bytes(n_rows) of device memory.  mn / mx / avg may be null (without extra, integer mn and mx
// are both given or both null); nonempty: the validity bitmap of min / max / avg (bit g = the group has a valid value), or
// null.  extra: integers also fold the double sum of avg, floats also fold min / max -- the single-key entry asks for neither.
cudaError_t launch_group_reduce(int dtype, bool extra, const void* val, const uint32_t* vvalid, const uint32_t* starts, long long n_groups, long long n_rows,
                                void* sum, long long* count, void* mn, void* mx, double* avg, uint32_t* nonempty, void* scratch, int sm_count, cudaStream_t s) {
    if (n_groups <= 0) return cudaSuccess;
    if (n_groups > 0x7fffffffLL * kWarpsPerCta) return cudaErrorInvalidConfiguration;
#define BDF_REDUCE(T) reduce_typed<T>(extra, val, vvalid, starts, n_groups, n_rows, sum, count, mn, mx, avg, nonempty, scratch, sm_count, s)
    switch (dtype) {
        case T_I8: return BDF_REDUCE(int8_t);
        case T_I16: return BDF_REDUCE(int16_t);
        case T_I32: return BDF_REDUCE(int32_t);
        case T_I64: return BDF_REDUCE(int64_t);
        case T_U8: return BDF_REDUCE(uint8_t);
        case T_U16: return BDF_REDUCE(uint16_t);
        case T_U32: return BDF_REDUCE(uint32_t);
        case T_U64: return BDF_REDUCE(uint64_t);
        case T_F32: return BDF_REDUCE(float);
        case T_F64: return BDF_REDUCE(double);
        default: return cudaErrorInvalidValue;
    }
#undef BDF_REDUCE
}

cudaError_t launch_group_bounds(const uint32_t* idx, const uint32_t* starts, long long n_groups, long long n_rows, uint32_t* first, uint32_t* last,
                                cudaStream_t s) {
    if (n_groups <= 0) return cudaSuccess;
    k_group_bounds<<<(unsigned)((n_groups + kThreads - 1) / kThreads), kThreads, 0, s>>>(idx, starts, n_groups, n_rows, first, last);
    return cudaGetLastError();
}

cudaError_t launch_group_distinct(const uint32_t* pos, long long n_pos, const uint32_t* starts, long long n_groups, long long n_rows, long long* out,
                                  uint32_t* first, cudaStream_t s) {
    if (n_groups <= 0) return cudaSuccess;
    k_group_distinct<<<(unsigned)((n_groups + kThreads - 1) / kThreads), kThreads, 0, s>>>(pos, n_pos, starts, n_groups, n_rows, out, first);
    return cudaGetLastError();
}

}  // namespace bdf
