// k_list.cu -- the kernels of the list functions (ArrayFunctions, src/functions/array.rs; runtime.cu list_* drives them).
//
// A list chunk is (Int32 offsets rebased to 0, list validity at bit 0, the child chunk's elements).  Equality everywhere is the key
// equality of sort / group-by / join: two values are equal iff their SortKey is (integers exact, NaNs one value, -0.0 == 0.0).
//   k_list_find      contains / position: LANES lanes per list (1, 8 or 32, by the average list length, as k_group_reduce picks
//                    them), in rounds of LANES consecutive elements; a list stops at the round of its first match.  A list longer
//                    than kLaneRounds rounds (kLaneRounds x LANES elements: one thread must not walk thousands of elements while
//                    its warp waits) is left to k_list_find_long, one CTA per segment of at most kLongList elements, whose first
//                    matches meet in an atomicMin on the element index (a minimum does not depend on the order it is formed in).
//   k_list_parent    the element -> list map of the sort-based functions and explode: every element finds its list by binary search
//                    of the offsets, so one huge list is spread over the whole GPU.  Writes the global list number and the bitmap of
//                    elements that belong to a valid list (whole words by ballot, OR-ed in: a word may straddle two chunks).
//   k_list_remove_mask  array_remove's keep bits (an element of a valid list that is not a valid element equal to v).
//   k_list_mark      distinct / except / intersect / union over the stable (list, value) sort: decides per sorted position from
//                    the group heads and the side the element came from, and sets the keep bit at the element's ORIGINAL position.
//   k_list_offsets   the offsets of a result from the list numbers of its kept elements (in list order): one binary search per list.
//   k_list_repeat    array_repeat's gather indices, one thread per OUTPUT element (binary search of the output offsets).
//   k_list_size / k_list_minmax_valid  size, and the validity / empty-list check of max and min (folded by k_group_reduce).
//   k_list_take_sizes  take / filter of whole lists, one thread per OUTPUT list: the size and first element of its source list (0 for
//                    a null index or a null list), and its validity bit (warp-aggregated atomicOr: an output chunk may start
//                    inside a word).  k_list_take_rows then gives every output element its source element, one thread per OUTPUT
//                    element (binary search of the scanned sizes, as k_list_repeat), so one hot list is spread over the GPU;
//                    take_dev gathers the elements.
//   k_list_rebase    Int32 offsets of one output chunk from the 64-bit scan of all output sizes.
//   k_list_ranks     collect_list / collect_set offsets: the rank of every group start among the sorted rows that are kept.
#include "sort_keys.cuh"

namespace bdf {

constexpr long long kLongList = 16384;   // elements per segment of k_list_find_long
constexpr long long kLaneRounds = 64;    // a list of more than kLaneRounds x LANES elements goes to k_list_find_long

__device__ __forceinline__ bool bit_at(const uint32_t* __restrict__ w, long long i) { return (__ldg(w + (i >> 5)) >> (i & 31)) & 1u; }

// The list of element e: the last j with off[j] <= e (empty lists share their offset with the next list).
__device__ __forceinline__ long long list_of(const int32_t* __restrict__ off, long long len, long long e) {
    long long lo = 0, hi = len - 1;
    while (lo < hi) {
        const long long mid = (lo + hi + 1) >> 1;
        if ((long long)__ldg(off + mid) <= e) lo = mid; else hi = mid - 1;
    }
    return lo;
}

__device__ __forceinline__ long long lower_bound_u32_list(const uint32_t* __restrict__ a, long long n, long long x) {
    long long lo = 0, hi = n;
    while (lo < hi) {
        const long long mid = (lo + hi) >> 1;
        if ((long long)__ldg(a + mid) < x) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// ---- contains / position ----------------------------------------------------------------------------------------------------------
struct LongList { unsigned long long list, b, e; unsigned int seg0, n_seg; };
// One 64-bit counter (lists << 32 | segments) hands out slot and first segment together, so items are in ascending seg0 order and a
// segment finds its item by binary search.
struct LongWork { unsigned long long counter; LongList item[1]; };   // item[capacity] follows, then the per-item minima

template <typename T>
struct FindArgs {
    const int32_t* off; const uint32_t* lvalid; long long len;
    const T* values; const uint32_t* vvalid; int vbit_off; unsigned long long key;
    int mode;                 // 0 contains, 1 position
    uint32_t* bits;           // contains: result bits (zeroed)
    int32_t* pos;             // position: result
};

template <typename T>
__device__ __forceinline__ bool find_hit(const FindArgs<T>& a, long long i) {
    if (a.vvalid && !bit_at(a.vvalid, a.vbit_off + i)) return false;
    return SortKey<T>::of(a.values[i]) == a.key;
}

template <typename T, int LANES>
__global__ void __launch_bounds__(kThreads)
k_list_find(const FindArgs<T> a, LongWork* __restrict__ work) {
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    const long long j = t / LANES;
    const int lane = threadIdx.x & 31, sub = lane & (LANES - 1);
    const bool mine = j < a.len;
    long long b = 0, e = 0;
    bool deferred = false;
    if (mine && (!a.lvalid || bit_at(a.lvalid, j))) { b = a.off[j]; e = a.off[j + 1]; }
    if (e - b > kLaneRounds * LANES) {
        if (sub == 0) {
            const unsigned int nseg = (unsigned int)((e - b + kLongList - 1) / kLongList);
            const unsigned long long old = atomicAdd(&work->counter, (1ull << 32) | nseg);
            work->item[old >> 32] = LongList{(unsigned long long)j, (unsigned long long)b, (unsigned long long)e, (unsigned int)old, nseg};
        }
        deferred = true;
        e = b;
    }
    long long found = -1;
    const unsigned group_mask = (LANES == 32 ? 0xffffffffu : ((1u << LANES) - 1u)) << (lane & ~(LANES - 1));
    for (long long r = 0;; r++) {
        const long long i = b + r * LANES + sub;
        const bool hit = found < 0 && i < e && find_hit(a, i);
        const unsigned mine_bits = __ballot_sync(0xffffffffu, hit) & group_mask;
        if (found < 0 && mine_bits) found = r * LANES + (__ffs(mine_bits) - 1 - (lane & ~(LANES - 1)));
        const bool more = found < 0 && b + (r + 1) * LANES < e;
        if (!__any_sync(0xffffffffu, more)) break;
    }
    if (!mine || sub != 0 || deferred) return;
    if (a.mode == 1) a.pos[j] = found >= 0 ? (int32_t)(found + 1) : 0;
    else if (found >= 0) atomicOr(&a.bits[j >> 5], 1u << (j & 31));
}

// One CTA per segment of a long list (grid-stride: the segment count is only known on the device); best[item] = the first match.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_list_find_long(const FindArgs<T> a, const LongWork* __restrict__ work, unsigned long long* __restrict__ best) {
    const unsigned long long cnt = work->counter;
    const unsigned int n_items = (unsigned int)(cnt >> 32), n_seg = (unsigned int)cnt;
    __shared__ unsigned long long s_best;
    for (unsigned int w = blockIdx.x; w < n_seg; w += gridDim.x) {
        unsigned int lo = 0, hi = n_items - 1;   // the last item whose first segment is <= w
        while (lo < hi) {
            const unsigned int mid = (lo + hi + 1) >> 1;
            if (work->item[mid].seg0 <= w) lo = mid; else hi = mid - 1;
        }
        const unsigned int k = lo;
        const LongList it = work->item[k];
        const long long sb = (long long)it.b + (long long)(w - it.seg0) * kLongList, se = min((long long)it.e, sb + kLongList);
        if (threadIdx.x == 0) s_best = ~0ull;
        __syncthreads();
        unsigned long long m = ~0ull;
        for (long long i = sb + threadIdx.x; i < se && m == ~0ull; i += kThreads)
            if (find_hit(a, i)) m = (unsigned long long)i;
        if (m != ~0ull) atomicMin(&s_best, m);
        __syncthreads();
        if (threadIdx.x == 0 && s_best != ~0ull) atomicMin(&best[k], s_best);
        __syncthreads();
    }
}

template <typename T>
__global__ void k_list_find_long_finish(const FindArgs<T> a, const LongWork* __restrict__ work, const unsigned long long* __restrict__ best) {
    const unsigned int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= (unsigned int)(work->counter >> 32)) return;
    const LongList it = work->item[k];
    const long long j = (long long)it.list;
    if (a.mode == 1) a.pos[j] = best[k] != ~0ull ? (int32_t)(best[k] - it.b + 1) : 0;
    else if (best[k] != ~0ull) atomicOr(&a.bits[j >> 5], 1u << (j & 31));
}

// Every deferred list has more than kLaneRounds elements (LANES >= 1).
static size_t long_capacity(long long n_elem) { return (size_t)(n_elem / kLaneRounds) + 2; }

size_t list_find_scratch_bytes(long long n_elem) {
    const size_t cap = long_capacity(n_elem);
    return 64 + cap * sizeof(LongList) + cap * 8 + 256;
}

template <typename T>
static cudaError_t find_typed(const int32_t* off, const uint32_t* lvalid, long long len, long long n_elem, const void* values, const uint32_t* vvalid,
                              int vbit_off, uint64_t value_bits, int mode, uint32_t* bits, int32_t* pos, void* scratch, int sm_count, cudaStream_t s) {
    T v;
    memcpy(&v, &value_bits, sizeof(T));
    FindArgs<T> a{off, lvalid, len, (const T*)values, vvalid, vbit_off, 0ull, mode, bits, pos};
    // the host computes the search key with the device's rule (SortKey is host-callable only through this copy)
    if constexpr (IsFloat<T>::value) {
        if (v != v) a.key = sizeof(T) == 4 ? 0xffffffffull : ~0ull;
        else {
            if (v == (T)0) v = (T)0;
            unsigned long long u = 0;
            memcpy(&u, &v, sizeof(T));
            const int sh = 8 * (int)sizeof(T) - 1;
            const unsigned long long all = sizeof(T) == 4 ? 0xffffffffull : ~0ull;
            a.key = (u >> sh) ? (~u & all) : (u | (1ull << sh));
        }
    } else if constexpr ((T)-1 < (T)0) {
        using U = typename UnsignedOf<T>::type;
        a.key = (unsigned long long)(U)((U)v ^ (U)((U)1 << (8 * sizeof(T) - 1)));
    } else {
        a.key = (unsigned long long)v;
    }
    LongWork* work = (LongWork*)scratch;
    const size_t cap = long_capacity(n_elem);
    unsigned long long* best = (unsigned long long*)((char*)scratch + 64 + cap * sizeof(LongList));
    best = (unsigned long long*)(((uintptr_t)best + 7) & ~(uintptr_t)7);
    cudaError_t e = cudaMemsetAsync(work, 0, 8, s);
    if (e == cudaSuccess) e = cudaMemsetAsync(best, 0xff, cap * 8, s);
    if (e != cudaSuccess) return e;
    const long long avg = n_elem / len;
    const int lanes = avg > 64 ? 32 : avg > 4 ? 8 : 1;
    const unsigned grid = (unsigned)((len * lanes + kThreads - 1) / kThreads);
    if (lanes == 32) k_list_find<T, 32><<<grid, kThreads, 0, s>>>(a, work);
    else if (lanes == 8) k_list_find<T, 8><<<grid, kThreads, 0, s>>>(a, work);
    else k_list_find<T, 1><<<grid, kThreads, 0, s>>>(a, work);
    if (n_elem > kLaneRounds * lanes) {   // a long list is possible: both kernels find nothing to do when there is none
        k_list_find_long<T><<<(unsigned)(sm_count * 4), kThreads, 0, s>>>(a, work, best);
        k_list_find_long_finish<T><<<(unsigned)((cap + 127) / 128), 128, 0, s>>>(a, work, best);
    }
    return cudaGetLastError();
}

// One list chunk.  scratch: list_find_scratch_bytes(n_elem).  bits (contains, zeroed by the caller) or pos (position).
cudaError_t launch_list_find(int dtype, const int32_t* off, const uint32_t* lvalid, long long len, long long n_elem, const void* values,
                             const uint32_t* vvalid, int vbit_off, uint64_t value_bits, int mode, uint32_t* bits, int32_t* pos, void* scratch,
                             int sm_count, cudaStream_t s) {
    if (len <= 0) return cudaSuccess;
#define BDF_FIND(T) find_typed<T>(off, lvalid, len, n_elem, values, vvalid, vbit_off, value_bits, mode, bits, pos, scratch, sm_count, s)
    switch (dtype) {
        case T_I8: return BDF_FIND(int8_t);
        case T_I16: return BDF_FIND(int16_t);
        case T_I32: return BDF_FIND(int32_t);
        case T_I64: return BDF_FIND(int64_t);
        case T_U8: return BDF_FIND(uint8_t);
        case T_U16: return BDF_FIND(uint16_t);
        case T_U32: return BDF_FIND(uint32_t);
        case T_U64: return BDF_FIND(uint64_t);
        case T_F32: return BDF_FIND(float);
        case T_F64: return BDF_FIND(double);
        default: return cudaErrorInvalidValue;
    }
#undef BDF_FIND
}

// ---- element -> list ------------------------------------------------------------------------------------------------------------
// Threads cover the global positions from elem0 rounded down to a word, so every warp writes one whole (or partial) word.
__global__ void __launch_bounds__(kThreads)
k_list_parent(const int32_t* __restrict__ off, const uint32_t* __restrict__ lvalid, const uint32_t* __restrict__ and_valid, long long len,
              long long n_elem, long long list0, long long elem0, uint32_t* __restrict__ parent, uint32_t* __restrict__ inlist) {
    const long long g = (elem0 & ~31LL) + (long long)blockIdx.x * kThreads + threadIdx.x;
    const long long e = g - elem0;
    bool v = false;
    if (e >= 0 && e < n_elem) {
        const long long j = list_of(off, len, e);
        parent[g] = (uint32_t)(list0 + j);
        v = (!lvalid || bit_at(lvalid, j)) && (!and_valid || bit_at(and_valid, j));
    }
    const unsigned w = __ballot_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && w) atomicOr(&inlist[g >> 5], w);
}

cudaError_t launch_list_parent(const int32_t* off, const uint32_t* lvalid, const uint32_t* and_valid, long long len, long long n_elem, long long list0,
                               long long elem0, uint32_t* parent, uint32_t* inlist, cudaStream_t s) {
    if (n_elem <= 0) return cudaSuccess;
    const long long n = elem0 - (elem0 & ~31LL) + n_elem;
    k_list_parent<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, s>>>(off, lvalid, and_valid, len, n_elem, list0, elem0, parent, inlist);
    return cudaGetLastError();
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_list_remove_mask(const T* __restrict__ values, const uint32_t* __restrict__ vvalid, int vbit_off, long long n_elem, long long elem0,
                   unsigned long long key, const uint32_t* __restrict__ inlist, uint32_t* __restrict__ keep) {
    const long long g = (elem0 & ~31LL) + (long long)blockIdx.x * kThreads + threadIdx.x;
    const long long e = g - elem0;
    bool k = false;
    if (e >= 0 && e < n_elem && bit_at(inlist, g)) {
        const bool valid = !vvalid || bit_at(vvalid, vbit_off + e);
        k = !(valid && SortKey<T>::of(values[e]) == key);
    }
    const unsigned w = __ballot_sync(0xffffffffu, k);
    if ((threadIdx.x & 31) == 0 && w) atomicOr(&keep[g >> 5], w);
}

template <typename T>
static cudaError_t remove_typed(const void* values, const uint32_t* vvalid, int vbit_off, long long n_elem, long long elem0, uint64_t value_bits,
                                const uint32_t* inlist, uint32_t* keep, cudaStream_t s) {
    T v;
    memcpy(&v, &value_bits, sizeof(T));
    unsigned long long key;
    if constexpr (IsFloat<T>::value) {
        if (v != v) key = sizeof(T) == 4 ? 0xffffffffull : ~0ull;
        else {
            if (v == (T)0) v = (T)0;
            unsigned long long u = 0;
            memcpy(&u, &v, sizeof(T));
            const int sh = 8 * (int)sizeof(T) - 1;
            const unsigned long long all = sizeof(T) == 4 ? 0xffffffffull : ~0ull;
            key = (u >> sh) ? (~u & all) : (u | (1ull << sh));
        }
    } else if constexpr ((T)-1 < (T)0) {
        using U = typename UnsignedOf<T>::type;
        key = (unsigned long long)(U)((U)v ^ (U)((U)1 << (8 * sizeof(T) - 1)));
    } else {
        key = (unsigned long long)v;
    }
    const long long n = elem0 - (elem0 & ~31LL) + n_elem;
    k_list_remove_mask<T><<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, s>>>((const T*)values, vvalid, vbit_off, n_elem, elem0, key, inlist, keep);
    return cudaGetLastError();
}

cudaError_t launch_list_remove_mask(int dtype, const void* values, const uint32_t* vvalid, int vbit_off, long long n_elem, long long elem0,
                                    uint64_t value_bits, const uint32_t* inlist, uint32_t* keep, cudaStream_t s) {
    if (n_elem <= 0) return cudaSuccess;
#define BDF_RM(T) remove_typed<T>(values, vvalid, vbit_off, n_elem, elem0, value_bits, inlist, keep, s)
    switch (dtype) {
        case T_I8: return BDF_RM(int8_t);
        case T_I16: return BDF_RM(int16_t);
        case T_I32: return BDF_RM(int32_t);
        case T_I64: return BDF_RM(int64_t);
        case T_U8: return BDF_RM(uint8_t);
        case T_U16: return BDF_RM(uint16_t);
        case T_U32: return BDF_RM(uint32_t);
        case T_U64: return BDF_RM(uint64_t);
        case T_F32: return BDF_RM(float);
        case T_F64: return BDF_RM(double);
        default: return cudaErrorInvalidValue;
    }
#undef BDF_RM
}

// ---- sort-based set functions ---------------------------------------------------------------------------------------------------
// Sorted position i: perm[i] = the element's position in the concatenated input, head bit i = a new (list, value) group starts here,
// pvalid bit i = the element belongs to a list that takes part.  Elements at positions >= split are the "a" side (the b side comes
// first in except / intersect, so a group is [b elements][a elements], each part in input order).
//   mode 0 (distinct, union)  keep the group head: the first occurrence in input order;
//   mode 1 (except)           keep the head if it is an a element: then the group has no b element;
//   mode 2 (intersect)        keep the first a element of a group that also has a b element.
__global__ void __launch_bounds__(kThreads)
k_list_mark(const uint32_t* __restrict__ perm, const uint32_t* __restrict__ head, const uint32_t* __restrict__ pvalid, long long n, long long split,
            int mode, uint32_t* __restrict__ keep) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= n || !bit_at(pvalid, i)) return;
    const long long p = perm[i];
    const bool h = bit_at(head, i), is_a = p >= split;
    bool k;
    if (mode == 0) k = h;
    else if (mode == 1) k = h && is_a;
    else k = !h && is_a && (long long)perm[i - 1] < split;
    if (k) atomicOr(&keep[p >> 5], 1u << (p & 31));
}

cudaError_t launch_list_mark(const uint32_t* perm, const uint32_t* head, const uint32_t* pvalid, long long n, long long split, int mode, uint32_t* keep,
                             cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_list_mark<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, s>>>(perm, head, pvalid, n, split, mode, keep);
    return cudaGetLastError();
}

// out[j] = mult * (the number of kept elements of lists before j), j = 0 .. n_lists; kp: the kept elements' list numbers, ascending.
__global__ void __launch_bounds__(kThreads)
k_list_offsets(const uint32_t* __restrict__ kp, long long n_kept, long long n_lists, long long mult, int32_t* __restrict__ out) {
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (j > n_lists) return;
    out[j] = (int32_t)(mult * (j == n_lists ? n_kept : lower_bound_u32_list(kp, n_kept, j)));
}

cudaError_t launch_list_offsets(const uint32_t* kp, long long n_kept, long long n_lists, long long mult, int32_t* out, cudaStream_t s) {
    k_list_offsets<<<(unsigned)((n_lists + 1 + kThreads - 1) / kThreads), kThreads, 0, s>>>(kp, n_kept, n_lists, mult, out);
    return cudaGetLastError();
}

// array_repeat: output element o of list j is kept element (o - count * base[j]) mod size_j of the list, whose input position is rows[..].
__global__ void __launch_bounds__(kThreads)
k_list_repeat(const int32_t* __restrict__ base, long long n_lists, long long count, const uint32_t* __restrict__ rows, long long n_out,
              uint32_t* __restrict__ src) {
    const long long o = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (o >= n_out) return;
    long long lo = 0, hi = n_lists - 1;   // the last list with count * base[j] <= o
    while (lo < hi) {
        const long long mid = (lo + hi + 1) >> 1;
        if (count * (long long)__ldg(base + mid) <= o) lo = mid; else hi = mid - 1;
    }
    const long long b = base[lo], size = (long long)base[lo + 1] - b;
    src[o] = rows[b + (o - count * b) % size];
}

cudaError_t launch_list_repeat(const int32_t* base, long long n_lists, long long count, const uint32_t* rows, long long n_out, uint32_t* src, cudaStream_t s) {
    if (n_out <= 0) return cudaSuccess;
    k_list_repeat<<<(unsigned)((n_out + kThreads - 1) / kThreads), kThreads, 0, s>>>(base, n_lists, count, rows, n_out, src);
    return cudaGetLastError();
}

// ---- size, and the validity of max / min ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_list_size(const int32_t* __restrict__ off, const uint32_t* __restrict__ lvalid, long long len, int32_t* __restrict__ out) {
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (j < len) out[j] = (!lvalid || bit_at(lvalid, j)) ? off[j + 1] - off[j] : -1;
}

cudaError_t launch_list_size(const int32_t* off, const uint32_t* lvalid, long long len, int32_t* out, cudaStream_t s) {
    if (len <= 0) return cudaSuccess;
    k_list_size<<<(unsigned)((len + kThreads - 1) / kThreads), kThreads, 0, s>>>(off, lvalid, len, out);
    return cudaGetLastError();
}

// valid = the list is valid and has a valid element (nonempty: k_group_reduce's bitmap); *empty = some valid list has no element.
__global__ void __launch_bounds__(kThreads)
k_list_minmax_valid(const int32_t* __restrict__ off, const uint32_t* __restrict__ lvalid, const uint32_t* __restrict__ nonempty, long long len,
                    uint32_t* __restrict__ valid, int* __restrict__ empty) {
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool v = false;
    if (j < len) {
        const bool lv = !lvalid || bit_at(lvalid, j);
        if (lv && off[j + 1] == off[j]) *empty = 1;
        v = lv && bit_at(nonempty, j);
    }
    const unsigned w = __ballot_sync(0xffffffffu, v);
    if ((threadIdx.x & 31) == 0 && j < len) valid[j >> 5] = w;
}

cudaError_t launch_list_minmax_valid(const int32_t* off, const uint32_t* lvalid, const uint32_t* nonempty, long long len, uint32_t* valid, int* empty,
                                     cudaStream_t s) {
    if (len <= 0) return cudaSuccess;
    k_list_minmax_valid<<<(unsigned)((len + kThreads - 1) / kThreads), kThreads, 0, s>>>(off, lvalid, nonempty, len, valid, empty);
    return cudaGetLastError();
}

// ---- take / filter of whole lists -----------------------------------------------------------------------------------------------
// The list chunk of global list row r: the last chunk whose start is <= r (empty chunks share their start with the next one).
__device__ __forceinline__ int list_chunk_of(const ListChunkDesc* __restrict__ t, int n, long long r) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (t[mid].start <= r) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// Output list i is source list idx[i] (take: a global row; local: a row of list chunk ic, where ic is the index chunk of i).
// sizes[i] = its element count, first[i] = its first element in the concatenated children; its validity bit goes to bit
// (i - chunk start) of vout[ic] (local) or bit i of vout[0]; nulls[ic or 0] counts the null outputs.
__global__ void __launch_bounds__(kThreads)
k_list_take_sizes(const SortChunk* __restrict__ idx, int n_idx, long long n, const ListChunkDesc* __restrict__ lists, int n_lists, long long total,
                  int local, uint32_t* const* __restrict__ vout, unsigned long long* __restrict__ sizes, uint32_t* __restrict__ first,
                  unsigned long long* __restrict__ nulls, int* __restrict__ flags) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool valid = false;
    int ic = 0;
    long long il = i;
    if (i < n) {
        ic = n_idx == 1 ? 0 : chunk_of(idx, n_idx, i);
        const SortChunk ich = idx[ic];
        il = i - ich.start;
        unsigned long long size = 0;
        uint32_t f = 0;
        if (!ich.validity || chunk_bit(ich.validity, ich.bit_off + il)) {
            const long long r0 = (long long)((const uint32_t*)ich.values)[il];
            const long long r = local ? lists[ic].start + r0 : r0;
            if (r >= total) atomicOr(flags, 1);   // arrow take: index out of bounds is an error
            else {
                const int lc = local ? ic : (n_lists == 1 ? 0 : list_chunk_of(lists, n_lists, r));
                const ListChunkDesc d = lists[lc];
                const long long j = r - d.start;
                if (!d.valid || bit_at(d.valid, j)) {
                    valid = true;
                    const int32_t b = __ldg(d.off + j);
                    size = (unsigned long long)(__ldg(d.off + j + 1) - b);
                    f = (uint32_t)(d.elem0 + b);
                }
            }
        }
        sizes[i] = size;
        first[i] = f;
    }
    const int key = i < n ? (local ? ic : 0) : -1;
    // validity: lanes that write the same word of the same chunk OR their bits together; one atomic per word
    const long long bit = local ? il : i;
    const unsigned long long word = i < n && valid ? (unsigned long long)(uintptr_t)(vout[key] + (bit >> 5)) : 0ull;
    const unsigned same = __match_any_sync(0xffffffffu, word);
    const unsigned bits = __reduce_or_sync(same, valid ? 1u << (bit & 31) : 0u);
    if (word && (threadIdx.x & 31) == __ffs(same) - 1) atomicOr((uint32_t*)(uintptr_t)word, bits);
    // null outputs per chunk, one atomic per chunk a warp touches
    const unsigned same_chunk = __match_any_sync(0xffffffffu, key);
    const unsigned n_null = __popc(__ballot_sync(0xffffffffu, i < n && !valid) & same_chunk);
    if (key >= 0 && n_null && (threadIdx.x & 31) == __ffs(same_chunk) - 1) atomicAdd(nulls + key, (unsigned long long)n_null);
}

cudaError_t launch_list_take_sizes(const void* idx_table, int n_idx, long long n, const void* list_table, int n_lists, long long total, int local,
                                   uint32_t* const* vout, unsigned long long* sizes, uint32_t* first, unsigned long long* nulls, int* flags,
                                   cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_list_take_sizes<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, s>>>((const SortChunk*)idx_table, n_idx, n,
                                                                                     (const ListChunkDesc*)list_table, n_lists, total, local, vout,
                                                                                     sizes, first, nulls, flags);
    return cudaGetLastError();
}

// Output element o belongs to output list p (the last p with off[p] <= o) and is element o - off[p] of its source list.
__global__ void __launch_bounds__(kThreads)
k_list_take_rows(const unsigned long long* __restrict__ off, long long n, const uint32_t* __restrict__ first, long long n_out, uint32_t* __restrict__ src) {
    const long long o = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (o >= n_out) return;
    long long lo = 0, hi = n - 1;
    while (lo < hi) {
        const long long mid = (lo + hi + 1) >> 1;
        if ((long long)__ldg(off + mid) <= o) lo = mid; else hi = mid - 1;
    }
    src[o] = __ldg(first + lo) + (uint32_t)(o - (long long)__ldg(off + lo));
}

cudaError_t launch_list_take_rows(const unsigned long long* off, long long n, const uint32_t* first, long long n_out, uint32_t* src, cudaStream_t s) {
    if (n_out <= 0) return cudaSuccess;
    k_list_take_rows<<<(unsigned)((n_out + kThreads - 1) / kThreads), kThreads, 0, s>>>(off, n, first, n_out, src);
    return cudaGetLastError();
}

__global__ void __launch_bounds__(kThreads)
k_list_rebase(const unsigned long long* __restrict__ off, long long len, int32_t* __restrict__ out) {
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (j <= len) out[j] = (int32_t)(off[j] - off[0]);
}

cudaError_t launch_list_rebase(const unsigned long long* off, long long len, int32_t* out, cudaStream_t s) {
    k_list_rebase<<<(unsigned)((len + 1 + kThreads - 1) / kThreads), kThreads, 0, s>>>(off, len, out);
    return cudaGetLastError();
}

// out[g] = the number of kept sorted rows before starts[g] (kept: ascending), g < n_groups; out[n_groups] = n_kept.
__global__ void __launch_bounds__(kThreads)
k_list_ranks(const uint32_t* __restrict__ kept, long long n_kept, const uint32_t* __restrict__ starts, long long n_groups, int32_t* __restrict__ out) {
    const long long g = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (g > n_groups) return;
    out[g] = (int32_t)(g == n_groups ? n_kept : lower_bound_u32_list(kept, n_kept, __ldg(starts + g)));
}

cudaError_t launch_list_ranks(const uint32_t* kept, long long n_kept, const uint32_t* starts, long long n_groups, int32_t* out, cudaStream_t s) {
    k_list_ranks<<<(unsigned)((n_groups + 1 + kThreads - 1) / kThreads), kThreads, 0, s>>>(kept, n_kept, starts, n_groups, out);
    return cudaGetLastError();
}

}  // namespace bdf
