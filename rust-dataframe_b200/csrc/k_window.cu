// k_window.cu -- window functions over PARTITION BY / ORDER BY (WindowFunctions, src/functions/window.rs:1-11, and WindowSpec,
// src/window.rs:8-22: stubs in the reference).
//
// The host (runtime.cu window_dev) sorts the rows by (partition keys ascending, order keys with their directions) with the stable
// radix lexsort, gathers the keys, marks the first row of every partition (P heads) and of every peer group (Q heads, a superset
// of P) with k_group_heads, and compacts the head positions with filter(iota, heads).  The kernels work in that sorted space,
// positions i = 0..n-1.  The host scans the popcounts of the head words first (launch_scan_popcount, k_scan.cu): prefix[w] is the
// number of runs starting before position 32w, so the run of position i -- and through the compacted starts its first and last
// position -- costs O(1) (no binary search per row).
//   k_window_rank    per position: partition and peer bounds -> row_number, rank, dense_rank, percent_rank, cume_dist, written
//                    to out[perm[i]] (the caller's row order), and the gather indices that bring a sorted-order column back to
//                    row order: i itself (the inverse permutation), the last peer of i, the last row of i's partition.
//   k_window_shift   lag / lead: x at position i -/+ k when that lies inside i's partition, else the default or NULL.
//   k_window_scan    segmented inclusive scan with the group fold's accumulators (group_acc.cuh): reduce-then-scan over a FIXED
//                    tile decomposition -- (1) every tile folds its rows into (a partition starts here, aggregate since the last
//                    start), (2) k_window_carry, one CTA, scans those tile records into every tile's carry-in, (3) every tile
//                    rescans its rows from its carry.  The order in which values are combined depends only on n, so float sums
//                    are the same bits on every run; a decoupled look-back would combine predecessors in a timing-dependent order.
//   k_window_level   bounded frames: one level of a radix-32 prefix / suffix hierarchy of the scan's accumulator.  Level 0 holds,
//                    for every position, the inclusive prefix and suffix of its aligned block of 32 values; level L + 1 does the
//                    same over the block totals of level L, up to the first level of at most 32 items (~2.07 n records in all).
//   k_window_frame_agg   per position: the frame [s, e] (frame_bounds: ROWS arithmetic, or a binary search of the order key for
//                    RANGE), then a fixed sequence of terms: while s and e lie in different blocks, suffix(s) on the left and
//                    prefix(e) on the right, one level up; then a fold of at most 32 items.  Every term is an aggregate of rows
//                    inside the frame, so float sums stay accurate relative to the frame, and the order of the terms depends only on
//                    (s, e): the same bits on every run and under any chunking.  The cost does not grow with the frame's width.
//   k_window_frame_value first_value / last_value / nth_value: a read at s, e or s + n - 1, or with IGNORE NULLS the rank of the valid
//                    slots (the popcount prefix of the validity words) and a search for the wanted rank inside [s, e].
// Values are read through a chunk table (SortChunk), so the call without keys reads the caller's chunks in place and writes row
// order directly.
#include "group_acc.cuh"
#include "sort_keys.cuh"

#include <cstring>

namespace bdf {

constexpr int kWinItems = 8;                       // consecutive rows per thread in the scan
constexpr int kWinTile = kThreads * kWinItems;     // 2048 rows per scan tile
constexpr int kWinCarryThreads = 1024;
enum : int { WIN_SUM = 0, WIN_COUNT, WIN_MIN, WIN_MAX, WIN_AVG };   // the aggregate a scan writes

// ---- runs ----------------------------------------------------------------------------------------------------------------
struct WinHeads { const uint32_t* words; const unsigned long long* prefix; const uint32_t* starts; long long n_runs; };
struct WinRuns {
    WinHeads p;   // partitions; words == null: the whole column is one partition
    WinHeads q;   // peer groups; words == null: every row of a partition is a peer
    long long n;
};

__device__ __forceinline__ long long run_of(const WinHeads& h, long long i) {
    const uint32_t w = __ldg(h.words + (i >> 5));
    const uint32_t below = (2u << (i & 31)) - 1u;   // bits 0..i&31 (all 32 when i&31 == 31: 2u << 31 wraps to 0)
    return (long long)__ldg(h.prefix + (i >> 5)) + __popc(w & below) - 1;
}
__device__ __forceinline__ void run_bounds(const WinHeads& h, long long n, long long r, long long* first, long long* last) {
    *first = __ldg(h.starts + r);
    *last = (r + 1 < h.n_runs ? (long long)__ldg(h.starts + r + 1) : n) - 1;
}

struct WinPos { long long ps, pe, qs, qe, dense; };
__device__ __forceinline__ WinPos win_pos(const WinRuns& r, long long i, bool need_q) {
    WinPos o;
    if (r.p.words) run_bounds(r.p, r.n, run_of(r.p, i), &o.ps, &o.pe);
    else { o.ps = 0; o.pe = r.n - 1; }
    o.qs = o.ps; o.qe = o.pe; o.dense = 1;
    if (need_q && r.q.words) {
        const long long q = run_of(r.q, i);
        run_bounds(r.q, r.n, q, &o.qs, &o.qe);
        o.dense = q - run_of(r.q, o.ps) + 1;   // a partition start is always a peer start
    }
    return o;
}

// ---- ranking functions and gather indices -------------------------------------------------------------------------------
struct WinRankOut {
    uint32_t *row_number, *rank, *dense_rank;
    double *percent_rank, *cume_dist;
    uint32_t *inv, *range_end, *part_end;   // row r -> its sorted position, its last peer's, its partition's last
};

__global__ void __launch_bounds__(kThreads)
k_window_rank(const WinRuns runs, const uint32_t* __restrict__ perm, const WinRankOut o) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= runs.n) return;
    const bool need_q = o.rank || o.dense_rank || o.percent_rank || o.cume_dist || o.range_end;
    const WinPos p = win_pos(runs, i, need_q);
    const long long r = perm ? (long long)perm[i] : i;
    const long long rows = p.pe - p.ps + 1;
    if (o.row_number) o.row_number[r] = (uint32_t)(i - p.ps + 1);
    if (o.rank) o.rank[r] = (uint32_t)(p.qs - p.ps + 1);
    if (o.dense_rank) o.dense_rank[r] = (uint32_t)p.dense;
    if (o.percent_rank) o.percent_rank[r] = rows == 1 ? 0.0 : (double)(p.qs - p.ps) / (double)(rows - 1);
    if (o.cume_dist) o.cume_dist[r] = (double)(p.qe - p.ps + 1) / (double)rows;
    if (o.inv) o.inv[r] = (uint32_t)i;
    if (o.range_end) o.range_end[r] = (uint32_t)p.qe;
    if (o.part_end) o.part_end[r] = (uint32_t)p.pe;
}

// ---- lag / lead ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool read_chunked(const SortChunk* __restrict__ x, int nx, long long j, const void** p, long long* local) {
    const int c = nx == 1 ? 0 : chunk_of(x, nx, j);
    const SortChunk ch = x[c];
    *local = j - ch.start;
    *p = ch.values;
    return ch.validity ? chunk_bit(ch.validity, ch.bit_off + *local) : true;
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_window_shift(const WinRuns runs, const SortChunk* __restrict__ x, int nx, long long k, int lead, T def, int has_def, T* __restrict__ out,
               uint32_t* __restrict__ vout) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool valid = false;
    if (i < runs.n) {
        const WinPos p = win_pos(runs, i, false);
        T v = (T)0;
        if (lead ? k <= p.pe - i : k <= i - p.ps) {   // the source row is inside the partition
            const long long j = lead ? i + k : i - k;
            const void* vals;
            long long local;
            valid = read_chunked(x, nx, j, &vals, &local);
            if (valid) v = ((const T*)vals)[local];
        } else if (has_def) {
            valid = true;
            v = def;
        }
        out[i] = v;
    }
    const unsigned word = __ballot_sync(0xffffffffu, valid);
    if ((threadIdx.x & 31) == 0 && i < runs.n) vout[i >> 5] = word;
}

// ---- segmented scan -----------------------------------------------------------------------------------------------------
template <typename T> struct WinAcc {
    GroupAggX<T> g;
    unsigned long long cnt;
    __device__ __forceinline__ void init() { g.init(); cnt = 0; }
    __device__ __forceinline__ void add(T x, bool ok) { g.add(x, ok, GroupFlip<T>::value); cnt += ok ? 1ull : 0ull; }
    __device__ __forceinline__ void merge(const WinAcc& o) { g.merge(o.g); cnt += o.cnt; }
};
// A segmented record: h = a partition starts inside the span, a = the aggregate from the last start (or the span's first row) on.
template <typename T> struct WinSeg { WinAcc<T> a; unsigned long long h; };

// (l then r): r alone when a partition starts inside r, else l's aggregate continued by r's.
template <typename T>
__device__ __forceinline__ WinSeg<T> seg_combine(const WinSeg<T>& l, const WinSeg<T>& r) {
    WinSeg<T> o = l;
    if (r.h) o.a = r.a;
    else o.a.merge(r.a);
    o.h = l.h | r.h;
    return o;
}
template <typename T>
__device__ __forceinline__ WinSeg<T> seg_identity() { WinSeg<T> s; s.a.init(); s.h = 0; return s; }

template <typename A>
__device__ __forceinline__ A shfl_up_rec(const A& a, int o) {
    static_assert(sizeof(A) % 8 == 0, "record of 64-bit words");
    A r;
    unsigned long long w[sizeof(A) / 8];
    memcpy(w, &a, sizeof(A));
#pragma unroll
    for (int k = 0; k < (int)(sizeof(A) / 8); k++) w[k] = __shfl_up_sync(0xffffffffu, w[k], o);
    memcpy(&r, w, sizeof(A));
    return r;
}

// The exclusive prefix of every thread's record over the CTA, combined in a fixed order: a warp scan, then the warp totals in
// warp order.  s_tot: NWARPS records of shared memory.
template <typename T, int NWARPS>
__device__ __forceinline__ WinSeg<T> block_exclusive(const WinSeg<T>& mine, WinSeg<T>* s_tot) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    WinSeg<T> inc = mine;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const WinSeg<T> up = shfl_up_rec(inc, o);
        if (lane >= o) inc = seg_combine(up, inc);
    }
    WinSeg<T> ex = shfl_up_rec(inc, 1);
    if (lane == 0) ex = seg_identity<T>();
    __syncthreads();   // s_tot may still be read by a previous call
    if (lane == 31) s_tot[warp] = inc;
    __syncthreads();
    WinSeg<T> pre = seg_identity<T>();
    for (int w = 0; w < warp; w++) pre = seg_combine(pre, s_tot[w]);
    return seg_combine(pre, ex);
}

template <typename T, int FN> struct WinOutT { using type = T; };
template <typename T> struct WinOutT<T, WIN_COUNT> { using type = long long; };
template <typename T> struct WinOutT<T, WIN_AVG> { using type = double; };

template <typename T, int FN>
__device__ __forceinline__ typename WinOutT<T, FN>::type win_result(const WinAcc<T>& a, bool* valid) {
    constexpr unsigned long long flip = GroupFlip<T>::value;
    *valid = true;
    if constexpr (FN == WIN_COUNT) return (long long)a.cnt;
    else if constexpr (FN == WIN_AVG) {
        *valid = a.cnt != 0;
        double s;
        if constexpr (IsFloat<T>::value) s = a.g.sum; else s = a.g.dsum;
        return a.cnt ? s / (double)a.cnt : 0.0;
    } else if constexpr (IsFloat<T>::value) {
        if constexpr (FN == WIN_SUM) return (T)a.g.sum;
        *valid = a.cnt != 0;
        return a.cnt ? FloatKey<T>::value(FN == WIN_MIN ? a.g.kmin : a.g.kmax) : (T)0;
    } else {
        using U = typename UnsignedOf<T>::type;
        if constexpr (FN == WIN_SUM) return (T)(U)a.g.a.sum;   // wrapping
        *valid = a.cnt != 0;
        return a.cnt ? (T)(U)((FN == WIN_MIN ? a.g.a.kmin : a.g.a.kmax) ^ flip) : (T)0;
    }
}

// Phase 1 (RESCAN false): tile b's record -> tiles[b].  Phase 3 (RESCAN true): every row's inclusive aggregate from carry[b].
// Rows go through shared memory both ways so that global loads and stores are coalesced while a thread owns 8 consecutive rows.
template <typename T, int FN, bool RESCAN>
__global__ void __launch_bounds__(kThreads)
k_window_scan(const SortChunk* __restrict__ x, int nx, const uint32_t* __restrict__ heads, long long n, WinSeg<T>* __restrict__ tiles,
              const WinAcc<T>* __restrict__ carry, typename WinOutT<T, FN>::type* __restrict__ out, uint32_t* __restrict__ vout) {
    using O = typename WinOutT<T, FN>::type;
    constexpr int kPad = kWinTile + kWinTile / kWinItems;   // one spare slot per 8 rows: thread t's rows start at 9t (no bank conflicts)
    __shared__ unsigned long long s_buf[kPad];
    __shared__ unsigned int s_ok[kWinTile / 32];
    __shared__ WinSeg<T> s_tot[kWarpsPerCta];
    const long long base = (long long)blockIdx.x * kWinTile;
    const int tid = threadIdx.x;
    // coalesced loads: slot e = k * 256 + tid
#pragma unroll
    for (int k = 0; k < kWinItems; k++) {   // every word of s_ok is one warp's ballot
        const int e = k * kThreads + tid;
        const long long j = base + e;
        T v = (T)0;
        bool ok = false;
        if (j < n) {
            const void* vals;
            long long local;
            ok = read_chunked(x, nx, j, &vals, &local);
            v = ((const T*)vals)[local];
        }
        *(T*)&s_buf[e + e / kWinItems] = v;
        const unsigned bal = __ballot_sync(0xffffffffu, ok);
        if ((tid & 31) == 0) s_ok[e >> 5] = bal;
    }
    __syncthreads();
    const long long r0 = base + (long long)tid * kWinItems;
    const unsigned okb = (s_ok[(tid * kWinItems) >> 5] >> ((tid * kWinItems) & 31)) & 0xffu;
    unsigned hb = 0;
    if (r0 < n) hb = heads ? (__ldg(heads + (r0 >> 5)) >> (r0 & 31)) & 0xffu : (r0 == 0 ? 1u : 0u);
    T v[kWinItems];
#pragma unroll
    for (int k = 0; k < kWinItems; k++) v[k] = *(const T*)&s_buf[tid * (kWinItems + 1) + k];
    WinSeg<T> mine = seg_identity<T>();
#pragma unroll
    for (int k = 0; k < kWinItems; k++) {
        if (r0 + k >= n) break;
        if ((hb >> k) & 1u) { mine.a.init(); mine.h = 1; }
        mine.a.add(v[k], (okb >> k) & 1u);
    }
    const WinSeg<T> ex = block_exclusive<T, kWarpsPerCta>(mine, s_tot);
    if constexpr (!RESCAN) {
        if (tid == kThreads - 1) tiles[blockIdx.x] = seg_combine(ex, mine);
    } else {
        WinSeg<T> from;
        from.a = carry[blockIdx.x];
        from.h = 0;
        WinAcc<T> a = seg_combine(from, ex).a;
        unsigned vb = 0;
        O res[kWinItems];
#pragma unroll
        for (int k = 0; k < kWinItems; k++) {
            res[k] = (O)0;
            if (r0 + k >= n) continue;
            if ((hb >> k) & 1u) a.init();
            a.add(v[k], (okb >> k) & 1u);
            bool valid;
            res[k] = win_result<T, FN>(a, &valid);
            vb |= (valid ? 1u : 0u) << k;
        }
        __syncthreads();   // every thread has read its rows out of s_buf
#pragma unroll
        for (int k = 0; k < kWinItems; k++) *(O*)&s_buf[tid * (kWinItems + 1) + k] = res[k];
        if (vout) store_bits<kWinItems>(vout, r0, vb, r0 < n);
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kWinItems; k++) {
            const int e = k * kThreads + tid;
            if (base + e < n) out[base + e] = *(const O*)&s_buf[e + e / kWinItems];
        }
    }
}

// Phase 2: one CTA turns the tile records into every tile's carry-in (the aggregate of its partition's rows before the tile).
// Thread t owns a contiguous range of tiles: a sequential fold, one block scan of the 1024 fold results, then the range again.
template <typename T>
__global__ void __launch_bounds__(kWinCarryThreads)
k_window_carry(const WinSeg<T>* __restrict__ tiles, long long n_tiles, WinAcc<T>* __restrict__ carry) {
    __shared__ WinSeg<T> s_tot[kWinCarryThreads / 32];
    const long long per = (n_tiles + kWinCarryThreads - 1) / kWinCarryThreads;
    const long long b = min(n_tiles, (long long)threadIdx.x * per), e = min(n_tiles, b + per);
    WinSeg<T> mine = seg_identity<T>();
    for (long long t = b; t < e; t++) mine = seg_combine(mine, tiles[t]);
    WinSeg<T> run = block_exclusive<T, kWinCarryThreads / 32>(mine, s_tot);
    for (long long t = b; t < e; t++) {
        carry[t] = run.a;
        run = seg_combine(run, tiles[t]);
    }
}

// ---- launchers ----------------------------------------------------------------------------------------------------------
// The three head arrays of one head bitmap (words, prefix from launch_scan_popcount, compacted starts) and the number of runs.
static WinRuns make_runs(const void* const* p, long long n_p, const void* const* q, long long n_q, long long n) {
    WinRuns r{};
    if (p) r.p = WinHeads{(const uint32_t*)p[0], (const unsigned long long*)p[1], (const uint32_t*)p[2], n_p};
    if (q) r.q = WinHeads{(const uint32_t*)q[0], (const unsigned long long*)q[1], (const uint32_t*)q[2], n_q};
    r.n = n;
    return r;
}

// p / q: {head words, prefix, starts} or null (one partition / peers = partition); outs: the 8 WinRankOut pointers in order, each
// may be null.
cudaError_t launch_window_rank(const void* const* p, long long n_p, const void* const* q, long long n_q, long long n, const uint32_t* perm,
                               void* const* outs, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const WinRankOut o{(uint32_t*)outs[0], (uint32_t*)outs[1], (uint32_t*)outs[2], (double*)outs[3], (double*)outs[4],
                       (uint32_t*)outs[5], (uint32_t*)outs[6], (uint32_t*)outs[7]};
    k_window_rank<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, s>>>(make_runs(p, n_p, q, n_q, n), perm, o);
    return cudaGetLastError();
}

// x: a chunk table (sort_table) of nx chunks; def_bits: the default's T::Native in the low bytes.
cudaError_t launch_window_shift(int dtype, const void* const* p, long long n_p, long long n, const void* x, int nx, long long k, int lead,
                                unsigned long long def_bits, int has_def, void* out, uint32_t* vout, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const WinRuns r = make_runs(p, n_p, nullptr, 0, n);
    const unsigned g = (unsigned)((n + kThreads - 1) / kThreads);
    const SortChunk* xc = (const SortChunk*)x;
    switch (dtype) {
#define BDF_SHIFT_CASE(ID, T)                                                                              \
    case ID: {                                                                                             \
        T d;                                                                                               \
        memcpy(&d, &def_bits, sizeof(T));                                                                  \
        k_window_shift<T><<<g, kThreads, 0, s>>>(r, xc, nx, k, lead, d, has_def, (T*)out, vout);          \
        break;                                                                                             \
    }
        BDF_SHIFT_CASE(0, int8_t) BDF_SHIFT_CASE(1, int16_t) BDF_SHIFT_CASE(2, int32_t) BDF_SHIFT_CASE(3, int64_t)
        BDF_SHIFT_CASE(4, uint8_t) BDF_SHIFT_CASE(5, uint16_t) BDF_SHIFT_CASE(6, uint32_t) BDF_SHIFT_CASE(7, uint64_t)
        BDF_SHIFT_CASE(8, float) BDF_SHIFT_CASE(9, double)
#undef BDF_SHIFT_CASE
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

size_t window_scan_scratch_bytes(long long n) {
    const size_t tiles = (size_t)((n + kWinTile - 1) / kWinTile);
    return tiles * (sizeof(WinSeg<long long>) + sizeof(WinAcc<long long>)) + 256;   // the largest records
}

template <typename T, int FN>
static cudaError_t scan_fn(const SortChunk* x, int nx, const uint32_t* heads, long long n, void* scratch, void* out, uint32_t* vout, cudaStream_t s) {
    const long long tiles = (n + kWinTile - 1) / kWinTile;
    WinSeg<T>* recs = (WinSeg<T>*)scratch;
    WinAcc<T>* carry = (WinAcc<T>*)((char*)scratch + (((size_t)tiles * sizeof(WinSeg<T>) + 15) & ~(size_t)15));
    using O = typename WinOutT<T, FN>::type;
    k_window_scan<T, WIN_SUM, false><<<(unsigned)tiles, kThreads, 0, s>>>(x, nx, heads, n, recs, nullptr, nullptr, nullptr);
    k_window_carry<T><<<1, kWinCarryThreads, 0, s>>>(recs, tiles, carry);
    k_window_scan<T, FN, true><<<(unsigned)tiles, kThreads, 0, s>>>(x, nx, heads, n, recs, carry, (O*)out, vout);
    return cudaGetLastError();
}

template <typename T>
static cudaError_t scan_typed(int fn, const SortChunk* x, int nx, const uint32_t* heads, long long n, void* scratch, void* out, uint32_t* vout,
                              cudaStream_t s) {
    switch (fn) {
        case WIN_SUM: return scan_fn<T, WIN_SUM>(x, nx, heads, n, scratch, out, vout, s);
        case WIN_COUNT: return scan_fn<T, WIN_COUNT>(x, nx, heads, n, scratch, out, vout, s);
        case WIN_MIN: return scan_fn<T, WIN_MIN>(x, nx, heads, n, scratch, out, vout, s);
        case WIN_MAX: return scan_fn<T, WIN_MAX>(x, nx, heads, n, scratch, out, vout, s);
        case WIN_AVG: return scan_fn<T, WIN_AVG>(x, nx, heads, n, scratch, out, vout, s);
        default: return cudaErrorInvalidValue;
    }
}

// fn: 0 sum, 1 count, 2 min, 3 max, 4 avg.  heads: the partition head words (null: one partition).  vout: the validity of min /
// max / avg (null for sum / count).  scratch: window_scan_scratch_bytes(n).
cudaError_t launch_window_scan(int dtype, int fn, const void* x, int nx, const uint32_t* heads, long long n, void* scratch, void* out, uint32_t* vout,
                               cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    if ((n + kWinTile - 1) / kWinTile > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    const SortChunk* xc = (const SortChunk*)x;
    switch (dtype) {
        case T_I8: return scan_typed<int8_t>(fn, xc, nx, heads, n, scratch, out, vout, s);
        case T_I16: return scan_typed<int16_t>(fn, xc, nx, heads, n, scratch, out, vout, s);
        case T_I32: return scan_typed<int32_t>(fn, xc, nx, heads, n, scratch, out, vout, s);
        case T_I64: return scan_typed<int64_t>(fn, xc, nx, heads, n, scratch, out, vout, s);
        case T_U8: return scan_typed<uint8_t>(fn, xc, nx, heads, n, scratch, out, vout, s);
        case T_U16: return scan_typed<uint16_t>(fn, xc, nx, heads, n, scratch, out, vout, s);
        case T_U32: return scan_typed<uint32_t>(fn, xc, nx, heads, n, scratch, out, vout, s);
        case T_U64: return scan_typed<uint64_t>(fn, xc, nx, heads, n, scratch, out, vout, s);
        case T_F32: return scan_typed<float>(fn, xc, nx, heads, n, scratch, out, vout, s);
        case T_F64: return scan_typed<double>(fn, xc, nx, heads, n, scratch, out, vout, s);
        default: return cudaErrorInvalidValue;
    }
}

// ---- bounded frames: [s, e] of every position -----------------------------------------------------------------------------
// The order key at sorted position j: its class (the numeric run is class 0 ascending, 1 descending; NaN sorts above every number,
// so it is class 1 ascending and 0 descending; null is class 2 both ways) and its value, exact in __int128 or as a double.
struct WinKey { int cls; __int128 i; double f; };

__device__ __forceinline__ WinKey win_key(const WinFrameDesc& f, long long j) {
    const void* p;
    long long local;
    const bool ok = read_chunked((const SortChunk*)f.key, f.key_chunks, j, &p, &local);
    WinKey k;
    k.i = 0;
    k.f = 0.0;
    int raw = 0;   // 0 number, 1 NaN, 2 null
    if (!ok) raw = 2;
    else switch (f.key_dtype) {
        case T_I8: k.i = ((const int8_t*)p)[local]; break;
        case T_I16: k.i = ((const int16_t*)p)[local]; break;
        case T_I32: k.i = ((const int32_t*)p)[local]; break;
        case T_I64: k.i = ((const long long*)p)[local]; break;
        case T_U8: k.i = ((const uint8_t*)p)[local]; break;
        case T_U16: k.i = ((const uint16_t*)p)[local]; break;
        case T_U32: k.i = ((const uint32_t*)p)[local]; break;
        case T_U64: k.i = (__int128)((const unsigned long long*)p)[local]; break;
        case T_F32: k.f = (double)((const float*)p)[local]; raw = k.f != k.f; break;
        default: k.f = ((const double*)p)[local]; raw = k.f != k.f; break;
    }
    k.cls = raw == 2 ? 2 : (f.key_desc ? 1 - raw : raw);
    return k;
}

// The first position j in [lo, hi) for which pred(j) holds (pred is false, then true, over the range); hi when there is none.
template <typename P>
__device__ __forceinline__ long long win_search(long long lo, long long hi, P pred) {
    while (lo < hi) {
        const long long mid = lo + ((hi - lo) >> 1);
        if (pred(mid)) hi = mid;
        else lo = mid + 1;
    }
    return lo;
}

__device__ __forceinline__ long long win_clamp(long long o) {   // offsets beyond any partition act alike; no overflow below
    const long long lim = 1ll << 34;
    return o < -lim ? -lim : (o > lim ? lim : o);
}

__device__ __forceinline__ void frame_bounds(const WinRuns& r, const WinFrameDesc& f, long long i, long long* s, long long* e) {
    const WinPos p = win_pos(r, i, f.kind == WIN_FR_PEERS);
    *s = p.ps;
    *e = p.pe;
    if (f.kind == WIN_FR_ROWS) {
        if (f.start != LLONG_MIN) *s = max(p.ps, i + win_clamp(f.start));
        if (f.end != LLONG_MAX) *e = min(p.pe, i + win_clamp(f.end));
        return;
    }
    if (f.kind == WIN_FR_PEERS) { *e = p.qe; return; }
    const bool is_f = f.key_dtype == T_F32 || f.key_dtype == T_F64;
    const bool s_unb = is_f ? f.start_f == -INFINITY : f.start == LLONG_MIN;
    const bool e_unb = is_f ? f.end_f == INFINITY : f.end == LLONG_MAX;
    if (s_unb && e_unb) return;
    const WinKey v = win_key(f, i);
    const int num = f.key_desc ? 1 : 0;
    const long long end = p.pe + 1;
    if (v.cls != num) {   // a null or NaN key: an offset bound is the edge of the row's own peer run
        if (!s_unb) *s = win_search(p.ps, end, [=](long long j) { return win_key(f, j).cls >= v.cls; });
        if (!e_unb) *e = win_search(p.ps, end, [=](long long j) { return win_key(f, j).cls > v.cls; }) - 1;
        return;
    }
    const long long a = win_search(p.ps, end, [=](long long j) { return win_key(f, j).cls >= num; });
    const long long b = win_search(a, end, [=](long long j) { return win_key(f, j).cls > num; });   // numbers: [a, b)
    // The keys of [a, b) run in the sort's direction.  Ascending: v + start <= k <= v + end; descending: v - end <= k <= v - start.
    if (!s_unb) {
        if (is_f) {
            const double t = f.key_desc ? __dsub_rn(v.f, f.start_f) : __dadd_rn(v.f, f.start_f);
            *s = win_search(a, b, [=](long long j) { const double k = win_key(f, j).f; return f.key_desc ? k <= t : k >= t; });
        } else {
            const __int128 t = f.key_desc ? v.i - (__int128)f.start : v.i + (__int128)f.start;
            *s = win_search(a, b, [=](long long j) { const __int128 k = win_key(f, j).i; return f.key_desc ? k <= t : k >= t; });
        }
    }
    if (!e_unb) {
        if (is_f) {
            const double t = f.key_desc ? __dsub_rn(v.f, f.end_f) : __dadd_rn(v.f, f.end_f);
            *e = win_search(a, b, [=](long long j) { const double k = win_key(f, j).f; return f.key_desc ? k < t : k > t; }) - 1;
        } else {
            const __int128 t = f.key_desc ? v.i - (__int128)f.end : v.i + (__int128)f.end;
            *e = win_search(a, b, [=](long long j) { const __int128 k = win_key(f, j).i; return f.key_desc ? k < t : k > t; }) - 1;
        }
    }
}

// ---- bounded frames: the prefix / suffix hierarchy --------------------------------------------------------------------------
constexpr int kWinMaxLevels = 8;   // 32^7 > 2^32 rows
template <typename T> struct WinLevels {
    WinAcc<T>* pre[kWinMaxLevels];
    WinAcc<T>* suf[kWinMaxLevels];
    long long cnt[kWinMaxLevels + 1];   // items of every level; cnt[levels] <= 32
    int levels;                         // levels with stored records
};

template <typename A>
__device__ __forceinline__ A shfl_down_rec(const A& a, int o) {
    static_assert(sizeof(A) % 8 == 0, "record of 64-bit words");
    A r;
    unsigned long long w[sizeof(A) / 8];
    memcpy(w, &a, sizeof(A));
#pragma unroll
    for (int k = 0; k < (int)(sizeof(A) / 8); k++) w[k] = __shfl_down_sync(0xffffffffu, w[k], o);
    memcpy(&r, w, sizeof(A));
    return r;
}

// Item j of level lvl: x at j on level 0, else the total of block j of the level below (its last prefix).
template <typename T>
__device__ __forceinline__ WinAcc<T> win_item(const WinLevels<T>& h, const SortChunk* __restrict__ x, int nx, int lvl, long long j) {
    WinAcc<T> a;
    if (lvl == 0) {
        const void* p;
        long long local;
        const bool ok = read_chunked(x, nx, j, &p, &local);
        a.init();
        a.add(ok ? ((const T*)p)[local] : (T)0, ok);
    } else {
        a = h.pre[lvl - 1][min(32 * j + 31, h.cnt[lvl - 1] - 1)];
    }
    return a;
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_window_level(const SortChunk* __restrict__ x, int nx, const WinLevels<T> h, int lvl) {
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    const int lane = threadIdx.x & 31;
    WinAcc<T> pre;
    pre.init();
    if (j < h.cnt[lvl]) pre = win_item(h, x, nx, lvl, j);
    WinAcc<T> suf = pre;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {   // a fixed-order warp scan each way over one aligned block of 32 items
        WinAcc<T> up = shfl_up_rec(pre, o);
        const WinAcc<T> dn = shfl_down_rec(suf, o);
        if (lane >= o) { up.merge(pre); pre = up; }
        if (lane + o < 32) suf.merge(dn);
    }
    if (j < h.cnt[lvl]) {
        h.pre[lvl][j] = pre;
        h.suf[lvl][j] = suf;
    }
}

// The aggregate of positions [s, e]: suffix / prefix terms level by level, then a fold of at most 32 items, in an order fixed by (s, e).
template <typename T>
__device__ __forceinline__ WinAcc<T> frame_fold(const WinLevels<T>& h, const SortChunk* __restrict__ x, int nx, long long s, long long e) {
    WinAcc<T> l, r;
    l.init();
    r.init();
    int lvl = 0;
    while (s <= e) {
        if ((s >> 5) == (e >> 5)) {
            for (long long j = s; j <= e; j++) l.merge(win_item(h, x, nx, lvl, j));
            break;
        }
        l.merge(h.suf[lvl][s]);
        WinAcc<T> t = h.pre[lvl][e];
        t.merge(r);
        r = t;
        s = (s >> 5) + 1;
        e = (e >> 5) - 1;
        lvl++;
    }
    l.merge(r);
    return l;
}

// __launch_bounds__(kThreads, 4) on the two frame kernels: without the occupancy hint ptxas held them to 32 registers and spilled.
template <typename T, int FN>
__global__ void __launch_bounds__(kThreads, 4)
k_window_frame_agg(const WinRuns runs, const WinFrameDesc f, const SortChunk* __restrict__ x, int nx, const WinLevels<T> h,
                   typename WinOutT<T, FN>::type* __restrict__ out, uint32_t* __restrict__ vout) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool valid = false;
    if (i < runs.n) {
        long long s, e;
        frame_bounds(runs, f, i, &s, &e);
        out[i] = win_result<T, FN>(frame_fold(h, x, nx, s, e), &valid);
    }
    const unsigned word = __ballot_sync(0xffffffffu, valid);
    if (vout && (threadIdx.x & 31) == 0 && i < runs.n) vout[i >> 5] = word;
}

// ---- bounded frames: first_value / last_value / nth_value ------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
k_window_valid_words(const SortChunk* __restrict__ x, int nx, long long n, uint32_t* __restrict__ words) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool ok = false;
    if (i < n) {
        const void* p;
        long long local;
        ok = read_chunked(x, nx, i, &p, &local);
    }
    const unsigned word = __ballot_sync(0xffffffffu, ok);
    if ((threadIdx.x & 31) == 0 && i < n) words[i >> 5] = word;
}

// Valid slots in [0, p] (p may be -1).
__device__ __forceinline__ long long valid_upto(const uint32_t* __restrict__ w, const unsigned long long* __restrict__ pre, long long p) {
    if (p < 0) return 0;
    const uint32_t below = (2u << (p & 31)) - 1u;
    return (long long)__ldg(pre + (p >> 5)) + __popc(__ldg(w + (p >> 5)) & below);
}

// The position of the r-th valid slot (1-based), known to lie in words [w0, w1].
__device__ __forceinline__ long long valid_select(const uint32_t* __restrict__ w, const unsigned long long* __restrict__ pre, long long r, long long w0,
                                                  long long w1) {
    const long long wd = win_search(w0, w1 + 1, [=](long long k) { return (long long)__ldg(pre + k) >= r; }) - 1;   // last word with prefix < r
    uint32_t bits = __ldg(w + wd);
    for (long long k = r - (long long)__ldg(pre + wd); k > 1; k--) bits &= bits - 1u;
    return 32 * wd + __ffs(bits) - 1;
}

// which: 0 first_value, 1 last_value, 2 nth_value (nth >= 1).  vwords / vprefix: the sorted validity and its popcount prefix for
// IGNORE NULLS, null for RESPECT NULLS.
template <typename T>
__global__ void __launch_bounds__(kThreads, 4)
k_window_frame_value(const WinRuns runs, const WinFrameDesc f, const SortChunk* __restrict__ x, int nx, int which, long long nth,
                     const uint32_t* __restrict__ vwords, const unsigned long long* __restrict__ vprefix, T* __restrict__ out,
                     uint32_t* __restrict__ vout) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    bool valid = false;
    if (i < runs.n) {
        long long s, e, j = -1;
        frame_bounds(runs, f, i, &s, &e);
        if (s <= e) {
            if (!vwords) {
                j = which == 0 ? s : which == 1 ? e : (nth - 1 <= e - s ? s + nth - 1 : -1);
            } else {
                const long long before = valid_upto(vwords, vprefix, s - 1), upto = valid_upto(vwords, vprefix, e);
                const long long have = upto - before;
                const long long k = which == 0 ? 1 : which == 1 ? have : nth;   // the k-th valid slot of the frame
                if (k >= 1 && k <= have) j = valid_select(vwords, vprefix, before + k, s >> 5, e >> 5);
            }
        }
        T v = (T)0;
        if (j >= 0) {
            const void* p;
            long long local;
            valid = read_chunked(x, nx, j, &p, &local);
            if (valid) v = ((const T*)p)[local];
        }
        out[i] = v;
    }
    const unsigned word = __ballot_sync(0xffffffffu, valid);
    if ((threadIdx.x & 31) == 0 && i < runs.n) vout[i >> 5] = word;
}

// ---- bounded frame launchers ------------------------------------------------------------------------------------------------
int window_frame_levels(long long n) {
    int l = 0;
    for (long long c = n; c > 32; c = (c + 31) / 32) l++;
    return l;
}

static size_t acc_bytes(int dtype) { return dtype_is_float(dtype) ? sizeof(WinAcc<double>) : sizeof(WinAcc<long long>); }
static size_t round256(size_t b) { return (b + 255) & ~(size_t)255; }

size_t window_frame_scratch_bytes(int dtype, long long n) {
    size_t b = 256;
    for (long long c = n; c > 32; c = (c + 31) / 32) b += 2 * round256((size_t)c * acc_bytes(dtype));
    return b;
}

template <typename T>
static WinLevels<T> levels_in(void* scratch, long long n) {
    WinLevels<T> h{};
    char* p = (char*)scratch;
    long long c = n;
    int l = 0;
    for (; c > 32; c = (c + 31) / 32, l++) {
        h.cnt[l] = c;
        h.pre[l] = (WinAcc<T>*)p;
        p += round256((size_t)c * sizeof(WinAcc<T>));
        h.suf[l] = (WinAcc<T>*)p;
        p += round256((size_t)c * sizeof(WinAcc<T>));
    }
    h.cnt[l] = c;
    h.levels = l;
    return h;
}

#define BDF_WIN_DTYPES(X) X(T_I8, int8_t) X(T_I16, int16_t) X(T_I32, int32_t) X(T_I64, int64_t) X(T_U8, uint8_t) X(T_U16, uint16_t) \
    X(T_U32, uint32_t) X(T_U64, uint64_t) X(T_F32, float) X(T_F64, double)

template <typename T>
static cudaError_t frame_build(const SortChunk* x, int nx, long long n, void* scratch, cudaStream_t s) {
    const WinLevels<T> h = levels_in<T>(scratch, n);
    for (int l = 0; l < h.levels; l++)
        k_window_level<T><<<(unsigned)((h.cnt[l] + kThreads - 1) / kThreads), kThreads, 0, s>>>(x, nx, h, l);
    return cudaGetLastError();
}

// Every level of x's hierarchy (window_frame_levels(n) launches) into scratch (window_frame_scratch_bytes).
cudaError_t launch_window_frame_build(int dtype, const void* x, int nx, long long n, void* scratch, cudaStream_t s) {
    const SortChunk* xc = (const SortChunk*)x;
    switch (dtype) {
#define BDF_BUILD_CASE(ID, T) case ID: return frame_build<T>(xc, nx, n, scratch, s);
        BDF_WIN_DTYPES(BDF_BUILD_CASE)
#undef BDF_BUILD_CASE
        default: return cudaErrorInvalidValue;
    }
}

template <typename T>
static cudaError_t frame_agg(int fn, const WinRuns& r, const WinFrameDesc& f, const SortChunk* x, int nx, long long n, void* scratch, void* out,
                             uint32_t* vout, cudaStream_t s) {
    const WinLevels<T> h = levels_in<T>(scratch, n);
    const unsigned g = (unsigned)((n + kThreads - 1) / kThreads);
    switch (fn) {
#define BDF_AGG_CASE(FN) \
    case FN: k_window_frame_agg<T, FN><<<g, kThreads, 0, s>>>(r, f, x, nx, h, (typename WinOutT<T, FN>::type*)out, vout); break;
        BDF_AGG_CASE(WIN_SUM) BDF_AGG_CASE(WIN_COUNT) BDF_AGG_CASE(WIN_MIN) BDF_AGG_CASE(WIN_MAX) BDF_AGG_CASE(WIN_AVG)
#undef BDF_AGG_CASE
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}

// fn: 0 sum, 1 count, 2 min, 3 max, 4 avg over the frames of f; scratch: x's hierarchy from launch_window_frame_build.
cudaError_t launch_window_frame_agg(int dtype, int fn, const void* const* p, long long n_p, const void* const* q, long long n_q, const WinFrameDesc& f,
                                    const void* x, int nx, long long n, void* scratch, void* out, uint32_t* vout, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const WinRuns r = make_runs(p, n_p, q, n_q, n);
    const SortChunk* xc = (const SortChunk*)x;
    switch (dtype) {
#define BDF_FAGG_CASE(ID, T) case ID: return frame_agg<T>(fn, r, f, xc, nx, n, scratch, out, vout, s);
        BDF_WIN_DTYPES(BDF_FAGG_CASE)
#undef BDF_FAGG_CASE
        default: return cudaErrorInvalidValue;
    }
}

cudaError_t launch_window_valid_words(const void* x, int nx, long long n, uint32_t* words, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    k_window_valid_words<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, s>>>((const SortChunk*)x, nx, n, words);
    return cudaGetLastError();
}

cudaError_t launch_window_frame_value(int dtype, int which, long long nth, const void* const* p, long long n_p, const void* const* q, long long n_q,
                                      const WinFrameDesc& f, const void* x, int nx, long long n, const uint32_t* vwords,
                                      const unsigned long long* vprefix, void* out, uint32_t* vout, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    const WinRuns r = make_runs(p, n_p, q, n_q, n);
    const unsigned g = (unsigned)((n + kThreads - 1) / kThreads);
    const SortChunk* xc = (const SortChunk*)x;
    switch (dtype) {
#define BDF_VALUE_CASE(ID, T)                                                                                              \
    case ID: k_window_frame_value<T><<<g, kThreads, 0, s>>>(r, f, xc, nx, which, nth, vwords, vprefix, (T*)out, vout); break;
        BDF_WIN_DTYPES(BDF_VALUE_CASE)
#undef BDF_VALUE_CASE
        default: return cudaErrorInvalidValue;
    }
    return cudaGetLastError();
}
#undef BDF_WIN_DTYPES

}  // namespace bdf
