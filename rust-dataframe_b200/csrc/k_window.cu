// k_window.cu -- window functions over PARTITION BY / ORDER BY (WindowFunctions, src/functions/window.rs:1-11, and WindowSpec,
// src/window.rs:8-22: stubs in the reference).
//
// The host (runtime.cu window_dev) sorts the rows by (partition keys ascending, order keys with their directions) with the stable
// radix lexsort, gathers the keys, marks the first row of every partition (P heads) and of every peer group (Q heads, a superset
// of P) with k_group_heads, and compacts the head positions with filter(iota, heads).  The kernels work in that sorted space,
// positions i = 0..n-1:
//   k_window_count   popcount of every head word and the total of every CTA, for the 64-bit scan of k_join.cu: afterwards
//                    prefix[w] is the number of runs starting before position 32w, so the run of position i -- and through the
//                    compacted starts its first and last position -- costs O(1) (no binary search per row).
//   k_window_rank    per position: partition and peer bounds -> row_number, rank, dense_rank, percent_rank, cume_dist, written
//                    to out[perm[i]] (the caller's row order), and the gather indices that bring a sorted-order column back to
//                    row order: i itself (the inverse permutation), the last peer of i, the last row of i's partition.
//   k_window_shift   lag / lead: x at position i -/+ k when that lies inside i's partition, else the default or NULL.
//   k_window_scan    segmented inclusive scan with the group fold's accumulators (group_acc.cuh): reduce-then-scan over a FIXED
//                    tile decomposition -- (1) every tile folds its rows into (a partition starts here, aggregate since the last
//                    start), (2) k_window_carry, one CTA, scans those tile records into every tile's carry-in, (3) every tile
//                    rescans its rows from its carry.  The order in which values are combined depends only on n, so float sums
//                    are the same bits on every run; a decoupled look-back would combine predecessors in a timing-dependent order.
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

// counts[w] = popcount(words[w]); block_sums[b] = the total of CTA b (kJoinTile words: 256 threads x 8) -- the input of launch_join_scan.
__global__ void __launch_bounds__(kThreads)
k_window_count(const uint32_t* __restrict__ words, long long n_words, unsigned long long* __restrict__ counts, unsigned long long* __restrict__ block_sums) {
    __shared__ unsigned long long s_warp[kWarpsPerCta];
    const long long base = (long long)blockIdx.x * kWinTile + (long long)threadIdx.x * kWinItems;
    unsigned long long sum = 0;
#pragma unroll
    for (int k = 0; k < kWinItems; k++)
        if (base + k < n_words) { const unsigned long long c = __popc(words[base + k]); counts[base + k] = c; sum += c; }
    sum = __reduce_add_sync(0xffffffffu, (unsigned)sum);
    if ((threadIdx.x & 31) == 0) s_warp[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
#pragma unroll
        for (int w = 0; w < kWarpsPerCta; w++) t += s_warp[w];
        block_sums[blockIdx.x] = t;
    }
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
// The three head arrays of one head bitmap (words, prefix from launch_join_scan, compacted starts) and the number of runs.
static WinRuns make_runs(const void* const* p, long long n_p, const void* const* q, long long n_q, long long n) {
    WinRuns r{};
    if (p) r.p = WinHeads{(const uint32_t*)p[0], (const unsigned long long*)p[1], (const uint32_t*)p[2], n_p};
    if (q) r.q = WinHeads{(const uint32_t*)q[0], (const unsigned long long*)q[1], (const uint32_t*)q[2], n_q};
    r.n = n;
    return r;
}

int window_count_tile() { return kWinTile; }

cudaError_t launch_window_count(const uint32_t* words, long long n_words, unsigned long long* counts, unsigned long long* block_sums, cudaStream_t s) {
    if (n_words <= 0) return cudaSuccess;
    k_window_count<<<(unsigned)((n_words + kWinTile - 1) / kWinTile), kThreads, 0, s>>>(words, n_words, counts, block_sums);
    return cudaGetLastError();
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

}  // namespace bdf
