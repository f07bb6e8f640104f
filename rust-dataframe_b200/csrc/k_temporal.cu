// k_temporal.cu -- calendar arithmetic on Date32 / Date64 / Timestamp / Time32 / Time64 columns (include/b200df.h "dates and
// timestamps"): ScalarFunctions::hour (src/functions/scalar.rs:267-273 -> arrow compute::hour) and the Spark date functions that are
// stubs in the reference.  One launch over all chunks, the descriptor walk, 16-byte loads and validity handling of k_cast.cu.
//
// A value is split by FLOOR division into (days, time of day) -- the divisor is a compile-time constant of the storage unit, so the
// split is a multiply-high, not a 64-bit division.  Civil fields come from days by Hinnant's civil_from_days / days_from_civil
// ("chrono-Compatible Low-Level Date Algorithms", PAPERS.md) in 32-bit arithmetic once the day is known to lie in chrono's range.
// The function is a uniform runtime switch (one kernel per (storage, unit, output width), 14 in all, instead of one per function as
// well): no kernel spills, at 40-48 registers.  The functions that go through the civil date are bound by integer issue, not by HBM
// (DESIGN.md §7 has the measurement and the SASS figures).
//
// Roofline: HBM, sizeof(In) + sizeof(Out) + 2/8 bytes/row (Timestamp -> Int32 field: 12 B/row plus validity); the two-column form
// sizeof(A) + sizeof(B) + sizeof(Out) (MONTHS_BETWEEN of two timestamps: 24 B/row).
#include "civil.cuh"
#include "common.cuh"

namespace bdf {

enum : int {
    TF_YEAR = 0, TF_QUARTER, TF_MONTH, TF_DAY_OF_MONTH, TF_DAY_OF_YEAR, TF_DAY_OF_WEEK, TF_HOUR, TF_MINUTE, TF_SECOND, TF_TO_DATE,
    TF_DATE_ADD, TF_DATE_SUB, TF_ADD_MONTHS, TF_LAST_DAY, TF_NEXT_DAY, TF_DATE_TRUNC, TF_UNIX_TIMESTAMP, TF_TO_TIMESTAMP
};
enum : int { TR_YEAR = 0, TR_QUARTER, TR_MONTH, TR_WEEK, TR_DAY, TR_HOUR, TR_MINUTE, TR_SECOND };
enum : int { TB_DATE_DIFF = 0, TB_MONTHS_BETWEEN };

template <int CFG> struct TUnit;
template <> struct TUnit<TC_DAYS> { static constexpr int64_t per_day = 1, per_sec = 1; };
template <> struct TUnit<TC_S> { static constexpr int64_t per_day = 86400LL, per_sec = 1; };
template <> struct TUnit<TC_MS> { static constexpr int64_t per_day = 86400000LL, per_sec = 1000LL; };
template <> struct TUnit<TC_US> { static constexpr int64_t per_day = 86400000000LL, per_sec = 1000000LL; };
template <> struct TUnit<TC_NS> { static constexpr int64_t per_day = 86400000000000LL, per_sec = 1000000000LL; };

__device__ __forceinline__ int32_t days_from_civil(int32_t y, uint32_t m, uint32_t d) {
    y -= m <= 2 ? 1 : 0;
    const int32_t era = (y >= 0 ? y : y - 399) / 400;
    const uint32_t yoe = (uint32_t)(y - era * 400);
    const uint32_t doy = (153 * (m > 2 ? m - 3 : m + 9) + 2) / 5 + d - 1;
    const uint32_t doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + (int32_t)doe - 719468;
}
__device__ __forceinline__ uint32_t days_in_month(int32_t y, uint32_t m) {
    if (m == 2) return (y % 4 == 0 && (y % 100 != 0 || y % 400 == 0)) ? 29u : 28u;
    return (m == 4 || m == 6 || m == 9 || m == 11) ? 30u : 31u;
}
__device__ __forceinline__ int32_t floor_mod7(int32_t x) { const int32_t r = x % 7; return r < 0 ? r + 7 : r; }
__device__ __forceinline__ int64_t floor_div_rt(int64_t v, int64_t q) { const int64_t a = v / q; return (v - a * q < 0) ? a - 1 : a; }
__device__ __forceinline__ bool day_ok(int64_t d) { return d >= kMinDay && d <= kMaxDay; }

// (days, time of day) of v by floor division, then the fixed tz offset (|off| < one day, in the same units) applied.
template <int CFG>
__device__ __forceinline__ void split_local(int64_t v, int64_t off, int64_t& days, int64_t& tod) {
    constexpr int64_t UPD = TUnit<CFG>::per_day;
    if constexpr (UPD == 1) { days = v; tod = 0; }
    else {
        days = v / UPD;
        tod = v - days * UPD;
        if (tod < 0) { tod += UPD; days -= 1; }
        tod += off;
        if (tod >= UPD) { tod -= UPD; days += 1; }
        else if (tod < 0) { tod += UPD; days -= 1; }
    }
}

template <int CFG>
__device__ __forceinline__ int32_t time_field(int fn, int64_t tod) {
    if constexpr (TUnit<CFG>::per_day == 1) return 0;   // Date32: midnight
    else {
        constexpr int64_t UPS = TUnit<CFG>::per_sec;
        if (fn == TF_HOUR) return (int32_t)(tod / (3600 * UPS));
        if (fn == TF_MINUTE) return (int32_t)((tod / (60 * UPS)) % 60);
        return (int32_t)((tod / UPS) % 60);
    }
}

// One slot: false = NULL.
template <typename In, typename Out, int CFG>
__device__ __forceinline__ bool temporal_one(In x, const TemporalParams& p, Out& out) {
    constexpr int64_t UPD = TUnit<CFG>::per_day;
    constexpr int64_t UPS = TUnit<CFG>::per_sec;
    const int64_t v = (int64_t)x;
    const int fn = p.fn;
    if (p.time_kind) {   // Time32 / Time64: HOUR / MINUTE / SECOND of a time of day
        if (v < 0 || v >= UPD) return false;
        out = (Out)time_field<CFG>(fn, v);
        return true;
    }
    if (fn == TF_UNIX_TIMESTAMP || fn == TF_TO_TIMESTAMP) {   // instants: the UTC date is range-checked, tz plays no part
        int64_t days, tod;
        split_local<CFG>(v, 0, days, tod);
        if (!day_ok(days)) return false;
        if (fn == TF_UNIX_TIMESTAMP) {
            out = (Out)(days * 86400 + tod / UPS);   // = floor(v / units per second), tod >= 0
            return true;
        }
        if (p.div > 1) { out = (Out)floor_div_rt(v, p.div); return true; }
        const __int128 r = (__int128)v * p.mul;
        if (r > (__int128)INT64_MAX || r < (__int128)INT64_MIN) return false;
        out = (Out)(int64_t)r;
        return true;
    }
    int64_t days, tod;
    split_local<CFG>(v, p.off, days, tod);
    if (!day_ok(days)) return false;
    const int32_t d = (int32_t)days;
    switch (fn) {
        case TF_HOUR: case TF_MINUTE: case TF_SECOND: out = (Out)time_field<CFG>(fn, tod); return true;
        case TF_TO_DATE: out = (Out)d; return true;
        case TF_DAY_OF_WEEK: out = (Out)(floor_mod7(d + 4) + 1); return true;   // 1970-01-01 was a Thursday (5)
        case TF_DATE_ADD: case TF_DATE_SUB: {
            const int64_t r = fn == TF_DATE_ADD ? (int64_t)d + p.arg : (int64_t)d - p.arg;
            if (!day_ok(r)) return false;
            out = (Out)r;
            return true;
        }
        case TF_NEXT_DAY: {
            int32_t delta = floor_mod7((int32_t)p.aux - (floor_mod7(d + 4) + 1));
            if (delta == 0) delta = 7;
            const int64_t r = (int64_t)d + delta;
            if (!day_ok(r)) return false;
            out = (Out)r;
            return true;
        }
        default: break;
    }
    int32_t y;
    uint32_t m, dd;
    civil_from_days(d, y, m, dd);
    switch (fn) {
        case TF_YEAR: out = (Out)y; return true;
        case TF_QUARTER: out = (Out)((m - 1) / 3 + 1); return true;
        case TF_MONTH: out = (Out)m; return true;
        case TF_DAY_OF_MONTH: out = (Out)dd; return true;
        case TF_DAY_OF_YEAR: out = (Out)(d - days_from_civil(y, 1, 1) + 1); return true;
        case TF_LAST_DAY: out = (Out)days_from_civil(y, m, days_in_month(y, m)); return true;
        case TF_ADD_MONTHS: {
            const int64_t total = (int64_t)y * 12 + (int64_t)(m - 1) + p.arg;
            const int64_t ny = total >= 0 ? total / 12 : -((-total + 11) / 12);
            if (ny < -262144 || ny > 262143) return false;
            const uint32_t nm = (uint32_t)(total - ny * 12) + 1;
            const uint32_t last = days_in_month((int32_t)ny, nm);
            const uint32_t nd = (dd == days_in_month(y, m) || dd > last) ? last : dd;   // Spark 2.4
            out = (Out)days_from_civil((int32_t)ny, nm, nd);
            return true;
        }
        case TF_DATE_TRUNC: {
            int32_t nd = d;
            int64_t ntod = tod;
            switch (p.aux) {
                case TR_YEAR: nd = days_from_civil(y, 1, 1); ntod = 0; break;
                case TR_QUARTER: nd = days_from_civil(y, (m - 1) / 3 * 3 + 1, 1); ntod = 0; break;
                case TR_MONTH: nd = days_from_civil(y, m, 1); ntod = 0; break;
                case TR_WEEK: nd = d - floor_mod7(d + 3); ntod = 0; break;   // Monday
                case TR_DAY: ntod = 0; break;
                case TR_HOUR: ntod = tod - tod % (3600 * UPS); break;
                case TR_MINUTE: ntod = tod - tod % (60 * UPS); break;
                default: ntod = tod - tod % UPS; break;
            }
            if (nd < kMinDay) return false;
            if constexpr (UPD == 1) { out = (Out)nd; return true; }
            const __int128 r = (__int128)nd * UPD + ntod - p.off;
            if (r > (__int128)INT64_MAX || r < (__int128)INT64_MIN) return false;
            out = (Out)(int64_t)r;
            return true;
        }
        default: return false;
    }
}

// Steps per thread of a full tile.  Four 4-element steps (Date32 -> Int32) inline sixteen copies of the switch and made ptxas spill;
// two steps keep every kernel spill-free at the same 8 elements per thread as the 8-byte kernels.
__host__ __device__ constexpr int temporal_unroll(int e) { return e >= 4 ? 2 : kUnroll; }

template <typename In, typename Out, int CFG>
__global__ void __launch_bounds__(kThreads)
k_temporal(const UnDesc* __restrict__ descs, int n_chunks, uint32_t* __restrict__ warp_counts, const TemporalParams p) {
    constexpr int W = sizeof(In) > sizeof(Out) ? (int)sizeof(In) : (int)sizeof(Out);
    constexpr int E = 16 / W;
    constexpr int U = temporal_unroll(E);
    constexpr int TILE = kThreads * U * E;
    constexpr uint32_t FULLMASK = (1u << E) - 1u;

    const int64_t tile = blockIdx.x;
    const int c = (n_chunks == 1) ? 0 : find_chunk(descs, n_chunks, tile);
    const In* __restrict__ pi = (const In*)descs[c].in;
    Out* __restrict__ po = (Out*)descs[c].out;
    const uint32_t* __restrict__ vi = descs[c].vin;
    uint32_t* __restrict__ vo = descs[c].vout;
    const int64_t len = descs[c].len;
    const int64_t off = descs[c].off;
    const int64_t base = (tile - descs[c].tile0) * TILE;

    unsigned int nvalid = 0;
    if (base + TILE <= len) {
        Vec<In, E> x[U];
#pragma unroll
        for (int j = 0; j < U; j++) x[j].load(pi + base + (int64_t)(j * kThreads + threadIdx.x) * E);
        MaskRaw<E, U> rv;
        if (vi) mask_issue<E, U>(rv, vi, off + base + (int64_t)threadIdx.x * E, (int64_t)kThreads * E);
        uint32_t m[U];
#pragma unroll
        for (int j = 0; j < U; j++) m[j] = vi ? mask_get<E, U>(rv, j) : FULLMASK;
#pragma unroll
        for (int j = 0; j < U; j++) {
            const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
            Vec<Out, E> r;
            uint32_t ok = 0;
#pragma unroll
            for (int e = 0; e < E; e++) {
                Out y = 0;
                const bool good = ((m[j] >> e) & 1u) && temporal_one<In, Out, CFG>(x[j].e[e], p, y);
                r.e[e] = good ? y : (Out)0;
                ok |= (good ? 1u : 0u) << e;
            }
            r.store(po + e0);
            store_bits<E>(vo, e0, ok, true);
            nvalid += __popc(ok);
        }
    } else {
#pragma unroll 1
        for (int j = 0; j < U; j++) {
            const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
            const uint32_t in_range = tail_mask<E>(e0, len);
            uint32_t m = in_range;
            if (in_range && vi) m &= load_bits<E>(vi, off + e0);
            uint32_t ok = 0;
#pragma unroll
            for (int e = 0; e < E; e++) {
                if ((in_range >> e) & 1u) {
                    Out y = 0;
                    const bool good = ((m >> e) & 1u) && temporal_one<In, Out, CFG>(pi[e0 + e], p, y);
                    po[e0 + e] = good ? y : (Out)0;
                    ok |= (good ? 1u : 0u) << e;
                }
            }
            store_bits<E>(vo, e0, ok, in_range != 0);
            nvalid += __popc(ok);
        }
    }
    const unsigned int wvalid = __reduce_add_sync(0xffffffffu, nvalid);   // per-warp count, plain store (no atomics)
    if ((threadIdx.x & 31) == 0) warp_counts[(int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)] = wvalid;
}

// ---- two columns: DATE_DIFF and MONTHS_BETWEEN ------------------------------------------------------------------------------
// Each side is split with its own unit (a uniform switch over the five storage units, each a constant division) into the local day
// and the whole seconds of the local time of day.
__device__ __forceinline__ bool side_split(int64_t v, int cfg, int64_t off, int32_t& day, int32_t& sec) {
    int64_t days = 0, tod = 0, ups = 1;
    switch (cfg) {
        case TC_DAYS: split_local<TC_DAYS>(v, 0, days, tod); break;
        case TC_S: split_local<TC_S>(v, off, days, tod); ups = TUnit<TC_S>::per_sec; break;
        case TC_MS: split_local<TC_MS>(v, off, days, tod); ups = TUnit<TC_MS>::per_sec; break;
        case TC_US: split_local<TC_US>(v, off, days, tod); ups = TUnit<TC_US>::per_sec; break;
        default: split_local<TC_NS>(v, off, days, tod); ups = TUnit<TC_NS>::per_sec; break;
    }
    if (!day_ok(days)) return false;
    day = (int32_t)days;
    sec = (int32_t)(tod / ups);
    return true;
}

template <typename Out>
__device__ __forceinline__ bool temporal_two(int64_t a, int64_t b, const TemporalParams2& p, Out& out) {
    int32_t da, sa, db, sb;
    if (!side_split(a, p.cfg_a, p.off_a, da, sa) || !side_split(b, p.cfg_b, p.off_b, db, sb)) return false;
    if (p.fn == TB_DATE_DIFF) { out = (Out)(da - db); return true; }
    int32_t y1, y2;
    uint32_t m1, d1, m2, d2;
    civil_from_days(da, y1, m1, d1);
    civil_from_days(db, y2, m2, d2);
    const double month_diff = (double)(((int64_t)y1 * 12 + m1) - ((int64_t)y2 * 12 + m2));
    if (d1 == d2 || (d1 == days_in_month(y1, m1) && d2 == days_in_month(y2, m2))) { out = (Out)month_diff; return true; }
    const double sec_diff = (double)(((int64_t)d1 - (int64_t)d2) * 86400 + ((int64_t)sa - (int64_t)sb));
    const double diff = __dadd_rn(month_diff, __ddiv_rn(sec_diff, 2678400.0));
    const double t = __dmul_rn(diff, 1e8);
    double k = floor(t);
    if (__dsub_rn(t, k) >= 0.5) k = __dadd_rn(k, 1.0);
    out = (Out)__ddiv_rn(k, 1e8);
    return true;
}

template <typename A, typename B, typename Out>
__global__ void __launch_bounds__(kThreads)
k_temporal2(const BinDesc* __restrict__ descs, int n_chunks, uint32_t* __restrict__ warp_counts, const TemporalParams2 p) {
    constexpr int WA = (int)sizeof(A) > (int)sizeof(B) ? (int)sizeof(A) : (int)sizeof(B);
    constexpr int W = WA > (int)sizeof(Out) ? WA : (int)sizeof(Out);
    constexpr int E = 16 / W;
    constexpr int TILE = kThreads * kUnroll * E;

    const int64_t tile = blockIdx.x;
    const int c = (n_chunks == 1) ? 0 : find_chunk(descs, n_chunks, tile);
    const A* __restrict__ pa = (const A*)descs[c].a;
    const B* __restrict__ pb = (const B*)descs[c].b;
    Out* __restrict__ po = (Out*)descs[c].out;
    const uint32_t* __restrict__ va = descs[c].va;
    const uint32_t* __restrict__ vb = descs[c].vb;
    uint32_t* __restrict__ vo = descs[c].vout;
    const int64_t len = descs[c].len;
    const int64_t base = (tile - descs[c].tile0) * TILE;
    const bool full = base + TILE <= len;

    unsigned int nvalid = 0;
#pragma unroll
    for (int j = 0; j < kUnroll; j++) {
        const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
        const uint32_t in_range = full ? ((1u << E) - 1u) : tail_mask<E>(e0, len);
        uint32_t m = in_range;
        if (in_range && va) m &= load_bits<E>(va, descs[c].offa + e0);
        if (in_range && vb) m &= load_bits<E>(vb, descs[c].offb + e0);
        uint32_t ok = 0;
        if (full) {
            Vec<A, E> xa;
            Vec<B, E> xb;
            Vec<Out, E> r;
            xa.load(pa + e0);
            xb.load(pb + e0);
#pragma unroll
            for (int e = 0; e < E; e++) {
                Out y = 0;
                const bool good = ((m >> e) & 1u) && temporal_two<Out>((int64_t)xa.e[e], (int64_t)xb.e[e], p, y);
                r.e[e] = good ? y : (Out)0;
                ok |= (good ? 1u : 0u) << e;
            }
            r.store(po + e0);
        } else {
            for (int e = 0; e < E; e++) {
                if ((in_range >> e) & 1u) {
                    Out y = 0;
                    const bool good = ((m >> e) & 1u) && temporal_two<Out>((int64_t)pa[e0 + e], (int64_t)pb[e0 + e], p, y);
                    po[e0 + e] = good ? y : (Out)0;
                    ok |= (good ? 1u : 0u) << e;
                }
            }
        }
        store_bits<E>(vo, e0, ok, in_range != 0);
        nvalid += __popc(ok);
    }
    const unsigned int wvalid = __reduce_add_sync(0xffffffffu, nvalid);
    if ((threadIdx.x & 31) == 0) warp_counts[(int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)] = wvalid;
}

// ---- launchers ----------------------------------------------------------------------------------------------------------------
int elems_per_tile_temporal(int in_dtype, int out_dtype) {
    const int w = dtype_width(in_dtype) > dtype_width(out_dtype) ? dtype_width(in_dtype) : dtype_width(out_dtype);
    return kThreads * temporal_unroll(16 / w) * (16 / w);
}
int elems_per_tile_temporal2(int a_dtype, int b_dtype, int out_dtype) {
    int w = dtype_width(a_dtype) > dtype_width(b_dtype) ? dtype_width(a_dtype) : dtype_width(b_dtype);
    w = w > dtype_width(out_dtype) ? w : dtype_width(out_dtype);
    return kTileBytes / w;
}

template <typename In, typename Out, int CFG>
static cudaError_t launch_t(const UnDesc* d, int n, int64_t tiles, uint32_t* vc, const TemporalParams& p, cudaStream_t s) {
    k_temporal<In, Out, CFG><<<(unsigned)tiles, kThreads, 0, s>>>(d, n, vc, p);
    return cudaGetLastError();
}

template <typename In, typename Out>
static cudaError_t launch_cfg(int cfg, const UnDesc* d, int n, int64_t tiles, uint32_t* vc, const TemporalParams& p, cudaStream_t s) {
    if constexpr (sizeof(In) == 4) {   // Date32 (days), Time32 (s / ms)
        switch (cfg) {
            case TC_DAYS: return launch_t<In, Out, TC_DAYS>(d, n, tiles, vc, p, s);
            case TC_S: return launch_t<In, Out, TC_S>(d, n, tiles, vc, p, s);
            case TC_MS: return launch_t<In, Out, TC_MS>(d, n, tiles, vc, p, s);
            default: return cudaErrorInvalidValue;
        }
    } else {
        switch (cfg) {
            case TC_S: return launch_t<In, Out, TC_S>(d, n, tiles, vc, p, s);
            case TC_MS: return launch_t<In, Out, TC_MS>(d, n, tiles, vc, p, s);
            case TC_US: return launch_t<In, Out, TC_US>(d, n, tiles, vc, p, s);
            case TC_NS: return launch_t<In, Out, TC_NS>(d, n, tiles, vc, p, s);
            default: return cudaErrorInvalidValue;
        }
    }
}

cudaError_t launch_temporal(int cfg, int in_dtype, int out_dtype, const TemporalParams& p, const UnDesc* d, int n, int64_t tiles, uint32_t* vc,
                            cudaStream_t s) {
    if (tiles <= 0) return cudaSuccess;
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    const bool in32 = in_dtype == T_I32, out32 = out_dtype == T_I32;
    if (in32) return out32 ? launch_cfg<int32_t, int32_t>(cfg, d, n, tiles, vc, p, s) : launch_cfg<int32_t, int64_t>(cfg, d, n, tiles, vc, p, s);
    return out32 ? launch_cfg<int64_t, int32_t>(cfg, d, n, tiles, vc, p, s) : launch_cfg<int64_t, int64_t>(cfg, d, n, tiles, vc, p, s);
}

template <typename A, typename B>
static cudaError_t launch_t2(int out_dtype, const BinDesc* d, int n, int64_t tiles, uint32_t* vc, const TemporalParams2& p, cudaStream_t s) {
    if (out_dtype == T_I32) k_temporal2<A, B, int32_t><<<(unsigned)tiles, kThreads, 0, s>>>(d, n, vc, p);
    else k_temporal2<A, B, double><<<(unsigned)tiles, kThreads, 0, s>>>(d, n, vc, p);
    return cudaGetLastError();
}

cudaError_t launch_temporal2(int a_dtype, int b_dtype, int out_dtype, const TemporalParams2& p, const BinDesc* d, int n, int64_t tiles,
                             uint32_t* vc, cudaStream_t s) {
    if (tiles <= 0) return cudaSuccess;
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    const bool a32 = a_dtype == T_I32, b32 = b_dtype == T_I32;
    if (a32) return b32 ? launch_t2<int32_t, int32_t>(out_dtype, d, n, tiles, vc, p, s) : launch_t2<int32_t, int64_t>(out_dtype, d, n, tiles, vc, p, s);
    return b32 ? launch_t2<int64_t, int32_t>(out_dtype, d, n, tiles, vc, p, s) : launch_t2<int64_t, int64_t>(out_dtype, d, n, tiles, vc, p, s);
}

}  // namespace bdf
