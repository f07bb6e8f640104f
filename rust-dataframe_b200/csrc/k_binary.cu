// k_binary.cu -- K1: c[i] = a[i] (op) b[i] over all chunks of a column pair in ONE launch, with the
// validity AND, the output null count and the divide-by-zero flag fused in.
//
// Replaces arrow::compute::{add,subtract,multiply,divide} as called per chunk by
// ScalarFunctions::{add,subtract,multiply,par_multiply,divide} (reference src/functions/scalar.rs:16-103)
// and the math_op binaries atan2/hypot/log (scalar.rs:148,274,291,499-523).
//
// Semantics kept (oracle/oracle.c states them with provenance):
//   * add/sub/mul compute every slot, also under nulls; integers wrap; IEEE ops round once (the
//     __*_rn intrinsics can never be contracted into FMAs);
//   * divide: a VALID slot with a zero divisor (ints and floats) raises the DivideByZero flag; null
//     slots divide by 1; iN::MIN / -1 wraps;
//   * math_op binaries: null slot -> payload 0;
//   * validity = a AND b at bit offset 0, zero padding bits; valid slots are counted per warp (plain stores).
//
// Roofline: HBM.  Algorithmic bytes/row = 3*sizeof(T) + (v_in + [v_in>0])/8  (24 B/row for f64, no nulls).
#include "common.cuh"
#include "math_exact.cuh"

namespace bdf {

enum : int { OP_ADD = 0, OP_SUB, OP_MUL, OP_DIV, OP_ATAN2, OP_HYPOT, OP_LOG };



template <size_t N> struct WideOf { using type = uint32_t; };
template <> struct WideOf<8> { using type = uint64_t; };



// apply(a, b, valid, divzero): valid = output slot is valid; divzero is OR-ed when a valid divisor is 0.
template <typename T, int OP>
__device__ __forceinline__ T bin_apply(T a, T b, bool valid, bool& divzero) {
    if constexpr (IsFloat<T>::value) {
        if constexpr (sizeof(T) == 8) {
            if constexpr (OP == OP_ADD) return __dadd_rn(a, b);
            else if constexpr (OP == OP_SUB) return __dsub_rn(a, b);
            else if constexpr (OP == OP_MUL) return __dmul_rn(a, b);
            else if constexpr (OP == OP_DIV) {
                divzero |= valid && (b == 0.0);
                return __ddiv_rn(a, valid ? b : 1.0);
            } else if constexpr (OP == OP_ATAN2) return valid ? atan2(a, b) : 0.0;
            else if constexpr (OP == OP_HYPOT) return valid ? hypot_exact(a, b) : 0.0;
            else return valid ? __ddiv_rn(log(a), log(b)) : 0.0;
        } else {
            if constexpr (OP == OP_ADD) return __fadd_rn(a, b);
            else if constexpr (OP == OP_SUB) return __fsub_rn(a, b);
            else if constexpr (OP == OP_MUL) return __fmul_rn(a, b);
            else if constexpr (OP == OP_DIV) {
                divzero |= valid && (b == 0.0f);
                return __fdiv_rn(a, valid ? b : 1.0f);
            } else if constexpr (OP == OP_ATAN2) return valid ? atan2f(a, b) : 0.0f;
            else if constexpr (OP == OP_HYPOT) return valid ? hypotf(a, b) : 0.0f;
            else return valid ? __fdiv_rn(logf(a), logf(b)) : 0.0f;
        }
    } else {
        using U = typename UnsignedOf<T>::type;
        using W = typename WideOf<sizeof(T)>::type;  // >= 32 bit unsigned: no signed-int promotion overflow
        if constexpr (OP == OP_ADD) return (T)(U)((W)(U)a + (W)(U)b);
        else if constexpr (OP == OP_SUB) return (T)(U)((W)(U)a - (W)(U)b);
        else if constexpr (OP == OP_MUL) return (T)(U)((W)(U)a * (W)(U)b);
        else {
            divzero |= valid && (b == (T)0);
            const T d = valid ? b : (T)1;
            if constexpr (((T)-1) < (T)0) {
                if (d == (T)-1) return (T)(U)((U)0 - (U)a);  // also covers MIN / -1 (wraps)
            }
            return (T)(a / (d == (T)0 ? (T)1 : d));  // d == 0 only on the error path; result is discarded
        }
    }
}

// FusedAgg (the per-thread accumulator of K5) lives in common.cuh: k_expr folds the result of a fused chain the same way.

template <typename T, int OP, bool AGG, int U>
__global__ void __launch_bounds__(kThreads)
k_binary(const BinDesc* __restrict__ descs, int n_chunks, uint32_t* __restrict__ warp_counts,
         int* __restrict__ flags, AggDev* __restrict__ tile_partials, unsigned long long flip) {
    constexpr int E = 16 / (int)sizeof(T);
    constexpr int TILE = kThreads * U * E;
    constexpr uint32_t FULLMASK = (E == 32) ? 0xffffffffu : ((1u << E) - 1u);

    const int64_t tile = blockIdx.x;
    const int c = (n_chunks == 1) ? 0 : find_chunk(descs, n_chunks, tile);
    const T* __restrict__ pa = (const T*)descs[c].a;
    const T* __restrict__ pb = (const T*)descs[c].b;
    T* __restrict__ po = (T*)descs[c].out;
    const uint32_t* __restrict__ va = descs[c].va;
    const uint32_t* __restrict__ vb = descs[c].vb;
    uint32_t* __restrict__ vo = descs[c].vout;
    const int64_t len = descs[c].len;
    const int64_t offa = descs[c].offa, offb = descs[c].offb;
    const int64_t base = (tile - descs[c].tile0) * TILE;

    unsigned int nvalid = 0;
    bool divzero = false;
    FusedAgg<T> agg;
    if constexpr (AGG) agg.init();

    if (base + TILE <= len) {
        // ---- full tile: 2 x U 16-byte loads in flight per thread before first use ----
        Vec<T, E> a[U], b[U];
#pragma unroll
        for (int j = 0; j < U; j++) {
            const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
            a[j].load(pa + e0);
            b[j].load(pb + e0);
        }
        // validity words of all U steps: issued as two batches (one uniform branch each), consumed afterwards
        MaskRaw<E, U> ra, rb;
        const int64_t e_first = base + (int64_t)threadIdx.x * E;
        if (va) mask_issue<E, U>(ra, va, offa + e_first, (int64_t)kThreads * E);
        if (vb) mask_issue<E, U>(rb, vb, offb + e_first, (int64_t)kThreads * E);
        uint32_t m[U];
#pragma unroll
        for (int j = 0; j < U; j++) {
            m[j] = FULLMASK;
            if (va) m[j] &= mask_get<E, U>(ra, j);
            if (vb) m[j] &= mask_get<E, U>(rb, j);
        }
#pragma unroll
        for (int j = 0; j < U; j++) {
            const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
            Vec<T, E> r;
#pragma unroll
            for (int e = 0; e < E; e++) {
                r.e[e] = bin_apply<T, OP>(a[j].e[e], b[j].e[e], (m[j] >> e) & 1u, divzero);
                if constexpr (AGG) agg.add(r.e[e], (m[j] >> e) & 1u, flip);
            }
            r.store(po + e0);
            if (vo) store_bits<E>(vo, e0, m[j], true);
            if (vo || AGG) nvalid += __popc(m[j]);
        }
    } else {
        // ---- tail tile of the chunk: element-wise guards ----
#pragma unroll 1
        for (int j = 0; j < U; j++) {
            const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
            const uint32_t in_range = tail_mask<E>(e0, len);
            uint32_t m = in_range;
            if (in_range) {
                if (va) m &= load_bits<E>(va, offa + e0);
                if (vb) m &= load_bits<E>(vb, offb + e0);
            }
#pragma unroll
            for (int e = 0; e < E; e++) {
                if ((in_range >> e) & 1u) {
                    const T x = pa[e0 + e], y = pb[e0 + e];
                    const T z = bin_apply<T, OP>(x, y, (m >> e) & 1u, divzero);
                    po[e0 + e] = z;
                    if constexpr (AGG) agg.add(z, (m >> e) & 1u, flip);
                }
            }
            if (vo) store_bits<E>(vo, e0, m, in_range != 0);
            if (vo || AGG) nvalid += __popc(m);
        }
    }

    if (vo || AGG) {
        // valid slots of this warp -> one plain store per warp (no atomics, no block barrier); the host sums
        // the per-warp counts of a chunk when a null count is asked for
        const unsigned int wvalid = __reduce_add_sync(0xffffffffu, nvalid);
        if ((threadIdx.x & 31) == 0 && vo) warp_counts[(int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)] = wvalid;
        if constexpr (AGG) {
            __shared__ unsigned int s_cnt[kThreads / 32];
            if ((threadIdx.x & 31) == 0) s_cnt[threadIdx.x >> 5] = wvalid;
            // fixed xor-shuffle tree inside each warp, then warp 0 folds the 8 warp results in warp order
            __shared__ FusedAgg<T> s_agg[kThreads / 32];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) agg.merge_shfl(o);
            if ((threadIdx.x & 31) == 0) s_agg[threadIdx.x >> 5] = agg;
            __syncthreads();
            if (threadIdx.x == 0) {
                FusedAgg<T> t = s_agg[0];
#pragma unroll
                for (int w = 1; w < kThreads / 32; w++) t.merge(s_agg[w]);
                unsigned long long total = 0;
#pragma unroll
                for (int w = 0; w < kThreads / 32; w++) total += s_cnt[w];
                t.store(&tile_partials[blockIdx.x], total);
            }
        }
    }
    if constexpr (OP == OP_DIV) {
        if (divzero) atomicOr(flags, 1);
    }
}

// Folds per-tile partials into one result.  Grid and per-thread assignment are fixed => deterministic.
template <bool IS_FLOAT>
__global__ void __launch_bounds__(kThreads)
k_finish(const AggDev* __restrict__ parts, long long n_parts, AggDev* __restrict__ stage, unsigned int* __restrict__ ticket,
         AggDev* __restrict__ result) {
    __shared__ AggDev s_part[kThreads / 32];
    __shared__ bool s_last;
    auto ident = [] { AggDev a; a.sum_bits = 0; a.min_bits = ~0ull; a.max_bits = 0; a.count = 0; return a; };
    auto merge = [](AggDev& a, const AggDev& b) {
        if constexpr (IS_FLOAT)
            a.sum_bits = (unsigned long long)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)a.sum_bits), __longlong_as_double((long long)b.sum_bits)));
        else a.sum_bits += b.sum_bits;
        a.min_bits = b.min_bits < a.min_bits ? b.min_bits : a.min_bits;
        a.max_bits = b.max_bits > a.max_bits ? b.max_bits : a.max_bits;
        a.count += b.count;
    };
    auto shfl = [](const AggDev& a, int o) {
        AggDev r;
        r.sum_bits = __shfl_xor_sync(0xffffffffu, a.sum_bits, o); r.min_bits = __shfl_xor_sync(0xffffffffu, a.min_bits, o);
        r.max_bits = __shfl_xor_sync(0xffffffffu, a.max_bits, o); r.count = __shfl_xor_sync(0xffffffffu, a.count, o);
        return r;
    };
    auto block_fold = [&](AggDev v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { AggDev t = shfl(v, o); merge(v, t); }
        __syncthreads();
        if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = v;
        __syncthreads();
        AggDev r = s_part[0];
        for (int w = 1; w < kThreads / 32; w++) merge(r, s_part[w]);
        return r;  // identical in every thread
    };
    AggDev acc = ident();
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n_parts; i += (long long)gridDim.x * kThreads) {
        AggDev p;
        p.sum_bits = __ldcg(&parts[i].sum_bits); p.min_bits = __ldcg(&parts[i].min_bits);
        p.max_bits = __ldcg(&parts[i].max_bits); p.count = __ldcg(&parts[i].count);
        merge(acc, p);
    }
    acc = block_fold(acc);
    if (threadIdx.x == 0) {
        stage[blockIdx.x] = acc;
        __threadfence();
        s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    AggDev fin = ident();
    for (unsigned int i = threadIdx.x; i < gridDim.x; i += kThreads) {
        AggDev p;
        p.sum_bits = __ldcg(&stage[i].sum_bits); p.min_bits = __ldcg(&stage[i].min_bits);
        p.max_bits = __ldcg(&stage[i].max_bits); p.count = __ldcg(&stage[i].count);
        merge(fin, p);
    }
    fin = block_fold(fin);
    if (threadIdx.x == 0) { *result = fin; __threadfence_system(); *ticket = 0; }  // result: device-mapped host memory
}

cudaError_t launch_finish(bool is_float, const AggDev* parts, int64_t n_parts, int sm_count, AggDev* stage, unsigned int* ticket,
                          AggDev* result, cudaStream_t s) {
    int64_t grid = (n_parts + 4 * kThreads - 1) / (4 * kThreads);
    if (grid > sm_count) grid = sm_count;
    if (grid < 1) grid = 1;
    if (is_float) k_finish<true><<<(unsigned)grid, kThreads, 0, s>>>(parts, n_parts, stage, ticket, result);
    else k_finish<false><<<(unsigned)grid, kThreads, 0, s>>>(parts, n_parts, stage, ticket, result);
    return cudaGetLastError();
}

// The same fold for several partial ranges at once (blockIdx.y = range): multi-column aggregates pay one launch, not one per column.
struct FinishJobs { FinishJob j[kFinishMany]; };
__global__ void __launch_bounds__(kThreads)
k_finish_many(const FinishJobs jobs, AggDev* __restrict__ stage_all, unsigned int* __restrict__ tickets) {
    __shared__ AggDev s_part[kThreads / 32];
    __shared__ bool s_last;
    const FinishJob& job = jobs.j[blockIdx.y];
    const AggDev* __restrict__ parts = job.parts;
    const long long n_parts = job.n_parts;
    const bool is_float = job.is_float != 0;
    AggDev* __restrict__ stage = stage_all + (size_t)blockIdx.y * gridDim.x;
    unsigned int* __restrict__ ticket = tickets + blockIdx.y;
    auto ident = [] { AggDev a; a.sum_bits = 0; a.min_bits = ~0ull; a.max_bits = 0; a.count = 0; return a; };
    auto merge = [is_float](AggDev& a, const AggDev& b) {
        if (is_float)
            a.sum_bits = (unsigned long long)__double_as_longlong(__dadd_rn(__longlong_as_double((long long)a.sum_bits), __longlong_as_double((long long)b.sum_bits)));
        else a.sum_bits += b.sum_bits;
        a.min_bits = b.min_bits < a.min_bits ? b.min_bits : a.min_bits;
        a.max_bits = b.max_bits > a.max_bits ? b.max_bits : a.max_bits;
        a.count += b.count;
    };
    auto shfl = [](const AggDev& a, int o) {
        AggDev r;
        r.sum_bits = __shfl_xor_sync(0xffffffffu, a.sum_bits, o); r.min_bits = __shfl_xor_sync(0xffffffffu, a.min_bits, o);
        r.max_bits = __shfl_xor_sync(0xffffffffu, a.max_bits, o); r.count = __shfl_xor_sync(0xffffffffu, a.count, o);
        return r;
    };
    auto block_fold = [&](AggDev v) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { AggDev t = shfl(v, o); merge(v, t); }
        __syncthreads();
        if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = v;
        __syncthreads();
        AggDev r = s_part[0];
        for (int w = 1; w < kThreads / 32; w++) merge(r, s_part[w]);
        return r;
    };
    AggDev acc = ident();
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n_parts; i += (long long)gridDim.x * kThreads) {
        AggDev p;
        p.sum_bits = __ldcg(&parts[i].sum_bits); p.min_bits = __ldcg(&parts[i].min_bits);
        p.max_bits = __ldcg(&parts[i].max_bits); p.count = __ldcg(&parts[i].count);
        merge(acc, p);
    }
    acc = block_fold(acc);
    if (threadIdx.x == 0) {
        stage[blockIdx.x] = acc;
        __threadfence();
        s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    AggDev fin = ident();
    for (unsigned int i = threadIdx.x; i < gridDim.x; i += kThreads) {
        AggDev p;
        p.sum_bits = __ldcg(&stage[i].sum_bits); p.min_bits = __ldcg(&stage[i].min_bits);
        p.max_bits = __ldcg(&stage[i].max_bits); p.count = __ldcg(&stage[i].count);
        merge(fin, p);
    }
    fin = block_fold(fin);
    if (threadIdx.x == 0) { *job.result = fin; __threadfence_system(); *ticket = 0; }
}

cudaError_t launch_finish_many(int n, const FinishJob* jobs, int sm_count, AggDev* stage, unsigned int* tickets, cudaStream_t s) {
    if (n < 1 || n > kFinishMany) return cudaErrorInvalidValue;
    FinishJobs jj;
    long long most = 1;
    for (int i = 0; i < n; i++) { jj.j[i] = jobs[i]; most = jobs[i].n_parts > most ? jobs[i].n_parts : most; }
    int64_t gx = (most + 4 * kThreads - 1) / (4 * kThreads);
    const int64_t cap = sm_count / (n < 4 ? 1 : 4) > 1 ? sm_count / (n < 4 ? 1 : 4) : 1;   // n ranges share the SMs
    if (gx > cap) gx = cap;
    if (gx < 1) gx = 1;
    k_finish_many<<<dim3((unsigned)gx, (unsigned)n), kThreads, 0, s>>>(jj, stage, tickets);
    return cudaGetLastError();
}

int elems_per_tile(int dtype) { return kTileBytes / dtype_width(dtype); }

// Compute-heavy binaries (divide and the libm ones) keep fewer vectors in registers per thread: the extra
// occupancy hides the long dependent instruction sequences better than deeper per-thread batching.
template <int OP> struct UnrollOf { static constexpr int value = (OP > OP_DIV) ? 2 : kUnroll; };
int elems_per_tile_binary(int op, int dtype) { return (op > OP_DIV ? kThreads * 2 * 16 : kTileBytes) / dtype_width(dtype); }

struct AggArgs { AggDev* partials; unsigned long long flip; };

template <typename T, int OP>
static cudaError_t launch_one(const BinDesc* d, int n, int64_t tiles, uint32_t* vc, int* flags, cudaStream_t s, AggArgs ag) {
    if constexpr (OP <= OP_DIV) {
        if (ag.partials) {
            k_binary<T, OP, true, UnrollOf<OP>::value><<<(unsigned)tiles, kThreads, 0, s>>>(d, n, vc, flags, ag.partials, ag.flip);
            return cudaGetLastError();
        }
    }
    k_binary<T, OP, false, UnrollOf<OP>::value><<<(unsigned)tiles, kThreads, 0, s>>>(d, n, vc, flags, nullptr, 0ull);
    return cudaGetLastError();
}

template <typename T>
static cudaError_t launch_wrapping(int op, const BinDesc* d, int n, int64_t tiles, uint32_t* vc, int* flags,
                                   cudaStream_t s, AggArgs ag) {
    switch (op) {
        case OP_ADD: return launch_one<T, OP_ADD>(d, n, tiles, vc, flags, s, ag);
        case OP_SUB: return launch_one<T, OP_SUB>(d, n, tiles, vc, flags, s, ag);
        default: return launch_one<T, OP_MUL>(d, n, tiles, vc, flags, s, ag);
    }
}

template <typename T>
static cudaError_t launch_float(int op, const BinDesc* d, int n, int64_t tiles, uint32_t* vc, int* flags,
                                cudaStream_t s, AggArgs ag) {
    switch (op) {
        case OP_ADD: return launch_one<T, OP_ADD>(d, n, tiles, vc, flags, s, ag);
        case OP_SUB: return launch_one<T, OP_SUB>(d, n, tiles, vc, flags, s, ag);
        case OP_MUL: return launch_one<T, OP_MUL>(d, n, tiles, vc, flags, s, ag);
        case OP_DIV: return launch_one<T, OP_DIV>(d, n, tiles, vc, flags, s, ag);
        case OP_ATAN2: return launch_one<T, OP_ATAN2>(d, n, tiles, vc, flags, s, ag);
        case OP_HYPOT: return launch_one<T, OP_HYPOT>(d, n, tiles, vc, flags, s, ag);
        default: return launch_one<T, OP_LOG>(d, n, tiles, vc, flags, s, ag);
    }
}

cudaError_t launch_binary(int op, int dtype, const BinDesc* d, int n, int64_t tiles, uint32_t* vc, int* flags,
                          cudaStream_t s, AggDev* tile_partials) {
    const int bits = 8 * dtype_width(dtype);
    AggArgs ag{tile_partials, dtype_is_signed_int(dtype) ? (1ull << (bits - 1)) : 0ull};
    if (tiles <= 0) return cudaSuccess;
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    if (dtype == T_F64) return launch_float<double>(op, d, n, tiles, vc, flags, s, ag);
    if (dtype == T_F32) return launch_float<float>(op, d, n, tiles, vc, flags, s, ag);
    if (op > OP_DIV) return cudaErrorInvalidValue;
    if (op == OP_DIV) {
        switch (dtype) {
            case T_I8: return launch_one<int8_t, OP_DIV>(d, n, tiles, vc, flags, s, ag);
            case T_I16: return launch_one<int16_t, OP_DIV>(d, n, tiles, vc, flags, s, ag);
            case T_I32: return launch_one<int32_t, OP_DIV>(d, n, tiles, vc, flags, s, ag);
            case T_I64: return launch_one<int64_t, OP_DIV>(d, n, tiles, vc, flags, s, ag);
            case T_U8: return launch_one<uint8_t, OP_DIV>(d, n, tiles, vc, flags, s, ag);
            case T_U16: return launch_one<uint16_t, OP_DIV>(d, n, tiles, vc, flags, s, ag);
            case T_U32: return launch_one<uint32_t, OP_DIV>(d, n, tiles, vc, flags, s, ag);
            default: return launch_one<uint64_t, OP_DIV>(d, n, tiles, vc, flags, s, ag);
        }
    }
    // add/sub/mul wrap: identical bits for signed and unsigned -> one instantiation per width
    switch (dtype_width(dtype)) {
        case 1: return launch_wrapping<uint8_t>(op, d, n, tiles, vc, flags, s, ag);
        case 2: return launch_wrapping<uint16_t>(op, d, n, tiles, vc, flags, s, ag);
        case 4: return launch_wrapping<uint32_t>(op, d, n, tiles, vc, flags, s, ag);
        default: return launch_wrapping<uint64_t>(op, d, n, tiles, vc, flags, s, ag);
    }
}

}  // namespace bdf
