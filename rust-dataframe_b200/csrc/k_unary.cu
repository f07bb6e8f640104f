// k_unary.cu -- K2: y[i] = f(x[i]) over all chunks of a column in ONE launch, validity passed through
// (re-aligned to bit offset 0) and counted.
//
// Replaces the reference's own scalar_op loop (src/functions/scalar.rs:525-540) behind
// ScalarFunctions::{abs,sin,cos,tan,acos,asin,atan,cbrt,ceil,cosh,degrees,exp,expm1,floor,log10,log2,
// radians,round,sinh,sqrt,tanh} (scalar.rs:106-457): null -> null with payload 0, else num::Float::f(x)
// (= platform libm on the CPU).  CUDA's double/float math functions are used at full precision (no
// fast-math); documented error <= 2 ulp (f64 sin/cos/tan), <= 2/2/4 ulp (f32 sinf/cosf/tanf), so results
// are compared with glibc under the ulp tolerance stated in tests/test_parity_gpu.py.  log2 (f64) and log10 (f32) go
// through math_exact.cuh, which returns the exact k at 2^k / 10^k where CUDA's result is 1 ulp off.
//
// Roofline: HBM, 2*sizeof(T) + 2*[nullable]/8 bytes/row (16 B/row for f64); f64 trig is close to the FP64
// pipe limit (see DESIGN.md).
#include "common.cuh"
#include "math_exact.cuh"

namespace bdf {

enum : int {
    UN_ABS = 0, UN_SIN, UN_COS, UN_TAN, UN_ACOS, UN_ASIN, UN_ATAN, UN_CBRT, UN_CEIL, UN_COSH, UN_DEGREES, UN_EXP,
    UN_EXPM1, UN_FLOOR, UN_LOG10, UN_LOG2, UN_RADIANS, UN_ROUND, UN_SINH, UN_SQRT, UN_TANH, UN_N
};

template <int OP>
__device__ __forceinline__ double un_apply(double x) {
    if constexpr (OP == UN_ABS) return fabs(x);
    else if constexpr (OP == UN_SIN) return sin(x);
    else if constexpr (OP == UN_COS) return cos(x);
    else if constexpr (OP == UN_TAN) return tan(x);
    else if constexpr (OP == UN_ACOS) return acos(x);
    else if constexpr (OP == UN_ASIN) return asin(x);
    else if constexpr (OP == UN_ATAN) return atan(x);
    else if constexpr (OP == UN_CBRT) return cbrt(x);
    else if constexpr (OP == UN_CEIL) return ceil(x);
    else if constexpr (OP == UN_COSH) return cosh(x);
    else if constexpr (OP == UN_DEGREES) return __dmul_rn(x, 180.0 / 3.14159265358979323846264338327950288);
    else if constexpr (OP == UN_EXP) return exp(x);
    else if constexpr (OP == UN_EXPM1) return expm1(x);
    else if constexpr (OP == UN_FLOOR) return floor(x);
    else if constexpr (OP == UN_LOG10) return log10(x);
    else if constexpr (OP == UN_LOG2) return log2_exact(x);
    else if constexpr (OP == UN_RADIANS) return __dmul_rn(x, 3.14159265358979323846264338327950288 / 180.0);
    else if constexpr (OP == UN_ROUND) return round(x);
    else if constexpr (OP == UN_SINH) return sinh(x);
    else if constexpr (OP == UN_SQRT) return __dsqrt_rn(x);
    else return tanh(x);
}

template <int OP>
__device__ __forceinline__ float un_apply(float x) {
    if constexpr (OP == UN_ABS) return fabsf(x);
    else if constexpr (OP == UN_SIN) return sinf(x);
    else if constexpr (OP == UN_COS) return cosf(x);
    else if constexpr (OP == UN_TAN) return tanf(x);
    else if constexpr (OP == UN_ACOS) return acosf(x);
    else if constexpr (OP == UN_ASIN) return asinf(x);
    else if constexpr (OP == UN_ATAN) return atanf(x);
    else if constexpr (OP == UN_CBRT) return cbrtf(x);
    else if constexpr (OP == UN_CEIL) return ceilf(x);
    else if constexpr (OP == UN_COSH) return coshf(x);
    else if constexpr (OP == UN_DEGREES) return __fmul_rn(x, 57.2957795130823208767981548141051703f);
    else if constexpr (OP == UN_EXP) return expf(x);
    else if constexpr (OP == UN_EXPM1) return expm1f(x);
    else if constexpr (OP == UN_FLOOR) return floorf(x);
    else if constexpr (OP == UN_LOG10) return log10_exact(x);
    else if constexpr (OP == UN_LOG2) return log2f(x);
    else if constexpr (OP == UN_RADIANS) return __fmul_rn(x, 3.14159265358979323846264338327950288f / 180.0f);
    else if constexpr (OP == UN_ROUND) return roundf(x);
    else if constexpr (OP == UN_SINH) return sinhf(x);
    else if constexpr (OP == UN_SQRT) return __fsqrt_rn(x);
    else return tanhf(x);
}

// abs on signed integers: num::abs, wraps at iN::MIN (release build).
template <int OP> __device__ __forceinline__ int8_t un_apply(int8_t x) { return (int8_t)(x < 0 ? (uint8_t)(0u - (uint8_t)x) : x); }
template <int OP> __device__ __forceinline__ int16_t un_apply(int16_t x) { return (int16_t)(x < 0 ? (uint16_t)(0u - (uint16_t)x) : x); }
template <int OP> __device__ __forceinline__ int32_t un_apply(int32_t x) { return (int32_t)(x < 0 ? 0u - (uint32_t)x : (uint32_t)x); }
template <int OP> __device__ __forceinline__ int64_t un_apply(int64_t x) { return (int64_t)(x < 0 ? 0ull - (uint64_t)x : (uint64_t)x); }

// Vectors kept in flight per thread.  The libm-class functions are long dependent instruction sequences, so the
// unroll trades occupancy against per-thread ILP; it was measured rather than guessed (see UnaryUnroll).
__host__ __device__ constexpr bool unary_is_heavy(int op) {
    return !(op == UN_ABS || op == UN_CEIL || op == UN_FLOOR || op == UN_ROUND || op == UN_SQRT || op == UN_DEGREES || op == UN_RADIANS);
}
template <int OP> struct UnaryUnroll { static constexpr int value = kUnroll; };  // f64 sin: U=2 slower than 4, U=8 no better and tan slower: keep 4

template <typename T, int OP, int U>
__global__ void __launch_bounds__(kThreads)
k_unary(const UnDesc* __restrict__ descs, int n_chunks, uint32_t* __restrict__ warp_counts) {
    constexpr int E = 16 / (int)sizeof(T);
    constexpr int TILE = kThreads * U * E;
    constexpr uint32_t FULLMASK = (1u << E) - 1u;

    const int64_t tile = blockIdx.x;
    const int c = (n_chunks == 1) ? 0 : find_chunk(descs, n_chunks, tile);
    const T* __restrict__ pi = (const T*)descs[c].in;
    T* __restrict__ po = (T*)descs[c].out;
    const uint32_t* __restrict__ vi = descs[c].vin;
    uint32_t* __restrict__ vo = descs[c].vout;
    const int64_t len = descs[c].len;
    const int64_t off = descs[c].off;
    const int64_t base = (tile - descs[c].tile0) * TILE;

    unsigned int nvalid = 0;
    if (base + TILE <= len) {
        Vec<T, E> x[U];
#pragma unroll
        for (int j = 0; j < U; j++) x[j].load(pi + base + (int64_t)(j * kThreads + threadIdx.x) * E);
        MaskRaw<E, U> rv;  // validity words of all steps in one batch (see common.cuh)
        if (vi) mask_issue<E, U>(rv, vi, off + base + (int64_t)threadIdx.x * E, (int64_t)kThreads * E);
        uint32_t m[U];
#pragma unroll
        for (int j = 0; j < U; j++) m[j] = vi ? mask_get<E, U>(rv, j) : FULLMASK;
#pragma unroll
        for (int j = 0; j < U; j++) {
            const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
            Vec<T, E> r;
#pragma unroll
            for (int e = 0; e < E; e++) {
                const T y = un_apply<OP>(x[j].e[e]);  // computed for every lane (no divergence), selected afterwards
                r.e[e] = ((m[j] >> e) & 1u) ? y : (T)0;
            }
            r.store(po + e0);
            if (vo) {
                store_bits<E>(vo, e0, m[j], true);
                nvalid += __popc(m[j]);
            }
        }
    } else {
#pragma unroll 1
        for (int j = 0; j < U; j++) {
            const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * E;
            const uint32_t in_range = tail_mask<E>(e0, len);
            uint32_t m = in_range;
            if (in_range && vi) m &= load_bits<E>(vi, off + e0);
#pragma unroll
            for (int e = 0; e < E; e++)
                if ((in_range >> e) & 1u) po[e0 + e] = ((m >> e) & 1u) ? un_apply<OP>(pi[e0 + e]) : (T)0;
            if (vo) {
                store_bits<E>(vo, e0, m, in_range != 0);
                nvalid += __popc(m);
            }
        }
    }
    if (vo) {
        const unsigned int wvalid = __reduce_add_sync(0xffffffffu, nvalid);  // per-warp count, plain store (no atomics)
        if ((threadIdx.x & 31) == 0) warp_counts[(int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5)] = wvalid;
    }
}

template <typename T, int OP>
static cudaError_t launch_one(const UnDesc* d, int n, int64_t tiles, uint32_t* vc, cudaStream_t s) {
    k_unary<T, OP, UnaryUnroll<OP>::value><<<(unsigned)tiles, kThreads, 0, s>>>(d, n, vc);
    return cudaGetLastError();
}

template <typename T>
static cudaError_t launch_float(int op, const UnDesc* d, int n, int64_t tiles, uint32_t* vc, cudaStream_t s) {
    switch (op) {
#define BDF_CASE(OP) case OP: return launch_one<T, OP>(d, n, tiles, vc, s);
        BDF_CASE(UN_ABS) BDF_CASE(UN_SIN) BDF_CASE(UN_COS) BDF_CASE(UN_TAN) BDF_CASE(UN_ACOS) BDF_CASE(UN_ASIN)
        BDF_CASE(UN_ATAN) BDF_CASE(UN_CBRT) BDF_CASE(UN_CEIL) BDF_CASE(UN_COSH) BDF_CASE(UN_DEGREES) BDF_CASE(UN_EXP)
        BDF_CASE(UN_EXPM1) BDF_CASE(UN_FLOOR) BDF_CASE(UN_LOG10) BDF_CASE(UN_LOG2) BDF_CASE(UN_RADIANS)
        BDF_CASE(UN_ROUND) BDF_CASE(UN_SINH) BDF_CASE(UN_SQRT) BDF_CASE(UN_TANH)
#undef BDF_CASE
        default: return cudaErrorInvalidValue;
    }
}

int elems_per_tile_unary(int op, int dtype) { return kTileBytes / dtype_width(dtype); }

cudaError_t launch_unary(int op, int dtype, const UnDesc* d, int n, int64_t tiles, uint32_t* vc, cudaStream_t s) {
    if (tiles <= 0) return cudaSuccess;
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    if (dtype == T_F64) return launch_float<double>(op, d, n, tiles, vc, s);
    if (dtype == T_F32) return launch_float<float>(op, d, n, tiles, vc, s);
    if (op != UN_ABS) return cudaErrorInvalidValue;
    switch (dtype) {
        case T_I8: return launch_one<int8_t, UN_ABS>(d, n, tiles, vc, s);
        case T_I16: return launch_one<int16_t, UN_ABS>(d, n, tiles, vc, s);
        case T_I32: return launch_one<int32_t, UN_ABS>(d, n, tiles, vc, s);
        case T_I64: return launch_one<int64_t, UN_ABS>(d, n, tiles, vc, s);
        default: return cudaErrorInvalidValue;
    }
}

}  // namespace bdf
