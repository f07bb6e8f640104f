// sort_keys.cuh -- the total order of DataFrame::sort over one criterion, shared by the radix lexsort (k_sort.cu) and the
// equi-join's search of the sorted build keys (k_join.cu).  The join finds its partners by binary search in the order the sort
// produced, so both must map a value to exactly the same key: a difference anywhere would silently lose matches.
#pragma once

#include "common.cuh"

namespace bdf {

template <typename To, typename From> __device__ __forceinline__ To bit_cast_to(From f) {
    static_assert(sizeof(To) == sizeof(From), "bit_cast_to: sizes differ");
    To t;
    memcpy(&t, &f, sizeof(To));
    return t;
}

struct SortChunk {          // one chunk of a column in the concatenated row space
    const void* values;
    const uint32_t* validity;
    int64_t start;          // first global row of the chunk
    int32_t bit_off;        // residual bit offset of the validity bitmap
    int32_t val_bit_off;    // boolean columns: residual bit offset of the values bitmap
};

__device__ __forceinline__ int chunk_of(const SortChunk* __restrict__ t, int n, int64_t row) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {   // last chunk whose start <= row (empty chunks share their start with the next one)
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(&t[mid].start) <= row) lo = mid; else hi = mid - 1;
    }
    return lo;
}
__device__ __forceinline__ bool chunk_bit(const uint32_t* __restrict__ bits, int64_t bit) {
    return (__ldg(bits + (bit >> 5)) >> (bit & 31)) & 1u;
}

// ---- order-preserving keys --------------------------------------------------------------------------------------
// Ascending key order = the sort's order of valid values: sign flip for integers; for floats every NaN is one value, greater
// than every number, and -0.0 == 0.0.
template <typename T> struct SortKey;
template <> struct SortKey<int8_t>   { static __device__ __forceinline__ unsigned long long of(int8_t x)   { return (uint8_t)x ^ 0x80u; } };
template <> struct SortKey<int16_t>  { static __device__ __forceinline__ unsigned long long of(int16_t x)  { return (uint16_t)x ^ 0x8000u; } };
template <> struct SortKey<int32_t>  { static __device__ __forceinline__ unsigned long long of(int32_t x)  { return (uint32_t)x ^ 0x80000000u; } };
template <> struct SortKey<int64_t>  { static __device__ __forceinline__ unsigned long long of(int64_t x)  { return (unsigned long long)x ^ (1ull << 63); } };
template <> struct SortKey<uint8_t>  { static __device__ __forceinline__ unsigned long long of(uint8_t x)  { return x; } };
template <> struct SortKey<uint16_t> { static __device__ __forceinline__ unsigned long long of(uint16_t x) { return x; } };
template <> struct SortKey<uint32_t> { static __device__ __forceinline__ unsigned long long of(uint32_t x) { return x; } };
template <> struct SortKey<uint64_t> { static __device__ __forceinline__ unsigned long long of(uint64_t x) { return x; } };
template <> struct SortKey<float> {
    static __device__ __forceinline__ unsigned long long of(float x) {
        if (x != x) return 0xffffffffull;            // every NaN is the same, greatest key
        if (x == 0.0f) x = 0.0f;                     // -0.0 == 0.0
        const uint32_t b = __float_as_uint(x);
        return (b >> 31) ? (uint32_t)~b : (b | 0x80000000u);
    }
};
template <> struct SortKey<double> {
    static __device__ __forceinline__ unsigned long long of(double x) {
        if (x != x) return ~0ull;
        if (x == 0.0) x = 0.0;
        const unsigned long long b = (unsigned long long)__double_as_longlong(x);
        return (b >> 63) ? ~b : (b | (1ull << 63));
    }
};

// The key of element i of a values buffer whose dtype is only known at run time (the criteria of one call may differ in type).
__device__ __forceinline__ unsigned long long sort_key_at(int dtype, const void* values, int64_t i) {
    switch (dtype) {
        case T_I8: return SortKey<int8_t>::of(((const int8_t*)values)[i]);
        case T_I16: return SortKey<int16_t>::of(((const int16_t*)values)[i]);
        case T_I32: return SortKey<int32_t>::of(((const int32_t*)values)[i]);
        case T_I64: return SortKey<int64_t>::of(((const int64_t*)values)[i]);
        case T_U8: return SortKey<uint8_t>::of(((const uint8_t*)values)[i]);
        case T_U16: return SortKey<uint16_t>::of(((const uint16_t*)values)[i]);
        case T_U32: return SortKey<uint32_t>::of(((const uint32_t*)values)[i]);
        case T_U64: return SortKey<uint64_t>::of(((const uint64_t*)values)[i]);
        case T_F32: return SortKey<float>::of(((const float*)values)[i]);
        default: return SortKey<double>::of(((const double*)values)[i]);
    }
}

}  // namespace bdf
