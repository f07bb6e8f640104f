// k_cond.cu -- null handling and conditional selection (include/b200df.h "null handling and conditional selection"):
//   coalesce / case_when   k_cond_select<T>   every row copies the bits of the first argument that supplies it
//   greatest / least       k_cond_extreme<T>  the sort's order (SortKey<T>), nulls skipped, the earliest of equal values
//   nanvl                  k_cond_nanvl<T>    a unless it is NaN, then b
//   Boolean values         k_cond_bool        the same selection done entirely in 32-row words
//   is_null / is_not_null  k_null_bits        a shifted (inverted) copy of the validity words
//   is_nan                 k_is_nan<T>
//
// The value kernels work one 32-row word at a time: every lane of a warp derives the same per-argument masks from the validity
// and condition bitmaps of the word (funnel-shifted by the chunk's bit offsets), lane l owns row l of the word and loads only
// from the argument that supplies that row.  A warp whose mask for argument k is empty issues no load of k's values, and a
// word is finished once no row is pending, so coalesce(a, b) reads b only around the nulls of a and a case_when reads each
// branch's values only where that branch is taken.  The output validity word is the OR of the taken masks, each ANDed with the
// validity of the argument that supplied the rows; its popcount is the warp's valid count (no second pass for null counts).
#include <type_traits>

#include "common.cuh"
#include "sort_keys.cuh"

namespace bdf {

enum : int { ROW_COALESCE = 0, ROW_GREATEST, ROW_LEAST, ROW_NANVL };
enum : int { NT_IS_NULL = 0, NT_IS_NOT_NULL, NT_IS_NAN };

constexpr int kCondWords = 8;                               // 32-row words per warp and tile
constexpr int kCondTile = kWarpsPerCta * kCondWords * 32;   // rows per tile of the value kernels
constexpr int kCondBoolTile = kThreads * kUnroll * 32;      // rows per tile of the word kernels (one word per lane and step)
constexpr int kBoolDtype = 10;

__device__ __forceinline__ const CondHead* cond_chunk(const char* __restrict__ descs, size_t stride, int n_chunks, int64_t tile) {
    int lo = 0, hi = n_chunks - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(&((const CondHead*)(descs + (size_t)mid * stride))->tile0) <= tile) lo = mid; else hi = mid - 1;
    }
    return (const CondHead*)(descs + (size_t)lo * stride);
}

// The rows of the word at e0 (mask `tail`) where argument a is valid.  A word no row asks about (tail == 0, e.g. a word past the
// chunk's end in the last tile) reads nothing: with a nonzero bit offset load_bits also reads the next bitmap word, which for such
// a word can lie past the end of the bitmap's allocation.
__device__ __forceinline__ uint32_t arg_valid(const CondArg& a, int64_t e0, uint32_t tail) {
    if (!tail || a.kind == COND_NULL) return 0u;
    if (a.kind == COND_SCALAR || !a.validity) return tail;
    return load_bits<32>(a.validity, (int64_t)a.bit_off + e0) & tail;
}
// The rows where condition c is valid and true (a NULL condition counts as false).
__device__ __forceinline__ uint32_t cond_true(const CondArg& c, int64_t e0, uint32_t tail) {
    if (!tail) return 0u;   // as arg_valid: nothing is read for a word no row asks about
    uint32_t v = load_bits<32>((const uint32_t*)c.values, (int64_t)c.val_bit_off + e0) & tail;
    if (c.validity) v &= load_bits<32>(c.validity, (int64_t)c.bit_off + e0);
    return v;
}
template <typename T>
__device__ __forceinline__ T arg_value(const CondArg& a, int64_t row) {
    if (a.kind == COND_COLUMN) return ((const T*)a.values)[row];
    // the low sizeof(T) bytes of the scalar's bits
    if constexpr (std::is_same<T, double>::value) return __longlong_as_double((long long)a.bits);
    else if constexpr (std::is_same<T, float>::value) return __uint_as_float((uint32_t)a.bits);
    else return (T)a.bits;
}

// Warp-level tail of every value kernel: store the values and the validity words of the warp's words, report its valid count.
template <typename T>
__device__ __forceinline__ void cond_store(const CondHead* h, int64_t base, const T (&val)[kCondWords], const uint32_t (&vw)[kCondWords],
                                           const uint32_t (&tail)[kCondWords], uint32_t* __restrict__ warp_counts) {
    const int lane = threadIdx.x & 31;
    T* __restrict__ out = (T*)h->out;
    uint32_t* __restrict__ vout = h->vout;
    unsigned int nvalid = 0;
#pragma unroll
    for (int w = 0; w < kCondWords; w++) {
        const int64_t e0 = base + w * 32;
        if ((tail[w] >> lane) & 1u) out[e0 + lane] = val[w];
        if (vout && lane == 0 && tail[w]) vout[e0 >> 5] = vw[w];
        nvalid += __popc(vw[w]);
    }
    if (vout && lane == 0) warp_counts[(int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5)] = nvalid;
}

// coalesce (n_conds == 0): take_k = pending & valid_k.  case_when (n_conds == n_vals - 1): hit_k = pending & cvalid_k & cval_k,
// the else takes what is still pending, and a row is valid where the value that took it is.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_cond_select(const char* __restrict__ descs, size_t stride, int n_chunks, uint32_t* __restrict__ warp_counts) {
    const CondHead* h = cond_chunk(descs, stride, n_chunks, blockIdx.x);
    const CondArg* __restrict__ args = (const CondArg*)(h + 1);
    const int n_conds = h->n_conds, n_vals = h->n_vals;
    const int lane = threadIdx.x & 31;
    const int64_t base = ((int64_t)blockIdx.x - h->tile0) * kCondTile + (int64_t)(threadIdx.x >> 5) * (kCondWords * 32);
    uint32_t tail[kCondWords], pend[kCondWords], vw[kCondWords];
    T val[kCondWords];
#pragma unroll
    for (int w = 0; w < kCondWords; w++) {
        tail[w] = pend[w] = tail_mask<32>(base + w * 32, h->len);
        vw[w] = 0u;
        val[w] = T(0);
    }
    for (int k = 0; k < n_vals; k++) {
        uint32_t any = 0u;
#pragma unroll
        for (int w = 0; w < kCondWords; w++) any |= pend[w];
        if (!any) break;   // the same in every lane: the masks are words, not rows
        const CondArg a = args[n_conds + k];
        const bool branch = k < n_conds;
#pragma unroll
        for (int w = 0; w < kCondWords; w++) {
            const int64_t e0 = base + w * 32;
            const uint32_t p = pend[w];   // a finished word reads nothing more
            const uint32_t hit = !p ? 0u : branch ? cond_true(args[k], e0, p) : p & (n_conds ? ~0u : arg_valid(a, e0, p));
            const uint32_t sel = n_conds && hit ? hit & arg_valid(a, e0, hit) : hit;
            pend[w] &= ~hit;
            vw[w] |= sel;
            if ((sel >> lane) & 1u) val[w] = arg_value<T>(a, e0 + lane);
        }
    }
    cond_store<T>(h, base, val, vw, tail, warp_counts);
}

// greatest / least: every valid argument is read; a later argument replaces the best only when its key is strictly greater
// (smaller), so the earliest of equal values wins and the bits of the value that won are kept.
template <typename T, bool GREATEST>
__global__ void __launch_bounds__(kThreads)
k_cond_extreme(const char* __restrict__ descs, size_t stride, int n_chunks, uint32_t* __restrict__ warp_counts) {
    const CondHead* h = cond_chunk(descs, stride, n_chunks, blockIdx.x);
    const CondArg* __restrict__ args = (const CondArg*)(h + 1);
    const int n_vals = h->n_vals;
    const int lane = threadIdx.x & 31;
    const int64_t base = ((int64_t)blockIdx.x - h->tile0) * kCondTile + (int64_t)(threadIdx.x >> 5) * (kCondWords * 32);
    uint32_t tail[kCondWords], vw[kCondWords];
    unsigned long long best[kCondWords];
    T val[kCondWords];
#pragma unroll
    for (int w = 0; w < kCondWords; w++) {
        tail[w] = tail_mask<32>(base + w * 32, h->len);
        vw[w] = 0u;
        best[w] = 0ull;
        val[w] = T(0);
    }
    for (int k = 0; k < n_vals; k++) {
        const CondArg a = args[k];
#pragma unroll
        for (int w = 0; w < kCondWords; w++) {
            const int64_t e0 = base + w * 32;
            const uint32_t m = arg_valid(a, e0, tail[w]);
            if ((m >> lane) & 1u) {
                const T x = arg_value<T>(a, e0 + lane);
                const unsigned long long key = SortKey<T>::of(x);
                if (!((vw[w] >> lane) & 1u) || (GREATEST ? key > best[w] : key < best[w])) { best[w] = key; val[w] = x; }
            }
            vw[w] |= m;
        }
    }
    cond_store<T>(h, base, val, vw, tail, warp_counts);
}

// nanvl(a, b): a where a is valid and not NaN, b where a is NaN (NULL where b is), NULL where a is NULL.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_cond_nanvl(const char* __restrict__ descs, size_t stride, int n_chunks, uint32_t* __restrict__ warp_counts) {
    const CondHead* h = cond_chunk(descs, stride, n_chunks, blockIdx.x);
    const CondArg* __restrict__ args = (const CondArg*)(h + 1);
    const CondArg a = args[0], b = args[1];
    const int lane = threadIdx.x & 31;
    const int64_t base = ((int64_t)blockIdx.x - h->tile0) * kCondTile + (int64_t)(threadIdx.x >> 5) * (kCondWords * 32);
    uint32_t tail[kCondWords], vw[kCondWords];
    T val[kCondWords];
#pragma unroll
    for (int w = 0; w < kCondWords; w++) {
        const int64_t e0 = base + w * 32;
        tail[w] = tail_mask<32>(e0, h->len);
        const uint32_t va = arg_valid(a, e0, tail[w]);
        T x = T(0);
        if ((va >> lane) & 1u) x = arg_value<T>(a, e0 + lane);
        const uint32_t nan = __ballot_sync(0xffffffffu, x != x) & va;
        const uint32_t vb = nan ? arg_valid(b, e0, nan) : 0u;
        if ((vb >> lane) & 1u) x = arg_value<T>(b, e0 + lane);
        else if ((nan >> lane) & 1u) x = T(0);
        val[w] = x;
        vw[w] = (va & ~nan) | vb;
    }
    cond_store<T>(h, base, val, vw, tail, warp_counts);
}

// Boolean values: the selection is done on whole words, out = OR_k(sel_k & vals_k); one word per lane and step.
__global__ void __launch_bounds__(kThreads)
k_cond_bool(const char* __restrict__ descs, size_t stride, int n_chunks, uint32_t* __restrict__ warp_counts) {
    const CondHead* h = cond_chunk(descs, stride, n_chunks, blockIdx.x);
    const CondArg* __restrict__ args = (const CondArg*)(h + 1);
    const int n_conds = h->n_conds, n_vals = h->n_vals;
    const int64_t base = ((int64_t)blockIdx.x - h->tile0) * kCondBoolTile;
    uint32_t* __restrict__ out = (uint32_t*)h->out;
    uint32_t* __restrict__ vout = h->vout;
    unsigned int nvalid = 0;
    for (int j = 0; j < kUnroll; j++) {
        const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * 32;
        const uint32_t tail = tail_mask<32>(e0, h->len);
        if (!tail) continue;
        uint32_t pend = tail, vw = 0u, ov = 0u;
        for (int k = 0; k < n_vals && pend; k++) {
            const CondArg& a = args[n_conds + k];
            const uint32_t hit = k < n_conds ? cond_true(args[k], e0, pend) : pend & (n_conds ? ~0u : arg_valid(a, e0, pend));
            const uint32_t sel = n_conds ? hit & arg_valid(a, e0, hit) : hit;
            if (sel) {
                const uint32_t vals = a.kind == COND_COLUMN ? load_bits<32>((const uint32_t*)a.values, (int64_t)a.val_bit_off + e0)
                                                            : (a.bits ? ~0u : 0u);
                ov |= sel & vals;
            }
            vw |= sel;
            pend &= ~hit;
        }
        out[e0 >> 5] = ov;
        if (vout) vout[e0 >> 5] = vw;
        nvalid += __popc(vw);
    }
    if (vout) {
        const unsigned int wvalid = __reduce_add_sync(0xffffffffu, nvalid);
        if ((threadIdx.x & 31) == 0) warp_counts[(int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5)] = wvalid;
    }
}

// is_null / is_not_null: the validity words shifted to bit 0 (inverted for is_null), the tail masked.  ZERO: all false (is_nan
// of a column that cannot hold a NaN).  The result has no bitmap.
enum : int { NB_IS_NULL = 0, NB_IS_NOT_NULL, NB_ZERO };
template <int MODE>
__global__ void __launch_bounds__(kThreads)
k_null_bits(const char* __restrict__ descs, size_t stride, int n_chunks) {
    const CondHead* h = cond_chunk(descs, stride, n_chunks, blockIdx.x);
    const CondArg a = *(const CondArg*)(h + 1);
    const int64_t base = ((int64_t)blockIdx.x - h->tile0) * kCondBoolTile;
    uint32_t* __restrict__ out = (uint32_t*)h->out;
#pragma unroll
    for (int j = 0; j < kUnroll; j++) {
        const int64_t e0 = base + (int64_t)(j * kThreads + threadIdx.x) * 32;
        const uint32_t tail = tail_mask<32>(e0, h->len);
        if (!tail) continue;
        uint32_t r = 0u;
        if (MODE != NB_ZERO) {
            const uint32_t v = arg_valid(a, e0, tail);
            r = MODE == NB_IS_NULL ? (~v & tail) : v;
        }
        out[e0 >> 5] = r;
    }
}

// is_nan: a valid slot holding a NaN; a NULL slot is false.
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_is_nan(const char* __restrict__ descs, size_t stride, int n_chunks) {
    const CondHead* h = cond_chunk(descs, stride, n_chunks, blockIdx.x);
    const CondArg a = *(const CondArg*)(h + 1);
    const int lane = threadIdx.x & 31;
    const int64_t base = ((int64_t)blockIdx.x - h->tile0) * kCondTile + (int64_t)(threadIdx.x >> 5) * (kCondWords * 32);
    uint32_t* __restrict__ out = (uint32_t*)h->out;
    uint32_t valid[kCondWords];
    T x[kCondWords];
#pragma unroll
    for (int w = 0; w < kCondWords; w++) {
        const int64_t e0 = base + w * 32;
        valid[w] = arg_valid(a, e0, tail_mask<32>(e0, h->len));
        x[w] = T(0);
        if ((valid[w] >> lane) & 1u) x[w] = ((const T*)a.values)[e0 + lane];
    }
#pragma unroll
    for (int w = 0; w < kCondWords; w++) {
        const int64_t e0 = base + w * 32;
        const uint32_t nan = __ballot_sync(0xffffffffu, x[w] != x[w]) & valid[w];
        if (lane == 0 && e0 < h->len) out[e0 >> 5] = nan;
    }
}

int cond_tile_elems(int dtype) { return dtype == kBoolDtype ? kCondBoolTile : kCondTile; }
int null_test_tile_elems(int dtype, int test) { return test == NT_IS_NAN && dtype_is_float(dtype) ? kCondTile : kCondBoolTile; }

template <typename T>
static void cond_value_kernel(int fn, dim3 grid, const char* d, size_t stride, int n, uint32_t* wc, cudaStream_t s) {
    if (fn == ROW_GREATEST) {
        k_cond_extreme<T, true><<<grid, kThreads, 0, s>>>(d, stride, n, wc);
    } else if (fn == ROW_LEAST) {
        k_cond_extreme<T, false><<<grid, kThreads, 0, s>>>(d, stride, n, wc);
    } else if (fn == ROW_NANVL) {
        if constexpr (IsFloat<T>::value) k_cond_nanvl<T><<<grid, kThreads, 0, s>>>(d, stride, n, wc);
    } else if constexpr (!IsFloat<T>::value && !std::is_signed<T>::value) {
        k_cond_select<T><<<grid, kThreads, 0, s>>>(d, stride, n, wc);   // a pure selection: only the width matters
    }
}

cudaError_t launch_cond(int fn, int dtype, const void* descs, int n_args, int n_chunks, int64_t tiles, uint32_t* warp_counts, cudaStream_t s) {
    if (tiles <= 0) return cudaSuccess;
    const dim3 grid((unsigned)tiles);
    const char* d = (const char*)descs;
    const size_t stride = cond_desc_bytes(n_args);
    if (dtype == kBoolDtype) {
        k_cond_bool<<<grid, kThreads, 0, s>>>(d, stride, n_chunks, warp_counts);
        return cudaGetLastError();
    }
    // coalesce only needs the width; greatest / least / nanvl need the type
    const int t = fn == ROW_COALESCE ? (dtype_width(dtype) == 1 ? T_U8 : dtype_width(dtype) == 2 ? T_U16 : dtype_width(dtype) == 4 ? T_U32 : T_U64) : dtype;
    switch (t) {
        case T_I8: cond_value_kernel<int8_t>(fn, grid, d, stride, n_chunks, warp_counts, s); break;
        case T_I16: cond_value_kernel<int16_t>(fn, grid, d, stride, n_chunks, warp_counts, s); break;
        case T_I32: cond_value_kernel<int32_t>(fn, grid, d, stride, n_chunks, warp_counts, s); break;
        case T_I64: cond_value_kernel<int64_t>(fn, grid, d, stride, n_chunks, warp_counts, s); break;
        case T_U8: cond_value_kernel<uint8_t>(fn, grid, d, stride, n_chunks, warp_counts, s); break;
        case T_U16: cond_value_kernel<uint16_t>(fn, grid, d, stride, n_chunks, warp_counts, s); break;
        case T_U32: cond_value_kernel<uint32_t>(fn, grid, d, stride, n_chunks, warp_counts, s); break;
        case T_U64: cond_value_kernel<uint64_t>(fn, grid, d, stride, n_chunks, warp_counts, s); break;
        case T_F32: cond_value_kernel<float>(fn, grid, d, stride, n_chunks, warp_counts, s); break;
        default: cond_value_kernel<double>(fn, grid, d, stride, n_chunks, warp_counts, s); break;
    }
    return cudaGetLastError();
}

cudaError_t launch_null_test(int test, int dtype, const void* descs, int n_chunks, int64_t tiles, cudaStream_t s) {
    if (tiles <= 0) return cudaSuccess;
    const dim3 grid((unsigned)tiles);
    const char* d = (const char*)descs;
    const size_t stride = cond_desc_bytes(1);
    if (test == NT_IS_NAN && dtype == T_F32) k_is_nan<float><<<grid, kThreads, 0, s>>>(d, stride, n_chunks);
    else if (test == NT_IS_NAN && dtype == T_F64) k_is_nan<double><<<grid, kThreads, 0, s>>>(d, stride, n_chunks);
    else if (test == NT_IS_NAN) k_null_bits<NB_ZERO><<<grid, kThreads, 0, s>>>(d, stride, n_chunks);
    else if (test == NT_IS_NULL) k_null_bits<NB_IS_NULL><<<grid, kThreads, 0, s>>>(d, stride, n_chunks);
    else k_null_bits<NB_IS_NOT_NULL><<<grid, kThreads, 0, s>>>(d, stride, n_chunks);
    return cudaGetLastError();
}

}  // namespace bdf
