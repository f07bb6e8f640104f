// common.cuh -- device helpers shared by the sm_90a kernels of libb200df.
//
// Data layout in HBM (DESIGN.md "Layout"): every chunk of a device column is an Arrow PrimitiveArray
// whose values start 256-byte aligned (element offset already applied at upload) and whose validity
// bitmap (LSB-first, 1 = valid) is a 4-byte-aligned array of 32-bit words with a residual BIT offset
// `off` (0..7 for uploaded slices, 0 for kernel-made columns).  Bitmaps are padded so that one word past
// the last used one may be read.
//
// Work decomposition: a *tile* is THREADS x U vectors of 16 bytes per array (coalesced: lane l of a warp
// touches vector j*THREADS + l).  A thread therefore owns E = 16/sizeof(T) consecutive elements per step
// and E consecutive validity bits; 32/E neighbouring lanes share one bitmap word, which they assemble
// with a log2(32/E)-step shuffle-OR so the warp writes whole 32-bit words.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace bdf {

enum : int { T_I8 = 0, T_I16, T_I32, T_I64, T_U8, T_U16, T_U32, T_U64, T_F32, T_F64, T_NTYPES };

__host__ __device__ inline int dtype_width(int t) {
    switch (t) {
        case T_I8: case T_U8: return 1;
        case T_I16: case T_U16: return 2;
        case T_I32: case T_U32: case T_F32: return 4;
        default: return 8;
    }
}
__host__ __device__ inline bool dtype_is_float(int t) { return t == T_F32 || t == T_F64; }
__host__ __device__ inline bool dtype_is_signed_int(int t) { return t >= T_I8 && t <= T_I64; }

constexpr int kThreads = 256;  // CTA size of every streaming kernel
constexpr int kUnroll = 4;     // 16-byte vectors in flight per thread per array
constexpr int kTileBytes = kThreads * kUnroll * 16;  // bytes of the widest array per tile (16 KiB)
constexpr int kWarpsPerCta = kThreads / 32;          // kernels report valid-slot counts per warp: [tile][warp] u32

// ---- 128-bit streaming loads/stores -----------------------------------------------------------
// Inputs are read exactly once and outputs written exactly once: bypass L1 allocation so the small
// validity words (which ARE re-read by neighbouring lanes) keep the L1.
__device__ __forceinline__ uint4 ld_stream16(const void* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint2 ld_stream8(const void* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t ld_stream4(const void* p) {
    uint32_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ uint16_t ld_stream2(const void* p) {
    uint16_t r;
    asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(r) : "l"(p));
    return r;
}
__device__ __forceinline__ void st_stream16(void* p, uint4 v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ void st_stream8(void* p, uint2 v) {
    asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" :: "l"(p), "r"(v.x), "r"(v.y) : "memory");
}
__device__ __forceinline__ void st_stream4(void* p, uint32_t v) {
    asm volatile("st.global.L1::no_allocate.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_stream2(void* p, uint16_t v) {
    asm volatile("st.global.L1::no_allocate.u16 [%0], %1;" :: "l"(p), "h"(v) : "memory");
}

// A register-resident vector of N elements of T moved with one access of N*sizeof(T) bytes (2..16).
template <typename T, int N>
struct Vec {
    static constexpr int kBytes = N * (int)sizeof(T);
    static_assert(kBytes == 16 || kBytes == 8 || kBytes == 4 || kBytes == 2, "unsupported vector size");
    union {
        T e[N];
        uint4 q;
        uint2 d;
        uint32_t w;
        uint16_t h;
    };
    __device__ __forceinline__ void load(const void* p) {
        if constexpr (kBytes == 16) q = ld_stream16(p);
        else if constexpr (kBytes == 8) d = ld_stream8(p);
        else if constexpr (kBytes == 4) w = ld_stream4(p);
        else h = ld_stream2(p);
    }
    __device__ __forceinline__ void store(void* p) const {
        if constexpr (kBytes == 16) st_stream16(p, q);
        else if constexpr (kBytes == 8) st_stream8(p, d);
        else if constexpr (kBytes == 4) st_stream4(p, w);
        else st_stream2(p, h);
    }
};

// ---- validity bitmap access ----------------------------------------------------------------------
// E consecutive bits starting at absolute bit index `bit` of word array v.
template <int E>
__device__ __forceinline__ uint32_t load_bits(const uint32_t* __restrict__ v, int64_t bit) {
    const int64_t w = bit >> 5;
    const int sh = (int)(bit & 31);
    const uint32_t lo = __ldg(v + w);
    const uint32_t hi = (sh + E > 32) ? __ldg(v + w + 1) : 0u;
    const uint32_t r = __funnelshift_r(lo, hi, sh);
    if constexpr (E == 32) return r;
    else return r & ((1u << E) - 1u);
}

// Batched form used on full tiles: issue the raw word loads of all U steps back to back (no consumer in
// between, so all of them are in flight together with the value loads), extract the bits later.  Wrap the
// issue in ONE uniform `if (bitmap present)`; per-step conditionals would make the compiler serialise the
// loads (load -> wait -> shift, U times), which costs U memory latencies per tile.
template <int E, int U>
struct MaskRaw {
    uint32_t lo[U], hi[U];
    int sh[U];
};
template <int E, int U>
__device__ __forceinline__ void mask_issue(MaskRaw<E, U>& r, const uint32_t* __restrict__ v, int64_t bit0, int64_t stride_bits) {
    // Every caller steps by kThreads * E bits, a whole number of 32-bit words: the shift is the same for all U steps and
    // the word addresses are one base pointer plus constants (the 64-bit shift/LEA chain per step that the general form
    // costs is most of the instruction count of a nullable tile).
    const uint32_t* __restrict__ p = v + (bit0 >> 5);
    const int sh = (int)(bit0 & 31);
    const int stride_words = (int)(stride_bits >> 5);
    const bool two = sh + E > 32;
#pragma unroll
    for (int j = 0; j < U; j++) {
        r.sh[j] = sh;
        r.lo[j] = __ldg(p + j * stride_words);
        r.hi[j] = two ? __ldg(p + j * stride_words + 1) : 0u;
    }
}
// The general form (a word index per step).  k_filter.cu keeps it: with three bitmaps in flight the base-pointer form above
// costs it registers (the filter scatter got slower when it was switched over).
template <int E, int U>
__device__ __forceinline__ void mask_issue_general(MaskRaw<E, U>& r, const uint32_t* __restrict__ v, int64_t bit0, int64_t stride_bits) {
#pragma unroll
    for (int j = 0; j < U; j++) {
        const int64_t bit = bit0 + (int64_t)j * stride_bits;
        const int64_t w = bit >> 5;
        r.sh[j] = (int)(bit & 31);
        r.lo[j] = __ldg(v + w);
        r.hi[j] = (r.sh[j] + E > 32) ? __ldg(v + w + 1) : 0u;
    }
}
// The same with the word pointer and the shift already known (a loop over consecutive tiles advances the pointer by a constant).
template <int E, int U>
__device__ __forceinline__ void mask_issue_at(MaskRaw<E, U>& r, const uint32_t* __restrict__ p, int sh, int stride_words) {
    const bool two = sh + E > 32;
#pragma unroll
    for (int j = 0; j < U; j++) {
        r.sh[j] = sh;
        r.lo[j] = __ldg(p + j * stride_words);
        r.hi[j] = two ? __ldg(p + j * stride_words + 1) : 0u;
    }
}
template <int E, int U>
__device__ __forceinline__ uint32_t mask_get(const MaskRaw<E, U>& r, int j) {
    const uint32_t x = __funnelshift_r(r.lo[j], r.hi[j], r.sh[j]);
    if constexpr (E == 32) return x;
    else return x & ((1u << E) - 1u);
}

// Each lane contributes E bits for elements [e0, e0+E) (e0 a multiple of E, bit offset 0 on output); the
// 32/E lanes that share a word OR their pieces together and the first of them stores the word.
// Must be executed by all 32 lanes of the warp.  `active` = this lane's e0 lies inside the chunk.
template <int E>
__device__ __forceinline__ void store_bits(uint32_t* __restrict__ vout, int64_t e0, uint32_t bits, bool active) {
    constexpr int G = 32 / E;
    const int lane = threadIdx.x & 31;
    uint32_t c = bits << (E * (lane % G));
#pragma unroll
    for (int o = 1; o < G; o <<= 1) c |= __shfl_xor_sync(0xffffffffu, c, o);
    if ((lane % G) == 0 && active) vout[e0 >> 5] = c;
}

// Mask of the elements of [e0, e0+E) that lie below len.
template <int E>
__device__ __forceinline__ uint32_t tail_mask(int64_t e0, int64_t len) {
    const int64_t rem = len - e0;
    if (rem >= E) return (E == 32) ? 0xffffffffu : ((1u << E) - 1u);
    if (rem <= 0) return 0u;
    return (1u << (int)rem) - 1u;
}

// Chunk lookup: descriptors are sorted by tile0 (first tile of the chunk); returns the chunk owning `tile`.
template <typename Desc>
__device__ __forceinline__ int find_chunk(const Desc* __restrict__ descs, int n_chunks, int64_t tile) {
    int lo = 0, hi = n_chunks - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(&descs[mid].tile0) <= tile) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ---- descriptors (one per chunk, device-resident array sorted by tile0) ------------------------
struct BinDesc {
    const void* a; const void* b; void* out;
    const uint32_t* va; const uint32_t* vb; uint32_t* vout;
    int64_t len; int64_t tile0;
    int32_t offa, offb;
};
struct UnDesc {
    const void* in; void* out;
    const uint32_t* vin; uint32_t* vout;
    int64_t len; int64_t tile0;
    int32_t off; int32_t pad;
};
struct RedDesc {
    const void* in; const uint32_t* vin;
    int64_t len; int64_t tile0;
    int32_t off; int32_t pad;
};
struct GenDesc {
    void* out; uint32_t* vout;
    int64_t len; int64_t tile0; int64_t row0;
};
// CSV writer (k_csv_write.cu): one per (chunk, column), chunk-major.
struct CsvwDesc {
    const void* values; const uint32_t* validity;
    int32_t bit_off;       // validity bit offset
    int32_t val_bit_off;   // Boolean values bit offset
    int32_t dtype; int32_t pad;
};
// JSON writer (k_json_write.cu): one JsonwDesc per (chunk, column), chunk-major; one JsonwCol per column.
struct JsonwDesc {
    const void* values; const uint32_t* validity;   // a scalar column's, or a list column's elements'
    const int32_t* loffs;       // list: len + 1 offsets from 0; nullptr for a scalar column
    const uint32_t* lvalid;     // list: the list validity at bit 0, or nullptr
    long long estart;           // list: elements in the column's earlier chunks
    int32_t bit_off;            // validity bit offset
    int32_t val_bit_off;        // Boolean values bit offset
};
struct JsonwCol {
    long long upd, ups, off;    // temporal text (json_format.cuh): units per day, per second, tz offset in units
    int32_t tkind, frac, suffix_len;
    int32_t dtype;              // a list's element dtype
    int32_t name_at, name_len;  // the column's "name": in the names buffer
    int32_t list;               // its index among the list columns; -1 for a scalar column
    char suffix[8];
};
// The tables of one write.  plan is the current window's plan (k_json_write.cu): [0] its end row, [1] its elements,
// [2 + L] the first element of list L in it, [2 + n_lists + L] where list L's elements start in the window's element scan.
struct JsonwArgs {
    const JsonwDesc* desc; const JsonwCol* cols; const char* names; const long long* chunk_start;
    const int32_t* list_cols;   // the column of list L
    long long* plan;
    int n_cols, n_chunks, n_lists, explicit_nulls;
};

// Null handling and conditional selection (k_cond.cu): one header per chunk followed by its arguments, so the stride of the
// descriptor array is cond_desc_bytes(n_conds + n_vals).  Arguments [0, n_conds) are the Boolean conditions of a case_when,
// [n_conds, n_conds + n_vals) the values (for a case_when the last one is the else).
enum : int { COND_COLUMN = 0, COND_SCALAR, COND_NULL };
struct CondArg {
    const void* values;         // COND_COLUMN: the chunk's values (a bitmap for Boolean columns)
    const uint32_t* validity;   // nullptr: every slot valid
    unsigned long long bits;    // COND_SCALAR: T::Native bits (Boolean 0 / 1)
    int16_t bit_off;            // validity bit offset
    int16_t val_bit_off;        // Boolean values bit offset
    int32_t kind;               // COND_COLUMN, COND_SCALAR or COND_NULL (a NULL literal)
};
struct CondHead {
    void* out; uint32_t* vout;  // vout nullptr: the result chunk has no bitmap
    int64_t len; int64_t tile0;
    int32_t n_conds, n_vals;
    int64_t pad;
};
__host__ __device__ inline size_t cond_desc_bytes(int n_args) { return sizeof(CondHead) + (size_t)n_args * sizeof(CondArg); }

// Partial / final aggregate as the kernels produce it.
struct AggDev {
    unsigned long long sum_bits;  // ints: 64-bit wrapping sum; floats: double bit pattern
    unsigned long long min_bits;  // ints only: order-preserving unsigned key of the minimum (identity ~0)
    unsigned long long max_bits;  // ints only: order-preserving unsigned key of the maximum (identity 0)
    unsigned long long count;     // valid slots
};

template <typename T> struct UnsignedOf { using type = T; };
template <> struct UnsignedOf<int8_t> { using type = uint8_t; };
template <> struct UnsignedOf<int16_t> { using type = uint16_t; };
template <> struct UnsignedOf<int32_t> { using type = uint32_t; };
template <> struct UnsignedOf<int64_t> { using type = uint64_t; };
template <typename T> struct IsFloat { static constexpr bool value = false; };
template <> struct IsFloat<float> { static constexpr bool value = true; };
template <> struct IsFloat<double> { static constexpr bool value = true; };

// ---- K5: aggregate of the OUTPUT fused into the same pass (sum/min/max/count of c while c is written) ----
// Integers: wrapping 64-bit sum of the zero-extended values (only the low sizeof(T) bytes are meaningful),
// min/max over order-preserving unsigned keys (value ^ sign flip).  Floats: sum in double.  One partial per
// CTA (= per tile) in tile order; k_finish folds them in a fixed order => deterministic.
template <typename T, bool F = IsFloat<T>::value> struct FusedAgg;
template <typename T> struct FusedAgg<T, false> {
    unsigned long long sum, kmin, kmax;
    __device__ __forceinline__ void init() { sum = 0; kmin = ~0ull; kmax = 0; }
    __device__ __forceinline__ void add(T x, bool valid, unsigned long long flip) {
        using U = typename UnsignedOf<T>::type;
        const unsigned long long z = (unsigned long long)(U)x;
        if (valid) { sum += z; const unsigned long long k = z ^ flip; kmin = k < kmin ? k : kmin; kmax = k > kmax ? k : kmax; }
    }
    __device__ __forceinline__ void merge_shfl(int o) {
        const unsigned long long s2 = __shfl_xor_sync(0xffffffffu, sum, o), a2 = __shfl_xor_sync(0xffffffffu, kmin, o),
                                 b2 = __shfl_xor_sync(0xffffffffu, kmax, o);
        sum += s2; kmin = a2 < kmin ? a2 : kmin; kmax = b2 > kmax ? b2 : kmax;
    }
    __device__ __forceinline__ void merge(const FusedAgg& o) { sum += o.sum; kmin = o.kmin < kmin ? o.kmin : kmin; kmax = o.kmax > kmax ? o.kmax : kmax; }
    __device__ __forceinline__ void store(AggDev* d, unsigned long long cnt) const { d->sum_bits = sum; d->min_bits = kmin; d->max_bits = kmax; d->count = cnt; }
};
template <typename T> struct FusedAgg<T, true> {
    double sum;
    __device__ __forceinline__ void init() { sum = 0.0; }
    __device__ __forceinline__ void add(T x, bool valid, unsigned long long) { sum = __dadd_rn(sum, valid ? (double)x : 0.0); }
    __device__ __forceinline__ void merge_shfl(int o) { sum = __dadd_rn(sum, __shfl_xor_sync(0xffffffffu, sum, o)); }
    __device__ __forceinline__ void merge(const FusedAgg& o) { sum = __dadd_rn(sum, o.sum); }
    __device__ __forceinline__ void store(AggDev* d, unsigned long long cnt) const {
        d->sum_bits = (unsigned long long)__double_as_longlong(sum); d->min_bits = ~0ull; d->max_bits = 0; d->count = cnt;
    }
};

// ---- launchers (defined in k_*.cu) ---------------------------------------------------------------
int elems_per_tile(int dtype);                 // tile size in elements for arrays of dtype
int elems_per_tile_binary(int op, int dtype);
int elems_per_tile_unary(int op, int dtype);   // K2 tile size (libm-class functions use shorter tiles)  // K1 tile size (divide/libm binaries use shorter tiles)
int elems_per_tile_cast(int from, int to);
// tile_partials != nullptr (add/sub/mul/div only): also write one AggDev per tile with the aggregate of the
// OUTPUT (K5); fold them with launch_finish.  Integer min/max partials are unsigned keys (value ^ sign flip).
cudaError_t launch_binary(int op, int dtype, const BinDesc* d_descs, int n_chunks, int64_t total_tiles,
                          uint32_t* d_warp_counts, int* d_flags, cudaStream_t s, AggDev* tile_partials = nullptr);
cudaError_t launch_finish(bool is_float, const AggDev* parts, int64_t n_parts, int sm_count, AggDev* stage, unsigned int* ticket,
                          AggDev* result, cudaStream_t s);
cudaError_t launch_unary(int op, int dtype, const UnDesc* d_descs, int n_chunks, int64_t total_tiles,
                         uint32_t* d_warp_counts, cudaStream_t s);
cudaError_t launch_cast(int from, int to, const UnDesc* d_descs, int n_chunks, int64_t total_tiles,
                        uint32_t* d_warp_counts, cudaStream_t s);
// K4: one AggDev partial per CTA (integer min/max as unsigned keys: extended value ^ 2^63 for signed types);
// fold with launch_finish.
cudaError_t launch_reduce(int dtype, const RedDesc* d_descs, int n_chunks, int64_t total_tiles, AggDev* d_cta_partials,
                          cudaStream_t s);
int64_t reduce_partials(int dtype, int64_t tiles);  // number of partials launch_reduce writes
// Several columns of ONE dtype can share a launch: concatenate their chunk descriptors and start every column's tile
// numbering on a multiple of reduce_tiles_per_cta(dtype) -- a CTA then never mixes columns, and column k's partials are the
// CTA range [tile0_k / K, ceil(tile_end_k / K)).
int reduce_tiles_per_cta(int dtype);
// Fold up to kFinishMany partial ranges in ONE launch (grid.y = range); stage: n x sm_count records, tickets: n zeroed counters.
constexpr int kFinishMany = 64;
struct FinishJob { const AggDev* parts; long long n_parts; AggDev* result; int is_float; int pad; };
cudaError_t launch_finish_many(int n, const FinishJob* jobs, int sm_count, AggDev* stage, unsigned int* tickets, cudaStream_t s);
cudaError_t launch_generate(int dtype, int kind, double lo, double hi, uint64_t seed, uint64_t col, uint32_t null_mod,
                            const GenDesc* d_descs, int n_chunks, int64_t total_tiles,
                            uint32_t* d_warp_counts, cudaStream_t s);
cudaError_t launch_fill(void* p, size_t bytes, int sm_count, cudaStream_t s);

// Dates and timestamps (k_temporal.cu).  Storage unit of a temporal input: days (Date32) or seconds .. nanoseconds.
enum : int { TC_DAYS = 0, TC_S, TC_MS, TC_US, TC_NS };
struct TemporalParams {
    int32_t fn;          // bdf_temporal_fn
    int32_t aux;         // DATE_TRUNC: bdf_trunc_unit; NEXT_DAY: weekday 1..7 (Spark numbering)
    int32_t time_kind;   // the input is Time32 / Time64 (a time of day)
    int32_t pad;
    int64_t arg;         // DATE_ADD / DATE_SUB days, ADD_MONTHS months
    int64_t off;         // fixed tz offset in input units (civil functions), |off| < one day
    int64_t mul, div;    // TO_TIMESTAMP: v * mul (overflow -> NULL) when div == 1, else floor(v / div)
};
struct TemporalParams2 {
    int32_t fn;          // bdf_temporal_binary_fn
    int32_t cfg_a, cfg_b;
    int32_t pad;
    int64_t off_a, off_b;
};
int elems_per_tile_temporal(int in_dtype, int out_dtype);
int elems_per_tile_temporal2(int a_dtype, int b_dtype, int out_dtype);
cudaError_t launch_temporal(int cfg, int in_dtype, int out_dtype, const TemporalParams& p, const UnDesc* d_descs, int n_chunks,
                            int64_t total_tiles, uint32_t* d_warp_counts, cudaStream_t s);
cudaError_t launch_temporal2(int a_dtype, int b_dtype, int out_dtype, const TemporalParams2& p, const BinDesc* d_descs, int n_chunks,
                             int64_t total_tiles, uint32_t* d_warp_counts, cudaStream_t s);

struct Moments;   // moments.cuh

// Comparisons, and / or / not, filter (k_filter.cu).
cudaError_t launch_compare(int op, const BinDesc* d, int n, int64_t tiles, int ta, int tb, bool scalar_rhs, double scalar, uint32_t* wc,
                           cudaStream_t s);
int compare_tile_elems();
int bool_tile_elems();
cudaError_t launch_boolean(int op, const void* d, int n, int64_t tiles, uint32_t* wc, cudaStream_t s);
cudaError_t launch_filter_count(const void* d, int n, int64_t tiles, int tile_elems, unsigned int* tile_counts, long long* tile_offsets,
                                long long* chunk_totals, cudaStream_t s);
cudaError_t launch_filter_scatter(int dtype, const void* d, int n, int64_t tiles, const long long* tile_offsets, cudaStream_t s);
size_t filter_desc_size();
size_t bool_desc_size();
void fill_filter_desc(void* base, int64_t i, const void* in, void* out, const uint32_t* vin, uint32_t* vout, const uint32_t* mval,
                      const uint32_t* mvalid, int64_t len, int64_t tile0, int off, int moff, int mvoff);
void fill_bool_desc(void* base, int64_t i, const uint32_t* a, const uint32_t* b, uint32_t* out, const uint32_t* va, const uint32_t* vb,
                    uint32_t* vout, int64_t len, int64_t tile0, int offa, int offb, int voffa, int voffb);

// A chain of Calculations fused into one pass (k_expr.cu).
int expr_tile_elems();
int expr_max_inputs();
int expr_max_nodes();
size_t expr_desc_size();
void fill_expr_desc(void* base, int64_t i, int n_inputs, const void* const* in, const uint32_t* const* vin, const int32_t* off, double* out,
                    uint32_t* vout, int64_t len, int64_t tile0);
size_t expr_prog_size();
void expr_prog_stats(const void* prog, int* n_instructions, int* n_temporaries);
int expr_compile(int n_inputs, const int* in_dtypes, int n_nodes, const int* op, const int* a, const int* b, void* prog);
cudaError_t launch_expr(const void* descs, int n_chunks, int64_t tiles, const void* prog, uint32_t* warp_counts, int* flags, AggDev* tile_partials,
                        cudaStream_t s);

// Null handling and conditional selection (k_cond.cu).  fn: bdf_row_fn (case_when is a COALESCE launch with n_conds > 0);
// test: bdf_null_test.  `descs` is the CondHead array of stride cond_desc_bytes(n_args).
int cond_tile_elems(int dtype);
int null_test_tile_elems(int dtype, int test);
cudaError_t launch_cond(int fn, int dtype, const void* descs, int n_args, int n_chunks, int64_t tiles, uint32_t* warp_counts, cudaStream_t s);
cudaError_t launch_null_test(int test, int dtype, const void* descs, int n_chunks, int64_t tiles, cudaStream_t s);

// Exclusive prefix scans (k_scan.cu).  launch_scan_one scans `count` entries in place in one CTA; *total = their sum unless total is
// null.  The others scan n 64-bit entries in place in a buffer of n + 1: afterwards data[i] = the sum of the entries before i and
// data[n] = the total; sums is scratch of scan_tile_sums(n) entries.  k...Launches: the kernels each launcher counts for.
template <typename T>
cudaError_t launch_scan_one(T* data, long long count, T* total, cudaStream_t s);
long long scan_tile_sums(long long n);
constexpr int kScanSumsLaunches = 2;   // sums already holds the tile sums (kScanTile entries per CTA, scan.cuh)
cudaError_t launch_scan_sums(unsigned long long* data, long long n, unsigned long long* sums, cudaStream_t s);
constexpr int kScanLaunches = 3;
cudaError_t launch_scan(unsigned long long* data, long long n, unsigned long long* sums, cudaStream_t s);
constexpr int kScanPopcountLaunches = 3;   // the entries are the popcounts of words[0, n_words): counts[w] = the set bits before word w
cudaError_t launch_scan_popcount(const uint32_t* words, long long n_words, unsigned long long* counts, unsigned long long* sums, cudaStream_t s);

// Sort indices and take (k_sort.cu).
size_t sort_chunk_size();
void fill_sort_chunk(void* base, int64_t i, const void* values, const uint32_t* validity, int64_t start, int32_t bit_off, int32_t val_bit_off);
int sort_tile_elems();
int take_tile_elems();
int sort_pass_ctas(int64_t n, int sm_count);
cudaError_t launch_iota(uint32_t* out, int64_t n, int sm_count, cudaStream_t s);
int sort_key_bytes(int dtype);
cudaError_t launch_sort_keys(int dtype, const void* chunks, int n_chunks, const uint32_t* idx, int64_t n, int mode, int descending,
                             void* keys, unsigned long long* agree, int sm_count, cudaStream_t s);
cudaError_t launch_radix_pass(int key_bytes, const void* keys_in, const uint32_t* idx_in, int64_t n, int shift, unsigned int* block_hist,
                              void* keys_out, uint32_t* idx_out, int sm_count, cudaStream_t s);
cudaError_t launch_take(int dtype, const void* vals, int n_vals, const void* idxs, int n_idxs, int64_t n, int64_t n_rows_values, void* out,
                        uint32_t* vout, uint32_t* warp_counts, int* flags, cudaStream_t s);

// Group-by (k_group.cu).
cudaError_t launch_group_heads(int n_keys, const void* const* values, const uint32_t* const* valid, const int* widths, const int* is_float,
                               int and_last_valid, long long n, uint32_t* words, cudaStream_t s);
cudaError_t launch_group_reduce(int dtype, bool extra, const void* val, const uint32_t* vvalid, const uint32_t* starts, long long n_groups, long long n_rows,
                                void* sum, long long* count, void* mn, void* mx, double* avg, uint32_t* nonempty, void* scratch, int sm_count, cudaStream_t s);
cudaError_t launch_group_bounds(const uint32_t* idx, const uint32_t* starts, long long n_groups, long long n_rows, uint32_t* first, uint32_t* last,
                                cudaStream_t s);
cudaError_t launch_group_distinct(const uint32_t* pos, long long n_pos, const uint32_t* starts, long long n_groups, long long n_rows, long long* out,
                                  uint32_t* first, cudaStream_t s);
cudaError_t launch_group_moments(int dtype, const void* val, const uint32_t* vvalid, const uint32_t* starts, long long n_groups, long long n_rows,
                                 Moments* mom, void* scratch, int sm_count, cudaStream_t s);
cudaError_t launch_group_stats(const Moments* mom, long long n_groups, int stat, double* out, uint32_t* valid, cudaStream_t s);
size_t group_big_scratch_bytes(long long n_rows);

// Statistical aggregates (k_moments.cu).
cudaError_t launch_moments(int dtype, const RedDesc* d, int n, int64_t tiles, Moments* partials, Moments* result, cudaStream_t s);
int64_t moments_partials(int64_t tiles);

// Column distributions (k_dist.cu).
int dist_tile_elems(int dtype);
cudaError_t launch_select_pass(int dtype, int key_bytes, bool compact, const RedDesc* d, int n, int64_t tiles, const unsigned long long* prefixes,
                               int m, unsigned long long pmask, int shift, unsigned long long* hist, unsigned long long* and_or,
                               const uint32_t* chosen, void* out, unsigned long long* cursor, int sm_count, cudaStream_t s);
cudaError_t launch_hist(int dtype, bool range, const RedDesc* d, int n, int64_t tiles, const double* edges, double lo, double hi, int nbins,
                        unsigned long long* out, int sm_count, cudaStream_t s);
cudaError_t launch_dist_groups(const uint32_t* starts, long long n_groups, long long n_rows, const uint32_t* pos, long long n_pos, const uint32_t* valid,
                               uint32_t* first_run, uint32_t* vend, cudaStream_t s);
cudaError_t launch_dist_runs(const uint32_t* pos, long long n_pos, const uint32_t* starts, long long n_groups, long long n_rows, const uint32_t* first_run,
                             const uint32_t* vend, long long* counts, unsigned long long* best, cudaStream_t s);
cudaError_t launch_dist_mode(const unsigned long long* best, long long n_groups, const uint32_t* first_run, const uint32_t* pos, uint32_t* row,
                             uint32_t* row_valid, long long* freq, cudaStream_t s);
cudaError_t launch_dist_median(int dtype, const void* sval, const uint32_t* starts, long long n_groups, const uint32_t* vend, double* out,
                               uint32_t* out_valid, cudaStream_t s);

// Joins (k_join.cu).
cudaError_t launch_join_count(int n_keys, const int* dtypes, const void* const* probe_tables, const int* probe_chunks, const void* const* build_keys,
                              const uint32_t* const* build_valid, long long n_probe, const uint32_t* run_starts, long long n_runs, long long n_build,
                              int outer, unsigned long long* counts, uint32_t* match_start, unsigned char* hit, unsigned long long* block_sums,
                              cudaStream_t s);
cudaError_t launch_join_emit(const unsigned long long* offs, long long n_probe, const uint32_t* match_start, const uint32_t* perm, unsigned long long probe_rows,
                             const uint32_t* unmatched, unsigned long long n_out, uint32_t* probe_out, uint32_t* probe_valid, uint32_t* build_out,
                             uint32_t* build_valid, cudaStream_t s);
cudaError_t launch_join_unmatched(const uint32_t* perm, long long n_build, const uint32_t* run_starts, long long n_runs, const unsigned char* hit,
                                  uint32_t* mask, int sm_count, cudaStream_t s);
cudaError_t launch_join_exists(int n_keys, const int* dtypes, const void* const* probe_tables, const int* probe_chunks, const void* const* build_keys,
                               const uint32_t* const* build_valid, long long n_probe, long long n_runs, int anti, uint32_t* mask, cudaStream_t s);
cudaError_t launch_join_asof(int n_by, const int* dtypes, const void* const* probe_tables, const int* probe_chunks, const void* const* build_keys,
                             const uint32_t* const* build_valid, int on_dtype, const void* on_table, int on_chunks, const void* on_build,
                             const uint32_t* on_build_valid, int direction, int exact, int has_tol, unsigned long long tol, double tol_f,
                             long long n_probe, const uint32_t* run_starts, long long n_runs, long long n_build, const uint32_t* perm, uint32_t* out,
                             uint32_t* out_valid, cudaStream_t s);

// Top-k (k_topk.cu).  chunks: topk_chunk_size() bytes each, filled by fill_topk_chunk, tiles of topk_tile_elems(dtype) elements.
// ids: the row of every tie-set position (gathered rounds) or null (positional).  tie and counts[0..1] are zeroed by the caller.
int topk_chunk_size();
int topk_tile_elems(int dtype);
void fill_topk_chunk(void* descs, int64_t i, const void* values, const uint32_t* validity, int64_t len, int64_t tile0, int64_t row0, int bit_off,
                     bool owns_words);
cudaError_t launch_topk_mark(int dtype, const void* chunks, int n_chunks, int64_t tiles, unsigned long long t, bool all_valid, bool descending,
                             const uint32_t* ids, uint32_t* chosen, uint32_t* tie, unsigned long long* counts, int sm_count, cudaStream_t s);
cudaError_t launch_topk_choose(const uint32_t* ids, long long count, uint32_t* chosen, cudaStream_t s);

// Distinct rows and set operations (k_setop.cu).  heads: {head words, per-word run prefix, run starts} of the sorted positions.
// mode: 0..2 bdf_keep (duplicated), 3 + bdf_setop.  words: one bit per output row at the row's original position, zeroed by the caller.
cudaError_t launch_setop_left_count(const void* const* heads, long long n_runs, long long n, const uint32_t* perm, long long n_left,
                                    uint32_t* run_left, cudaStream_t s);
cudaError_t launch_setop_mark(const void* const* heads, long long n_runs, long long n, const uint32_t* perm, long long n_out, int mode,
                              const uint32_t* run_left, uint32_t* words, cudaStream_t s);
cudaError_t launch_setop_widen_bool(const void* bits, long long off, long long len, unsigned char* out, cudaStream_t s);
cudaError_t launch_bitmap_rebase(const void* src, long long off, long long len, uint32_t* dst, cudaStream_t s);

// Window functions (k_window.cu).
cudaError_t launch_window_rank(const void* const* p, long long n_p, const void* const* q, long long n_q, long long n, const uint32_t* perm,
                               void* const* outs, cudaStream_t s);
cudaError_t launch_window_shift(int dtype, const void* const* p, long long n_p, long long n, const void* x, int nx, long long k, int lead,
                                unsigned long long def_bits, int has_def, void* out, uint32_t* vout, cudaStream_t s);
size_t window_scan_scratch_bytes(long long n);
cudaError_t launch_window_scan(int dtype, int fn, const void* x, int nx, const uint32_t* heads, long long n, void* scratch, void* out, uint32_t* vout,
                               cudaStream_t s);
// Bounded frames: how every sorted position finds its frame [s, e] inside its partition (the rules are in include/b200df.h).
enum : int { WIN_FR_ROWS = 0, WIN_FR_PEERS, WIN_FR_RANGE };
struct WinFrameDesc {
    int kind;                 // ROWS: offsets from the position; PEERS: partition start .. last peer; RANGE: offsets of the order key
    int key_dtype, key_desc, key_chunks;
    long long start, end;     // ROWS and integer RANGE; LLONG_MIN / LLONG_MAX = UNBOUNDED
    double start_f, end_f;    // float RANGE; -inf / +inf = UNBOUNDED
    const void* key;          // RANGE: the order key in sorted order, as a chunk table (sort_table)
};
int window_frame_levels(long long n);
size_t window_frame_scratch_bytes(int dtype, long long n);
cudaError_t launch_window_frame_build(int dtype, const void* x, int nx, long long n, void* scratch, cudaStream_t s);
cudaError_t launch_window_frame_agg(int dtype, int fn, const void* const* p, long long n_p, const void* const* q, long long n_q, const WinFrameDesc& f,
                                    const void* x, int nx, long long n, void* scratch, void* out, uint32_t* vout, cudaStream_t s);
cudaError_t launch_window_valid_words(const void* x, int nx, long long n, uint32_t* words, cudaStream_t s);
cudaError_t launch_window_frame_value(int dtype, int which, long long nth, const void* const* p, long long n_p, const void* const* q, long long n_q,
                                      const WinFrameDesc& f, const void* x, int nx, long long n, const uint32_t* vwords,
                                      const unsigned long long* vprefix, void* out, uint32_t* vout, cudaStream_t s);

// CSV reader (k_csv.cu).
int csv_tile_bytes();
int csv_parse_rows();
size_t csv_desc_bytes();
size_t csv_slow_bytes();
size_t csv_patch_bytes();
cudaError_t launch_csv_tokenize(const uint8_t* text, long long n, uint8_t delim, uint32_t* agg, uint8_t* start, int* final_state, uint16_t* fe,
                                uint16_t* re, unsigned long long* block_counts, cudaStream_t s);
cudaError_t launch_csv_index(const uint16_t* fe, const uint16_t* re, long long n, const unsigned long long* block_offsets, unsigned long long* ends,
                             unsigned long long* first_rec, cudaStream_t s);
cudaError_t launch_csv_check(const unsigned long long* ends, long long n_fields, long long k, unsigned long long* bad, int sm_count, cudaStream_t s);
cudaError_t launch_csv_infer(const uint8_t* text, const unsigned long long* ends, long long f0, long long f1, long long k, unsigned int* col_bits,
                             int sm_count, cudaStream_t s);
cudaError_t launch_csv_parse(const uint8_t* text, const unsigned long long* ends, const void* cols, int n_cols, long long f0, long long k, long long n_rows,
                             long long batch, unsigned long long* err_key, void* slow, unsigned long long* n_slow, long long slow_cap, cudaStream_t s);
cudaError_t launch_csv_scatter(const void* patches, long long n, cudaStream_t s);

// Parquet reader (k_parquet.cu; the page, tile, output and run records are parquet_decode.cuh's pq::Page, Tile, Out and Run).
size_t pq_page_bytes();
size_t pq_tile_bytes();
size_t pq_out_bytes();
size_t pq_run_bytes();
cudaError_t launch_pq_snappy(const void* pages, int n_pages, const uint8_t* upload, uint8_t* scratch, int* err, int sm_count, cudaStream_t s);
cudaError_t launch_pq_runs(const void* pages, int n_pages, const uint8_t* upload, const uint8_t* scratch, void* runs, void* meta, int* err,
                           cudaStream_t s);
cudaError_t launch_pq_levels(const void* pages, const void* tiles, int n_tiles, const uint8_t* upload, const uint8_t* scratch, const void* runs,
                             const void* meta, const void* outs, long long batch, int* tile_valid, unsigned long long* nulls, int* err,
                             cudaStream_t s);
cudaError_t launch_pq_values(const void* pages, const void* tiles, int n_tiles, const uint8_t* upload, const uint8_t* scratch, const void* runs,
                             const void* meta, const void* outs, long long batch, const int* tile_valid, int* err, cudaStream_t s);

// line-delimited JSON reader (k_json.cu).
int json_tile_bytes();
int json_parse_rows();
size_t json_member_bytes();
size_t json_key_bytes();
size_t json_desc_bytes();
size_t json_slow_bytes();
size_t json_list_chunk_bytes();
cudaError_t launch_json_nl_count(const uint8_t* text, long long n, unsigned long long* counts, cudaStream_t s);
cudaError_t launch_json_nl_index(const uint8_t* text, long long n, const unsigned long long* offsets, unsigned long long* nl, cudaStream_t s);
cudaError_t launch_json_lex(const uint8_t* text, long long n, const unsigned long long* nl, long long n_nl, unsigned long long* members,
                            unsigned long long* is_rec, unsigned long long* bad, int sm_count, cudaStream_t s);
cudaError_t launch_json_members(const uint8_t* text, long long n, const unsigned long long* nl, long long n_nl, const unsigned long long* first_member,
                                const unsigned long long* rec_of, void* members, int sm_count, cudaStream_t s);
cudaError_t launch_json_keys(const uint8_t* text, const void* members, long long n_members, void* table, unsigned cap, unsigned int* full, int sm_count,
                             cudaStream_t s);
cudaError_t launch_json_resolve(const uint8_t* text, const void* members, long long n_members, const void* table, unsigned cap, const int* col_of, int n_cols,
                                unsigned int* slots, unsigned int* collision, int sm_count, cudaStream_t s);
cudaError_t launch_json_infer(const void* members, const unsigned int* slots, long long n_slots, int n_cols, unsigned int* col_bits, int sm_count, cudaStream_t s);
cudaError_t launch_json_parse(const uint8_t* text, const void* members, const unsigned int* slots, int n_file_cols, const void* cols, int n_cols, long long n_rows,
                              long long batch, void* slow, unsigned long long* n_slow, long long slow_cap, cudaStream_t s);
cudaError_t launch_json_list_count(const uint8_t* text, const void* members, const unsigned int* slots, int n_file_cols, int file_col, long long n_rows,
                                   long long batch, unsigned long long* counts, uint32_t* valid_words, unsigned long long* chunk_nulls, cudaStream_t s);
cudaError_t launch_json_bounds(const unsigned long long* offs, long long n_rows, long long batch, long long n_chunks, unsigned long long* bounds, cudaStream_t s);
cudaError_t launch_json_list_fill(const uint8_t* text, const void* members, const unsigned int* slots, int n_file_cols, int file_col, int dtype, long long n_rows,
                                  long long batch, const unsigned long long* offs, const uint32_t* valid_words, const void* out, unsigned long long* elem_nulls,
                                  void* slow, unsigned long long* n_slow, long long slow_cap, cudaStream_t s);

// CSV writer (k_csv_write.cu).
cudaError_t launch_csvw_measure(const CsvwDesc* cols, const long long* chunk_start, int n_cols, int n_chunks, long long row0, long long rows,
                                unsigned long long* lens, unsigned long long* block_sums, cudaStream_t s);
cudaError_t launch_csvw_emit(const CsvwDesc* cols, const long long* chunk_start, int n_cols, int n_chunks, long long row0, long long rows, int delim,
                             const unsigned long long* offs, char* out, cudaStream_t s);

// JSON writer (k_json_write.cu).
cudaError_t launch_jsonw_window(const JsonwArgs& a, long long row0, long long rows, long long max_rows, long long elem_cap, cudaStream_t s);
cudaError_t launch_jsonw_elem_len(const JsonwArgs& a, long long n_elems, unsigned long long* elens, unsigned long long* block_sums, cudaStream_t s);
cudaError_t launch_jsonw_measure(const JsonwArgs& a, long long row0, long long rows, const unsigned long long* escan, unsigned long long* lens,
                                 unsigned long long* block_sums, cudaStream_t s);
cudaError_t launch_jsonw_cut(const JsonwArgs& a, long long row0, long long rows, const unsigned long long* offs, unsigned long long cap, int max_cuts,
                             long long* cuts, cudaStream_t s);
cudaError_t launch_jsonw_emit(const JsonwArgs& a, long long wrow0, long long r0, long long r1, const unsigned long long* offs, unsigned long long base,
                              const unsigned long long* escan, long long* lpos, long long lpos_stride, char* out, cudaStream_t s);
cudaError_t launch_jsonw_elem_emit(const JsonwArgs& a, int list, long long e0, long long e1, long long wrow0, const unsigned long long* escan,
                                   const long long* lpos, long long lpos_stride, unsigned long long base, char* out, cudaStream_t s);

// Parquet writer (k_parquet_write.cu; the page, tile and page-result records are parquet_encode.cuh's pq::WPage, WTile and WPageOut).
size_t pqw_page_bytes();
size_t pqw_tile_bytes();
size_t pqw_out_bytes();
cudaError_t launch_pqw_rgid(const long long* rg_start, int n_rg, long long n, uint32_t* out, int sm_count, cudaStream_t s);
cudaError_t launch_pqw_dict(const uint32_t* run_rg, const uint32_t* run_valid, long long n_runs, const uint32_t* head, const unsigned long long* prefix,
                            const uint32_t* perm, long long n, unsigned int* count, unsigned int* first, uint32_t* ids, int sm_count, cudaStream_t s);
cudaError_t launch_pqw_encode(const void* pages, int n_pages, const void* tiles, int n_tiles, unsigned int* tile_valid, unsigned int* tile_base, void* lay,
                              uint8_t* raw, void* out, cudaStream_t s);
cudaError_t launch_pqw_snappy(const void* pages, const int* frag_page, int n_frags, uint8_t* raw, void* out, uint8_t* frag, unsigned int* frag_len,
                              cudaStream_t s);

// List columns (k_list.cu).
size_t list_find_scratch_bytes(long long n_elem);
cudaError_t launch_list_find(int dtype, const int32_t* off, const uint32_t* lvalid, long long len, long long n_elem, const void* values,
                             const uint32_t* vvalid, int vbit_off, uint64_t value_bits, int mode, uint32_t* bits, int32_t* pos, void* scratch,
                             int sm_count, cudaStream_t s);
cudaError_t launch_list_parent(const int32_t* off, const uint32_t* lvalid, const uint32_t* and_valid, long long len, long long n_elem, long long list0,
                               long long elem0, uint32_t* parent, uint32_t* inlist, cudaStream_t s);
cudaError_t launch_list_remove_mask(int dtype, const void* values, const uint32_t* vvalid, int vbit_off, long long n_elem, long long elem0,
                                    uint64_t value_bits, const uint32_t* inlist, uint32_t* keep, cudaStream_t s);
cudaError_t launch_list_mark(const uint32_t* perm, const uint32_t* head, const uint32_t* pvalid, long long n, long long split, int mode, uint32_t* keep,
                             cudaStream_t s);
cudaError_t launch_list_offsets(const uint32_t* kp, long long n_kept, long long n_lists, long long mult, int32_t* out, cudaStream_t s);
cudaError_t launch_list_repeat(const int32_t* base, long long n_lists, long long count, const uint32_t* rows, long long n_out, uint32_t* src, cudaStream_t s);
cudaError_t launch_list_size(const int32_t* off, const uint32_t* lvalid, long long len, int32_t* out, cudaStream_t s);
cudaError_t launch_list_minmax_valid(const int32_t* off, const uint32_t* lvalid, const uint32_t* nonempty, long long len, uint32_t* valid, int* empty,
                                     cudaStream_t s);
struct ListChunkDesc {         // one list chunk in the concatenated list rows and elements of a take / filter
    const int32_t* off;        // len + 1 offsets from 0
    const uint32_t* valid;     // list validity at bit 0, or nullptr
    long long start, elem0;    // first global list row and first global element of the chunk
};
cudaError_t launch_list_take_sizes(const void* idx_table, int n_idx, long long n, const void* list_table, int n_lists, long long total, int local,
                                   uint32_t* const* vout, unsigned long long* sizes, uint32_t* first, unsigned long long* nulls, int* flags,
                                   cudaStream_t s);
cudaError_t launch_list_take_rows(const unsigned long long* off, long long n, const uint32_t* first, long long n_out, uint32_t* src, cudaStream_t s);
cudaError_t launch_list_rebase(const unsigned long long* off, long long len, int32_t* out, cudaStream_t s);
cudaError_t launch_list_ranks(const uint32_t* kept, long long n_kept, const uint32_t* starts, long long n_groups, int32_t* out, cudaStream_t s);

}  // namespace bdf
