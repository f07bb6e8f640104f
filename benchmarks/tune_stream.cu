// tune_stream.cu -- developer micro-benchmark used to pick the tile shape / grid policy of the streaming kernels
// (K1 add, K4 sum, K5 fused add+sum) on an H100.  Not part of the product library.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo benchmarks/tune_stream.cu -o benchmarks/bin/tune_stream
//   ./benchmarks/bin/tune_stream [rows]
// Every variant is timed with CUDA events over inputs far larger than L2 (1e8 f64 rows), best and median of 20.
//
// Sections:
//   ceiling   plain read-only (sum), copy (1 read + 1 write) and c = a + b (2 reads + 1 write) kernels: the best rate of
//             each is the achievable HBM rate that the product kernels are judged against
//   k5        candidates for K5 (k_binary<double,ADD,AGG=true>): c = a + b with one 32-byte partial per 2048-row tile, folded
//             exactly as the product folds it (lane order, xor tree, warps in order); threads x U, one tile per CTA or a
//             persistent grid walking a contiguous tile range, an L2 evict_first policy, and a cp.async.bulk (TMA) pipeline
//
// Result on one H100 80GB HBM3 at a 400 W power limit (details in DESIGN.md sections 4 and 5): ceiling read-only 3.07, copy
// 2.99, 2R1W 3.04 TB/s; K5 at 256 threads x U = 4, one tile per CTA, 0.805 ms = 2.98 TB/s, and no candidate more than 0.7 %
// faster (persistent -5 to -6 %, cp.async.bulk -3 to -4 %), so K5 keeps that shape.
// Only 16-byte accesses are swept: 256-bit ld/st.global need sm_100.
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1); } } while (0)

struct V16 { union { uint4 q; double d[2]; }; };

__device__ __forceinline__ void ld16(V16& v, const void* p) {
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.q.x), "=r"(v.q.y), "=r"(v.q.z), "=r"(v.q.w) : "l"(p));
}
__device__ __forceinline__ void st16(void* p, const V16& v) {
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" :: "l"(p), "r"(v.q.x), "r"(v.q.y), "r"(v.q.z), "r"(v.q.w) : "memory");
}
__device__ __forceinline__ uint64_t policy_evict_first() {
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void ld16_ef(V16& v, const void* p, uint64_t pol) {
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=r"(v.q.x), "=r"(v.q.y), "=r"(v.q.z), "=r"(v.q.w) : "l"(p), "l"(pol));
}
__device__ __forceinline__ void st16_ef(void* p, const V16& v, uint64_t pol) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.u32 [%0], {%1,%2,%3,%4}, %5;"
                 :: "l"(p), "r"(v.q.x), "r"(v.q.y), "r"(v.q.z), "r"(v.q.w), "l"(pol) : "memory");
}

// ---- ceiling: copy c = a (1R1W) and add c = a + b (2R1W) ------------------------------------------------
template <int THREADS, int U, bool PERSIST>
__global__ void __launch_bounds__(THREADS) k_copy(const double* __restrict__ a, double* __restrict__ c, long n_tiles) {
    constexpr long TILE = (long)THREADS * U * 2;
    for (long tile = blockIdx.x; tile < n_tiles; tile += PERSIST ? gridDim.x : n_tiles) {
        const long base = tile * TILE;
        V16 x[U];
#pragma unroll
        for (int j = 0; j < U; j++) ld16(x[j], a + base + (long)(j * THREADS + threadIdx.x) * 2);
#pragma unroll
        for (int j = 0; j < U; j++) st16(c + base + (long)(j * THREADS + threadIdx.x) * 2, x[j]);
    }
}

template <int THREADS, int U, bool PERSIST>
__global__ void __launch_bounds__(THREADS) k_add(const double* __restrict__ a, const double* __restrict__ b, double* __restrict__ c, long n_tiles) {
    constexpr long TILE = (long)THREADS * U * 2;
    for (long tile = blockIdx.x; tile < n_tiles; tile += PERSIST ? gridDim.x : n_tiles) {
        const long base = tile * TILE;
        V16 x[U], y[U];
#pragma unroll
        for (int j = 0; j < U; j++) { const long e = base + (long)(j * THREADS + threadIdx.x) * 2; ld16(x[j], a + e); ld16(y[j], b + e); }
#pragma unroll
        for (int j = 0; j < U; j++) {
            const long e = base + (long)(j * THREADS + threadIdx.x) * 2;
            V16 r;
            r.d[0] = __dadd_rn(x[j].d[0], y[j].d[0]);
            r.d[1] = __dadd_rn(x[j].d[1], y[j].d[1]);
            st16(c + e, r);
        }
    }
}

// ---- sum (read only) ----------------------------------------------------------------------------------
__device__ __forceinline__ double block_sum(double v, double* smem) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) smem[warp] = v;
    __syncthreads();
    double r = 0;
    if (warp == 0) {
        r = lane < (int)(blockDim.x >> 5) ? smem[lane] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
    }
    return r;
}

template <int THREADS, int U>
__global__ void __launch_bounds__(THREADS) k_sum(const double* __restrict__ a, long n_tiles, double* __restrict__ partials) {
    constexpr long TILE = (long)THREADS * U * 2;
    __shared__ double smem[32];
    double acc[2] = {0.0, 0.0};
    for (long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const long base = tile * TILE;
        V16 x[U];
#pragma unroll
        for (int j = 0; j < U; j++) ld16(x[j], a + base + (long)(j * THREADS + threadIdx.x) * 2);
#pragma unroll
        for (int j = 0; j < U; j++) { acc[0] = __dadd_rn(acc[0], x[j].d[0]); acc[1] = __dadd_rn(acc[1], x[j].d[1]); }
    }
    const double s = block_sum(acc[0] + acc[1], smem);
    if (threadIdx.x == 0) partials[blockIdx.x] = s;
}

// ---- K5 candidates ------------------------------------------------------------------------------------
// The per-tile partial of the product: 32 bytes (sum, min key, max key, count); sum folded per thread in element order,
// xor tree inside the warp, warps in order by thread 0.
struct Part { unsigned long long sum_bits, min_bits, max_bits, count; };

template <int THREADS>
__device__ __forceinline__ void tile_partial(double s, double* s_w, Part* out) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = s_w[0];
#pragma unroll
        for (int w = 1; w < THREADS / 32; w++) t = __dadd_rn(t, s_w[w]);
        *out = Part{(unsigned long long)__double_as_longlong(t), ~0ull, 0ull, 0ull};
    }
}

// One tile of THREADS x U x 16 B per array.  EF: loads and stores carry an L2 evict_first policy.
template <int THREADS, int U, bool EF>
__device__ __forceinline__ void k5_tile(const double* __restrict__ a, const double* __restrict__ b, double* __restrict__ c, long base,
                                        double* s_w, Part* out, uint64_t pol) {
    V16 x[U], y[U];
#pragma unroll
    for (int j = 0; j < U; j++) {
        const long e = base + (long)(j * THREADS + threadIdx.x) * 2;
        if constexpr (EF) { ld16_ef(x[j], a + e, pol); ld16_ef(y[j], b + e, pol); } else { ld16(x[j], a + e); ld16(y[j], b + e); }
    }
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < U; j++) {
        const long e = base + (long)(j * THREADS + threadIdx.x) * 2;
        V16 r;
        r.d[0] = __dadd_rn(x[j].d[0], y[j].d[0]); s = __dadd_rn(s, r.d[0]);
        r.d[1] = __dadd_rn(x[j].d[1], y[j].d[1]); s = __dadd_rn(s, r.d[1]);
        if constexpr (EF) st16_ef(c + e, r, pol); else st16(c + e, r);
    }
    tile_partial<THREADS>(s, s_w, out);
}

// PERSIST = false: one tile per CTA (the product's shape before this probe).  PERSIST = true: gridDim.x CTAs, CTA g walks
// the contiguous tiles [g * n / G, (g + 1) * n / G) with a bumped pointer; s_w is double-buffered so one barrier per tile holds.
template <int THREADS, int U, bool PERSIST, bool EF>
__global__ void __launch_bounds__(THREADS) k5(const double* __restrict__ a, const double* __restrict__ b, double* __restrict__ c, long n_tiles,
                                              Part* __restrict__ parts) {
    constexpr long TILE = (long)THREADS * U * 2;
    __shared__ double s_w[2][THREADS / 32];
    const uint64_t pol = EF ? policy_evict_first() : 0ull;
    if constexpr (!PERSIST) {
        k5_tile<THREADS, U, EF>(a, b, c, (long)blockIdx.x * TILE, s_w[0], &parts[blockIdx.x], pol);
    } else {
        const long t0 = (long)blockIdx.x * n_tiles / gridDim.x, t1 = (long)(blockIdx.x + 1) * n_tiles / gridDim.x;
        for (long t = t0; t < t1; t++) k5_tile<THREADS, U, EF>(a, b, c, t * TILE, s_w[t & 1], &parts[t], pol);
    }
}

// TMA: persistent, contiguous tile range per CTA; S stages of (a tile, b tile) filled by cp.async.bulk on an mbarrier each;
// threads add out of shared memory with the product's lane -> element order, write c over the a slot, and one thread
// stores it with a bulk shared -> global copy.  256 threads, 2048-row tiles (16 KiB per array).
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    unsigned done = 0;
    while (!done)
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst, const void* src, unsigned bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_u32(src)), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}

template <int S>
__global__ void __launch_bounds__(256) k5_tma(const double* __restrict__ a, const double* __restrict__ b, double* __restrict__ c, long n_tiles,
                                              Part* __restrict__ parts) {
    constexpr int THREADS = 256, U = 4;
    constexpr long TILE = (long)THREADS * U * 2;
    constexpr unsigned TB = (unsigned)(TILE * 8);
    extern __shared__ __align__(128) unsigned char smem[];
    double* sa = (double*)smem;                 // [S][TILE]
    double* sb = sa + (size_t)S * TILE;         // [S][TILE]
    __shared__ unsigned long long bar[S];
    __shared__ double s_w[2][THREADS / 32];
    const long t0 = (long)blockIdx.x * n_tiles / gridDim.x, t1 = (long)(blockIdx.x + 1) * n_tiles / gridDim.x;
    if (threadIdx.x == 0) {
        for (int s = 0; s < S; s++) mbar_init(&bar[s], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        for (int s = 0; s < S && t0 + s < t1; s++) {
            mbar_expect_tx(&bar[s], 2 * TB);
            bulk_g2s(sa + (size_t)s * TILE, a + (t0 + s) * TILE, TB, &bar[s]);
            bulk_g2s(sb + (size_t)s * TILE, b + (t0 + s) * TILE, TB, &bar[s]);
        }
    }
    __syncthreads();
    for (long t = t0; t < t1; t++) {
        const long i = t - t0;
        const int s = (int)(i % S);
        mbar_wait(&bar[s], (unsigned)((i / S) & 1));
        double* pa = sa + (size_t)s * TILE;
        const double* pb = sb + (size_t)s * TILE;
        double acc = 0.0;
#pragma unroll
        for (int j = 0; j < U; j++) {
            const int e = (j * THREADS + threadIdx.x) * 2;
            const double2 x = *(const double2*)(pa + e), y = *(const double2*)(pb + e);
            double2 r;
            r.x = __dadd_rn(x.x, y.x); acc = __dadd_rn(acc, r.x);
            r.y = __dadd_rn(x.y, y.y); acc = __dadd_rn(acc, r.y);
            *(double2*)(pa + e) = r;
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // c in shared memory is read by the bulk store next
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc = __dadd_rn(acc, __shfl_xor_sync(0xffffffffu, acc, o));
        if ((threadIdx.x & 31) == 0) s_w[i & 1][threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            bulk_s2g(c + t * TILE, pa, TB);
            double v = s_w[i & 1][0];
#pragma unroll
            for (int w = 1; w < THREADS / 32; w++) v = __dadd_rn(v, s_w[i & 1][w]);
            parts[t] = Part{(unsigned long long)__double_as_longlong(v), ~0ull, 0ull, 0ull};
            if (t + S < t1) {
                asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // the store has read the a slot
                mbar_expect_tx(&bar[s], 2 * TB);
                bulk_g2s(pa, a + (t + S) * TILE, TB, &bar[s]);
                bulk_g2s(sb + (size_t)s * TILE, b + (t + S) * TILE, TB, &bar[s]);
            }
        }
    }
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// ---- harness -----------------------------------------------------------------------------------------
static cudaEvent_t e0, e1;
template <typename F>
static float run(const char* name, double bytes, F launch) {
    for (int i = 0; i < 3; i++) launch();
    CK(cudaDeviceSynchronize());
    std::vector<float> ms(20);
    for (auto& m : ms) {
        CK(cudaEventRecord(e0));
        launch();
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        CK(cudaEventElapsedTime(&m, e0, e1));
    }
    CK(cudaGetLastError());
    std::sort(ms.begin(), ms.end());
    printf("%-52s best %.4f ms %7.1f GB/s | median %.4f ms %7.1f GB/s\n", name, ms[0], bytes / ms[0] / 1e6, ms[10], bytes / ms[10] / 1e6);
    return ms[0];
}

template <typename K>
static int resident(K kernel, int threads, size_t smem) {
    int n = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, threads, smem));
    return n;
}

int main(int argc, char** argv) {
    const long rows = argc > 1 ? atol(argv[1]) : 100000000L;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    printf("device %s, %d SMs, rows %ld\n", prop.name, sms, rows);
    double *a, *b, *c, *partials;
    const size_t bytes = (size_t)rows * 8 + (1 << 20);
    CK(cudaMalloc(&a, bytes)); CK(cudaMalloc(&b, bytes)); CK(cudaMalloc(&c, bytes)); CK(cudaMalloc(&partials, (size_t)rows / 64 * sizeof(Part) + (1 << 20)));
    CK(cudaMemset(a, 0, bytes)); CK(cudaMemset(b, 0, bytes)); CK(cudaMemset(c, 0, bytes));
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    const double B_ADD = 24.0 * rows, B_SUM = 8.0 * rows, B_COPY = 16.0 * rows;
    Part* parts = (Part*)partials;

    printf("== ceiling ==\n");
    float best_r = 1e30f, best_c = 1e30f, best_a = 1e30f;
    best_c = std::min(best_c, run("memcpy d2d (1R1W)", B_COPY, [&] { cudaMemcpyAsync(c, a, (size_t)rows * 8, cudaMemcpyDeviceToDevice); }));
#define COPY(T, U, P, CPS) { constexpr long TILE = (long)T * U * 2; const long nt = rows / TILE; \
        const long grid = P ? (long)sms * CPS : nt; char nm[96]; snprintf(nm, 96, "copy 1R1W T=%d U=%d %s", T, U, P ? "persist x" #CPS : "tile/CTA"); \
        best_c = std::min(best_c, run(nm, B_COPY, [&] { k_copy<T, U, P><<<(unsigned)grid, T>>>(a, c, nt); })); }
    COPY(256, 4, false, 0) COPY(256, 8, false, 0) COPY(512, 4, false, 0) COPY(256, 4, true, 8) COPY(256, 8, true, 4)
#define ADD(T, U, P, CPS) { constexpr long TILE = (long)T * U * 2; const long nt = rows / TILE; \
        const long grid = P ? (long)sms * CPS : nt; char nm[96]; snprintf(nm, 96, "add 2R1W T=%d U=%d %s", T, U, P ? "persist x" #CPS : "tile/CTA"); \
        best_a = std::min(best_a, run(nm, B_ADD, [&] { k_add<T, U, P><<<(unsigned)grid, T>>>(a, b, c, nt); })); }
    ADD(256, 4, false, 0) ADD(256, 2, false, 0) ADD(256, 8, false, 0) ADD(512, 4, false, 0) ADD(128, 4, false, 0)
    ADD(256, 4, true, 4) ADD(256, 4, true, 6) ADD(256, 4, true, 8) ADD(512, 2, true, 4) ADD(1024, 2, true, 2)
#define SUM(T, U, CPS) { constexpr long TILE = (long)T * U * 2; const long nt = rows / TILE; char nm[96]; \
        snprintf(nm, 96, "read-only sum T=%d U=%d grid=SMs x" #CPS, T, U); \
        best_r = std::min(best_r, run(nm, B_SUM, [&] { k_sum<T, U><<<sms * CPS, T>>>(a, nt, partials); })); }
    SUM(256, 4, 5) SUM(256, 4, 8) SUM(256, 8, 4) SUM(256, 8, 8) SUM(256, 16, 4) SUM(512, 4, 4) SUM(512, 8, 2) SUM(512, 8, 4)
    printf("CEILING read-only %.1f GB/s, copy 1R1W %.1f GB/s, add 2R1W %.1f GB/s (best of each class)\n",
           B_SUM / best_r / 1e6, B_COPY / best_c / 1e6, B_ADD / best_a / 1e6);

    printf("== k5 candidates (c = a + b, one 32-byte partial per tile) ==\n");
#define K5(T, U, P, EF) { constexpr long TILE = (long)T * U * 2; const long nt = rows / TILE; \
        const int occ = resident(k5<T, U, P, EF>, T, 0); const long grid = P ? (long)sms * occ : nt; char nm[96]; \
        snprintf(nm, 96, "k5 T=%d U=%d %s%s tile=%ld", T, U, P ? "persist contiguous" : "tile/CTA", EF ? " evict_first" : "", TILE); \
        if (P) printf("   (%d resident CTAs/SM)\n", occ); \
        run(nm, B_ADD, [&] { k5<T, U, P, EF><<<(unsigned)grid, T>>>(a, b, c, nt, parts); }); }
    K5(256, 4, false, false) K5(256, 2, false, false) K5(256, 8, false, false) K5(512, 2, false, false) K5(512, 4, false, false) K5(512, 8, false, false)
    K5(256, 4, true, false) K5(256, 2, true, false) K5(256, 8, true, false) K5(512, 2, true, false) K5(512, 4, true, false)
    K5(256, 4, false, true) K5(256, 4, true, true) K5(512, 2, false, true)
#define K5TMA(S) { constexpr long TILE = 2048; const long nt = rows / TILE; const size_t sm = (size_t)S * 2 * TILE * 8; \
        CK(cudaFuncSetAttribute(k5_tma<S>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm)); \
        const int occ = resident(k5_tma<S>, 256, sm); char nm[96]; snprintf(nm, 96, "k5 TMA bulk T=256 stages=%d (%d CTAs/SM)", S, occ); \
        run(nm, B_ADD, [&] { k5_tma<S><<<(unsigned)(sms * occ), 256, sm>>>(a, b, c, nt, parts); }); }
    K5TMA(2) K5TMA(3) K5TMA(4) K5TMA(6)

    // sequence as the product runs it: K5 back to back, events around the pair -> the launch-to-launch cost
    {
        constexpr long TILE = 2048; const long nt = rows / TILE;
        std::vector<float> ms(10);
        for (auto& m : ms) {
            CK(cudaEventRecord(e0));
            for (int k = 0; k < 10; k++) k5<256, 4, false, false><<<(unsigned)nt, 256>>>(a, b, c, nt, parts);
            CK(cudaEventRecord(e1));
            CK(cudaEventSynchronize(e1));
            CK(cudaEventElapsedTime(&m, e0, e1));
        }
        std::sort(ms.begin(), ms.end());
        printf("%-52s best %.4f ms per launch %7.1f GB/s\n", "k5 T=256 U=4 tile/CTA, 10 back to back", ms[0] / 10, B_ADD / (ms[0] / 10) / 1e6);
    }
    return 0;
}
