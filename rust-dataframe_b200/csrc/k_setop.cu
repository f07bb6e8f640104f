// k_setop.cu -- distinct rows and set operations (pandas' duplicated / drop_duplicates, Spark's intersect / intersectAll / subtract /
// exceptAll; the rules are in include/b200df.h), and the bit copies of the device concatenation.
//
// The host (runtime.cu setop_mask) sorts the key tuples stably with the radix lexsort -- for a set operation the left rows and then
// the right rows as one column, so that a run's left rows come first and in row order -- gathers them, marks the run heads with
// k_group_heads (group-by's key equality: one NULL, one NaN, -0.0 == 0.0), scans the popcounts of the head words and compacts the run
// starts, so that a position finds its run and the run's bounds in O(1), as k_window does.  The kernels here:
//   k_setop_left_count  set operations: the LAST left position of every run writes the run's left count cl.  One writer per run, no
//                       atomics; a run without left rows is never read.
//   k_setop_mark        per sorted position: the run bounds, then the decision -- duplicated (keep FIRST / LAST / NONE), or for a left
//                       position of a set operation "its rank among the run's left rows < q(cl, cr)" -- OR-ed as one bit into a
//                       zeroed bitmap of all left rows at the row's original position perm[i] (atomicOr: the 1e8-row bitmap is
//                       12.5 MB and stays in L2, where a byte per row did not; DESIGN §8 has both measured).  k_bitmap_rebase then
//                       copies every output chunk's bits to bit 0 of its own bitmap.
//   k_setop_widen_bool  a Boolean chunk (values bitmap at any bit offset) as one UInt8 per row, 0 or 1; Boolean keys are sorted and
//                       compared as UInt8.
//   k_bitmap_rebase     a bitmap that starts at bit `off` of its first byte, copied to bit 0 of another (the mask's chunks, the
//                       concatenation of sliced chunks and the widened Boolean's validity).
#include "common.cuh"

namespace bdf {

struct SetopRuns {
    const uint32_t* words;                 // bit i: sorted position i starts a run
    const unsigned long long* prefix;      // per head word: the runs that start before it
    const uint32_t* starts;                // the first position of every run
    long long n_runs, n;
};

__device__ __forceinline__ long long setop_run_of(const SetopRuns& h, long long i) {
    const uint32_t w = __ldg(h.words + (i >> 5));
    const uint32_t below = (2u << (i & 31)) - 1u;   // bits 0..i&31 (all 32 when i&31 == 31: 2u << 31 wraps to 0)
    return (long long)__ldg(h.prefix + (i >> 5)) + __popc(w & below) - 1;
}
__device__ __forceinline__ long long setop_run_end(const SetopRuns& h, long long r) {   // one past the run's last position
    return r + 1 < h.n_runs ? (long long)__ldg(h.starts + r + 1) : h.n;
}

__global__ void __launch_bounds__(kThreads)
k_setop_left_count(const SetopRuns runs, const uint32_t* __restrict__ perm, unsigned long long n_left, uint32_t* __restrict__ run_left) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= runs.n || __ldg(perm + i) >= n_left) return;
    const long long r = setop_run_of(runs, i);
    const long long e = setop_run_end(runs, r);
    if (i + 1 < e && __ldg(perm + i + 1) < n_left) return;   // not the run's last left position
    run_left[r] = (uint32_t)(i - __ldg(runs.starts + r) + 1);
}

// The decision of sorted position i, whose row is below n_out.  mode: 0..2 bdf_keep (duplicated), 3 + bdf_setop (set operations,
// which read run_left).
__device__ __forceinline__ bool setop_decide(const SetopRuns& runs, long long i, int mode, const uint32_t* __restrict__ run_left) {
    const long long r = setop_run_of(runs, i);
    const long long s = __ldg(runs.starts + r), e = setop_run_end(runs, r);
    if (mode < 3) return mode == 0 ? i > s : mode == 1 ? i + 1 < e : e - s > 1;
    const long long cl = __ldg(run_left + r), cr = e - s - cl;
    long long q;
    switch (mode - 3) {
        case 0: q = cr > 0 ? 1 : 0; break;              // INTERSECT (cl > 0: this row is one)
        case 1: q = cl < cr ? cl : cr; break;           // INTERSECT ALL
        case 2: q = cr == 0 ? 1 : 0; break;             // EXCEPT
        default: q = cl > cr ? cl - cr : 0; break;      // EXCEPT ALL
    }
    return i - s < q;   // the run's left rows come first, in row order: i - s is this row's rank among them
}

// words: one bit per output row, zeroed; only the true decisions are OR-ed in.
__global__ void __launch_bounds__(kThreads)
k_setop_mark(const SetopRuns runs, const uint32_t* __restrict__ perm, unsigned long long n_out, int mode, const uint32_t* __restrict__ run_left,
             uint32_t* __restrict__ words) {
    const long long i = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (i >= runs.n) return;
    const uint32_t row = __ldg(perm + i);
    if (row >= n_out) return;
    if (setop_decide(runs, i, mode, run_left)) atomicOr(words + (row >> 5), 1u << (row & 31));
}

// Bit `off + j` of src, for j < len; src is read byte-wise and never past its last byte that holds one of those bits.
__device__ __forceinline__ uint32_t rebased_word(const unsigned char* __restrict__ src, long long off, long long len, long long w) {
    const long long bit0 = off + 32 * w;
    const long long last = (off + len - 1) >> 3;
    unsigned long long acc = 0;
    for (int b = 0; b < 5; b++) {
        const long long k = (bit0 >> 3) + b;
        if (k <= last) acc |= (unsigned long long)__ldg(src + k) << (8 * b);
    }
    uint32_t word = (uint32_t)(acc >> (bit0 & 7));
    const long long rest = len - 32 * w;
    if (rest < 32) word &= (1u << rest) - 1u;
    return word;
}

__global__ void __launch_bounds__(kThreads)
k_bitmap_rebase(const unsigned char* __restrict__ src, long long off, long long len, uint32_t* __restrict__ dst) {
    const long long w = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (w * 32 >= len) return;
    dst[w] = rebased_word(src, off, len, w);
}

__global__ void __launch_bounds__(kThreads)
k_setop_widen_bool(const unsigned char* __restrict__ bits, long long off, long long len, unsigned char* __restrict__ out) {
    const long long j = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (j >= len) return;
    const long long b = off + j;
    out[j] = (__ldg(bits + (b >> 3)) >> (b & 7)) & 1u;
}

static cudaError_t grid_of(long long n, unsigned* blocks) {
    const long long b = (n + kThreads - 1) / kThreads;
    if (b > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    *blocks = (unsigned)b;
    return cudaSuccess;
}

static SetopRuns setop_runs(const void* const* heads, long long n_runs, long long n) {
    return SetopRuns{(const uint32_t*)heads[0], (const unsigned long long*)heads[1], (const uint32_t*)heads[2], n_runs, n};
}

cudaError_t launch_setop_left_count(const void* const* heads, long long n_runs, long long n, const uint32_t* perm, long long n_left,
                                    uint32_t* run_left, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    unsigned blocks = 0;
    cudaError_t e = grid_of(n, &blocks);
    if (e != cudaSuccess) return e;
    k_setop_left_count<<<blocks, kThreads, 0, s>>>(setop_runs(heads, n_runs, n), perm, (unsigned long long)n_left, run_left);
    return cudaGetLastError();
}

cudaError_t launch_setop_mark(const void* const* heads, long long n_runs, long long n, const uint32_t* perm, long long n_out, int mode,
                              const uint32_t* run_left, uint32_t* words, cudaStream_t s) {
    if (n <= 0) return cudaSuccess;
    if (mode < 0 || mode > 6) return cudaErrorInvalidValue;
    unsigned blocks = 0;
    cudaError_t e = grid_of(n, &blocks);
    if (e != cudaSuccess) return e;
    k_setop_mark<<<blocks, kThreads, 0, s>>>(setop_runs(heads, n_runs, n), perm, (unsigned long long)n_out, mode, run_left, words);
    return cudaGetLastError();
}

cudaError_t launch_bitmap_rebase(const void* src, long long off, long long len, uint32_t* dst, cudaStream_t s) {
    if (len <= 0) return cudaSuccess;
    unsigned blocks = 0;
    cudaError_t e = grid_of((len + 31) / 32, &blocks);
    if (e != cudaSuccess) return e;
    k_bitmap_rebase<<<blocks, kThreads, 0, s>>>((const unsigned char*)src, off, len, dst);
    return cudaGetLastError();
}

cudaError_t launch_setop_widen_bool(const void* bits, long long off, long long len, unsigned char* out, cudaStream_t s) {
    if (len <= 0) return cudaSuccess;
    unsigned blocks = 0;
    cudaError_t e = grid_of(len, &blocks);
    if (e != cudaSuccess) return e;
    k_setop_widen_bool<<<blocks, kThreads, 0, s>>>((const unsigned char*)bits, off, len, out);
    return cudaGetLastError();
}

}  // namespace bdf
