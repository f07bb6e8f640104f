// k_expr.cu -- SURVEY 8(f) N3: several consecutive Calculations of the evaluator fused into ONE pass.
//
// The reference's Evaluate::calculate (src/evaluation.rs:66-96, 97-323) materialises every Calculation as a new
// column: for BASELINE config 2 (e=a+b; f=e*c; g=f/d; h=sin(g)) that is 24+24+24+16 = 88 B/row of HBM traffic.
// When the intermediates are not kept (an optimiser pass like src/optimiser.rs can tell), the same chain needs only
// its inputs and its final column: 4 x 8 + 8 = 40 B/row.  Every node is exactly the operator the unfused path would
// run (__dadd_rn/__dmul_rn/__ddiv_rn, CUDA libm), so the final column is bit-identical to the unfused CUDA chain.
// Validity = AND of the inputs a node depends on; a divide node raises DivideByZero iff a slot that is valid FOR
// THAT NODE has a zero divisor (exactly what the materialised chain would report).  Null slots of the result carry
// payload 0.
//
// Execution model: the host compiles the straight-line DAG into an ACCUMULATOR program (expr_compile below): one
// register accumulator; the input tiles and up to two temporaries staged in shared memory (see k_expr).
#include "common.cuh"
#include "math_exact.cuh"

#include <cstdlib>
#include <vector>

namespace bdf {

constexpr int kExprMaxInputs = 6;
constexpr int kExprMaxNodes = 12;
constexpr int kExprMaxIns = 40;
constexpr int kExprUnroll = 4;       // 16-byte loads per lane and input: tile = 256 x 4 x 2 = 2048 rows (U=3 was slower)
constexpr int kExprMinCtas = 4;      // 64 registers: 4 CTAs/SM (U=4 unbounded: 80 regs, 3 CTAs, slower on the config-2 chain)
constexpr int kExprUnaryBase = 100;  // node op (C ABI): 0..6 = bdf_binop, 100 + bdf_unop = unary (operand a)

// Accumulator-machine opcodes.  Operand codes: shared-memory slot (0..ni-1 input column, ni.. temporary) or the accumulator itself.
enum : uint8_t { XI_BIN = 0 /* +binop: acc = acc OP operand */, XI_RBIN = 16 /* +binop: acc = operand OP acc */, XI_LOAD = 32, XI_STORE = 33, XI_UN = 64 /* +unop */ };
constexpr int kOperandAcc = 255;
constexpr int kExprMaxTemps = 2;

struct ExprProg {
    int n_inputs, n_ins, n_slots;   // n_slots = inputs + temporaries the program uses
    uint8_t op[kExprMaxIns], src[kExprMaxIns];
    uint8_t in_dtype[kExprMaxInputs];   // element type of every input column (read through `as f64`: Function::Cast to Float64)
};
struct ExprDesc {
    const void* in[kExprMaxInputs];
    const uint32_t* vin[kExprMaxInputs];
    int32_t off[kExprMaxInputs];
    double* out; uint32_t* vout;
    int64_t len; int64_t tile0;
};

template <int F>
__device__ __forceinline__ double expr_unary(double x) {
    if constexpr (F == 0) return fabs(x);
    else if constexpr (F == 1) return sin(x);
    else if constexpr (F == 2) return cos(x);
    else if constexpr (F == 3) return tan(x);
    else if constexpr (F == 4) return acos(x);
    else if constexpr (F == 5) return asin(x);
    else if constexpr (F == 6) return atan(x);
    else if constexpr (F == 7) return cbrt(x);
    else if constexpr (F == 8) return ceil(x);
    else if constexpr (F == 9) return cosh(x);
    else if constexpr (F == 10) return __dmul_rn(x, 180.0 / 3.14159265358979323846264338327950288);
    else if constexpr (F == 11) return exp(x);
    else if constexpr (F == 12) return expm1(x);
    else if constexpr (F == 13) return floor(x);
    else if constexpr (F == 14) return log10(x);
    else if constexpr (F == 15) return log2_exact(x);
    else if constexpr (F == 16) return __dmul_rn(x, 3.14159265358979323846264338327950288 / 180.0);
    else if constexpr (F == 17) return round(x);
    else if constexpr (F == 18) return sinh(x);
    else if constexpr (F == 19) return __dsqrt_rn(x);
    else return tanh(x);
}

// One warp-uniform dispatch per node, then the U x 2 elements in a straight line (the compiler interleaves the
// libm bodies like k_unary does); scalar_op semantics: a null slot gets payload 0 and the function is not run.
template <int U, int F>
__device__ __forceinline__ void expr_apply_unary(Vec<double, 2> (&acc)[U], uint32_t am) {
#pragma unroll
    for (int j = 0; j < U; j++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const double y = expr_unary<F>(acc[j].e[e]);   // computed for every lane (no divergence), selected afterwards
            acc[j].e[e] = ((am >> (j * 2 + e)) & 1u) ? y : 0.0;
        }
}
template <int U>
__device__ __forceinline__ void expr_dispatch_unary(int f, Vec<double, 2> (&acc)[U], uint32_t am) {
    switch (f) {
#define BDF_EXPR_UN(F) case F: expr_apply_unary<U, F>(acc, am); break;
        BDF_EXPR_UN(0) BDF_EXPR_UN(1) BDF_EXPR_UN(2) BDF_EXPR_UN(3) BDF_EXPR_UN(4) BDF_EXPR_UN(5) BDF_EXPR_UN(6)
        BDF_EXPR_UN(7) BDF_EXPR_UN(8) BDF_EXPR_UN(9) BDF_EXPR_UN(10) BDF_EXPR_UN(11) BDF_EXPR_UN(12) BDF_EXPR_UN(13)
        BDF_EXPR_UN(14) BDF_EXPR_UN(15) BDF_EXPR_UN(16) BDF_EXPR_UN(17) BDF_EXPR_UN(18) BDF_EXPR_UN(19)
#undef BDF_EXPR_UN
        default: expr_apply_unary<U, 20>(acc, am); break;
    }
}

// Shared-memory staging.  The operands of the accumulator machine live in shared memory, laid out
// [slot][j][thread] as 16-byte pairs (conflict-free; every thread only ever touches its own entries, so no CTA
// barrier is needed): the input tiles arrive there by cp.async, which keeps n_inputs x U x 16 B per thread in flight
// WITHOUT holding a register per byte -- a register-resident version (6 inputs + 2 temporaries + libm) needed 90-128
// registers, ran 2 CTAs/SM and was far from the roofline on a plain fused add; the loads in flight, not the interpreter, were
// the limit.  Validity bits travel as one packed word per [slot][thread] (bit j*2+e).
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
    const unsigned saddr = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(saddr), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async8(void* smem_dst, const void* gsrc) {
    const unsigned saddr = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"(saddr), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
    const unsigned saddr = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(saddr), "l"(gsrc) : "memory");
}
// The two elements a lane staged for one step, as doubles.  Non-Float64 inputs were staged as raw bytes (2 x width in
// the low bytes of the 16-byte slot) and are converted here: the infallible `as f64` of Function::Cast to Float64.
__device__ __forceinline__ Vec<double, 2> expr_as_f64(int t, const Vec<double, 2>& raw) {
    if (t == T_F64) return raw;
    const unsigned long long lo = (unsigned long long)__double_as_longlong(raw.e[0]), hi = (unsigned long long)__double_as_longlong(raw.e[1]);
    const uint32_t w0 = (uint32_t)lo, w1 = (uint32_t)(lo >> 32);
    Vec<double, 2> r;
    switch (t) {
        case T_I64: r.e[0] = (double)(long long)lo; r.e[1] = (double)(long long)hi; break;
        case T_U64: r.e[0] = (double)lo; r.e[1] = (double)hi; break;
        case T_F32: r.e[0] = (double)__uint_as_float(w0); r.e[1] = (double)__uint_as_float(w1); break;
        case T_I32: r.e[0] = (double)(int)w0; r.e[1] = (double)(int)w1; break;
        case T_U32: r.e[0] = (double)w0; r.e[1] = (double)w1; break;
        case T_I16: r.e[0] = (double)(short)(w0 & 0xffffu); r.e[1] = (double)(short)(w0 >> 16); break;
        case T_U16: r.e[0] = (double)(w0 & 0xffffu); r.e[1] = (double)(w0 >> 16); break;
        case T_I8: r.e[0] = (double)(signed char)(w0 & 0xffu); r.e[1] = (double)(signed char)((w0 >> 8) & 0xffu); break;
        default: r.e[0] = (double)(w0 & 0xffu); r.e[1] = (double)((w0 >> 8) & 0xffu); break;
    }
    return r;
}
__device__ __forceinline__ double expr_load1(int t, const void* __restrict__ p, int64_t i) {
    switch (t) {
        case T_F64: return ((const double*)p)[i];
        case T_I64: return (double)((const long long*)p)[i];
        case T_U64: return (double)((const unsigned long long*)p)[i];
        case T_F32: return (double)((const float*)p)[i];
        case T_I32: return (double)((const int*)p)[i];
        case T_U32: return (double)((const unsigned*)p)[i];
        case T_I16: return (double)((const short*)p)[i];
        case T_U16: return (double)((const unsigned short*)p)[i];
        case T_I8: return (double)((const signed char*)p)[i];
        default: return (double)((const unsigned char*)p)[i];
    }
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;\n" ::: "memory");
}

// l OP r for every element; validity AND; DivideByZero on a zero divisor in a slot valid for this node.
template <int U, int OP>
__device__ __forceinline__ void expr_binop(Vec<double, 2> (&out)[U], const Vec<double, 2> (&l)[U], const Vec<double, 2> (&r)[U], uint32_t ok, bool& divzero) {
#pragma unroll
    for (int j = 0; j < U; j++)
#pragma unroll
        for (int e = 0; e < 2; e++) {
            const double a = l[j].e[e], b = r[j].e[e];
            const bool v = (ok >> (j * 2 + e)) & 1u;
            double q;
            if constexpr (OP == 0) q = __dadd_rn(a, b);
            else if constexpr (OP == 1) q = __dsub_rn(a, b);
            else if constexpr (OP == 2) q = __dmul_rn(a, b);
            else if constexpr (OP == 3) { divzero |= v && (b == 0.0); q = __ddiv_rn(a, v ? b : 1.0); }
            else if constexpr (OP == 4) { const double y = atan2(a, b); q = v ? y : 0.0; }
            else if constexpr (OP == 5) { const double y = hypot_exact(a, b); q = v ? y : 0.0; }
            else { const double y = __ddiv_rn(log(a), log(b)); q = v ? y : 0.0; }
            out[j].e[e] = q;
        }
}

template <int U>
__device__ __forceinline__ void expr_dispatch(int op, Vec<double, 2> (&out)[U], const Vec<double, 2> (&l)[U], const Vec<double, 2> (&r)[U], uint32_t ok, bool& divzero) {
    switch (op) {
        case 0: expr_binop<U, 0>(out, l, r, ok, divzero); break;
        case 1: expr_binop<U, 1>(out, l, r, ok, divzero); break;
        case 2: expr_binop<U, 2>(out, l, r, ok, divzero); break;
        case 3: expr_binop<U, 3>(out, l, r, ok, divzero); break;
        case 4: expr_binop<U, 4>(out, l, r, ok, divzero); break;
        case 5: expr_binop<U, 5>(out, l, r, ok, divzero); break;
        default: expr_binop<U, 6>(out, l, r, ok, divzero); break;
    }
}

// AGG: also fold sum/count of the RESULT column into one partial per tile (k_finish folds them, like K5); the result
// column itself is optional then (d.out == nullptr: aggregate only, nothing is written but the partials).
// TYPED: some input column is not Float64: its raw bytes are staged and converted to doubles in place (`as f64`) before
// the node loop.  The all-Float64 instantiation carries none of that code (one kernel for both slowed the Float64 chain:
// 64 registers spilled in the node loop).
template <int U, int MINB, bool AGG, bool TYPED>
__global__ void __launch_bounds__(kThreads, MINB)
k_expr(const ExprDesc* __restrict__ descs, int n_chunks, const ExprProg prog, uint32_t* __restrict__ warp_counts, int* __restrict__ flags,
       AggDev* __restrict__ tile_partials) {
    constexpr int E = 2;
    constexpr int TILE = kThreads * U * E;
    constexpr uint32_t ALL = (1u << (U * E)) - 1u;
    extern __shared__ __align__(16) unsigned char expr_smem[];
    const int ni = prog.n_inputs;
    const int tid = threadIdx.x;
    Vec<double, 2>* sv = reinterpret_cast<Vec<double, 2>*>(expr_smem);                                   // [slot][j][tid]
    uint32_t* sm = reinterpret_cast<uint32_t*>(expr_smem + (size_t)prog.n_slots * U * kThreads * 16);   // [slot][tid]

    const int64_t tile = blockIdx.x;
    const int c = (n_chunks == 1) ? 0 : find_chunk(descs, n_chunks, tile);
    const ExprDesc& d = descs[c];
    const int64_t len = d.len;
    const int64_t base = (tile - d.tile0) * TILE;
    double* __restrict__ po = d.out;
    uint32_t* __restrict__ vo = d.vout;
    const bool full = base + TILE <= len;
    const int64_t e_first = base + (int64_t)tid * E;

    if (full) {
        // All descriptor fields first (independent loads, one latency), then every copy, then the validity words:
        // a rolled loop here serialises n_inputs descriptor->copy round trips before the tile is in flight.
        const char* in[kExprMaxInputs];
        const uint32_t* vin[kExprMaxInputs];
        int32_t off[kExprMaxInputs];
#pragma unroll
        for (int i = 0; i < kExprMaxInputs; i++) { in[i] = (const char*)d.in[i]; vin[i] = d.vin[i]; off[i] = d.off[i]; }
#pragma unroll
        for (int i = 0; i < kExprMaxInputs; i++)
            if (i < ni) {
                const int w = TYPED ? dtype_width(prog.in_dtype[i]) : 8;   // warp-uniform
#pragma unroll
                for (int j = 0; j < U; j++) {
                    void* dst = &sv[(i * U + j) * kThreads + tid];
                    const char* src = in[i] + (e_first + (int64_t)j * kThreads * E) * w;
                    if (w == 8) cp_async16(dst, src);
                    else if (w == 4) cp_async8(dst, src);
                    else if (w == 2) cp_async4(dst, src);
                    else *reinterpret_cast<uint16_t*>(dst) = ld_stream2(src);
                }
            }
        asm volatile("cp.async.commit_group;\n" ::: "memory");
#pragma unroll
        for (int i = 0; i < kExprMaxInputs; i++)
            if (i < ni) {
                uint32_t m = ALL;
                if (vin[i]) {
                    MaskRaw<E, U> r;
                    mask_issue<E, U>(r, vin[i], off[i] + e_first, (int64_t)kThreads * E);
                    m = 0;
#pragma unroll
                    for (int j = 0; j < U; j++) m |= mask_get<E, U>(r, j) << (j * E);
                }
                sm[i * kThreads + tid] = m;
            }
        cp_async_wait_all();
        if constexpr (TYPED) {   // raw bytes -> doubles, in place, once per tile (every thread converts the slots it staged itself)
#pragma unroll 1
            for (int i = 0; i < ni; i++) {
                const int t = prog.in_dtype[i];
                if (t == T_F64) continue;
#pragma unroll
                for (int j = 0; j < U; j++) {
                    Vec<double, 2>* slot = &sv[(i * U + j) * kThreads + tid];
                    *slot = expr_as_f64(t, *slot);
                }
            }
        }
    } else {
#pragma unroll 1
        for (int i = 0; i < ni; i++) {
            uint32_t m = 0;
#pragma unroll
            for (int j = 0; j < U; j++) {
                const int64_t e0 = e_first + (int64_t)j * kThreads * E;
                uint32_t in_range = tail_mask<E>(e0, len);
                Vec<double, 2> x;
                x.e[0] = 0.0; x.e[1] = 0.0;
                if (in_range) {
#pragma unroll
                    for (int e = 0; e < E; e++) if ((in_range >> e) & 1u) x.e[e] = expr_load1(TYPED ? (int)prog.in_dtype[i] : (int)T_F64, d.in[i], e0 + e);
                    if (d.vin[i]) in_range &= load_bits<E>(d.vin[i], d.off[i] + e0);
                }
                sv[(i * U + j) * kThreads + tid] = x;
                m |= in_range << (j * E);
            }
            sm[i * kThreads + tid] = m;
        }
    }

    Vec<double, 2> acc[U];
    uint32_t am = 0;
#pragma unroll
    for (int j = 0; j < U; j++) { acc[j].e[0] = 0.0; acc[j].e[1] = 0.0; }
    bool divzero = false;
#pragma unroll 1
    for (int k = 0; k < prog.n_ins; k++) {
        const int op = prog.op[k], src = prog.src[k];
        if (op >= XI_UN) {
            expr_dispatch_unary<U>(op - XI_UN, acc, am);
        } else if (op == XI_STORE) {
#pragma unroll
            for (int j = 0; j < U; j++) sv[(src * U + j) * kThreads + tid] = acc[j];
            sm[src * kThreads + tid] = am;
        } else {
            Vec<double, 2> o[U];
            uint32_t om = am;
            if (src == kOperandAcc) {
#pragma unroll
                for (int j = 0; j < U; j++) o[j] = acc[j];
            } else {
#pragma unroll
                for (int j = 0; j < U; j++) o[j] = sv[(src * U + j) * kThreads + tid];
                om = sm[src * kThreads + tid];
            }
            if (op == XI_LOAD) {
#pragma unroll
                for (int j = 0; j < U; j++) acc[j] = o[j];
                am = om;
            } else {
                const uint32_t ok = am & om;
                if (op >= XI_RBIN) expr_dispatch<U>(op - XI_RBIN, acc, o, acc, ok, divzero);
                else expr_dispatch<U>(op, acc, acc, o, ok, divzero);
                am = ok;
            }
        }
    }

    unsigned int nvalid = 0;
    FusedAgg<double> agg;
    if constexpr (AGG) agg.init();
#pragma unroll
    for (int j = 0; j < U; j++) {
        const int64_t e0 = e_first + (int64_t)j * kThreads * E;
        const uint32_t in_range = full ? 3u : tail_mask<E>(e0, len);
        const uint32_t okbits = (am >> (j * E)) & in_range;
        Vec<double, E> r;
#pragma unroll
        for (int e = 0; e < E; e++) {
            r.e[e] = ((okbits >> e) & 1u) ? acc[j].e[e] : 0.0;
            if constexpr (AGG) agg.add(r.e[e], (okbits >> e) & 1u, 0ull);
        }
        if (po) {
            if (full) r.store(po + e0);
            else {
#pragma unroll
                for (int e = 0; e < E; e++) if ((in_range >> e) & 1u) po[e0 + e] = r.e[e];
            }
        }
        if (vo) store_bits<E>(vo, e0, okbits, in_range != 0);
        if (vo || AGG) nvalid += __popc(okbits);
    }
    if (vo || AGG) {
        const unsigned int wvalid = __reduce_add_sync(0xffffffffu, nvalid);
        if ((threadIdx.x & 31) == 0 && vo) warp_counts[(int64_t)blockIdx.x * kWarpsPerCta + (threadIdx.x >> 5)] = wvalid;
        if constexpr (AGG) {   // same fixed fold as K5: xor-shuffle tree per warp, warp 0 folds the 8 warp results in order
            __shared__ unsigned int s_cnt[kWarpsPerCta];
            __shared__ FusedAgg<double> s_agg[kWarpsPerCta];
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) agg.merge_shfl(o);
            if ((threadIdx.x & 31) == 0) { s_cnt[threadIdx.x >> 5] = wvalid; s_agg[threadIdx.x >> 5] = agg; }
            __syncthreads();
            if (threadIdx.x == 0) {
                FusedAgg<double> t = s_agg[0];
                unsigned long long total = s_cnt[0];
#pragma unroll
                for (int w = 1; w < kWarpsPerCta; w++) { t.merge(s_agg[w]); total += s_cnt[w]; }
                t.store(&tile_partials[blockIdx.x], total);
            }
        }
    }
    if (divzero) atomicOr(flags, 1);
}

// ---- EXPERIMENT (not the default, see launch_expr): the all-Float64 chain with bulk asynchronous copies (1-D TMA) -------------
// k_expr above loads a tile, waits, computes: loads and math of ONE CTA never overlap, only the 3 CTAs of an SM overlap each
// other.  Here a CTA walks its tiles in HALF tiles (1024 rows = 8 KiB per
// input) through two shared-memory stages: while the warps interpret the program over stage s, ONE thread has already asked the
// copy engine for the next half tile into stage s ^ 1 (`cp.async.bulk.shared.global`, UBLKCP in SASS, completion counted in
// bytes on an mbarrier), so no lane spends issue slots on 16-byte LDGSTS and the next tile is always in flight.  The layout of a
// stage is the one k_expr uses ([slot][j][thread] 16-byte pairs == the half tile's rows in order), so a bulk copy of
// U * 256 * 16 bytes per input drops in.  Partial half tiles at the end of a chunk are filled by the threads themselves.
constexpr int kBulkU = 2;   // half tile = 256 threads x 2 vectors x 2 rows = 1024 rows

__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
    const unsigned addr = (unsigned)__cvta_generic_to_shared(bar);
    unsigned done = 0;
    while (!done) {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(done) : "r"(addr), "r"(parity) : "memory");
    }
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gsrc), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar)) : "memory");
}

template <bool AGG>
__global__ void __launch_bounds__(kThreads, 2)
k_expr_bulk(const ExprDesc* __restrict__ descs, int n_chunks, long long total_tiles, const ExprProg prog, uint32_t* __restrict__ warp_counts,
            int* __restrict__ flags, AggDev* __restrict__ tile_partials) {
    constexpr int U = kBulkU, E = 2;
    constexpr int HALF = kThreads * U * E;             // rows per half tile
    constexpr int TILE = kThreads * kExprUnroll * E;   // rows per tile, as the host numbers them
    constexpr int SLOT = U * kThreads;                 // 16-byte pairs per slot
    constexpr uint32_t ALL = (1u << (U * E)) - 1u;
    extern __shared__ __align__(128) unsigned char expr_smem[];
    const int ni = prog.n_inputs, nt = prog.n_slots - ni;
    const int tid = threadIdx.x;
    Vec<double, 2>* stage[2];
    stage[0] = reinterpret_cast<Vec<double, 2>*>(expr_smem);
    stage[1] = stage[0] + (size_t)ni * SLOT;
    Vec<double, 2>* temps = stage[1] + (size_t)ni * SLOT;
    uint32_t* sm = reinterpret_cast<uint32_t*>(temps + (size_t)nt * SLOT);   // [slot][thread] validity bits of the current half tile
    unsigned long long* bar = reinterpret_cast<unsigned long long*>(sm + (size_t)prog.n_slots * kThreads);
    int* s_full = reinterpret_cast<int*>(bar + 2);                           // was stage s filled by the copy engine?
    __shared__ unsigned int s_cnt[kWarpsPerCta];
    __shared__ FusedAgg<double> s_agg[kWarpsPerCta];

    if (tid == 0) {
        mbar_init(&bar[0], 1); mbar_init(&bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const long long my_tiles = (total_tiles - (long long)blockIdx.x + (long long)gridDim.x - 1) / (long long)gridDim.x;   // blockIdx.x < total_tiles
    const long long n_half = my_tiles * 2;
    auto tile_of = [&](long long q) { return (long long)blockIdx.x + (q >> 1) * (long long)gridDim.x; };
    // thread 0: start the copies of half tile q into stage s (or note that the threads must fill it themselves)
    auto issue = [&](long long q, int s) {
        const long long tile = tile_of(q);
        const int c = (n_chunks == 1) ? 0 : find_chunk(descs, n_chunks, tile);
        const ExprDesc& d = descs[c];
        const long long base = (tile - d.tile0) * TILE + (q & 1) * HALF;
        const bool full = base + HALF <= d.len;
        s_full[s] = full ? 1 : 0;
        if (full) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the stage was read through the generic proxy a moment ago
            mbar_expect_tx(&bar[s], (unsigned)(ni * SLOT * 16));
            for (int i = 0; i < ni; i++) bulk_g2s(stage[s] + (size_t)i * SLOT, (const char*)d.in[i] + base * 8, SLOT * 16, &bar[s]);
        }
    };
    if (tid == 0 && n_half > 0) issue(0, 0);
    __syncthreads();

    unsigned phase[2] = {0u, 0u};
    unsigned int nvalid = 0;
    FusedAgg<double> agg;
    if constexpr (AGG) agg.init();
    bool divzero = false;
#pragma unroll 1
    for (long long q = 0; q < n_half; q++) {
        const int s = (int)(q & 1);
        if (tid == 0 && q + 1 < n_half) issue(q + 1, s ^ 1);   // stage s ^ 1 was released by the barrier that ended iteration q - 1
        const long long tile = tile_of(q);
        const int c = (n_chunks == 1) ? 0 : find_chunk(descs, n_chunks, tile);
        const ExprDesc& d = descs[c];
        const long long len = d.len;
        const long long base = (tile - d.tile0) * TILE + (q & 1) * HALF;
        const long long e_first = base + (long long)tid * E;
        double* __restrict__ po = d.out;
        uint32_t* __restrict__ vo = d.vout;
        const bool full = s_full[s] != 0;
        Vec<double, 2>* in_stage = stage[s];
        auto slot_ptr = [&](int slot) { return slot < ni ? in_stage + (size_t)slot * SLOT : temps + (size_t)(slot - ni) * SLOT; };
        if (full) {
            // validity words first (they are in flight while the thread waits for the copy engine)
            for (int i = 0; i < ni; i++) {
                uint32_t m = ALL;
                const uint32_t* vin = d.vin[i];
                if (vin) {
                    MaskRaw<E, U> r;
                    mask_issue<E, U>(r, vin, d.off[i] + e_first, (int64_t)kThreads * E);
                    m = 0;
#pragma unroll
                    for (int j = 0; j < U; j++) m |= mask_get<E, U>(r, j) << (j * E);
                }
                sm[i * kThreads + tid] = m;
            }
            mbar_wait(&bar[s], phase[s]);
            phase[s] ^= 1u;
        } else {
#pragma unroll 1
            for (int i = 0; i < ni; i++) {
                uint32_t m = 0;
#pragma unroll
                for (int j = 0; j < U; j++) {
                    const long long e0 = e_first + (long long)j * kThreads * E;
                    uint32_t in_range = tail_mask<E>(e0, len);
                    Vec<double, 2> x;
                    x.e[0] = 0.0; x.e[1] = 0.0;
                    if (in_range) {
#pragma unroll
                        for (int e = 0; e < E; e++) if ((in_range >> e) & 1u) x.e[e] = ((const double*)d.in[i])[e0 + e];
                        if (d.vin[i]) in_range &= load_bits<E>(d.vin[i], d.off[i] + e0);
                    }
                    in_stage[(i * U + j) * kThreads + tid] = x;
                    m |= in_range << (j * E);
                }
                sm[i * kThreads + tid] = m;
            }
        }

        Vec<double, 2> acc[U];
        uint32_t am = 0;
#pragma unroll
        for (int j = 0; j < U; j++) { acc[j].e[0] = 0.0; acc[j].e[1] = 0.0; }
#pragma unroll 1
        for (int k = 0; k < prog.n_ins; k++) {
            const int op = prog.op[k], src = prog.src[k];
            if (op >= XI_UN) {
                expr_dispatch_unary<U>(op - XI_UN, acc, am);
            } else if (op == XI_STORE) {
                Vec<double, 2>* t = slot_ptr(src);
#pragma unroll
                for (int j = 0; j < U; j++) t[j * kThreads + tid] = acc[j];
                sm[src * kThreads + tid] = am;
            } else {
                Vec<double, 2> o[U];
                uint32_t om = am;
                if (src == kOperandAcc) {
#pragma unroll
                    for (int j = 0; j < U; j++) o[j] = acc[j];
                } else {
                    const Vec<double, 2>* t = slot_ptr(src);
#pragma unroll
                    for (int j = 0; j < U; j++) o[j] = t[j * kThreads + tid];
                    om = sm[src * kThreads + tid];
                }
                if (op == XI_LOAD) {
#pragma unroll
                    for (int j = 0; j < U; j++) acc[j] = o[j];
                    am = om;
                } else {
                    const uint32_t ok = am & om;
                    if (op >= XI_RBIN) expr_dispatch<U>(op - XI_RBIN, acc, o, acc, ok, divzero);
                    else expr_dispatch<U>(op, acc, acc, o, ok, divzero);
                    am = ok;
                }
            }
        }

#pragma unroll
        for (int j = 0; j < U; j++) {
            const long long e0 = e_first + (long long)j * kThreads * E;
            const uint32_t in_range = full ? 3u : tail_mask<E>(e0, len);
            const uint32_t okbits = (am >> (j * E)) & in_range;
            Vec<double, E> r;
#pragma unroll
            for (int e = 0; e < E; e++) {
                r.e[e] = ((okbits >> e) & 1u) ? acc[j].e[e] : 0.0;
                if constexpr (AGG) agg.add(r.e[e], (okbits >> e) & 1u, 0ull);
            }
            if (po) {
                if (full) r.store(po + e0);
                else {
#pragma unroll
                    for (int e = 0; e < E; e++) if ((in_range >> e) & 1u) po[e0 + e] = r.e[e];
                }
            }
            if (vo) store_bits<E>(vo, e0, okbits, in_range != 0);
            if (vo || AGG) nvalid += __popc(okbits);
        }
        __syncthreads();   // every warp is done with stage s (and with the temporaries): thread 0 may refill it next iteration

        if (q & 1) {       // second half: the host's tile is complete -> its per-warp valid counts and its aggregate partial
            if (vo || AGG) {
                const unsigned int wvalid = __reduce_add_sync(0xffffffffu, nvalid);
                if ((tid & 31) == 0 && vo) warp_counts[tile * kWarpsPerCta + (tid >> 5)] = wvalid;
                if constexpr (AGG) {
#pragma unroll
                    for (int o = 16; o > 0; o >>= 1) agg.merge_shfl(o);
                    if ((tid & 31) == 0) { s_cnt[tid >> 5] = wvalid; s_agg[tid >> 5] = agg; }
                    __syncthreads();
                    if (tid == 0) {
                        FusedAgg<double> t = s_agg[0];
                        unsigned long long total = s_cnt[0];
#pragma unroll
                        for (int w = 1; w < kWarpsPerCta; w++) { t.merge(s_agg[w]); total += s_cnt[w]; }
                        t.store(&tile_partials[tile], total);
                    }
                    agg.init();
                }
            }
            nvalid = 0;
        }
    }
    if (divzero) atomicOr(flags, 1);
}

static size_t expr_bulk_smem(const ExprProg& p) {
    const size_t slot = (size_t)kBulkU * kThreads * 16;
    return (size_t)(2 * p.n_inputs + (p.n_slots - p.n_inputs)) * slot + (size_t)p.n_slots * kThreads * 4 + 2 * 8 + 2 * 4 + 16;
}

template <bool AGG>
static cudaError_t launch_expr_bulk(const ExprDesc* dd, int n_chunks, int64_t tiles, const ExprProg& pp, uint32_t* warp_counts, int* flags,
                                    AggDev* tile_partials, int sm_count, cudaStream_t s) {
    constexpr int kMaxSmem = (2 * kExprMaxInputs + kExprMaxTemps) * kBulkU * kThreads * 16 + (kExprMaxInputs + kExprMaxTemps) * kThreads * 4 + 64;
    static const cudaError_t attr = cudaFuncSetAttribute(k_expr_bulk<AGG>, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxSmem);
    if (attr != cudaSuccess) return attr;
    const size_t smem = expr_bulk_smem(pp);
    int per_sm = (int)((size_t)(227 * 1024) / (smem + 1024));
    per_sm = per_sm < 1 ? 1 : (per_sm > 2 ? 2 : per_sm);   // 96-104 registers: two CTAs per SM
    int64_t grid = (int64_t)sm_count * per_sm;
    if (grid > tiles) grid = tiles;
    k_expr_bulk<AGG><<<(unsigned)grid, kThreads, smem, s>>>(dd, n_chunks, tiles, pp, warp_counts, flags, tile_partials);
    return cudaGetLastError();
}

int expr_tile_elems() { return kThreads * kExprUnroll * 2; }
int expr_max_inputs() { return kExprMaxInputs; }
int expr_max_nodes() { return kExprMaxNodes; }
size_t expr_desc_size() { return sizeof(ExprDesc); }
size_t expr_prog_size() { return sizeof(ExprProg); }
void expr_prog_stats(const void* prog, int* n_instructions, int* n_temporaries) {
    const ExprProg* p = (const ExprProg*)prog;
    *n_instructions = p->n_ins;
    *n_temporaries = p->n_slots - p->n_inputs;
}

void fill_expr_desc(void* base, int64_t i, int n_inputs, const void* const* in, const uint32_t* const* vin, const int32_t* off, double* out,
                    uint32_t* vout, int64_t len, int64_t tile0) {
    ExprDesc* d = (ExprDesc*)base + i;
    for (int k = 0; k < kExprMaxInputs; k++) {
        d->in[k] = k < n_inputs ? in[k] : nullptr;
        d->vin[k] = k < n_inputs ? vin[k] : nullptr;
        d->off[k] = k < n_inputs ? off[k] : 0;
    }
    d->out = out; d->vout = vout; d->len = len; d->tile0 = tile0;
}

// ---- host: straight-line DAG -> accumulator program ------------------------------------------------------------
// Slots 0..ni-1 are inputs, slot ni+k is node k (validated by the caller: operands refer to earlier slots only).
// Every node is evaluated exactly once (the set of divide nodes that can raise is the materialised chain's), so a
// node nobody uses is rejected rather than dropped.  A node used more than once, and the first-evaluated operand of
// a node whose operands are both intermediate, live in one of two temporaries.
// Returns 0 ok, 1 dead node, 2 needs more than two live temporaries, 3 program too long.
namespace {
struct ExprCompiler {
    int ni, nn;
    const int *op, *a, *b;
    int uses[kExprMaxInputs + kExprMaxNodes];
    int where[kExprMaxInputs + kExprMaxNodes];   // node slots: operand code of the temporary holding it, or -1
    bool busy[2] = {false, false};
    int err = 0;
    ExprProg* p;

    void emit(int o, int s) {
        if (p->n_ins >= kExprMaxIns) { err = err ? err : 3; return; }
        p->op[p->n_ins] = (uint8_t)o; p->src[p->n_ins] = (uint8_t)s; p->n_ins++;
    }
    bool leaf(int s) const { return s < ni || where[s] >= 0; }
    int operand(int s) const { return s < ni ? s : where[s]; }
    void consume(int s) {
        if (s < ni) return;
        if (--uses[s] == 0 && where[s] >= 0) { busy[where[s] - ni] = false; where[s] = -1; }
    }
    void hold(int s) {   // keep the accumulator's value of slot s in a temporary
        const int tmp = !busy[0] ? 0 : (!busy[1] ? 1 : -1);
        if (tmp < 0) { err = err ? err : 2; return; }
        busy[tmp] = true; where[s] = ni + tmp;
        if (ni + tmp + 1 > p->n_slots) p->n_slots = ni + tmp + 1;
        emit(XI_STORE, ni + tmp);
    }
    void eval(int s) {   // slot s -> accumulator; consumes one reference to s
        if (err) return;
        if (leaf(s)) { emit(XI_LOAD, operand(s)); consume(s); return; }
        const int k = s - ni, o = op[k], x = a[k], y = b[k];
        if (o >= kExprUnaryBase) { eval(x); emit(XI_UN + (o - kExprUnaryBase), 0); }
        else if (x == y) { eval(x); emit(XI_BIN + o, kOperandAcc); consume(x); }
        else if (leaf(y)) { eval(x); emit(XI_BIN + o, operand(y)); consume(y); }
        else if (leaf(x)) { eval(y); emit(XI_RBIN + o, operand(x)); consume(x); }
        else { uses[y]++; eval(y); eval(x); if (!err) emit(XI_BIN + o, operand(y)); consume(y); }
        if (err) return;
        if (uses[s] > 1) hold(s);
        consume(s);
    }
};
}  // namespace

int expr_compile(int n_inputs, const int* in_dtypes, int n_nodes, const int* op, const int* a, const int* b, void* prog) {
    ExprProg* p = (ExprProg*)prog;
    for (int i = 0; i < kExprMaxInputs; i++) p->in_dtype[i] = (uint8_t)(i < n_inputs ? in_dtypes[i] : T_F64);
    ExprCompiler c{};
    c.ni = n_inputs; c.nn = n_nodes; c.op = op; c.a = a; c.b = b; c.p = p;
    p->n_inputs = n_inputs; p->n_ins = 0; p->n_slots = n_inputs;
    for (int s = 0; s < n_inputs + n_nodes; s++) { c.uses[s] = 0; c.where[s] = -1; }
    c.uses[n_inputs + n_nodes - 1] = 1;   // the result column
    for (int k = 0; k < n_nodes; k++) {
        c.uses[a[k]]++;
        if (op[k] < kExprUnaryBase) c.uses[b[k]]++;
    }
    for (int k = 0; k < n_nodes; k++) if (c.uses[n_inputs + k] == 0) return 1;
    c.eval(n_inputs + n_nodes - 1);
    return c.err;
}

size_t expr_smem_bytes(const ExprProg& p, int unroll) { return (size_t)p.n_slots * kThreads * ((size_t)unroll * 16 + 4); }

template <int U, int MINB, bool AGG, bool TYPED>
static cudaError_t launch_expr_u(const ExprDesc* dd, int n_chunks, int64_t tiles, const ExprProg& pp, uint32_t* warp_counts, int* flags,
                                 AggDev* tile_partials, cudaStream_t s) {
    static const cudaError_t attr = cudaFuncSetAttribute(k_expr<U, MINB, AGG, TYPED>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                         (int)((kExprMaxInputs + kExprMaxTemps) * kThreads * (U * 16 + 4)));
    if (attr != cudaSuccess) return attr;
    k_expr<U, MINB, AGG, TYPED><<<(unsigned)tiles, kThreads, expr_smem_bytes(pp, U), s>>>(dd, n_chunks, pp, warp_counts, flags, tile_partials);
    return cudaGetLastError();
}

// tile_partials != nullptr: also one AggDev per tile with sum/count of the result (fold with launch_finish(is_float = true)).
cudaError_t launch_expr(const void* descs, int n_chunks, int64_t tiles, const void* prog, uint32_t* warp_counts, int* flags,
                        AggDev* tile_partials, cudaStream_t s) {
    if (tiles <= 0) return cudaSuccess;
    if (tiles > 0x7fffffffLL) return cudaErrorInvalidConfiguration;
    const ExprDesc* dd = (const ExprDesc*)descs;
    const ExprProg& pp = *(const ExprProg*)prog;
    bool typed = false;
    for (int i = 0; i < pp.n_inputs; i++) typed = typed || pp.in_dtype[i] != T_F64;
    // Off by default: slower than k_expr when it was measured (arithmetic chain, sin chain and a + b at 1e8 rows; not
    // re-measured on H100) -- two CTAs of 96-104 registers per SM, one block barrier
    // per half tile and a single stage of look-ahead (32-64 KiB in flight per SM) lose to three independent cp.async CTAs.  Kept
    // for the next iteration (deeper pipeline / warp-specialised producer); BDF_EXPR_BULK=1 selects it, results are identical.
    static const bool use_bulk = [] { const char* e = getenv("BDF_EXPR_BULK"); return e && e[0] == '1'; }();
    if (!typed && use_bulk) {
        int dev = 0, sms = 132;
        if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        if (tile_partials) return launch_expr_bulk<true>(dd, n_chunks, tiles, pp, warp_counts, flags, tile_partials, sms, s);
        return launch_expr_bulk<false>(dd, n_chunks, tiles, pp, warp_counts, flags, nullptr, sms, s);
    }
    if (tile_partials) {
        if (typed) return launch_expr_u<kExprUnroll, kExprMinCtas, true, true>(dd, n_chunks, tiles, pp, warp_counts, flags, tile_partials, s);
        return launch_expr_u<kExprUnroll, kExprMinCtas, true, false>(dd, n_chunks, tiles, pp, warp_counts, flags, tile_partials, s);
    }
    if (typed) return launch_expr_u<kExprUnroll, kExprMinCtas, false, true>(dd, n_chunks, tiles, pp, warp_counts, flags, nullptr, s);
    return launch_expr_u<kExprUnroll, kExprMinCtas, false, false>(dd, n_chunks, tiles, pp, warp_counts, flags, nullptr, s);
}

}  // namespace bdf
