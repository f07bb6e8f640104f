// runtime.cu -- host runtime and C ABI of libb200df.so (see include/b200df.h for the contract).
//
// One bdf_ctx per GPU (one process per GPU).  Three non-blocking streams: h2d (uploads), compute (all
// kernels, all stream-ordered allocations), d2h (downloads).  Columns are device-resident lists of Arrow
// chunks carved out of two arenas (values, validity).  Chunks become ready in *groups*; every group has
// an event, so the kernels of group g run while group g+1 is still crossing PCIe and group g-1 is
// already on its way back.  When all inputs are already resident an operator is ONE batched launch over
// every chunk of the column.
#include <algorithm>
#include <atomic>
#include <cerrno>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <memory>
#include <mutex>
#include <new>
#include <deque>
#include <limits>
#include <functional>
#include <sched.h>
#include <fcntl.h>
#include <locale.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/b200df.h"
#include "common.cuh"
#include "comm.cuh"
#include "moments.cuh"
#include "dist.cuh"
#include "json_parse.cuh"
#include "json_format.cuh"
#define PQ_HOST_PLAN
#include "parquet_decode.cuh"
#define PQ_HOST_WRITE
#include "parquet_encode.cuh"
#include "ipc_schema.cuh"

using namespace bdf;

// ---------------------------------------------------------------------------------------------------
// errors

static thread_local std::string g_err;

static int fail(int status, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_err = buf;
    return status;
}

namespace bdf {
int set_error(int status, const char* msg) {   // for the host-only translation units of the library (ipc.cu)
    g_err = msg;
    return status;
}
}  // namespace bdf

static int cuda_status(cudaError_t e) { return e == cudaErrorMemoryAllocation ? BDF_OOM : BDF_CUDA; }

// Set by the communicator layer (comm.cu reports NCCL failures as text + cudaErrorUnknown): turns the next
// fail_cuda into BDF_NCCL.
static thread_local std::string g_nccl_err;
// Reports a failed CUDA call and clears the runtime's last error, so that the next call does not see it again.
static int fail_cuda(cudaError_t e, const char* what) {
    cudaGetLastError();
    if (!g_nccl_err.empty()) {
        const std::string m = g_nccl_err;
        g_nccl_err.clear();
        return fail(BDF_NCCL, "%s: %s", what, m.c_str());
    }
    return fail(cuda_status(e), "%s failed: %s", what, cudaGetErrorString(e));
}

#define CK(call)                                                                                       \
    do {                                                                                               \
        cudaError_t _e = (call);                                                                       \
        if (_e != cudaSuccess) {                                                                       \
            cudaGetLastError();                                                                        \
            return fail(cuda_status(_e), "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
        }                                                                                              \
    } while (0)

#define TRY(expr)                  \
    do {                           \
        int _st = (expr);          \
        if (_st != BDF_OK) return _st; \
    } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---------------------------------------------------------------------------------------------------
// objects

struct Group {
    int64_t begin, end;  // chunks [begin, end)
    cudaEvent_t ev;      // chunks are complete in HBM once ev has fired
};

struct DevChunk {
    char* values;
    uint32_t* validity;  // nullptr = no bitmap
    int64_t len;
    int32_t bit_off;      // residual bit offset of the validity bitmap
    int32_t val_bit_off;  // boolean columns only: residual bit offset of the VALUES bitmap
};

struct bdf_col {
    int dtype = 0;
    int64_t total_len = 0;
    std::vector<DevChunk> chunks;
    char* arena_values = nullptr;
    char* arena_validity = nullptr;
    uint32_t* d_warp_counts = nullptr;             // valid slots per warp per tile ([tile][8]), written by the producing kernel
    int64_t tile_elems = 0;                        // tile size (elements) the producing kernel used
    std::vector<int64_t> tile0;                    // column-global first tile of each chunk (n+1 entries)
    bool counts_on_device = false;                 // d_warp_counts not yet folded into null_counts
    std::vector<int64_t> null_counts;              // -1 = unknown
    std::vector<Group> groups;
    std::vector<uint32_t> dl_counts;               // staging of d_warp_counts during a split download
    bdf_col* dl_tmp = nullptr;                     // re-aligned copy used by a split download of a sliced column
    struct StagedCopy { void* dst; const void* src; size_t bytes; };
    std::vector<StagedCopy> dl_staged;             // device->pageable-host copies carried out in download_finish
    // A column of a multi-GPU context (bdf_init_multi): the logical chunks are cut into row ranges, each range lives as one
    // chunk of a per-GPU sub-column.  Empty for the columns of a one-GPU context.
    struct Piece { int kid; int64_t local; int64_t row0, rows; };   // rows [row0, row0 + rows) of a logical chunk = chunk `local` of fparts[kid]
    std::vector<bdf_col*> fparts;                  // one sub-column per GPU (possibly without chunks)
    std::vector<std::vector<Piece>> fmap;          // per logical chunk, in row order
    std::vector<int64_t> flens;                    // logical chunk lengths
};

// Result of an aggregate that is still in flight (or done): a pinned slot + the event that guards it.
struct bdf_future {
    int n = 1;                   // number of aggregates the future carries (one per column of a multi-column call)
    int fused = 1;               // which kernel produced the keys: 1 = k_binary AGG, 2 = k_reduce (see convert_agg)
    int slot = 0;                // first index into h_agg: n records, or 2n ({AggDev, {rows, panics, chunks}}) when global
    bool global = false;         // combined across the ranks of the communicator (comm.cuh)
    int lslot = 0;               // global only: first index into d_local (the per-rank records the collective reads)
    std::vector<int> dtypes;
    std::vector<int64_t> rows;   // local rows per aggregate
    std::vector<uint32_t> panics;  // local chunks that are empty or all-null (max/min .unwrap() would panic)
    std::vector<uint32_t> chunks;  // local chunk count
    cudaEvent_t ev = nullptr;
    std::vector<bdf_future*> fparts;   // multi-GPU context: the per-GPU futures (every one yields the same, global, records)
};

struct ProfEntry {
    bdf_launch_record rec;
    cudaEvent_t e0, e1;
};

// Persistent host threads for the staged copies of PAGEABLE buffers (Arrow MutableBuffers, a mapped IPC file): a copy
// is cut into 512 KiB jobs that the workers and the calling thread pull until it is done.  (Spawning threads per 8 MiB
// slot, the first version, stopped scaling at 4 threads because the spawn/join cost was comparable to the copy.)
class CopyPool {
  public:
    explicit CopyPool(int workers) {
        for (int i = 0; i < workers; i++) th_.emplace_back([this] { work(); });
    }
    ~CopyPool() {
        { std::lock_guard<std::mutex> g(m_); stop_ = true; }
        cv_work_.notify_all();
        for (auto& t : th_) t.join();
    }
    int workers() const { return (int)th_.size(); }
    // populate: the destination may be memory nobody has touched yet (a fresh Arrow MutableBuffer): every job first asks
    // the kernel for its pages in ONE call (MADV_POPULATE_WRITE) instead of taking a fault per 4 KiB page inside the
    // copy (faster into fresh memory, benchmarks/staging_probe2.cu); a no-op for resident pages.
    static void job_copy(char* dst, const char* src, size_t n, bool populate) {
        if (populate) {
            const uintptr_t a = ((uintptr_t)dst + 4095) & ~(uintptr_t)4095, b = ((uintptr_t)dst + n) & ~(uintptr_t)4095;
            if (b > a) madvise((void*)a, b - a, 23 /* MADV_POPULATE_WRITE (Linux 5.14+); an error only means: fault as usual */);
        }
        memcpy(dst, src, n);
    }
    void copy(char* dst, const char* src, size_t n, bool populate = false) {
        constexpr size_t kJob = (size_t)512 << 10;
        if (th_.empty() || n < 2 * kJob) { job_copy(dst, src, n, populate); return; }
        run((n + kJob - 1) / kJob, [=](size_t j) { job_copy(dst + j * kJob, src + j * kJob, std::min(kJob, n - j * kJob), populate); });
    }
    // fn(0) .. fn(jobs - 1) on the workers and the calling thread; returns when all have finished.
    void run(size_t jobs, const std::function<void(size_t)>& fn) {
        std::unique_lock<std::mutex> lk(m_);
        fn_ = &fn; next_ = 0; jobs_ = jobs; done_ = 0;
        lk.unlock();
        cv_work_.notify_all();
        lk.lock();
        while (next_ < jobs_) {   // the caller works too
            const size_t j = next_++;
            lk.unlock();
            fn(j);
            lk.lock();
            done_++;
        }
        cv_done_.wait(lk, [this] { return done_ == jobs_; });
        jobs_ = 0; next_ = 0; done_ = 0; fn_ = nullptr;
    }

  private:
    void work() {
        std::unique_lock<std::mutex> lk(m_);
        for (;;) {
            cv_work_.wait(lk, [this] { return stop_ || next_ < jobs_; });
            if (stop_) return;
            const size_t j = next_++;
            const std::function<void(size_t)>* fn = fn_;
            lk.unlock();
            (*fn)(j);
            lk.lock();
            if (++done_ == jobs_) cv_done_.notify_all();
        }
    }
    std::mutex m_;
    std::condition_variable cv_work_, cv_done_;
    std::vector<std::thread> th_;
    const std::function<void(size_t)>* fn_ = nullptr;
    size_t next_ = 0, jobs_ = 0, done_ = 0;
    bool stop_ = false;
};

struct bdf_ctx {
    int device = 0;
    int sm_count = 0, cc_major = 0, cc_minor = 0;
    size_t hbm_bytes = 0;
    cudaStream_t s_compute = nullptr, s_h2d = nullptr, s_d2h = nullptr;
    cudaStream_t s_desc = nullptr;  // descriptor copies: run ahead of the compute stream, off its critical path
    cudaStream_t s_fin = nullptr;   // k_finish of fused aggregates: overlaps the next operator (highest priority)
    std::mutex mu;
    // pinned staging: descriptor ring + small result area
    char* ring = nullptr;           // pinned host side of the descriptor ring
    char* dring = nullptr;          // device side, same offsets
    size_t ring_cap = 0, ring_head = 0;
    std::vector<cudaEvent_t> ev_pool;  // recycled cudaEventDisableTiming events
    AggDev* h_agg = nullptr;        // pinned + device-mapped: kernels write results straight into it
    AggDev* h_agg_dev = nullptr;    // device-side address of h_agg
    int* h_flag = nullptr;          // pinned
    unsigned long long* h_sort_agree = nullptr;   // pinned: OR and AND of the sort keys of one criterion
    int64_t last_sort_passes = 0;
    // device scratch
    AggDev* d_partials = nullptr;       // per-CTA partials of k_reduce (compute stream only)
    size_t red_part_cap = 0;
    AggDev* d_stage2 = nullptr;         // k_finish staging for the k_reduce path
    AggDev* d_stage_many = nullptr;     // k_finish_many staging (kFinishMany x sm_count) and tickets, allocated on first use
    unsigned int* d_tickets_many = nullptr;
    unsigned int* d_ticket = nullptr;   // k_finish tickets: [0] reduce path (compute stream), [1] fused aggregates (finish stream)
    AggDev* d_stage = nullptr;          // k_finish per-CTA staging, sm_count entries
    int* d_flag = nullptr;
    int fut_next = 0;                   // ring cursor over the future half of h_agg
    struct PartBuf { AggDev* p = nullptr; size_t cap = 0; cudaEvent_t done = nullptr; bool used = false; } part[3];
    int part_next = 0;                  // per-tile partials of fused aggregates: 3 persistent buffers in rotation
    // staging for PAGEABLE host buffers: pinned slots filled/drained by a few host threads while the DMA of the
    // previous slot is in flight (cudaMemcpyAsync straight from pageable memory is a single-threaded driver copy)
    struct StageSlot { char* p = nullptr; cudaEvent_t ev = nullptr; bool busy = false; };
    std::vector<StageSlot> stage;
    int stage_next = 0;
    int copy_threads = 8;
    std::unique_ptr<CopyPool> pool;
    cudaEvent_t ev_tmp = nullptr, ev_t0 = nullptr, ev_t1 = nullptr;
    void* flush_buf = nullptr;
    size_t flush_bytes = 0;
    size_t pipeline_bytes = (size_t)32 << 20;
    bool pipeline_split = false;   // BDF_PIPELINE_SPLIT: split operators at every input group end, landed or not
    bool profiling = false;
    std::vector<ProfEntry> prof;
    std::vector<cudaEvent_t> prof_pool;   // recycled timing events
    int64_t launches = 0;
    // multi-GPU: the communicator this context is a rank of (nullptr = a lone GPU) -- comm.cuh
    Comm* comm = nullptr;
    bool collective = true;             // aggregates are combined across the ranks (every rank makes the same calls)
    AggDev* d_local = nullptr;          // per-rank aggregate records awaiting their collective (ring of kAggSlots)
    int local_next = 0;
    int64_t collectives = 0;            // grouped NCCL calls enqueued since the communicator was attached
    struct Fleet* fleet = nullptr;      // non-null: this is a multi-GPU context (bdf_init_multi); it owns no device itself
};

static constexpr int kAggSlots = 4096;

// ---------------------------------------------------------------------------------------------------
// small helpers

static constexpr int kBool = 10;  // BDF_BOOL: bit-packed boolean column (N2)

static inline size_t value_bytes(int dtype, int64_t len, int bit_off) {
    return dtype == kBool ? (size_t)((len + bit_off + 7) / 8) : (size_t)len * dtype_width(dtype);
}

static int check_dtype(int t) {
    if (t < 0 || t >= BDF_NTYPES) return fail(BDF_INVALID, "invalid dtype %d", t);
    return BDF_OK;
}

// Descriptor ring: host writes descriptors into pinned memory, one async copy moves them to the same offset
// of the device ring, kernels read them there.  No per-call allocation.
static int ring_alloc(bdf_ctx* c, size_t bytes, void** host, void** dev) {
    bytes = align_up(std::max<size_t>(bytes, 1), 256);
    if (bytes > c->ring_cap) return fail(BDF_OOM, "descriptor ring too small for %zu bytes", bytes);
    if (c->ring_head + bytes > c->ring_cap) {
        CK(cudaStreamSynchronize(c->s_desc));
        CK(cudaStreamSynchronize(c->s_compute));  // everything that read the ring has finished
        c->ring_head = 0;
    }
    *host = c->ring + c->ring_head;
    *dev = c->dring + c->ring_head;
    c->ring_head += bytes;
    return BDF_OK;
}

static cudaError_t ev_get(bdf_ctx* c, cudaEvent_t* ev) {
    if (!c->ev_pool.empty()) { *ev = c->ev_pool.back(); c->ev_pool.pop_back(); return cudaSuccess; }
    return cudaEventCreateWithFlags(ev, cudaEventDisableTiming);
}
static void ev_put(bdf_ctx* c, cudaEvent_t ev) { if (ev) c->ev_pool.push_back(ev); }

// Chunks [begin, end) of col are complete once the work enqueued on s so far has run: record that as one of its groups.
static cudaError_t record_group(bdf_ctx* c, bdf_col* col, int64_t begin, int64_t end, cudaStream_t s) {
    Group g{begin, end, nullptr};
    cudaError_t e = ev_get(c, &g.ev);
    if (e == cudaSuccess) e = cudaEventRecord(g.ev, s);
    col->groups.push_back(g);
    return e;
}
static cudaError_t finish_single_group(bdf_ctx* c, bdf_col* o) { return record_group(c, o, 0, (int64_t)o->chunks.size(), c->s_compute); }

// Copy descriptors host ring -> device ring on the descriptor stream and make the compute stream wait for
// them: the copy itself runs while the previous kernel is still busy.
static cudaError_t desc_upload(bdf_ctx* c, void* dev, const void* host, size_t bytes) {
    if (!bytes) return cudaSuccess;
    cudaError_t e = cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, c->s_desc);
    cudaEvent_t ev = nullptr;
    if (e == cudaSuccess) e = ev_get(c, &ev);
    if (e == cudaSuccess) e = cudaEventRecord(ev, c->s_desc);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(c->s_compute, ev, 0);
    ev_put(c, ev);  // the wait has captured this record; re-recording later does not affect it
    return e;
}

struct LaunchTimer {  // brackets one launch with events when profiling is on
    bdf_ctx* c;
    ProfEntry e{};
    bool on;
    LaunchTimer(bdf_ctx* ctx, int kernel, int dtype, int64_t rows, int64_t bytes) : c(ctx), on(ctx->profiling) {
        c->launches++;
        if (!on) return;
        e.rec.kernel = kernel; e.rec.dtype = dtype; e.rec.rows = rows; e.rec.bytes = bytes; e.rec.ms = 0.f;
        // timing events come from a pool (bdf_profile_read returns them): creating two events per launch cost more host time
        // than the launch itself and showed up as a few percent of the headline step at 8 GPUs
        auto take = [&](cudaEvent_t* ev) {
            if (!c->prof_pool.empty()) { *ev = c->prof_pool.back(); c->prof_pool.pop_back(); } else cudaEventCreate(ev);
        };
        take(&e.e0); take(&e.e1);
        cudaEventRecord(e.e0, c->s_compute);
    }
    ~LaunchTimer() {
        if (!on) return;
        cudaEventRecord(e.e1, c->s_compute);
        c->prof.push_back(e);
    }
};

static void col_destroy_host(bdf_ctx* c, bdf_col* col) {
    for (auto& g : col->groups) ev_put(c, g.ev);
    delete col;
}

// Free device memory of a column in stream order on the compute stream.
static void col_release(bdf_ctx* c, bdf_col* col) {
    if (!col) return;
    if (col->dl_tmp) { cudaStreamSynchronize(c->s_d2h); col_release(c, col->dl_tmp); col->dl_tmp = nullptr; }
    if (!col->dl_counts.empty()) cudaStreamSynchronize(c->s_d2h);  // a split download is still writing into it
    for (auto& g : col->groups) if (g.ev) cudaStreamWaitEvent(c->s_compute, g.ev, 0);
    if (col->arena_values) cudaFreeAsync(col->arena_values, c->s_compute);
    if (col->arena_validity) cudaFreeAsync(col->arena_validity, c->s_compute);
    if (col->d_warp_counts) cudaFreeAsync(col->d_warp_counts, c->s_compute);
    col_destroy_host(c, col);
}

// What an owner does with an object it still holds.  No drop writes g_err, so after a failure the caller reads the error of
// the step that failed.
static void drop(bdf_ctx* c, bdf_col* col) { col_release(c, col); }
static void drop(bdf_ctx* c, bdf_future* f) {   // its event goes back to the pool
    ev_put(c, f->ev);
    delete f;
}

// Owns what an operator body made until the body hands it to its caller with release(); every other exit drops it.
template <class T>
class Owned {
  public:
    explicit Owned(bdf_ctx* c, T* p = nullptr) : c_(c), p_(p) {}
    Owned(Owned&& o) noexcept : c_(o.c_), p_(o.release()) {}
    Owned& operator=(Owned&& o) noexcept {
        if (this != &o) {
            if (p_) drop(c_, p_);
            c_ = o.c_;
            p_ = o.release();
        }
        return *this;
    }
    ~Owned() { if (p_) drop(c_, p_); }
    T* get() const { return p_; }
    T* operator->() const { return p_; }
    T** out() { return &p_; }   // where a maker writes the object: only on an empty owner
    T* release() { T* p = p_; p_ = nullptr; return p; }

  private:
    bdf_ctx* c_;
    T* p_;
};
using ColOwner = Owned<bdf_col>;
using FutOwner = Owned<bdf_future>;

// One stream-ordered allocation on the compute stream, freed in the same stream order when the scope ends.
template <class T>
class Scratch {
  public:
    Scratch() = default;
    Scratch(const Scratch&) = delete;
    Scratch& operator=(const Scratch&) = delete;
    ~Scratch() { if (p_) cudaFreeAsync(p_, c_->s_compute); }
    cudaError_t alloc(bdf_ctx* c, size_t bytes) {
        c_ = c;
        return cudaMallocAsync((void**)&p_, bytes, c->s_compute);
    }
    T* get() const { return p_; }
    operator T*() const { return p_; }

  private:
    bdf_ctx* c_ = nullptr;
    T* p_ = nullptr;
};

struct ChunkPlan {
    int64_t len;
    bool has_validity;
};

// Allocate arenas for a column with the given chunk plan (validity at bit offset `bit_off[i]`).
// tile_elems > 0: the column will be produced by a kernel with that tile size (per-warp valid counts are kept).
static int col_alloc(bdf_ctx* c, int dtype, const std::vector<ChunkPlan>& plan, const std::vector<int32_t>* bit_offs,
                     int64_t tile_elems, bdf_col** out) {
    bdf_col* col = new (std::nothrow) bdf_col();
    if (!col) return fail(BDF_OOM, "host allocation failed");
    col->dtype = dtype;
    const int w = dtype_width(dtype);
    const size_t n = plan.size();
    std::vector<size_t> voff(n), boff(n);
    size_t vbytes = 0, bbytes = 0;
    for (size_t i = 0; i < n; i++) {
        voff[i] = vbytes;
        vbytes += align_up(value_bytes(dtype, plan[i].len, bit_offs ? (*bit_offs)[i] : 0) + (dtype == kBool ? 8 : 0), 256);
        boff[i] = bbytes;
        if (plan[i].has_validity) {
            const int bo = bit_offs ? (*bit_offs)[i] : 0;
            bbytes += align_up(((size_t)plan[i].len + bo + 7) / 8 + 8, 256);
        }
        col->total_len += plan[i].len;
    }
    cudaError_t e = cudaSuccess;
    if (vbytes) e = cudaMallocAsync((void**)&col->arena_values, vbytes, c->s_compute);
    if (e == cudaSuccess && bbytes) e = cudaMallocAsync((void**)&col->arena_validity, bbytes, c->s_compute);
    col->tile_elems = tile_elems;
    col->tile0.assign(n + 1, 0);
    if (tile_elems > 0)
        for (size_t i = 0; i < n; i++) col->tile0[i + 1] = col->tile0[i] + (plan[i].len + tile_elems - 1) / tile_elems;
    const size_t n_tiles = (size_t)col->tile0[n];
    if (e == cudaSuccess && bbytes && n_tiles)
        e = cudaMallocAsync((void**)&col->d_warp_counts, n_tiles * kWarpsPerCta * sizeof(uint32_t), c->s_compute);
    if (e == cudaSuccess && bbytes) e = cudaMemsetAsync(col->arena_validity, 0, bbytes, c->s_compute);
    if (e != cudaSuccess) {
        cudaGetLastError();
        col_release(c, col);
        return fail(cuda_status(e), "device allocation of %zu bytes failed: %s", vbytes + bbytes, cudaGetErrorString(e));
    }
    col->chunks.resize(n);
    col->null_counts.assign(n, 0);
    for (size_t i = 0; i < n; i++) {
        DevChunk& ch = col->chunks[i];
        ch.values = col->arena_values ? col->arena_values + voff[i] : nullptr;
        ch.validity = plan[i].has_validity ? (uint32_t*)(col->arena_validity + boff[i]) : nullptr;
        ch.len = plan[i].len;
        ch.bit_off = bit_offs ? (*bit_offs)[i] : 0;
        ch.val_bit_off = (dtype == kBool && bit_offs) ? (*bit_offs)[i] : 0;
    }
    *out = col;
    return BDF_OK;
}

// True when every group event of the column has already fired.
static bool col_complete(const bdf_col* col) {
    for (auto& g : col->groups)
        if (cudaEventQuery(g.ev) != cudaSuccess) { cudaGetLastError(); return false; }
    return true;
}

// A group whose event has already fired adds no wait to the stream.
static void wait_groups(cudaStream_t s, const bdf_col* col, int64_t begin, int64_t end) {
    for (auto& g : col->groups)
        if (g.begin < end && g.end > begin && cudaEventQuery(g.ev) != cudaSuccess) {
            cudaGetLastError();   // NotReady must not reach a later launch check
            cudaStreamWaitEvent(s, g.ev, 0);
        }
}

// Group boundaries for an operator over `n` chunks: a single group when the inputs are resident, else
// the union of the inputs' group ends (so work starts as soon as its own inputs have landed).  A context made with
// BDF_PIPELINE_SPLIT=1 always splits at the group ends, so that the grouped launches run whether or not the copies have landed.
static std::vector<int64_t> plan_groups(const bdf_ctx* c, int64_t n, const bdf_col* const* inputs, size_t n_inputs) {
    bool all_done = !c->pipeline_split;
    for (size_t j = 0; j < n_inputs; j++) all_done = all_done && (!inputs[j] || col_complete(inputs[j]));
    std::vector<int64_t> ends;
    if (!all_done)
        for (size_t j = 0; j < n_inputs; j++)
            if (inputs[j])
                for (auto& g : inputs[j]->groups)
                    if (g.end < n) ends.push_back(g.end);
    ends.push_back(n);
    std::sort(ends.begin(), ends.end());
    ends.erase(std::unique(ends.begin(), ends.end()), ends.end());
    return ends;
}
static std::vector<int64_t> plan_groups(const bdf_ctx* c, int64_t n, std::initializer_list<const bdf_col*> inputs) {
    return plan_groups(c, n, inputs.begin(), inputs.size());
}

static int64_t bitmap_bytes(int64_t len) { return (len + 7) / 8; }

// Fold the per-warp valid counts of every chunk into null_counts (host side; chunk i owns tiles [tile0[i], tile0[i+1])).
static void fold_counts(bdf_col* col, const uint32_t* counts) {
    const size_t n = col->chunks.size();
    for (size_t i = 0; i < n; i++) {
        if (!col->chunks[i].validity) { col->null_counts[i] = 0; continue; }
        int64_t valid = 0;
        for (int64_t k = col->tile0[i] * kWarpsPerCta; k < col->tile0[i + 1] * kWarpsPerCta; k++) valid += counts[k];
        col->null_counts[i] = col->chunks[i].len - valid;
    }
    col->counts_on_device = false;
}

// Mirror kernel-written valid counts into host null_counts (one small D2H + sync on the compute stream).
static int fetch_counts(bdf_ctx* c, bdf_col* col) {
    if (!col->counts_on_device) return BDF_OK;
    const size_t n = col->chunks.size();
    const size_t total = (size_t)col->tile0[n] * kWarpsPerCta;
    std::vector<uint32_t> tmp(std::max<size_t>(total, 1));
    if (total) {
        wait_groups(c->s_compute, col, 0, (int64_t)n);
        CK(cudaMemcpyAsync(tmp.data(), col->d_warp_counts, total * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->s_compute));
        CK(cudaStreamSynchronize(c->s_compute));
    }
    fold_counts(col, tmp.data());
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// reduce plumbing

static int64_t reduce_bytes(const bdf_col* col, int64_t begin, int64_t end) {
    int64_t b = 0;
    const int w = dtype_width(col->dtype);
    for (int64_t i = begin; i < end; i++)
        b += col->chunks[i].len * w + (col->chunks[i].validity ? bitmap_bytes(col->chunks[i].len) : 0);
    return b;
}

// Launch one reduce over chunks [begin,end) of col into *result (device-mapped host memory: c->h_agg_dev + slot, or a
// device record that a collective will read).  Caller has made the stream wait.
static int reduce_range(bdf_ctx* c, const bdf_col* col, int64_t begin, int64_t end, AggDev* result) {
    const int64_t n = end - begin;
    const int tile = elems_per_tile(col->dtype);
    void *hp = nullptr, *dp = nullptr;
    TRY(ring_alloc(c, (size_t)n * sizeof(RedDesc), &hp, &dp));
    RedDesc* hd = (RedDesc*)hp;
    int64_t tiles = 0, rows = 0;
    for (int64_t i = 0; i < n; i++) {
        const DevChunk& ch = col->chunks[begin + i];
        hd[i].in = ch.values; hd[i].vin = ch.validity; hd[i].len = ch.len; hd[i].tile0 = tiles; hd[i].off = ch.bit_off; hd[i].pad = 0;
        tiles += (ch.len + tile - 1) / tile;
        rows += ch.len;
    }
    RedDesc* dd = (RedDesc*)dp;
    CK(desc_upload(c, dd, hd, (size_t)n * sizeof(RedDesc)));
    if ((size_t)tiles > c->red_part_cap) {  // grow the per-CTA partials buffer (rare): drain its users first
        CK(cudaStreamSynchronize(c->s_compute));
        if (c->d_partials) CK(cudaFree(c->d_partials));
        c->d_partials = nullptr; c->red_part_cap = 0;
        const size_t cap = std::max<size_t>((size_t)tiles * 2, 65536);
        CK(cudaMalloc((void**)&c->d_partials, cap * sizeof(AggDev)));
        c->red_part_cap = cap;
    }
    {
        LaunchTimer t(c, BDF_K_REDUCE, col->dtype, rows, reduce_bytes(col, begin, end));  // k_reduce + k_finish
        CK(launch_reduce(col->dtype, dd, (int)n, tiles, c->d_partials, c->s_compute));
        c->launches++;
        CK(launch_finish(dtype_is_float(col->dtype), c->d_partials, reduce_partials(col->dtype, tiles), c->sm_count, c->d_stage2, c->d_ticket, result, c->s_compute));
    }
    return BDF_OK;
}

// Make sure every chunk's null count is known on the host (metadata for count / would_panic).
static int ensure_null_counts(bdf_ctx* c, bdf_col* col) {
    TRY(fetch_counts(c, col));
    std::vector<int64_t> unknown;
    for (size_t i = 0; i < col->chunks.size(); i++)
        if (col->null_counts[i] < 0) unknown.push_back((int64_t)i);
    if (unknown.empty()) return BDF_OK;
    if (col->dtype == kBool) return fail(BDF_UNSUPPORTED, "null count of an uploaded boolean column is unknown: pass null_count in the view");
    wait_groups(c->s_compute, col, 0, (int64_t)col->chunks.size());
    for (size_t k = 0; k < unknown.size(); k += kAggSlots) {
        const size_t m = std::min<size_t>(kAggSlots, unknown.size() - k);
        for (size_t j = 0; j < m; j++) TRY(reduce_range(c, col, unknown[k + j], unknown[k + j] + 1, c->h_agg_dev + j));
        CK(cudaStreamSynchronize(c->s_compute));
        for (size_t j = 0; j < m; j++) {
            const int64_t i = unknown[k + j];
            col->null_counts[i] = col->chunks[i].len - (int64_t)c->h_agg[j].count;
        }
    }
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// pageable host memory: staged copies

static constexpr size_t kStageBytes = (size_t)8 << 20;
static constexpr int kStageSlots = 6;
static constexpr size_t kStageMin = (size_t)1 << 20;  // smaller copies go straight through the driver

static bool is_pageable(const void* p) {
    cudaPointerAttributes attr;
    if (cudaPointerGetAttributes(&attr, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return attr.type == cudaMemoryTypeUnregistered;
}

static int ensure_stage(bdf_ctx* c) {
    if (!c->stage.empty()) return BDF_OK;
    // built in locals and committed to the context only when complete: a failure part-way leaves the context unstaged
    std::vector<bdf_ctx::StageSlot> slots(kStageSlots);
    cudaError_t e = cudaSuccess;
    for (auto& sl : slots) {
        if (e == cudaSuccess) e = cudaHostAlloc((void**)&sl.p, kStageBytes, cudaHostAllocDefault);
        if (e == cudaSuccess) e = cudaEventCreateWithFlags(&sl.ev, cudaEventDisableTiming);
    }
    const char* t = getenv("BDF_COPY_THREADS");
    const int hw = (int)std::thread::hardware_concurrency();
    const int threads = t && atoi(t) > 0 ? atoi(t) : std::max(1, std::min(8, hw > 0 ? hw : 8));
    std::unique_ptr<CopyPool> pool;
    if (e == cudaSuccess) pool.reset(new (std::nothrow) CopyPool(threads - 1));   // the calling thread is the last worker
    if (e != cudaSuccess || !pool) {
        cudaGetLastError();
        for (auto& sl : slots) { if (sl.p) cudaFreeHost(sl.p); if (sl.ev) cudaEventDestroy(sl.ev); }
        return e != cudaSuccess ? fail(cuda_status(e), "pinned staging allocation failed: %s", cudaGetErrorString(e)) : fail(BDF_OOM, "host allocation failed");
    }
    c->copy_threads = threads;
    c->pool = std::move(pool);
    c->stage = std::move(slots);
    return BDF_OK;
}

// host -> device on the h2d stream; pageable sources are staged through pinned slots (the source has been read
// completely when this returns).
static cudaError_t h2d_copy(bdf_ctx* c, void* dst, const void* src, size_t bytes) {
    if (bytes < kStageMin || !is_pageable(src)) return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, c->s_h2d);
    if (ensure_stage(c) != BDF_OK) return cudaErrorMemoryAllocation;
    for (size_t off = 0; off < bytes; off += kStageBytes) {
        const size_t n = std::min(kStageBytes, bytes - off);
        bdf_ctx::StageSlot& sl = c->stage[c->stage_next++ % kStageSlots];
        if (sl.busy) { cudaError_t e = cudaEventSynchronize(sl.ev); if (e != cudaSuccess) return e; }
        c->pool->copy(sl.p, (const char*)src + off, n);
        cudaError_t e = cudaMemcpyAsync((char*)dst + off, sl.p, n, cudaMemcpyHostToDevice, c->s_h2d);
        if (e == cudaSuccess) e = cudaEventRecord(sl.ev, c->s_h2d);
        if (e != cudaSuccess) return e;
        sl.busy = true;
    }
    return cudaSuccess;
}

// device -> pageable host, pipelined: DMA into slot k+1.. while host threads drain slot k into the user's buffer.
static cudaError_t d2h_staged(bdf_ctx* c, const std::vector<bdf_col::StagedCopy>& copies) {
    if (copies.empty()) return cudaSuccess;
    if (ensure_stage(c) != BDF_OK) return cudaErrorMemoryAllocation;
    struct Pending { bdf_ctx::StageSlot* sl; char* dst; size_t n; };
    std::deque<Pending> pending;
    auto retire = [&]() -> cudaError_t {
        Pending p = pending.front();
        pending.pop_front();
        cudaError_t e = cudaEventSynchronize(p.sl->ev);
        if (e == cudaSuccess) c->pool->copy(p.dst, p.sl->p, p.n, true);
        p.sl->busy = false;
        return e;
    };
    for (auto& cp : copies)
        for (size_t off = 0; off < cp.bytes; off += kStageBytes) {
            const size_t n = std::min(kStageBytes, cp.bytes - off);
            if ((int)pending.size() >= kStageSlots - 1) { cudaError_t e = retire(); if (e != cudaSuccess) return e; }
            bdf_ctx::StageSlot& sl = c->stage[c->stage_next++ % kStageSlots];
            if (sl.busy) { cudaError_t e = cudaEventSynchronize(sl.ev); if (e != cudaSuccess) return e; }  // an earlier upload's slot
            cudaError_t e = cudaMemcpyAsync(sl.p, (const char*)cp.src + off, n, cudaMemcpyDeviceToHost, c->s_d2h);
            if (e == cudaSuccess) e = cudaEventRecord(sl.ev, c->s_d2h);
            if (e != cudaSuccess) return e;
            sl.busy = true;
            pending.push_back(Pending{&sl, (char*)cp.dst + off, n});
        }
    while (!pending.empty()) { cudaError_t e = retire(); if (e != cudaSuccess) return e; }
    return cudaSuccess;
}

// ---------------------------------------------------------------------------------------------------
// upload / download

struct UploadSpec {
    int dtype;
    int64_t n;
    const bdf_view* views;
};

// Upload K columns with their chunks interleaved (a0,b0,a1,b1,...) so that a binary operator can start on
// chunk i as soon as BOTH of its inputs have landed.
static int upload_many(bdf_ctx* c, const std::vector<UploadSpec>& specs, bool async, std::vector<bdf_col*>& out) {
    int64_t max_n = 0;
    std::vector<ColOwner> cols;
    for (size_t k = 0; k < specs.size(); k++) {
        const UploadSpec& s = specs[k];
        std::vector<ChunkPlan> plan((size_t)s.n);
        std::vector<int32_t> offs((size_t)s.n);
        for (int64_t i = 0; i < s.n; i++) {
            const bdf_view& v = s.views[i];
            if (v.len < 0 || v.offset < 0 || (v.len > 0 && !v.values)) return fail(BDF_INVALID, "bad view %lld", (long long)i);
            plan[i] = {v.len, v.validity != nullptr};
            offs[i] = (int32_t)(v.offset & 7);
        }
        cols.emplace_back(c);
        TRY(col_alloc(c, s.dtype, plan, &offs, 0, cols[k].out()));
        for (int64_t i = 0; i < s.n; i++)
            cols[k]->null_counts[i] = s.views[i].validity ? (s.views[i].null_count >= 0 ? s.views[i].null_count : -1) : 0;
        max_n = std::max(max_n, s.n);
    }
    // allocations are stream-ordered on the compute stream: let the copy stream see them
    cudaError_t e = cudaEventRecord(c->ev_tmp, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(c->s_h2d, c->ev_tmp, 0);
    size_t pending = 0;
    int64_t group_begin = 0;
    for (int64_t i = 0; i < max_n && e == cudaSuccess; i++) {
        for (size_t k = 0; k < specs.size() && e == cudaSuccess; k++) {
            if (i >= specs[k].n) continue;
            const bdf_view& v = specs[k].views[i];
            const DevChunk& ch = cols[k]->chunks[i];
            const int w = dtype_width(specs[k].dtype);
            if (v.len) {
                const bool is_bool = specs[k].dtype == kBool;
                const size_t vb = value_bytes(specs[k].dtype, v.len, (int)(v.offset & 7));
                e = h2d_copy(c, ch.values, (const char*)v.values + (is_bool ? (v.offset >> 3) : v.offset * w), vb);
                pending += vb;
                if (e == cudaSuccess && v.validity)
                    e = cudaMemcpyAsync(ch.validity, v.validity + (v.offset >> 3), (size_t)((v.len + (v.offset & 7) + 7) / 8),
                                        cudaMemcpyHostToDevice, c->s_h2d);
            }
        }
        if (e == cudaSuccess && (pending >= c->pipeline_bytes || i == max_n - 1)) {
            for (size_t k = 0; k < specs.size() && e == cudaSuccess; k++) {
                const int64_t b = std::min(group_begin, specs[k].n), en = std::min(i + 1, specs[k].n);
                if (en <= b) continue;
                e = record_group(c, cols[k].get(), b, en, c->s_h2d);
            }
            pending = 0;
            group_begin = i + 1;
        }
    }
    if (e == cudaSuccess && !async) e = cudaStreamSynchronize(c->s_h2d);
    if (e != cudaSuccess) {
        const int st = fail_cuda(e, "upload");
        cudaStreamSynchronize(c->s_h2d);   // no copy may still write into the columns when they are freed
        return st;
    }
    out.clear();
    for (ColOwner& col : cols) out.push_back(col.release());
    return BDF_OK;
}

static int realign(bdf_ctx* c, const bdf_col* in, bdf_col** out);  // identity cast: bit offset -> 0

// Downloads are split in two so that callers can overlap them with later work: enqueue puts the D2H copies
// on the d2h stream behind the group events; finish waits for them and fills in the metadata.
static int download_enqueue(bdf_ctx* c, bdf_col* col, bdf_out* out) {
    bool misaligned = false;
    for (auto& ch : col->chunks) misaligned = misaligned || (ch.validity && ch.bit_off != 0) || ch.val_bit_off != 0;
    if (misaligned) {  // an uploaded slice downloaded as-is: shift its bitmap to offset 0 first
        ColOwner tmp(c);
        TRY(realign(c, col, tmp.out()));
        TRY(download_enqueue(c, tmp.get(), out));
        col->dl_tmp = tmp.release();
        return BDF_OK;
    }
    const int w = dtype_width(col->dtype);
    const int64_t n = (int64_t)col->chunks.size();
    for (int64_t i = 0; i < n; i++) {
        const DevChunk& ch = col->chunks[i];
        if (out[i].len != ch.len) return fail(BDF_INVALID, "output chunk %lld has capacity %lld, result has %lld rows", (long long)i, (long long)out[i].len, (long long)ch.len);
        if (ch.len && !out[i].values) return fail(BDF_INVALID, "output chunk %lld has no values buffer", (long long)i);
        if (ch.validity && ch.len && !out[i].validity) return fail(BDF_INVALID, "output chunk %lld needs a validity buffer", (long long)i);
    }
    for (auto& g : col->groups) {
        CK(cudaStreamWaitEvent(c->s_d2h, g.ev, 0));
        for (int64_t i = g.begin; i < g.end; i++) {
            const DevChunk& ch = col->chunks[i];
            if (!ch.len) continue;
            const size_t vbytes = value_bytes(col->dtype, ch.len, 0);
            if (vbytes >= kStageMin && is_pageable(out[i].values)) col->dl_staged.push_back({out[i].values, ch.values, vbytes});
            else CK(cudaMemcpyAsync(out[i].values, ch.values, vbytes, cudaMemcpyDeviceToHost, c->s_d2h));
            if (ch.validity) CK(cudaMemcpyAsync(out[i].validity, ch.validity, (size_t)bitmap_bytes(ch.len), cudaMemcpyDeviceToHost, c->s_d2h));
        }
    }
    if (col->counts_on_device && col->tile0[n] > 0) {
        col->dl_counts.resize((size_t)col->tile0[n] * kWarpsPerCta);
        CK(cudaMemcpyAsync(col->dl_counts.data(), col->d_warp_counts, col->dl_counts.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, c->s_d2h));
    }
    return BDF_OK;
}

static int download_finish(bdf_ctx* c, bdf_col* col, bdf_out* out) {
    if (col->dl_tmp) {
        bdf_col* tmp = col->dl_tmp;
        col->dl_tmp = nullptr;
        int st = download_finish(c, tmp, out);
        col_release(c, tmp);
        return st;
    }
    const int64_t n = (int64_t)col->chunks.size();
    if (!col->dl_staged.empty()) {  // the d2h stream already waits for the group events of this column
        cudaError_t e = d2h_staged(c, col->dl_staged);
        col->dl_staged.clear();
        if (e != cudaSuccess) { cudaGetLastError(); return fail(cuda_status(e), "staged download failed: %s", cudaGetErrorString(e)); }
    }
    CK(cudaStreamSynchronize(c->s_d2h));
    if (col->counts_on_device && (int64_t)col->dl_counts.size() == col->tile0[n] * kWarpsPerCta) {
        fold_counts(col, col->dl_counts.data());
        col->dl_counts.clear();
    }
    TRY(ensure_null_counts(c, col));
    for (int64_t i = 0; i < n; i++) {
        out[i].len = col->chunks[i].len;
        out[i].has_validity = col->chunks[i].validity != nullptr;
        out[i].null_count = col->null_counts[i];
    }
    return BDF_OK;
}

static int download(bdf_ctx* c, bdf_col* col, bdf_out* out) {
    TRY(download_enqueue(c, col, out));
    return download_finish(c, col, out);
}

// ---------------------------------------------------------------------------------------------------
// operators on device columns

static bool cast_is_fallible(int from, int to) {
    if (from == to || dtype_is_float(to)) return false;
    if (dtype_is_float(from)) return true;
    const bool fs = dtype_is_signed_int(from), ts = dtype_is_signed_int(to);
    const int fw = dtype_width(from), tw = dtype_width(to);
    if (fs == ts) return tw < fw;
    if (fs) return true;        // signed -> unsigned: negatives fail
    return tw <= fw;            // unsigned -> signed: needs a strictly wider target
}

static int future_new(bdf_ctx* c, int dtype, int fused, int64_t rows, bdf_future** out, int n = 1);
static bool is_global(const bdf_ctx* c) { return c->comm != nullptr && c->collective; }
static AggDev* future_target(bdf_ctx* c, const bdf_future* f, int i);
static cudaError_t future_combine(bdf_ctx* c, bdf_future* f, cudaStream_t s);
// The DivideByZero flag of a sharded divide: max over the ranks, so that every rank returns the same status.
static cudaError_t flag_allreduce(bdf_ctx* c) {
    std::string err;
    c->collectives++;
    cudaError_t e = comm_allreduce_max_i32(c->comm, c->d_flag, 1, c->s_compute, &err);
    if (e != cudaSuccess && !err.empty()) g_nccl_err = err;
    return e;
}

// One of three rotating per-tile partial buffers (K5 and fused expressions): grown on demand, reused once the
// k_finish that last read it has run.
static cudaError_t part_acquire(bdf_ctx* c, int64_t total_tiles, bdf_ctx::PartBuf** out) {
    bdf_ctx::PartBuf* pb = &c->part[c->part_next++ % 3];
    cudaError_t e = cudaSuccess;
    const size_t need = std::max<size_t>(1, (size_t)total_tiles);
    if (pb->cap < need) {  // grow (rare): nothing may still be using the old buffer
        cudaStreamSynchronize(c->s_fin); cudaStreamSynchronize(c->s_compute);
        if (pb->p) cudaFree(pb->p);
        pb->p = nullptr; pb->cap = 0;
        e = cudaMalloc((void**)&pb->p, need * sizeof(AggDev));
        if (e == cudaSuccess) pb->cap = need;
    }
    if (e == cudaSuccess && !pb->done) e = cudaEventCreateWithFlags(&pb->done, cudaEventDisableTiming);
    if (e == cudaSuccess && pb->used) {  // its previous k_finish has read it: wait on the device only while that is still pending
        e = cudaEventQuery(pb->done);
        if (e == cudaErrorNotReady) {
            cudaGetLastError();   // NotReady must not reach a later launch check
            e = cudaStreamWaitEvent(c->s_compute, pb->done, 0);
        }
    }
    *out = pb;
    return e;
}

// zip() of k columns whose paired chunks must have the same length: *n = the number of chunk tuples.
static int zip_chunks(const bdf_col* const* cols, int k, int64_t* n) {
    *n = (int64_t)cols[0]->chunks.size();
    for (int j = 1; j < k; j++) *n = std::min<int64_t>(*n, (int64_t)cols[j]->chunks.size());
    for (int j = 1; j < k; j++)
        for (int64_t i = 0; i < *n; i++)
            if (cols[j]->chunks[i].len != cols[0]->chunks[i].len)
                return fail(BDF_LENGTH_MISMATCH, "Cannot perform math operation on arrays of different length");
    return BDF_OK;
}

// Reads back the device flag the kernels raise (DivideByZero, an index out of bounds, an empty list): waits for the compute stream.
// all_ranks: the max over the ranks of the communicator, so that every rank takes the same exit.
static cudaError_t flag_read(bdf_ctx* c, bool all_ranks, int* flag) {
    cudaError_t e = all_ranks ? flag_allreduce(c) : cudaSuccess;
    if (e == cudaSuccess) e = cudaMemcpyAsync(c->h_flag, c->d_flag, sizeof(int), cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
    *flag = e == cudaSuccess ? *c->h_flag : 0;
    return e;
}

// Folds the per-tile partials of a fused aggregate (K5, fused expressions) into the future on the finish stream, so that the next
// operator on the compute stream does not wait for it.  The caller has made the finish stream wait for the launch that wrote them.
static cudaError_t fused_finish(bdf_ctx* c, bdf_future* f, bdf_ctx::PartBuf* pb, int64_t tiles, int64_t n_chunks) {
    c->launches++;
    cudaError_t e = launch_finish(dtype_is_float(f->dtypes[0]), pb->p, tiles, c->sm_count, c->d_stage, c->d_ticket + 1, future_target(c, f, 0), c->s_fin);
    if (e == cudaSuccess) e = cudaEventRecord(pb->done, c->s_fin);
    pb->used = true;
    f->chunks[0] = (uint32_t)n_chunks;
    if (e == cudaSuccess) e = future_combine(c, f, c->s_fin);   // ranks of a communicator: one grouped NCCL reduction
    if (e == cudaSuccess) e = cudaEventRecord(f->ev, c->s_fin);
    return e;
}

// The launch loop of the element-wise operators.  Allocates the output column (plan, dtype, tile) and, for every chunk group
// [begin, end) up to each of `ends`: fills the descriptors of its chunks, makes the compute stream wait for the inputs' groups,
// uploads the descriptors, launches under one LaunchTimer and records the group's event on the output.  A group without chunks
// launches nothing.
//   fill(host descriptors, chunk i, tile0 of i within its group, output chunk i) -> the chunk's bytes for the launch record
//   launch(device descriptors of the group, begin, end, tiles, tile_base = tiles of the groups before, warp counts) -> cudaError_t
template <class Fill, class Launch>
static int launch_groups(bdf_ctx* c, const bdf_col* const* inputs, size_t n_inputs, const std::vector<int64_t>& ends, int dtype,
                         const std::vector<ChunkPlan>& plan, int tile, size_t desc_bytes, int kernel, const char* what, Fill fill,
                         Launch launch, bdf_col** out) {
    ColOwner o(c);
    TRY(col_alloc(c, dtype, plan, nullptr, tile, o.out()));
    o->counts_on_device = o->d_warp_counts != nullptr;
    void *hp = nullptr, *dp = nullptr;
    TRY(ring_alloc(c, plan.size() * desc_bytes, &hp, &dp));
    char *hd = (char*)hp, *dd = (char*)dp;
    cudaError_t e = cudaSuccess;
    int64_t begin = 0, tile_base = 0;
    for (size_t gi = 0; gi < ends.size() && e == cudaSuccess; gi++) {
        const int64_t end = ends[gi];
        int64_t tiles = 0, rows = 0, bytes = 0;
        for (int64_t i = begin; i < end; i++) {
            bytes += fill((void*)hd, i, tiles, o->chunks[i]);
            tiles += (plan[i].len + tile - 1) / tile;
            rows += plan[i].len;
        }
        for (size_t j = 0; j < n_inputs; j++)
            if (inputs[j]) wait_groups(c->s_compute, inputs[j], begin, end);
        if (end > begin) {
            e = desc_upload(c, dd + begin * desc_bytes, hd + begin * desc_bytes, (size_t)(end - begin) * desc_bytes);
            if (e == cudaSuccess) {
                LaunchTimer t(c, kernel, dtype, rows, bytes);
                e = launch((const void*)(dd + begin * desc_bytes), begin, end, tiles, tile_base,
                           o->d_warp_counts ? o->d_warp_counts + o->tile0[begin] * kWarpsPerCta : nullptr);
            }
        }
        if (e == cudaSuccess) e = record_group(c, o.get(), begin, end, c->s_compute);
        begin = end;
        tile_base += tiles;
    }
    if (e != cudaSuccess) return fail_cuda(e, what);
    *out = o.release();
    return BDF_OK;
}
template <class Fill, class Launch>
static int launch_groups(bdf_ctx* c, std::initializer_list<const bdf_col*> inputs, const std::vector<int64_t>& ends, int dtype,
                         const std::vector<ChunkPlan>& plan, int tile, size_t desc_bytes, int kernel, const char* what, Fill fill,
                         Launch launch, bdf_col** out) {
    return launch_groups(c, inputs.begin(), inputs.size(), ends, dtype, plan, tile, desc_bytes, kernel, what, fill, launch, out);
}

static int binary_dev(bdf_ctx* c, int op, const bdf_col* l, const bdf_col* r, bdf_col** out, bdf_future** fut = nullptr) {
    if (op < 0 || op >= BDF_NBINARY) return fail(BDF_INVALID, "invalid binary op %d", op);
    if (l->dtype != r->dtype) return fail(BDF_INVALID, "binary op on columns of different types (%d, %d)", l->dtype, r->dtype);
    if (l->dtype == kBool) return fail(BDF_UNSUPPORTED, "arithmetic on a boolean column");
    const int dtype = l->dtype;
    if (op > BDF_DIV && !dtype_is_float(dtype)) return fail(BDF_UNSUPPORTED, "atan2/hypot/log need a float column (T::Native: Float)");
    const bdf_col* in[] = {l, r};
    int64_t n = 0;
    TRY(zip_chunks(in, 2, &n));
    std::vector<ChunkPlan> plan((size_t)n);
    for (int64_t i = 0; i < n; i++)
        plan[i] = {l->chunks[i].len, op > BDF_DIV || l->chunks[i].validity || r->chunks[i].validity};
    const int tile = elems_per_tile_binary(op, dtype);
    const int w = dtype_width(dtype);
    cudaError_t e = cudaSuccess;
    // K5: aggregate of the output fused into the same pass -> one partial per tile, folded by k_finish
    bdf_ctx::PartBuf* pb = nullptr;
    int64_t total_tiles = 0, total_rows = 0;
    FutOwner f(c);
    if (fut) {
        if (op > BDF_DIV) return fail(BDF_UNSUPPORTED, "fused aggregate is available for add/subtract/multiply/divide");
        for (int64_t i = 0; i < n; i++) { total_tiles += (plan[i].len + tile - 1) / tile; total_rows += plan[i].len; }
        TRY(future_new(c, dtype, 1, total_rows, f.out()));
        e = part_acquire(c, total_tiles, &pb);
    }
    const std::vector<int64_t> ends = plan_groups(c, n, {l, r});
    if (e == cudaSuccess && op == BDF_DIV) e = cudaMemsetAsync(c->d_flag, 0, sizeof(int), c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "binary op");
    ColOwner o(c);
    TRY(launch_groups(c, {l, r}, ends, dtype, plan, tile, sizeof(BinDesc), BDF_K_BINARY, "binary op",
        [&](void* hd, int64_t i, int64_t tile0, const DevChunk& oc) {
            const DevChunk &a = l->chunks[i], &b = r->chunks[i];
            ((BinDesc*)hd)[i] = BinDesc{a.values, b.values, oc.values, a.validity, b.validity, oc.validity, a.len, tile0, a.bit_off, b.bit_off};
            return 3 * a.len * w + ((a.validity ? 1 : 0) + (b.validity ? 1 : 0) + (oc.validity ? 1 : 0)) * bitmap_bytes(a.len);
        },
        [&](const void* dd, int64_t begin, int64_t end, int64_t tiles, int64_t tile_base, uint32_t* wc) {
            return launch_binary(op, dtype, (const BinDesc*)dd, (int)(end - begin), tiles, wc, c->d_flag, c->s_compute, pb ? pb->p + tile_base : nullptr);
        },
        o.out()));
    if (f.get()) {
        for (auto& g : o->groups) cudaStreamWaitEvent(c->s_fin, g.ev, 0);
        e = fused_finish(c, f.get(), pb, total_tiles, n);
    }
    // DivideByZero must be returned INSTEAD of data: wait for the flag (every rank of a communicator takes the same exit).
    int flag = 0;
    if (e == cudaSuccess && op == BDF_DIV) e = flag_read(c, is_global(c), &flag);
    if (e != cudaSuccess) return fail_cuda(e, "binary op");
    if (flag) return fail(BDF_DIVIDE_BY_ZERO, "Divide by zero error");
    *out = o.release();
    if (fut) *fut = f.release();
    return BDF_OK;
}

// Shared body of unary ops and casts (one input column, one output column).
static int map_dev(bdf_ctx* c, bool is_cast, int op_or_to, const bdf_col* in, bdf_col** out) {
    const int from = in->dtype;
    int to = from;
    if (from == kBool) return fail(BDF_UNSUPPORTED, "numeric function on a boolean column");
    if (is_cast) {
        to = op_or_to;
        TRY(check_dtype(to));
    } else {
        const int op = op_or_to;
        if (op < 0 || op >= BDF_NUNARY) return fail(BDF_INVALID, "invalid unary op %d", op);
        if (op == BDF_ABS) {
            if (!dtype_is_float(from) && !dtype_is_signed_int(from)) return fail(BDF_UNSUPPORTED, "abs needs a signed type (T::Native: Signed)");
        } else if (!dtype_is_float(from)) {
            return fail(BDF_UNSUPPORTED, "float function on a non-float column (T::Native: Float)");
        }
    }
    const int64_t n = (int64_t)in->chunks.size();
    const bool fallible = is_cast && cast_is_fallible(from, to);
    std::vector<ChunkPlan> plan((size_t)n);
    for (int64_t i = 0; i < n; i++) plan[i] = {in->chunks[i].len, in->chunks[i].validity != nullptr || fallible};
    const int tile = is_cast ? elems_per_tile_cast(from, to) : elems_per_tile_unary(op_or_to, from);
    const int wf = dtype_width(from), wt = dtype_width(to);
    return launch_groups(c, {in}, plan_groups(c, n, {in}), to, plan, tile, sizeof(UnDesc), is_cast ? BDF_K_CAST : BDF_K_UNARY,
        is_cast ? "cast" : "unary op",
        [&](void* hd, int64_t i, int64_t tile0, const DevChunk& oc) {
            const DevChunk& a = in->chunks[i];
            ((UnDesc*)hd)[i] = UnDesc{a.values, oc.values, a.validity, oc.validity, a.len, tile0, a.bit_off, 0};
            return a.len * (wf + wt) + ((a.validity ? 1 : 0) + (oc.validity ? 1 : 0)) * bitmap_bytes(a.len);
        },
        [&](const void* dd, int64_t begin, int64_t end, int64_t tiles, int64_t, uint32_t* wc) {
            return is_cast ? launch_cast(from, to, (const UnDesc*)dd, (int)(end - begin), tiles, wc, c->s_compute)
                           : launch_unary(op_or_to, from, (const UnDesc*)dd, (int)(end - begin), tiles, wc, c->s_compute);
        },
        out);
}

// ---- dates and timestamps (k_temporal.cu; the rules are stated in include/b200df.h) ----------------------------------------------

static int64_t temporal_per_sec(int cfg) { return cfg == TC_MS ? 1000LL : cfg == TC_US ? 1000000LL : cfg == TC_NS ? 1000000000LL : 1LL; }

// A valid (kind, unit) -> its physical dtype and storage unit; anything else is BDF_INVALID.
static int temporal_storage(const bdf_temporal_type* t, int* dtype, int* cfg) {
    const int u = t->unit;
    switch (t->kind) {
        case BDF_DATE32: *dtype = BDF_I32; *cfg = TC_DAYS; return BDF_OK;
        case BDF_DATE64: if (u == BDF_MILLISECOND) { *dtype = BDF_I64; *cfg = TC_MS; return BDF_OK; } break;
        case BDF_TIMESTAMP: if (u >= BDF_SECOND && u <= BDF_NANOSECOND) { *dtype = BDF_I64; *cfg = TC_S + u; return BDF_OK; } break;
        case BDF_TIME32: if (u == BDF_SECOND || u == BDF_MILLISECOND) { *dtype = BDF_I32; *cfg = TC_S + u; return BDF_OK; } break;
        case BDF_TIME64: if (u == BDF_MICROSECOND || u == BDF_NANOSECOND) { *dtype = BDF_I64; *cfg = TC_S + u; return BDF_OK; } break;
        default: return fail(BDF_INVALID, "unknown temporal kind %d", t->kind);
    }
    return fail(BDF_INVALID, "temporal kind %d does not take time unit %d", t->kind, u);
}

// The fixed offset of a Timestamp's tz in seconds; false for a tz the device cannot apply (a named zone).
static bool temporal_tz_offset(const char* tz, int64_t* sec) {
    *sec = 0;
    if (!tz || !strcmp(tz, "UTC") || !strcmp(tz, "Z")) return true;
    const auto dig = [](char ch) { return ch >= '0' && ch <= '9'; };
    if (strlen(tz) != 6 || (tz[0] != '+' && tz[0] != '-') || !dig(tz[1]) || !dig(tz[2]) || tz[3] != ':' || !dig(tz[4]) || !dig(tz[5])) return false;
    const int hh = (tz[1] - '0') * 10 + (tz[2] - '0'), mm = (tz[4] - '0') * 10 + (tz[5] - '0');
    if (hh > 23 || mm > 59) return false;
    *sec = (tz[0] == '-' ? -1 : 1) * (int64_t)(hh * 3600 + mm * 60);
    return true;
}

struct TemporalPlan {
    int in_dtype = 0, cfg = 0, out_dtype = 0;
    bdf_temporal_type out_type{};
    TemporalParams p{};
};

// Validates (fn, type, arg) and plans the launch: what bdf_temporal_result reports and every entry checks first.
static int temporal_plan(int fn, const bdf_temporal_type* t, int64_t arg, TemporalPlan* pl) {
    if (!t) return fail(BDF_INVALID, "null temporal type");
    if (fn < 0 || fn >= BDF_NTEMPORAL) return fail(BDF_INVALID, "unknown temporal function %d", fn);
    TRY(temporal_storage(t, &pl->in_dtype, &pl->cfg));
    const bool time_kind = t->kind == BDF_TIME32 || t->kind == BDF_TIME64;
    const bool field_of_day = fn == BDF_TEMPORAL_HOUR || fn == BDF_TEMPORAL_MINUTE || fn == BDF_TEMPORAL_SECOND;
    if (time_kind && !field_of_day) return fail(BDF_UNSUPPORTED, "temporal function %d needs a date or a timestamp, not a time of day", fn);
    const bool int32_arg = fn == BDF_TEMPORAL_DATE_ADD || fn == BDF_TEMPORAL_DATE_SUB || fn == BDF_TEMPORAL_ADD_MONTHS;
    if (int32_arg && (arg < INT32_MIN || arg > INT32_MAX)) return fail(BDF_INVALID, "the argument %lld is outside the Int32 range", (long long)arg);
    if (fn == BDF_TEMPORAL_NEXT_DAY && (arg < 1 || arg > 7)) return fail(BDF_INVALID, "next_day takes a day of week 1..7 (1 = Sunday), not %lld", (long long)arg);
    if (fn == BDF_TEMPORAL_DATE_TRUNC && (arg < BDF_TRUNC_YEAR || arg > BDF_TRUNC_SECOND)) return fail(BDF_INVALID, "unknown date_trunc unit %lld", (long long)arg);
    if (fn == BDF_TEMPORAL_TO_TIMESTAMP && (arg < BDF_SECOND || arg > BDF_NANOSECOND)) return fail(BDF_INVALID, "unknown time unit %lld", (long long)arg);
    const bool instant = fn == BDF_TEMPORAL_UNIX_TIMESTAMP || fn == BDF_TEMPORAL_TO_TIMESTAMP;
    int64_t off_sec = 0;
    if (t->kind == BDF_TIMESTAMP && !instant && !temporal_tz_offset(t->tz, &off_sec))
        return fail(BDF_UNSUPPORTED, "time zone '%s' is not a fixed offset: named zones need a tz database the device does not have", t->tz);
    TemporalParams& p = pl->p;
    p.fn = fn;
    p.time_kind = time_kind ? 1 : 0;
    p.arg = int32_arg ? arg : 0;
    p.aux = (fn == BDF_TEMPORAL_NEXT_DAY || fn == BDF_TEMPORAL_DATE_TRUNC) ? (int32_t)arg : 0;
    p.off = off_sec * temporal_per_sec(pl->cfg);
    p.mul = 1; p.div = 1;
    pl->out_type = bdf_temporal_type{BDF_TEMPORAL_NONE, 0, nullptr};
    switch (fn) {
        case BDF_TEMPORAL_TO_DATE: case BDF_TEMPORAL_DATE_ADD: case BDF_TEMPORAL_DATE_SUB: case BDF_TEMPORAL_ADD_MONTHS:
        case BDF_TEMPORAL_LAST_DAY: case BDF_TEMPORAL_NEXT_DAY:
            pl->out_dtype = BDF_I32; pl->out_type = bdf_temporal_type{BDF_DATE32, 0, nullptr}; break;
        case BDF_TEMPORAL_DATE_TRUNC: pl->out_dtype = pl->in_dtype; pl->out_type = *t; break;
        case BDF_TEMPORAL_UNIX_TIMESTAMP: pl->out_dtype = BDF_I64; break;
        case BDF_TEMPORAL_TO_TIMESTAMP: {
            pl->out_dtype = BDF_I64;
            pl->out_type = bdf_temporal_type{BDF_TIMESTAMP, (int32_t)arg, t->kind == BDF_TIMESTAMP ? t->tz : nullptr};
            const int64_t dst = temporal_per_sec(TC_S + (int)arg);
            if (pl->cfg == TC_DAYS) p.mul = 86400 * dst;
            else {
                const int64_t src = temporal_per_sec(pl->cfg);
                if (dst >= src) p.mul = dst / src; else p.div = src / dst;
            }
            break;
        }
        default: pl->out_dtype = BDF_I32; break;   // the Int32 fields
    }
    return BDF_OK;
}

static int temporal_dev(bdf_ctx* c, const TemporalPlan& pl, const bdf_col* in, bdf_col** out) {
    if (in->dtype != pl.in_dtype) return fail(BDF_INVALID, "a column of dtype %d does not hold this temporal type (dtype %d)", in->dtype, pl.in_dtype);
    const int64_t n = (int64_t)in->chunks.size();
    std::vector<ChunkPlan> plan((size_t)n);
    for (int64_t i = 0; i < n; i++) plan[i] = {in->chunks[i].len, true};   // range rules can turn any slot NULL
    const int tile = elems_per_tile_temporal(pl.in_dtype, pl.out_dtype);
    const int wi = dtype_width(pl.in_dtype), wo = dtype_width(pl.out_dtype);
    return launch_groups(c, {in}, plan_groups(c, n, {in}), pl.out_dtype, plan, tile, sizeof(UnDesc), BDF_K_TEMPORAL, "temporal function",
        [&](void* hd, int64_t i, int64_t tile0, const DevChunk& oc) {
            const DevChunk& a = in->chunks[i];
            ((UnDesc*)hd)[i] = UnDesc{a.values, oc.values, a.validity, oc.validity, a.len, tile0, a.bit_off, 0};
            return a.len * (wi + wo) + ((a.validity ? 1 : 0) + 1) * bitmap_bytes(a.len);
        },
        [&](const void* dd, int64_t begin, int64_t end, int64_t tiles, int64_t, uint32_t* wc) {
            return launch_temporal(pl.cfg, pl.in_dtype, pl.out_dtype, pl.p, (const UnDesc*)dd, (int)(end - begin), tiles, wc, c->s_compute);
        },
        out);
}

// One side of a two-column temporal function: a date kind, its storage and its fixed offset in its own units.
static int temporal_side(const bdf_temporal_type* t, const bdf_col* col, int* cfg, int64_t* off) {
    if (!t || !col) return fail(BDF_INVALID, "null argument");
    int dtype = 0;
    TRY(temporal_storage(t, &dtype, cfg));
    if (t->kind == BDF_TIME32 || t->kind == BDF_TIME64) return fail(BDF_UNSUPPORTED, "date_diff / months_between need dates or timestamps, not times of day");
    int64_t sec = 0;
    if (t->kind == BDF_TIMESTAMP && !temporal_tz_offset(t->tz, &sec))
        return fail(BDF_UNSUPPORTED, "time zone '%s' is not a fixed offset: named zones need a tz database the device does not have", t->tz);
    if (col->dtype != dtype) return fail(BDF_INVALID, "a column of dtype %d does not hold this temporal type (dtype %d)", col->dtype, dtype);
    *off = sec * temporal_per_sec(*cfg);
    return BDF_OK;
}

static int temporal_binary_dev(bdf_ctx* c, int fn, const bdf_temporal_type* ta, const bdf_col* a, const bdf_temporal_type* tb, const bdf_col* b,
                               bdf_col** out) {
    if (fn != BDF_TEMPORAL_DATE_DIFF && fn != BDF_TEMPORAL_MONTHS_BETWEEN) return fail(BDF_INVALID, "unknown two-column temporal function %d", fn);
    TemporalParams2 p{};
    p.fn = fn;
    TRY(temporal_side(ta, a, &p.cfg_a, &p.off_a));
    TRY(temporal_side(tb, b, &p.cfg_b, &p.off_b));
    const int out_dtype = fn == BDF_TEMPORAL_DATE_DIFF ? BDF_I32 : BDF_F64;
    const bdf_col* in[] = {a, b};
    int64_t n = 0;
    TRY(zip_chunks(in, 2, &n));
    std::vector<ChunkPlan> plan((size_t)n);
    for (int64_t i = 0; i < n; i++) plan[i] = {a->chunks[i].len, true};
    const int tile = elems_per_tile_temporal2(a->dtype, b->dtype, out_dtype);
    const int wrow = dtype_width(a->dtype) + dtype_width(b->dtype) + dtype_width(out_dtype);
    return launch_groups(c, {a, b}, plan_groups(c, n, {a, b}), out_dtype, plan, tile, sizeof(BinDesc), BDF_K_TEMPORAL, "temporal function",
        [&](void* hd, int64_t i, int64_t tile0, const DevChunk& oc) {
            const DevChunk &x = a->chunks[i], &y = b->chunks[i];
            ((BinDesc*)hd)[i] = BinDesc{x.values, y.values, oc.values, x.validity, y.validity, oc.validity, x.len, tile0, x.bit_off, y.bit_off};
            return x.len * wrow + ((x.validity ? 1 : 0) + (y.validity ? 1 : 0) + 1) * bitmap_bytes(x.len);
        },
        [&](const void* dd, int64_t begin, int64_t end, int64_t tiles, int64_t, uint32_t* wc) {
            return launch_temporal2(a->dtype, b->dtype, out_dtype, p, (const BinDesc*)dd, (int)(end - begin), tiles, wc, c->s_compute);
        },
        out);
}

static int boolean_dev(bdf_ctx* c, int op, const bdf_col* a, const bdf_col* b, bdf_col** out);
static int realign(bdf_ctx* c, const bdf_col* in, bdf_col** out) {
    if (in->dtype == kBool) return boolean_dev(c, 1 /* OR: x | x = x, validity AND itself */, in, in, out);
    return map_dev(c, true, in->dtype, in, out);
}

// A future over n aggregates.  On a context that is a rank of a communicator (collective mode) the kernels write their
// per-rank records to device memory (d_local) and future_combine enqueues the grouped NCCL reduction that delivers the
// GLOBAL records to the pinned slots; otherwise the kernels write the pinned slots themselves.
static int future_new(bdf_ctx* c, int dtype, int fused, int64_t rows, bdf_future** out, int n) {
    if (n < 1 || n > kCommMaxCols) return fail(BDF_INVALID, "an aggregate call takes 1..%d columns", kCommMaxCols);
    bdf_future* f = new (std::nothrow) bdf_future();
    if (!f) return fail(BDF_OOM, "host allocation failed");
    f->n = n; f->fused = fused; f->global = is_global(c);
    f->dtypes.assign((size_t)n, dtype); f->rows.assign((size_t)n, rows); f->panics.assign((size_t)n, 0u); f->chunks.assign((size_t)n, 1u);
    const int words = f->global ? 2 * n : n;
    if (c->fut_next % kAggSlots + words > kAggSlots) c->fut_next += kAggSlots - c->fut_next % kAggSlots;  // keep the block contiguous
    f->slot = kAggSlots + c->fut_next % kAggSlots;  // upper half of h_agg is the future ring
    c->fut_next += words;
    if (f->global) {
        if (c->local_next % kAggSlots + n > kAggSlots) c->local_next += kAggSlots - c->local_next % kAggSlots;
        f->lslot = c->local_next % kAggSlots;
        c->local_next += n;
    }
    cudaError_t e = ev_get(c, &f->ev);
    if (e != cudaSuccess) { delete f; return fail_cuda(e, "event creation"); }
    *out = f;
    return BDF_OK;
}

// Where the kernels of aggregate i of the future deliver their folded record.
static AggDev* future_target(bdf_ctx* c, const bdf_future* f, int i) {
    return f->global ? c->d_local + f->lslot + i : c->h_agg_dev + f->slot + i;
}

// Global futures: enqueue the ONE grouped collective on the stream that produced the records (no host round trip).
static cudaError_t future_combine(bdf_ctx* c, bdf_future* f, cudaStream_t s) {
    if (!f->global) return cudaSuccess;
    unsigned long long fmask = 0, rows[kCommMaxCols];
    for (int i = 0; i < f->n; i++) {
        if (dtype_is_float(f->dtypes[i])) fmask |= 1ull << i;
        rows[i] = (unsigned long long)f->rows[i];
    }
    std::string err;
    c->collectives++;
    c->launches += 2;  // pack + unpack (the NCCL kernel itself is not ours)
    cudaError_t e = comm_combine(c->comm, fmask, f->n, c->d_local + f->lslot, rows, f->panics.data(), f->chunks.data(), c->h_agg_dev + f->slot, s, &err);
    if (e != cudaSuccess && !err.empty()) g_nccl_err = err;
    return e;
}

// AggDev (device format) -> bdf_agg4 (ABI format: T::Native bit patterns)
static void convert_agg(int dtype, int fused, const AggDev& a, int64_t rows, bdf_agg4* out) {
    memset(out, 0, sizeof *out);
    const int w = dtype_width(dtype);
    const uint64_t mask = w == 8 ? ~0ull : ((1ull << (8 * w)) - 1ull);
    if (dtype == BDF_F64) {
        out->sum = a.sum_bits;
    } else if (dtype == BDF_F32) {
        double d; memcpy(&d, &a.sum_bits, 8);
        const float f = (float)d;
        uint32_t fb; memcpy(&fb, &f, 4);
        out->sum = fb;
    } else {
        // k_binary AGG (fused == 1) keys flip the sign bit of T; k_reduce (fused == 2) keys flip bit 63 of the extended value
        const uint64_t flip = !dtype_is_signed_int(dtype) ? 0ull : (fused == 1 ? (1ull << (8 * w - 1)) : (1ull << 63));
        out->sum = a.sum_bits & mask;
        out->min = (a.min_bits ^ flip) & mask;
        out->max = (a.max_bits ^ flip) & mask;
    }
    out->count = (int64_t)a.count;
    out->rows = rows;
    out->any_valid = a.count > 0;
}

// sum/min/max/count of several columns with as few launches as possible: the columns of one dtype share ONE k_reduce launch
// (their chunk descriptors are concatenated, every column starting on a CTA boundary), and ONE k_finish_many folds every
// column's partials.  BASELINE config 3 (8 x Int64) is 2 launches instead of 16 -- what matters once the rows are split
// over several GPUs and a column's reduction takes microseconds.
static int reduce_columns(bdf_ctx* c, int n_cols, bdf_col* const* cols, bdf_future* f) {
    struct Range { int64_t cta0, ctas; };
    std::vector<Range> range((size_t)n_cols);
    int64_t total_ctas = 0, total_chunks = 0;
    for (int k = 0; k < n_cols; k++) total_chunks += (int64_t)cols[k]->chunks.size();
    void *hp = nullptr, *dp = nullptr;
    TRY(ring_alloc(c, (size_t)total_chunks * sizeof(RedDesc), &hp, &dp));
    RedDesc* hd = (RedDesc*)hp;
    RedDesc* dd = (RedDesc*)dp;
    struct Launch { int dtype; int64_t desc0, n_desc, tiles, cta0; int64_t rows, bytes; };
    std::vector<Launch> launches;
    std::vector<char> done((size_t)n_cols, 0);
    int64_t di = 0;
    for (int k0 = 0; k0 < n_cols; k0++) {
        if (done[k0]) continue;
        const int dtype = cols[k0]->dtype;
        const int K = reduce_tiles_per_cta(dtype), tile = elems_per_tile(dtype);
        Launch L{dtype, di, 0, 0, total_ctas, 0, 0};
        int64_t tiles = 0;
        for (int k = k0; k < n_cols; k++) {
            if (done[k] || cols[k]->dtype != dtype) continue;
            done[k] = 1;
            tiles = (tiles + K - 1) / K * K;   // the column starts on a CTA boundary
            const int64_t col_tile0 = tiles;
            for (const DevChunk& ch : cols[k]->chunks) {
                hd[di] = RedDesc{ch.values, ch.validity, ch.len, tiles, ch.bit_off, 0};
                di++;
                tiles += (ch.len + tile - 1) / tile;
                L.rows += ch.len;
            }
            L.bytes += reduce_bytes(cols[k], 0, (int64_t)cols[k]->chunks.size());
            range[k] = Range{L.cta0 + col_tile0 / K, (tiles - col_tile0 + K - 1) / K};
        }
        L.n_desc = di - L.desc0;
        L.tiles = tiles;
        total_ctas += (tiles + K - 1) / K;
        launches.push_back(L);
    }
    CK(desc_upload(c, dd, hd, (size_t)total_chunks * sizeof(RedDesc)));
    if ((size_t)total_ctas > c->red_part_cap) {
        CK(cudaStreamSynchronize(c->s_compute));
        if (c->d_partials) CK(cudaFree(c->d_partials));
        c->d_partials = nullptr; c->red_part_cap = 0;
        const size_t cap = std::max<size_t>((size_t)total_ctas * 2, 65536);
        CK(cudaMalloc((void**)&c->d_partials, cap * sizeof(AggDev)));
        c->red_part_cap = cap;
    }
    if (!c->d_stage_many) {
        CK(cudaMalloc((void**)&c->d_stage_many, (size_t)kFinishMany * c->sm_count * sizeof(AggDev)));
        CK(cudaMalloc((void**)&c->d_tickets_many, kFinishMany * sizeof(unsigned int)));
        CK(cudaMemset(c->d_tickets_many, 0, kFinishMany * sizeof(unsigned int)));
    }
    for (const Launch& L : launches) {
        LaunchTimer t(c, BDF_K_REDUCE, L.dtype, L.rows, L.bytes);
        CK(launch_reduce(L.dtype, dd + L.desc0, (int)L.n_desc, L.tiles, c->d_partials + L.cta0, c->s_compute));
    }
    FinishJob jobs[kFinishMany];
    for (int k = 0; k < n_cols; k++)
        jobs[k] = FinishJob{c->d_partials + range[k].cta0, (long long)range[k].ctas, future_target(c, f, k), dtype_is_float(cols[k]->dtype) ? 1 : 0, 0};
    c->launches++;
    CK(launch_finish_many(n_cols, jobs, c->sm_count, c->d_stage_many, c->d_tickets_many, c->s_compute));
    return BDF_OK;
}

// Chunks of the column that are empty or all-null: the reference's max/min .unwrap() a None there (aggregate.rs:19,29).
static int count_panic_chunks(bdf_ctx* c, bdf_col* col, uint32_t* out) {
    TRY(ensure_null_counts(c, col));
    uint32_t k = 0;
    for (size_t i = 0; i < col->chunks.size(); i++)
        if (col->chunks[i].len - col->null_counts[i] == 0) k++;
    *out = k;
    return BDF_OK;
}

// sum/min/max/count of n columns: one k_reduce + k_finish per column on the compute stream and -- on a rank of a
// communicator -- ONE grouped collective for all of them.  need_counts: also evaluate the would-panic rule (may
// synchronise to learn null counts of uploaded columns).
static int aggregate_many_dev_async(bdf_ctx* c, int n_cols, bdf_col* const* cols, bool need_counts, bdf_future** fut) {
    if (n_cols < 1 || n_cols > kCommMaxCols) return fail(BDF_INVALID, "an aggregate call takes 1..%d columns", kCommMaxCols);
    for (int k = 0; k < n_cols; k++) {
        if (!cols[k]) return fail(BDF_INVALID, "null column");
        if (cols[k]->dtype == kBool) return fail(BDF_UNSUPPORTED, "aggregate of a boolean column");
    }
    std::vector<uint32_t> panics((size_t)n_cols, 0u);
    if (need_counts)
        for (int k = 0; k < n_cols; k++) TRY(count_panic_chunks(c, cols[k], &panics[k]));
    FutOwner f(c);
    TRY(future_new(c, cols[0]->dtype, 2, 0, f.out(), n_cols));
    for (int k = 0; k < n_cols; k++) {
        bdf_col* col = cols[k];
        const int64_t n = (int64_t)col->chunks.size();
        f->dtypes[k] = col->dtype; f->rows[k] = col->total_len; f->panics[k] = panics[k]; f->chunks[k] = (uint32_t)n;
        wait_groups(c->s_compute, col, 0, n);
    }
    if (n_cols == 1) TRY(reduce_range(c, cols[0], 0, (int64_t)cols[0]->chunks.size(), future_target(c, f.get(), 0)));
    else TRY(reduce_columns(c, n_cols, cols, f.get()));
    cudaError_t e = future_combine(c, f.get(), c->s_compute);
    if (e == cudaSuccess) e = cudaEventRecord(f->ev, c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "aggregate");
    *fut = f.release();
    return BDF_OK;
}

static int aggregate_all_dev_async(bdf_ctx* c, bdf_col* col, bdf_future** fut) {
    return aggregate_many_dev_async(c, 1, &col, false, fut);
}

// Waits for the future, converts its n records into out[0..n) and consumes it.
static int future_wait(bdf_ctx* c, bdf_future* f, bdf_agg4* out) {
    cudaError_t e = cudaEventSynchronize(f->ev);
    if (e == cudaSuccess && out)
        for (int i = 0; i < f->n; i++) {
            if (f->global) {
                const AggDev& x = c->h_agg[f->slot + 2 * i + 1];   // {rows, panics, chunks} summed over the ranks
                convert_agg(f->dtypes[i], f->fused, c->h_agg[f->slot + 2 * i], (int64_t)x.sum_bits, &out[i]);
                out[i].would_panic = x.min_bits != 0;
                out[i].n_chunks = (int64_t)x.max_bits;
            } else {
                convert_agg(f->dtypes[i], f->fused, c->h_agg[f->slot + i], f->rows[i], &out[i]);
                out[i].would_panic = f->panics[i] != 0;
                out[i].n_chunks = (int64_t)f->chunks[i];
            }
        }
    drop(c, f);
    if (e != cudaSuccess) return fail(cuda_status(e), "waiting for an aggregate failed: %s", cudaGetErrorString(e));
    return BDF_OK;
}

static int aggregate_all_dev(bdf_ctx* c, bdf_col* col, bool need_counts, bdf_agg4* out) {
    bdf_future* f = nullptr;
    TRY(aggregate_many_dev_async(c, 1, &col, need_counts, &f));
    return future_wait(c, f, out);
}

// count is metadata (aggregate.rs:70-80); on a rank of a communicator the other ranks' chunks count too.
static int count_global(bdf_ctx* c, int64_t* total) {
    if (!is_global(c)) return BDF_OK;
    std::vector<int64_t> all((size_t)comm_world(c->comm));
    std::string err;
    c->collectives++;
    cudaError_t e = comm_host_allgather(c->comm, total, all.data(), sizeof(int64_t), c->s_compute, &err);
    if (e != cudaSuccess) { g_nccl_err = err; return fail_cuda(e, "count"); }
    *total = 0;
    for (int64_t v : all) *total += v;
    return BDF_OK;
}

static int aggregate_dev(bdf_ctx* c, int op, bdf_col* col, void* out_scalar, int32_t* is_some) {
    if (op < 0 || op >= BDF_NAGG) return fail(BDF_INVALID, "invalid aggregate op %d", op);
    const int dtype = col->dtype;
    const int w = dtype_width(dtype);
    if (op == BDF_COUNT) {  // metadata only, as in the reference (aggregate.rs:70-80)
        TRY(ensure_null_counts(c, col));
        int64_t total = 0;
        for (size_t i = 0; i < col->chunks.size(); i++) total += col->chunks[i].len - col->null_counts[i];
        TRY(count_global(c, &total));
        *(int64_t*)out_scalar = total;
        *is_some = 1;
        return BDF_OK;
    }
    if ((op == BDF_MIN || op == BDF_MAX) && dtype_is_float(dtype))
        return fail(BDF_UNSUPPORTED, "min/max need T::Native: Ord (integers only)");
    bdf_agg4 a;
    TRY(aggregate_all_dev(c, col, op != BDF_SUM, &a));
    if (op == BDF_SUM) {
        memcpy(out_scalar, &a.sum, (size_t)w);
        *is_some = 1;
        return BDF_OK;
    }
    if (a.would_panic) return fail(BDF_WOULD_PANIC, "max/min on an empty or all-null chunk: the reference unwraps None");
    *is_some = a.n_chunks == 0 ? 0 : 1;   // Iterator::max of an empty Vec is None
    if (*is_some) memcpy(out_scalar, op == BDF_MIN ? &a.min : &a.max, (size_t)w);
    return BDF_OK;
}

// avg (aggregate.rs:32-65): per-chunk mean from an exact/double sum and the valid count, then the
// reference's weighted merge in chunk order.
static int avg_dev(bdf_ctx* c, bdf_col* col, double* out, int32_t* is_some) {
    const int dtype = col->dtype;
    if (dtype == BDF_I64 || dtype == BDF_U64) return fail(BDF_UNSUPPORTED, "avg needs f64: From<T::Native>");
    const int64_t n = (int64_t)col->chunks.size();
    wait_groups(c->s_compute, col, 0, n);
    double mean = 0.0;
    int64_t count = 0;
    for (int64_t k = 0; k < n; k += kAggSlots) {
        const int64_t m = std::min<int64_t>(kAggSlots, n - k);
        for (int64_t j = 0; j < m; j++) TRY(reduce_range(c, col, k + j, k + j + 1, c->h_agg_dev + j));
        CK(cudaStreamSynchronize(c->s_compute));
        for (int64_t j = 0; j < m; j++) {
            const AggDev& a = c->h_agg[j];
            const int64_t len = (int64_t)a.count;
            double s;
            if (dtype_is_float(dtype)) memcpy(&s, &a.sum_bits, 8);
            else if (dtype_is_signed_int(dtype)) s = (double)(int64_t)a.sum_bits;
            else s = (double)a.sum_bits;
            const double mch = len ? s / (double)len : 0.0;
            // A rank of a communicator sees only SOME chunks of the column: an empty local chunk contributes nothing there
            // (the reference's 0/0 = NaN when the column's FIRST chunk has no valid slot is a statement about the whole
            // column's chunk order; the one-GPU context and the multi-GPU context reproduce it, see fleet_avg_dev).
            if (len == 0 && is_global(c)) continue;
            count += len;
            mean = mean + ((mch - mean) * (double)len) / (double)count;
        }
    }
    if (is_global(c)) {
        // The reference merges per-chunk means in chunk order (aggregate.rs:44-63); the chunks of the other ranks are
        // merged as one (mean, count) pair per rank, in rank order, with the same formula.
        struct Pair { double mean; int64_t count; } mine{mean, count};
        std::vector<Pair> all((size_t)comm_world(c->comm));
        std::string err;
        c->collectives++;
        cudaError_t e = comm_host_allgather(c->comm, &mine, all.data(), sizeof(Pair), c->s_compute, &err);
        if (e != cudaSuccess) { g_nccl_err = err; return fail_cuda(e, "avg"); }
        mean = 0.0; count = 0;
        for (const Pair& p : all) {
            if (!p.count) continue;
            count += p.count;
            mean = mean + ((p.mean - mean) * (double)p.count) / (double)count;
        }
    }
    *is_some = count != 0;
    *out = mean;
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// N2: BooleanFilter comparisons, boolean kernels, filter (k_filter.cu)

// BooleanFilter::{Gt,..,Le}: cast both sides to Float64 (as the reference does, expression.rs:820-845), compare.  The casts are
// fused into the kernel's loads.
static int compare_dev(bdf_ctx* c, int op, const bdf_col* l, const bdf_col* r, double scalar, bdf_col** out) {
    if (op < 0 || op > 5) return fail(BDF_INVALID, "invalid comparison op %d", op);
    if (l->dtype == kBool || (r && r->dtype == kBool)) return fail(BDF_UNSUPPORTED, "comparison of boolean columns is not part of this path");
    const bdf_col* in[] = {l, r};
    int64_t n = 0;
    TRY(zip_chunks(in, r ? 2 : 1, &n));
    std::vector<ChunkPlan> plan((size_t)n);
    for (int64_t i = 0; i < n; i++) plan[i] = {l->chunks[i].len, l->chunks[i].validity != nullptr || (r && r->chunks[i].validity != nullptr)};
    const int wrow = dtype_width(l->dtype) + (r ? dtype_width(r->dtype) : 0);
    return launch_groups(c, {l, r}, {n}, kBool, plan, compare_tile_elems(), sizeof(BinDesc), BDF_K_COMPARE, "compare",
        [&](void* hd, int64_t i, int64_t tile0, const DevChunk& oc) {
            const DevChunk& a = l->chunks[i];
            const DevChunk* b = r ? &r->chunks[i] : nullptr;
            ((BinDesc*)hd)[i] = BinDesc{a.values, b ? b->values : nullptr, oc.values, a.validity, b ? b->validity : nullptr, oc.validity, a.len, tile0,
                                        a.bit_off, b ? b->bit_off : 0};
            return wrow * a.len + bitmap_bytes(a.len) * (1 + (a.validity ? 1 : 0) + (b && b->validity ? 1 : 0) + (oc.validity ? 1 : 0));
        },
        [&](const void* dd, int64_t begin, int64_t end, int64_t tiles, int64_t, uint32_t* wc) {
            return launch_compare(op, (const BinDesc*)dd, (int)(end - begin), tiles, l->dtype, r ? r->dtype : BDF_F64, r == nullptr, scalar, wc, c->s_compute);
        },
        out);
}

static int boolean_dev(bdf_ctx* c, int op, const bdf_col* a, const bdf_col* b, bdf_col** out) {
    if (op < 0 || op > 2) return fail(BDF_INVALID, "invalid boolean op %d", op);
    if (a->dtype != kBool || (op != 2 && (!b || b->dtype != kBool))) return fail(BDF_UNSUPPORTED, "and/or/not need boolean columns");
    if (op == 2) b = nullptr;
    const bdf_col* in[] = {a, b};
    int64_t n = 0;
    TRY(zip_chunks(in, b ? 2 : 1, &n));
    std::vector<ChunkPlan> plan((size_t)n);
    for (int64_t i = 0; i < n; i++) plan[i] = {a->chunks[i].len, a->chunks[i].validity != nullptr || (b && b->chunks[i].validity != nullptr)};
    int64_t rows = 0;
    return launch_groups(c, {a, b}, {n}, kBool, plan, bool_tile_elems(), bool_desc_size(), BDF_K_COMPARE, "boolean op",
        [&](void* hd, int64_t i, int64_t tile0, const DevChunk& oc) {
            const DevChunk& x = a->chunks[i];
            const DevChunk* y = b ? &b->chunks[i] : nullptr;
            fill_bool_desc(hd, i, (const uint32_t*)x.values, y ? (const uint32_t*)y->values : nullptr, (uint32_t*)oc.values, x.validity,
                           y ? y->validity : nullptr, oc.validity, x.len, tile0, x.val_bit_off, y ? y->val_bit_off : 0, x.bit_off, y ? y->bit_off : 0);
            // the record counts (rows / 8) * (2 or 3) bytes for the whole launch: each chunk adds its step of rows / 8
            const int64_t before = rows / 8;
            rows += x.len;
            return (rows / 8 - before) * (b ? 3 : 2);
        },
        [&](const void* dd, int64_t begin, int64_t end, int64_t tiles, int64_t, uint32_t* wc) {
            return launch_boolean(op, dd, (int)(end - begin), tiles, wc, c->s_compute);
        },
        out);
}

// ---------------------------------------------------------------------------------------------------
// Null handling and conditional selection (k_cond.cu): coalesce, greatest, least, nanvl, case_when, is_null / is_nan

static constexpr int kCondMaxArgs = 64;

// The checks of a row-wise call, shared by the one-GPU and multi-GPU forms and made before any device work.  *dtype: the type of
// the value columns (they give the result type, so at least one value must be a column).
static int cond_check(int fn, int32_t n_conds, const bdf_col* const* conds, int32_t n_vals, const bdf_arg* vals, int* dtype) {
    *dtype = -1;
    for (int32_t k = 0; k < n_conds; k++) {
        if (!conds[k]) return fail(BDF_INVALID, "null condition %d", (int)k);
        if (conds[k]->dtype != kBool) return fail(BDF_INVALID, "condition %d is not a Boolean column", (int)k);
    }
    for (int32_t k = 0; k < n_vals; k++) {
        const bdf_col* col = vals[k].column;
        if (!col) continue;
        if (*dtype < 0) *dtype = col->dtype;
        else if (col->dtype != *dtype) return fail(BDF_INVALID, "arguments of different types (%d, %d): cast them first", *dtype, col->dtype);
    }
    if (*dtype < 0) return fail(BDF_INVALID, "no value argument is a column, so nothing gives the result type");
    if (*dtype == kBool && fn != BDF_ROW_COALESCE) return fail(BDF_UNSUPPORTED, "greatest / least / nanvl of Boolean columns");
    if (fn == BDF_ROW_NANVL && !dtype_is_float(*dtype)) return fail(BDF_UNSUPPORTED, "nanvl needs Float32 or Float64 arguments");
    for (int32_t k = 0; k < n_vals; k++)
        if (*dtype == kBool && !vals[k].column && vals[k].valid && vals[k].bits > 1)
            return fail(BDF_INVALID, "a Boolean scalar is 0 or 1, not %llu", (unsigned long long)vals[k].bits);
    return BDF_OK;
}

// Every column of the call: the conditions, then the value columns in argument order.
static std::vector<const bdf_col*> cond_columns(int32_t n_conds, const bdf_col* const* conds, int32_t n_vals, const bdf_arg* vals) {
    std::vector<const bdf_col*> cols(conds, conds + n_conds);
    for (int32_t k = 0; k < n_vals; k++)
        if (vals[k].column) cols.push_back(vals[k].column);
    return cols;
}

static CondArg cond_arg(const DevChunk* ch, const bdf_arg& v) {
    if (ch) return CondArg{ch->values, ch->validity, 0ull, (int16_t)ch->bit_off, (int16_t)ch->val_bit_off, COND_COLUMN};
    return CondArg{nullptr, nullptr, v.valid ? (unsigned long long)v.bits : 0ull, 0, 0, v.valid ? COND_SCALAR : COND_NULL};
}

// fn: bdf_row_fn; a case_when is a COALESCE with n_conds = n_vals - 1 conditions (the last value is the else).
static int cond_dev(bdf_ctx* c, int fn, int32_t n_conds, const bdf_col* const* conds, int32_t n_vals, const bdf_arg* vals, bdf_col** out) {
    int dtype = 0;
    TRY(cond_check(fn, n_conds, conds, n_vals, vals, &dtype));
    const std::vector<const bdf_col*> cols = cond_columns(n_conds, conds, n_vals, vals);
    int64_t n = 0;
    TRY(zip_chunks(cols.data(), (int)cols.size(), &n));
    bool null_literal = false;
    for (int32_t k = 0; k < n_vals; k++) null_literal = null_literal || (!vals[k].column && !vals[k].valid);
    std::vector<ChunkPlan> plan((size_t)n);
    for (int64_t i = 0; i < n; i++) {
        bool nullable = null_literal;
        for (int32_t k = 0; k < n_vals; k++) nullable = nullable || (vals[k].column && vals[k].column->chunks[i].validity);
        plan[i] = {cols[0]->chunks[i].len, nullable};
    }
    const int n_args = n_conds + n_vals;
    const size_t stride = cond_desc_bytes(n_args);
    const int64_t w = dtype == kBool ? 0 : dtype_width(dtype);
    int64_t value_cols = 0;
    for (int32_t k = 0; k < n_vals; k++) value_cols += vals[k].column ? 1 : 0;
    // the launch record's bytes: one value read per row for a selection (every value column for greatest / least), the write, and
    // every bitmap read and written
    const int64_t reads = (fn == BDF_ROW_GREATEST || fn == BDF_ROW_LEAST) ? value_cols : 1;
    // grouped as the other element-wise operators: a group starts once its own chunks of every input have landed
    return launch_groups(c, cols.data(), cols.size(), plan_groups(c, n, cols.data(), cols.size()), dtype, plan, cond_tile_elems(dtype), stride, BDF_K_BINARY, "row-wise selection",
        [&](void* hd, int64_t i, int64_t tile0, const DevChunk& oc) {
            const int64_t len = plan[i].len;
            CondHead* h = (CondHead*)((char*)hd + i * stride);
            *h = CondHead{oc.values, oc.validity, len, tile0, n_conds, n_vals, 0};
            CondArg* a = (CondArg*)(h + 1);
            int64_t bitmaps = (oc.validity ? 1 : 0) + (dtype == kBool ? 1 + reads : 0);
            for (int32_t k = 0; k < n_conds; k++) {
                const DevChunk& ch = conds[k]->chunks[i];
                a[k] = cond_arg(&ch, bdf_arg{});
                bitmaps += 1 + (ch.validity ? 1 : 0);
            }
            for (int32_t k = 0; k < n_vals; k++) {
                const DevChunk* ch = vals[k].column ? &vals[k].column->chunks[i] : nullptr;
                a[n_conds + k] = cond_arg(ch, vals[k]);
                bitmaps += ch && ch->validity ? 1 : 0;
            }
            return (reads + 1) * w * len + bitmaps * bitmap_bytes(len);
        },
        [&](const void* dd, int64_t begin, int64_t end, int64_t tiles, int64_t, uint32_t* wc) {
            return launch_cond(fn, dtype, dd, n_args, (int)(end - begin), tiles, wc, c->s_compute);
        },
        out);
}

static int null_test_dev(bdf_ctx* c, int test, const bdf_col* in, bdf_col** out) {
    const int64_t n = (int64_t)in->chunks.size();
    std::vector<ChunkPlan> plan((size_t)n);
    for (int64_t i = 0; i < n; i++) plan[i] = {in->chunks[i].len, false};
    const size_t stride = cond_desc_bytes(1);
    const bool reads_values = test == BDF_IS_NAN && dtype_is_float(in->dtype);
    const int64_t w = reads_values ? dtype_width(in->dtype) : 0;
    return launch_groups(c, {in}, plan_groups(c, n, {in}), kBool, plan, null_test_tile_elems(in->dtype, test), stride, BDF_K_COMPARE, "null test",
        [&](void* hd, int64_t i, int64_t tile0, const DevChunk& oc) {
            const DevChunk& ch = in->chunks[i];
            CondHead* h = (CondHead*)((char*)hd + i * stride);
            *h = CondHead{oc.values, nullptr, ch.len, tile0, 0, 1, 0};
            *(CondArg*)(h + 1) = cond_arg(&ch, bdf_arg{});
            return w * ch.len + (1 + (ch.validity ? 1 : 0)) * bitmap_bytes(ch.len);
        },
        [&](const void* dd, int64_t begin, int64_t end, int64_t tiles, int64_t, uint32_t*) {
            return launch_null_test(test, in->dtype, dd, (int)(end - begin), tiles, c->s_compute);
        },
        out);
}

// ChunkedArray::filter: arrow compute::filter(chunk, mask chunk) for every chunk pair (src/table.rs:97-107).
static int filter_dev(bdf_ctx* c, const bdf_col* values, const bdf_col* mask, bdf_col** out) {
    if (mask->dtype != kBool) return fail(BDF_INVALID, "the filter mask must be a boolean column");
    if (values->dtype == kBool) return fail(BDF_UNSUPPORTED, "filtering a boolean column is not part of this path");
    const int64_t n = std::min<int64_t>((int64_t)values->chunks.size(), (int64_t)mask->chunks.size());  // zip()
    for (int64_t i = 0; i < n; i++)
        if (values->chunks[i].len != mask->chunks[i].len)
            return fail(BDF_LENGTH_MISMATCH, "Filter array must have the same length as the data");
    const int dtype = values->dtype;
    const int tile = elems_per_tile(dtype);
    int64_t tiles = 0, rows = 0;
    std::vector<int64_t> tile0((size_t)n + 1, 0);
    for (int64_t i = 0; i < n; i++) { tile0[i] = tiles; tiles += (values->chunks[i].len + tile - 1) / tile; rows += values->chunks[i].len; }
    void *hp = nullptr, *dp = nullptr;
    TRY(ring_alloc(c, (size_t)n * filter_desc_size(), &hp, &dp));
    Scratch<unsigned int> d_counts;
    Scratch<long long> d_offsets, d_totals;
    cudaError_t e = d_counts.alloc(c, std::max<size_t>(1, (size_t)tiles) * sizeof(unsigned int));
    if (e == cudaSuccess) e = d_offsets.alloc(c, std::max<size_t>(1, (size_t)tiles) * sizeof(long long));
    if (e == cudaSuccess) e = d_totals.alloc(c, std::max<size_t>(1, (size_t)n) * sizeof(long long));
    if (e != cudaSuccess) return fail_cuda(e, "filter scratch allocation");
    // pass 1: counts + scan (output pointers are not needed yet)
    for (int64_t i = 0; i < n; i++) {
        const DevChunk &v = values->chunks[i], &m = mask->chunks[i];
        fill_filter_desc(hp, i, v.values, nullptr, v.validity, nullptr, (const uint32_t*)m.values, m.validity, v.len, tile0[i], v.bit_off, m.val_bit_off, m.bit_off);
    }
    wait_groups(c->s_compute, values, 0, n);
    wait_groups(c->s_compute, mask, 0, n);
    e = desc_upload(c, dp, hp, (size_t)n * filter_desc_size());
    std::vector<long long> totals((size_t)std::max<int64_t>(n, 1), 0);
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_FILTER, dtype, rows, rows / 4);
        c->launches++;  // count + scan
        e = launch_filter_count(dp, (int)n, tiles, tile, d_counts, d_offsets, d_totals, c->s_compute);
    }
    if (e == cudaSuccess && n) e = cudaMemcpyAsync(totals.data(), d_totals, (size_t)n * sizeof(long long), cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);  // output lengths are needed to size the result
    if (e != cudaSuccess) return fail_cuda(e, "filter (count)");
    std::vector<ChunkPlan> plan((size_t)n);
    int64_t kept = 0;
    for (int64_t i = 0; i < n; i++) { plan[i] = {(int64_t)totals[i], values->chunks[i].validity != nullptr}; kept += totals[i]; }
    ColOwner o(c);
    TRY(col_alloc(c, dtype, plan, nullptr, 0, o.out()));
    for (int64_t i = 0; i < n; i++) o->null_counts[i] = o->chunks[i].validity ? -1 : 0;  // counted on demand
    // pass 2: scatter
    void *hp2 = nullptr, *dp2 = nullptr;
    TRY(ring_alloc(c, (size_t)n * filter_desc_size(), &hp2, &dp2));
    for (int64_t i = 0; i < n; i++) {
        const DevChunk &v = values->chunks[i], &m = mask->chunks[i], &oc = o->chunks[i];
        fill_filter_desc(hp2, i, v.values, oc.values, v.validity, oc.validity, (const uint32_t*)m.values, m.validity, v.len, tile0[i], v.bit_off, m.val_bit_off, m.bit_off);
    }
    e = desc_upload(c, dp2, hp2, (size_t)n * filter_desc_size());
    if (e == cudaSuccess) {
        const int w = dtype_width(dtype);
        LaunchTimer t(c, BDF_K_FILTER, dtype, rows, rows * w + kept * w + rows / 4);
        e = launch_filter_scatter(dtype, dp2, (int)n, tiles, d_offsets, c->s_compute);
    }
    if (e == cudaSuccess) e = finish_single_group(c, o.get());
    if (e != cudaSuccess) return fail_cuda(e, "filter (scatter)");
    *out = o.release();
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// N3: a chain of Calculations fused into one pass (k_expr.cu)

// Validation + host compilation of a fused program (shared by the evaluation entry and bdf_expr_check; needs no device).
static int expr_prepare(int n_inputs, const int* in_dtypes, int n_nodes, const bdf_expr_node* nodes, unsigned char (&prog)[256], bool* has_div) {
    if (n_inputs < 1 || n_inputs > expr_max_inputs()) return fail(BDF_INVALID, "an expression takes 1..%d input columns", expr_max_inputs());
    if (n_nodes < 1 || n_nodes > expr_max_nodes()) return fail(BDF_INVALID, "an expression has 1..%d nodes", expr_max_nodes());
    std::vector<int> op(n_nodes), a(n_nodes), b(n_nodes);
    *has_div = false;
    for (int k = 0; k < n_nodes; k++) {
        op[k] = nodes[k].op; a[k] = nodes[k].a; b[k] = nodes[k].b;
        const bool unary = op[k] >= BDF_EXPR_UNARY;
        if (unary ? (op[k] - BDF_EXPR_UNARY >= BDF_NUNARY) : (op[k] < 0 || op[k] >= BDF_NBINARY)) return fail(BDF_INVALID, "node %d: invalid op %d", k, op[k]);
        if (a[k] < 0 || a[k] >= n_inputs + k || (!unary && (b[k] < 0 || b[k] >= n_inputs + k)))
            return fail(BDF_INVALID, "node %d refers to a slot that is not computed yet", k);
        if (unary) b[k] = a[k];
        *has_div = *has_div || op[k] == BDF_DIV;
    }
    static_assert(sizeof(prog) >= 8 + 2 * 40, "ExprProg must fit");
    if (expr_prog_size() > sizeof(prog)) return fail(BDF_INVALID, "internal: expression program too large");
    for (int i = 0; i < n_inputs; i++)
        if (in_dtypes[i] < 0 || in_dtypes[i] >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "fused expressions take numeric columns");
    switch (expr_compile(n_inputs, in_dtypes, n_nodes, op.data(), a.data(), b.data(), prog)) {
        case 0: return BDF_OK;
        case 1: return fail(BDF_INVALID, "a node's result is never used: the materialised chain would still evaluate it, split the expression");
        case 2: return fail(BDF_UNSUPPORTED, "the expression keeps more than two intermediates alive at once: split it");
        default: return fail(BDF_UNSUPPORTED, "the expression is too long to fuse: split it");
    }
}

// out == nullptr (only with fut): aggregate only, the result column is never written.
static int expr_dev(bdf_ctx* c, int n_inputs, const bdf_col* const* inputs, int n_nodes, const bdf_expr_node* nodes, bdf_col** out,
                    bdf_future** fut = nullptr) {
    if (!inputs) return fail(BDF_INVALID, "null argument");
    int in_dtypes[8] = {0};
    for (int i = 0; i < n_inputs && i < 8; i++) {
        if (!inputs[i]) return fail(BDF_INVALID, "null input column");
        in_dtypes[i] = inputs[i]->dtype;
    }
    alignas(8) unsigned char prog[256];
    bool has_div = false;
    TRY(expr_prepare(n_inputs, in_dtypes, n_nodes, nodes, prog, &has_div));
    for (int i = 0; i < n_inputs; i++)
        if (!inputs[i]) return fail(BDF_INVALID, "null input column");
    int64_t n = 0;
    TRY(zip_chunks(inputs, n_inputs, &n));
    std::vector<ChunkPlan> plan((size_t)n);
    for (int64_t ch = 0; ch < n; ch++) {
        bool hv = false;
        for (int i = 0; i < n_inputs; i++) hv = hv || inputs[i]->chunks[ch].validity != nullptr;
        plan[ch] = {inputs[0]->chunks[ch].len, hv};
    }
    const int tile = expr_tile_elems();
    ColOwner o(c);
    if (out) {
        TRY(col_alloc(c, BDF_F64, plan, nullptr, tile, o.out()));
        o->counts_on_device = o->d_warp_counts != nullptr;
    }
    int64_t total_tiles = 0, total_rows = 0;
    for (int64_t ch = 0; ch < n; ch++) { total_tiles += (plan[ch].len + tile - 1) / tile; total_rows += plan[ch].len; }
    void *hp = nullptr, *dp = nullptr;
    TRY(ring_alloc(c, (size_t)n * expr_desc_size(), &hp, &dp));
    cudaError_t e = cudaSuccess;
    FutOwner f(c);
    bdf_ctx::PartBuf* pb = nullptr;
    if (fut) {
        TRY(future_new(c, BDF_F64, 1, total_rows, f.out()));
        e = part_acquire(c, total_tiles, &pb);
    }
    cudaEvent_t ev_done = nullptr;   // the launch's completion on the compute stream, for the finish stream
    if (e == cudaSuccess) {
        int64_t tiles = 0, bytes = 0;
        for (int64_t ch = 0; ch < n; ch++) {
            const void* in[8]; const uint32_t* vin[8]; int32_t off[8];
            const int64_t len = plan[ch].len;
            for (int i = 0; i < n_inputs; i++) {
                const DevChunk& x = inputs[i]->chunks[ch];
                in[i] = x.values; vin[i] = x.validity; off[i] = x.bit_off;
                if ((uintptr_t)x.values & 15) e = cudaErrorMisalignedAddress;
                bytes += (int64_t)dtype_width(inputs[i]->dtype) * x.len + (x.validity ? bitmap_bytes(x.len) : 0);
            }
            double* po = o.get() ? (double*)o->chunks[ch].values : nullptr;
            uint32_t* vo = o.get() ? o->chunks[ch].validity : nullptr;
            fill_expr_desc(hp, ch, n_inputs, in, vin, off, po, vo, len, tiles);
            tiles += (len + tile - 1) / tile;
            if (o.get()) bytes += 8 * len + (vo ? bitmap_bytes(len) : 0);
        }
        for (int i = 0; i < n_inputs; i++) wait_groups(c->s_compute, inputs[i], 0, n);
        if (e == cudaSuccess) e = desc_upload(c, dp, hp, (size_t)n * expr_desc_size());
        if (e == cudaSuccess && has_div) e = cudaMemsetAsync(c->d_flag, 0, sizeof(int), c->s_compute);
        if (e == cudaSuccess) {
            LaunchTimer t(c, BDF_K_EXPR, BDF_F64, total_rows, bytes);
            e = launch_expr(dp, (int)n, total_tiles, prog, o.get() ? o->d_warp_counts : nullptr, c->d_flag, pb ? pb->p : nullptr, c->s_compute);
        }
        if (e == cudaSuccess && o.get()) e = finish_single_group(c, o.get());
        if (e == cudaSuccess && f.get()) {
            e = ev_get(c, &ev_done);
            if (e == cudaSuccess) e = cudaEventRecord(ev_done, c->s_compute);
            if (e == cudaSuccess) e = cudaStreamWaitEvent(c->s_fin, ev_done, 0);
            if (e == cudaSuccess) e = fused_finish(c, f.get(), pb, total_tiles, n);
            if (ev_done) ev_put(c, ev_done);
        }
    }
    int flag = 0;
    if (e == cudaSuccess && has_div) e = flag_read(c, is_global(c), &flag);
    if (e != cudaSuccess) return fail_cuda(e, "fused expression");
    if (flag) return fail(BDF_DIVIDE_BY_ZERO, "Divide by zero error");
    if (out) *out = o.release();
    if (fut) *fut = f.release();
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// DataFrame::sort = lexsort_to_indices + take (k_sort.cu)

// The chunk table of a column in the concatenated row space (descriptor ring, uploaded on the descriptor stream).
static int sort_table(bdf_ctx* c, const bdf_col* col, void** dev, int* n_chunks, bool* nullable) {
    const int64_t n = (int64_t)col->chunks.size();
    void* hp = nullptr;
    TRY(ring_alloc(c, (size_t)std::max<int64_t>(n, 1) * sort_chunk_size(), &hp, dev));
    int64_t start = 0;
    bool any = false;
    for (int64_t i = 0; i < n; i++) {
        const DevChunk& ch = col->chunks[i];
        fill_sort_chunk(hp, i, ch.values, ch.validity, start, ch.bit_off, ch.val_bit_off);
        start += ch.len;
        any = any || ch.validity != nullptr;
    }
    if (n == 0) fill_sort_chunk(hp, 0, nullptr, nullptr, 0, 0, 0);
    wait_groups(c->s_compute, col, 0, n);
    cudaError_t e = desc_upload(c, *dev, hp, (size_t)std::max<int64_t>(n, 1) * sort_chunk_size());
    if (e != cudaSuccess) return fail_cuda(e, "descriptor upload");
    *n_chunks = (int)std::max<int64_t>(n, 1);
    if (nullable) *nullable = any;
    return BDF_OK;
}

// The checks of the sort's criteria, shared with top-k.
static int sort_check(int n_keys, const bdf_sort_key* keys) {
    if (n_keys < 1) return fail(BDF_INVALID, "Sort criteria cannot be empty");
    for (int k = 0; k < n_keys; k++) {
        if (!keys[k].column) return fail(BDF_INVALID, "null sort column");
        const int dt = keys[k].column->dtype;
        if (dt < 0 || dt >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "sort criteria must be numeric columns");
        if (keys[k].column->total_len != keys[0].column->total_len) return fail(BDF_LENGTH_MISMATCH, "sort columns have different lengths");
    }
    if (keys[0].column->total_len > 0xffffffffLL) return fail(BDF_UNSUPPORTED, "sort indices are UInt32: at most 2^32-1 rows");
    return BDF_OK;
}

static int sort_indices_dev(bdf_ctx* c, int n_keys, const bdf_sort_key* keys, bdf_col** out) {
    TRY(sort_check(n_keys, keys));
    const int64_t n = keys[0].column->total_len;
    ColOwner o(c);
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{n, false}}, nullptr, sort_tile_elems(), o.out()));
    cudaError_t e = cudaSuccess;
    int st = BDF_OK;
    if (n > 0) {
        Scratch<unsigned long long> kbuf[2];
        Scratch<uint32_t> ibuf[2];
        Scratch<unsigned int> block_hist;
        Scratch<unsigned long long> agree;   // [0] OR, [1] AND of the keys of the current criterion
        if (!c->h_sort_agree) e = cudaHostAlloc((void**)&c->h_sort_agree, 2 * sizeof(unsigned long long), cudaHostAllocDefault);
        for (int b = 0; b < 2 && e == cudaSuccess; b++) {
            e = kbuf[b].alloc(c, (size_t)n * 8);
            if (e == cudaSuccess) e = ibuf[b].alloc(c, (size_t)n * 4);
        }
        if (e == cudaSuccess) e = block_hist.alloc(c, (size_t)256 * sort_pass_ctas(n, c->sm_count) * sizeof(unsigned int));
        if (e == cudaSuccess) e = agree.alloc(c, 2 * sizeof(unsigned long long));
        int cur = 0;
        int64_t passes = 0, pass_bytes = 0;
        if (e == cudaSuccess) {
            LaunchTimer t(c, BDF_K_SORT, keys[0].column->dtype, n, 0);
            e = launch_iota(ibuf[0], n, c->sm_count, c->s_compute);
            for (int k = n_keys - 1; k >= 0 && e == cudaSuccess && st == BDF_OK; k--) {
                const bdf_col* col = keys[k].column;
                void* table = nullptr; int nch = 0; bool nullable = false;
                st = sort_table(c, col, &table, &nch, &nullable);
                for (int mode = 0; mode < (nullable ? 2 : 1) && e == cudaSuccess && st == BDF_OK; mode++) {
                    e = cudaMemsetAsync(agree, 0, sizeof(unsigned long long), c->s_compute);
                    if (e == cudaSuccess) e = cudaMemsetAsync(agree + 1, 0xff, sizeof(unsigned long long), c->s_compute);
                    if (e == cudaSuccess) e = launch_sort_keys(col->dtype, table, nch, ibuf[cur], n, mode, keys[k].descending != 0, kbuf[cur], agree, c->sm_count, c->s_compute);
                    if (e == cudaSuccess) e = cudaMemcpyAsync(c->h_sort_agree, agree, 2 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->s_compute);
                    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
                    const int digits = mode ? 1 : dtype_width(col->dtype);
                    const unsigned long long differ = e == cudaSuccess ? (c->h_sort_agree[0] ^ c->h_sort_agree[1]) : 0ull;   // bits that are not the same in all keys
                    for (int d = 0; d < digits && e == cudaSuccess; d++) {
                        if (((differ >> (8 * d)) & 0xff) == 0) continue;   // every key has the same digit: the pass would be the identity
                        const int kb = sort_key_bytes(col->dtype);
                        e = launch_radix_pass(kb, kbuf[cur], ibuf[cur], n, 8 * d, block_hist, kbuf[cur ^ 1], ibuf[cur ^ 1], c->sm_count, c->s_compute);
                        cur ^= 1;
                        passes++;
                        pass_bytes += (int64_t)(3 * kb + 8) * n;   // histogram read + keys and indices read and written
                    }
                }
            }
            if (e == cudaSuccess && st == BDF_OK)
                e = cudaMemcpyAsync(o->chunks[0].values, ibuf[cur], (size_t)n * 4, cudaMemcpyDeviceToDevice, c->s_compute);
            c->last_sort_passes = passes;
        }
        if (c->profiling && !c->prof.empty() && c->prof.back().rec.kernel == BDF_K_SORT) c->prof.back().rec.bytes = 8 * n + pass_bytes + 4 * n;
    }
    TRY(st);
    if (e == cudaSuccess) e = finish_single_group(c, o.get());
    if (e != cudaSuccess) return fail_cuda(e, "sort");
    *out = o.release();
    return BDF_OK;
}

static int col_borrow(int dtype, const std::vector<DevChunk>& chunks, bdf_col** out);

// keep_chunks: chunk k of the result is the take of index chunk k (one launch per chunk) instead of one chunk for all indices.
static int take_dev(bdf_ctx* c, const bdf_col* values, const bdf_col* indices, bdf_col** out, bool keep_chunks = false) {
    if (indices->dtype != BDF_U32) return fail(BDF_UNSUPPORTED, "take indices must be a UInt32 column");
    const int64_t n = indices->total_len;
    void *vt = nullptr, *it = nullptr;
    int nv = 0, ni = 0;
    bool vnull = false, inull = false;
    TRY(sort_table(c, values, &vt, &nv, &vnull));
    TRY(sort_table(c, indices, &it, &ni, &inull));
    ColOwner o(c);
    std::vector<ChunkPlan> plan;
    if (keep_chunks) for (const DevChunk& ch : indices->chunks) plan.push_back(ChunkPlan{ch.len, vnull || inull});
    else plan.push_back(ChunkPlan{n, vnull || inull});
    TRY(col_alloc(c, values->dtype, plan, nullptr, take_tile_elems(), o.out()));
    o->counts_on_device = o->d_warp_counts != nullptr;
    cudaError_t e = cudaMemsetAsync(c->d_flag, 0, sizeof(int), c->s_compute);
    if (e == cudaSuccess) {
        const int w = values->dtype == kBool ? 1 : dtype_width(values->dtype);
        LaunchTimer t(c, BDF_K_TAKE, values->dtype, n, n * (4 + 2 * (int64_t)w));
        if (!keep_chunks)
            e = launch_take(values->dtype, vt, nv, it, ni, n, values->total_len, o->chunks[0].values, o->chunks[0].validity, o->d_warp_counts, c->d_flag,
                            c->s_compute);
        for (size_t k = 0; keep_chunks && k < plan.size() && e == cudaSuccess; k++) {
            if (!plan[k].len) continue;
            ColOwner one(c);
            void* kt = nullptr;
            int nk = 0;
            int st = col_borrow(BDF_U32, {indices->chunks[k]}, one.out());
            if (st == BDF_OK) st = sort_table(c, one.get(), &kt, &nk, nullptr);
            if (st != BDF_OK) return st;
            const DevChunk& oc = o->chunks[k];
            e = launch_take(values->dtype, vt, nv, kt, nk, plan[k].len, values->total_len, oc.values, oc.validity,
                            o->d_warp_counts ? o->d_warp_counts + o->tile0[k] * kWarpsPerCta : nullptr, c->d_flag, c->s_compute);
        }
    }
    if (e == cudaSuccess) e = finish_single_group(c, o.get());
    int flag = 0;
    if (e == cudaSuccess) e = flag_read(c, false, &flag);
    if (e != cudaSuccess) return fail_cuda(e, "take");
    if (flag) return fail(BDF_INVALID, "take: index out of bounds");
    *out = o.release();
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// top-k = the first k rows of DataFrame::sort, chosen by a radix select of the sort keys (k_topk.cu)
//   Rounds, one per criterion, over a tie set (round 0: every row; later: the ascending row ids that tie on every earlier criterion)
//   and `need`, the rows still to choose.  select_keys finds the key t of rank need - 1 (ascending) or v - need (descending) among
//   the v valid keys of the tie set; k_topk_mark ORs the rows before t into the chosen bitmap and marks the rows equal to t.  When
//   need > v every valid row is chosen and the nulls are the ties.  Once the ties hold exactly the rows still needed, or the last
//   criterion is reached, the first `need` ties in row order are chosen: rows equal on every criterion keep row order, as in the
//   stable sort.  The chosen rows (ascending) are then sorted on their gathered criteria and mapped back.

static int select_keys(bdf_ctx* c, const bdf_col* col, const std::function<std::vector<int64_t>(int64_t)>& ranks_of, int max_targets,
                       std::vector<uint64_t>* keys, int64_t* n_valid);

// k above this share of the rows: one sort of all rows costs less than the rounds plus a sort of k rows (DESIGN §8).
constexpr int64_t kTopkSortNum = 5, kTopkSortDen = 8;

// A Boolean column over a bitmap the caller owns (bit 0 is row 0).
static int bits_borrow(uint32_t* words, int64_t n, bdf_col** out) { return col_borrow(kBool, {DevChunk{(char*)words, nullptr, n, 0, 0}}, out); }

// One mark pass over col: positional (ids null: the tie set is every row, chunk by chunk) or over one gathered chunk whose position i
// is row ids[i].  tie: a bitmap over col's positions.  counts: BEFORE, TIE.
static int topk_mark(bdf_ctx* c, const bdf_col* col, const uint32_t* ids, uint64_t t, bool all_valid, bool descending, uint32_t* chosen, uint32_t* tie,
                     unsigned long long* d_counts, int64_t counts[2]) {
    const int64_t nch = (int64_t)col->chunks.size(), n = col->total_len;
    const int tile = topk_tile_elems(col->dtype);
    void *hp = nullptr, *dp = nullptr;
    TRY(ring_alloc(c, (size_t)std::max<int64_t>(nch, 1) * topk_chunk_size(), &hp, &dp));
    int64_t tiles = 0, row0 = 0;
    for (int64_t i = 0; i < nch; i++) {
        const DevChunk& ch = col->chunks[i];
        const int64_t end = row0 + ch.len;
        fill_topk_chunk(hp, i, ch.values, ch.validity, ch.len, tiles, row0, ch.bit_off, row0 % 32 == 0 && (end % 32 == 0 || end == n));
        tiles += (ch.len + tile - 1) / tile;
        row0 = end;
    }
    wait_groups(c->s_compute, col, 0, nch);
    CK(desc_upload(c, dp, hp, (size_t)std::max<int64_t>(nch, 1) * topk_chunk_size()));
    const int64_t n_words = (n + 31) / 32;
    CK(cudaMemsetAsync(tie, 0, (size_t)n_words * 4, c->s_compute));
    CK(cudaMemsetAsync(d_counts, 0, 2 * sizeof(unsigned long long), c->s_compute));
    {
        LaunchTimer lt(c, BDF_K_SELECT, col->dtype, n, reduce_bytes(col, 0, nch) + 2 * n_words * 4);
        CK(launch_topk_mark(col->dtype, dp, (int)std::max<int64_t>(nch, 1), tiles, t, all_valid, descending, ids, chosen, tie, d_counts, c->sm_count,
                            c->s_compute));
    }
    unsigned long long h[2] = {0, 0};
    CK(cudaMemcpyAsync(h, d_counts, sizeof h, cudaMemcpyDeviceToHost, c->s_compute));
    CK(cudaStreamSynchronize(c->s_compute));
    counts[0] = (int64_t)h[0];
    counts[1] = (int64_t)h[1];
    return BDF_OK;
}

static int top_k_indices_dev(bdf_ctx* c, int n_keys, const bdf_sort_key* keys, int64_t k, bdf_col** out) {
    TRY(sort_check(n_keys, keys));
    if (k < 0) return fail(BDF_INVALID, "top-k needs k >= 0");
    const int64_t n = keys[0].column->total_len, k_out = std::min(k, n);
    ColOwner o(c);
    if (k_out == 0 || k_out * kTopkSortDen > n * kTopkSortNum) {   // no rows, or the whole sort and its first k entries
        ColOwner full(c);
        if (k_out) TRY(sort_indices_dev(c, n_keys, keys, full.out()));
        TRY(col_alloc(c, BDF_U32, {ChunkPlan{k_out, false}}, nullptr, 0, o.out()));
        cudaError_t e = cudaSuccess;
        if (k_out) e = cudaMemcpyAsync(o->chunks[0].values, full->chunks[0].values, (size_t)k_out * 4, cudaMemcpyDeviceToDevice, c->s_compute);
        if (e == cudaSuccess) e = finish_single_group(c, o.get());
        if (e != cudaSuccess) return fail_cuda(e, "top-k");
        *out = o.release();
        return BDF_OK;
    }

    const int64_t n_words = (n + 31) / 32;
    Scratch<uint32_t> chosen, tie;
    Scratch<unsigned long long> d_counts;
    CK(chosen.alloc(c, (size_t)n_words * 4));
    CK(tie.alloc(c, (size_t)n_words * 4));
    CK(d_counts.alloc(c, 2 * sizeof(unsigned long long)));
    CK(cudaMemsetAsync(chosen, 0, (size_t)n_words * 4, c->s_compute));
    ColOwner iota(c);
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{n, false}}, nullptr, 0, iota.out()));
    c->launches++;
    CK(launch_iota((uint32_t*)iota->chunks[0].values, n, c->sm_count, c->s_compute));
    CK(finish_single_group(c, iota.get()));

    ColOwner ids(c);   // the tie set's rows once it is not every row
    bool all_rows = true;
    int64_t need = k_out;
    for (int j = 0; j < n_keys && need > 0; j++) {
        const bool desc = keys[j].descending != 0;
        ColOwner gathered(c);
        const bdf_col* col = keys[j].column;
        if (!all_rows) {
            TRY(take_dev(c, col, ids.get(), gathered.out()));
            col = gathered.get();
        }
        std::vector<uint64_t> t;
        int64_t v = 0;
        auto rank = [&](int64_t nv) { return std::vector<int64_t>{need > nv ? 0 : desc ? nv - need : need - 1}; };
        TRY(select_keys(c, col, rank, 1, &t, &v));
        const bool all_valid = need > v;
        int64_t counts[2];
        TRY(topk_mark(c, col, all_rows ? nullptr : (const uint32_t*)ids->chunks[0].values, all_valid ? 0 : t[0], all_valid, desc, chosen, tie,
                      d_counts, counts));
        need -= counts[0];
        if (need == 0) break;
        const bool last = counts[1] == need || j + 1 == n_keys;
        if (all_rows && counts[1] == n && !last) continue;   // every row ties: the next criterion is read in place
        ColOwner mask(c), tie_ids(c);
        TRY(bits_borrow(tie, col->total_len, mask.out()));
        TRY(filter_dev(c, all_rows ? iota.get() : ids.get(), mask.get(), tie_ids.out()));
        if (last) {   // the first `need` ties in row order
            LaunchTimer lt(c, BDF_K_SELECT, BDF_U32, need, need * 4);
            CK(launch_topk_choose((const uint32_t*)tie_ids->chunks[0].values, need, chosen, c->s_compute));
            break;
        }
        ids = std::move(tie_ids);
        all_rows = false;
    }

    // the chosen rows in ascending order, sorted on their gathered criteria, mapped back to row numbers
    ColOwner mask(c), rows(c), perm(c);
    TRY(bits_borrow(chosen, n, mask.out()));
    TRY(filter_dev(c, iota.get(), mask.get(), rows.out()));
    if (rows->total_len != k_out) return fail(BDF_INVALID, "internal: top-k chose a wrong number of rows");
    std::vector<ColOwner> gathered;
    std::vector<bdf_sort_key> gk;
    for (int j = 0; j < n_keys; j++) {
        gathered.emplace_back(c);
        TRY(take_dev(c, keys[j].column, rows.get(), gathered.back().out()));
        gk.push_back(bdf_sort_key{gathered.back().get(), keys[j].descending});
    }
    TRY(sort_indices_dev(c, n_keys, gk.data(), perm.out()));
    return take_dev(c, rows.get(), perm.get(), out);
}

// ---------------------------------------------------------------------------------------------------
// group-by (k_group.cu): sort the keys, gather them, mark group heads, compact keys and group starts, fold every requested
// value column once per group; first / last are a take of each group's first / last original row; count_distinct sorts
// (keys..., value) once more and counts the distinct-value heads inside every group.

static bool group_is_stat(int fn) { return fn == BDF_GROUP_KURTOSIS || fn == BDF_GROUP_SKEWNESS || fn == BDF_GROUP_STDDEV || fn == BDF_GROUP_VARIANCE ||
                                           fn == BDF_GROUP_STDDEV_POP || fn == BDF_GROUP_VAR_POP; }
static int group_stat_of(int fn) {   // bdf_group_fn -> bdf_stat
    switch (fn) {
        case BDF_GROUP_KURTOSIS: return BDF_STAT_KURTOSIS;
        case BDF_GROUP_SKEWNESS: return BDF_STAT_SKEWNESS;
        case BDF_GROUP_STDDEV: return BDF_STAT_STDDEV;
        case BDF_GROUP_VARIANCE: return BDF_STAT_VARIANCE;
        case BDF_GROUP_STDDEV_POP: return BDF_STAT_STDDEV_POP;
        default: return BDF_STAT_VAR_POP;
    }
}

// Head bitmap (a boolean column of n rows) over one-chunk columns in sorted order.  kernel >= 0: the launch gets a launch record
// under that bdf_kernel_id (the window's heads); group-by and join keep theirs unrecorded.
static int group_heads(bdf_ctx* c, const std::vector<const bdf_col*>& cols, bool and_last_valid, int64_t n, bdf_col** out, int kernel = -1) {
    ColOwner head(c);
    TRY(col_alloc(c, kBool, {ChunkPlan{n, false}}, nullptr, 0, head.out()));
    std::vector<const void*> vals(cols.size());
    std::vector<const uint32_t*> valid(cols.size());
    std::vector<int> widths(cols.size()), is_float(cols.size());
    int64_t key_bytes = 0;
    for (size_t k = 0; k < cols.size(); k++) {
        wait_groups(c->s_compute, cols[k], 0, 1);
        vals[k] = cols[k]->chunks[0].values;
        valid[k] = cols[k]->chunks[0].validity;
        widths[k] = dtype_width(cols[k]->dtype);
        is_float[k] = dtype_is_float(cols[k]->dtype) ? 1 : 0;
        key_bytes += widths[k];
    }
    cudaError_t e;
    {
        std::unique_ptr<LaunchTimer> t;
        if (kernel >= 0) t.reset(new LaunchTimer(c, kernel, kBool, n, n * key_bytes + bitmap_bytes(n)));
        else c->launches++;
        e = launch_group_heads((int)cols.size(), vals.data(), valid.data(), widths.data(), is_float.data(), and_last_valid ? 1 : 0, n,
                               (uint32_t*)head->chunks[0].values, c->s_compute);
    }
    if (e == cudaSuccess) e = finish_single_group(c, head.get());
    if (e != cudaSuccess) return fail_cuda(e, "group heads");
    *out = head.release();
    return BDF_OK;
}

// A copy of a one-chunk column made on the compute stream (the same aggregate requested twice gets two columns).
static int group_clone(bdf_ctx* c, const bdf_col* src, bdf_col** out) {
    const DevChunk& s = src->chunks[0];
    ColOwner o(c);
    TRY(col_alloc(c, src->dtype, {ChunkPlan{s.len, s.validity != nullptr}}, nullptr, 0, o.out()));
    cudaError_t e = cudaSuccess;
    if (s.len) e = cudaMemcpyAsync(o->chunks[0].values, s.values, (size_t)s.len * dtype_width(src->dtype), cudaMemcpyDeviceToDevice, c->s_compute);
    if (e == cudaSuccess && s.len && s.validity)
        e = cudaMemcpyAsync(o->chunks[0].validity, s.validity, (size_t)bitmap_bytes(s.len), cudaMemcpyDeviceToDevice, c->s_compute);
    if (e == cudaSuccess) e = finish_single_group(c, o.get());
    if (e != cudaSuccess) return fail_cuda(e, "group result copy");
    o->null_counts[0] = src->null_counts[0];
    *out = o.release();
    return BDF_OK;
}

// The runs of equal key tuples in sorted order: group-by's groups, and the join's build side.
struct SortedRuns {
    explicit SortedRuns(bdf_ctx* c) : perm(c), head(c), iota(c), starts(c) {}
    ColOwner perm;                   // the stable sort permutation (sorted position -> row)
    std::vector<ColOwner> sorted;    // the key columns in sorted order
    ColOwner head;                   // bit i: sorted row i starts a run
    std::vector<ColOwner> distinct;  // the key tuple of every run
    ColOwner iota;                   // 0, 1, .., n-1
    ColOwner starts;                 // the first sorted row of every run
    int64_t n_runs = 0;
};

// Sort the keys, gather them in sorted order, mark the heads, compact the distinct key tuples and the run starts.  Only the first
// n_cut keys cut runs; the keys after them order the rows inside a run (the as-of join's `on` key).  n_cut == 0: the whole side is one
// run (none when it is empty), and no heads, distinct tuples or starts are made.  `what` names the caller's iota in a CUDA failure.
static int sorted_runs(bdf_ctx* c, int n_keys, int n_cut, const bdf_col* const* keys, const char* what, SortedRuns* r) {
    const int64_t n = keys[0]->total_len;
    std::vector<bdf_sort_key> sk((size_t)n_keys);
    for (int k = 0; k < n_keys; k++) sk[k] = bdf_sort_key{keys[k], 0};
    TRY(sort_indices_dev(c, n_keys, sk.data(), r->perm.out()));
    std::vector<const bdf_col*> sorted;
    for (int k = 0; k < n_keys; k++) {
        r->sorted.emplace_back(c);
        TRY(take_dev(c, keys[k], r->perm.get(), r->sorted[k].out()));
        sorted.push_back(r->sorted[k].get());
    }
    if (n_cut == 0) {
        r->n_runs = n > 0 ? 1 : 0;
        return BDF_OK;
    }
    sorted.resize((size_t)n_cut);
    TRY(group_heads(c, sorted, false, n, r->head.out()));
    for (int k = 0; k < n_cut; k++) {
        r->distinct.emplace_back(c);
        TRY(filter_dev(c, sorted[k], r->head.get(), r->distinct[k].out()));
    }
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{n, false}}, nullptr, 0, r->iota.out()));
    c->launches++;
    cudaError_t e = n > 0 ? launch_iota((uint32_t*)r->iota->chunks[0].values, n, c->sm_count, c->s_compute) : cudaSuccess;
    if (e == cudaSuccess) e = finish_single_group(c, r->iota.get());
    if (e != cudaSuccess) return fail_cuda(e, what);
    TRY(filter_dev(c, r->iota.get(), r->head.get(), r->starts.out()));
    r->n_runs = r->starts->chunks.empty() ? 0 : r->starts->chunks[0].len;
    return BDF_OK;
}

// One head bitmap and what k_window and k_setop need to find the run of a position in O(1).
struct WinHeadsHost {
    explicit WinHeadsHost(bdf_ctx* c) : bits(c), starts(c) {}
    ColOwner bits;                        // bit i: sorted position i starts a run
    Scratch<unsigned long long> prefix;   // per head word: the runs that start before it
    ColOwner starts;                      // the first position of every run
    int64_t n_runs = 0;
    const void* arrays[3] = {nullptr, nullptr, nullptr};   // {words, prefix, starts} as the kernels take them
};

// The per-word run prefix of h->bits and the compacted run starts; the scan's launches are recorded under `kernel`.
static int window_runs(bdf_ctx* c, const bdf_col* iota, int64_t n, WinHeadsHost* h, int kernel = BDF_K_WINDOW) {
    const int64_t words = (n + 31) / 32;
    Scratch<unsigned long long> block_sums;
    cudaError_t e = h->prefix.alloc(c, (size_t)(words + 1) * sizeof(unsigned long long));
    if (e == cudaSuccess) e = block_sums.alloc(c, (size_t)scan_tile_sums(words) * sizeof(unsigned long long));
    if (e == cudaSuccess) {
        LaunchTimer t(c, kernel, BDF_U64, n, words * (4 + 8 + 16));   // popcounts written, then read and written by the scan
        c->launches += kScanPopcountLaunches - 1;                        // the timer counts one
        e = launch_scan_popcount((const uint32_t*)h->bits->chunks[0].values, words, h->prefix, block_sums, c->s_compute);
    }
    if (e != cudaSuccess) return fail_cuda(e, "window run prefix");
    TRY(filter_dev(c, iota, h->bits.get(), h->starts.out()));
    h->n_runs = h->starts->chunks[0].len;
    h->arrays[0] = h->bits->chunks[0].values;
    h->arrays[1] = h->prefix.get();
    h->arrays[2] = h->starts->chunks[0].values;
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// distinct rows and set operations (k_setop.cu): the key tuples are sorted stably once -- a set operation sorts the left rows and then
// the right rows as one column, borrowing both sides' chunks -- gathered, and cut into runs by the head kernel, whose equality is
// group-by's.  One pass over the sorted positions decides every row from its run's bounds (and, for a set operation, the run's left
// count, which the run's last left position writes) and stores a byte at the row's original position; a second pass packs the bytes
// of every output chunk into its bitmap.  The result is a Boolean mask over the (left) rows, chunked like the keys, for the filter.

// A Boolean column as one UInt8 per row (0 / 1), chunked like it, its validity copied to bit 0: the sort and the head kernel compare
// Boolean keys as UInt8.
static int bool_widen(bdf_ctx* c, const bdf_col* in, bdf_col** out) {
    std::vector<ChunkPlan> plan;
    for (const DevChunk& ch : in->chunks) plan.push_back(ChunkPlan{ch.len, ch.validity != nullptr});
    ColOwner o(c);
    TRY(col_alloc(c, BDF_U8, plan, nullptr, 0, o.out()));
    TRY(fetch_counts(c, const_cast<bdf_col*>(in)));   // a computed column's null counts may still be on the device
    wait_groups(c->s_compute, in, 0, (int64_t)in->chunks.size());
    cudaError_t e = cudaSuccess;
    {
        LaunchTimer t(c, BDF_K_GROUP, BDF_U8, in->total_len, in->total_len + in->total_len / 4);
        int launches = 0;
        for (size_t i = 0; i < in->chunks.size() && e == cudaSuccess; i++) {
            const DevChunk& s = in->chunks[i];
            if (!s.len) continue;
            e = launch_setop_widen_bool(s.values, s.val_bit_off, s.len, (unsigned char*)o->chunks[i].values, c->s_compute);
            launches++;
            if (e == cudaSuccess && s.validity) {
                e = launch_bitmap_rebase(s.validity, s.bit_off, s.len, o->chunks[i].validity, c->s_compute);
                launches++;
            }
        }
        c->launches += std::max(launches - 1, 0);   // the timer counts one
    }
    if (e == cudaSuccess) e = finish_single_group(c, o.get());
    if (e != cudaSuccess) return fail_cuda(e, "Boolean widening");
    o->null_counts = in->null_counts;
    *out = o.release();
    return BDF_OK;
}

// The chunks of cols[0], then those of cols[1], ...: values copied device to device, bitmaps copied to bit 0 of their new chunk.
static int concat_dev(bdf_ctx* c, int n, const bdf_col* const* cols, bdf_col** out) {
    if (n < 1) return fail(BDF_INVALID, "concat takes at least one column");
    if (!cols || !out) return fail(BDF_INVALID, "null argument");
    for (int k = 0; k < n; k++)
        if (!cols[k]) return fail(BDF_INVALID, "null column");
    const int dt = cols[0]->dtype;
    if (!((dt >= 0 && dt < BDF_NTYPES) || dt == kBool)) return fail(BDF_UNSUPPORTED, "concat takes numeric or Boolean columns");
    for (int k = 0; k < n; k++)
        if (cols[k]->dtype != dt) return fail(BDF_UNSUPPORTED, "concatenated columns must have the same dtype");
    std::vector<ChunkPlan> plan;
    std::vector<const DevChunk*> src;
    std::vector<int64_t> nulls;
    for (int k = 0; k < n; k++) {
        TRY(fetch_counts(c, const_cast<bdf_col*>(cols[k])));   // a computed column's null counts may still be on the device
        for (size_t i = 0; i < cols[k]->chunks.size(); i++) {
            const DevChunk& ch = cols[k]->chunks[i];
            plan.push_back(ChunkPlan{ch.len, ch.validity != nullptr});
            src.push_back(&ch);
            nulls.push_back(cols[k]->null_counts[i]);
        }
        wait_groups(c->s_compute, cols[k], 0, (int64_t)cols[k]->chunks.size());
    }
    ColOwner o(c);
    TRY(col_alloc(c, dt, plan, nullptr, 0, o.out()));
    cudaError_t e = cudaSuccess;
    int64_t rows = 0, bytes = 0;   // read and written
    for (const DevChunk* s : src) {
        rows += s->len;
        bytes += 2 * ((dt == kBool ? bitmap_bytes(s->len) : s->len * dtype_width(dt)) + (s->validity ? bitmap_bytes(s->len) : 0));
    }
    {
        LaunchTimer t(c, BDF_K_GROUP, dt, rows, bytes);
        int launches = 0;
        for (size_t i = 0; i < src.size() && e == cudaSuccess; i++) {
            const DevChunk &s = *src[i], &d = o->chunks[i];
            if (!s.len) continue;
            if (dt == kBool) {
                e = launch_bitmap_rebase(s.values, s.val_bit_off, s.len, (uint32_t*)d.values, c->s_compute);
                launches++;
            } else {
                e = cudaMemcpyAsync(d.values, s.values, (size_t)s.len * dtype_width(dt), cudaMemcpyDeviceToDevice, c->s_compute);
            }
            if (e == cudaSuccess && s.validity) {
                e = launch_bitmap_rebase(s.validity, s.bit_off, s.len, d.validity, c->s_compute);
                launches++;
            }
        }
        c->launches += launches - 1;   // the timer counts one
    }
    if (e == cudaSuccess) e = finish_single_group(c, o.get());
    if (e != cudaSuccess) return fail_cuda(e, "concat");
    o->null_counts = nulls;
    *out = o.release();
    return BDF_OK;
}

// A mask over the rows of `left` (one bitmap of all left rows, then copied to every chunk's bitmap).  mode 0..2: duplicated with that bdf_keep, right == null;
// mode 3 + bdf_setop: the set operation against `right`.  The arguments are checked by the entries.
static int setop_mask(bdf_ctx* c, int mode, int n_keys, const bdf_col* const* left, const bdf_col* const* right, bdf_col** out) {
    const int64_t nl = left[0]->total_len, nr = right ? right[0]->total_len : 0, n = nl + nr;
    if (n > 0xffffffffLL) return fail(BDF_UNSUPPORTED, "sort indices are UInt32: at most 2^32-1 rows");
    std::vector<ChunkPlan> plan;
    for (const DevChunk& ch : left[0]->chunks) plan.push_back(ChunkPlan{ch.len, false});
    ColOwner mask(c);
    TRY(col_alloc(c, kBool, plan, nullptr, 0, mask.out()));
    if (nl == 0) {
        cudaError_t e = finish_single_group(c, mask.get());
        if (e != cudaSuccess) return fail_cuda(e, "distinct rows");
        *out = mask.release();
        return BDF_OK;
    }

    // the keys: Boolean ones widened, the two sides of a set operation borrowed as one column
    std::vector<ColOwner> owned;
    owned.reserve((size_t)n_keys * 4);
    std::vector<bdf_sort_key> sk;
    for (int k = 0; k < n_keys; k++) {
        const bdf_col* side[2] = {left[k], right ? right[k] : nullptr};
        for (int j = 0; j < 2 && side[j]; j++)
            if (side[j]->dtype == kBool) {
                owned.emplace_back(c);
                TRY(bool_widen(c, side[j], owned.back().out()));
                side[j] = owned.back().get();
            }
        if (side[1]) {
            std::vector<DevChunk> chunks(side[0]->chunks);
            chunks.insert(chunks.end(), side[1]->chunks.begin(), side[1]->chunks.end());
            wait_groups(c->s_compute, side[0], 0, (int64_t)side[0]->chunks.size());
            wait_groups(c->s_compute, side[1], 0, (int64_t)side[1]->chunks.size());
            owned.emplace_back(c);
            TRY(col_borrow(side[0]->dtype, chunks, owned.back().out()));
            side[0] = owned.back().get();
        }
        sk.push_back(bdf_sort_key{side[0], 0});
    }

    // sort, gather, heads, run prefix and starts
    ColOwner perm(c), iota(c);
    TRY(sort_indices_dev(c, n_keys, sk.data(), perm.out()));
    std::vector<ColOwner> sorted;
    std::vector<const bdf_col*> sorted_keys;
    for (int k = 0; k < n_keys; k++) {
        sorted.emplace_back(c);
        TRY(take_dev(c, sk[k].column, perm.get(), sorted.back().out()));
        sorted_keys.push_back(sorted.back().get());
    }
    WinHeadsHost H(c);
    TRY(group_heads(c, sorted_keys, false, n, H.bits.out(), BDF_K_GROUP));
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{n, false}}, nullptr, 0, iota.out()));
    c->launches++;
    cudaError_t e = launch_iota((uint32_t*)iota->chunks[0].values, n, c->sm_count, c->s_compute);
    if (e == cudaSuccess) e = finish_single_group(c, iota.get());
    if (e != cudaSuccess) return fail_cuda(e, "distinct rows iota");
    TRY(window_runs(c, iota.get(), n, &H, BDF_K_GROUP));

    // the decisions at every left row's original position, then one bitmap per chunk
    const uint32_t* perm_d = (const uint32_t*)perm->chunks[0].values;
    Scratch<uint32_t> run_left;
    if (mode >= 3) e = run_left.alloc(c, (size_t)std::max<int64_t>(H.n_runs, 1) * sizeof(uint32_t));
    if (e != cudaSuccess) return fail_cuda(e, "distinct rows scratch allocation");
    if (mode >= 3) {
        LaunchTimer t(c, BDF_K_GROUP, BDF_U32, n, n * 4 + nl * 24 / 32 + H.n_runs * 4);   // perm; head words, prefix and starts of left rows
        e = launch_setop_left_count(H.arrays, H.n_runs, n, perm_d, nl, run_left, c->s_compute);
    }
    Scratch<uint32_t> words;   // one bit per left row, the true ones OR-ed in
    const int64_t n_words = (nl + 31) / 32;
    if (e == cudaSuccess) e = words.alloc(c, (size_t)n_words * sizeof(uint32_t));
    if (e == cudaSuccess) e = cudaMemsetAsync(words, 0, (size_t)n_words * sizeof(uint32_t), c->s_compute);
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_GROUP, kBool, n, n * (4 + 4 + 8) + n_words * 4 + (mode >= 3 ? nl * 4 : 0));
        e = launch_setop_mark(H.arrays, H.n_runs, n, perm_d, nl, mode, run_left.get(), words, c->s_compute);
    }
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_GROUP, kBool, nl, 2 * n_words * 4);
        int64_t row0 = 0;
        int launches = 0;
        for (size_t i = 0; i < mask->chunks.size() && e == cudaSuccess; i++) {
            const DevChunk& d = mask->chunks[i];
            if (d.len) {
                e = launch_bitmap_rebase(words.get(), row0, d.len, (uint32_t*)d.values, c->s_compute);
                launches++;
            }
            row0 += d.len;
        }
        c->launches += launches - 1;   // the timer counts one
    }
    if (e == cudaSuccess) e = finish_single_group(c, mask.get());
    if (e != cudaSuccess) return fail_cuda(e, "distinct rows");
    *out = mask.release();
    return BDF_OK;
}

// The checks of the two entries; right == null for duplicated.
static int setop_check(int n_keys, const bdf_col* const* left, const bdf_col* const* right, bool two_sides) {
    if (n_keys < 1 || n_keys > 16) return fail(BDF_INVALID, "1..16 key columns");
    if (!left || (two_sides && !right)) return fail(BDF_INVALID, "null argument");
    for (int k = 0; k < n_keys; k++)
        if (!left[k] || (two_sides && !right[k])) return fail(BDF_INVALID, "null key column");
    auto keyable = [](int dt) { return (dt >= 0 && dt < BDF_NTYPES) || dt == kBool; };
    for (int k = 0; k < n_keys; k++)
        if (!keyable(left[k]->dtype) || (two_sides && !keyable(right[k]->dtype)))
            return fail(BDF_UNSUPPORTED, "distinct rows and set operations take numeric or Boolean key columns");
    for (int k = 0; two_sides && k < n_keys; k++)
        if (left[k]->dtype != right[k]->dtype) return fail(BDF_UNSUPPORTED, "Union can only be performed on tables with compatible column types");
    for (int k = 0; k < n_keys; k++)
        if (left[k]->total_len != left[0]->total_len || (two_sides && right[k]->total_len != right[0]->total_len))
            return fail(BDF_LENGTH_MISMATCH, "key columns of one side have different lengths");
    return BDF_OK;
}

// The distinct valid values of x inside every group: a second stable lexsort over (keys..., x) -- the groups occupy the same row
// ranges in both sort orders -- and the heads of (keys..., x) on a valid x, each of which starts a distinct value of its group.
// n_keys == 0: the whole column is one group.  sval: x in that order; pos: the sorted rows of the heads (ascending value order
// inside every group).
struct DistinctRuns {
    explicit DistinctRuns(bdf_ctx* c) : sval(c), dhead(c), pos(c) {}
    ColOwner sval, dhead, pos;
};

static int distinct_runs(bdf_ctx* c, int n_keys, const bdf_col* const* keys, const std::vector<const bdf_col*>& sorted_keys, const bdf_col* x,
                         const bdf_col* iota, int64_t n, DistinctRuns* r) {
    std::vector<bdf_sort_key> sk2((size_t)n_keys);
    for (int k = 0; k < n_keys; k++) sk2[k] = bdf_sort_key{keys[k], 0};
    sk2.push_back(bdf_sort_key{x, 0});
    ColOwner idx2(c);
    TRY(sort_indices_dev(c, n_keys + 1, sk2.data(), idx2.out()));
    TRY(take_dev(c, x, idx2.get(), r->sval.out()));
    std::vector<const bdf_col*> cols = sorted_keys;
    cols.push_back(r->sval.get());
    TRY(group_heads(c, cols, true, n, r->dhead.out()));
    TRY(filter_dev(c, iota, r->dhead.get(), r->pos.out()));
    return BDF_OK;
}

// sum_distinct: the distinct values (the head values, in ascending order inside every group) folded per group by the SUM fold of
// launch_group_reduce; d_first: the first distinct value of every group (launch_group_distinct's `first`).
static int distinct_sum(bdf_ctx* c, const DistinctRuns& dr, const uint32_t* d_first, int64_t n_groups, bdf_col** out) {
    const int dt = dr.sval->dtype;
    const int w = dtype_width(dt);
    ColOwner dvals(c), sum(c), cnt(c);
    TRY(filter_dev(c, dr.sval.get(), dr.dhead.get(), dvals.out()));
    const int64_t nd = dvals->chunks.empty() ? 0 : dvals->chunks[0].len;
    TRY(col_alloc(c, dt, {ChunkPlan{n_groups, false}}, nullptr, 0, sum.out()));
    TRY(col_alloc(c, BDF_I64, {ChunkPlan{n_groups, false}}, nullptr, 0, cnt.out()));
    if (nd) wait_groups(c->s_compute, dvals.get(), 0, 1);
    cudaError_t e;
    {
        LaunchTimer t(c, BDF_K_GROUP, dt, nd, nd * w + n_groups * (4 + w + 8));
        Scratch<void> scratch;
        e = scratch.alloc(c, group_big_scratch_bytes(nd));
        c->launches += 3;
        if (e == cudaSuccess)
            e = launch_group_reduce(dt, false, nd ? dvals->chunks[0].values : nullptr, nd ? dvals->chunks[0].validity : nullptr, d_first, n_groups, nd,
                                    sum->chunks[0].values, (long long*)cnt->chunks[0].values, nullptr, nullptr, nullptr, nullptr, scratch, c->sm_count,
                                    c->s_compute);
    }
    if (e == cudaSuccess) e = finish_single_group(c, sum.get());
    if (e != cudaSuccess) return fail_cuda(e, "distinct sum");
    *out = sum.release();
    return BDF_OK;
}

// Median / mode per group (k_dist.cu) over distinct_runs: in the second sort each group's valid values come first, in key order.
// vend: the end of every group's valid prefix; first_run: the first distinct run of every group (mode only).
static int dist_group_bounds(bdf_ctx* c, const DistinctRuns& dr, const uint32_t* d_starts, int64_t n_groups, int64_t n, bool runs,
                             Scratch<uint32_t>* first_run, Scratch<uint32_t>* vend) {
    const size_t bytes = (size_t)std::max<int64_t>(n_groups, 1) * sizeof(uint32_t);
    cudaError_t e = vend->alloc(c, bytes);
    if (e == cudaSuccess && runs) e = first_run->alloc(c, bytes);
    const int64_t n_pos = dr.pos->chunks.empty() ? 0 : dr.pos->chunks[0].len;
    if (n_pos) wait_groups(c->s_compute, dr.pos.get(), 0, 1);
    wait_groups(c->s_compute, dr.sval.get(), 0, 1);
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_GROUP, BDF_U32, n_groups, n_groups * 12);
        e = launch_dist_groups(d_starts, n_groups, n, runs && n_pos ? (const uint32_t*)dr.pos->chunks[0].values : nullptr, n_pos,
                               dr.sval->chunks[0].validity, runs ? first_run->get() : nullptr, vend->get(), c->s_compute);
    }
    if (e != cudaSuccess) return fail_cuda(e, "distribution group bounds");
    return BDF_OK;
}

static int group_median(bdf_ctx* c, const DistinctRuns& dr, const uint32_t* d_starts, int64_t n_groups, int64_t n, bdf_col** out) {
    ColOwner res(c);
    TRY(col_alloc(c, BDF_F64, {ChunkPlan{n_groups, true}}, nullptr, 0, res.out()));
    Scratch<uint32_t> first_run, vend;
    TRY(dist_group_bounds(c, dr, d_starts, n_groups, n, false, &first_run, &vend));
    cudaError_t e;
    {
        LaunchTimer t(c, BDF_K_GROUP, BDF_F64, n_groups, n_groups * (4 + 4 + 2 * dtype_width(dr.sval->dtype) + 8));
        e = launch_dist_median(dr.sval->dtype, dr.sval->chunks[0].values, d_starts, n_groups, vend, (double*)res->chunks[0].values,
                               res->chunks[0].validity, c->s_compute);
    }
    if (e == cudaSuccess) e = finish_single_group(c, res.get());
    if (e != cudaSuccess) return fail_cuda(e, "group median");
    res->null_counts[0] = -1;   // learnt on demand (ensure_null_counts)
    *out = res.release();
    return BDF_OK;
}

// The mode of every group: the sorted row of its most frequent (then smallest) distinct run, gathered from the sorted values; d_freq
// (may be null): the run's row count per group, 0 without a valid value.
static int group_mode(bdf_ctx* c, const DistinctRuns& dr, const uint32_t* d_starts, int64_t n_groups, int64_t n, bdf_col** out, long long* d_freq) {
    Scratch<uint32_t> first_run, vend;
    TRY(dist_group_bounds(c, dr, d_starts, n_groups, n, true, &first_run, &vend));
    const int64_t n_pos = dr.pos->chunks.empty() ? 0 : dr.pos->chunks[0].len;
    const uint32_t* pos = n_pos ? (const uint32_t*)dr.pos->chunks[0].values : nullptr;
    ColOwner rows(c);
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{n_groups, true}}, nullptr, 0, rows.out()));
    Scratch<unsigned long long> best;
    cudaError_t e = best.alloc(c, (size_t)std::max<int64_t>(n_groups, 1) * 8);
    if (e == cudaSuccess) e = cudaMemsetAsync(best, 0, (size_t)std::max<int64_t>(n_groups, 1) * 8, c->s_compute);
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_GROUP, BDF_I64, n_pos, n_pos * 8 + n_groups * 16);
        e = launch_dist_runs(pos, n_pos, d_starts, n_groups, n, first_run, vend, nullptr, best, c->s_compute);
    }
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_GROUP, BDF_U32, n_groups, n_groups * 20);
        e = launch_dist_mode(best, n_groups, first_run, pos, (uint32_t*)rows->chunks[0].values, rows->chunks[0].validity, d_freq, c->s_compute);
    }
    if (e == cudaSuccess) e = finish_single_group(c, rows.get());
    if (e != cudaSuccess) return fail_cuda(e, "group mode");
    rows->null_counts[0] = -1;
    return take_dev(c, dr.sval.get(), rows.get(), out);
}

static bool group_is_collect(int fn) { return fn == BDF_GROUP_COLLECT_LIST || fn == BDF_GROUP_COLLECT_SET; }
static void drop(bdf_ctx* c, bdf_list* l);
static int group_collect(bdf_ctx* c, const SortedRuns& runs, const bdf_col* x, int fn, const DistinctRuns* dr, bdf_list** out);

// out_lists == nullptr: the entry without list outputs (bdf_group_by_dev), which does not know the collect functions.
static int group_by_dev(bdf_ctx* c, int n_keys, const bdf_col* const* keys, int n_aggs, const bdf_group_agg* aggs, bdf_col** out_keys, bdf_col** out,
                        bdf_list** out_lists, int64_t* n_groups_out) {
    if (n_keys < 1 || n_keys > 16) return fail(BDF_INVALID, "1..16 group key columns");
    for (int k = 0; k < n_keys; k++) {
        if (!keys[k]) return fail(BDF_INVALID, "null key column");
        if (keys[k]->dtype < 0 || keys[k]->dtype >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "the group key must be a numeric column");
        if (keys[k]->total_len != keys[0]->total_len) return fail(BDF_LENGTH_MISMATCH, "key columns have different lengths");
    }
    for (int j = 0; j < n_aggs; j++) {
        const bdf_col* v = aggs[j].column;
        if (!v) return fail(BDF_INVALID, "null value column");
        if (v->dtype < 0 || v->dtype >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "aggregated columns must be numeric");
        const int fn = aggs[j].function;
        if (!((fn >= BDF_GROUP_SUM && fn <= BDF_GROUP_VAR_POP) || fn == BDF_GROUP_MEDIAN || fn == BDF_GROUP_MODE || (out_lists && group_is_collect(fn))))
            return fail(BDF_UNSUPPORTED, "unknown group function %d", fn);
        if (aggs[j].function == BDF_GROUP_AVG && (v->dtype == BDF_I64 || v->dtype == BDF_U64)) return fail(BDF_UNSUPPORTED, "avg needs f64: From<T::Native>");
        if (v->total_len != keys[0]->total_len) return fail(BDF_LENGTH_MISMATCH, "key and value columns have different lengths");
    }
    const int64_t n = keys[0]->total_len;
    SortedRuns runs(c);
    TRY(sorted_runs(c, n_keys, n_keys, keys, "group iota", &runs));
    const bdf_col* idx = runs.perm.get();
    const int64_t n_groups = runs.n_runs;
    const uint32_t* d_starts = (const uint32_t*)runs.starts->chunks[0].values;
    std::vector<ColOwner> res;
    for (int j = 0; j < n_aggs; j++) res.emplace_back(c);
    cudaError_t e = cudaSuccess;

    // sum / count / min / max / avg: every distinct value column is gathered once and folded once
    std::vector<bool> done((size_t)n_aggs, false);
    for (int j0 = 0; j0 < n_aggs; j0++) {
        const int f0 = aggs[j0].function;
        if (done[j0] || f0 == BDF_GROUP_COUNT_DISTINCT || f0 == BDF_GROUP_FIRST || f0 == BDF_GROUP_LAST || f0 > BDF_GROUP_LAST) continue;
        const bdf_col* v = aggs[j0].column;
        bool want[5] = {false, false, false, false, false};   // sum, max, min, avg, count (bdf_group_fn order)
        for (int j = j0; j < n_aggs; j++)
            if (aggs[j].column == v && aggs[j].function <= BDF_GROUP_COUNT) want[aggs[j].function] = true;
        const int dt = v->dtype;
        const bool is_float = dtype_is_float(dt);
        const bool mm = want[BDF_GROUP_MAX] || want[BDF_GROUP_MIN];
        // the accumulators the single-key entry never needed: only EXTRA folds write avg, and a float column's min / max
        const bool extra = want[BDF_GROUP_AVG] || (is_float && mm);
        ColOwner sval(c), csum(c), ccnt(c), cmin(c), cmax(c), cavg(c);   // what nobody asks for is dropped with the owner
        TRY(take_dev(c, v, idx, sval.out()));
        TRY(col_alloc(c, dt, {ChunkPlan{n_groups, false}}, nullptr, 0, csum.out()));
        TRY(col_alloc(c, BDF_I64, {ChunkPlan{n_groups, false}}, nullptr, 0, ccnt.out()));
        // integers without extra: the kernel writes min and max together
        if (want[BDF_GROUP_MIN] || (mm && !is_float)) TRY(col_alloc(c, dt, {ChunkPlan{n_groups, true}}, nullptr, 0, cmin.out()));
        if (want[BDF_GROUP_MAX] || (mm && !is_float)) TRY(col_alloc(c, dt, {ChunkPlan{n_groups, true}}, nullptr, 0, cmax.out()));
        if (want[BDF_GROUP_AVG]) TRY(col_alloc(c, BDF_F64, {ChunkPlan{n_groups, true}}, nullptr, 0, cavg.out()));
        bdf_col* const validity_of[3] = {cmin.get(), cmax.get(), cavg.get()};
        bdf_col* nonempty = nullptr;   // the kernel sets this bitmap; the others get a copy
        for (bdf_col* r : validity_of) if (r && !nonempty) nonempty = r;
        wait_groups(c->s_compute, sval.get(), 0, 1);
        wait_groups(c->s_compute, runs.starts.get(), 0, 1);
        {
            const int w = dtype_width(dt);
            const int outs = 1 + (cmin.get() ? 1 : 0) + (cmax.get() ? 1 : 0);
            LaunchTimer t(c, BDF_K_GROUP, dt, n, n * w + (sval->chunks[0].validity ? bitmap_bytes(n) : 0) + n_groups * (4 + outs * w + 8 + (cavg.get() ? 8 : 0)));
            Scratch<void> scratch;
            e = scratch.alloc(c, group_big_scratch_bytes(n));
            c->launches += 3;   // long groups among short ones: k_group_medium; hot keys: k_group_big + k_group_big_finish
            if (e == cudaSuccess)
                e = launch_group_reduce(dt, extra, sval->chunks[0].values, sval->chunks[0].validity, d_starts, n_groups, n, csum->chunks[0].values,
                                        (long long*)ccnt->chunks[0].values, cmin.get() ? cmin->chunks[0].values : nullptr, cmax.get() ? cmax->chunks[0].values : nullptr,
                                        cavg.get() ? (double*)cavg->chunks[0].values : nullptr, nonempty ? nonempty->chunks[0].validity : nullptr, scratch,
                                        c->sm_count, c->s_compute);
        }
        // min / max / avg share one validity pattern: copy the bitmap rather than set it several times with atomics
        for (bdf_col* r : validity_of)
            if (e == cudaSuccess && r && r != nonempty && n_groups)
                e = cudaMemcpyAsync(r->chunks[0].validity, nonempty->chunks[0].validity, (size_t)bitmap_bytes(n_groups), cudaMemcpyDeviceToDevice, c->s_compute);
        for (bdf_col* r : {csum.get(), ccnt.get(), cmin.get(), cmax.get(), cavg.get()})
            if (r && e == cudaSuccess) {
                e = finish_single_group(c, r);
                if (r->chunks[0].validity) r->null_counts[0] = -1;   // learnt on demand (ensure_null_counts)
            }
        if (e != cudaSuccess) return fail_cuda(e, "group aggregate");
        ColOwner* const by_fn[5] = {&csum, &cmax, &cmin, &cavg, &ccnt};
        bdf_col* const made[5] = {csum.get(), cmax.get(), cmin.get(), cavg.get(), ccnt.get()};
        for (int j = j0; j < n_aggs; j++) {
            const int fn = aggs[j].function;
            if (aggs[j].column != v || fn > BDF_GROUP_COUNT) continue;
            if (by_fn[fn]->get()) res[j] = std::move(*by_fn[fn]);   // first request: the column itself
            else TRY(group_clone(c, made[fn], res[j].out()));       // the same aggregate again: a copy
            done[j] = true;
        }
    }

    // first / last: the original row of every group's first / last sorted row, then a take of the original column
    bool need_first = false, need_last = false;
    for (int j = 0; j < n_aggs; j++) { need_first |= aggs[j].function == BDF_GROUP_FIRST; need_last |= aggs[j].function == BDF_GROUP_LAST; }
    ColOwner first_rows(c), last_rows(c);
    if (need_first) TRY(col_alloc(c, BDF_U32, {ChunkPlan{n_groups, false}}, nullptr, 0, first_rows.out()));
    if (need_last) TRY(col_alloc(c, BDF_U32, {ChunkPlan{n_groups, false}}, nullptr, 0, last_rows.out()));
    if (need_first || need_last) {
        wait_groups(c->s_compute, idx, 0, 1);
        c->launches++;
        e = launch_group_bounds((const uint32_t*)idx->chunks[0].values, d_starts, n_groups, n, first_rows.get() ? (uint32_t*)first_rows->chunks[0].values : nullptr,
                                last_rows.get() ? (uint32_t*)last_rows->chunks[0].values : nullptr, c->s_compute);
        for (bdf_col* r : {first_rows.get(), last_rows.get()})
            if (r && e == cudaSuccess) e = finish_single_group(c, r);
        if (e != cudaSuccess) return fail_cuda(e, "group bounds");
    }
    for (int j = 0; j < n_aggs; j++)
        if (aggs[j].function == BDF_GROUP_FIRST || aggs[j].function == BDF_GROUP_LAST)
            TRY(take_dev(c, aggs[j].column, aggs[j].function == BDF_GROUP_FIRST ? first_rows.get() : last_rows.get(), res[j].out()));

    // variance / stddev / skewness / kurtosis (and the population forms): every value column is gathered once and folded once into
    // a moment record per group; every requested statistic is then one small kernel over the records
    std::vector<bool> stat_done((size_t)n_aggs, false);
    for (int j0 = 0; j0 < n_aggs; j0++) {
        if (stat_done[j0] || !group_is_stat(aggs[j0].function)) continue;
        const bdf_col* v = aggs[j0].column;
        ColOwner sval(c);
        TRY(take_dev(c, v, idx, sval.out()));
        for (int j = j0; j < n_aggs; j++)
            if (aggs[j].column == v && group_is_stat(aggs[j].function)) TRY(col_alloc(c, BDF_F64, {ChunkPlan{n_groups, true}}, nullptr, 0, res[j].out()));
        wait_groups(c->s_compute, sval.get(), 0, 1);
        wait_groups(c->s_compute, runs.starts.get(), 0, 1);
        Scratch<void> scratch;
        Scratch<Moments> mom;
        {
            const int w = dtype_width(v->dtype);
            LaunchTimer t(c, BDF_K_GROUP, v->dtype, n, n * w + (sval->chunks[0].validity ? bitmap_bytes(n) : 0) + n_groups * (4 + (int64_t)sizeof(Moments)));
            e = scratch.alloc(c, group_big_scratch_bytes(n));
            if (e == cudaSuccess) e = mom.alloc(c, (size_t)std::max<int64_t>(n_groups, 1) * sizeof(Moments));
            c->launches += 3;   // as for the other folds: k_group_medium, k_group_big, k_group_big_finish
            if (e == cudaSuccess)
                e = launch_group_moments(v->dtype, sval->chunks[0].values, sval->chunks[0].validity, d_starts, n_groups, n, mom, scratch, c->sm_count,
                                         c->s_compute);
        }
        for (int j = j0; j < n_aggs && e == cudaSuccess; j++) {
            if (aggs[j].column != v || !group_is_stat(aggs[j].function)) continue;
            bdf_col* r = res[j].get();
            {
                LaunchTimer t(c, BDF_K_GROUP, BDF_F64, n_groups, n_groups * ((int64_t)sizeof(Moments) + 8) + bitmap_bytes(n_groups));
                e = launch_group_stats(mom, n_groups, group_stat_of(aggs[j].function), (double*)r->chunks[0].values, r->chunks[0].validity, c->s_compute);
            }
            if (e == cudaSuccess) e = finish_single_group(c, r);
            r->null_counts[0] = -1;   // learnt on demand (ensure_null_counts)
            stat_done[j] = true;
        }
        if (e != cudaSuccess) return fail_cuda(e, "group statistics");
    }

    // count_distinct / sum_distinct: the distinct valid values of every group (distinct_runs); count_distinct counts them, sum_distinct
    // folds them -- in ascending order, with the SUM fold of launch_group_reduce over their own group starts
    for (int j = 0; j < n_aggs; j++) {
        const int fn = aggs[j].function;
        if (fn != BDF_GROUP_COUNT_DISTINCT && fn != BDF_GROUP_SUM_DISTINCT) continue;
        std::vector<const bdf_col*> sorted_keys;
        for (const ColOwner& s : runs.sorted) sorted_keys.push_back(s.get());
        DistinctRuns dr(c);
        TRY(distinct_runs(c, n_keys, keys, sorted_keys, aggs[j].column, runs.iota.get(), n, &dr));
        if (fn == BDF_GROUP_COUNT_DISTINCT) {
            TRY(col_alloc(c, BDF_I64, {ChunkPlan{n_groups, false}}, nullptr, 0, res[j].out()));
            bdf_col* cd = res[j].get();
            wait_groups(c->s_compute, dr.pos.get(), 0, 1);
            c->launches++;
            {
                LaunchTimer t(c, BDF_K_GROUP, BDF_I64, n_groups, n_groups * 16);
                e = launch_group_distinct((const uint32_t*)dr.pos->chunks[0].values, dr.pos->chunks[0].len, d_starts, n_groups, n,
                                          (long long*)cd->chunks[0].values, nullptr, c->s_compute);
            }
            if (e == cudaSuccess) e = finish_single_group(c, cd);
            if (e != cudaSuccess) return fail_cuda(e, "group distinct count");
        } else {
            ColOwner dstarts(c);
            TRY(col_alloc(c, BDF_U32, {ChunkPlan{n_groups, false}}, nullptr, 0, dstarts.out()));
            wait_groups(c->s_compute, dr.pos.get(), 0, 1);
            c->launches++;
            {
                LaunchTimer t(c, BDF_K_GROUP, BDF_U32, n_groups, n_groups * 12);
                e = launch_group_distinct((const uint32_t*)dr.pos->chunks[0].values, dr.pos->chunks[0].len, d_starts, n_groups, n, nullptr,
                                          (uint32_t*)dstarts->chunks[0].values, c->s_compute);
            }
            if (e == cudaSuccess) e = finish_single_group(c, dstarts.get());
            if (e != cudaSuccess) return fail_cuda(e, "group distinct starts");
            TRY(distinct_sum(c, dr, (const uint32_t*)dstarts->chunks[0].values, n_groups, res[j].out()));
        }
    }

    // median / mode: the same second sort; the median reads the two middle valid values of every group, the mode counts the distinct
    // runs (k_dist.cu)
    for (int j = 0; j < n_aggs; j++) {
        const int fn = aggs[j].function;
        if (fn != BDF_GROUP_MEDIAN && fn != BDF_GROUP_MODE) continue;
        std::vector<const bdf_col*> sorted_keys;
        for (const ColOwner& s : runs.sorted) sorted_keys.push_back(s.get());
        DistinctRuns dr(c);
        TRY(distinct_runs(c, n_keys, keys, sorted_keys, aggs[j].column, runs.iota.get(), n, &dr));
        if (fn == BDF_GROUP_MEDIAN) TRY(group_median(c, dr, d_starts, n_groups, n, res[j].out()));
        else TRY(group_mode(c, dr, d_starts, n_groups, n, res[j].out(), nullptr));
    }

    // collect_list / collect_set: lists of n_groups rows; collect_set shares one second sort per value column
    std::vector<Owned<bdf_list>> lists;
    for (int j = 0; j < n_aggs; j++) lists.emplace_back(c);
    for (int j = 0; j < n_aggs; j++) {
        const int fn = aggs[j].function;
        if (!group_is_collect(fn)) continue;
        if (fn == BDF_GROUP_COLLECT_LIST) { TRY(group_collect(c, runs, aggs[j].column, fn, nullptr, lists[j].out())); continue; }
        if (lists[j].get()) continue;   // made with an earlier collect_set of the same column
        std::vector<const bdf_col*> sorted_keys;
        for (const ColOwner& s : runs.sorted) sorted_keys.push_back(s.get());
        DistinctRuns dr(c);
        TRY(distinct_runs(c, n_keys, keys, sorted_keys, aggs[j].column, runs.iota.get(), n, &dr));
        for (int j2 = j; j2 < n_aggs; j2++)
            if (aggs[j2].function == BDF_GROUP_COLLECT_SET && aggs[j2].column == aggs[j].column)
                TRY(group_collect(c, runs, aggs[j].column, fn, &dr, lists[j2].out()));
    }
    for (int k = 0; k < n_keys; k++) out_keys[k] = runs.distinct[k].release();
    for (int j = 0; j < n_aggs; j++) out[j] = res[j].release();
    for (int j = 0; out_lists && j < n_aggs; j++) out_lists[j] = lists[j].release();
    if (n_groups_out) *n_groups_out = n_groups;
    return BDF_OK;
}

// The single-key entry of round 2: sum / count per value column, min / max for integer columns (floats: NULL pointers).
static int group_aggregate_dev(bdf_ctx* c, const bdf_col* key, int n_values, const bdf_col* const* values, bdf_col** out_keys,
                               bdf_group_out* outs, int64_t* n_groups_out) {
    if (key->dtype < 0 || key->dtype >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "the group key must be a numeric column");
    if (n_values < 0 || n_values > 64) return fail(BDF_INVALID, "0..64 value columns");
    std::vector<bdf_group_agg> aggs;
    for (int j = 0; j < n_values; j++) {
        if (!values[j]) return fail(BDF_INVALID, "null value column");
        if (values[j]->dtype < 0 || values[j]->dtype >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "aggregated columns must be numeric");
        aggs.push_back(bdf_group_agg{values[j], BDF_GROUP_SUM});
        aggs.push_back(bdf_group_agg{values[j], BDF_GROUP_COUNT});
        if (!dtype_is_float(values[j]->dtype)) {
            aggs.push_back(bdf_group_agg{values[j], BDF_GROUP_MIN});
            aggs.push_back(bdf_group_agg{values[j], BDF_GROUP_MAX});
        }
    }
    std::vector<bdf_col*> res(aggs.size(), nullptr);
    const int st = group_by_dev(c, 1, &key, (int)aggs.size(), aggs.data(), out_keys, res.data(), nullptr, n_groups_out);
    if (st != BDF_OK) {
        for (int j = 0; j < n_values; j++) outs[j] = bdf_group_out{nullptr, nullptr, nullptr, nullptr};
        return st;
    }
    size_t r = 0;
    for (int j = 0; j < n_values; j++) {
        const bool is_int = !dtype_is_float(values[j]->dtype);
        outs[j].sum = res[r++];
        outs[j].count = res[r++];
        outs[j].min = is_int ? res[r++] : nullptr;
        outs[j].max = is_int ? res[r++] : nullptr;
    }
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// statistical aggregates (k_moments.cu, moments.cuh): the moment record of a whole column, and its distinct values

static_assert(sizeof(Moments) == sizeof(bdf_moment_rec) && offsetof(bdf_moment_rec, m4) == offsetof(Moments, m4), "bdf_moment_rec layout");

// One launch of k_moments over every chunk and its finish; on a rank of a communicator the records of all ranks are all-gathered
// and merged in rank order, so every rank returns the same bits.
static int moments_dev(bdf_ctx* c, const bdf_col* col, Moments* out) {
    if (col->dtype < 0 || col->dtype >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "the statistics need a numeric column");
    const int64_t n = (int64_t)col->chunks.size();
    wait_groups(c->s_compute, col, 0, n);
    const int tile = elems_per_tile(col->dtype);
    void *hp = nullptr, *dp = nullptr;
    TRY(ring_alloc(c, (size_t)std::max<int64_t>(n, 1) * sizeof(RedDesc), &hp, &dp));
    RedDesc* hd = (RedDesc*)hp;
    int64_t tiles = 0, rows = 0;
    for (int64_t i = 0; i < n; i++) {
        const DevChunk& ch = col->chunks[i];
        hd[i].in = ch.values; hd[i].vin = ch.validity; hd[i].len = ch.len; hd[i].tile0 = tiles; hd[i].off = ch.bit_off; hd[i].pad = 0;
        tiles += (ch.len + tile - 1) / tile;
        rows += ch.len;
    }
    CK(desc_upload(c, dp, hd, (size_t)n * sizeof(RedDesc)));
    Scratch<Moments> parts;
    Moments* result = (Moments*)c->h_agg_dev;   // device-mapped pinned memory: the finish writes the record straight to the host
    {
        LaunchTimer t(c, BDF_K_MOMENTS, col->dtype, rows, reduce_bytes(col, 0, n));   // k_moments + k_moments_finish
        CK(parts.alloc(c, (size_t)std::max<int64_t>(moments_partials(tiles), 1) * sizeof(Moments)));
        CK(launch_moments(col->dtype, (const RedDesc*)dp, (int)n, tiles, parts, result, c->s_compute));
        c->launches++;
    }
    CK(cudaStreamSynchronize(c->s_compute));
    Moments mine;
    memcpy(&mine, (const void*)c->h_agg, sizeof mine);
    if (is_global(c)) {
        std::vector<Moments> all((size_t)comm_world(c->comm));
        std::string err;
        c->collectives++;
        cudaError_t e = comm_host_allgather(c->comm, &mine, all.data(), sizeof(Moments), c->s_compute, &err);
        if (e != cudaSuccess) { g_nccl_err = err; return fail_cuda(e, "moments"); }
        mine = Moments{0, 0.0, 0.0, 0.0, 0.0};
        for (const Moments& m : all) mine = moments_merge(mine, m);
    }
    *out = mine;
    return BDF_OK;
}

// The distinct runs of a whole column of n > 0 rows, handled as one group (starts: that group's start, 0).
static int column_runs(bdf_ctx* c, const bdf_col* x, DistinctRuns* dr, ColOwner* starts) {
    const int64_t n = x->total_len;
    ColOwner iota(c);
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{n, false}}, nullptr, 0, iota.out()));
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{1, false}}, nullptr, 0, starts->out()));
    c->launches++;
    cudaError_t e = launch_iota((uint32_t*)iota->chunks[0].values, n, c->sm_count, c->s_compute);
    if (e == cudaSuccess) e = cudaMemsetAsync((*starts)->chunks[0].values, 0, sizeof(uint32_t), c->s_compute);   // the one group starts at 0
    if (e == cudaSuccess) e = finish_single_group(c, iota.get());
    if (e == cudaSuccess) e = finish_single_group(c, starts->get());
    if (e != cudaSuccess) return fail_cuda(e, "distinct iota");
    return distinct_runs(c, 0, nullptr, {}, x, iota.get(), n, dr);
}

// count_distinct / sum_distinct of a whole column: the group-by's distinct machinery with the column as one group.
static int distinct_dev(bdf_ctx* c, const bdf_col* x, bdf_distinct_rec* out) {
    if (x->dtype < 0 || x->dtype >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "count_distinct / sum_distinct need a numeric column");
    if (is_global(c))
        return fail(BDF_UNSUPPORTED, "distinct values need every row of the column on one GPU (as sort / group-by / join): use a one-GPU context");
    const int64_t n = x->total_len;
    if (n == 0) { *out = bdf_distinct_rec{0, 0}; return BDF_OK; }
    ColOwner first(c), sum(c);
    DistinctRuns dr(c);
    TRY(column_runs(c, x, &dr, &first));
    const int64_t count = dr.pos->chunks.empty() ? 0 : dr.pos->chunks[0].len;
    TRY(distinct_sum(c, dr, (const uint32_t*)first->chunks[0].values, 1, sum.out()));
    uint64_t bits = 0;
    CK(cudaMemcpyAsync(&bits, sum->chunks[0].values, (size_t)dtype_width(x->dtype), cudaMemcpyDeviceToHost, c->s_compute));
    CK(cudaStreamSynchronize(c->s_compute));
    *out = bdf_distinct_rec{count, bits};
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// distributions (k_dist.cu, dist.cuh): exact percentiles by an MSD radix select, the histogram, mode and uniques

static int dist_check(bdf_ctx* c, const bdf_col* x) {
    if (x->dtype < 0 || x->dtype >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "the distributions need a numeric column");
    if (is_global(c)) return fail(BDF_UNSUPPORTED, "the distributions need every row of the column on one GPU: use a one-GPU context");
    if (x->total_len > 0xffffffffLL) return fail(BDF_UNSUPPORTED, "sort indices are UInt32: at most 2^32-1 rows");
    return BDF_OK;
}

// The chunks of col as k_reduce descriptors with tiles of dist_tile_elems(dtype) elements.
static int dist_descs(bdf_ctx* c, const bdf_col* col, const RedDesc** d, int64_t* tiles) {
    const int64_t n = (int64_t)col->chunks.size();
    wait_groups(c->s_compute, col, 0, n);
    const int tile = dist_tile_elems(col->dtype);
    void *hp = nullptr, *dp = nullptr;
    TRY(ring_alloc(c, (size_t)std::max<int64_t>(n, 1) * sizeof(RedDesc), &hp, &dp));
    RedDesc* hd = (RedDesc*)hp;
    int64_t t = 0;
    for (int64_t i = 0; i < n; i++) {
        const DevChunk& ch = col->chunks[i];
        hd[i].in = ch.values; hd[i].vin = ch.validity; hd[i].len = ch.len; hd[i].tile0 = t; hd[i].off = ch.bit_off; hd[i].pad = 0;
        t += (ch.len + tile - 1) / tile;
    }
    CK(desc_upload(c, dp, hd, (size_t)n * sizeof(RedDesc)));
    *d = (const RedDesc*)dp;
    *tiles = t;
    return BDF_OK;
}

// The value a sort key stands for, read as f64 (+0.0 for a zero, the positive quiet NaN for NaN).
static double key_value(int dtype, uint64_t k) {
    switch (dtype) {
        case BDF_I8: return (double)(int8_t)(uint8_t)(k ^ 0x80u);
        case BDF_I16: return (double)(int16_t)(uint16_t)(k ^ 0x8000u);
        case BDF_I32: return (double)(int32_t)(uint32_t)(k ^ 0x80000000u);
        case BDF_I64: return (double)(int64_t)(k ^ (1ull << 63));
        case BDF_F32: {
            const uint32_t b = (k >> 31) ? (uint32_t)k ^ 0x80000000u : ~(uint32_t)k;
            float f;
            memcpy(&f, &b, sizeof f);
            return dist_canonical((double)f);
        }
        case BDF_F64: {
            const uint64_t b = (k >> 63) ? k ^ (1ull << 63) : ~k;
            double f;
            memcpy(&f, &b, sizeof f);
            return dist_canonical(f);
        }
        default: return (double)k;
    }
}

constexpr int kMaxPercentiles = 1024;

// MSD radix select: the keys of the valid values at the given ranks (0-based in key order).  ranks_of(n_valid) gives the wanted ranks,
// ascending and distinct, once the first pass has counted the valid values; n_valid = 0 selects nothing.
//   A level histograms one 8-bit digit of every candidate (a key whose decided high bits equal a target's prefix), then every target
//   takes the bucket holding its rank.  Bits below the digit on which every candidate agrees (their AND equals their OR there) are
//   decided at once.  When the chosen buckets hold fewer keys than the candidates, those keys are compacted into a scratch that the
//   next level reads instead; otherwise (a column of one value, or every bucket chosen) the next level reads the same source again.
static int select_keys(bdf_ctx* c, const bdf_col* col, const std::function<std::vector<int64_t>(int64_t)>& ranks_of, int max_targets,
                       std::vector<uint64_t>* keys, int64_t* n_valid) {
    const int dt = col->dtype, w = dtype_width(dt), kb = w <= 4 ? 4 : 8;
    const RedDesc* cd = nullptr;
    int64_t col_tiles = 0;
    TRY(dist_descs(c, col, &cd, &col_tiles));
    const int64_t col_bytes = reduce_bytes(col, 0, (int64_t)col->chunks.size());
    const size_t max_bins = (size_t)max_targets * 256;
    Scratch<unsigned long long> hist, small, d_pre;   // small: AND, OR, cursor
    Scratch<uint32_t> chosen;
    CK(hist.alloc(c, max_bins * 8));
    CK(small.alloc(c, 3 * 8));
    CK(d_pre.alloc(c, (size_t)max_targets * 8));
    CK(chosen.alloc(c, max_bins / 8));
    std::unique_ptr<Scratch<void>> cur;   // the candidates of the current source when it is a scratch
    const RedDesc* src = cd;              // the current source: the column (key_bytes 0) or the scratch (raw keys)
    int src_n = (int)col->chunks.size(), src_kb = 0;
    int64_t src_tiles = col_tiles, src_bytes = col_bytes, cand = 0;
    struct Target { uint64_t prefix; int64_t rank; };
    std::vector<Target> tg;
    std::vector<uint64_t> pre{0}, hh(max_bins), ao(2);
    uint64_t pmask = 0;
    int s_top = 8 * w;   // bits at and above s_top are decided (zero above the type's width)
    for (int level = 0; s_top > 0; level++) {
        const int shift = std::max(0, s_top - 8), m = (int)pre.size();
        const uint64_t ao0[3] = {~0ull, 0ull, 0ull};
        CK(cudaMemcpyAsync(d_pre, pre.data(), (size_t)m * 8, cudaMemcpyHostToDevice, c->s_compute));
        CK(cudaMemcpyAsync(small, ao0, sizeof ao0, cudaMemcpyHostToDevice, c->s_compute));
        CK(cudaMemsetAsync(hist, 0, (size_t)m * 256 * 8, c->s_compute));
        {
            LaunchTimer t(c, BDF_K_SELECT, dt, src_kb ? cand : col->total_len, src_bytes);
            CK(launch_select_pass(dt, src_kb, false, src, src_n, src_tiles, d_pre, m, pmask, shift, hist, small, nullptr, nullptr, nullptr,
                                  c->sm_count, c->s_compute));
        }
        CK(cudaMemcpyAsync(hh.data(), hist, (size_t)m * 256 * 8, cudaMemcpyDeviceToHost, c->s_compute));
        CK(cudaMemcpyAsync(ao.data(), small, 2 * 8, cudaMemcpyDeviceToHost, c->s_compute));
        CK(cudaStreamSynchronize(c->s_compute));
        if (level == 0) {
            cand = 0;
            for (int d = 0; d < 256; d++) cand += (int64_t)hh[d];
            *n_valid = cand;
            if (!cand) return BDF_OK;
            for (int64_t r : ranks_of(cand)) tg.push_back(Target{0, r});
        }
        // every target takes the bucket of its rank inside its class (targets ascend, so do their prefixes)
        std::vector<uint32_t> chosen_bits((size_t)m * 8, 0u);
        int64_t kept = 0;
        size_t ci = 0;
        for (Target& t : tg) {
            while (pre[ci] != t.prefix) ci++;
            const uint64_t* h = &hh[ci * 256];
            int64_t cum = 0;
            int d = 0;
            while (cum + (int64_t)h[d] <= t.rank) cum += (int64_t)h[d++];
            t.rank -= cum;
            t.prefix |= (uint64_t)d << shift;
            const size_t bin = ci * 256 + (size_t)d;
            if (!((chosen_bits[bin >> 5] >> (bin & 31)) & 1u)) {
                chosen_bits[bin >> 5] |= 1u << (bin & 31);
                kept += (int64_t)h[d];
            }
        }
        // bits below the digit on which every candidate agrees are decided too
        const uint64_t low = shift ? (1ull << shift) - 1 : 0ull, diff = (ao[0] ^ ao[1]) & low;
        const int new_top = diff ? 64 - __builtin_clzll(diff) : 0;
        const uint64_t agreed = low & ~(new_top ? (new_top == 64 ? ~0ull : (1ull << new_top) - 1) : 0ull);
        for (Target& t : tg) t.prefix |= ao[0] & agreed;
        if (new_top == 0) break;
        if (kept < cand) {   // compact the chosen buckets (this level's prefixes and digit)
            std::unique_ptr<Scratch<void>> next(new Scratch<void>());
            CK(next->alloc(c, (size_t)kept * kb));
            CK(cudaMemcpyAsync(chosen, chosen_bits.data(), chosen_bits.size() * 4, cudaMemcpyHostToDevice, c->s_compute));
            CK(cudaMemsetAsync(small.get() + 2, 0, 8, c->s_compute));
            {
                LaunchTimer t(c, BDF_K_SELECT, dt, src_kb ? cand : col->total_len, src_bytes + kept * kb);
                CK(launch_select_pass(dt, src_kb, true, src, src_n, src_tiles, d_pre, m, pmask, shift, nullptr, nullptr, chosen, next->get(),
                                      small.get() + 2, c->sm_count, c->s_compute));
            }
            void *hp = nullptr, *dp = nullptr;
            TRY(ring_alloc(c, sizeof(RedDesc), &hp, &dp));
            RedDesc* hd = (RedDesc*)hp;
            const int tile = kThreads * kUnroll * (16 / kb);
            hd->in = next->get(); hd->vin = nullptr; hd->len = kept; hd->tile0 = 0; hd->off = 0; hd->pad = 0;
            CK(desc_upload(c, dp, hd, sizeof(RedDesc)));
            cur = std::move(next);   // the previous scratch is freed in stream order, after the compaction that read it
            src = (const RedDesc*)dp; src_n = 1; src_kb = kb;
            src_tiles = (kept + tile - 1) / tile;
            src_bytes = kept * kb;
            cand = kept;
        }
        pre.clear();
        for (const Target& t : tg)
            if (pre.empty() || pre.back() != t.prefix) pre.push_back(t.prefix);
        s_top = new_top;
        pmask = ~((1ull << s_top) - 1) & (kb == 4 ? 0xffffffffull : ~0ull);
    }
    keys->clear();
    for (const Target& t : tg) keys->push_back(t.prefix);
    return BDF_OK;
}

static int percentile_dev(bdf_ctx* c, const bdf_col* col, int n_p, const double* p, double* out, int32_t* is_some) {
    TRY(dist_check(c, col));
    std::vector<double> pos((size_t)n_p);
    std::vector<int64_t> ranks;
    auto ranks_of = [&](int64_t n) {
        for (int i = 0; i < n_p; i++) {
            pos[i] = dist_mul((double)(n - 1), p[i]);
            ranks.push_back((int64_t)floor(pos[i]));
            ranks.push_back((int64_t)ceil(pos[i]));
        }
        std::sort(ranks.begin(), ranks.end());
        ranks.erase(std::unique(ranks.begin(), ranks.end()), ranks.end());
        return ranks;
    };
    std::vector<uint64_t> keys;
    int64_t n_valid = 0;
    TRY(select_keys(c, col, ranks_of, 2 * n_p, &keys, &n_valid));
    for (int i = 0; i < n_p; i++) {
        if (!n_valid) { out[i] = 0.0; is_some[i] = 0; continue; }
        const double lo = floor(pos[i]), hi = ceil(pos[i]);
        const size_t a = std::lower_bound(ranks.begin(), ranks.end(), (int64_t)lo) - ranks.begin();
        const size_t b = std::lower_bound(ranks.begin(), ranks.end(), (int64_t)hi) - ranks.begin();
        out[i] = dist_interp(key_value(col->dtype, keys[a]), key_value(col->dtype, keys[b]), pos[i], lo, hi);
        is_some[i] = 1;
    }
    return BDF_OK;
}

static int mode_dev(bdf_ctx* c, const bdf_col* x, uint64_t* bits, int64_t* freq, int32_t* is_some) {
    TRY(dist_check(c, x));
    const int64_t n = x->total_len;
    if (n == 0) { *bits = 0; *freq = 0; *is_some = 0; return BDF_OK; }
    ColOwner first(c), val(c);
    DistinctRuns dr(c);
    TRY(column_runs(c, x, &dr, &first));
    Scratch<long long> d_freq;
    CK(d_freq.alloc(c, sizeof(long long)));
    TRY(group_mode(c, dr, (const uint32_t*)first->chunks[0].values, 1, n, val.out(), d_freq));
    uint64_t b = 0;
    long long f = 0;
    wait_groups(c->s_compute, val.get(), 0, 1);
    CK(cudaMemcpyAsync(&b, val->chunks[0].values, (size_t)dtype_width(x->dtype), cudaMemcpyDeviceToHost, c->s_compute));
    CK(cudaMemcpyAsync(&f, d_freq, sizeof f, cudaMemcpyDeviceToHost, c->s_compute));
    CK(cudaStreamSynchronize(c->s_compute));
    *bits = f ? b : 0;
    *freq = f;
    *is_some = f ? 1 : 0;
    return BDF_OK;
}

static int uniques_dev(bdf_ctx* c, const bdf_col* x, bdf_col** values, bdf_col** counts) {
    TRY(dist_check(c, x));
    const int64_t n = x->total_len;
    ColOwner v(c), cnt(c);
    if (n == 0) {
        TRY(col_alloc(c, x->dtype, {ChunkPlan{0, false}}, nullptr, 0, v.out()));
        if (counts) TRY(col_alloc(c, BDF_I64, {ChunkPlan{0, false}}, nullptr, 0, cnt.out()));
    } else {
        ColOwner first(c);
        DistinctRuns dr(c);
        TRY(column_runs(c, x, &dr, &first));
        TRY(filter_dev(c, dr.sval.get(), dr.dhead.get(), v.out()));
        if (counts) {
            const int64_t n_pos = dr.pos->chunks.empty() ? 0 : dr.pos->chunks[0].len;
            const uint32_t* d_starts = (const uint32_t*)first->chunks[0].values;
            Scratch<uint32_t> first_run, vend;
            TRY(dist_group_bounds(c, dr, d_starts, 1, n, true, &first_run, &vend));
            TRY(col_alloc(c, BDF_I64, {ChunkPlan{n_pos, false}}, nullptr, 0, cnt.out()));
            cudaError_t e;
            {
                LaunchTimer t(c, BDF_K_GROUP, BDF_I64, n_pos, n_pos * 12);
                e = launch_dist_runs(n_pos ? (const uint32_t*)dr.pos->chunks[0].values : nullptr, n_pos, d_starts, 1, n, first_run, vend,
                                     n_pos ? (long long*)cnt->chunks[0].values : nullptr, nullptr, c->s_compute);
            }
            if (e == cudaSuccess) e = finish_single_group(c, cnt.get());
            if (e != cudaSuccess) return fail_cuda(e, "uniques counts");
        }
    }
    *values = v.release();
    if (counts) *counts = cnt.release();
    return BDF_OK;
}

// numpy's linspace of the bin edges (dist.cuh's operations: one rounding each).
static void hist_edges(double lo, double hi, int nbins, double* edges) {
    const double delta = dist_sub(hi, lo), step = delta / (double)nbins;
    for (int i = 0; i < nbins; i++)
        edges[i] = step == 0.0 ? dist_add(dist_mul((double)i / (double)nbins, delta), lo) : dist_add(dist_mul((double)i, step), lo);
    edges[nbins] = hi;
}

static int hist_dev(bdf_ctx* c, const bdf_col* x, int nbins, const double* range, double* edges_out, int64_t* counts_out) {
    TRY(dist_check(c, x));
    double lo = 0.0, hi = 1.0;
    if (range) {
        lo = range[0];
        hi = range[1];
        if (lo > hi) return fail(BDF_INVALID, "max must be larger than min in range parameter.");
        if (!std::isfinite(lo) || !std::isfinite(hi)) return fail(BDF_INVALID, "supplied range of [%.17g, %.17g] is not finite", lo, hi);
    }
    const RedDesc* d = nullptr;
    int64_t tiles = 0;
    TRY(dist_descs(c, x, &d, &tiles));
    const int64_t bytes = reduce_bytes(x, 0, (int64_t)x->chunks.size());
    Scratch<unsigned long long> dev;
    Scratch<double> d_edges;
    CK(dev.alloc(c, (size_t)std::max(nbins, 2) * 8));   // the range pass writes two keys
    CK(d_edges.alloc(c, (size_t)(nbins + 1) * 8));
    if (!range) {   // [min, max] of the valid non-NaN values
        const unsigned long long init[2] = {~0ull, 0ull};
        unsigned long long mm[2];
        CK(cudaMemcpyAsync(dev, init, sizeof init, cudaMemcpyHostToDevice, c->s_compute));
        {
            LaunchTimer t(c, BDF_K_HIST, x->dtype, x->total_len, bytes);
            CK(launch_hist(x->dtype, true, d, (int)x->chunks.size(), tiles, nullptr, 0.0, 0.0, 0, dev, c->sm_count, c->s_compute));
        }
        CK(cudaMemcpyAsync(mm, dev, sizeof mm, cudaMemcpyDeviceToHost, c->s_compute));
        CK(cudaStreamSynchronize(c->s_compute));
        if (mm[0] <= mm[1]) {
            lo = key_value(x->dtype, mm[0]);
            hi = key_value(x->dtype, mm[1]);
            if (!std::isfinite(lo) || !std::isfinite(hi)) return fail(BDF_INVALID, "autodetected range of [%.17g, %.17g] is not finite", lo, hi);
        }
    }
    if (lo == hi) { lo = dist_sub(lo, 0.5); hi = dist_add(hi, 0.5); }
    std::vector<double> edges((size_t)nbins + 1);
    std::vector<int64_t> counts((size_t)nbins);
    hist_edges(lo, hi, nbins, edges.data());
    CK(cudaMemcpyAsync(d_edges, edges.data(), edges.size() * 8, cudaMemcpyHostToDevice, c->s_compute));
    CK(cudaMemsetAsync(dev, 0, (size_t)nbins * 8, c->s_compute));
    {
        LaunchTimer t(c, BDF_K_HIST, x->dtype, x->total_len, bytes);
        CK(launch_hist(x->dtype, false, d, (int)x->chunks.size(), tiles, d_edges, lo, hi, nbins, dev, c->sm_count, c->s_compute));
    }
    CK(cudaMemcpyAsync(counts.data(), dev, (size_t)nbins * 8, cudaMemcpyDeviceToHost, c->s_compute));
    CK(cudaStreamSynchronize(c->s_compute));
    memcpy(edges_out, edges.data(), edges.size() * 8);
    memcpy(counts_out, counts.data(), counts.size() * 8);
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// equi-join (k_join.cu): the build side (the right side; the left side for RIGHT) is sorted, gathered and cut into runs of equal
// key tuples by sorted_runs, as group-by's groups are; every probe row binary-searches the distinct tuples, the counts are scanned into
// output offsets (one host wait for the total), and the emit writes the index pairs by output position.  FULL appends the build
// rows of the runs no probe row hit, listed in row order by a compaction of an iota.  LEFT SEMI / ANTI write one bit per left row
// instead and compact an iota of the left rows with it.

// What the probe kernels read of every criterion: the probe column's chunk table and the build side's distinct keys.
struct JoinProbe {
    std::vector<const void*> tables, build;
    std::vector<const uint32_t*> build_valid;
    std::vector<int> chunks, dtypes;
    int64_t key_bytes = 0;
};

static int join_probe(bdf_ctx* c, int n_keys, const bdf_col* const* probe, const SortedRuns& runs, JoinProbe* p) {
    for (int k = 0; k < n_keys; k++) {
        void* t = nullptr;
        int n_chunks = 0;
        TRY(sort_table(c, probe[k], &t, &n_chunks, nullptr));
        p->tables.push_back(t);
        p->chunks.push_back(n_chunks);
        p->build.push_back(runs.distinct[k]->chunks[0].values);
        p->build_valid.push_back(runs.distinct[k]->chunks[0].validity);
        p->dtypes.push_back(probe[k]->dtype);
        p->key_bytes += dtype_width(probe[k]->dtype);
    }
    return BDF_OK;
}

// LEFT SEMI / ANTI: the left rows with (without) a partner, ascending.  No counts and no host wait for a total: a bit per left row
// compacts an iota, as FULL lists its unmatched rows.
static int join_exists_dev(bdf_ctx* c, bool anti, int n_keys, const bdf_col* const* lk, const bdf_col* const* rk, bdf_col** out_l, bdf_col** out_r,
                           int64_t* n_rows_out) {
    const int64_t np = lk[0]->total_len;
    SortedRuns runs(c);
    TRY(sorted_runs(c, n_keys, n_keys, rk, "join iota", &runs));
    JoinProbe p;
    TRY(join_probe(c, n_keys, lk, runs, &p));
    ColOwner mask(c), iota(c), rows(c);
    TRY(col_alloc(c, kBool, {ChunkPlan{np, false}}, nullptr, 0, mask.out()));
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{np, false}}, nullptr, 0, iota.out()));
    cudaError_t e;
    {
        LaunchTimer t(c, BDF_K_JOIN, kBool, np, np * p.key_bytes + bitmap_bytes(np));
        e = launch_join_exists(n_keys, p.dtypes.data(), p.tables.data(), p.chunks.data(), p.build.data(), p.build_valid.data(), np, runs.n_runs,
                               anti ? 1 : 0, (uint32_t*)mask->chunks[0].values, c->s_compute);
    }
    c->launches++;
    if (e == cudaSuccess && np > 0) e = launch_iota((uint32_t*)iota->chunks[0].values, np, c->sm_count, c->s_compute);
    if (e == cudaSuccess) e = finish_single_group(c, mask.get());
    if (e == cudaSuccess) e = finish_single_group(c, iota.get());
    if (e != cudaSuccess) return fail_cuda(e, "join existence mask");
    TRY(filter_dev(c, iota.get(), mask.get(), rows.out()));
    if (n_rows_out) *n_rows_out = rows->chunks[0].len;
    *out_l = rows.release();
    if (out_r) *out_r = nullptr;
    return BDF_OK;
}

static int join_dev(bdf_ctx* c, int how, int n_keys, const bdf_col* const* lk, const bdf_col* const* rk, bdf_col** out_l, bdf_col** out_r,
                    int64_t* n_rows_out) {
    if (n_keys == 0) return fail(BDF_INVALID, "Join criteria cannot be empty");
    if (n_keys < 0 || n_keys > 16) return fail(BDF_INVALID, "1..16 join criteria");
    if (!lk || !rk) return fail(BDF_INVALID, "null argument");
    for (int k = 0; k < n_keys; k++)
        if (!lk[k] || !rk[k]) return fail(BDF_INVALID, "null join column");
    if (how < BDF_JOIN_LEFT || how > BDF_JOIN_LEFT_ANTI) return fail(BDF_UNSUPPORTED, "unknown join type %d", how);
    for (int k = 0; k < n_keys; k++)
        if (lk[k]->dtype < 0 || lk[k]->dtype >= BDF_NTYPES || rk[k]->dtype < 0 || rk[k]->dtype >= BDF_NTYPES)
            return fail(BDF_UNSUPPORTED, "join columns must be numeric");
    for (int k = 0; k < n_keys; k++)
        if (lk[k]->dtype != rk[k]->dtype) return fail(BDF_UNSUPPORTED, "Join columns must have compatible types");
    for (int k = 0; k < n_keys; k++)
        if (lk[k]->total_len != lk[0]->total_len || rk[k]->total_len != rk[0]->total_len)
            return fail(BDF_LENGTH_MISMATCH, "join columns of one side have different lengths");
    if (lk[0]->total_len > 0xffffffffLL || rk[0]->total_len > 0xffffffffLL) return fail(BDF_UNSUPPORTED, "sort indices are UInt32: at most 2^32-1 rows");
    if (how == BDF_JOIN_LEFT_SEMI || how == BDF_JOIN_LEFT_ANTI) return join_exists_dev(c, how == BDF_JOIN_LEFT_ANTI, n_keys, lk, rk, out_l, out_r, n_rows_out);
    const bool swap = how == BDF_JOIN_RIGHT, full = how == BDF_JOIN_FULL, outer = how != BDF_JOIN_INNER;
    const bdf_col* const* probe = swap ? rk : lk;
    const bdf_col* const* build = swap ? lk : rk;
    const int64_t np = probe[0]->total_len, nb = build[0]->total_len;

    // the build side: sorted row numbers, the distinct key tuples, the first sorted row of every run
    SortedRuns runs(c);
    TRY(sorted_runs(c, n_keys, n_keys, build, "join iota", &runs));
    const int64_t n_runs = runs.n_runs;
    const uint32_t* perm = (const uint32_t*)runs.perm->chunks[0].values;
    const uint32_t* starts = (const uint32_t*)runs.starts->chunks[0].values;

    // the probe side is read in place, through the chunk tables of its key columns
    JoinProbe jp;
    TRY(join_probe(c, n_keys, probe, runs, &jp));
    const int64_t blocks = scan_tile_sums(np);
    Scratch<unsigned long long> counts, block_sums;
    Scratch<uint32_t> mstart;
    Scratch<unsigned char> hit;
    cudaError_t e = counts.alloc(c, (size_t)(np + 1) * sizeof(unsigned long long));
    if (e == cudaSuccess) e = mstart.alloc(c, (size_t)std::max<int64_t>(np, 1) * sizeof(uint32_t));
    if (e == cudaSuccess) e = block_sums.alloc(c, (size_t)blocks * sizeof(unsigned long long));
    if (e == cudaSuccess && full) e = hit.alloc(c, (size_t)std::max<int64_t>(n_runs, 1));
    if (e == cudaSuccess && full) e = cudaMemsetAsync(hit, 0, (size_t)std::max<int64_t>(n_runs, 1), c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "join scratch allocation");
    unsigned long long total = 0;   // output rows of the probe part
    {
        LaunchTimer t(c, BDF_K_JOIN, BDF_U32, np, np * (jp.key_bytes + 8 + 4));
        e = launch_join_count(n_keys, jp.dtypes.data(), jp.tables.data(), jp.chunks.data(), jp.build.data(), jp.build_valid.data(), np, starts, n_runs, nb,
                              outer ? 1 : 0, counts, mstart, hit, block_sums, c->s_compute);
    }
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_JOIN, BDF_U64, np, np > 0 ? np * 16 + blocks * 16 : 0);   // no probe rows: a memset of the total
        c->launches += kScanSumsLaunches - 1;   // the timer counts one
        e = launch_scan_sums(counts, np, block_sums, c->s_compute);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&total, counts + np, sizeof(total), cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);   // the output length sizes the result
    if (e != cudaSuccess) return fail_cuda(e, "join count");

    // FULL: the build rows of runs nobody hit, in row order
    ColOwner mask(c), unm(c);
    int64_t n_unm = 0;
    if (full) {
        TRY(col_alloc(c, kBool, {ChunkPlan{nb, false}}, nullptr, 0, mask.out()));
        e = nb > 0 ? cudaMemsetAsync(mask->chunks[0].values, 0, (size_t)(nb + 31) / 32 * 4, c->s_compute) : cudaSuccess;
        if (e == cudaSuccess) {
            LaunchTimer t(c, BDF_K_JOIN, kBool, nb, nb * 8 + n_runs * 5);
            e = launch_join_unmatched(perm, nb, starts, n_runs, hit, (uint32_t*)mask->chunks[0].values, c->sm_count, c->s_compute);
        }
        if (e == cudaSuccess) e = finish_single_group(c, mask.get());
        if (e != cudaSuccess) return fail_cuda(e, "join unmatched rows");
        TRY(filter_dev(c, runs.iota.get(), mask.get(), unm.out()));
        n_unm = unm->chunks[0].len;
    }

    const unsigned long long n_out = total + (unsigned long long)n_unm;
    if ((long double)n_out * 8.25L > (long double)c->hbm_bytes)   // two UInt32 columns and their bitmaps
        return fail(BDF_OOM, "a join output of %llu rows does not fit in device memory", n_out);
    ColOwner pidx(c), bidx(c);
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{(int64_t)n_out, full}}, nullptr, 0, pidx.out()));
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{(int64_t)n_out, outer}}, nullptr, 0, bidx.out()));
    {
        LaunchTimer t(c, BDF_K_JOIN, BDF_U32, (int64_t)n_out, (int64_t)n_out * 12 + (int64_t)bitmap_bytes((int64_t)n_out) * 2);
        e = launch_join_emit(counts, np, mstart, perm, total, unm.get() ? (const uint32_t*)unm->chunks[0].values : nullptr, n_out,
                             (uint32_t*)pidx->chunks[0].values, pidx->chunks[0].validity, (uint32_t*)bidx->chunks[0].values, bidx->chunks[0].validity,
                             c->s_compute);
    }
    if (e == cudaSuccess) e = finish_single_group(c, pidx.get());
    if (e == cudaSuccess) e = finish_single_group(c, bidx.get());
    if (e != cudaSuccess) return fail_cuda(e, "join emit");
    pidx->null_counts[0] = full ? n_unm : 0;
    bidx->null_counts[0] = outer ? -1 : 0;   // the probe rows without a partner: counted on demand
    bdf_col* p = pidx.release();
    bdf_col* b = bidx.release();
    *out_l = swap ? b : p;
    *out_r = swap ? p : b;
    if (n_rows_out) *n_rows_out = (int64_t)n_out;
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// as-of join (k_join.cu k_join_asof): the right side is sorted once by (by..., on), stably, and cut into runs on the `by` keys only;
// every left row finds its run with the equi-join's search and its `on` key inside the run, reading the left chunks in place.

static int join_asof_dev(bdf_ctx* c, const bdf_col* lon, const bdf_col* ron, int n_by, const bdf_col* const* lby, const bdf_col* const* rby,
                         const bdf_asof_spec* spec, bdf_col** out) {
    if (n_by < 0 || n_by > 16) return fail(BDF_INVALID, "0..16 as-of by keys");
    if (!lon || !ron || !spec || !out || (n_by && (!lby || !rby))) return fail(BDF_INVALID, "null argument");
    std::vector<const bdf_col*> lk, rk;   // by..., on
    for (int k = 0; k < n_by; k++) {
        if (!lby[k] || !rby[k]) return fail(BDF_INVALID, "null join column");
        lk.push_back(lby[k]);
        rk.push_back(rby[k]);
    }
    lk.push_back(lon);
    rk.push_back(ron);
    const int nk = n_by + 1;
    if (spec->direction < BDF_ASOF_BACKWARD || spec->direction > BDF_ASOF_NEAREST) return fail(BDF_UNSUPPORTED, "unknown as-of direction %d", spec->direction);
    for (int k = 0; k < nk; k++)
        if (lk[k]->dtype < 0 || lk[k]->dtype >= BDF_NTYPES || rk[k]->dtype < 0 || rk[k]->dtype >= BDF_NTYPES)
            return fail(BDF_UNSUPPORTED, "join columns must be numeric");
    for (int k = 0; k < nk; k++)
        if (lk[k]->dtype != rk[k]->dtype) return fail(BDF_UNSUPPORTED, "Join columns must have compatible types");
    if (spec->has_tolerance && (dtype_is_float(lon->dtype) ? !(spec->tolerance_f >= 0.0) : spec->tolerance < 0))
        return fail(BDF_INVALID, "the as-of tolerance must be >= 0");
    for (int k = 0; k < nk; k++)
        if (lk[k]->total_len != lon->total_len || rk[k]->total_len != ron->total_len)
            return fail(BDF_LENGTH_MISMATCH, "join columns of one side have different lengths");
    if (ron->total_len > 0xffffffffLL) return fail(BDF_UNSUPPORTED, "sort indices are UInt32: at most 2^32-1 rows");
    const int64_t nl = lon->total_len, nr = ron->total_len;

    SortedRuns runs(c);
    TRY(sorted_runs(c, nk, n_by, rk.data(), "as-of join iota", &runs));
    JoinProbe p;
    TRY(join_probe(c, n_by, lk.data(), runs, &p));
    void* on_table = nullptr;
    int on_chunks = 0;
    TRY(sort_table(c, lon, &on_table, &on_chunks, nullptr));
    const DevChunk& son = runs.sorted[n_by]->chunks[0];   // the right `on` key in sorted order
    ColOwner o(c);
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{nl, true}}, nullptr, 0, o.out()));
    cudaError_t e;
    {
        LaunchTimer t(c, BDF_K_JOIN, lon->dtype, nl, nl * (p.key_bytes + dtype_width(lon->dtype) + 4) + bitmap_bytes(nl));
        e = launch_join_asof(n_by, p.dtypes.data(), p.tables.data(), p.chunks.data(), p.build.data(), p.build_valid.data(), lon->dtype, on_table,
                             on_chunks, son.values, son.validity, spec->direction, spec->allow_exact_matches ? 1 : 0, spec->has_tolerance ? 1 : 0,
                             (unsigned long long)spec->tolerance, spec->tolerance_f, nl,
                             n_by ? (const uint32_t*)runs.starts->chunks[0].values : nullptr, runs.n_runs, nr,
                             (const uint32_t*)runs.perm->chunks[0].values, (uint32_t*)o->chunks[0].values, o->chunks[0].validity, c->s_compute);
    }
    if (e == cudaSuccess) e = finish_single_group(c, o.get());
    if (e != cudaSuccess) return fail_cuda(e, "as-of join");
    o->null_counts[0] = -1;   // the rows without a partner: counted on demand
    *out = o.release();
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// window functions (k_window.cu): the rows are sorted by (partition keys, order keys) once for all calls; the partition heads (P) and
// the peer heads (Q = P OR the order keys' heads) are marked with k_group_heads, and each gets a per-word prefix of its runs and the
// compacted run starts, so a position finds its partition and peer bounds in O(1).  Ranking functions are written straight to row
// order through the permutation; lag / lead and the scans work in sorted order and come back through one take each, whose index
// is the frame's last sorted position of every row.  Without any key nothing is sorted: the kernels read the caller's chunks in place.

static bool win_is_rank(int f) { return f >= BDF_WIN_ROW_NUMBER && f <= BDF_WIN_CUME_DIST; }
static bool win_is_shift(int f) { return f == BDF_WIN_LAG || f == BDF_WIN_LEAD; }
static bool win_is_value(int f) { return f >= BDF_WIN_FIRST_VALUE && f <= BDF_WIN_NTH_VALUE; }
static bool win_bounded(int fr) { return fr == BDF_FRAME_ROWS_BETWEEN || fr == BDF_FRAME_RANGE_BETWEEN; }

// The bounded frame of a call as the kernels resolve it: an equivalent specification becomes the existing frame (same bits), and a
// value function's existing frame becomes bounds (ROWS and PARTITION as row offsets, RANGE as partition start .. last peer).
static bdf_window_call win_normalise(bdf_window_call k, bool float_key) {
    if (k.frame == BDF_FRAME_ROWS_BETWEEN && k.start == INT64_MIN && (k.end == 0 || k.end == INT64_MAX))
        k.frame = k.end == 0 ? BDF_FRAME_ROWS : BDF_FRAME_PARTITION;
    if (k.frame == BDF_FRAME_RANGE_BETWEEN) {
        const bool s_unb = float_key ? k.start_f == -INFINITY : k.start == INT64_MIN;
        const bool e_zero = float_key ? k.end_f == 0.0 : k.end == 0, e_unb = float_key ? k.end_f == INFINITY : k.end == INT64_MAX;
        if (s_unb && (e_zero || e_unb)) k.frame = e_zero ? BDF_FRAME_RANGE : BDF_FRAME_PARTITION;
    }
    return k;
}

static WinFrameDesc win_frame_desc(const bdf_window_call& k) {
    WinFrameDesc f{};
    f.kind = WIN_FR_ROWS;
    f.start = k.start;
    f.end = k.end;
    f.start_f = k.start_f;
    f.end_f = k.end_f;
    if (k.frame == BDF_FRAME_ROWS) { f.start = INT64_MIN; f.end = 0; }
    else if (k.frame == BDF_FRAME_PARTITION) { f.start = INT64_MIN; f.end = INT64_MAX; }
    else if (k.frame == BDF_FRAME_RANGE) f.kind = WIN_FR_PEERS;
    else if (k.frame == BDF_FRAME_RANGE_BETWEEN) f.kind = WIN_FR_RANGE;
    return f;
}

// The checks of a bounded frame's offsets (the key type decides which pair is read for RANGE).
static int win_check_bounds(const bdf_window_call& k, bool float_key) {
    if (k.frame == BDF_FRAME_RANGE_BETWEEN && float_key) {
        if (k.start_f != k.start_f || k.end_f != k.end_f) return fail(BDF_INVALID, "a RANGE offset is NaN");
        if (k.start_f > k.end_f) return fail(BDF_INVALID, "the frame starts after it ends");
        if (k.start_f == INFINITY || k.end_f == -INFINITY) return fail(BDF_INVALID, "a frame cannot start at UNBOUNDED FOLLOWING or end at UNBOUNDED PRECEDING");
        return BDF_OK;
    }
    if (k.start > k.end) return fail(BDF_INVALID, "the frame starts after it ends");
    if (k.start == INT64_MAX || k.end == INT64_MIN) return fail(BDF_INVALID, "a frame cannot start at UNBOUNDED FOLLOWING or end at UNBOUNDED PRECEDING");
    return BDF_OK;
}

static int win_out_dtype(const bdf_window_call& k) {
    switch (k.function) {
        case BDF_WIN_ROW_NUMBER: case BDF_WIN_RANK: case BDF_WIN_DENSE_RANK: return BDF_U32;
        case BDF_WIN_PERCENT_RANK: case BDF_WIN_CUME_DIST: case BDF_WIN_AVG: return BDF_F64;
        case BDF_WIN_COUNT: return BDF_I64;
        default: return k.column->dtype;
    }
}

// The prefix / suffix hierarchy of the last column a bounded aggregate read: the aggregates of one column share it.
struct WinHierarchy {
    std::unique_ptr<Scratch<void>> bytes;
    const bdf_col* of = nullptr;
};

// One bounded-frame aggregate or value function, in sorted order, into *out (one chunk).  src / table: x in sorted order; key: the
// single order key (RANGE BETWEEN), which source() brings into sorted order (null source: nothing is sorted).
static int window_frame_call(bdf_ctx* c, const bdf_window_call& k, const void* const* p, int64_t n_p, const void* const* q, int64_t n_q,
                             const bdf_col* src, void* table, int n_chunks, bool nullable, bdf_sort_key key,
                             const std::function<int(const bdf_col*, const bdf_col**)>* source, int64_t n, WinHierarchy* hier, bdf_col** out) {
    WinFrameDesc f = win_frame_desc(k);
    if (f.kind == WIN_FR_RANGE) {
        const bdf_col* ks = key.column;
        if (source) TRY((*source)(key.column, &ks));
        bool key_nullable = false;
        TRY(sort_table(c, ks, (void**)&f.key, &f.key_chunks, &key_nullable));
        f.key_dtype = key.column->dtype;
        f.key_desc = key.descending ? 1 : 0;
    }
    const int dt = k.column->dtype, w = dtype_width(dt);
    const int64_t run_bytes = (p ? 16 : 0) + (q ? 16 : 0) + (f.kind == WIN_FR_RANGE ? 2 * dtype_width(f.key_dtype) : 0);
    ColOwner tmp(c);
    cudaError_t e = cudaSuccess;
    if (win_is_value(k.function)) {
        TRY(col_alloc(c, dt, {ChunkPlan{n, true}}, nullptr, 0, tmp.out()));
        const int64_t words = (n + 31) / 32;
        Scratch<uint32_t> vwords;
        Scratch<unsigned long long> vprefix, block_sums;
        const bool ranks = k.ignore_nulls && nullable;   // IGNORE NULLS over a column with nulls: the popcount prefix of its validity
        if (ranks) {
            e = vwords.alloc(c, (size_t)words * sizeof(uint32_t));
            if (e == cudaSuccess) e = vprefix.alloc(c, (size_t)(words + 1) * sizeof(unsigned long long));
            if (e == cudaSuccess) e = block_sums.alloc(c, (size_t)scan_tile_sums(words) * sizeof(unsigned long long));
            if (e == cudaSuccess) {
                LaunchTimer t(c, BDF_K_WINDOW, BDF_U32, n, bitmap_bytes(n) * 2 + words * (8 + 16));   // validity words, popcounts, scan
                c->launches += kScanPopcountLaunches;                                                  // the timer counts the first
                e = launch_window_valid_words(table, n_chunks, n, vwords, c->s_compute);
                if (e == cudaSuccess) e = launch_scan_popcount(vwords, words, vprefix, block_sums, c->s_compute);
            }
        }
        if (e == cudaSuccess) {
            LaunchTimer t(c, BDF_K_WINDOW, dt, n, n * (2 * w + run_bytes) + (nullable ? bitmap_bytes(n) : 0) + bitmap_bytes(n) + (ranks ? words * 12 : 0));
            const int which = k.function - BDF_WIN_FIRST_VALUE;   // 0 first, 1 last, 2 nth
            e = launch_window_frame_value(dt, which, k.offset, p, n_p, q, n_q, f, table, n_chunks, n, ranks ? vwords.get() : nullptr,
                                          ranks ? vprefix.get() : nullptr, tmp->chunks[0].values, tmp->chunks[0].validity, c->s_compute);
        }
    } else {
        const int fn = k.function - BDF_WIN_SUM;   // SUM, COUNT, MIN, MAX, AVG: the order of k_window.cu's scans
        const int od = win_out_dtype(k);
        const bool out_nullable = k.function == BDF_WIN_MIN || k.function == BDF_WIN_MAX || k.function == BDF_WIN_AVG;
        TRY(col_alloc(c, od, {ChunkPlan{n, out_nullable}}, nullptr, 0, tmp.out()));
        const int levels = window_frame_levels(n);
        if (hier->of != src) {
            hier->of = nullptr;
            hier->bytes.reset(new Scratch<void>());
            e = hier->bytes->alloc(c, window_frame_scratch_bytes(dt, n));
            if (e == cudaSuccess && levels > 0) {
                const int64_t rec = dtype_is_float(dt) ? 32 : 40;   // sizeof(WinAcc<T>)
                LaunchTimer t(c, BDF_K_WINDOW, dt, n, n * w + (nullable ? bitmap_bytes(n) : 0) + (int64_t)((double)n * 2.07 * rec));
                c->launches += levels - 1;
                e = launch_window_frame_build(dt, table, n_chunks, n, hier->bytes->get(), c->s_compute);
            }
            if (e == cudaSuccess) hier->of = src;
        }
        if (e == cudaSuccess) {
            const int64_t rec = dtype_is_float(dt) ? 32 : 40;
            LaunchTimer t(c, BDF_K_WINDOW, od, n, n * (dtype_width(od) + run_bytes + 2 * (levels + 1) * rec) + (out_nullable ? bitmap_bytes(n) : 0));
            e = launch_window_frame_agg(dt, fn, p, n_p, q, n_q, f, table, n_chunks, n, hier->bytes->get(), tmp->chunks[0].values,
                                        out_nullable ? tmp->chunks[0].validity : nullptr, c->s_compute);
        }
    }
    if (e != cudaSuccess) return fail_cuda(e, "window frame");
    *out = tmp.release();
    return BDF_OK;
}

static int window_dev(bdf_ctx* c, int n_part, const bdf_col* const* part, int n_order, const bdf_sort_key* order, int n_calls,
                      const bdf_window_call* calls, bdf_col** out) {
    if (n_part < 0 || n_part > 16 || n_order < 0 || n_order > 16) return fail(BDF_INVALID, "0..16 partition and 0..16 order columns");
    if (n_calls < 0 || n_calls > 64) return fail(BDF_INVALID, "0..64 window calls");
    if ((n_part && !part) || (n_order && !order) || (n_calls && (!calls || !out))) return fail(BDF_INVALID, "null argument");
    std::vector<const bdf_col*> cols;   // every column of the call, for the type and length checks
    for (int k = 0; k < n_part; k++) cols.push_back(part[k]);
    for (int k = 0; k < n_order; k++) cols.push_back(order[k].column);
    for (const bdf_col* x : cols)
        if (!x) return fail(BDF_INVALID, "null partition or order column");
    for (int j = 0; j < n_calls; j++) {
        const bdf_window_call& k = calls[j];
        if (k.function < BDF_WIN_ROW_NUMBER || k.function > BDF_WIN_NTH_VALUE) return fail(BDF_UNSUPPORTED, "unknown window function %d", k.function);
        if (win_is_rank(k.function) && k.column) return fail(BDF_INVALID, "a ranking function takes no column");
        if (!win_is_rank(k.function) && !k.column) return fail(BDF_INVALID, "lag, lead and the aggregates need a column");
        if (win_is_shift(k.function) && k.offset < 0) return fail(BDF_INVALID, "lag / lead offset must be >= 0");
        if (!win_is_rank(k.function) && !win_is_shift(k.function) && (k.frame < BDF_FRAME_ROWS || k.frame > BDF_FRAME_RANGE_BETWEEN))
            return fail(BDF_UNSUPPORTED, "unknown window frame %d", k.frame);
        if (k.ignore_nulls && !win_is_value(k.function)) return fail(BDF_INVALID, "IGNORE NULLS is for first_value, last_value and nth_value");
        if (k.function == BDF_WIN_NTH_VALUE && k.offset < 1) return fail(BDF_INVALID, "nth_value needs n >= 1");
        if (k.frame == BDF_FRAME_RANGE_BETWEEN && !win_is_rank(k.function) && !win_is_shift(k.function) && n_order != 1)
            return fail(BDF_INVALID, "RANGE BETWEEN needs exactly one order column");
        if (k.column) cols.push_back(k.column);
    }
    for (const bdf_col* x : cols)
        if (x->dtype < 0 || x->dtype >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "window columns must be numeric");
    for (int j = 0; j < n_calls; j++)
        if (calls[j].function == BDF_WIN_AVG && (calls[j].column->dtype == BDF_I64 || calls[j].column->dtype == BDF_U64))
            return fail(BDF_UNSUPPORTED, "avg needs f64: From<T::Native>");
    const bool float_key = n_order == 1 && (order[0].column->dtype == BDF_F32 || order[0].column->dtype == BDF_F64);
    std::vector<bdf_window_call> norm(calls, calls + n_calls);   // the calls with their frames resolved (win_normalise)
    for (auto& k : norm) {
        if (win_is_rank(k.function) || win_is_shift(k.function)) continue;
        if (win_bounded(k.frame)) TRY(win_check_bounds(k, float_key));
        k = win_normalise(k, float_key);
    }
    calls = norm.data();
    if (cols.empty()) {
        if (n_calls == 0) return BDF_OK;
        return fail(BDF_INVALID, "a window without partition, order or value columns has no rows to number");
    }
    for (const bdf_col* x : cols)
        if (x->total_len != cols[0]->total_len) return fail(BDF_LENGTH_MISMATCH, "window columns have different lengths");
    const int64_t n = cols[0]->total_len;
    if (n > 0xffffffffLL) return fail(BDF_UNSUPPORTED, "sort indices are UInt32: at most 2^32-1 rows");
    if (n_calls == 0) return BDF_OK;

    std::vector<ColOwner> res;
    for (int j = 0; j < n_calls; j++) res.emplace_back(c);
    cudaError_t e = cudaSuccess;
    if (n == 0) {
        for (int j = 0; j < n_calls; j++) {
            TRY(col_alloc(c, win_out_dtype(calls[j]), {ChunkPlan{0, false}}, nullptr, 0, res[j].out()));
            e = finish_single_group(c, res[j].get());
            if (e != cudaSuccess) return fail_cuda(e, "window");
        }
        for (int j = 0; j < n_calls; j++) out[j] = res[j].release();
        return BDF_OK;
    }

    // what the calls need: peer bounds, and the gather index of each frame
    const bool sorted = n_part + n_order > 0;
    bool need_q = false, need_inv = false, need_range = false, need_part = false;
    for (int j = 0; j < n_calls; j++) {
        const int f = calls[j].function;
        if (f == BDF_WIN_RANK || f == BDF_WIN_DENSE_RANK || f == BDF_WIN_PERCENT_RANK || f == BDF_WIN_CUME_DIST) need_q = true;
        else if (win_is_shift(f)) need_inv = need_inv || sorted;
        else if (win_is_value(f) || win_bounded(calls[j].frame)) {   // bounded frames: computed in sorted order, one take back
            need_inv = need_inv || sorted;
            if (calls[j].frame == BDF_FRAME_RANGE) need_q = true;
        } else if (!win_is_rank(f)) {
            const int fr = calls[j].frame;
            if (fr == BDF_FRAME_ROWS) need_inv = need_inv || sorted;
            else if (fr == BDF_FRAME_RANGE && sorted) { need_q = true; need_range = true; }
            else need_part = true;   // PARTITION, and RANGE without keys: every row is a peer
        }
    }
    const bool has_p = n_part > 0, has_q = need_q && n_order > 0;

    ColOwner perm(c), iota(c);
    WinHeadsHost P(c), Q(c);
    if (sorted) {
        std::vector<bdf_sort_key> sk;
        for (int k = 0; k < n_part; k++) sk.push_back(bdf_sort_key{part[k], 0});
        for (int k = 0; k < n_order; k++) sk.push_back(order[k]);
        TRY(sort_indices_dev(c, (int)sk.size(), sk.data(), perm.out()));
        TRY(col_alloc(c, BDF_U32, {ChunkPlan{n, false}}, nullptr, 0, iota.out()));
        c->launches++;
        e = launch_iota((uint32_t*)iota->chunks[0].values, n, c->sm_count, c->s_compute);
        if (e == cudaSuccess) e = finish_single_group(c, iota.get());
        if (e != cudaSuccess) return fail_cuda(e, "window iota");
        // the two bitmaps take two launches: 16 + 16 keys exceed what one k_group_heads compares
        auto heads_of = [&](int k0, int k1, bdf_col** h) -> int {
            std::vector<ColOwner> keys;
            std::vector<const bdf_col*> sorted_keys;
            for (int k = k0; k < k1; k++) {
                keys.emplace_back(c);
                TRY(take_dev(c, sk[k].column, perm.get(), keys.back().out()));
                sorted_keys.push_back(keys.back().get());
            }
            return group_heads(c, sorted_keys, false, n, h, BDF_K_WINDOW);
        };
        if (has_p) {
            TRY(heads_of(0, n_part, P.bits.out()));
            TRY(window_runs(c, iota.get(), n, &P));
        }
        if (has_q) {
            ColOwner oh(c);
            TRY(heads_of(n_part, n_part + n_order, oh.out()));
            if (has_p) TRY(boolean_dev(c, BDF_OR, P.bits.get(), oh.get(), Q.bits.out()));
            else Q.bits = std::move(oh);
            TRY(window_runs(c, iota.get(), n, &Q));
        }
    }
    const void* const* p_arrays = has_p ? P.arrays : nullptr;
    const uint32_t* perm_d = sorted ? (const uint32_t*)perm->chunks[0].values : nullptr;

    // ranking functions (the first call of each; a repeated call gets a copy) and the gather indices, in one pass
    int first_of[5] = {-1, -1, -1, -1, -1};
    void* rank_outs[8] = {};
    ColOwner inv(c), range_end(c), part_end(c);
    int64_t u32_outs = 0, f64_outs = 0;
    for (int j = 0; j < n_calls; j++) {
        const int f = calls[j].function;
        if (!win_is_rank(f) || first_of[f] >= 0) continue;
        first_of[f] = j;
        TRY(col_alloc(c, win_out_dtype(calls[j]), {ChunkPlan{n, false}}, nullptr, 0, res[j].out()));
        rank_outs[f] = res[j]->chunks[0].values;
        (win_out_dtype(calls[j]) == BDF_F64 ? f64_outs : u32_outs)++;
    }
    ColOwner* const index_cols[3] = {&inv, &range_end, &part_end};
    const bool need_index[3] = {need_inv, need_range, need_part};
    for (int k = 0; k < 3; k++)
        if (need_index[k]) {
            TRY(col_alloc(c, BDF_U32, {ChunkPlan{n, false}}, nullptr, 0, index_cols[k]->out()));
            rank_outs[5 + k] = (*index_cols[k])->chunks[0].values;
            u32_outs++;
        }
    if (u32_outs + f64_outs) {
        LaunchTimer t(c, BDF_K_WINDOW, BDF_U32, n, n * ((sorted ? 4 : 0) + (has_p ? 8 : 0) + (has_q ? 16 : 0) + 4 * u32_outs + 8 * f64_outs));
        e = launch_window_rank(p_arrays, P.n_runs, has_q ? Q.arrays : nullptr, Q.n_runs, n, perm_d, rank_outs, c->s_compute);
    }
    for (int j = 0; j < n_calls && e == cudaSuccess; j++)
        if (res[j].get()) e = finish_single_group(c, res[j].get());
    for (int k = 0; k < 3 && e == cudaSuccess; k++)
        if (index_cols[k]->get()) e = finish_single_group(c, index_cols[k]->get());
    if (e != cudaSuccess) return fail_cuda(e, "window ranks");
    for (int j = 0; j < n_calls; j++)
        if (win_is_rank(calls[j].function) && first_of[calls[j].function] != j) TRY(group_clone(c, res[first_of[calls[j].function]].get(), res[j].out()));

    // lag / lead and the scans read x in sorted order: one gather per distinct column
    std::vector<std::pair<const bdf_col*, ColOwner>> gathered;
    auto source = [&](const bdf_col* x, const bdf_col** src) -> int {
        if (!sorted) { *src = x; return BDF_OK; }
        for (auto& g : gathered)
            if (g.first == x) { *src = g.second.get(); return BDF_OK; }
        gathered.emplace_back(x, ColOwner(c));
        TRY(take_dev(c, x, perm.get(), gathered.back().second.out()));
        *src = gathered.back().second.get();
        return BDF_OK;
    };
    const std::function<int(const bdf_col*, const bdf_col**)> source_fn = source;
    WinHierarchy hier;
    for (int j = 0; j < n_calls; j++) {
        const bdf_window_call& k = calls[j];
        if (win_is_rank(k.function)) continue;
        const bdf_col* src = nullptr;
        TRY(source(k.column, &src));
        void* table = nullptr;
        int n_chunks = 0;
        bool nullable = false;
        TRY(sort_table(c, src, &table, &n_chunks, &nullable));
        const int dt = k.column->dtype, w = dtype_width(dt);
        ColOwner tmp(c);
        const bdf_col* idx = nullptr;   // sorted order back to row order; null: tmp already is in row order
        if (win_is_value(k.function) || win_bounded(k.frame)) {
            TRY(window_frame_call(c, k, has_p ? P.arrays : nullptr, P.n_runs, has_q ? Q.arrays : nullptr, Q.n_runs, src, table, n_chunks, nullable,
                                  n_order == 1 && sorted ? order[0] : bdf_sort_key{nullptr, 0}, sorted ? &source_fn : nullptr, n, &hier, tmp.out()));
            idx = sorted ? inv.get() : nullptr;
        } else if (win_is_shift(k.function)) {
            TRY(col_alloc(c, dt, {ChunkPlan{n, true}}, nullptr, 0, tmp.out()));
            LaunchTimer t(c, BDF_K_WINDOW, dt, n, n * (2 * w + (has_p ? 8 : 0)) + (nullable ? bitmap_bytes(n) : 0) + bitmap_bytes(n));
            e = launch_window_shift(dt, p_arrays, P.n_runs, n, table, n_chunks, k.offset, k.function == BDF_WIN_LEAD ? 1 : 0, k.default_bits,
                                    k.has_default ? 1 : 0, tmp->chunks[0].values, tmp->chunks[0].validity, c->s_compute);
            idx = inv.get();
        } else {
            const int fn = k.function - BDF_WIN_SUM;   // SUM, COUNT, MIN, MAX, AVG: the order of k_window.cu's scans
            const int od = win_out_dtype(k);
            const bool out_nullable = k.function == BDF_WIN_MIN || k.function == BDF_WIN_MAX || k.function == BDF_WIN_AVG;
            TRY(col_alloc(c, od, {ChunkPlan{n, out_nullable}}, nullptr, 0, tmp.out()));
            Scratch<void> scratch;
            e = scratch.alloc(c, window_scan_scratch_bytes(n));
            if (e == cudaSuccess) {
                LaunchTimer t(c, BDF_K_WINDOW, od, n, n * (w + dtype_width(od)) + (nullable ? bitmap_bytes(n) : 0) + (has_p ? bitmap_bytes(n) : 0) +
                                                       (out_nullable ? bitmap_bytes(n) : 0));
                c->launches += 2;   // tile reduce, carry scan, tile rescan
                e = launch_window_scan(dt, fn, table, n_chunks, has_p ? (const uint32_t*)P.arrays[0] : nullptr, n, scratch, tmp->chunks[0].values,
                                       out_nullable ? tmp->chunks[0].validity : nullptr, c->s_compute);
            }
            idx = k.frame == BDF_FRAME_ROWS ? inv.get() : (k.frame == BDF_FRAME_RANGE && sorted) ? range_end.get() : part_end.get();
        }
        if (e == cudaSuccess) e = finish_single_group(c, tmp.get());
        if (e != cudaSuccess) return fail_cuda(e, "window");
        if (tmp->chunks[0].validity) tmp->null_counts[0] = -1;   // learnt on demand (ensure_null_counts)
        if (idx) TRY(take_dev(c, tmp.get(), idx, res[j].out()));
        else res[j] = std::move(tmp);
    }
    for (int j = 0; j < n_calls; j++) out[j] = res[j].release();
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// CSV reader (k_csv.cu; the rules are in include/b200df.h): the file is mapped and its bytes go to HBM through the pageable staging
// path; the tokenizer scan builds the field index there, the field counts are checked and the schema inferred on the device.  The
// bytes and the index stay until bdf_csv_close; a read parses only the requested columns.

// A text file as the readers hold it: mapped, and its bytes after a leading UTF-8 BOM in HBM (zero-padded to whole tiles).
struct MappedText {
    int fd = -1;
    const uint8_t* map = nullptr;   // the whole file
    size_t size = 0;
    size_t off = 0;                 // 3 when the file starts with a UTF-8 BOM
    int64_t n = 0;                  // bytes after the BOM (what the device holds)
    uint8_t* d_text = nullptr;
    double upload_ms = 0;           // host time of the upload
};

static void text_free(bdf_ctx* c, MappedText* t) {
    if (t->d_text) cudaFreeAsync(t->d_text, c->s_compute);
    if (t->map) munmap((void*)t->map, t->size);
    if (t->fd >= 0) close(t->fd);
}

// Map `path`, step over a BOM, and upload the rest through the pageable staging path: page cache -> pinned staging -> HBM.  The
// device buffer is padded with zeros to whole tiles of `tile` bytes.  `what` names the reader in the messages.
static int text_open(bdf_ctx* c, const char* path, int64_t tile, const char* what, MappedText* f) {
    f->fd = open(path, O_RDONLY | O_CLOEXEC);
    struct stat sb;
    if (f->fd < 0 || fstat(f->fd, &sb) != 0) return fail(BDF_INVALID, "cannot open %s: %s", path, strerror(errno));
    f->size = (size_t)sb.st_size;
    if (f->size) {
        void* m = mmap(nullptr, f->size, PROT_READ, MAP_PRIVATE, f->fd, 0);
        if (m == MAP_FAILED) return fail(BDF_INVALID, "cannot map %s: %s", path, strerror(errno));
        f->map = (const uint8_t*)m;
    }
    if (f->size >= 3 && f->map[0] == 0xEF && f->map[1] == 0xBB && f->map[2] == 0xBF) f->off = 3;
    f->n = (int64_t)(f->size - f->off);
    const int64_t tiles = std::max<int64_t>((f->n + tile - 1) / tile, 1);
    if ((long double)tiles * tile * 1.3L > (long double)c->hbm_bytes) return fail(BDF_OOM, "a %s file of %lld bytes does not fit in device memory", what, (long long)f->n);
    cudaError_t e = cudaMallocAsync((void**)&f->d_text, (size_t)(tiles * tile), c->s_compute);
    if (e == cudaSuccess) e = cudaMemsetAsync(f->d_text + f->n, 0, (size_t)(tiles * tile - f->n), c->s_compute);
    if (e == cudaSuccess) e = cudaEventRecord(c->ev_tmp, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(c->s_h2d, c->ev_tmp, 0);
    const auto t0 = std::chrono::steady_clock::now();
    if (e == cudaSuccess && f->n) e = h2d_copy(c, f->d_text, f->map + f->off, (size_t)f->n);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_h2d);
    f->upload_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (e != cudaSuccess) {
        const int st = fail_cuda(e, (std::string(what) + " upload").c_str());
        cudaStreamSynchronize(c->s_h2d);   // no copy may still read the mapping when it is unmapped
        return st;
    }
    return BDF_OK;
}

struct bdf_csv : MappedText {
    unsigned long long* d_ends = nullptr;   // per field: end byte | bit 63 when it ends its record
    int64_t n_fields = 0, k = 0, n_rows = 0, f0 = 0, batch = 1024;
    int has_header = 1;
    uint8_t delim = ',';
    std::vector<std::string> names;
    std::vector<int32_t> dtypes, nullable;
    mutable int64_t exact_fields = 0;
};

static constexpr unsigned long long kCsvRec = 1ull << 63;

static void csv_free(bdf_ctx* c, bdf_csv* f) {
    if (!f) return;
    if (f->d_ends) cudaFreeAsync(f->d_ends, c->s_compute);
    text_free(c, f);
    delete f;
}
static void drop(bdf_ctx* c, bdf_csv* f) { csv_free(c, f); }

// The unquoted value of raw field bytes [s, e) of the mapping (the rules of csv_parse.cuh's Unquote).
static std::string csv_unquote(const uint8_t* s, const uint8_t* e) {
    std::string out;
    int st = 0;
    if (s < e && *s == '"') { st = 1; s++; }
    for (; s < e; s++) {
        const uint8_t b = *s;
        if (st == 0) out += (char)b;
        else if (st == 1) { if (b == '"') st = 2; else out += (char)b; }
        else if (b == '"') { st = 1; out += '"'; }
        else { st = 0; out += (char)b; }
    }
    return out;
}

// Raw span of field f from two entries of the index (prev: the entry of f - 1, or none for f == 0).
static void csv_span(const bdf_csv* f, bool has_prev, unsigned long long prev, unsigned long long cur, int64_t* s, int64_t* e) {
    const unsigned long long mask = kCsvRec - 1;
    *e = (int64_t)(cur & mask);
    int64_t a = has_prev ? (int64_t)(prev & mask) + 1 : 0;
    if (!has_prev || (prev & kCsvRec))
        while (a < *e && (f->map[f->off + a] == '\r' || f->map[f->off + a] == '\n')) a++;
    *s = a;
}

static int csv_fetch(bdf_ctx* c, const bdf_csv* f, int64_t first, int64_t count, std::vector<unsigned long long>& out) {
    out.resize((size_t)std::max<int64_t>(count, 1));
    if (count > 0) {
        CK(cudaMemcpyAsync(out.data(), f->d_ends + first, (size_t)count * sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->s_compute));
        CK(cudaStreamSynchronize(c->s_compute));
    }
    return BDF_OK;
}

// The field at index `bad` disagrees with the first record's field count: the csv crate's UnequalLengths text.
static int csv_unequal(bdf_ctx* c, bdf_csv* f, int64_t bad) {
    const int64_t r = bad / f->k, first = r * f->k;
    std::vector<unsigned long long> v;
    TRY(csv_fetch(c, f, first, bad - first + 1, v));
    int64_t n_found = bad - first + 1;
    if (!(v[(size_t)(bad - first)] & kCsvRec)) {   // more fields than the first record: find this record's end
        for (int64_t i = bad + 1; i < f->n_fields; i += 65536) {
            std::vector<unsigned long long> w;
            const int64_t cnt = std::min<int64_t>(65536, f->n_fields - i);
            TRY(csv_fetch(c, f, i, cnt, w));
            int64_t j = 0;
            while (j < cnt && !(w[(size_t)j] & kCsvRec)) j++;
            if (j < cnt) { n_found = i + j - first + 1; break; }
        }
    }
    unsigned long long prev = 0;
    std::vector<unsigned long long> p;
    if (first > 0) { TRY(csv_fetch(c, f, first - 1, 1, p)); prev = p[0]; }
    int64_t s, e;
    csv_span(f, first > 0, prev, v[0], &s, &e);
    const int64_t byte = (int64_t)f->off + s;
    int64_t line = 1;
    for (int64_t i = 0; i < byte; i++) line += f->map[i] == '\n';
    return fail(BDF_INVALID, "CSV error: record %lld (line: %lld, byte: %lld): found record with %lld fields, but the previous record has %lld fields",
                (long long)r, (long long)line, (long long)byte, (long long)n_found, (long long)f->k);
}

static int csv_open(bdf_ctx* c, const char* path, const bdf_csv_options* o, int n_schema, const int32_t* schema, bdf_csv** out) {
    if (!path || !o || !out) return fail(BDF_INVALID, "null argument");
    if (o->batch_size < 1) return fail(BDF_INVALID, "batch_size must be at least 1");
    if (o->delimiter == '"' || o->delimiter == '\r' || o->delimiter == '\n') return fail(BDF_INVALID, "the delimiter cannot be a quote or a line terminator");
    if (schema) {
        if (n_schema < 1) return fail(BDF_INVALID, "an explicit schema needs at least one column");
        for (int i = 0; i < n_schema; i++)
            if (!((schema[i] >= 0 && schema[i] <= kBool) || schema[i] == BDF_UTF8 || schema[i] == -1))
                return fail(BDF_UNSUPPORTED, "schema column %d: type %d is not read from CSV (numeric, Boolean or Utf8)", i, schema[i]);
    }
    Owned<bdf_csv> f(c, new (std::nothrow) bdf_csv());
    if (!f.get()) return fail(BDF_OOM, "host allocation failed");
    f->has_header = o->has_header ? 1 : 0;
    f->delim = o->delimiter;
    f->batch = o->batch_size;
    const int64_t tile = csv_tile_bytes();
    TRY(text_open(c, path, tile, "CSV", f.get()));
    const int64_t tiles = std::max<int64_t>((f->n + tile - 1) / tile, 1);

    Scratch<uint32_t> agg;
    Scratch<uint8_t> start;
    Scratch<uint16_t> fe, re;
    Scratch<unsigned long long> counts, small;   // small: [0] final state, [1] first record end, [2] first bad field
    Scratch<unsigned int> bits;

    // tokenize: the state at every CTA, the field / record end masks, the field count
    cudaError_t e = agg.alloc(c, (size_t)tiles * 4);
    if (e == cudaSuccess) e = start.alloc(c, (size_t)tiles);
    if (e == cudaSuccess) e = fe.alloc(c, (size_t)tiles * kThreads * 2);
    if (e == cudaSuccess) e = re.alloc(c, (size_t)tiles * kThreads * 2);
    if (e == cudaSuccess) e = counts.alloc(c, (size_t)(tiles + 1) * 8);
    if (e == cudaSuccess) e = small.alloc(c, 4 * 8);
    if (e == cudaSuccess) e = cudaMemsetAsync(small, 0xff, 4 * 8, c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "CSV tokenizer scratch allocation");
    {
        LaunchTimer t(c, BDF_K_CSV, kBool, f->n, f->n * 2 + tiles * kThreads * 4);
        c->launches += 3;   // reduce, CTA-state scan, mark, count scan
        e = launch_csv_tokenize(f->d_text, f->n, f->delim, agg, start, (int*)small.get(), fe, re, counts, c->s_compute);
    }
    unsigned long long host_small[4] = {0, 0, 0, 0}, total = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&total, counts + tiles, 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaMemcpyAsync(host_small, small, 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "CSV tokenizer");
    const int final_state = (int)(host_small[0] & 0xffffffffu);
    const bool eof_field = final_state != 0;   // the last record has no terminator: end of file ends it
    f->n_fields = (int64_t)total + (eof_field ? 1 : 0);
    if (f->n_fields == 0) return fail(BDF_WOULD_PANIC, "the CSV file has no records: the reference panics at batches[0]");

    // the field index
    e = cudaMallocAsync((void**)&f->d_ends, (size_t)f->n_fields * 8, c->s_compute);
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_CSV, BDF_U64, f->n, tiles * kThreads * 4 + (int64_t)total * 8);
        e = launch_csv_index(fe, re, f->n, counts, f->d_ends, small + 1, c->s_compute);
    }
    unsigned long long eof_entry = (unsigned long long)f->n | kCsvRec;
    if (e == cudaSuccess && eof_field) e = cudaMemcpyAsync(f->d_ends + total, &eof_entry, 8, cudaMemcpyHostToDevice, c->s_compute);
    if (e == cudaSuccess) e = cudaMemcpyAsync(host_small, small, 4 * 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "CSV field index");
    const unsigned long long first_rec = std::min<unsigned long long>(host_small[1], eof_field ? total : ~0ull);
    f->k = (int64_t)first_rec + 1;

    // every record has the first record's field count
    {
        LaunchTimer t(c, BDF_K_CSV, BDF_U64, f->n_fields, f->n_fields * 8);
        e = launch_csv_check(f->d_ends, f->n_fields, f->k, small + 2, c->sm_count, c->s_compute);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(host_small, small, 4 * 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "CSV record check");
    if (host_small[2] != ~0ull) return csv_unequal(c, f.get(), (int64_t)host_small[2]);
    const int64_t n_records = f->n_fields / f->k;
    f->f0 = f->has_header ? f->k : 0;
    f->n_rows = n_records - f->has_header;
    if (f->k > 0x7fffffffLL) return fail(BDF_UNSUPPORTED, "more than 2^31-1 columns");
    const int k = (int)f->k;

    // names
    if (f->has_header) {
        std::vector<unsigned long long> h;
        TRY(csv_fetch(c, f.get(), 0, f->k, h));
        for (int i = 0; i < k; i++) {
            int64_t s, en;
            csv_span(f.get(), i > 0, i > 0 ? h[(size_t)i - 1] : 0, h[(size_t)i], &s, &en);
            f->names.push_back(csv_unquote(f->map + f->off + s, f->map + f->off + en));
        }
    } else {
        for (int i = 0; i < k; i++) f->names.push_back("column_" + std::to_string(i + 1));
    }
    if (f->n_rows == 0) return fail(BDF_WOULD_PANIC, "the CSV file has no data records: the reference panics at batches[0]");

    // schema
    if (schema) {
        if (n_schema != k) return fail(BDF_INVALID, "the schema has %d columns, the file %d", n_schema, k);
        for (int i = 0; i < k; i++) {
            f->dtypes.push_back(schema[i] == BDF_UTF8 ? -1 : schema[i]);
            f->nullable.push_back(1);
        }
    } else {
        const int64_t rows = o->max_records < 0 ? f->n_rows : std::min<int64_t>(o->max_records, f->n_rows);
        std::vector<unsigned int> hb((size_t)k, 0u);
        e = bits.alloc(c, (size_t)k * 4);
        if (e == cudaSuccess) e = cudaMemsetAsync(bits, 0, (size_t)k * 4, c->s_compute);
        if (e == cudaSuccess) {
            LaunchTimer t(c, BDF_K_CSV, BDF_U32, rows * f->k, rows * f->k * 16);
            e = launch_csv_infer(f->d_text, f->d_ends, f->f0, f->f0 + rows * f->k, f->k, bits, c->sm_count, c->s_compute);
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(hb.data(), bits, (size_t)k * 4, cudaMemcpyDeviceToHost, c->s_compute);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
        if (e != cudaSuccess) return fail_cuda(e, "CSV schema inference");
        for (int i = 0; i < k; i++) {
            const unsigned int types = hb[(size_t)i] & ~1u;   // bit 0: an empty field (a null)
            int dt = -1;                                       // Utf8: other, a mix, or no type at all
            if (types == 2u) dt = kBool;
            else if (types == 4u) dt = BDF_I64;
            else if (types == 8u || types == 12u) dt = BDF_F64;
            f->dtypes.push_back(dt);
            f->nullable.push_back((hb[(size_t)i] & 1u) ? 1 : 0);
        }
    }
    *out = f.release();
    return BDF_OK;
}

static int csv_read(bdf_ctx* c, const bdf_csv* f, int n_cols, const int32_t* cols, bdf_col** out) {
    if (!f || !out || (n_cols > 0 && !cols)) return fail(BDF_INVALID, "null argument");
    if (n_cols < 0 || n_cols > 65535) return fail(BDF_INVALID, "0..65535 columns");
    for (int i = 0; i < n_cols; i++) {
        if (cols[i] < 0 || cols[i] >= (int)f->k) return fail(BDF_INVALID, "column %d out of range (the file has %lld)", cols[i], (long long)f->k);
        if (f->dtypes[(size_t)cols[i]] < 0)
            return fail(BDF_UNSUPPORTED, "column %d (%s) is Utf8: not on the device path", cols[i], f->names[(size_t)cols[i]].c_str());
    }
    const int64_t batch = f->batch, n_chunks = (f->n_rows + batch - 1) / batch;
    const int rows_per_tile = csv_parse_rows();
    std::vector<ChunkPlan> plan((size_t)n_chunks);
    for (int64_t i = 0; i < n_chunks; i++) plan[(size_t)i] = ChunkPlan{std::min(batch, f->n_rows - i * batch), true};
    std::vector<ColOwner> res;
    Scratch<char> descs;
    Scratch<unsigned long long> small;   // [0] first failing field key, [1] slow-path fields
    Scratch<void> slow, patches;
    const size_t dsz = csv_desc_bytes();
    std::vector<char> hdesc((size_t)std::max(n_cols, 1) * dsz, 0);
    int64_t float_fields = 0, out_bytes = 0;
    for (int i = 0; i < n_cols; i++) {
        const int dt = f->dtypes[(size_t)cols[i]];
        res.emplace_back(c);
        TRY(col_alloc(c, dt, plan, nullptr, rows_per_tile, res[(size_t)i].out()));
        bdf_col* col = res[(size_t)i].get();
        const DevChunk& c0 = col->chunks[0];
        const long long vs = n_chunks > 1 ? (long long)(col->chunks[1].values - c0.values) : 0;
        const long long bs = n_chunks > 1 ? (long long)((char*)col->chunks[1].validity - (char*)c0.validity) : 0;
        const DevChunk& cl = col->chunks[(size_t)n_chunks - 1];
        if (cl.values != c0.values + vs * (n_chunks - 1) || (char*)cl.validity != (char*)c0.validity + bs * (n_chunks - 1))
            return fail(BDF_INVALID, "internal: CSV output chunks are not evenly spaced");
        struct Desc { char* values; long long vstride; uint32_t* validity; long long bstride; uint32_t* warp_counts; int dtype; int file_col; } d{
            c0.values, vs, c0.validity, bs, col->d_warp_counts, dt, cols[i]};
        static_assert(sizeof(Desc) == 48, "CsvColDesc layout");
        memcpy(hdesc.data() + (size_t)i * dsz, &d, sizeof d);
        if (dt == BDF_F32 || dt == BDF_F64) float_fields += f->n_rows;
        out_bytes += (int64_t)value_bytes(dt, f->n_rows, 0) + bitmap_bytes(f->n_rows);
    }
    const long long slow_cap = std::max<long long>(65536, float_fields / 64);
    cudaError_t e = descs.alloc(c, hdesc.size());
    if (e == cudaSuccess) e = cudaMemcpyAsync(descs, hdesc.data(), hdesc.size(), cudaMemcpyHostToDevice, c->s_compute);
    if (e == cudaSuccess) e = small.alloc(c, 16);
    if (e == cudaSuccess) e = cudaMemsetAsync(small, 0xff, 8, c->s_compute);
    if (e == cudaSuccess) e = cudaMemsetAsync(small + 1, 0, 8, c->s_compute);
    if (e == cudaSuccess && float_fields) e = slow.alloc(c, (size_t)slow_cap * csv_slow_bytes());
    if (e != cudaSuccess) return fail_cuda(e, "CSV read scratch allocation");
    unsigned long long hs[2] = {~0ull, 0};
    {
        const int64_t fields = f->n_rows * n_cols;
        LaunchTimer t(c, BDF_K_CSV, n_cols == 1 ? f->dtypes[(size_t)cols[0]] : -1, fields,
                      f->n * n_cols / std::max<int64_t>(f->k, 1) + fields * 16 + out_bytes);
        e = launch_csv_parse(f->d_text, f->d_ends, descs, n_cols, f->f0, f->k, f->n_rows, batch, small, slow, small + 1, slow_cap, c->s_compute);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(hs, small, 16, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "CSV parse");
    if (hs[0] != ~0ull) {   // the first failing field: (batch, column in the request, row)
        const unsigned long long key = hs[0];
        const int64_t row = (int64_t)(key % (unsigned long long)batch), rest = (int64_t)(key / (unsigned long long)batch);
        const int p = (int)(rest % n_cols);
        const int64_t chunk = rest / n_cols, r = chunk * batch + row, fld = f->f0 + r * f->k + cols[p];
        std::vector<unsigned long long> v;
        TRY(csv_fetch(c, f, fld > 0 ? fld - 1 : 0, fld > 0 ? 2 : 1, v));
        int64_t s, en;
        csv_span(f, fld > 0, fld > 0 ? v[0] : 0, fld > 0 ? v[1] : v[0], &s, &en);
        g_err = "Error while parsing value " + csv_unquote(f->map + f->off + s, f->map + f->off + en) + " for column " + std::to_string(cols[p]) +
                " at line " + std::to_string(r + f->has_header);
        return BDF_PARSE;
    }
    int64_t n_slow = (int64_t)hs[1];
    if (n_slow > slow_cap)
        return fail(BDF_UNSUPPORTED, "%lld float fields need exact rounding, more than the %lld one read resolves", (long long)n_slow, slow_cap);
    if (n_slow > 0) {   // exact rounding on the host, in the C locale, written back by one scatter
        struct Slow { long long start, end; int col, pad; long long chunk, row; };
        struct Patch { unsigned long long dst, bits; int width, pad; };
        std::vector<Slow> sl((size_t)n_slow);
        e = cudaMemcpyAsync(sl.data(), slow, (size_t)n_slow * sizeof(Slow), cudaMemcpyDeviceToHost, c->s_compute);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
        if (e != cudaSuccess) return fail_cuda(e, "CSV exact rounding");
        static locale_t cloc = newlocale(LC_ALL_MASK, "C", (locale_t)0);
        std::vector<Patch> hp;
        for (size_t i = 0; i < sl.size(); i++) {
            const Slow& x = sl[i];
            const std::string v = csv_unquote(f->map + f->off + x.start, f->map + f->off + x.end);
            const bdf_col* col = res[(size_t)x.col].get();
            Patch pt{};
            if (col->dtype == BDF_F64) {
                const double d = strtod_l(v.c_str(), nullptr, cloc);
                memcpy(&pt.bits, &d, 8);
                pt.width = 8;
            } else {
                const float fl = strtof_l(v.c_str(), nullptr, cloc);
                uint32_t b;
                memcpy(&b, &fl, 4);
                pt.bits = b;
                pt.width = 4;
            }
            pt.dst = (unsigned long long)(uintptr_t)(col->chunks[(size_t)x.chunk].values + x.row * pt.width);
            hp.push_back(pt);
        }
        static_assert(sizeof(Patch) == 24, "CsvPatch layout");
        e = patches.alloc(c, hp.size() * sizeof(Patch));
        if (e == cudaSuccess) e = cudaMemcpyAsync(patches, hp.data(), hp.size() * sizeof(Patch), cudaMemcpyHostToDevice, c->s_compute);
        if (e == cudaSuccess) {
            LaunchTimer t(c, BDF_K_CSV, -1, (int64_t)hp.size(), (int64_t)hp.size() * 32);
            e = launch_csv_scatter(patches, (long long)hp.size(), c->s_compute);
        }
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);   // hp is read by the copy
        if (e != cudaSuccess) return fail_cuda(e, "CSV exact rounding");
    }
    for (int i = 0; i < n_cols; i++) {
        bdf_col* col = res[(size_t)i].get();
        col->counts_on_device = true;
        TRY(fetch_counts(c, col));
        for (size_t j = 0; j < col->chunks.size(); j++)
            if (col->null_counts[j] == 0) col->chunks[j].validity = nullptr;   // no bitmap in a chunk without nulls
        e = finish_single_group(c, col);
        if (e != cudaSuccess) return fail_cuda(e, "CSV read");
    }
    f->exact_fields = n_slow;
    for (int i = 0; i < n_cols; i++) out[i] = res[(size_t)i].release();
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// CSV writer (k_csv_write.cu; DataFrame::to_csv, src/dataframe.rs:527-543).  The rows go in blocks whose text surely fits one of two
// fixed device buffers: while block k is measured, scanned and formatted, block k-1 crosses PCIe through the pinned staging slots
// and the CopyPool threads pwrite every slot at its offset in the file (known from the scan), so neither HBM nor pinned memory
// grows with the file.

static constexpr size_t kCsvwText = (size_t)64 << 20;        // bytes of each of the two device text buffers
static constexpr int64_t kCsvwMaxRows = (int64_t)1 << 21;    // rows per block at most (their lengths and offsets: 16 MiB)
// The longest field of each dtype (BDF_I8 .. BDF_F64, BDF_BOOL).  A positional float whose last digit sits at 10^e (e < 0) is 2 - e
// bytes plus its sign, and the shortest digits never need e below the rounding interval's width (2^-1074 > 10^-324, 2^-149 > 10^-45):
// at most 327 bytes for Float64 (-0.000...0005, the negative smallest subnormal) and 48 for Float32; above 1, 310 and 40.
static const int kCsvwMaxField[11] = {4, 6, 11, 20, 3, 5, 10, 20, 48, 327, 5};

// The delimiter must not occur in any value's text, so that no value needs quotes.
static bool csvw_delim_ok(int d) {
    return !((d >= '0' && d <= '9') || strchr("-.\"\r\nNaintruefls", d) || d == 0);
}

// The header record, quoted as the csv crate's QuoteStyle::Necessary quotes.
static std::string csvw_header(int n_cols, const char* const* names, char delim) {
    std::string h;
    for (int j = 0; j < n_cols; j++) {
        if (j) h += delim;
        const char* s = names[j];
        const bool quote = (n_cols == 1 && !*s) || strpbrk(s, "\"\r\n") || strchr(s, delim);
        if (!quote) { h += s; continue; }
        h += '"';
        for (; *s; s++) { if (*s == '"') h += '"'; h += *s; }
        h += '"';
    }
    return h + '\n';
}

static int pwrite_all(int fd, const char* p, size_t n, off_t off) {   // 0 or an errno
    while (n) {
        const ssize_t w = pwrite(fd, p, n, off);
        if (w < 0) { if (errno == EINTR) continue; return errno; }
        if (w == 0) return EIO;
        p += w; n -= (size_t)w; off += w;
    }
    return 0;
}

// Text blocks from device buffers to a file, in order: each block crosses PCIe through the context's pinned staging slots (at most
// kStageSlots - 1 in flight) and the CopyPool threads pwrite every slot at its offset in the file.  The CSV and JSON writers share it.
struct FileSink {
    bdf_ctx* c;
    int fd;
    const char* path;
    off_t file_off;
    struct Pending { bdf_ctx::StageSlot* sl; off_t off; size_t n; };
    std::deque<Pending> pending;

    int retire() {
        const Pending p = pending.front();
        pending.pop_front();
        CK(cudaEventSynchronize(p.sl->ev));
        p.sl->busy = false;
        constexpr size_t kJob = (size_t)512 << 10;
        std::atomic<int> werr{0};
        c->pool->run((p.n + kJob - 1) / kJob, [&](size_t j) {
            const int we = pwrite_all(fd, p.sl->p + j * kJob, std::min(kJob, p.n - j * kJob), p.off + (off_t)(j * kJob));
            if (we) werr = we;
        });
        if (werr) return fail(BDF_INVALID, "writing %s failed: %s", path, strerror(werr));
        return BDF_OK;
    }
    // `bytes` of `text`, complete once `ready` has fired, go next in the file; `left` is recorded on the copy stream once they have
    // left `text`.
    int put(const char* text, size_t bytes, cudaEvent_t ready, cudaEvent_t left) {
        CK(cudaStreamWaitEvent(c->s_d2h, ready, 0));
        for (size_t off = 0; off < bytes; off += kStageBytes) {
            const size_t n = std::min(kStageBytes, bytes - off);
            if ((int)pending.size() >= kStageSlots - 1) TRY(retire());
            bdf_ctx::StageSlot& sl = c->stage[c->stage_next++ % kStageSlots];
            if (sl.busy) CK(cudaEventSynchronize(sl.ev));   // an upload's slot
            CK(cudaMemcpyAsync(sl.p, text + off, n, cudaMemcpyDeviceToHost, c->s_d2h));
            CK(cudaEventRecord(sl.ev, c->s_d2h));
            sl.busy = true;
            pending.push_back(Pending{&sl, file_off + (off_t)off, n});
        }
        CK(cudaEventRecord(left, c->s_d2h));
        file_off += (off_t)bytes;
        return BDF_OK;
    }
    int flush() {
        while (!pending.empty()) TRY(retire());
        return BDF_OK;
    }
};

static int csv_write(bdf_ctx* c, const char* path, int n_cols, const char* const* names, const bdf_col* const* cols, const bdf_csv_write_options* opt) {
    if (!path || !names || !cols) return fail(BDF_INVALID, "null argument");
    if (n_cols <= 0) return fail(BDF_INVALID, "no columns to write");
    const int delim = opt ? opt->delimiter : ',';
    if (!csvw_delim_ok(delim)) return fail(BDF_INVALID, "delimiter 0x%02x can occur in a formatted value", delim);
    int64_t n_chunks = -1, max_row = n_cols + 2;
    for (int j = 0; j < n_cols; j++) {
        const bdf_col* col = cols[j];
        if (!col || !names[j]) return fail(BDF_INVALID, "null column or name");
        if (!col->fparts.empty()) return fail(BDF_INVALID, "a column of a multi-GPU context was passed to a one-GPU context");
        if (!((col->dtype >= 0 && col->dtype < BDF_NTYPES) || col->dtype == kBool)) return fail(BDF_UNSUPPORTED, "column '%s': dtype %d", names[j], col->dtype);
        const int64_t nc = (int64_t)col->chunks.size();
        if (n_chunks < 0) n_chunks = nc;
        if (nc != n_chunks)
            return fail(BDF_LENGTH_MISMATCH, "columns have different numbers of chunks (%lld, %lld)", (long long)nc, (long long)n_chunks);
        for (int64_t b = 0; b < nc; b++)
            if (col->chunks[b].len != cols[0]->chunks[b].len)
                return fail(BDF_LENGTH_MISMATCH, "chunk %lld: column '%s' has %lld rows, column '%s' has %lld", (long long)b, names[j],
                            (long long)col->chunks[b].len, names[0], (long long)cols[0]->chunks[b].len);
        max_row += kCsvwMaxField[col->dtype];
    }
    std::vector<long long> starts((size_t)n_chunks + 1, 0);
    std::vector<CsvwDesc> descs((size_t)n_chunks * n_cols);
    for (int64_t b = 0; b < n_chunks; b++) {
        starts[b + 1] = starts[b] + cols[0]->chunks[b].len;
        for (int j = 0; j < n_cols; j++) {
            const DevChunk& ch = cols[j]->chunks[b];
            descs[b * n_cols + j] = CsvwDesc{ch.values, ch.validity, ch.bit_off, ch.val_bit_off, cols[j]->dtype, 0};
        }
    }
    const int64_t rows = starts[n_chunks];
    const size_t text_cap = std::max<size_t>(kCsvwText, (size_t)max_row);
    const int64_t block_rows = std::max<int64_t>(1, std::min<int64_t>(kCsvwMaxRows, (int64_t)(text_cap / (size_t)max_row)));

    const int fd = open(path, O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
    if (fd < 0) return fail(BDF_INVALID, "cannot create %s: %s", path, strerror(errno));
    struct FdGuard { int fd; ~FdGuard() { if (fd >= 0) close(fd); } } fdg{fd};
    off_t file_off = 0;
    if (!opt || opt->has_header) {
        const std::string h = csvw_header(n_cols, names, (char)delim);
        const int we = pwrite_all(fd, h.data(), h.size(), 0);
        if (we) return fail(BDF_INVALID, "writing %s failed: %s", path, strerror(we));
        file_off = (off_t)h.size();
    }
    auto finish = [&]() {
        const int fdv = fdg.fd;
        fdg.fd = -1;
        if (close(fdv) != 0) return fail(BDF_INVALID, "closing %s failed: %s", path, strerror(errno));
        return (int)BDF_OK;
    };
    if (rows == 0) return finish();

    for (int j = 0; j < n_cols; j++) wait_groups(c->s_compute, cols[j], 0, n_chunks);
    TRY(ensure_stage(c));
    Scratch<CsvwDesc> d_desc;
    Scratch<long long> d_starts;
    Scratch<char> text[2];
    Scratch<unsigned long long> lens, sums;
    cudaError_t e = d_desc.alloc(c, descs.size() * sizeof(CsvwDesc));
    if (e == cudaSuccess) e = d_starts.alloc(c, starts.size() * sizeof(long long));
    if (e == cudaSuccess) e = text[0].alloc(c, text_cap);
    if (e == cudaSuccess) e = text[1].alloc(c, text_cap);
    if (e == cudaSuccess) e = lens.alloc(c, (size_t)(block_rows + 1) * sizeof(unsigned long long));
    if (e == cudaSuccess) e = sums.alloc(c, (size_t)scan_tile_sums(block_rows) * sizeof(unsigned long long));
    // pageable sources: the copies have read them when they return
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_desc, descs.data(), descs.size() * sizeof(CsvwDesc), cudaMemcpyHostToDevice, c->s_compute);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_starts, starts.data(), starts.size() * sizeof(long long), cudaMemcpyHostToDevice, c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "CSV write setup");
    struct Pinned { unsigned long long* p = nullptr; ~Pinned() { if (p) cudaFreeHost(p); } } tot;
    struct Events { bdf_ctx* c; cudaEvent_t ev[4] = {}; ~Events() { for (auto x : ev) ev_put(c, x); } } evs{c};
    CK(cudaHostAlloc((void**)&tot.p, 2 * sizeof(unsigned long long), cudaHostAllocDefault));
    for (auto& x : evs.ev) CK(ev_get(c, &x));
    cudaEvent_t* ev_emit = evs.ev;       // block k's text is complete in text[k & 1]
    cudaEvent_t* ev_d2h = evs.ev + 2;    // block k's text has left text[k & 1]
    // Declared after the buffers, so it runs first on every exit: no copy may still read a text buffer when it is freed.
    struct DrainD2H { cudaStream_t s; ~DrainD2H() { cudaStreamSynchronize(s); } } drain_guard{c->s_d2h};

    const int64_t n_blocks = (rows + block_rows - 1) / block_rows;
    size_t emit_rec[2] = {0, 0};
    auto enqueue = [&](int64_t k) -> int {
        const int b = (int)(k & 1);
        const int64_t row0 = k * block_rows, n = std::min(block_rows, rows - row0);
        cudaError_t e2 = k >= 2 ? cudaStreamWaitEvent(c->s_compute, ev_d2h[b], 0) : cudaSuccess;
        if (e2 == cudaSuccess) {
            LaunchTimer t(c, BDF_K_CSV_WRITE, BDF_U64, n, n * (8 + 16));   // lengths written, then read and written by the scan
            c->launches += kScanSumsLaunches;                                // the timer counts the measure
            e2 = launch_csvw_measure(d_desc, d_starts, n_cols, (int)n_chunks, row0, n, lens, sums, c->s_compute);
            if (e2 == cudaSuccess) e2 = launch_scan_sums(lens, n, sums, c->s_compute);
        }
        if (e2 == cudaSuccess) e2 = cudaMemcpyAsync(tot.p + b, lens + n, sizeof(unsigned long long), cudaMemcpyDeviceToHost, c->s_compute);
        if (e2 == cudaSuccess) {
            LaunchTimer t(c, BDF_K_CSV_WRITE, BDF_U8, n, n * 8);   // + the text, once the block's size is known
            e2 = launch_csvw_emit(d_desc, d_starts, n_cols, (int)n_chunks, row0, n, delim, lens, text[b], c->s_compute);
        }
        if (c->profiling) emit_rec[b] = c->prof.size() - 1;
        if (e2 == cudaSuccess) e2 = cudaEventRecord(ev_emit[b], c->s_compute);
        return e2 == cudaSuccess ? BDF_OK : fail_cuda(e2, "CSV write kernels");
    };
    FileSink sink{c, fd, path, file_off, {}};
    auto drain = [&](int64_t k) -> int {
        const int b = (int)(k & 1);
        CK(cudaEventSynchronize(ev_emit[b]));
        const size_t bytes = (size_t)tot.p[b];
        if (c->profiling) c->prof[emit_rec[b]].rec.bytes += (int64_t)bytes;
        return sink.put(text[b], bytes, ev_emit[b], ev_d2h[b]);
    };
    TRY(enqueue(0));
    for (int64_t k = 0; k < n_blocks; k++) {
        if (k + 1 < n_blocks) TRY(enqueue(k + 1));
        TRY(drain(k));
    }
    TRY(sink.flush());
    return finish();
}

// ---------------------------------------------------------------------------------------------------
// Parquet writer (k_parquet_write.cu; DataFrame::to_parquet, src/dataframe.rs:545-560; the rules are in include/b200df.h).  The
// dictionary of every column is found first (sorted_runs over (row group, value bits): a fixed number of launches per column).  Then
// the pages go in blocks of consecutive pages in file order, as the CSV writer's text does: while block k is encoded (and
// compressed) into one of two fixed device buffers, block k-1's page results come back in one small copy, the host serialises its
// page headers, and the headers and bodies cross to the file through the pinned staging slots, pwrite by the CopyPool threads.

static constexpr int64_t kPqwPageRows = (int64_t)1 << 17;
static constexpr size_t kPqwRaw = (size_t)64 << 20;     // bytes of each of the two page-body buffers
static constexpr size_t kPqwFrag = (size_t)80 << 20;    // bytes of the snappy fragment buffer
static constexpr int64_t kPqwDictLimit = (int64_t)1 << 20;
static constexpr int64_t kPqwMaxChunks = (int64_t)1 << 20;   // column chunks (row groups x columns) per file: the host's per-chunk tables

namespace {
struct PqwCol {
    int dtype = 0, phys = 0, width = 0, in_width = 0, conv = pq::CONV_NONE, ord = pq::ORD_SIGNED;
    pq::WColumn meta;
    // per row group, for a column with a dictionary: whether the chunk keeps it, its entries, their first index in the kept
    // entries, and the index in the kept ids of the row group's first row
    std::vector<char> keep;
    std::vector<unsigned int> dcount;
    std::vector<int64_t> dfirst, id0;
};
}  // namespace

// The Parquet type of a column (b200df.h's table).
static int pqw_type(const bdf_col* col, const bdf_temporal_type* tt, const char* name, PqwCol* o) {
    const int dt = col->dtype;
    o->dtype = dt;
    o->meta.name = name;
    pq::WColumn& m = o->meta;
    const bool tagged = tt && tt->kind;
    if (tagged) {   // the tag is checked as bdf_ipc_write_typed checks it: the temporal functions' validation, then the physical dtype
        int32_t rd = 0;
        int st = bdf_temporal_result(BDF_TEMPORAL_UNIX_TIMESTAMP, tt, 0, &rd, nullptr);
        if (st == BDF_UNSUPPORTED) st = bdf_temporal_result(BDF_TEMPORAL_HOUR, tt, 0, &rd, nullptr);   // time kinds
        if (st != BDF_OK) return st;
        const int phys = (tt->kind == BDF_DATE32 || tt->kind == BDF_TIME32) ? BDF_I32 : BDF_I64;
        if (dt != phys) return fail(BDF_INVALID, "column '%s' of dtype %d does not hold temporal kind %d", name, dt, tt->kind);
    }
    if (dt == kBool) { o->phys = pq::PHYS_BOOLEAN; o->width = 0; o->in_width = 0; o->ord = pq::ORD_UNSIGNED; return BDF_OK; }
    if (dt < 0 || dt >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "column '%s': dtype %d is not written to Parquet", name, dt);
    o->in_width = dtype_width(dt);
    if (dt == BDF_F32 || dt == BDF_F64) {
        o->phys = dt == BDF_F32 ? pq::PHYS_FLOAT : pq::PHYS_DOUBLE;
        o->width = o->in_width;
        o->ord = dt == BDF_F32 ? pq::ORD_FLOAT : pq::ORD_DOUBLE;
    } else {
        const bool sg = dtype_is_signed_int(dt);
        const int bits = 8 * o->in_width;
        o->phys = bits == 64 ? pq::PHYS_INT64 : pq::PHYS_INT32;
        o->width = bits == 64 ? 8 : 4;
        o->conv = sg && bits < 32 ? pq::CONV_SEXT : pq::CONV_NONE;
        o->ord = sg ? pq::ORD_SIGNED : pq::ORD_UNSIGNED;
        m.logical = 10; m.int_bits = bits; m.int_signed = sg ? 1 : 0;
        static const int conv_sg[4] = {15, 16, 17, 18}, conv_us[4] = {11, 12, 13, 14};   // INT_8 .. INT_64, UINT_8 .. UINT_64
        const int k = bits == 8 ? 0 : bits == 16 ? 1 : bits == 32 ? 2 : 3;
        m.converted = sg ? conv_sg[k] : conv_us[k];
    }
    m.phys = o->phys;
    if (!tagged) return BDF_OK;
    const int kind = tt->kind, unit = tt->unit;
    o->ord = pq::ORD_SIGNED;
    o->conv = pq::CONV_NONE;
    m.int_bits = 0;
    switch (kind) {
        case BDF_DATE32: case BDF_DATE64:
            o->phys = pq::PHYS_INT32; o->width = 4; m.logical = 6; m.converted = 6;
            if (kind == BDF_DATE64) o->conv = pq::CONV_DAYS;
            break;
        case BDF_TIME32:
            o->phys = pq::PHYS_INT32; o->width = 4; m.logical = 7; m.converted = 7; m.time_unit = 1; m.utc = true;
            if (unit == BDF_SECOND) o->conv = pq::CONV_MUL1000;
            break;
        case BDF_TIME64:
            o->phys = pq::PHYS_INT64; o->width = 8; m.logical = 7; m.time_unit = unit; m.utc = true;
            m.converted = unit == BDF_MICROSECOND ? 8 : -1;
            break;
        default:   // BDF_TIMESTAMP
            o->phys = pq::PHYS_INT64; o->width = 8; m.logical = 8; m.utc = tt->tz != nullptr;
            m.time_unit = unit == BDF_SECOND ? 1 : unit;
            if (unit == BDF_SECOND) o->conv = pq::CONV_MUL1000;
            m.converted = m.utc && m.time_unit == 1 ? 9 : m.utc && m.time_unit == 2 ? 10 : -1;   // TIMESTAMP_MILLIS / _MICROS mean UTC
            break;
    }
    m.phys = o->phys;
    return BDF_OK;
}

// Device-to-device copies of the ranges [from, from + len) of src to consecutive places of dst (elements of `w` bytes).
static cudaError_t pqw_gather(bdf_ctx* c, const char* src, char* dst, const std::vector<std::pair<int64_t, int64_t>>& ranges, int w) {
    int64_t at = 0;
    for (const auto& r : ranges) {
        cudaError_t e = cudaMemcpyAsync(dst + at * w, src + r.first * w, (size_t)(r.second * w), cudaMemcpyDeviceToDevice, c->s_compute);
        if (e != cudaSuccess) return e;
        at += r.second;
    }
    return cudaSuccess;
}

// The dictionary of every row group of one column.  Found over the whole column: ids (one per row, its entry in its row group's
// dictionary) and the distinct values (every row group's valid runs, ascending bits).  Kept: only what the chunks that keep a
// dictionary read -- their rows' ids and their entries (at most kPqwDictLimit bytes each) -- in *ids and *dvals; both stay empty when
// no chunk keeps one.
static int pqw_dictionary(bdf_ctx* c, const bdf_col* col, const bdf_col* rg_col, const std::vector<int64_t>& rg_start, PqwCol* pc, ColOwner* ids,
                          ColOwner* dvals) {
    const int64_t n = col->total_len;
    const int n_rg = (int)rg_start.size() - 1;
    static const int as_unsigned[4] = {BDF_U8, BDF_U16, BDF_U32, BDF_U64};
    const int w = dtype_width(col->dtype);
    ColOwner view(c);
    {
        bdf_col* v = new (std::nothrow) bdf_col();   // the column's chunks read as unsigned integers of its width: no arenas of its own
        if (!v) return fail(BDF_OOM, "host allocation failed");
        v->dtype = as_unsigned[w == 1 ? 0 : w == 2 ? 1 : w == 4 ? 2 : 3];
        v->total_len = n;
        v->chunks = col->chunks;
        v->null_counts = col->null_counts;
        *view.out() = v;
    }
    wait_groups(c->s_compute, col, 0, (int64_t)col->chunks.size());
    const bdf_col* keys[2] = {rg_col, view.get()};
    ColOwner all_ids(c);
    std::vector<unsigned int> first((size_t)n_rg, 0);
    pc->dcount.assign((size_t)n_rg, 0);
    SortedRuns r(c);
    TRY(sorted_runs(c, 2, 2, keys, "Parquet dictionary iota", &r));
    {
        TRY(col_alloc(c, BDF_U32, {ChunkPlan{n, false}}, nullptr, 0, all_ids.out()));
        const int64_t words = (n + 31) / 32;
        Scratch<unsigned int> cf;
        Scratch<unsigned long long> prefix, block_sums;
        cudaError_t e = cf.alloc(c, (size_t)2 * n_rg * sizeof(unsigned int));
        if (e == cudaSuccess) e = prefix.alloc(c, (size_t)(words + 1) * sizeof(unsigned long long));
        if (e == cudaSuccess) e = block_sums.alloc(c, (size_t)scan_tile_sums(words) * sizeof(unsigned long long));
        if (e == cudaSuccess) e = cudaMemsetAsync(cf, 0, (size_t)n_rg * sizeof(unsigned int), c->s_compute);
        if (e == cudaSuccess) e = cudaMemsetAsync(cf + n_rg, 0xff, (size_t)n_rg * sizeof(unsigned int), c->s_compute);
        const int64_t n_runs = r.n_runs;
        const uint32_t* head = (const uint32_t*)r.head->chunks[0].values;
        if (e == cudaSuccess) {
            LaunchTimer t(c, BDF_K_PARQUET_WRITE, BDF_U32, n, words * (4 + 8 + 16) + n * 16 + n_runs * 8);   // head prefix; perm, ids; runs
            c->launches += kScanPopcountLaunches + 1;                                                        // and runs, ids
            e = launch_scan_popcount(head, words, prefix, block_sums, c->s_compute);
            if (e == cudaSuccess)
                e = launch_pqw_dict((const uint32_t*)r.distinct[0]->chunks[0].values, r.distinct[1]->chunks[0].validity, n_runs, head, prefix,
                                    (const uint32_t*)r.perm->chunks[0].values, n, cf, cf + n_rg, (uint32_t*)all_ids->chunks[0].values, c->sm_count,
                                    c->s_compute);
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(pc->dcount.data(), cf, (size_t)n_rg * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->s_compute);
        if (e == cudaSuccess) e = cudaMemcpyAsync(first.data(), cf + n_rg, (size_t)n_rg * sizeof(unsigned int), cudaMemcpyDeviceToHost, c->s_compute);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
        if (e != cudaSuccess) return fail_cuda(e, "Parquet dictionary");
    }
    // which chunks keep a dictionary, and the ranges of ids and entries they read (adjacent row groups merged)
    pc->keep.assign((size_t)n_rg, 0);
    pc->dfirst.assign((size_t)n_rg, 0);
    pc->id0.assign((size_t)n_rg, 0);
    std::vector<std::pair<int64_t, int64_t>> id_ranges, entry_ranges;
    int64_t kept_ids = 0, kept_entries = 0;
    for (int g = 0; g < n_rg; g++) {
        const int64_t cnt = pc->dcount[(size_t)g];
        if (cnt == 0 || cnt * pc->width > kPqwDictLimit) continue;   // the limit counts physical bytes
        pc->keep[(size_t)g] = 1;
        const int64_t rows = rg_start[g + 1] - rg_start[g];
        pc->id0[(size_t)g] = kept_ids;
        pc->dfirst[(size_t)g] = kept_entries;
        if (!id_ranges.empty() && id_ranges.back().first + id_ranges.back().second == rg_start[g]) id_ranges.back().second += rows;
        else id_ranges.push_back({rg_start[g], rows});
        if (!entry_ranges.empty() && entry_ranges.back().first + entry_ranges.back().second == (int64_t)first[(size_t)g]) entry_ranges.back().second += cnt;
        else entry_ranges.push_back({(int64_t)first[(size_t)g], cnt});
        kept_ids += rows;
        kept_entries += cnt;
    }
    if (kept_ids == 0) return BDF_OK;   // every chunk is written PLAIN: nothing is kept
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{kept_ids, false}}, nullptr, 0, ids->out()));
    TRY(col_alloc(c, view->dtype, {ChunkPlan{kept_entries, false}}, nullptr, 0, dvals->out()));
    cudaError_t e = pqw_gather(c, all_ids->chunks[0].values, (*ids)->chunks[0].values, id_ranges, 4);
    if (e == cudaSuccess) e = pqw_gather(c, r.distinct[1]->chunks[0].values, (*dvals)->chunks[0].values, entry_ranges, w);
    if (e == cudaSuccess) e = finish_single_group(c, ids->get());
    if (e == cudaSuccess) e = finish_single_group(c, dvals->get());
    if (e != cudaSuccess) return fail_cuda(e, "Parquet dictionary (kept entries)");
    return BDF_OK;
}

static int parquet_write(bdf_ctx* c, const char* path, int n_cols, const char* const* names, const bdf_col* const* cols, const bdf_temporal_type* types,
                         const bdf_parquet_write_options* opt) {
    if (!path || !names || !cols) return fail(BDF_INVALID, "null argument");
    if (n_cols <= 0) return fail(BDF_INVALID, "no columns to write");
    const int compression = opt ? opt->compression : 0, use_dict = opt ? opt->dictionary : 1;
    const int64_t rg_rows_opt = opt ? opt->row_group_rows : 0;
    if (compression != 0 && compression != 1) return fail(BDF_INVALID, "compression must be 0 (UNCOMPRESSED) or 1 (SNAPPY), not %d", compression);
    if (use_dict != 0 && use_dict != 1) return fail(BDF_INVALID, "dictionary must be 0 or 1, not %d", use_dict);
    if (rg_rows_opt < 0) return fail(BDF_INVALID, "row_group_rows must be at least 0");
    std::vector<PqwCol> pc((size_t)n_cols);
    std::vector<int32_t> dtypes((size_t)n_cols);
    int64_t n_chunks = -1;
    for (int j = 0; j < n_cols; j++) {
        const bdf_col* col = cols[j];
        if (!col || !names[j]) return fail(BDF_INVALID, "null column or name");
        if (!col->fparts.empty()) return fail(BDF_INVALID, "a column of a multi-GPU context was passed to a one-GPU context");
        TRY(pqw_type(col, types ? &types[j] : nullptr, names[j], &pc[(size_t)j]));
        dtypes[(size_t)j] = col->dtype;
        const int64_t nc = (int64_t)col->chunks.size();
        if (n_chunks < 0) n_chunks = nc;
        if (nc != n_chunks)
            return fail(BDF_LENGTH_MISMATCH, "columns have different numbers of chunks (%lld, %lld)", (long long)nc, (long long)n_chunks);
        for (int64_t b = 0; b < nc; b++)
            if (col->chunks[b].len != cols[0]->chunks[b].len)
                return fail(BDF_LENGTH_MISMATCH, "chunk %lld: column '%s' has %lld rows, column '%s' has %lld", (long long)b, names[j],
                            (long long)col->chunks[b].len, names[0], (long long)cols[0]->chunks[b].len);
    }
    std::vector<int64_t> starts((size_t)n_chunks + 1, 0);
    for (int64_t b = 0; b < n_chunks; b++) starts[b + 1] = starts[b] + cols[0]->chunks[b].len;
    const int64_t rows = starts[n_chunks];
    if (rows > 0xffffffffLL) return fail(BDF_UNSUPPORTED, "at most 2^32-1 rows per file (the dictionary's UInt32 row numbers)");
    // row groups: one per non-empty chunk, or row_group_rows rows each across the chunks
    int64_t n_rg64 = 0;
    if (rg_rows_opt == 0) { for (int64_t b = 0; b < n_chunks; b++) n_rg64 += starts[b + 1] > starts[b]; }
    else n_rg64 = (rows + rg_rows_opt - 1) / rg_rows_opt;
    if (n_rg64 * n_cols > kPqwMaxChunks)
        return fail(BDF_INVALID, "%lld row groups x %d columns: at most %lld column chunks per file (use larger row groups)", (long long)n_rg64, n_cols,
                    (long long)kPqwMaxChunks);
    const int n_rg = (int)n_rg64;
    std::vector<int64_t> rg_start;
    if (rg_rows_opt == 0) { for (int64_t b = 0; b < n_chunks; b++) if (starts[b + 1] > starts[b]) rg_start.push_back(starts[b]); }
    else for (int64_t r = 0; r < rows; r += rg_rows_opt) rg_start.push_back(r);
    rg_start.push_back(rows);
    std::string arrow_schema;
    {
        std::vector<bdf_temporal_type> tts((size_t)n_cols, bdf_temporal_type{0, 0, nullptr});
        if (types) for (int j = 0; j < n_cols; j++) tts[(size_t)j] = types[j];
        arrow_schema = pq::base64(bdf::arrow_schema_message(n_cols, names, dtypes.data(), tts.data()));
    }
    std::vector<pq::WColumn> wcols;
    for (auto& p : pc) wcols.push_back(p.meta);

    // dictionaries (every non-Boolean column when dictionary = 1)
    std::vector<ColOwner> ids, dvals;
    for (int j = 0; j < n_cols; j++) { ids.emplace_back(c); dvals.emplace_back(c); }
    if (use_dict && rows > 0) {
        ColOwner rg_col(c);
        TRY(col_alloc(c, BDF_U32, {ChunkPlan{rows, false}}, nullptr, 0, rg_col.out()));
        Scratch<long long> d_rg;
        cudaError_t e = d_rg.alloc(c, (size_t)n_rg * sizeof(long long));
        if (e == cudaSuccess) e = cudaMemcpyAsync(d_rg, rg_start.data(), (size_t)n_rg * sizeof(long long), cudaMemcpyHostToDevice, c->s_compute);
        if (e == cudaSuccess) {
            LaunchTimer t(c, BDF_K_PARQUET_WRITE, BDF_U32, rows, rows * 4);
            e = launch_pqw_rgid(d_rg, n_rg, rows, (uint32_t*)rg_col->chunks[0].values, c->sm_count, c->s_compute);
        }
        if (e == cudaSuccess) e = finish_single_group(c, rg_col.get());
        if (e != cudaSuccess) return fail_cuda(e, "Parquet row-group ids");
        for (int j = 0; j < n_cols; j++)
            if (cols[j]->dtype != kBool) TRY(pqw_dictionary(c, cols[j], rg_col.get(), rg_start, &pc[(size_t)j], &ids[(size_t)j], &dvals[(size_t)j]));
    }

    // the page, tile and fragment tables of every block, in file order
    const bool snappy = compression == 1;
    const uint32_t frag_cap = pq::snappy_bound(pq::kFragment);
    struct Blk { size_t p0, p1, t0, t1, f0, f1; size_t raw; };
    struct PageRef { int rg, col; };
    std::vector<pq::WPage> pages;
    std::vector<pq::WTile> tiles;
    std::vector<int> frag_page;
    std::vector<PageRef> pref;
    std::vector<Blk> blocks;
    std::vector<std::vector<int>> chunk_dict((size_t)n_rg, std::vector<int>((size_t)n_cols, 0));   // the chunk is dictionary-encoded
    Blk cur{0, 0, 0, 0, 0, 0, 0};
    size_t frag_used = 0;
    auto add_page = [&](pq::WPage pg, size_t raw_worst, int rg, int j, const std::function<void(int)>& make_tiles) {
        pg.n_frags = snappy ? (int)((raw_worst + pq::kFragment - 1) / pq::kFragment) : 0;
        size_t slot = raw_worst;
        if (snappy) slot = raw_worst + raw_worst / 6 + 32 * (size_t)pg.n_frags + 8;
        slot = align_up(slot, 16);
        const size_t frags = (size_t)pg.n_frags * frag_cap;
        if (pages.size() > cur.p0 && (cur.raw + slot > kPqwRaw || frag_used + frags > kPqwFrag)) {
            cur.p1 = pages.size(); cur.t1 = tiles.size(); cur.f1 = frag_page.size();
            blocks.push_back(cur);
            cur = Blk{pages.size(), 0, tiles.size(), 0, frag_page.size(), 0, 0};
            frag_used = 0;
        }
        pg.slot = (long long)cur.raw;
        pg.frag0 = (long long)(frag_page.size() - cur.f0);
        pg.tile0 = (int)(tiles.size() - cur.t0);
        for (int f = 0; f < pg.n_frags; f++) frag_page.push_back((int)(pages.size() - cur.p0));
        make_tiles((int)(pages.size() - cur.p0));
        pg.n_tiles = (int)(tiles.size() - cur.t0) - pg.tile0;
        cur.raw += slot;
        frag_used += frags;
        pages.push_back(pg);
        pref.push_back(PageRef{rg, j});
    };
    for (int g = 0; g < n_rg; g++)
        for (int j = 0; j < n_cols; j++) {
            const PqwCol& p = pc[(size_t)j];
            const bdf_col* col = cols[j];
            pq::WPage base{};
            base.width = p.width; base.in_width = p.in_width; base.conv = p.conv; base.ord = p.ord;
            const bool dict = dvals[(size_t)j].get() && p.keep[(size_t)g];
            chunk_dict[(size_t)g][(size_t)j] = dict;
            if (dict) {
                pq::WPage pg = base;
                pg.kind = pq::KIND_DICT;
                pg.rows = (int)p.dcount[(size_t)g];
                const DevChunk& dv = dvals[(size_t)j]->chunks[0];
                const long long first = p.dfirst[(size_t)g];
                add_page(pg, (size_t)pg.rows * p.width, g, j, [&](int page) {
                    for (int e0 = 0; e0 < pg.rows; e0 += pq::kWTileRows)
                        tiles.push_back(pq::WTile{dv.values, nullptr, nullptr, first + e0, 0, 0, page, e0, std::min(pq::kWTileRows, pg.rows - e0), 0});
                });
                base.id_bw = pq::id_bit_width(p.dcount[(size_t)g]);
            }
            for (int64_t r0 = rg_start[g]; r0 < rg_start[g + 1]; r0 += kPqwPageRows) {
                const int64_t r1 = std::min(rg_start[g + 1], r0 + kPqwPageRows);
                pq::WPage pg = base;
                pg.kind = pq::KIND_V1;
                pg.rows = (int)(r1 - r0);
                const size_t nr = (size_t)pg.rows, bits = (nr + 7) / 8;
                const size_t values = pg.id_bw ? 1 + 5 + bits * (size_t)pg.id_bw : p.width ? nr * (size_t)p.width : bits;
                add_page(pg, 4 + 5 + bits + values, g, j, [&](int page) {
                    int64_t b = std::upper_bound(starts.begin(), starts.end(), r0) - starts.begin() - 1;
                    for (int64_t r = r0; r < r1;) {
                        while (starts[b + 1] <= r) b++;
                        const DevChunk& ch = col->chunks[(size_t)b];
                        const int64_t end = std::min({r1, starts[b + 1], r + (int64_t)pq::kWTileRows});
                        const uint32_t* idp = dict ? (const uint32_t*)ids[(size_t)j]->chunks[0].values + p.id0[(size_t)g] + (r - rg_start[g]) : nullptr;
                        tiles.push_back(pq::WTile{ch.values, ch.validity, idp, r - starts[b], ch.bit_off, ch.val_bit_off, page, (int)(r - r0), (int)(end - r), 0});
                        r = end;
                    }
                });
            }
        }
    if (pages.size() > cur.p0) { cur.p1 = pages.size(); cur.t1 = tiles.size(); cur.f1 = frag_page.size(); blocks.push_back(cur); }
    if (tiles.size() > (size_t)0x7fffffff) return fail(BDF_UNSUPPORTED, "the file has more tiles than one launch covers");

    // device buffers, then the file
    for (int j = 0; j < n_cols; j++) wait_groups(c->s_compute, cols[j], 0, n_chunks);
    const size_t np = std::max<size_t>(pages.size(), 1), nt = std::max<size_t>(tiles.size(), 1), nf = std::max<size_t>(frag_page.size(), 1);
    Scratch<char> d_pages, d_tiles, d_out, d_lay;
    Scratch<unsigned int> d_tvalid, d_tbase, d_flen;
    Scratch<int> d_fpage;
    Scratch<uint8_t> raw[2], frag;
    struct Pinned { pq::WPageOut* p = nullptr; ~Pinned() { if (p) cudaFreeHost(p); } } h_out;
    cudaError_t e = d_pages.alloc(c, np * sizeof(pq::WPage));
    if (e == cudaSuccess) e = d_tiles.alloc(c, nt * sizeof(pq::WTile));
    if (e == cudaSuccess) e = d_out.alloc(c, np * sizeof(pq::WPageOut));
    if (e == cudaSuccess) e = d_lay.alloc(c, np * sizeof(uint2));
    if (e == cudaSuccess) e = d_tvalid.alloc(c, nt * sizeof(unsigned int));
    if (e == cudaSuccess) e = d_tbase.alloc(c, nt * sizeof(unsigned int));
    if (e == cudaSuccess) e = d_fpage.alloc(c, nf * sizeof(int));
    if (e == cudaSuccess) e = d_flen.alloc(c, nf * sizeof(unsigned int));
    if (e == cudaSuccess && !blocks.empty()) e = raw[0].alloc(c, kPqwRaw);
    if (e == cudaSuccess && blocks.size() > 1) e = raw[1].alloc(c, kPqwRaw);
    if (e == cudaSuccess && snappy && !blocks.empty()) e = frag.alloc(c, kPqwFrag);
    if (e == cudaSuccess && !pages.empty()) e = cudaMemcpyAsync(d_pages, pages.data(), pages.size() * sizeof(pq::WPage), cudaMemcpyHostToDevice, c->s_compute);
    if (e == cudaSuccess && !tiles.empty()) e = cudaMemcpyAsync(d_tiles, tiles.data(), tiles.size() * sizeof(pq::WTile), cudaMemcpyHostToDevice, c->s_compute);
    if (e == cudaSuccess && !frag_page.empty()) e = cudaMemcpyAsync(d_fpage, frag_page.data(), frag_page.size() * sizeof(int), cudaMemcpyHostToDevice, c->s_compute);
    if (e == cudaSuccess) e = cudaHostAlloc((void**)&h_out.p, np * sizeof(pq::WPageOut), cudaHostAllocDefault);
    if (e != cudaSuccess) return fail_cuda(e, "Parquet write setup");
    TRY(ensure_stage(c));
    struct Events { bdf_ctx* c; cudaEvent_t ev[4] = {}; ~Events() { for (auto x : ev) ev_put(c, x); } } evs{c};
    for (auto& x : evs.ev) CK(ev_get(c, &x));
    cudaEvent_t* ev_done = evs.ev;       // block k's page results are on the host and its bodies complete in raw[k & 1]
    cudaEvent_t* ev_d2h = evs.ev + 2;    // block k's bodies have left raw[k & 1]

    const int fd = open(path, O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
    if (fd < 0) return fail(BDF_INVALID, "cannot create %s: %s", path, strerror(errno));
    struct FdGuard { int fd; ~FdGuard() { if (fd >= 0) close(fd); } } fdg{fd};
    // Declared after the buffers, so it runs first on every exit: no copy may still read a body buffer when it is freed.
    struct DrainD2H { cudaStream_t s; ~DrainD2H() { cudaStreamSynchronize(s); } } drain_guard{c->s_d2h};
    off_t file_off = 0;

    size_t rec_enc[2] = {0, 0}, rec_snappy[2] = {0, 0};
    auto enqueue = [&](size_t k) -> int {
        const Blk& B = blocks[k];
        const int b = (int)(k & 1);
        cudaError_t e2 = k >= 2 ? cudaStreamWaitEvent(c->s_compute, ev_d2h[b], 0) : cudaSuccess;
        if (e2 == cudaSuccess) e2 = cudaMemsetAsync(raw[b], 0, B.raw, c->s_compute);
        const int n_p = (int)(B.p1 - B.p0), n_t = (int)(B.t1 - B.t0), n_f = (int)(B.f1 - B.f0);
        if (e2 == cudaSuccess) {
            int64_t in_rows = 0, in_bytes = 0;
            for (size_t t = B.t0; t < B.t1; t++) {
                const pq::WPage& pg = pages[B.p0 + (size_t)tiles[t].page];
                in_rows += tiles[t].rows;
                in_bytes += pg.in_width ? (int64_t)tiles[t].rows * pg.in_width : tiles[t].rows / 8;
            }
            LaunchTimer t(c, BDF_K_PARQUET_WRITE, -1, in_rows, in_bytes);   // + the bodies, once their sizes are known
            c->launches += 2;                                                // count, layout, encode
            e2 = launch_pqw_encode(d_pages + B.p0 * sizeof(pq::WPage), n_p, d_tiles + B.t0 * sizeof(pq::WTile), n_t, d_tvalid + B.t0, d_tbase + B.t0,
                                   d_lay + B.p0 * sizeof(uint2), raw[b], d_out + B.p0 * sizeof(pq::WPageOut), c->s_compute);
        }
        if (c->profiling) rec_enc[b] = c->prof.size() - 1;
        if (e2 == cudaSuccess && snappy) {
            LaunchTimer t(c, BDF_K_PARQUET_WRITE, BDF_U8, n_p, 0);   // bytes: the bodies read and written, once known
            c->launches++;                                           // snappy, compaction
            e2 = launch_pqw_snappy(d_pages + B.p0 * sizeof(pq::WPage), d_fpage + B.f0, n_f, raw[b], d_out + B.p0 * sizeof(pq::WPageOut), frag,
                                   d_flen + B.f0, c->s_compute);
            if (c->profiling) rec_snappy[b] = c->prof.size() - 1;
        }
        if (e2 == cudaSuccess)
            e2 = cudaMemcpyAsync(h_out.p + B.p0, d_out + B.p0 * sizeof(pq::WPageOut), (size_t)n_p * sizeof(pq::WPageOut), cudaMemcpyDeviceToHost, c->s_compute);
        if (e2 == cudaSuccess) e2 = cudaEventRecord(ev_done[b], c->s_compute);
        return e2 == cudaSuccess ? BDF_OK : fail_cuda(e2, "Parquet write kernels");
    };
    struct Pending { bdf_ctx::StageSlot* sl; off_t off; size_t n; };
    std::deque<Pending> pending;
    auto retire = [&]() -> int {
        const Pending p = pending.front();
        pending.pop_front();
        CK(cudaEventSynchronize(p.sl->ev));
        p.sl->busy = false;
        constexpr size_t kJob = (size_t)512 << 10;
        std::atomic<int> werr{0};
        c->pool->run((p.n + kJob - 1) / kJob, [&](size_t j) {
            const int we = pwrite_all(fd, p.sl->p + j * kJob, std::min(kJob, p.n - j * kJob), p.off + (off_t)(j * kJob));
            if (we) werr = we;
        });
        if (werr) return fail(BDF_INVALID, "writing %s failed: %s", path, strerror(werr));
        return BDF_OK;
    };
    // The file's bytes go through the staging slots in order: a header is copied in by the host, a body by a D2H copy.
    bdf_ctx::StageSlot* sl = nullptr;
    size_t fill = 0;
    off_t slot_off = 0;
    auto close_slot = [&]() -> int {
        if (!sl) return BDF_OK;
        CK(cudaEventRecord(sl->ev, c->s_d2h));
        sl->busy = true;
        pending.push_back(Pending{sl, slot_off, fill});
        sl = nullptr;
        return BDF_OK;
    };
    auto put = [&](const char* src, size_t n, bool device) -> int {
        while (n) {
            if (!sl || fill == kStageBytes) {
                TRY(close_slot());
                if ((int)pending.size() >= kStageSlots - 1) TRY(retire());
                sl = &c->stage[c->stage_next++ % kStageSlots];
                if (sl->busy) CK(cudaEventSynchronize(sl->ev));   // an upload's slot
                fill = 0;
                slot_off = file_off;
            }
            const size_t m = std::min(n, kStageBytes - fill);
            if (device) CK(cudaMemcpyAsync(sl->p + fill, src, m, cudaMemcpyDeviceToHost, c->s_d2h));
            else memcpy(sl->p + fill, src, m);
            fill += m; src += m; n -= m; file_off += (off_t)m;
        }
        return BDF_OK;
    };
    TRY(put("PAR1", 4, false));
    std::vector<std::vector<pq::WChunkMeta>> meta((size_t)n_rg, std::vector<pq::WChunkMeta>((size_t)n_cols));
    std::vector<std::vector<pq::Stats>> cst((size_t)n_rg, std::vector<pq::Stats>((size_t)n_cols, pq::stats_empty()));
    auto drain = [&](size_t k) -> int {
        const Blk& B = blocks[k];
        const int b = (int)(k & 1);
        CK(cudaEventSynchronize(ev_done[b]));
        CK(cudaStreamWaitEvent(c->s_d2h, ev_done[b], 0));
        int64_t raw_sum = 0, comp_sum = 0;
        for (size_t i = B.p0; i < B.p1; i++) {
            const pq::WPage& pg = pages[i];
            const pq::WPageOut& o = h_out.p[i];
            if (o.err) return fail(BDF_INVALID, "a snappy fragment outgrew its worst-case bound");
            const PageRef& pr = pref[i];
            pq::WChunkMeta& m = meta[(size_t)pr.rg][(size_t)pr.col];
            const bool dict = chunk_dict[(size_t)pr.rg][(size_t)pr.col] != 0;
            const int enc = pg.kind == pq::KIND_DICT || pg.id_bw ? pq::ENC_PLAIN_DICTIONARY : pq::ENC_PLAIN;
            const std::string h = pq::page_header(pg.kind, (int)o.raw_len, (int)o.comp_len, pg.rows, enc);
            if (pg.kind == pq::KIND_DICT) m.dict_page_offset = file_off;
            else if (m.num_values == 0) m.data_page_offset = file_off;
            if (pg.kind != pq::KIND_DICT) { m.num_values += pg.rows; pq::stats_merge(&cst[(size_t)pr.rg][(size_t)pr.col], o.st); }
            m.total_uncompressed += (long long)(h.size() + o.raw_len);
            m.total_compressed += (long long)(h.size() + o.comp_len);
            m.phys = pc[(size_t)pr.col].phys;
            m.codec = snappy ? 1 : 0;
            m.encodings = dict ? std::vector<int>{pq::ENC_PLAIN_DICTIONARY, pq::ENC_RLE} : std::vector<int>{pq::ENC_PLAIN, pq::ENC_RLE};
            raw_sum += o.raw_len;
            comp_sum += o.comp_len;
            TRY(put(h.data(), h.size(), false));
            TRY(put((const char*)raw[b].get() + pg.slot, o.comp_len, true));
        }
        if (c->profiling) {
            c->prof[rec_enc[b]].rec.bytes += raw_sum;
            if (snappy) c->prof[rec_snappy[b]].rec.bytes += raw_sum + comp_sum;
        }
        CK(cudaEventRecord(ev_d2h[b], c->s_d2h));
        return BDF_OK;
    };
    if (!blocks.empty()) TRY(enqueue(0));
    for (size_t k = 0; k < blocks.size(); k++) {
        if (k + 1 < blocks.size()) TRY(enqueue(k + 1));
        TRY(drain(k));
    }
    // the footer: chunk statistics in the stored physical values
    for (int g = 0; g < n_rg; g++)
        for (int j = 0; j < n_cols; j++) {
            pq::WChunkMeta& m = meta[(size_t)g][(size_t)j];
            const pq::Stats& s = cst[(size_t)g][(size_t)j];
            const PqwCol& p = pc[(size_t)j];
            const int w = p.width ? p.width : 1;
            m.has_stats = true;
            m.null_count = (long long)s.nulls;
            m.has_minmax = s.count > 0;
            if (m.has_minmax) {
                const uint64_t lo = pq::stat_value(p.ord, w, s.kmin, false), hi = pq::stat_value(p.ord, w, s.kmax, true);
                m.min_value.assign((const char*)&lo, (size_t)w);   // little-endian
                m.max_value.assign((const char*)&hi, (size_t)w);
            }
        }
    std::vector<long long> rg_rows((size_t)n_rg);
    for (int g = 0; g < n_rg; g++) rg_rows[(size_t)g] = rg_start[g + 1] - rg_start[g];
    std::string tail = pq::file_metadata(wcols, rg_rows, meta, arrow_schema);
    const uint32_t flen = (uint32_t)tail.size();
    tail.append((const char*)&flen, 4);
    tail += "PAR1";
    TRY(put(tail.data(), tail.size(), false));
    TRY(close_slot());
    while (!pending.empty()) TRY(retire());
    const int fdv = fdg.fd;
    fdg.fd = -1;
    if (close(fdv) != 0) return fail(BDF_INVALID, "closing %s failed: %s", path, strerror(errno));
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// Multi-GPU context (bdf_init_multi): ONE process, every GPU of the box.  The library owns the sharding that the
// reference leaves to rayon (par_iter over chunks, src/functions/scalar.rs:28-31,99-102): the rows of a call are cut into
// one contiguous range per GPU (cuts on 64-row boundaries inside a chunk, so a piece is a zero-copy Arrow slice whose
// validity starts on a byte boundary), every GPU runs the ordinary one-GPU path on its pieces -- its own PCIe link, its
// own staging threads -- and aggregates are combined by the grouped ncclAllReduce of comm.cu (ncclCommInitAll).
// A fleet context owns no device; its "kids" are complete one-GPU contexts driven by one persistent host thread each
// (a blocking collective must be entered by all ranks at once, and uploads of different GPUs should overlap).

struct Fleet {
    std::vector<bdf_ctx*> kids;
    struct Worker {
        std::thread th;
        std::mutex m;
        std::condition_variable cv;
        std::function<int()> job;
        bool has_job = false, done = false, stop = false;
        int status = BDF_OK;
        std::string err;
    };
    std::vector<std::unique_ptr<Worker>> workers;
    std::mutex run_mu;   // one fan-out at a time: two caller threads must not interleave their jobs (or the order of the kids' collectives)
};

static void fleet_worker_main(Fleet::Worker* w, int device) {
    // run near the GPU: host<->device copies and the staging threads this thread creates stay on the GPU's NUMA node
    char bus[32];
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) == cudaSuccess) {
        for (char* p = bus; *p; p++) *p = (char)tolower(*p);
        const std::string base = std::string("/sys/bus/pci/devices/") + bus + "/numa_node";
        int node = -1;
        if (FILE* f = fopen(base.c_str(), "r")) { if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f); }
        if (node >= 0) {
            const std::string cl = "/sys/devices/system/node/node" + std::to_string(node) + "/cpulist";
            if (FILE* f = fopen(cl.c_str(), "r")) {
                char buf[4096];
                if (fgets(buf, sizeof buf, f)) {
                    cpu_set_t set, cur; CPU_ZERO(&set);
                    int n = 0;
                    for (char* tok = strtok(buf, ",\n"); tok; tok = strtok(nullptr, ",\n")) {
                        int lo, hi;
                        if (sscanf(tok, "%d-%d", &lo, &hi) == 2) { for (int cpu = lo; cpu <= hi && cpu < CPU_SETSIZE; cpu++) { CPU_SET(cpu, &set); n++; } }
                        else if (sscanf(tok, "%d", &lo) == 1 && lo < CPU_SETSIZE) { CPU_SET(lo, &set); n++; }
                    }
                    if (n && sched_getaffinity(0, sizeof cur, &cur) == 0) {
                        CPU_AND(&set, &set, &cur);
                        if (CPU_COUNT(&set) > 0) sched_setaffinity(0, sizeof set, &set);
                    }
                }
                fclose(f);
            }
        }
    }
    cudaGetLastError();
    std::unique_lock<std::mutex> lk(w->m);
    for (;;) {
        w->cv.wait(lk, [w] { return w->has_job || w->stop; });
        if (w->stop) return;
        std::function<int()> job = std::move(w->job);
        w->has_job = false;
        lk.unlock();
        g_err.clear();
        int st;
        try { st = job(); } catch (...) { st = fail(BDF_INVALID, "internal error in a fleet worker"); }
        lk.lock();
        w->status = st;
        w->err = g_err;
        w->done = true;
        w->cv.notify_all();
    }
}

// Run fn(k) for every kid, each on its own thread, and wait.  The first failing status (lowest kid) is returned with its message.
static int fleet_run(Fleet* f, const std::function<int(int)>& fn) {
    std::lock_guard<std::mutex> one_at_a_time(f->run_mu);   // the jobs run on the workers and never fan out themselves: no recursion
    const int n = (int)f->kids.size();
    for (int k = 0; k < n; k++) {
        Fleet::Worker* w = f->workers[k].get();
        std::lock_guard<std::mutex> g(w->m);
        w->job = [&fn, k] { return fn(k); };
        w->has_job = true; w->done = false;
        w->cv.notify_all();
    }
    int status = BDF_OK;
    std::string err;
    for (int k = 0; k < n; k++) {
        Fleet::Worker* w = f->workers[k].get();
        std::unique_lock<std::mutex> lk(w->m);
        w->cv.wait(lk, [w] { return w->done; });
        if (w->status != BDF_OK && status == BDF_OK) { status = w->status; err = w->err; }
    }
    if (status != BDF_OK) g_err = err;
    return status;
}

static bool is_fleet_col(const bdf_col* col) { return col && !col->fparts.empty(); }

// Cut the rows of the logical chunks into one contiguous range per kid (balanced by rows; cuts inside a chunk are
// multiples of 64 rows).  Returns the pieces per logical chunk; `local` numbers a kid's pieces in order.
static std::vector<std::vector<bdf_col::Piece>> fleet_plan(const std::vector<int64_t>& lens, int n_kids) {
    const size_t n = lens.size();
    int64_t total = 0;
    std::vector<int64_t> start(n + 1, 0);
    for (size_t i = 0; i < n; i++) { start[i] = total; total += lens[i]; }
    start[n] = total;
    auto snap = [&](int64_t g) {   // a global cut -> an aligned row of the chunk it falls into
        if (g <= 0) return (int64_t)0;
        if (g >= total) return total;
        size_t i = (size_t)(std::upper_bound(start.begin(), start.begin() + (ptrdiff_t)n, g) - start.begin()) - 1;
        return start[i] + (g - start[i]) / 64 * 64;
    };
    std::vector<int64_t> cut((size_t)n_kids + 1);
    for (int k = 0; k <= n_kids; k++) cut[k] = snap((int64_t)((__int128)total * k / n_kids));
    cut[n_kids] = total;
    std::vector<std::vector<bdf_col::Piece>> map(n);
    std::vector<int64_t> next_local((size_t)n_kids, 0);
    for (size_t i = 0; i < n; i++)
        for (int k = 0; k < n_kids; k++) {
            const int64_t b = std::max(cut[k], start[i]), e = std::min(cut[k + 1], start[i] + lens[i]);
            if (e > b) map[i].push_back(bdf_col::Piece{k, next_local[k]++, b - start[i], e - b});
        }
    // an empty logical chunk still needs a home (it keeps the chunk structure and the reference's panic rule intact)
    for (size_t i = 0; i < n; i++)
        if (lens[i] == 0) map[i].push_back(bdf_col::Piece{(int)(i % (size_t)n_kids), next_local[i % (size_t)n_kids]++, 0, 0});
    return map;
}

// The host views of kid k under a plan (zero-copy slices of the caller's chunks), in the kid's local chunk order.
static std::vector<bdf_view> fleet_views(const std::vector<std::vector<bdf_col::Piece>>& map, int n_kids, int kid, const bdf_view* in) {
    std::vector<std::pair<int64_t, bdf_view>> mine;
    for (size_t i = 0; i < map.size(); i++)
        for (const auto& pc : map[i])
            if (pc.kid == kid) {
                bdf_view v = in[i];
                v.offset += pc.row0;
                v.len = pc.rows;
                if (!(pc.row0 == 0 && pc.rows == in[i].len)) v.null_count = v.validity ? -1 : 0;   // a proper slice: unknown
                mine.push_back({pc.local, v});
            }
    (void)n_kids;
    std::sort(mine.begin(), mine.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    std::vector<bdf_view> out;
    for (auto& m : mine) out.push_back(m.second);
    return out;
}

static std::vector<bdf_out> fleet_outs(const std::vector<std::vector<bdf_col::Piece>>& map, int kid, int out_dtype, const bdf_out* out) {
    std::vector<std::pair<int64_t, bdf_out>> mine;
    const int w = out_dtype == kBool ? 0 : dtype_width(out_dtype);
    for (size_t i = 0; i < map.size(); i++)
        for (const auto& pc : map[i])
            if (pc.kid == kid) {
                bdf_out o = out[i];
                if (o.values) o.values = (char*)o.values + (out_dtype == kBool ? pc.row0 / 8 : pc.row0 * w);
                if (o.validity) o.validity = o.validity + pc.row0 / 8;   // row0 is a multiple of 64
                o.len = pc.rows;
                mine.push_back({pc.local, o});
            }
    std::sort(mine.begin(), mine.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
    std::vector<bdf_out> res;
    for (auto& m : mine) res.push_back(m.second);
    return res;
}

// Fold the kids' per-piece results back into the caller's per-chunk bdf_out entries.
static void fleet_merge_outs(const std::vector<std::vector<bdf_col::Piece>>& map, const std::vector<std::vector<bdf_out>>& kid_outs,
                             const std::vector<int64_t>& lens, bdf_out* out) {
    for (size_t i = 0; i < map.size(); i++) {
        int64_t nulls = 0;
        int32_t hv = 0;
        for (const auto& pc : map[i]) {
            const bdf_out& o = kid_outs[(size_t)pc.kid][(size_t)pc.local];
            nulls += o.null_count;
            hv |= o.has_validity;
        }
        out[i].len = lens[i];
        out[i].null_count = nulls;
        out[i].has_validity = hv;
    }
}

static bool fleet_same_map(const bdf_col* a, const bdf_col* b, int64_t n) {
    if ((int64_t)a->fmap.size() < n || (int64_t)b->fmap.size() < n) return false;
    for (int64_t i = 0; i < n; i++) {
        if (a->fmap[i].size() != b->fmap[i].size()) return false;
        for (size_t j = 0; j < a->fmap[i].size(); j++) {
            const auto &x = a->fmap[i][j], &y = b->fmap[i][j];
            if (x.kid != y.kid || x.local != y.local || x.row0 != y.row0 || x.rows != y.rows) return false;
        }
    }
    return true;
}

static bdf_col* fleet_col_new(int dtype, int n_kids) {
    bdf_col* col = new (std::nothrow) bdf_col();
    if (!col) return nullptr;
    col->dtype = dtype;
    col->fparts.assign((size_t)n_kids, nullptr);
    return col;
}

static void fleet_col_free(Fleet* f, bdf_col* col) {
    if (!col) return;
    for (size_t k = 0; k < col->fparts.size(); k++)
        if (col->fparts[k]) bdf_col_free(f->kids[k], col->fparts[k]);
    delete col;
}

// A result column with the logical structure of `like` (elementwise operators keep it), parts filled by the kids.
static bdf_col* fleet_col_like(const bdf_col* like, int dtype, int n_kids, int64_t n_chunks) {
    bdf_col* col = fleet_col_new(dtype, n_kids);
    if (!col) return nullptr;
    col->fmap.assign(like->fmap.begin(), like->fmap.begin() + (ptrdiff_t)n_chunks);
    col->flens.assign(like->flens.begin(), like->flens.begin() + (ptrdiff_t)n_chunks);
    col->total_len = 0;
    for (int64_t v : col->flens) col->total_len += v;
    return col;
}

static int fleet_upload_many(bdf_ctx* c, int64_t n_cols, const int32_t* dtypes, const int64_t* n_chunks, const bdf_view* const* in, int flags, bdf_col** out) {
    Fleet* f = c->fleet;
    const int nk = (int)f->kids.size();
    // all columns of one call share ONE plan when their chunk lengths agree (a RecordBatch list), so that operators over them line up
    std::vector<bdf_col*> cols((size_t)n_cols, nullptr);
    std::vector<std::vector<std::vector<bdf_view>>> views((size_t)n_cols);
    for (int64_t j = 0; j < n_cols; j++) {
        std::vector<int64_t> lens((size_t)n_chunks[j]);
        for (int64_t i = 0; i < n_chunks[j]; i++) {
            if (in[j][i].len < 0 || in[j][i].offset < 0) { for (auto* x : cols) fleet_col_free(f, x); return fail(BDF_INVALID, "bad view %lld", (long long)i); }
            lens[i] = in[j][i].len;
        }
        cols[j] = fleet_col_new(dtypes[j], nk);
        if (!cols[j]) { for (auto* x : cols) fleet_col_free(f, x); return fail(BDF_OOM, "host allocation failed"); }
        cols[j]->fmap = fleet_plan(lens, nk);
        cols[j]->flens = lens;
        for (int64_t v : lens) cols[j]->total_len += v;
        views[j].resize((size_t)nk);
        for (int k = 0; k < nk; k++) views[j][k] = fleet_views(cols[j]->fmap, nk, k, in[j]);
    }
    int st = fleet_run(f, [&](int k) {
        std::vector<int32_t> dt((size_t)n_cols);
        std::vector<int64_t> cnt((size_t)n_cols);
        std::vector<const bdf_view*> ptr((size_t)n_cols);
        std::vector<bdf_col*> res((size_t)n_cols, nullptr);
        for (int64_t j = 0; j < n_cols; j++) { dt[j] = dtypes[j]; cnt[j] = (int64_t)views[j][k].size(); ptr[j] = views[j][k].data(); }
        int s2 = bdf_upload_many(f->kids[k], n_cols, dt.data(), cnt.data(), ptr.data(), flags, res.data());
        for (int64_t j = 0; j < n_cols; j++) cols[j]->fparts[k] = res[j];
        return s2;
    });
    if (st != BDF_OK) { const std::string keep = g_err; for (auto* x : cols) fleet_col_free(f, x); g_err = keep; return st; }
    for (int64_t j = 0; j < n_cols; j++) out[j] = cols[j];
    return BDF_OK;
}

static int fleet_download(bdf_ctx* c, const bdf_col* col, bdf_out* out, int phase /* 0 both, 1 begin, 2 end */) {
    Fleet* f = c->fleet;
    const int nk = (int)f->kids.size();
    const int64_t n = (int64_t)col->fmap.size();
    for (int64_t i = 0; i < n; i++)
        if (out[i].len != col->flens[i]) return fail(BDF_INVALID, "output chunk %lld has capacity %lld, result has %lld rows", (long long)i, (long long)out[i].len, (long long)col->flens[i]);
    std::vector<std::vector<bdf_out>> kouts((size_t)nk);
    for (int k = 0; k < nk; k++) kouts[k] = fleet_outs(col->fmap, k, col->dtype, out);
    int st = fleet_run(f, [&](int k) {
        bdf_out dummy{};
        bdf_out* o = kouts[k].empty() ? &dummy : kouts[k].data();
        if (phase == 1) return bdf_download_begin(f->kids[k], col->fparts[k], o);
        if (phase == 2) return bdf_download_end(f->kids[k], col->fparts[k], o);
        return bdf_download(f->kids[k], col->fparts[k], o);
    });
    if (st != BDF_OK) return st;
    if (phase != 1) fleet_merge_outs(col->fmap, kouts, col->flens, out);
    return BDF_OK;
}

// The inputs of one elementwise call on a fleet context: fleet columns whose chunks pair up as zip() pairs them, cut by one plan.
// `*n` is the number of pairs.  Unequal chunk lengths are reported as `mismatch` and unequal chunk counts as `uneven`, because
// the entries answer them differently (BDF_LENGTH_MISMATCH or BDF_INVALID, BDF_UNSUPPORTED or BDF_INVALID).
static int fleet_zip(const bdf_col* const* cols, size_t n_cols, int mismatch, int uneven, int64_t* n) {
    auto differ = [](int st) {
        if (st == BDF_LENGTH_MISMATCH) return fail(st, "Cannot perform math operation on arrays of different length");
        if (st == BDF_UNSUPPORTED) return fail(st, "columns with different numbers of chunks on a multi-GPU context");
        return fail(BDF_INVALID, "the columns are sharded differently over the GPUs (upload them in one bdf_upload_many call)");
    };
    const bdf_col* first = cols[0];
    *n = (int64_t)first->fmap.size();
    for (size_t j = 0; j < n_cols; j++) {
        if (!is_fleet_col(cols[j])) return fail(BDF_INVALID, "a column of a one-GPU context was passed to a multi-GPU context");
        *n = std::min<int64_t>(*n, (int64_t)cols[j]->fmap.size());
    }
    for (size_t j = 0; j < n_cols; j++) {
        for (int64_t i = 0; i < *n; i++)
            if (cols[j]->flens[i] != first->flens[i]) return differ(mismatch);
        if (!fleet_same_map(first, cols[j], *n)) return differ(BDF_INVALID);
        if (cols[j]->fmap.size() != first->fmap.size()) return differ(uneven);
    }
    return BDF_OK;
}

// One elementwise operator over fleet columns: `call(k, parts of the inputs on kid k, &result part)`.
static int fleet_map(bdf_ctx* c, int out_dtype, const bdf_col* const* inputs, size_t n_inputs, bdf_col** out,
                     const std::function<int(int, bdf_col**)>& call) {
    Fleet* f = c->fleet;
    const int nk = (int)f->kids.size();
    int64_t n = 0;
    TRY(fleet_zip(inputs, n_inputs, BDF_LENGTH_MISMATCH, BDF_UNSUPPORTED, &n));
    bdf_col* o = fleet_col_like(inputs[0], out_dtype, nk, n);
    if (!o) return fail(BDF_OOM, "host allocation failed");
    int st = fleet_run(f, [&](int k) { return call(k, &o->fparts[k]); });
    if (st != BDF_OK) { const std::string keep = g_err; fleet_col_free(f, o); g_err = keep; return st; }
    *out = o;
    return BDF_OK;
}
static int fleet_map(bdf_ctx* c, int out_dtype, std::initializer_list<const bdf_col*> inputs, bdf_col** out,
                     const std::function<int(int, bdf_col**)>& call) {
    return fleet_map(c, out_dtype, inputs.begin(), inputs.size(), out, call);
}

static bdf_future* fleet_future_new(int n_kids) {
    bdf_future* fu = new (std::nothrow) bdf_future();
    if (fu) fu->fparts.assign((size_t)n_kids, nullptr);
    return fu;
}

static int fleet_future_wait(bdf_ctx* c, bdf_future* fu, bdf_agg4* out) {
    Fleet* f = c->fleet;
    const int n = fu->n;
    std::vector<std::vector<bdf_agg4>> res(f->kids.size(), std::vector<bdf_agg4>((size_t)std::max(n, 1)));
    int st = fleet_run(f, [&](int k) { return fu->fparts[k] ? bdf_future_wait(f->kids[k], fu->fparts[k], res[k].data()) : BDF_OK; });
    if (st == BDF_OK && out) for (int i = 0; i < n; i++) out[i] = res[0][i];   // every rank holds the same global records
    delete fu;
    return st;
}

// Aggregates of n columns: every kid reduces its parts, the collective inside the kids' call makes the result global.
static int fleet_aggregate_many(bdf_ctx* c, int32_t n_cols, const bdf_col* const* cols, bdf_future** fut) {
    Fleet* f = c->fleet;
    if (n_cols < 1 || n_cols > kCommMaxCols) return fail(BDF_INVALID, "an aggregate call takes 1..%d columns", kCommMaxCols);
    for (int32_t j = 0; j < n_cols; j++)
        if (!is_fleet_col(cols[j])) return fail(BDF_INVALID, "a column of a one-GPU context was passed to a multi-GPU context");
    bdf_future* fu = fleet_future_new((int)f->kids.size());
    if (!fu) return fail(BDF_OOM, "host allocation failed");
    fu->n = n_cols;
    int st = fleet_run(f, [&](int k) {
        std::vector<const bdf_col*> parts((size_t)n_cols);
        for (int32_t j = 0; j < n_cols; j++) parts[j] = cols[j]->fparts[k];
        return bdf_aggregate_all_many_dev_async(f->kids[k], n_cols, parts.data(), &fu->fparts[k]);
    });
    if (st != BDF_OK) { const std::string keep = g_err; fleet_future_wait(c, fu, nullptr); g_err = keep; return st; }
    *fut = fu;
    return BDF_OK;
}

// Logical chunks of a fleet column without a valid slot (empty or all-null): the reference's max/min unwrap() a None there.
// Evaluated over the caller's chunks -- a piece may be all-null while its chunk is not.
static int fleet_panic_chunks(bdf_ctx* c, const bdf_col* col, int* out) {
    Fleet* f = c->fleet;
    const size_t n = col->fmap.size();
    std::vector<int64_t> valid(n, 0);
    std::mutex m;
    int st = fleet_run(f, [&](int k) {
        for (size_t i = 0; i < n; i++)
            for (const auto& pc : col->fmap[i])
                if (pc.kid == k) {
                    int64_t len = 0, nulls = 0; int32_t hv = 0;
                    int s2 = bdf_col_chunk_info(f->kids[k], col->fparts[k], pc.local, &len, &nulls, &hv);
                    if (s2 != BDF_OK) return s2;
                    std::lock_guard<std::mutex> g(m);
                    valid[i] += len - (hv ? nulls : 0);
                }
        return (int)BDF_OK;
    });
    if (st != BDF_OK) return st;
    int k = 0;
    for (size_t i = 0; i < n; i++) if (valid[i] == 0) k++;
    *out = k;
    return BDF_OK;
}

static int fleet_aggregate_dev(bdf_ctx* c, int op, const bdf_col* col, void* out_scalar, int32_t* is_some) {
    if (op < 0 || op >= BDF_NAGG) return fail(BDF_INVALID, "invalid aggregate op %d", op);
    if (!is_fleet_col(col)) return fail(BDF_INVALID, "a column of a one-GPU context was passed to a multi-GPU context");
    const int dtype = col->dtype;
    if ((op == BDF_MIN || op == BDF_MAX) && dtype_is_float(dtype)) return fail(BDF_UNSUPPORTED, "min/max need T::Native: Ord (integers only)");
    if (dtype == kBool) return fail(BDF_UNSUPPORTED, "aggregate of a boolean column");
    bdf_future* fu = nullptr;
    TRY(fleet_aggregate_many(c, 1, &col, &fu));
    bdf_agg4 a;
    TRY(fleet_future_wait(c, fu, &a));
    const int w = dtype_width(dtype);
    if (op == BDF_COUNT) { *(int64_t*)out_scalar = a.count; *is_some = 1; return BDF_OK; }
    if (op == BDF_SUM) { memcpy(out_scalar, &a.sum, (size_t)w); *is_some = 1; return BDF_OK; }
    int panics = 0;
    TRY(fleet_panic_chunks(c, col, &panics));
    if (panics) return fail(BDF_WOULD_PANIC, "max/min on an empty or all-null chunk: the reference unwraps None");
    *is_some = col->fmap.empty() ? 0 : 1;
    if (*is_some) memcpy(out_scalar, op == BDF_MIN ? &a.min : &a.max, (size_t)w);
    return BDF_OK;
}

static int fleet_aggregate_all_blocking(bdf_ctx* c, int32_t n_cols, const bdf_col* const* cols, bdf_agg4* out) {
    bdf_future* fu = nullptr;
    TRY(fleet_aggregate_many(c, n_cols, cols, &fu));
    TRY(fleet_future_wait(c, fu, out));
    for (int32_t j = 0; j < n_cols; j++) {
        int panics = 0;
        TRY(fleet_panic_chunks(c, cols[j], &panics));
        out[j].would_panic = panics != 0;
        out[j].n_chunks = (int64_t)cols[j]->fmap.size();
    }
    return BDF_OK;
}

static int fleet_chunk_info(bdf_ctx* c, const bdf_col* col, int64_t chunk, int64_t* len, int64_t* null_count, int32_t* has_validity);

static int fleet_avg_dev(bdf_ctx* c, const bdf_col* col, double* out, int32_t* is_some) {
    Fleet* f = c->fleet;
    if (!is_fleet_col(col)) return fail(BDF_INVALID, "a column of a one-GPU context was passed to a multi-GPU context");
    std::vector<double> v(f->kids.size(), 0.0);
    std::vector<int32_t> some(f->kids.size(), 0);
    TRY(fleet_run(f, [&](int k) { return bdf_avg_dev(f->kids[k], col->fparts[k], &v[k], &some[k]); }));
    *out = v[0]; *is_some = some[0];
    // aggregate.rs:57-60: `mean + (m - mean) * len / count` is 0/0 when the first chunk has no valid slot, and NaN sticks
    if (!col->fmap.empty()) {
        int64_t len = 0, nulls = 0; int32_t hv = 0;
        TRY(fleet_chunk_info(c, col, 0, &len, &nulls, &hv));
        if (len - (hv ? nulls : 0) == 0) *out = std::numeric_limits<double>::quiet_NaN();
    }
    return BDF_OK;
}

// Every GPU computes the record of its row ranges; the kids of a fleet of several GPUs are the ranks of one communicator, so each
// of them all-gathers the records and merges them in rank order (moments_dev) and returns the same bits.  A fleet of one GPU is the
// one-GPU context's call.
static int fleet_moments_dev(bdf_ctx* c, const bdf_col* col, bdf_moment_rec* out) {
    Fleet* f = c->fleet;
    if (!is_fleet_col(col)) return fail(BDF_INVALID, "a column of a one-GPU context was passed to a multi-GPU context");
    std::vector<bdf_moment_rec> rec(f->kids.size());
    TRY(fleet_run(f, [&](int k) { return bdf_moments_dev(f->kids[k], col->fparts[k], &rec[k]); }));
    *out = rec[0];
    return BDF_OK;
}

// Fused operator + aggregate: every kid runs the one-GPU entry on its parts; the future yields the global records.
static int fleet_with_future(bdf_ctx* c, int out_dtype, std::initializer_list<const bdf_col*> inputs, bool want_col, bdf_col** out, bdf_future** fut,
                             const std::function<int(int, bdf_col**, bdf_future**)>& call) {
    Fleet* f = c->fleet;
    const int nk = (int)f->kids.size();
    int64_t n = 0;
    TRY(fleet_zip(inputs.begin(), inputs.size(), BDF_LENGTH_MISMATCH, BDF_INVALID, &n));
    bdf_col* o = want_col ? fleet_col_like(*inputs.begin(), out_dtype, nk, n) : nullptr;
    bdf_future* fu = fleet_future_new(nk);
    if ((want_col && !o) || !fu) { fleet_col_free(f, o); delete fu; return fail(BDF_OOM, "host allocation failed"); }
    fu->n = 1;
    int st = fleet_run(f, [&](int k) { return call(k, o ? &o->fparts[k] : nullptr, &fu->fparts[k]); });
    if (st != BDF_OK) {
        const std::string keep = g_err;
        fleet_future_wait(c, fu, nullptr);
        fleet_col_free(f, o);
        g_err = keep;
        return st;
    }
    if (out) *out = o;
    *fut = fu;
    return BDF_OK;
}

// Host in / host out over every GPU: shard the views of the inputs (chunk i of every input has the same length) by one plan,
// run the one-GPU drop-in entry per kid on its pieces (its own PCIe link), fold the metadata into `out`.
// `call(kid, pieces, views of every input, outs)`.
template <class F>
static int fleet_host_map(bdf_ctx* c, std::initializer_list<const bdf_view*> inputs, int64_t n, int out_dtype, bdf_out* out, F&& call) {
    Fleet* f = c->fleet;
    const int nk = (int)f->kids.size();
    const size_t ni = inputs.size();
    const bdf_view* first = *inputs.begin();
    std::vector<int64_t> lens((size_t)n);
    for (int64_t i = 0; i < n; i++) {
        for (const bdf_view* in : inputs)
            if (in[i].len != first[i].len) return fail(BDF_LENGTH_MISMATCH, "Cannot perform math operation on arrays of different length");
        for (const bdf_view* in : inputs)
            if (in[i].len < 0 || in[i].offset < 0) return fail(BDF_INVALID, "bad view %lld", (long long)i);
        lens[i] = first[i].len;
    }
    const auto map = fleet_plan(lens, nk);
    std::vector<std::vector<bdf_view>> iv((size_t)nk * ni);   // kid k, input j at k * ni + j
    std::vector<std::vector<bdf_out>> ov((size_t)nk);
    for (int k = 0; k < nk; k++) {
        size_t j = 0;
        for (const bdf_view* in : inputs) iv[k * ni + j++] = fleet_views(map, nk, k, in);
        ov[k] = fleet_outs(map, k, out_dtype, out);
    }
    TRY(fleet_run(f, [&](int k) {
        bdf_view dv{}; bdf_out dummy{};
        std::vector<const bdf_view*> v(ni);
        for (size_t j = 0; j < ni; j++) v[j] = iv[k * ni + j].empty() ? &dv : iv[k * ni + j].data();
        return call(f->kids[k], (int64_t)ov[k].size(), v.data(), ov[k].empty() ? &dummy : ov[k].data());
    }));
    fleet_merge_outs(map, ov, lens, out);
    return BDF_OK;
}

// A reduction of a host column over every GPU: upload the pieces (every GPU its own), run `body(fleet column)`, and wait for the
// uploads before the column goes: host inputs must not be touched after return.
template <class F>
static int fleet_host_reduce(bdf_ctx* c, int dtype, int64_t n, const bdf_view* in, F&& body) {
    bdf_col* col = nullptr;
    const int32_t dt = dtype;
    TRY(fleet_upload_many(c, 1, &dt, &n, &in, BDF_ASYNC, &col));
    const int st = body(col);
    const std::string keep = g_err;
    Fleet* f = c->fleet;
    fleet_run(f, [&](int k) { return bdf_col_wait(f->kids[k], col->fparts[k]); });
    fleet_col_free(f, col);
    g_err = keep;
    return st;
}

static int fleet_generate(bdf_ctx* c, int dtype, int kind, double lo, double hi, uint64_t seed, uint64_t col_id, int64_t n_chunks,
                          const int64_t* chunk_lens, int64_t row0, uint32_t null_mod, bdf_col** out) {
    Fleet* f = c->fleet;
    const int nk = (int)f->kids.size();
    std::vector<int64_t> lens((size_t)n_chunks);
    for (int64_t i = 0; i < n_chunks; i++) { if (chunk_lens[i] < 0) return fail(BDF_INVALID, "negative chunk length"); lens[i] = chunk_lens[i]; }
    bdf_col* col = fleet_col_new(dtype, nk);
    if (!col) return fail(BDF_OOM, "host allocation failed");
    col->fmap = fleet_plan(lens, nk);
    col->flens = lens;
    for (int64_t v : lens) col->total_len += v;
    // a kid's pieces cover one contiguous range of global rows: generate them as one column starting at that row
    std::vector<std::vector<int64_t>> klens((size_t)nk);
    std::vector<int64_t> krow0((size_t)nk, -1);
    int64_t start = 0;
    for (int64_t i = 0; i < n_chunks; i++) {
        for (const auto& pc : col->fmap[i]) {
            if ((int64_t)klens[pc.kid].size() <= pc.local) klens[pc.kid].resize((size_t)pc.local + 1, 0);
            klens[pc.kid][pc.local] = pc.rows;
            if (krow0[pc.kid] < 0 && pc.rows > 0) krow0[pc.kid] = start + pc.row0;
        }
        start += lens[i];
    }
    int st = fleet_run(f, [&](int k) {
        const int64_t dummy = 0;
        return bdf_generate(f->kids[k], dtype, kind, lo, hi, seed, col_id, (int64_t)klens[k].size(), klens[k].empty() ? &dummy : klens[k].data(),
                            row0 + std::max<int64_t>(krow0[k], 0), null_mod, &col->fparts[k]);
    });
    if (st != BDF_OK) { const std::string keep = g_err; fleet_col_free(f, col); g_err = keep; return st; }
    *out = col;
    return BDF_OK;
}

static int fleet_chunk_info(bdf_ctx* c, const bdf_col* col, int64_t chunk, int64_t* len, int64_t* null_count, int32_t* has_validity) {
    Fleet* f = c->fleet;
    if (!is_fleet_col(col) || chunk < 0 || chunk >= (int64_t)col->fmap.size()) return fail(BDF_INVALID, "bad chunk index");
    if (len) *len = col->flens[chunk];
    if (!null_count && !has_validity) return BDF_OK;
    int64_t nulls = 0; int32_t hv = 0;
    for (const auto& pc : col->fmap[chunk]) {   // a handful of pieces: the calling thread asks the kids in turn
        int64_t l = 0, nc = 0; int32_t h = 0;
        TRY(bdf_col_chunk_info(f->kids[pc.kid], col->fparts[pc.kid], pc.local, &l, null_count ? &nc : nullptr, &h));
        nulls += nc; hv |= h;
    }
    if (null_count) *null_count = nulls;
    if (has_validity) *has_validity = hv;
    return BDF_OK;
}

static void fleet_destroy(bdf_ctx* c) {
    Fleet* f = c->fleet;
    for (auto& w : f->workers) {
        { std::lock_guard<std::mutex> g(w->m); w->stop = true; }
        w->cv.notify_all();
        if (w->th.joinable()) w->th.join();
    }
    for (bdf_ctx* k : f->kids) bdf_destroy(k);
    delete f;
    delete c;
}

// ---------------------------------------------------------------------------------------------------
// list columns and ArrayFunctions (k_list.cu).  Contains / position / max / min / size work chunk by chunk on the list's own
// offsets.  The functions that return lists work in the element space of the call (every element of the input lists, counted
// through the chunks): a parent column (the element's global list number, NULL for an element of a null list) and the stable
// lexsort over (parent, value) turn them into the existing sort / take / heads / filter steps, and the result's offsets come from
// the list numbers of the kept elements.  They return one chunk, as take and sort do.

struct bdf_list {
    int dtype = 0;
    bdf_col* values = nullptr;               // chunk i = the elements of list chunk i
    std::vector<int64_t> lens, null_counts;  // lists and null lists per chunk
    std::vector<int64_t> valid_elems;        // elements that belong to a valid list, per chunk
    std::vector<int32_t*> off;               // device: len + 1 offsets from 0
    std::vector<uint32_t*> valid;            // device: the list validity at bit 0, or nullptr
    char* arena = nullptr;                   // the offsets and validity of every chunk
    int64_t total_len = 0;
};

static void list_release(bdf_ctx* c, bdf_list* l) {
    if (!l) return;
    if (l->values) col_release(c, l->values);
    if (l->arena) cudaFreeAsync(l->arena, c->s_compute);
    delete l;
}
static void drop(bdf_ctx* c, bdf_list* l) { list_release(c, l); }
using ListOwner = Owned<bdf_list>;

static constexpr int64_t kListMaxChunkElems = 0x7fffffffLL;    // Int32 offsets
static constexpr int64_t kListMaxCallElems = 0xffffffffLL;     // the sort's UInt32 row numbers

// A list whose offsets (and validity, where has_valid) live in one device arena; the caller fills them and sets `values`.
static int list_alloc(bdf_ctx* c, int dtype, const std::vector<int64_t>& lens, const std::vector<bool>& has_valid, bdf_list** out) {
    ListOwner l(c, new (std::nothrow) bdf_list());
    if (!l.get()) return fail(BDF_OOM, "host allocation failed");
    l->dtype = dtype;
    l->lens = lens;
    const size_t n = lens.size();
    std::vector<size_t> ooff(n), voff(n);
    size_t bytes = 0;
    for (size_t i = 0; i < n; i++) {
        ooff[i] = bytes;
        bytes += align_up((size_t)(lens[i] + 1) * 4, 256);
        voff[i] = bytes;
        if (has_valid[i]) bytes += align_up((size_t)(lens[i] + 31) / 32 * 4 + 8, 256);
        l->total_len += lens[i];
    }
    cudaError_t e = cudaMallocAsync((void**)&l->arena, std::max<size_t>(bytes, 256), c->s_compute);
    if (e != cudaSuccess) { cudaGetLastError(); l->arena = nullptr; return fail(cuda_status(e), "list allocation of %zu bytes failed", bytes); }
    for (size_t i = 0; i < n; i++) {
        l->off.push_back((int32_t*)(l->arena + ooff[i]));
        l->valid.push_back(has_valid[i] ? (uint32_t*)(l->arena + voff[i]) : nullptr);
    }
    l->null_counts.assign(n, 0);
    l->valid_elems.assign(n, 0);
    *out = l.release();
    return BDF_OK;
}

static bool host_bit(const uint8_t* bits, int64_t i) { return (bits[i >> 3] >> (i & 7)) & 1u; }

static int list_upload(bdf_ctx* c, int dtype, int64_t n, const bdf_list_view* in, bool async, bdf_list** out) {
    if (dtype < 0 || dtype >= BDF_NTYPES) return fail(BDF_UNSUPPORTED, "list columns on the device have one of the ten numeric child types");
    std::vector<bdf_view> child((size_t)n);
    std::vector<std::vector<int32_t>> offs((size_t)n);
    std::vector<std::vector<uint32_t>> bits((size_t)n);
    std::vector<int64_t> lens((size_t)n), nulls((size_t)n, 0), valid_elems((size_t)n, 0);
    std::vector<bool> has_valid((size_t)n);
    int64_t total = 0;
    for (int64_t i = 0; i < n; i++) {
        const bdf_list_view& v = in[i];
        if (v.len < 0 || v.offset < 0 || (v.len > 0 && !v.offsets) || v.values.len < 0 || v.values.offset < 0)
            return fail(BDF_INVALID, "bad list view %lld", (long long)i);
        const int32_t* o = v.offsets ? v.offsets + v.offset : nullptr;
        const int64_t first = o ? o[0] : 0, last = o ? o[v.len] : 0;
        if (first < 0 || last > v.values.len) return fail(BDF_INVALID, "list chunk %lld: offsets outside the child array", (long long)i);
        offs[i].resize((size_t)v.len + 1);
        offs[i][0] = 0;
        for (int64_t k = 0; k < v.len; k++) {
            if (o[k + 1] < o[k]) return fail(BDF_INVALID, "list chunk %lld: offsets decrease at %lld", (long long)i, (long long)k);
            offs[i][k + 1] = (int32_t)(o[k + 1] - first);
        }
        if (last - first >= kListMaxChunkElems) return fail(BDF_UNSUPPORTED, "list chunk %lld: 2^31 or more elements", (long long)i);
        lens[i] = v.len;
        has_valid[i] = v.validity != nullptr;
        if (v.validity) bits[i].assign((size_t)(v.len + 31) / 32 + 2, 0u);
        for (int64_t k = 0; k < v.len; k++) {
            const bool ok = !v.validity || host_bit(v.validity, v.offset + k);
            if (v.validity && ok) bits[i][k >> 5] |= 1u << (k & 31);
            if (ok) valid_elems[i] += o[k + 1] - o[k];
            else nulls[i]++;
        }
        child[i] = bdf_view{v.values.values, v.values.validity, last - first, v.values.offset + first,
                            (first == 0 && last == v.values.len) ? v.values.null_count : -1};
        total += last - first;
    }
    if (total >= kListMaxCallElems) return fail(BDF_UNSUPPORTED, "a list call holds 2^32 or more elements (the sort's UInt32 row numbers)");
    ListOwner l(c);
    TRY(list_alloc(c, dtype, lens, has_valid, l.out()));
    l->null_counts = nulls;
    l->valid_elems = valid_elems;
    std::vector<bdf_col*> cols;
    TRY(upload_many(c, {UploadSpec{dtype, n, child.data()}}, async, cols));
    ColOwner values(c, cols[0]);
    bool misaligned = false;
    for (auto& ch : values->chunks) misaligned = misaligned || (ch.validity && ch.bit_off != 0);
    if (misaligned) {   // the fold of max / min reads validity at bit 0
        ColOwner re(c);
        TRY(realign(c, values.get(), re.out()));
        values = std::move(re);
    }
    for (int64_t i = 0; i < n; i++) {
        CK(cudaMemcpyAsync(l->off[i], offs[i].data(), offs[i].size() * 4, cudaMemcpyHostToDevice, c->s_compute));
        if (l->valid[i]) CK(cudaMemcpyAsync(l->valid[i], bits[i].data(), bits[i].size() * 4, cudaMemcpyHostToDevice, c->s_compute));
    }
    CK(cudaStreamSynchronize(c->s_compute));   // the host vectors go out of scope
    l->values = values.release();
    *out = l.release();
    return BDF_OK;
}

static int list_download(bdf_ctx* c, const bdf_list* l, bdf_list_out* out) {
    const int64_t n = (int64_t)l->lens.size();
    std::vector<bdf_out> vo((size_t)std::max<int64_t>(n, 1));
    for (int64_t i = 0; i < n; i++) {
        if (!out[i].offsets) return fail(BDF_INVALID, "list output chunk %lld has no offsets buffer", (long long)i);
        if (l->valid[i] && l->lens[i] && !out[i].validity) return fail(BDF_INVALID, "list output chunk %lld needs a validity buffer", (long long)i);
        vo[i] = bdf_out{out[i].values, out[i].value_validity, l->values->chunks[i].len, 0, 0};
    }
    TRY(download(c, l->values, vo.data()));
    // the offsets and validity are written by kernels on the compute stream (k_list_offsets is the last step of every list-returning
    // function): copy them in that stream's order
    std::vector<uint32_t> words;
    for (int64_t i = 0; i < n; i++) {
        CK(cudaMemcpyAsync(out[i].offsets, l->off[i], (size_t)(l->lens[i] + 1) * 4, cudaMemcpyDeviceToHost, c->s_compute));
        CK(cudaStreamSynchronize(c->s_compute));
        out[i].has_validity = l->valid[i] != nullptr;
        out[i].null_count = l->null_counts[i];
        if (l->valid[i] && l->lens[i]) {
            words.resize((size_t)(l->lens[i] + 31) / 32);
            CK(cudaMemcpyAsync(words.data(), l->valid[i], words.size() * 4, cudaMemcpyDeviceToHost, c->s_compute));
            CK(cudaStreamSynchronize(c->s_compute));
            memcpy(out[i].validity, words.data(), (size_t)bitmap_bytes(l->lens[i]));
        }
        out[i].has_value_validity = vo[i].has_validity;
        out[i].value_null_count = vo[i].null_count;
    }
    return BDF_OK;
}

// A column that borrows device memory owned by other columns (no arenas, no events): views for the sort keys and the concatenated
// children of two lists.  Everything that reads it runs on the compute stream after the owners were produced.
static int col_borrow(int dtype, const std::vector<DevChunk>& chunks, bdf_col** out) {
    bdf_col* col = new (std::nothrow) bdf_col();
    if (!col) return fail(BDF_OOM, "host allocation failed");
    col->dtype = dtype;
    col->chunks = chunks;
    for (auto& ch : chunks) col->total_len += ch.len;
    col->null_counts.assign(chunks.size(), -1);
    col->tile0.assign(chunks.size() + 1, 0);
    *out = col;
    return BDF_OK;
}

// The element space of one call over the children of `parts` in order.  and_valid[k]: a list whose validity also gates part k's
// elements (union: b's elements take part only where a's list is valid), or null.
struct ListElems {
    explicit ListElems(bdf_ctx* c) : parent(c), inlist(c), iota(c), keyed(c), child(c) {}
    ColOwner parent;   // UInt32: the global list number of every element
    ColOwner inlist;   // Boolean: the element belongs to a valid list
    ColOwner iota;     // UInt32: 0 .. n-1
    ColOwner keyed;    // parent with inlist as its validity: the first sort key, elements of null lists sort last
    ColOwner child;    // the children of the parts, chunk after chunk (borrowed)
    int64_t n = 0;
};

static int list_elems(bdf_ctx* c, const std::vector<const bdf_list*>& parts, const std::vector<const bdf_list*>& and_valid, ListElems* x) {
    std::vector<DevChunk> chunks;
    for (const bdf_list* l : parts) {
        wait_groups(c->s_compute, l->values, 0, (int64_t)l->values->chunks.size());
        for (auto& ch : l->values->chunks) chunks.push_back(ch);
        x->n += l->values->total_len;
    }
    const int64_t n = x->n;
    TRY(col_borrow(parts[0]->dtype, chunks, x->child.out()));
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{n, false}}, nullptr, 0, x->parent.out()));
    TRY(col_alloc(c, kBool, {ChunkPlan{n, false}}, nullptr, 0, x->inlist.out()));
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{n, false}}, nullptr, 0, x->iota.out()));
    uint32_t* parent = (uint32_t*)x->parent->chunks[0].values;
    uint32_t* inlist = (uint32_t*)x->inlist->chunks[0].values;
    cudaError_t e = n ? cudaMemsetAsync(inlist, 0, align_up((size_t)bitmap_bytes(n), 4), c->s_compute) : cudaSuccess;
    {
        LaunchTimer t(c, BDF_K_LIST, BDF_U32, n, 4 * n + n / 8);
        int64_t elem0 = 0;
        for (size_t k = 0; k < parts.size() && e == cudaSuccess; k++) {
            const bdf_list* l = parts[k];
            int64_t list0 = 0;
            for (size_t i = 0; i < l->lens.size() && e == cudaSuccess; i++) {
                const int64_t ne = l->values->chunks[i].len;
                e = launch_list_parent(l->off[i], l->valid[i], and_valid[k] ? and_valid[k]->valid[i] : nullptr, l->lens[i], ne, list0, elem0, parent,
                                       inlist, c->s_compute);
                list0 += l->lens[i];
                elem0 += ne;
            }
        }
    }
    c->launches++;
    if (e == cudaSuccess && n) e = launch_iota((uint32_t*)x->iota->chunks[0].values, n, c->sm_count, c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "list parents");
    DevChunk kc = x->parent->chunks[0];
    kc.validity = inlist;
    TRY(col_borrow(BDF_U32, {kc}, x->keyed.out()));
    return BDF_OK;
}

// The one-chunk result list: values = child[rows], offsets from kp (the kept elements' list numbers, ascending), times mult.
static int list_result(bdf_ctx* c, int dtype, const bdf_col* child, const bdf_col* rows, const bdf_col* kp, int64_t n_lists, int64_t mult,
                       bdf_list** out) {
    const int64_t n_kept = kp->total_len;
    if (n_kept * mult >= kListMaxChunkElems) return fail(BDF_UNSUPPORTED, "a list result of 2^31 or more elements (one chunk of Int32 offsets)");
    ListOwner l(c);
    TRY(list_alloc(c, dtype, {n_lists}, {false}, l.out()));
    l->valid_elems[0] = n_kept * mult;
    ColOwner values(c);
    TRY(take_dev(c, child, rows, values.out()));
    cudaError_t e;
    {
        LaunchTimer t(c, BDF_K_LIST, BDF_I32, n_lists, 4 * (n_lists + 1));
        e = launch_list_offsets(n_kept ? (const uint32_t*)kp->chunks[0].values : nullptr, n_kept, n_lists, mult, l->off[0], c->s_compute);
    }
    if (e != cudaSuccess) return fail_cuda(e, "list offsets");
    l->values = values.release();
    *out = l.release();
    return BDF_OK;
}

static int bool_zeroed(bdf_ctx* c, int64_t n, bdf_col** out) {
    ColOwner b(c);
    TRY(col_alloc(c, kBool, {ChunkPlan{n, false}}, nullptr, 0, b.out()));
    if (n) CK(cudaMemsetAsync(b->chunks[0].values, 0, align_up((size_t)bitmap_bytes(n), 4), c->s_compute));
    *out = b.release();
    return BDF_OK;
}

static int list_find(bdf_ctx* c, int fn, const bdf_list* l, uint64_t bits, bdf_col** out) {
    if (fn != BDF_LIST_CONTAINS && fn != BDF_LIST_POSITION) return fail(BDF_INVALID, "unknown list find function %d", fn);
    const bool contains = fn == BDF_LIST_CONTAINS;
    const size_t n = l->lens.size();
    std::vector<ChunkPlan> plan(n);
    int64_t max_elems = 0, rows = 0;
    for (size_t i = 0; i < n; i++) {
        plan[i] = {l->lens[i], contains && l->valid[i] != nullptr};
        max_elems = std::max(max_elems, l->values->chunks[i].len);
        rows += l->values->chunks[i].len;
    }
    ColOwner o(c);
    TRY(col_alloc(c, contains ? kBool : BDF_I32, plan, nullptr, 0, o.out()));
    Scratch<void> scratch;
    CK(scratch.alloc(c, list_find_scratch_bytes(max_elems)));
    wait_groups(c->s_compute, l->values, 0, (int64_t)n);
    cudaError_t e = cudaSuccess;
    {
        const int64_t w = dtype_width(l->dtype);
        LaunchTimer t(c, BDF_K_LIST, contains ? kBool : BDF_I32, rows, rows * w + 4 * (l->total_len + (int64_t)n) + (contains ? l->total_len / 4 : 4 * l->total_len));
        for (size_t i = 0; i < n && e == cudaSuccess; i++) {
            const DevChunk& ch = l->values->chunks[i];
            DevChunk& oc = o->chunks[i];
            if (contains && l->lens[i]) {
                e = cudaMemsetAsync(oc.values, 0, align_up((size_t)bitmap_bytes(l->lens[i]), 4), c->s_compute);
                if (e == cudaSuccess && oc.validity)
                    e = cudaMemcpyAsync(oc.validity, l->valid[i], (size_t)bitmap_bytes(l->lens[i]), cudaMemcpyDeviceToDevice, c->s_compute);
            }
            if (e == cudaSuccess)
                e = launch_list_find(l->dtype, l->off[i], l->valid[i], l->lens[i], ch.len, ch.values, ch.validity, ch.bit_off, bits, contains ? 0 : 1,
                                     (uint32_t*)oc.values, (int32_t*)oc.values, scratch, c->sm_count, c->s_compute);
            o->null_counts[i] = oc.validity ? l->null_counts[i] : 0;
        }
    }
    if (e == cudaSuccess) e = finish_single_group(c, o.get());
    if (e != cudaSuccess) return fail_cuda(e, "list find");
    *out = o.release();
    return BDF_OK;
}

static int list_reduce(bdf_ctx* c, int fn, const bdf_list* l, bdf_col** out) {
    if (fn < BDF_LIST_MAX || fn > BDF_LIST_SIZE) return fail(BDF_INVALID, "unknown list reduce function %d", fn);
    const size_t n = l->lens.size();
    const bool size = fn == BDF_LIST_SIZE;
    std::vector<ChunkPlan> plan(n);
    int64_t max_len = 0, max_elems = 0, rows = 0;
    for (size_t i = 0; i < n; i++) {
        plan[i] = {l->lens[i], !size};
        max_len = std::max(max_len, l->lens[i]);
        max_elems = std::max(max_elems, l->values->chunks[i].len);
        rows += l->values->chunks[i].len;
    }
    const int dt = size ? BDF_I32 : l->dtype;
    ColOwner o(c);
    TRY(col_alloc(c, dt, plan, nullptr, 0, o.out()));
    wait_groups(c->s_compute, l->values, 0, (int64_t)n);
    cudaError_t e = cudaSuccess;
    if (size) {
        LaunchTimer t(c, BDF_K_LIST, BDF_I32, l->total_len, 8 * l->total_len);
        for (size_t i = 0; i < n && e == cudaSuccess; i++) e = launch_list_size(l->off[i], l->valid[i], l->lens[i], (int32_t*)o->chunks[i].values, c->s_compute);
    } else {
        // the group-by fold with the offsets as group starts: sum / count / the other extreme are scratch
        const int w = dtype_width(l->dtype);
        Scratch<char> sum, other, big;
        Scratch<long long> count;
        Scratch<uint32_t> nonempty;
        e = sum.alloc(c, (size_t)std::max<int64_t>(max_len, 1) * 8);
        if (e == cudaSuccess) e = other.alloc(c, (size_t)std::max<int64_t>(max_len, 1) * w);
        if (e == cudaSuccess) e = count.alloc(c, (size_t)std::max<int64_t>(max_len, 1) * 8);
        if (e == cudaSuccess) e = nonempty.alloc(c, ((size_t)max_len + 31) / 32 * 4 + 8);
        if (e == cudaSuccess) e = big.alloc(c, group_big_scratch_bytes(max_elems));
        if (e == cudaSuccess) e = cudaMemsetAsync(c->d_flag, 0, sizeof(int), c->s_compute);
        {
            LaunchTimer t(c, BDF_K_LIST, dt, rows, rows * w + 4 * (l->total_len + (int64_t)n) + l->total_len * w + l->total_len / 8);
            for (size_t i = 0; i < n && e == cudaSuccess; i++) {
                const DevChunk& ch = l->values->chunks[i];
                DevChunk& oc = o->chunks[i];
                const int64_t len = l->lens[i];
                if (!len) continue;
                e = cudaMemsetAsync(nonempty, 0, ((size_t)len + 31) / 32 * 4, c->s_compute);
                void* mn = fn == BDF_LIST_MIN ? oc.values : (void*)other.get();
                void* mx = fn == BDF_LIST_MAX ? oc.values : (void*)other.get();
                c->launches += 3;
                if (e == cudaSuccess)
                    e = launch_group_reduce(l->dtype, true, ch.values, ch.validity, (const uint32_t*)l->off[i], len, ch.len, sum, count, mn, mx, nullptr, nonempty,
                                            big, c->sm_count, c->s_compute);
                if (e == cudaSuccess) e = launch_list_minmax_valid(l->off[i], l->valid[i], nonempty, len, oc.validity, c->d_flag, c->s_compute);
                o->null_counts[i] = -1;
            }
        }
        int flag = 0;
        if (e == cudaSuccess) e = flag_read(c, false, &flag);
        if (e == cudaSuccess && flag) return fail(BDF_WOULD_PANIC, "array_max / array_min of an empty list: the reference's .max().unwrap() panics");
    }
    if (e == cudaSuccess) e = finish_single_group(c, o.get());
    if (e != cudaSuccess) return fail_cuda(e, "list reduce");
    *out = o.release();
    return BDF_OK;
}

// Keep the elements whose bit is set in `keep` (element space of x), in element order.
static int list_keep(bdf_ctx* c, const ListElems& x, const bdf_col* keep, int dtype, int64_t n_lists, bdf_list** out) {
    ColOwner rows(c), kp(c);
    TRY(filter_dev(c, x.iota.get(), keep, rows.out()));
    TRY(filter_dev(c, x.parent.get(), keep, kp.out()));
    return list_result(c, dtype, x.child.get(), rows.get(), kp.get(), n_lists, 1, out);
}

// The stable (list, value) sort of the element space, its group heads, and the keep bits `mode` of k_list_mark sets from them.
static int list_mark(bdf_ctx* c, const ListElems& x, int64_t split, int mode, bdf_col** keep) {
    const bdf_sort_key keys[2] = {{x.keyed.get(), 0}, {x.child.get(), 0}};
    ColOwner perm(c), sp(c), sv(c), head(c), k(c);
    TRY(sort_indices_dev(c, 2, keys, perm.out()));
    TRY(take_dev(c, x.keyed.get(), perm.get(), sp.out()));
    TRY(take_dev(c, x.child.get(), perm.get(), sv.out()));
    TRY(group_heads(c, {sv.get(), sp.get()}, false, x.n, head.out()));
    TRY(bool_zeroed(c, x.n, k.out()));
    cudaError_t e;
    {
        LaunchTimer t(c, BDF_K_LIST, kBool, x.n, 4 * x.n + x.n / 4);
        e = launch_list_mark((const uint32_t*)perm->chunks[0].values, (const uint32_t*)head->chunks[0].values, sp->chunks[0].validity, x.n, split, mode,
                             (uint32_t*)k->chunks[0].values, c->s_compute);
    }
    if (e != cudaSuccess) return fail_cuda(e, "list mark");
    *keep = k.release();
    return BDF_OK;
}

static int list_transform(bdf_ctx* c, int fn, const bdf_list* l, uint64_t bits, int64_t count, bdf_list** out) {
    if (fn < BDF_LIST_REMOVE || fn > BDF_LIST_REPEAT) return fail(BDF_INVALID, "unknown list transform function %d", fn);
    if (fn == BDF_LIST_REPEAT && count < 0) return fail(BDF_INVALID, "array_repeat: count %lld < 0", (long long)count);
    ListElems x(c);
    TRY(list_elems(c, {l}, {nullptr}, &x));
    const int64_t N = l->total_len;
    if (fn == BDF_LIST_REMOVE) {
        ColOwner keep(c);
        TRY(bool_zeroed(c, x.n, keep.out()));
        cudaError_t e = cudaSuccess;
        {
            LaunchTimer t(c, BDF_K_LIST, kBool, x.n, x.n * dtype_width(l->dtype) + x.n / 4);
            int64_t elem0 = 0;
            for (size_t i = 0; i < l->lens.size() && e == cudaSuccess; i++) {
                const DevChunk& ch = l->values->chunks[i];
                e = launch_list_remove_mask(l->dtype, ch.values, ch.validity, ch.bit_off, ch.len, elem0, bits, (const uint32_t*)x.inlist->chunks[0].values,
                                            (uint32_t*)keep->chunks[0].values, c->s_compute);
                elem0 += ch.len;
            }
        }
        if (e != cudaSuccess) return fail_cuda(e, "array_remove");
        return list_keep(c, x, keep.get(), l->dtype, N, out);
    }
    if (fn == BDF_LIST_DISTINCT) {
        ColOwner keep(c);
        TRY(list_mark(c, x, 0, 0, keep.out()));
        return list_keep(c, x, keep.get(), l->dtype, N, out);
    }
    if (fn == BDF_LIST_SORT) {
        // elements of null lists have a null first key and sort after all others: the first K sorted rows are the result
        int64_t K = 0;
        for (int64_t v : l->valid_elems) K += v;
        const bdf_sort_key keys[2] = {{x.keyed.get(), 0}, {x.child.get(), 0}};
        ColOwner perm(c), head(c), kp(c);
        TRY(sort_indices_dev(c, 2, keys, perm.out()));
        DevChunk pc = perm->chunks[0];
        pc.len = K;
        TRY(col_borrow(BDF_U32, {pc}, head.out()));
        TRY(take_dev(c, x.parent.get(), head.get(), kp.out()));
        return list_result(c, l->dtype, x.child.get(), head.get(), kp.get(), N, 1, out);
    }
    // REPEAT
    ColOwner rows(c), kp(c), src(c);
    TRY(filter_dev(c, x.iota.get(), x.inlist.get(), rows.out()));
    TRY(filter_dev(c, x.parent.get(), x.inlist.get(), kp.out()));
    const int64_t K = rows->total_len;
    if (K > 0 && count >= kListMaxChunkElems / K)
        return fail(BDF_UNSUPPORTED, "array_repeat: a result of 2^31 or more elements (one chunk of Int32 offsets)");
    const int64_t n_out = K * count;
    Scratch<int32_t> base;
    CK(base.alloc(c, (size_t)(N + 1) * 4));
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{n_out, false}}, nullptr, 0, src.out()));
    cudaError_t e;
    {
        LaunchTimer t(c, BDF_K_LIST, BDF_U32, n_out, 8 * n_out + 8 * (N + 1));
        e = launch_list_offsets(K ? (const uint32_t*)kp->chunks[0].values : nullptr, K, N, 1, base, c->s_compute);
        if (e == cudaSuccess)
            e = launch_list_repeat(base, N, count, K ? (const uint32_t*)rows->chunks[0].values : nullptr, n_out, (uint32_t*)src->chunks[0].values, c->s_compute);
    }
    if (e == cudaSuccess) e = finish_single_group(c, src.get());
    if (e != cudaSuccess) return fail_cuda(e, "array_repeat");
    // the offsets of the result are count x those of the kept elements
    return list_result(c, l->dtype, x.child.get(), src.get(), kp.get(), N, count, out);
}

static int list_same_shape(const bdf_list* a, const bdf_list* b) {
    if (a->dtype != b->dtype) return fail(BDF_UNSUPPORTED, "the two lists have different element types");
    if (a->lens.size() != b->lens.size()) return fail(BDF_LENGTH_MISMATCH, "Expected array a and b to have the same length");
    for (size_t i = 0; i < a->lens.size(); i++)
        if (a->lens[i] != b->lens[i]) return fail(BDF_LENGTH_MISMATCH, "Expected array a and b to have the same length");
    return BDF_OK;
}

static int list_set(bdf_ctx* c, int fn, const bdf_list* a, const bdf_list* b, bdf_list** out) {
    if (fn < BDF_LIST_EXCEPT || fn > BDF_LIST_UNION) return fail(BDF_INVALID, "unknown list set function %d", fn);
    TRY(list_same_shape(a, b));
    if (a->values->total_len + b->values->total_len >= kListMaxCallElems)
        return fail(BDF_UNSUPPORTED, "a list call holds 2^32 or more elements (the sort's UInt32 row numbers)");
    ListElems x(c);
    ColOwner keep(c);
    if (fn == BDF_LIST_UNION) {   // a then b: a group's head is its first appearance in a ++ b
        TRY(list_elems(c, {a, b}, {nullptr, a}, &x));
        TRY(list_mark(c, x, 0, 0, keep.out()));
        // kept elements in element order are a's, then b's: a stable sort by list number puts every list's a part before its b part
        ColOwner rows(c), kp(c), q(c), rows2(c), kp2(c);
        TRY(filter_dev(c, x.iota.get(), keep.get(), rows.out()));
        TRY(filter_dev(c, x.parent.get(), keep.get(), kp.out()));
        const bdf_sort_key key{kp.get(), 0};
        TRY(sort_indices_dev(c, 1, &key, q.out()));
        TRY(take_dev(c, rows.get(), q.get(), rows2.out()));
        TRY(take_dev(c, kp.get(), q.get(), kp2.out()));
        return list_result(c, a->dtype, x.child.get(), rows2.get(), kp2.get(), a->total_len, 1, out);
    }
    // b then a: a group is [b elements][a elements], so its first a element tells whether b has the value
    TRY(list_elems(c, {b, a}, {nullptr, nullptr}, &x));
    TRY(list_mark(c, x, b->values->total_len, fn == BDF_LIST_EXCEPT ? 1 : 2, keep.out()));
    return list_keep(c, x, keep.get(), a->dtype, a->total_len, out);
}

static int list_explode(bdf_ctx* c, const bdf_list* l, bdf_col** rows_out, bdf_col** values_out) {
    ListElems x(c);
    TRY(list_elems(c, {l}, {nullptr}, &x));
    ColOwner rows(c), pos(c), values(c);
    TRY(filter_dev(c, x.parent.get(), x.inlist.get(), rows.out()));
    TRY(filter_dev(c, x.iota.get(), x.inlist.get(), pos.out()));
    TRY(take_dev(c, x.child.get(), pos.get(), values.out()));
    *rows_out = rows.release();
    *values_out = values.release();
    return BDF_OK;
}

// Take / filter of whole lists: output list i is source list rows[i].  local (filter): rows chunk k holds rows of list chunk k and
// becomes output chunk k; otherwise rows count through the chunks and the result is one chunk.  A null row or a null list gives a
// null list of no element; only the elements of valid lists are copied.
static int list_gather(bdf_ctx* c, const bdf_list* l, const bdf_col* rows, bool local, bdf_list** out) {
    const int64_t n = rows->total_len, n_lc = (int64_t)l->lens.size();
    const size_t n_out = local ? rows->chunks.size() : 1;
    std::vector<int64_t> out_lens;
    if (local) for (const DevChunk& ch : rows->chunks) out_lens.push_back(ch.len);
    else out_lens.push_back(n);
    ListOwner res(c);
    TRY(list_alloc(c, l->dtype, out_lens, std::vector<bool>(n_out, true), res.out()));
    // the list chunk table and the output validity pointers, uploaded together
    std::vector<ListChunkDesc> lt((size_t)std::max<int64_t>(n_lc, 1), ListChunkDesc{nullptr, nullptr, 0, 0});
    int64_t start = 0, elem0 = 0;
    for (int64_t i = 0; i < n_lc; i++) {
        lt[i] = ListChunkDesc{l->off[i], l->valid[i], (long long)start, (long long)elem0};
        start += l->lens[i];
        elem0 += l->values->chunks[i].len;
    }
    void* it = nullptr;
    int ni = 0;
    TRY(sort_table(c, rows, &it, &ni, nullptr));
    wait_groups(c->s_compute, l->values, 0, n_lc);
    Scratch<char> tables;
    Scratch<unsigned long long> sizes, scan_sums, nulls;
    Scratch<uint32_t> first;
    const size_t lt_bytes = lt.size() * sizeof(ListChunkDesc);
    CK(tables.alloc(c, lt_bytes + n_out * sizeof(uint32_t*)));
    CK(sizes.alloc(c, (size_t)(n + 1) * 8));
    CK(scan_sums.alloc(c, (size_t)scan_tile_sums(n) * 8));
    CK(nulls.alloc(c, n_out * 8));
    CK(first.alloc(c, (size_t)std::max<int64_t>(n, 1) * 4));
    std::vector<char> host(lt_bytes + n_out * sizeof(uint32_t*));
    memcpy(host.data(), lt.data(), lt_bytes);
    memcpy(host.data() + lt_bytes, res->valid.data(), n_out * sizeof(uint32_t*));
    CK(cudaMemcpyAsync(tables.get(), host.data(), host.size(), cudaMemcpyHostToDevice, c->s_compute));
    CK(cudaMemsetAsync(nulls, 0, n_out * 8, c->s_compute));
    for (size_t k = 0; k < n_out; k++)
        if (out_lens[k]) CK(cudaMemsetAsync(res->valid[k], 0, align_up((size_t)bitmap_bytes(out_lens[k]), 4), c->s_compute));
    CK(cudaMemsetAsync(c->d_flag, 0, sizeof(int), c->s_compute));
    cudaError_t e;
    {
        LaunchTimer t(c, BDF_K_LIST, BDF_U64, n, n * (4 + 8 + 8 + 4) + n / 8);   // index, two offsets, size and first element
        c->launches += kScanLaunches;   // the timer counts the sizes
        e = launch_list_take_sizes(it, ni, n, tables.get(), (int)std::max<int64_t>(n_lc, 1), l->total_len, local ? 1 : 0,
                                   (uint32_t* const*)(tables.get() + lt_bytes), sizes, first, nulls, c->d_flag, c->s_compute);
        if (e == cudaSuccess) e = launch_scan(sizes, n, scan_sums, c->s_compute);
    }
    // the host needs the element count of every output chunk (scan entries at the chunk bounds), the null counts and the flag
    std::vector<unsigned long long> bounds(n_out + 1), h_nulls(n_out);
    int64_t p = 0;
    for (size_t k = 0; k <= n_out && e == cudaSuccess; k++) {
        e = cudaMemcpyAsync(&bounds[k], sizes + p, 8, cudaMemcpyDeviceToHost, c->s_compute);
        if (k < n_out) p += out_lens[k];
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(h_nulls.data(), nulls, n_out * 8, cudaMemcpyDeviceToHost, c->s_compute);
    int flag = 0;
    if (e == cudaSuccess) e = flag_read(c, false, &flag);   // synchronises the compute stream
    if (e != cudaSuccess) return fail_cuda(e, "list take (sizes)");
    if (flag) return fail(BDF_INVALID, "take: index out of bounds");
    const int64_t n_elem = (int64_t)bounds[n_out];
    if (n_elem > kListMaxChunkElems) return fail(BDF_UNSUPPORTED, "a list result of 2^31 or more elements (Int32 offsets)");
    ColOwner src(c), src_view(c), values(c);
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{n_elem, false}}, nullptr, 0, src.out()));
    {
        LaunchTimer t(c, BDF_K_LIST, BDF_U32, n_elem, n_elem * 4 + 4 * (int64_t)n_out + 4 * (n + (int64_t)n_out));
        e = launch_list_take_rows(sizes, n, first, n_elem, (uint32_t*)src->chunks[0].values, c->s_compute);
        p = 0;
        for (size_t k = 0; k < n_out && e == cudaSuccess; k++) {
            e = launch_list_rebase(sizes + p, out_lens[k], res->off[k], c->s_compute);
            p += out_lens[k];
        }
    }
    if (e == cudaSuccess) e = finish_single_group(c, src.get());
    if (e != cudaSuccess) return fail_cuda(e, "list take (rows)");
    if (local) {   // one view of src per output chunk: the element gather keeps the chunks
        std::vector<DevChunk> views(n_out);
        for (size_t k = 0; k < n_out; k++)
            views[k] = DevChunk{src->chunks[0].values + 4 * bounds[k], nullptr, (int64_t)(bounds[k + 1] - bounds[k]), 0, 0};
        TRY(col_borrow(BDF_U32, views, src_view.out()));
    }
    TRY(take_dev(c, l->values, local ? src_view.get() : src.get(), values.out(), local));
    for (size_t k = 0; k < n_out; k++) {
        res->null_counts[k] = (int64_t)h_nulls[k];
        res->valid_elems[k] = (int64_t)(bounds[k + 1] - bounds[k]);
        if (!h_nulls[k]) res->valid[k] = nullptr;   // every list is valid: no bitmap (its bytes stay in the arena)
    }
    res->values = values.release();
    *out = res.release();
    return BDF_OK;
}

static int list_take(bdf_ctx* c, const bdf_list* l, const bdf_col* indices, bdf_list** out) {
    if (indices->dtype != BDF_U32) return fail(BDF_UNSUPPORTED, "take indices must be a UInt32 column");
    return list_gather(c, l, indices, false, out);
}

// collect_list: the valid values of x in sorted-row order (row order inside a group: the sort is stable).  collect_set: the heads
// of the distinct runs of dr (the first occurrence in row order of every distinct valid value, ascending inside a group).  Either
// way the groups keep their sorted row ranges, so list g starts at the rank of the group's first sorted row among the kept rows.
static int group_collect(bdf_ctx* c, const SortedRuns& runs, const bdf_col* x, int fn, const DistinctRuns* dr, bdf_list** out) {
    const int64_t n = runs.perm->total_len, n_groups = runs.n_runs;
    ColOwner sval(c), valid(c), vals(c), kept(c);
    const bdf_col* kv = nullptr;   // the kept values in sorted order
    const bdf_col* kr = nullptr;   // their sorted rows
    if (fn == BDF_GROUP_COLLECT_SET) {
        TRY(filter_dev(c, dr->sval.get(), dr->dhead.get(), vals.out()));
        kv = vals.get();
        kr = dr->pos.get();
    } else {
        TRY(take_dev(c, x, runs.perm.get(), sval.out()));
        if (sval->chunks[0].validity) {   // the validity of x in sorted order is the mask of the kept rows
            TRY(col_borrow(kBool, {DevChunk{(char*)sval->chunks[0].validity, nullptr, n, 0, 0}}, valid.out()));
            TRY(filter_dev(c, sval.get(), valid.get(), vals.out()));
            TRY(filter_dev(c, runs.iota.get(), valid.get(), kept.out()));
            kv = vals.get();
            kr = kept.get();
        } else {
            kv = sval.get();
            kr = runs.iota.get();
        }
    }
    const int64_t n_elem = kv->total_len;
    if (n_elem > kListMaxChunkElems) return fail(BDF_UNSUPPORTED, "a list result of 2^31 or more elements (Int32 offsets)");
    ListOwner l(c);
    TRY(list_alloc(c, x->dtype, {n_groups}, {false}, l.out()));
    wait_groups(c->s_compute, kr, 0, 1);
    wait_groups(c->s_compute, runs.starts.get(), 0, 1);
    cudaError_t e;
    {
        LaunchTimer t(c, BDF_K_LIST, BDF_I32, n_groups, n_groups * 8 + 4);
        e = launch_list_ranks(n_elem ? (const uint32_t*)kr->chunks[0].values : nullptr, n_elem, (const uint32_t*)runs.starts->chunks[0].values, n_groups,
                              l->off[0], c->s_compute);
    }
    if (e != cudaSuccess) return fail_cuda(e, "collect offsets");
    l->valid_elems[0] = n_elem;
    l->values = kv == sval.get() ? sval.release() : vals.release();
    *out = l.release();
    return BDF_OK;
}

// The kept row numbers of every list chunk (a filter of 0 .. len-1 per chunk), then the gather with the chunks kept.
static int list_filter(bdf_ctx* c, const bdf_list* l, const bdf_col* mask, bdf_list** out) {
    if (mask->dtype != kBool) return fail(BDF_INVALID, "the filter mask must be a boolean column");
    if (mask->chunks.size() != l->lens.size()) return fail(BDF_LENGTH_MISMATCH, "Filter array must have the same length as the data");
    int64_t max_len = 0;
    for (size_t i = 0; i < l->lens.size(); i++) {
        if (mask->chunks[i].len != l->lens[i]) return fail(BDF_LENGTH_MISMATCH, "Filter array must have the same length as the data");
        max_len = std::max(max_len, l->lens[i]);
    }
    ColOwner iota(c), rows_of(c), kept(c);
    TRY(col_alloc(c, BDF_U32, {ChunkPlan{max_len, false}}, nullptr, 0, iota.out()));
    c->launches++;
    cudaError_t e = max_len ? launch_iota((uint32_t*)iota->chunks[0].values, max_len, c->sm_count, c->s_compute) : cudaSuccess;
    if (e != cudaSuccess) return fail_cuda(e, "list filter rows");
    std::vector<DevChunk> views;
    for (int64_t len : l->lens) views.push_back(DevChunk{iota->chunks[0].values, nullptr, len, 0, 0});
    TRY(col_borrow(BDF_U32, views, rows_of.out()));
    TRY(filter_dev(c, rows_of.get(), mask, kept.out()));
    return list_gather(c, l, kept.get(), true, out);
}

// The lists of ls[0], then those of ls[1], ...: offsets and list validity copied device to device, the elements concatenated with
// concat_dev (chunk i of the elements stays the elements of list chunk i).
static int list_concat(bdf_ctx* c, int n, const bdf_list* const* ls, bdf_list** out) {
    if (n < 1) return fail(BDF_INVALID, "concat takes at least one list column");
    if (!ls || !out) return fail(BDF_INVALID, "null argument");
    for (int k = 0; k < n; k++)
        if (!ls[k]) return fail(BDF_INVALID, "null list column");
    for (int k = 0; k < n; k++)
        if (ls[k]->dtype != ls[0]->dtype) return fail(BDF_UNSUPPORTED, "concatenated list columns must have the same child dtype");
    std::vector<int64_t> lens, nulls, valid_elems;
    std::vector<bool> has_valid;
    std::vector<const bdf_col*> values;
    for (int k = 0; k < n; k++) {
        const bdf_list* l = ls[k];
        lens.insert(lens.end(), l->lens.begin(), l->lens.end());
        nulls.insert(nulls.end(), l->null_counts.begin(), l->null_counts.end());
        valid_elems.insert(valid_elems.end(), l->valid_elems.begin(), l->valid_elems.end());
        for (uint32_t* v : l->valid) has_valid.push_back(v != nullptr);
        values.push_back(l->values);
    }
    int64_t elems = 0;
    for (int k = 0; k < n; k++) elems += ls[k]->values->total_len;
    if (elems >= kListMaxCallElems) return fail(BDF_UNSUPPORTED, "a list call holds 2^32 or more elements (the sort's UInt32 row numbers)");
    ListOwner o(c);
    TRY(list_alloc(c, ls[0]->dtype, lens, has_valid, o.out()));
    TRY(concat_dev(c, n, values.data(), &o->values));   // waits for every input's elements, whose groups cover the offsets too
    cudaError_t e = cudaSuccess;
    size_t j = 0;
    for (int k = 0; k < n && e == cudaSuccess; k++)
        for (size_t i = 0; i < ls[k]->lens.size() && e == cudaSuccess; i++, j++) {
            const int64_t len = ls[k]->lens[i];
            e = cudaMemcpyAsync(o->off[j], ls[k]->off[i], (size_t)(len + 1) * 4, cudaMemcpyDeviceToDevice, c->s_compute);
            if (e == cudaSuccess && ls[k]->valid[i] && len)
                e = cudaMemcpyAsync(o->valid[j], ls[k]->valid[i], (size_t)(len + 31) / 32 * 4, cudaMemcpyDeviceToDevice, c->s_compute);
        }
    if (e != cudaSuccess) return fail_cuda(e, "list concat");
    o->null_counts = nulls;
    o->valid_elems = valid_elems;
    *out = o.release();
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// line-delimited JSON reader (k_json.cu; the rules are in include/b200df.h): the file goes to HBM as for the CSV reader; the lines
// are found, checked and walked on the device, which lists every member of every record's object.  The host decodes the distinct
// keys into the dictionary and applies the inference's coercion table; the members and the (record, column) slots stay on the
// device until bdf_json_close, and a read converts only the requested columns.

struct bdf_json : MappedText {
    void* d_members = nullptr;          // JsonMember per member of every record, in file order
    unsigned int* d_slots = nullptr;    // [record][column]: 1 + the member that gives the value, 0 for none
    int64_t n_members = 0, n_rows = 0, batch = 1024;
    std::vector<std::string> names;
    std::vector<int32_t> dtypes, nullable;
    mutable int64_t exact_fields = 0;
};

static void json_free(bdf_ctx* c, bdf_json* f) {
    if (!f) return;
    if (f->d_members) cudaFreeAsync(f->d_members, c->s_compute);
    if (f->d_slots) cudaFreeAsync(f->d_slots, c->s_compute);
    text_free(c, f);
    delete f;
}
static void drop(bdf_ctx* c, bdf_json* f) { json_free(c, f); }

static constexpr unsigned kJsonKeyCap = 1u << 16;   // distinct raw keys per file

struct JsonKeyH { unsigned long long hash, first, kstart; uint32_t klen, rec; };    // k_json.cu's JsonKey
struct JsonSlowH { long long start, end; int col, pad; long long chunk, row; };    // k_json.cu's JsonSlow

static void put_utf8(std::string& out, uint32_t cp) {
    if (cp < 0x80) out += (char)cp;
    else if (cp < 0x800) { out += (char)(0xC0 | cp >> 6); out += (char)(0x80 | (cp & 0x3F)); }
    else if (cp < 0x10000) { out += (char)(0xE0 | cp >> 12); out += (char)(0x80 | ((cp >> 6) & 0x3F)); out += (char)(0x80 | (cp & 0x3F)); }
    else { out += (char)(0xF0 | cp >> 18); out += (char)(0x80 | ((cp >> 12) & 0x3F)); out += (char)(0x80 | ((cp >> 6) & 0x3F)); out += (char)(0x80 | (cp & 0x3F)); }
}

// The key a string's raw bytes [s, e) (between the quotes, already checked) stand for: escapes decoded, \uXXXX pairs of surrogates
// joined, and a lone surrogate as U+FFFD.
static std::string json_unescape(const uint8_t* s, const uint8_t* e) {
    std::string out;
    auto hex4 = [](const uint8_t* p) { uint32_t v = 0; for (int k = 0; k < 4; k++) { const int c = p[k]; v = v * 16 + (uint32_t)(c <= '9' ? c - '0' : (c | 32) - 'a' + 10); } return v; };
    while (s < e) {
        if (*s != '\\') { out += (char)*s++; continue; }
        const uint8_t x = s[1];
        s += 2;
        switch (x) {
            case 'b': out += '\b'; break;
            case 'f': out += '\f'; break;
            case 'n': out += '\n'; break;
            case 'r': out += '\r'; break;
            case 't': out += '\t'; break;
            case 'u': {
                uint32_t cp = hex4(s);
                s += 4;
                if (cp >= 0xD800 && cp < 0xDC00 && e - s >= 6 && s[0] == '\\' && s[1] == 'u') {
                    const uint32_t lo = hex4(s + 2);
                    if (lo >= 0xDC00 && lo < 0xE000) { cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00); s += 6; }
                }
                put_utf8(out, cp >= 0xD800 && cp < 0xE000 ? 0xFFFD : cp);
                break;
            }
            default: out += (char)x; break;   // " \ /
        }
    }
    return out;
}

struct JsonNoMembers {
    void member(const uint8_t*, const uint8_t*, const uint8_t*, const uint8_t*, int, bool) {}
};

// Line `line` (from 0) is malformed: walk it on the host with the device's rules to say where and why.
static int json_bad_line(bdf_ctx* c, const bdf_json* f, const unsigned long long* d_nl, int64_t n_nl, int64_t line) {
    unsigned long long b[2] = {0, 0};
    if (line > 0) CK(cudaMemcpyAsync(&b[0], d_nl + line - 1, 8, cudaMemcpyDeviceToHost, c->s_compute));
    if (line < n_nl) CK(cudaMemcpyAsync(&b[1], d_nl + line, 8, cudaMemcpyDeviceToHost, c->s_compute));
    CK(cudaStreamSynchronize(c->s_compute));
    const uint8_t* text = f->map + f->off;
    const int64_t s = line > 0 ? (int64_t)b[0] + 1 : 0, e = line < n_nl ? (int64_t)b[1] : f->n;
    json::Cursor cur{text + s, text + e, 0, nullptr};
    JsonNoMembers v;
    json::record(cur, v);
    static const char* const what[] = {"malformed record", "the record is not an object", "expected a key (a string)", "expected ':'",
                                       "expected a value", "expected ',' or a closing bracket", "unterminated string", "invalid escape",
                                       "control character in a string", "invalid number", "invalid literal", "trailing characters after the object",
                                       "nesting deeper than 128 levels"};
    const int code = cur.err >= 0 && cur.err <= json::eDepth ? cur.err : 0;
    const long long byte = (long long)f->off + (long long)((cur.at ? cur.at : text + s) - text);
    return fail(BDF_INVALID, "JSON error at line %lld, byte %lld: %s", (long long)line + 1, byte, what[code]);
}

// The coercion table over the class bits of one column (json_parse.cuh): its dtype, or -1 off the device path.
static int json_coerce(unsigned bits) {
    const unsigned t = bits & ~(unsigned)(json::kNull | json::kMissing);
    if (t & (json::kStr | json::kObj | json::kListOther)) return -1;
    if (t & json::kBool) return t == json::kBool ? kBool : -1;
    const bool list = (t & (json::kListInt | json::kListFloat | json::kListEmpty)) != 0;
    const bool fl = (t & (json::kFloat | json::kListFloat)) != 0, in = (t & (json::kInt | json::kListInt)) != 0;
    if (!fl && !in) return -1;   // only nulls, or lists that never had a typed element
    const int scalar = fl ? BDF_F64 : BDF_I64;
    return list ? BDF_LIST_BASE + scalar : scalar;
}

static bool json_dtype_ok(int t) {
    return (t >= 0 && t <= kBool) || (t >= BDF_LIST_BASE && t < BDF_LIST_BASE + BDF_NTYPES) || t == BDF_UTF8 || t == -1;
}

static int json_open(bdf_ctx* c, const char* path, const bdf_json_options* o, int n_schema, const char* const* schema_names, const int32_t* schema,
                     bdf_json** out) {
    if (!path || !o || !out) return fail(BDF_INVALID, "null argument");
    if (o->batch_size < 1) return fail(BDF_INVALID, "batch_size must be at least 1");
    if (schema || schema_names) {
        if (!schema || !schema_names || n_schema < 1) return fail(BDF_INVALID, "an explicit schema needs at least one (name, dtype) pair");
        for (int i = 0; i < n_schema; i++) {
            if (!schema_names[i]) return fail(BDF_INVALID, "schema column %d has no name", i);
            if (!json_dtype_ok(schema[i]))
                return fail(BDF_UNSUPPORTED, "schema column %d: type %d is not read from JSON (numeric, Boolean, List of a numeric type or Utf8)", i, schema[i]);
            for (int j = 0; j < i; j++)
                if (strcmp(schema_names[i], schema_names[j]) == 0) return fail(BDF_INVALID, "schema name '%s' repeats", schema_names[i]);
        }
    }
    Owned<bdf_json> f(c, new (std::nothrow) bdf_json());
    if (!f.get()) return fail(BDF_OOM, "host allocation failed");
    f->batch = o->batch_size;
    const int64_t tile = json_tile_bytes();
    TRY(text_open(c, path, tile, "JSON", f.get()));
    const int64_t tiles = std::max<int64_t>((f->n + tile - 1) / tile, 1);

    Scratch<unsigned long long> counts, nl, members, is_rec, sums, small;   // small: [0] first bad line
    Scratch<void> table;
    Scratch<unsigned int> flags, bits;   // flags: [0] the key table is full, [1] a hash collision
    Scratch<int> col_of;

    // the '\n' positions
    cudaError_t e = counts.alloc(c, (size_t)(tiles + 1) * 8);
    if (e == cudaSuccess) e = small.alloc(c, 8);
    if (e == cudaSuccess) e = cudaMemsetAsync(small, 0xff, 8, c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "JSON line index scratch allocation");
    unsigned long long n_nl = 0;
    {
        LaunchTimer t(c, BDF_K_JSON, BDF_U8, f->n, f->n);
        c->launches++;   // count, scan
        e = launch_json_nl_count(f->d_text, f->n, counts, c->s_compute);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&n_nl, counts + tiles, 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
    if (e == cudaSuccess) e = nl.alloc(c, (size_t)std::max<unsigned long long>(n_nl, 1) * 8);
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_JSON, BDF_U64, f->n, f->n + (int64_t)n_nl * 8);
        e = launch_json_nl_index(f->d_text, f->n, counts, nl, c->s_compute);
    }
    if (e != cudaSuccess) return fail_cuda(e, "JSON line index");

    // every line checked; its members, and whether it is a record
    const int64_t lines = (int64_t)n_nl + 1;
    e = members.alloc(c, (size_t)(lines + 1) * 8);
    if (e == cudaSuccess) e = is_rec.alloc(c, (size_t)(lines + 1) * 8);
    if (e == cudaSuccess) e = sums.alloc(c, (size_t)scan_tile_sums(lines) * 8);
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_JSON, BDF_U64, lines, f->n + lines * 16);
        e = launch_json_lex(f->d_text, f->n, nl, (long long)n_nl, members, is_rec, small, c->sm_count, c->s_compute);
    }
    unsigned long long bad = ~0ull;
    if (e == cudaSuccess) e = cudaMemcpyAsync(&bad, small, 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "JSON record check");
    if (bad != ~0ull) return json_bad_line(c, f.get(), nl, (int64_t)n_nl, (int64_t)bad);
    {
        LaunchTimer t(c, BDF_K_JSON, BDF_U64, lines, lines * 32);
        c->launches += 2 * kScanLaunches - 1;   // two scans; the timer counts one
        e = launch_scan(members, lines, sums, c->s_compute);
        if (e == cudaSuccess) e = launch_scan(is_rec, lines, sums, c->s_compute);
    }
    unsigned long long tot[2] = {0, 0};
    if (e == cudaSuccess) e = cudaMemcpyAsync(&tot[0], members + lines, 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&tot[1], is_rec + lines, 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "JSON record scan");
    f->n_members = (int64_t)tot[0];
    f->n_rows = (int64_t)tot[1];
    if (f->n_rows == 0) return fail(BDF_WOULD_PANIC, "the JSON file has no records: the reference panics at batches[0]");
    if (tot[0] >= 0xffffffffull) return fail(BDF_UNSUPPORTED, "2^32 - 1 or more object members in one file");

    // the members, and the distinct keys
    e = cudaMallocAsync(&f->d_members, (size_t)std::max<int64_t>(f->n_members, 1) * json_member_bytes(), c->s_compute);
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_JSON, -1, lines, f->n + f->n_members * (int64_t)json_member_bytes());
        e = launch_json_members(f->d_text, f->n, nl, (long long)n_nl, members, is_rec, f->d_members, c->sm_count, c->s_compute);
    }
    if (e == cudaSuccess) e = table.alloc(c, (size_t)kJsonKeyCap * json_key_bytes());
    if (e == cudaSuccess) e = cudaMemsetAsync(table, 0xff, (size_t)kJsonKeyCap * json_key_bytes(), c->s_compute);
    if (e == cudaSuccess) e = flags.alloc(c, 8);
    if (e == cudaSuccess) e = cudaMemsetAsync(flags, 0, 8, c->s_compute);
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_JSON, -1, f->n_members, f->n_members * 32);
        c->launches++;   // insert, gather
        e = launch_json_keys(f->d_text, f->d_members, f->n_members, table, kJsonKeyCap, flags, c->sm_count, c->s_compute);
    }
    static_assert(sizeof(JsonKeyH) == 32, "JsonKey layout");
    std::vector<JsonKeyH> keys(kJsonKeyCap);
    unsigned int hflags[2] = {0, 0};
    if (e == cudaSuccess) e = cudaMemcpyAsync(keys.data(), table, (size_t)kJsonKeyCap * sizeof(JsonKeyH), cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaMemcpyAsync(hflags, flags, 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "JSON key table");
    if (hflags[0]) return fail(BDF_UNSUPPORTED, "more than %u distinct keys in one file", kJsonKeyCap);

    // the dictionary: every raw key decoded (escapes are rare: only those need work); a name's first member over its spellings
    struct Name { unsigned long long first; uint32_t rec; };
    std::vector<std::string> names;
    std::vector<Name> seen;
    std::vector<int> name_of(kJsonKeyCap, -1);
    std::unordered_map<std::string, size_t> index;   // up to kJsonKeyCap names: no linear search
    for (unsigned s = 0; s < kJsonKeyCap; s++) {
        const JsonKeyH& k = keys[s];
        if (k.hash == ~0ull) continue;
        const uint8_t* p = f->map + f->off + k.kstart;
        const std::string name = memchr(p, '\\', k.klen) ? json_unescape(p, p + k.klen) : std::string((const char*)p, k.klen);
        const size_t j = index.emplace(name, names.size()).first->second;
        if (j == names.size()) { names.push_back(name); seen.push_back(Name{k.first, k.rec}); }
        else if (k.first < seen[j].first) seen[j] = Name{k.first, k.rec};
        name_of[s] = (int)j;
    }
    const int64_t n_inf = o->max_records < 0 ? f->n_rows : std::min<int64_t>(o->max_records, f->n_rows);
    std::vector<int> col_of_name(names.size(), -1);
    if (schema) {
        for (int i = 0; i < n_schema; i++) {
            f->names.push_back(schema_names[i]);
            f->dtypes.push_back(schema[i] == BDF_UTF8 ? -1 : schema[i]);
            f->nullable.push_back(1);
            for (size_t j = 0; j < names.size(); j++)
                if (names[j] == schema_names[i] && f->dtypes.back() >= 0) col_of_name[j] = i;
        }
    } else {   // the keys of the inferred records, in the order they are first seen
        std::vector<size_t> order;
        for (size_t j = 0; j < names.size(); j++)
            if ((int64_t)seen[j].rec < n_inf) order.push_back(j);
        std::sort(order.begin(), order.end(), [&](size_t a, size_t b) { return seen[a].first < seen[b].first; });
        for (size_t i = 0; i < order.size(); i++) {
            col_of_name[order[i]] = (int)i;
            f->names.push_back(names[order[i]]);
        }
    }
    const int n_cols = (int)f->names.size();
    if (n_cols > 65535) return fail(BDF_UNSUPPORTED, "more than 65535 columns");
    std::vector<int> hcol(kJsonKeyCap, -1);
    for (unsigned s = 0; s < kJsonKeyCap; s++)
        if (name_of[s] >= 0) hcol[s] = col_of_name[(size_t)name_of[s]];

    // the slots: which member gives each (record, column)
    const size_t slot_bytes = (size_t)f->n_rows * (size_t)n_cols * 4;
    if (n_cols) {
        e = cudaMallocAsync((void**)&f->d_slots, slot_bytes, c->s_compute);
        if (e == cudaSuccess) e = cudaMemsetAsync(f->d_slots, 0, slot_bytes, c->s_compute);
        if (e == cudaSuccess) e = col_of.alloc(c, (size_t)kJsonKeyCap * 4);
        if (e == cudaSuccess) e = cudaMemcpyAsync(col_of, hcol.data(), (size_t)kJsonKeyCap * 4, cudaMemcpyHostToDevice, c->s_compute);
        if (e == cudaSuccess) {
            LaunchTimer t(c, BDF_K_JSON, BDF_U32, f->n_members, f->n_members * 48);
            e = launch_json_resolve(f->d_text, f->d_members, f->n_members, table, kJsonKeyCap, col_of, n_cols, f->d_slots, flags + 1, c->sm_count, c->s_compute);
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(hflags, flags, 8, cudaMemcpyDeviceToHost, c->s_compute);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);   // hcol is read by the copy
        if (e != cudaSuccess) return fail_cuda(e, "JSON key resolution");
        if (hflags[1]) return fail(BDF_UNSUPPORTED, "two different keys of the file share a 64-bit hash");
    }

    // inference: the class bits of every column over the first n_inf records
    if (!schema && n_cols) {
        std::vector<unsigned int> hb((size_t)n_cols, 0u);
        e = bits.alloc(c, (size_t)n_cols * 4);
        if (e == cudaSuccess) e = cudaMemsetAsync(bits, 0, (size_t)n_cols * 4, c->s_compute);
        if (e == cudaSuccess) {
            LaunchTimer t(c, BDF_K_JSON, BDF_U32, n_inf * n_cols, n_inf * n_cols * 8);
            e = launch_json_infer(f->d_members, f->d_slots, n_inf * n_cols, n_cols, bits, c->sm_count, c->s_compute);
        }
        if (e == cudaSuccess) e = cudaMemcpyAsync(hb.data(), bits, (size_t)n_cols * 4, cudaMemcpyDeviceToHost, c->s_compute);
        if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
        if (e != cudaSuccess) return fail_cuda(e, "JSON schema inference");
        for (int i = 0; i < n_cols; i++) {
            f->dtypes.push_back(json_coerce(hb[(size_t)i]));
            f->nullable.push_back((hb[(size_t)i] & (json::kNull | json::kMissing)) ? 1 : 0);
        }
    }
    *out = f.release();
    return BDF_OK;
}

// The floats the device could not round: rounded exactly on the host (C locale) and written back by k_csv_scatter.  Entry x goes
// to element x.row of chunk x.chunk of cols[x.col].
static int json_exact(bdf_ctx* c, const bdf_json* f, const void* slow, int64_t n_slow, const std::vector<const bdf_col*>& cols) {
    struct Patch { unsigned long long dst, bits; int width, pad; };   // k_csv.cu's CsvPatch
    static_assert(sizeof(Patch) == 24, "CsvPatch layout");
    std::vector<JsonSlowH> sl((size_t)n_slow);
    CK(cudaMemcpyAsync(sl.data(), slow, (size_t)n_slow * sizeof(JsonSlowH), cudaMemcpyDeviceToHost, c->s_compute));
    CK(cudaStreamSynchronize(c->s_compute));
    static locale_t cloc = newlocale(LC_ALL_MASK, "C", (locale_t)0);
    std::vector<Patch> hp;
    for (const JsonSlowH& x : sl) {
        const std::string v((const char*)f->map + f->off + x.start, (size_t)(x.end - x.start));
        const bdf_col* col = cols[(size_t)x.col];
        Patch pt{};
        if (col->dtype == BDF_F64) {
            const double d = strtod_l(v.c_str(), nullptr, cloc);
            memcpy(&pt.bits, &d, 8);
            pt.width = 8;
        } else {
            const float fl = strtof_l(v.c_str(), nullptr, cloc);
            uint32_t b;
            memcpy(&b, &fl, 4);
            pt.bits = b;
            pt.width = 4;
        }
        pt.dst = (unsigned long long)(uintptr_t)(col->chunks[(size_t)x.chunk].values + x.row * pt.width);
        hp.push_back(pt);
    }
    Scratch<void> patches;
    cudaError_t e = patches.alloc(c, hp.size() * sizeof(Patch));
    if (e == cudaSuccess) e = cudaMemcpyAsync(patches, hp.data(), hp.size() * sizeof(Patch), cudaMemcpyHostToDevice, c->s_compute);
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_JSON, -1, (int64_t)hp.size(), (int64_t)hp.size() * 32);
        e = launch_csv_scatter(patches, (long long)hp.size(), c->s_compute);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);   // hp is read by the copy
    if (e != cudaSuccess) return fail_cuda(e, "JSON exact rounding");
    return BDF_OK;
}

static int json_check_col(const bdf_json* f, int col) {
    if (col < 0 || col >= (int)f->names.size()) return fail(BDF_INVALID, "column %d out of range (the file has %zu)", col, f->names.size());
    if (f->dtypes[(size_t)col] < 0)
        return fail(BDF_UNSUPPORTED, "column %d (%s) is not on the device path (a string, an object or a mix of kinds)", col, f->names[(size_t)col].c_str());
    return BDF_OK;
}

static int json_read(bdf_ctx* c, const bdf_json* f, int n_cols, const int32_t* cols, bdf_col** out) {
    if (!f || !out || (n_cols > 0 && !cols)) return fail(BDF_INVALID, "null argument");
    if (n_cols < 0 || n_cols > 65535) return fail(BDF_INVALID, "0..65535 columns");
    for (int i = 0; i < n_cols; i++) {
        TRY(json_check_col(f, cols[i]));
        if (f->dtypes[(size_t)cols[i]] > kBool)
            return fail(BDF_UNSUPPORTED, "column %d (%s) is a List: read it with bdf_json_read_list", cols[i], f->names[(size_t)cols[i]].c_str());
    }
    const int64_t batch = f->batch, n_chunks = (f->n_rows + batch - 1) / batch;
    std::vector<ChunkPlan> plan((size_t)n_chunks);
    for (int64_t i = 0; i < n_chunks; i++) plan[(size_t)i] = ChunkPlan{std::min(batch, f->n_rows - i * batch), true};
    std::vector<ColOwner> res;
    Scratch<char> descs;
    Scratch<unsigned long long> small;   // [0] slow-path values
    Scratch<void> slow;
    const size_t dsz = json_desc_bytes();
    std::vector<char> hdesc((size_t)std::max(n_cols, 1) * dsz, 0);
    int64_t float_fields = 0, out_bytes = 0;
    for (int i = 0; i < n_cols; i++) {
        const int dt = f->dtypes[(size_t)cols[i]];
        res.emplace_back(c);
        TRY(col_alloc(c, dt, plan, nullptr, json_parse_rows(), res[(size_t)i].out()));
        bdf_col* col = res[(size_t)i].get();
        const DevChunk& c0 = col->chunks[0];
        const long long vs = n_chunks > 1 ? (long long)(col->chunks[1].values - c0.values) : 0;
        const long long bs = n_chunks > 1 ? (long long)((char*)col->chunks[1].validity - (char*)c0.validity) : 0;
        const DevChunk& cl = col->chunks[(size_t)n_chunks - 1];
        if (cl.values != c0.values + vs * (n_chunks - 1) || (char*)cl.validity != (char*)c0.validity + bs * (n_chunks - 1))
            return fail(BDF_INVALID, "internal: JSON output chunks are not evenly spaced");
        struct Desc { char* values; long long vstride; uint32_t* validity; long long bstride; uint32_t* warp_counts; int dtype; int file_col; } d{
            c0.values, vs, c0.validity, bs, col->d_warp_counts, dt, cols[i]};
        static_assert(sizeof(Desc) == 48, "JsonColDesc layout");
        memcpy(hdesc.data() + (size_t)i * dsz, &d, sizeof d);
        if (dt == BDF_F32 || dt == BDF_F64) float_fields += f->n_rows;
        out_bytes += (int64_t)value_bytes(dt, f->n_rows, 0) + bitmap_bytes(f->n_rows);
    }
    const long long slow_cap = std::max<long long>(65536, float_fields / 64);
    cudaError_t e = descs.alloc(c, hdesc.size());
    if (e == cudaSuccess) e = cudaMemcpyAsync(descs, hdesc.data(), hdesc.size(), cudaMemcpyHostToDevice, c->s_compute);
    if (e == cudaSuccess) e = small.alloc(c, 8);
    if (e == cudaSuccess) e = cudaMemsetAsync(small, 0, 8, c->s_compute);
    if (e == cudaSuccess && float_fields) e = slow.alloc(c, (size_t)slow_cap * json_slow_bytes());
    if (e != cudaSuccess) return fail_cuda(e, "JSON read scratch allocation");
    unsigned long long n_slow = 0;
    {
        const int64_t cells = f->n_rows * n_cols;
        LaunchTimer t(c, BDF_K_JSON, n_cols == 1 ? f->dtypes[(size_t)cols[0]] : -1, cells, cells * 48 + out_bytes);
        e = launch_json_parse(f->d_text, f->d_members, f->d_slots, (int)f->names.size(), descs, n_cols, f->n_rows, batch, slow, small, slow_cap, c->s_compute);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(&n_slow, small, 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);   // hdesc is read by the copy
    if (e != cudaSuccess) return fail_cuda(e, "JSON parse");
    if ((long long)n_slow > slow_cap)
        return fail(BDF_UNSUPPORTED, "%llu float values need exact rounding, more than the %lld one read resolves", n_slow, slow_cap);
    if (n_slow) {
        std::vector<const bdf_col*> targets;
        for (auto& r : res) targets.push_back(r.get());
        TRY(json_exact(c, f, slow, (int64_t)n_slow, targets));
    }
    for (int i = 0; i < n_cols; i++) {
        bdf_col* col = res[(size_t)i].get();
        col->counts_on_device = true;
        TRY(fetch_counts(c, col));
        for (size_t j = 0; j < col->chunks.size(); j++)
            if (col->null_counts[j] == 0) col->chunks[j].validity = nullptr;   // no bitmap in a chunk without nulls
        e = finish_single_group(c, col);
        if (e != cudaSuccess) return fail_cuda(e, "JSON read");
    }
    f->exact_fields = (int64_t)n_slow;
    for (int i = 0; i < n_cols; i++) out[i] = res[(size_t)i].release();
    return BDF_OK;
}

static int json_read_list(bdf_ctx* c, const bdf_json* f, int col, bdf_list** out) {
    if (!f || !out) return fail(BDF_INVALID, "null argument");
    TRY(json_check_col(f, col));
    const int ldt = f->dtypes[(size_t)col];
    if (ldt < BDF_LIST_BASE) return fail(BDF_UNSUPPORTED, "column %d (%s) is not a List: read it with bdf_json_read", col, f->names[(size_t)col].c_str());
    const int dt = ldt - BDF_LIST_BASE;
    const int64_t batch = f->batch, n_rows = f->n_rows, n_chunks = (n_rows + batch - 1) / batch, words = (batch + 31) / 32;
    const int n_file_cols = (int)f->names.size();
    Scratch<unsigned long long> counts, sums, bounds, nulls, small;   // nulls: [chunk] null lists, then [chunk] null elements; small: slow values
    Scratch<uint32_t> vwords;
    Scratch<void> descs, slow;
    cudaError_t e = counts.alloc(c, (size_t)(n_rows + 1) * 8);
    if (e == cudaSuccess) e = sums.alloc(c, (size_t)scan_tile_sums(n_rows) * 8);
    if (e == cudaSuccess) e = bounds.alloc(c, (size_t)(n_chunks + 1) * 8);
    if (e == cudaSuccess) e = nulls.alloc(c, (size_t)n_chunks * 16);
    if (e == cudaSuccess) e = cudaMemsetAsync(nulls, 0, (size_t)n_chunks * 16, c->s_compute);
    if (e == cudaSuccess) e = vwords.alloc(c, (size_t)(n_chunks * words) * 4);
    if (e != cudaSuccess) return fail_cuda(e, "JSON list scratch allocation");
    {
        LaunchTimer t(c, BDF_K_JSON, ldt, n_rows, n_rows * 16);
        c->launches += kScanLaunches + 1;   // the timer counts the count; and bounds
        e = launch_json_list_count(f->d_text, f->d_members, f->d_slots, n_file_cols, col, n_rows, batch, counts, vwords, nulls, c->s_compute);
        if (e == cudaSuccess) e = launch_scan(counts, n_rows, sums, c->s_compute);
        if (e == cudaSuccess) e = launch_json_bounds(counts, n_rows, batch, n_chunks, bounds, c->s_compute);
    }
    std::vector<unsigned long long> hb((size_t)n_chunks + 1), hn((size_t)n_chunks * 2);
    if (e == cudaSuccess) e = cudaMemcpyAsync(hb.data(), bounds, hb.size() * 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaMemcpyAsync(hn.data(), nulls, (size_t)n_chunks * 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "JSON list count");
    if (hb[(size_t)n_chunks] >= (unsigned long long)kListMaxCallElems)
        return fail(BDF_UNSUPPORTED, "a list call holds 2^32 or more elements (the sort's UInt32 row numbers)");
    std::vector<int64_t> lens((size_t)n_chunks), elems((size_t)n_chunks);
    std::vector<ChunkPlan> plan((size_t)n_chunks);
    for (int64_t i = 0; i < n_chunks; i++) {
        lens[(size_t)i] = std::min(batch, n_rows - i * batch);
        elems[(size_t)i] = (int64_t)(hb[(size_t)i + 1] - hb[(size_t)i]);
        if (elems[(size_t)i] >= kListMaxChunkElems) return fail(BDF_UNSUPPORTED, "list chunk %lld: 2^31 or more elements", (long long)i);
        plan[(size_t)i] = ChunkPlan{elems[(size_t)i], true};
    }
    ListOwner l(c);
    TRY(list_alloc(c, dt, lens, std::vector<bool>((size_t)n_chunks, true), l.out()));
    ColOwner child(c);
    TRY(col_alloc(c, dt, plan, nullptr, 0, child.out()));
    struct Chunk { int32_t* offsets; uint32_t* validity; char* values; uint32_t* value_validity; };
    static_assert(sizeof(Chunk) == 32, "JsonListChunk layout");
    std::vector<Chunk> hc((size_t)n_chunks);
    for (int64_t i = 0; i < n_chunks; i++) {
        const DevChunk& ch = child->chunks[(size_t)i];
        hc[(size_t)i] = Chunk{l->off[(size_t)i], l->valid[(size_t)i], ch.values, ch.validity};
    }
    const int64_t total = (int64_t)hb[(size_t)n_chunks];
    const long long slow_cap = std::max<long long>(65536, total / 64);
    e = descs.alloc(c, hc.size() * sizeof(Chunk));
    if (e == cudaSuccess) e = cudaMemcpyAsync(descs, hc.data(), hc.size() * sizeof(Chunk), cudaMemcpyHostToDevice, c->s_compute);
    if (e == cudaSuccess) e = small.alloc(c, 8);
    if (e == cudaSuccess) e = cudaMemsetAsync(small, 0, 8, c->s_compute);
    if (e == cudaSuccess && dtype_is_float(dt)) e = slow.alloc(c, (size_t)slow_cap * json_slow_bytes());
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_JSON, dt, total, n_rows * 48 + total * (dtype_width(dt) + 16));
        e = launch_json_list_fill(f->d_text, f->d_members, f->d_slots, n_file_cols, col, dt, n_rows, batch, counts, vwords, descs, nulls + n_chunks, slow,
                                  small, slow_cap, c->s_compute);
    }
    unsigned long long n_slow = 0;
    if (e == cudaSuccess) e = cudaMemcpyAsync(hn.data() + n_chunks, nulls + n_chunks, (size_t)n_chunks * 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&n_slow, small, 8, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);   // hc is read by the copy
    if (e != cudaSuccess) return fail_cuda(e, "JSON list fill");
    if ((long long)n_slow > slow_cap)
        return fail(BDF_UNSUPPORTED, "%llu float values need exact rounding, more than the %lld one read resolves", n_slow, slow_cap);
    if (n_slow) TRY(json_exact(c, f, slow, (int64_t)n_slow, {child.get()}));
    for (int64_t i = 0; i < n_chunks; i++) {
        const size_t k = (size_t)i;
        l->null_counts[k] = (int64_t)hn[k];
        l->valid_elems[k] = elems[k];   // a null list has no elements
        if (hn[k] == 0) l->valid[k] = nullptr;   // no bitmap in a chunk without null lists
        child->null_counts[k] = (int64_t)hn[(size_t)n_chunks + k];
        if (child->null_counts[k] == 0) child->chunks[k].validity = nullptr;
    }
    e = finish_single_group(c, child.get());
    if (e != cudaSuccess) return fail_cuda(e, "JSON list read");
    f->exact_fields = (int64_t)n_slow;
    l->values = child.release();
    *out = l.release();
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// Parquet reader (parquet.cu reads the footers and page headers and plans the read; k_parquet.cu decodes; the rules are in
// include/b200df.h): the projected column chunks go to HBM still compressed, through the pageable staging path, with the page and
// tile tables; four launches over the whole page table decompress, walk the runs, write the validity and write the values straight
// into the output chunks.  The per-page error words and per-chunk null counts come back in one copy at the end.

static int parquet_read(bdf_ctx* c, const bdf_parquet* f, int n_cols, const int32_t* cols, bdf_col** out) {
    if (!f || !out || (n_cols > 0 && !cols)) return fail(BDF_INVALID, "null argument");
    if (n_cols < 0 || n_cols > 65535) return fail(BDF_INVALID, "0..65535 columns");
    pq::Plan P;
    TRY(pq::plan(f, n_cols, cols, &P));
    const int64_t n_chunks = (int64_t)P.chunk_lens.size(), n_out = n_chunks * n_cols;
    const int n_pages = (int)P.pages.size(), n_tiles = (int)P.tiles.size();
    std::vector<int32_t> dtypes((size_t)n_cols), nullable((size_t)n_cols);
    int64_t out_bytes = 0, rows = 0;
    for (int i = 0; i < n_cols; i++) {
        TRY(bdf_parquet_column(f, cols[i], nullptr, &dtypes[(size_t)i], &nullable[(size_t)i]));
        for (int64_t len : P.chunk_lens) out_bytes += (int64_t)align_up(value_bytes(dtypes[(size_t)i], len, 0) + 8, 256) + (nullable[(size_t)i] ? (int64_t)align_up((size_t)len / 8 + 9, 256) : 0);
    }
    for (int64_t len : P.chunk_lens) rows += len;
    const size_t err_bytes = align_up((size_t)std::max(n_pages, 1) * 4, 8);
    const size_t small_bytes = err_bytes + (size_t)std::max<int64_t>(n_out, 1) * 8;
    const long double need = (long double)out_bytes + P.upload_bytes + P.scratch_bytes + (long double)P.run_entries * pq_run_bytes() +
                             (long double)n_pages * (pq_page_bytes() + 16) + (long double)n_tiles * (pq_tile_bytes() + 4) +
                             (long double)n_out * pq_out_bytes() + small_bytes;
    if (need * 1.1L > (long double)c->hbm_bytes)
        return fail(BDF_OOM, "a Parquet read of %.0Lf bytes (compressed chunks, scratch and outputs) does not fit in device memory", need);

    std::vector<ColOwner> res;
    std::vector<pq::Out> houts((size_t)std::max<int64_t>(n_out, 1));
    for (int i = 0; i < n_cols; i++) {
        std::vector<ChunkPlan> plan((size_t)n_chunks);
        for (int64_t j = 0; j < n_chunks; j++) plan[(size_t)j] = ChunkPlan{P.chunk_lens[(size_t)j], nullable[(size_t)i] != 0};
        res.emplace_back(c);
        TRY(col_alloc(c, dtypes[(size_t)i], plan, nullptr, 0, res[(size_t)i].out()));
        bdf_col* col = res[(size_t)i].get();
        if (dtypes[(size_t)i] == kBool && col->arena_values) {   // Boolean values are OR-ed in bit by bit
            size_t vb = 0;
            for (int64_t len : P.chunk_lens) vb += align_up(value_bytes(kBool, len, 0) + 8, 256);
            CK(cudaMemsetAsync(col->arena_values, 0, vb, c->s_compute));
        }
        for (int64_t j = 0; j < n_chunks; j++)
            houts[(size_t)(i * n_chunks + j)] = pq::Out{col->chunks[(size_t)j].values, col->chunks[(size_t)j].validity};
    }
    Scratch<uint8_t> upload, scratch, small;
    Scratch<char> pages, tiles, outs, runs, meta;
    Scratch<int> tile_valid;
    cudaError_t e = upload.alloc(c, (size_t)std::max<long long>(P.upload_bytes, 16));
    if (e == cudaSuccess) e = scratch.alloc(c, (size_t)std::max<long long>(P.scratch_bytes, 16));
    if (e == cudaSuccess) e = runs.alloc(c, (size_t)std::max<long long>(P.run_entries, 1) * pq_run_bytes());
    if (e == cudaSuccess) e = meta.alloc(c, (size_t)std::max(n_pages, 1) * 16);
    if (e == cudaSuccess) e = pages.alloc(c, (size_t)std::max(n_pages, 1) * pq_page_bytes());
    if (e == cudaSuccess) e = tiles.alloc(c, (size_t)std::max(n_tiles, 1) * pq_tile_bytes());
    if (e == cudaSuccess) e = tile_valid.alloc(c, (size_t)std::max(n_tiles, 1) * 4);
    if (e == cudaSuccess) e = outs.alloc(c, houts.size() * pq_out_bytes());
    if (e == cudaSuccess) e = small.alloc(c, small_bytes);
    if (e == cudaSuccess) e = cudaMemsetAsync(small, 0, small_bytes, c->s_compute);
    if (e == cudaSuccess && n_pages) e = cudaMemcpyAsync(pages, P.pages.data(), (size_t)n_pages * pq_page_bytes(), cudaMemcpyHostToDevice, c->s_compute);
    if (e == cudaSuccess && n_tiles) e = cudaMemcpyAsync(tiles, P.tiles.data(), (size_t)n_tiles * pq_tile_bytes(), cudaMemcpyHostToDevice, c->s_compute);
    if (e == cudaSuccess) e = cudaMemcpyAsync(outs, houts.data(), houts.size() * pq_out_bytes(), cudaMemcpyHostToDevice, c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "Parquet read allocation");
    // the compressed chunks: page cache -> pinned staging -> HBM on the copy stream, after the allocations
    e = cudaEventRecord(c->ev_tmp, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(c->s_h2d, c->ev_tmp, 0);
    const auto t0 = std::chrono::steady_clock::now();
    for (size_t s = 0; s < P.segs.size() && e == cudaSuccess; s++)
        if (P.segs[s].len) e = h2d_copy(c, upload.get() + P.segs[s].dst, P.segs[s].src, (size_t)P.segs[s].len);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_h2d);
    const double upload_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (e != cudaSuccess) {
        const int st = fail_cuda(e, "Parquet upload");
        cudaStreamSynchronize(c->s_h2d);   // no copy may still write into the buffers when they are freed
        return st;
    }
    int* err = (int*)small.get();
    unsigned long long* nulls = (unsigned long long*)(small.get() + err_bytes);
    int64_t comp_bytes = 0;
    for (const auto& sg : P.segs) comp_bytes += sg.len;
    {
        LaunchTimer t(c, BDF_K_PARQUET, BDF_U8, n_pages, comp_bytes + P.scratch_bytes);
        e = launch_pq_snappy(pages, n_pages, upload, scratch, err, c->sm_count, c->s_compute);
    }
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_PARQUET, BDF_U32, n_pages, P.run_entries * (int64_t)pq_run_bytes());
        e = launch_pq_runs(pages, n_pages, upload, scratch, runs, meta, err, c->s_compute);
    }
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_PARQUET, kBool, rows * n_cols, rows * n_cols / 8);
        e = launch_pq_levels(pages, tiles, n_tiles, upload, scratch, runs, meta, outs, P.batch, tile_valid, nulls, err, c->s_compute);
    }
    if (e == cudaSuccess) {
        LaunchTimer t(c, BDF_K_PARQUET, n_cols == 1 ? dtypes[0] : -1, rows * n_cols, out_bytes);
        e = launch_pq_values(pages, tiles, n_tiles, upload, scratch, runs, meta, outs, P.batch, tile_valid, err, c->s_compute);
    }
    std::vector<char> hs(small_bytes);
    if (e == cudaSuccess) e = cudaMemcpyAsync(hs.data(), small, small_bytes, cudaMemcpyDeviceToHost, c->s_compute);
    if (e == cudaSuccess) e = cudaStreamSynchronize(c->s_compute);   // the host tables are read by the copies
    if (e != cudaSuccess) return fail_cuda(e, "Parquet decode");
    const int* herr = (const int*)hs.data();
    for (int p = 0; p < n_pages; p++)
        if (herr[p]) return pq::page_error(f, P, p, herr[p]);
    const unsigned long long* hn = (const unsigned long long*)(hs.data() + err_bytes);
    for (int i = 0; i < n_cols; i++) {
        bdf_col* col = res[(size_t)i].get();
        for (int64_t j = 0; j < n_chunks; j++) {
            col->null_counts[(size_t)j] = (int64_t)hn[i * n_chunks + j];
            if (col->null_counts[(size_t)j] == 0) col->chunks[(size_t)j].validity = nullptr;   // no bitmap in a chunk without nulls
        }
        e = finish_single_group(c, col);
        if (e != cudaSuccess) return fail_cuda(e, "Parquet read");
    }
    pq::set_stats(f, n_pages, comp_bytes, upload_ms);
    for (int i = 0; i < n_cols; i++) out[i] = res[(size_t)i].release();
    return BDF_OK;
}

// ---------------------------------------------------------------------------------------------------
// C ABI

#define NEED_CTX(ctx) \
    if (!(ctx)) return fail(BDF_INVALID, "null context")

// An entry checks its arguments first (after NEED_CTX where the null context answers first), then hands a multi-GPU context to
// the fleet, then ENTERs.  ENTER stays after the fleet dispatch: a fleet branch may call back into an entry with the same context,
// and the context's mutex is not recursive.
#define ENTER(ctx)                                                   \
    NEED_CTX(ctx);                                                   \
    std::lock_guard<std::mutex> _lock((ctx)->mu);                    \
    CK(cudaSetDevice((ctx)->device));

// Host in / host out on one GPU: upload the views (the copies run ahead of the operator), run `body(uploaded columns)`, and wait
// for the copies before the inputs go: the caller may reuse its host buffers as soon as the call returns.
template <class F>
static int host_call(bdf_ctx* c, const std::vector<UploadSpec>& specs, F&& body) {
    std::vector<bdf_col*> cols;
    TRY(upload_many(c, specs, true, cols));
    const int st = body(cols.data());
    const std::string keep = g_err;
    cudaStreamSynchronize(c->s_h2d);
    for (bdf_col* col : cols) col_release(c, col);
    g_err = keep;
    return st;
}

extern "C" {

int bdf_abi_version(void) { return BDF_ABI_VERSION; }

const char* bdf_last_error(void) { return g_err.c_str(); }

void bdf_destroy(bdf_ctx* c) {
    if (c && c->fleet) { fleet_destroy(c); return; }
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->s_compute) cudaStreamSynchronize(c->s_compute);
    if (c->s_h2d) cudaStreamSynchronize(c->s_h2d);
    if (c->s_d2h) cudaStreamSynchronize(c->s_d2h);
    if (c->s_desc) cudaStreamSynchronize(c->s_desc);
    if (c->s_fin) cudaStreamSynchronize(c->s_fin);
    for (auto& p : c->prof) { cudaEventDestroy(p.e0); cudaEventDestroy(p.e1); }
    for (auto ev : c->prof_pool) cudaEventDestroy(ev);
    for (auto ev : c->ev_pool) cudaEventDestroy(ev);
    c->pool.reset();
    for (auto& sl : c->stage) { if (sl.p) cudaFreeHost(sl.p); if (sl.ev) cudaEventDestroy(sl.ev); }
    for (auto& b : c->part) { if (b.p) cudaFree(b.p); if (b.done) cudaEventDestroy(b.done); }
    if (c->ring) cudaFreeHost(c->ring);
    if (c->dring) cudaFree(c->dring);
    if (c->d_stage) cudaFree(c->d_stage);
    if (c->h_agg) cudaFreeHost(c->h_agg);
    if (c->h_flag) cudaFreeHost(c->h_flag);
    if (c->h_sort_agree) cudaFreeHost(c->h_sort_agree);
    if (c->d_partials) cudaFree(c->d_partials);
    if (c->d_stage2) cudaFree(c->d_stage2);
    if (c->d_stage_many) cudaFree(c->d_stage_many);
    if (c->d_tickets_many) cudaFree(c->d_tickets_many);
    if (c->d_ticket) cudaFree(c->d_ticket);
    if (c->d_flag) cudaFree(c->d_flag);
    if (c->flush_buf) cudaFree(c->flush_buf);
    if (c->comm) { comm_destroy(c->comm); c->comm = nullptr; }
    if (c->d_local) cudaFree(c->d_local);
    if (c->ev_tmp) cudaEventDestroy(c->ev_tmp);
    if (c->ev_t0) cudaEventDestroy(c->ev_t0);
    if (c->ev_t1) cudaEventDestroy(c->ev_t1);
    if (c->s_compute) cudaStreamDestroy(c->s_compute);
    if (c->s_h2d) cudaStreamDestroy(c->s_h2d);
    if (c->s_d2h) cudaStreamDestroy(c->s_d2h);
    if (c->s_desc) cudaStreamDestroy(c->s_desc);
    if (c->s_fin) cudaStreamDestroy(c->s_fin);
    delete c;
}

static int init_impl(bdf_ctx* c, int device) {
    int n_dev = 0;
    cudaError_t e = cudaGetDeviceCount(&n_dev);
    if (e != cudaSuccess || n_dev == 0) {
        cudaGetLastError();
        return fail(BDF_CUDA, "no usable CUDA device (%s); this library has no CPU fallback", e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    if (device < 0 || device >= n_dev) return fail(BDF_INVALID, "device %d out of range (0..%d)", device, n_dev - 1);
    c->device = device;
    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    c->sm_count = prop.multiProcessorCount; c->cc_major = prop.major; c->cc_minor = prop.minor; c->hbm_bytes = prop.totalGlobalMem;
    if (prop.major != 9 || prop.minor != 0) return fail(BDF_CUDA, "device %d is sm_%d%d; libb200df is built for sm_90a only", device, prop.major, prop.minor);
    CK(cudaStreamCreateWithFlags(&c->s_compute, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&c->s_h2d, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&c->s_d2h, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&c->s_desc, cudaStreamNonBlocking));
    // The finish stream's few CTAs are scheduled ahead of the CTAs still queued from the next operator's grid: at the default
    // priority a k_finish waited for the whole next K5 grid to be dispatched, so the host saw the step's result one step late.
    int prio_least = 0, prio_greatest = 0;
    CK(cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest));
    CK(cudaStreamCreateWithPriority(&c->s_fin, cudaStreamNonBlocking, prio_greatest));
    cudaMemPool_t pool;
    CK(cudaDeviceGetDefaultMemPool(&pool, device));
    uint64_t keep = ~0ull;  // keep freed arenas cached: operators allocate their outputs per call
    CK(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
    c->ring_cap = (size_t)32 << 20;  // ~400k chunk descriptors per operator call
    CK(cudaHostAlloc((void**)&c->ring, c->ring_cap, cudaHostAllocDefault));
    CK(cudaMalloc((void**)&c->dring, c->ring_cap));
    CK(cudaHostAlloc((void**)&c->h_agg, 2 * kAggSlots * sizeof(AggDev), cudaHostAllocMapped));
    CK(cudaHostGetDevicePointer((void**)&c->h_agg_dev, c->h_agg, 0));
    CK(cudaHostAlloc((void**)&c->h_flag, sizeof(int), cudaHostAllocDefault));
    CK(cudaMalloc((void**)&c->d_stage2, (size_t)c->sm_count * sizeof(AggDev)));
    CK(cudaMalloc((void**)&c->d_stage, (size_t)c->sm_count * sizeof(AggDev)));
    CK(cudaMalloc((void**)&c->d_ticket, 4 * sizeof(unsigned int)));
    CK(cudaMalloc((void**)&c->d_flag, sizeof(int)));
    CK(cudaMalloc((void**)&c->d_local, (size_t)kAggSlots * sizeof(AggDev)));
    CK(cudaMemset(c->d_ticket, 0, 4 * sizeof(unsigned int)));
    CK(cudaMemset(c->d_flag, 0, sizeof(int)));
    CK(cudaEventCreateWithFlags(&c->ev_tmp, cudaEventDisableTiming));
    CK(cudaEventCreate(&c->ev_t0));
    CK(cudaEventCreate(&c->ev_t1));
    // experiment knob: L2 fetch granularity hint (32 / 64 / 128 bytes) -- random gathers (take) fetch whole 128-byte lines by default
    if (const char* fg = getenv("BDF_L2_FETCH")) { if (atoi(fg) > 0) cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)atoi(fg)); cudaGetLastError(); }
    const char* pb = getenv("BDF_PIPELINE_BYTES");
    if (pb && atoll(pb) > 0) c->pipeline_bytes = (size_t)atoll(pb);
    const char* ps = getenv("BDF_PIPELINE_SPLIT");
    c->pipeline_split = ps && atoi(ps) > 0;
    return BDF_OK;
}

int bdf_init(int device, bdf_ctx** out) {
    if (!out) return fail(BDF_INVALID, "null out pointer");
    *out = nullptr;
    bdf_ctx* c = new (std::nothrow) bdf_ctx();
    if (!c) return fail(BDF_OOM, "host allocation failed");
    int st = init_impl(c, device);
    if (st != BDF_OK) { std::string keep = g_err; bdf_destroy(c); g_err = keep; return st; }
    *out = c;
    return BDF_OK;
}

namespace bdf { int ctx_attach_comm(bdf_ctx* c, Comm* cm) { c->comm = cm; c->collective = true; c->collectives = 0; return BDF_OK; } }

int bdf_init_multi(int n_gpus, const int* devices, bdf_ctx** out) {
    if (!out) return fail(BDF_INVALID, "null out pointer");
    *out = nullptr;
    int n_dev = 0;
    cudaError_t e = cudaGetDeviceCount(&n_dev);
    if (e != cudaSuccess || n_dev == 0) {
        cudaGetLastError();
        return fail(BDF_CUDA, "no usable CUDA device (%s); this library has no CPU fallback", e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    }
    if (n_gpus == 0) n_gpus = n_dev;
    if (n_gpus < 1 || n_gpus > n_dev) return fail(BDF_INVALID, "%d GPUs requested, %d visible", n_gpus, n_dev);
    std::vector<int> devs((size_t)n_gpus);
    for (int i = 0; i < n_gpus; i++) {
        devs[i] = devices ? devices[i] : i;
        if (devs[i] < 0 || devs[i] >= n_dev) return fail(BDF_INVALID, "device %d out of range (0..%d)", devs[i], n_dev - 1);
        for (int j = 0; j < i; j++) if (devs[j] == devs[i]) return fail(BDF_INVALID, "device %d listed twice", devs[i]);
    }
    bdf_ctx* c = new (std::nothrow) bdf_ctx();
    Fleet* f = new (std::nothrow) Fleet();
    if (!c || !f) { delete c; delete f; return fail(BDF_OOM, "host allocation failed"); }
    c->fleet = f;
    c->device = devs[0];
    int st = BDF_OK;
    for (int i = 0; i < n_gpus && st == BDF_OK; i++) {
        bdf_ctx* kid = nullptr;
        st = bdf_init(devs[i], &kid);
        if (st == BDF_OK) f->kids.push_back(kid);
    }
    if (st == BDF_OK && n_gpus > 1) {   // ncclCommInitAll: one communicator, one rank per GPU, all in this process
        std::vector<Comm*> comms((size_t)n_gpus, nullptr);
        std::string err;
        if (comm_create_all(n_gpus, devs.data(), comms.data(), &err) != 0) st = fail(BDF_NCCL, "%s", err.c_str());
        else {
            for (int i = 0; i < n_gpus; i++) ctx_attach_comm(f->kids[i], comms[i]);
            const char* mode = getenv("BDF_COMBINE");
            if (!(mode && strcmp(mode, "nccl") == 0)) {
                std::string perr;
                if (comm_enable_p2p_all(n_gpus, comms.data(), &perr) == 0) for (Comm* cm : comms) comm_set_p2p(cm, true);
                else if (mode && strcmp(mode, "p2p") == 0) st = fail(BDF_NCCL, "BDF_COMBINE=p2p: %s", perr.c_str());
            }
        }
    }
    if (st == BDF_OK)
        for (int i = 0; i < n_gpus; i++) {
            f->workers.emplace_back(new Fleet::Worker());
            Fleet::Worker* w = f->workers.back().get();
            w->th = std::thread(fleet_worker_main, w, devs[i]);
        }
    if (st != BDF_OK) { const std::string keep = g_err; fleet_destroy(c); g_err = keep; return st; }
    *out = c;
    return BDF_OK;
}

int bdf_fleet_size(bdf_ctx* c) { return c ? (c->fleet ? (int)c->fleet->kids.size() : 1) : 0; }

int bdf_synchronize(bdf_ctx* c) {
    if (c && c->fleet) { Fleet* f = c->fleet; return fleet_run(f, [f](int k) { return bdf_synchronize(f->kids[k]); }); }
    ENTER(c);
    CK(cudaStreamSynchronize(c->s_h2d));
    CK(cudaStreamSynchronize(c->s_compute));
    CK(cudaStreamSynchronize(c->s_fin));
    CK(cudaStreamSynchronize(c->s_d2h));
    return BDF_OK;
}

int bdf_device_info(bdf_ctx* c, int32_t* sm_count, int32_t* cc_major, int32_t* cc_minor, int64_t* hbm_bytes) {
    if (c && c->fleet) {   // the first GPU's shape, the HBM of all of them
        int64_t total = 0, one = 0;
        for (bdf_ctx* k : c->fleet->kids) { TRY(bdf_device_info(k, sm_count, cc_major, cc_minor, &one)); total += one; }
        TRY(bdf_device_info(c->fleet->kids[0], sm_count, cc_major, cc_minor, &one));
        if (hbm_bytes) *hbm_bytes = total;
        return BDF_OK;
    }
    if (!c) return fail(BDF_INVALID, "null context");
    if (sm_count) *sm_count = c->sm_count;
    if (cc_major) *cc_major = c->cc_major;
    if (cc_minor) *cc_minor = c->cc_minor;
    if (hbm_bytes) *hbm_bytes = (int64_t)c->hbm_bytes;
    return BDF_OK;
}

int bdf_host_alloc(bdf_ctx* c, size_t bytes, void** out) {
    if (c && c->fleet) return bdf_host_alloc(c->fleet->kids[0], bytes, out);   // pinned memory is usable from every GPU (unified addressing)
    ENTER(c);
    if (!out) return fail(BDF_INVALID, "null out pointer");
    CK(cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault));
    return BDF_OK;
}
int bdf_host_free(bdf_ctx* c, void* p) {
    if (c && c->fleet) return bdf_host_free(c->fleet->kids[0], p);
    ENTER(c);
    if (p) CK(cudaFreeHost(p));
    return BDF_OK;
}
int bdf_host_register(bdf_ctx* c, void* p, size_t bytes) {
    if (c && c->fleet) return bdf_host_register(c->fleet->kids[0], p, bytes);
    ENTER(c);
    CK(cudaHostRegister(p, bytes, cudaHostRegisterDefault));
    return BDF_OK;
}
int bdf_host_unregister(bdf_ctx* c, void* p) {
    if (c && c->fleet) return bdf_host_unregister(c->fleet->kids[0], p);
    ENTER(c);
    CK(cudaHostUnregister(p));
    return BDF_OK;
}

// ---- multi-GPU: communicator -------------------------------------------------------------------------

int bdf_comm_unique_id(uint8_t* id) {
    if (!id) return fail(BDF_INVALID, "null id");
    std::string err;
    if (comm_unique_id(id, &err) != 0) return fail(BDF_NCCL, "%s", err.c_str());
    return BDF_OK;
}

int bdf_comm_attach(bdf_ctx* c, const uint8_t* id, int rank, int world) {
    if (c && c->fleet) return fail(BDF_INVALID, "a multi-GPU context already owns its communicator (ncclCommInitAll)");
    ENTER(c);
    if (!id || world < 1 || rank < 0 || rank >= world) return fail(BDF_INVALID, "bad communicator arguments (rank %d of %d)", rank, world);
    if (c->comm) return fail(BDF_INVALID, "the context already belongs to a communicator");
    CK(cudaStreamSynchronize(c->s_compute));
    std::string err;
    Comm* cm = comm_create(id, rank, world, &err);
    if (!cm) return fail(BDF_NCCL, "%s", err.c_str());
    c->comm = cm;
    c->collective = true;
    c->collectives = 0;
    // The combine itself can run over NVLink peer memory instead of NCCL (comm.cuh); every rank reads the same environment.
    const char* mode = getenv("BDF_COMBINE");
    if (world > 1 && !(mode && strcmp(mode, "nccl") == 0)) {
        std::string perr;
        // Default transport: the mailboxes up to 4 ranks, NCCL above unless asked for.  When it was chosen, a blocking combine
        // was cheaper over the mailboxes than over NCCL at 2 / 4 / 8 GPUs, but the pipelined weak series at 8 GPUs ran slower
        // with the mailboxes.  Not re-measured on H100 boxes.
        if (comm_enable_p2p(cm, &perr) == 0) comm_set_p2p(cm, world <= 4 || (mode && strcmp(mode, "p2p") == 0));
        else if (mode && strcmp(mode, "p2p") == 0) { comm_destroy(cm); c->comm = nullptr; return fail(BDF_NCCL, "BDF_COMBINE=p2p: %s", perr.c_str()); }
    }
    return BDF_OK;
}

int bdf_comm_set_combine(bdf_ctx* c, int mode) {
    if (c && c->fleet) { for (bdf_ctx* k : c->fleet->kids) TRY(bdf_comm_set_combine(k, mode)); return BDF_OK; }
    ENTER(c);
    if (mode != 0 && mode != 1) return fail(BDF_INVALID, "combine mode is 0 (NCCL) or 1 (peer memory)");
    if (!c->comm) return mode == 0 ? BDF_OK : fail(BDF_UNSUPPORTED, "the context is not a rank of a communicator");
    CK(cudaStreamSynchronize(c->s_compute));
    CK(cudaStreamSynchronize(c->s_fin));
    if (comm_set_p2p(c->comm, mode == 1) != 0) return fail(BDF_UNSUPPORTED, "peer-memory mailboxes are not available on this communicator");
    return BDF_OK;
}

int bdf_comm_get_combine(bdf_ctx* c) {
    if (c && c->fleet) return bdf_comm_get_combine(c->fleet->kids[0]);
    return c && c->comm && comm_uses_p2p(c->comm) ? 1 : 0;
}

int bdf_comm_detach(bdf_ctx* c) {
    if (c && c->fleet) return fail(BDF_INVALID, "the communicator of a multi-GPU context lives as long as the context");
    ENTER(c);
    if (!c->comm) return BDF_OK;
    CK(cudaStreamSynchronize(c->s_compute));
    CK(cudaStreamSynchronize(c->s_fin));
    comm_destroy(c->comm);
    c->comm = nullptr;
    return BDF_OK;
}

int bdf_comm_info(bdf_ctx* c, int32_t* rank, int32_t* world, int32_t* nccl_version, int64_t* collectives) {
    if (c && c->fleet) {
        TRY(bdf_comm_info(c->fleet->kids[0], rank, world, nccl_version, collectives));
        if (rank) *rank = 0;
        return BDF_OK;
    }
    if (!c) return fail(BDF_INVALID, "null context");
    if (rank) *rank = c->comm ? comm_rank(c->comm) : 0;
    if (world) *world = c->comm ? comm_world(c->comm) : 1;
    if (nccl_version) *nccl_version = c->comm ? comm_version() : 0;
    if (collectives) *collectives = c->collectives;
    return BDF_OK;
}

int bdf_comm_collective(bdf_ctx* c, int on) {
    if (c && c->fleet) return on ? BDF_OK : fail(BDF_UNSUPPORTED, "a multi-GPU context always returns the aggregates of the whole column");
    ENTER(c);
    c->collective = on != 0;
    return BDF_OK;
}

int bdf_comm_all_reduce_f64(bdf_ctx* c, int op, int64_t n, double* inout) {
    if (c && c->fleet) return BDF_OK;   // one process: the caller's value is already the job's value
    ENTER(c);
    if (n < 0 || (n && !inout) || (op != BDF_SUM && op != BDF_MIN && op != BDF_MAX)) return fail(BDF_INVALID, "bad arguments");
    if (!c->comm || n == 0) return BDF_OK;   // a lone GPU: the value is already the result
    std::string err;
    c->collectives++;
    cudaError_t e = comm_host_allreduce_f64(c->comm, op == BDF_SUM ? 0 : op == BDF_MIN ? 1 : 2, inout, (int)n, c->s_compute, &err);
    if (e != cudaSuccess) { g_nccl_err = err; return fail_cuda(e, "all-reduce"); }
    return BDF_OK;
}

int bdf_comm_barrier(bdf_ctx* c) {
    if (c && c->fleet) return bdf_synchronize(c);
    {
        ENTER(c);
        CK(cudaStreamSynchronize(c->s_h2d));
        CK(cudaStreamSynchronize(c->s_compute));
        CK(cudaStreamSynchronize(c->s_fin));
        CK(cudaStreamSynchronize(c->s_d2h));
    }
    double one = 1.0;
    return bdf_comm_all_reduce_f64(c, BDF_SUM, 1, &one);   // returns once every rank has arrived
}

int bdf_aggregate_all_many_dev_async(bdf_ctx* c, int32_t n_cols, const bdf_col* const* cols, bdf_future** fut) {
    NEED_CTX(c);
    if (!cols || !fut) return fail(BDF_INVALID, "null argument");
    if (c->fleet) return fleet_aggregate_many(c, n_cols, cols, fut);
    ENTER(c);
    return aggregate_many_dev_async(c, n_cols, const_cast<bdf_col* const*>(cols), false, fut);
}

int bdf_aggregate_all_many_dev(bdf_ctx* c, int32_t n_cols, const bdf_col* const* cols, bdf_agg4* out) {
    NEED_CTX(c);
    if (!cols || !out) return fail(BDF_INVALID, "null argument");
    if (c->fleet) return fleet_aggregate_all_blocking(c, n_cols, cols, out);
    ENTER(c);
    bdf_future* f = nullptr;
    TRY(aggregate_many_dev_async(c, n_cols, const_cast<bdf_col* const*>(cols), true, &f));
    return future_wait(c, f, out);
}

int bdf_future_count(const bdf_future* fut) { return fut ? fut->n : 0; }

// ---- device-resident API -----------------------------------------------------------------------

int bdf_upload(bdf_ctx* c, int dtype, int64_t n_chunks, const bdf_view* in, int flags, bdf_col** out) {
    NEED_CTX(c);
    if (dtype != kBool) TRY(check_dtype(dtype));
    if (!out || n_chunks < 0 || (n_chunks && !in)) return fail(BDF_INVALID, "bad arguments");
    if (c->fleet) {
        const int32_t dt = dtype;
        return fleet_upload_many(c, 1, &dt, &n_chunks, &in, flags, out);
    }
    ENTER(c);
    std::vector<bdf_col*> cols;
    TRY(upload_many(c, {UploadSpec{dtype, n_chunks, in}}, (flags & BDF_ASYNC) != 0, cols));
    *out = cols[0];
    return BDF_OK;
}

int bdf_upload_many(bdf_ctx* c, int64_t n_cols, const int32_t* dtypes, const int64_t* n_chunks, const bdf_view* const* in,
                    int flags, bdf_col** out) {
    NEED_CTX(c);
    if (n_cols < 0 || (n_cols && (!dtypes || !n_chunks || !in || !out))) return fail(BDF_INVALID, "bad arguments");
    for (int64_t k = 0; k < n_cols; k++) {
        if (dtypes[k] != kBool) TRY(check_dtype(dtypes[k]));
        if (n_chunks[k] < 0 || (n_chunks[k] && !in[k])) return fail(BDF_INVALID, "bad arguments for column %lld", (long long)k);
    }
    if (c->fleet) return fleet_upload_many(c, n_cols, dtypes, n_chunks, in, flags, out);
    ENTER(c);
    std::vector<UploadSpec> specs;
    for (int64_t k = 0; k < n_cols; k++) specs.push_back(UploadSpec{dtypes[k], n_chunks[k], in[k]});
    std::vector<bdf_col*> cols;
    TRY(upload_many(c, specs, (flags & BDF_ASYNC) != 0, cols));
    for (int64_t k = 0; k < n_cols; k++) out[k] = cols[k];
    return BDF_OK;
}

int bdf_col_wait(bdf_ctx* c, const bdf_col* col) {
    if (c && c->fleet) { if (!is_fleet_col(col)) return fail(BDF_INVALID, "null column"); Fleet* f = c->fleet; return fleet_run(f, [f, col](int k) { return bdf_col_wait(f->kids[k], col->fparts[k]); }); }
    ENTER(c);
    if (!col) return fail(BDF_INVALID, "null column");
    for (auto& g : col->groups) CK(cudaEventSynchronize(g.ev));
    return BDF_OK;
}

int bdf_col_describe(const bdf_col* col, int32_t* dtype, int64_t* n_chunks, int64_t* total_len) {
    if (is_fleet_col(col)) {
        if (dtype) *dtype = col->dtype;
        if (n_chunks) *n_chunks = (int64_t)col->fmap.size();
        if (total_len) *total_len = col->total_len;
        return BDF_OK;
    }
    if (!col) return fail(BDF_INVALID, "null column");
    if (dtype) *dtype = col->dtype;
    if (n_chunks) *n_chunks = (int64_t)col->chunks.size();
    if (total_len) *total_len = col->total_len;
    return BDF_OK;
}

int bdf_col_chunk_info(bdf_ctx* c, const bdf_col* col, int64_t chunk, int64_t* len, int64_t* null_count, int32_t* has_validity) {
    if (c && c->fleet) return fleet_chunk_info(c, col, chunk, len, null_count, has_validity);
    ENTER(c);
    if (!col || chunk < 0 || chunk >= (int64_t)col->chunks.size()) return fail(BDF_INVALID, "bad chunk index");
    if (len) *len = col->chunks[chunk].len;
    if (has_validity) *has_validity = col->chunks[chunk].validity != nullptr;
    if (null_count) {
        TRY(ensure_null_counts(c, const_cast<bdf_col*>(col)));
        *null_count = col->null_counts[chunk];
    }
    return BDF_OK;
}

int bdf_binary_dev(bdf_ctx* c, int op, const bdf_col* l, const bdf_col* r, bdf_col** out) {
    NEED_CTX(c);
    if (!l || !r || !out) return fail(BDF_INVALID, "null argument");
    if (Fleet* f = c->fleet)
        return fleet_map(c, l->dtype, {l, r}, out, [=](int k, bdf_col** o) { return bdf_binary_dev(f->kids[k], op, l->fparts[k], r->fparts[k], o); });
    ENTER(c);
    return binary_dev(c, op, l, r, out);
}

int bdf_unary_dev(bdf_ctx* c, int op, const bdf_col* in, bdf_col** out) {
    NEED_CTX(c);
    if (!in || !out) return fail(BDF_INVALID, "null argument");
    if (Fleet* f = c->fleet)
        return fleet_map(c, in->dtype, {in}, out, [=](int k, bdf_col** o) { return bdf_unary_dev(f->kids[k], op, in->fparts[k], o); });
    ENTER(c);
    return map_dev(c, false, op, in, out);
}

int bdf_cast_dev(bdf_ctx* c, int to, const bdf_col* in, bdf_col** out) {
    NEED_CTX(c);
    if (!in || !out) return fail(BDF_INVALID, "null argument");
    if (Fleet* f = c->fleet)
        return fleet_map(c, to, {in}, out, [=](int k, bdf_col** o) { return bdf_cast_dev(f->kids[k], to, in->fparts[k], o); });
    ENTER(c);
    return map_dev(c, true, to, in, out);
}

int bdf_temporal_result(int fn, const bdf_temporal_type* type, int64_t arg, int32_t* out_dtype, bdf_temporal_type* out_type) {
    TemporalPlan pl;
    TRY(temporal_plan(fn, type, arg, &pl));
    if (out_dtype) *out_dtype = pl.out_dtype;
    if (out_type) *out_type = pl.out_type;
    return BDF_OK;
}

int bdf_temporal_dev(bdf_ctx* c, int fn, const bdf_temporal_type* type, int64_t arg, const bdf_col* in, bdf_col** out) {
    TemporalPlan pl;
    TRY(temporal_plan(fn, type, arg, &pl));
    NEED_CTX(c);
    if (!in || !out) return fail(BDF_INVALID, "null argument");
    if (Fleet* f = c->fleet) {
        if (in->dtype != pl.in_dtype) return fail(BDF_INVALID, "a column of dtype %d does not hold this temporal type (dtype %d)", in->dtype, pl.in_dtype);
        return fleet_map(c, pl.out_dtype, {in}, out, [=](int k, bdf_col** o) { return bdf_temporal_dev(f->kids[k], fn, type, arg, in->fparts[k], o); });
    }
    ENTER(c);
    return temporal_dev(c, pl, in, out);
}

int bdf_temporal_binary_dev(bdf_ctx* c, int fn, const bdf_temporal_type* ta, const bdf_col* a, const bdf_temporal_type* tb, const bdf_col* b,
                            bdf_col** out) {
    NEED_CTX(c);
    if (!a || !b || !out) return fail(BDF_INVALID, "null argument");
    if (c->fleet) {
        if (!ta || !tb) return fail(BDF_INVALID, "null argument");
        if (fn != BDF_TEMPORAL_DATE_DIFF && fn != BDF_TEMPORAL_MONTHS_BETWEEN) return fail(BDF_INVALID, "unknown two-column temporal function %d", fn);
        int cfg = 0;
        int64_t off = 0;
        TRY(temporal_side(ta, a, &cfg, &off));
        TRY(temporal_side(tb, b, &cfg, &off));
        Fleet* f = c->fleet;
        return fleet_map(c, fn == BDF_TEMPORAL_DATE_DIFF ? BDF_I32 : BDF_F64, {a, b}, out,
                         [=](int k, bdf_col** o) { return bdf_temporal_binary_dev(f->kids[k], fn, ta, a->fparts[k], tb, b->fparts[k], o); });
    }
    ENTER(c);
    return temporal_binary_dev(c, fn, ta, a, tb, b, out);
}

int bdf_aggregate_dev(bdf_ctx* c, int op, const bdf_col* in, void* out_scalar, int32_t* is_some) {
    NEED_CTX(c);
    if (!in || !out_scalar || !is_some) return fail(BDF_INVALID, "null argument");
    if (c->fleet) return fleet_aggregate_dev(c, op, in, out_scalar, is_some);
    ENTER(c);
    return aggregate_dev(c, op, const_cast<bdf_col*>(in), out_scalar, is_some);
}

int bdf_aggregate_all_dev(bdf_ctx* c, const bdf_col* in, bdf_agg4* out) {
    NEED_CTX(c);
    if (!in || !out) return fail(BDF_INVALID, "null argument");
    if (c->fleet) return fleet_aggregate_all_blocking(c, 1, &in, out);
    ENTER(c);
    return aggregate_all_dev(c, const_cast<bdf_col*>(in), true, out);
}

int bdf_avg_dev(bdf_ctx* c, const bdf_col* in, double* out, int32_t* is_some) {
    NEED_CTX(c);
    if (!in || !out || !is_some) return fail(BDF_INVALID, "null argument");
    if (c->fleet) return fleet_avg_dev(c, in, out, is_some);
    ENTER(c);
    return avg_dev(c, const_cast<bdf_col*>(in), out, is_some);
}

int bdf_moments_dev(bdf_ctx* c, const bdf_col* in, bdf_moment_rec* out) {
    NEED_CTX(c);
    if (!in || !out) return fail(BDF_INVALID, "null argument");
    if (c->fleet) return fleet_moments_dev(c, in, out);
    ENTER(c);
    Moments m;
    TRY(moments_dev(c, in, &m));
    memcpy(out, &m, sizeof m);
    return BDF_OK;
}

int bdf_distinct_dev(bdf_ctx* c, const bdf_col* in, bdf_distinct_rec* out) {
    if (c && c->fleet)
        return fail(BDF_UNSUPPORTED, "distinct values need every row of the column on one GPU (as sort / group-by / join): use a one-GPU context");
    ENTER(c);
    if (!in || !out) return fail(BDF_INVALID, "null argument");
    return distinct_dev(c, in, out);
}

static const char* kDistFleet = "the distributions need every row of the column on one GPU: use a one-GPU context";

static int check_percentiles(int32_t n_p, const double* p, const double* out, const int32_t* is_some) {
    if (!p || !out || !is_some) return fail(BDF_INVALID, "null argument");
    if (n_p < 1 || n_p > kMaxPercentiles) return fail(BDF_INVALID, "1..%d percentiles per call", kMaxPercentiles);
    for (int32_t i = 0; i < n_p; i++)
        if (!(p[i] >= 0.0 && p[i] <= 1.0)) return fail(BDF_INVALID, "percentile %d is %g: it must be in [0, 1]", i, p[i]);
    return BDF_OK;
}

static int check_hist(int32_t nbins, const double* edges, const int64_t* counts) {
    if (!edges || !counts) return fail(BDF_INVALID, "null argument");
    if (nbins < 1 || nbins > (1 << 24)) return fail(BDF_INVALID, "nbins must be in 1..2^24, not %d", nbins);
    return BDF_OK;
}

int bdf_percentile_dev(bdf_ctx* c, const bdf_col* in, int32_t n_p, const double* p, double* out, int32_t* is_some) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "%s", kDistFleet);
    ENTER(c);
    if (!in) return fail(BDF_INVALID, "null argument");
    TRY(check_percentiles(n_p, p, out, is_some));
    std::vector<double> o((size_t)n_p);
    std::vector<int32_t> some((size_t)n_p);
    TRY(percentile_dev(c, in, n_p, p, o.data(), some.data()));
    memcpy(out, o.data(), o.size() * sizeof(double));
    memcpy(is_some, some.data(), some.size() * sizeof(int32_t));
    return BDF_OK;
}

int bdf_mode_dev(bdf_ctx* c, const bdf_col* in, uint64_t* bits, int64_t* freq, int32_t* is_some) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "%s", kDistFleet);
    ENTER(c);
    if (!in || !bits || !freq || !is_some) return fail(BDF_INVALID, "null argument");
    uint64_t b = 0;
    int64_t f = 0;
    int32_t some = 0;
    TRY(mode_dev(c, in, &b, &f, &some));
    *bits = b; *freq = f; *is_some = some;
    return BDF_OK;
}

int bdf_uniques_dev(bdf_ctx* c, const bdf_col* in, bdf_col** values, bdf_col** counts) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "%s", kDistFleet);
    ENTER(c);
    if (!in || !values) return fail(BDF_INVALID, "null argument");
    return uniques_dev(c, in, values, counts);
}

int bdf_hist_dev(bdf_ctx* c, const bdf_col* in, int32_t nbins, const double* range, double* edges, int64_t* counts) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "%s", kDistFleet);
    ENTER(c);
    if (!in) return fail(BDF_INVALID, "null argument");
    TRY(check_hist(nbins, edges, counts));
    return hist_dev(c, in, nbins, range, edges, counts);
}

int bdf_hist_density(int32_t nbins, const double* edges, const int64_t* counts, double* out) {
    TRY(check_hist(nbins, edges, counts));
    if (!out) return fail(BDF_INVALID, "null argument");
    int64_t total = 0;
    for (int32_t i = 0; i < nbins; i++) total += counts[i];
    for (int32_t i = 0; i < nbins; i++) out[i] = ((double)counts[i] / dist_sub(edges[i + 1], edges[i])) / (double)total;
    return BDF_OK;
}

int bdf_moments_stat(const bdf_moment_rec* m, int stat, double* out, int32_t* is_some) {
    if (!m || !out || !is_some) return fail(BDF_INVALID, "null argument");
    if (stat < BDF_STAT_VARIANCE || stat > BDF_STAT_KURTOSIS) return fail(BDF_INVALID, "unknown statistic %d", stat);
    Moments r;
    memcpy(&r, m, sizeof r);
    double v = 0.0;
    *is_some = moments_stat(r, stat, &v) ? 1 : 0;
    *out = v;
    return BDF_OK;
}

int bdf_moments_merge(const bdf_moment_rec* a, const bdf_moment_rec* b, bdf_moment_rec* out) {
    if (!a || !b || !out) return fail(BDF_INVALID, "null argument");
    Moments x, y;
    memcpy(&x, a, sizeof x);
    memcpy(&y, b, sizeof y);
    const Moments r = moments_merge(x, y);
    memcpy(out, &r, sizeof r);
    return BDF_OK;
}

int bdf_binary_agg_dev_async(bdf_ctx* c, int op, const bdf_col* l, const bdf_col* r, bdf_col** out, bdf_future** fut) {
    NEED_CTX(c);
    if (!l || !r || !out || !fut) return fail(BDF_INVALID, "null argument");
    if (Fleet* f = c->fleet)
        return fleet_with_future(c, l->dtype, {l, r}, true, out, fut,
                                 [=](int k, bdf_col** o, bdf_future** fu) { return bdf_binary_agg_dev_async(f->kids[k], op, l->fparts[k], r->fparts[k], o, fu); });
    ENTER(c);
    return binary_dev(c, op, l, r, out, fut);
}

int bdf_binary_agg_dev(bdf_ctx* c, int op, const bdf_col* l, const bdf_col* r, bdf_col** out, bdf_agg4* agg) {
    NEED_CTX(c);
    if (!l || !r || !out || !agg) return fail(BDF_INVALID, "null argument");
    if (c->fleet) {
        bdf_future* fu = nullptr;
        TRY(bdf_binary_agg_dev_async(c, op, l, r, out, &fu));
        return fleet_future_wait(c, fu, agg);
    }
    ENTER(c);
    bdf_future* f = nullptr;
    TRY(binary_dev(c, op, l, r, out, &f));
    return future_wait(c, f, agg);
}

int bdf_eval_expr_agg_dev_async(bdf_ctx* c, int32_t n_inputs, const bdf_col* const* inputs, int32_t n_nodes, const bdf_expr_node* nodes,
                                bdf_col** out, bdf_future** fut) {
    NEED_CTX(c);
    if (Fleet* f = c->fleet) {
        if (!inputs || !nodes || !fut || n_inputs < 1 || n_inputs > 8) return fail(BDF_INVALID, "bad arguments");
        for (int i = 0; i < n_inputs; i++) if (!is_fleet_col(inputs[i])) return fail(BDF_INVALID, "null input column");
        int64_t n = 0;
        TRY(fleet_zip(inputs, (size_t)n_inputs, BDF_INVALID, BDF_INVALID, &n));
        return fleet_with_future(c, BDF_F64, {inputs[0]}, out != nullptr, out, fut, [=](int k, bdf_col** o, bdf_future** fu) {
            const bdf_col* parts[8];
            for (int i = 0; i < n_inputs; i++) parts[i] = inputs[i]->fparts[k];
            return bdf_eval_expr_agg_dev_async(f->kids[k], n_inputs, parts, n_nodes, nodes, o, fu);
        });
    }
    ENTER(c);
    if (!inputs || !nodes || !fut) return fail(BDF_INVALID, "null argument");
    return expr_dev(c, n_inputs, inputs, n_nodes, nodes, out, fut);
}

int bdf_eval_expr_agg_dev(bdf_ctx* c, int32_t n_inputs, const bdf_col* const* inputs, int32_t n_nodes, const bdf_expr_node* nodes, bdf_col** out,
                          bdf_agg4* agg) {
    NEED_CTX(c);
    if (!agg) return fail(BDF_INVALID, "null argument");
    if (c->fleet) {
        bdf_future* fu = nullptr;
        TRY(bdf_eval_expr_agg_dev_async(c, n_inputs, inputs, n_nodes, nodes, out, &fu));
        return fleet_future_wait(c, fu, agg);
    }
    ENTER(c);
    if (!inputs || !nodes) return fail(BDF_INVALID, "null argument");
    bdf_future* f = nullptr;
    TRY(expr_dev(c, n_inputs, inputs, n_nodes, nodes, out, &f));
    return future_wait(c, f, agg);
}

int bdf_aggregate_all_dev_async(bdf_ctx* c, const bdf_col* in, bdf_future** fut) {
    NEED_CTX(c);
    if (!in || !fut) return fail(BDF_INVALID, "null argument");
    if (c->fleet) return fleet_aggregate_many(c, 1, &in, fut);
    ENTER(c);
    return aggregate_all_dev_async(c, const_cast<bdf_col*>(in), fut);
}

int bdf_future_wait(bdf_ctx* c, bdf_future* fut, bdf_agg4* out) {
    NEED_CTX(c);
    if (!fut) return fail(BDF_INVALID, "null future");
    if (c->fleet) return fleet_future_wait(c, fut, out);
    ENTER(c);
    return future_wait(c, fut, out);
}

int bdf_expr_check(int32_t n_inputs, const int32_t* input_dtypes, int32_t n_nodes, const bdf_expr_node* nodes, int32_t* n_instructions,
                   int32_t* n_temporaries) {
    if (!nodes) return fail(BDF_INVALID, "null argument");
    int dt[8];
    for (int i = 0; i < 8; i++) dt[i] = (input_dtypes && i < n_inputs) ? input_dtypes[i] : BDF_F64;
    alignas(8) unsigned char prog[256];
    bool has_div = false;
    TRY(expr_prepare(n_inputs, dt, n_nodes, nodes, prog, &has_div));
    int ni = 0, nt = 0;
    expr_prog_stats(prog, &ni, &nt);
    if (n_instructions) *n_instructions = ni;
    if (n_temporaries) *n_temporaries = nt;
    return BDF_OK;
}

int bdf_eval_expr_dev(bdf_ctx* c, int32_t n_inputs, const bdf_col* const* inputs, int32_t n_nodes, const bdf_expr_node* nodes, bdf_col** out) {
    NEED_CTX(c);
    if (Fleet* f = c->fleet) {
        if (!inputs || !nodes || !out || n_inputs < 1 || n_inputs > 8) return fail(BDF_INVALID, "bad arguments");
        for (int i = 0; i < n_inputs; i++) if (!is_fleet_col(inputs[i])) return fail(BDF_INVALID, "null input column");
        int64_t n = 0;
        TRY(fleet_zip(inputs, (size_t)n_inputs, BDF_INVALID, BDF_INVALID, &n));
        return fleet_map(c, BDF_F64, {inputs[0]}, out, [=](int k, bdf_col** o) {
            const bdf_col* parts[8];
            for (int i = 0; i < n_inputs; i++) parts[i] = inputs[i]->fparts[k];
            return bdf_eval_expr_dev(f->kids[k], n_inputs, parts, n_nodes, nodes, o);
        });
    }
    ENTER(c);
    if (!inputs || !nodes || !out) return fail(BDF_INVALID, "null argument");
    return expr_dev(c, n_inputs, inputs, n_nodes, nodes, out);
}

int bdf_sort_indices_dev(bdf_ctx* c, int32_t n_keys, const bdf_sort_key* keys, bdf_col** indices) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "sort / take / filter move rows between chunks: use a one-GPU context (bdf_init) for them");
    ENTER(c);
    if (!keys || !indices) return fail(BDF_INVALID, "null argument");
    return sort_indices_dev(c, n_keys, keys, indices);
}

int bdf_top_k_indices_dev(bdf_ctx* c, int32_t n_keys, const bdf_sort_key* keys, int64_t k, bdf_col** indices) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "sort / take / filter move rows between chunks: use a one-GPU context (bdf_init) for them");
    ENTER(c);
    if (!keys || !indices) return fail(BDF_INVALID, "null argument");
    return top_k_indices_dev(c, n_keys, keys, k, indices);
}

int bdf_group_aggregate_dev(bdf_ctx* c, const bdf_col* key, int32_t n_values, const bdf_col* const* values, bdf_col** out_keys, bdf_group_out* out,
                            int64_t* n_groups) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "group-by moves rows between chunks: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    if (!key || !out_keys || (n_values && (!values || !out))) return fail(BDF_INVALID, "null argument");
    return group_aggregate_dev(c, key, n_values, values, out_keys, out, n_groups);
}

int bdf_group_by_dev(bdf_ctx* c, int32_t n_keys, const bdf_col* const* keys, int32_t n_aggs, const bdf_group_agg* aggs, bdf_col** out_keys, bdf_col** out,
                     int64_t* n_groups) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "group-by moves rows between chunks: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    if (!keys || !out_keys || (n_aggs && (!aggs || !out))) return fail(BDF_INVALID, "null argument");
    if (n_aggs < 0 || n_aggs > 64) return fail(BDF_INVALID, "0..64 aggregations");
    return group_by_dev(c, n_keys, keys, n_aggs, aggs, out_keys, out, nullptr, n_groups);
}

int bdf_group_by_lists_dev(bdf_ctx* c, int32_t n_keys, const bdf_col* const* keys, int32_t n_aggs, const bdf_group_agg* aggs, bdf_col** out_keys,
                           bdf_col** out, bdf_list** out_lists, int64_t* n_groups) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "group-by moves rows between chunks: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    if (!keys || !out_keys || (n_aggs && (!aggs || !out || !out_lists))) return fail(BDF_INVALID, "null argument");
    if (n_aggs < 0 || n_aggs > 64) return fail(BDF_INVALID, "0..64 aggregations");
    return group_by_dev(c, n_keys, keys, n_aggs, aggs, out_keys, out, out_lists, n_groups);
}

int bdf_join_indices_dev(bdf_ctx* c, int32_t join_type, int32_t n_keys, const bdf_col* const* left_keys, const bdf_col* const* right_keys,
                         bdf_col** left_indices, bdf_col** right_indices, int64_t* n_rows) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "a join moves rows between chunks: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    if (!left_indices || (!right_indices && join_type != BDF_JOIN_LEFT_SEMI && join_type != BDF_JOIN_LEFT_ANTI)) return fail(BDF_INVALID, "null argument");
    return join_dev(c, join_type, n_keys, left_keys, right_keys, left_indices, right_indices, n_rows);
}

int bdf_join_asof_dev(bdf_ctx* c, const bdf_col* left_on, const bdf_col* right_on, int32_t n_by, const bdf_col* const* left_by,
                      const bdf_col* const* right_by, const bdf_asof_spec* spec, bdf_col** right_indices) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "a join moves rows between chunks: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return join_asof_dev(c, left_on, right_on, n_by, left_by, right_by, spec, right_indices);
}

int bdf_window_dev(bdf_ctx* c, int32_t n_partition, const bdf_col* const* partition_by, int32_t n_order, const bdf_sort_key* order_by,
                   int32_t n_calls, const bdf_window_call* calls, bdf_col** out) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "a window moves rows between chunks: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return window_dev(c, n_partition, partition_by, n_order, order_by, n_calls, calls, out);
}

int bdf_csv_open(bdf_ctx* c, const char* path, const bdf_csv_options* options, int32_t n_schema, const int32_t* schema_dtypes, bdf_csv** out) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "the CSV reader reads into one GPU: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return csv_open(c, path, options, n_schema, schema_dtypes, out);
}

int bdf_csv_describe(const bdf_csv* f, int32_t* n_columns, int64_t* n_batches, int64_t* n_rows) {
    if (!f) return fail(BDF_INVALID, "null file");
    if (n_columns) *n_columns = (int32_t)f->k;
    if (n_batches) *n_batches = (f->n_rows + f->batch - 1) / f->batch;
    if (n_rows) *n_rows = f->n_rows;
    return BDF_OK;
}

int bdf_csv_column(const bdf_csv* f, int32_t col, const char** name, int32_t* dtype, int32_t* nullable) {
    if (!f) return fail(BDF_INVALID, "null file");
    if (col < 0 || col >= (int32_t)f->k) return fail(BDF_INVALID, "column %d out of range", col);
    if (name) *name = f->names[(size_t)col].c_str();
    if (dtype) *dtype = f->dtypes[(size_t)col];
    if (nullable) *nullable = f->nullable[(size_t)col];
    return BDF_OK;
}

int bdf_csv_read(bdf_ctx* c, const bdf_csv* f, int32_t n_cols, const int32_t* cols, bdf_col** out) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "the CSV reader reads into one GPU: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return csv_read(c, f, n_cols, cols, out);
}

int bdf_csv_stats(const bdf_csv* f, int64_t* n_fields, int64_t* exact_fields, double* upload_ms) {
    if (!f) return fail(BDF_INVALID, "null file");
    if (n_fields) *n_fields = f->n_fields;
    if (exact_fields) *exact_fields = f->exact_fields;
    if (upload_ms) *upload_ms = f->upload_ms;
    return BDF_OK;
}

void bdf_csv_close(bdf_ctx* c, bdf_csv* f) {
    if (!c || !f || c->fleet) return;
    std::lock_guard<std::mutex> lock(c->mu);
    cudaSetDevice(c->device);
    csv_free(c, f);
}

int bdf_json_open(bdf_ctx* c, const char* path, const bdf_json_options* options, int32_t n_schema, const char* const* schema_names,
                  const int32_t* schema_dtypes, bdf_json** out) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "the JSON reader reads into one GPU: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return json_open(c, path, options, n_schema, schema_names, schema_dtypes, out);
}

int bdf_json_describe(const bdf_json* f, int32_t* n_columns, int64_t* n_batches, int64_t* n_rows) {
    if (!f) return fail(BDF_INVALID, "null file");
    if (n_columns) *n_columns = (int32_t)f->names.size();
    if (n_batches) *n_batches = (f->n_rows + f->batch - 1) / f->batch;
    if (n_rows) *n_rows = f->n_rows;
    return BDF_OK;
}

int bdf_json_column(const bdf_json* f, int32_t col, const char** name, int32_t* dtype, int32_t* nullable) {
    if (!f) return fail(BDF_INVALID, "null file");
    if (col < 0 || col >= (int32_t)f->names.size()) return fail(BDF_INVALID, "column %d out of range", col);
    if (name) *name = f->names[(size_t)col].c_str();
    if (dtype) *dtype = f->dtypes[(size_t)col];
    if (nullable) *nullable = f->nullable[(size_t)col];
    return BDF_OK;
}

int bdf_json_read(bdf_ctx* c, const bdf_json* f, int32_t n_cols, const int32_t* cols, bdf_col** out) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "the JSON reader reads into one GPU: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return json_read(c, f, n_cols, cols, out);
}

int bdf_json_read_list(bdf_ctx* c, const bdf_json* f, int32_t col, bdf_list** out) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "the JSON reader reads into one GPU: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return json_read_list(c, f, col, out);
}

int bdf_json_stats(const bdf_json* f, int64_t* n_members, int64_t* exact_fields, double* upload_ms) {
    if (!f) return fail(BDF_INVALID, "null file");
    if (n_members) *n_members = f->n_members;
    if (exact_fields) *exact_fields = f->exact_fields;
    if (upload_ms) *upload_ms = f->upload_ms;
    return BDF_OK;
}

void bdf_json_close(bdf_ctx* c, bdf_json* f) {
    if (!c || !f || c->fleet) return;
    std::lock_guard<std::mutex> lock(c->mu);
    cudaSetDevice(c->device);
    json_free(c, f);
}

int bdf_parquet_read(bdf_ctx* c, const bdf_parquet* f, int32_t n_cols, const int32_t* cols, bdf_col** out) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "the Parquet reader reads into one GPU: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return parquet_read(c, f, n_cols, cols, out);
}

// ---------------------------------------------------------------------------------------------------
// JSON writer (k_json_write.cu; the rules are in include/b200df.h).  A list row has no longest text, so the rows go in WINDOWS of at
// most kJsonwMaxRows rows and kJsonwElems list elements (one row at least): the window's elements and rows are measured and
// scanned, and its text is cut into blocks that fill a text buffer (a row longer than the buffer is a block in a buffer of its own).
// As in the CSV writer, block k is formatted into one of two fixed buffers while block k-1 crosses PCIe to the file (FileSink).

static constexpr size_t kJsonwText = (size_t)64 << 20;        // bytes of each of the two device text buffers
static constexpr int64_t kJsonwMaxRows = (int64_t)1 << 21;    // rows per window
static constexpr int64_t kJsonwElems = (int64_t)1 << 23;      // list elements per window, unless one row has more
static constexpr int kJsonwMaxCuts = 4096;                    // blocks per window (a window with more ends at the last one)

// A column name as serde_json writes a string, and the ':' after it.
static std::string jsonw_name(const char* s) {
    std::string o = "\"";
    for (; *s; s++) {
        const unsigned char ch = (unsigned char)*s;
        switch (ch) {
            case '"': o += "\\\""; break;
            case '\\': o += "\\\\"; break;
            case '\b': o += "\\b"; break;
            case '\f': o += "\\f"; break;
            case '\n': o += "\\n"; break;
            case '\r': o += "\\r"; break;
            case '\t': o += "\\t"; break;
            default:
                if (ch < 0x20) {
                    char buf[8];
                    snprintf(buf, sizeof buf, "\\u%04x", ch);
                    o += buf;
                } else {
                    o += (char)ch;
                }
        }
    }
    return o + "\":";
}

// The temporal text of column j (types[j]): its JsonwCol fields, or BDF_INVALID / BDF_UNSUPPORTED as the temporal functions refuse.
static int jsonw_temporal(const bdf_temporal_type* t, const bdf_col* col, const char* name, JsonwCol* jc) {
    int dtype = 0, cfg = 0;
    TRY(temporal_storage(t, &dtype, &cfg));
    if (col->dtype != dtype) return fail(BDF_INVALID, "column '%s' of dtype %d does not hold temporal kind %d", name, col->dtype, t->kind);
    int64_t off_sec = 0;
    if (t->kind == BDF_TIMESTAMP && !temporal_tz_offset(t->tz, &off_sec))
        return fail(BDF_UNSUPPORTED, "column '%s': time zone '%s' is not a fixed offset: named zones need a tz database the device does not have", name, t->tz);
    const int64_t ups = temporal_per_sec(cfg);
    jc->ups = ups;
    jc->upd = cfg == TC_DAYS ? 1 : 86400 * ups;
    jc->off = off_sec * ups;
    jc->frac = t->kind == BDF_DATE32 || t->kind == BDF_DATE64 ? 0 : 3 * t->unit;
    jc->tkind = t->kind == BDF_DATE32 || t->kind == BDF_DATE64 ? JT_DATE : t->kind == BDF_TIMESTAMP ? JT_TIMESTAMP : JT_TIME;
    if (t->kind == BDF_TIMESTAMP && t->tz) {
        const bool utc = !strcmp(t->tz, "UTC") || !strcmp(t->tz, "Z") || !strcmp(t->tz, "+00:00");
        const char* sfx = utc ? "Z" : t->tz;   // a fixed offset is 6 bytes (temporal_tz_offset)
        jc->suffix_len = (int32_t)strlen(sfx);
        memcpy(jc->suffix, sfx, (size_t)jc->suffix_len);
    }
    return BDF_OK;
}

// Every date of a temporal column must lie in chrono's range and every time of day in [0, one day): its min and max decide.
static int jsonw_check_range(bdf_ctx* c, const bdf_col* col, const JsonwCol& jc, const char* name) {
    const int64_t n = (int64_t)col->chunks.size();
    if (col->total_len == 0) return BDF_OK;
    wait_groups(c->s_compute, col, 0, n);
    TRY(reduce_range(c, col, 0, n, c->h_agg_dev));
    CK(cudaStreamSynchronize(c->s_compute));
    const AggDev a = c->h_agg[0];
    if (a.count == 0) return BDF_OK;
    const int64_t lo = (int64_t)(a.min_bits ^ (1ull << 63)), hi = (int64_t)(a.max_bits ^ (1ull << 63));   // k_reduce's sign-flipped keys
    if (jc.tkind == JT_TIME) {
        if (lo < 0) return fail(BDF_INVALID, "column '%s': the time of day %lld is outside [0, %lld)", name, (long long)lo, (long long)jc.upd);
        if (hi >= jc.upd) return fail(BDF_INVALID, "column '%s': the time of day %lld is outside [0, %lld)", name, (long long)hi, (long long)jc.upd);
        return BDF_OK;
    }
    for (const int64_t v : {lo, hi}) {
        int64_t days = 0, tod = 0;
        jsonf_split(v, jc.tkind, jc.upd, jc.off, days, tod);
        if (days < kMinDay || days > kMaxDay)
            return fail(BDF_INVALID, "column '%s': the value %lld is a date outside chrono's range (years -262144 ..= 262143)", name, (long long)v);
    }
    return BDF_OK;
}

static int json_write(bdf_ctx* c, const char* path, int n_cols, const char* const* names, const bdf_col* const* cols, const bdf_temporal_type* types,
                      const bdf_list* const* lists, const bdf_json_write_options* opt) {
    if (!path || !names || !cols) return fail(BDF_INVALID, "null argument");
    if (n_cols <= 0) return fail(BDF_INVALID, "no columns to write");
    std::vector<JsonwCol> jcols((size_t)n_cols);
    std::vector<int32_t> list_cols;
    std::string name_text;
    int64_t n_chunks = -1;
    auto chunk_rows = [&](int j, int64_t b) { return lists && lists[j] ? lists[j]->lens[(size_t)b] : cols[j]->chunks[(size_t)b].len; };
    for (int j = 0; j < n_cols; j++) {
        const bdf_list* l = lists ? lists[j] : nullptr;
        if (!names[j] || (l ? cols[j] != nullptr : cols[j] == nullptr))
            return fail(BDF_INVALID, "column %d: null column or name, or both a column and a list", j);
        const bdf_col* col = l ? l->values : cols[j];
        if (!col->fparts.empty()) return fail(BDF_INVALID, "a column of a multi-GPU context was passed to a one-GPU context");
        JsonwCol& jc = jcols[(size_t)j];
        jc = JsonwCol{};
        jc.list = -1;
        jc.dtype = col->dtype;
        if (l) {
            if (types && types[j].kind) return fail(BDF_INVALID, "list column '%s' cannot carry a temporal type", names[j]);
            jc.list = (int32_t)list_cols.size();
            list_cols.push_back(j);
        } else if (!((col->dtype >= 0 && col->dtype < BDF_NTYPES) || col->dtype == kBool)) {
            return fail(BDF_UNSUPPORTED, "column '%s': dtype %d", names[j], col->dtype);
        } else if (types && types[j].kind) {
            TRY(jsonw_temporal(&types[j], col, names[j], &jc));
        }
        const int64_t nc = l ? (int64_t)l->lens.size() : (int64_t)col->chunks.size();
        if (n_chunks < 0) n_chunks = nc;
        if (nc != n_chunks)
            return fail(BDF_LENGTH_MISMATCH, "columns have different numbers of chunks (%lld, %lld)", (long long)nc, (long long)n_chunks);
        for (int64_t b = 0; b < nc; b++)
            if (chunk_rows(j, b) != chunk_rows(0, b))
                return fail(BDF_LENGTH_MISMATCH, "chunk %lld: column '%s' has %lld rows, column '%s' has %lld", (long long)b, names[j],
                            (long long)chunk_rows(j, b), names[0], (long long)chunk_rows(0, b));
        const std::string nm = jsonw_name(names[j]);
        jc.name_at = (int32_t)name_text.size();
        jc.name_len = (int32_t)nm.size();
        name_text += nm;
    }
    const int n_lists = (int)list_cols.size();
    std::vector<long long> starts((size_t)n_chunks + 1, 0);
    std::vector<JsonwDesc> descs((size_t)n_chunks * n_cols);
    std::vector<long long> estart((size_t)n_cols, 0);
    for (int64_t b = 0; b < n_chunks; b++) {
        starts[b + 1] = starts[b] + chunk_rows(0, b);
        for (int j = 0; j < n_cols; j++) {
            const bdf_list* l = lists ? lists[j] : nullptr;
            const DevChunk& ch = l ? l->values->chunks[(size_t)b] : cols[j]->chunks[(size_t)b];
            JsonwDesc& d = descs[b * n_cols + j];
            d = JsonwDesc{ch.values, ch.validity, nullptr, nullptr, 0, ch.bit_off, ch.val_bit_off};
            if (l) {
                d.loffs = l->off[(size_t)b];
                d.lvalid = l->valid[(size_t)b];
                d.estart = estart[(size_t)j];
                estart[(size_t)j] += ch.len;
            }
        }
    }
    const int64_t rows = starts[(size_t)n_chunks];
    for (int j = 0; j < n_cols; j++) {   // before the file is touched: a refused value leaves it as it was
        const bdf_col* col = lists && lists[j] ? lists[j]->values : cols[j];
        wait_groups(c->s_compute, col, 0, (int64_t)col->chunks.size());
        if (jcols[(size_t)j].tkind != JT_NONE) TRY(jsonw_check_range(c, col, jcols[(size_t)j], names[j]));
    }

    const int fd = open(path, O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
    if (fd < 0) return fail(BDF_INVALID, "cannot create %s: %s", path, strerror(errno));
    struct FdGuard { int fd; ~FdGuard() { if (fd >= 0) close(fd); } } fdg{fd};
    auto finish = [&]() {
        const int fdv = fdg.fd;
        fdg.fd = -1;
        if (close(fdv) != 0) return fail(BDF_INVALID, "closing %s failed: %s", path, strerror(errno));
        return (int)BDF_OK;
    };
    if (rows == 0) return finish();

    TRY(ensure_stage(c));
    // the column tables in one buffer: descriptors, columns, chunk starts, list columns, names, the window plan
    const int cut_stride = 2 + n_lists;
    const size_t plan_n = 2 + 2 * (size_t)n_lists, cuts_n = 1 + (size_t)(kJsonwMaxCuts + 1) * cut_stride;
    auto al = [](size_t x) { return (x + 15) & ~(size_t)15; };
    const size_t o_cols = al(descs.size() * sizeof(JsonwDesc)), o_starts = o_cols + al(jcols.size() * sizeof(JsonwCol));
    const size_t o_lists = o_starts + al(starts.size() * sizeof(long long)), o_names = o_lists + al(list_cols.size() * sizeof(int32_t) + 4);
    const size_t o_plan = o_names + al(name_text.size() + 1), o_cuts = o_plan + al(plan_n * sizeof(long long)), meta_bytes = o_cuts + cuts_n * sizeof(long long);
    std::vector<char> hmeta(o_plan, 0);
    memcpy(hmeta.data(), descs.data(), descs.size() * sizeof(JsonwDesc));
    memcpy(hmeta.data() + o_cols, jcols.data(), jcols.size() * sizeof(JsonwCol));
    memcpy(hmeta.data() + o_starts, starts.data(), starts.size() * sizeof(long long));
    if (n_lists) memcpy(hmeta.data() + o_lists, list_cols.data(), list_cols.size() * sizeof(int32_t));
    memcpy(hmeta.data() + o_names, name_text.data(), name_text.size());

    Scratch<char> meta;
    Scratch<char> text[2];
    Scratch<unsigned long long> lens, sums, elens_fixed, esums_fixed;
    Scratch<long long> lpos;
    cudaError_t e = meta.alloc(c, meta_bytes);
    if (e == cudaSuccess) e = text[0].alloc(c, kJsonwText);
    if (e == cudaSuccess) e = text[1].alloc(c, kJsonwText);
    if (e == cudaSuccess) e = lens.alloc(c, (size_t)(kJsonwMaxRows + 1) * sizeof(unsigned long long));
    if (e == cudaSuccess) e = sums.alloc(c, (size_t)scan_tile_sums(kJsonwMaxRows) * sizeof(unsigned long long));
    if (e == cudaSuccess && n_lists) e = elens_fixed.alloc(c, (size_t)(kJsonwElems + 1) * sizeof(unsigned long long));
    if (e == cudaSuccess && n_lists) e = esums_fixed.alloc(c, (size_t)scan_tile_sums(kJsonwElems) * sizeof(unsigned long long));
    if (e == cudaSuccess && n_lists) e = lpos.alloc(c, (size_t)n_lists * kJsonwMaxRows * sizeof(long long));
    // pageable source: the copy has read it when it returns
    if (e == cudaSuccess) e = cudaMemcpyAsync(meta.get(), hmeta.data(), hmeta.size(), cudaMemcpyHostToDevice, c->s_compute);
    if (e != cudaSuccess) return fail_cuda(e, "JSON write setup");
    std::unique_ptr<Scratch<unsigned long long>> elens_big, esums_big;   // the elements of a row longer than the window's cap
    std::unique_ptr<Scratch<char>> text_big;                             // the text of a row longer than a text buffer
    int64_t elem_cap = kJsonwElems;
    size_t big_cap = 0;
    unsigned long long* elens = elens_fixed.get();
    unsigned long long* esums = esums_fixed.get();
    struct Pinned { long long* p = nullptr; ~Pinned() { if (p) cudaFreeHost(p); } } hp;
    struct Events { bdf_ctx* c; cudaEvent_t ev[4] = {}; ~Events() { for (auto x : ev) ev_put(c, x); } } evs{c};
    CK(cudaHostAlloc((void**)&hp.p, (plan_n + cuts_n) * sizeof(long long), cudaHostAllocDefault));
    for (auto& x : evs.ev) CK(ev_get(c, &x));
    cudaEvent_t* ev_emit = evs.ev;       // block k's text is complete in its buffer
    cudaEvent_t* ev_d2h = evs.ev + 2;    // block k's text has left its buffer
    // Declared after the buffers, so it runs first on every exit: no copy may still read a text buffer when it is freed.
    struct DrainD2H { cudaStream_t s; ~DrainD2H() { cudaStreamSynchronize(s); } } drain_guard{c->s_d2h};

    JsonwArgs a;
    a.desc = (const JsonwDesc*)meta.get();
    a.cols = (const JsonwCol*)(meta.get() + o_cols);
    a.chunk_start = (const long long*)(meta.get() + o_starts);
    a.list_cols = (const int32_t*)(meta.get() + o_lists);
    a.names = meta.get() + o_names;
    a.plan = (long long*)(meta.get() + o_plan);
    a.n_cols = n_cols; a.n_chunks = (int)n_chunks; a.n_lists = n_lists; a.explicit_nulls = opt && opt->explicit_nulls ? 1 : 0;
    long long* d_cuts = (long long*)(meta.get() + o_cuts);
    long long* h_plan = hp.p;
    long long* h_cuts = hp.p + plan_n;

    FileSink sink{c, fd, path, 0, {}};
    struct Block { const char* text; size_t bytes; int b; };
    Block prev{nullptr, 0, 0};
    bool have_prev = false;
    auto put_prev = [&]() -> int {
        if (!have_prev) return BDF_OK;
        have_prev = false;
        return sink.put(prev.text, prev.bytes, ev_emit[prev.b], ev_d2h[prev.b]);
    };
    int64_t k = 0;   // blocks so far
    for (int64_t w0 = 0; w0 < rows;) {
        TRY(put_prev());
        int64_t w1 = std::min<int64_t>(rows, w0 + kJsonwMaxRows), n_el = 0;
        if (n_lists) {
            {
                LaunchTimer t(c, BDF_K_JSON_WRITE, -1, 1, 0);
                CK(launch_jsonw_window(a, w0, rows, kJsonwMaxRows, kJsonwElems, c->s_compute));
            }
            CK(cudaMemcpyAsync(h_plan, a.plan, plan_n * sizeof(long long), cudaMemcpyDeviceToHost, c->s_compute));
            CK(cudaStreamSynchronize(c->s_compute));
            w1 = h_plan[0];
            n_el = h_plan[1];
            if (n_el > elem_cap) {   // one row with more elements than the cap: buffers of its size (freed in stream order)
                elens_big.reset(new Scratch<unsigned long long>());
                esums_big.reset(new Scratch<unsigned long long>());
                e = elens_big->alloc(c, (size_t)(n_el + 1) * sizeof(unsigned long long));
                if (e == cudaSuccess) e = esums_big->alloc(c, (size_t)scan_tile_sums(n_el) * sizeof(unsigned long long));
                if (e != cudaSuccess) return fail_cuda(e, "JSON write: the elements of a long list");
                elens = elens_big->get(); esums = esums_big->get(); elem_cap = n_el;
            }
            if (n_el > 0) {
                {
                    LaunchTimer t(c, BDF_K_JSON_WRITE, BDF_U64, n_el, n_el * 8);
                    CK(launch_jsonw_elem_len(a, n_el, elens, esums, c->s_compute));
                }
                LaunchTimer t(c, BDF_K_JSON_WRITE, BDF_U32, n_el, n_el * 16);
                c->launches += kScanSumsLaunches - 1;
                CK(launch_scan_sums(elens, n_el, esums, c->s_compute));
            }
        }
        const int64_t wn = w1 - w0;
        {
            LaunchTimer t(c, BDF_K_JSON_WRITE, BDF_U64, wn, wn * 8);
            CK(launch_jsonw_measure(a, w0, wn, elens, lens, sums, c->s_compute));
        }
        {
            LaunchTimer t(c, BDF_K_JSON_WRITE, BDF_U32, wn, wn * 16);
            c->launches += kScanSumsLaunches - 1;
            CK(launch_scan_sums(lens, wn, sums, c->s_compute));
        }
        {
            LaunchTimer t(c, BDF_K_JSON_WRITE, -1, 1, 0);
            CK(launch_jsonw_cut(a, w0, wn, lens, kJsonwText, kJsonwMaxCuts, d_cuts, c->s_compute));
        }
        CK(cudaMemcpyAsync(h_cuts, d_cuts, cuts_n * sizeof(long long), cudaMemcpyDeviceToHost, c->s_compute));
        CK(cudaStreamSynchronize(c->s_compute));
        const int64_t nb = h_cuts[0];
        for (int64_t q = 0; q < nb; q++) {
            const long long* ce = h_cuts + 1 + q * cut_stride;
            const long long* cn = ce + cut_stride;
            const int64_t r0 = w0 + ce[0], r1 = w0 + cn[0];
            const unsigned long long base = (unsigned long long)ce[1];
            const size_t bytes = (size_t)(cn[1] - ce[1]);
            const int b = (int)(k & 1);
            char* out = text[b].get();
            if (bytes > kJsonwText) {   // one row longer than a text buffer
                TRY(put_prev());
                // An earlier long row's text may still be crossing out of text_big.  Every copy queued so far precedes block k-1's
                // `left` event on the copy stream (its put is done: just above, or at the start of this window), so the emit waits on it.
                if (k >= 1) CK(cudaStreamWaitEvent(c->s_compute, ev_d2h[prev.b], 0));
                if (bytes > big_cap) {
                    CK(cudaStreamSynchronize(c->s_d2h));   // the last long row's text has left its buffer
                    text_big.reset(new Scratch<char>());
                    e = text_big->alloc(c, bytes);
                    if (e != cudaSuccess) return fail_cuda(e, "JSON write: the text of a long row");
                    big_cap = bytes;
                }
                out = text_big->get();
            }
            if (k >= 2) CK(cudaStreamWaitEvent(c->s_compute, ev_d2h[b], 0));
            {
                LaunchTimer t(c, BDF_K_JSON_WRITE, BDF_U8, r1 - r0, (int64_t)bytes);
                CK(launch_jsonw_emit(a, w0, r0, r1, lens, base, elens, lpos.get(), kJsonwMaxRows, out, c->s_compute));
            }
            for (int L = 0; L < n_lists; L++) {
                if (cn[2 + L] <= ce[2 + L]) continue;
                LaunchTimer t(c, BDF_K_JSON_WRITE, BDF_U8, cn[2 + L] - ce[2 + L], 0);
                CK(launch_jsonw_elem_emit(a, L, ce[2 + L], cn[2 + L], w0, elens, lpos.get(), kJsonwMaxRows, base, out, c->s_compute));
            }
            CK(cudaEventRecord(ev_emit[b], c->s_compute));
            TRY(put_prev());   // block k-1 crosses while block k is formatted
            prev = Block{out, bytes, b};
            have_prev = true;
            k++;
        }
        w0 += h_cuts[1 + nb * cut_stride];
    }
    TRY(put_prev());
    TRY(sink.flush());
    return finish();
}

int bdf_csv_write(bdf_ctx* c, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols,
                  const bdf_csv_write_options* options) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "the CSV writer writes from one GPU: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return csv_write(c, path, n_cols, names, cols, options);
}

int bdf_json_write(bdf_ctx* c, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols, const bdf_temporal_type* types,
                   const bdf_list* const* lists, const bdf_json_write_options* options) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "the JSON writer writes from one GPU: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return json_write(c, path, n_cols, names, cols, types, lists, options);
}

int bdf_parquet_write(bdf_ctx* c, const char* path, int32_t n_cols, const char* const* names, const bdf_col* const* cols, const bdf_temporal_type* types,
                      const bdf_parquet_write_options* options) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "the Parquet writer writes from one GPU: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return parquet_write(c, path, n_cols, names, cols, types, options);
}

int bdf_take_dev(bdf_ctx* c, const bdf_col* values, const bdf_col* indices, bdf_col** out) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "sort / take / filter move rows between chunks: use a one-GPU context (bdf_init) for them");
    ENTER(c);
    if (!values || !indices || !out) return fail(BDF_INVALID, "null argument");
    return take_dev(c, values, indices, out);
}

int bdf_compare_dev(bdf_ctx* c, int op, const bdf_col* left, const bdf_col* right, double scalar, bdf_col** out) {
    if (c && c->fleet) {
        if (!left || !out) return fail(BDF_INVALID, "null argument");
        Fleet* f = c->fleet;
        if (right) return fleet_map(c, kBool, {left, right}, out, [=](int k, bdf_col** o) { return bdf_compare_dev(f->kids[k], op, left->fparts[k], right->fparts[k], scalar, o); });
        return fleet_map(c, kBool, {left}, out, [=](int k, bdf_col** o) { return bdf_compare_dev(f->kids[k], op, left->fparts[k], nullptr, scalar, o); });
    }
    ENTER(c);
    if (!left || !out) return fail(BDF_INVALID, "null argument");
    return compare_dev(c, op, left, right, scalar, out);
}

int bdf_boolean_dev(bdf_ctx* c, int op, const bdf_col* a, const bdf_col* b, bdf_col** out) {
    if (c && c->fleet) {
        if (!a || !out) return fail(BDF_INVALID, "null argument");
        Fleet* f = c->fleet;
        if (b && op != BDF_NOT) return fleet_map(c, kBool, {a, b}, out, [=](int k, bdf_col** o) { return bdf_boolean_dev(f->kids[k], op, a->fparts[k], b->fparts[k], o); });
        return fleet_map(c, kBool, {a}, out, [=](int k, bdf_col** o) { return bdf_boolean_dev(f->kids[k], op, a->fparts[k], nullptr, o); });
    }
    ENTER(c);
    if (!a || !out) return fail(BDF_INVALID, "null argument");
    return boolean_dev(c, op, a, b, out);
}

// A row-wise call on a multi-GPU context: the checks once, then the same call on every GPU's parts.
static int fleet_cond(bdf_ctx* c, int fn, int32_t n_conds, const bdf_col* const* conds, int32_t n_vals, const bdf_arg* vals, bdf_col** out) {
    int dtype = 0;
    TRY(cond_check(fn, n_conds, conds, n_vals, vals, &dtype));
    const std::vector<const bdf_col*> cols = cond_columns(n_conds, conds, n_vals, vals);
    Fleet* f = c->fleet;
    return fleet_map(c, dtype, cols.data(), cols.size(), out, [&](int k, bdf_col** o) {
        std::vector<const bdf_col*> kc((size_t)n_conds);
        std::vector<bdf_arg> kv(vals, vals + n_vals);
        for (int32_t j = 0; j < n_conds; j++) kc[j] = conds[j]->fparts[k];
        for (auto& v : kv)
            if (v.column) v.column = v.column->fparts[k];
        return n_conds ? bdf_case_when_dev(f->kids[k], n_conds, kc.data(), kv.data(), o) : bdf_rowwise_dev(f->kids[k], fn, n_vals, kv.data(), o);
    });
}

int bdf_rowwise_dev(bdf_ctx* c, int fn, int32_t n_args, const bdf_arg* args, bdf_col** out) {
    NEED_CTX(c);
    if (!args || !out) return fail(BDF_INVALID, "null argument");
    if (fn < BDF_ROW_COALESCE || fn > BDF_ROW_NANVL) return fail(BDF_INVALID, "invalid row-wise function %d", fn);
    const int lo = fn == BDF_ROW_COALESCE ? 1 : 2, hi = fn == BDF_ROW_NANVL ? 2 : kCondMaxArgs;
    if (n_args < lo || n_args > hi) return fail(BDF_INVALID, "this function takes %d..%d arguments, not %d", lo, hi, (int)n_args);
    if (c->fleet) return fleet_cond(c, fn, 0, nullptr, n_args, args, out);
    ENTER(c);
    return cond_dev(c, fn, 0, nullptr, n_args, args, out);
}

int bdf_case_when_dev(bdf_ctx* c, int32_t n_branches, const bdf_col* const* conditions, const bdf_arg* values, bdf_col** out) {
    NEED_CTX(c);
    if (!conditions || !values || !out) return fail(BDF_INVALID, "null argument");
    if (n_branches < 1 || n_branches > kCondMaxArgs) return fail(BDF_INVALID, "case_when takes 1..%d branches, not %d", kCondMaxArgs, (int)n_branches);
    if (c->fleet) return fleet_cond(c, BDF_ROW_COALESCE, n_branches, conditions, n_branches + 1, values, out);
    ENTER(c);
    return cond_dev(c, BDF_ROW_COALESCE, n_branches, conditions, n_branches + 1, values, out);
}

int bdf_null_test_dev(bdf_ctx* c, int fn, const bdf_col* in, bdf_col** out) {
    NEED_CTX(c);
    if (!in || !out) return fail(BDF_INVALID, "null argument");
    if (fn < BDF_IS_NULL || fn > BDF_IS_NAN) return fail(BDF_INVALID, "invalid null test %d", fn);
    if (Fleet* f = c->fleet)
        return fleet_map(c, kBool, {in}, out, [=](int k, bdf_col** o) { return bdf_null_test_dev(f->kids[k], fn, in->fparts[k], o); });
    ENTER(c);
    return null_test_dev(c, fn, in, out);
}

int bdf_filter_dev(bdf_ctx* c, const bdf_col* values, const bdf_col* mask, bdf_col** out) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "sort / take / filter move rows between chunks: use a one-GPU context (bdf_init) for them");
    ENTER(c);
    if (!values || !mask || !out) return fail(BDF_INVALID, "null argument");
    return filter_dev(c, values, mask, out);
}

static int download_entry(bdf_ctx* c, const bdf_col* col, bdf_out* out, int phase /* 0 both, 1 begin, 2 end */) {
    NEED_CTX(c);
    if (c->fleet) {
        if (!is_fleet_col(col) || (!out && !col->fmap.empty())) return fail(BDF_INVALID, "null argument");
        return fleet_download(c, col, out, phase);
    }
    ENTER(c);
    if (!col || (!out && !col->chunks.empty())) return fail(BDF_INVALID, "null argument");
    if (phase == 1) return download_enqueue(c, const_cast<bdf_col*>(col), out);
    if (phase == 2) return download_finish(c, const_cast<bdf_col*>(col), out);
    return download(c, const_cast<bdf_col*>(col), out);
}

int bdf_download_begin(bdf_ctx* c, const bdf_col* col, bdf_out* out) { return download_entry(c, col, out, 1); }
int bdf_download_end(bdf_ctx* c, const bdf_col* col, bdf_out* out) { return download_entry(c, col, out, 2); }
int bdf_download(bdf_ctx* c, const bdf_col* col, bdf_out* out) { return download_entry(c, col, out, 0); }

void bdf_col_free(bdf_ctx* c, bdf_col* col) {
    if (c && c->fleet) { fleet_col_free(c->fleet, col); return; }
    if (!c || !col) return;
    std::lock_guard<std::mutex> lock(c->mu);
    cudaSetDevice(c->device);
    col_release(c, col);
}

// ---- host in / host out ------------------------------------------------------------------------

int bdf_binary(bdf_ctx* c, int op, int dtype, int64_t n_left, const bdf_view* left, int64_t n_right, const bdf_view* right, bdf_out* out) {
    NEED_CTX(c);
    if (c->fleet && !out && std::min(n_left, n_right) > 0) return fail(BDF_INVALID, "bad arguments");
    TRY(check_dtype(dtype));
    if (n_left < 0 || n_right < 0 || (n_left && !left) || (n_right && !right)) return fail(BDF_INVALID, "bad arguments");
    const int64_t n = std::min(n_left, n_right);
    if (c->fleet)
        return fleet_host_map(c, {left, right}, n, dtype, out, [=](bdf_ctx* kid, int64_t m, const bdf_view* const* v, bdf_out* o) {
            return bdf_binary(kid, op, dtype, m, v[0], m, v[1], o);
        });
    ENTER(c);
    for (int64_t i = 0; i < n; i++)  // reject before moving a byte
        if (left[i].len != right[i].len) return fail(BDF_LENGTH_MISMATCH, "Cannot perform math operation on arrays of different length");
    return host_call(c, {UploadSpec{dtype, n, left}, UploadSpec{dtype, n, right}}, [&](bdf_col* const* in) {
        ColOwner o(c);
        TRY(binary_dev(c, op, in[0], in[1], o.out()));
        return download(c, o.get(), out);
    });
}

static int map_host(bdf_ctx* c, bool is_cast, int op_or_to, int dtype, int64_t n, const bdf_view* in, bdf_out* out) {
    NEED_CTX(c);
    if (c->fleet && is_cast) TRY(check_dtype(op_or_to));
    TRY(check_dtype(dtype));
    if (n < 0 || (n && !in)) return fail(BDF_INVALID, "bad arguments");
    if (c->fleet)
        return fleet_host_map(c, {in}, n, is_cast ? op_or_to : dtype, out, [=](bdf_ctx* kid, int64_t m, const bdf_view* const* v, bdf_out* o) {
            return is_cast ? bdf_cast(kid, dtype, op_or_to, m, v[0], o) : bdf_unary(kid, op_or_to, dtype, m, v[0], o);
        });
    ENTER(c);
    return host_call(c, {UploadSpec{dtype, n, in}}, [&](bdf_col* const* cols) {
        ColOwner o(c);
        TRY(map_dev(c, is_cast, op_or_to, cols[0], o.out()));
        return download(c, o.get(), out);
    });
}

int bdf_unary(bdf_ctx* c, int op, int dtype, int64_t n, const bdf_view* in, bdf_out* out) { return map_host(c, false, op, dtype, n, in, out); }

int bdf_cast(bdf_ctx* c, int from, int to, int64_t n, const bdf_view* in, bdf_out* out) { return map_host(c, true, to, from, n, in, out); }

int bdf_temporal(bdf_ctx* c, int fn, const bdf_temporal_type* type, int64_t arg, int64_t n, const bdf_view* in, bdf_out* out) {
    NEED_CTX(c);
    TemporalPlan pl;
    TRY(temporal_plan(fn, type, arg, &pl));
    if (n < 0 || (n && (!in || !out))) return fail(BDF_INVALID, "bad arguments");
    if (c->fleet)
        return fleet_host_map(c, {in}, n, pl.out_dtype, out, [=](bdf_ctx* kid, int64_t m, const bdf_view* const* v, bdf_out* o) {
            return bdf_temporal(kid, fn, type, arg, m, v[0], o);
        });
    ENTER(c);
    return host_call(c, {UploadSpec{pl.in_dtype, n, in}}, [&](bdf_col* const* cols) {
        ColOwner o(c);
        TRY(temporal_dev(c, pl, cols[0], o.out()));
        return download(c, o.get(), out);
    });
}

int bdf_aggregate(bdf_ctx* c, int op, int dtype, int64_t n, const bdf_view* in, void* out_scalar, int32_t* is_some) {
    NEED_CTX(c);
    if (c->fleet && (!out_scalar || !is_some)) return fail(BDF_INVALID, "bad arguments");
    TRY(check_dtype(dtype));
    if (n < 0 || (n && !in) || !out_scalar || !is_some) return fail(BDF_INVALID, "bad arguments");
    if (c->fleet) return fleet_host_reduce(c, dtype, n, in, [&](const bdf_col* col) { return fleet_aggregate_dev(c, op, col, out_scalar, is_some); });
    ENTER(c);
    if (op == BDF_COUNT) {  // metadata only when every null_count is known: no bytes move
        bool known = true;
        int64_t total = 0;
        for (int64_t i = 0; i < n; i++) {
            if (in[i].validity && in[i].null_count < 0) known = false;
            total += in[i].len - (in[i].validity ? in[i].null_count : 0);
        }
        if (known) { TRY(count_global(c, &total)); *(int64_t*)out_scalar = total; *is_some = 1; return BDF_OK; }
    }
    return host_call(c, {UploadSpec{dtype, n, in}}, [&](bdf_col* const* cols) { return aggregate_dev(c, op, cols[0], out_scalar, is_some); });
}

int bdf_aggregate_all(bdf_ctx* c, int dtype, int64_t n, const bdf_view* in, bdf_agg4* out) {
    NEED_CTX(c);
    if (c->fleet && !out) return fail(BDF_INVALID, "bad arguments");
    TRY(check_dtype(dtype));
    if (n < 0 || (n && !in) || !out) return fail(BDF_INVALID, "bad arguments");
    if (c->fleet) return fleet_host_reduce(c, dtype, n, in, [&](const bdf_col* col) { return fleet_aggregate_all_blocking(c, 1, &col, out); });
    ENTER(c);
    return host_call(c, {UploadSpec{dtype, n, in}}, [&](bdf_col* const* cols) { return aggregate_all_dev(c, cols[0], true, out); });
}

int bdf_avg(bdf_ctx* c, int dtype, int64_t n, const bdf_view* in, double* out, int32_t* is_some) {
    NEED_CTX(c);
    if (c->fleet && (!out || !is_some)) return fail(BDF_INVALID, "bad arguments");
    TRY(check_dtype(dtype));
    if (n < 0 || (n && !in) || !out || !is_some) return fail(BDF_INVALID, "bad arguments");
    if (c->fleet) return fleet_host_reduce(c, dtype, n, in, [&](const bdf_col* col) { return fleet_avg_dev(c, col, out, is_some); });
    ENTER(c);
    return host_call(c, {UploadSpec{dtype, n, in}}, [&](bdf_col* const* cols) { return avg_dev(c, cols[0], out, is_some); });
}

// Host-in entries of the statistics: a Boolean column is a type the operators do not take (BDF_UNSUPPORTED), not a bad dtype.
static int check_stat_dtype(int dtype) {
    if (dtype == kBool) return fail(BDF_UNSUPPORTED, "the statistics need a numeric column");
    return check_dtype(dtype);
}

int bdf_moments(bdf_ctx* c, int dtype, int64_t n, const bdf_view* in, bdf_moment_rec* out) {
    NEED_CTX(c);
    TRY(check_stat_dtype(dtype));
    if (n < 0 || (n && !in) || !out) return fail(BDF_INVALID, "bad arguments");
    if (c->fleet) return fleet_host_reduce(c, dtype, n, in, [&](const bdf_col* col) { return fleet_moments_dev(c, col, out); });
    ENTER(c);
    return host_call(c, {UploadSpec{dtype, n, in}}, [&](bdf_col* const* cols) {
        Moments m;
        TRY(moments_dev(c, cols[0], &m));
        memcpy(out, &m, sizeof m);
        return (int)BDF_OK;
    });
}

int bdf_distinct(bdf_ctx* c, int dtype, int64_t n, const bdf_view* in, bdf_distinct_rec* out) {
    if (c && c->fleet)
        return fail(BDF_UNSUPPORTED, "distinct values need every row of the column on one GPU (as sort / group-by / join): use a one-GPU context");
    ENTER(c);
    TRY(check_stat_dtype(dtype));
    if (n < 0 || (n && !in) || !out) return fail(BDF_INVALID, "bad arguments");
    if (is_global(c))
        return fail(BDF_UNSUPPORTED, "distinct values need every row of the column on one GPU (as sort / group-by / join): use a one-GPU context");
    return host_call(c, {UploadSpec{dtype, n, in}}, [&](bdf_col* const* cols) { return distinct_dev(c, cols[0], out); });
}

int bdf_percentile(bdf_ctx* c, int dtype, int64_t n, const bdf_view* in, int32_t n_p, const double* p, double* out, int32_t* is_some) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "%s", kDistFleet);
    ENTER(c);
    TRY(check_stat_dtype(dtype));
    if (n < 0 || (n && !in)) return fail(BDF_INVALID, "bad arguments");
    TRY(check_percentiles(n_p, p, out, is_some));
    if (is_global(c)) return fail(BDF_UNSUPPORTED, "%s", kDistFleet);
    std::vector<double> o((size_t)n_p);
    std::vector<int32_t> some((size_t)n_p);
    TRY(host_call(c, {UploadSpec{dtype, n, in}}, [&](bdf_col* const* cols) { return percentile_dev(c, cols[0], n_p, p, o.data(), some.data()); }));
    memcpy(out, o.data(), o.size() * sizeof(double));
    memcpy(is_some, some.data(), some.size() * sizeof(int32_t));
    return BDF_OK;
}

int bdf_mode(bdf_ctx* c, int dtype, int64_t n, const bdf_view* in, uint64_t* bits, int64_t* freq, int32_t* is_some) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "%s", kDistFleet);
    ENTER(c);
    TRY(check_stat_dtype(dtype));
    if (n < 0 || (n && !in) || !bits || !freq || !is_some) return fail(BDF_INVALID, "bad arguments");
    if (is_global(c)) return fail(BDF_UNSUPPORTED, "%s", kDistFleet);
    uint64_t b = 0;
    int64_t f = 0;
    int32_t some = 0;
    TRY(host_call(c, {UploadSpec{dtype, n, in}}, [&](bdf_col* const* cols) { return mode_dev(c, cols[0], &b, &f, &some); }));
    *bits = b; *freq = f; *is_some = some;
    return BDF_OK;
}

// ---- measurement support -------------------------------------------------------------------------

int bdf_profile_enable(bdf_ctx* c, int on) {
    if (c && c->fleet) { for (bdf_ctx* k : c->fleet->kids) TRY(bdf_profile_enable(k, on)); return BDF_OK; }
    ENTER(c);
    c->profiling = on != 0;
    return BDF_OK;
}

int bdf_profile_read(bdf_ctx* c, bdf_launch_record* buf, int64_t cap, int64_t* n) {
    if (c && c->fleet) {   // the records of all GPUs, GPU by GPU
        int64_t total = 0;
        for (bdf_ctx* k : c->fleet->kids) {
            int64_t got = 0;
            TRY(bdf_profile_read(k, buf ? buf + total : nullptr, buf ? cap - total : 0, &got));
            total += got;
        }
        if (n) *n = total;
        return BDF_OK;
    }
    ENTER(c);
    CK(cudaStreamSynchronize(c->s_compute));
    int64_t k = 0;
    for (auto& p : c->prof) {
        float ms = 0.f;
        cudaEventElapsedTime(&ms, p.e0, p.e1);
        p.rec.ms = ms;
        if (buf && k < cap) buf[k++] = p.rec;
        c->prof_pool.push_back(p.e0); c->prof_pool.push_back(p.e1);
    }
    c->prof.clear();
    if (n) *n = k;
    return BDF_OK;
}

int64_t bdf_launch_count(bdf_ctx* c) {
    if (c && c->fleet) { int64_t t = 0; for (bdf_ctx* k : c->fleet->kids) t += bdf_launch_count(k); return t; }
    return c ? c->launches : 0;
}

int bdf_timer_start(bdf_ctx* c) {
    if (c && c->fleet) { for (bdf_ctx* k : c->fleet->kids) TRY(bdf_timer_start(k)); return BDF_OK; }
    ENTER(c);
    CK(cudaEventRecord(c->ev_t0, c->s_compute));
    return BDF_OK;
}

int bdf_timer_stop(bdf_ctx* c, float* ms) {
    if (c && c->fleet) {   // the slowest GPU
        float worst = 0.f;
        for (bdf_ctx* k : c->fleet->kids) { float one = 0.f; TRY(bdf_timer_stop(k, &one)); worst = std::max(worst, one); }
        if (ms) *ms = worst;
        return BDF_OK;
    }
    ENTER(c);
    CK(cudaEventRecord(c->ev_t1, c->s_compute));
    CK(cudaEventSynchronize(c->ev_t1));
    if (ms) CK(cudaEventElapsedTime(ms, c->ev_t0, c->ev_t1));
    return BDF_OK;
}

int bdf_flush_l2(bdf_ctx* c, size_t bytes) {
    if (c && c->fleet) { for (bdf_ctx* k : c->fleet->kids) TRY(bdf_flush_l2(k, bytes)); return BDF_OK; }
    ENTER(c);
    if (bytes > c->flush_bytes) {
        if (c->flush_buf) CK(cudaFree(c->flush_buf));
        c->flush_buf = nullptr; c->flush_bytes = 0;
        CK(cudaMalloc(&c->flush_buf, bytes));
        c->flush_bytes = bytes;
    }
    CK(launch_fill(c->flush_buf, bytes, c->sm_count, c->s_compute));
    return BDF_OK;
}

int bdf_generate(bdf_ctx* c, int dtype, int kind, double lo, double hi, uint64_t seed, uint64_t col_id, int64_t n_chunks,
                 const int64_t* chunk_lens, int64_t row0, uint32_t null_mod, bdf_col** out) {
    NEED_CTX(c);
    TRY(check_dtype(dtype));
    if (!out || n_chunks < 0 || (n_chunks && !chunk_lens) || kind < 0 || kind > 3) return fail(BDF_INVALID, "bad arguments");
    if (c->fleet) return fleet_generate(c, dtype, kind, lo, hi, seed, col_id, n_chunks, chunk_lens, row0, null_mod, out);
    ENTER(c);
    std::vector<ChunkPlan> plan((size_t)n_chunks);
    for (int64_t i = 0; i < n_chunks; i++) {
        if (chunk_lens[i] < 0) return fail(BDF_INVALID, "negative chunk length");
        plan[i] = {chunk_lens[i], null_mod != 0};
    }
    const int w = dtype_width(dtype);
    int64_t rows = 0;
    return launch_groups(c, {}, {n_chunks}, dtype, plan, elems_per_tile(dtype), sizeof(GenDesc), BDF_K_GENERATE, "generate",
        [&](void* hd, int64_t i, int64_t tile0, const DevChunk& oc) {
            ((GenDesc*)hd)[i] = GenDesc{oc.values, oc.validity, oc.len, tile0, row0 + rows};
            rows += oc.len;
            return oc.len * w;
        },
        [&](const void* dd, int64_t begin, int64_t end, int64_t tiles, int64_t, uint32_t* wc) {
            return launch_generate(dtype, kind, lo, hi, seed, col_id, null_mod, (const GenDesc*)dd, (int)(end - begin), tiles, wc, c->s_compute);
        },
        out);
}


// ---- list columns ------------------------------------------------------------------------------

#define LIST_ENTER(ctx)                                                                                                   \
    if ((ctx) && (ctx)->fleet) return fail(BDF_UNSUPPORTED, "list columns live on one GPU: use a one-GPU context (bdf_init) for them"); \
    ENTER(ctx)

int bdf_list_upload(bdf_ctx* c, int child_dtype, int64_t n_chunks, const bdf_list_view* in, int flags, bdf_list** out) {
    LIST_ENTER(c);
    if (!out || n_chunks < 0 || (n_chunks && !in)) return fail(BDF_INVALID, "bad arguments");
    return list_upload(c, child_dtype, n_chunks, in, (flags & BDF_ASYNC) != 0, out);
}

int bdf_list_describe(const bdf_list* l, int32_t* child_dtype, int64_t* n_chunks, int64_t* total_len) {
    if (!l) return fail(BDF_INVALID, "null list");
    if (child_dtype) *child_dtype = l->dtype;
    if (n_chunks) *n_chunks = (int64_t)l->lens.size();
    if (total_len) *total_len = l->total_len;
    return BDF_OK;
}

int bdf_list_chunk_info(bdf_ctx* c, const bdf_list* l, int64_t chunk, int64_t* len, int64_t* null_count, int64_t* n_elements) {
    LIST_ENTER(c);
    if (!l || chunk < 0 || chunk >= (int64_t)l->lens.size()) return fail(BDF_INVALID, "bad chunk index");
    if (len) *len = l->lens[chunk];
    if (null_count) *null_count = l->null_counts[chunk];
    if (n_elements) *n_elements = l->values->chunks[chunk].len;
    return BDF_OK;
}

int bdf_list_download(bdf_ctx* c, const bdf_list* l, bdf_list_out* out) {
    LIST_ENTER(c);
    if (!l || (!out && !l->lens.empty())) return fail(BDF_INVALID, "null argument");
    return list_download(c, l, out);
}

const bdf_col* bdf_list_values(const bdf_list* l) { return l ? l->values : nullptr; }

void bdf_list_free(bdf_ctx* c, bdf_list* l) {
    if (!c || !l || c->fleet) return;
    std::lock_guard<std::mutex> lock(c->mu);
    cudaSetDevice(c->device);
    list_release(c, l);
}

int bdf_list_find_dev(bdf_ctx* c, int fn, const bdf_list* l, uint64_t value_bits, bdf_col** out) {
    LIST_ENTER(c);
    if (!l || !out) return fail(BDF_INVALID, "null argument");
    return list_find(c, fn, l, value_bits, out);
}

int bdf_list_reduce_dev(bdf_ctx* c, int fn, const bdf_list* l, bdf_col** out) {
    LIST_ENTER(c);
    if (!l || !out) return fail(BDF_INVALID, "null argument");
    return list_reduce(c, fn, l, out);
}

int bdf_list_transform_dev(bdf_ctx* c, int fn, const bdf_list* l, uint64_t value_bits, int64_t count, bdf_list** out) {
    LIST_ENTER(c);
    if (!l || !out) return fail(BDF_INVALID, "null argument");
    return list_transform(c, fn, l, value_bits, count, out);
}

int bdf_list_set_dev(bdf_ctx* c, int fn, const bdf_list* a, const bdf_list* b, bdf_list** out) {
    LIST_ENTER(c);
    if (!a || !b || !out) return fail(BDF_INVALID, "null argument");
    return list_set(c, fn, a, b, out);
}

int bdf_list_explode_dev(bdf_ctx* c, const bdf_list* l, bdf_col** rows, bdf_col** values) {
    LIST_ENTER(c);
    if (!l || !rows || !values) return fail(BDF_INVALID, "null argument");
    return list_explode(c, l, rows, values);
}

int bdf_list_take_dev(bdf_ctx* c, const bdf_list* l, const bdf_col* indices, bdf_list** out) {
    LIST_ENTER(c);
    if (!l || !indices || !out) return fail(BDF_INVALID, "null argument");
    return list_take(c, l, indices, out);
}

int bdf_list_filter_dev(bdf_ctx* c, const bdf_list* l, const bdf_col* mask, bdf_list** out) {
    LIST_ENTER(c);
    if (!l || !mask || !out) return fail(BDF_INVALID, "null argument");
    return list_filter(c, l, mask, out);
}

// ---- distinct rows and set operations ---------------------------------------------------------------------------------------

int bdf_duplicated_dev(bdf_ctx* c, int32_t n_keys, const bdf_col* const* keys, int32_t keep, bdf_col** mask) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "distinct rows move rows between chunks: use a one-GPU context (bdf_init) for them");
    ENTER(c);
    if (!mask) return fail(BDF_INVALID, "null argument");
    if (keep < BDF_KEEP_FIRST || keep > BDF_KEEP_NONE) return fail(BDF_INVALID, "unknown keep %d", keep);
    TRY(setop_check(n_keys, keys, nullptr, false));
    return setop_mask(c, keep, n_keys, keys, nullptr, mask);
}

int bdf_set_op_dev(bdf_ctx* c, int32_t op, int32_t n_keys, const bdf_col* const* left, const bdf_col* const* right, bdf_col** mask) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "set operations move rows between chunks: use a one-GPU context (bdf_init) for them");
    ENTER(c);
    if (!mask) return fail(BDF_INVALID, "null argument");
    if (op < BDF_SETOP_INTERSECT || op > BDF_SETOP_EXCEPT_ALL) return fail(BDF_INVALID, "unknown set operation %d", op);
    TRY(setop_check(n_keys, left, right, true));
    return setop_mask(c, 3 + op, n_keys, left, right, mask);
}

int bdf_bool_widen_dev(bdf_ctx* c, const bdf_col* in, bdf_col** out) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "use a one-GPU context (bdf_init) for the Boolean widening");
    ENTER(c);
    if (!in || !out) return fail(BDF_INVALID, "null argument");
    if (in->dtype != kBool) return fail(BDF_UNSUPPORTED, "the widening takes a Boolean column");
    return bool_widen(c, in, out);
}

int bdf_concat_dev(bdf_ctx* c, int32_t n, const bdf_col* const* cols, bdf_col** out) {
    if (c && c->fleet) return fail(BDF_UNSUPPORTED, "concat moves chunks between columns: use a one-GPU context (bdf_init) for it");
    ENTER(c);
    return concat_dev(c, n, cols, out);
}

int bdf_list_concat_dev(bdf_ctx* c, int32_t n, const bdf_list* const* lists, bdf_list** out) {
    LIST_ENTER(c);
    return list_concat(c, n, lists, out);
}

}  // extern "C"
