// libbsc_b200/csrc/common.cuh -- shared device/host plumbing for the GPU block-sorting path.
//
// One `Ctx` = one CUDA stream + one bump-allocated HBM arena + small pinned mailboxes.  Every
// stage takes a Ctx and enqueues its kernels on ctx->stream; nothing here is global except the
// per-device context pool in api.cu.  Blocks are independent (SURVEY.md 8e), so concurrency is
// simply "several Ctx in flight".
#pragma once

#include <cuda_runtime.h>
#include <vector>
#include <mutex>
#include <atomic>
#include <condition_variable>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

typedef uint8_t  u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;

// libbsc error codes (libbsc/libbsc.h:41-51)
#define LIBBSC_NO_ERROR                0
#define LIBBSC_BAD_PARAMETER          -1
#define LIBBSC_NOT_ENOUGH_MEMORY      -2
#define LIBBSC_NOT_COMPRESSIBLE       -3
#define LIBBSC_NOT_SUPPORTED          -4
#define LIBBSC_UNEXPECTED_EOB         -5
#define LIBBSC_DATA_CORRUPT           -6
#define LIBBSC_GPU_ERROR              -7
#define LIBBSC_GPU_NOT_SUPPORTED      -8
#define LIBBSC_GPU_NOT_ENOUGH_MEMORY  -9

#define LIBBSC_FEATURE_FASTMODE        1
#define LIBBSC_FEATURE_MULTITHREADING  2
#define LIBBSC_FEATURE_LARGEPAGES      4
#define LIBBSC_FEATURE_CUDA            8

#define LIBBSC_HEADER_SIZE 28

// SMs of `device` (132 on an H100 SXM), read once per device: grid sizes and the decoder layout scale with it
static inline u32 device_sms(int device)
{
    static std::atomic<int> sms[16];
    int v = sms[device & 15].load(std::memory_order_relaxed);
    if (v <= 0) {
        if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device) != cudaSuccess || v <= 0) { cudaGetLastError(); v = 132; }
        sms[device & 15].store(v, std::memory_order_relaxed);
    }
    return (u32)v;
}

struct CudaFail { cudaError_t err; const char *file; int line; };

#define CUDA_TRY(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { \
        if (getenv("BSCB200_DEBUG")) fprintf(stderr, "[libbsc_b200] %s:%d: %s -> %s\n", __FILE__, __LINE__, #expr, cudaGetErrorString(e_)); \
        throw CudaFail{e_, __FILE__, __LINE__}; } } while (0)

#define KERNEL_CHECK() CUDA_TRY(cudaGetLastError())

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
static inline u32 ceil_div(u64 a, u64 b) { return (u32)((a + b - 1) / b); }
static inline int bits_for(u64 max_value) { int b = 0; while (b < 64 && (max_value >> b) != 0) ++b; return b > 0 ? b : 1; }

// Bump allocator over one cudaMalloc'd slab.  reset() between blocks; grows (realloc) on demand
// only while empty, so pointers handed out stay valid for the duration of a block.
struct Arena {
    u8    *base = nullptr;
    size_t cap = 0, used = 0;

    void reserve(size_t bytes) {
        if (bytes <= cap) return;
        if (used != 0) throw CudaFail{cudaErrorMemoryAllocation, __FILE__, __LINE__};
        if (base) { cudaFree(base); base = nullptr; cap = 0; }
        cudaError_t e = cudaMalloc((void **)&base, bytes);
        if (e != cudaSuccess) { cudaGetLastError(); throw CudaFail{cudaErrorMemoryAllocation, __FILE__, __LINE__}; }
        cap = bytes;
    }
    // what get<T>(count) takes from the arena: 256 B slack after every buffer, 256-byte aligned
    template <typename T> static size_t bytes_for(size_t count) { return align_up(count * sizeof(T) + 256, 256); }
    template <typename T> T *get(size_t count) {
        size_t bytes = bytes_for<T>(count);
        if (used + bytes > cap) throw CudaFail{cudaErrorMemoryAllocation, __FILE__, __LINE__};
        T *p = (T *)(base + used); used += bytes; return p;
    }
    size_t mark() const { return used; }
    void release(size_t m) { used = m; }
    void reset() { used = 0; }
    void destroy() { if (base) cudaFree(base); base = nullptr; cap = used = 0; }
};

// one timed kernel launch (profiling mode only): CUDA events on the launching stream
struct ProfRec { const char *name; cudaEvent_t a, b; double bytes; };

// A large scratch slab for the SORT stages (forward BWT ~58 n, ST-k ~30 n, inverse ST ~41 n), shared by all contexts of a device:
// a sort holds it for some tens of milliseconds of a block whose coder stage runs for seconds, so a handful of slabs serve any
// number of blocks in flight (api.cu: scratch pool).  `idle` is recorded on the last user's stream when it hands the slab back.
struct Scratch {
    Arena       arena;
    cudaEvent_t idle = nullptr;
    bool        idle_valid = false;
};

struct Ctx {
    int          device = 0;
    cudaStream_t stream = nullptr;
    bool         owns_stream = false;
    Arena        arena;                 // per-block state: staged block, coder stage, inverse BWT
    Scratch     *scratch = nullptr;     // held only while a sort stage runs (ScratchLease in api.cu); sort stages fall back to `arena`
    Arena       &sort_arena() { return scratch ? scratch->arena : arena; }
    long long    sort_budget = 0;       // > 0: the forward BWT sorts in batches when its standard working set is larger (bscb200_ctx_set_sort_budget)
    u32         *h_mail = nullptr;      // pinned host mailbox (64 words) for small D2H read-backs
    u32         *d_mail = nullptr;      // device mailbox (64 words)
    u64          kernels_launched = 0;  // our own kernel launches enqueued through this ctx
    bool         profile = false;       // bracket every launch with CUDA events (bench.py roofline leg)
    double       next_bytes = 0;        // algorithmic bytes of the next launch (PROF_BYTES)
    std::vector<ProfRec>     prof;
    std::vector<cudaEvent_t> ev_pool;
    size_t       ev_used = 0;
    cudaEvent_t ev() {
        if (ev_used == ev_pool.size()) { cudaEvent_t e; CUDA_TRY(cudaEventCreate(&e)); ev_pool.push_back(e); }
        return ev_pool[ev_used++];
    }

    // Host wait for this context's stream.  cudaStreamSynchronize spins (cudaDeviceScheduleAuto), and in a full pipeline the sort kernels a
    // thread waits for are queued behind other blocks' coder CTAs for tens of milliseconds: dozens of threads per GPU (x 8 ranks per host)
    // would burn a core each.  So the wait BLOCKS on an event created with cudaEventBlockingSync (the thread sleeps until the driver's
    // interrupt, a little later than a spin would see it).  BSCB200_SYNC=spin restores the spinning wait (A/B).
    cudaEvent_t ev_sync = nullptr;
    void sync() {
        static const bool spin = [] { const char *e = getenv("BSCB200_SYNC"); return e && e[0] == 's'; }();
        if (spin) { CUDA_TRY(cudaStreamSynchronize(stream)); return; }
        if (!ev_sync) CUDA_TRY(cudaEventCreateWithFlags(&ev_sync, cudaEventBlockingSync | cudaEventDisableTiming));
        CUDA_TRY(cudaEventRecord(ev_sync, stream));
        CUDA_TRY(cudaEventSynchronize(ev_sync));
    }
    // Wait for a kernel that runs for 0.01 - 2 s (the coder kernels) WITHOUT putting anything behind it on the stream and without
    // driver calls.  A process has at most 32 hardware work queues per GPU (CUDA_DEVICE_MAX_CONNECTIONS), so with 40+ blocks in
    // flight two streams share a queue; an event record or a copy enqueued behind the 2 s kernel of one of them holds the queue's head
    // until that kernel ENDS and the other stream's work waits behind it, so blocks in flight run as waves of 32.  Polling
    // cudaStreamQuery from dozens of threads instead slows the launch-heavy sort stages of the other blocks (driver lock).  So the
    // kernel itself reports: its last CTA writes a sequence
    // number into this context's pinned mailbox (signal_done below) and the host thread sleeps on that word.
    // Stream priorities (BSCB200_PRIO=0 turns them off).  When SM slots free up, the CTA scheduler places pending CTAs of higher-priority
    // streams first, whichever block launched first.  Three levels per context:
    //   stream     (highest)  everything that is short: the sort / scan / rank kernels.  A coder CTA holds its slot for 0.1 - 4 s, a sort
    //                         CTA for microseconds; at equal priority the sort launches of a full pipeline wait behind coder CTAs
    //                         for many times their own duration while the coder slots of their blocks stand empty;
    //   stream_hi  (middle)   the LONG streams of a coder launch (qlfc.cu: split launches): longest-stream-first ACROSS blocks without any
    //                         coordination between the host threads;
    //   stream_lo  (lowest)   the other coder streams.
    cudaStream_t stream_hi = nullptr, stream_lo = nullptr;
    cudaEvent_t  ev_fork = nullptr, ev_join = nullptr, ev_join_lo = nullptr;
    static bool priorities_on() { static const bool on = [] { const char *e = getenv("BSCB200_PRIO"); return !(e && e[0] == '0'); }(); return on; }
    void ensure_hi() {
        if (stream_hi) return;
        int lo = 0, hi = 0; CUDA_TRY(cudaDeviceGetStreamPriorityRange(&lo, &hi));       // lo = least (numerically greatest), hi = greatest priority
        const bool on = priorities_on();
        CUDA_TRY(cudaStreamCreateWithPriority(&stream_hi, cudaStreamNonBlocking, on ? (lo + hi) / 2 : hi));
        if (on) { CUDA_TRY(cudaStreamCreateWithPriority(&stream_lo, cudaStreamNonBlocking, lo)); CUDA_TRY(cudaEventCreateWithFlags(&ev_join_lo, cudaEventDisableTiming)); }
        CUDA_TRY(cudaEventCreateWithFlags(&ev_fork, cudaEventDisableTiming));
        CUDA_TRY(cudaEventCreateWithFlags(&ev_join, cudaEventDisableTiming));
    }
    // the stream the SHORT streams of a coder launch go to (the main stream when priorities are off)
    cudaStream_t coder_stream() { ensure_hi(); return stream_lo ? stream_lo : stream; }
    u32 done_seq = 0;
    struct DoneSignalArgs { u32 *ctr; u32 *host_flag; u32 seq; };
    DoneSignalArgs next_signal() { ++done_seq; return DoneSignalArgs{d_mail + 128, h_mail + 250, done_seq}; }
    // `a`, `b`: the streams the reporting kernels were launched on (default: the context's own stream)
    void wait_signal(cudaStream_t a = nullptr, cudaStream_t b = nullptr) {
        if (!a) a = stream;
        volatile u32 *flag = (volatile u32 *)(h_mail + 250);
        // 20 us steps growing to 0.4 ms, and to 2 ms once the kernel has run for 50 ms (a coder launch takes 0.1 - 2 s; with 8 ranks x 64+
        // waiting threads per host the wake-ups themselves must stay cheap)
        unsigned us = 20, slept = 0, total = 0;
        while (*flag != done_seq) {
            struct timespec ts = {0, (long)us * 1000L}; nanosleep(&ts, nullptr);
            slept += us; total += us; if (us < (total > 50000 ? 2000u : 400u)) us += us / 2;
            if (slept > 200000) {                            // every 0.2 s: has the stream died (launch failure, kernel fault)?
                slept = 0;
                cudaError_t e = cudaStreamQuery(a);
                if (e == cudaSuccess && b) e = cudaStreamQuery(b);
                if (e == cudaSuccess) { if (*flag != done_seq) { cudaGetLastError(); throw CudaFail{cudaErrorUnknown, __FILE__, __LINE__}; } break; }
                if (e != cudaErrorNotReady) { cudaGetLastError(); throw CudaFail{e, __FILE__, __LINE__}; }
            }
        }
    }
    // Read `words` u32 from the device mailbox (blocks the host on this stream only).
    void fetch_mail(int words) {
        CUDA_TRY(cudaMemcpyAsync(h_mail, d_mail, sizeof(u32) * words, cudaMemcpyDeviceToHost, stream));
        sync();
    }
};

// Optional cap on the coder CTAs in flight per device (BSCB200_CODER_SLOTS, default: none).  A coder CTA pins half an SM's shared memory for
// 0.1 - 2 s; the sort kernels of other blocks need shared memory too and can only run where a half is free.  With every half taken by
// coders the sorts starve in a saturated pipeline, so a caller that keeps
// both directions in flight can leave a share of the SMs to the sorts.  Host-side counting semaphore; a launch waits for its CTAs' worth.
struct CoderSlots {
    static int limit() { static const int v = [] { const char *e = getenv("BSCB200_CODER_SLOTS"); int k = e ? atoi(e) : 0; return k >= 8 ? k : 0; }(); return v; }
    struct State { std::mutex m; std::condition_variable cv; int used = 0; };
    static State &state(int device) { static State s[16]; return s[device & 15]; }
    struct Lease {
        int device, n;
        Lease(int dev, int ctas) : device(dev), n(limit() ? (ctas < limit() ? ctas : limit()) : 0) {
            if (!n) return;
            State &S = state(device); std::unique_lock<std::mutex> lk(S.m);
            S.cv.wait(lk, [&] { return S.used + n <= limit(); });
            S.used += n;
        }
        ~Lease() { if (!n) return; State &S = state(device); { std::lock_guard<std::mutex> lk(S.m); S.used -= n; } S.cv.notify_all(); }
    };
};

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (kernel, device): the call is not free and
// must not sit in front of every launch of a kernel that other streams are running.
template <typename F> static inline void ensure_dyn_smem(F *kernel, int device, size_t bytes)
{
    static const void *seen[64]; static int seen_dev[64]; static int count = 0;   // per translation unit; tiny
    static std::mutex m;
    std::lock_guard<std::mutex> lk(m);
    for (int i = 0; i < count; ++i) if (seen[i] == (const void *)kernel && seen_dev[i] == device) return;
    CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
    if (count < 64) { seen[count] = (const void *)kernel; seen_dev[count] = device; ++count; }
}

#define PROF_BYTES(ctx, b) do { (ctx)->next_bytes = (double)(b); } while (0)
#define LAUNCH(ctx, kernel, grid, block, smem, ...) LAUNCH_NAMED(ctx, #kernel, kernel, grid, block, smem, __VA_ARGS__)
// the same for a kernel chosen at run time (a function pointer): `name` is what the profile reports
#define LAUNCH_NAMED(ctx, name, kernel, grid, block, smem, ...) do { \
        Ctx *c_ = (ctx); cudaEvent_t ea_ = nullptr, eb_ = nullptr; const bool p_ = c_->profile; \
        if (p_) { ea_ = c_->ev(); eb_ = c_->ev(); CUDA_TRY(cudaEventRecord(ea_, c_->stream)); } \
        kernel<<<(grid), (block), (smem), c_->stream>>>(__VA_ARGS__); KERNEL_CHECK(); \
        if (p_) { CUDA_TRY(cudaEventRecord(eb_, c_->stream)); c_->prof.push_back(ProfRec{name, ea_, eb_, c_->next_bytes}); } \
        c_->next_bytes = 0; c_->kernels_launched++; } while (0)

// A launch that the host waits for before anything else goes onto the stream (Ctx::wait_signal): the kernel takes a DoneSignal as its
// LAST parameter and calls signal_done once per CTA; the closing profile event is recorded after the wait, not behind the kernel.
#define LAUNCH_LONG(ctx, kernel, grid, block, smem, ...) do { \
        Ctx *c_ = (ctx); cudaEvent_t ea_ = nullptr, eb_ = nullptr; const bool p_ = c_->profile; const double nb_ = c_->next_bytes; \
        CoderSlots::Lease lease_(c_->device, (int)(grid)); \
        if (p_) { ea_ = c_->ev(); eb_ = c_->ev(); CUDA_TRY(cudaEventRecord(ea_, c_->stream)); } \
        const Ctx::DoneSignalArgs sg_ = c_->next_signal(); \
        kernel<<<(grid), (block), (smem), c_->stream>>>(__VA_ARGS__, DoneSignal{sg_.ctr, sg_.host_flag, sg_.seq, (u32)(grid)}); KERNEL_CHECK(); \
        c_->next_bytes = 0; c_->kernels_launched++; \
        c_->wait_signal(); \
        if (p_) { CUDA_TRY(cudaEventRecord(eb_, c_->stream)); c_->prof.push_back(ProfRec{#kernel, ea_, eb_, nb_}); } } while (0)

// ---- small device helpers// ---- small device helpers ------------------------------------------------------------------
__device__ __forceinline__ u32 lane_id() { return threadIdx.x & 31; }

// Completion report of a long kernel (LAUNCH_LONG): ONE thread per CTA calls it after the CTA's results are in global memory; the
// last CTA of the grid re-arms the counter and writes `seq` into the context's pinned host mailbox.
struct DoneSignal { u32 *ctr; u32 *host_flag; u32 seq; u32 total; };   // total = CTAs that report (one launch, or the two launches of a split)
__device__ __forceinline__ void signal_done(const DoneSignal &s)
{
    __threadfence();
    if (atomicAdd(s.ctr, 1u) == s.total - 1u) {
        *s.ctr = 0;
        __threadfence_system();
        *(volatile u32 *)s.host_flag = s.seq;
    }
}
__device__ __forceinline__ u32 lanemask_lt() { u32 m; asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m)); return m; }

// Lanes of the warp that hold the same `bits`-bit digit as this lane, from one ballot per digit bit (all 32 lanes must call it).
// Against __match_any_sync: as a DEPENDENT operation match.any is slow for many distinct values, but its THROUGHPUT with many warps in
// flight is better than 8 ballots + 8 selects, so the multisplits (rs_onesweep, unbwt_lf) keep match.any; the grid-stride histogram
// (one item per thread and iteration, little else to overlap with) is faster with the ballots and keeps them.
__device__ __forceinline__ u32 warp_peers(u32 d, int bits)
{
    u32 m = 0xffffffffu;
#pragma unroll
    for (int b = 0; b < 9; ++b) {
        if (b < bits) {                                  // warp-uniform
            const u32 bit = (d >> b) & 1u, v = __ballot_sync(0xffffffffu, bit);
            m &= bit ? v : ~v;
        }
    }
    return m;
}

// relaxed, device-scope single-word accesses for decoupled look-back descriptors
__device__ __forceinline__ u64 ld_relaxed(const u64 *p) { u64 v; asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ void st_relaxed(u64 *p, u64 v) { asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" :: "l"(p), "l"(v) : "memory"); }

// ---- TMA bulk copies (cp.async.bulk, SASS UBLKCP) completing on an mbarrier in shared memory -----------------------------------
__device__ __forceinline__ u32 smem_addr(const void *p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(u64 *bar, u32 arrivals)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_addr(bar)), "r"(arrivals) : "memory");
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// one arrival + the number of bytes the bulk copies issued next will deliver
__device__ __forceinline__ void mbar_arrive_expect_tx(u64 *bar, u32 bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(u64 *bar, u32 parity)
{
    asm volatile("{\n\t.reg .pred P1;\n\tMBAR_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t@P1 bra MBAR_DONE;\n\tbra MBAR_WAIT;\n\tMBAR_DONE:\n\t}"
                 :: "r"(smem_addr(bar)), "r"(parity) : "memory");
}
// global -> shared, `bytes` a multiple of 16, both addresses 16-byte aligned; completes (complete_tx) on `bar`
__device__ __forceinline__ void bulk_copy_g2s(void *dst_smem, const void *src_gmem, u32 bytes, u64 *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_addr(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_addr(bar)) : "memory");
}
// orders earlier generic-proxy accesses to shared memory (ld/st.shared of all threads, after a barrier) before later async-proxy writes (TMA)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// streaming 128-bit loads that do not pollute L1 (inputs that are read exactly once)
__device__ __forceinline__ uint4 ld_stream_v4(const void *p) {
    uint4 v; asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}
