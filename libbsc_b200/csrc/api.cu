// libbsc_b200/csrc/api.cu -- the C-ABI boundary (include/libbsc_b200.h).
//
// Host glue only: parameter validation, the 28-byte block header, error codes, H2D/D2H copies and
// the per-device context pool.  Every byte-touching stage (BWT / ST / QLFC / Adler-32) runs as
// CUDA kernels on the current device; there is NO CPU implementation of those stages in this
// library -- if CUDA is unavailable every entry point returns LIBBSC_GPU_NOT_SUPPORTED.
//
// Mirrors libbsc/libbsc/libbsc.cpp (bsc_store 68-81, bsc_compress 213-338, bsc_block_info 340-418,
// bsc_decompress 522-617) and the stage entry points libbsc.cpp calls:
// bsc_bwt_encode/decode (bwt.h:56,68), bsc_st_encode (st.h:57), bsc_coder_compress/decompress
// (coder.h:56,66), bsc_adler32 (adler32.h).
#include "common.cuh"
#include "stages.cuh"
#include "lzp_host.h"
#include "../../include/libbsc_b200.h"

#include <condition_variable>
#include <new>
#include <mutex>
#include <vector>
#include <sys/mman.h>
#include <unistd.h>

// ---------------------------------------------------------------------------------------------
// context pool
// ---------------------------------------------------------------------------------------------
namespace {

constexpr int MAX_DEVICES = 16;
std::mutex g_pool_mutex;
std::vector<Ctx *> g_pool[MAX_DEVICES];
void *(*g_malloc)(size_t) = nullptr;
void *(*g_zero_malloc)(size_t) = nullptr;
void (*g_free)(void *) = nullptr;
unsigned long long g_launches_retired = 0;

Ctx *ctx_new(int device, cudaStream_t stream, bool own)
{
    Ctx *c = new Ctx();
    c->device = device;
    try {
        CUDA_TRY(cudaSetDevice(device));
        if (own) {                                   // the context's own stream carries the short kernels: highest priority (Ctx::stream_hi)
            int lo = 0, hi = 0; CUDA_TRY(cudaDeviceGetStreamPriorityRange(&lo, &hi));
            CUDA_TRY(cudaStreamCreateWithPriority(&c->stream, cudaStreamNonBlocking, Ctx::priorities_on() ? hi : lo)); c->owns_stream = true;
        }
        else c->stream = stream;
        CUDA_TRY(cudaMallocHost((void **)&c->h_mail, 1024));
        CUDA_TRY(cudaMalloc((void **)&c->d_mail, 1024));
        CUDA_TRY(cudaMemsetAsync(c->d_mail, 0, 1024, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
    } catch (...) { delete c; throw; }
    return c;
}

// Destroys a context; its kernel launches stay counted in bscb200_total_kernel_launches.
void ctx_delete(Ctx *c)
{
    if (!c) return;
    { std::lock_guard<std::mutex> lk(g_pool_mutex); g_launches_retired += c->kernels_launched; }
    cudaSetDevice(c->device);
    c->arena.destroy();
    if (c->h_mail) cudaFreeHost(c->h_mail);
    if (c->d_mail) cudaFree(c->d_mail);
    for (cudaEvent_t e : c->ev_pool) cudaEventDestroy(e);
    if (c->stream_hi) cudaStreamDestroy(c->stream_hi);
    if (c->stream_lo) cudaStreamDestroy(c->stream_lo);
    if (c->ev_join_lo) cudaEventDestroy(c->ev_join_lo);
    if (c->ev_fork) cudaEventDestroy(c->ev_fork);
    if (c->ev_join) cudaEventDestroy(c->ev_join);
    if (c->ev_sync) cudaEventDestroy(c->ev_sync);
    if (c->owns_stream && c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

Ctx *ctx_acquire()
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    if (dev < 0 || dev >= MAX_DEVICES) return nullptr;
    {
        std::lock_guard<std::mutex> lk(g_pool_mutex);
        if (!g_pool[dev].empty()) { Ctx *c = g_pool[dev].back(); g_pool[dev].pop_back(); return c; }
    }
    try { return ctx_new(dev, nullptr, true); } catch (...) { cudaGetLastError(); return nullptr; }
}

void ctx_release(Ctx *c)
{
    if (!c) return;
    c->arena.reset();
    std::lock_guard<std::mutex> lk(g_pool_mutex);
    g_pool[c->device].push_back(c);
}

// ---- scratch pool: a few large slabs per device for the sort stages, shared by every context of that device -----------------
// BSCB200_SORT_SLABS (default 6) bounds how many exist; a sort waits (host side) for a free one.  Handing a slab from one stream to
// another is ordered by an event recorded at release and waited for at acquisition, so no host synchronisation is needed.
// Slabs are made on demand.  With the coder at five streams per SM the pipeline turns over 12+ blocks a second while a forward BWT that
// shares the SMs with coder CTAs holds its slab for ~0.3 s: three slabs (round 2's first setting) made the sorts queue for memory.
// A slab that cannot be allocated any more (the caller filled the HBM) lowers the bound to what exists instead of failing the block.
struct ScratchPool { std::mutex m; std::condition_variable cv; std::vector<Scratch *> free_list; int created = 0, cap = -1; };
ScratchPool g_scratch[MAX_DEVICES];
int scratch_limit()
{
    static const int v = [] { const char *e = getenv("BSCB200_SORT_SLABS"); int k = e ? atoi(e) : 0; return k >= 1 && k <= 64 ? k : 6; }();
    return v;
}

// Frees a slab (null: nothing) once its last user is done with it.
void scratch_destroy(Scratch *s)
{
    if (!s) return;
    if (s->idle_valid) cudaEventSynchronize(s->idle);
    s->arena.destroy();
    if (s->idle) cudaEventDestroy(s->idle);
    delete s;
}

Scratch *scratch_acquire(Ctx *c, size_t bytes)
{
    ScratchPool &P = g_scratch[c->device];
    for (;;) {
        Scratch *s = nullptr;
        {
            std::unique_lock<std::mutex> lk(P.m);
            for (;;) {
                if (!P.free_list.empty()) { s = P.free_list.back(); P.free_list.pop_back(); break; }
                if (P.created < (P.cap >= 0 ? P.cap : scratch_limit())) { P.created++; break; }      // make a new one outside the lock
                P.cv.wait(lk);
            }
        }
        const bool fresh = (s == nullptr);
        try {
            if (!s) { s = new Scratch(); CUDA_TRY(cudaEventCreateWithFlags(&s->idle, cudaEventDisableTiming)); }
            if (s->idle_valid) CUDA_TRY(cudaStreamWaitEvent(c->stream, s->idle, 0));
            if (s->arena.cap < bytes) {
                if (s->idle_valid) CUDA_TRY(cudaEventSynchronize(s->idle));         // the slab is about to be freed: its last user must be done
                s->arena.reset(); s->arena.reserve(bytes);
            }
        } catch (const CudaFail &f) {
            std::unique_lock<std::mutex> lk(P.m);
            if (fresh && f.err == cudaErrorMemoryAllocation && P.created > 1) {       // no room for one more slab: live with the ones there are
                cudaGetLastError();
                scratch_destroy(s);
                P.created--; P.cap = P.created;
                P.cv.notify_all();
                continue;
            }
            if (fresh) { scratch_destroy(s); P.created--; } else P.free_list.push_back(s);
            P.cv.notify_one();
            throw;
        } catch (...) {
            std::lock_guard<std::mutex> lk(P.m);
            if (s && !fresh) { P.free_list.push_back(s); } else { P.created--; }
            P.cv.notify_one();
            throw;
        }
        s->arena.reset();
        return s;
    }
}

void scratch_release(Ctx *c, Scratch *s)
{
    if (!s) return;
    s->idle_valid = cudaEventRecord(s->idle, c->stream) == cudaSuccess;
    if (!s->idle_valid) { cudaGetLastError(); cudaStreamSynchronize(c->stream); cudaGetLastError(); }
    ScratchPool &P = g_scratch[c->device];
    { std::lock_guard<std::mutex> lk(P.m); P.free_list.push_back(s); }
    P.cv.notify_one();
}

// holds a scratch slab for the duration of one sort stage
struct ScratchLease {
    Ctx *c;
    ScratchLease(Ctx *ctx, size_t bytes) : c(ctx) { c->scratch = scratch_acquire(c, bytes); }
    ~ScratchLease() { Scratch *s = c->scratch; c->scratch = nullptr; scratch_release(c, s); }
    ScratchLease(const ScratchLease &) = delete; ScratchLease &operator=(const ScratchLease &) = delete;
};

// ---- the three context lifetimes of an entry point ------------------------------------------------------------------------------
// Runs `body()` and returns its result, or the libbsc code of what it threw: nothing may unwind through the extern "C" boundary.
// `failed` tells whether it threw, which may leave the context mid-stage.
template <class F> int run_mapped(F &&body, bool &failed)
{
    failed = true;
    int r;
    try { r = body(); failed = false; }
    catch (const CudaFail &f) { cudaGetLastError(); r = f.err == cudaErrorMemoryAllocation ? LIBBSC_GPU_NOT_ENOUGH_MEMORY : LIBBSC_GPU_ERROR; }
    catch (const std::bad_alloc &) { r = LIBBSC_NOT_ENOUGH_MEMORY; }
    catch (...) { r = LIBBSC_GPU_ERROR; }
    return r;
}

// run `body(ctx)` on a pooled context.  A context that failed mid-stage is destroyed instead of pooled (its device mailbox may hold
// partial Adler-32 sums that the next block would inherit).
template <class F> int with_ctx(F body)
{
    Ctx *c = ctx_acquire();
    if (!c) return LIBBSC_GPU_NOT_SUPPORTED;
    bool failed;
    const int r = run_mapped([&] { return body(c); }, failed);
    if (failed) { cudaStreamSynchronize(c->stream); cudaGetLastError(); ctx_delete(c); }
    else ctx_release(c);
    return r;
}

// run `body(ctx)` on a context of its own, destroyed afterwards so that none of its HBM outlives the call
template <class F> int with_own_ctx(F body)
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return LIBBSC_GPU_NOT_SUPPORTED; }
    Ctx *c = nullptr;
    bool failed;
    const int r = run_mapped([&] { c = ctx_new(dev, nullptr, true); return body(c); }, failed);
    if (c) { cudaStreamSynchronize(c->stream); cudaGetLastError(); ctx_delete(c); }
    return r;
}

// run `body()` on the caller's context, which a failure leaves reset for its next call
template <class F> int guarded(Ctx *c, F body)
{
    bool failed;
    const int r = run_mapped(body, failed);
    if (failed) {
        cudaStreamSynchronize(c->stream); cudaGetLastError(); c->arena.reset();
        cudaMemsetAsync(c->d_mail, 0, 1024, c->stream); cudaStreamSynchronize(c->stream); cudaGetLastError();   // adler32.cu expects zeroed accumulators
    }
    return r;
}

// arena sizes (bytes) generous enough for each sort stage at block length n
size_t need_bwt_encode(size_t n) { return 58 * n + (64u << 20); }
size_t need_st_encode(size_t n)  { return 30 * n + (16u << 20); }
size_t need_st_decode(size_t n)  { return 41 * n + (16u << 20); }
// The coder stage in either direction, from the buffers it takes (at most about 8.5 n + 28 MB)
size_t need_coder(size_t n)      { return std::max(coder_compress_bytes((u32)n), coder_decompress_bytes()); }
// A context's arena on the device-resident entry points: the block's working copy and the coder stage (compress), or the coder stage and
// then the inverse BWT in the same space (decompress, about 8.7 n).  The sort stages work in the shared slabs.
size_t ctx_workspace(size_t n)   { return std::max(Arena::bytes_for<u8>(n + 64) + need_coder(n), bwt_decode_bytes((u32)n)); }
// bsc_compress on a pooled context: the staged block and the output beside that workspace
size_t host_compress_bytes(size_t n) { return Arena::bytes_for<u8>(n + 64) + Arena::bytes_for<u8>(n + 4096) + ctx_workspace(n); }
// bsc_decompress of a block of `block` bytes that holds n bytes of data: the staged block and the output beside the coder stage, then
// the inverse BWT in the same space.  Above 1 GiB (BWT and stored blocks) this is about 10.7 n + 28 MB, which large_bound holds.
size_t host_decompress_bytes(size_t block, size_t n)
{
    return Arena::bytes_for<u8>(block + 128) + Arena::bytes_for<u8>(n + 128) + std::max(need_coder(n), bwt_decode_bytes((u32)n));
}

unsigned int host_adler32(const unsigned char *p, size_t n)
{
    unsigned int a = 1, b = 0;
    while (n) { size_t k = n < 5552 ? n : 5552; n -= k; while (k--) { a += *p++; b += a; } a %= 65521u; b %= 65521u; }
    return (b << 16) | a;
}
void put32(unsigned char *p, unsigned int v) { memcpy(p, &v, 4); }
unsigned int get32(const unsigned char *p) { unsigned int v; memcpy(&v, p, 4); return v; }

// number of bytes starting at p (up to `want`) that lie in mapped pages
size_t readable_prefix(const void *p, size_t want)
{
    const size_t page = (size_t)sysconf(_SC_PAGESIZE);
    size_t addr = (size_t)p, first = addr & ~(page - 1), ok = 0;
    unsigned char vec;
    for (size_t pg = first; pg < addr + want; pg += page) {
        if (mincore((void *)pg, page, &vec) != 0) break;
        ok = pg + page - addr;
    }
    return ok < want ? ok : want;
}

// the parameter ranges of libbsc: arguments outside them are LIBBSC_BAD_PARAMETER, header fields outside them LIBBSC_DATA_CORRUPT
bool sorter_valid(int s) { return s == 1 || (s >= 3 && s <= 8); }
bool coder_valid(int c) { return c >= 1 && c <= 3; }
bool lzp_valid(int hash, int min) { return hash >= 10 && hash <= 28 && min >= 4 && min <= 255; }
bool st_order_valid(int k) { return k >= 3 && k <= 8; }

// ---- the 28-byte block header (libbsc.cpp:68-81, 340-418) ------------------------------------------------------------------------
// The mode word: block sorter in bits 0..4, coder in 5..7, LZP minimum length in 8..15, LZP hash size in 16..23; 0 for a stored block.
struct Mode {
    int word = 0;
    static Mode of(int sorter, int coder, int lzpHash, int lzpMin) { return Mode{sorter | (coder << 5) | (lzpMin << 8) | (lzpHash << 16)}; }
    int sorter() const { return word & 0x1f; }
    int coder() const { return (word >> 5) & 7; }
    int lzp_min() const { return (word >> 8) & 0xff; }
    int lzp_hash() const { return (word >> 16) & 0xff; }
    bool has_lzp() const { return word != (word & 0xff); }
};

struct BlockHeader {
    int block_size = 0, data_size = 0;
    Mode mode;
    int index = 0;
    u32 adler_data = 0, adler_payload = 0;

    int payload() const { return block_size - LIBBSC_HEADER_SIZE; }
    // the 28 bytes at h, the header's own Adler-32 last
    void write(unsigned char *h) const
    {
        put32(h, (u32)block_size); put32(h + 4, (u32)data_size); put32(h + 8, (u32)mode.word); put32(h + 12, (u32)index);
        put32(h + 16, adler_data); put32(h + 20, adler_payload); put32(h + 24, host_adler32(h, 24));
    }
    // Reads the header at h (headerSize readable bytes) with bsc_block_info's checks, its codes in its order.
    int read(const unsigned char *h, int headerSize)
    {
        if (headerSize < LIBBSC_HEADER_SIZE) return LIBBSC_UNEXPECTED_EOB;
        if (get32(h + 24) != host_adler32(h, 24)) return LIBBSC_DATA_CORRUPT;
        *this = BlockHeader{(int)get32(h), (int)get32(h + 4), Mode{(int)get32(h + 8)}, (int)get32(h + 12), get32(h + 16), get32(h + 20)};
        const Mode m = mode;
        if (m.sorter() != 0 && !sorter_valid(m.sorter())) return LIBBSC_DATA_CORRUPT;
        if (m.coder() != 0 && !coder_valid(m.coder())) return LIBBSC_DATA_CORRUPT;
        if ((m.lzp_min() != 0 || m.lzp_hash() != 0) && !lzp_valid(m.lzp_hash(), m.lzp_min())) return LIBBSC_DATA_CORRUPT;
        if (Mode::of(m.sorter(), m.coder(), m.lzp_hash(), m.lzp_min()).word != m.word) return LIBBSC_DATA_CORRUPT;    // bits 24..31 set
        if (block_size < LIBBSC_HEADER_SIZE || block_size > LIBBSC_HEADER_SIZE + data_size) return LIBBSC_DATA_CORRUPT;
        if (index < 0 || index > data_size) return LIBBSC_DATA_CORRUPT;
        return LIBBSC_NO_ERROR;
    }
};

// Forward BWT of a block on this context, its sort in a shared slab: the standard sorter, or the batched one when the context's sort
// budget (bscb200_ctx_set_sort_budget) is smaller than the standard working set.
int bwt_encode_leased(Ctx *ctx, u8 *d_T, int n, unsigned char *num_indexes, int *indexes)
{
    if (ctx->sort_budget <= 0 || n <= 1 || (long long)need_bwt_encode((size_t)n) <= ctx->sort_budget) {
        ScratchLease lease(ctx, need_bwt_encode((size_t)n));
        return stage_bwt_encode(ctx, d_T, n, num_indexes, indexes);
    }
    const u32 B = bwt_batch_entries((u32)n, ctx->sort_budget);
    ScratchLease lease(ctx, bwt_batched_bytes((u32)n, B));
    return stage_bwt_encode_batched(ctx, d_T, n, num_indexes, indexes, B);
}

// The same for the forward sort transform of order k (block sorters 3..8)
int st_encode_leased(Ctx *ctx, u8 *d_T, int n, int k)
{
    if (ctx->sort_budget <= 0 || n <= 1 || (long long)need_st_encode((size_t)n) <= ctx->sort_budget) {
        ScratchLease lease(ctx, need_st_encode((size_t)n));
        return stage_st_encode(ctx, d_T, n, k);
    }
    const u32 B = st_batch_entries((u32)n, ctx->sort_budget);
    ScratchLease lease(ctx, st_batched_bytes((u32)n, B));
    return stage_st_encode_batched(ctx, d_T, n, k, B);
}

// ---------------------------------------------------------------------------------------------
// block compress
// ---------------------------------------------------------------------------------------------
// Stored block (libbsc.cpp:68-81) built on the device: header on host, data D2D.
int store_dev(Ctx *ctx, const u8 *d_in, int n, u8 *d_out, u32 adler_data)
{
    if (n > 0) CUDA_TRY(cudaMemcpyAsync(d_out + LIBBSC_HEADER_SIZE, d_in, (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
    BlockHeader{n + LIBBSC_HEADER_SIZE, n, Mode{0}, 0, adler_data, adler_data}.write((unsigned char *)(ctx->h_mail + 64));
    CUDA_TRY(cudaMemcpyAsync(d_out, ctx->h_mail + 64, LIBBSC_HEADER_SIZE, cudaMemcpyHostToDevice, ctx->stream));
    ctx->sync();
    return n + LIBBSC_HEADER_SIZE;
}

// The LZP stage of a block before compression, on the host and not in place (libbsc.cpp:139-154, 264-276).  After run(), `stream` holds
// the LZP stream of the block, or is null: LZP was not asked for, or it did not shrink the block, which goes on without it (mode &= 0xff).
struct LzpPass {
    unsigned char *stream = nullptr;
    int size = 0, hash = 0, min = 0, orig_n = 0;
    u32 adler_orig = 0;

    LzpPass() = default;
    LzpPass(const LzpPass &) = delete; LzpPass &operator=(const LzpPass &) = delete;
    ~LzpPass() { if (stream) bsc_free(stream); }
    int run(const unsigned char *data, int n, int lzpHashSize, int lzpMinLen, int features)
    {
        if (lzpMinLen == 0) return LIBBSC_NO_ERROR;
        stream = (unsigned char *)bsc_malloc((size_t)n + 64);
        if (!stream) return LIBBSC_NOT_ENOUGH_MEMORY;
        size = lzp_host::compress(data, stream, n, lzpHashSize, lzpMinLen, (features & LIBBSC_FEATURE_MULTITHREADING) != 0);
        if (size < 0) { bsc_free(stream); stream = nullptr; return LIBBSC_NO_ERROR; }
        hash = lzpHashSize; min = lzpMinLen; orig_n = n; adler_orig = host_adler32(data, (size_t)n);
        return LIBBSC_NO_ERROR;
    }
};

// The rest of a block once the coder stage returned `result` (its output at d_out + 28, or a code), as libbsc.cpp:181-210 and 311-337
// frame it: LIBBSC_NOT_COMPRESSIBLE unless the block shrinks, else the secondary indexes after the coder output and the header.  H
// describes the block but for its size and the payload Adler-32.  Returns the block's size.
int finish_dev(Ctx *ctx, u8 *d_out, int result, unsigned char num_indexes, const int *indexes, BlockHeader H)
{
    if (result == LIBBSC_NOT_SUPPORTED) return result;
    if (result < 0 || result + 1 + 4 * num_indexes >= H.data_size) return LIBBSC_NOT_COMPRESSIBLE;
    unsigned char *tail = (unsigned char *)(ctx->h_mail + 96);            // pinned, <= 4*255+1 bytes needs care: num_indexes <= 15 here
    memcpy(tail, indexes, 4 * (size_t)num_indexes);
    tail[4 * num_indexes] = num_indexes;
    CUDA_TRY(cudaMemcpyAsync(d_out + LIBBSC_HEADER_SIZE + result, tail, 4 * (size_t)num_indexes + 1, cudaMemcpyHostToDevice, ctx->stream));
    result += 1 + 4 * num_indexes;
    H.block_size = result + LIBBSC_HEADER_SIZE;
    H.adler_payload = stage_adler32(ctx, d_out + LIBBSC_HEADER_SIZE, result);
    unsigned char *h = (unsigned char *)(ctx->h_mail + 64);
    H.write(h);
    CUDA_TRY(cudaMemcpyAsync(d_out, h, LIBBSC_HEADER_SIZE, cudaMemcpyHostToDevice, ctx->stream));
    ctx->sync();
    return H.block_size;
}

// bsc_compress with LZP disabled, everything in HBM.  d_out must hold n + 28 bytes.
// `lz` (host-pointer bsc_compress with LZP parameters only): d_in holds the LZP stream of a block of lz->orig_n bytes; the header describes
// the original block, and a block that does not shrink is reported as LIBBSC_NOT_COMPRESSIBLE (the caller stores the ORIGINAL data,
// libbsc.cpp:315-318).
int compress_dev(Ctx *ctx, const u8 *d_in, int n, u8 *d_out, int blockSorter, int coder, int features, bool inplace_rules, const LzpPass *lz = nullptr)
{
    if (!sorter_valid(blockSorter) || !coder_valid(coder)) return LIBBSC_BAD_PARAMETER;
    if (n < 0 || n > 1073741824) return LIBBSC_BAD_PARAMETER;
    if (lz && n <= LIBBSC_HEADER_SIZE) blockSorter = 1;                  // libbsc.cpp:278-282: a tiny LZP stream is always BWT-sorted
    BlockHeader H;
    H.data_size = lz ? lz->orig_n : n;
    H.mode = Mode::of(blockSorter, coder, lz ? lz->hash : 0, lz ? lz->min : 0);
    H.adler_data = lz ? lz->adler_orig : stage_adler32(ctx, d_in, n);
    if (!lz && n <= LIBBSC_HEADER_SIZE) return store_dev(ctx, d_in, n, d_out, H.adler_data);

    Arena &A = ctx->arena;
    const size_t mark = A.mark();
    u8 *work = A.get<u8>((size_t)n + 64);
    CUDA_TRY(cudaMemcpyAsync(work, d_in, (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));

    int indexes[256]; unsigned char num_indexes = 0;
    if (blockSorter == 1) H.index = bwt_encode_leased(ctx, work, n, &num_indexes, indexes);      // the sort's ~58 n live in a shared slab
    else H.index = st_encode_leased(ctx, work, n, blockSorter);
    if (H.data_size < 64 * 1024) num_indexes = 0;       // libbsc.cpp:303
    if (H.index < 0) { A.release(mark); return H.index; }

    const int result = stage_coder_compress(ctx, work, d_out + LIBBSC_HEADER_SIZE, n, coder, features);
    A.release(mark);
    const int size = finish_dev(ctx, d_out, result, num_indexes, indexes, H);
    if (size == LIBBSC_NOT_COMPRESSIBLE && !inplace_rules && !lz) return store_dev(ctx, d_in, n, d_out, H.adler_data);   // libbsc.cpp:315-318
    return size;
}

// ---------------------------------------------------------------------------------------------
// block decompress, step by step (libbsc.cpp:522-617).  The callers checked the header H (BlockHeader::read) and the sizes, and the
// block's payload lies at d_payload with 64 readable bytes after it.  Only the inverse sort and where the buffers sit differ by path.
// ---------------------------------------------------------------------------------------------
// The coder stage into d_L: returns the length of the sorted (and LZP-coded) data or a code.  A stored block may be empty, so the
// empty payload is rejected here, after the stored blocks have left.
int decode_coder(Ctx *ctx, const BlockHeader &H, const u8 *d_payload, u8 *d_L, int features)
{
    if (H.payload() < 1) return LIBBSC_DATA_CORRUPT;
    return stage_coder_decompress(ctx, d_payload, H.payload(), d_L, H.data_size, H.mode.coder(), features);
}

// libbsc.cpp:599-613: undo the LZP stage of a block on the host, from the lzSize-byte LZP stream at d_lz
int undo_lzp_host(Ctx *ctx, const BlockHeader &H, const u8 *d_lz, int lzSize, unsigned char *output)
{
    const int dataSize = H.data_size;
    // the LZP stream, then the data after it: the caller's buffer is written only once the data is known to be right
    unsigned char *lz = (unsigned char *)bsc_malloc((size_t)lzSize + (size_t)dataSize + 1);
    if (!lz) return LIBBSC_NOT_ENOUGH_MEMORY;
    unsigned char *data = lz + lzSize;
    if (lzSize > 0) { CUDA_TRY(cudaMemcpyAsync(lz, d_lz, (size_t)lzSize, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
    int r = lzp_host::decompress(lz, lzSize, data, dataSize, H.mode.lzp_hash(), H.mode.lzp_min());
    if (r >= 0) r = (r == dataSize && H.adler_data == host_adler32(data, (size_t)dataSize)) ? LIBBSC_NO_ERROR : LIBBSC_DATA_CORRUPT;
    if (r == LIBBSC_NO_ERROR && dataSize > 0) memcpy(output, data, (size_t)dataSize);
    bsc_free(lz);
    return r;
}

// The last step, once the inverse sort left lzSize bytes at d_T: undo LZP on the host, or check the length and the data Adler-32 and
// copy the data to `output` (null on the device-resident entry point).  `output` is written only once the data is known to be right.
int deliver(Ctx *ctx, const BlockHeader &H, const u8 *d_T, int lzSize, unsigned char *output)
{
    if (H.mode.has_lzp()) return undo_lzp_host(ctx, H, d_T, lzSize, output);
    if (lzSize != H.data_size || H.adler_data != stage_adler32(ctx, d_T, H.data_size)) return LIBBSC_DATA_CORRUPT;
    if (output && H.data_size > 0) { CUDA_TRY(cudaMemcpyAsync(output, d_T, (size_t)H.data_size, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
    return LIBBSC_NO_ERROR;
}

// The secondary indexes at the end of a BWT block's payload (`payload` bytes at d_payload) for a text of n bytes.  The product's inverse
// BWT does not use them, but the reference does whenever their count is the one bsc_bwt_encode writes for n (bwt.cpp:295-310), and
// then libsais_unbwt_aux rejects values outside 0..n - 1 with LIBBSC_BAD_PARAMETER before it decodes.  True for such a block.
bool secondary_indexes_out_of_range(Ctx *ctx, const u8 *d_payload, int payload, int n, int index)
{
    if (n <= 1 || index <= 0 || index > n) return false;                  // stage_bwt_decode answers first, as bsc_bwt_decode does
    int mod = n / 8;
    mod |= mod >> 1; mod |= mod >> 2; mod |= mod >> 4; mod |= mod >> 8; mod |= mod >> 16; mod >>= 1;
    const int want = (unsigned char)((n - 1) / (mod + 1));               // at most 15
    unsigned char tail[1 + 4 * 16];
    const int k = payload < (int)sizeof(tail) ? payload : (int)sizeof(tail);
    CUDA_TRY(cudaMemcpyAsync(tail, d_payload + payload - k, (size_t)k, cudaMemcpyDeviceToHost, ctx->stream));
    ctx->sync();
    const int count = tail[k - 1];
    if (count != want || 4 * count + 1 > k) return false;
    for (int t = 0; t < count; ++t) {
        const long long v = (long long)(int)get32(tail + k - 1 - 4 * count + 4 * t) + 1;
        if (v <= 0 || v > n) return true;
    }
    return false;
}

// bsc_decompress of the block at d_block on a context's arena: the inverse BWT in the arena, ST3..ST8 in a shared slab.  The data lands
// at d_out, and in `output` for host callers.  The device-resident entry point passes no `output`: LZP stays on the host side of the
// boundary.
int decompress_dev(Ctx *ctx, const BlockHeader &H, const u8 *d_block, u8 *d_out, unsigned char *output, int features)
{
    const u8 *d_payload = d_block + LIBBSC_HEADER_SIZE;
    if (H.adler_payload != stage_adler32(ctx, d_payload, H.payload())) return LIBBSC_DATA_CORRUPT;
    if (H.mode.word == 0) {
        // A stored block carries exactly dataSize payload bytes (bsc_store, libbsc.cpp:68-81).  The reference copies dataSize bytes
        // whatever blockSize says (libbsc.cpp:550-555), reading past a shorter block; here such a header is corrupt.  Like the reference,
        // the data Adler-32 of a stored block is not checked: the payload Adler-32 above covers the same bytes.
        if (H.payload() != H.data_size) return LIBBSC_DATA_CORRUPT;
        if (H.data_size > 0) CUDA_TRY(cudaMemcpyAsync(d_out, d_payload, (size_t)H.data_size, cudaMemcpyDeviceToDevice, ctx->stream));
        ctx->sync();
        if (output && H.data_size > 0) { CUDA_TRY(cudaMemcpyAsync(output, d_out, (size_t)H.data_size, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return LIBBSC_NO_ERROR;
    }
    if (H.mode.has_lzp() && !output) return LIBBSC_NOT_SUPPORTED;
    const int lzSize = decode_coder(ctx, H, d_payload, d_out, features);
    if (lzSize < 0) return lzSize;
    const int sorter = H.mode.sorter();
    if (!sorter_valid(sorter)) return LIBBSC_DATA_CORRUPT;               // sorter field 0 with a coder: libbsc.cpp:593, after the coder stage
    int r;
    if (sorter == 1) {
        if (secondary_indexes_out_of_range(ctx, d_payload, H.payload(), lzSize, H.index)) return LIBBSC_BAD_PARAMETER;
        r = stage_bwt_decode(ctx, d_out, lzSize, H.index);
    }
    else { ScratchLease lease(ctx, need_st_decode((size_t)lzSize)); r = stage_st_decode(ctx, d_out, lzSize, sorter, H.index); }   // libbsc.cpp:584-589
    if (r < 0) return r;
    return deliver(ctx, H, d_out, lzSize, output);
}

// ---------------------------------------------------------------------------------------------
// blocks above 1 GiB: in-place bsc_compress, and bsc_decompress of such blocks
// ---------------------------------------------------------------------------------------------
// On the pooled path a block of n bytes holds about 31 n of HBM: the staged block, its working copy, the output and the coder stage in
// the context, and a 16.5 n sort slab that the pool keeps after the call.  A block above 1 GiB instead runs on a context made for the
// call and destroyed after it, in ONE allocation: the block, sorted in place (an in-place call may destroy its input, libbsc.cpp:160),
// and a region that first holds the batched forward BWT (16 n + 32 B) and then the coder stage with its output (about 9.5 n + 28 MB).
// The caller's buffer is written only once the block is done.  In place, ST3..ST8 compress only up to 1 GiB; bsc_st_encode above it has
// a bounded path of its own (st_encode_large below), and their inverse a lean layout (decompress_large_st below).
// The arena is 17.5 n + 128 MiB: the batched sort at batches of about n / 64 entries (16.5 n) or the coder stage with its output
// (at most 9.5 n + 28 MB) after the block.  The bound adds n / 2 + 128 MiB for what lies outside the arena: the context, the coder
// tables, kernel images loaded on first use and the driver's own transient allocations (about 0.55 GB measured at the largest n).
constexpr int LARGE_N = 1073741824;                  // blocks above this take the path below
// Where bsc_compress (in place) and bsc_decompress route: LARGE_N, or BSCB200_LARGE_N=<bytes> (read once per process) when it lies in
// 0..LARGE_N.  The switch is for tests only: it lets blocks of a few bytes up take the paths below, which blocks above 1 GiB take in
// production.  The argument limits, the HBM bounds and the CLI stay keyed on LARGE_N itself.
int large_route_n()
{
    static const int v = [] {
        const char *e = getenv("BSCB200_LARGE_N");
        char *end = nullptr;
        const long long t = e ? strtoll(e, &end, 10) : -1;
        return (e && end != e && *end == '\0' && t >= 0 && t <= LARGE_N) ? (int)t : LARGE_N;
    }();
    return v;
}
constexpr size_t LARGE_FIXED = 256u << 20;
size_t large_bound(size_t n) { return 18 * n + LARGE_FIXED; }
size_t large_arena(size_t n) { return 17 * n + n / 2 + LARGE_FIXED / 2; }
// bsc_decompress of an ST3..ST8 block whose data size n is above 1 GiB: ONE arena holds L (n + 128) and a region of
// st_decode_lean_bytes(n) = 25 n + 1 MiB after it.  The compressed block (at most n + 28) sits at the top end of that region while the
// coder stage (at most 12 n + 64 MB) works below it; the inverse ST then takes the whole region in its lean layout (st_decode.cu), and
// its output lands there too.  26 n + 1 MiB in all, the block included.  The bound adds n / 2 + 255 MiB for what lies outside the
// arena, as large_bound does: 26.5 n + 256 MiB, 57.2 GB at n = 2146435072.
// Below about 5.3 MiB (a routed test block) the block and the coder stage need more than 25 n + 1 MiB: the decoder alone takes 3.4 MB
// of model state per stream.  The region is then the block plus the coder stage, which stays within the bound.
size_t large_st_region(size_t n) { return std::max(st_decode_lean_bytes(n), align_up(n + 28 + 128, 256) + need_coder(n)); }
size_t large_st_arena(size_t n) { return align_up(n + 128 + 256, 256) + align_up(large_st_region(n), 256); }
size_t large_st_bound(size_t n) { return 26 * n + n / 2 + LARGE_FIXED; }
// bsc_st_encode of a block above 1 GiB: ONE arena of 5.5 n + 128 MiB holds the staged block (n + 64) and the batched forward ST after it
// (st_batched_bytes: L, n bytes, and 28 bytes per batch entry), whose batches take what is left: about n / 8 entries.  The bound adds
// n / 2 + 128 MiB for what lies outside the arena, as large_bound does: 6 n + 256 MiB, 13.1 GB at n = 2146435072.
size_t st_large_arena(size_t n) { return 5 * n + n / 2 + LARGE_FIXED / 2; }
size_t st_large_bound(size_t n) { return 6 * n + LARGE_FIXED; }

// In-place bsc_compress of a block of n > 1 GiB bytes with the BWT sorter (libbsc.cpp:124-210).
int compress_large(unsigned char *data, int n, int lzpHashSize, int lzpMinLen, int coder, int features)
{
    size_t fr = 0, total = 0;
    if (cudaMemGetInfo(&fr, &total) != cudaSuccess) { cudaGetLastError(); return LIBBSC_GPU_NOT_SUPPORTED; }
    if (fr < large_bound((size_t)n)) return LIBBSC_GPU_NOT_ENOUGH_MEMORY;

    LzpPass lz;
    const int e = lz.run(data, n, lzpHashSize, lzpMinLen, features);
    if (e != LIBBSC_NO_ERROR) return e;
    const unsigned char *src = lz.stream ? lz.stream : data;
    const int m = lz.stream ? lz.size : n;                  // bytes that go through the sort and the coder
    return with_own_ctx([&](Ctx *ctx) {
        Arena &A = ctx->arena;
        A.reserve(large_arena((size_t)n));
        u8 *d_blk = A.get<u8>((size_t)m + 64);
        CUDA_TRY(cudaMemcpyAsync(d_blk, src, (size_t)m, cudaMemcpyHostToDevice, ctx->stream));
        BlockHeader H;
        H.data_size = n;
        H.mode = Mode::of(1, coder, lz.hash, lz.min);
        H.adler_data = lz.stream ? lz.adler_orig : stage_adler32(ctx, d_blk, m);
        // the sort may use the whole region after the block (less a margin for the arena's rounding): batches of about n / 64 entries
        const u32 B = bwt_batch_entries((u32)m, (long long)(A.cap - A.used) - (16ll << 20));
        int indexes[256]; unsigned char num_indexes = 0;
        H.index = stage_bwt_encode_batched(ctx, d_blk, m, &num_indexes, indexes, B);
        if (H.index < 0) return H.index;
        u8 *d_out = A.get<u8>((size_t)m + 4096) + 4;       // payload (offset 28) lands 16-byte aligned
        const int result = stage_coder_compress(ctx, d_blk, d_out + LIBBSC_HEADER_SIZE, m, coder, features);
        const int size = finish_dev(ctx, d_out, result, num_indexes, indexes, H);
        if (size < 0) return size;
        CUDA_TRY(cudaMemcpyAsync(data, d_out, (size_t)size, cudaMemcpyDeviceToHost, ctx->stream));
        ctx->sync();
        return size;
    });
}

// bsc_decompress of a block with block sorter 3..8 whose data size is above 1 GiB (large_st_arena above).  The caller checked the header
// and the sizes.  The caller's buffer is written only on success.
int decompress_large_st(const unsigned char *input, const BlockHeader &H, unsigned char *output, int features)
{
    size_t fr = 0, total = 0;
    if (cudaMemGetInfo(&fr, &total) != cudaSuccess) { cudaGetLastError(); return LIBBSC_GPU_NOT_SUPPORTED; }
    if (fr < large_st_bound((size_t)H.data_size)) return LIBBSC_GPU_NOT_ENOUGH_MEMORY;
    return with_own_ctx([&](Ctx *ctx) {
        Arena &A = ctx->arena;
        A.reserve(large_st_arena((size_t)H.data_size));
        u8 *d_L = A.get<u8>((size_t)H.data_size + 128);
        const size_t full = A.cap, blk = align_up((size_t)H.block_size + 128, 256);
        u8 *d_blk = A.base + full - blk + 4;                 // the top end of the region; payload (offset 28) lands 16-byte aligned
        CUDA_TRY(cudaMemcpyAsync(d_blk, input, (size_t)H.block_size, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(cudaMemsetAsync(d_blk + H.block_size, 0, 64, ctx->stream));
        const u8 *d_payload = d_blk + LIBBSC_HEADER_SIZE;
        if (H.adler_payload != stage_adler32(ctx, d_payload, H.payload())) return LIBBSC_DATA_CORRUPT;
        A.cap = full - blk;                                  // the coder stage stays below the block
        const int lzSize = decode_coder(ctx, H, d_payload, d_L, features);
        A.cap = full;
        if (lzSize < 0) return lzSize;
        u8 *d_T = nullptr;                                   // the block is dead: the inverse ST takes the whole region after L
        const int r = stage_st_decode_lean(ctx, d_L, lzSize, H.mode.sorter(), H.index, &d_T);
        if (r < 0) return r;
        return deliver(ctx, H, d_T, lzSize, output);
    });
}

// bsc_st_encode of T (n bytes) above the routing threshold (st_large_arena above).  The caller checked the arguments.  T is written only
// on success.
int st_encode_large(unsigned char *T, int n, int k)
{
    size_t fr = 0, total = 0;
    if (cudaMemGetInfo(&fr, &total) != cudaSuccess) { cudaGetLastError(); return LIBBSC_GPU_NOT_SUPPORTED; }
    if (fr < st_large_bound((size_t)n)) return LIBBSC_GPU_NOT_ENOUGH_MEMORY;
    return with_own_ctx([&](Ctx *ctx) {
        Arena &A = ctx->arena;
        A.reserve(st_large_arena((size_t)n));
        u8 *d = A.get<u8>((size_t)n + 64);
        CUDA_TRY(cudaMemcpyAsync(d, T, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        // the sort may use the rest of the arena (less a margin for its rounding)
        const u32 B = st_batch_entries((u32)n, (long long)(A.cap - A.used) - (16ll << 20));
        const int r = stage_st_encode_batched(ctx, d, n, k, B);
        if (r >= 0) { CUDA_TRY(cudaMemcpyAsync(T, d, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
}

// ---------------------------------------------------------------------------------------------
// host-pointer stage entry points: the data goes in, through one stage on the device, and back when the stage succeeds
// ---------------------------------------------------------------------------------------------
// T (n bytes) through `stage(ctx, d_T)`, which works in place; T is written back when the stage returns r >= 0.
template <class F> int stage_in_place(unsigned char *T, int n, size_t reserve, F stage)
{
    return with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve(reserve);
        u8 *d = ctx->arena.get<u8>((size_t)n + 64);
        if (n > 0) CUDA_TRY(cudaMemcpyAsync(d, T, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        const int r = stage(ctx, d);
        if (r >= 0 && n > 0) { CUDA_TRY(cudaMemcpyAsync(T, d, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
}

// inSize bytes at `input` through `stage(ctx, d_in, d_out)` into a device buffer of out_room bytes; the r > 0 bytes the stage returns
// go to `output`.  The decoders (`pad`) read ahead: 64 zero bytes follow their input.
template <class F> int stage_to_output(const unsigned char *input, int inSize, unsigned char *output, size_t out_room, size_t reserve, bool pad, F stage)
{
    return with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve(reserve);
        u8 *d_in = ctx->arena.get<u8>((size_t)inSize + (pad ? 128 : 64));
        u8 *d_out = ctx->arena.get<u8>(out_room);
        CUDA_TRY(cudaMemcpyAsync(d_in, input, (size_t)inSize, cudaMemcpyHostToDevice, ctx->stream));
        if (pad) CUDA_TRY(cudaMemsetAsync(d_in + inSize, 0, 64, ctx->stream));
        const int r = stage(ctx, d_in, d_out);
        if (r > 0) { CUDA_TRY(cudaMemcpyAsync(output, d_out, (size_t)r, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// exported C ABI
// ---------------------------------------------------------------------------------------------
extern "C" {

int bsc_platform_init(int features, void *(*malloc_fn)(size_t), void *(*zero_malloc_fn)(size_t), void (*free_fn)(void *))
{
    (void)features;
    if (malloc_fn && zero_malloc_fn && free_fn) { g_malloc = malloc_fn; g_zero_malloc = zero_malloc_fn; g_free = free_fn; }
    return LIBBSC_NO_ERROR;
}
void *bsc_malloc(size_t size) { return g_malloc ? g_malloc(size) : malloc(size); }
void *bsc_zero_malloc(size_t size) { return g_zero_malloc ? g_zero_malloc(size) : calloc(1, size); }
void bsc_free(void *p) { if (g_free) g_free(p); else free(p); }

int bsc_init_full(int features, void *(*malloc_fn)(size_t), void *(*zero_malloc_fn)(size_t), void (*free_fn)(void *))
{
    bsc_platform_init(features, malloc_fn, zero_malloc_fn, free_fn);
    // Blocks run on independent streams; give every stream its own hardware queue (default 8 would
    // alias streams and serialise long coder kernels).  Only effective before the CUDA context exists.
    setenv("CUDA_DEVICE_MAX_CONNECTIONS", "32", 0);
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count < 1) { cudaGetLastError(); return LIBBSC_GPU_NOT_SUPPORTED; }
    return LIBBSC_NO_ERROR;
}
int bsc_init(int features) { return bsc_init_full(features, nullptr, nullptr, nullptr); }
int bsc_bwt_init(int) { return LIBBSC_NO_ERROR; }
int bsc_st_init(int) { return LIBBSC_NO_ERROR; }
int bsc_coder_init(int) { return LIBBSC_NO_ERROR; }
int bsc_qlfc_init(int) { return LIBBSC_NO_ERROR; }

unsigned int bsc_adler32(const unsigned char *T, int n, int features)
{
    (void)features;
    if (n < (1 << 16)) return host_adler32(T, (size_t)(n > 0 ? n : 0));   // headers / tiny buffers
    unsigned int value = 0;
    int r = with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve((size_t)n + (1u << 20));
        u8 *d = ctx->arena.get<u8>((size_t)n + 64);
        CUDA_TRY(cudaMemcpyAsync(d, T, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        value = stage_adler32(ctx, d, n);
        return 0;
    });
    return r == 0 ? value : host_adler32(T, (size_t)n);
}

int bsc_store(const unsigned char *input, unsigned char *output, int n, int features)
{
    (void)features;
    if (n < 0) return LIBBSC_BAD_PARAMETER;
    unsigned int a = bsc_adler32(input, n, features);
    memmove(output + LIBBSC_HEADER_SIZE, input, (size_t)n);
    BlockHeader{n + LIBBSC_HEADER_SIZE, n, Mode{0}, 0, a, a}.write(output);
    return n + LIBBSC_HEADER_SIZE;
}

int bsc_block_info(const unsigned char *blockHeader, int headerSize, int *pBlockSize, int *pDataSize, int features)
{
    (void)features;
    BlockHeader H;
    const int r = H.read(blockHeader, headerSize);
    if (r != LIBBSC_NO_ERROR) return r;
    if (pBlockSize) *pBlockSize = H.block_size;
    if (pDataSize) *pDataSize = H.data_size;
    return LIBBSC_NO_ERROR;
}

int bsc_compress(const unsigned char *input, unsigned char *output, int n, int lzpHashSize, int lzpMinLen, int blockSorter, int coder, int features)
{
    if (!sorter_valid(blockSorter) || !coder_valid(coder)) return LIBBSC_BAD_PARAMETER;
    if (lzpMinLen != 0 || lzpHashSize != 0) {
        if (!lzp_valid(lzpHashSize, lzpMinLen)) return LIBBSC_BAD_PARAMETER;
        // The LZP stage runs on the host (lzp_host.h: all five x86-64 variants of the reference; north star: libbsc/lzp stays on the host).
        if (!lzp_host::supported(lzpHashSize, lzpMinLen)) return LIBBSC_NOT_SUPPORTED;
    }
    const bool inplace = (input == output);
    if (n < 0 || n > (inplace ? 2146435072 : 1073741824)) return LIBBSC_BAD_PARAMETER;
    if (n <= LIBBSC_HEADER_SIZE) return bsc_store(input, output, n, features);
    // In place only: compress_large works on its argument in place.  Out of place, blocks above 1 GiB were refused above, and below it a
    // lowered routing threshold (tests) keeps them on the pooled path.
    if (inplace && n > large_route_n()) return blockSorter == 1 ? compress_large(output, n, lzpHashSize, lzpMinLen, coder, features) : LIBBSC_NOT_SUPPORTED;
    LzpPass lz;
    int r = lz.run(input, n, lzpHashSize, lzpMinLen, features);
    if (r != LIBBSC_NO_ERROR) return r;
    const unsigned char *src = lz.stream ? lz.stream : input;
    const int m = lz.stream ? lz.size : n;
    r = with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve(host_compress_bytes(n));
        u8 *d_in = ctx->arena.get<u8>((size_t)m + 64);
        u8 *d_out = ctx->arena.get<u8>((size_t)n + 4096) + 4;      // payload (offset 28) lands 16-byte aligned
        if (m > 0) CUDA_TRY(cudaMemcpyAsync(d_in, src, (size_t)m, cudaMemcpyHostToDevice, ctx->stream));
        const int size = compress_dev(ctx, d_in, m, d_out, blockSorter, coder, features, inplace, lz.stream ? &lz : nullptr);
        if (size > 0) { CUDA_TRY(cudaMemcpyAsync(output, d_out, (size_t)size, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return size;
    });
    if (r == LIBBSC_NOT_COMPRESSIBLE && lz.stream && !inplace) return bsc_store(input, output, n, features);
    return r;
}

int bsc_decompress(const unsigned char *input, int inputSize, unsigned char *output, int outputSize, int features)
{
    BlockHeader H;
    const int info = H.read(input, inputSize);
    if (info != LIBBSC_NO_ERROR) return info;
    if (inputSize < H.block_size || outputSize < H.data_size) return LIBBSC_UNEXPECTED_EOB;
    const bool large = H.data_size > large_route_n();
    if (large && H.mode.sorter() >= 3) return decompress_large_st(input, H, output, features);
    // Above 1 GiB (BWT and stored blocks): on a context of its own that does not keep its HBM after the call.
    auto body = [&](Ctx *ctx) {
        ctx->arena.reserve(host_decompress_bytes((size_t)H.block_size, (size_t)H.data_size));
        u8 *d_blk = ctx->arena.get<u8>((size_t)H.block_size + 128) + 4;
        u8 *d_out = ctx->arena.get<u8>((size_t)H.data_size + 128);
        CUDA_TRY(cudaMemcpyAsync(d_blk, input, (size_t)H.block_size, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(cudaMemsetAsync(d_blk + H.block_size, 0, 64, ctx->stream));
        return decompress_dev(ctx, H, d_blk, d_out, output, features);
    };
    return large ? with_own_ctx(body) : with_ctx(body);
}

int bsc_bwt_encode(unsigned char *T, int n, unsigned char *num_indexes, int *indexes, int features)
{
    (void)features;
    if (T == nullptr || n < 0) return LIBBSC_BAD_PARAMETER;
    return stage_in_place(T, n, (size_t)n + 4096, [&](Ctx *ctx, u8 *d) { return bwt_encode_leased(ctx, d, n, num_indexes, indexes); });
}

int bsc_bwt_decode(unsigned char *T, int n, int index, unsigned char num_indexes, int *indexes, int features)
{
    (void)num_indexes; (void)indexes; (void)features;    // secondary indexes are CPU accelerators only (bwt.cpp:263 ignores them on the GPU too)
    if (T == nullptr || n < 0 || index <= 0 || index > n) return LIBBSC_BAD_PARAMETER;
    if (n <= 1) return LIBBSC_NO_ERROR;
    return stage_in_place(T, n, Arena::bytes_for<u8>((size_t)n + 64) + bwt_decode_bytes((u32)n),
                          [&](Ctx *ctx, u8 *d) { return stage_bwt_decode(ctx, d, n, index); });
}

int bsc_st_encode(unsigned char *T, int n, int k, int features)
{
    (void)features;
    if (T == nullptr || n < 0) return LIBBSC_BAD_PARAMETER;
    if (!st_order_valid(k)) return LIBBSC_BAD_PARAMETER;
    if (n <= 1) return 0;
    if (n > large_route_n()) return st_encode_large(T, n, k);
    return stage_in_place(T, n, (size_t)n + 4096, [&](Ctx *ctx, u8 *d) { return st_encode_leased(ctx, d, n, k); });
}

int bsc_st_decode(unsigned char *T, int n, int k, int index, int features)
{
    (void)features;
    if (T == nullptr || n < 0) return LIBBSC_BAD_PARAMETER;       // st.cpp:1493-1496
    if (index < 0 || index >= n) return LIBBSC_BAD_PARAMETER;
    if (!st_order_valid(k)) return LIBBSC_BAD_PARAMETER;
    if (n <= 1) return LIBBSC_NO_ERROR;
    return stage_in_place(T, n, (size_t)n + 4096, [&](Ctx *ctx, u8 *d) { ScratchLease lease(ctx, need_st_decode(n)); return stage_st_decode(ctx, d, n, k, index); });
}

int bsc_coder_compress(const unsigned char *input, unsigned char *output, int n, int coder, int features)
{
    if (!coder_valid(coder)) return LIBBSC_BAD_PARAMETER;
    if (n <= 0) return LIBBSC_BAD_PARAMETER;
    return stage_to_output(input, n, output, (size_t)n + 4096, 2 * (size_t)n + 16384 + need_coder(n), false,
                           [&](Ctx *ctx, const u8 *d_in, u8 *d_out) { return stage_coder_compress(ctx, d_in, d_out, n, coder, features); });
}

// Size-aware variant used by bsc_decompress and exported for integrators.
int bscb200_coder_decompress(const unsigned char *input, int inputSize, unsigned char *output, int outputCapacity, int coder, int features)
{
    if (!coder_valid(coder)) return LIBBSC_BAD_PARAMETER;
    if (inputSize < 1 || outputCapacity < 0) return LIBBSC_BAD_PARAMETER;
    return stage_to_output(input, inputSize, output, (size_t)outputCapacity + 128,
                           (size_t)inputSize + (size_t)outputCapacity + 16384 + need_coder((size_t)outputCapacity), true,
                           [&](Ctx *ctx, const u8 *d_in, u8 *d_out) { return stage_coder_decompress(ctx, d_in, inputSize, d_out, outputCapacity, coder, features); });
}

// The uncompressed size n of a QLFC stream = its first 32 range-coded bits, each with p = 1/2 (qlfc.cpp:852; rangecoder.h:203-240).
// Needs 14 readable bytes.  Returns -1 for n > 2^31 - 1.
static long long qlfc_stream_size(const unsigned char *p)
{
    unsigned int code = ((unsigned)p[2] | ((unsigned)p[3] << 8)) << 16 | ((unsigned)p[4] | ((unsigned)p[5] << 8));
    unsigned int range = 0xffffffffu, nn = 0; int pos = 6;
    for (int b = 0; b < 32; ++b) {
        if (range < 0x10000u) { range <<= 16; code = (code << 16) | ((unsigned)p[pos] | ((unsigned)p[pos + 1] << 8)); pos += 2; }
        unsigned int r = (range >> 12) * 2048u;
        if (code >= r) { code -= r; range -= r; nn = (nn << 1) | 1u; } else { range = r; nn <<= 1; }
    }
    return nn > 0x7fffffffu ? -1 : (long long)nn;
}

// libbsc's own signature carries no sizes (coder.h:66).  They are recovered from the container: the sub-block table for
// nBlocks > 1; for a single sub-block the uncompressed size n is coded in the stream and the stream itself is shorter than n
// (bsc_coder_compress stores a sub-block raw otherwise).  CALLER CONTRACT for the size-less ABI: the n + 17 bytes after `input`
// are either part of the stream or unmapped -- they are copied to the device as far as they are mapped (never read by the decoder
// beyond the stream's end).  Integrators that know their sizes should call bscb200_coder_decompress.
int bsc_coder_decompress(const unsigned char *input, unsigned char *output, int coder, int features)
{
    if (!coder_valid(coder)) return LIBBSC_BAD_PARAMETER;
    int nBlocks = input[0];
    long long inSize = 0, outSize = 0;
    if (nBlocks == 1) {
        outSize = qlfc_stream_size(input + 1);
        if (outSize < 0) return LIBBSC_DATA_CORRUPT;
        inSize = (long long)readable_prefix(input, (size_t)outSize + 1 + 16);
    } else {
        if (nBlocks > 8) return LIBBSC_DATA_CORRUPT;        // nBlocks == 0: an empty container, 0 bytes (coder.cpp:339-346)
        inSize = 1 + 8 * nBlocks;
        for (int b = 0; b < nBlocks; ++b) { outSize += (int)get32(input + 1 + 8 * b); inSize += (int)get32(input + 5 + 8 * b); }
    }
    if (inSize > 0x7fffffffLL || outSize > 0x7fffffffLL) return LIBBSC_DATA_CORRUPT;
    return bscb200_coder_decompress(input, (int)inSize, output, (int)outSize, coder, features);
}

// ---- one QLFC stream at a time (libbsc/coder/qlfc/qlfc.h:55-99; qlfc.cpp:2138-2226) ------------------------------------------
static int qlfc_encode_block(int coder, const unsigned char *input, unsigned char *output, int inputSize, int outputSize)
{
    if (inputSize <= 0 || outputSize < 0) return LIBBSC_BAD_PARAMETER;
    const size_t room = (size_t)(outputSize > inputSize ? outputSize : inputSize);
    return stage_to_output(input, inputSize, output, room + 4096, 2 * room + (size_t)inputSize + 16384 + need_coder(room), false,
                           [&](Ctx *ctx, const u8 *d_in, u8 *d_out) { return stage_coder_compress(ctx, d_in, d_out, inputSize, coder, 0, outputSize); });
}
// Size-less like the reference's: n comes from the stream; the stream is taken to be at most n + 16 bytes long (what
// bsc_qlfc_*_encode_block produces with outputSize <= inputSize; same caller contract as bsc_coder_decompress above).
static int qlfc_decode_block(int coder, const unsigned char *input, unsigned char *output)
{
    const long long n = qlfc_stream_size(input);
    if (n < 0) return LIBBSC_DATA_CORRUPT;
    const int inSize = (int)readable_prefix(input, (size_t)n + 16);
    if (inSize < 14) return LIBBSC_UNEXPECTED_EOB;
    return stage_to_output(input, inSize, output, (size_t)n + 128, (size_t)inSize + (size_t)n + 16384 + need_coder((size_t)n), true,
                           [&](Ctx *ctx, const u8 *d_in, u8 *d_out) { return stage_coder_decompress(ctx, d_in, inSize, d_out, (int)n, coder, 0, true); });
}
int bsc_qlfc_static_encode_block(const unsigned char *input, unsigned char *output, int inputSize, int outputSize) { return qlfc_encode_block(1, input, output, inputSize, outputSize); }
int bsc_qlfc_adaptive_encode_block(const unsigned char *input, unsigned char *output, int inputSize, int outputSize) { return qlfc_encode_block(2, input, output, inputSize, outputSize); }
int bsc_qlfc_fast_encode_block(const unsigned char *input, unsigned char *output, int inputSize, int outputSize) { return qlfc_encode_block(3, input, output, inputSize, outputSize); }
int bsc_qlfc_static_decode_block(const unsigned char *input, unsigned char *output) { return qlfc_decode_block(1, input, output); }
int bsc_qlfc_adaptive_decode_block(const unsigned char *input, unsigned char *output) { return qlfc_decode_block(2, input, output); }
int bsc_qlfc_fast_decode_block(const unsigned char *input, unsigned char *output) { return qlfc_decode_block(3, input, output); }

// ---- extensions: explicit contexts and device-resident operation ------------------------------
void *bscb200_ctx_create(int device, void *cuda_stream)
{
    try { return ctx_new(device, (cudaStream_t)cuda_stream, cuda_stream == nullptr); } catch (...) { cudaGetLastError(); return nullptr; }
}
void bscb200_ctx_destroy(void *ctx) { ctx_delete((Ctx *)ctx); }
int bscb200_ctx_reserve(void *ctx, long long bytes)
{
    Ctx *c = (Ctx *)ctx;
    return guarded(c, [&]() { CUDA_TRY(cudaSetDevice(c->device)); c->arena.reset(); c->arena.reserve((size_t)bytes); return 0; });
}
// Bounds the working set of the forward sorts on this context, the BWT and the sort transforms (block sorters 3..8): each sorts in
// batches whenever its standard sorter would need more than `bytes` (0 = no bound).
int bscb200_ctx_set_sort_budget(void *ctx, long long bytes)
{
    if (!ctx || bytes < 0) return LIBBSC_BAD_PARAMETER;
    ((Ctx *)ctx)->sort_budget = bytes;
    return LIBBSC_NO_ERROR;
}
// Per-context workspace: the staged block + the coder stage (the inverse BWT reuses the coder's space).  The sort stages work in
// the device-wide scratch slabs (scratch pool above), which is what lets dozens of blocks be in flight per GPU.
long long bscb200_workspace_bytes(int n, int blockSorter)
{
    (void)blockSorter;
    return (long long)ctx_workspace((size_t)n);
}
long long bscb200_scratch_bytes(int n, int blockSorter)     /* size of one shared sort slab for blocks of n bytes */
{
    size_t s = (blockSorter == 1 ? need_bwt_encode((size_t)n) : need_st_encode((size_t)n));
    size_t d = blockSorter == 1 ? 0 : need_st_decode((size_t)n);
    return (long long)(s > d ? s : d);
}
// HBM that an in-place bsc_compress of a block above 1 GiB, or bsc_decompress of one, takes at most: 18 n + 256 MiB (large_bound)
long long bscb200_inplace_bytes(int n, int blockSorter, int coder)
{
    if (n < 0 || n > 2146435072 || !sorter_valid(blockSorter) || !coder_valid(coder)) return LIBBSC_BAD_PARAMETER;
    if (blockSorter != 1) return LIBBSC_NOT_SUPPORTED;      // the in-place bsc_compress does not encode ST3..ST8 above 1 GiB
    return (long long)large_bound((size_t)n);
}
// HBM that bsc_st_encode of n bytes takes at most: above 1 GiB the bound of its own context (st_large_bound), else the pooled cost, the
// staged block in a context and one shared sort slab
long long bscb200_st_encode_bytes(int n)
{
    if (n < 0 || n > 2146435072) return LIBBSC_BAD_PARAMETER;
    if (n > LARGE_N) return (long long)st_large_bound((size_t)n);
    return (long long)((size_t)n + 4096 + need_st_encode((size_t)n));
}
// HBM that bsc_decompress of a block with data size n takes at most: above 1 GiB the bound of its own context (large_bound for the BWT,
// large_st_bound for ST3..ST8), else the pooled cost, one context's workspace and one shared sort slab
long long bscb200_decompress_bytes(int n, int blockSorter)
{
    if (n < 0 || n > 2146435072 || !sorter_valid(blockSorter)) return LIBBSC_BAD_PARAMETER;
    if (n > LARGE_N) return (long long)(blockSorter == 1 ? large_bound((size_t)n) : large_st_bound((size_t)n));
    return bscb200_workspace_bytes(n, blockSorter) + bscb200_scratch_bytes(n, blockSorter);
}
// host-only: the inverse LZP stage by itself (what bsc_decompress runs after the GPU stages), for CPU tests against the reference
int bscb200_lzp_decompress_host(const unsigned char *input, int n, unsigned char *output, int outputCapacity, int lzpHashSize, int lzpMinLen)
{
    if (!input || !output || n < 0 || outputCapacity < 0 || !lzp_valid(lzpHashSize, lzpMinLen)) return LIBBSC_BAD_PARAMETER;
    return lzp_host::decompress(input, n, output, outputCapacity, lzpHashSize, lzpMinLen);
}

// host-only: the forward LZP stage by itself (bsc_lzp_compress, lzp.h); LIBBSC_NOT_SUPPORTED for the parameter classes whose
// reference variant is not restated (lzp_host.h)
int bscb200_lzp_compress_host(const unsigned char *input, unsigned char *output, int n, int lzpHashSize, int lzpMinLen, int features)
{
    if (!input || !output || n < 0 || !lzp_valid(lzpHashSize, lzpMinLen)) return LIBBSC_BAD_PARAMETER;
    if (!lzp_host::supported(lzpHashSize, lzpMinLen)) return LIBBSC_NOT_SUPPORTED;
    return lzp_host::compress(input, output, n, lzpHashSize, lzpMinLen, (features & LIBBSC_FEATURE_MULTITHREADING) != 0);
}

// Multi-GPU callers (libbsc_b200/cli/bsc_b200.cpp, one worker thread per GPU slot): every entry point works on the CURRENT device
// of the calling thread, so a worker only has to bind itself once.  Plain wrappers, so that callers need no CUDA headers.
// free HBM on the current device (callers size their number of blocks in flight with it: libbsc_b200/cli/bsc_b200.cpp)
long long bscb200_device_free_bytes(void) { size_t f = 0, t = 0; if (cudaMemGetInfo(&f, &t) != cudaSuccess) { cudaGetLastError(); return -1; } return (long long)f; }
// Frees everything the library caches on every device: pooled contexts (bsc_* host-pointer entry points) and the sort slabs.  Only when no
// call is in flight.  Contexts made with bscb200_ctx_create belong to their owner.
void bscb200_release_pools(void)
{
    int cur = 0; cudaGetDevice(&cur);
    for (int d = 0; d < MAX_DEVICES; ++d) {
        std::vector<Ctx *> ctxs; std::vector<Scratch *> slabs;
        { std::lock_guard<std::mutex> lk(g_pool_mutex); ctxs.swap(g_pool[d]); }
        { std::lock_guard<std::mutex> lk(g_scratch[d].m); slabs.swap(g_scratch[d].free_list); g_scratch[d].created -= (int)slabs.size(); g_scratch[d].cap = -1; }
        for (Ctx *c : ctxs) ctx_delete(c);
        if (!slabs.empty()) cudaSetDevice(d);
        for (Scratch *s : slabs) scratch_destroy(s);
    }
    cudaSetDevice(cur); cudaGetLastError();
}
int bscb200_device_count(void) { int n = 0; return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0; }
int bscb200_set_device(int device) { return cudaSetDevice(device) == cudaSuccess ? LIBBSC_NO_ERROR : LIBBSC_GPU_ERROR; }

// workspace of a context that only ever DEcompresses blocks of n bytes: the same as bscb200_workspace_bytes
long long bscb200_workspace_bytes_decode(int n) { return bscb200_workspace_bytes(n, 1); }
unsigned long long bscb200_ctx_kernel_launches(void *ctx) { return ((Ctx *)ctx)->kernels_launched; }

int bscb200_compress_device(void *ctx, const unsigned char *d_input, unsigned char *d_output, int n, int blockSorter, int coder, int features)
{
    Ctx *c = (Ctx *)ctx;
    return guarded(c, [&]() { c->arena.reset(); c->arena.reserve((size_t)bscb200_workspace_bytes(n, blockSorter)); return compress_dev(c, d_input, n, d_output, blockSorter, coder, features, false); });
}
int bscb200_decompress_device(void *ctx, const unsigned char *d_input, int inputSize, unsigned char *d_output, int outputSize, int features)
{
    Ctx *c = (Ctx *)ctx;
    return guarded(c, [&]() {
        if (inputSize < LIBBSC_HEADER_SIZE) return LIBBSC_UNEXPECTED_EOB;
        CUDA_TRY(cudaMemcpyAsync(c->h_mail + 64, d_input, LIBBSC_HEADER_SIZE, cudaMemcpyDeviceToHost, c->stream));
        c->sync();
        c->arena.reset(); c->arena.reserve((size_t)bscb200_workspace_bytes_decode(outputSize));   // no-op for a context that already compressed
        BlockHeader H;
        const int info = H.read((const unsigned char *)(c->h_mail + 64), inputSize);
        if (info != LIBBSC_NO_ERROR) return info;
        if (inputSize < H.block_size || outputSize < H.data_size) return LIBBSC_UNEXPECTED_EOB;
        return decompress_dev(c, H, d_input, d_output, nullptr, features);
    });
}
int bscb200_bwt_encode_device(void *ctx, unsigned char *d_T, int n, unsigned char *num_indexes, int *indexes)
{
    Ctx *c = (Ctx *)ctx;
    return guarded(c, [&]() { c->arena.reset(); return bwt_encode_leased(c, d_T, n, num_indexes, indexes); });
}
int bscb200_bwt_decode_device(void *ctx, unsigned char *d_T, int n, int index)
{
    Ctx *c = (Ctx *)ctx;
    if (d_T == nullptr || n < 0 || index <= 0 || index > n) return LIBBSC_BAD_PARAMETER;      // before any workspace is sized from n
    return guarded(c, [&]() { c->arena.reset(); c->arena.reserve(bwt_decode_bytes((u32)n)); int r = stage_bwt_decode(c, d_T, n, index); c->sync(); return r; });
}
int bscb200_st_encode_device(void *ctx, unsigned char *d_T, int n, int k)
{
    Ctx *c = (Ctx *)ctx;
    if (d_T == nullptr || n < 0 || !st_order_valid(k)) return LIBBSC_BAD_PARAMETER;
    return guarded(c, [&]() { c->arena.reset(); return st_encode_leased(c, d_T, n, k); });
}
int bscb200_st_decode_device(void *ctx, unsigned char *d_T, int n, int k, int index)
{
    Ctx *c = (Ctx *)ctx;
    if (d_T == nullptr || n < 0 || index < 0 || index >= n || !st_order_valid(k)) return LIBBSC_BAD_PARAMETER;     // st.cpp:1493-1495
    return guarded(c, [&]() { c->arena.reset(); ScratchLease lease(c, need_st_decode((size_t)n)); int r = stage_st_decode(c, d_T, n, k, index); c->sync(); return r; });
}
int bscb200_coder_compress_device(void *ctx, const unsigned char *d_in, unsigned char *d_out, int n, int coder, int features)
{
    Ctx *c = (Ctx *)ctx;
    if (!coder_valid(coder) || n <= 0) return LIBBSC_BAD_PARAMETER;
    return guarded(c, [&]() { c->arena.reset(); c->arena.reserve(need_coder((size_t)n)); return stage_coder_compress(c, d_in, d_out, n, coder, features); });
}
int bscb200_coder_decompress_device(void *ctx, const unsigned char *d_in, int inputSize, unsigned char *d_out, int outputCapacity, int coder, int features)
{
    Ctx *c = (Ctx *)ctx;
    if (!coder_valid(coder) || inputSize < 1 || outputCapacity < 0) return LIBBSC_BAD_PARAMETER;
    return guarded(c, [&]() { c->arena.reset(); c->arena.reserve(need_coder((size_t)outputCapacity)); return stage_coder_decompress(c, d_in, inputSize, d_out, outputCapacity, coder, features); });
}
unsigned int bscb200_adler32_device(void *ctx, const unsigned char *d_p, int n)
{
    Ctx *c = (Ctx *)ctx; unsigned int v = 0;
    guarded(c, [&]() { v = stage_adler32(c, d_p, n); return 0; });
    return v;
}

// Per-kernel timing: bracket every launch of this context with CUDA events on its stream.
void bscb200_ctx_set_profile(void *ctx, int on)
{
    Ctx *c = (Ctx *)ctx; c->profile = on != 0; c->prof.clear(); c->ev_used = 0;
}
// Writes one line per kernel name: "<name>\t<launches>\t<total_ms>\t<algorithmic_bytes>\n"; returns bytes written.
int bscb200_ctx_profile_report(void *ctx, char *buf, int cap)
{
    Ctx *c = (Ctx *)ctx;
    cudaStreamSynchronize(c->stream);
    struct Acc { const char *name; int n; double ms, bytes; };
    std::vector<Acc> acc;
    for (const ProfRec &r : c->prof) {
        float ms = 0; if (cudaEventElapsedTime(&ms, r.a, r.b) != cudaSuccess) { cudaGetLastError(); continue; }
        size_t i = 0; for (; i < acc.size(); ++i) if (strcmp(acc[i].name, r.name) == 0) break;
        if (i == acc.size()) acc.push_back(Acc{r.name, 0, 0, 0});
        acc[i].n++; acc[i].ms += ms; acc[i].bytes += r.bytes;
    }
    int w = 0;
    for (const Acc &a : acc) { int k = snprintf(buf + w, cap > w ? (size_t)(cap - w) : 0, "%.*s\t%d\t%.6f\t%.0f\n", (int)strcspn(a.name + (a.name[0] == '('), "<"), a.name + (a.name[0] == '('), a.n, a.ms, a.bytes);   /* template arguments are not part of the reported name */ if (k < 0 || w + k >= cap) break; w += k; }
    c->prof.clear(); c->ev_used = 0;
    return w;
}

// total kernel launches issued through pooled + destroyed contexts (bench.py's gpu_launches)
unsigned long long bscb200_total_kernel_launches(void)
{
    std::lock_guard<std::mutex> lk(g_pool_mutex);
    unsigned long long t = g_launches_retired;
    for (int d = 0; d < MAX_DEVICES; ++d) for (Ctx *c : g_pool[d]) t += c->kernels_launched;
    return t;
}
const char *bscb200_version(void) { return "libbsc_b200 0.1 (libbsc 3.3.5 block format)"; }

}  // extern "C"
