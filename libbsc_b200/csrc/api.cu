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
bool g_initialised = false;
int g_features = 0;
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

void ctx_delete(Ctx *c)
{
    if (!c) return;
    cudaSetDevice(c->device);
    c->arena.destroy();
    if (c->h_mail) cudaFreeHost(c->h_mail);
    if (c->d_mail) cudaFree(c->d_mail);
    if (c->h_stage) cudaFreeHost(c->h_stage);
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
                if (s) { if (s->idle) cudaEventDestroy(s->idle); s->arena.destroy(); delete s; }
                P.created--; P.cap = P.created;
                P.cv.notify_all();
                continue;
            }
            if (s && !fresh) { P.free_list.push_back(s); } else { if (s) { if (s->idle) cudaEventDestroy(s->idle); s->arena.destroy(); delete s; } P.created--; }
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

int map_failure(const CudaFail &f)
{
    cudaGetLastError();
    return f.err == cudaErrorMemoryAllocation ? LIBBSC_GPU_NOT_ENOUGH_MEMORY : LIBBSC_GPU_ERROR;
}

// run `body(ctx)` on a pooled context, translating CUDA failures into libbsc error codes.  Nothing may unwind through the
// extern "C" boundary, and a context that failed mid-stage is destroyed instead of pooled (its device mailbox may hold partial
// Adler-32 sums that the next block would inherit).
template <class F> int with_ctx(F body)
{
    Ctx *c = ctx_acquire();
    if (!c) return LIBBSC_GPU_NOT_SUPPORTED;
    int r; bool broken = true;
    try { r = body(c); broken = false; }
    catch (const CudaFail &f) { r = map_failure(f); }
    catch (const std::bad_alloc &) { r = LIBBSC_NOT_ENOUGH_MEMORY; }
    catch (...) { r = LIBBSC_GPU_ERROR; }
    if (broken) {
        cudaStreamSynchronize(c->stream); cudaGetLastError();
        { std::lock_guard<std::mutex> lk(g_pool_mutex); g_launches_retired += c->kernels_launched; }
        ctx_delete(c);
    } else ctx_release(c);
    return r;
}
template <class F> int guarded(Ctx *c, F body)
{
    int r;
    try { return body(); }
    catch (const CudaFail &f) { r = map_failure(f); }
    catch (const std::bad_alloc &) { r = LIBBSC_NOT_ENOUGH_MEMORY; }
    catch (...) { r = LIBBSC_GPU_ERROR; }
    cudaStreamSynchronize(c->stream); cudaGetLastError(); c->arena.reset();
    cudaMemsetAsync(c->d_mail, 0, 1024, c->stream); cudaStreamSynchronize(c->stream); cudaGetLastError();   // adler32.cu expects zeroed accumulators
    return r;
}

// arena sizes (bytes) generous enough for each stage at block length n
size_t need_bwt_encode(size_t n) { return 58 * n + (64u << 20); }
size_t need_bwt_decode(size_t n) { return 10 * n + (16u << 20); }   // L n, LF 4n, look-back n/2, nodes + 128-byte slabs 3.3 n
size_t need_st_encode(size_t n)  { return 30 * n + (16u << 20); }
size_t need_st_decode(size_t n)  { return 41 * n + (16u << 20); }
size_t need_coder(size_t n)      { return 12 * n + (64u << 20); }

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

bool sorter_valid(int s) { return s == 1 || (s >= 3 && s <= 8); }

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

// ---------------------------------------------------------------------------------------------
// device-resident block compress / decompress
// ---------------------------------------------------------------------------------------------
// Stored block (libbsc.cpp:68-81) built on the device: header on host, data D2D.
int store_dev(Ctx *ctx, const u8 *d_in, int n, u8 *d_out, u32 adler_data)
{
    unsigned char h[LIBBSC_HEADER_SIZE];
    put32(h, (u32)(n + LIBBSC_HEADER_SIZE)); put32(h + 4, (u32)n); put32(h + 8, 0); put32(h + 12, 0);
    put32(h + 16, adler_data); put32(h + 20, adler_data); put32(h + 24, host_adler32(h, 24));
    if (n > 0) CUDA_TRY(cudaMemcpyAsync(d_out + LIBBSC_HEADER_SIZE, d_in, (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
    memcpy(ctx->h_mail + 64, h, LIBBSC_HEADER_SIZE);
    CUDA_TRY(cudaMemcpyAsync(d_out, ctx->h_mail + 64, LIBBSC_HEADER_SIZE, cudaMemcpyHostToDevice, ctx->stream));
    ctx->sync();
    return n + LIBBSC_HEADER_SIZE;
}

// bsc_compress with LZP disabled, everything in HBM.  d_out must hold n + 28 bytes.
// `lz` (host-pointer bsc_compress with LZP parameters only): d_in holds the LZP stream of a block of lz->orig_n bytes whose Adler-32
// is lz->adler_orig; the header describes the original block, and a block that does not shrink is reported as LIBBSC_NOT_COMPRESSIBLE
// (the caller stores the ORIGINAL data, libbsc.cpp:315-318).
struct LzpInfo { int orig_n; u32 adler_orig; int mode_bits; };
int finish_dev(Ctx *ctx, u8 *d_out, int result, unsigned char num_indexes, const int *indexes, int orig_n, int mode, int index, u32 adler_data);

int compress_dev(Ctx *ctx, const u8 *d_in, int n, u8 *d_out, int blockSorter, int coder, int features, bool inplace_rules, const LzpInfo *lz = nullptr)
{
    if (!sorter_valid(blockSorter)) return LIBBSC_BAD_PARAMETER;
    if (coder < 1 || coder > 3) return LIBBSC_BAD_PARAMETER;
    if (n < 0 || n > 1073741824) return LIBBSC_BAD_PARAMETER;
    if (lz && n <= LIBBSC_HEADER_SIZE) blockSorter = 1;                  // libbsc.cpp:278-282: a tiny LZP stream is always BWT-sorted
    int mode = blockSorter | (coder << 5) | (lz ? lz->mode_bits : 0);
    const u32 adler_data = lz ? lz->adler_orig : stage_adler32(ctx, d_in, n);
    if (!lz && n <= LIBBSC_HEADER_SIZE) return store_dev(ctx, d_in, n, d_out, adler_data);
    const int orig_n = lz ? lz->orig_n : n;

    Arena &A = ctx->arena;
    const size_t mark = A.mark();
    u8 *work = A.get<u8>((size_t)n + 64);
    CUDA_TRY(cudaMemcpyAsync(work, d_in, (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));

    int indexes[256]; unsigned char num_indexes = 0; int index;
    if (blockSorter == 1) index = bwt_encode_leased(ctx, work, n, &num_indexes, indexes);      // the sort's ~58 n live in a shared slab
    else { ScratchLease lease(ctx, need_st_encode(n)); index = stage_st_encode(ctx, work, n, blockSorter); }
    if (orig_n < 64 * 1024) num_indexes = 0;              // libbsc.cpp:303
    if (index < 0) { A.release(mark); return index; }

    int result = stage_coder_compress(ctx, work, d_out + LIBBSC_HEADER_SIZE, n, coder, features);
    A.release(mark);
    if (result == LIBBSC_NOT_SUPPORTED) return result;
    if (result < 0 || result + 1 + 4 * num_indexes >= orig_n) {
        if (inplace_rules || lz) return LIBBSC_NOT_COMPRESSIBLE;         // libbsc.cpp:188-191
        return store_dev(ctx, d_in, n, d_out, adler_data);               // libbsc.cpp:315-318
    }
    return finish_dev(ctx, d_out, result, num_indexes, indexes, orig_n, mode, index, adler_data);
}

// The secondary indexes and the header of a compressed block whose coder output (`result` bytes) is at d_out + 28.
int finish_dev(Ctx *ctx, u8 *d_out, int result, unsigned char num_indexes, const int *indexes, int orig_n, int mode, int index, u32 adler_data)
{
    unsigned char *tail = (unsigned char *)(ctx->h_mail + 96);            // pinned, <= 4*255+1 bytes needs care: num_indexes <= 15 here
    memcpy(tail, indexes, 4 * (size_t)num_indexes);
    tail[4 * num_indexes] = num_indexes;
    CUDA_TRY(cudaMemcpyAsync(d_out + LIBBSC_HEADER_SIZE + result, tail, 4 * (size_t)num_indexes + 1, cudaMemcpyHostToDevice, ctx->stream));
    result += 1 + 4 * num_indexes;
    const u32 adler_payload = stage_adler32(ctx, d_out + LIBBSC_HEADER_SIZE, result);
    unsigned char *h = (unsigned char *)(ctx->h_mail + 64);
    put32(h, (u32)(result + LIBBSC_HEADER_SIZE)); put32(h + 4, (u32)orig_n); put32(h + 8, (u32)mode); put32(h + 12, (u32)index);
    put32(h + 16, adler_data); put32(h + 20, adler_payload); put32(h + 24, host_adler32(h, 24));
    CUDA_TRY(cudaMemcpyAsync(d_out, h, LIBBSC_HEADER_SIZE, cudaMemcpyHostToDevice, ctx->stream));
    ctx->sync();
    return result + LIBBSC_HEADER_SIZE;
}

int block_info_host(const unsigned char *h, int headerSize, int *pBlockSize, int *pDataSize)
{
    if (headerSize < LIBBSC_HEADER_SIZE) return LIBBSC_UNEXPECTED_EOB;
    if (get32(h + 24) != host_adler32(h, 24)) return LIBBSC_DATA_CORRUPT;
    int blockSize = (int)get32(h), dataSize = (int)get32(h + 4), mode = (int)get32(h + 8), index = (int)get32(h + 12);
    int lzpHash = (mode >> 16) & 0xff, lzpMin = (mode >> 8) & 0xff, coder = (mode >> 5) & 7, sorter = mode & 0x1f;
    int rebuilt = 0;
    if (sorter_valid(sorter)) rebuilt = sorter; else if (sorter > 0) return LIBBSC_DATA_CORRUPT;
    if (coder >= 1 && coder <= 3) rebuilt += coder << 5; else if (coder > 0) return LIBBSC_DATA_CORRUPT;
    if (lzpMin != 0 || lzpHash != 0) {
        if (lzpMin < 4 || lzpMin > 255) return LIBBSC_DATA_CORRUPT;
        if (lzpHash < 10 || lzpHash > 28) return LIBBSC_DATA_CORRUPT;
        rebuilt += (lzpMin << 8) + (lzpHash << 16);
    }
    if (rebuilt != mode) return LIBBSC_DATA_CORRUPT;
    if (blockSize < LIBBSC_HEADER_SIZE || blockSize > LIBBSC_HEADER_SIZE + dataSize) return LIBBSC_DATA_CORRUPT;
    if (index < 0 || index > dataSize) return LIBBSC_DATA_CORRUPT;
    if (pBlockSize) *pBlockSize = blockSize;
    if (pDataSize) *pDataSize = dataSize;
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

// bsc_decompress body once the 28-byte header `h` is on the host and the block is in HBM.
// `lz_out` (host-pointer entry point only): blocks with an LZP stage (mode bits 8..23) are decoded up to the LZP stream, whose
// length goes to *lz_out; the caller undoes LZP on the host (lzp_host.h) and checks length and Adler-32 of the data there.
int decompress_dev(Ctx *ctx, const unsigned char *h, const u8 *d_block, int inputSize, u8 *d_out, int outputSize, int features, int *lz_out = nullptr)
{
    int blockSize = 0, dataSize = 0;
    int info = block_info_host(h, inputSize, &blockSize, &dataSize);
    if (info != LIBBSC_NO_ERROR) return info;
    if (inputSize < blockSize || outputSize < dataSize) return LIBBSC_UNEXPECTED_EOB;
    const int payload = blockSize - LIBBSC_HEADER_SIZE;
    if (get32(h + 20) != stage_adler32(ctx, d_block + LIBBSC_HEADER_SIZE, payload)) return LIBBSC_DATA_CORRUPT;
    const int mode = (int)get32(h + 8);
    if (mode == 0) {
        // A stored block carries exactly dataSize payload bytes (bsc_store, libbsc.cpp:68-81).  The reference copies dataSize bytes
        // whatever blockSize says (libbsc.cpp:550-555), reading past a shorter block; here such a header is corrupt.  Like the reference,
        // the data Adler-32 of a stored block is not checked: the payload Adler-32 above covers the same bytes.
        if (payload != dataSize) return LIBBSC_DATA_CORRUPT;
        if (dataSize > 0) CUDA_TRY(cudaMemcpyAsync(d_out, d_block + LIBBSC_HEADER_SIZE, (size_t)dataSize, cudaMemcpyDeviceToDevice, ctx->stream));
        ctx->sync();
        return LIBBSC_NO_ERROR;
    }
    const bool lzp = mode != (mode & 0xff);
    if (lzp && !lz_out) return LIBBSC_NOT_SUPPORTED;                     // device-resident API: LZP stays on the host side of the boundary
    const int index = (int)get32(h + 12); const u32 adler_data = get32(h + 16);
    const int coder = (mode >> 5) & 7, sorter = mode & 0x1f;
    if (payload < 1) return LIBBSC_DATA_CORRUPT;

    int lzSize = stage_coder_decompress(ctx, d_block + LIBBSC_HEADER_SIZE, payload, d_out, dataSize, coder, features);
    if (lzSize < 0) return lzSize;
    if (!sorter_valid(sorter)) return LIBBSC_DATA_CORRUPT;               // sorter field 0 with a coder: libbsc.cpp:593, after the coder stage
    if (sorter == 1 && secondary_indexes_out_of_range(ctx, d_block + LIBBSC_HEADER_SIZE, payload, lzSize, index)) return LIBBSC_BAD_PARAMETER;
    int r;
    if (sorter == 1) r = stage_bwt_decode(ctx, d_out, lzSize, index);
    else { ScratchLease lease(ctx, need_st_decode((size_t)lzSize)); r = stage_st_decode(ctx, d_out, lzSize, sorter, index); }   // libbsc.cpp:584-589
    if (r < 0) return r;
    if (lzp) { *lz_out = lzSize; return LIBBSC_NO_ERROR; }
    if (lzSize != dataSize) return LIBBSC_DATA_CORRUPT;
    return adler_data == stage_adler32(ctx, d_out, dataSize) ? LIBBSC_NO_ERROR : LIBBSC_DATA_CORRUPT;
}

// ---------------------------------------------------------------------------------------------
// blocks above 1 GiB: in-place bsc_compress, and bsc_decompress of such blocks
// ---------------------------------------------------------------------------------------------
// On the pooled path a block of n bytes holds about 31 n of HBM: the staged block, its working copy, the output and the coder stage in
// the context, and a 16.5 n sort slab that the pool keeps after the call.  A block above 1 GiB instead runs on a context made for the
// call and destroyed after it, in ONE allocation: the block, sorted in place (an in-place call may destroy its input, libbsc.cpp:160),
// and a region that first holds the batched forward BWT (16 n + 32 B) and then the coder stage with its output (about 13 n + 64 MB).
// The caller's buffer is written only once the block is done.  Only the BWT has a bounded forward sorter: the forward ST needs about
// 30 n (need_st_encode), so ST3..ST8 compress only up to 1 GiB.  Their inverse has a lean layout (decompress_large_st below).
// The arena is 17.5 n + 128 MiB: the batched sort at batches of about n / 64 entries (16.5 n) or the coder stage with its output
// (at most 13 n + 64 MB) after the block.  The bound adds n / 2 + 128 MiB for what lies outside the arena: the context, the coder
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

// run `body(ctx)` on a context of its own, destroyed afterwards so that none of its HBM outlives the call
template <class F> int with_own_ctx(F body)
{
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return LIBBSC_GPU_NOT_SUPPORTED; }
    Ctx *c = nullptr;
    try { c = ctx_new(dev, nullptr, true); }
    catch (const CudaFail &f) { return map_failure(f); }
    catch (...) { cudaGetLastError(); return LIBBSC_GPU_ERROR; }
    int r;
    try { r = body(c); }
    catch (const CudaFail &f) { r = map_failure(f); }
    catch (const std::bad_alloc &) { r = LIBBSC_NOT_ENOUGH_MEMORY; }
    catch (...) { r = LIBBSC_GPU_ERROR; }
    cudaStreamSynchronize(c->stream); cudaGetLastError();
    { std::lock_guard<std::mutex> lk(g_pool_mutex); g_launches_retired += c->kernels_launched; }
    ctx_delete(c);
    return r;
}

// In-place bsc_compress of a block of n > 1 GiB bytes with the BWT sorter (libbsc.cpp:124-210).
int compress_large(unsigned char *data, int n, int lzpHashSize, int lzpMinLen, int coder, int features)
{
    size_t fr = 0, total = 0;
    if (cudaMemGetInfo(&fr, &total) != cudaSuccess) { cudaGetLastError(); return LIBBSC_GPU_NOT_SUPPORTED; }
    if (fr < large_bound((size_t)n)) return LIBBSC_GPU_NOT_ENOUGH_MEMORY;

    int m = n, mode_bits = 0; u32 adler_orig = 0;          // m: bytes that go through the sort and the coder
    unsigned char *lzbuf = nullptr;
    if (lzpMinLen != 0) {                                   // libbsc.cpp:139-154: LZP on the host, not in place
        lzbuf = (unsigned char *)bsc_malloc((size_t)n + 64);
        if (!lzbuf) return LIBBSC_NOT_ENOUGH_MEMORY;
        const int lzSize = lzp_host::compress(data, lzbuf, n, lzpHashSize, lzpMinLen, (features & LIBBSC_FEATURE_MULTITHREADING) != 0);
        if (lzSize >= 0) { m = lzSize; mode_bits = (lzpMinLen << 8) | (lzpHashSize << 16); adler_orig = host_adler32(data, (size_t)n); }
        else { bsc_free(lzbuf); lzbuf = nullptr; }         // LZP did not shrink the block: continue without it (mode &= 0xff)
    }
    const unsigned char *src = lzbuf ? lzbuf : data;
    const int r = with_own_ctx([&](Ctx *ctx) {
        Arena &A = ctx->arena;
        A.reserve(large_arena((size_t)n));
        u8 *d_blk = A.get<u8>((size_t)m + 64);
        CUDA_TRY(cudaMemcpyAsync(d_blk, src, (size_t)m, cudaMemcpyHostToDevice, ctx->stream));
        const u32 adler_data = lzbuf ? adler_orig : stage_adler32(ctx, d_blk, m);
        // the sort may use the whole region after the block (less a margin for the arena's rounding): batches of about n / 64 entries
        const u32 B = bwt_batch_entries((u32)m, (long long)(A.cap - A.used) - (16ll << 20));
        int indexes[256]; unsigned char num_indexes = 0;
        const int index = stage_bwt_encode_batched(ctx, d_blk, m, &num_indexes, indexes, B);
        if (index < 0) return index;
        u8 *d_out = A.get<u8>((size_t)m + 4096) + 4;       // payload (offset 28) lands 16-byte aligned
        const int result = stage_coder_compress(ctx, d_blk, d_out + LIBBSC_HEADER_SIZE, m, coder, features);
        if (result == LIBBSC_NOT_SUPPORTED) return result;
        if (result < 0 || result + 1 + 4 * num_indexes >= n) return LIBBSC_NOT_COMPRESSIBLE;     // libbsc.cpp:188-191
        const int size = finish_dev(ctx, d_out, result, num_indexes, indexes, n, 1 | (coder << 5) | mode_bits, index, adler_data);
        CUDA_TRY(cudaMemcpyAsync(data, d_out, (size_t)size, cudaMemcpyDeviceToHost, ctx->stream));
        ctx->sync();
        return size;
    });
    if (lzbuf) bsc_free(lzbuf);
    return r;
}

// libbsc.cpp:599-613: undo the LZP stage of a block (header h) on the host, from the lzSize-byte LZP stream at d_lz
int undo_lzp_host(Ctx *ctx, const unsigned char *h, const u8 *d_lz, int lzSize, unsigned char *output, int dataSize)
{
    const int mode = (int)get32(h + 8);
    // the LZP stream, then the data after it: the caller's buffer is written only once the data is known to be right
    unsigned char *lz = (unsigned char *)bsc_malloc((size_t)lzSize + (size_t)dataSize + 1);
    if (!lz) return LIBBSC_NOT_ENOUGH_MEMORY;
    unsigned char *data = lz + lzSize;
    if (lzSize > 0) { CUDA_TRY(cudaMemcpyAsync(lz, d_lz, (size_t)lzSize, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
    int r = lzp_host::decompress(lz, lzSize, data, dataSize, (mode >> 16) & 0xff, (mode >> 8) & 0xff);
    if (r >= 0) r = (r == dataSize && get32(h + 16) == host_adler32(data, (size_t)dataSize)) ? LIBBSC_NO_ERROR : LIBBSC_DATA_CORRUPT;
    if (r == LIBBSC_NO_ERROR && dataSize > 0) memcpy(output, data, (size_t)dataSize);
    bsc_free(lz);
    return r;
}

// bsc_decompress of a block with block sorter 3..8 whose data size is above 1 GiB (large_st_arena above).  The caller checked the header
// (block_info_host) and the sizes.  The caller's buffer is written only on success.
int decompress_large_st(const unsigned char *input, const unsigned char *h, int blockSize, int dataSize, unsigned char *output, int features)
{
    size_t fr = 0, total = 0;
    if (cudaMemGetInfo(&fr, &total) != cudaSuccess) { cudaGetLastError(); return LIBBSC_GPU_NOT_SUPPORTED; }
    if (fr < large_st_bound((size_t)dataSize)) return LIBBSC_GPU_NOT_ENOUGH_MEMORY;
    return with_own_ctx([&](Ctx *ctx) {
        Arena &A = ctx->arena;
        A.reserve(large_st_arena((size_t)dataSize));
        u8 *d_L = A.get<u8>((size_t)dataSize + 128);
        const size_t full = A.cap, blk = align_up((size_t)blockSize + 128, 256);
        u8 *d_blk = A.base + full - blk + 4;                 // the top end of the region; payload (offset 28) lands 16-byte aligned
        CUDA_TRY(cudaMemcpyAsync(d_blk, input, (size_t)blockSize, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(cudaMemsetAsync(d_blk + blockSize, 0, 64, ctx->stream));
        const int payload = blockSize - LIBBSC_HEADER_SIZE, mode = (int)get32(h + 8), index = (int)get32(h + 12);
        if (payload < 1) return LIBBSC_DATA_CORRUPT;
        if (get32(h + 20) != stage_adler32(ctx, d_blk + LIBBSC_HEADER_SIZE, payload)) return LIBBSC_DATA_CORRUPT;
        A.cap = full - blk;                                  // the coder stage stays below the block
        const int lzSize = stage_coder_decompress(ctx, d_blk + LIBBSC_HEADER_SIZE, payload, d_L, dataSize, (mode >> 5) & 7, features);
        A.cap = full;
        if (lzSize < 0) return lzSize;
        u8 *d_T = nullptr;                                   // the block is dead: the inverse ST takes the whole region after L
        const int r = stage_st_decode_lean(ctx, d_L, lzSize, mode & 0x1f, index, &d_T);
        if (r < 0) return r;
        if (mode != (mode & 0xff)) return undo_lzp_host(ctx, h, d_T, lzSize, output, dataSize);
        if (lzSize != dataSize || get32(h + 16) != stage_adler32(ctx, d_T, dataSize)) return LIBBSC_DATA_CORRUPT;
        CUDA_TRY(cudaMemcpyAsync(output, d_T, (size_t)dataSize, cudaMemcpyDeviceToHost, ctx->stream));
        ctx->sync();
        return LIBBSC_NO_ERROR;
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
    g_features = features; g_initialised = true;
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
    put32(output, (u32)(n + LIBBSC_HEADER_SIZE)); put32(output + 4, (u32)n); put32(output + 8, 0); put32(output + 12, 0);
    put32(output + 16, a); put32(output + 20, a); put32(output + 24, host_adler32(output, 24));
    return n + LIBBSC_HEADER_SIZE;
}

int bsc_block_info(const unsigned char *blockHeader, int headerSize, int *pBlockSize, int *pDataSize, int features)
{
    (void)features;
    return block_info_host(blockHeader, headerSize, pBlockSize, pDataSize);
}

int bsc_compress(const unsigned char *input, unsigned char *output, int n, int lzpHashSize, int lzpMinLen, int blockSorter, int coder, int features)
{
    if (!sorter_valid(blockSorter)) return LIBBSC_BAD_PARAMETER;
    if (coder < 1 || coder > 3) return LIBBSC_BAD_PARAMETER;
    if (lzpMinLen != 0 || lzpHashSize != 0) {
        if (lzpMinLen < 4 || lzpMinLen > 255) return LIBBSC_BAD_PARAMETER;
        if (lzpHashSize < 10 || lzpHashSize > 28) return LIBBSC_BAD_PARAMETER;
        // The LZP stage runs on the host (lzp_host.h: all five x86-64 variants of the reference; north star: libbsc/lzp stays on the host).
        if (!lzp_host::supported(lzpHashSize, lzpMinLen)) return LIBBSC_NOT_SUPPORTED;
    }
    const bool inplace = (input == output);
    if (n < 0 || n > (inplace ? 2146435072 : 1073741824)) return LIBBSC_BAD_PARAMETER;
    if (n <= LIBBSC_HEADER_SIZE) return bsc_store(input, output, n, features);
    // In place only: compress_large works on its argument in place.  Out of place, blocks above 1 GiB were refused above, and below it a
    // lowered routing threshold (tests) keeps them on the pooled path.
    if (inplace && n > large_route_n()) return blockSorter == 1 ? compress_large(output, n, lzpHashSize, lzpMinLen, coder, features) : LIBBSC_NOT_SUPPORTED;
    if (lzpMinLen != 0) {                                   // libbsc.cpp:264-276
        unsigned char *lzbuf = (unsigned char *)bsc_malloc((size_t)n + 64);
        if (!lzbuf) return LIBBSC_NOT_ENOUGH_MEMORY;
        const int lzSize = lzp_host::compress(input, lzbuf, n, lzpHashSize, lzpMinLen, (features & LIBBSC_FEATURE_MULTITHREADING) != 0);
        if (lzSize >= 0) {
            const LzpInfo lz = {n, host_adler32(input, (size_t)n), (lzpMinLen << 8) | (lzpHashSize << 16)};
            int r = with_ctx([&](Ctx *ctx) {
                ctx->arena.reserve(3 * (size_t)n + 16384 + need_coder(n));
                u8 *d_in = ctx->arena.get<u8>((size_t)lzSize + 64);
                u8 *d_out = ctx->arena.get<u8>((size_t)n + 4096) + 4;
                if (lzSize > 0) CUDA_TRY(cudaMemcpyAsync(d_in, lzbuf, (size_t)lzSize, cudaMemcpyHostToDevice, ctx->stream));
                int rr = compress_dev(ctx, d_in, lzSize, d_out, blockSorter, coder, features, inplace, &lz);
                if (rr > 0) { CUDA_TRY(cudaMemcpyAsync(output, d_out, (size_t)rr, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
                return rr;
            });
            bsc_free(lzbuf);
            if (r == LIBBSC_NOT_COMPRESSIBLE && !inplace) return bsc_store(input, output, n, features);
            return r;
        }
        bsc_free(lzbuf);                                    // LZP did not shrink the block: continue without it (mode &= 0xff)
    }
    return with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve(3 * (size_t)n + 16384 + need_coder(n));
        u8 *d_in = ctx->arena.get<u8>((size_t)n + 64);
        u8 *d_out = ctx->arena.get<u8>((size_t)n + 4096) + 4;      // payload (offset 28) lands 16-byte aligned
        CUDA_TRY(cudaMemcpyAsync(d_in, input, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        int r = compress_dev(ctx, d_in, n, d_out, blockSorter, coder, features, inplace);
        if (r > 0) { CUDA_TRY(cudaMemcpyAsync(output, d_out, (size_t)r, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
}

int bsc_decompress(const unsigned char *input, int inputSize, unsigned char *output, int outputSize, int features)
{
    int blockSize = 0, dataSize = 0;
    int info = block_info_host(input, inputSize, &blockSize, &dataSize);
    if (info != LIBBSC_NO_ERROR) return info;
    if (inputSize < blockSize || outputSize < dataSize) return LIBBSC_UNEXPECTED_EOB;
    unsigned char h[LIBBSC_HEADER_SIZE]; memcpy(h, input, LIBBSC_HEADER_SIZE);
    const bool large = dataSize > large_route_n();
    if (large && (get32(h + 8) & 0x1f) >= 3) return decompress_large_st(input, h, blockSize, dataSize, output, features);
    // Above 1 GiB (BWT and stored blocks): about 14 n + 64 MB (large_bound holds it), on a context of its own that does not keep it after the call.
    auto body = [&](Ctx *ctx) {
        ctx->arena.reserve((size_t)blockSize + (size_t)dataSize + 8192 + need_coder((size_t)dataSize));      // coder stage, then the inverse BWT in the same space
        u8 *d_blk = ctx->arena.get<u8>((size_t)blockSize + 128) + 4;
        u8 *d_out = ctx->arena.get<u8>((size_t)dataSize + 128);
        CUDA_TRY(cudaMemcpyAsync(d_blk, input, (size_t)blockSize, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(cudaMemsetAsync(d_blk + blockSize, 0, 64, ctx->stream));
        int lzSize = -1;
        int r = decompress_dev(ctx, h, d_blk, blockSize, d_out, dataSize, features, &lzSize);
        if (r == LIBBSC_NO_ERROR && lzSize >= 0) return undo_lzp_host(ctx, h, d_out, lzSize, output, dataSize);
        if (r == LIBBSC_NO_ERROR && dataSize > 0) { CUDA_TRY(cudaMemcpyAsync(output, d_out, (size_t)dataSize, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    };
    return large ? with_own_ctx(body) : with_ctx(body);
}

int bsc_bwt_encode(unsigned char *T, int n, unsigned char *num_indexes, int *indexes, int features)
{
    (void)features;
    if (T == nullptr || n < 0) return LIBBSC_BAD_PARAMETER;
    return with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve((size_t)n + 4096);
        u8 *d = ctx->arena.get<u8>((size_t)n + 64);
        if (n > 0) CUDA_TRY(cudaMemcpyAsync(d, T, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        int r = bwt_encode_leased(ctx, d, n, num_indexes, indexes);
        if (r >= 0 && n > 0) { CUDA_TRY(cudaMemcpyAsync(T, d, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
}

int bsc_bwt_decode(unsigned char *T, int n, int index, unsigned char num_indexes, int *indexes, int features)
{
    (void)num_indexes; (void)indexes; (void)features;    // secondary indexes are CPU accelerators only (bwt.cpp:263 ignores them on the GPU too)
    if (T == nullptr || n < 0 || index <= 0 || index > n) return LIBBSC_BAD_PARAMETER;
    if (n <= 1) return LIBBSC_NO_ERROR;
    return with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve((size_t)n + 4096 + need_bwt_decode(n));
        u8 *d = ctx->arena.get<u8>((size_t)n + 64);
        CUDA_TRY(cudaMemcpyAsync(d, T, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        int r = stage_bwt_decode(ctx, d, n, index);
        if (r == 0) { CUDA_TRY(cudaMemcpyAsync(T, d, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
}

int bsc_st_encode(unsigned char *T, int n, int k, int features)
{
    (void)features;
    if (T == nullptr || n < 0) return LIBBSC_BAD_PARAMETER;
    if (k < 3 || k > 8) return LIBBSC_BAD_PARAMETER;
    if (n <= 1) return 0;
    return with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve((size_t)n + 4096);
        u8 *d = ctx->arena.get<u8>((size_t)n + 64);
        CUDA_TRY(cudaMemcpyAsync(d, T, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        ScratchLease lease(ctx, need_st_encode(n));
        int r = stage_st_encode(ctx, d, n, k);
        if (r >= 0) { CUDA_TRY(cudaMemcpyAsync(T, d, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
}

int bsc_st_decode(unsigned char *T, int n, int k, int index, int features)
{
    (void)features;
    if (T == nullptr || n < 0) return LIBBSC_BAD_PARAMETER;       // st.cpp:1493-1496
    if (index < 0 || index >= n) return LIBBSC_BAD_PARAMETER;
    if (k < 3 || k > 8) return LIBBSC_BAD_PARAMETER;
    if (n <= 1) return LIBBSC_NO_ERROR;
    return with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve((size_t)n + 4096);
        u8 *d = ctx->arena.get<u8>((size_t)n + 64);
        CUDA_TRY(cudaMemcpyAsync(d, T, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        ScratchLease lease(ctx, need_st_decode(n));
        int r = stage_st_decode(ctx, d, n, k, index);
        if (r == 0) { CUDA_TRY(cudaMemcpyAsync(T, d, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
}

int bsc_coder_compress(const unsigned char *input, unsigned char *output, int n, int coder, int features)
{
    if (coder < 1 || coder > 3) return LIBBSC_BAD_PARAMETER;
    if (n <= 0) return LIBBSC_BAD_PARAMETER;
    return with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve(2 * (size_t)n + 16384 + need_coder(n));
        u8 *d_in = ctx->arena.get<u8>((size_t)n + 64);
        u8 *d_out = ctx->arena.get<u8>((size_t)n + 4096);
        CUDA_TRY(cudaMemcpyAsync(d_in, input, (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
        int r = stage_coder_compress(ctx, d_in, d_out, n, coder, features);
        if (r > 0) { CUDA_TRY(cudaMemcpyAsync(output, d_out, (size_t)r, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
}

// Size-aware variant used by bsc_decompress and exported for integrators.
int bscb200_coder_decompress(const unsigned char *input, int inputSize, unsigned char *output, int outputCapacity, int coder, int features)
{
    if (coder < 1 || coder > 3) return LIBBSC_BAD_PARAMETER;
    if (inputSize < 1 || outputCapacity < 0) return LIBBSC_BAD_PARAMETER;
    return with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve((size_t)inputSize + (size_t)outputCapacity + 16384 + need_coder((size_t)outputCapacity));
        u8 *d_in = ctx->arena.get<u8>((size_t)inputSize + 128);
        u8 *d_out = ctx->arena.get<u8>((size_t)outputCapacity + 128);
        CUDA_TRY(cudaMemcpyAsync(d_in, input, (size_t)inputSize, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(cudaMemsetAsync(d_in + inputSize, 0, 64, ctx->stream));
        int r = stage_coder_decompress(ctx, d_in, inputSize, d_out, outputCapacity, coder, features);
        if (r > 0) { CUDA_TRY(cudaMemcpyAsync(output, d_out, (size_t)r, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
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
    if (coder < 1 || coder > 3) return LIBBSC_BAD_PARAMETER;
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
    return with_ctx([&](Ctx *ctx) {
        const size_t room = (size_t)(outputSize > inputSize ? outputSize : inputSize);
        ctx->arena.reserve(2 * room + (size_t)inputSize + 16384 + need_coder(room));
        u8 *d_in = ctx->arena.get<u8>((size_t)inputSize + 64);
        u8 *d_out = ctx->arena.get<u8>(room + 4096);
        CUDA_TRY(cudaMemcpyAsync(d_in, input, (size_t)inputSize, cudaMemcpyHostToDevice, ctx->stream));
        int r = stage_coder_compress(ctx, d_in, d_out, inputSize, coder, 0, outputSize);
        if (r > 0) { CUDA_TRY(cudaMemcpyAsync(output, d_out, (size_t)r, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
}
// Size-less like the reference's: n comes from the stream; the stream is taken to be at most n + 16 bytes long (what
// bsc_qlfc_*_encode_block produces with outputSize <= inputSize; same caller contract as bsc_coder_decompress above).
static int qlfc_decode_block(int coder, const unsigned char *input, unsigned char *output)
{
    const long long n = qlfc_stream_size(input);
    if (n < 0) return LIBBSC_DATA_CORRUPT;
    const int inSize = (int)readable_prefix(input, (size_t)n + 16);
    if (inSize < 14) return LIBBSC_UNEXPECTED_EOB;
    return with_ctx([&](Ctx *ctx) {
        ctx->arena.reserve((size_t)inSize + (size_t)n + 16384 + need_coder((size_t)n));
        u8 *d_in = ctx->arena.get<u8>((size_t)inSize + 128);
        u8 *d_out = ctx->arena.get<u8>((size_t)n + 128);
        CUDA_TRY(cudaMemcpyAsync(d_in, input, (size_t)inSize, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(cudaMemsetAsync(d_in + inSize, 0, 64, ctx->stream));
        int r = stage_coder_decompress(ctx, d_in, inSize, d_out, (int)n, coder, 0, true);
        if (r > 0) { CUDA_TRY(cudaMemcpyAsync(output, d_out, (size_t)r, cudaMemcpyDeviceToHost, ctx->stream)); ctx->sync(); }
        return r;
    });
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
void bscb200_ctx_destroy(void *ctx)
{
    Ctx *c = (Ctx *)ctx;
    if (c) { std::lock_guard<std::mutex> lk(g_pool_mutex); g_launches_retired += c->kernels_launched; }
    ctx_delete(c);
}
int bscb200_ctx_reserve(void *ctx, long long bytes)
{
    Ctx *c = (Ctx *)ctx;
    return guarded(c, [&]() { CUDA_TRY(cudaSetDevice(c->device)); c->arena.reset(); c->arena.reserve((size_t)bytes); return 0; });
}
// Bounds the forward BWT's working set on this context: it sorts in batches whenever the standard sorter would need more than `bytes`
// (0 = no bound).  Block sorters 3..8 ignore it.
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
    return (long long)(need_coder((size_t)n) + (size_t)n + 8192);
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
    if (n < 0 || n > 2146435072 || !sorter_valid(blockSorter) || coder < 1 || coder > 3) return LIBBSC_BAD_PARAMETER;
    if (blockSorter != 1) return LIBBSC_NOT_SUPPORTED;      // no bounded sort transform
    return (long long)large_bound((size_t)n);
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
    if (!input || !output || n < 0 || outputCapacity < 0 || lzpHashSize < 10 || lzpHashSize > 28 || lzpMinLen < 4 || lzpMinLen > 255) return LIBBSC_BAD_PARAMETER;
    return lzp_host::decompress(input, n, output, outputCapacity, lzpHashSize, lzpMinLen);
}

// host-only: the forward LZP stage by itself (bsc_lzp_compress, lzp.h); LIBBSC_NOT_SUPPORTED for the parameter classes whose
// reference variant is not restated (lzp_host.h)
int bscb200_lzp_compress_host(const unsigned char *input, unsigned char *output, int n, int lzpHashSize, int lzpMinLen, int features)
{
    if (!input || !output || n < 0 || lzpHashSize < 10 || lzpHashSize > 28 || lzpMinLen < 4 || lzpMinLen > 255) return LIBBSC_BAD_PARAMETER;
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
        { std::lock_guard<std::mutex> lk(g_pool_mutex); ctxs.swap(g_pool[d]); for (Ctx *c : ctxs) g_launches_retired += c->kernels_launched; }
        { std::lock_guard<std::mutex> lk(g_scratch[d].m); slabs.swap(g_scratch[d].free_list); g_scratch[d].created -= (int)slabs.size(); g_scratch[d].cap = -1; }
        for (Ctx *c : ctxs) ctx_delete(c);
        if (!slabs.empty()) cudaSetDevice(d);
        for (Scratch *s : slabs) { if (s->idle_valid) cudaEventSynchronize(s->idle); s->arena.destroy(); if (s->idle) cudaEventDestroy(s->idle); delete s; }
    }
    cudaSetDevice(cur); cudaGetLastError();
}
int bscb200_device_count(void) { int n = 0; return cudaGetDeviceCount(&n) == cudaSuccess ? n : 0; }
int bscb200_set_device(int device) { return cudaSetDevice(device) == cudaSuccess ? LIBBSC_NO_ERROR : LIBBSC_GPU_ERROR; }

// workspace of a context that only ever DEcompresses blocks of n bytes (inverse BWT + coder stage: ~21 n instead of ~71 n)
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
        unsigned char h[LIBBSC_HEADER_SIZE];
        CUDA_TRY(cudaMemcpyAsync(c->h_mail + 64, d_input, LIBBSC_HEADER_SIZE, cudaMemcpyDeviceToHost, c->stream));
        c->sync(); memcpy(h, c->h_mail + 64, LIBBSC_HEADER_SIZE);
        c->arena.reset(); c->arena.reserve((size_t)bscb200_workspace_bytes_decode(outputSize));   // no-op for a context that already compressed
        return decompress_dev(c, h, d_input, inputSize, d_output, outputSize, features);
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
    return guarded(c, [&]() { c->arena.reset(); c->arena.reserve(need_bwt_decode((size_t)n)); int r = stage_bwt_decode(c, d_T, n, index); c->sync(); return r; });
}
int bscb200_st_encode_device(void *ctx, unsigned char *d_T, int n, int k)
{
    Ctx *c = (Ctx *)ctx;
    if (d_T == nullptr || n < 0 || k < 3 || k > 8) return LIBBSC_BAD_PARAMETER;
    return guarded(c, [&]() { c->arena.reset(); ScratchLease lease(c, need_st_encode((size_t)n)); return stage_st_encode(c, d_T, n, k); });
}
int bscb200_st_decode_device(void *ctx, unsigned char *d_T, int n, int k, int index)
{
    Ctx *c = (Ctx *)ctx;
    if (d_T == nullptr || n < 0 || index < 0 || index >= n || k < 3 || k > 8) return LIBBSC_BAD_PARAMETER;     // st.cpp:1493-1495
    return guarded(c, [&]() { c->arena.reset(); ScratchLease lease(c, need_st_decode((size_t)n)); int r = stage_st_decode(c, d_T, n, k, index); c->sync(); return r; });
}
int bscb200_coder_compress_device(void *ctx, const unsigned char *d_in, unsigned char *d_out, int n, int coder, int features)
{
    Ctx *c = (Ctx *)ctx;
    if (coder < 1 || coder > 3 || n <= 0) return LIBBSC_BAD_PARAMETER;
    return guarded(c, [&]() { c->arena.reset(); c->arena.reserve(need_coder((size_t)n)); return stage_coder_compress(c, d_in, d_out, n, coder, features); });
}
int bscb200_coder_decompress_device(void *ctx, const unsigned char *d_in, int inputSize, unsigned char *d_out, int outputCapacity, int coder, int features)
{
    Ctx *c = (Ctx *)ctx;
    if (coder < 1 || coder > 3 || inputSize < 1 || outputCapacity < 0) return LIBBSC_BAD_PARAMETER;
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
