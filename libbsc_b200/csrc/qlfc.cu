// libbsc_b200/csrc/qlfc.cu -- QLFC entropy stage (static model, coder id 1) on the device.
//
// Replaces bsc_coder_compress / bsc_coder_decompress (libbsc/coder/coder.cpp:244-347) and the
// static QLFC coder under them (libbsc/coder/qlfc/qlfc.cpp:200-255 transform, 829-1129 encoder,
// 1672-1927 decoder; coder/common/rangecoder.h; coder/common/predictor.h:45-61;
// qlfc_model.h:115-241).  The bit stream is reproduced exactly; the data that define it (two
// state tables + the F_* constants) come from qlfc_tables.inc.
//
// Device decomposition of the encoder:
//   q_split      sub-block boundaries of the container (coder.cpp:70-109), one CTA.
//   q_run_*      parallel run detection over the whole block: run start positions + symbols.
//   q_rank_*     stage 1 of QLFC (backward move-to-front rank per run) as tiled parallel ranks (qlfc_ranks.cuh);
//                also emits the MTF-order table.
//   q_encode5    stage 2: context model + binary range coder.  The format fixes <= 8 independent
//                streams per block and each stream is a serial recurrence (adaptive counters +
//                range/low): a six-warp pipeline per stream (qlfc_encoder.cuh), two streams per SM.
//                Throughput comes from running many blocks' streams concurrently.
//   q_decode6    inverse of both stages, one lock-step warp per stream (qlfc_decoder6.cuh), two per SM.
#include "common.cuh"
#include "stages.cuh"
#include <algorithm>
#include <atomic>
#include "qlfc_tables.inc"
#include "qlfc_tables2.inc"

#define Q_MAX_SUB 8

namespace {



enum { K_RANK_T, K_RANK_E, K_RANK_M, K_RANK_P, K_RUN_T, K_RUN_E, K_RUN_M };

__constant__ short c_params[7][15];

struct SubBlock {
    u32 in_start, in_size;       // slice of the block
    u32 run_begin, run_end;      // slice of the run arrays
    u32 out_off, out_cap;        // slice of the temp output / (decode) input stream offset, size
    int result;                  // bytes produced or error
    u32 nsym;
    u32 tile_base, tiles;        // slice of the rank tiles (qlfc_ranks.cuh)
    u32 stat_cached, stat_miss;  // rare-counter cache statistics of the coder kernel
};

// ---------------------------------------------------------------------------------------------
// sub-block split (coder.cpp:70-109): sample i = 1, 33, 65, ...; cut after every (total/nBlocks)
// sampled changes.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) q_split(const u8 *__restrict__ in, u32 n, u32 nBlocks, u32 *__restrict__ start, u32 *__restrict__ size)
{
    __shared__ u32 s_warp[32];
    __shared__ u32 s_total;
    __shared__ u32 s_cut[Q_MAX_SUB];
    const u32 samples = n > 1 ? (n - 2) / 32 + 1 : 0;    // i = 1 + 32*j < n
    const u32 per_thread = (samples + 1023) / 1024;
    const u32 b = threadIdx.x * per_thread, e = min(b + per_thread, samples);
    u32 cnt = 0;
    for (u32 j = b; j < e; ++j) { u32 i = 1 + 32 * j; cnt += (in[i] != in[i - 1]); }
    u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5, incl = cnt;
    for (int o = 1; o < 32; o <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl += t; }
    if (lane == 31) s_warp[w] = incl;
    if (threadIdx.x < Q_MAX_SUB) s_cut[threadIdx.x] = 0;
    __syncthreads();
    u32 pre = 0; for (u32 i = 0; i < w; ++i) pre += s_warp[i];
    u32 excl = pre + incl - cnt;
    if (threadIdx.x == 1023) s_total = pre + incl;
    __syncthreads();
    const u32 total = s_total;
    if (total > nBlocks) {
        const u32 per = total / nBlocks;
        // cut id (1..nBlocks-1) happens at the sample where the running change count reaches id*per
        u32 run = excl;
        for (u32 j = b; j < e; ++j) {
            u32 i = 1 + 32 * j;
            if (in[i] != in[i - 1]) { ++run; if (run % per == 0) { u32 id = run / per; if (id < nBlocks) s_cut[id] = i; } }
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            u32 prev = 0;
            for (u32 id = 0; id < nBlocks; ++id) {
                u32 nxt = (id + 1 < nBlocks) ? s_cut[id + 1] : n;
                start[id] = prev; size[id] = nxt - prev; prev = nxt;
            }
        }
    } else if (threadIdx.x == 0) {
        for (u32 p = 0; p < nBlocks; ++p) { start[p] = (n / nBlocks) * p; size[p] = (p != nBlocks - 1) ? n / nBlocks : n - (n / nBlocks) * (nBlocks - 1); }
    }
}

// ---------------------------------------------------------------------------------------------
// run detection: a run starts where the byte changes or a sub-block starts.
// ---------------------------------------------------------------------------------------------
#define RUN_THREADS 256
#define RUN_ITEMS   16
#define RUN_TILE    (RUN_THREADS * RUN_ITEMS)

__device__ __forceinline__ bool is_run_head(const u8 *__restrict__ in, u32 i, const u32 *s_start, u32 nBlocks)
{
    if (i == 0 || in[i] != in[i - 1]) return true;
    for (u32 s = 1; s < nBlocks; ++s) if (s_start[s] == i) return true;
    return false;
}

__global__ void __launch_bounds__(RUN_THREADS) q_run_count(const u8 *__restrict__ in, u32 n, const u32 *__restrict__ sb_start, u32 nBlocks, u32 *__restrict__ tile_count)
{
    __shared__ u32 s_w[RUN_THREADS / 32];
    __shared__ u32 s_start[Q_MAX_SUB];
    if (threadIdx.x < nBlocks) s_start[threadIdx.x] = sb_start[threadIdx.x];
    __syncthreads();
    u32 base = blockIdx.x * RUN_TILE + threadIdx.x * RUN_ITEMS, c = 0;
    for (int k = 0; k < RUN_ITEMS; ++k) { u32 i = base + k; if (i < n) c += is_run_head(in, i, s_start, nBlocks); }
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((threadIdx.x & 31) == 0) s_w[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) { u32 t = 0; for (int i = 0; i < RUN_THREADS / 32; ++i) t += s_w[i]; tile_count[blockIdx.x] = t; }
}

// exclusive scan of tile counts in place (single CTA); total -> *total_out
__global__ void __launch_bounds__(1024) q_scan_tiles(u32 *__restrict__ tile_count, u32 tiles, u32 *__restrict__ total_out)
{
    __shared__ u32 s_w[32];
    u32 per = (tiles + 1023) / 1024, b = threadIdx.x * per, e = min(b + per, tiles), c = 0;
    for (u32 i = b; i < e; ++i) c += tile_count[i];
    u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5, incl = c;
    for (int o = 1; o < 32; o <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl += t; }
    if (lane == 31) s_w[w] = incl;
    __syncthreads();
    u32 pre = 0; for (u32 i = 0; i < w; ++i) pre += s_w[i];
    u32 run = pre + incl - c;
    for (u32 i = b; i < e; ++i) { u32 t = tile_count[i]; tile_count[i] = run; run += t; }
    if (threadIdx.x == 1023) *total_out = pre + incl;
}

__global__ void __launch_bounds__(RUN_THREADS) q_run_write(const u8 *__restrict__ in, u32 n, const u32 *__restrict__ sb_start, u32 nBlocks,
                                                           const u32 *__restrict__ tile_excl, u32 *__restrict__ run_pos, u8 *__restrict__ run_sym)
{
    __shared__ u32 s_w[RUN_THREADS / 32];
    __shared__ u32 s_start[Q_MAX_SUB];
    if (threadIdx.x < nBlocks) s_start[threadIdx.x] = sb_start[threadIdx.x];
    __syncthreads();
    u32 base = blockIdx.x * RUN_TILE + threadIdx.x * RUN_ITEMS, c = 0;
    bool hd[RUN_ITEMS];
    for (int k = 0; k < RUN_ITEMS; ++k) { u32 i = base + k; hd[k] = (i < n) && is_run_head(in, i, s_start, nBlocks); c += hd[k]; }
    u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5, incl = c;
    for (int o = 1; o < 32; o <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl += t; }
    if (lane == 31) s_w[w] = incl;
    __syncthreads();
    u32 pre = tile_excl[blockIdx.x]; for (u32 i = 0; i < w; ++i) pre += s_w[i];
    u32 o = pre + incl - c;
    for (int k = 0; k < RUN_ITEMS; ++k) if (hd[k]) { run_pos[o] = base + k; run_sym[o] = in[base + k]; ++o; }
}

// run index of each sub-block's first run (binary search over run_pos) + sentinel
__global__ void q_run_bounds(u32 *run_pos, u32 R, u32 n, const u32 *__restrict__ sb_start, const u32 *__restrict__ sb_size, u32 nBlocks,
                             SubBlock *__restrict__ sb)
{
    u32 s = threadIdx.x;
    if (s == 0) run_pos[R] = n;                          // sentinel: run t spans [run_pos[t], run_pos[t+1])
    if (s >= nBlocks) return;
    u32 lo = 0, hi = R;                                  // first run with pos >= sb_start[s]
    while (lo < hi) { u32 mid = (lo + hi) >> 1; if (run_pos[mid] < sb_start[s]) lo = mid + 1; else hi = mid; }
    sb[s].in_start = sb_start[s]; sb[s].in_size = sb_size[s]; sb[s].run_begin = lo;
    u32 endpos = sb_start[s] + sb_size[s];
    u32 lo2 = lo, hi2 = R;
    while (lo2 < hi2) { u32 mid = (lo2 + hi2) >> 1; if (run_pos[mid] < endpos) lo2 = mid + 1; else hi2 = mid; }
    sb[s].run_end = lo2;
}

// ---------------------------------------------------------------------------------------------
// model helpers
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) q_model_init(short *__restrict__ models, size_t total_shorts)
{
    size_t i = ((size_t)blockIdx.x * 256 + threadIdx.x) * 8;
    if (i + 8 <= total_shorts) *(uint4 *)(models + i) = make_uint4(0x08000800u, 0x08000800u, 0x08000800u, 0x08000800u);
    else for (; i < total_shorts; ++i) models[i] = 2048;
}

__device__ __forceinline__ int ilog2_dev(u32 v) { return 31 - __clz(v | 1u); }

// which symbols can still appear in the MTF-order header (qlfc.cpp:857-891): lane l owns symbols 8l..8l+7
__device__ __forceinline__ void header_options(u32 used8, int prev, int prefix, int bit, bool &can0, bool &can1)
{
    u32 lane = lane_id(); bool c0 = false, c1 = false;
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        int c = 8 * (int)lane + k;
        bool cand = (c == prev || !((used8 >> k) & 1u)) && ((c >> (bit + 1)) == prefix);
        if (cand) { if (c & (1 << bit)) c1 = true; else c0 = true; }
    }
    can0 = __any_sync(0xffffffffu, c0); can1 = __any_sync(0xffffffffu, c1);
}

struct QTables { u8 rank_state[32768]; u8 run_state[8192]; };

#include "qlfc_ranks.cuh"
#include "qlfc_coder.cuh"
#include "qlfc_lanes.cuh"
#include "qlfc_fast.cuh"
#include "qlfc_decoder6.cuh"
#include "qlfc_adaptive.cuh"
#include "qlfc_encoder.cuh"

constexpr size_t MODEL_SHORTS_PAD = 2 * (size_t)COLD_PAD;     // by-state + by-symbol cold arrays per stream

}  // namespace

// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static int coder_num_blocks(int n)                        // coder.cpp:52-59
{
    if (n < 256 * 1024) return 1;
    if (n < 4 * 1024 * 1024) return 2;
    if (n < 16 * 1024 * 1024) return 4;
    return 8;
}

// ONE copy of the constant tables per device (never freed: 58 KB), shared by every context: the coders that read the state tables
// through L1 (LayoutDietTG) then share their cache lines between the CTAs of different blocks on an SM.
static const QTables *get_tables(Ctx *ctx)
{
    static std::mutex m; static QTables *per_device[16] = {};
    std::lock_guard<std::mutex> lk(m);
    QTables *&d = per_device[ctx->device & 15];
    if (!d) {
        // multipliers of the hot counter moves (qlfc_decoder6.cuh), stored right after the tables
        int h_moves[QD6_MOVES]; qd6_fill_moves(h_moves);
        // device image: QTables | moves (padded to 128 B) | stretch | squash (the adaptive coder's tables, qlfc_adaptive.cuh)
        static_assert(sizeof(h_moves) <= 128, "moves table slot");
        QTables *t = nullptr;
        CUDA_TRY(cudaMalloc((void **)&t, sizeof(QTables) + 128 + 2 * QA_TAB_BYTES));
        CUDA_TRY(cudaMemcpy(t->rank_state, bscb_rank_state_tab, 32768, cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(t->run_state, bscb_run_state_tab, 8192, cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy(t + 1, h_moves, sizeof(h_moves), cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy((u8 *)(t + 1) + 128, bscb_stretch_le16, 2 * 4097, cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpy((u8 *)(t + 1) + 128 + QA_TAB_BYTES, bscb_squash_le16, 2 * 4097, cudaMemcpyHostToDevice));
        CUDA_TRY(cudaMemcpyToSymbol(c_params, bscb_static_params, sizeof(c_params), 0, cudaMemcpyHostToDevice));
        CUDA_TRY(cudaDeviceSynchronize());
        d = t;
    }
    return d;
}

// Coder ids (libbsc.h:60-62): 1 static, 2 adaptive, 3 fast -- all three run on the device.
static int coder_gate(int coder) { return (coder >= 1 && coder <= 3) ? LIBBSC_NO_ERROR : LIBBSC_BAD_PARAMETER; }
static_assert(QF_COLD <= 2 * (size_t)COLD_PAD, "the fast coder's cold counters must fit the per-stream model allocation");

static void init_models(Ctx *ctx, short *models, int count)
{
    size_t total = (size_t)count * MODEL_SHORTS_PAD;
    LAUNCH(ctx, q_model_init, ceil_div(total, 256 * 8), 256, 0, models, total);
}

// Split launch of a static-coder kernel: the streams of `order[0 .. n_hi)` (the long ones; `order` is sorted longest first) go to the
// context's middle-priority side stream, the rest to its lowest-priority one; both halves report to ONE completion signal.  See Ctx::stream_hi.
// BSCB200_CODER_SPLIT=0 turns it off (A/B).
static bool coder_split_enabled() { static const bool on = [] { const char *e = getenv("BSCB200_CODER_SPLIT"); return !(e && e[0] == '0'); }(); return on; }
static int coder_split_point(const u32 *weight, const u32 *order, int n)
{
    if (!coder_split_enabled() || n < 3) return 0;
    int k = 0;
    while (k < n && (u64)weight[order[k]] * 20 >= (u64)weight[order[0]] * 11) ++k;      // >= 55 % of the longest
    return (k == n) ? 0 : k;
}
// blocks inside a coder stage (either direction) per device: the decoder layout is chosen by this load
struct CodersInFlight {
    static std::atomic<int> &ctr(int device) { static std::atomic<int> c[16]; return c[device & 15]; }
    int device, count;
    explicit CodersInFlight(int dev) : device(dev), count(++ctr(dev)) {}
    ~CodersInFlight() { --ctr(device); }
    static int now(int device) { return ctr(device).load(); }
};
// decoder streams per SM chosen by load (see stage_coder_decompress); sticky per device so that the layouts do not alternate
static int decoder_layout_by_load(int device)
{
    static std::atomic<int> mode[16];
    const int load = CodersInFlight::now(device);
    std::atomic<int> &m = mode[device & 15];
    if (load * Q_MAX_SUB > (int)device_sms(device)) m.store(5);
    else if (load <= 4) m.store(4);
    const int v = m.load();
    return v ? v : 4;
}
struct SplitLaunch {
    Ctx *c; cudaEvent_t ea = nullptr, eb = nullptr; bool prof; double bytes; Ctx::DoneSignalArgs sg; CoderSlots::Lease lease; int n_hi;
    cudaStream_t s_long, s_short;                      // where the long / the other streams of the launch go (Ctx::stream_hi)
    SplitLaunch(Ctx *ctx, int total, int hi) : c(ctx), prof(ctx->profile), bytes(ctx->next_bytes), lease(ctx->device, total), n_hi(hi) {
        if (prof) { ea = c->ev(); eb = c->ev(); CUDA_TRY(cudaEventRecord(ea, c->stream)); }
        sg = c->next_signal();
        s_short = c->coder_stream(); s_long = c->stream_hi;
        if (n_hi > 0 || s_short != c->stream) {
            CUDA_TRY(cudaEventRecord(c->ev_fork, c->stream));
            if (n_hi > 0) CUDA_TRY(cudaStreamWaitEvent(s_long, c->ev_fork, 0));
            if (s_short != c->stream) CUDA_TRY(cudaStreamWaitEvent(s_short, c->ev_fork, 0));
        }
    }
    void finish(const char *name, int launches) {
        c->next_bytes = 0; c->kernels_launched += launches;
        c->wait_signal(s_short, n_hi > 0 ? s_long : nullptr);
        // every kernel of the launch has reported: the joins below never make anything wait
        if (n_hi > 0) { CUDA_TRY(cudaEventRecord(c->ev_join, s_long)); CUDA_TRY(cudaStreamWaitEvent(c->stream, c->ev_join, 0)); }
        if (s_short != c->stream) { CUDA_TRY(cudaEventRecord(c->ev_join_lo, s_short)); CUDA_TRY(cudaStreamWaitEvent(c->stream, c->ev_join_lo, 0)); }
        if (prof) { CUDA_TRY(cudaEventRecord(eb, c->stream)); c->prof.push_back(ProfRec{name, ea, eb, bytes}); }
    }
};

int stage_coder_compress(Ctx *ctx, const u8 *d_in, u8 *d_out, int n_, int coder, int features, int bare_out_size)
{
    { const int g = coder_gate(coder); if (g != LIBBSC_NO_ERROR) return g; }
    const bool fast = coder == 3;
    if (n_ <= 0) return LIBBSC_BAD_PARAMETER;
    CodersInFlight load_(ctx->device);
    const u32 n = (u32)n_;
    // bare_out_size >= 0: ONE stream without the container byte, output capacity as given (bsc_qlfc_*_encode_block, qlfc.h:55-77)
    const bool bare = bare_out_size >= 0;
    const int nBlocks = bare ? 1 : coder_num_blocks(n_);
    const QTables *tables = get_tables(ctx);
    Arena &A = ctx->arena;
    const size_t mark = A.mark();

    u32 *d_start = A.get<u32>(2 * Q_MAX_SUB), *d_size = d_start + Q_MAX_SUB;
    SubBlock *d_sb = A.get<SubBlock>(Q_MAX_SUB);
    const u32 run_tiles = ceil_div(n, RUN_TILE);
    u32 *tile_cnt = A.get<u32>(run_tiles + 1);
    u8 *mtf = A.get<u8>(256 * Q_MAX_SUB);
    short *models = A.get<short>((size_t)nBlocks * MODEL_SHORTS_PAD);
    u8 *tmp = A.get<u8>((size_t)(bare && (u32)bare_out_size > n ? (u32)bare_out_size : n) + (4096 + 256) * Q_MAX_SUB);

    // 1. split
    if (nBlocks > 1) LAUNCH(ctx, q_split, 1, 1024, 0, d_in, n, (u32)nBlocks, d_start, d_size);
    else { u32 *h = ctx->h_mail + 240; h[0] = 0; h[1] = n;   /* pinned: pageable async copies serialise concurrent blocks */CUDA_TRY(cudaMemcpyAsync(d_start, &h[0], 4, cudaMemcpyHostToDevice, ctx->stream)); CUDA_TRY(cudaMemcpyAsync(d_size, &h[1], 4, cudaMemcpyHostToDevice, ctx->stream)); ctx->sync(); }
    // 2. runs
    LAUNCH(ctx, q_run_count, run_tiles, RUN_THREADS, 0, d_in, n, d_start, (u32)nBlocks, tile_cnt);
    LAUNCH(ctx, q_scan_tiles, 1, 1024, 0, tile_cnt, run_tiles, ctx->d_mail);
    CUDA_TRY(cudaMemcpyAsync(ctx->d_mail + 8, d_start, sizeof(u32) * 2 * Q_MAX_SUB, cudaMemcpyDeviceToDevice, ctx->stream));
    ctx->fetch_mail(8 + 2 * Q_MAX_SUB);
    const u32 R = ctx->h_mail[0];
    u32 h_start[Q_MAX_SUB], h_size[Q_MAX_SUB];
    for (int b = 0; b < nBlocks; ++b) { h_start[b] = ctx->h_mail[8 + b]; h_size[b] = ctx->h_mail[8 + Q_MAX_SUB + b]; }

    u32 *run_pos = A.get<u32>((size_t)R + 2);
    u8 *run_sym = A.get<u8>((size_t)R + 32);
    u8 *run_rank = A.get<u8>((size_t)R + 32);
    LAUNCH(ctx, q_run_write, run_tiles, RUN_THREADS, 0, d_in, n, d_start, (u32)nBlocks, tile_cnt, run_pos, run_sym);
    LAUNCH(ctx, q_run_bounds, 1, 32, 0, run_pos, R, n, d_start, d_size, (u32)nBlocks, d_sb);
    // output slices in tmp (256-byte aligned, 4 KB slack each); capacity = the sub-block's input size (coder.cpp:193)
    // All small host<->device copies go through the context's PINNED mailbox.  A cudaMemcpyAsync to or
    // from pageable memory blocks inside the driver until the stream drains (here: a ~1 s coder
    // kernel) and, measured, stalls the pageable copies of every other block's thread meanwhile.
    SubBlock *h_sb = (SubBlock *)(ctx->h_mail + 128);
    CUDA_TRY(cudaMemcpyAsync(h_sb, d_sb, sizeof(SubBlock) * nBlocks, cudaMemcpyDeviceToHost, ctx->stream));
    ctx->sync();
    u32 total_tiles = 0;
    for (u32 b = 0, off = 0; b < (u32)nBlocks; ++b) {
        h_sb[b].out_off = off; off += (u32)align_up((size_t)h_size[b] + 4096, 256);   // 16-bit stores need even offsets
        h_sb[b].out_cap = bare ? (u32)bare_out_size : (nBlocks == 1) ? n - 1 : h_size[b];
        h_sb[b].result = 0; h_sb[b].nsym = 0; h_sb[b].stat_cached = 0; h_sb[b].stat_miss = 0;
        h_sb[b].tile_base = total_tiles; h_sb[b].tiles = ceil_div(h_sb[b].run_end - h_sb[b].run_begin, RK_TILE); total_tiles += h_sb[b].tiles;
    }
    CUDA_TRY(cudaMemcpyAsync(d_sb, h_sb, sizeof(SubBlock) * nBlocks, cudaMemcpyHostToDevice, ctx->stream));
    // Longest stream first: the format's sub-blocks differ 3.5x in length (coder.cpp:70-109 cuts at data-dependent places), a
    // coder CTA runs for as long as its stream has runs, and CTAs start in blockIdx order -- so the order decides how long the
    // last SM of the launch stays busy while the others idle (or pick up another block's streams).
    u32 *enc_order = ctx->h_mail + 224;                     // pinned
    u32 *d_order = A.get<u32>(Q_MAX_SUB);
    for (int b = 0; b < nBlocks; ++b) enc_order[b] = (u32)b;
    std::stable_sort(enc_order, enc_order + nBlocks, [&](u32 x, u32 y) { return h_sb[x].run_end - h_sb[x].run_begin > h_sb[y].run_end - h_sb[y].run_begin; });
    CUDA_TRY(cudaMemcpyAsync(d_order, enc_order, sizeof(u32) * Q_MAX_SUB, cudaMemcpyHostToDevice, ctx->stream));
    // 3. ranks, 4. encode
    {
        u32 *first_tab = A.get<u32>((size_t)total_tiles * 256), *next_tab = A.get<u32>((size_t)total_tiles * 256);
        LAUNCH(ctx, q_rank_first, ceil_div(total_tiles, 4), 128, 0, run_sym, d_sb, (u32)nBlocks, total_tiles, first_tab);
        LAUNCH(ctx, q_rank_scan, nBlocks, 256, 0, d_sb, first_tab, next_tab, mtf);
        PROF_BYTES(ctx, 2.0 * R);
        LAUNCH(ctx, q_rank_tile, ceil_div(total_tiles, 4), 128, 0, run_sym, run_rank, d_sb, (u32)nBlocks, total_tiles, next_tab);
    }
    // The counter file of the static coder is the "diet" layout (qlfc_decoder6.cuh: 106 KB + 5.6 KB of pipe state for the encoder,
    // 110 KB for the decoder), so that TWO coder CTAs share an SM: a coder CTA keeps one scheduler only partly busy (it waits on a
    // dependency chain), so a second stream on the SM costs the first one little.
    static_assert(((sizeof(CoderSmemT<LayoutEncDiet>) + 15) & ~(size_t)15) + sizeof(EncPipe) <= 232448 / 2 - 1024, "two encoders must fit one SM");
    static_assert(3 * (((sizeof(CoderSmemT<LayoutEncDietTG>) + 15) & ~(size_t)15) + sizeof(EncPipe) + 1024) <= 232448, "three encoders without resident state tables must fit one SM");
    static_assert(4 * (((sizeof(CoderSmemT<LayoutEncDiet4>) + 15) & ~(size_t)15) + sizeof(EncPipe) + 1024) <= 232448, "four encoders per SM");
    // Encoder streams per SM: BSCB200_ENC_PER_SM = 2 (state tables resident, LayoutEncDiet), 3 (tables through L1, LayoutEncDietTG; default),
    // 4 (LayoutEncDiet4).  BSCB200_ENC_TG=0 is the old spelling of 2.
    static const int enc_per_sm = [] { const char *t = getenv("BSCB200_ENC_TG"); if (t && t[0] == '0') return 2;
                                       const char *e = getenv("BSCB200_ENC_PER_SM"); const int v = e ? atoi(e) : 0; return (v >= 2 && v <= 4) ? v : 3; }();
    const size_t enc_image = enc_per_sm == 2 ? sizeof(CoderSmemT<LayoutEncDiet>) : enc_per_sm == 3 ? sizeof(CoderSmemT<LayoutEncDietTG>) : sizeof(CoderSmemT<LayoutEncDiet4>);
    const size_t enc_smem = ((enc_image + 15) & ~(size_t)15) + sizeof(EncPipe);
    auto *const enc_kernel = enc_per_sm == 2 ? q_encode5<LayoutEncDiet, 2> : enc_per_sm == 3 ? q_encode5<LayoutEncDietTG, 3> : q_encode5<LayoutEncDiet4, 4>;
    if (fast) {
        LAUNCH(ctx, q_fast_model_init, 256, 256, 0, models, (u32)nBlocks);
        ensure_dyn_smem(q_fast_encode, ctx->device, sizeof(FastSmem));
        PROF_BYTES(ctx, (double)n);
        LAUNCH_LONG(ctx, q_fast_encode, nBlocks, 32, sizeof(FastSmem), run_pos, run_sym, run_rank, d_sb, mtf, models, tmp, (const u32 *)d_order);
    } else if (coder == 2) {
        init_models(ctx, models, nBlocks);
        ensure_dyn_smem(q_adaptive_encode, ctx->device, QA_BYTES);
        PROF_BYTES(ctx, (double)n);
        LAUNCH_LONG(ctx, q_adaptive_encode, nBlocks, 32, QA_BYTES, run_pos, run_sym, run_rank, d_sb, mtf, models, tables, tmp, (const u32 *)d_order);
    } else {
        init_models(ctx, models, nBlocks);
        PROF_BYTES(ctx, (double)n);                      // + c written; the launch is latency-, not bandwidth-bound
        ensure_dyn_smem(enc_kernel, ctx->device, enc_smem);
        u32 runs[Q_MAX_SUB]; for (int b = 0; b < nBlocks; ++b) runs[b] = h_sb[b].run_end - h_sb[b].run_begin;
        const int n_hi = coder_split_point(runs, enc_order, nBlocks);
        SplitLaunch sl(ctx, nBlocks, n_hi);
        const DoneSignal done{sl.sg.ctr, sl.sg.host_flag, sl.sg.seq, (u32)nBlocks};
        if (n_hi > 0) { enc_kernel<<<n_hi, QE_THREADS, enc_smem, sl.s_long>>>(run_pos, run_sym, run_rank, d_sb, mtf, models, tables, tmp, (const u32 *)d_order, done); KERNEL_CHECK(); }
        enc_kernel<<<nBlocks - n_hi, QE_THREADS, enc_smem, sl.s_short>>>(run_pos, run_sym, run_rank, d_sb, mtf, models, tables, tmp, (const u32 *)(d_order + n_hi), done); KERNEL_CHECK();
        sl.finish("q_encode5", n_hi > 0 ? 2 : 1);
    }
    CUDA_TRY(cudaMemcpyAsync(h_sb, d_sb, sizeof(SubBlock) * nBlocks, cudaMemcpyDeviceToHost, ctx->stream));
    ctx->sync();                                         // short: the encoder (0.01 - 0.7 s) was waited for by LAUNCH_LONG

    if (getenv("BSCB200_QSTATS"))
        for (int b = 0; b < nBlocks; ++b) fprintf(stderr, "[qstats enc] sub %d: in %u runs %u out %d rare-accesses %u misses %u\n", b, h_sb[b].in_size, h_sb[b].run_end - h_sb[b].run_begin, h_sb[b].result, h_sb[b].stat_cached, h_sb[b].stat_miss);
    int result;
    if (bare) {
        result = h_sb[0].result;
        if (result > 0) { CUDA_TRY(cudaMemcpyAsync(d_out, tmp + h_sb[0].out_off, (size_t)result, cudaMemcpyDeviceToDevice, ctx->stream)); ctx->sync(); }
        A.release(mark);
        return result;
    }
    if (nBlocks == 1) {                                   // coder.cpp:113-119
        result = h_sb[0].result;
        if (result >= 0) {
            u8 *one = (u8 *)(ctx->h_mail + 240); *one = 1;
            CUDA_TRY(cudaMemcpyAsync(d_out, one, 1, cudaMemcpyHostToDevice, ctx->stream));
            CUDA_TRY(cudaMemcpyAsync(d_out + 1, tmp + h_sb[0].out_off, (size_t)result, cudaMemcpyDeviceToDevice, ctx->stream));
            ctx->sync();
            result += 1;
        }
        A.release(mark);
        return result;
    }

    int res[Q_MAX_SUB];
    const bool parallel_rules = (features & LIBBSC_FEATURE_MULTITHREADING) != 0;
    int ptr = 1 + 8 * nBlocks;
    result = 0;
    if (parallel_rules) {                                 // coder.cpp:159-240
        int total = ptr;
        for (int b = 0; b < nBlocks; ++b) { res[b] = h_sb[b].result < 0 ? (int)h_size[b] : h_sb[b].result; total += res[b]; }
        if (total >= n_) result = LIBBSC_NOT_COMPRESSIBLE;
    } else {                                              // coder.cpp:111-155
        for (int b = 0; b < nBlocks && result == 0; ++b) {
            int room = (int)h_size[b]; if (room > n_ - ptr) room = n_ - ptr;
            int r = h_sb[b].result;
            if (room != (int)h_size[b]) {                 // clipped output size: redo this sub-block with the clipped room
                h_sb[b].out_cap = (u32)(room > 0 ? room : 0); h_sb[b].result = 0;
                u32 *d_list = A.get<u32>(1); u32 &one = ctx->h_mail[240]; one = (u32)b;
                CUDA_TRY(cudaMemcpyAsync(d_sb + b, &h_sb[b], sizeof(SubBlock), cudaMemcpyHostToDevice, ctx->stream));
                CUDA_TRY(cudaMemcpyAsync(d_list, &one, 4, cudaMemcpyHostToDevice, ctx->stream));
                ctx->sync();
                if (fast) {                                // q_fast_encode indexes the cold counters by sub-block id
                    LAUNCH(ctx, q_fast_model_init, 256, 256, 0, models, (u32)nBlocks);
                    LAUNCH_LONG(ctx, q_fast_encode, 1, 32, sizeof(FastSmem), run_pos, run_sym, run_rank, d_sb, mtf, models, tmp, (const u32 *)d_list);
                } else if (coder == 2) {
                    init_models(ctx, models + (size_t)b * MODEL_SHORTS_PAD, 1);
                    LAUNCH_LONG(ctx, q_adaptive_encode, 1, 32, QA_BYTES, run_pos, run_sym, run_rank, d_sb, mtf, models, tables, tmp, (const u32 *)d_list);
                } else {
                    init_models(ctx, models + (size_t)b * MODEL_SHORTS_PAD, 1);
                    LAUNCH_LONG(ctx, enc_kernel, 1, QE_THREADS, enc_smem, run_pos, run_sym, run_rank, d_sb, mtf, models, tables, tmp, (const u32 *)d_list);
                }
                CUDA_TRY(cudaMemcpyAsync(&h_sb[b], d_sb + b, sizeof(SubBlock), cudaMemcpyDeviceToHost, ctx->stream));
                ctx->sync();
                r = h_sb[b].result;
            }
            if (r < 0) { if (ptr + (int)h_size[b] >= n_) { result = LIBBSC_NOT_COMPRESSIBLE; break; } r = (int)h_size[b]; h_sb[b].result = -1; }
            res[b] = r; ptr += r;
        }
        ptr = 1 + 8 * nBlocks;
    }
    if (result == 0) {
        u8 *hdr = (u8 *)(ctx->h_mail + 32);               // pinned scratch (<= 65 bytes)
        hdr[0] = (u8)nBlocks;
        for (int b = 0; b < nBlocks; ++b) {
            u32 a = h_size[b], c = (u32)res[b];
            memcpy(hdr + 1 + 8 * b, &a, 4); memcpy(hdr + 5 + 8 * b, &c, 4);
        }
        CUDA_TRY(cudaMemcpyAsync(d_out, hdr, (size_t)(1 + 8 * nBlocks), cudaMemcpyHostToDevice, ctx->stream));
        for (int b = 0; b < nBlocks; ++b) {
            // coder.cpp:137-141, 224-231: a sub-block whose stored size equals its input size is raw
            const u8 *src = (res[b] == (int)h_size[b]) ? d_in + h_start[b] : tmp + h_sb[b].out_off;
            CUDA_TRY(cudaMemcpyAsync(d_out + ptr, src, (size_t)res[b], cudaMemcpyDeviceToDevice, ctx->stream));
            ptr += res[b];
        }
        ctx->sync();
        result = ptr;
    }
    A.release(mark);
    return result;
}

int stage_coder_decompress(Ctx *ctx, const u8 *d_in, int in_size, u8 *d_out, int out_cap, int coder, int features, bool bare)
{
    (void)features;
    { const int g = coder_gate(coder); if (g != LIBBSC_NO_ERROR) return g; }
    if (in_size < 1) return LIBBSC_UNEXPECTED_EOB;
    CodersInFlight load_(ctx->device);
    const QTables *tables = get_tables(ctx);
    Arena &A = ctx->arena;
    const size_t mark = A.mark();

    u8 hdr[1 + 8 * 255];
    {
        int want = in_size < 65 ? in_size : 65;
        CUDA_TRY(cudaMemcpyAsync(ctx->h_mail + 32, d_in, (size_t)want, cudaMemcpyDeviceToHost, ctx->stream));
        ctx->sync();
        memcpy(hdr, ctx->h_mail + 32, (size_t)want);
    }
    const int nBlocks = bare ? 1 : hdr[0];               // bare: ONE stream without the container byte (bsc_qlfc_*_decode_block, qlfc.h:79-99)
    SubBlock *h_sb = (SubBlock *)(ctx->h_mail + 128); u32 *list = ctx->h_mail + 232; int nlist = 0;   // pinned (see stage_coder_compress)
    memset(h_sb, 0, sizeof(SubBlock) * Q_MAX_SUB); memset(list, 0, sizeof(u32) * Q_MAX_SUB);
    if (nBlocks == 1) {
        h_sb[0].in_start = 0; h_sb[0].in_size = (u32)out_cap; h_sb[0].out_off = bare ? 0 : 1; h_sb[0].out_cap = (u32)(in_size - (bare ? 0 : 1));
        list[nlist++] = 0;
    } else {
        if (nBlocks == 0) { A.release(mark); return 0; }   // an empty container decodes to 0 bytes, as in the reference (coder.cpp:339-346)
        if (nBlocks > Q_MAX_SUB || in_size < 1 + 8 * nBlocks) { A.release(mark); return LIBBSC_DATA_CORRUPT; }
        long long inPtr = 1 + 8 * nBlocks, outPtr = 0;
        for (int b = 0; b < nBlocks; ++b) {
            int rawSize, packed; memcpy(&rawSize, hdr + 1 + 8 * b, 4); memcpy(&packed, hdr + 5 + 8 * b, 4);
            if (rawSize < 0 || packed < 0 || outPtr + rawSize > out_cap) { A.release(mark); return LIBBSC_DATA_CORRUPT; }
            // Every sub-stream lies inside the payload.  The reference never uses the packed size of the LAST coded sub-block
            // (coder.cpp:318-336: it only places the sub-blocks after it), so that one is bounded by the payload's end instead of being
            // rejected; a stored sub-block is copied whole and must fit.
            const long long avail = in_size - inPtr;
            if (packed > avail && (b != nBlocks - 1 || packed == rawSize)) { A.release(mark); return LIBBSC_DATA_CORRUPT; }
            h_sb[b].in_start = (u32)outPtr; h_sb[b].in_size = (u32)rawSize; h_sb[b].out_off = (u32)inPtr; h_sb[b].out_cap = (u32)std::min<long long>(packed, avail);
            if (packed != rawSize) list[nlist++] = (u32)b;
            else { h_sb[b].result = rawSize; if (rawSize) CUDA_TRY(cudaMemcpyAsync(d_out + outPtr, d_in + inPtr, (size_t)rawSize, cudaMemcpyDeviceToDevice, ctx->stream)); }
            inPtr += packed; outPtr += rawSize;
        }
    }
    // longest stream first (see stage_coder_compress); the packed size is the best proxy for the number of decisions
    std::stable_sort(list, list + nlist, [&](u32 x, u32 y) { return h_sb[x].out_cap > h_sb[y].out_cap; });
    if (nlist > 0) {
        SubBlock *d_sb = A.get<SubBlock>(Q_MAX_SUB);
        u32 *d_list = A.get<u32>(Q_MAX_SUB);
        short *models = A.get<short>((size_t)nlist * MODEL_SHORTS_PAD);
        CUDA_TRY(cudaMemcpyAsync(d_sb, h_sb, sizeof(SubBlock) * Q_MAX_SUB, cudaMemcpyHostToDevice, ctx->stream));
        CUDA_TRY(cudaMemcpyAsync(d_list, list, sizeof(u32) * Q_MAX_SUB, cudaMemcpyHostToDevice, ctx->stream));
        ctx->sync();
        if (coder == 3) {
            LAUNCH(ctx, q_fast_model_init, 256, 256, 0, models, (u32)nlist);
            ensure_dyn_smem(q_fast_decode, ctx->device, sizeof(FastSmem));
            PROF_BYTES(ctx, (double)in_size + (double)out_cap);
            LAUNCH_LONG(ctx, q_fast_decode, nlist, 32, sizeof(FastSmem), d_in, d_sb, models, d_out, (const u32 *)d_list);
        } else if (coder == 2) {
            init_models(ctx, models, nlist);
            ensure_dyn_smem(q_adaptive_decode, ctx->device, QA_BYTES);
            PROF_BYTES(ctx, (double)in_size + (double)out_cap);
            LAUNCH_LONG(ctx, q_adaptive_decode, nlist, 32, QA_BYTES, d_in, d_sb, models, tables, d_out, (const u32 *)d_list);
        } else {
            init_models(ctx, models, nlist);
            PROF_BYTES(ctx, (double)in_size + (double)out_cap);
            static const bool prof = getenv("BSCB200_QDEC_PROF") != nullptr;          // per-phase cycle counts (diagnostic)
            static_assert(LayoutDiet::BYTES <= 232448 / 2 - 1024, "two decoder streams must fit one SM");
            if (prof) { ensure_dyn_smem(q_decode6<LayoutDiet, true>, ctx->device, LayoutDiet::BYTES);
                        LAUNCH_LONG(ctx, (q_decode6<LayoutDiet, true>), nlist, 32, LayoutDiet::BYTES, d_in, d_sb, models, tables, d_out, d_list); }
            else {
                u32 packed[Q_MAX_SUB]; for (int b = 0; b < Q_MAX_SUB; ++b) packed[b] = h_sb[b].out_cap;
                const int n_hi = coder_split_point(packed, list, nlist);
                // Streams per SM = how much of the counter file is resident (qlfc_decoder6.cuh).  BSCB200_DEC_PER_SM = 2: LayoutDiet (state
                // tables resident, 110 KB); 3: LayoutDietTG (tables through L1, 71 KB); 4: LayoutDiet4 (55 KB, rank exponent 4 row-wise);
                // 5: LayoutDiet5 (39 KB; slower per stream when alone, more streams in flight in a full pipeline).
                // Default: by load, with hysteresis -- 4 per SM while every stream of the blocks in coder stages on this device can have an SM
                // share of its own choosing (blocks x 8 streams <= the device's SMs, 16 blocks on an H100: a caller with a handful of blocks
                // wants the short latency); 5 per SM
                // once streams have to share SMs anyway, and then until the device has drained to 4 blocks: a MIX of 55 KB and 39 KB CTAs packs
                // an SM badly (a load hovering around a single threshold was slower than either layout alone in a full pipeline).
                static const int forced = [] { const char *e = getenv("BSCB200_DEC_PER_SM"); const int v = e ? atoi(e) : 0; return (v >= 2 && v <= 5) ? v : 0; }();
                const int per_sm = forced ? forced : decoder_layout_by_load(ctx->device);
                auto launch = [&](auto kernel, size_t smem) {
                    ensure_dyn_smem(kernel, ctx->device, smem);
                    SplitLaunch sl(ctx, nlist, n_hi);
                    const DoneSignal done{sl.sg.ctr, sl.sg.host_flag, sl.sg.seq, (u32)nlist};
                    if (n_hi > 0) { kernel<<<n_hi, 32, smem, sl.s_long>>>(d_in, d_sb, models, tables, d_out, (const u32 *)d_list, done); KERNEL_CHECK(); }
                    kernel<<<nlist - n_hi, 32, smem, sl.s_short>>>(d_in, d_sb, models + (size_t)n_hi * MODEL_SHORTS_PAD, tables, d_out, (const u32 *)(d_list + n_hi), done); KERNEL_CHECK();
                    sl.finish("q_decode6", n_hi > 0 ? 2 : 1);
                };
                switch (per_sm) {
                case 2:  launch(q_decode6<LayoutDiet, false>, LayoutDiet::BYTES); break;
                case 3:  launch(q_decode6<LayoutDietTG, false>, LayoutDietTG::BYTES); break;
                case 4:  launch(q_decode6<LayoutDiet4, false>, LayoutDiet4::BYTES); break;
                default: launch(q_decode6<LayoutDiet5, false>, LayoutDiet5::BYTES); break;
                }
            }
        }
        CUDA_TRY(cudaMemcpyAsync(h_sb, d_sb, sizeof(SubBlock) * Q_MAX_SUB, cudaMemcpyDeviceToHost, ctx->stream));
    }
    ctx->sync();                                         // short: the decoder (up to 2 s) was waited for by LAUNCH_LONG
    if (getenv("BSCB200_QSTATS"))
        for (int b = 0; b < (nBlocks == 1 ? 1 : nBlocks); ++b) fprintf(stderr, "[qstats dec] sub %d: out %d rare-accesses %u misses %u\n", b, h_sb[b].result, h_sb[b].stat_cached, h_sb[b].stat_miss);
    int total = 0, err = 0;
    for (int b = 0; b < (nBlocks == 1 ? 1 : nBlocks); ++b) { if (h_sb[b].result < 0) err = h_sb[b].result; total += h_sb[b].result; }
    A.release(mark);
    return err ? err : total;
}
