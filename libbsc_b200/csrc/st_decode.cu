// libbsc_b200/csrc/st_decode.cu -- inverse sort transform of order k (k = 3..8) on the device.
//
// Replaces bsc_st_decode (libbsc/st/st.cpp:1491-1527; context-boundary sort 1014-1093 / 1248-1330, reconstruction
// 1095-1244 / 1332-1480).  The reference prepares per-context counters and then walks the whole text as ONE serial chain
// of n dependent steps (both its serial and its OpenMP variant: only the preparation is parallel there).
//
// What is computed (SURVEY.md B.2): rows = the n cyclic rotations of T stably sorted by their first k bytes, L[j] = the byte
// preceding rotation j, `index` = the row of rotation 0.  Rows with equal k-byte context form a k-GROUP and stand in text
// order inside it.  Going backwards through the text from a row of group G with L = c always lands in the group
// G' = (c, first k-1 bytes of G), and the rows of G' are consumed from the last one to the first one (text order again).
// So T read backwards is a walk over a graph whose nodes are k-groups and whose edges are rows.
//
// Design here -- as much of that walk as possible becomes a STATIC permutation that is ranked in parallel:
//   * LF = destination of the stable counting sort of L (lf_map.cuh, shared with the inverse BWT) maps the rows of a
//     (k-1)-group that carry symbol c ONTO the group G' = (c, that (k-1)-group), in row order.
//   * When all those source rows lie in ONE k-group, row order = text order on both sides, so LF is exactly the walk's
//     step (STATIC edge).  When they come from several k-groups their interleaving in text order is only known to the
//     walk itself: G' is a DYNAMIC group, its rows are list heads and the edges into it are list ends.
//   * The text being cyclic, rotation 0 (first of its group, visited FIRST) pairs with the LAST row of its target group: if
//     that group is otherwise static its edges are the LF edges shifted by one (st_link), else it is dynamic anyway.
//   st_round x k   group boundaries for context orders 1..k: flag_{r+1}[LF[i]] = "i is the first row with its symbol in its
//                  r-group" = r-group of i differs from the r-group of the previous row with the same symbol; one fused
//                  pass per order: decoupled look-back max-scan (group start per row) + scatter through LF
//   st_groups      last row (= stack top) of every k-group, dynamic flag (sources from more than one k-group)
//   st_link        per row: static successor, or list end + the dynamic group it pops from
//   lr_jump x log  in-place Wyllie pointer jumping on 64-bit (successor, distance) pairs (list_rank.cuh) -> list end + distance per row;
//                  rounds after convergence return at once (device-side flag, no host round trip)
//   st_heads       per list head: list length and the dynamic group its end pops from
//   st_serial      the part that is inherently serial: one lane pops list heads, one step per LIST (not per byte) -- n/4 steps
//                  on English text at k = 6, a few hundred on the 32 MiB high-entropy blocks of BASELINE config 5
//   st_place/emit  text offset of every list, then every row writes its byte to its final place
// Memory ~ 39 n in the pooled layout; 25 n after L in the lean layout of the blocks above 1 GiB (st_decode_run below).
// Latency/sector bound (random 4/8-byte gathers), not stream bound.
#include "common.cuh"
#include "stages.cuh"
#include "lf_map.cuh"
#include "list_rank.cuh"

#include <chrono>

#define SR_THREADS 256
#define SR_ITEMS   8
#define SR_TILE    (SR_THREADS * SR_ITEMS)

#define ST_DONE   LR_DONE
#define ST_NONE   0xffffffffu

namespace {

// Rows that start a 1-byte context bucket: f1[C[c]] = 1 for every symbol that occurs.
__global__ void st_flag1(const u32 *__restrict__ cbase, u32 n, u8 *__restrict__ f1)
{
    u32 c = threadIdx.x;
    u32 lo = cbase[c], hi = c == 255 ? n : cbase[c + 1];
    if (lo < hi) f1[lo] = 1;
}

// One context order: g[j] = start row of j's r-group (inclusive max-scan of "j starts a group ? j : 0"; row 0 always starts one),
// then tmp_out[LF[j]] = g[j].  flag_r[j] = f1[j] | (tmp_in[j] != tmp_in[j-1]) for r > 1 (tmp_in = previous order's scatter).
template <bool FIRST, bool LAST>
__global__ void __launch_bounds__(SR_THREADS)
st_round(const u8 *__restrict__ f1, const u32 *__restrict__ tmp_in, const u32 *__restrict__ LF, u32 n,
         u32 *tile_counter, u64 *lookback, u32 *__restrict__ tmp_out, u32 *__restrict__ gk)
{
    __shared__ u32 s_tile, s_warp[SR_THREADS / 32], s_prefix;
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) s_tile = atomicAdd(tile_counter, 1u);
    __syncthreads();
    const u32 tile = s_tile, base = tile * SR_TILE + tid * SR_ITEMS;

    u32 g[SR_ITEMS];
    u32 prev = 0;
    if (!FIRST && base > 0 && base < n) prev = tmp_in[base - 1];
    u32 run = 0;
#pragma unroll
    for (int i = 0; i < SR_ITEMS; ++i) {
        const u32 j = base + i;
        bool fl = false;
        if (j < n) {
            fl = f1[j] != 0;
            if (!FIRST) { u32 t = tmp_in[j]; fl = fl || (t != prev); prev = t; }
        }
        if (fl) run = j;
        g[i] = run;
    }
    // block-wide inclusive max-scan of the per-thread maxima
    u32 incl = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl = max(incl, t); }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    u32 excl = __shfl_up_sync(0xffffffffu, incl, 1); if (lane == 0) excl = 0;
    for (u32 w = 0; w < warp; ++w) excl = max(excl, s_warp[w]);
    if (tid == 0) {
        u32 total = 0;
        for (u32 w = 0; w < SR_THREADS / 32; ++w) total = max(total, s_warp[w]);
        u64 *mine = lookback + tile;
        u32 pre = 0;
        if (tile == 0) st_relaxed(mine, LB_FLAG_PREFIX | (u64)total);
        else {
            st_relaxed(mine, LB_FLAG_AGG | (u64)total);
            for (u32 t = tile; t-- > 0; ) {
                u64 v;
                do { v = ld_relaxed(lookback + t); } while ((v & LB_FLAG_MASK) == 0);
                pre = max(pre, (u32)v);
                if ((v & LB_FLAG_MASK) == LB_FLAG_PREFIX) break;
            }
            st_relaxed(mine, LB_FLAG_PREFIX | (u64)max(pre, total));
        }
        s_prefix = pre;
    }
    __syncthreads();
    excl = max(excl, s_prefix);
#pragma unroll
    for (int i = 0; i < SR_ITEMS; ++i) {
        const u32 j = base + i;
        if (j < n) {
            const u32 v = max(g[i], excl);
            tmp_out[LF[j]] = v;
            if (LAST) gk[j] = v;
        }
    }
}

// Per k-group (keyed by its start row a): top[a] = its last row; dynf[a] = 1 when the rows that map INTO it come from more than
// one k-group (tmpk[j] = k-group of the LF-source of row j; sources of a group are increasing rows, so first != last decides).
__global__ void __launch_bounds__(256) st_groups(const u32 *__restrict__ gk, const u32 *__restrict__ tmpk, u32 n, u32 *__restrict__ top, u8 *__restrict__ dynf)
{
    u32 j = blockIdx.x * 256 + threadIdx.x;
    if (j >= n) return;
    const u32 a = gk[j];
    if (j + 1 == n || gk[j + 1] != a) {
        top[a] = j;
        if (tmpk[a] != tmpk[j]) dynf[a] = 1;
    }
}

// params[0] = the group rotation 0 steps into (its edges are LF shifted by one when it is static)
__global__ void st_special(const u32 *__restrict__ gk, const u32 *__restrict__ LF, u32 index, u32 *params) { params[0] = gk[LF[index]]; }

// pair[i] = (successor | distance << 32): a list end points to itself with distance 0 and carries ST_DONE.
__global__ void __launch_bounds__(256) st_link(const u32 *__restrict__ LF, const u32 *__restrict__ gk, const u8 *__restrict__ dynf, const u32 *__restrict__ top,
                                               const u32 *__restrict__ params, u32 n, u32 index, u64 *__restrict__ pair, u32 *__restrict__ tgt)
{
    u32 i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const u32 lf = LF[i], t = gk[lf];
    u32 nx = lf, target = ST_NONE;
    bool end = false;
    if (dynf[t]) { end = true; target = t; }
    else {
        if (t == params[0]) nx = (i == index) ? top[t] : lf - 1;
        if (nx == index) end = true;                     // the walk ends in front of rotation 0
    }
    tgt[i] = target;
    pair[i] = end ? ((u64)i | ((u64)ST_DONE << 32)) : ((u64)nx | (1ull << 32));
}

// rec[h] = (list length | dynamic group its end pops from << 32) for every list head h (rows of dynamic groups + rotation 0)
__global__ void __launch_bounds__(256) st_heads(const u64 *__restrict__ pair, const u32 *__restrict__ gk, const u8 *__restrict__ dynf, const u32 *__restrict__ tgt,
                                                u32 n, u32 index, u64 *__restrict__ rec)
{
    u32 h = blockIdx.x * 256 + threadIdx.x;
    if (h >= n) return;
    if (h != index && !dynf[gk[h]]) return;
    const u64 p = pair[h];
    const u32 e = (u32)p, len = ((u32)(p >> 32) & ~ST_DONE) + 1;
    rec[h] = (u64)len | ((u64)tgt[e] << 32);
}

// The serial part: list after list, backwards through the text.  posh[h] = text offset of the END of list h (its lowest offset).
__global__ void st_serial(const u64 *__restrict__ rec, u32 *top, u32 n, u32 index, u32 *__restrict__ posh, u32 *status, DoneSignal done)
{
    if (threadIdx.x != 0) return;
    long long cur = n;
    u32 h = index, steps = 0;
    for (;;) {
        const u64 r = rec[h];
        u32 len = (u32)r; if (len == 0) len = 1;         // only unvisited garbage on corrupt input
        cur -= len;
        posh[h] = cur > 0 ? (u32)cur : 0;
        if (cur <= 0) break;
        const u32 g = (u32)(r >> 32);
        if (g >= n || ++steps > n) break;                // corrupt input guard
        const u32 t = top[g]; top[g] = t - 1;
        if (t >= n) break;
        h = t;
    }
    status[0] = cur == 0 ? 0u : 1u;                      // 1: the lists do not tile the text (corrupt input)
    signal_done(done);
}

__global__ void __launch_bounds__(256) st_place(const u64 *__restrict__ pair, const u32 *__restrict__ gk, const u8 *__restrict__ dynf, const u32 *__restrict__ posh,
                                                u32 n, u32 index, u32 *__restrict__ posE)
{
    u32 h = blockIdx.x * 256 + threadIdx.x;
    if (h >= n) return;
    if (h != index && !dynf[gk[h]]) return;
    posE[(u32)pair[h]] = posh[h];
}

__global__ void __launch_bounds__(256) st_emit(const u64 *__restrict__ pair, const u32 *__restrict__ posE, const u8 *__restrict__ L, u32 n, u8 *__restrict__ out)
{
    u32 i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const u64 p = pair[i];
    const u64 pos = (u64)posE[(u32)p] + ((u32)(p >> 32) & ~ST_DONE);
    if (pos < n) out[pos] = L[i];
}

// ---- the lean layout (blocks above 1 GiB): the same steps, with `rec` split into two u32 arrays that live in dead space -------------
// rlen[h] = list length (in LF's space, zeroed after st_link); the dynamic group its end pops from is written IN PLACE over tgt.
// In place is safe: the lists are disjoint and only heads are written.  Thread h reads tgt[e], e = end(h); e is h itself (a one-row list:
// the same thread reads, then writes) or a row that heads no list, whose tgt no thread writes and only h's list ends at.
__global__ void __launch_bounds__(256) st_heads_lean(const u64 *__restrict__ pair, const u32 *__restrict__ gk, const u8 *__restrict__ dynf, u32 *tgt,
                                                     u32 n, u32 index, u32 *__restrict__ rlen)
{
    u32 h = blockIdx.x * 256 + threadIdx.x;
    if (h >= n) return;
    if (h != index && !dynf[gk[h]]) return;
    const u64 p = pair[h];
    const u32 e = (u32)p;
    rlen[h] = ((u32)(p >> 32) & ~ST_DONE) + 1;
    tgt[h] = tgt[e];
}

// st_serial on the two arrays.  posh[h] is written IN PLACE over rlen[h]: the one lane reads a head's length before it writes that
// head's offset, and each head is visited once on valid input (a second visit on corrupt input reads an offset as a length: the
// same bounded loop, the same status).
__global__ void st_serial_lean(u32 *rlen_posh, const u32 *__restrict__ rgrp, u32 *top, u32 n, u32 index, u32 *status, DoneSignal done)
{
    if (threadIdx.x != 0) return;
    long long cur = n;
    u32 h = index, steps = 0;
    for (;;) {
        u32 len = rlen_posh[h]; if (len == 0) len = 1;   // only unvisited garbage on corrupt input
        const u32 g = rgrp[h];
        ++steps;
        cur -= len;
        rlen_posh[h] = cur > 0 ? (u32)cur : 0;
        if (cur <= 0) break;
        if (g >= n || steps > n) break;                 // corrupt input guard
        const u32 t = top[g]; top[g] = t - 1;
        if (t >= n) break;
        h = t;
    }
    status[0] = cur == 0 ? 0u : 1u;                      // 1: the lists do not tile the text (corrupt input)
    status[1] = steps;                                   // lists visited (BSCB200_STSTATS)
    signal_done(done);
}

// st_place with posE written IN PLACE over posh: head h reads pos[h] and writes pos[end(h)].  end(h) is h itself or a row that heads no
// list, and only heads are read, so no thread reads an entry that another thread writes.  Ends that no head reaches keep a stale value
// (corrupt input only): st_emit's `pos < n` guard keeps every write inside the output.
__global__ void __launch_bounds__(256) st_place_lean(const u64 *__restrict__ pair, const u32 *__restrict__ gk, const u8 *__restrict__ dynf, u32 *pos,
                                                     u32 n, u32 index)
{
    u32 h = blockIdx.x * 256 + threadIdx.x;
    if (h >= n) return;
    if (h != index && !dynf[gk[h]]) return;
    const u32 v = pos[h];
    pos[(u32)pair[h]] = v;
}

}  // namespace

size_t st_decode_lean_bytes(size_t n) { return 25 * n + (1u << 20); }

// Both layouts enqueue the same kernels in the same order.
// POOLED (stage_st_decode): every array lives for the whole stage, about 39 n in a sort slab, next to the caller's block.
// LEAN (stage_st_decode_lean): L is read where it lies and arrays that are dead take the place of later ones, 25 n after L:
//   LF 4 | gk 4 | f1 1 | tmp[0] 4 | tmp[1] 4 | pair 8       (u32 arrays n + 2 words, `pair` n + 2 u64)
//   lb, slb (the look-back descriptors, n / 2 + n / 32)   in `pair`, which st_link writes first, after the last use of both
//   dynf                                                  in f1, dead after the last st_round (zeroed again)
//   top                                                   in the tmp buffer the last round read; st_groups reads only tmpk
//   tgt                                                   in tmpk, dead after st_groups (st_special and st_link do not read it)
//   rlen, then posh, then posE                            in LF, dead after st_link (st_heads_lean, st_serial_lean, st_place_lean)
//   group of each head's end                              in place over tgt (st_heads_lean)
//   the output                                            in gk, dead after st_place
// The peak is the whole region at st_link: L 1 + LF 4 + gk 4 + dynf 1 + top 4 + tgt 4 + pair 8 = 26 n.
static int st_decode_run(Ctx *ctx, u8 *d_T, int n_, int k, int index_, u8 **lean_out)
{
    if (d_T == nullptr || n_ < 0) return LIBBSC_BAD_PARAMETER;       // st.cpp:1493-1496, same order
    if (index_ < 0 || index_ >= n_) return LIBBSC_BAD_PARAMETER;
    if (k < 3 || k > 8) return LIBBSC_BAD_PARAMETER;
    if (lean_out) *lean_out = d_T;
    if (n_ <= 1) return LIBBSC_NO_ERROR;
    const bool lean = lean_out != nullptr;
    const u32 n = (u32)n_, index = (u32)index_;
    Arena &A = lean ? ctx->arena : ctx->sort_arena();
    const size_t mark = A.mark();

    const u32 lf_tiles = ceil_div(n, LF_TILE), sr_tiles = ceil_div(n, SR_TILE), nb = ceil_div(n, 256);
    u8 *Lp, *f1, *dynf;
    u32 *LF, *hist, *tmp[2], *gk, *top, *small;
    u64 *lb, *pair, *rec, *slb;
    if (!lean) {
        Lp    = A.get<u8>((size_t)n + 64);
        LF    = A.get<u32>((size_t)n + 2);
        hist  = A.get<u32>(256 + 64);
        lb    = A.get<u64>((size_t)lf_tiles * 256);
        f1    = A.get<u8>((size_t)n + 64);
        dynf  = A.get<u8>((size_t)n + 64);
        tmp[0] = A.get<u32>((size_t)n + 2); tmp[1] = A.get<u32>((size_t)n + 2);
        gk    = A.get<u32>((size_t)n + 2);
        top   = A.get<u32>((size_t)n + 2);
        pair  = A.get<u64>((size_t)n + 2);
        rec   = A.get<u64>((size_t)n + 2);
        slb   = A.get<u64>((size_t)sr_tiles * 8);            // look-back descriptors, one set per context order
        small = A.get<u32>(128);                             // [0..7] tile counters, [8] params, [9] status, [16..63] jump flags
    } else {
        const size_t lb_words = align_up((size_t)lf_tiles * 256, 32);
        Lp    = d_T;
        LF    = A.get<u32>((size_t)n + 2);
        gk    = A.get<u32>((size_t)n + 2);
        f1    = A.get<u8>((size_t)n + 64);
        tmp[0] = A.get<u32>((size_t)n + 2); tmp[1] = A.get<u32>((size_t)n + 2);
        pair  = A.get<u64>(std::max((size_t)n + 2, lb_words + (size_t)sr_tiles * 8));
        hist  = A.get<u32>(256 + 64);
        small = A.get<u32>(128);
        lb = pair; slb = pair + lb_words;
        dynf = f1; top = nullptr; rec = nullptr;             // placed below, once their space is dead
    }

    if (!lean) CUDA_TRY(cudaMemcpyAsync(Lp, d_T, n, cudaMemcpyDeviceToDevice, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(Lp + n, 0, 64, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(hist, 0, sizeof(u32) * (256 + 64), ctx->stream));
    CUDA_TRY(cudaMemsetAsync(lb, 0, sizeof(u64) * (size_t)lf_tiles * 256, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(f1, 0, (size_t)n, ctx->stream));
    if (!lean) CUDA_TRY(cudaMemsetAsync(dynf, 0, (size_t)n, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(slb, 0, sizeof(u64) * (size_t)sr_tiles * 8, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(small, 0, sizeof(u32) * 128, ctx->stream));
    if (!lean) CUDA_TRY(cudaMemsetAsync(rec, 0, sizeof(u64) * (size_t)n, ctx->stream));

    LAUNCH(ctx, unbwt_hist, min(ceil_div(n, 256 * 64), device_sms(ctx->device) * 8), 256, 0, Lp, n, hist);
    LAUNCH(ctx, unbwt_scan256, 1, 32, 0, hist);
    PROF_BYTES(ctx, 5.0 * n);
    LAUNCH(ctx, unbwt_lf<false>, lf_tiles, LF_THREADS, 0, Lp, n, n, hist, hist + 256, lb, LF);
    LAUNCH(ctx, st_flag1, 1, 256, 0, hist, n, f1);

    int cur = 0;                                             // tmp[cur] = scatter of the previous order
    for (int r = 1; r <= k; ++r) {
        PROF_BYTES(ctx, 13.0 * n);
        u32 *tc = small + (r - 1); u64 *lbr = slb + (size_t)(r - 1) * sr_tiles;
        if (r == 1)      LAUNCH(ctx, (st_round<true, false>),  sr_tiles, SR_THREADS, 0, f1, (const u32 *)nullptr, LF, n, tc, lbr, tmp[0], gk);
        else if (r < k)  LAUNCH(ctx, (st_round<false, false>), sr_tiles, SR_THREADS, 0, f1, tmp[cur], LF, n, tc, lbr, tmp[cur ^ 1], gk);
        else             LAUNCH(ctx, (st_round<false, true>),  sr_tiles, SR_THREADS, 0, f1, tmp[cur], LF, n, tc, lbr, tmp[cur ^ 1], gk);
        if (r > 1) cur ^= 1;
    }
    u32 *tmpk = tmp[cur], *tgt = tmp[cur ^ 1];
    if (lean) {
        top = tmp[cur ^ 1]; tgt = tmpk;                      // the last round's input is dead; tmpk is dead after st_groups
        CUDA_TRY(cudaMemsetAsync(dynf, 0, (size_t)n, ctx->stream));   // f1's bytes: dead after the last round
    }
    LAUNCH(ctx, st_groups, nb, 256, 0, gk, tmpk, n, top, dynf);
    LAUNCH(ctx, st_special, 1, 1, 0, gk, LF, index, small + 8);
    PROF_BYTES(ctx, 25.0 * n);
    LAUNCH(ctx, st_link, nb, 256, 0, LF, gk, dynf, top, small + 8, n, index, pair, tgt);
    lr_rank(ctx, pair, n, n, small + 16);
    if (!lean) {
        LAUNCH(ctx, st_heads, nb, 256, 0, pair, gk, dynf, tgt, n, index, rec);
        u32 *posh = LF, *posE = tmpk;                        // both free from here on
        CUDA_TRY(cudaMemsetAsync(posE, 0, sizeof(u32) * (size_t)n, ctx->stream));
        LAUNCH_LONG(ctx, st_serial, 1, 32, 0, rec, top, n, index, posh, small + 9);   // up to seconds on text (one step per list): nothing queued behind it
        LAUNCH(ctx, st_place, nb, 256, 0, pair, gk, dynf, posh, n, index, posE);
        PROF_BYTES(ctx, 14.0 * n);
        LAUNCH(ctx, st_emit, nb, 256, 0, pair, posE, Lp, n, d_T);
        A.release(mark);
        return LIBBSC_NO_ERROR;
    }
    u32 *pos = LF;                                           // rlen, then posh, then posE: LF is dead after st_link
    u8 *out = (u8 *)gk;                                      // gk is dead after st_place
    CUDA_TRY(cudaMemsetAsync(pos, 0, sizeof(u32) * (size_t)n, ctx->stream));
    LAUNCH(ctx, st_heads_lean, nb, 256, 0, pair, gk, dynf, tgt, n, index, pos);
    static const bool stats = getenv("BSCB200_STSTATS") != nullptr;      // one line per block on stderr: lists and st_serial time
    if (stats) ctx->sync();
    const auto t0 = std::chrono::steady_clock::now();
    LAUNCH_LONG(ctx, st_serial_lean, 1, 32, 0, pos, tgt, top, n, index, small + 9);
    const double serial_s = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    LAUNCH(ctx, st_place_lean, nb, 256, 0, pair, gk, dynf, pos, n, index);
    PROF_BYTES(ctx, 14.0 * n);
    LAUNCH(ctx, st_emit, nb, 256, 0, pair, pos, Lp, n, out);
    CUDA_TRY(cudaMemcpyAsync(ctx->h_mail + 240, small + 9, 2 * sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
    ctx->sync();
    if (stats) fprintf(stderr, "[ststats] n %u k %d lists %u st_serial %.3f s\n", n, k, ctx->h_mail[241], serial_s);
    *lean_out = out;                                         // the caller's region: not released
    return ctx->h_mail[240] == 0 ? LIBBSC_NO_ERROR : LIBBSC_DATA_CORRUPT;
}

int stage_st_decode(Ctx *ctx, u8 *d_T, int n, int k, int index) { return st_decode_run(ctx, d_T, n, k, index, nullptr); }

int stage_st_decode_lean(Ctx *ctx, u8 *d_L, int n, int k, int index, u8 **d_result)
{
    if (d_result == nullptr) return LIBBSC_BAD_PARAMETER;
    return st_decode_run(ctx, d_L, n, k, index, d_result);
}
