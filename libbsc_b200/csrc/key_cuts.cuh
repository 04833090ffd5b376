// libbsc_b200/csrc/key_cuts.cuh -- what the batched sorters (bwt_encode_batched.cu, st_encode_batched.cu) share: cutting the keys of a
// "segment" into ranges of at most B entries, and order-preserving compaction of the entries a predicate picks.
//
// A segment is a functor with key(i) and pos(i) for its entries i = 0..cnt-1.  Its keys (KB significant bits) are cut by a 65536-bin
// histogram of the top 16 key bits, refined by the next 16 bits only inside bins that hold more than B entries, down to the last key
// bit.  A range then holds at most B entries, or is a single key value with more than B of them.
#pragma once
#include "common.cuh"
#include "bwt_rounds.cuh"

#include <vector>

#define CP_THREADS 256
#define CP_ITEMS   8
#define CP_TILE    (CP_THREADS * CP_ITEMS)                // == SC_TILE: the compactions share the tile aggregates and bwt_tile_scan
static_assert(CP_TILE == SC_TILE, "compaction tiles must match the scan tiles");

namespace {

// T[pos..pos+8) as a big-endian word, zero past n.  T need not be aligned or padded.
__device__ __forceinline__ u64 text8(const u8 *T, u32 n, u32 pos)
{
    if ((u64)pos + 16 <= n) {
        const uintptr_t a = (uintptr_t)(T + pos);
        const u64 *W = (const u64 *)(a & ~(uintptr_t)7);  // two aligned words around T[pos..pos+8), inside the allocation
        const u32 sh = (u32)(a & 7) * 8u;
        const u64 v = sh ? ((W[0] >> sh) | (W[1] << (64u - sh))) : W[0];
        return ((u64)__byte_perm((u32)v, 0, 0x0123) << 32) | (u64)__byte_perm((u32)(v >> 32), 0, 0x0123);
    }
    u64 v = 0;
    for (u32 b = 0; b < 8; ++b) v = (v << 8) | ((u64)pos + b < n ? T[pos + b] : 0u);
    return v;
}

// 16-bit digit histogram over the entries whose key matches `pval` under `pmask`
template <class Seg>
__global__ void __launch_bounds__(256) bb_hist16(Seg s, u32 cnt, u64 pmask, u64 pval, int shift, u32 *__restrict__ hist)
{
    for (u32 i0 = blockIdx.x * 256; i0 < cnt; i0 += gridDim.x * 256) {    // whole warps stay in the loop (match_any is warp-collective)
        const u32 i = i0 + threadIdx.x;
        u32 d = 0xffffffffu;
        if (i < cnt) { const u64 k = s.key(i); if ((k & pmask) == pval) d = (u32)(k >> shift) & 0xffffu; }
        const u32 m = __match_any_sync(0xffffffffu, d);
        if (d != 0xffffffffu && (m & lanemask_lt()) == 0) atomicAdd(&hist[d], (u32)__popc(m));
    }
}

// ---- order-preserving compaction: count per tile, bwt_tile_scan, write ----------------------------------------------------------
template <class Pick>
__global__ void __launch_bounds__(CP_THREADS) bb_count(Pick p, u32 cnt, TileAgg *__restrict__ agg)
{
    __shared__ u32 s_cnt[CP_THREADS / 32];
    const u32 base = blockIdx.x * CP_TILE;
    u32 c = 0;
#pragma unroll
    for (int k = 0; k < CP_ITEMS; ++k) { const u32 i = base + k * CP_THREADS + threadIdx.x; if (i < cnt && p.pred(i)) ++c; }
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0) s_cnt[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        u32 t = 0;
        for (int w = 0; w < CP_THREADS / 32; ++w) t += s_cnt[w];
        agg[blockIdx.x] = TileAgg{0, t, 0, 0};
    }
}

template <class Pick>
__global__ void __launch_bounds__(CP_THREADS) bb_write(Pick p, u32 cnt, const TileAgg *__restrict__ agg)
{
    __shared__ u32 s_cnt[CP_THREADS / 32];
    const u32 base = blockIdx.x * CP_TILE, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    u32 run = agg[blockIdx.x].active;                   // exclusive prefix of this tile
    for (int k = 0; k < CP_ITEMS; ++k) {
        const u32 i = base + k * CP_THREADS + threadIdx.x;
        const bool f = i < cnt && p.pred(i);
        const u32 b = __ballot_sync(0xffffffffu, f);
        if (lane == 0) s_cnt[warp] = __popc(b);
        __syncthreads();
        u32 off = run, tot = 0;
        for (u32 w = 0; w < CP_THREADS / 32; ++w) { const u32 c = s_cnt[w]; if (w < warp) off += c; tot += c; }
        if (f) p.emit(i, off + __popc(b & lanemask_lt()));
        run += tot;
        __syncthreads();
    }
}

// the entries of a segment whose key lies in [lo, hi], into the batch buffers
template <class Seg> struct PickRange {
    Seg s; u64 lo, hi; u64 *k; u32 *v;
    __device__ __forceinline__ bool pred(u32 i) const { const u64 x = s.key(i); return x >= lo && x <= hi; }
    __device__ __forceinline__ void emit(u32 i, u32 x) const { k[x] = s.key(i); v[x] = s.pos(i); }
};

// keys [lo, hi] holding `count` entries, the first of which is entry `cum` of the segment in key order
struct Range { u64 lo, hi; u32 count, cum; };

struct KeyCuts {
    Ctx *ctx; u32 B;
    u32 *hist;                                           // 65536 bins
    TileAgg *agg;                                        // one per compaction tile of the largest segment
    std::vector<u32> h_hist;

    u32 grid_for(u32 cnt) const { return min(ceil_div(cnt, 256), device_sms(ctx->device) * 8); }

    // ordered compaction of `cnt` entries; returns how many were picked
    template <class Pick> u32 compact(const Pick &p, u32 cnt) {
        const u32 tiles = ceil_div(cnt, CP_TILE);
        LAUNCH(ctx, bb_count<Pick>, tiles, CP_THREADS, 0, p, cnt, agg);
        LAUNCH(ctx, bwt_tile_scan, 1, 1024, 0, agg, tiles, ctx->d_mail);
        LAUNCH(ctx, bb_write<Pick>, tiles, CP_THREADS, 0, p, cnt, (const TileAgg *)agg);
        ctx->fetch_mail(1);
        return ctx->h_mail[0];
    }

    // Cut the keys of a segment (KB significant bits) into ranges of at most B entries, or single values.  Below the top 16 key bits
    // a level takes the next 16, or what is left of the KB (8 bits when KB is 24, 40 or 56): its digit then also holds low prefix
    // bits, which equal pval's there, so OR-ing it into pval still gives the bin's keys.
    template <class Seg> void plan(const Seg &s, u32 cnt, int KB, u64 pval, int plen, std::vector<Range> &R, Range &run, u32 &cum) {
        const int shift = KB - plen > 16 ? KB - plen - 16 : 0;
        const u64 pmask = plen ? (~0ull << (KB - plen)) : 0ull;
        CUDA_TRY(cudaMemsetAsync(hist, 0, 65536 * sizeof(u32), ctx->stream));
        LAUNCH(ctx, bb_hist16<Seg>, grid_for(cnt), 256, 0, s, cnt, pmask, pval, shift, hist);
        CUDA_TRY(cudaMemcpyAsync(h_hist.data(), hist, 65536 * sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
        ctx->sync();
        const std::vector<u32> h = h_hist;                 // the recursion below reuses h_hist
        for (u32 d = 0; d < 65536; ++d) {
            const u32 c = h[d];
            if (!c) continue;
            const u64 lo = pval | ((u64)d << shift), hi = lo | ((1ull << shift) - 1);
            if (c <= B) {
                if (run.count && run.count + c > B) { R.push_back(run); run.count = 0; }
                if (!run.count) { run.lo = lo; run.cum = cum; }
                run.hi = hi; run.count += c; cum += c;
            } else {
                if (run.count) { R.push_back(run); run.count = 0; }
                if (shift == 0) { R.push_back(Range{lo, lo, c, cum}); cum += c; }
                else plan(s, cnt, KB, lo, plen + 16, R, run, cum);
            }
        }
    }

    // the ranges of a whole segment in key order; false when they do not add up to its entries
    template <class Seg> bool cut(const Seg &s, u32 cnt, int KB, std::vector<Range> &R) {
        Range run{0, 0, 0, 0}; u32 cum = 0;
        plan(s, cnt, KB, 0, 0, R, run, cum);
        if (run.count) R.push_back(run);
        return cum == cnt;
    }
};

}  // namespace
