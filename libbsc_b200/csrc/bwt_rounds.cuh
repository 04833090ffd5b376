// libbsc_b200/csrc/bwt_rounds.cuh -- the kernels that split sorted suffix groups and emit the BWT, shared by the standard
// forward BWT (bwt_encode.cu) and the batched one (bwt_encode_batched.cu).
#pragma once
#include "common.cuh"

#define SC_THREADS 256
#define SC_ITEMS   8
#define SC_TILE    (SC_THREADS * SC_ITEMS)

namespace {

__global__ void __launch_bounds__(256) bwt_gather_key2(const u32 *__restrict__ sa, const u32 *__restrict__ rank, u32 *__restrict__ key2, u32 m, u32 n, u32 h)
{
    u32 t = blockIdx.x * 256 + threadIdx.x;
    if (t >= m) return;
    u64 p = (u64)sa[t] + h;
    key2[t] = p < n ? __ldg(rank + p) : 0u;
}

struct TileAgg { u32 maxhead, active, groups, pad; };

// A tile of SC_TILE slots (+ one neighbour on each side) staged in shared memory with coalesced loads.
// Each thread then works on 8 CONSECUTIVE slots (what the scans want); one pad entry per 8 keeps the
// 64-byte lane stride off the same banks (the unstaged version was measured to be bank-conflict bound).
struct ScTile {
    u64 key[(SC_TILE + 2) + (SC_TILE + 2) / 8 + 1];
    u32 sa[(SC_TILE + 2) + (SC_TILE + 2) / 8 + 1];
    u32 idx[SC_TILE + SC_TILE / 8 + 1];
};
__device__ __forceinline__ u32 sc_pad(u32 i) { return i + (i >> 3); }

// entry j of the staged arrays holds global slot base + j - 1.  IDX: the slots come from idx[] (else slot = index)
template <bool INIT, bool IDX = !INIT>
__device__ __forceinline__ void sc_load(ScTile &S, const u64 *__restrict__ key, const u32 *__restrict__ sa, const u32 *__restrict__ idx, u32 base, u32 m)
{
    for (u32 j = threadIdx.x; j < SC_TILE + 2; j += SC_THREADS) {
        const long long g = (long long)base + j - 1;
        const bool ok = g >= 0 && g < (long long)m;
        S.key[sc_pad(j)] = ok ? key[g] : 0ull;
        S.sa[sc_pad(j)] = ok ? sa[g] : 0u;
    }
    if (IDX) for (u32 j = threadIdx.x; j < SC_TILE; j += SC_THREADS) S.idx[sc_pad(j)] = (base + j < m) ? idx[base + j] : 0u;
    __syncthreads();
}

// per-slot classification shared by the reduce and apply kernels; i = slot index inside the tile
template <bool INIT>
__device__ __forceinline__ void classify(const ScTile &S, u32 i, u32 t, u32 m, u32 n, bool &head, bool &single)
{
    const u64 k = S.key[sc_pad(i + 1)];
    bool h0 = (t == 0) || S.key[sc_pad(i)] != k;
    bool h1 = (t + 1 == m) || S.key[sc_pad(i + 2)] != k;
    if (INIT) {                                          // suffixes shorter than 8 are complete: own group
        if (t > 0 && (u64)S.sa[sc_pad(i)] + 8 > n) h0 = true;
        if ((u64)S.sa[sc_pad(i + 1)] + 8 > n) h1 = true;
    }
    head = h0; single = h0 && h1;
}

template <bool INIT, bool IDX = !INIT>
__global__ void __launch_bounds__(SC_THREADS) bwt_tile_reduce(const u64 *__restrict__ key, const u32 *__restrict__ sa, const u32 *__restrict__ idx,
                                                              u32 m, u32 n, TileAgg *__restrict__ agg)
{
    __shared__ u32 s_max[SC_THREADS / 32], s_act[SC_THREADS / 32], s_grp[SC_THREADS / 32];
    __shared__ ScTile T;
    sc_load<INIT, IDX>(T, key, sa, idx, blockIdx.x * SC_TILE, m);
    u32 base = blockIdx.x * SC_TILE + threadIdx.x * SC_ITEMS;
    u32 mx = 0, act = 0, grp = 0;
#pragma unroll
    for (int i = 0; i < SC_ITEMS; ++i) {
        u32 t = base + i;
        if (t < m) {
            const u32 li = threadIdx.x * SC_ITEMS + i;
            bool head, single; classify<INIT>(T, li, t, m, n, head, single);
            u32 iv = IDX ? T.idx[sc_pad(li)] : t;
            if (head) mx = iv + 1;                       // idx is increasing in t
            act += !single; grp += (head && !single);
        }
    }
    for (int o = 16; o; o >>= 1) { mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o)); act += __shfl_xor_sync(0xffffffffu, act, o); grp += __shfl_xor_sync(0xffffffffu, grp, o); }
    u32 w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) { s_max[w] = mx; s_act[w] = act; s_grp[w] = grp; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int i = 1; i < SC_THREADS / 32; ++i) { mx = max(mx, s_max[i]); act += s_act[i]; grp += s_grp[i]; }
        agg[blockIdx.x] = TileAgg{mx, act, grp, 0};
    }
}

// exclusive scan of the tile aggregates (single CTA), totals -> mailbox[0..1]
__global__ void __launch_bounds__(1024) bwt_tile_scan(TileAgg *agg, u32 tiles, u32 *mail)
{
    __shared__ u32 s_max[32], s_act[32], s_grp[32];
    u32 per = (tiles + 1023) / 1024;
    u32 b = threadIdx.x * per, e = min(b + per, tiles);
    u32 mx = 0, act = 0, grp = 0;
    for (u32 i = b; i < e; ++i) { TileAgg a = agg[i]; mx = max(mx, a.maxhead); act += a.active; grp += a.groups; }
    u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    u32 imx = mx, iact = act, igrp = grp;
    for (int o = 1; o < 32; o <<= 1) {
        u32 a = __shfl_up_sync(0xffffffffu, imx, o), c = __shfl_up_sync(0xffffffffu, iact, o), d = __shfl_up_sync(0xffffffffu, igrp, o);
        if (lane >= (u32)o) { imx = max(imx, a); iact += c; igrp += d; }
    }
    if (lane == 31) { s_max[w] = imx; s_act[w] = iact; s_grp[w] = igrp; }
    __syncthreads();
    u32 pmx = 0, pact = 0, pgrp = 0;
    for (u32 i = 0; i < w; ++i) { pmx = max(pmx, s_max[i]); pact += s_act[i]; pgrp += s_grp[i]; }
    // exclusive prefix for this thread's chunk
    u32 xmx = max(pmx, __shfl_up_sync(0xffffffffu, imx, 1)), xact = pact + iact - act, xgrp = pgrp + igrp - grp;
    if (lane == 0) xmx = pmx;
    for (u32 i = b; i < e; ++i) {
        TileAgg a = agg[i];
        agg[i] = TileAgg{xmx, xact, xgrp, 0};
        xmx = max(xmx, a.maxhead); xact += a.active; xgrp += a.groups;
    }
    if (threadIdx.x == 1023) { mail[0] = pact + iact; mail[1] = pgrp + igrp; }
}

// STAGE: instead of storing rank[sa] directly, write the pair (rank << 32 | sa) of slot t to rank_pairs[t], coalesced through the
// tile's key array; bwt_encode.cu partitions the pairs by position window and stores them with bwt_stage_scatter.
template <bool INIT, bool IDX = !INIT, bool STAGE = false>
__global__ void __launch_bounds__(SC_THREADS) bwt_apply(const u64 *__restrict__ key, const u32 *__restrict__ sa, const u32 *__restrict__ idx,
                                                        u32 m, u32 n, const TileAgg *__restrict__ agg, u32 *__restrict__ rank,
                                                        u32 *__restrict__ sa_out, u32 *__restrict__ idx_out, u32 *__restrict__ grp_out,
                                                        u64 *__restrict__ rank_pairs = nullptr)
{
    __shared__ u32 s_max[SC_THREADS / 32], s_act[SC_THREADS / 32], s_grp[SC_THREADS / 32];
    __shared__ ScTile T;
    sc_load<INIT, IDX>(T, key, sa, idx, blockIdx.x * SC_TILE, m);
    const u32 base = blockIdx.x * SC_TILE + threadIdx.x * SC_ITEMS;
    const u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    bool head[SC_ITEMS], single[SC_ITEMS]; u32 iv[SC_ITEMS], sv[SC_ITEMS];
    u32 mx = 0, act = 0, grp = 0;
#pragma unroll
    for (int i = 0; i < SC_ITEMS; ++i) {
        u32 t = base + i; head[i] = false; single[i] = true; iv[i] = 0; sv[i] = 0;
        if (t < m) {
            const u32 li = threadIdx.x * SC_ITEMS + i;
            classify<INIT>(T, li, t, m, n, head[i], single[i]);
            iv[i] = IDX ? T.idx[sc_pad(li)] : t; sv[i] = T.sa[sc_pad(li + 1)];
            if (head[i]) mx = iv[i] + 1;
            act += !single[i]; grp += (head[i] && !single[i]);
        }
    }
    u32 imx = mx, iact = act, igrp = grp;
    for (int o = 1; o < 32; o <<= 1) {
        u32 a = __shfl_up_sync(0xffffffffu, imx, o), c = __shfl_up_sync(0xffffffffu, iact, o), d = __shfl_up_sync(0xffffffffu, igrp, o);
        if (lane >= (u32)o) { imx = max(imx, a); iact += c; igrp += d; }
    }
    if (lane == 31) { s_max[w] = imx; s_act[w] = iact; s_grp[w] = igrp; }
    __syncthreads();
    TileAgg carry = agg[blockIdx.x];
    u32 pmx = carry.maxhead, pact = carry.active, pgrp = carry.groups;
    for (u32 i = 0; i < w; ++i) { pmx = max(pmx, s_max[i]); pact += s_act[i]; pgrp += s_grp[i]; }
    u32 up = __shfl_up_sync(0xffffffffu, imx, 1);
    u32 xmx = lane == 0 ? pmx : max(pmx, up), xact = pact + iact - act, xgrp = pgrp + igrp - grp;
#pragma unroll
    for (int i = 0; i < SC_ITEMS; ++i) {
        u32 t = base + i;
        if (t < m) {
            if (head[i]) { xmx = iv[i] + 1; if (!single[i]) xgrp++; }
            if (STAGE) T.key[sc_pad(threadIdx.x * SC_ITEMS + i)] = ((u64)xmx << 32) | sv[i];   // T.key was last read before the barrier above
            else       rank[sv[i]] = xmx;                // = 1 + SA slot of the group head
            if (!single[i]) { sa_out[xact] = sv[i]; idx_out[xact] = iv[i]; grp_out[xact] = xgrp - 1; xact++; }
        }
    }
    if (STAGE) {
        __syncthreads();
        const u32 tbase = blockIdx.x * SC_TILE;
        for (u32 j = threadIdx.x; j < SC_TILE && tbase + j < m; j += SC_THREADS) rank_pairs[tbase + j] = T.key[sc_pad(j)];
    }
}

// L, primary index and secondary indexes from the final ranks (Appendix B.1 of SURVEY.md)
// STAGE: row 0 is stored here; the other rows go as pairs (byte << 32 | row) to L_pairs[i - 1], for bwt_stage_scatter.
template <bool STAGE = false>
__global__ void __launch_bounds__(256) bwt_emit(const u8 *__restrict__ T, const u32 *__restrict__ rank, u8 *__restrict__ L, u32 n,
                                                u64 *__restrict__ L_pairs = nullptr)
{
    u32 i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    u32 p = __ldg(rank) - 1;                             // SA slot of suffix 0
    if (i == 0) { L[0] = T[n - 1]; return; }
    u32 j = rank[i] - 1;
    if (STAGE) L_pairs[i - 1] = ((u64)T[i - 1] << 32) | (j < p ? j + 1 : j);
    else       L[j < p ? j + 1 : j] = T[i - 1];
}

__global__ void bwt_emit_indexes(const u32 *__restrict__ rank, u32 n, u32 r, u32 count, u32 *mail)
{
    u32 t = threadIdx.x;
    if (t == 0) mail[0] = rank[0];                       // primary index = ISA[0] + 1
    if (t < count) mail[1 + t] = rank[(size_t)(t + 1) * r] - 1;
}

}  // namespace
