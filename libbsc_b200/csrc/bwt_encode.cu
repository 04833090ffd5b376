// libbsc_b200/csrc/bwt_encode.cu -- forward Burrows-Wheeler transform on the device.
//
// Replaces bsc_bwt_encode's sorters (libbsc/bwt/bwt.cpp:178-231: libsais on the CPU,
// libcubwt_bwt_aux on the GPU, libcubwt.cu:2031-2223).  Same result by construction: the BWT,
// the primary index and the secondary indexes are pure functions of the suffix order
// (SURVEY.md 7.2 / Appendix B.1), and any correct suffix sorter yields that order.
//
// Algorithm (prefix doubling, all of it radix passes + scans; no DC3, no segmented sort):
//   1. ONE 8-pass onesweep radix sort of all n suffixes by their first 8 bytes (keys are
//      synthesised from the text inside the sort, never materialised).  Suffixes are fed in
//      descending position order so that among equal zero-padded keys the shorter suffix comes
//      first, which is the "sentinel is smallest" rule.
//   2. rank[i] = 1 + SA slot of the head of suffix i's group.  Groups of size 1 are final.
//   3. While unsorted groups remain (depth h = 8, 16, 32, ...): for the still-active suffixes
//      only, key2 = rank[i+h] (0 = ran off the end); radix sort (dense group id, key2) pairs;
//      re-split groups, scatter the new ranks, compact away the newly unique suffixes.
//   4. Emit L, the primary index and the secondary indexes straight from rank[].
//
// All intermediate arrays live in the Ctx arena (about 53 n bytes).
#include "radix_sort.cuh"
#include "stages.cuh"

#define SC_THREADS 256
#define SC_ITEMS   8
#define SC_TILE    (SC_THREADS * SC_ITEMS)

namespace {

// keys of the initial sort: element e <-> text position n-1-e
struct SrcTextDesc {
    const u8 *T; u32 n;
    __device__ __forceinline__ u64 key(u32 e) const { return load_be64(T, n - 1 - e); }
    __device__ __forceinline__ u32 val(u32 e) const { return n - 1 - e; }
};

// keys of a refinement round
struct SrcRound {
    const u32 *grp, *key2, *sa;
    __device__ __forceinline__ u64 key(u32 e) const { return ((u64)grp[e] << 32) | key2[e]; }
    __device__ __forceinline__ u32 val(u32 e) const { return sa[e]; }
};

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

// entry j of the staged arrays holds global slot base + j - 1
template <bool INIT>
__device__ __forceinline__ void sc_load(ScTile &S, const u64 *__restrict__ key, const u32 *__restrict__ sa, const u32 *__restrict__ idx, u32 base, u32 m)
{
    for (u32 j = threadIdx.x; j < SC_TILE + 2; j += SC_THREADS) {
        const long long g = (long long)base + j - 1;
        const bool ok = g >= 0 && g < (long long)m;
        S.key[sc_pad(j)] = ok ? key[g] : 0ull;
        S.sa[sc_pad(j)] = ok ? sa[g] : 0u;
    }
    if (!INIT) for (u32 j = threadIdx.x; j < SC_TILE; j += SC_THREADS) S.idx[sc_pad(j)] = (base + j < m) ? idx[base + j] : 0u;
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

template <bool INIT>
__global__ void __launch_bounds__(SC_THREADS) bwt_tile_reduce(const u64 *__restrict__ key, const u32 *__restrict__ sa, const u32 *__restrict__ idx,
                                                              u32 m, u32 n, TileAgg *__restrict__ agg)
{
    __shared__ u32 s_max[SC_THREADS / 32], s_act[SC_THREADS / 32], s_grp[SC_THREADS / 32];
    __shared__ ScTile T;
    sc_load<INIT>(T, key, sa, idx, blockIdx.x * SC_TILE, m);
    u32 base = blockIdx.x * SC_TILE + threadIdx.x * SC_ITEMS;
    u32 mx = 0, act = 0, grp = 0;
#pragma unroll
    for (int i = 0; i < SC_ITEMS; ++i) {
        u32 t = base + i;
        if (t < m) {
            const u32 li = threadIdx.x * SC_ITEMS + i;
            bool head, single; classify<INIT>(T, li, t, m, n, head, single);
            u32 iv = INIT ? t : T.idx[sc_pad(li)];
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

template <bool INIT>
__global__ void __launch_bounds__(SC_THREADS) bwt_apply(const u64 *__restrict__ key, const u32 *__restrict__ sa, const u32 *__restrict__ idx,
                                                        u32 m, u32 n, const TileAgg *__restrict__ agg, u32 *__restrict__ rank,
                                                        u32 *__restrict__ sa_out, u32 *__restrict__ idx_out, u32 *__restrict__ grp_out)
{
    __shared__ u32 s_max[SC_THREADS / 32], s_act[SC_THREADS / 32], s_grp[SC_THREADS / 32];
    __shared__ ScTile T;
    sc_load<INIT>(T, key, sa, idx, blockIdx.x * SC_TILE, m);
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
            iv[i] = INIT ? t : T.idx[sc_pad(li)]; sv[i] = T.sa[sc_pad(li + 1)];
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
            rank[sv[i]] = xmx;                           // = 1 + SA slot of the group head
            if (!single[i]) { sa_out[xact] = sv[i]; idx_out[xact] = iv[i]; grp_out[xact] = xgrp - 1; xact++; }
        }
    }
}

// L, primary index and secondary indexes from the final ranks (Appendix B.1 of SURVEY.md)
__global__ void __launch_bounds__(256) bwt_emit(const u8 *__restrict__ T, const u32 *__restrict__ rank, u8 *__restrict__ L, u32 n)
{
    u32 i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    u32 p = __ldg(rank) - 1;                             // SA slot of suffix 0
    if (i == 0) { L[0] = T[n - 1]; return; }
    u32 j = rank[i] - 1;
    L[j < p ? j + 1 : j] = T[i - 1];
}

__global__ void bwt_emit_indexes(const u32 *__restrict__ rank, u32 n, u32 r, u32 count, u32 *mail)
{
    u32 t = threadIdx.x;
    if (t == 0) mail[0] = rank[0];                       // primary index = ISA[0] + 1
    if (t < count) mail[1 + t] = rank[(size_t)(t + 1) * r] - 1;
}

}  // namespace

// Forward BWT of d_T[0..n) (device, in place).  Returns the primary index (>= 1) or an error.
// If indexes != NULL also reports the secondary indexes exactly as bwt.cpp:127-131 does.
int stage_bwt_encode(Ctx *ctx, u8 *d_T, int n_, unsigned char *num_indexes, int *indexes)
{
    if (n_ < 0) return LIBBSC_BAD_PARAMETER;
    const bool want_aux = (num_indexes != nullptr && indexes != nullptr);
    u32 r = 0;
    if (want_aux) {
        int mod = n_ / 8;
        mod |= mod >> 1; mod |= mod >> 2; mod |= mod >> 4; mod |= mod >> 8; mod |= mod >> 16; mod >>= 1;
        r = (u32)mod + 1;
        if (r < 2) return LIBBSC_BAD_PARAMETER;          // libsais.c:6869 (r must be a power of two >= 2)
    }
    if (n_ <= 1) return n_;                              // libsais.c:6845-6850
    const u32 n = (u32)n_;

    Arena &A = ctx->sort_arena();
    const size_t mark = A.mark();
    u8  *Tp      = A.get<u8>((size_t)n + 32);
    u64 *k[2]    = { A.get<u64>(n), A.get<u64>(n) };
    u32 *v[2]    = { A.get<u32>(n), A.get<u32>(n) };
    u32 *rank    = A.get<u32>((size_t)n + 1);
    u32 *sa_act  = A.get<u32>(n);
    u32 *idx[2]  = { A.get<u32>(n), A.get<u32>(n) };
    u32 *grp     = A.get<u32>(n);
    u32 *key2    = A.get<u32>(n);
    const u32 sc_tiles_max = ceil_div(n, SC_TILE);
    TileAgg *agg = A.get<TileAgg>(sc_tiles_max);
    void *scratch = A.get<u8>(rs_scratch_bytes(n, RS_MAX_PASSES));

    CUDA_TRY(cudaMemcpyAsync(Tp, d_T, n, cudaMemcpyDeviceToDevice, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(Tp + n, 0, 32, ctx->stream));

    // 1. initial sort by the first 8 bytes
    DigitPasses p8 = make_passes(0, 64);
    int cur = rs_sort<u64, true>(ctx, SrcTextDesc{Tp, n}, k, v, n, p8, scratch);

    // 2. first split
    u32 m = n, tiles = ceil_div(m, SC_TILE);
    LAUNCH(ctx, bwt_tile_reduce<true>, tiles, SC_THREADS, 0, k[cur], v[cur], (const u32 *)nullptr, m, n, agg);
    LAUNCH(ctx, bwt_tile_scan, 1, 1024, 0, agg, tiles, ctx->d_mail);
    int ib = 0;
    LAUNCH(ctx, bwt_apply<true>, tiles, SC_THREADS, 0, k[cur], v[cur], (const u32 *)nullptr, m, n, agg, rank, sa_act, idx[ib], grp);
    ctx->fetch_mail(2);
    m = ctx->h_mail[0]; u32 G = ctx->h_mail[1];

    // 3. doubling rounds
    const int bits_k2 = bits_for(n);
    for (u64 h = 8; m > 0; h <<= 1) {
        if (h >= ((u64)1 << 31)) { A.release(mark); return LIBBSC_GPU_ERROR; }   // cannot happen for n <= 2^30
        LAUNCH(ctx, bwt_gather_key2, ceil_div(m, 256), 256, 0, sa_act, rank, key2, m, n, (u32)h);
        DigitPasses pr = make_passes(0, bits_k2, 32, 32 + (G > 1 ? bits_for(G - 1) : 0));
        cur = rs_sort<u64, true>(ctx, SrcRound{grp, key2, sa_act}, k, v, m, pr, scratch);
        tiles = ceil_div(m, SC_TILE);
        LAUNCH(ctx, bwt_tile_reduce<false>, tiles, SC_THREADS, 0, k[cur], v[cur], idx[ib], m, n, agg);
        LAUNCH(ctx, bwt_tile_scan, 1, 1024, 0, agg, tiles, ctx->d_mail);
        LAUNCH(ctx, bwt_apply<false>, tiles, SC_THREADS, 0, k[cur], v[cur], idx[ib], m, n, agg, rank, sa_act, idx[ib ^ 1], grp);
        ib ^= 1;
        ctx->fetch_mail(2);
        m = ctx->h_mail[0]; G = ctx->h_mail[1];
    }

    // 4. emit
    LAUNCH(ctx, bwt_emit, ceil_div(n, 256), 256, 0, Tp, rank, d_T, n);
    u32 cnt = want_aux ? (n - 1) / r : 0;
    LAUNCH(ctx, bwt_emit_indexes, 1, 256, 0, rank, n, r ? r : 1u, cnt, ctx->d_mail);
    ctx->fetch_mail(1 + (int)cnt);
    int index = (int)ctx->h_mail[0];
    if (want_aux) {
        *num_indexes = (unsigned char)cnt;
        for (u32 t = 0; t < cnt; ++t) indexes[t] = (int)ctx->h_mail[1 + t];
    }
    A.release(mark);
    return index;
}
