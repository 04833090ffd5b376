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
#include "bwt_rounds.cuh"

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
        if (h >= ((u64)1 << 31)) { A.release(mark); return LIBBSC_GPU_ERROR; }   // cannot happen for n < 2^31: no group survives h >= n, so the last round needed is h = 2^30
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
