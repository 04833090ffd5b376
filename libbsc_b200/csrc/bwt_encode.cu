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
// Segmented rounds (BSCB200_BWT_SEG = S, default 256; 0 = off).  Each group already occupies a contiguous range of the round's
// slots and only needs ordering by key2 inside it, so step 3's global sort over (group, key2) can be split by group size:
//   - groups of at most S entries are sorted inside one CTA (bwt_seg_sort): a CTA owns the groups that START in its
//     SEG_TILE slots, loads them whole (at most SEG_TILE - 1 + S <= SEG_CAP entries) into shared memory, places each
//     entry by counting the smaller key2 of its group and writes it to its slot -- one read and one write instead of up to 8
//     radix passes;
//   - the larger groups are compacted (bwt_seg_compact), radix-sorted by (dense large-group id, key2) -- fewer group bits
//     than the dense id over all groups -- and written back to their slot ranges (bwt_seg_scatter).
// The result is the array the global sort gives, up to the order of equal (group, key2) entries, which the split does not
// see: it gives them one rank.  So L and the indexes are unchanged.  The group starts live in idx[ib ^ 1] (free until
// bwt_apply writes it) and the large entries in k[] / v[], so the arena is the same size.
// On a 64 MiB text block S = 256 takes the forward BWT from 37.4 to 35.4 ms (DESIGN 4.2): larger S spend more on counting
// inside large groups than they save in radix passes, smaller ones leave more entries to the radix sort.
//
// Staged rank and L stores (BSCB200_BWT_STAGE: 0 = direct, 1 = staged, unset = by size, stage_on).  rank[sa] = value in bwt_apply
// and L[row] = byte in bwt_emit are random stores into arrays larger than the L2; each one leaves a sector partly written.  Staged,
// the kernels write (value << 32 | position) pairs in slot order instead, one keys-only radix pass partitions them by the top 8
// position bits, and bwt_stage_scatter stores them in that order: the resident CTAs then write into a few windows at a time, whose
// sectors the L2 merges whole.  The pairs of a split go to k[cur ^ 1] (idle during bwt_apply) and are partitioned into k[cur] (dead
// once bwt_apply has read it); those of the emit use k[1] and k[0].  So the arena is unchanged.  A 64 MiB text block, every store
// staged: 36.4 -> 28.8 ms.
//
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

#define SEG_TILE    1024                              // slots whose groups one bwt_seg_sort CTA owns
#define SEG_CAP     2048                              // entries it can hold: SEG_TILE - 1 + S for the largest S
#define SEG_MAX     (SEG_CAP - SEG_TILE)
#define SEG_DEFAULT 256                               // measured best of 64 / 256 / 1024 on a 64 MiB text block (DESIGN 4.2)

// the group-size bound of the segmented rounds (0: every group goes through the global radix sort), read once per process
static u32 bwt_seg_limit()
{
    static const u32 v = [] { const char *e = getenv("BSCB200_BWT_SEG"); const int k = e ? atoi(e) : SEG_DEFAULT; return (u32)(k < 0 ? 0 : k > SEG_MAX ? SEG_MAX : k); }();
    return v;
}

// gstart[g] = first slot of group g, gstart[G] = m (grp[] is dense and ascending in slot order)
__global__ void __launch_bounds__(256) bwt_seg_starts(const u32 *__restrict__ grp, u32 *__restrict__ gstart, u32 m, u32 G)
{
    const u32 t = blockIdx.x * 256 + threadIdx.x;
    if (t >= m) return;
    const u32 g = grp[t];
    if (t == 0 || grp[t - 1] != g) gstart[g] = t;
    if (t == 0) gstart[G] = m;
}

// The entries of groups of more than S entries, per SC_TILE slots (warp w takes slots w*256 + 32 i + lane, which keeps slot order).
//   SEG_COUNT:   tile totals of large entries and large groups -> agg (then bwt_tile_scan makes them exclusive prefixes)
//   SEG_COMPACT: large entry number e <- ((dense large-group id) << 32 | key2, sa)
//   SEG_SCATTER: slot t <- (grp << 32 | key2 of sorted entry e, its sa)
enum { SEG_COUNT, SEG_COMPACT, SEG_SCATTER };
template <int MODE>
__global__ void __launch_bounds__(SC_THREADS) bwt_seg_large(const u32 *__restrict__ grp, const u32 *__restrict__ key2, const u32 *__restrict__ sa,
                                                            const u32 *__restrict__ gstart, u32 m, u32 S, TileAgg *__restrict__ agg,
                                                            const u64 *__restrict__ kin, const u32 *__restrict__ vin, u64 *__restrict__ kout, u32 *__restrict__ vout)
{
    __shared__ u32 s_cnt[SC_THREADS / 32], s_hd[SC_THREADS / 32];
    const u32 lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const u32 base = blockIdx.x * SC_TILE + w * (32 * SC_ITEMS) + lane;
    u32 g[SC_ITEMS], big[SC_ITEMS], head[SC_ITEMS], cnt = 0, hds = 0;
#pragma unroll
    for (int i = 0; i < SC_ITEMS; ++i) {
        const u32 t = base + 32 * i;
        bool L = false, H = false;
        g[i] = 0;
        if (t < m) { g[i] = grp[t]; const u32 s0 = gstart[g[i]]; L = gstart[g[i] + 1] - s0 > S; H = s0 == t; }
        big[i] = __ballot_sync(0xffffffffu, L); head[i] = __ballot_sync(0xffffffffu, L && H);
        cnt += __popc(big[i]); hds += __popc(head[i]);
    }
    if (lane == 0) { s_cnt[w] = cnt; s_hd[w] = hds; }
    __syncthreads();
    if (MODE == SEG_COUNT) {
        if (threadIdx.x == 0) {
            for (int i = 1; i < SC_THREADS / 32; ++i) { cnt += s_cnt[i]; hds += s_hd[i]; }
            agg[blockIdx.x] = TileAgg{0, cnt, hds, 0};
        }
        return;
    }
    const TileAgg carry = agg[blockIdx.x];
    u32 e = carry.active, lid = carry.groups;
    for (u32 i = 0; i < w; ++i) { e += s_cnt[i]; lid += s_hd[i]; }
    const u32 lt = lanemask_lt(), le = lt | (1u << lane);
#pragma unroll
    for (int i = 0; i < SC_ITEMS; ++i) {
        const u32 t = base + 32 * i;
        if ((big[i] >> lane) & 1u) {
            const u32 my = e + __popc(big[i] & lt);
            if (MODE == SEG_COMPACT) { kout[my] = ((u64)(lid + __popc(head[i] & le) - 1) << 32) | key2[t]; vout[my] = sa[t]; }
            else                     { kout[t] = ((u64)g[i] << 32) | (u32)kin[my]; vout[t] = vin[my]; }
        }
        e += __popc(big[i]); lid += __popc(head[i]);
    }
}

// The groups of at most S entries that start in slots [blockIdx.x * SEG_TILE, + SEG_TILE): loaded whole (a group of more than S
// entries at the end is left out; one in the middle is loaded but skipped) into shared memory.  Each entry's place in its group is
// the number of entries of the group with a smaller key2, or an equal one at a smaller slot: a count over the group, which the warp
// reads as broadcasts.  That costs s steps per entry of a group of s, far fewer than a sorting network over the CTA's 2048 entries
// for the small groups that hold most entries.  16 KB of shared memory, so a CTA fits next to the coder CTAs of the pipeline.
__global__ void __launch_bounds__(256) bwt_seg_sort(const u32 *__restrict__ grp, const u32 *__restrict__ key2, const u32 *__restrict__ sa,
                                                    const u32 *__restrict__ gstart, u32 m, u32 S, u64 *__restrict__ kout, u32 *__restrict__ vout)
{
    __shared__ u32 sk[SEG_CAP];
    __shared__ u32 sv[SEG_CAP];
    __shared__ u32 s_a, s_b;
    const u32 tid = threadIdx.x, base = blockIdx.x * SEG_TILE, end = min(base + SEG_TILE, m);
    if (tid == 0) {
        const u32 g0 = grp[base];
        const u32 a = gstart[g0] == base ? base : gstart[g0 + 1];
        u32 b = a;
        if (a < end) {
            const u32 g1 = grp[end - 1], s1 = gstart[g1];
            b = gstart[g1 + 1];
            if (b - s1 > S) b = s1;
        }
        s_a = a; s_b = max(a, b);
    }
    __syncthreads();
    const u32 a = s_a, len = s_b - a;
    if (len == 0) return;
    for (u32 j = tid; j < len; j += 256) { sk[j] = key2[a + j]; sv[j] = sa[a + j]; }
    __syncthreads();
    for (u32 j = tid; j < len; j += 256) {
        const u32 g = grp[a + j], gs = gstart[g], ge = gstart[g + 1];
        if (ge - gs > S) continue;
        const u32 my = sk[j], lo = gs - a, hi = ge - a;
        u32 pos = 0;
        for (u32 i = lo; i < hi; ++i) { const u32 x = sk[i]; pos += (x < my) | ((x == my) & (i < j)); }
        kout[gs + pos] = ((u64)g << 32) | my;
        vout[gs + pos] = sv[j];
    }
}

// dst[pos] = value for the pairs (value << 32 | pos), read in order: after the partition by window, the stores of the resident CTAs
// fall into a few windows, whose sectors the L2 fills completely before it writes them back
template <typename T>
__global__ void __launch_bounds__(256) bwt_stage_scatter(const u64 *__restrict__ pairs, T *__restrict__ dst, u32 cnt)
{
    const u32 t = blockIdx.x * 256 + threadIdx.x;
    if (t >= cnt) return;
    const u64 p = pairs[t];
    dst[(u32)p] = (T)(p >> 32);
}

// Staged scatter: the pairs (value << 32 | pos) in pairs[0..cnt), with every pos < 2^pos_bits, are partitioned by the top 8 bits of
// pos (one keys-only radix pass, stable, into `parted`), then stored window after window.  The stores land where the direct
// scatter puts them; only their order changes.
template <typename T>
static void bwt_stage_store(Ctx *ctx, const char *name, const u64 *pairs, u64 *parted, u32 cnt, int pos_bits, T *dst, void *scratch)
{
    u64 *const kk[2] = { parted, parted };              // one pass: it writes kk[0] only
    u32 *const vv[2] = { nullptr, nullptr };
    rs_sort<u64, false>(ctx, SrcArray<u64, false>{pairs, nullptr}, kk, vv, cnt, make_passes(pos_bits > 8 ? pos_bits - 8 : 0, pos_bits), scratch,
                        "bwt_stage_part");
    LAUNCH_NAMED(ctx, name, bwt_stage_scatter<T>, ceil_div(cnt, 256), 256, 0, parted, dst, cnt);
}

// Measured on an H100 (DESIGN 4.2): staged wins for 7.9 M entries and up, loses at 0.45 M; it loses on an L of 25 MiB (which the
// 50 MB L2 holds) and wins on one of 64 MiB and on rank arrays of 100 and 256 MiB.
#define STAGE_MIN_ENTRIES (1u << 22)
#define STAGE_MIN_BYTES   ((size_t)50000000)

// BSCB200_BWT_STAGE: 0 = every rank and L store direct, 1 = every one staged, unset = by size (stage_on); read once per process
static int bwt_stage_switch()
{
    static const int v = [] { const char *e = getenv("BSCB200_BWT_STAGE"); return e && (e[0] == '0' || e[0] == '1') ? e[0] - '0' : -1; }();
    return v;
}

// staged or direct store of cnt entries into an array of `bytes`
static bool stage_on(u32 cnt, size_t bytes)
{
    const int s = bwt_stage_switch();
    return s >= 0 ? s == 1 : (cnt >= STAGE_MIN_ENTRIES && bytes > STAGE_MIN_BYTES);
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
    // the pairs of a staged rank store go to k[cur ^ 1], idle during bwt_apply, and are partitioned into k[cur], dead once it has run
    const int pos_bits = bits_for(n - 1);
    if (stage_on(m, (size_t)4 * n)) {
        LAUNCH_NAMED(ctx, "bwt_apply_staged", (bwt_apply<true, false, true>), tiles, SC_THREADS, 0, k[cur], v[cur], (const u32 *)nullptr, m, n, agg,
                     rank, sa_act, idx[ib], grp, k[cur ^ 1]);
        bwt_stage_store(ctx, "bwt_stage_rank", k[cur ^ 1], k[cur], m, pos_bits, rank, scratch);
    } else {
        LAUNCH(ctx, bwt_apply<true>, tiles, SC_THREADS, 0, k[cur], v[cur], (const u32 *)nullptr, m, n, agg, rank, sa_act, idx[ib], grp);
    }
    ctx->fetch_mail(2);
    m = ctx->h_mail[0]; u32 G = ctx->h_mail[1];

    // 3. doubling rounds
    const int bits_k2 = bits_for(n);
    const u32 S = bwt_seg_limit();
    for (u64 h = 8; m > 0; h <<= 1) {
        if (h >= ((u64)1 << 31)) { A.release(mark); return LIBBSC_GPU_ERROR; }   // cannot happen for n < 2^31: no group survives h >= n, so the last round needed is h = 2^30
        LAUNCH(ctx, bwt_gather_key2, ceil_div(m, 256), 256, 0, sa_act, rank, key2, m, n, (u32)h);
        if (S == 0) {
            DigitPasses pr = make_passes(0, bits_k2, 32, 32 + (G > 1 ? bits_for(G - 1) : 0));
            cur = rs_sort<u64, true>(ctx, SrcRound{grp, key2, sa_act}, k, v, m, pr, scratch);
        } else {
            u32 *gstart = idx[ib ^ 1];                   // G + 1 <= m / 2 + 1 words; bwt_apply writes idx[ib ^ 1] only after the sort
            LAUNCH(ctx, bwt_seg_starts, ceil_div(m, 256), 256, 0, grp, gstart, m, G);
            tiles = ceil_div(m, SC_TILE);
            LAUNCH_NAMED(ctx, "bwt_seg_count", bwt_seg_large<SEG_COUNT>, tiles, SC_THREADS, 0, grp, key2, sa_act, gstart, m, S, agg,
                         (const u64 *)nullptr, (const u32 *)nullptr, (u64 *)nullptr, (u32 *)nullptr);
            LAUNCH(ctx, bwt_tile_scan, 1, 1024, 0, agg, tiles, ctx->d_mail);
            ctx->fetch_mail(2);
            const u32 ml = ctx->h_mail[0], nl = ctx->h_mail[1];   // entries and number of the groups of more than S entries
            cur = 0;
            if (ml > 0) {
                LAUNCH_NAMED(ctx, "bwt_seg_compact", bwt_seg_large<SEG_COMPACT>, tiles, SC_THREADS, 0, grp, key2, sa_act, gstart, m, S, agg,
                             (const u64 *)nullptr, (const u32 *)nullptr, k[1], v[1]);
                DigitPasses pl = make_passes(0, bits_k2, 32, 32 + (nl > 1 ? bits_for(nl - 1) : 0));
                const int c = rs_sort<u64, true>(ctx, SrcArray<u64, true>{k[1], v[1]}, k, v, ml, pl, scratch);   // pass 0 reads k[1] before pass 1 writes it
                cur = c ^ 1;
                LAUNCH_NAMED(ctx, "bwt_seg_scatter", bwt_seg_large<SEG_SCATTER>, tiles, SC_THREADS, 0, grp, key2, sa_act, gstart, m, S, agg,
                             (const u64 *)k[c], (const u32 *)v[c], k[cur], v[cur]);
            }
            if (ml < m) LAUNCH(ctx, bwt_seg_sort, ceil_div(m, SEG_TILE), 256, 0, grp, key2, sa_act, gstart, m, S, k[cur], v[cur]);
        }
        tiles = ceil_div(m, SC_TILE);
        LAUNCH(ctx, bwt_tile_reduce<false>, tiles, SC_THREADS, 0, k[cur], v[cur], idx[ib], m, n, agg);
        LAUNCH(ctx, bwt_tile_scan, 1, 1024, 0, agg, tiles, ctx->d_mail);
        if (stage_on(m, (size_t)4 * n)) {
            LAUNCH_NAMED(ctx, "bwt_apply_staged", (bwt_apply<false, true, true>), tiles, SC_THREADS, 0, k[cur], v[cur], idx[ib], m, n, agg,
                         rank, sa_act, idx[ib ^ 1], grp, k[cur ^ 1]);
            bwt_stage_store(ctx, "bwt_stage_rank", k[cur ^ 1], k[cur], m, pos_bits, rank, scratch);
        } else {
            LAUNCH(ctx, bwt_apply<false>, tiles, SC_THREADS, 0, k[cur], v[cur], idx[ib], m, n, agg, rank, sa_act, idx[ib ^ 1], grp);
        }
        ib ^= 1;
        ctx->fetch_mail(2);
        m = ctx->h_mail[0]; G = ctx->h_mail[1];
    }

    // 4. emit (every k / v buffer is free now)
    if (stage_on(n - 1, n)) {
        LAUNCH_NAMED(ctx, "bwt_emit_staged", bwt_emit<true>, ceil_div(n, 256), 256, 0, Tp, rank, d_T, n, k[1]);
        bwt_stage_store(ctx, "bwt_stage_L", k[1], k[0], n - 1, pos_bits, d_T, scratch);
    } else {
        LAUNCH(ctx, bwt_emit, ceil_div(n, 256), 256, 0, Tp, rank, d_T, n);
    }
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
