// libbsc_b200/csrc/radix_sort.cuh -- device-wide stable LSD radix sort, "onesweep" style.
//
// This is the workhorse of the forward BWT (prefix-doubling suffix sort) and of ST-k.  It replaces
// the reference's cub::DeviceRadixSort / DeviceSegmentedSort calls (libcubwt.cu:713-739,
// 1686-1703, 2136-2163; st.cu:187-193, 273-279) with our own kernels:
//
//   rs_hist1      : 256-bin histogram of the FIRST digit only (one read of the source keys).
//   rs_onesweep   : per digit pass, ONE read + ONE write of every (key,value): each CTA scans the
//                   digit histogram into global bases, ranks a tile with warp match-any multisplit,
//                   obtains its per-digit global offsets by decoupled look-back over the preceding
//                   tiles (single pass, no separate upsweep), reorders the tile in shared memory and
//                   stores digit-contiguous, fully coalesced runs.  While storing, it accumulates
//                   the histogram of the NEXT digit, so no pass ever re-reads the keys for
//                   counting (profile r1d: the up-front 8-digit histogram kernel cost 4 sort passes).
//
// Keys come from a "source" functor so that the first pass can synthesise keys on the fly (text
// 8-grams, ST context words) instead of reading a materialised key array: that removes one write
// + two reads of 8n bytes from every sort.
//
// HBM traffic per pass: (sizeof(K) + 4) bytes read + the same written per element -- the
// algorithmic floor for an LSD pass (ncu r1d: 1.615 GB measured vs 1.611 GB algorithmic for
// n = 2^26 pairs) -- plus 2 KB of look-back descriptors per 4096-element tile.
#pragma once

#include "common.cuh"

#define RS_THREADS 256
#define RS_ITEMS   16
#define RS_TILE    (RS_THREADS * RS_ITEMS)
#define RS_WARPS   (RS_THREADS / 32)
#define RS_MAX_PASSES 8

struct DigitPasses {
    int count;
    unsigned char shift[RS_MAX_PASSES];
    unsigned char bits[RS_MAX_PASSES];
};

// Build the list of <=8-bit digit passes covering key bit ranges [lo0,hi0) then [lo1,hi1) (LSD order).
static inline DigitPasses make_passes(int lo0, int hi0, int lo1 = 0, int hi1 = 0)
{
    DigitPasses p; p.count = 0;
    int lo[2] = {lo0, lo1}, hi[2] = {hi0, hi1};
    for (int f = 0; f < 2; ++f) {
        int total = hi[f] - lo[f];
        if (total <= 0) continue;
        int np = (total + 7) / 8;
        for (int s = lo[f], k = 0; k < np; ++k) {      // spread the bits evenly over the passes
            int b = (total + np - 1 - k) / np; if (b > hi[f] - s) b = hi[f] - s;
            p.shift[p.count] = (unsigned char)s; p.bits[p.count] = (unsigned char)b; p.count++; s += b;
        }
    }
    return p;
}

// ---- key sources ---------------------------------------------------------------------------
template <typename K, bool HAS_VAL> struct SrcArray {
    const K *keys; const u32 *vals;
    __device__ __forceinline__ K   key(u32 i) const { return keys[i]; }
    __device__ __forceinline__ u32 val(u32 i) const { return HAS_VAL ? vals[i] : 0u; }
};

// 8 bytes T[pos..pos+7] as one big-endian word.  T must be 8-byte aligned and readable (zero
// padded) up to pos+15.
__device__ __forceinline__ u64 load_be64(const u8 *T, u32 pos)
{
    const u64 *W = (const u64 *)T;
    u64 a = W[pos >> 3], b = W[(pos >> 3) + 1];
    u32 sh = (pos & 7u) * 8u;
    u64 v = sh ? ((a >> sh) | (b << (64u - sh))) : a;   // little-endian bytes pos..pos+7
    u32 lo = (u32)v, hi = (u32)(v >> 32);
    return ((u64)__byte_perm(lo, 0, 0x0123) << 32) | (u64)__byte_perm(hi, 0, 0x0123);
}

// ---- histogram of the first digit ------------------------------------------------------------
template <class Src>
__global__ void __launch_bounds__(RS_THREADS) rs_hist1(Src src, u32 n, int shift, int bits, u32 *__restrict__ ghist)
{
    __shared__ u32 sh[256];
    sh[threadIdx.x] = 0;
    __syncthreads();
    const u32 stride = gridDim.x * RS_THREADS, dmask = (1u << bits) - 1u;
    for (u32 i0 = blockIdx.x * RS_THREADS; i0 < n; i0 += stride) {       // whole warps stay in the loop (warp_peers is warp-collective)
        const u32 i = i0 + threadIdx.x;
        const u32 d = i < n ? ((u32)(src.key(i) >> shift) & dmask) : 256u;    // 256: "no item", a class of its own (bit 8)
        const u32 m = warp_peers(d, 9);                              // warp-aggregate: text digits are skewed
        if (i < n && (m & lanemask_lt()) == 0) atomicAdd(&sh[d], __popc(m));
    }
    __syncthreads();
    if (sh[threadIdx.x]) atomicAdd(&ghist[threadIdx.x], sh[threadIdx.x]);
}

// ---- one digit pass ------------------------------------------------------------------------
#define RS_FLAG_AGG    (1ull << 62)
#define RS_FLAG_PREFIX (2ull << 62)
#define RS_FLAG_MASK   (3ull << 62)

template <typename K> __device__ __forceinline__ K rs_all_ones();
template <> __device__ __forceinline__ u64 rs_all_ones<u64>() { return ~0ull; }
template <> __device__ __forceinline__ u32 rs_all_ones<u32>() { return ~0u; }

// 55 KB for (u64, u32) pairs: with the 1 KB the system reserves per CTA, TWO sort CTAs fit the half SM that a coder CTA (<= 113 KB) leaves
// free -- in the compress / decompress pipeline the sorts run in those halves, and at 59 KB (u32 warp histograms) only one fitted.
template <typename K, bool HAS_VAL> struct RsSmem {
    u16 whist[RS_WARPS][256];                            // per-warp digit counts (<= 512), then exclusive prefixes over the warps (< 4096)
    u32 dstart[256];                                     // (folding dstart into whist saves a load per item but made ptxas spill 40 - 100 bytes: kept apart)
    u32 gbase[256];
    u32 nexthist[256];
    u32 scan_tmp[RS_WARPS];
    u32 tile;
    K   keys[RS_TILE];
    u32 vals[HAS_VAL ? RS_TILE : 1];
};

// exclusive scan of one value per thread over the 256 threads of the CTA (tmp: RS_WARPS words)
__device__ __forceinline__ u32 rs_block_excl_scan(u32 v, u32 *tmp, u32 lane, u32 warp)
{
    u32 incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { u32 t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl += t; }
    if (lane == 31) tmp[warp] = incl;
    __syncthreads();
    u32 woff = 0;
#pragma unroll
    for (int w = 0; w < RS_WARPS; ++w) if (w < (int)warp) woff += tmp[w];
    __syncthreads();
    return woff + incl - v;
}

// MINB = CTAs per SM the register budget is cut for: 3 -> 80 registers (37 % occupancy), 4 -> 64 registers without spills (50 %); four
// 56 KB CTAs fill the 228 KB of an SM.
template <typename K, bool HAS_VAL, class Src, int MINB>
__global__ void __launch_bounds__(RS_THREADS, MINB)
rs_onesweep(Src src, K *__restrict__ kout, u32 *__restrict__ vout, u32 n, int shift, int bits,
            const u32 *__restrict__ hist_in, u32 *__restrict__ hist_next, int shift2, int bits2,
            u32 *tile_counter, u64 *lookback)
{
    extern __shared__ __align__(16) unsigned char rs_smem_raw[];
    RsSmem<K, HAS_VAL> &S = *reinterpret_cast<RsSmem<K, HAS_VAL> *>(rs_smem_raw);

    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 dmask = (1u << bits) - 1u;

    if (tid == 0) S.tile = atomicAdd(tile_counter, 1u);
    for (int i = tid; i < RS_WARPS * 256 / 2; i += RS_THREADS) ((u32 *)&S.whist[0][0])[i] = 0;
    S.nexthist[tid] = 0;
    // global digit bases = exclusive scan of this digit's histogram (complete: the previous kernel ended)
    const u32 gdigit_base = rs_block_excl_scan(hist_in[tid], S.scan_tmp, lane, warp);   // contains __syncthreads
    const u32 tile = S.tile;
    const u32 base = tile * RS_TILE;                     // n <= 2^30 so this cannot overflow
    const u32 valid = min((u32)RS_TILE, n - base);
    const u32 wbase = warp * (32 * RS_ITEMS) + lane;     // warp-striped: item i of this lane = wbase + 32*i

    K keys[RS_ITEMS];
#pragma unroll
    for (int i = 0; i < RS_ITEMS; ++i) {
        u32 off = wbase + 32 * i;
        keys[i] = off < valid ? src.key(base + off) : rs_all_ones<K>();
    }

    // --- warp-level multisplit ranking (stable: items in (i, lane) order) ---
    u32 pos[RS_ITEMS];
#pragma unroll
    for (int i = 0; i < RS_ITEMS; ++i) {
        u32 d = (u32)(keys[i] >> shift) & dmask;
        u32 m = __match_any_sync(0xffffffffu, d);
        u32 leader = __ffs(m) - 1;
        u32 pre = 0;
        if (lane == leader) { pre = S.whist[warp][d]; S.whist[warp][d] = (u16)(pre + __popc(m)); }
        pre = __shfl_sync(0xffffffffu, pre, leader);
        pos[i] = pre + __popc(m & lanemask_lt());
        __syncwarp();
    }
    __syncthreads();

    // --- per digit (thread = digit): warp offsets, tile offsets, decoupled look-back ---
    {
        const u32 d = tid;                               // RS_THREADS == 256 digits
        u32 run = 0;
#pragma unroll
#pragma unroll
        for (int w = 0; w < RS_WARPS; ++w) { u32 t = S.whist[w][d]; S.whist[w][d] = (u16)run; run += t; }
        const u32 count = run;
        const u32 excl = rs_block_excl_scan(count, S.scan_tmp, lane, warp);
        S.dstart[d] = excl;

        u64 *mine = lookback + (size_t)tile * 256 + d;
        u32 gexcl = 0;
        if (tile == 0) {
            st_relaxed(mine, RS_FLAG_PREFIX | (u64)count);
        } else {
            st_relaxed(mine, RS_FLAG_AGG | (u64)count);
            for (u32 t = tile; t-- > 0; ) {
                const u64 *theirs = lookback + (size_t)t * 256 + d;
                u64 v;
                do { v = ld_relaxed(theirs); } while ((v & RS_FLAG_MASK) == 0);
                gexcl += (u32)v;
                if ((v & RS_FLAG_MASK) == RS_FLAG_PREFIX) break;
            }
            st_relaxed(mine, RS_FLAG_PREFIX | (u64)(gexcl + count));
        }
        S.gbase[d] = gdigit_base + gexcl - excl;         // u32 wrap-around arithmetic is intended
    }
    __syncthreads();

    // --- reorder the tile in shared memory, then store digit-contiguous runs ---
#pragma unroll
    for (int i = 0; i < RS_ITEMS; ++i) {
        u32 d = (u32)(keys[i] >> shift) & dmask;
        pos[i] += S.dstart[d] + S.whist[warp][d];
        S.keys[pos[i]] = keys[i];
    }
    if (HAS_VAL) {
#pragma unroll
        for (int i = 0; i < RS_ITEMS; ++i) {
            u32 off = wbase + 32 * i;
            if (off < valid) S.vals[pos[i]] = src.val(base + off);
        }
    }
    __syncthreads();
    const u32 dmask2 = (1u << bits2) - 1u;
#pragma unroll 4
    for (u32 j = tid; j < valid; j += RS_THREADS) {
        K k = S.keys[j];
        u32 d = (u32)(k >> shift) & dmask;
        u32 g = S.gbase[d] + j;
        kout[g] = k;
        if (HAS_VAL) vout[g] = S.vals[j];
        if (hist_next) atomicAdd(&S.nexthist[(u32)(k >> shift2) & dmask2], 1u);   // next digit's histogram, for free
    }
    if (hist_next) {
        __syncthreads();
        const u32 c = S.nexthist[tid];
        if (c) atomicAdd(&hist_next[tid], c);
    }
}

// ---- one digit pass over MATERIALISED keys: persistent CTAs, tiles staged by TMA, two stages ------------------------------------
// Every pass but the first reads (key, value) arrays.  Here a CTA keeps taking tiles (ordered tile ids from an atomic counter, as
// the look-back needs) and the NEXT tile's 32 KB of keys + 16 KB of values are already on their way into the other shared-memory
// stage -- one elected thread issues two cp.async.bulk (TMA, SASS UBLKCP) that complete on the stage's mbarrier -- while the
// current tile is ranked, reordered in place in its stage and stored.  No load instruction sits between the tile and the ranking,
// the registers hold only the current tile, and HBM reads run a full tile ahead of the compute.
template <typename K, bool HAS_VAL> struct RsSmemTma {
    alignas(128) K   keys[2][RS_TILE];
    alignas(128) u32 vals[2][HAS_VAL ? RS_TILE : 4];
    u32 whist[RS_WARPS][256];
    u32 dstart[256];
    u32 gbase[256];
    u32 nexthist[256];
    u32 scan_tmp[RS_WARPS];
    u32 tile[2];
    alignas(8) u64 full[2];                              // mbarriers: "stage s holds its tile"
};

template <typename K, bool HAS_VAL>
__global__ void __launch_bounds__(RS_THREADS, 2)
rs_onesweep_tma(const K *__restrict__ kin, const u32 *__restrict__ vin, K *__restrict__ kout, u32 *__restrict__ vout, u32 n, u32 tiles, int shift, int bits,
                const u32 *__restrict__ hist_in, u32 *__restrict__ hist_next, int shift2, int bits2, u32 *tile_counter, u64 *lookback)
{
    extern __shared__ __align__(128) unsigned char rs_smem_raw[];
    RsSmemTma<K, HAS_VAL> &S = *reinterpret_cast<RsSmemTma<K, HAS_VAL> *>(rs_smem_raw);
    const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const u32 dmask = (1u << bits) - 1u, dmask2 = (1u << bits2) - 1u;

    // stage s <- tile t (thread 0 only): expect the bytes, then the two bulk copies; sizes rounded up to 16 (the arrays are padded)
    auto fill = [&](u32 s, u32 t) {
        const u32 base = t * RS_TILE, valid = min((u32)RS_TILE, n - base);
        const u32 kb = (valid * (u32)sizeof(K) + 15u) & ~15u, vb = HAS_VAL ? ((valid * 4u + 15u) & ~15u) : 0u;
        mbar_arrive_expect_tx(&S.full[s], kb + vb);
        bulk_copy_g2s(S.keys[s], kin + base, kb, &S.full[s]);
        if (HAS_VAL) bulk_copy_g2s(S.vals[s], vin + base, vb, &S.full[s]);
    };

    if (tid == 0) { mbar_init(&S.full[0], 1); mbar_init(&S.full[1], 1); mbar_init_fence(); }
    S.nexthist[tid] = 0;
    const u32 gdigit_base = rs_block_excl_scan(hist_in[tid], S.scan_tmp, lane, warp);   // contains __syncthreads: the barriers are initialised
    if (tid == 0) {
        for (u32 s = 0; s < 2; ++s) { const u32 t = atomicAdd(tile_counter, 1u); S.tile[s] = t; if (t < tiles) fill(s, t); }
    }
    u32 parity0 = 0, parity1 = 0;
    const u32 wbase = warp * (32 * RS_ITEMS) + lane;     // warp-striped: item i of this lane = wbase + 32*i

    for (u32 s = 0; ; s ^= 1) {
        __syncthreads();                                 // tile[s] is visible; every read of the previous tile's stage is done
        const u32 tile = S.tile[s];
        if (tile >= tiles) break;                        // ids grow with time: the other stage has no tile either
        const u32 base = tile * RS_TILE, valid = min((u32)RS_TILE, n - base);
        for (int i = tid; i < RS_WARPS * 256; i += RS_THREADS) (&S.whist[0][0])[i] = 0;
        if (s == 0) { mbar_wait(&S.full[0], parity0); parity0 ^= 1; } else { mbar_wait(&S.full[1], parity1); parity1 ^= 1; }

        K keys[RS_ITEMS]; u32 vals[RS_ITEMS];
#pragma unroll
        for (int i = 0; i < RS_ITEMS; ++i) {
            const u32 off = wbase + 32 * i;
            keys[i] = off < valid ? S.keys[s][off] : rs_all_ones<K>();
            if (HAS_VAL) vals[i] = S.vals[s][off];
        }
        __syncthreads();                                 // the tile lives in registers: its stage can take the reordered tile; whist is zero

        u32 pos[RS_ITEMS];
#pragma unroll
        for (int i = 0; i < RS_ITEMS; ++i) {
            const u32 d = (u32)(keys[i] >> shift) & dmask;
            const u32 m = __match_any_sync(0xffffffffu, d);
            const u32 leader = __ffs(m) - 1;
            u32 pre = 0;
            if (lane == leader) { pre = S.whist[warp][d]; S.whist[warp][d] = pre + __popc(m); }
            pre = __shfl_sync(0xffffffffu, pre, leader);
            pos[i] = pre + __popc(m & lanemask_lt());
            __syncwarp();
        }
        __syncthreads();
        {
            const u32 d = tid;
            u32 run = 0;
#pragma unroll
            for (int w = 0; w < RS_WARPS; ++w) { u32 t = S.whist[w][d]; S.whist[w][d] = run; run += t; }
            const u32 count = run;
            const u32 excl = rs_block_excl_scan(count, S.scan_tmp, lane, warp);
            S.dstart[d] = excl;
            u64 *mine = lookback + (size_t)tile * 256 + d;
            u32 gexcl = 0;
            if (tile == 0) {
                st_relaxed(mine, RS_FLAG_PREFIX | (u64)count);
            } else {
                st_relaxed(mine, RS_FLAG_AGG | (u64)count);
                for (u32 t = tile; t-- > 0; ) {
                    const u64 *theirs = lookback + (size_t)t * 256 + d;
                    u64 v;
                    do { v = ld_relaxed(theirs); } while ((v & RS_FLAG_MASK) == 0);
                    gexcl += (u32)v;
                    if ((v & RS_FLAG_MASK) == RS_FLAG_PREFIX) break;
                }
                st_relaxed(mine, RS_FLAG_PREFIX | (u64)(gexcl + count));
            }
            S.gbase[d] = gdigit_base + gexcl - excl;
        }
        __syncthreads();
#pragma unroll
        for (int i = 0; i < RS_ITEMS; ++i) {
            const u32 d = (u32)(keys[i] >> shift) & dmask;
            const u32 q = pos[i] + S.dstart[d] + S.whist[warp][d];
            S.keys[s][q] = keys[i];
            if (HAS_VAL) S.vals[s][q] = vals[i];
        }
        __syncthreads();
#pragma unroll 4
        for (u32 j = tid; j < valid; j += RS_THREADS) {
            const K k = S.keys[s][j];
            const u32 g = S.gbase[(u32)(k >> shift) & dmask] + j;
            kout[g] = k;
            if (HAS_VAL) vout[g] = S.vals[s][j];
            if (hist_next) atomicAdd(&S.nexthist[(u32)(k >> shift2) & dmask2], 1u);
        }
        __syncthreads();                                 // stage s has been read for the last time
        if (tid == 0) {
            const u32 t = atomicAdd(tile_counter, 1u);
            S.tile[s] = t;
            if (t < tiles) { fence_proxy_async_smem(); fill(s, t); }
        }
    }
    if (hist_next) {
        const u32 c = S.nexthist[tid];                   // all atomics on it precede the loop's final barrier
        if (c) atomicAdd(&hist_next[tid], c);
    }
}

// ---- host driver ---------------------------------------------------------------------------
// BSCB200_SORT_TMA=1: passes over materialised keys through rs_onesweep_tma.  The TMA-staged
// persistent kernel is slower than rs_onesweep -- a persistent CTA holds the id of its PREFETCHED
// tile while it still works on the current one, so that tile's aggregate reaches the look-back a whole tile time later and the chain of
// waits grows (long-scoreboard and branch-resolving stalls dominate); it also takes 109 KB of shared memory per CTA, which
// no SM half next to a coder CTA can give.  So it is not the default; it stays selectable and parity-tested.
static inline int rs_min_blocks() { static const int v = [] { const char *e = getenv("BSCB200_SORT_OCC"); return (e && e[0] == '3') ? 3 : 4; }(); return v; }
static inline bool rs_use_tma() { static const bool on = [] { const char *e = getenv("BSCB200_SORT_TMA"); return e && e[0] == '1'; }(); return on; }

// Scratch needed by one sort (histograms, tile counters, look-back descriptors).
static inline size_t rs_scratch_bytes(u32 n, int npasses)
{
    size_t tiles = ceil_div(n, RS_TILE);
    return align_up(sizeof(u32) * 256 * RS_MAX_PASSES + sizeof(u32) * 64, 256) + (size_t)npasses * tiles * 256 * sizeof(u64);
}

// Sort n elements.  Pass 0 reads from `first`; later passes ping-pong between (k[0],v[0]) and
// (k[1],v[1]), pass p writing to buffer (p & 1).  Returns the index of the buffer holding the
// sorted result.  `scratch` must hold rs_scratch_bytes(n, passes.count).  `name`: the passes' name in the profile.
template <typename K, bool HAS_VAL, class FirstSrc>
static int rs_sort(Ctx *ctx, FirstSrc first, K *const k[2], u32 *const v[2], u32 n, const DigitPasses &passes, void *scratch,
                   const char *name = "rs_onesweep")
{
    if (passes.count == 0 || n == 0) return -1;
    const u32 tiles = ceil_div(n, RS_TILE);
    u32 *ghist = (u32 *)scratch;
    u32 *counters = ghist + 256 * RS_MAX_PASSES;
    u64 *lookback = (u64 *)((u8 *)scratch + align_up(sizeof(u32) * 256 * RS_MAX_PASSES + sizeof(u32) * 64, 256));
    CUDA_TRY(cudaMemsetAsync(scratch, 0, rs_scratch_bytes(n, passes.count), ctx->stream));

    u32 hgrid = min(tiles, device_sms(ctx->device) * 8);
    const double pass_bytes = 2.0 * (double)n * (sizeof(K) + (HAS_VAL ? 4 : 0));   // read + write of every element
    PROF_BYTES(ctx, (double)n * sizeof(K));
    LAUNCH(ctx, (rs_hist1<FirstSrc>), hgrid, RS_THREADS, 0, first, n, (int)passes.shift[0], (int)passes.bits[0], ghist);

    const size_t smem = sizeof(RsSmem<K, HAS_VAL>);
    const bool occ4 = rs_min_blocks() == 4;
    auto *const k_first = occ4 ? rs_onesweep<K, HAS_VAL, FirstSrc, 4> : rs_onesweep<K, HAS_VAL, FirstSrc, 3>;
    auto *const k_next  = occ4 ? rs_onesweep<K, HAS_VAL, SrcArray<K, HAS_VAL>, 4> : rs_onesweep<K, HAS_VAL, SrcArray<K, HAS_VAL>, 3>;
    ensure_dyn_smem(k_first, ctx->device, smem);
    ensure_dyn_smem(k_next, ctx->device, smem);
    const size_t smem_tma = sizeof(RsSmemTma<K, HAS_VAL>);
    ensure_dyn_smem(rs_onesweep_tma<K, HAS_VAL>, ctx->device, smem_tma);

    for (int p = 0; p < passes.count; ++p) {
        int dst = p & 1;
        u64 *lb = lookback + (size_t)p * tiles * 256;
        const bool more = p + 1 < passes.count;
        u32 *hnext = more ? ghist + 256 * (p + 1) : nullptr;
        const int s2 = more ? (int)passes.shift[p + 1] : 0, b2 = more ? (int)passes.bits[p + 1] : 1;
        PROF_BYTES(ctx, pass_bytes);
        if (p == 0) {
            LAUNCH_NAMED(ctx, name, k_first, tiles, RS_THREADS, smem,
                   first, k[dst], v[dst], n, (int)passes.shift[p], (int)passes.bits[p], ghist + 256 * p, hnext, s2, b2, counters + p, lb);
        } else if (!rs_use_tma()) {
            SrcArray<K, HAS_VAL> src{k[dst ^ 1], v[dst ^ 1]};
            LAUNCH_NAMED(ctx, name, k_next, tiles, RS_THREADS, smem,
                   src, k[dst], v[dst], n, (int)passes.shift[p], (int)passes.bits[p], ghist + 256 * p, hnext, s2, b2, counters + p, lb);
        } else {
            const u32 grid = min(tiles, device_sms(ctx->device) * 2);                // persistent: two CTAs per SM, each loops over tiles
            LAUNCH(ctx, (rs_onesweep_tma<K, HAS_VAL>), grid, RS_THREADS, smem_tma,
                   (const K *)k[dst ^ 1], (const u32 *)v[dst ^ 1], k[dst], v[dst], n, tiles, (int)passes.shift[p], (int)passes.bits[p], ghist + 256 * p, hnext, s2, b2, counters + p, lb);
        }
    }
    return (passes.count - 1) & 1;
}
