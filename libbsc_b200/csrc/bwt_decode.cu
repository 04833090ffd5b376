// libbsc_b200/csrc/bwt_decode.cu -- inverse Burrows-Wheeler transform on the device.
//
// Replaces bsc_bwt_decode (libbsc/bwt/bwt.cpp:283-332: libsais_unbwt on the CPU,
// libcubwt_unbwt on the GPU, libcubwt.cu:2953-3132).
//
// Conventions (SURVEY.md B.1): the conceptual matrix of T$ has n+1 rows; row 0 starts with '$',
// and L is its last column with the '$' entry (row `index`) removed.  LF(row) = 1 + C[c] +
// occ_c(row); walking LF from row 0 yields T backwards.
//
//   unbwt_hist   256-bin histogram of L                                   (reads n)
//   unbwt_lf     LF mapping = destination of a STABLE counting sort by symbol: per 4 KB tile a
//                warp match-any multisplit ranks the bytes, per-symbol decoupled look-back gives
//                the tile's global offsets in the same pass              (reads n, writes 4n)
//   unbwt_walk   K ~ n/64 start rows (one per 64-row window, jittered); one thread per segment chases LF until it
//                reaches another start row -- ONCE: the bytes it meets are staged in 128-byte slabs (node k = segment k's first
//                slab; a segment longer than 128 bytes takes further nodes from an atomic counter and links them), so the
//                pointer chase, which is sector/latency bound (one dependent 4-byte gather per output byte), is never repeated
//                (an earlier version walked twice; the reference stages too, libcubwt.cu:2744-2906)
//   lr_jump      device-side pointer-jumping list ranking over the nodes (list_rank.cuh; no host round trip, cf.
//                libcubwt.cu:3077-3086): bytes from the start of every node to the end of the walk
//   unbwt_place  every staged byte goes to its final place (coalesced reads, contiguous reversed writes)
#include "common.cuh"
#include "stages.cuh"
#include "lf_map.cuh"
#include "list_rank.cuh"

namespace {

// Segment starts ("marks"): one row per window of 64 rows, at a pseudo-random offset inside the window.  Evenly spaced marks would
// be correct too, but on structured inputs LF advances rows in arithmetic progressions (a text of period 8 and length 2^26 keeps the
// row's residue mod 64 for millions of steps), and then one thread walks a chain of millions of rows alone.  The reference jitters its
// marks for the same reason (libcubwt.cu:2727-2742).  Window 0 starts at row 0, where the walk begins.
__device__ __forceinline__ u32 mark_row(u32 w, u32 n)
{
    u32 h = w * 0x9E3779B1u; h ^= h >> 15; h *= 0x85EBCA77u; h ^= h >> 13;
    const u32 r = (w << 6) + (w == 0 ? 0u : (h & 63u));
    return r <= n ? r : (w << 6);                        // rows are 0 .. n; the last window may be short
}
__device__ __forceinline__ bool is_mark(u32 row, u32 n) { return mark_row(row >> 6, n) == row; }

#define UW_SLAB 128u                                    // bytes per node: a segment (mean 64 bytes, geometric) needs a second node in 13 % of the cases

// One thread per segment k (start row mark_row(k)); node ids: k for the first slab, K + (atomic counter) for the others.
// pair[node] = (next node | bytes in this node << 32) for lr_jump; the node whose walk reaches row `index` ends the text's list.
__global__ void __launch_bounds__(256) unbwt_walk(const u32 *__restrict__ LF, const u8 *__restrict__ L, u32 n, u32 index, u32 K, u32 max_nodes,
                                                  u32 *node_counter, u64 *__restrict__ pair, u8 *__restrict__ node_len, u32 *__restrict__ stage)
{
    u32 k = blockIdx.x * 256 + threadIdx.x;
    if (k >= K) return;
    u32 row = mark_row(k, n), node = k, j = 0, w = 0, extra = 0;
    u32 *slab = stage + (size_t)node * (UW_SLAB / 4);
    u64 link;
    for (;;) {
        if (row == index) { link = (u64)node | ((u64)(j | LR_DONE) << 32); break; }                    // the walk ends in front of the '$' row
        w = (w >> 8) | ((u32)L[row < index ? row : row - 1] << 24);                                      // byte j of the node, little-endian packing
        if ((++j & 3u) == 0) slab[(j >> 2) - 1] = w;
        row = __ldg(LF + row);
        if (is_mark(row, n)) { link = (u64)(row >> 6) | ((u64)j << 32); break; }                        // the next segment starts here
        if (j == UW_SLAB) {                                                                             // slab full: link a fresh node and go on
            const u32 fresh = K + atomicAdd(node_counter, 1u);
            if (fresh >= max_nodes || ++extra > n / UW_SLAB + 1) { link = (u64)node | ((u64)(j | LR_DONE) << 32); break; }   // corrupt input: LF is not a permutation
            pair[node] = (u64)fresh | ((u64)j << 32); node_len[node] = (u8)j;
            node = fresh; j = 0; slab = stage + (size_t)node * (UW_SLAB / 4);
        }
    }
    if (j & 3u) slab[j >> 2] = w >> (8u * (4u - (j & 3u)));
    pair[node] = link; node_len[node] = (u8)j;
}

// Byte j (walk order) of node i is text position D(i) - 1 - j, D(i) = bytes from the start of node i to the end of the walk.
// One thread per 4 staged bytes: a warp reads 128 contiguous bytes and writes 128 contiguous bytes (reversed).
__global__ void __launch_bounds__(256) unbwt_place(const u64 *__restrict__ pair, const u8 *__restrict__ node_len, const u32 *__restrict__ stage, const u32 *__restrict__ node_counter,
                                                   u32 K, u32 n, u8 *__restrict__ out)
{
    const u64 t = (u64)blockIdx.x * 256 + threadIdx.x;     // word index into the slabs
    const u32 node = (u32)(t / (UW_SLAB / 4)), j0 = (u32)(t % (UW_SLAB / 4)) * 4u;
    if (node >= K + min(*node_counter, n / UW_SLAB + 1u)) return;
    const u32 len = node_len[node];
    if (j0 >= len) return;
    const u32 D = (u32)(pair[node] >> 32) & ~LR_DONE;
    const u32 w = stage[t];
#pragma unroll
    for (u32 b = 0; b < 4; ++b) {
        const u32 j = j0 + b;
        const u64 pos = (u64)D - 1 - j;
        if (j < len && D > j && pos < n) out[pos] = (u8)(w >> (8 * b));
    }
}

// one segment per window of 64 rows (mark_row); every further node of a segment holds 64 bytes of text
u32 unbwt_segments(u32 n) { return ceil_div((u64)n + 1, 64); }
u32 unbwt_max_nodes(u32 n) { return unbwt_segments(n) + n / UW_SLAB + 2; }

}  // namespace

size_t bwt_decode_bytes(u32 n)
{
    const size_t nodes = unbwt_max_nodes(n);
    return Arena::bytes_for<u8>((size_t)n + 64) + Arena::bytes_for<u32>((size_t)n + 2) + Arena::bytes_for<u32>(256 + 64 + 64)
         + Arena::bytes_for<u64>((size_t)ceil_div(n, LF_TILE) * 256) + Arena::bytes_for<u64>(nodes) + Arena::bytes_for<u8>(nodes)
         + Arena::bytes_for<u32>(nodes * (UW_SLAB / 4));
}

int stage_bwt_decode(Ctx *ctx, u8 *d_T, int n_, int index_)
{
    if (d_T == nullptr || n_ < 0 || index_ <= 0 || index_ > n_) return LIBBSC_BAD_PARAMETER;
    if (n_ <= 1) return LIBBSC_NO_ERROR;
    const u32 n = (u32)n_, index = (u32)index_;
    Arena &A = ctx->arena;
    const size_t mark = A.mark();

    // the buffers below are what bwt_decode_bytes(n) counts
    const u32 tiles = ceil_div(n, LF_TILE);
    const u32 K = unbwt_segments(n);
    const u32 max_nodes = unbwt_max_nodes(n);
    u8  *Lp    = A.get<u8>((size_t)n + 64);
    u32 *LF    = A.get<u32>((size_t)n + 2);
    u32 *hist  = A.get<u32>(256 + 64 + 64);                  // [0..255] counts / bases, [256] tile counter, [320] node counter, [321..] jump flags
    u64 *lb    = A.get<u64>((size_t)tiles * 256);
    u64 *pair  = A.get<u64>((size_t)max_nodes);
    u8  *nlen  = A.get<u8>((size_t)max_nodes);
    u32 *stage = A.get<u32>((size_t)max_nodes * (UW_SLAB / 4));

    CUDA_TRY(cudaMemcpyAsync(Lp, d_T, n, cudaMemcpyDeviceToDevice, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(Lp + n, 0, 64, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(hist, 0, sizeof(u32) * (256 + 64 + 64), ctx->stream));
    CUDA_TRY(cudaMemsetAsync(lb, 0, sizeof(u64) * (size_t)tiles * 256, ctx->stream));
    CUDA_TRY(cudaMemsetAsync(nlen, 0, (size_t)max_nodes, ctx->stream));                                  // unused nodes: empty ...
    CUDA_TRY(cudaMemsetAsync(pair, 0xff, sizeof(u64) * (size_t)max_nodes, ctx->stream));                 // ... and LR_DONE, so the ranking skips them

    LAUNCH(ctx, unbwt_hist, min(ceil_div(n, 256 * 64), device_sms(ctx->device) * 8), 256, 0, Lp, n, hist);
    LAUNCH(ctx, unbwt_scan256, 1, 32, 0, hist);
    PROF_BYTES(ctx, 5.0 * n);
    LAUNCH(ctx, unbwt_lf<true>, tiles, LF_THREADS, 0, Lp, n, index, hist, hist + 256, lb, LF);

    PROF_BYTES(ctx, 6.0 * n);                                // 4 n of LF gathered, n of L gathered, n staged
    LAUNCH(ctx, unbwt_walk, ceil_div(K, 256), 256, 0, LF, Lp, n, index, K, max_nodes, hist + 320, pair, nlen, stage);
    lr_rank(ctx, pair, max_nodes, max_nodes, hist + 321);
    PROF_BYTES(ctx, 2.0 * n);
    LAUNCH(ctx, unbwt_place, ceil_div((u64)max_nodes * (UW_SLAB / 4), 256), 256, 0, pair, nlen, (const u32 *)stage, hist + 320, K, n, d_T);
    A.release(mark);
    return LIBBSC_NO_ERROR;
}
