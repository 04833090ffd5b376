// libbsc_b200/csrc/list_rank.cuh -- in-place Wyllie pointer jumping on 64-bit (successor | distance << 32) pairs, shared by the inverse
// BWT (bwt_decode.cu: lists of segment nodes) and the inverse sort transform (st_decode.cu: lists of rows).
//
// pair[i] = successor | weight << 32.  A list END points to itself and carries LR_DONE in its distance word (its own weight counts).
// After convergence every element holds (its list's end, sum of the weights from itself to the end inclusive of the end's) | LR_DONE.
// Any 64-bit snapshot of pair[j] is a valid (successor, distance) statement, so reading a pair that another thread has already
// advanced in the same round only speeds convergence up: no ping-pong buffers.  Rounds after convergence return at once (device-side
// flag per round, no host round trip); launch ceil(log8(longest list)) + 1 of them (LR_HOPS jumps per element and launch).
#pragma once
#include "common.cuh"

#define LR_DONE 0x80000000u

namespace {

// LR_HOPS jumps per element and launch.  If every unfinished pointer spans >= D elements before a launch, every element it reads
// during the launch spans >= D too (its state from the previous launch, or better), so after k hops the pointer spans >= (k + 1) D: the
// span grows by LR_HOPS + 1 = 8 per launch instead of 2 -- 8 launches for 1.5 M nodes instead of 22, with no more memory traffic per
// element (an element stops hopping the moment it is done).  The pair is stored once, after the last hop.
#define LR_HOPS 7
__global__ void __launch_bounds__(256) lr_jump(u64 *pair, u32 n, u32 *flags, int round)
{
    if (round > 0 && flags[round - 1] == 0) return;     // converged in an earlier round (uniform for the whole grid)
    const u32 i = blockIdx.x * 256 + threadIdx.x;
    bool more = false;
    if (i < n) {
        u64 p = ld_relaxed(pair + i);
        u32 d = (u32)(p >> 32);
        if (!(d & LR_DONE)) {
#pragma unroll 1
            for (int h = 0; h < LR_HOPS && !(d & LR_DONE); ++h) {
                const u64 q = ld_relaxed(pair + (u32)p);
                const u32 qd = (u32)(q >> 32);
                d = (d + (qd & ~LR_DONE)) | (qd & LR_DONE);
                p = (u64)(u32)q | ((u64)d << 32);
            }
            st_relaxed(pair + i, p);
            more = !(d & LR_DONE);
        }
    }
    // ONE store per CTA: two million threads storing to the same word serialise
    if (__syncthreads_or(more) && threadIdx.x == 0) flags[round] = 1;
}

}  // namespace

// enqueue enough rounds for lists of up to `longest` elements; flags: >= 40 zeroed words
static inline void lr_rank(Ctx *ctx, u64 *pair, u32 n, u32 longest, u32 *flags)
{
    int rounds = 1; u64 span = LR_HOPS + 1; while (span < (u64)longest) { span *= LR_HOPS + 1; ++rounds; }
    for (int r = 0; r <= rounds; ++r) LAUNCH(ctx, lr_jump, ceil_div(n, 256), 256, 0, pair, n, flags, r);
}
