// libbsc_b200/csrc/st_encode_batched.cu -- Sort Transform of order k (k = 3..8) whose working set is bounded: n + 28 bytes per
// batch entry.
//
// Same definition and result as st_encode.cu: P = the STABLE sort of the n cyclic rotations by their first k bytes,
// L[j] = T[(P[j] - 1) mod n], index = the j with P[j] = 0.  The standard sorter radix-sorts all n rotations at once (about 30 n bytes);
// ST-k has no doubling rounds, so one stable sort by at most 64 key bits is the whole job, and here it runs in batches of at most B
// entries.  The key of rotation i is T[i .. i+k) taken cyclically as a big-endian word (KB = 8 k bits).
//
// All rotations form one segment, read straight from the text (key_cuts.cuh).  Its key space is cut into ranges of at most B entries.
// Each range is compacted out of the segment in ASCENDING position order, which is what makes the result stable, radix-sorted on the
// key bits below the range's common prefix, and its L bytes are written at the range's rows of a separate L buffer.  A single key
// value with more than B entries needs no sort: its positions in ascending order are its rows, so they are compacted straight into L.
// The text is only read until the last range is done; then L is copied over it.
//
// Every range, every oversized key value and every histogram level scans the whole text, so the work grows with n / B; B is kept at
// least bwt_batch_floor(n) = max(65536, n / 64) for the same reason as in bwt_encode_batched.cu.
#include "radix_sort.cuh"
#include "stages.cuh"
#include "key_cuts.cuh"

namespace {

// the segment: rotation i is entry i, its key the k bytes T[i .. i+k) taken cyclically (a context wraps around the text more than
// once when n < 8).  T need not be aligned or padded.
struct SegRot {
    const u8 *T; u32 n; int k;
    __device__ __forceinline__ u64 key(u32 i) const {
        u64 v = 0;
        if ((u64)i + 16 <= n) v = text8(T, n, i);
        else for (u32 b = 0, j = i; b < 8; ++b, j = j + 1 == n ? 0u : j + 1) v = (v << 8) | T[j];
        return v >> (64 - 8 * k);
    }
    __device__ __forceinline__ u32 pos(u32 i) const { return i; }
};

// the L byte of rotation p at row `row`; the row of rotation 0 is the index
__device__ __forceinline__ void st_put(const u8 *T, u32 n, u32 p, u8 *L, u32 row, u32 *index)
{
    L[row] = T[p ? p - 1 : n - 1];
    if (p == 0) *index = row;
}

// the rotations whose key is `val` (more than a batch of them), in ascending position order = their order in P: rows base, base + 1, ..
struct PickRows {
    SegRot s; u64 val; u8 *L; u32 base; u32 *index;
    __device__ __forceinline__ bool pred(u32 i) const { return s.key(i) == val; }
    __device__ __forceinline__ void emit(u32 i, u32 x) const { st_put(s.T, s.n, i, L, base + x, index); }
};

// the sorted positions of one range -> rows base ..
__global__ void __launch_bounds__(256) st_batch_emit(const u32 *__restrict__ pos, u32 cnt, const u8 *__restrict__ T, u32 n,
                                                     u8 *__restrict__ L, u32 base, u32 *index)
{
    const u32 j = blockIdx.x * 256 + threadIdx.x;
    if (j < cnt) st_put(T, n, pos[j], L, base + j, index);
}

}  // namespace

size_t st_batched_bytes(u32 n, u32 B)
{
    return Arena::bytes_for<u8>(n) + Arena::bytes_for<TileAgg>(ceil_div(n, CP_TILE)) + Arena::bytes_for<u32>(65536) + Arena::bytes_for<u32>(1)
         + 2 * Arena::bytes_for<u64>(B) + 2 * Arena::bytes_for<u32>(B) + Arena::bytes_for<u8>(rs_scratch_bytes(B, RS_MAX_PASSES));
}

u32 st_batch_entries(u32 n, long long budget)
{
    const long long fixed = (long long)st_batched_bytes(n, 0), per = 28;    // per entry: keys 2 x 8, values 2 x 4, look-back 4
    long long b = budget > fixed ? (budget - fixed) / per : 0;
    if (b > (long long)n) b = n;
    if (b > ST_BATCH_MAX) b = ST_BATCH_MAX;
    const u32 floor = bwt_batch_floor(n);
    return b < (long long)floor ? floor : (u32)b;
}

// Sort transform of d_T[0..n) in place, sorting in batches of at most B entries.  Same results as stage_st_encode.
int stage_st_encode_batched(Ctx *ctx, u8 *d_T, int n_, int k, u32 B)
{
    if (n_ < 0) return LIBBSC_BAD_PARAMETER;
    if (k < 3 || k > 8) return LIBBSC_BAD_PARAMETER;
    if (n_ <= 1) return 0;
    const u32 n = (u32)n_;
    if (B < bwt_batch_floor(n)) B = bwt_batch_floor(n);

    Arena &A = ctx->sort_arena();
    const size_t mark = A.mark();
    KeyCuts C;
    C.ctx = ctx; C.B = B;
    u8 *L = A.get<u8>(n);
    C.agg = A.get<TileAgg>(ceil_div(n, CP_TILE));
    C.hist = A.get<u32>(65536);
    u32 *index = A.get<u32>(1);
    u64 *kb[2] = { A.get<u64>(B), A.get<u64>(B) };
    u32 *vb[2] = { A.get<u32>(B), A.get<u32>(B) };
    void *scratch = A.get<u8>(rs_scratch_bytes(B, RS_MAX_PASSES));
    C.h_hist.resize(65536);
    CUDA_TRY(cudaMemsetAsync(index, 0xff, sizeof(u32), ctx->stream));

    const SegRot s{d_T, n, k};
    std::vector<Range> R;
    bool ok = C.cut(s, n, 8 * k, R);
    for (size_t i = 0; ok && i < R.size(); ++i) {
        const Range &r = R[i];
        if (r.count > B) { ok = C.compact(PickRows{s, r.lo, L, r.cum, index}, n) == r.count; continue; }
        ok = C.compact(PickRange<SegRot>{s, r.lo, r.hi, kb[1], vb[1]}, n) == r.count;
        const int bits = r.lo == r.hi ? 0 : 64 - __builtin_clzll(r.lo ^ r.hi);       // the range's keys agree above these bits
        int cur = 1;
        if (ok && bits) cur = rs_sort<u64, true>(ctx, SrcArray<u64, true>{kb[1], vb[1]}, kb, vb, r.count, make_passes(0, bits), scratch);
        if (ok) LAUNCH(ctx, st_batch_emit, ceil_div(r.count, 256), 256, 0, (const u32 *)vb[cur], r.count, (const u8 *)d_T, n, L, r.cum, index);
    }
    if (!ok) { A.release(mark); return LIBBSC_GPU_ERROR; }

    CUDA_TRY(cudaMemcpyAsync(d_T, L, n, cudaMemcpyDeviceToDevice, ctx->stream));
    CUDA_TRY(cudaMemcpyAsync(ctx->h_mail, index, sizeof(u32), cudaMemcpyDeviceToHost, ctx->stream));
    ctx->sync();
    A.release(mark);
    return ctx->h_mail[0] < n ? (int)ctx->h_mail[0] : LIBBSC_GPU_ERROR;
}
