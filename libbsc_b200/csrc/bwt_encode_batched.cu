// libbsc_b200/csrc/bwt_encode_batched.cu -- forward BWT whose working set is bounded: 16 n bytes + 32 bytes per batch entry.
//
// Same prefix doubling as bwt_encode.cu and the same result (the BWT is a pure function of the suffix order).  The standard sorter
// radix-sorts every active suffix of a round at once, which takes about 58 n bytes.  This one keeps only four global u32 arrays
//   rank[p]  1 + SA slot of the head of suffix p's group (as in bwt_encode.cu),
//   sa[i]    positions of the ACTIVE suffixes (those in unsorted groups) in slot order,
//   idx[i]   their slots,
//   key2[i]  the round's second key of active entry i,
// and sorts in batches of at most B entries in one workspace (keys and values double-buffered, radix scratch).
//
// Initial sort by the first 8 bytes.  All n suffixes form one "segment" (entry e = position n-1-e, so equal keys keep the
// shorter suffix first, as in the standard sorter).  A segment is cut into key ranges of at most B entries: a 65536-bin histogram of
// the top 16 key bits, refined by the next 16 bits only inside bins that hold more than B entries.  Each range is compacted out of the
// segment in entry order, radix-sorted and split into groups (rank[]), and its sorted positions go to the segment's slots in
// idx[], used as a temporary.  A single key value with more than B entries is one group already: it is compacted straight into its
// slots, unsorted.  Finally the segment's non-singleton slots are compacted into sa[] / idx[].
//
// Doubling rounds.  key2[i] = rank[sa[i] + h] is gathered for ALL active entries before any rank of the round changes; ranks written
// later in the round stay inside the written group's slot range, so the batches of one round are independent.  The active list is cut
// into batches of whole groups of at most B entries, each sorted by (head slot of its group, key2) and split like a standard round.  A
// group of more than B entries is a segment of its own, keyed by key2, and is cut into key2 ranges as above.
#include "radix_sort.cuh"
#include "stages.cuh"
#include "key_cuts.cuh"

namespace {

// entries of a segment: key and position of entry i
struct SegText {                                         // the initial segment: every suffix, descending position
    const u8 *T; u32 n;
    __device__ __forceinline__ u64 key(u32 i) const { return text8(T, n, n - 1 - i); }
    __device__ __forceinline__ u32 pos(u32 i) const { return n - 1 - i; }
};
struct SegRound {                                        // one oversized group of a round
    const u32 *key2, *sa;
    __device__ __forceinline__ u64 key(u32 i) const { return key2[i]; }
    __device__ __forceinline__ u32 pos(u32 i) const { return sa[i]; }
};

// sort keys of a round batch: (head slot of the group - base, key2)
struct SrcBatch {
    const u32 *rank, *key2, *sa; u32 base;
    __device__ __forceinline__ u64 key(u32 e) const { return ((u64)(rank[sa[e]] - 1u - base) << 32) | key2[e]; }
    __device__ __forceinline__ u32 val(u32 e) const { return sa[e]; }
};

// the entries of a segment whose key is `val` (more than a batch of them): already one group, written unsorted to their slots.
// Initial segment: suffixes shorter than 8 bytes come first (largest positions first) and are groups of their own.
template <class Seg, bool INIT> struct PickValue {
    Seg s; u64 val; u32 *out; u32 *rank; u32 head; u32 n;     // head = 1 + slot of the range's first entry
    __device__ __forceinline__ bool pred(u32 i) const { return s.key(i) == val; }
    __device__ __forceinline__ void emit(u32 i, u32 x) const {
        const u32 p = s.pos(i);
        out[x] = p;
        u32 r = head;
        if (INIT) {
            if ((u64)p + 8 > n) r = head + x;
            else for (u32 e = 0; e < 7 && e < n; ++e) r += (s.key(e) == val);   // entries 0..6 are the short suffixes
        }
        rank[p] = r;
    }
};

// after a segment is sorted: its slots that are not singleton groups, into the active list
struct PickActive {
    const u32 *sa, *rank; u32 slot0, left; u32 *sa_out, *idx_out;      // sa: the segment's positions from slot0 on, `left` of them
    __device__ __forceinline__ bool pred(u32 j) const {
        const u32 s = slot0 + j;
        if (rank[sa[j]] - 1u != s) return true;             // not the head of its group
        return j + 1 < left && rank[sa[j + 1]] - 1u == s;   // a head whose group goes on
    }
    __device__ __forceinline__ void emit(u32 j, u32 x) const { sa_out[x] = sa[j]; idx_out[x] = slot0 + j; }
};

__global__ void __launch_bounds__(256) bb_iota(u32 *__restrict__ a, u32 cnt, u32 first)
{
    const u32 t = blockIdx.x * 256 + threadIdx.x;
    if (t < cnt) a[t] = first + t;
}

// last (LAST) or first group start among active entries [lo, hi) -> atomicMax / atomicMin on *out
template <bool LAST>
__global__ void __launch_bounds__(256) bb_find_start(const u32 *__restrict__ sa, const u32 *__restrict__ idx, const u32 *__restrict__ rank, u32 lo, u32 hi, u32 *out)
{
    u32 best = LAST ? 0u : 0xffffffffu;
    for (u32 i = lo + blockIdx.x * 256 + threadIdx.x; i < hi; i += gridDim.x * 256)
        if (rank[sa[i]] - 1u == idx[i]) best = LAST ? max(best, i) : min(best, i);
    best = LAST ? __reduce_max_sync(0xffffffffu, best) : __reduce_min_sync(0xffffffffu, best);
    if ((threadIdx.x & 31) == 0) { if (LAST) atomicMax(out, best); else atomicMin(out, best); }
}

struct Batched : KeyCuts {
    u8 *T; u32 n;
    u32 *rank, *sa, *idx, *key2, *ib;
    u64 *k[2]; u32 *v[2];
    void *scratch;

    // Sort a segment of `cnt` entries whose slots start at `slot0` and split it into groups; its positions in slot order go to
    // out[0..cnt).  Then its unsorted groups are appended to the active list at *m_out.  Returns false on an inconsistency.
    template <bool INIT, class Seg> bool segment(const Seg &s, u32 cnt, int KB, u32 slot0, u32 *out, u32 &m_out) {
        std::vector<Range> R;
        if (!cut(s, cnt, KB, R)) return false;
        for (const Range &r : R) {
            if (r.count > B) {                               // one key value, one group
                if (compact(PickValue<Seg, INIT>{s, r.lo, out + r.cum, rank, 1 + slot0 + r.cum, n}, cnt) != r.count) return false;
                continue;
            }
            if (compact(PickRange<Seg>{s, r.lo, r.hi, k[1], v[1]}, cnt) != r.count) return false;
            const int bits = r.lo == r.hi ? 0 : 64 - __builtin_clzll(r.lo ^ r.hi);
            int cur = 1;
            if (bits) cur = rs_sort<u64, true>(ctx, SrcArray<u64, true>{k[1], v[1]}, k, v, r.count, make_passes(0, bits), scratch);
            CUDA_TRY(cudaMemcpyAsync(out + r.cum, v[cur], (size_t)r.count * 4, cudaMemcpyDeviceToDevice, ctx->stream));
            LAUNCH(ctx, bb_iota, ceil_div(r.count, 256), 256, 0, ib, r.count, slot0 + r.cum);
            split<INIT>(k[cur], v[cur], r.count, (u32 *)k[cur ^ 1], (u32 *)k[cur ^ 1] + B, v[cur ^ 1]);
        }
        // the segment's unsorted groups -> active list, B slots at a time through ib (the writes never pass the reads: see below)
        for (u32 c0 = 0; c0 < cnt; c0 += B) {
            const u32 left = cnt - c0, take = min(left, B + 1);
            CUDA_TRY(cudaMemcpyAsync(ib, out + c0, (size_t)take * 4, cudaMemcpyDeviceToDevice, ctx->stream));
            m_out += compact(PickActive{ib, rank, slot0 + c0, left, sa + m_out, idx + m_out}, min(left, B));
        }
        return true;
    }

    // split sorted (key, position) pairs whose slots are in ib into groups: rank[] only (the compacted outputs go to scratch)
    template <bool INIT> void split(const u64 *key, const u32 *pos, u32 cnt, u32 *sa_out, u32 *idx_out, u32 *grp_out) {
        const u32 tiles = ceil_div(cnt, SC_TILE);
        LAUNCH(ctx, (bwt_tile_reduce<INIT, true>), tiles, SC_THREADS, 0, key, pos, ib, cnt, n, agg);
        LAUNCH(ctx, bwt_tile_scan, 1, 1024, 0, agg, tiles, ctx->d_mail);
        LAUNCH(ctx, (bwt_apply<INIT, true>), tiles, SC_THREADS, 0, key, pos, ib, cnt, n, agg, rank, sa_out, idx_out, grp_out);
    }

    u32 find_start(bool last, u32 lo, u32 hi) {
        if (lo >= hi) return last ? 0u : 0xffffffffu;
        CUDA_TRY(cudaMemsetAsync(ctx->d_mail, last ? 0x00 : 0xff, 4, ctx->stream));
        if (last) LAUNCH(ctx, bb_find_start<true>, grid_for(hi - lo), 256, 0, sa, idx, rank, lo, hi, ctx->d_mail);
        else      LAUNCH(ctx, bb_find_start<false>, grid_for(hi - lo), 256, 0, sa, idx, rank, lo, hi, ctx->d_mail);
        ctx->fetch_mail(1);
        return ctx->h_mail[0];
    }
    u32 peek(const u32 *p) {
        CUDA_TRY(cudaMemcpyAsync(ctx->h_mail, p, 4, cudaMemcpyDeviceToHost, ctx->stream));
        ctx->sync();
        return ctx->h_mail[0];
    }

    // one doubling round over the m active entries; returns the new number of active entries (or -1)
    long long round(u32 m, u32 h) {
        LAUNCH(ctx, bwt_gather_key2, ceil_div(m, 256), 256, 0, sa, rank, key2, m, n, h);
        const int bits_k2 = bits_for(n);
        u32 out = 0;
        for (u32 b0 = 0; b0 < m; ) {
            u32 c = m;
            if (m - b0 > B) c = find_start(true, b0 + 1, b0 + B + 1);
            if (c > b0) {                                    // whole groups [b0, c), at most B entries
                const u32 cnt = c - b0, base = peek(idx + b0), span = peek(idx + c - 1) - base;
                CUDA_TRY(cudaMemcpyAsync(ib, idx + b0, (size_t)cnt * 4, cudaMemcpyDeviceToDevice, ctx->stream));
                const int cur = rs_sort<u64, true>(ctx, SrcBatch{rank, key2 + b0, sa + b0, base}, k, v, cnt,
                                                   make_passes(0, bits_k2, 32, 32 + bits_for(span)), scratch);
                const u32 tiles = ceil_div(cnt, SC_TILE);
                LAUNCH(ctx, bwt_tile_reduce<false>, tiles, SC_THREADS, 0, k[cur], v[cur], ib, cnt, n, agg);
                LAUNCH(ctx, bwt_tile_scan, 1, 1024, 0, agg, tiles, ctx->d_mail);
                LAUNCH(ctx, bwt_apply<false>, tiles, SC_THREADS, 0, k[cur], v[cur], ib, cnt, n, agg, rank, sa + out, idx + out, (u32 *)k[cur ^ 1]);
                ctx->fetch_mail(1);
                out += ctx->h_mail[0];
            } else {                                         // one group of more than B entries
                const u32 e0 = find_start(false, b0 + B + 1, m);
                c = e0 == 0xffffffffu ? m : e0;
                if (!segment<false>(SegRound{key2 + b0, sa + b0}, c - b0, 32, peek(idx + b0), idx + b0, out)) return -1;
            }
            b0 = c;
        }
        return out;
    }
};

}  // namespace

size_t bwt_batched_bytes(u32 n, u32 B)
{
    auto piece = [](size_t count, size_t size) { return align_up(count * size + 256, 256); };    // Arena::get's rounding
    return 4 * piece((size_t)n + 1, 4) + piece(ceil_div(n, SC_TILE), sizeof(TileAgg)) + piece(65536, 4)
         + 2 * piece(B, 8) + 2 * piece(B, 4) + piece((size_t)B + 1, 4) + piece(rs_scratch_bytes(B, RS_MAX_PASSES), 1);
}

// Each key range, each oversized key value and each histogram level scans its whole segment once, and a segment is cut into a few
// ranges per B entries.  So a segment of S entries costs O(S * S / B) work: B >= n / 64 keeps that to a bounded number of passes over
// the block whatever the budget.
u32 bwt_batch_floor(u32 n) { const u32 f = n / BWT_BATCH_FLOOR_DIV; return f > 65536 ? f : 65536; }

u32 bwt_batch_entries(u32 n, long long budget)
{
    const long long fixed = (long long)bwt_batched_bytes(n, 0), per = 32;   // per entry: keys 2 x 8, values 2 x 4, slots 4, look-back 4
    long long b = budget > fixed ? (budget - fixed) / per : 0;
    if (b > (long long)n) b = n;
    const u32 floor = bwt_batch_floor(n);
    return b < (long long)floor ? floor : (u32)b;
}

// Forward BWT of d_T[0..n) in place, sorting in batches of at most B entries.  Same results as stage_bwt_encode.
int stage_bwt_encode_batched(Ctx *ctx, u8 *d_T, int n_, unsigned char *num_indexes, int *indexes, u32 B)
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
    if (B < bwt_batch_floor(n)) B = bwt_batch_floor(n);

    Arena &A = ctx->sort_arena();
    const size_t mark = A.mark();
    Batched S;
    S.ctx = ctx; S.T = d_T; S.n = n; S.B = B;
    S.rank = A.get<u32>((size_t)n + 1); S.sa = A.get<u32>((size_t)n + 1); S.idx = A.get<u32>((size_t)n + 1); S.key2 = A.get<u32>((size_t)n + 1);
    S.agg = A.get<TileAgg>(ceil_div(n, SC_TILE));
    S.hist = A.get<u32>(65536);
    S.k[0] = A.get<u64>(B); S.k[1] = A.get<u64>(B); S.v[0] = A.get<u32>(B); S.v[1] = A.get<u32>(B);
    S.ib = A.get<u32>((size_t)B + 1);
    S.scratch = A.get<u8>(rs_scratch_bytes(B, RS_MAX_PASSES));
    S.h_hist.resize(65536);

    // 1. initial sort by the first 8 bytes: idx[] holds the sorted positions until they are compacted into sa[] / idx[]
    u32 m = 0;
    if (!S.segment<true>(SegText{d_T, n}, n, 64, 0, S.idx, m)) { A.release(mark); return LIBBSC_GPU_ERROR; }

    // 2. doubling rounds.  The last round needed is h = 2^30: no group survives a round with h >= n, and n < 2^31.
    for (u64 h = 8; m > 0; h <<= 1) {
        if (h >= ((u64)1 << 31)) { A.release(mark); return LIBBSC_GPU_ERROR; }
        const long long next = S.round(m, (u32)h);
        if (next < 0) { A.release(mark); return LIBBSC_GPU_ERROR; }
        m = (u32)next;
    }

    // 3. emit: L goes to key2 (free now) and then over the text
    u8 *L = (u8 *)S.key2;
    LAUNCH(ctx, bwt_emit, ceil_div(n, 256), 256, 0, d_T, S.rank, L, n);
    CUDA_TRY(cudaMemcpyAsync(d_T, L, n, cudaMemcpyDeviceToDevice, ctx->stream));
    u32 cnt = want_aux ? (n - 1) / r : 0;
    LAUNCH(ctx, bwt_emit_indexes, 1, 256, 0, S.rank, n, r ? r : 1u, cnt, ctx->d_mail);
    ctx->fetch_mail(1 + (int)cnt);
    int index = (int)ctx->h_mail[0];
    if (want_aux) {
        *num_indexes = (unsigned char)cnt;
        for (u32 t = 0; t < cnt; ++t) indexes[t] = (int)ctx->h_mail[1 + t];
    }
    A.release(mark);
    return index;
}
