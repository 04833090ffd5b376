// libbsc_b200/csrc/qlfc_encoder.cuh -- QLFC stage 2 ENCODER as a five-warp pipeline.
// Included by qlfc.cu after qlfc_coder.cuh (uses CoderSmem, the counter-file layout, Rc2Enc).
//
// Facts this design rests on (qlfc.cpp:829-1129):
//   * every model context is a function of the INPUT (symbols, ranks, run lengths) only -- never of
//     the coder state -- so probabilities can be produced ahead of the range coder;
//   * a probability is a weighted sum of THREE counters (by state, by symbol, shared) and each counter
//     moves as a function of its own value and the coded bit only -- never of the mixed probability --
//     so the three counter files evolve independently of each other;
//   * the four decision groups of a run -- rank first-bit + exponent, rank mantissa (or escape),
//     run-length first-bit + exponent, run-length mantissa -- use disjoint counter arrays, so four
//     different warps can evaluate them without any ordering between them;
//   * the only truly serial recurrence is the range coder (range/low, rangecoder.h:83-177).
//
//   warp 0..3  "model" : 32 decisions of this warp's group at a time, one lane per decision
//   warp 4     "coder" : consumes the (bit, p) records in stream order from a shared-memory ring
//
// Work is organised in batches of (up to) 32 runs.  The per-run CONTEXTS are computed one lane per run
// ("vector prologue"): sliding-window contexts come from warp ballots, the per-symbol histories from
// match_any chains, avgRank from a 32-step serial integer loop, ring offsets from a warp scan, and
// the state-table look-ups are one vector shared-memory load.  Then each model warp flattens the
// decisions of its group over the whole batch and evaluates them 32 at a time, one lane per DECISION:
// decisions that hit the same counter inside a chunk are ordered by __match_any_sync and resolved in
// occurrence order (usually a single round), separately for each of the three counter kinds.
//
// All model warps derive the ring position of every decision from the same arithmetic (the number of
// decisions of a run follows from rank, run length, maxRank and the escape flag), so they never talk
// to each other; the coder consumes up to the minimum of the four progress counters.  A batch is cut
// short so that its records never exceed half the ring.
//
// The critical model warp's instruction count per run fell with each step -- one warp doing everything, two model warps, a
// vector prologue, four model warps with a lane per decision of one run, a lane per decision of 32 runs (this file) -- until
// the range-coder warp became the limit.
#pragma once

#define QE_RING 1024
#define QE_BIT  0x2000u                                     // record: bits 0..12 p, bit 13 the coded bit, bit 14 run start
#define QE_RUN  0x4000u
#define QE_MODELS 4
#define QE_THREADS ((QE_MODELS + 2) * 32)
#ifdef QE_DIAG      // where does each warp spend its time?  (nvcc -DQE_DIAG; prints for sub-block 0)
#define QE_DIAG_DECL long long dg_wait = 0, dg_t0 = 0, dg_start = clock64();
#define QE_DIAG_T0 dg_t0 = clock64();
#define QE_DIAG_T1 dg_wait += clock64() - dg_t0;
#define QE_DIAG_END(name) if (sid == 0 && lane == 0) printf("%s warp %u: total %lld waiting %lld\n", name, warp, clock64() - dg_start, dg_wait);
#define QE_DIAG_ROUNDS(k) , dg_rounds[k]
#define QE_DIAG_ROUNDS_PARAM , unsigned long long &dg_r
#define QE_DIAG_ROUNDS_ADD dg_r += maxocc + 1;
#else
#define QE_DIAG_ROUNDS(k)
#define QE_DIAG_ROUNDS_PARAM
#define QE_DIAG_ROUNDS_ADD
#define QE_DIAG_DECL
#define QE_DIAG_T0
#define QE_DIAG_T1
#define QE_DIAG_END(name)
#endif

struct EncPipe {
    alignas(16) u32 ring[QE_RING];                          // model warps: record; after the range warp: the addend of `low`
    alignas(16) int prm[7][2][12];                          // [class][bit] = w0 w1 w2 | Ms Ks | Mc Kc | Mg Kg
    volatile u32 prog[QE_MODELS], done[QE_MODELS];          // records completed by each model warp / its end flag
    volatile u32 mid, mid_done, final_range;                // records passed through the range warp / its end flag / range at the end
    volatile u32 head;                                      // records consumed by the low warp (ring space free again)
    volatile u32 hdr_len, hdr_ready, max_rank;              // published by warp 0 after the stream header
    volatile u32 fail;
    u8  hist2[2][256];                                      // private history copies of warps 1 and 3 (warps 0, 2 use CoderSmem's)
};

// parameters of one decision class for one outcome, in the (p*M + K) >> 12 form of the counter moves
__device__ __forceinline__ void enc_fill_params(EncPipe &P, u32 lane)
{
    for (int i = lane; i < 14; i += 32) {
        const int k = i >> 1, b = i & 1;
        int *q = P.prm[k][b];
        q[0] = bscb_param(k, 0); q[1] = bscb_param(k, 1); q[2] = bscb_param(k, 2);
        for (int who = 0; who < 3; ++who) {
            const int th0 = bscb_param(k, 3 + 4 * who), ar0 = bscb_param(k, 4 + 4 * who), th1 = bscb_param(k, 5 + 4 * who), ar1 = bscb_param(k, 6 + 4 * who);
            q[3 + 2 * who] = b ? 4096 - ar1 : 4096 - ar0;
            q[4 + 2 * who] = b ? th1 * ar1 + 4095 : (4096 - th0) * ar0;
        }
        q[9] = q[10] = q[11] = 0;
    }
}

// One counter kind of one chunk of decisions.  Lane `act` uses counter S.s16[x] (or, when `cached`, the
// rare counter `key` through this kind's direct-mapped write-back cache): returns the counter's value
// BEFORE this lane's decision and applies the move (v*M + Kc) >> 12.  Lanes that share a counter -- or
// a cache slot -- are served in lane (= stream) order, one per round.
template <class LY, int KIND>   // 0 by state, 1 by symbol, 2 shared (never cached)
__device__ __forceinline__ int enc_resolve(CoderSmemT<LY> &S, bool act, u32 x, bool cached, u32 key, int M, int Kc, short *__restrict__ cold, u32 lane, u32 &misses QE_DIAG_ROUNDS_PARAM)
{
    u16 *tags = KIND == 0 ? S.tag_state : S.tag_char;
    const u32 vbase = KIND == 0 ? LY::C_STATE_VAL : LY::C_CHAR_VAL;
    if (KIND != 2 && cached) x = vbase + LY::cache_slot(key);
    const u32 m = __match_any_sync(0xffffffffu, act ? x : (0x80000000u | lane));
    const u32 below = m & lanemask_lt();
    const u32 occ = __popc(below);
    const u32 maxocc = __reduce_max_sync(0xffffffffu, act ? occ : 0u);
    const u32 prevl = below ? 31u - (u32)__clz(below) : lane;      // the previous user of my counter
    int v = 0;
    QE_DIAG_ROUNDS_ADD
    // two different rare counters on one cache slot inside a chunk (very rare): take turns through shared memory
    bool clash = false;
    if (KIND != 2) { const u32 pk = __shfl_sync(0xffffffffu, key, prevl); clash = __any_sync(0xffffffffu, act && cached && below && pk != key); }
    if (!clash) {
        // The first user of a counter reads it, the value then travels down the chain of users by shuffles,
        // the last one writes it back: one round per link, no shared-memory round trip in between.
        if (act && occ == 0) {
            if (KIND != 2 && cached) {
                const u32 slot = x - vbase, t = tags[slot];
                if (t != LY::cache_tag(key)) {
                    if (t) cold[LY::cache_unslot(slot, t)] = (short)S.s16[x];
                    S.s16[x] = (u16)cold[key]; tags[slot] = (u16)LY::cache_tag(key); ++misses;
                }
            }
            v = S.s16[x];
        }
        int vn = (v * M + Kc) >> 12;
        for (u32 round = 1; round <= maxocc; ++round) {
            const int t = __shfl_sync(0xffffffffu, vn, prevl);
            if (occ == round) { v = t; vn = (v * M + Kc) >> 12; }
        }
        if (act && (m >> lane) == 1u) S.s16[x] = (u16)vn;
        __syncwarp();
        return v;
    }
    for (u32 round = 0; round <= maxocc; ++round) {
        if (act && occ == round) {
            if (KIND != 2 && cached) {
                const u32 slot = x - vbase, t = tags[slot];
                if (t != LY::cache_tag(key)) {
                    if (t) cold[LY::cache_unslot(slot, t)] = (short)S.s16[x];
                    S.s16[x] = (u16)cold[key]; tags[slot] = (u16)LY::cache_tag(key); ++misses;
                }
            }
            v = S.s16[x];
            S.s16[x] = (u16)((v * M + Kc) >> 12);
        }
        __syncwarp();
    }
    return v;
}

// bits [32-lane, ...) of (prev:cur): the flags of the runs before this lane's run, most recent in bit 0
__device__ __forceinline__ u32 enc_window(u32 prev_rev, u32 cur_rev, u32 lane) { return (u32)((((u64)prev_rev << 32) | cur_rev) >> (32u - lane)); }

// LY: layout of the counter file (qlfc_decoder6.cuh).  The product instantiates LayoutEncDiet: fewer mantissa rows resident, 106 KB
// + 5.6 KB of pipe state, so that two six-warp encoders share an SM (same time per stream as the 205 KB layout when alone).
// (A one-multiply-add form of the range recurrence was tried and was slower.)
// MINB: encoder CTAs per SM the REGISTER budget must allow (192 threads: 122 registers fit two CTAs, <= 112 three, <= 80 four)
template <class LY, int MINB> __global__ void __launch_bounds__(QE_THREADS, MINB) q_encode5(const u32 *__restrict__ run_pos, const u8 *__restrict__ run_sym, const u8 *__restrict__ run_rank,
                                                    SubBlock *__restrict__ sbs, const u8 *__restrict__ mtf_all, short *__restrict__ cold_all,
                                                    const QTables *__restrict__ tables, u8 *__restrict__ out_all, const u32 *__restrict__ sb_list, DoneSignal done)
{
    extern __shared__ __align__(16) u8 q_smem_raw[];
    CoderSmemT<LY> &S = *reinterpret_cast<CoderSmemT<LY> *>(q_smem_raw);
    EncPipe &P = *reinterpret_cast<EncPipe *>(q_smem_raw + ((sizeof(CoderSmemT<LY>) + 15) & ~(size_t)15));
    const u32 warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const u32 sid = sb_list ? sb_list[blockIdx.x] : blockIdx.x;
    SubBlock &sb = sbs[sid];

    if (warp == 0) coder_smem_init_t<LY>(S, tables);
    if (warp == 1) {
        enc_fill_params(P, lane);
        for (int i = lane; i < 512; i += 32) (&P.hist2[0][0])[i] = 0;
        if (lane < QE_MODELS) { P.prog[lane] = lane ? 0xffffffffu : 0u; P.done[lane] = 0; }
        if (lane == 0) { P.head = 0; P.hdr_len = 0; P.hdr_ready = 0; P.max_rank = 7; P.fail = 0; P.mid = 0; P.mid_done = 0; P.final_range = 0; }
    }
    __syncthreads();

    const u32 rb = sb.run_begin, re = sb.run_end;
    u8 *flg = S.inwin;                                         // 2 flags per record, 4 records per byte: bit k = renormalise before record k, bit 4+k = run start

    if (warp == QE_MODELS) {
        // ------------------------- range warp: the `range` recurrence only (rangecoder.h:83-177) -------------------------
        // Turns each record (bit, p) into the addend of `low` and a "renormalise first" flag, in place.
        u32 range = 0xffffffffu, h = 0;
        bool bad = false;
        QE_DIAG_DECL
        for (;;) {
            u32 limit, spins = 0;
            bool fin;
            QE_DIAG_T0
            for (;;) {
                fin = P.done[0] && P.done[1] && P.done[2] && P.done[3];          // read before the counters: then they are final
                limit = min(min(P.prog[0], P.prog[1]), min(P.prog[2], P.prog[3]));
                if (!fin) limit &= ~3u;                                        // whole groups of four until the very end
                if (limit != h || fin) break;
                if (P.fail || ++spins > (1u << 27)) { bad = true; break; }
            }
            QE_DIAG_T1
            if (bad || limit == h) break;
            __threadfence_block();
            if ((h & 3u) == 0 && limit - h >= 4u) {
                u32 groups = (limit - h) >> 2;
                uint4 q = *reinterpret_cast<const uint4 *>(&P.ring[h & (QE_RING - 1)]);
                for (; groups; --groups) {
                    const u32 slot = h & (QE_RING - 1);
                    uint4 nq = q;
                    if (groups > 1) nq = *reinterpret_cast<const uint4 *>(&P.ring[(h + 4) & (QE_RING - 1)]);    // prefetch the next group
                    u32 recs[4] = {q.x, q.y, q.z, q.w}, f = 0;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        const u32 rec = recs[k];
                        const bool sh = range < 0x10000u;
                        const bool bit = rec & QE_BIT;
                        if (sh) range <<= 16;
                        const u32 r = (range >> 12) * (rec & 0x1fffu);
                        range = bit ? range - r : r;
                        recs[k] = bit ? r : 0u;
                        f |= (sh ? 1u << k : 0u) | ((rec & QE_RUN) ? 16u << k : 0u);
                    }
                    *reinterpret_cast<uint4 *>(&P.ring[slot]) = make_uint4(recs[0], recs[1], recs[2], recs[3]);
                    if (lane == 0) flg[slot >> 2] = (u8)f;
                    h += 4; q = nq;
                }
            }
            while (h != limit) {                                               // the last few records of the stream
                const u32 slot = h & (QE_RING - 1);
                const u32 rec = P.ring[slot], k = h & 3u;
                const bool sh = range < 0x10000u;
                if (sh) range <<= 16;
                const u32 r = (range >> 12) * (rec & 0x1fffu);
                const bool bit = rec & QE_BIT;
                range = bit ? range - r : r;
                u32 f = k ? flg[slot >> 2] : 0u;
                f |= (sh ? 1u << k : 0u) | ((rec & QE_RUN) ? 16u << k : 0u);
                __syncwarp();
                if (lane == 0) { P.ring[slot] = bit ? r : 0u; flg[slot >> 2] = (u8)f; }
                __syncwarp();
                ++h;
            }
            __syncwarp();
            __threadfence_block();
            if (lane == 0) P.mid = h;
        }
        __syncwarp();
        __threadfence_block();
        QE_DIAG_END("range")
        if (lane == 0) { P.final_range = range; P.mid = h; if (bad && !P.fail) P.fail = 2; __threadfence_block(); P.mid_done = 1; }
        return;
    }
    if (warp == QE_MODELS + 1) {
        // ------------------------- low warp: carries, output units and the end-of-buffer rule -------------------------
        Rc2Enc rc; rc.init(out_all + sb.out_off);
        const long long eob = (long long)sb.out_cap - 16;
        u32 h = 0; int result = 0; bool eob_hit = eob <= 0;
        QE_DIAG_DECL
        for (;;) {
            u32 limit, spins = 0;
            QE_DIAG_T0
            for (;;) {
                limit = P.mid;
                if (limit != h) break;
                if (P.mid_done && P.mid == h) break;
                if (P.fail == 2 || ++spins > (1u << 27)) { result = LIBBSC_GPU_ERROR; break; }
            }
            QE_DIAG_T1
            if (result || limit == h) break;
            __threadfence_block();
            while (h != limit) {
                const u32 slot = h & (QE_RING - 1);
                if (!eob_hit && (h & 3u) == 0 && limit - h >= 4u) {
                    // fast path: four records per 128-bit shared-memory load, no end-of-buffer test.  The
                    // test of qlfc.cpp:898-901 can only start to matter after a renormalisation moved the
                    // write position past the limit; from then on the checked path below takes over.
                    u32 groups = (limit - h) >> 2;
                    uint4 q = *reinterpret_cast<const uint4 *>(&P.ring[slot]);
                    u32 f = flg[slot >> 2];
                    for (; groups && !eob_hit; --groups) {
                        uint4 nq = q; u32 nf = f;
                        if (groups > 1) {                             // prefetch the next group
                            const u32 ns = (h + 4) & (QE_RING - 1);
                            nq = *reinterpret_cast<const uint4 *>(&P.ring[ns]); nf = flg[ns >> 2];
                        }
                        if (__builtin_expect((f & 15u) == 0, 1)) {    // no renormalisation inside the group: just add
                            rc.low += ((u64)q.x + q.y) + ((u64)q.z + q.w);
                            h += 4;
                        } else {
                            u32 a0 = q.x, a1 = q.y, a2 = q.z, a3 = q.w;
#pragma unroll 1
                            for (u32 k = 0, ff = f; k < 4; ++k, ff >>= 1) {
                                ++h;
                                if (ff & 1u) { rc.shift(); eob_hit = (long long)rc.pos >= eob; }
                                rc.low += a0; a0 = a1; a1 = a2; a2 = a3;
                                if (eob_hit) break;
                            }
                        }
                        if (lane == 0 && (h & 63u) == 0) P.head = h;
                        q = nq; f = nf;
                    }
                    continue;
                }
                const u32 a = P.ring[slot], f = (u32)flg[slot >> 2] >> (h & 3u); ++h;
                if (eob_hit && (f & 16u)) { result = LIBBSC_NOT_COMPRESSIBLE; break; }        // qlfc.cpp:898-901
                if (f & 1u) { rc.shift(); eob_hit = (long long)rc.pos >= eob; }
                rc.low += a;
            }
            if (lane == 0) P.head = h;
            if (result) break;
        }
        QE_DIAG_END("low")
        if (result == 0) {
            for (u32 spins = 0; !P.mid_done; ) if (++spins > (1u << 27)) { result = LIBBSC_GPU_ERROR; break; }
            __threadfence_block();
            rc.range = P.final_range;
            if (result == 0 && P.fail == 2) result = LIBBSC_GPU_ERROR;
            if (result == 0) result = (int)rc.finish();
        }
        __syncwarp();
        if (lane == 0) { if (result < 0 && P.fail == 0) P.fail = 1; sb.result = result; signal_done(done); }   // the stream's bytes are all written by this (LOW) warp
        return;
    }

    // ------------------------------------------ model warps ------------------------------------------
    const bool rank_side = warp < 2;                          // warps 0,1: rank decisions; warps 2,3: run-length decisions
    u8 *my_hist = warp == 0 ? S.rankHist : warp == 2 ? S.runHist : warp == 1 ? P.hist2[0] : P.hist2[1];
    short *cold_s = cold_all + (size_t)sid * 2 * COLD_PAD, *cold_c = cold_s + COLD_PAD;
    u32 n_cached = 0, misses = 0;
    u32 maxRank = 7;
    u32 base_off = 0;                                          // ring position (record index) of the current batch of runs

    u32 head_seen = 0;
    bool stop = false;
    if (warp == 0) {
        // ----------------------- stream header: n as 32 raw bits, then the MTF order (qlfc.cpp:851-891) -----------------------
        // Warps 1..3 keep their progress counters at "infinity" meanwhile, so the coder follows warp 0 alone.
        const u32 n = sb.in_size;
        P.ring[lane] = 2048u | (((n >> (31 - lane)) & 1u) ? QE_BIT : 0u);
        u32 off = 32;
        {
            const u8 *mtf = mtf_all + sid * 256;
            u32 used8 = 0; int prev = -1;
            for (int d = 0; d < 256 && !stop; ++d) {
                const int c = mtf[d];
                for (int bit = 7; bit >= 0; --bit) {
                    bool can0, can1; header_options(used8, prev, c >> (bit + 1), bit, can0, can1);
                    if (can0 && can1) {
                        if (off - head_seen >= QE_RING) {       // the header can be longer than the ring: hand over what is there
                            __syncwarp();
                            __threadfence_block();
                            if (lane == 0) P.prog[0] = off;
                            for (u32 spins = 0; off - (head_seen = P.head) >= QE_RING; ) if (P.fail || ++spins > (1u << 26)) { if (!P.fail) P.fail = 2; stop = true; break; }
                            if (stop) break;
                        }
                        if (lane == 0) P.ring[off & (QE_RING - 1)] = 2048u | (((c >> bit) & 1) ? QE_BIT : 0u);
                        ++off;
                    }
                }
                if (c == prev) { maxRank = (u32)ilog2_dev((u32)(d - 1)); break; }
                prev = c; if ((u32)(c >> 3) == lane) used8 |= 1u << (c & 7);
            }
        }
        base_off = off;
        __syncwarp();
        __threadfence_block();
        if (lane == 0) { P.max_rank = maxRank; P.hdr_len = off; P.prog[0] = off; __threadfence_block(); P.hdr_ready = 1; }
        // nobody may publish beyond the header before every model warp has dropped from "infinity" to the header length
        for (u32 spins = 0; !stop && (P.prog[1] == 0xffffffffu || P.prog[2] == 0xffffffffu || P.prog[3] == 0xffffffffu); )
            if (P.fail || ++spins > (1u << 27)) { if (!P.fail) P.fail = 2; stop = true; }
    } else {
        for (u32 spins = 0; !P.hdr_ready; ) if (P.fail || ++spins > (1u << 27)) { if (!P.fail) P.fail = 2; stop = true; break; }
        __threadfence_block();
        maxRank = P.max_rank; base_off = P.hdr_len;
        __syncwarp();
        if (lane == 0) P.prog[warp] = base_off;
    }

    // ---- state carried from batch to batch ----
    QE_DIAG_DECL
#ifdef QE_DIAG
    unsigned long long dg_rounds[3] = {0, 0, 0}, dg_chunks = 0; long long dg_cyc = 0, dg_c0 = 0;
#endif
    u32 avg = 0;                                               // avgRank after the last run of the previous batch
    u32 pf0 = 0, plo = 0, phi = 0, prn = 0;                    // bit-reversed flag ballots of the previous batch

    for (u32 t0 = rb; t0 < re && !stop; ) {
        // ================= vector prologue: lane j <-> run t0 + j =================
        u32 cnt = min(32u, re - t0);
        bool live = lane < cnt;
        u32 sym = 256u + lane, rank = 1, len = 1;              // dead lanes: unique pseudo-symbols, no decisions
        if (live) { sym = run_sym[t0 + lane]; rank = run_rank[t0 + lane]; len = run_pos[t0 + lane + 1] - run_pos[t0 + lane]; }
        const u32 er = (u32)ilog2_dev(rank), eu = (u32)ilog2_dev(len), rank0 = rank - 1;
        u32 my_avg = 0;                                        // avgRank seen by this lane's run (qlfc.cpp:1048: serial integer recurrence)
        {
            u32 a = avg;
#pragma unroll 8
            for (u32 j = 0; j < 32; ++j) {
                const u32 r = __shfl_sync(0xffffffffu, rank, j);
                if (lane == j) my_avg = a;
                if (j < cnt) a = (a * 124u + r * 4u) >> 7;
            }
            avg = a;
        }
        const bool esc = my_avg >= 32u;
        const u32 nE = (!esc && rank != 1) ? (er - 1) + (er < maxRank ? 1u : 0u) : 0u;
        const u32 nM = esc ? maxRank + 1u : (rank != 1 ? er : 0u);
        u32 nA = live ? (esc ? 0u : 1u) + nE + nM : 0u;
        u32 nB = live ? 1u + (len != 1 ? 2u * eu : 0u) : 0u;
        u32 incl = nA + nB;                                    // ring offsets: exclusive warp scan of the decision counts
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const u32 t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (u32)o) incl += t; }
        const u32 my_off = incl - (nA + nB);
        u32 batch_total = __shfl_sync(0xffffffffu, incl, 31);
        if (batch_total > QE_RING / 2) {                       // long runs: cut the batch so that its records fit half the ring
            cnt = (u32)__popc(__ballot_sync(0xffffffffu, live && incl <= QE_RING / 2));   // >= 1: a run has at most 78 decisions
            avg = __shfl_sync(0xffffffffu, my_avg, cnt);       // cnt < 32 here; nothing before this point had side effects
            batch_total = __shfl_sync(0xffffffffu, incl, cnt - 1);
            live = lane < cnt;
            if (!live) { sym = 256u + lane; nA = nB = 0; }
        }
        // sliding-window contexts (qlfc.cpp:1123-1125) from ballots; most recent run in the low bits
        const u32 q3 = rank0 < 3 ? rank0 : 3;
        const u32 bf0 = __brev(__ballot_sync(0xffffffffu, live && rank0 == 0));
        const u32 blo = __brev(__ballot_sync(0xffffffffu, live && (q3 & 1u))), bhi = __brev(__ballot_sync(0xffffffffu, live && (q3 & 2u)));
        const u32 brn = __brev(__ballot_sync(0xffffffffu, live && len < 3));
        const u32 sh = 32u - cnt;                              // a short batch shifts less history out of the windows
        const u32 ctxRank0 = enc_window(pf0, bf0, lane) & 7u, ctxRun = enc_window(prn, brn, lane) & 15u;
        const u32 wl = enc_window(plo, blo, lane) & 15u, wh = enc_window(phi, bhi, lane) & 15u;
        const u32 ctxRank4 = (wl & 1u) | ((wh & 1u) << 1) | ((wl & 2u) << 1) | ((wh & 2u) << 2) | ((wl & 4u) << 2) | ((wh & 4u) << 3) | ((wl & 8u) << 3) | ((wh & 8u) << 4);
        // carry: the flags of the last 32 runs, most recent in bit 0 (for a full batch this is just the new ballot)
        pf0 = (u32)(((((u64)pf0 << 32) | bf0) >> sh)); plo = (u32)(((((u64)plo << 32) | blo) >> sh));
        phi = (u32)(((((u64)phi << 32) | bhi) >> sh)); prn = (u32)(((((u64)prn << 32) | brn) >> sh));
        // per-symbol histories: value left by the previous run of the same symbol
        const u32 same = __match_any_sync(0xffffffffu, sym);
        const u32 below = same & lanemask_lt();
        const u32 prevl = below ? 31u - (u32)__clz(below) : lane;
        const bool last_of_sym = live && (same >> lane) == 1u;   // no later run of this symbol in the batch
        u32 my_st;
        if (rank_side) {
            const u32 er_prev = __shfl_sync(0xffffffffu, er, prevl);
            const u32 rh = below ? er_prev : (u32)my_hist[sym & 255u];             // rankHistory = exponent of the previous rank (0 for rank 1)
            { const u32 ti = (ctxRun << 11) | (ctxRank4 << 3) | rh; my_st = LY::TG ? (u32)__ldg(tables->rank_state + ti) : (u32)S.rank_state[LY::TG ? 0 : ti]; }
            __syncwarp();
            if (last_of_sym) my_hist[sym] = (u8)er;
        } else {
            const u32 occ = __popc(below), maxocc = __reduce_max_sync(0xffffffffu, live ? occ : 0u);
            u32 vin = my_hist[sym & 255u], vout = 0;
            for (u32 round = 0; round <= maxocc; ++round) {       // resolve same-symbol chains in occurrence order
                const u32 t = __shfl_sync(0xffffffffu, vout, prevl);
                if (occ == round) { if (round) vin = t; vout = (len == 1) ? (vin + 2u) >> 2 : (vin + 3u * eu + 3u) >> 2; }
            }
            { const u32 ti = (ctxRank0 << 10) | (ctxRun << 6) | ((rank0 < 7 ? rank0 : 7u) << 3) | (vin < 7 ? vin : 7u); my_st = LY::TG ? (u32)__ldg(tables->run_state + ti) : (u32)S.run_state[LY::TG ? 0 : ti]; }
            __syncwarp();
            if (last_of_sym) my_hist[sym] = (u8)vout;
        }
        const u32 pack = er | (eu << 3) | ((esc ? 1u : 0u) << 8) | (nE << 9) | (nM << 12);
        // this warp's group: number of decisions per run, and where they sit inside the run's records
        u32 gcnt, gpos;
        if (warp == 0)      { gcnt = esc ? 0u : 1u + nE;               gpos = 0; }
        else if (warp == 1) { gcnt = nM;                               gpos = esc ? 0u : 1u + nE; }
        else if (warp == 2) { gcnt = len != 1 ? 1u + eu : 1u;          gpos = nA; }
        else                { gcnt = len != 1 ? eu : 0u;               gpos = nA + 1u + eu; }
        if (!live) gcnt = 0;
        u32 gincl = gcnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const u32 t = __shfl_up_sync(0xffffffffu, gincl, o); if (lane >= (u32)o) gincl += t; }
        const u32 goff = gincl - gcnt, gtotal = __shfl_sync(0xffffffffu, gincl, 31);
        const u32 rpos = my_off + gpos;                        // batch-relative record index of this run's first decision of the group
        const u32 val = rank_side ? rank : len;
        __syncwarp();

        // room in the ring for the whole batch (re-read the consumer's head only when needed)
        QE_DIAG_T0
        for (u32 spins = 0; (int)(base_off + batch_total - head_seen) > QE_RING; ) {
            head_seen = P.head;
            if (P.fail || ++spins > (1u << 26)) { if (!P.fail) P.fail = 2; stop = true; break; }
        }
        QE_DIAG_T1
        if (stop) break;

        // ================= 32 decisions of this warp's group at a time, one lane per decision =================
#ifdef QE_DIAG
        dg_c0 = clock64(); dg_chunks += (gtotal + 31) / 32;
#endif
        for (u32 cb = 0; cb < gtotal; cb += 32) {
            const u32 g = cb + lane;
            const bool act = g < gtotal;
            u32 r = 0;                                         // the run of decision g: largest r with goff[r] <= g
#pragma unroll
            for (u32 step = 16; step; step >>= 1) { const u32 v = __shfl_sync(0xffffffffu, goff, r + step); if (v <= g) r += step; }
            const u32 c = __shfl_sync(0xffffffffu, sym, r) & 255u, v_ = __shfl_sync(0xffffffffu, val, r);
            const u32 pk = __shfl_sync(0xffffffffu, pack, r), st = __shfl_sync(0xffffffffu, my_st, r);
            const u32 rp = __shfl_sync(0xffffffffu, rpos, r), go = __shfl_sync(0xffffffffu, goff, r);
            const u32 d = act ? g - go : 0u;
            const u32 r_er = pk & 7u, r_eu = (pk >> 3) & 31u;
            const bool r_esc = (pk >> 8) & 1u;
            int K; u32 bit, is, ic, ig, cs = 0, cc = 0; bool cached = false, runflag = false;
            if (warp == 0) {            // rank: first bit (d = 0) and unary exponent (d = 1..nE)
                const u32 k = d - 1; const bool isT = d == 0;
                K = isT ? K_RANK_T : K_RANK_E;
                bit = isT ? (v_ != 1) : (k + 1 < r_er);
                is = isT ? LY::R_RT_STATE + st : LY::R_RE_STATE + st * 8 + k;
                ic = isT ? LY::R_RT_CHAR + c : LY::R_RE_CHAR + c * 8 + k;
                ig = isT ? LY::R_RT_SHARED : LY::R_RE_SHARED + k;
                runflag = isT;
            } else if (warp == 1) {     // rank: mantissa tree of depth e (or the escape tree of depth maxRank+1)
                const u32 e_m = r_esc ? maxRank + 1u : r_er, v = r_esc ? (v_ | (1u << e_m)) : v_;
                const u32 bp = e_m - 1 - (d < e_m ? d : 0), node = v >> (bp + 1);
                const u32 bank = r_esc ? 8u : r_er;
                const u32 rowoff = (1u << r_er) - 2u + node;
                K = r_esc ? K_RANK_P : K_RANK_M;
                bit = (v >> bp) & 1u;
                cached = r_esc || r_er > LY::MAXE_R;
                is = LY::R_RM_STATE + st * LY::ROW_R + rowoff; ic = LY::R_RM_CHAR + c * LY::ROW_R + rowoff; ig = LY::R_WIDE_SHARED + bank * 256 + node;
                cs = wide_idx(bank, st, node); cc = wide_idx(bank, c, node);
                runflag = r_esc && d == 0;
            } else if (warp == 2) {     // run length: first bit (d = 0) and unary exponent (d = 1..eu)
                const u32 k = d - 1; const bool isT = d == 0;
                K = isT ? K_RUN_T : K_RUN_E;
                bit = isT ? (v_ != 1) : (k + 1 < r_eu);
                cached = !isT && k >= UE_RES;
                is = isT ? LY::R_UT_STATE + st : LY::R_UE_STATE + st * UE_RES + k;
                ic = isT ? LY::R_UT_CHAR + c : LY::R_UE_CHAR + c * UE_RES + k;
                ig = isT ? LY::R_UT_SHARED : LY::R_UE_SHARED + k;
                cs = ue_idx(st, k); cc = ue_idx(c, k);
            } else {                    // run length: mantissa (tree for exponents <= 5, linear contexts above; qlfc.cpp:1119)
                const u32 bp = r_eu - 1 - (d < r_eu ? d : 0);
                const bool tree = r_eu <= 5u;                                   // the FORMAT's rule (qlfc.cpp:1119), not a residency question
                const u32 node = tree ? (v_ >> (bp + 1)) : 1u + d;
                const u32 rowoff = (1u << r_eu) - 2u + node;
                K = K_RUN_M;
                bit = (v_ >> bp) & 1u;
                cached = LY::MAXE_U >= 5u ? !tree : r_eu > LY::MAXE_U;          // full layout: exactly the tree rows are resident
                is = LY::R_UM_STATE + st * LY::ROW_U + rowoff; ic = LY::R_UM_CHAR + c * LY::ROW_U + rowoff; ig = LY::R_NARROW_SHARED + r_eu * 32 + node;
                cs = narrow_idx(r_eu, st, node); cc = narrow_idx(r_eu, c, node);
            }
            cached = cached && act;
            if (__any_sync(0xffffffffu, cached)) n_cached += 2u * (u32)__popc(__ballot_sync(0xffffffffu, cached));
            const int4 *q = reinterpret_cast<const int4 *>(P.prm[K][bit & 1u]);
            const int4 qa = q[0], qb = q[1]; const int qg = P.prm[K][bit & 1u][8];
            const int vs = enc_resolve<LY, 0>(S, act, is, cached, cs, qa.w, qb.x, cold_s, lane, misses QE_DIAG_ROUNDS(0));
            const int vc = enc_resolve<LY, 1>(S, act, ic, cached, cc, qb.y, qb.z, cold_c, lane, misses QE_DIAG_ROUNDS(1));
            const int vg = enc_resolve<LY, 2>(S, act, ig, false, 0, qb.w, qg, nullptr, lane, misses QE_DIAG_ROUNDS(2));
            const u32 p = (u32)((vc * qa.x + vs * qa.y + vg * qa.z) >> 5);
            if (act) P.ring[(base_off + rp + d) & (QE_RING - 1)] = p | (bit ? QE_BIT : 0u) | (runflag ? QE_RUN : 0u);
        }
#ifdef QE_DIAG
        dg_cyc += clock64() - dg_c0;
#endif
        base_off += batch_total;
        __syncwarp();
        __threadfence_block();
        if (lane == 0) P.prog[warp] = base_off;
        if (P.fail) stop = true;
        t0 += cnt;
    }
    __syncwarp();
    __threadfence_block();
    if (lane == 0) { P.prog[warp] = base_off; P.done[warp] = 1; }
    QE_DIAG_END("model")
#ifdef QE_DIAG
    if (sid == 0 && lane == 0 && warp == 0) printf("records %u runs %u\n", base_off, re - rb);
    if (sid == 0 && lane == 0) printf("model warp %u: chunks %llu rounds s %llu c %llu g %llu, cycles in chunks %lld\n", warp, dg_chunks, dg_rounds[0], dg_rounds[1], dg_rounds[2], dg_cyc);
#endif
    misses = __reduce_add_sync(0xffffffffu, misses);
    if (lane == 0) { atomicAdd(&sb.stat_cached, n_cached); atomicAdd(&sb.stat_miss, misses); }
}
