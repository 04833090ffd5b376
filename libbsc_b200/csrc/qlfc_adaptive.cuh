// libbsc_b200/csrc/qlfc_adaptive.cuh -- the ADAPTIVE QLFC coder (coder id 2, `-e2`): encoder qlfc.cpp:463-823, decoder 1366-1666,
// ProbabilityMixer predictor.h:74-213, constants qlfc_model.h:38-113 (M_*), mixer arrays 225-231, start values
// qlfc_model.cpp:49-71, stretch / squash tables.h:38-558.  Included by qlfc.cu after qlfc_decoder6.cuh (uses its layout
// template, range-decoder step and prologue, the fast coder's range ENcoder, SM3 and the QD3_* dual-compile macros); ALSO
// compiled for the host by tools/qdec3_host.cpp and checked there against the oracle (tests/test_qdec3_host.py).
//
// The adaptive coder makes exactly the decisions of the static coder with exactly the same three counters per decision
// (other move constants); only the probability differs: the three counters are stretched, combined with per-context
// on-line weights, squashed, refined through a 17-point probability map, and weights and map learn from the coded bit.
// So a decision costs about three times the instructions of a static one, and the working set grows by 1896 mixers x 48 B
// and 16 KB of tables: counter file in the two-streams-per-SM layout of qlfc_decoder6.cuh (110 KB) + 107 KB = 215 KB,
// one stream per SM.  Both directions are one lock-step warp per stream (decision by decision).
// STATUS: bit-exact in host emulation and on the GPU (tests/test_gpu_other_coders.py, tests/test_gpu_pipeline.py); enabled
// without any switch (coder_gate in qlfc.cu).
#pragma once

typedef QLayout<4, 2, 10> ALY;                                  // counter file (qlfc_decoder6.cuh)
constexpr u32 QA_TAB_BYTES = 8208;                              // 4097 x int16, padded to 16
constexpr u32 OA_STRETCH = (ALY::BYTES + 15u) & ~15u, OA_SQUASH = OA_STRETCH + QA_TAB_BYTES, OA_MIX = OA_SQUASH + QA_TAB_BYTES;
constexpr u32 QA_MIXERS = 256 + 64 + 8 + 256 + 256 + 1024 + 32, QA_MIX_BYTES = 48;   // {int w0, w1, w2; short map[17]; pad}
constexpr u32 MX_RANK = 0, MX_RANKEXP = 256, MX_RANKMAN = 320, MX_RANKESC = 328, MX_RUN = 584, MX_RUNEXP = 840, MX_RUNMAN = 1864;
constexpr u32 QA_BYTES = OA_MIX + QA_MIXERS * QA_MIX_BYTES;
static_assert(QA_BYTES <= 227 * 1024, "the adaptive coder's working set must fit one SM");
static_assert(MX_RUNMAN + 32 == QA_MIXERS, "mixer index space");

QD3_FN int qa_ld_s16(const SM3 &sm, u32 off) { return (int)(short)sm.ld16(off); }
#ifdef QD3_HOST
QD3_FN int qa_ld_s32(const SM3 &sm, u32 off) { return (int)sm.ld32(off); }
QD3_FN void qa_st_s32(const SM3 &sm, u32 off, int v) { memcpy(sm.b + off, &v, 4); }
#else
QD3_FN int qa_ld_s32(const SM3 &sm, u32 off) { return (int)sm.ld32(off); }
QD3_FN void qa_st_s32(const SM3 &sm, u32 off, int v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(sm.b + off), "r"(v) : "memory"); }
#endif

// counter moves with the adaptive constants, same closed forms as q_up / q_down (exact for any integers):
//   bit 0: p + (((4096 - TH0 - p) * AR0) >> 12) = (p * (4096 - AR0) + (4096 - TH0) * AR0) >> 12
//   bit 1: p - (((p - TH1) * AR1) >> 12)        = (p * (4096 - AR1) + TH1 * AR1 + 4095) >> 12
template <int K, int WHO> QD3_FN int qa_move(int p, u32 bit)          // WHO: 0 state, 1 symbol, 2 shared, 3 the mixer's map
{
    const int up = p * (4096 - bscb_aparam(K, 4 * WHO + 1)) + (4096 - bscb_aparam(K, 4 * WHO)) * bscb_aparam(K, 4 * WHO + 1);
    const int dn = p * (4096 - bscb_aparam(K, 4 * WHO + 3)) + bscb_aparam(K, 4 * WHO + 2) * bscb_aparam(K, 4 * WHO + 3) + 4095;
    return (bit ? dn : up) >> 12;
}

struct QaMix { int s0, s1, s2, mixed; u32 moff, ioff; };        // stretched inputs, the mixed probability, mixer / map-entry byte offsets

// predictor.h:105-123 Mixup(charProbability, stateProbability, staticProbability)
QD3_FN int qa_mixup(const SM3 &sm, QaMix &m, u32 mixer, int pc, int ps, int pg)
{
    m.moff = OA_MIX + mixer * QA_MIX_BYTES;
    m.s0 = qa_ld_s16(sm, OA_STRETCH + 2u * (u32)pc); m.s1 = qa_ld_s16(sm, OA_STRETCH + 2u * (u32)ps); m.s2 = qa_ld_s16(sm, OA_STRETCH + 2u * (u32)pg);
    const int w0 = qa_ld_s32(sm, m.moff), w1 = qa_ld_s32(sm, m.moff + 4), w2 = qa_ld_s32(sm, m.moff + 8);
    int sp = (int)(short)((m.s0 * w0 + m.s1 * w1 + m.s2 * w2) >> 17);          // the reference keeps this in a short
    sp = sp < -2047 ? -2047 : sp; sp = sp > 2047 ? 2047 : sp;
    const u32 index = (u32)(sp + 2048) >> 8;
    const int weight = sp & 255, probability = qa_ld_s16(sm, OA_SQUASH + 2u * (u32)(2048 + sp));
    m.ioff = m.moff + 12u + 2u * index;
    const int m0 = qa_ld_s16(sm, m.ioff), m1 = qa_ld_s16(sm, m.ioff + 2);
    const int mapped = m0 + (((m1 - m0) * weight) >> 8);
    return m.mixed = (3 * probability + mapped) >> 2;
}
// predictor.h:185-211 UpdateBit0 / UpdateBit1 (int products wrap like the reference's)
template <int K> QD3_FN void qa_learn(const SM3 &sm, const QaMix &m, u32 bit)
{
    const int m0 = qa_ld_s16(sm, m.ioff), m1 = qa_ld_s16(sm, m.ioff + 2);
    sm.st16(m.ioff, (u32)qa_move<K, 3>(m0, bit)); sm.st16(m.ioff + 2, (u32)qa_move<K, 3>(m1, bit));
    const int eps = m.mixed - (bit ? 1 : 4095);
    const int w0 = qa_ld_s32(sm, m.moff), w1 = qa_ld_s32(sm, m.moff + 4), w2 = qa_ld_s32(sm, m.moff + 8);
    qa_st_s32(sm, m.moff,     w0 - ((int)((u32)(bscb_aparam(K, 16) * eps) * (u32)m.s0) >> 16));
    qa_st_s32(sm, m.moff + 4, w1 - ((int)((u32)(bscb_aparam(K, 17) * eps) * (u32)m.s1) >> 16));
    qa_st_s32(sm, m.moff + 8, w2 - ((int)((u32)(bscb_aparam(K, 18) * eps) * (u32)m.s2) >> 16));
}

// one decision: probability from (counters is, ic, ig through mixer `mixer`), then everything learns from the bit
template <int K> QD3_FN u32 qa_dec(const SM3 &sm, Rc3 &rc, u32 mixer, u32 is, u32 ic, u32 ig)
{
    const int s = sm.cnt(is), c = sm.cnt(ic), g = sm.cnt(ig);
    QaMix m; const int p = qa_mixup(sm, m, mixer, c, s, g);
    const u32 b = qd6_step<ALY>(sm, rc, (u32)p);
    sm.set(is, qa_move<K, 0>(s, b)); sm.set(ic, qa_move<K, 1>(c, b)); sm.set(ig, qa_move<K, 2>(g, b));
    qa_learn<K>(sm, m, b);
    return b;
}
template <int K> QD3_FN void qa_enc(const SM3 &sm, QfEnc &rc, u32 mixer, u32 is, u32 ic, u32 ig, u32 b)
{
    const int s = sm.cnt(is), c = sm.cnt(ic), g = sm.cnt(ig);
    QaMix m; const int p = qa_mixup(sm, m, mixer, c, s, g);
    sm.set(is, qa_move<K, 0>(s, b)); sm.set(ic, qa_move<K, 1>(c, b)); sm.set(ig, qa_move<K, 2>(g, b));
    qa_learn<K>(sm, m, b);
    qf_encode<12>(rc, b, (u32)p);
}

// counter index of a rank-mantissa / escape / run-exponent / run-mantissa decision: resident rows or the write-back caches
#define QA_RANK_M(e, st, c, node, IS, IC) do { if ((e) <= LY::MAXE_R) { IS = LY::R_RM_STATE + (st) * LY::ROW_R + (1u << (e)) - 2u + (node); IC = LY::R_RM_CHAR + (c) * LY::ROW_R + (1u << (e)) - 2u + (node); } \
        else { IS = qd6_cache_get<LY>(sm, LY::C_STATE_VAL, LY::O_TAG_STATE, cold_s, wide_idx((e), (st), (node)), st_miss); IC = qd6_cache_get<LY>(sm, LY::C_CHAR_VAL, LY::O_TAG_CHAR, cold_c, wide_idx((e), (c), (node)), st_miss); st_cached += 2; } } while (0)
#define QA_RUN_E(st2, c, k, IS, IC) do { if ((k) < UE_RES) { IS = LY::R_UE_STATE + (st2) * UE_RES + (k); IC = LY::R_UE_CHAR + (c) * UE_RES + (k); } \
        else { IS = qd6_cache_get<LY>(sm, LY::C_STATE_VAL, LY::O_TAG_STATE, cold_s, ue_idx((st2), (k)), st_miss); IC = qd6_cache_get<LY>(sm, LY::C_CHAR_VAL, LY::O_TAG_CHAR, cold_c, ue_idx((c), (k)), st_miss); st_cached += 2; } } while (0)
#define QA_RUN_M(e, st2, c, node, IS, IC) do { if ((e) <= LY::MAXE_U) { IS = LY::R_UM_STATE + (st2) * LY::ROW_U + (1u << (e)) - 2u + (node); IC = LY::R_UM_CHAR + (c) * LY::ROW_U + (1u << (e)) - 2u + (node); } \
        else { IS = qd6_cache_get<LY>(sm, LY::C_STATE_VAL, LY::O_TAG_STATE, cold_s, narrow_idx((e), (st2), (node)), st_miss); IC = qd6_cache_get<LY>(sm, LY::C_CHAR_VAL, LY::O_TAG_CHAR, cold_c, narrow_idx((e), (c), (node)), st_miss); st_cached += 2; } } while (0)

// ---- decoder (qlfc.cpp:1366-1666) --------------------------------------------------------------------------------------
QD3_FN int qa_decode_stream(const SM3 &sm, const u8 *__restrict__ in, u32 in_limit, u8 *__restrict__ out, u32 out_cap,
                            short *__restrict__ cold_s, short *__restrict__ cold_c, u32 &st_cached, u32 &st_miss)
{
    typedef ALY LY;
    QD3_LREGS;
#ifndef QD3_HOST
    const u32 lane = threadIdx.x & 31u;
#endif
    Rc3 rc; u32 n; int maxRank;
    { const int err = qd6_prologue<LY>(sm, rc, lr, in, in_limit, out_cap, n, maxRank); if (err) return err; }   // the stream header is the static coder's

    u32 ctxRank0 = 0, ctxRank4 = 0, ctxRun = 0; int avgRank = 0;
    u32 c, m1, m2, m3;
    { const u32 f = sm.ld32(LY::O_MTF); c = f & 255u; m1 = (f >> 8) & 255u; m2 = (f >> 16) & 255u; m3 = f >> 24; }
    for (u32 i = 0; i < n; ) {
        if (rc.pos - rc.wbase > QD3_RUN_ROOM) QD6_REFILL();
        u32 rank = 1, b, is, ic;
        const u32 h = sm.ld8(LY::O_RANK_HIST + c);
        const u32 st = sm.ld8(LY::O_RANK_STATE + ((ctxRun << 11) | (ctxRank4 << 3) | h));
        if (avgRank < 32) {
            b = qa_dec<K_RANK_T>(sm, rc, MX_RANK + c, LY::R_RT_STATE + st, LY::R_RT_CHAR + c, LY::R_RT_SHARED);
            if (!b) sm.st8(LY::O_RANK_HIST + c, 0);
            else {
                u32 e = 1;
                while ((int)e != maxRank) {
                    b = qa_dec<K_RANK_E>(sm, rc, MX_RANKEXP + (h > e ? h : e) * 8u + e, LY::R_RE_STATE + st * 8 + e - 1, LY::R_RE_CHAR + c * 8 + e - 1, LY::R_RE_SHARED + e - 1);
                    if (!b) break;
                    if (++e >= 7) break;
                }
                sm.st8(LY::O_RANK_HIST + c, e);
                for (u32 bit = e; bit > 0; --bit) {
                    QA_RANK_M(e, st, c, rank, is, ic);
                    b = qa_dec<K_RANK_M>(sm, rc, MX_RANKMAN + e, is, ic, LY::R_WIDE_SHARED + e * 256u + rank);
                    rank = 2u * rank + b;
                }
            }
        } else {
            rank = 0;
            for (u32 node = 1, bit = (u32)maxRank + 1u; bit > 0; --bit) {
                QA_RANK_M(8u, st, c, node, is, ic);                                   // bank 8 = escape (never resident)
                b = qa_dec<K_RANK_P>(sm, rc, MX_RANKESC + node, is, ic, LY::R_WIDE_SHARED + 8u * 256u + node);
                node = 2u * node + b; rank = 2u * rank + b;
            }
            sm.st8(LY::O_RANK_HIST + c, (u32)qd3_ilog2(rank));
        }
        rank &= 255u;
        const u32 cur = c;
        if (rank == 1) { c = m1; m1 = cur; }
        else if (rank == 2) { c = m1; m1 = m2; m2 = cur; }
        else if (rank == 3) { c = m1; m1 = m2; m2 = m3; m3 = cur; }
        else if (rank != 0) {
            sm.st8(LY::O_MTF, c); sm.st8(LY::O_MTF + 1, m1); sm.st8(LY::O_MTF + 2, m2); sm.st8(LY::O_MTF + 3, m3);
            QD3_SYNC();
            for (u32 basep = 0; basep < rank; basep += 32) {
                QD3_LANES { QD3_L(lr).tmp = sm.ld8(LY::O_MTF + basep + lane + 1u); }
                QD3_SYNC();
                QD3_LANES { if (basep + lane < rank) sm.st8(LY::O_MTF + basep + lane, QD3_L(lr).tmp); }
                QD3_SYNC();
            }
            sm.st8(LY::O_MTF + rank, cur);
            QD3_SYNC();
            const u32 f = sm.ld32(LY::O_MTF); c = f & 255u; m1 = (f >> 8) & 255u; m2 = (f >> 16) & 255u; m3 = f >> 24;
        }
        avgRank = (avgRank * 124 + (int)rank * 4) >> 7;
        const u32 rank0 = rank - 1u, hU = sm.ld8(LY::O_RUN_HIST + cur);
        const u32 st2 = sm.ld8(LY::O_RUN_STATE + ((ctxRank0 << 10) | (ctxRun << 6) | ((rank0 < 7u ? rank0 : 7u) << 3) | (hU < 7 ? hU : 7)));
        u32 run = 1;
        b = qa_dec<K_RUN_T>(sm, rc, MX_RUN + cur, LY::R_UT_STATE + st2, LY::R_UT_CHAR + cur, LY::R_UT_SHARED);
        if (!b) sm.st8(LY::O_RUN_HIST + cur, (hU + 2u) >> 2);
        else {
            u32 eu = 1;
            for (;;) {
                QA_RUN_E(st2, cur, eu - 1u, is, ic);
                b = qa_dec<K_RUN_E>(sm, rc, MX_RUNEXP + (hU > eu ? hU : eu) * 32u + eu, is, ic, LY::R_UE_SHARED + eu - 1u);
                if (!b) break;
                if (++eu >= 31u) break;                                              // corrupt-input guard
            }
            sm.st8(LY::O_RUN_HIST + cur, ((hU + 3u * eu + 3u) >> 2) & 255u);
            for (u32 node = 1, bit = eu; bit > 0; --bit) {
                QA_RUN_M(eu, st2, cur, node, is, ic);
                b = qa_dec<K_RUN_M>(sm, rc, MX_RUNMAN + eu, is, ic, LY::R_NARROW_SHARED + eu * 32u + node);
                run = 2u * run + b; node = eu <= 5u ? 2u * node + b : node + 1u;     // qlfc.cpp:1119
            }
        }
        ctxRank0 = ((ctxRank0 << 1) | (rank0 == 0u ? 1u : 0u)) & 0x7u;
        ctxRank4 = ((ctxRank4 << 2) | (rank0 < 3u ? rank0 : 3u)) & 0xffu;
        ctxRun   = ((ctxRun << 1) | (run < 3u ? 1u : 0u)) & 0xfu;
        if (run <= 32u && i + 32u <= n) { QD3_LANES { out[i + ((lane - i) & 31u)] = (u8)cur; } }
        else {
            if (run > n - i) run = n - i;
            QD3_LANES { for (u32 k = (lane - i) & 31u; k < run; k += 32) out[i + k] = (u8)cur; }
        }
        i += run;
    }
    return (int)n;
}

// ---- encoder (qlfc.cpp:463-823) ---------------------------------------------------------------------------------------
QD3_FN int qa_encode_stream(const SM3 &sm, const u32 *__restrict__ run_pos, const u8 *__restrict__ run_sym, const u8 *__restrict__ run_rank,
                            u32 run_begin, u32 run_end, u32 in_size, const u8 *__restrict__ mtf, u8 *__restrict__ out, u32 out_cap,
                            short *__restrict__ cold_s, short *__restrict__ cold_c, u32 &st_cached, u32 &st_miss)
{
    typedef ALY LY;
    QF_LREGS;
#ifndef QD3_HOST
    const u32 lane = threadIdx.x & 31u;
#endif
    QD3_LANES { QD3_L(lr).used8 = 0; QD3_L(lr).tmp = 0; }
    QfEnc rc; rc.low = 0; rc.range = 0xffffffffu; rc.cache = 0; rc.pending = 0; rc.pos = 0; rc.out = out;
    const long long eob = (long long)out_cap - 16;
    for (int b = 31; b >= 0; --b) qf_encode<12>(rc, (in_size >> b) & 1u, 2048u);
    int maxRank = 7;
    {
        int prev = -1;
        for (int d = 0; d < 256; ++d) {
            const int c = mtf[d];
            for (int bit = 7; bit >= 0; --bit) {
                bool can0, can1; QD3_HEADER_OPTIONS(prev, c >> (bit + 1), bit, can0, can1);
                if (can0 && can1) qf_encode<12>(rc, (u32)(c >> bit) & 1u, 2048u);
            }
            if (c == prev) { maxRank = qd3_ilog2((u32)(d - 1)); break; }
            prev = c;
            QD3_LANES { if ((u32)(c >> 3) == lane) QD3_L(lr).used8 |= 1u << (c & 7); }
        }
    }
    u32 ctxRank0 = 0, ctxRank4 = 0, ctxRun = 0; int avgRank = 0;
    for (u32 t0 = run_begin; t0 < run_end; t0 += 32) {
        const u32 cnt = run_end - t0 < 32u ? run_end - t0 : 32u;
        QD3_LANES {
            QfLane &r = QD3_L(lr);
            r.sym = 0; r.rank = 1; r.len = 1;
            if (lane < cnt) { r.sym = run_sym[t0 + lane]; r.rank = run_rank[t0 + lane]; r.len = run_pos[t0 + lane + 1] - run_pos[t0 + lane]; }
        }
        for (u32 j = 0; j < cnt; ++j) {
            if ((long long)rc.pos >= eob) return LIBBSC_NOT_COMPRESSIBLE;             // qlfc.cpp:531-534
            const u32 c = QF_BCAST(sym, j), rank = QF_BCAST(rank, j), run = QF_BCAST(len, j);
            u32 is, ic;
            const u32 h = sm.ld8(LY::O_RANK_HIST + c);
            const u32 st = sm.ld8(LY::O_RANK_STATE + ((ctxRun << 11) | (ctxRank4 << 3) | h));
            if (avgRank < 32) {
                qa_enc<K_RANK_T>(sm, rc, MX_RANK + c, LY::R_RT_STATE + st, LY::R_RT_CHAR + c, LY::R_RT_SHARED, rank != 1u ? 1u : 0u);
                if (rank == 1u) sm.st8(LY::O_RANK_HIST + c, 0);
                else {
                    const u32 e = (u32)qd3_ilog2(rank);
                    sm.st8(LY::O_RANK_HIST + c, e);
                    for (u32 b = 1; b < e; ++b)
                        qa_enc<K_RANK_E>(sm, rc, MX_RANKEXP + (h > b ? h : b) * 8u + b, LY::R_RE_STATE + st * 8 + b - 1, LY::R_RE_CHAR + c * 8 + b - 1, LY::R_RE_SHARED + b - 1, 1u);
                    if ((int)e < maxRank)
                        qa_enc<K_RANK_E>(sm, rc, MX_RANKEXP + (h > e ? h : e) * 8u + e, LY::R_RE_STATE + st * 8 + e - 1, LY::R_RE_CHAR + c * 8 + e - 1, LY::R_RE_SHARED + e - 1, 0u);
                    for (u32 node = 1, bit = e; bit > 0; --bit) {
                        const u32 b = (rank >> (bit - 1u)) & 1u;
                        QA_RANK_M(e, st, c, node, is, ic);
                        qa_enc<K_RANK_M>(sm, rc, MX_RANKMAN + e, is, ic, LY::R_WIDE_SHARED + e * 256u + node, b);
                        node = 2u * node + b;
                    }
                }
            } else {
                sm.st8(LY::O_RANK_HIST + c, (u32)qd3_ilog2(rank));
                for (u32 node = 1, bit = (u32)maxRank + 1u; bit > 0; --bit) {
                    const u32 b = (rank >> (bit - 1u)) & 1u;
                    QA_RANK_M(8u, st, c, node, is, ic);
                    qa_enc<K_RANK_P>(sm, rc, MX_RANKESC + node, is, ic, LY::R_WIDE_SHARED + 8u * 256u + node, b);
                    node = 2u * node + b;
                }
            }
            avgRank = (avgRank * 124 + (int)rank * 4) >> 7;
            const u32 rank0 = rank - 1u, hU = sm.ld8(LY::O_RUN_HIST + c);
            const u32 st2 = sm.ld8(LY::O_RUN_STATE + ((ctxRank0 << 10) | (ctxRun << 6) | ((rank0 < 7u ? rank0 : 7u) << 3) | (hU < 7 ? hU : 7)));
            qa_enc<K_RUN_T>(sm, rc, MX_RUN + c, LY::R_UT_STATE + st2, LY::R_UT_CHAR + c, LY::R_UT_SHARED, run != 1u ? 1u : 0u);
            if (run == 1u) sm.st8(LY::O_RUN_HIST + c, (hU + 2u) >> 2);
            else {
                const u32 e = (u32)qd3_ilog2(run);
                sm.st8(LY::O_RUN_HIST + c, ((hU + 3u * e + 3u) >> 2) & 255u);
                for (u32 b = 1; b <= e; ++b) {                                        // b < e: continue (1), b == e: stop (0)
                    QA_RUN_E(st2, c, b - 1u, is, ic);
                    qa_enc<K_RUN_E>(sm, rc, MX_RUNEXP + (hU > b ? hU : b) * 32u + b, is, ic, LY::R_UE_SHARED + b - 1u, b < e ? 1u : 0u);
                }
                for (u32 node = 1, bit = e; bit > 0; --bit) {
                    const u32 b = (run >> (bit - 1u)) & 1u;
                    QA_RUN_M(e, st2, c, node, is, ic);
                    qa_enc<K_RUN_M>(sm, rc, MX_RUNMAN + e, is, ic, LY::R_NARROW_SHARED + e * 32u + node, b);
                    node = e <= 5u ? 2u * node + b : node + 1u;
                }
            }
            ctxRank0 = ((ctxRank0 << 1) | (rank0 == 0u ? 1u : 0u)) & 0x7u;
            ctxRank4 = ((ctxRank4 << 2) | (rank0 < 3u ? rank0 : 3u)) & 0xffu;
            ctxRun   = ((ctxRun << 1) | (run < 3u ? 1u : 0u)) & 0xfu;
        }
    }
    if (rc.range < 0x10000u) qf_shift(rc);
    qf_shift(rc); qf_shift(rc); qf_shift(rc);
    return (int)rc.pos;
}

// mixers at their start values (predictor.h:96-103): weights 2048 << 5, 2048 << 5, 0; map[p] = squash((p - 8) * 256)
QD3_FN void qa_init_mixer(const SM3 &sm, u32 mixer)
{
    const u32 o = OA_MIX + mixer * QA_MIX_BYTES;
    qa_st_s32(sm, o, 2048 << 5); qa_st_s32(sm, o + 4, 2048 << 5); qa_st_s32(sm, o + 8, 0);
    for (u32 p = 0; p < 17; ++p) sm.st16(o + 12u + 2u * p, (u32)qa_ld_s16(sm, OA_SQUASH + 2u * (2048u + (p - 8u) * 256u)));
    sm.st16(o + 46u, 0);
}

#ifndef QD3_HOST
// `tables` points at {QTables, moves (128 B), stretch (QA_TAB_BYTES), squash (QA_TAB_BYTES)} (qlfc.cu:get_tables)
__device__ __forceinline__ void qa_smem_init(u8 *raw, const QTables *__restrict__ tables)
{
    qd6_smem_init<ALY>(raw, tables);
    const u32 lane = threadIdx.x & 31;
    const uint4 *src = (const uint4 *)((const u8 *)(tables + 1) + 128); uint4 *dst = (uint4 *)(raw + OA_STRETCH);
    for (u32 i = lane; i < 2 * QA_TAB_BYTES / 16; i += 32) dst[i] = src[i];
    __syncwarp();
    SM3 sm; sm.b = (u32)__cvta_generic_to_shared(raw);
    for (u32 m = lane; m < QA_MIXERS; m += 32) qa_init_mixer(sm, m);
    __syncwarp();
}

__global__ void __launch_bounds__(32, 1) q_adaptive_decode(const u8 *__restrict__ in_all, SubBlock *__restrict__ sbs, short *__restrict__ cold_all,
                                                           const QTables *__restrict__ tables, u8 *__restrict__ out_all, const u32 *__restrict__ sb_list, DoneSignal done)
{
    extern __shared__ __align__(16) u8 q_smem_raw[];
    qa_smem_init(q_smem_raw, tables);
    SM3 sm; sm.b = (u32)__cvta_generic_to_shared(q_smem_raw);
    asm volatile("" : "+r"(sm.b) :: "memory");
    const u32 sid = sb_list[blockIdx.x];
    SubBlock &sb = sbs[sid];
    short *cold_s = cold_all + (size_t)blockIdx.x * 2 * COLD_PAD, *cold_c = cold_s + COLD_PAD;
    u32 st_cached = 0, st_miss = 0;
    const int r = qa_decode_stream(sm, in_all + sb.out_off, sb.out_cap, out_all + sb.in_start, sb.in_size, cold_s, cold_c, st_cached, st_miss);
    __syncwarp();                                        // every lane's output stores precede lane 0's report
    if (threadIdx.x == 0) { sb.result = r; sb.stat_cached = st_cached; sb.stat_miss = st_miss; signal_done(done); }
}

__global__ void __launch_bounds__(32, 1) q_adaptive_encode(const u32 *__restrict__ run_pos, const u8 *__restrict__ run_sym, const u8 *__restrict__ run_rank,
                                                           SubBlock *__restrict__ sbs, const u8 *__restrict__ mtf_all, short *__restrict__ cold_all,
                                                           const QTables *__restrict__ tables, u8 *__restrict__ out_all, const u32 *__restrict__ sb_list, DoneSignal done)
{
    extern __shared__ __align__(16) u8 q_smem_raw[];
    qa_smem_init(q_smem_raw, tables);
    SM3 sm; sm.b = (u32)__cvta_generic_to_shared(q_smem_raw);
    asm volatile("" : "+r"(sm.b) :: "memory");
    const u32 sid = sb_list ? sb_list[blockIdx.x] : blockIdx.x;
    SubBlock &sb = sbs[sid];
    short *cold_s = cold_all + (size_t)sid * 2 * COLD_PAD, *cold_c = cold_s + COLD_PAD;
    u32 st_cached = 0, st_miss = 0;
    const int r = qa_encode_stream(sm, run_pos, run_sym, run_rank, sb.run_begin, sb.run_end, sb.in_size, mtf_all + sid * 256, out_all + sb.out_off, sb.out_cap,
                                   cold_s, cold_c, st_cached, st_miss);
    __syncwarp();                                        // every lane's output stores precede lane 0's report
    if (threadIdx.x == 0) { sb.result = r; sb.stat_cached = st_cached; sb.stat_miss = st_miss; signal_done(done); }
}
#endif
