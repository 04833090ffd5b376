// libbsc_b200/csrc/qlfc_decoder6.cuh -- the QLFC static DECODER (qlfc.cpp:1672-1927): one lock-step warp per stream, with the LAYOUT
// of the counter file as a template parameter so that it fits TWO streams per SM.  Included by qlfc.cu after qlfc_lanes.cuh; also
// compiled for the host (tools/qdec3_host.cpp), where the 32 lanes are emulated and the output is compared with reference streams.
//
// Why two per SM: the decoder is a serial recurrence (the context of every decision depends on the previous decisions); one warp
// issues well under one instruction per cycle on ONE of the SM's four schedulers -- most of its cycles are fixed-latency
// dependency waits -- so a second stream on the same SM costs the first one little.  The "diet" layout keeps resident only what is hot:
//     state tables 40 KB | first-bit / exponent / shared counters 25 KB | rank mantissa trees for exponents 1..4 (30 nodes
//     per state / symbol) 30 KB | run mantissa trees for exponents 1..3 | staged rows
// = 110 KB.  Everything else (rank exponent 5, the escape bank, long runs) is used ROW-wise from HBM: the counters one run can
// touch in such a bank are one contiguous row per state and one per symbol, fetched with one coalesced access each, staged in
// 1 KB of shared memory for the decisions and written back whole (qd6_rows_in / qd6_rows_out).
// Instruction-count measures (a lone warp's time is its instruction count): the multipliers of the hot counter moves live in
// registers (q_move6), the exponent / mantissa loops address their counters through absolute shared-memory addresses that advance
// with the node, positions 0..31 of the MTF list live in the lanes (one shuffle per run instead of shared-memory traffic and
// three warp barriers for every rank > 3, i.e. 58 % of the runs on text).
// QLayout<5, 5, 12> (LayoutFull, 205 KB) is the layout of qlfc_coder.cuh; the adaptive coder derives its own from it.
#pragma once

template <u32 MAXE_R_, u32 MAXE_U_, int CLOG_> struct QLayout {
    static constexpr u32 MAXE_R = MAXE_R_, MAXE_U = MAXE_U_;                 // resident mantissa exponents (rank, run length)
    static constexpr bool BR = false;                                        // renormalisation of the range decoder as a rarely taken branch (q_decode8)
    static constexpr bool TG = false;                                        // state tables resident in shared memory (TablesInGlobal: read through L1)
    static constexpr u32  SHIFT = 0;                                         // bytes cut off the front of the shared-memory image
    static constexpr u32 ROW_R = (2u << MAXE_R_) - 2u, ROW_U = (2u << MAXE_U_) - 2u;   // compact row: exponent e at offsets 2^e-2 .. 2^(e+1)-3
    // counter file, indices in u16 units (same order as qlfc_coder.cuh)
    static constexpr u32 R_RT_SHARED = 0, R_RT_STATE = 2, R_RT_CHAR = R_RT_STATE + 256;
    static constexpr u32 R_RE_SHARED = R_RT_CHAR + 256, R_RE_STATE = R_RE_SHARED + 8, R_RE_CHAR = R_RE_STATE + 2048;
    static constexpr u32 R_UT_SHARED = R_RE_CHAR + 2048, R_UT_STATE = R_UT_SHARED + 2, R_UT_CHAR = R_UT_STATE + 256;
    static constexpr u32 R_UE_SHARED = R_UT_CHAR + 256, R_UE_STATE = R_UE_SHARED + 32, R_UE_CHAR = R_UE_STATE + 256 * UE_RES;
    static constexpr u32 R_WIDE_SHARED = R_UE_CHAR + 256 * UE_RES, R_NARROW_SHARED = R_WIDE_SHARED + 9 * 256;
    static constexpr u32 R_RM_STATE = R_NARROW_SHARED + 32 * 32, R_RM_CHAR = R_RM_STATE + 256 * ROW_R;
    static constexpr u32 R_UM_STATE = R_RM_CHAR + 256 * ROW_R, R_UM_CHAR = R_UM_STATE + 256 * ROW_U, R_END = R_UM_CHAR + 256 * ROW_U;
    static constexpr u32 SLOTS = 1u << CLOG_, HB = CLOG_ - 2, HMASK = (1u << HB) - 1u;   // 2 class bits + HB hashed bits per cache
    static constexpr u32 C_STATE_VAL = R_END, C_CHAR_VAL = C_STATE_VAL + SLOTS, S16_COUNT = (C_CHAR_VAL + SLOTS + 1) & ~1u;
    // shared-memory image (byte offsets); the counters start where CoderSmem's do, so SM3::cnt / SM3::set apply
    static constexpr u32 O_RANK_STATE = 0, O_RUN_STATE = 32768, O_S16 = 40960, O_TAG_STATE = O_S16 + 2 * S16_COUNT, O_TAG_CHAR = O_TAG_STATE + 2 * SLOTS;
    static constexpr u32 O_RANK_HIST = O_TAG_CHAR + 2 * SLOTS, O_RUN_HIST = O_RANK_HIST + 256, O_MTF = (O_RUN_HIST + 256 + 15u) & ~15u, O_WIN = O_MTF + 288;
    // decoder only: two staged rows [256] of the escape bank (state row, symbol row), addressed like counters
    static constexpr u32 O_ROWS = O_WIN + 272, BYTES = O_ROWS + 1024;
    static constexpr u32 R_ROW_STATE = (O_ROWS - O_S16) / 2u, R_ROW_CHAR = R_ROW_STATE + 256u;
    // cache slot of a cold index: classes as in qlfc_coder.cuh (0,1 rank banks, 2 run mantissa, 3 run exponent >= 8)
    static QD3_FN_MEMBER u32 cache_slot(u32 idx)
    {
        const u32 h = idx >> HB;
        const u32 cls = idx < 9u * 65536u ? (h & 1u) : (idx < 9u * 65536u + 32u * 8192u ? 2u : 3u);
        return (cls << HB) | ((idx ^ (h * 1237u)) & HMASK);
    }
    static QD3_FN_MEMBER u32 cache_tag(u32 idx) { return (idx >> HB) + 1u; }
    static QD3_FN_MEMBER u32 cache_unslot(u32 slot, u32 tag) { const u32 h = tag - 1u; return (h << HB) | (((slot & HMASK) ^ (h * 1237u)) & HMASK); }
};
// the same image as a struct (what the encoder uses); for QLayout<5, 5, 12> it is CoderSmem, member for member
template <class LY> struct CoderSmemT {
    u8    rank_state[LY::TG ? 16 : 32768];                   // TablesInGlobal: not resident (16-byte placeholders keep the alignment)
    u8    run_state[LY::TG ? 16 : 8192];
    u16   s16[LY::S16_COUNT];
    u16   tag_state[LY::SLOTS];
    u16   tag_char[LY::SLOTS];
    u8    rankHist[256], runHist[256];
    u8    mtf[256 + 32];
    alignas(16) u8 inwin[256];
};
template <class LY_> struct WithBranchRenorm : LY_ { static constexpr bool BR = true; };   // same image, other range-decoder step (qd6_step)
// The same image WITHOUT its first 40 KB (the two state tables): they are read-only and identical for every stream, so they are read
// through L1 from the ONE copy per device in global memory (4 one-byte look-ups per run, two of them issued a decision ahead of
// their use).  All offsets stay as they are: the accessor's base is moved back by SHIFT instead (SM3::b = image - SHIFT; offsets
// below SHIFT are never used).  70 KB per decoder stream instead of 110: THREE streams per SM.
template <class LY_> struct TablesInGlobal : LY_ {
    static constexpr bool TG = true;
    static constexpr u32  SHIFT = LY_::O_S16;
    static constexpr u32  BYTES = LY_::BYTES - LY_::O_S16;
};
typedef QLayout<5, 5, 12> LayoutFull;     // = qlfc_coder.cuh: 205 KB, one stream per SM
typedef QLayout<4, 3, 2> LayoutDiet;      // 110 KB, two DEcoder streams per SM: q_decode6 uses no caches (rows instead, see qd6_rows_in), so
                                          // their 8 KB hold the run-mantissa exponent 3 (run lengths 8..15) instead
typedef TablesInGlobal<LayoutDiet> LayoutDietTG;   // 70.7 KB: three decoder streams per SM
typedef TablesInGlobal<QLayout<3, 3, 2> > LayoutDiet4;   // 54.7 KB: FOUR per SM; the rank mantissa of exponent 4 (ranks 16..31) goes row-wise too
typedef TablesInGlobal<QLayout<2, 2, 2> > LayoutDiet5;   // 38.7 KB: five per SM (rank exponents 3, 4 and run exponent 3 row-wise)
typedef QLayout<4, 1, 10> LayoutEncDiet;  // 106 KB + the encoder's pipe state (5.6 KB): two six-warp encoders per SM
typedef TablesInGlobal<QLayout<3, 1, 10> > LayoutEncDiet4;   // 50 KB + 5.6 KB: four per SM (rank exponent 4 through the write-back cache)
typedef TablesInGlobal<LayoutEncDiet> LayoutEncDietTG;   // 66 KB + 5.6 KB: three per SM (the model warps gather their states through L1, a batch of 32 runs at a time)
static_assert(LayoutFull::R_END == R_END && LayoutFull::S16_COUNT == S16_COUNT && LayoutFull::O_S16 == O3_S16, "LayoutFull must reproduce qlfc_coder.cuh");
static_assert(LayoutFull::R_RM_STATE == R_RM_STATE && LayoutFull::R_UM_CHAR == R_UM_CHAR && LayoutFull::C_CHAR_VAL == C_CHAR_VAL, "LayoutFull must reproduce qlfc_coder.cuh");
static_assert(sizeof(CoderSmemT<LayoutFull>) == sizeof(CoderSmem) && offsetof(CoderSmemT<LayoutFull>, tag_state) == offsetof(CoderSmem, tag_state) &&
              offsetof(CoderSmemT<LayoutFull>, rankHist) == offsetof(CoderSmem, rankHist) && offsetof(CoderSmemT<LayoutFull>, inwin) == offsetof(CoderSmem, inwin),
              "CoderSmemT<LayoutFull> must be CoderSmem");
static_assert(LayoutDiet::BYTES <= 113 * 1024, "two diet decoders must fit one SM (227 KB, 1 KB reserved per CTA)");
static_assert(LayoutDiet::O_S16 == O3_S16 && (LayoutDiet::O_WIN & 15u) == 0 && (LayoutDiet::O_MTF & 3u) == 0, "alignment of the shared-memory image");
static_assert((LayoutDiet::O_ROWS & 15u) == 0 && (LayoutFull::O_ROWS & 15u) == 0 && (LayoutDiet::O_TAG_STATE & 3u) == 0, "staged rows are moved 16 bytes at a time");
static_assert(LayoutFull::BYTES <= 232448, "one full decoder per SM");
static_assert(3 * (LayoutDietTG::BYTES + 1024) <= 232448, "three decoders without resident state tables must fit one SM");
static_assert(4 * (LayoutDiet4::BYTES + 1024) <= 232448 && 5 * (LayoutDiet5::BYTES + 1024) <= 232448, "four / five decoders per SM");
static_assert((LayoutDiet4::O_ROWS & 15u) == 0 && (LayoutDiet5::O_ROWS & 15u) == 0 && (LayoutDiet4::O_WIN & 15u) == 0 && (LayoutDiet5::O_WIN & 15u) == 0 &&
              (LayoutDiet4::O_MTF & 3u) == 0 && (LayoutDiet5::O_MTF & 3u) == 0 && (LayoutDiet4::O_TAG_STATE & 3u) == 0 && (LayoutDiet5::O_TAG_STATE & 3u) == 0, "alignment of the smaller images");

// state-table look-ups: resident image, or the per-device copy in global memory through L1 (LY::TG)
#ifndef QD6_TABSIM_TOUCH
#define QD6_TABSIM_TOUCH(i) do { } while (0)     // tools/qdec3_host.cpp -DQD6_TABSIM: LRU model of the L1 lines these look-ups touch
#endif
template <class LY> QD3_FN u32 qd6_rank_state(const SM3 &sm, const u8 *__restrict__ tab, u32 idx)
{
    if (LY::TG) {
#ifdef QD3_HOST
        QD6_TABSIM_TOUCH(idx);
        return tab[idx];
#else
        return (u32)__ldg(tab + idx);
#endif
    }
    return sm.ld8(LY::O_RANK_STATE + idx);
}
template <class LY> QD3_FN u32 qd6_run_state(const SM3 &sm, const u8 *__restrict__ tab, u32 idx)
{
    if (LY::TG) {
#ifdef QD3_HOST
        QD6_TABSIM_TOUCH(32768u + idx);
        return tab[32768u + idx];
#else
        return (u32)__ldg(tab + 32768u + idx);
#endif
    }
    return sm.ld8(LY::O_RUN_STATE + idx);
}

// Index (into the counter file) of rare counter `idx` through the direct-mapped write-back cache (uniform).
template <class LY> QD3_FN u32 qd6_cache_get(const SM3 &sm, u32 val_base, u32 tags_off, short *__restrict__ cold, u32 idx, u32 &misses)
{
    const u32 slot = LY::cache_slot(idx), want = LY::cache_tag(idx);
    const u32 t = sm.ld16(tags_off + 2u * slot);
    if (t != want) {
        if (t) cold[LY::cache_unslot(slot, t)] = (short)sm.cnt(val_base + slot);
        sm.set(val_base + slot, (u16)cold[idx]);
        sm.st16(tags_off + 2u * slot, want);
        ++misses;
    }
    return val_base + slot;
}


// 16-byte accesses: a row of the escape bank in global memory <-> the staged copy in shared memory
QD3_FN U4 qd6_ldg128(const short *p)
{
#ifdef QD3_HOST
    U4 v; memcpy(&v, p, 16); return v;
#else
    const uint4 t = *(const uint4 *)p; U4 v; v.x = t.x; v.y = t.y; v.z = t.z; v.w = t.w; return v;
#endif
}
QD3_FN void qd6_stg128(short *p, const U4 &v)
{
#ifdef QD3_HOST
    memcpy(p, &v, 16);
#else
    *(uint4 *)p = make_uint4(v.x, v.y, v.z, v.w);
#endif
}
QD3_FN void qd6_sts128(const SM3 &sm, u32 off, const U4 &v)
{
#ifdef QD3_HOST
    memcpy(sm.b + off, &v, 16);
#else
    asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" :: "r"(sm.b + off), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
#endif
}

// Everything that is not resident (rank mantissa exponents > MAXE_R, the escape bank, run exponent indices >= UE_RES, run
// mantissa exponents > MAXE_U) is used ROW-wise: the counters one run can touch in such a bank are one contiguous row per
// (state) and one per (symbol) -- 2^e entries of a wide bank, 256 of the escape bank, 32 of a narrow bank or of the run exponent
// file -- so the two rows are fetched with one coalesced access each (lane l always owns bytes [16 l, 16 l + 16) of a row, which
// makes the global traffic program-ordered per address), staged in shared memory for the decisions and written back whole.
// One global round trip per event, where the write-back caches of qlfc_coder.cuh cost one per MISS: measured with this source
// on the host (first sub-blocks of BWT output, layout <4,2>): Python sources 0.99 cached accesses / 0.53 misses per run, an
// x86-64 shared object 2.2 / 1.3, G_skew 16 / 9.7 -- against 0.11, 0.13 and 1.0 row events per run.
template <class LY> QD3_FN void qd6_rows_in(const SM3 &sm, const short *__restrict__ cold_s, const short *__restrict__ cold_c, u32 rs_at, u32 rc_at, u32 nb)
{
#ifndef QD3_HOST
    const u32 lane = threadIdx.x & 31u;
#endif
    QD3_LANES {
        if (16u * lane < nb) {
            qd6_sts128(sm, LY::O_ROWS + 16u * lane, qd6_ldg128(cold_s + rs_at + 8u * lane));
            qd6_sts128(sm, LY::O_ROWS + 512u + 16u * lane, qd6_ldg128(cold_c + rc_at + 8u * lane));
        }
    }
    QD3_SYNC();
}
template <class LY> QD3_FN void qd6_rows_out(const SM3 &sm, short *__restrict__ cold_s, short *__restrict__ cold_c, u32 rs_at, u32 rc_at, u32 nb)
{
#ifndef QD3_HOST
    const u32 lane = threadIdx.x & 31u;
#endif
    QD3_SYNC();
    QD3_LANES {
        if (16u * lane < nb) {
            qd6_stg128(cold_s + rs_at + 8u * lane, sm.ld128(LY::O_ROWS + 16u * lane));
            qd6_stg128(cold_c + rc_at + 8u * lane, sm.ld128(LY::O_ROWS + 512u + 16u * lane));
        }
    }
    QD3_SYNC();
}

// The 16-bit renormalisation (rangecoder.h:213-219) as a function of its own: q_decode8 calls it from a rarely taken branch (once per
// 16 coded bits) instead of carrying seven always-executed instructions and a shared-memory load in every decision.
struct Qd6Norm { u32 code, pos; };
#ifdef QD3_HOST
static inline
#else
__device__ __noinline__
#endif
Qd6Norm qd6_renorm_cold(const SM3 sm, u32 win_off, u32 code, u32 pos, u32 wbase)
{
    Qd6Norm r;
    r.code = (code << 16) | sm.ld16(win_off + (pos - wbase));
    r.pos = pos + 2u;
    return r;
}

// one decision with P(bit = 0) = p / 4096
template <class LY> QD3_FN u32 qd6_step(const SM3 &sm, Rc3 &rc, u32 p)
{
    if (LY::BR) {
        if (rc.range < 0x10000u) {
            const Qd6Norm t = qd6_renorm_cold(sm, LY::O_WIN, rc.code, rc.pos, rc.wbase);
            rc.code = t.code; rc.pos = t.pos; rc.range <<= 16;
        }
        const u32 r = (rc.range >> 12) * p;
        const bool bit = rc.code >= r;
        rc.code -= bit ? r : 0u;
        rc.range = bit ? rc.range - r : r;
        return bit ? 1u : 0u;
    }
    const bool need = rc.range < 0x10000u;
    rc.code = need ? (rc.code << 16) | rc.nx : rc.code;
    rc.range = need ? rc.range << 16 : rc.range;
    rc.pos += need ? 2u : 0u;
    rc.nx = sm.ld16(LY::O_WIN + (rc.pos - rc.wbase));
    const u32 r = (rc.range >> 12) * p;
    const bool bit = rc.code >= r;
    rc.code -= bit ? r : 0u;
    rc.range = bit ? rc.range - r : r;
    return bit ? 1u : 0u;
}


// Counter moves (p * M + K) >> 12 as in qlfc_coder.cuh.  IMAD takes ONE immediate (the addend), so ptxas re-materialises
// every multiplier with a MOV in front of every use -- a visible share of the instructions of a mantissa decision -- and it folds any constant it can see.  The multipliers of the four hot decision classes are therefore
// LOADED (from a small table in global memory) into registers once per stream: 24 registers, no MOVs.
QD3_FN constexpr int qd6_hot(int k) { return k == K_RANK_T ? 0 : k == K_RANK_E ? 1 : k == K_RANK_M ? 2 : k == K_RUN_T ? 3 : -1; }
constexpr int QD6_HOT_CLASSES[4] = {K_RANK_T, K_RANK_E, K_RANK_M, K_RUN_T};
constexpr int QD6_MOVES = 4 * 3 * 2;                                       // table layout: [hot class][state, symbol, shared][bit]
struct Qd6Mv { int m[4][3][2]; };
QD3_FN void qd6_load_moves(Qd6Mv &mv, const int *__restrict__ moves)
{
#pragma unroll
    for (int h = 0; h < 4; ++h)
#pragma unroll
        for (int w = 0; w < 3; ++w) { mv.m[h][w][0] = moves[(h * 3 + w) * 2]; mv.m[h][w][1] = moves[(h * 3 + w) * 2 + 1]; }
}
// host side of the table (also used by the host emulation): multiplier 4096 - AR0 for bit 0, 4096 - AR1 for bit 1
static inline void qd6_fill_moves(int *moves)
{
    for (int h = 0; h < 4; ++h) for (int w = 0; w < 3; ++w) {
        moves[(h * 3 + w) * 2]     = 4096 - bscb_static_params[QD6_HOT_CLASSES[h]][4 + 4 * w];
        moves[(h * 3 + w) * 2 + 1] = 4096 - bscb_static_params[QD6_HOT_CLASSES[h]][6 + 4 * w];
    }
}
template <int K, int WHO> QD3_FN int q_move6(int p, u32 bit, const Qd6Mv &mv)
{
    constexpr int h = qd6_hot(K);
    const int m0 = h >= 0 ? mv.m[h >= 0 ? h : 0][WHO][0] : 4096 - bscb_param(K, 4 + 4 * WHO);
    const int m1 = h >= 0 ? mv.m[h >= 0 ? h : 0][WHO][1] : 4096 - bscb_param(K, 6 + 4 * WHO);
    const int up = p * m0 + (4096 - bscb_param(K, 3 + 4 * WHO)) * bscb_param(K, 4 + 4 * WHO);
    const int dn = p * m1 + bscb_param(K, 5 + 4 * WHO) * bscb_param(K, 6 + 4 * WHO) + 4095;
    return (bit ? dn : up) >> 12;
}

// one serial decision against three counters given by their ABSOLUTE shared-memory addresses (SM3::at)
template <class LY, int K> QD3_FN u32 qd6_dec3a(const SM3 &sm, Rc3 &rc, const Qd6Mv &mv, u32 as, u32 ac, u32 ag)
{
    const int s = (int)sm.ld16a(as), c = (int)sm.ld16a(ac), g = (int)sm.ld16a(ag);
    const u32 b = qd6_step<LY>(sm, rc, (u32)q_mix<K>(s, c, g));
    sm.st16a(as, (u32)q_move6<K, 0>(s, b, mv));
    sm.st16a(ac, (u32)q_move6<K, 1>(c, b, mv));
    sm.st16a(ag, (u32)q_move6<K, 2>(g, b, mv));
    return b;
}
// the same by counter index
template <class LY, int K> QD3_FN u32 qd6_dec3(const SM3 &sm, Rc3 &rc, const Qd6Mv &mv, u32 is, u32 ic, u32 ig)
{
    return qd6_dec3a<LY, K>(sm, rc, mv, sm.at(LY::O_S16 + 2u * is), sm.at(LY::O_S16 + 2u * ic), sm.at(LY::O_S16 + 2u * ig));
}
// ... with the counter values already loaded
template <class LY, int K> QD3_FN u32 qd6_dec3v(const SM3 &sm, Rc3 &rc, const Qd6Mv &mv, u32 is, u32 ic, u32 ig, int s, int c, int g)
{
    const u32 b = qd6_step<LY>(sm, rc, (u32)q_mix<K>(s, c, g));
    sm.set(is, q_move6<K, 0>(s, b, mv));
    sm.set(ic, q_move6<K, 1>(c, b, mv));
    sm.set(ig, q_move6<K, 2>(g, b, mv));
    return b;
}

// the same multipliers as compile-time constants, for the cold functions of q_decode8 (no 24-register argument)
QD3_FN Qd6Mv qd6_const_moves()
{
    Qd6Mv mv;
#define QD6_CM(h, K) mv.m[h][0][0] = 4096 - bscb_param(K, 4); mv.m[h][0][1] = 4096 - bscb_param(K, 6); mv.m[h][1][0] = 4096 - bscb_param(K, 8); \
                     mv.m[h][1][1] = 4096 - bscb_param(K, 10); mv.m[h][2][0] = 4096 - bscb_param(K, 12); mv.m[h][2][1] = 4096 - bscb_param(K, 14);
    QD6_CM(0, K_RANK_T) QD6_CM(1, K_RANK_E) QD6_CM(2, K_RANK_M) QD6_CM(3, K_RUN_T)
#undef QD6_CM
    return mv;
}
// what a cold decision function hands back: the range-coder registers it advanced and its result
struct Qd6Cold { u32 code, range, pos, nx, val; };

// (re)load the input window at rc.pos: 8 bytes per lane + 16 more by lanes 0..15
#define QD6_REFILL() do { rc.wbase = rc.pos; QD3_SYNC(); \
        QD3_LANES { for (u32 k_ = 0; k_ < 8; ++k_) { const u32 w_ = lane * 8u + k_, o_ = rc.wbase + w_; sm.st8(LY::O_WIN + w_, o_ < rc.limit ? rc.in[o_] : 0u); } \
                    if (lane < 16u) { const u32 w_ = 256u + lane, o_ = rc.wbase + w_; sm.st8(LY::O_WIN + w_, o_ < rc.limit ? rc.in[o_] : 0u); } } \
        QD3_SYNC(); } while (0)


// Stream prologue shared by both decoders: coder start-up, the 32-bit length, the MTF-order table.  Returns 0 or an error.
template <class LY> QD3_FN int qd6_prologue(const SM3 &sm, Rc3 &rc, QD3_LREGS_PARAM, const u8 *__restrict__ in, u32 in_limit, u32 out_cap, u32 &n, int &maxRank)
{
#ifndef QD3_HOST
    const u32 lane = threadIdx.x & 31u;
#endif
    QD3_LANES { QD3_L(lr).used8 = 0; QD3_L(lr).tmp = 0; }

    rc.in = in; rc.limit = in_limit; rc.code = 0; rc.range = 0xffffffffu; rc.pos = 0; rc.wbase = 0; rc.nx = 0;
    QD6_REFILL();
    rc.code = (sm.ld16(LY::O_WIN + 2) << 16) | sm.ld16(LY::O_WIN + 4);            // rangecoder.h:203-211: three units, the first falls out of 32 bits
    rc.pos = 6; rc.nx = sm.ld16(LY::O_WIN + 6);
    n = 0;
    for (int b = 0; b < 32; ++b) n = (n << 1) | qd6_step<LY>(sm, rc, 2048u);
    if (n > out_cap) return LIBBSC_DATA_CORRUPT;                            // would overrun the output slice

    maxRank = 7;
    int prev = -1;
    for (int d = 0; d < 256; ++d) {
        int c = 0;
        for (int bit = 7; bit >= 0; --bit) {
            bool can0, can1; QD3_HEADER_OPTIONS(prev, c, bit, can0, can1);
            if (can0 && can1) {
                if (rc.pos - rc.wbase > 256u) QD6_REFILL();
                c = 2 * c + (int)qd6_step<LY>(sm, rc, 2048u);
            }
            else if (can1) c = 2 * c + 1;
            else if (can0) c = 2 * c;
        }
        c &= 255;
        sm.st8(LY::O_MTF + d, (u32)c);
        if (c == prev) { maxRank = qd3_ilog2((u32)(d - 1)); break; }
        prev = c;
        QD3_LANES { if ((u32)(c >> 3) == lane) QD3_L(lr).used8 |= 1u << (c & 7); }
    }
    QD3_SYNC();
    return 0;
}


#define QD6_STREAM qd6_decode_stream
#define QD6_SUFFIX _i
#define QD6_ROLL
#define QD6_COLD QD3_FN
#include "qlfc_decoder6_stream.inc"
#undef QD6_STREAM
#undef QD6_SUFFIX
#undef QD6_ROLL
#undef QD6_COLD


#ifndef QD3_HOST
// coder_smem_init (qlfc_coder.cuh) for any layout: same statements, sizes from LY
template <class LY> __device__ __forceinline__ void coder_smem_init_t(CoderSmemT<LY> &S, const QTables *__restrict__ g)
{
    const u32 lane = threadIdx.x & 31;
    if (!LY::TG) {
        const uint4 *src = (const uint4 *)g; uint4 *dst = (uint4 *)S.rank_state;  // rank_state and run_state are contiguous
        for (u32 i = lane; i < sizeof(QTables) / 16; i += 32) dst[i] = src[i];
    }
    u32 *w = (u32 *)S.s16;
    for (u32 i = lane; i < LY::S16_COUNT / 2; i += 32) w[i] = 0x08000800u;        // every counter starts at 2048
    u32 *t = (u32 *)S.tag_state;
    for (u32 i = lane; i < (2 * LY::SLOTS * 2 + 512 + 288) / 4; i += 32) t[i] = 0; // tags, histories, mtf
    __syncwarp();
}

template <class LY> __device__ __forceinline__ void qd6_smem_init(u8 *raw, const QTables *__restrict__ g)
{
    const u32 lane = threadIdx.x & 31;
    if (!LY::TG) {
        const uint4 *src = (const uint4 *)g; uint4 *dst = (uint4 *)raw;                               // rank_state and run_state are contiguous
        for (u32 i = lane; i < sizeof(QTables) / 16; i += 32) dst[i] = src[i];
    }
    u32 *w = (u32 *)(raw + (LY::O_S16 - LY::SHIFT));
    for (u32 i = lane; i < LY::S16_COUNT / 2; i += 32) w[i] = 0x08000800u;                            // every counter starts at 2048
    u32 *t = (u32 *)(raw + (LY::O_TAG_STATE - LY::SHIFT));
    for (u32 i = lane; i < (LY::BYTES + LY::SHIFT - LY::O_TAG_STATE) / 4; i += 32) t[i] = 0;          // tags, histories, mtf, window
    __syncwarp();
}

template <class LY, bool PROF> __global__ void __launch_bounds__(32) q_decode6(const u8 *__restrict__ in_all, SubBlock *__restrict__ sbs, short *__restrict__ cold_all,
                                                                              const QTables *__restrict__ tables, u8 *__restrict__ out_all, const u32 *__restrict__ sb_list, DoneSignal done)   // the moves table (QD6_MOVES ints) follows the QTables
{
    extern __shared__ __align__(16) u8 q_smem_raw[];
    qd6_smem_init<LY>(q_smem_raw, tables);
    SM3 sm; sm.b = (u32)__cvta_generic_to_shared(q_smem_raw) - LY::SHIFT;        // u32 wrap-around is intended: every offset used is >= SHIFT
    asm volatile("" : "+r"(sm.b) :: "memory");
    const u32 sid = sb_list[blockIdx.x];
    SubBlock &sb = sbs[sid];
    short *cold_s = cold_all + (size_t)blockIdx.x * 2 * COLD_PAD, *cold_c = cold_s + COLD_PAD;
    u32 st_cached = 0, st_miss = 0;
    const int r = qd6_decode_stream<LY, PROF>(sm, in_all + sb.out_off, sb.out_cap, out_all + sb.in_start, sb.in_size, cold_s, cold_c, (const int *)(tables + 1), (const u8 *)tables, st_cached, st_miss);
    __syncwarp();                                        // every lane's output stores precede lane 0's report
    if (threadIdx.x == 0) { sb.result = r; sb.stat_cached = st_cached; sb.stat_miss = st_miss; signal_done(done); }
}

#endif
