// libbsc_b200/csrc/qlfc_lanes.cuh -- plumbing shared by the single-warp QLFC coders (static decoder qlfc_decoder6.cuh, adaptive
// coder qlfc_adaptive.cuh, fast coder qlfc_fast.cuh): the shared-memory image accessor SM3, the range-decoder registers Rc3, the
// per-lane registers Qd3Lane, and the QD3_* macros that let THE SAME SOURCE compile for the host (tools/qdec3_host.cpp, QD3_HOST):
// there the 32 lanes are emulated one after the other, so the lane logic is checked bit-for-bit against the reference's streams on
// the CPU (tests/test_qdec3_host.py).  (Three more decoder generations
// once lived in this file; they lost the A/B and are gone.)
#pragma once

#include <cstddef>

#ifdef QD3_HOST
#define QD3_FN static inline
#define QD3_FN_MEMBER
#define QD3_LANES for (u32 lane = 0; lane < 32; ++lane)
#define QD3_L(x) x[lane]
#define QD3_SYNC() do { } while (0)
#define QD3_PARAM(k, i) ((int)bscb_static_params[k][i])
#else
#define QD3_PARAM(k, i) ((int)c_params[k][i])     // lane-dependent class: a run-time look-up (once per stream)
#define QD3_FN __device__ __forceinline__
#define QD3_FN_MEMBER __device__ __forceinline__
#define QD3_LANES
#define QD3_L(x) x
#define QD3_SYNC() __syncwarp()
#endif

struct Dec3Smem {
    CoderSmem cs;
    alignas(16) u16 px[16];      // [0] rank first-bit, [1..7] rank exponent k = 0..6, [8..15] run first-bit for rank class q = 0..7
    alignas(16) u8  st2[16];     // [q] run state for rank class q
    alignas(16) u16 pm[128];     // rank mantissa probabilities at the compact row offsets 1..61 (+ slack for the pair loads)
    alignas(16) u8  win[272];    // staged window of the input stream
};
constexpr u32 O3_PX = (u32)offsetof(Dec3Smem, px), O3_ST2 = (u32)offsetof(Dec3Smem, st2), O3_PM = (u32)offsetof(Dec3Smem, pm), O3_WIN = (u32)offsetof(Dec3Smem, win);
constexpr u32 O3_RANK_STATE = (u32)offsetof(CoderSmem, rank_state), O3_RUN_STATE = (u32)offsetof(CoderSmem, run_state);
constexpr u32 O3_TAG_STATE = (u32)offsetof(CoderSmem, tag_state), O3_TAG_CHAR = (u32)offsetof(CoderSmem, tag_char);
constexpr u32 O3_RANK_HIST = (u32)offsetof(CoderSmem, rankHist), O3_RUN_HIST = (u32)offsetof(CoderSmem, runHist);
constexpr u32 O3_MTF = (u32)offsetof(CoderSmem, mtf), O3_S16 = (u32)offsetof(CoderSmem, s16);
constexpr u32 QD3_WIN_BYTES = 272, QD3_RUN_ROOM = 100;      // refill at a run start when more than this is consumed: 100 + 152 + 2 < 272

struct U4 { u32 x, y, z, w; };
struct U2 { u32 x, y; };

// shared-memory accessors on an explicit base (byte offsets inside Dec3Smem); an explicit base keeps the address arithmetic in 32 bits
struct SM3 {
#ifdef QD3_HOST
    u8 *b;
    u32 ld8(u32 off) const { return b[off]; }
    u32 ld16(u32 off) const { u16 v; memcpy(&v, b + off, 2); return v; }
    u32 ld32(u32 off) const { u32 v; memcpy(&v, b + off, 4); return v; }
    U2  ld64(u32 off) const { U2 v; memcpy(&v, b + off, 8); return v; }
    U4  ld128(u32 off) const { U4 v; memcpy(&v, b + off, 16); return v; }
    void st8(u32 off, u32 v) const { b[off] = (u8)v; }
    void st16(u32 off, u32 v) const { u16 t = (u16)v; memcpy(b + off, &t, 2); }
    u32 at(u32 off) const { return off; }                              // "absolute address" of an offset (host: the offset itself)
    u32 ld16a(u32 a) const { return ld16(a); }
    void st16a(u32 a, u32 v) const { st16(a, v); }
#else
    u32 b;
    __device__ __forceinline__ u32 ld8(u32 off) const { u32 v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(b + off)); return v; }
    __device__ __forceinline__ u32 ld16(u32 off) const { u32 v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(b + off)); return v; }
    __device__ __forceinline__ u32 ld32(u32 off) const { u32 v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(b + off)); return v; }
    __device__ __forceinline__ U2  ld64(u32 off) const { U2 v; asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(b + off)); return v; }
    __device__ __forceinline__ U4  ld128(u32 off) const { U4 v; asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(b + off)); return v; }
    __device__ __forceinline__ void st8(u32 off, u32 v) const { asm volatile("st.shared.u8 [%0], %1;" :: "r"(b + off), "r"(v) : "memory"); }
    __device__ __forceinline__ void st16(u32 off, u32 v) const { asm volatile("st.shared.u16 [%0], %1;" :: "r"(b + off), "r"(v) : "memory"); }
    __device__ __forceinline__ u32 at(u32 off) const { return b + off; }     // absolute shared-memory address of an offset
    __device__ __forceinline__ u32 ld16a(u32 a) const { u32 v; asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
    __device__ __forceinline__ void st16a(u32 a, u32 v) const { asm volatile("st.shared.u16 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
#endif
    // counters (indices in u16 units, as in qlfc_coder.cuh)
    QD3_FN_MEMBER int cnt(u32 idx) const { return (int)ld16(O3_S16 + 2u * idx); }
    QD3_FN_MEMBER void set(u32 idx, int v) const { st16(O3_S16 + 2u * idx, (u32)v); }
};

QD3_FN int qd3_ilog2(u32 v) {
#ifdef QD3_HOST
    return 31 - __builtin_clz(v | 1u);
#else
    return 31 - __clz(v | 1u);
#endif
}

// Index (into the counter file) of rare counter `idx` through the direct-mapped write-back cache (uniform).
QD3_FN u32 qd3_cache_get(const SM3 &sm, u32 val_base, u32 tags_off, short *__restrict__ cold, u32 idx, u32 &misses)
{
    const u32 slot = cache_slot(idx), want = cache_tag(idx);
    const u32 t = sm.ld16(tags_off + 2u * slot);
    if (t != want) {
        if (t) cold[cache_unslot(slot, t)] = (short)sm.cnt(val_base + slot);
        sm.set(val_base + slot, (u16)cold[idx]);
        sm.st16(tags_off + 2u * slot, want);
        ++misses;
    }
    return val_base + slot;
}

// ---- range decoder (rangecoder.h:203-240), branch-free step ---------------------------------------------------
struct Rc3 {
    const u8 *in; u32 limit;
    u32 code, range;
    u32 nx;                          // the 16-bit unit at `pos`, already loaded
    u32 pos, wbase;                  // next unread unit (byte offset in the stream, always even); window = [wbase, wbase + 272)
};

// one decision with P(bit = 0) = p / 4096
QD3_FN u32 qd3_step(const SM3 &sm, Rc3 &rc, u32 p)
{
    const bool need = rc.range < 0x10000u;
    rc.code = need ? (rc.code << 16) | rc.nx : rc.code;
    rc.range = need ? rc.range << 16 : rc.range;
    rc.pos += need ? 2u : 0u;
    rc.nx = sm.ld16(O3_WIN + (rc.pos - rc.wbase));
    const u32 r = (rc.range >> 12) * p;
    const bool bit = rc.code >= r;
    rc.code -= bit ? r : 0u;
    rc.range = bit ? rc.range - r : r;
    return bit ? 1u : 0u;
}

// one serial decision against three counters of the shared counter file (the rare paths)
template <int K> QD3_FN u32 qd3_dec3(const SM3 &sm, Rc3 &rc, u32 is, u32 ic, u32 ig)
{
    const int s = sm.cnt(is), c = sm.cnt(ic), g = sm.cnt(ig);
    const u32 b = qd3_step(sm, rc, (u32)q_mix<K>(s, c, g));
    sm.set(is, b ? q_down<K, 0>(s) : q_up<K, 0>(s));
    sm.set(ic, b ? q_down<K, 1>(c) : q_up<K, 1>(c));
    sm.set(ig, b ? q_down<K, 2>(g) : q_up<K, 2>(g));
    return b;
}

// ---- per-lane registers ------------------------------------------------------------------------------------------
struct Qd3Lane {
    // two mantissa-tree slots: compact row offsets lane and lane + 32
    u32 okA, eA, jA, dA, gxA;        // is a real node; its exponent (level), node number, depth of the node, shared-counter index
    u32 okB, eB, jB, dB, gxB;
    // slot X: lane 0 rank first-bit, 1..7 rank exponent k = lane - 1, 8..15 run first-bit for rank class q = lane - 8 (16..31 mirror 0..15, never store)
    u32 xS, xC, xG, xMul;            // state index = xS + (state) * xMul, symbol index = xC + c * xMul, shared index = xG
    int xw0, xw1, xw2;               // mix weights (symbol, state, shared)
    int xMs0, xKs0, xMs1, xKs1, xMc0, xKc0, xMc1, xKc1, xMg0, xKg0, xMg1, xKg1;   // counter moves (state/symbol/shared, bit 0/1): v' = (v * M + K) >> 12
    // values loaded by the evaluation phase, used again by the update phase
    int sA, cA, gA, sB, cB, gB, sX, cX, gX;
    u32 iSX, iCX;
    u32 used8, tmp;
    u32 mtfv;                        // qlfc_decoder6.cuh: lane l holds position l of the MTF list
};

QD3_FN void qd3_lane_init(Qd3Lane &r, u32 lane)
{
#define QD3_SLOT(o_, OK, E, J, D, GX) { const u32 o = (o_); const u32 e = (u32)qd3_ilog2(o + 2u), j = o + 2u - (1u << e); \
        const u32 ok = (j >= 1u && e >= 1u && e <= M_MAXE && o < M_ROW) ? 1u : 0u; \
        r.OK = ok; r.E = e; r.J = j; r.D = (u32)qd3_ilog2(j); r.GX = R_WIDE_SHARED + (ok ? e * 256u + j : 0u); }
    QD3_SLOT(lane, okA, eA, jA, dA, gxA) QD3_SLOT(lane + 32u, okB, eB, jB, dB, gxB)
#undef QD3_SLOT
    const u32 l = lane & 15u;
    int k;
    if (l == 0)     { k = K_RANK_T; r.xS = R_RT_STATE; r.xC = R_RT_CHAR; r.xG = R_RT_SHARED; r.xMul = 1; }
    else if (l < 8) { k = K_RANK_E; r.xS = R_RE_STATE + (l - 1); r.xC = R_RE_CHAR + (l - 1); r.xG = R_RE_SHARED + (l - 1); r.xMul = 8; }
    else            { k = K_RUN_T;  r.xS = R_UT_STATE; r.xC = R_UT_CHAR; r.xG = R_UT_SHARED; r.xMul = 1; }
    r.xw0 = QD3_PARAM(k, 0); r.xw1 = QD3_PARAM(k, 1); r.xw2 = QD3_PARAM(k, 2);
#define QD3_MOVE(who, M0, K0, M1, K1) { const int th0 = QD3_PARAM(k, 3 + 4 * who), ar0 = QD3_PARAM(k, 4 + 4 * who), th1 = QD3_PARAM(k, 5 + 4 * who), ar1 = QD3_PARAM(k, 6 + 4 * who); \
        r.M0 = 4096 - ar0; r.K0 = (4096 - th0) * ar0;  /* q_up */  r.M1 = 4096 - ar1; r.K1 = th1 * ar1 + 4095;  /* q_down */ }
    QD3_MOVE(0, xMs0, xKs0, xMs1, xKs1) QD3_MOVE(1, xMc0, xKc0, xMc1, xKc1) QD3_MOVE(2, xMg0, xKg0, xMg1, xKg1)
#undef QD3_MOVE
    r.sA = r.cA = r.gA = r.sB = r.cB = r.gB = r.sX = r.cX = r.gX = 0; r.iSX = r.iCX = 0; r.used8 = 0; r.tmp = 0;
}

#ifdef QD3_HOST
#define QD3_LREGS Qd3Lane lr[32]
#define QD3_LREGS_PARAM Qd3Lane (&lr)[32]
#else
#define QD3_LREGS Qd3Lane lr
#define QD3_LREGS_PARAM Qd3Lane &lr
#endif

// (re)load the input window at rc.pos: 8 bytes per lane + 16 more by lanes 0..15
#define QD3_REFILL() do { rc.wbase = rc.pos; QD3_SYNC(); \
        QD3_LANES { for (u32 k_ = 0; k_ < 8; ++k_) { const u32 w_ = lane * 8u + k_, o_ = rc.wbase + w_; sm.st8(O3_WIN + w_, o_ < rc.limit ? rc.in[o_] : 0u); } \
                    if (lane < 16u) { const u32 w_ = 256u + lane, o_ = rc.wbase + w_; sm.st8(O3_WIN + w_, o_ < rc.limit ? rc.in[o_] : 0u); } } \
        QD3_SYNC(); } while (0)

// which symbols can still appear in the MTF-order header (qlfc.cpp:857-891): lane l owns symbols 8l..8l+7
#ifdef QD3_HOST
#define QD3_HEADER_OPTIONS(prev, prefix, bit, can0, can1) do { can0 = can1 = false; \
        for (u32 lane = 0; lane < 32; ++lane) for (int k_ = 0; k_ < 8; ++k_) { const int c_ = 8 * (int)lane + k_; \
            if ((c_ == (prev) || !((lr[lane].used8 >> k_) & 1u)) && ((c_ >> ((bit) + 1)) == (prefix))) { if (c_ & (1 << (bit))) can1 = true; else can0 = true; } } } while (0)
#else
#define QD3_HEADER_OPTIONS(prev, prefix, bit, can0, can1) header_options(lr.used8, (prev), (prefix), (bit), can0, can1)
#endif

// PROF (device only, BSCB200_QDEC_PROF=1): cycle counts per phase, printed for the first stream of the launch.
#ifdef QD3_HOST
#define QD3_T(k) do { } while (0)
#else
#define QD3_T(k) do { if (PROF) { const long long t_ = clock64(); prof_t[k] += t_ - prof_last; prof_last = t_; } } while (0)
#endif
