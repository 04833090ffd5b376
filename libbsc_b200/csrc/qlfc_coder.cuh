// libbsc_b200/csrc/qlfc_coder.cuh -- QLFC stage 2 (context model + binary range coder), device engine.
// Included by qlfc.cu inside its anonymous namespace (needs SubBlock, QTables, K_*, bscb_param).
//
// Why this looks the way it does.  One coder stream is a strictly serial recurrence (every binary
// decision reads three adaptive counters whose addresses depend on the previous decisions, then
// updates them and the range coder).  The format allows only <= 8 streams per block
// (coder.cpp:52-59), so per-stream LATENCY is everything.  Counters in global memory cost an L2 round
// trip per load, and small shared-memory caches in front of them did not hold the working set, so the counter file is now laid out for shared memory: one SM per stream holds
//
//   * state tables                                  40 KB  (tables.h data, qlfc_tables.inc)
//   * first-bit, unary-exponent (index < 8) and model-wide shared counters      25 KB
//   * mantissa counters for exponents 1..5, stored COMPACTLY (2^e - 1 tree nodes per row instead of
//     the reference's 256/32-wide rows: 62 entries per state / symbol)          124 KB
//   * two small direct-mapped write-back caches (4 K entries each) for everything rare: rank
//     exponents 6-7, the escape bank, run exponents >= 6 and run-exponent indices >= 8; the
//     1.7 M counters behind them live in HBM                                    24 KB
//
// The decoder (qlfc_decoder6.cuh) is one lock-step warp per stream; the encoder (qlfc_encoder.cuh) is a
// six-warp pipeline per stream.
#pragma once

// ---- shared-memory counter file (indices in u16 units) ---------------------------------------------
constexpr u32 R_RT_SHARED = 0, R_RT_STATE = 2, R_RT_CHAR = R_RT_STATE + 256;
constexpr u32 R_RE_SHARED = R_RT_CHAR + 256, R_RE_STATE = R_RE_SHARED + 8, R_RE_CHAR = R_RE_STATE + 2048;
constexpr u32 R_UT_SHARED = R_RE_CHAR + 2048, R_UT_STATE = R_UT_SHARED + 2, R_UT_CHAR = R_UT_STATE + 256;
constexpr u32 UE_RES = 8;                                   // run-exponent indices kept resident
constexpr u32 R_UE_SHARED = R_UT_CHAR + 256, R_UE_STATE = R_UE_SHARED + 32, R_UE_CHAR = R_UE_STATE + 256 * UE_RES;
constexpr u32 R_WIDE_SHARED = R_UE_CHAR + 256 * UE_RES;    // 9 banks x 256 (rank mantissa e=0..7, escape)
constexpr u32 R_NARROW_SHARED = R_WIDE_SHARED + 9 * 256;   // 32 banks x 32 (run mantissa)
constexpr u32 M_ROW = 62;                                   // compact row: exponents 1..5 -> offsets 2^e-2 .. 2^(e+1)-3
constexpr u32 M_MAXE = 5;
constexpr u32 R_RM_STATE = R_NARROW_SHARED + 32 * 32, R_RM_CHAR = R_RM_STATE + 256 * M_ROW;
constexpr u32 R_UM_STATE = R_RM_CHAR + 256 * M_ROW, R_UM_CHAR = R_UM_STATE + 256 * M_ROW;
constexpr u32 R_END = R_UM_CHAR + 256 * M_ROW;

constexpr int  QC_LOG = 12;                                 // 4 K entries per cache
constexpr u32  QC_SLOTS = 1u << QC_LOG, QC_MASK = QC_SLOTS - 1;
constexpr u32  C_STATE_VAL = R_END;                         // cache of the by-state rare banks
constexpr u32  C_CHAR_VAL = C_STATE_VAL + QC_SLOTS;         // cache of the by-symbol rare banks
constexpr u32  S16_COUNT = (C_CHAR_VAL + QC_SLOTS + 1) & ~1u;
// index space behind each cache: 9 wide banks x [256][256], 32 narrow banks x [256][32], run exponent [256][32]
constexpr u32  COLD_WIDE = 65536, COLD_NARROW = 8192;
constexpr u32  COLD_UE = 9 * COLD_WIDE + 32 * COLD_NARROW;
constexpr u32  COLD_COUNT = COLD_UE + 8192;
constexpr u32  COLD_PAD = (COLD_COUNT + 255) & ~255u;
// Slot of a cold index: 11 hashed bits + 1 class bit (rank banks / run banks never share a slot, so the
// encoder's rank-model warp and run-model warp can use the caches concurrently).
// 10 hashed bits + 2 class bits: classes 0,1 = rank banks (rank mantissa e>5, escape), 2 = run mantissa
// e>5, 3 = run exponent index >= 8.  The encoder's model warps each touch exactly one class group, so
// they can use the caches concurrently without ever sharing a slot.
__device__ __forceinline__ u32 cache_slot(u32 idx)
{
    const u32 h = idx >> 10;
    const u32 cls = idx < 9u * 65536u ? (h & 1u) : (idx < 9u * 65536u + 32u * 8192u ? 2u : 3u);
    return (cls << 10) | ((idx ^ (h * 1237u)) & 1023u);
}
__device__ __forceinline__ u32 cache_tag(u32 idx) { return (idx >> 10) + 1u; }
__device__ __forceinline__ u32 cache_unslot(u32 slot, u32 tag) { const u32 h = tag - 1u; return (h << 10) | (((slot & 1023u) ^ (h * 1237u)) & 1023u); }

struct CoderSmem {
    u8    rank_state[32768];
    u8    run_state[8192];
    u16   s16[S16_COUNT];
    u16   tag_state[QC_SLOTS];   // 0 = empty, else 1 + (cold index >> 11)
    u16   tag_char[QC_SLOTS];
    u8    rankHist[256], runHist[256];
    u8    mtf[256 + 32];
    __align__(16) u8 inwin[256];     // decoder: staged window of the input stream
};

__device__ __forceinline__ void coder_smem_init(CoderSmem &S, const QTables *__restrict__ g)
{
    const u32 lane = threadIdx.x & 31;
    const uint4 *src = (const uint4 *)g; uint4 *dst = (uint4 *)S.rank_state;      // rank_state and run_state are contiguous
    for (u32 i = lane; i < sizeof(QTables) / 16; i += 32) dst[i] = src[i];
    u32 *w = (u32 *)S.s16;
    for (u32 i = lane; i < S16_COUNT / 2; i += 32) w[i] = 0x08000800u;            // every counter starts at 2048
    u32 *t = (u32 *)S.tag_state;
    for (u32 i = lane; i < (2 * QC_SLOTS * 2 + 512 + 288) / 4; i += 32) t[i] = 0; // tags, histories, mtf
    __syncwarp();
}

__device__ __forceinline__ u32 wide_idx(u32 bank, u32 x, u32 node) { return bank * COLD_WIDE + x * 256 + node; }
__device__ __forceinline__ u32 narrow_idx(u32 e, u32 x, u32 node) { return 9 * COLD_WIDE + e * COLD_NARROW + x * 32 + node; }
__device__ __forceinline__ u32 ue_idx(u32 x, u32 k) { return COLD_UE + x * 32 + k; }
__device__ __forceinline__ u32 m_off(u32 e, u32 node) { return (1u << e) - 2u + node; }   // position inside a compact row

// ---- counters ---------------------------------------------------------------------------------------
// All parameters are compile-time immediates (bscb_param is constexpr).  Counters provably stay in
// [1, 4095] from their start value 2048 for every parameter set, so they are kept as unsigned 16-bit.
template <int K> __device__ __forceinline__ int q_mix(int s, int c, int g)
{
    return (c * bscb_param(K, 0) + s * bscb_param(K, 1) + g * bscb_param(K, 2)) >> 5;
}
// Counter moves as ONE multiply-add and ONE shift.  With integer p:
//   bit 0 (predictor.h:50-53):  p + floor(((4096-TH0-p)*AR0)/4096) = floor((p*(4096-AR0) + (4096-TH0)*AR0) / 4096)
//   bit 1 (predictor.h:55-58):  p - floor(((p-TH1)*AR1)/4096)      = floor((p*(4096-AR1) + TH1*AR1 + 4095) / 4096)
// (checked exhaustively for p in [0,4096] and all 21 parameter sets; tests/test_oracle.py)
template <int K, int WHO> __device__ __forceinline__ int q_up(int p)
{
    return (p * (4096 - bscb_param(K, 4 + 4 * WHO)) + (4096 - bscb_param(K, 3 + 4 * WHO)) * bscb_param(K, 4 + 4 * WHO)) >> 12;
}
template <int K, int WHO> __device__ __forceinline__ int q_down(int p)
{
    return (p * (4096 - bscb_param(K, 6 + 4 * WHO)) + bscb_param(K, 5 + 4 * WHO) * bscb_param(K, 6 + 4 * WHO) + 4095) >> 12;
}

// ---- range coder (rangecoder.h:38-271), 16-bit units -------------------------------------------------
struct Rc2Enc {
    u64 low;                          // bits 0..31 = low32, bit 32 = pending carry (rangecoder.h:43-52 `ari.low`)
    u32 range, cache, pending, pos;
    u8 *out;
    __device__ __forceinline__ void init(u8 *o) { low = 0; range = 0xffffffffu; cache = 0; pending = 0; pos = 0; out = o; }
    __device__ __forceinline__ void put16(u32 v) { *(u16 *)(out + pos) = (u16)v; pos += 2; }   // all lanes store the same value
    __device__ __forceinline__ void shift() {
        const u32 low32 = (u32)low, carry = (u32)(low >> 32);
        if (low32 < 0xffff0000u || carry) {
            put16(cache + carry);
#pragma unroll 1
            for (; pending; --pending) put16(carry - 1);        // one time in 65536: keep it small
            cache = low32 >> 16;
        } else pending++;
        low = (u64)(u32)(low32 << 16);
    }
    // branch-free step: low += bit ? r : 0 ; range = bit ? range - r : r
    __device__ __forceinline__ void step(u32 bit, u32 p) {
        const u32 r = (range >> 12) * p;
        low += bit ? (u64)r : 0ull;
        range = bit ? range - r : r;
    }
    __device__ __forceinline__ void encode(u32 bit, int p) {
        if (range < 0x10000u) { shift(); range <<= 16; }
        step(bit, (u32)p);
    }
    __device__ u32 finish() { if (range < 0x10000u) shift(); shift(); shift(); shift(); return pos; }
};
