// libbsc_b200/csrc/qlfc_fast.cuh -- the FAST QLFC coder (coder id 3, `-e0`): encoder qlfc.cpp:1135-1336, decoder 1933-2127,
// model qlfc_model.h:243-259 (QlfcStatisticalModel2), start values qlfc_model.cpp:73-74, counter moves predictor.h:63-71,
// range coder rangecoder.h:145-177 / 213-240 with the precision template (13 bits for ranks, 11 for run lengths).
// Included by qlfc.cu after qlfc_lanes.cuh (uses SM3, Rc3 and the QD3_* dual-compile macros); ALSO compiled for the
// host by tools/qdec3_host.cpp, which runs this very source with 32 emulated lanes against the oracle on the CPU
// (tests/test_qdec3_host.py).
//
// The fast coder has ONE adaptive counter per binary decision, picked by the run's symbol and the position inside the
// code only (no states, no mixing), so the whole counter file is 84 KB: exponent rows [256][8] and [256][32], mantissa
// trees for exponents 1..5 stored compactly (62 nodes per symbol, as in qlfc_coder.cuh), and one small direct-mapped
// write-back cache in front of the rare remainder (rank exponents 6-7, run exponents > 5; 768 KB in HBM per stream).
// Both directions are one lock-step warp per stream for now: a decision is one shared-memory load, one shift-update
// and one branch-free range-coder step.
// STATUS: bit-exact in host emulation and on the GPU (tests/test_gpu_other_coders.py, tests/test_gpu_pipeline.py); enabled
// without any switch (coder_gate in qlfc.cu).
#pragma once

constexpr u32 QF_ROW = 62, QF_MAXE = 5;                        // compact mantissa row: exponents 1..5 at offsets 2^e-2 .. 2^(e+1)-3
constexpr u32 QF_CLOG = 12, QF_CSLOTS = 1u << QF_CLOG;         // write-back cache entries
constexpr u32 QF_COLD_RANK = 256u * 2u * 256u;                 // [symbol][exponent 6..7][node]
constexpr u32 QF_COLD_RUN = 256u * 32u * 32u;                  // [symbol][exponent][context]
constexpr u32 QF_COLD = QF_COLD_RANK + QF_COLD_RUN;            // shorts per stream in HBM

struct FastSmem {
    u16 re[256 * 8];             // rank exponent counters   (13-bit probabilities, start 4096)
    u16 rm[256 * QF_ROW];        // rank mantissa, exponents 1..5
    u16 ue[256 * 32];            // run exponent counters    (11-bit probabilities, start 1024)
    u16 um[256 * QF_ROW];        // run mantissa, exponents 1..5
    u16 cval[QF_CSLOTS];         // cache of the cold counters
    u16 ctag[QF_CSLOTS];         // 0 = empty, else 1 + (cold index >> QF_CLOG)
    alignas(16) u8 mtf[256 + 32];
    alignas(16) u8 win[272];     // decoder: staged window of the input stream
};
constexpr u32 OF_RE = (u32)offsetof(FastSmem, re), OF_RM = (u32)offsetof(FastSmem, rm), OF_UE = (u32)offsetof(FastSmem, ue), OF_UM = (u32)offsetof(FastSmem, um);
constexpr u32 OF_CVAL = (u32)offsetof(FastSmem, cval), OF_CTAG = (u32)offsetof(FastSmem, ctag), OF_MTF = (u32)offsetof(FastSmem, mtf), OF_WIN = (u32)offsetof(FastSmem, win);

// byte offset (in shared memory) of cold counter `idx`, through the cache (uniform: every lane does the same)
QD3_FN u32 qf_cold(const SM3 &sm, short *__restrict__ cold, u32 idx, u32 &misses)
{
    const u32 slot = idx & (QF_CSLOTS - 1u), want = (idx >> QF_CLOG) + 1u;
    const u32 t = sm.ld16(OF_CTAG + 2u * slot);
    if (t != want) {
        if (t) cold[((t - 1u) << QF_CLOG) | slot] = (short)sm.ld16(OF_CVAL + 2u * slot);
        sm.st16(OF_CVAL + 2u * slot, (u16)cold[idx]);
        sm.st16(OF_CTAG + 2u * slot, want);
        ++misses;
    }
    return OF_CVAL + 2u * slot;
}

struct QfLane { u32 used8, tmp, sym, rank, len; };             // per-lane registers (header bookkeeping, MTF rotation, run records)
#ifdef QD3_HOST
#define QF_LREGS QfLane lr[32]
#else
#define QF_LREGS QfLane lr
#endif

// counter move predictor.h:63-71: p -= (p - target) >> R   (arithmetic shift of a signed difference)
template <int R, int TO0, int TO1> QD3_FN int qf_move(int p, u32 bit) { return p - ((p - (bit ? TO1 : TO0)) >> R); }

// ---- decoder ----------------------------------------------------------------------------------------------------
#define QF_REFILL() do { rc.wbase = rc.pos; QD3_SYNC(); \
        QD3_LANES { for (u32 k_ = 0; k_ < 8; ++k_) { const u32 w_ = lane * 8u + k_, o_ = rc.wbase + w_; sm.st8(OF_WIN + w_, o_ < rc.limit ? rc.in[o_] : 0u); } \
                    if (lane < 16u) { const u32 w_ = 256u + lane, o_ = rc.wbase + w_; sm.st8(OF_WIN + w_, o_ < rc.limit ? rc.in[o_] : 0u); } } \
        QD3_SYNC(); } while (0)

// one decision with P(bit = 0) = p / 2^P  (rangecoder.h:224-240), branch-free, next unit preloaded
template <int P> QD3_FN u32 qf_step(const SM3 &sm, Rc3 &rc, u32 p)
{
    const bool need = rc.range < 0x10000u;
    rc.code = need ? (rc.code << 16) | rc.nx : rc.code;
    rc.range = need ? rc.range << 16 : rc.range;
    rc.pos += need ? 2u : 0u;
    rc.nx = sm.ld16(OF_WIN + (rc.pos - rc.wbase));
    const u32 r = (rc.range >> P) * p;
    const bool bit = rc.code >= r;
    rc.code -= bit ? r : 0u;
    rc.range = bit ? rc.range - r : r;
    return bit ? 1u : 0u;
}

// decision against the counter at shared-memory byte offset `off`
template <int P, int R, int TO0, int TO1> QD3_FN u32 qf_dec(const SM3 &sm, Rc3 &rc, u32 off)
{
    const int x = (int)sm.ld16(off);
    const u32 b = qf_step<P>(sm, rc, (u32)x);
    sm.st16(off, (u32)qf_move<R, TO0, TO1>(x, b));
    return b;
}

// Decodes one fast-coder stream into out[0 .. n).  `sm` points at an initialised FastSmem (counters at their start
// values, the rest zero), `cold` at QF_COLD initialised shorts.  Returns the decoded length or a libbsc error code.
QD3_FN int qf_decode_stream(const SM3 &sm, const u8 *__restrict__ in, u32 in_limit, u8 *__restrict__ out, u32 out_cap,
                            short *__restrict__ cold, u32 &st_cached, u32 &st_miss)
{
    QF_LREGS;
#ifndef QD3_HOST
    const u32 lane = threadIdx.x & 31u;
#endif
    QD3_LANES { QD3_L(lr).used8 = 0; QD3_L(lr).tmp = 0; }
    Rc3 rc; rc.in = in; rc.limit = in_limit; rc.code = 0; rc.range = 0xffffffffu; rc.pos = 0; rc.wbase = 0; rc.nx = 0;
    QF_REFILL();
    rc.code = (sm.ld16(OF_WIN + 2) << 16) | sm.ld16(OF_WIN + 4);
    rc.pos = 6; rc.nx = sm.ld16(OF_WIN + 6);
    u32 n = 0;
    for (int b = 0; b < 32; ++b) n = (n << 1) | qf_step<12>(sm, rc, 2048u);          // DecodeWord: 32 plain bits
    if (n > out_cap) return LIBBSC_DATA_CORRUPT;
    {
        int prev = -1;
        for (int d = 0; d < 256; ++d) {
            int c = 0;
            for (int bit = 7; bit >= 0; --bit) {
                bool can0, can1; QD3_HEADER_OPTIONS(prev, c, bit, can0, can1);
                if (can0 && can1) {
                    if (rc.pos - rc.wbase > 256u) QF_REFILL();
                    c = 2 * c + (int)qf_step<1>(sm, rc, 1u);                          // qlfc.cpp:1970: DecodeBit<1>(1)
                }
                else if (can1) c = 2 * c + 1;
                else if (can0) c = 2 * c;
            }
            c &= 255;
            sm.st8(OF_MTF + d, (u32)c);
            if (c == prev) break;
            prev = c;
            QD3_LANES { if ((u32)(c >> 3) == lane) QD3_L(lr).used8 |= 1u << (c & 7); }
        }
    }
    QD3_SYNC();

    u32 c, m1, m2, m3;
    { const u32 f = sm.ld32(OF_MTF); c = f & 255u; m1 = (f >> 8) & 255u; m2 = (f >> 16) & 255u; m3 = f >> 24; }
    for (u32 i = 0; i < n; ) {
        if (rc.pos - rc.wbase > QD3_RUN_ROOM) QF_REFILL();
        // ---- rank (qlfc.cpp:1992-2051) ----
        u32 rank = 1, b;
        const u32 reb = OF_RE + 2u * (c * 8u);
        b = qf_dec<13, 4, 8016, 83>(sm, rc, reb);
        if (b) {
            u32 e = 1;
            while (e < 7) { b = qf_dec<13, 4, 8114, 122>(sm, rc, reb + 2u * e); if (!b) break; ++e; }
            if (e <= QF_MAXE) {
                const u32 mb = OF_RM + 2u * (c * QF_ROW + (1u << e) - 2u);
                for (u32 bit = e; bit > 0; --bit) { b = qf_dec<13, 7, 7999, 235>(sm, rc, mb + 2u * rank); rank = 2u * rank + b; }
            } else {
                for (u32 bit = e; bit > 0; --bit) {
                    const u32 off = qf_cold(sm, cold, (c * 2u + (e - 6u)) * 256u + rank, st_miss); ++st_cached;
                    b = qf_dec<13, 7, 7999, 235>(sm, rc, off); rank = 2u * rank + b;
                }
            }
        }
        rank &= 255u;
        // ---- push c `rank` places back; positions 0..3 of the list live in (c, m1, m2, m3) ----
        const u32 cur = c;
        if (rank == 1) { c = m1; m1 = cur; }
        else if (rank == 2) { c = m1; m1 = m2; m2 = cur; }
        else if (rank == 3) { c = m1; m1 = m2; m2 = m3; m3 = cur; }
        else if (rank != 0) {
            sm.st8(OF_MTF, c); sm.st8(OF_MTF + 1, m1); sm.st8(OF_MTF + 2, m2); sm.st8(OF_MTF + 3, m3);
            QD3_SYNC();
            for (u32 basep = 0; basep < rank; basep += 32) {
                QD3_LANES { QD3_L(lr).tmp = sm.ld8(OF_MTF + basep + lane + 1u); }
                QD3_SYNC();
                QD3_LANES { if (basep + lane < rank) sm.st8(OF_MTF + basep + lane, QD3_L(lr).tmp); }
                QD3_SYNC();
            }
            sm.st8(OF_MTF + rank, cur);
            QD3_SYNC();
            const u32 f = sm.ld32(OF_MTF); c = f & 255u; m1 = (f >> 8) & 255u; m2 = (f >> 16) & 255u; m3 = f >> 24;
        }
        // ---- run length (qlfc.cpp:2053-2121) ----
        u32 run = 1;
        const u32 ueb = OF_UE + 2u * (cur * 32u);
        b = qf_dec<11, 5, 2025, 42>(sm, rc, ueb);
        if (b) {
            u32 e = 1;
            for (;;) { b = qf_dec<11, 4, 1962, 142>(sm, rc, ueb + 2u * e); if (!b) break; if (++e >= 31u) break; }   // 31: corrupt-input guard
            if (e <= QF_MAXE) {
                const u32 mb = OF_UM + 2u * (cur * QF_ROW + (1u << e) - 2u);
                for (u32 bit = e; bit > 0; --bit) { b = qf_dec<11, 6, 1951, 147>(sm, rc, mb + 2u * run); run = 2u * run + b; }
            } else {
                for (u32 ctx = 1; ctx <= e; ++ctx) {
                    const u32 off = qf_cold(sm, cold, QF_COLD_RANK + (cur * 32u + e) * 32u + ctx, st_miss); ++st_cached;
                    b = qf_dec<11, 5, 1987, 46>(sm, rc, off); run = 2u * run + b;
                }
            }
        }
        // ---- run expansion: byte address A is always written by lane A mod 32 ----
        if (run <= 32u && i + 32u <= n) { QD3_LANES { out[i + ((lane - i) & 31u)] = (u8)cur; } }
        else {
            if (run > n - i) run = n - i;
            QD3_LANES { for (u32 k = (lane - i) & 31u; k < run; k += 32) out[i + k] = (u8)cur; }
        }
        i += run;
    }
    return (int)n;
}

// ---- encoder ----------------------------------------------------------------------------------------------------
// rangecoder.h:38-177 with the precision template; 64-bit low (carry in bit 32), 16-bit output units
struct QfEnc {
    u64 low; u32 range, cache, pending, pos; u8 *out;
};
QD3_FN void qf_put16(QfEnc &e, u32 v) { e.out[e.pos] = (u8)v; e.out[e.pos + 1] = (u8)(v >> 8); e.pos += 2; }   // all lanes store the same bytes
QD3_FN void qf_shift(QfEnc &e)
{
    const u32 low32 = (u32)e.low, carry = (u32)(e.low >> 32);
    if (low32 < 0xffff0000u || carry) {
        qf_put16(e, e.cache + carry);
        for (; e.pending; --e.pending) qf_put16(e, carry - 1u);
        e.cache = low32 >> 16;
    } else e.pending++;
    e.low = (u64)(u32)(low32 << 16);
}
template <int P> QD3_FN void qf_encode(QfEnc &e, u32 bit, u32 p)
{
    if (e.range < 0x10000u) { qf_shift(e); e.range <<= 16; }
    const u32 r = (e.range >> P) * p;
    e.low += bit ? (u64)r : 0ull;
    e.range = bit ? e.range - r : r;
}
// EncodeBit<1>(value, 1) with an UNNORMALISED bit value (qlfc.cpp:1174 passes `c & (1 << bit)`): the reference masks
// with (0 - value), which clears the low bits of the addend for value = 2^k -- reproduced exactly.
QD3_FN void qf_encode_half_masked(QfEnc &e, u32 bitval)
{
    if (e.range < 0x10000u) { qf_shift(e); e.range <<= 16; }
    const u32 r = e.range >> 1, m = 0u - bitval;
    e.low += (u64)(m & r);
    e.range = r + (m & (e.range - r - r));
}
template <int P, int R, int TO0, int TO1> QD3_FN void qf_enc(const SM3 &sm, QfEnc &e, u32 off, u32 bit)
{
    const int x = (int)sm.ld16(off);
    sm.st16(off, (u32)qf_move<R, TO0, TO1>(x, bit));
    qf_encode<P>(e, bit, (u32)x);
}

#ifdef QD3_HOST
#define QF_BCAST(field, j) (lr[(j)].field)
#else
#define QF_BCAST(field, j) __shfl_sync(0xffffffffu, lr.field, (int)(j))
#endif

// Encodes runs [run_begin, run_end) (symbols, ranks, positions from the run-detection and rank kernels) of one sub-block.
// Returns the stream length or LIBBSC_NOT_COMPRESSIBLE (qlfc.cpp:1192-1195: output within 16 bytes of its capacity).
QD3_FN int qf_encode_stream(const SM3 &sm, const u32 *__restrict__ run_pos, const u8 *__restrict__ run_sym, const u8 *__restrict__ run_rank,
                            u32 run_begin, u32 run_end, u32 in_size, const u8 *__restrict__ mtf, u8 *__restrict__ out, u32 out_cap,
                            short *__restrict__ cold, u32 &st_cached, u32 &st_miss)
{
    QF_LREGS;
#ifndef QD3_HOST
    const u32 lane = threadIdx.x & 31u;
#endif
    QD3_LANES { QD3_L(lr).used8 = 0; QD3_L(lr).tmp = 0; }
    QfEnc rc; rc.low = 0; rc.range = 0xffffffffu; rc.cache = 0; rc.pending = 0; rc.pos = 0; rc.out = out;
    const long long eob = (long long)out_cap - 16;
    for (int b = 31; b >= 0; --b) qf_encode<12>(rc, (in_size >> b) & 1u, 2048u);
    {
        int prev = -1;
        for (int d = 0; d < 256; ++d) {
            const int c = mtf[d];
            for (int bit = 7; bit >= 0; --bit) {
                bool can0, can1; QD3_HEADER_OPTIONS(prev, c >> (bit + 1), bit, can0, can1);
                if (can0 && can1) qf_encode_half_masked(rc, (u32)(c & (1 << bit)));
            }
            if (c == prev) break;
            prev = c;
            QD3_LANES { if ((u32)(c >> 3) == lane) QD3_L(lr).used8 |= 1u << (c & 7); }
        }
    }
    for (u32 t0 = run_begin; t0 < run_end; t0 += 32) {
        const u32 cnt = run_end - t0 < 32u ? run_end - t0 : 32u;
        // lane j fetches run t0 + j (coalesced); the serial loop below broadcasts one run at a time
        QD3_LANES {
            QfLane &r = QD3_L(lr);
            r.sym = 0; r.rank = 1; r.len = 1;
            if (lane < cnt) { r.sym = run_sym[t0 + lane]; r.rank = run_rank[t0 + lane]; r.len = run_pos[t0 + lane + 1] - run_pos[t0 + lane]; }
        }
        for (u32 j = 0; j < cnt; ++j) {
            if ((long long)rc.pos >= eob) return LIBBSC_NOT_COMPRESSIBLE;
            const u32 c = QF_BCAST(sym, j), rank = QF_BCAST(rank, j), run = QF_BCAST(len, j);
            // ---- rank (qlfc.cpp:1240-1275) ----
            const u32 reb = OF_RE + 2u * (c * 8u);
            qf_enc<13, 4, 8016, 83>(sm, rc, reb, rank != 1u ? 1u : 0u);
            if (rank != 1u) {
                const u32 e = (u32)qd3_ilog2(rank);
                for (u32 b = 1; b < e; ++b) qf_enc<13, 4, 8114, 122>(sm, rc, reb + 2u * b, 1u);
                if (e < 7u)                 qf_enc<13, 4, 8114, 122>(sm, rc, reb + 2u * e, 0u);
                if (e <= QF_MAXE) {
                    const u32 mb = OF_RM + 2u * (c * QF_ROW + (1u << e) - 2u);
                    for (u32 node = 1, bit = e; bit > 0; --bit) { const u32 b = (rank >> (bit - 1u)) & 1u; qf_enc<13, 7, 7999, 235>(sm, rc, mb + 2u * node, b); node = 2u * node + b; }
                } else {
                    for (u32 node = 1, bit = e; bit > 0; --bit) {
                        const u32 b = (rank >> (bit - 1u)) & 1u;
                        const u32 off = qf_cold(sm, cold, (c * 2u + (e - 6u)) * 256u + node, st_miss); ++st_cached;
                        qf_enc<13, 7, 7999, 235>(sm, rc, off, b); node = 2u * node + b;
                    }
                }
            }
            // ---- run length (qlfc.cpp:1277-1331) ----
            const u32 ueb = OF_UE + 2u * (c * 32u);
            qf_enc<11, 5, 2025, 42>(sm, rc, ueb, run != 1u ? 1u : 0u);
            if (run != 1u) {
                const u32 e = (u32)qd3_ilog2(run);
                for (u32 b = 1; b < e; ++b) qf_enc<11, 4, 1962, 142>(sm, rc, ueb + 2u * b, 1u);
                qf_enc<11, 4, 1962, 142>(sm, rc, ueb + 2u * e, 0u);
                if (e <= QF_MAXE) {
                    const u32 mb = OF_UM + 2u * (c * QF_ROW + (1u << e) - 2u);
                    for (u32 node = 1, bit = e; bit > 0; --bit) { const u32 b = (run >> (bit - 1u)) & 1u; qf_enc<11, 6, 1951, 147>(sm, rc, mb + 2u * node, b); node = 2u * node + b; }
                } else {
                    for (u32 ctx = 1, bit = e; bit > 0; --bit, ++ctx) {
                        const u32 b = (run >> (bit - 1u)) & 1u;
                        const u32 off = qf_cold(sm, cold, QF_COLD_RANK + (c * 32u + e) * 32u + ctx, st_miss); ++st_cached;
                        qf_enc<11, 5, 1987, 46>(sm, rc, off, b);
                    }
                }
            }
        }
    }
    if (rc.range < 0x10000u) qf_shift(rc);
    qf_shift(rc); qf_shift(rc); qf_shift(rc);
    return (int)rc.pos;
}

#ifndef QD3_HOST
// start values: rank counters 4096, run counters 1024 (qlfc_model.cpp:73-74)
__device__ __forceinline__ void qf_smem_init(FastSmem &F)
{
    const u32 lane = threadIdx.x & 31u;
    u32 *w = (u32 *)F.re;
    for (u32 i = lane; i < (256 * 8 + 256 * QF_ROW) / 2; i += 32) w[i] = 0x10001000u;     // re and rm are contiguous
    w = (u32 *)F.ue;
    for (u32 i = lane; i < (256 * 32 + 256 * QF_ROW) / 2; i += 32) w[i] = 0x04000400u;    // ue and um are contiguous
    w = (u32 *)F.cval;
    for (u32 i = lane; i < (sizeof(FastSmem) - offsetof(FastSmem, cval)) / 4; i += 32) w[i] = 0;
    __syncwarp();
}

__global__ void __launch_bounds__(256) q_fast_model_init(short *__restrict__ cold, u32 streams)
{
    const size_t total = (size_t)streams * QF_COLD;
    for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (size_t)gridDim.x * 256)
        cold[i] = (i % QF_COLD) < QF_COLD_RANK ? (short)4096 : (short)1024;
}

__global__ void __launch_bounds__(32, 1) q_fast_decode(const u8 *__restrict__ in_all, SubBlock *__restrict__ sbs, short *__restrict__ cold_all,
                                                       u8 *__restrict__ out_all, const u32 *__restrict__ sb_list, DoneSignal done)
{
    extern __shared__ __align__(16) u8 q_smem_raw[];
    qf_smem_init(*reinterpret_cast<FastSmem *>(q_smem_raw));
    SM3 sm; sm.b = (u32)__cvta_generic_to_shared(q_smem_raw);
    asm volatile("" : "+r"(sm.b) :: "memory");
    const u32 sid = sb_list[blockIdx.x];
    SubBlock &sb = sbs[sid];
    u32 st_cached = 0, st_miss = 0;
    const int r = qf_decode_stream(sm, in_all + sb.out_off, sb.out_cap, out_all + sb.in_start, sb.in_size, cold_all + (size_t)blockIdx.x * QF_COLD, st_cached, st_miss);
    __syncwarp();                                        // every lane's output stores precede lane 0's report
    if (threadIdx.x == 0) { sb.result = r; sb.stat_cached = st_cached; sb.stat_miss = st_miss; signal_done(done); }
}

__global__ void __launch_bounds__(32, 1) q_fast_encode(const u32 *__restrict__ run_pos, const u8 *__restrict__ run_sym, const u8 *__restrict__ run_rank,
                                                       SubBlock *__restrict__ sbs, const u8 *__restrict__ mtf_all, short *__restrict__ cold_all,
                                                       u8 *__restrict__ out_all, const u32 *__restrict__ sb_list, DoneSignal done)
{
    extern __shared__ __align__(16) u8 q_smem_raw[];
    qf_smem_init(*reinterpret_cast<FastSmem *>(q_smem_raw));
    SM3 sm; sm.b = (u32)__cvta_generic_to_shared(q_smem_raw);
    asm volatile("" : "+r"(sm.b) :: "memory");
    const u32 sid = sb_list ? sb_list[blockIdx.x] : blockIdx.x;
    SubBlock &sb = sbs[sid];
    u32 st_cached = 0, st_miss = 0;
    const int r = qf_encode_stream(sm, run_pos, run_sym, run_rank, sb.run_begin, sb.run_end, sb.in_size, mtf_all + sid * 256, out_all + sb.out_off, sb.out_cap,
                                   cold_all + (size_t)sid * QF_COLD, st_cached, st_miss);
    __syncwarp();                                        // every lane's output stores precede lane 0's report
    if (threadIdx.x == 0) { sb.result = r; sb.stat_cached = st_cached; sb.stat_miss = st_miss; signal_done(done); }
}
#endif
