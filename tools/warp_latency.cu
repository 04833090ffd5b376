// tools/warp_latency.cu -- dependent-chain latency (cycles) of the warp primitives the QLFC coder leans on,
// measured with ONE resident warp (the situation of a coder warp: nothing else hides latency).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o warp_latency tools/warp_latency.cu && ./warp_latency
#include <cstdio>
#include <cuda_runtime.h>

#define REPS 256

template <int WHAT> __global__ void k(unsigned *out, long long *cyc, unsigned seed, int distinct)
{
    __shared__ unsigned sm[1024];
    const unsigned lane = threadIdx.x;
    for (int i = lane; i < 1024; i += 32) sm[i] = (i * 7 + 1) & 1023;
    __syncwarp();
    unsigned v = seed + lane, acc = 0;
    unsigned key = distinct >= 32 ? lane : lane % distinct;
    long long t0 = clock64();
#pragma unroll 1
    for (int r = 0; r < REPS; ++r) {
        if (WHAT == 0) { v = __shfl_sync(0xffffffffu, v, (lane + 1) & 31) + 1; }
        if (WHAT == 1) { v = __match_any_sync(0xffffffffu, key + (v & 0x40000000u)) ; acc += v; v = acc & 0x40000000u; }
        if (WHAT == 2) { v = __reduce_max_sync(0xffffffffu, v) + lane; }
        if (WHAT == 3) { v = sm[v & 1023]; }
        if (WHAT == 4) { v = __ballot_sync(0xffffffffu, v & 1) + lane; }
        if (WHAT == 5) { v = (v * 4093u + 77u) >> 12; }
        if (WHAT == 6) { sm[lane] = v; __syncwarp(); v = sm[(lane + 1) & 31] + 1; __syncwarp(); }
        if (WHAT == 7) { if ((v & 31) == (unsigned)(r & 31)) v = v * 3 + 1; __syncwarp(); }
        if (WHAT == 8) { v = __reduce_add_sync(0xffffffffu, v) + lane; }
    }
    // ---- issue rate of a LONE warp (round 2: does "one instruction per 4-5 cycles whatever the dependency structure" hold?) ----
    // N independent multiply-add chains in one instruction stream: cycles per INSTRUCTION = t / (REPS * N)
    if (WHAT >= 100 && WHAT < 110) {
        unsigned a0 = v, a1 = v + 1, a2 = v + 2, a3 = v + 3, a4 = v + 4, a5 = v + 5, a6 = v + 6, a7 = v + 7;
        t0 = clock64();
#pragma unroll 1
        for (int r = 0; r < REPS; ++r) {
            a0 = a0 * 4093u + 77u;
            if (WHAT >= 102) { a1 = a1 * 4091u + 79u; }
            if (WHAT >= 104) { a2 = a2 * 4089u + 81u; a3 = a3 * 4087u + 83u; }
            if (WHAT >= 108) { a4 = a4 * 4085u + 85u; a5 = a5 * 4083u + 87u; a6 = a6 * 4081u + 89u; a7 = a7 * 4079u + 91u; }
        }
        acc = a0 + a1 + a2 + a3 + a4 + a5 + a6 + a7;
    }
    // ---- straight-line issue: 64 independent operations per iteration (branch amortised) ----
    //   110: 64 IMAD (one pipe)   111: 32 IMAD + 32 LOP3 alternating (two pipes)
    if (WHAT == 110 || WHAT == 111 || WHAT == 112) {     // 112: as 110 but 2048 instructions (32 KB) of straight-line code per iteration
        unsigned a[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) a[j] = v + j;
        t0 = clock64();
#pragma unroll 1
        for (int r = 0; r < REPS; ++r) {
#pragma unroll
            for (int u = 0; u < (WHAT == 112 ? 256 : 8); ++u)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (WHAT == 110 || WHAT == 112 || (j & 1) == 0) asm volatile("mad.lo.u32 %0, %0, %1, 77;" : "+r"(a[j]) : "r"(seed));
                    else asm volatile("lop3.b32 %0, %0, %1, %2, 0x96;" : "+r"(a[j]) : "r"(seed), "r"(lane));
                }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) acc += a[j];
    }
    // ---- control flow of a lone warp ----
    //   120: 8 forward branches per iteration, ALWAYS taken (uniform, condition known long before): cost of a taken branch
    //   121: the same branches, NEVER taken
    //   122: one forward branch per iteration whose condition is computed right before it (multiply -> compare -> branch), taken
    //   123: as 122 but the compare feeds a predicated instruction instead of a branch
    if (WHAT == 120 || WHAT == 121) {
        const unsigned flag = (WHAT == 120) ? (v | 1u) : (v & (unsigned)(distinct >> 20));   // per-lane runtime values (vector predicate, like the coder's): 120 -> non-zero, 121 -> 0
        t0 = clock64();
#pragma unroll 1
        for (int r = 0; r < REPS; ++r) {
#pragma unroll
            for (int j = 0; j < 8; ++j)
                asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\t@p bra.uni SKIP;\n\t"
                             "mad.lo.u32 %0, %0, 4093, 77;\n\tmad.lo.u32 %0, %0, 4091, 79;\n\tmad.lo.u32 %0, %0, 4089, 81;\n\tmad.lo.u32 %0, %0, 4087, 83;\n\t"
                             "mad.lo.u32 %0, %0, 4093, 77;\n\tmad.lo.u32 %0, %0, 4091, 79;\n\tmad.lo.u32 %0, %0, 4089, 81;\n\tmad.lo.u32 %0, %0, 4087, 83;\n\t"
                             "SKIP:\n\tadd.u32 %0, %0, 1;\n\t}" : "+r"(v) : "r"(flag));
        }
    }
    //   124 / 125 / 126: the instruction-fetch question.  NB branches per iteration, all taken, each jumping over SKIP dead multiply-adds, so
    //   that the loop's code footprint is NB x (SKIP + 3) x 16 bytes: 124 = 32 x 16 (9.5 KB), 125 = 32 x 64 (34 KB), 126 = 64 x 64 (68 KB),
    //   against 120 (8 x 8, 1.5 KB).  If a taken branch costs the same in all four, instruction fetch is not what limits a lone warp whose
    //   hot path does not fit the L0 instruction cache; if it grows with the footprint, it is (DESIGN.md 4.5, round 2).
    if (WHAT >= 124 && WHAT <= 126) {
        constexpr int NB = WHAT == 126 ? 64 : 32, SK = WHAT == 124 ? 16 : 64;
        const unsigned flag = v | 1u;
        t0 = clock64();
#pragma unroll 1
        for (int r = 0; r < REPS; ++r) {
#pragma unroll
            for (int j = 0; j < NB; ++j) {
                if (SK == 16)
                    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\t@p bra.uni SKIP;\n\t"
                                 "mad.lo.u32 %0, %0, 4093, 77;\n\tmad.lo.u32 %0, %0, 4091, 79;\n\tmad.lo.u32 %0, %0, 4089, 81;\n\tmad.lo.u32 %0, %0, 4087, 83;\n\t"
                                 "mad.lo.u32 %0, %0, 4093, 77;\n\tmad.lo.u32 %0, %0, 4091, 79;\n\tmad.lo.u32 %0, %0, 4089, 81;\n\tmad.lo.u32 %0, %0, 4087, 83;\n\t"
                                 "mad.lo.u32 %0, %0, 4093, 77;\n\tmad.lo.u32 %0, %0, 4091, 79;\n\tmad.lo.u32 %0, %0, 4089, 81;\n\tmad.lo.u32 %0, %0, 4087, 83;\n\t"
                                 "mad.lo.u32 %0, %0, 4093, 77;\n\tmad.lo.u32 %0, %0, 4091, 79;\n\tmad.lo.u32 %0, %0, 4089, 81;\n\tmad.lo.u32 %0, %0, 4087, 83;\n\t"
                                 "SKIP:\n\tadd.u32 %0, %0, 1;\n\t}" : "+r"(v) : "r"(flag));
                else
                    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0;\n\t@p bra.uni SKIP;\n\t"
#define M4 "mad.lo.u32 %0, %0, 4093, 77;\n\tmad.lo.u32 %0, %0, 4091, 79;\n\tmad.lo.u32 %0, %0, 4089, 81;\n\tmad.lo.u32 %0, %0, 4087, 83;\n\t"
#define M16 M4 M4 M4 M4
                                 M16 M16 M16 M16
                                 "SKIP:\n\tadd.u32 %0, %0, 1;\n\t}" : "+r"(v) : "r"(flag));
            }
        }
    }
    if (WHAT == 122 || WHAT == 123) {
        unsigned w = seed | 0x80000000u;                                     // stays >= 2^31 >= thr: the compare below is always true, but ptxas cannot know
        const unsigned thr = (unsigned)distinct;
        t0 = clock64();
#pragma unroll 1
        for (int r = 0; r < REPS; ++r) {
            if (WHAT == 122)
                asm volatile("{\n\t.reg .pred p;\n\t.reg .u32 t;\n\tmad.lo.u32 %0, %0, 1, %1;\n\tshr.u32 t, %0, 12;\n\tsetp.ge.u32 p, t, %2;\n\t@p bra.uni SKIP;\n\t"
                             "mad.lo.u32 %0, %0, 4093, 77;\n\tmad.lo.u32 %0, %0, 4091, 79;\n\tmad.lo.u32 %0, %0, 4089, 81;\n\tmad.lo.u32 %0, %0, 4087, 83;\n\t"
                             "mad.lo.u32 %0, %0, 4093, 77;\n\tmad.lo.u32 %0, %0, 4091, 79;\n\tmad.lo.u32 %0, %0, 4089, 81;\n\tmad.lo.u32 %0, %0, 4087, 83;\n\t"
                             "SKIP:\n\t}" : "+r"(w) : "r"(lane), "r"(thr));
            else
                asm volatile("{\n\t.reg .pred p;\n\t.reg .u32 t;\n\tmad.lo.u32 %0, %0, 1, %1;\n\tshr.u32 t, %0, 12;\n\tsetp.ge.u32 p, t, %2;\n\t@p add.u32 %0, %0, 2;\n\t}"
                             : "+r"(w) : "r"(lane), "r"(thr));
        }
        acc += w;
    }
    // ---- 130: LDS.U16 pointer chase (the counter loads of the coder are 16-bit) ----
    if (WHAT == 130) {
        unsigned short *s16 = (unsigned short *)sm;
        unsigned x = v & 1023u;
        t0 = clock64();
#pragma unroll 1
        for (int r = 0; r < REPS; ++r) x = s16[x] & 1023u;
        acc += x;
    }
    long long t1 = clock64();
    out[lane] = v + acc;
    if (lane == 0) *cyc = t1 - t0;
}

template <int WHAT> static void run(const char *name, int distinct = 32)
{
    unsigned *out; long long *cyc, h;
    cudaMalloc(&out, 128); cudaMalloc(&cyc, 8);
    k<WHAT><<<1, 32>>>(out, cyc, 12345u, distinct);
    k<WHAT><<<1, 32>>>(out, cyc, 12345u, distinct);
    cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
    printf("%-44s %7.1f cycles per dependent op\n", name, (double)h / REPS);
    cudaFree(out); cudaFree(cyc);
}

int main()
{
    run<5>("IMAD + SHF (counter move)");
    run<0>("__shfl_sync");
    run<4>("__ballot_sync");
    run<2>("__reduce_max_sync");
    run<8>("__reduce_add_sync");
    run<3>("LDS (pointer chase)");
    run<6>("STS + syncwarp + LDS + syncwarp");
    run<7>("divergent if + syncwarp");
    run<1>("__match_any_sync, 32 distinct values", 32);
    run<1>("__match_any_sync, 16 distinct values", 16);
    run<1>("__match_any_sync, 8 distinct values", 8);
    run<1>("__match_any_sync, 4 distinct values", 4);
    run<1>("__match_any_sync, 1 distinct value", 1);
    // cycles per LOOP ITERATION below; divide by the number of chains for cycles per instruction
    run<100>("lone warp, 1 IMAD chain  (per iteration)");
    run<102>("lone warp, 2 independent IMAD chains");
    run<104>("lone warp, 4 independent IMAD chains");
    run<108>("lone warp, 8 independent IMAD chains");
    run<110>("lone warp, 64 independent IMAD, straight line (per iteration of 64)");
    run<111>("lone warp, 32 IMAD + 32 LOP3 alternating   (per iteration of 64)");
    run<112>("lone warp, 2048 independent IMAD, 32 KB of straight-line code (per iteration of 2048)");
    run<120>("8 uniform forward branches, all TAKEN      (per iteration of 8)");
    run<121>("8 uniform forward branches, none taken     (per iteration of 8 x 9 instr)");
    run<124>("32 taken forward branches, footprint 9.5 KB (per iteration of 32)");
    run<125>("32 taken forward branches, footprint 34 KB  (per iteration of 32)");
    run<126>("64 taken forward branches, footprint 68 KB  (per iteration of 64)");
    run<122>("IMAD -> SHF -> ISETP -> taken BRA chain     (per iteration)");
    run<123>("IMAD -> SHF -> ISETP -> predicated IADD     (per iteration)");
    run<130>("LDS.U16 pointer chase (+ LOP3)");
    return 0;
}
