/* oracle/ref_driver.c -- TEST/BENCH INFRASTRUCTURE ONLY.
 *
 * A block loop around the UNMODIFIED reference's public API (bsc_compress / bsc_decompress from
 * oracle/_ref/libbsc_ref.so), mirroring what the reference CLI does (bsc.cpp:184-199, 354, 594):
 *   T = omp_get_max_threads(); if (T <= nBlocks) intra-block multithreading is switched off;
 *   T = min(T, nBlocks); one block per OpenMP thread.
 * When the host has more threads than there are blocks, the CLI leaves FEATURE_MULTITHREADING on, but
 * its intra-block OpenMP regions only get threads if nested parallelism is enabled, which the CLI does
 * not do.  refdrv_set_nested(1) enables two active levels with inner teams of max_threads / nBlocks
 * threads.  Nesting was measured not to help the reference, so the default is the stock CLI behaviour.
 * Used by bench.py for the `cpu_baseline` object and for `--impl reference`.
 * Links against libbsc_ref.so only (no product code, no oracle port).
 */
#include <omp.h>
#include <stddef.h>

int bsc_init(int features);
int bsc_compress(const unsigned char *input, unsigned char *output, int n, int lzpHashSize, int lzpMinLen, int blockSorter, int coder, int features);
int bsc_decompress(const unsigned char *input, int inputSize, unsigned char *output, int outputSize, int features);

#define FEATURE_FASTMODE 1
#define FEATURE_MULTITHREADING 2

static int g_nested = 0;
void refdrv_set_nested(int on) { g_nested = on; }
static int inner_threads(int nBlocks)
{
    int T = omp_get_max_threads();
    return (g_nested && T > nBlocks && nBlocks > 0) ? T / nBlocks : 1;
}

static int cli_features(int nBlocks, int *threads_out)
{
    int features = FEATURE_FASTMODE | FEATURE_MULTITHREADING;
    int T = omp_get_max_threads();
    if (T <= nBlocks) features &= ~FEATURE_MULTITHREADING;    /* bsc.cpp:188 */
    if (T >= nBlocks) T = nBlocks;                             /* bsc.cpp:189 */
    *threads_out = T > 0 ? T : 1;
    return features;
}

int refdrv_init(void) { return bsc_init(FEATURE_FASTMODE | FEATURE_MULTITHREADING); }
int refdrv_max_threads(void) { return omp_get_max_threads(); }
/* The launcher's environment must not decide the baseline: torchrun exports OMP_NUM_THREADS=1 to its ranks, which made
 * rank 0 run 18 x 64 MiB blocks on one thread (round 1, SCALE N = 2/4/8: rc 124).  bench.py passes the host's thread count. */
void refdrv_set_threads(int n) { if (n > 0) omp_set_num_threads(n); }

/* compress nBlocks independent blocks; out[b] must hold size[b] + 28 bytes; outSize[b] = result */
int refdrv_compress(const unsigned char *const *in, const int *size, int nBlocks, unsigned char *const *out, int *outSize, int sorter, int coder)
{
    int T, features = cli_features(nBlocks, &T), b, inner = inner_threads(nBlocks);
    omp_set_max_active_levels(inner > 1 ? 2 : 1);
#pragma omp parallel for schedule(dynamic, 1) num_threads(T)
    for (b = 0; b < nBlocks; ++b) { omp_set_num_threads(inner); outSize[b] = bsc_compress(in[b], out[b], size[b], 0, 0, sorter, coder, features); }
    return T * inner;
}

int refdrv_decompress(const unsigned char *const *in, const int *inSize, int nBlocks, unsigned char *const *out, const int *outSize, int *result)
{
    int T, features = cli_features(nBlocks, &T), b, inner = inner_threads(nBlocks);
    omp_set_max_active_levels(inner > 1 ? 2 : 1);
#pragma omp parallel for schedule(dynamic, 1) num_threads(T)
    for (b = 0; b < nBlocks; ++b) { omp_set_num_threads(inner); result[b] = bsc_decompress(in[b], inSize[b], out[b], outSize[b], features); }
    return T * inner;
}
