/* include/libbsc_b200.h -- C ABI of the GPU (H100, sm_90a) block-sorting hot path.
 *
 * Drop-in boundary: the first group of functions has EXACTLY the names, argument meaning, buffer
 * ownership and error behaviour of the libbsc 3.3.5 entry points it replaces (reference file:line
 * cited per function), so that libbsc/libbsc/libbsc.cpp -- or any program linking libbsc.a --
 * can bind to this library instead of bwt.o / st.o / coder.o / qlfc.o (see INTEGRATION.md).
 * All pointers in that group are HOST pointers; the library moves the block to the current CUDA
 * device, runs the stage there and moves the result back.  Plain pointers and ints only.
 *
 * There is no CPU implementation behind these symbols: without a usable CUDA device they return
 * LIBBSC_GPU_NOT_SUPPORTED.
 *
 * The second group (bscb200_*) are extensions for callers that keep blocks resident in HBM and
 * manage their own streams (bench.py, the multi-GPU block scheduler).
 */
#ifndef LIBBSC_B200_H
#define LIBBSC_B200_H

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

/* error codes, features, ids: libbsc/libbsc.h:41-76 */
#ifndef LIBBSC_NO_ERROR
#define LIBBSC_NO_ERROR                0
#define LIBBSC_BAD_PARAMETER          -1
#define LIBBSC_NOT_ENOUGH_MEMORY      -2
#define LIBBSC_NOT_COMPRESSIBLE       -3
#define LIBBSC_NOT_SUPPORTED          -4
#define LIBBSC_UNEXPECTED_EOB         -5
#define LIBBSC_DATA_CORRUPT           -6
#define LIBBSC_GPU_ERROR              -7
#define LIBBSC_GPU_NOT_SUPPORTED      -8
#define LIBBSC_GPU_NOT_ENOUGH_MEMORY  -9
#define LIBBSC_FEATURE_FASTMODE        1
#define LIBBSC_FEATURE_MULTITHREADING  2
#define LIBBSC_FEATURE_LARGEPAGES      4
#define LIBBSC_FEATURE_CUDA            8
#define LIBBSC_HEADER_SIZE             28
#endif
#define LIBBSC_BLOCKSORTER_BWT         1   /* 3..8 = ST3..ST8 */
#define LIBBSC_CODER_QLFC_STATIC       1
#define LIBBSC_CODER_QLFC_ADAPTIVE     2   /* csrc/qlfc_adaptive.cuh */
#define LIBBSC_CODER_QLFC_FAST         3   /* csrc/qlfc_fast.cuh */

/* ---- group 1: libbsc-compatible entry points -------------------------------------------- */

/* libbsc/libbsc.h:95,104 ; libbsc/libbsc/libbsc.cpp:46-66.  Call once before anything else. */
int bsc_init(int features);
int bsc_init_full(int features, void *(*malloc_fn)(size_t), void *(*zero_malloc_fn)(size_t), void (*free_fn)(void *));

/* libbsc/libbsc.h:118 ; libbsc.cpp:213-338.  output holds n + 28 bytes; input may equal output.
 * bsc_compress: LZP (lzpHashSize/lzpMinLen != 0) is outside the replaced path: LIBBSC_NOT_SUPPORTED.
 * bsc_decompress: blocks with an LZP stage are accepted (the inverse stage runs on the host after the GPU stages).
 * Block size: n <= 1 GiB (1073741824), and in place (input == output) up to 2146435072 bytes as in the reference; out of place,
 * n > 1 GiB is LIBBSC_BAD_PARAMETER as in the reference.  An in-place block above 1 GiB is sorted in place with the batched forward
 * BWT on a context of its own, in at most bscb200_inplace_bytes() = 18 n + 256 MiB of HBM, all of it freed when the call returns;
 * LIBBSC_GPU_NOT_ENOUGH_MEMORY (nothing written) when the device has less free.  The caller's buffer is written only on success.
 * Above 1 GiB bsc_compress with the sort transforms (blockSorter 3..8) returns LIBBSC_NOT_SUPPORTED; bsc_st_encode itself takes such
 * blocks (below), so libbsc's own bsc_compress linked against this library's stages writes them.  bsc_decompress reads every block the reference writes, up to 2146435072 bytes with every sorter: a block
 * above 1 GiB runs on a context of its own, in at most bscb200_decompress_bytes() of HBM (18 n + 256 MiB for the BWT, 26.5 n + 256 MiB
 * for ST3..ST8), all of it freed when the call returns; LIBBSC_GPU_NOT_ENOUGH_MEMORY when the device has less free. */
int bsc_compress(const unsigned char *input, unsigned char *output, int n, int lzpHashSize, int lzpMinLen, int blockSorter, int coder, int features);
/* libbsc/libbsc.h:128 ; libbsc.cpp:68-81 */
int bsc_store(const unsigned char *input, unsigned char *output, int n, int features);
/* libbsc/libbsc.h:139 ; libbsc.cpp:340-418 */
int bsc_block_info(const unsigned char *blockHeader, int headerSize, int *pBlockSize, int *pDataSize, int features);
/* libbsc/libbsc.h:150 ; libbsc.cpp:522-617 */
int bsc_decompress(const unsigned char *input, int inputSize, unsigned char *output, int outputSize, int features);

/* libbsc/bwt/bwt.h:45,56,68 ; libbsc/bwt/bwt.cpp:54-69, 178-231, 283-332.  In place on T. */
int bsc_bwt_init(int features);
int bsc_bwt_encode(unsigned char *T, int n, unsigned char *num_indexes, int *indexes, int features);
int bsc_bwt_decode(unsigned char *T, int n, int index, unsigned char num_indexes, int *indexes, int features);

/* libbsc/st/st.h:47,57,68 ; libbsc/st/st.cpp:990-1012 (k = 3..8; st.cu:334 for 7, 8).  In place on T. */
int bsc_st_init(int features);
/* bsc_st_encode above 1 GiB sorts in batches on a context of its own, in at most bscb200_st_encode_bytes(n) = 6 n + 256 MiB of HBM, all of
 * it freed when the call returns; LIBBSC_GPU_NOT_ENOUGH_MEMORY (T untouched) when the device has less free.  T is written only on success. */
int bsc_st_encode(unsigned char *T, int n, int k, int features);
int bsc_st_decode(unsigned char *T, int n, int k, int index, int features);   /* st.h:68 ; st.cpp:1491-1527 (csrc/st_decode.cu) */

/* libbsc/coder/coder.h:45,56,66 ; libbsc/coder/coder.cpp:244-347.  output of compress holds n + 4096 bytes. */
int bsc_coder_init(int features);
int bsc_coder_compress(const unsigned char *input, unsigned char *output, int n, int coder, int features);
int bsc_coder_decompress(const unsigned char *input, unsigned char *output, int coder, int features);
int bsc_qlfc_init(int features);                                              /* libbsc/coder/qlfc/qlfc.h:45 */
/* libbsc/coder/qlfc/qlfc.h:55-99 ; qlfc.cpp:2138-2226: ONE QLFC stream (what the container holds per sub-block).  encode: fails
 * with LIBBSC_NOT_COMPRESSIBLE when the stream would come within 16 bytes of outputSize (rangecoder.h:118-127).  decode: size-less
 * like the reference's; the stream is taken to end at most n + 16 bytes after `input` (n = the size coded in the stream). */
int bsc_qlfc_static_encode_block(const unsigned char *input, unsigned char *output, int inputSize, int outputSize);
int bsc_qlfc_adaptive_encode_block(const unsigned char *input, unsigned char *output, int inputSize, int outputSize);
int bsc_qlfc_fast_encode_block(const unsigned char *input, unsigned char *output, int inputSize, int outputSize);
int bsc_qlfc_static_decode_block(const unsigned char *input, unsigned char *output);
int bsc_qlfc_adaptive_decode_block(const unsigned char *input, unsigned char *output);
int bsc_qlfc_fast_decode_block(const unsigned char *input, unsigned char *output);

/* libbsc/adler32/adler32.h ; adler32.cpp:83 */
unsigned int bsc_adler32(const unsigned char *T, int n, int features);

/* libbsc/platform/platform.h:190-216 ; platform.cpp:192-260 (allocator hooks honoured for host temporaries) */
int   bsc_platform_init(int features, void *(*malloc_fn)(size_t), void *(*zero_malloc_fn)(size_t), void (*free_fn)(void *));
void *bsc_malloc(size_t size);
void *bsc_zero_malloc(size_t size);
void  bsc_free(void *address);

/* ---- group 2: extensions ---------------------------------------------------------------- */

/* bsc_coder_decompress with explicit bounds (what bsc_decompress uses internally) */
int bscb200_coder_decompress(const unsigned char *input, int inputSize, unsigned char *output, int outputCapacity, int coder, int features);

/* A context = one CUDA stream + one HBM workspace on `device`.  cuda_stream may be a
 * cudaStream_t owned by the caller (e.g. a torch stream) or NULL for a private stream.
 * One block at a time per context; use several contexts for concurrency. */
void              *bscb200_ctx_create(int device, void *cuda_stream);
void               bscb200_ctx_destroy(void *ctx);
int                bscb200_ctx_reserve(void *ctx, long long bytes);
/* Bounds the working set of the forward sorts on this context.  BWT: whenever the standard sorter would need more than `bytes` (about
 * 58 n + 64 MB for a block of n), the sort runs in batches of B = (bytes - 16 n) / 32 entries in about 16 n + 32 B bytes.  Sort
 * transforms (block sorters 3..8, bscb200_st_encode_device and bscb200_compress_device): whenever the standard sorter would need more
 * than `bytes` (30 n + 16 MB), in batches of B = (bytes - n) / 28 entries in about n + 28 B bytes.  Same results either way.
 * B is at least max(65536, n / 64): every key range rescans the text (or an oversized group of the BWT), so the work grows with n / B,
 * and the floor keeps it within about 64 passes over the block per such segment.  Smaller batches cost time: see DESIGN.md 4.2 and 4.3
 * for measured times.  0 (the default) = no bound; negative = LIBBSC_BAD_PARAMETER.
 * bscb200_compress_device keeps its 1 GiB limit; blocks above it go through the in-place bsc_compress. */
int                bscb200_ctx_set_sort_budget(void *ctx, long long bytes);
int                bscb200_lzp_decompress_host(const unsigned char *input, int n, unsigned char *output, int outputCapacity, int lzpHashSize, int lzpMinLen);   /* inverse of the reference LZP stage (libbsc/lzp/lzp.h), host only */
int                bscb200_lzp_compress_host(const unsigned char *input, unsigned char *output, int n, int lzpHashSize, int lzpMinLen, int features);   /* the reference LZP stage forward (libbsc/lzp/lzp.h), host only */
int                bscb200_device_count(void);                    /* CUDA devices visible to the process */
long long          bscb200_device_free_bytes(void);               /* free HBM on the current device, -1 on error */
void               bscb200_release_pools(void);                   /* free the pooled contexts and sort slabs of every device (no call in flight) */
int                bscb200_set_device(int device);                /* bind the calling thread: all entry points use the current device */
long long          bscb200_workspace_bytes(int n, int blockSorter);   /* per-context workspace (~9 n): working copy + coder stage, or the inverse BWT */
long long          bscb200_workspace_bytes_decode(int n);         /* the same (kept for callers of the round-1 ABI) */
long long          bscb200_scratch_bytes(int n, int blockSorter);  /* one device-wide sort slab (~58 n for BWT); BSCB200_SORT_SLABS of them per GPU (default 3) */
/* HBM that an in-place bsc_compress of a block of n > 1 GiB, or bsc_decompress of one, takes at most: 18 n + 256 MiB (about 39 GB at
 * n = 2146435072), none of it kept after the call.  Same for the three coders and with LZP.  Blocks of at most 1 GiB take the pooled path
 * instead (bscb200_workspace_bytes + bscb200_scratch_bytes).  blockSorter 3..8: LIBBSC_NOT_SUPPORTED; bad arguments: LIBBSC_BAD_PARAMETER. */
long long          bscb200_inplace_bytes(int n, int blockSorter, int coder);
/* HBM that bsc_decompress of a block with data size n and this blockSorter takes at most.  Above 1 GiB: 18 n + 256 MiB for the BWT
 * (= bscb200_inplace_bytes(n, 1, 1)) and 26.5 n + 256 MiB for ST3..ST8 (about 57.2 GB at n = 2146435072), none of it kept after the call.
 * Up to 1 GiB: the pooled cost, bscb200_workspace_bytes + bscb200_scratch_bytes.  Bad arguments: LIBBSC_BAD_PARAMETER. */
long long          bscb200_decompress_bytes(int n, int blockSorter);
/* HBM that bsc_st_encode of n bytes takes at most: above 1 GiB 6 n + 256 MiB (about 13.1 GB at n = 2146435072), none of it kept after
 * the call; up to 1 GiB the pooled cost, the staged block (n + 4096) and one sort slab (30 n + 16 MiB).  Bad arguments: LIBBSC_BAD_PARAMETER. */
long long          bscb200_st_encode_bytes(int n);
unsigned long long bscb200_ctx_kernel_launches(void *ctx);
unsigned long long bscb200_total_kernel_launches(void);
/* per-kernel CUDA-event timing of everything launched through ctx (bench.py's roofline leg) */
void               bscb200_ctx_set_profile(void *ctx, int on);
int                bscb200_ctx_profile_report(void *ctx, char *buf, int cap);
const char        *bscb200_version(void);

/* Device-resident variants: all d_* pointers are device pointers on the context's device.
 * Same return values as their host-pointer counterparts.  bscb200_compress_device takes n <= 1 GiB (LIBBSC_BAD_PARAMETER above);
 * bscb200_bwt_encode_device takes any n >= 0, but the standard sorter needs about 58 n bytes, so above a few hundred MiB on an
 * 80 GB card a context needs a sort budget (bscb200_ctx_set_sort_budget). */
int bscb200_compress_device(void *ctx, const unsigned char *d_input, unsigned char *d_output /* n+28 */, int n, int blockSorter, int coder, int features);
int bscb200_decompress_device(void *ctx, const unsigned char *d_input, int inputSize, unsigned char *d_output, int outputSize, int features);
int bscb200_bwt_encode_device(void *ctx, unsigned char *d_T, int n, unsigned char *num_indexes /* host */, int *indexes /* host */);
int bscb200_bwt_decode_device(void *ctx, unsigned char *d_T, int n, int index);
int bscb200_st_encode_device(void *ctx, unsigned char *d_T, int n, int k);
int bscb200_st_decode_device(void *ctx, unsigned char *d_T, int n, int k, int index);
int bscb200_coder_compress_device(void *ctx, const unsigned char *d_in, unsigned char *d_out /* n+4096 */, int n, int coder, int features);
int bscb200_coder_decompress_device(void *ctx, const unsigned char *d_in, int inputSize, unsigned char *d_out, int outputCapacity, int coder, int features);
unsigned int bscb200_adler32_device(void *ctx, const unsigned char *d_p, int n);

#ifdef __cplusplus
}
#endif
#endif
