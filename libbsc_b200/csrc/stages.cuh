// libbsc_b200/csrc/stages.cuh -- device-resident stage entry points (host functions that enqueue
// kernels on ctx->stream; all data pointers are DEVICE pointers unless noted).
#pragma once
#include "common.cuh"

// Forward BWT in place (bsc_bwt_encode, bwt.cpp:178).  num_indexes/indexes are HOST pointers (may be NULL).
int stage_bwt_encode(Ctx *ctx, u8 *d_T, int n, unsigned char *num_indexes, int *indexes);
// The same result with a bounded working set (bwt_encode_batched.cu): sorts in batches of at most B entries (raised to
// bwt_batch_floor(n) if smaller) and takes bwt_batched_bytes(n, B) from ctx->sort_arena(); d_T needs no padding or alignment.
int stage_bwt_encode_batched(Ctx *ctx, u8 *d_T, int n, unsigned char *num_indexes, int *indexes, u32 B);
size_t bwt_batched_bytes(u32 n, u32 B);
// smallest batch: max(65536, n / BWT_BATCH_FLOOR_DIV), which bounds the passes over the block
#define BWT_BATCH_FLOOR_DIV 64
u32 bwt_batch_floor(u32 n);
// batch entries that a working set of `budget` bytes allows at block length n (at least bwt_batch_floor(n), at most that or n)
u32 bwt_batch_entries(u32 n, long long budget);
// Inverse BWT in place (bsc_bwt_decode, bwt.cpp:283).  Takes bwt_decode_bytes(n) from ctx->arena.
int stage_bwt_decode(Ctx *ctx, u8 *d_T, int n, int index);
size_t bwt_decode_bytes(u32 n);
// Sort transform of order k in place (bsc_st_encode, st.cpp:990; k = 3..8).
int stage_st_encode(Ctx *ctx, u8 *d_T, int n, int k);
// The same result with a bounded working set (st_encode_batched.cu): sorts in batches of at most B entries (raised to bwt_batch_floor(n)
// if smaller) and takes st_batched_bytes(n, B) from ctx->sort_arena(); d_T needs no padding or alignment and is written only at the end.
int stage_st_encode_batched(Ctx *ctx, u8 *d_T, int n, int k, u32 B);
size_t st_batched_bytes(u32 n, u32 B);
// batch entries that a working set of `budget` bytes allows at block length n (at least bwt_batch_floor(n), at most that, n or
// ST_BATCH_MAX, which keeps every radix sort far below the 2^30 entries rs_onesweep assumes whatever the block length)
#define ST_BATCH_MAX (1 << 28)
u32 st_batch_entries(u32 n, long long budget);
// Inverse sort transform in place (bsc_st_decode, st.cpp:1491; k = 3..8, index = row of rotation 0).
int stage_st_decode(Ctx *ctx, u8 *d_T, int n, int k, int index);
// The same inverse in the lean layout of the blocks above 1 GiB (st_decode.cu): L is read at d_L, which needs n + 64 writable bytes, and
// the stage takes st_decode_lean_bytes(n) from ctx->arena and keeps it.  The result lands there, at *d_result (d_L itself for n <= 1).
// LIBBSC_DATA_CORRUPT when the lists do not tile the text; the stage never writes outside its region on any input.
int stage_st_decode_lean(Ctx *ctx, u8 *d_L, int n, int k, int index, u8 **d_result);
size_t st_decode_lean_bytes(size_t n);
// Coder container (bsc_coder_compress, coder.cpp:244).  d_out must hold n + 4096 bytes.
// bare_out_size >= 0: one QLFC stream without the container (bsc_qlfc_*_encode_block, qlfc.h:55-77), output capacity bare_out_size.
int stage_coder_compress(Ctx *ctx, const u8 *d_in, u8 *d_out, int n, int coder, int features, int bare_out_size = -1);
// bsc_coder_decompress (coder.cpp:273).  `in_size` bounds the readable input (device padded by >= 64 bytes);
// out_cap bounds the writable output.
int stage_coder_decompress(Ctx *ctx, const u8 *d_in, int in_size, u8 *d_out, int out_cap, int coder, int features, bool bare = false);   // bare: one stream, no container byte
// the most each coder stage takes from ctx->arena, over every input (qlfc.cu)
size_t coder_compress_bytes(u32 n);
size_t coder_decompress_bytes();
// Adler-32 of a device buffer (bsc_adler32, adler32.cpp:83).  Result lands in ctx->d_mail[slot]
// (asynchronously); adler32_fetch() waits and returns it.
void stage_adler32_async(Ctx *ctx, const u8 *d_p, int n, int slot);
u32  stage_adler32(Ctx *ctx, const u8 *d_p, int n);
