// libbsc_b200/cli/bsc_b200.cpp -- file-level front end: the `bsc1` container of the reference CLI (bsc.cpp:50-57, 163-178,
// 401-417, 470-600) around the block API of libbsc_b200, with a multi-GPU block scheduler.
//
//   bsc_b200 e <input> <archive> [-b<MiB>] [-m<0|3..8>] [-e<0|1|2>] [-l [-H<bits>] [-M<len>]] [-g<dev[,dev...]>] [-j<blocks in flight per GPU>]
//   bsc_b200 d <archive> <output>              [-g...] [-j...]
//
// Format (SURVEY.md Appendix A.4): 'b','s','c',0x31 | int32 nBlocks | per block { int64 blockOffset, int8 recordSize,
// int8 sortingContexts } + one libbsc block.  This front end always WRITES recordSize = 1 and sortingContexts =
// FOLLOWING (the reference's filters off), so the stock `bsc` reads everything it writes; LZP
// is off by default (= `bsc e ... -p`) and on with -l (= `bsc e ...` without -s / -r).  It READS every bsc archive whose blocks the
// library decodes: the inverses of the reference's filters (reversed contexts, record reordering) are applied after decoding;
// the detectors that choose them on the compression side stay in the reference (BASELINE.json north_star: filters on the host).
//
// Scheduling: blocks are independent (SURVEY.md 8e).  One worker thread per (GPU, slot): a worker binds to its GPU once, takes the
// next block index, reads it with pread, calls bsc_compress / bsc_decompress (the library stages the block through pinned memory on
// a private stream of the CURRENT device), and hands the result to an in-order writer (compression) or writes it at its offset
// (decompression).  No collective, no peer traffic; GPUs never share a block.
//
// The same source builds against the UNMODIFIED reference library (-DBSCB200_CLI_REF, CPU) -- that build exists only for
// tests/test_cli_container.py, which checks the container byte-for-byte against the reference's own CLI without a GPU.
#include <algorithm>
#include <condition_variable>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include <fcntl.h>
#include <sys/stat.h>
#include <sys/time.h>
#include <unistd.h>

#ifdef BSCB200_CLI_REF
extern "C" {
int bsc_init(int features);
int bsc_compress(const unsigned char *input, unsigned char *output, int n, int lzpHashSize, int lzpMinLen, int blockSorter, int coder, int features);
int bsc_store(const unsigned char *input, unsigned char *output, int n, int features);
int bsc_block_info(const unsigned char *blockHeader, int headerSize, int *pBlockSize, int *pDataSize, int features);
int bsc_decompress(const unsigned char *input, int inputSize, unsigned char *output, int outputSize, int features);
}
static int bscb200_device_count(void) { return 1; }
static long long bscb200_device_free_bytes(void) { return -1; }
static long long bscb200_workspace_bytes(int, int) { return 0; }
static long long bscb200_scratch_bytes(int, int) { return 0; }
static long long bscb200_inplace_bytes(int, int, int) { return 0; }
static long long bscb200_decompress_bytes(int, int) { return 0; }
static void bscb200_release_pools(void) {}
static int bscb200_set_device(int) { return 0; }
#define LIBBSC_HEADER_SIZE 28
#define LIBBSC_NO_ERROR 0
#define LIBBSC_NOT_COMPRESSIBLE -3
#define LIBBSC_NOT_SUPPORTED -4
#else
#include "../../include/libbsc_b200.h"
#endif

namespace {

const unsigned char kSign[4] = {'b', 's', 'c', 0x31};
enum { kFeatures = 1 | 2, kContextsFollowing = 1, kContextsPreceding = 2, kRecordBytes = 10 };
const int kMaxOutOfPlace = 1 << 30;                                       // larger blocks are compressed in place (libbsc.cpp:124-210)

struct Options {
    int block_bytes = 25 << 20, sorter = 1, coder = 1, slots = 96;
    int lzp_hash = 0, lzp_min = 0;                                       // -l: the reference's LZP stage (host side of the library), off by default
    std::vector<int> devices;
};

double now() { timeval tv; gettimeofday(&tv, nullptr); return tv.tv_sec + tv.tv_usec * 1e-6; }

[[noreturn]] void die(const char *fmt, const char *arg = "")
{
    fprintf(stderr, fmt, arg); fputc('\n', stderr);
    exit(2);
}
const char *error_text(int code)
{
    switch (code) {
    case -2: return "not enough memory";
    case -4: return "method not supported by this build (see DESIGN.md 1: -m3..8 above -b1024)";
    case -5: return "unexpected end of block";
    case -6: return "the compressed data is corrupted";
    case -7: return "general GPU failure";
    case -8: return "no usable GPU";
    case -9: return "not enough GPU memory";
    default: return "internal error";
    }
}

void pread_all(int fd, void *buf, size_t n, off_t off, const char *name)
{
    unsigned char *p = (unsigned char *)buf;
    while (n) { ssize_t r = pread(fd, p, n, off); if (r <= 0) die("IO error on file: %s", name); p += r; n -= (size_t)r; off += r; }
}
void pwrite_all(int fd, const void *buf, size_t n, off_t off, const char *name)
{
    const unsigned char *p = (const unsigned char *)buf;
    while (n) { ssize_t r = pwrite(fd, p, n, off); if (r <= 0) die("IO error on file: %s", name); p += r; n -= (size_t)r; off += r; }
}

void put_record(unsigned char *rec, long long offset, int recordSize, int contexts)
{
    for (int i = 0; i < 8; ++i) rec[i] = (unsigned char)((unsigned long long)offset >> (8 * i));
    rec[8] = (unsigned char)recordSize; rec[9] = (unsigned char)contexts;
}

// Blocks in flight per GPU, bounded by its free memory: a context holds the staged block + the coder stage (~15 n + 64 MB); the sort
// slabs (~58 n each for BWT; three are reserved here, the library makes up to six while memory lasts) are shared by all of them.  At -b1024 that is one or two blocks, at -b25 the full -j.
// A block above 1 GiB takes the library's bounded path on a context of its own, no slabs: bscb200_inplace_bytes to compress (18 n + 256 MiB,
// BWT only), bscb200_decompress_bytes of the block's sorter to decompress (the same for the BWT, 26.5 n + 256 MiB for ST3..ST8); at -b2047 an
// 80 GB card runs one at a time.
int fit_slots(const Options &opt, int want, bool decode = false)
{
    int slots = want;
    const bool big = opt.block_bytes > kMaxOutOfPlace;
    for (int dev : opt.devices) {
        if (bscb200_set_device(dev) != 0) die("cannot select GPU");
        const long long fr = bscb200_device_free_bytes();
        if (fr < 0) continue;
        const long long per = big ? (decode ? bscb200_decompress_bytes(opt.block_bytes, opt.sorter) : bscb200_inplace_bytes(opt.block_bytes, 1, 1))
                                  : 2LL * opt.block_bytes + bscb200_workspace_bytes(opt.block_bytes, opt.sorter) + (64LL << 20);
        const long long avail = fr - fr / 10 - (big ? 0 : 3 * bscb200_scratch_bytes(opt.block_bytes, opt.sorter));
        const int fit = per > 0 ? (int)std::max(1LL, avail / per) : want;
        slots = std::min(slots, fit);
    }
    return std::max(1, slots);
}

// worker w of W runs on devices[w % devices.size()]
template <class F> void run_workers(const Options &opt, F body)
{
    const int W = (int)opt.devices.size() * opt.slots;
    std::vector<std::thread> th;
    for (int w = 0; w < W; ++w)
        th.emplace_back([&, w] {
            if (bscb200_set_device(opt.devices[(size_t)w % opt.devices.size()]) != 0) die("cannot select GPU");
            body(w);
        });
    for (auto &t : th) t.join();
}

// ------------------------------------------------------------------------------------------------------------------
int compress_file(const char *in_name, const char *out_name, Options opt)
{
    const int fin = open(in_name, O_RDONLY);
    if (fin < 0) die("Can't open input file: %s!", in_name);
    struct stat st; if (fstat(fin, &st) != 0) die("IO error on file: %s!", in_name);
    const long long size = (long long)st.st_size;
    FILE *fout = fopen(out_name, "wb");
    if (!fout) die("Can't create output file: %s!", out_name);

    if (opt.block_bytes > size) opt.block_bytes = (int)size;                          // bsc.cpp:159-162
    const int nBlocks = opt.block_bytes > 0 ? (int)((size + opt.block_bytes - 1) / opt.block_bytes) : 0;
    unsigned char head[8]; memcpy(head, kSign, 4); memcpy(head + 4, &nBlocks, 4);
    if (fwrite(head, 8, 1, fout) != 1) die("IO error on file: %s!", out_name);
    long long out_size = 8;

    const double t0 = now();
    std::mutex mu; std::condition_variable cv;
    int next = 0, next_to_write = 0;
    std::map<int, std::vector<unsigned char>> done;                                   // finished blocks waiting for their turn
    opt.slots = fit_slots(opt, opt.slots);
    const int W = std::max(1, std::min((int)opt.devices.size() * opt.slots, nBlocks));
    opt.slots = (W + (int)opt.devices.size() - 1) / (int)opt.devices.size();

    run_workers(opt, [&](int) {
        std::vector<unsigned char> in, out;
        for (;;) {
            int b;
            {   // bounded look-ahead: a worker may run at most 2 W blocks ahead of the writer
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return next >= nBlocks || next < next_to_write + 2 * W; });
                if (next >= nBlocks) return;
                b = next++;
            }
            const long long off = (long long)b * opt.block_bytes;
            const int n = (int)std::min<long long>(opt.block_bytes, size - off);
            out.assign((size_t)n + LIBBSC_HEADER_SIZE + kRecordBytes, 0);
            put_record(out.data(), off, 1, kContextsFollowing);
            unsigned char *blk = out.data() + kRecordBytes;
            int r;
            if (n <= kMaxOutOfPlace) {
                if (in.size() < (size_t)n) in.resize((size_t)n);
                pread_all(fin, in.data(), (size_t)n, (off_t)off, in_name);
                r = bsc_compress(in.data(), blk, n, opt.lzp_hash, opt.lzp_min, opt.sorter, opt.coder, kFeatures);   // stores incompressible blocks itself
            } else {                                                              // in place, as bsc.cpp:354-376 compresses every block
                pread_all(fin, blk, (size_t)n, (off_t)off, in_name);
                r = bsc_compress(blk, blk, n, opt.lzp_hash, opt.lzp_min, opt.sorter, opt.coder, kFeatures);
                if (r == LIBBSC_NOT_COMPRESSIBLE) {                              // the reference's library destroys the buffer here (this one does not)
                    pread_all(fin, blk, (size_t)n, (off_t)off, in_name);
                    r = bsc_store(blk, blk, n, kFeatures);
                }
            }
            if (r < LIBBSC_NO_ERROR) die("\nCompression failed: %s", error_text(r));
            out.resize((size_t)r + kRecordBytes);
            std::unique_lock<std::mutex> lk(mu);
            done.emplace(b, std::move(out));
            while (!done.empty() && done.begin()->first == next_to_write) {           // in-order writer (whoever finishes the next block writes)
                auto &blk = done.begin()->second;
                if (fwrite(blk.data(), 1, blk.size(), fout) != blk.size()) die("IO error on file: %s!", out_name);
                out_size += (long long)blk.size();
                done.erase(done.begin()); ++next_to_write;
            }
            cv.notify_all();
        }
    });
    if (fclose(fout) != 0) die("IO error on file: %s!", out_name);
    close(fin);
    const double dt = now() - t0;
    fprintf(stdout, "%.55s encoded %lld => %lld in %.3fs (%.2f MB/s)\n", in_name, size, out_size, dt, size / 1e6 / (dt > 0 ? dt : 1e-9));
    return 0;
}

// ------------------------------------------------------------------------------------------------------------------
struct BlockRef { long long file_pos, out_offset; int block_size, data_size, record_size, contexts, sorter; };

// inverses of the reference's host-side filters, applied after the block is decoded (bsc.cpp:614-647):
// reversed contexts (preprocessing.cpp:41-66) and record reordering (preprocessing.cpp:123-178: column-major back to records)
void undo_filters(std::vector<unsigned char> &buf, int n, int record_size, int contexts, std::vector<unsigned char> &tmp)
{
    if (contexts == kContextsPreceding) std::reverse(buf.begin(), buf.begin() + n);
    if (record_size > 1) {
        tmp.assign(buf.begin(), buf.begin() + n);
        const int rows = n / record_size;
        for (int i = 0; i < rows; ++i) for (int j = 0; j < record_size; ++j) buf[(size_t)record_size * i + j] = tmp[(size_t)j * rows + i];
    }
}

int decompress_file(const char *in_name, const char *out_name, Options opt)
{
    const int fin = open(in_name, O_RDONLY);
    if (fin < 0) die("Can't open input file: %s!", in_name);
    struct stat st; if (fstat(fin, &st) != 0) die("IO error on file: %s!", in_name);
    const long long size = (long long)st.st_size;
    const int fout = open(out_name, O_WRONLY | O_CREAT | O_TRUNC, 0644);
    if (fout < 0) die("Can't create output file: %s!", out_name);

    unsigned char head[8];
    if (size < 8) die("This is not bsc archive!");
    pread_all(fin, head, 8, 0, in_name);
    if (memcmp(head, kSign, 4) != 0) die("This is not bsc archive or invalid compression method!");
    // The block count in the header is only what the writer expected (segmentation, `bsc -s`, cuts blocks differently):
    // like the reference (bsc.cpp:520-524) read records until the file ends.
    // pass 1 (sequential, headers only): where is every block and where does it go
    std::vector<BlockRef> blocks;
    long long pos = 8;
    while (pos < size) {
        unsigned char rec[kRecordBytes + LIBBSC_HEADER_SIZE];
        if (pos + (long long)sizeof rec > size) die("Unexpected end of file: %s!", in_name);
        pread_all(fin, rec, sizeof rec, (off_t)pos, in_name);
        long long off = 0; for (int i = 0; i < 8; ++i) off |= (long long)rec[i] << (8 * i);
        const int recordSize = (signed char)rec[8], contexts = (signed char)rec[9];
        if (recordSize < 1 || (contexts != kContextsFollowing && contexts != kContextsPreceding)) die("This is not bsc archive or invalid compression method!");
        BlockRef r; r.file_pos = pos + kRecordBytes; r.out_offset = off; r.record_size = recordSize; r.contexts = contexts;
        if (bsc_block_info(rec + kRecordBytes, LIBBSC_HEADER_SIZE, &r.block_size, &r.data_size, kFeatures) != LIBBSC_NO_ERROR) die("This is not bsc archive or invalid compression method!");
        if (r.file_pos + r.block_size > size) die("Unexpected end of file: %s!", in_name);
        r.sorter = rec[kRecordBytes + 8] & 0x1f;                         // header mode, bits 0..4 (0: a stored block)
        blocks.push_back(r);
        pos = r.file_pos + r.block_size;
    }

    const int nBlocks = (int)blocks.size();
    const double t0 = now();
    std::mutex mu; int next = 0; long long out_size = 0;
    {   // sized for the largest block, with its sorter above 1 GiB (an ST block of equal size needs more than a BWT one)
        Options o2 = opt; o2.block_bytes = 0; o2.sorter = 1;
        for (const BlockRef &r : blocks)
            if (r.data_size > o2.block_bytes || (r.data_size == o2.block_bytes && r.sorter >= 3)) { o2.block_bytes = r.data_size; o2.sorter = r.sorter >= 3 ? r.sorter : 1; }
        if (o2.block_bytes <= kMaxOutOfPlace) o2.sorter = 6;
        opt.slots = fit_slots(o2, opt.slots, true);
    }
    const int W = std::max(1, std::min((int)opt.devices.size() * opt.slots, nBlocks));
    opt.slots = (W + (int)opt.devices.size() - 1) / (int)opt.devices.size();
    run_workers(opt, [&](int) {
        std::vector<unsigned char> in, out, tmp;
        for (;;) {
            int b;
            { std::lock_guard<std::mutex> lk(mu); if (next >= nBlocks) return; b = next++; }
            const BlockRef &r = blocks[(size_t)b];
            in.resize((size_t)r.block_size); out.resize((size_t)r.data_size + 1);
            pread_all(fin, in.data(), in.size(), (off_t)r.file_pos, in_name);
            const int rc = bsc_decompress(in.data(), r.block_size, out.data(), r.data_size, kFeatures);
            if (rc < LIBBSC_NO_ERROR) die("\nDecompression failed: %s", error_text(rc));
            undo_filters(out, r.data_size, r.record_size, r.contexts, tmp);
            pwrite_all(fout, out.data(), (size_t)r.data_size, (off_t)r.out_offset, out_name);
            std::lock_guard<std::mutex> lk(mu); out_size += r.data_size;
        }
    });
    close(fin); if (close(fout) != 0) die("IO error on file: %s!", out_name);
    const double dt = now() - t0;
    fprintf(stdout, "%.55s decoded %lld => %lld in %.3fs (%.2f MB/s)\n", in_name, size, out_size, dt, out_size / 1e6 / (dt > 0 ? dt : 1e-9));
    return 0;
}

void usage()
{
    fprintf(stdout,
            "bsc_b200 -- libbsc-compatible block-sorting compressor on NVIDIA H100 GPUs (bsc1 container)\n\n"
            "Usage: bsc_b200 <e|d> inputfile outputfile <options>\n"
            "  -b<size>  block size in MiB, default -b25 (1..2047; blocks above 1024 are compressed in place in at most 18 n + 256 MiB of HBM\n"
            "            each, -m0 only: -m3..8 above 1024 decode, in at most 26.5 n + 256 MiB each, but do not encode)\n"
            "  -m<algo>  block sorter: -m0 Burrows-Wheeler transform (default), -m3..-m8 sort transform of order n\n"
            "  -e<algo>  entropy coder: -e1 static QLFC (default), -e0 fast, -e2 adaptive\n"
            "  -l        LZP preprocessing on (host stage; -H<10..28> hash bits, -M<4..255> minimum match; bsc's defaults 15 / 128)\n"
            "  -g<list>  GPUs to use, e.g. -g0,1,2,3 (default: all visible)\n"
            "  -j<n>     blocks in flight per GPU, default -j96, fewer when HBM is short (8 coder streams per block, up to five per SM)\n"
            "Writes what `bsc e in out -p` writes; reads `bsc` archives made without -r / -c (LZP is undone on the host).\n");
    exit(0);
}

}  // namespace

int main(int argc, char **argv)
{
    if (argc < 4 || (argv[1][0] != 'e' && argv[1][0] != 'd') || argv[1][1] != 0) usage();
    Options opt;
    for (int i = 4; i < argc; ++i) {
        const char *a = argv[i];
        if (a[0] != '-' || !a[1]) usage();
        const int v = atoi(a + 2);
        switch (a[1]) {
        case 'b': if (v < 1 || v > 2047) usage(); opt.block_bytes = v << 20; break;            // bsc.cpp:761: up to 2047 MiB
        case 'm': if (v != 0 && (v < 3 || v > 8)) usage(); opt.sorter = v == 0 ? 1 : v; break;
        case 'e': if (v < 0 || v > 2) usage(); opt.coder = v == 0 ? 3 : v; break;
        case 'j': if (v < 1 || v > 64) usage(); opt.slots = v; break;
        case 'g': { opt.devices.clear(); for (const char *p = a + 2; *p; ) { opt.devices.push_back(atoi(p)); while (*p && *p != ',') ++p; if (*p == ',') ++p; } break; }
        case 'l': if (!opt.lzp_hash) { opt.lzp_hash = 15; opt.lzp_min = 128; } break;   // bsc's defaults (libbsc.h:78-79)
        case 'H': if (v < 10 || v > 28) usage(); opt.lzp_hash = v; if (!opt.lzp_min) opt.lzp_min = 128; break;
        case 'M': if (v < 4 || v > 255) usage(); opt.lzp_min = v; if (!opt.lzp_hash) opt.lzp_hash = 15; break;
        case 'p': opt.lzp_hash = opt.lzp_min = 0; break;                             // bsc compatibility: all preprocessing off (the default here)
        default: usage();
        }
    }
    if (opt.devices.empty()) { const int n = bscb200_device_count(); for (int d = 0; d < n; ++d) opt.devices.push_back(d); }
    if (opt.devices.empty()) die("no usable GPU (libbsc_b200 has no CPU path)");
    const int rc = bsc_init(kFeatures);
    if (rc != LIBBSC_NO_ERROR) die("Initialisation failed: %s", error_text(rc));
    const int rc2 = argv[1][0] == 'e' ? compress_file(argv[2], argv[3], opt) : decompress_file(argv[2], argv[3], opt);
    bscb200_release_pools();
    return rc2;
}
