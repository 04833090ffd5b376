// libbsc_b200/csrc/lzp_host.h -- the INVERSE of libbsc's LZP preprocessing stage, on the host (lzp.cpp:564-674 decoder, 813-887
// chunk container) and two of the five forward variants (see below).  BASELINE.json's north star keeps libbsc/lzp on the host: this
// is host code by design, sequential byte work before / after the GPU stages -- not a fallback for them.  Unlike the reference the
// decoder never writes past the caller's capacity (corrupt streams return LIBBSC_DATA_CORRUPT).
#pragma once
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

namespace lzp_host {

enum { kMatchFlag = 0xf2 };

// one chunk: literals, escaped flags (flag, 255) and matches (flag, length bytes: 254 = "254 more and continue") against the
// position last seen under the hash of the previous four bytes
inline int decode_chunk(const unsigned char *in, const unsigned char *in_end, unsigned char *out, long cap, int hash_bits, int min_len)
{
    if (in_end - in < 4) return -5;                                         // LIBBSC_UNEXPECTED_EOB
    if (cap < 4) return -6;
    const uint32_t mask = (uint32_t(1) << hash_bits) - 1u;
    int *seen = (int *)calloc((size_t)mask + 1, sizeof(int));
    if (!seen) return -2;
    long o = 0;
    while (o < 4) out[o++] = *in++;
    auto last4 = [&]() { return uint32_t(out[o - 1]) | (uint32_t(out[o - 2]) << 8) | (uint32_t(out[o - 3]) << 16) | (uint32_t(out[o - 4]) << 24); };
    uint32_t ctx = last4();
    int rc = 0;
    while (in < in_end) {
        const uint32_t slot = ((ctx >> 15) ^ ctx ^ (ctx >> 3)) & mask;
        const int from = seen[slot]; seen[slot] = (int)o;
        const unsigned char b = *in++;
        if (b != kMatchFlag || from <= 0) {                                 // plain literal
            if (o >= cap) { rc = -6; break; }
            out[o++] = b; ctx = (ctx << 8) | b;
            continue;
        }
        if (in >= in_end) { rc = -6; break; }
        if (*in == 255) {                                                   // escaped flag byte
            ++in;
            if (o >= cap) { rc = -6; break; }
            out[o++] = kMatchFlag; ctx = (ctx << 8) | kMatchFlag;
            continue;
        }
        long len = min_len;
        for (;;) { if (in >= in_end) { rc = -6; break; } const unsigned char l = *in++; len += l; if (l != 254) break; }
        if (rc || o + len > cap) { rc = -6; break; }
        for (const unsigned char *src = out + from; len > 0; --len) out[o++] = *src++;   // forward byte copy: source and target may overlap
        ctx = last4();
    }
    free(seen);
    return rc ? rc : (int)o;
}

// bsc_lzp_decompress: byte 0 = number of chunks; if > 1: {int32 rawSize, int32 packedSize} per chunk, then the chunks (raw when equal)
inline int decompress(const unsigned char *in, int n, unsigned char *out, int cap, int hash_bits, int min_len)
{
    if (n < 1) return -5;
    const int chunks = in[0];
    if (chunks == 1) return decode_chunk(in + 1, in + n, out, cap, hash_bits, min_len);
    if (chunks == 0 || n < 1 + 8 * chunks) return -6;
    long ip = 1 + 8L * chunks, op = 0;
    for (int c = 0; c < chunks; ++c) {
        int32_t raw, packed; memcpy(&raw, in + 1 + 8 * c, 4); memcpy(&packed, in + 5 + 8 * c, 4);
        if (raw < 0 || packed < 0 || ip + packed > n || op + raw > cap) return -6;
        int r = packed;
        if (packed != raw) r = decode_chunk(in + ip, in + ip + packed, out + op, raw, hash_bits, min_len);
        else memcpy(out + op, in + ip, (size_t)packed);
        if (r < 0) return r;
        if (r != raw) return -6;
        ip += packed; op += raw;
    }
    return (int)op;
}

// ---- forward stage ------------------------------------------------------------------------------------------------------------
// The reference picks one of five encoder variants by (hashSize, minLen) and platform (lzp.cpp:533-562), and they do NOT produce the
// same bytes (different match verification and length counting), so "the reference's output" means the variant an x86-64 build
// takes: `generic` for hashSize > 17, else `small` (minLen 4, 8), `small2x` (16), `medium` (5-7, 9-15), `large` (> 16, which includes
// the default 15 / 128).  All of them are restated here.
inline bool supported(int hash_bits, int min_len) { (void)hash_bits; (void)min_len; return true; }

inline uint64_t load64(const unsigned char *p) { uint64_t v; memcpy(&v, p, 8); return v; }
inline uint32_t load32(const unsigned char *p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline uint32_t hash_of(const unsigned char *p) { const uint32_t c = uint32_t(p[-1]) | (uint32_t(p[-2]) << 8) | (uint32_t(p[-3]) << 16) | (uint32_t(p[-4]) << 24); return (c >> 15) ^ c ^ (c >> 3); }

// match length bytes after the flag (lzp.cpp:398): 254 = "254 more, continue"; the early exit at the end-of-buffer mark only happens
// when the chunk is about to be declared incompressible anyway
inline void put_length(unsigned char *&out, const unsigned char *eob, long len)
{
    *out++ = kMatchFlag;
    while (len >= 254) { len -= 254; *out++ = 254; if (out >= eob) break; }
    *out++ = (unsigned char)len;
}

// tail of every variant (lzp.cpp:421-433): literals only, flags escaped when the decoder would take them for a match
inline int finish_literals(const unsigned char *in, const unsigned char *in_start, const unsigned char *in_end, unsigned char *out, const unsigned char *out_start,
                           const unsigned char *eob, int *seen, uint32_t mask)
{
    while (in < in_end && out < eob) {
        const uint32_t slot = hash_of(in) & mask;
        const int from = seen[slot]; seen[slot] = (int)(in - in_start);
        const unsigned char b = *out++ = *in++;
        if (b == kMatchFlag && from > 0) *out++ = 255;
    }
    return out >= eob ? -3 : (int)(out - out_start);                        // LIBBSC_NOT_COMPRESSIBLE
}

// lzp.cpp:337-436 bsc_lzp_encode_large<unsigned long long>: positions are examined in groups of four that restart after every event
inline int encode_large(const unsigned char *in, const unsigned char *in_end, unsigned char *out, unsigned char *out_end, int *seen, uint32_t mask, int min_len)
{
    const unsigned char *in_start = in, *out_start = out, *eob = out_end - 8;
    const unsigned char *heuristic = in, *scan_end = in_end - min_len - 32;
    for (int i = 0; i < 4; ++i) *out++ = *in++;
    while (in < scan_end && out < eob) {
        int from = 0, good = -1, bad = -1;
        for (int k = 0; k < 4; ++k) {
            const uint32_t slot = hash_of(in + k) & mask;
            from = seen[slot]; seen[slot] = (int)(in + k - in_start);
            if (from > 0 && in > heuristic && load64(in + k + min_len - 8) == load64(in_start + from + min_len - 8) && load64(in + k) == load64(in_start + from)) { good = k; break; }
            if (from > 0 && in[k] == kMatchFlag) { bad = k; break; }
        }
        if (good < 0 && bad < 0) { memcpy(out, in, 4); in += 4; out += 4; continue; }
        if (bad >= 0) { memcpy(out, in, (size_t)bad + 1); in += bad + 1; out += bad + 1; *out++ = 255; continue; }
        memcpy(out, in, (size_t)good); in += good; out += good;
        const unsigned char *ref = in_start + from;
        long len = 8;
        for (; in + len < scan_end; len += 8) {
            const uint64_t x = load64(in + len) ^ load64(ref + len);
            if (x) { len += __builtin_ctzll(x) / 8; break; }
        }
        if (len < min_len) {                                                 // too short: remember how far it went, emit one literal
            heuristic = in + len;
            if ((*out++ = *in++) == kMatchFlag) *out++ = 255;
            continue;
        }
        in += len;
        put_length(out, eob, len - min_len);
    }
    return finish_literals(in, in_start, in_end, out, out_start, eob, seen, mask);
}

// lzp.cpp:55-147 small<T>, 149-241 small2x<T>, 243-335 medium<T>: one skeleton -- groups of four positions, a candidate is taken
// when one or two machine words agree (no "too short" path: the words cover min_len), the length is then counted in 8-byte steps.
//   word       4 or 8 bytes (T)
//   second_at  offset of the second word that must agree, or -1 (small)
//   guard      bytes kept clear at the end of the chunk: word (small) or 2 * word (small2x, medium)
// Always inlined, so that each of encode_chunk's five calls is its own copy with these as constants.  Left to the compiler, the choice
// follows how much else api.cu inlines, and an out-of-line copy becomes one more symbol the library exports.
inline __attribute__((always_inline)) int encode_short(const unsigned char *in, const unsigned char *in_end, unsigned char *out, unsigned char *out_end, int *seen, uint32_t mask,
                        int min_len, int word, int second_at, int guard)
{
    const unsigned char *in_start = in, *out_start = out, *eob = out_end - 8;
    const unsigned char *scan_end = in_end - guard - 32;
    auto same = [&](const unsigned char *a, const unsigned char *b) { return word == 8 ? load64(a) == load64(b) : load32(a) == load32(b); };
    for (int i = 0; i < 4; ++i) *out++ = *in++;
    while (in < scan_end && out < eob) {
        int from = 0, good = -1, bad = -1;
        for (int k = 0; k < 4; ++k) {
            const uint32_t slot = hash_of(in + k) & mask;
            from = seen[slot]; seen[slot] = (int)(in + k - in_start);
            if (from > 0 && (second_at < 0 || same(in + k + second_at, in_start + from + second_at)) && same(in + k, in_start + from)) { good = k; break; }
            if (from > 0 && in[k] == kMatchFlag) { bad = k; break; }
        }
        if (good < 0 && bad < 0) { memcpy(out, in, 4); in += 4; out += 4; continue; }
        if (bad >= 0) { memcpy(out, in, (size_t)bad + 1); in += bad + 1; out += bad + 1; *out++ = 255; continue; }
        memcpy(out, in, (size_t)good); in += good; out += good;
        const unsigned char *ref = in_start + from;
        long len = min_len;
        for (; in + len < scan_end; len += 8) {
            const uint64_t x = load64(in + len) ^ load64(ref + len);
            if (x) { len += __builtin_ctzll(x) / 8; break; }
        }
        in += len;
        put_length(out, eob, len - min_len);
    }
    return finish_literals(in, in_start, in_end, out, out_start, eob, seen, mask);
}

// lzp.cpp:441-531 bsc_lzp_encode_generic (the unaligned-access build)
inline int encode_generic(const unsigned char *in, const unsigned char *in_end, unsigned char *out, unsigned char *out_end, int *seen, uint32_t mask, int min_len)
{
    const unsigned char *in_start = in, *out_start = out, *eob = out_end - 8;
    const unsigned char *heuristic = in, *scan_end = in_end - min_len - 32;
    for (int i = 0; i < 4; ++i) *out++ = *in++;
    while (in < scan_end && out < eob) {
        const uint32_t slot = hash_of(in) & mask;
        const int from = seen[slot]; seen[slot] = (int)(in - in_start);
        if (from <= 0) { *out++ = *in++; continue; }
        const unsigned char *ref = in_start + from;
        bool take = load32(in + min_len - 4) == load32(ref + min_len - 4) && load32(in) == load32(ref);
        if (take && heuristic > in && load32(heuristic) != load32(ref + (heuristic - in))) take = false;
        long len = 0;
        if (take) {
            for (len = 4; in + len < scan_end; len += 4) if (load32(in + len) != load32(ref + len)) break;
            if (len < min_len) { if (heuristic < in + len) heuristic = in + len; take = false; }
        }
        if (!take) { const unsigned char b = *out++ = *in++; if (b == kMatchFlag) *out++ = 255; continue; }
        { uint16_t a, b; memcpy(&a, in + len, 2); memcpy(&b, ref + len, 2); if (a == b) len += 2; }
        if (in[len] == ref[len]) len += 1;
        in += len;
        put_length(out, eob, len - min_len);
    }
    return finish_literals(in, in_start, in_end, out, out_start, eob, seen, mask);
}

// lzp.cpp:533-562
inline int encode_chunk(const unsigned char *in, const unsigned char *in_end, unsigned char *out, unsigned char *out_end, int hash_bits, int min_len)
{
    if (in_end - in - min_len < 32) return -3;
    int *seen = (int *)calloc((size_t)1 << hash_bits, sizeof(int));
    if (!seen) return -2;
    const uint32_t mask = (uint32_t(1) << hash_bits) - 1u;
    int r;
    if (hash_bits > 17)      r = encode_generic(in, in_end, out, out_end, seen, mask, min_len);
    else if (min_len == 4)   r = encode_short(in, in_end, out, out_end, seen, mask, min_len, 4, -1, 4);            // small<unsigned int>
    else if (min_len == 8)   r = encode_short(in, in_end, out, out_end, seen, mask, min_len, 8, -1, 8);            // small<unsigned long long>
    else if (min_len == 16)  r = encode_short(in, in_end, out, out_end, seen, mask, min_len, 8, 8, 16);            // small2x<unsigned long long>
    else if (min_len < 8)    r = encode_short(in, in_end, out, out_end, seen, mask, min_len, 4, min_len - 4, 8);   // medium<unsigned int>
    else if (min_len < 16)   r = encode_short(in, in_end, out, out_end, seen, mask, min_len, 8, min_len - 8, 16);  // medium<unsigned long long>
    else                     r = encode_large(in, in_end, out, out_end, seen, mask, min_len);
    free(seen);
    return r;
}

inline int chunk_count(int n) { return n < 256 * 1024 ? 1 : n < 4 * 1024 * 1024 ? 2 : n < 16 * 1024 * 1024 ? 4 : 8; }     // lzp.cpp:44-51

// bsc_lzp_compress (lzp.cpp:676-717 serial rules, 719-796 parallel rules = LIBBSC_FEATURE_MULTITHREADING with more than one chunk)
inline int compress(const unsigned char *in, unsigned char *out, int n, int hash_bits, int min_len, bool parallel_rules)
{
    const int chunks = chunk_count(n);
    if (chunks == 1) {
        const int r = encode_chunk(in, in + n, out + 1, out + n - 1, hash_bits, min_len);
        if (r < 0) return r;
        out[0] = 1;
        return r + 1;
    }
    const int each = n / chunks;
    out[0] = (unsigned char)chunks;
    if (parallel_rules) {
        unsigned char *tmp = (unsigned char *)malloc((size_t)n);
        if (!tmp) return -2;
        int32_t packed[8]; long total = 1 + 8L * chunks;
        for (int c = 0; c < chunks; ++c) {
            const int start = c * each, size = c != chunks - 1 ? each : n - start;
            int r = encode_chunk(in + start, in + start + size, tmp + start, tmp + start + size, hash_bits, min_len);
            if (r < 0) r = size;
            packed[c] = r; total += r;
        }
        if (total >= n) { free(tmp); return -3; }
        long op = 1 + 8L * chunks;
        for (int c = 0; c < chunks; ++c) {
            const int start = c * each; const int32_t size = c != chunks - 1 ? each : n - start;
            memcpy(out + 1 + 8 * c, &size, 4); memcpy(out + 5 + 8 * c, &packed[c], 4);
            memcpy(out + op, (packed[c] != size ? tmp : in) + start, (size_t)packed[c]);
            op += packed[c];
        }
        free(tmp);
        return (int)op;
    }
    long op = 1 + 8L * chunks;
    for (int c = 0; c < chunks; ++c) {
        const int start = c * each; const int32_t size = c != chunks - 1 ? each : n - start;
        long room = size; if (room > n - op) room = n - op;
        int32_t r = encode_chunk(in + start, in + start + size, out + op, out + op + room, hash_bits, min_len);
        if (r < 0) {
            if (op + size >= n) return -3;
            r = size; memcpy(out + op, in + start, (size_t)size);
        }
        memcpy(out + 1 + 8 * c, &size, 4); memcpy(out + 5 + 8 * c, &r, 4);
        op += r;
    }
    return (int)op;
}

}  // namespace lzp_host
