"""A deterministic battery of malformed blocks for bsc_decompress and the stages behind it.

Every base block is at most 1 MiB.  All but one are made by the C port (oracle/bsc_oracle.c, pinned byte for byte to the reference by
tests/test_golden.py); the block with an LZP stage is a reference fixture (tests/golden/rep700x900.block.lzp), since the port has no
forward LZP.  Each mutation is a pure function of the base block and a seed, and names itself: "<base>/<family>/<detail>".

The header mutations recompute the header Adler-32, so that they reach the checks behind it.  The payload mutations recompute the
payload Adler-32 as well, so that the corruption reaches the coder kernels and the inverse transforms.  A case also carries the sizes
bsc_decompress is called with (inputSize, outputSize), which the call-argument family changes.

tests/golden/make_reference_results_malformed.py records the reference's answer to every case, out of place and in place, in
tests/golden/reference_results_malformed.json; tests/test_gpu_malformed.py runs the product on the same cases."""
import os
import zlib

import numpy as np

HDR = 28
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
LZP_BLOCK = os.path.join(GOLD, "rep700x900.block.lzp")      # reference: bsc_compress(np.tile(text(3, 700), 900), lzp 15/128, BWT, coder 1)
SEED = 20261017


def adler32(a):
    return zlib.adler32(memoryview(np.ascontiguousarray(a, dtype=np.uint8)))


def get32(b, off):
    return int(np.asarray(b[off:off + 4], dtype=np.uint8).view("<i4")[0])


def put32(b, off, v):
    b[off:off + 4] = np.array([v & 0xffffffff], dtype="<u4").view(np.uint8)


def seal(b, payload=False):
    """recompute the payload Adler-32 (when asked) and the header Adler-32 of block b, in place; returns b"""
    if payload:
        put32(b, 20, adler32(b[HDR:]))
    put32(b, 24, adler32(b[:24]))
    return b


# ---- base blocks ------------------------------------------------------------------------------------------------------------------
def container8(port, data):
    """A BWT block of `data` whose coder stage is a container of eight sub-blocks, the sixth stored raw (packed size == raw size).
    bsc_compress writes eight sub-blocks only for blocks of 16 MiB and more; the format and the decoders take them at any size."""
    r, L, _ = port.bwt_encode(data, aux=False)
    assert r > 0
    cuts = np.linspace(0, L.size, 9).astype(int)
    table, streams = [], []
    for b in range(8):
        part = L[cuts[b]:cuts[b + 1]]
        z, s = port.encode_block(part) if b != 5 else (-1, None)
        s = s if z > 0 else part
        table += [part.size, s.size]
        streams.append(s)
    payload = np.concatenate([np.array([8], np.uint8), np.array(table, dtype="<i4").view(np.uint8)] + streams + [np.zeros(1, np.uint8)])
    blk = np.zeros(HDR + payload.size, np.uint8)
    blk[HDR:] = payload
    for off, v in ((0, blk.size), (4, data.size), (8, 1 | (1 << 5)), (12, r), (16, adler32(data))):
        put32(blk, off, v)
    return seal(blk, payload=True)


def base_blocks(gen, port):
    """{name: (block, data)}: the blocks every mutation starts from and the data each decodes to"""
    text3, skew, text5 = gen.text(7, 300000), gen.skew(3, 100000), gen.text(5, 200000)
    out = {}
    for name, a, sorter, coder in (("bwt_e1", text3, 1, 1), ("bwt_e2", skew, 1, 2), ("bwt_e3", text5, 1, 3),
                                   ("st3_e1", gen.skew(4, 150000), 3, 1), ("st6_e2", gen.text(6, 120000), 6, 2), ("st8_e3", text5, 8, 3)):
        z, blk = port.compress(a, sorter, coder, 3)
        assert z > 0 and get32(blk, 8) == sorter | (coder << 5), name
        out[name] = (blk, a)
    out["container8"] = (container8(port, gen.text(2, 1 << 20)), gen.text(2, 1 << 20))
    out["lzp"] = (np.fromfile(LZP_BLOCK, dtype=np.uint8), np.tile(gen.text(3, 700), 900))
    z, blk = port.store(gen.text(4, 5000))
    out["stored"] = (blk[:z].copy(), gen.text(4, 5000))
    return out


def sub_streams(blk):
    """(offset, size, raw size) in the block of every sub-stream of the coder container (a single stream: its size is unknown, -1)"""
    if get32(blk, 8) == 0:
        return []
    nb = int(blk[HDR])
    if nb == 1:
        return [(HDR + 1, get32(blk, 0) - HDR - 2, -1)]
    off, out = HDR + 1 + 8 * nb, []
    for b in range(nb):
        raw, packed = get32(blk, HDR + 1 + 8 * b), get32(blk, HDR + 5 + 8 * b)
        out.append((off, packed, raw))
        off += packed
    return out


# ---- mutations ----------------------------------------------------------------------------------------------------------------
def mutations(name, blk, seed=SEED):
    """[(case name, block, inputSize, outputSize)] of base block `blk`; a pure function of (blk, seed)"""
    rng = np.random.default_rng([seed, zlib.crc32(name.encode())])
    n, bs, mode, index = get32(blk, 4), get32(blk, 0), get32(blk, 8), get32(blk, 12)
    cases = []

    def add(detail, b, in_size=None, out_size=None):
        cases.append(("%s/%s" % (name, detail), b, b.size if in_size is None else in_size, n if out_size is None else out_size))

    def header(field_off, v):
        b = blk.copy()
        put32(b, field_off, v)
        return seal(b)

    add("valid", blk.copy())
    # header fields, header Adler-32 recomputed
    for s in (0, 2, 9, 31):
        add("sorter=%d" % s, header(8, (mode & ~0x1f) | s))
    for c in (0, 4, 7):
        add("coder=%d" % c, header(8, (mode & ~0xe0) | (c << 5)))
    for h, m in ((15, 128), (10, 4), (28, 255), (0, 0), (9, 128), (29, 128), (15, 3), (15, 0), (0, 128)):
        add("lzp=%d,%d" % (h, m), header(8, (mode & 0xff) | (m << 8) | (h << 16)))
    for v in sorted({27, 28, bs - 1, bs + 1, HDR + n + 1}):
        add("blockSize=%d" % v, header(0, v))
    for v in (n - 1, n + 1):
        add("dataSize=%d" % v, header(4, v))
    for v in sorted({0, 1, n, n + 1}):
        add("index=%d" % v, header(12, v))
    for off, what in ((16, "data"), (20, "payload")):
        add("adler_%s_forged" % what, header(off, get32(blk, off) ^ 0x00010001))
    # payload, payload Adler-32 recomputed
    for i, (off, size, raw) in enumerate(sub_streams(blk)):
        for where, lo, hi in (("head", 0, min(size, 14)), ("body", min(size, 14), size)):
            if hi > lo:
                b = blk.copy()
                p = off + int(rng.integers(lo, hi))
                b[p] ^= np.uint8(1 << int(rng.integers(0, 8)))
                add("flip/sub%d/%s@%d" % (i, where, p - HDR), seal(b, payload=True))
    if mode == 0:
        b = blk.copy()
        b[HDR + int(rng.integers(0, n))] ^= 0x10
        add("flip/stored", seal(b, payload=True))
    else:
        nb = int(blk[HDR])
        for v in (0, 2, 8, 9, 255):
            if v != nb:
                b = blk.copy()
                b[HDR] = v
                add("count=%d" % v, seal(b, payload=True))
        if nb > 1:
            last = HDR + 1 + 8 * (nb - 1)
            for detail, off, v in (("raw0=-1", HDR + 1, -1), ("packed0=-1", HDR + 5, -1),
                                   ("packed_last_overruns_input", last + 4, get32(blk, last + 4) + 64),
                                   ("raw0_overruns_dataSize", HDR + 1, get32(blk, HDR + 1) + n),
                                   ("packed0=raw0", HDR + 5, get32(blk, HDR + 1))):
                b = blk.copy()
                put32(b, off, v)
                add("table/%s" % detail, seal(b, payload=True))
        for v in sorted({0, 1, 255} - {int(blk[bs - 1])}):     # the count of secondary indexes
            b = blk.copy()
            b[bs - 1] = v
            add("num_indexes=%d" % v, seal(b, payload=True))
        count = int(blk[bs - 1])
        if get32(blk, 8) & 0x1f == 1 and 0 < count and 4 * count + 1 < bs - HDR:
            first = bs - 1 - 4 * count                          # the values of the secondary indexes, the count kept
            for detail, v in (("+1", get32(blk, first) + 1), ("=n", n), ("=-1", -1)):
                b = blk.copy()
                put32(b, first, v)
                add("index_value0%s" % detail, seal(b, payload=True))
    for cut in (bs // 2, bs - 2):
        b = blk[:cut].copy()
        put32(b, 0, cut)
        add("truncated@%d" % cut, seal(b, payload=True))
    # call arguments
    add("inputSize-1", blk.copy(), in_size=bs - 1)
    add("outputSize-1", blk.copy(), out_size=n - 1)
    return cases


def battery(gen, port):
    """(base blocks, [(case name, block, inputSize, outputSize)]) of every base"""
    bases = base_blocks(gen, port)
    return bases, [c for name, (blk, _) in bases.items() for c in mutations(name, blk)]


def corrupt_bwt_inputs():
    """(name, L, index) of random L with a random valid primary index: an LF map with many cycles for the inverse BWT"""
    rng = np.random.default_rng(SEED)
    for n in (1000, 70000, 1 << 20):
        yield "randL%d" % n, rng.integers(0, 256, n, dtype=np.uint8), int(rng.integers(1, n + 1))


def stage_calls():
    """(name, stage, args) of the stage-level calls with bad arguments; the data they run on is 1000 bytes of rng(SEED)"""
    return [("bwt_decode/index=0", "bwt_decode", dict(n=1000, index=0)),
            ("bwt_decode/index=n+1", "bwt_decode", dict(n=1000, index=1001)),
            ("bwt_decode/n=-1", "bwt_decode", dict(n=-1, index=1)),
            ("st_encode/k=2", "st_encode", dict(n=1000, k=2)),
            ("st_encode/k=9", "st_encode", dict(n=1000, k=9)),
            ("st_decode/k=2", "st_decode", dict(n=1000, k=2, index=5)),
            ("st_decode/k=9", "st_decode", dict(n=1000, k=9, index=5)),
            ("st_decode/index=n", "st_decode", dict(n=1000, k=4, index=1000)),
            ("coder_compress/coder=0", "coder_compress", dict(n=1000, coder=0)),
            ("coder_compress/coder=4", "coder_compress", dict(n=1000, coder=4)),
            ("coder_compress/n=0", "coder_compress", dict(n=0, coder=1)),
            ("coder_decompress/coder=0", "coder_decompress", dict(n=1000, coder=0)),
            ("coder_decompress/coder=4", "coder_decompress", dict(n=1000, coder=4)),
            ("block_info/headerSize=27", "block_info", dict(n=27))]


def stage_data():
    return np.random.default_rng(SEED).integers(0, 256, 1000, dtype=np.uint8)
