"""GPU parity tests: every stage of the CUDA path, called through the C ABI (host-pointer bsc_* entry
points of include/libbsc_b200.h), must be bit-identical to the oracle -- the unmodified reference when
oracle/_ref was built, else our C port -- on the same seeded inputs, to the reference's outputs stored in
tests/golden/reference_results.json, to the known-answer values of SURVEY.md Appendix C at BASELINE.json's
full sizes, and must satisfy the size-independent round-trip properties."""
import hashlib
import json
import os
import zlib

import numpy as np
import pytest

import reference_inputs as ri

pytestmark = pytest.mark.gpu

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_results.json")))


def digest(b):
    b = np.ascontiguousarray(b, dtype=np.uint8)
    return {"size": int(b.size), "sha256": hashlib.sha256(b.tobytes()).hexdigest()}


def small_inputs(gen):
    rng = np.random.default_rng(11)
    yield "text300k", gen.text(7, 300000)
    yield "text1M", gen.text(2, 1 << 20)
    yield "skew300k", gen.skew(3, 300000)
    yield "rand70k", gen.rand(1, 70000)
    yield "alpha4", rng.integers(0, 4, 5000, dtype=np.uint8)
    yield "alpha2_64k", rng.integers(0, 2, 65536, dtype=np.uint8)
    yield "allsame3000", np.full(3000, 65, dtype=np.uint8)
    yield "zeros1000", np.zeros(1000, dtype=np.uint8)
    yield "period7", np.tile(np.frombuffer(b"abcabcd", dtype=np.uint8), 3000)
    yield "withzeros", np.concatenate([gen.text(3, 5000), np.zeros(40, np.uint8), gen.text(4, 3000), np.zeros(9, np.uint8)])
    yield "ragged4097", gen.text(8, 4097)
    yield "tiny29", gen.text(1, 29)
    yield "tiny100", gen.text(1, 100)


def test_adler32_device(bsc):
    rng = np.random.default_rng(3)
    for n in (1 << 16, (1 << 16) + 1, 100000, (1 << 20) + 37, 5 << 20):
        a = rng.integers(0, 256, n, dtype=np.uint8)
        assert bsc.adler32(a) == zlib.adler32(a.tobytes()), n
    assert bsc.adler32(np.full(3 << 20, 255, dtype=np.uint8)) == zlib.adler32(b"\xff" * (3 << 20))


def test_st_encode_matches_oracle(bsc, gen, port, checker):
    for name, a in small_inputs(gen):
        for k in (3, 4, 5, 6, 7, 8):
            ref_impl = checker if k <= 6 else port          # k = 7, 8 exist only in the reference's CUDA build
            i2, L2 = ref_impl.st_encode(a, k)
            i1, L1 = bsc.st_encode(a, k)
            assert i1 == i2, (name, k, i1, i2)
            assert np.array_equal(L1, L2), (name, k)


def test_st_tiny_sizes(bsc, port):
    for n in (2, 3, 4, 5, 7, 8, 9, 16, 17):
        a = ((np.arange(n) * 5 + 1) % 3).astype(np.uint8)
        for k in (3, 6, 8):
            i2, L2 = port.st_encode(a, k)
            i1, L1 = bsc.st_encode(a, k)
            assert i1 == i2 and np.array_equal(L1, L2), (n, k)


def test_st_decode_matches_oracle(bsc, gen, port, checker):
    """bsc_st_decode (st.cpp:1491): inverse of every order on every input class, against the input and against the oracle's inverse."""
    for name, a in small_inputs(gen):
        for k in (3, 4, 5, 6, 7, 8):
            i, L = port.st_encode(a, k) if k > 6 else checker.st_encode(a, k)
            r, T = bsc.st_decode(L, k, i)
            assert r == 0 and np.array_equal(T, a), (name, k)
            r2, T2 = checker.st_decode(L, k, i)
            assert r2 == 0 and np.array_equal(T, T2), (name, k)
    for n in (2, 3, 4, 5, 7, 8, 9, 16, 17):
        a = ((np.arange(n) * 5 + 1) % 3).astype(np.uint8)
        for k in (3, 6, 8):
            i, L = port.st_encode(a, k)
            r, T = bsc.st_decode(L, k, i)
            assert r == 0 and np.array_equal(T, a), (n, k)
    a = gen.text(1, 100)
    assert bsc.st_decode(a, 6, 100)[0] == -1 and bsc.st_decode(a, 6, -1)[0] == -1 and bsc.st_decode(a, 2, 0)[0] == -1 and bsc.st_decode(a, 9, 0)[0] == -1


def test_st_decode_corrupt_input_terminates(bsc, gen):
    """An L / index pair that no text produces must come back (garbage, like the reference) without hanging or faulting."""
    rng = np.random.default_rng(5)
    for n in (1000, 70000, 1 << 20):
        L = rng.integers(0, 7, n, dtype=np.uint8)
        for k in (3, 6):
            r, T = bsc.st_decode(L, k, int(rng.integers(0, n)))
            assert r == 0 and T.size == n


def test_st_blocks_round_trip_all_orders(bsc, gen, checker):
    """-m3..8 archives: our blocks through our decoder and the reference's, the reference's (k <= 6 on its CPU build) through ours."""
    for name, a in small_inputs(gen):
        for sorter in (3, 4, 5, 6, 7, 8):
            z, blk = bsc.compress(a, sorter, 1, 3)
            q, u = bsc.decompress(blk)
            assert q == 0 and np.array_equal(u, a), (name, sorter)
            q, u = checker.decompress(blk)
            assert q == 0 and np.array_equal(u, a), (name, sorter)
            if sorter <= 6:
                z2, b2 = checker.compress(a, sorter, 1, 3)
                assert z == z2 and np.array_equal(blk, b2), (name, sorter)


def test_bwt_encode_matches_oracle(bsc, gen, checker):
    for name, a in small_inputs(gen):
        r2, L2, x2 = checker.bwt_encode(a)
        r1, L1, x1 = bsc.bwt_encode(a)
        assert r1 == r2, (name, r1, r2)
        assert x1 == x2, (name, x1, x2)
        assert np.array_equal(L1, L2), name


def test_bwt_small_n_conventions(bsc, port):
    for n in (0, 1, 2, 3, 7, 8, 9, 15, 16, 17, 31, 33):
        a = ((np.arange(n) * 7 + 3) % 5).astype(np.uint8)
        assert bsc.bwt_encode(a, aux=True)[0] == port.bwt_encode(a, aux=True)[0], n
        r1, L1, _ = bsc.bwt_encode(a, aux=False)
        r2, L2, _ = port.bwt_encode(a, aux=False)
        assert r1 == r2 and np.array_equal(L1, L2), n


def test_bwt_decode_matches_oracle(bsc, gen, checker):
    for name, a in small_inputs(gen):
        r, L, _ = checker.bwt_encode(a)
        d, T = bsc.bwt_decode(L, r)
        assert d == 0 and np.array_equal(T, a), name
    assert bsc.bwt_decode(np.zeros(10, np.uint8), 0)[0] == -1
    assert bsc.bwt_decode(np.zeros(10, np.uint8), 11)[0] == -1


def test_coder_compress_matches_oracle(bsc, gen, checker):
    for name, a in list(small_inputs(gen)) + [("text5M", gen.text(9, 5 << 20))]:
        _, L, _ = checker.bwt_encode(a)
        for feats in (3, 1):
            c2, s2 = checker.coder_compress(L, 1, feats)
            c1, s1 = bsc.coder_compress(L, 1, feats)
            assert c1 == c2, (name, feats, c1, c2)
            if c2 > 0:
                assert np.array_equal(s1, s2), (name, feats)


def test_coder_decompress_matches_oracle(bsc, gen, checker):
    for name, a in list(small_inputs(gen)) + [("text5M", gen.text(9, 5 << 20))]:
        _, L, _ = checker.bwt_encode(a)
        c, s = checker.coder_compress(L, 1, 3)
        if c <= 0:
            continue
        n, out = bsc.coder_decompress(s, L.size)
        assert n == L.size, (name, n)
        assert np.array_equal(out, L), name


def test_block_bytes_and_cross_decoding(bsc, gen, checker):
    for name, a in small_inputs(gen):
        for sorter in (1, 6):
            z2, b2 = checker.compress(a, sorter, 1, 3)
            z1, b1 = bsc.compress(a, sorter, 1, 3)
            assert z1 == z2, (name, sorter, z1, z2)
            assert np.array_equal(b1, b2), (name, sorter)
        z, blk = bsc.compress(a, 1, 1, 3)
        q, u = checker.decompress(blk)                    # ours -> reference decoder
        assert q == 0 and np.array_equal(u, a), name
        z, blk = checker.compress(a, 1, 1, 3)
        q, u = bsc.decompress(blk)                        # reference -> our decoder
        assert q == 0 and np.array_equal(u, a), name


def test_inplace_compress_and_decompress(bsc, gen):
    """The CLI's calls (bsc.cpp:354, 594): bsc_compress(buf, buf, ...) and bsc_decompress(buf, size, buf, n) on ONE buffer, against the
    reference's in-place results.  In place, an incompressible block answers LIBBSC_NOT_COMPRESSIBLE instead of being stored
    (libbsc.cpp:188-191)."""
    L = bsc.lib
    for name, (a, sorter) in ri.inplace_inputs(gen).items():
        n = a.size
        buf = np.zeros(n + 28 + 64, dtype=np.uint8); buf[:n] = a
        r = L.bsc_compress(buf.ctypes.data, buf.ctypes.data, n, 0, 0, sorter, 1, 3)
        assert r > 0 and digest(buf[:r]) == GOLD["inplace"][name], (name, r)
        q = L.bsc_decompress(buf.ctypes.data, r, buf.ctypes.data, n, 3)
        assert q == 0 and np.array_equal(buf[:n], a), sorter
    a = gen.rand(1, 300000)
    buf = np.zeros(a.size + 28 + 64, dtype=np.uint8); buf[:a.size] = a
    assert L.bsc_compress(buf.ctypes.data, buf.ctypes.data, a.size, 0, 0, 1, 1, 3) == -3
    assert np.array_equal(buf[:a.size], a)                           # the input is left alone


def test_degenerate_blocks_at_full_size(bsc):
    """64 MiB all-zero, period-7, period-8 (a power of two: LF keeps row residues) and two-symbol blocks: every suffix stays in an unsorted
    group for ~23 doubling rounds, and the inverse walks arithmetic progressions of rows.  Bounded in time, bit-exact against the reference."""
    import time
    for name, a in ri.degenerate_inputs().items():
        want = GOLD["degenerate"][name]
        t0 = time.time()
        r, L, aux = bsc.bwt_encode(a)
        t1 = time.time()
        assert r == want["index"] and aux == want["aux"] and digest(L) == want["L"], name
        t2 = time.time()
        q, T = bsc.bwt_decode(L, r)
        t3 = time.time()
        assert q == 0 and np.array_equal(T, a), name
        z, blk = bsc.compress(a)
        assert z > 0 and digest(blk) == want["block"], name
        q, u = bsc.decompress(blk)
        assert q == 0 and np.array_equal(u, a), name
        assert t1 - t0 < 30 and t3 - t2 < 30, (name, t1 - t0, t3 - t2)


def test_error_codes(bsc, gen):
    a = gen.text(1, 1000)
    assert bsc.compress(a, sorter=2)[0] == -1
    assert bsc.compress(a, coder=0)[0] == -1
    assert bsc.compress(a, lzp_hash=5, lzp_min=128)[0] == -1
    z, blk = bsc.compress(a)
    bad = blk.copy(); bad[40] ^= 1
    assert bsc.decompress(bad)[0] == -6
    bad = blk.copy(); bad[3] ^= 1
    assert bsc.block_info(bad)[0] == -6
    r, s = bsc.compress(gen.text(1, 20))                          # n <= 28: stored
    assert r == 48 and int.from_bytes(bytes(s[8:12]), "little") == 0


def test_k1_random_block_is_stored(bsc, gen):
    a = gen.rand(1, 1048576)
    r, L, aux = bsc.bwt_encode(a)
    assert r == 791385 and aux == [633903, 252159, 118572, 805028, 426935, 565037, 575571]
    assert gen.adler32(L) == 0x5ce80fec
    assert bsc.coder_compress(L, 1, 3)[0] == -3
    z, blk = bsc.compress(a)
    assert z == 1048604 and gen.adler32(blk) == 0x242115a8
    q, u = bsc.decompress(blk)
    assert q == 0 and np.array_equal(u, a)


def test_k2_text_25mb(bsc, gen):
    a = gen.text(2, 26214400)
    r, L, aux = bsc.bwt_encode(a)
    assert r == 4197692
    assert aux == [19656645, 17965358, 3119786, 16132698, 10774871, 18082751, 1296587, 1120570, 2626855, 2680633, 25151113, 17332296]
    assert gen.adler32(L) == 0x77ffc0f7
    c, s = bsc.coder_compress(L, 1, 3)
    assert c == 5019497 and gen.adler32(s) == 0xe6f2f8c5
    z, blk = bsc.compress(a)
    assert z == 5019574 and gen.adler32(blk) == 0xed300f73
    q, u = bsc.decompress(blk)
    assert q == 0 and np.array_equal(u, a)


def test_k3_text_64mb(bsc, gen):
    a = gen.text(2, 67108864)
    z, blk = bsc.compress(a)
    assert z == 12686186 and gen.adler32(blk) == 0xf21848c1
    assert int.from_bytes(bytes(blk[12:16]), "little") == 10745360
    q, u = bsc.decompress(blk)
    assert q == 0 and np.array_equal(u, a)


def test_k5_st6_skew_32mb(bsc, gen):
    a = gen.skew(3, 33554432)
    i, L = bsc.st_encode(a, 6)
    assert i == 28690215 and gen.adler32(L) == 0x3141fea1
    z, blk = bsc.compress(a, sorter=6)
    assert z == 32294018 and gen.adler32(blk) == 0x8d12e56b
    r, T = bsc.st_decode(L, 6, i)                                 # BASELINE config 5, decode side
    assert r == 0 and np.array_equal(T, a)
    q, u = bsc.decompress(blk)
    assert q == 0 and np.array_equal(u, a)


def test_decompress_blocks_made_with_reference_default_options(bsc, gen):
    """bsc_decompress accepts blocks with an LZP stage (the reference's default lzpHashSize 15 / lzpMinLen 128): GPU stages, then
    the inverse LZP stage on the host (csrc/lzp_host.h).  The blocks are the reference's own: same size and SHA-256."""
    for name, a in list(ri.lzp_inputs(gen).items())[:3]:
        z, blk = bsc.compress(a, 1, 1, 3, lzp_hash=15, lzp_min=128)
        assert z > 0 and digest(blk) == GOLD["lzp"][name + "/f3"], name
        q, u = bsc.decompress(blk)
        assert q == 0 and np.array_equal(u, a)
        bad = blk.copy(); bad[-5] ^= 1
        assert bsc.decompress(bad)[0] == -6


def test_compress_with_reference_default_options(bsc, gen):
    """bsc_compress(lzpHashSize 15, lzpMinLen 128) = the reference's default call: host LZP stage, then the GPU stages."""
    for name, a in ri.lzp_inputs(gen).items():
        for feats in (3, 1):
            z1, b1 = bsc.compress(a, 1, 1, feats, lzp_hash=15, lzp_min=128)
            assert z1 > 0 and digest(b1) == GOLD["lzp"]["%s/f%d" % (name, feats)], (name, feats)
        q, u = bsc.decompress(b1)
        assert q == 0 and np.array_equal(u, a)
