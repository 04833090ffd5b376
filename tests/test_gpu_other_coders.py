"""GPU parity tests of the ADAPTIVE (coder id 2, csrc/qlfc_adaptive.cuh) and FAST (coder id 3, csrc/qlfc_fast.cuh) QLFC coders
through the C ABI (SURVEY 8(f) #1): byte-identical streams, containers and blocks against the reference, and decoding of the
reference's streams."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

def _inputs(gen):
    rng = np.random.default_rng(11)
    yield "text300k", gen.text(7, 300000)
    yield "text1M", gen.text(2, 1 << 20)
    yield "text5M", gen.text(9, 5 << 20)
    yield "skew300k", gen.skew(3, 300000)
    yield "rand70k", gen.rand(1, 70000)
    yield "alpha4", rng.integers(0, 4, 5000, dtype=np.uint8)
    yield "alpha2_64k", rng.integers(0, 2, 65536, dtype=np.uint8)
    yield "allsame3000", np.full(3000, 65, dtype=np.uint8)
    yield "long runs", np.repeat(rng.integers(0, 200, 2000, dtype=np.uint8), rng.integers(1, 3000, 2000))
    yield "tiny100", gen.text(1, 100)


@pytest.mark.parametrize("coder", [2, 3])
def test_coder_matches_oracle(bsc, gen, checker, coder):
    for name, a in _inputs(gen):
        _, L, _ = checker.bwt_encode(a)
        for feats in (3, 1):
            c2, s2 = checker.coder_compress(L, coder, feats)
            c1, s1 = bsc.coder_compress(L, coder, feats)
            assert c1 == c2, (name, feats, c1, c2)
            if c2 > 0:
                assert np.array_equal(s1, s2), (name, feats)
        c, s = checker.coder_compress(L, coder, 3)
        if c > 0:
            n, out = bsc.coder_decompress(s, L.size, coder)
            assert n == L.size and np.array_equal(out, L), name
        z2, b2 = checker.compress(a, 1, coder, 3)
        z1, b1 = bsc.compress(a, 1, coder, 3)
        assert z1 == z2 and np.array_equal(b1, b2), name
        q, u = bsc.decompress(b2)
        assert q == 0 and np.array_equal(u, a), name


@pytest.mark.parametrize("coder", [1, 2, 3])
def test_qlfc_block_entry_points(bsc, gen, checker, coder):
    """bsc_qlfc_{static,adaptive,fast}_{encode,decode}_block (qlfc.h:55-99): one stream at a time, byte-identical to the reference, both the
    default capacity (= inputSize) and a clipped one (the EOB rule of rangecoder.h:118-127 decides compressible / not compressible)."""
    rng = np.random.default_rng(3)
    for name, a in (("bwt text 300k", checker.bwt_encode(gen.text(7, 300000))[1]), ("bwt text 2M", checker.bwt_encode(gen.text(2, 2 << 20))[1]),
                    ("skew 200k", gen.skew(3, 200000)), ("alpha4", rng.integers(0, 4, 50000, dtype=np.uint8)), ("allsame", np.full(3000, 65, dtype=np.uint8)),
                    ("rand 70k", gen.rand(1, 70000)), ("tiny", gen.text(1, 40))):
        for cap in (None, a.size // 3, a.size // 2):
            r2, s2 = checker.encode_block(a, cap, coder)
            r1, s1 = bsc.encode_block(a, cap, coder)
            assert r1 == r2, (name, cap, r1, r2)
            if r2 > 0:
                assert np.array_equal(s1, s2), (name, cap)
                n, out = bsc.decode_block(s2, a.size, coder)
                assert n == a.size and np.array_equal(out, a), (name, cap)
