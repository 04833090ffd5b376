"""Seeded inputs of the GPU tests that compare with tests/golden/reference_results.json (written by
tests/golden/make_reference_results.py from the same functions)."""
import numpy as np

CLI_OPTS = ["-b8"]


def lzp_inputs(gen):
    """blocks made with the reference's default LZP stage (lzpHashSize 15, lzpMinLen 128)"""
    return {"rep700x900": np.tile(gen.text(3, 700), 900), "text2_1M_x5": np.tile(gen.text(2, 1 << 20), 5), "text6_200k": gen.text(6, 200000),
            "A3000": np.full(3000, 65, np.uint8), "rand1_300k": gen.rand(1, 300000)}


def inplace_inputs(gen):
    """(input, sorter) of the in-place bsc_compress calls"""
    return {"text2_1M": (gen.text(2, 1 << 20), 1), "text5_300k": (gen.text(5, 300000), 1), "skew3_1M": (gen.skew(3, 1 << 20), 6),
            "text9_70k": (gen.text(9, 70000), 4)}


def degenerate_inputs():
    """64 MiB blocks on which every suffix stays in an unsorted group for many doubling rounds"""
    n = 64 << 20
    rng = np.random.default_rng(17)
    return {"zeros": np.zeros(n, dtype=np.uint8),
            "period7": np.tile(np.frombuffer(b"abcabcd", dtype=np.uint8), n // 7 + 1)[:n],
            "period8": np.tile(np.frombuffer(b"abcdefgh", dtype=np.uint8), n // 8),
            "two-symbol runs": np.repeat(rng.integers(0, 2, n // 4096, dtype=np.uint8), 4096)}


def cli_input(gen):
    return gen.text(2, 40 << 20)
