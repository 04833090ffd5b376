"""Seeded inputs of the blocks above 1 GiB (tests/test_gpu_large_blocks.py), shared with tests/golden/make_reference_results_large.py,
which records what the reference returns for them in tests/golden/reference_results_large.json.

The inputs are built to keep the QLFC coder's work small (few runs after the BWT: it is a serial recurrence per sub-block stream) while
giving the batched forward BWT its hard cases: a long zero run, a long periodic stretch and long repeats keep most suffixes in unsorted
groups for many doubling rounds."""
import numpy as np

N_MAX = 2146435072                      # the largest block the reference compresses (in place, libbsc.cpp; its CLI's -b2047)
GIB, MIB = 1 << 30, 1 << 20
CLI_OPTS = ["-b2047"]


def tiled_text(gen, n, seed=11):
    """a 32 MiB generated text, repeated up to n bytes"""
    t = gen.text(seed, 32 * MIB)
    return np.tile(t, n // t.size + 1)[:n]


def mixed(gen, n=N_MAX):
    """64 MiB of text, a 1 GiB zero run, a period-7 stretch and 16 MiB of random bytes at the end"""
    a = np.empty(n, dtype=np.uint8)
    a[:64 * MIB] = gen.text(12, 64 * MIB)
    a[64 * MIB:64 * MIB + GIB] = 0
    p = n - 16 * MIB - (64 * MIB + GIB)
    a[64 * MIB + GIB:n - 16 * MIB] = np.tile(np.frombuffer(b"abcabcd", dtype=np.uint8), p // 7 + 1)[:p]
    a[n - 16 * MIB:] = gen.rand(13, 16 * MIB)
    return a


def zeros(n=N_MAX):
    return np.zeros(n, dtype=np.uint8)


# name -> (input, lzpHashSize, lzpMinLen, coder) of the in-place bsc_compress calls; block sorter 1 (BWT)
CASES = {
    "text_1G+1/e1": (lambda gen: tiled_text(gen, GIB + 1), 0, 0, 1),
    "mixed_max/e1": (mixed, 0, 0, 1),
    "mixed_max/e3": (mixed, 0, 0, 3),
    "mixed_max/lzp_e1": (mixed, 15, 128, 1),
    "zeros_max/e1": (lambda gen: zeros(), 0, 0, 1),
}


def cli_input(gen):
    """a file larger than 2 GiB: one -b2047 block of `mixed` and a 64 MiB text block after it"""
    return np.concatenate([mixed(gen), gen.text(14, 64 * MIB)])
