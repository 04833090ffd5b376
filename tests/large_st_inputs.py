"""Seeded inputs of the sort-transform blocks above 1 GiB (tests/test_gpu_large_st_decode.py), shared with
tests/golden/make_reference_results_st_large.py, which records what the reference returns for them in
tests/golden/reference_results_st_large.json.  The text, zero and size helpers are those of the BWT blocks (large_block_inputs.py).
"""
import numpy as np

from large_block_inputs import GIB, MIB, N_MAX, tiled_text, zeros

# The inverse ST's serial part takes one step per list, and every row of a context that is followed by more than one distinct byte
# heads a list.  So these inputs are mostly made of contexts with ONE successor (a period of distinct bytes), which the inverse ranks in
# parallel and the QLFC coder codes as a few long runs; the other parts are kept small enough that the list count stays bounded.

def period251(n):
    """the bytes 0..250 over and over: every context of order 1..8 has one successor"""
    return np.tile(np.arange(251, dtype=np.uint8), n // 251 + 1)[:n]


def st_mix(gen, n=N_MAX):
    """n bytes: 16 MiB of text (lists of its own), a 4 MiB zero run (its order-k context is followed by 0 and by one other byte, so every
    row of the run heads a list: 4 M lists), a period-251 stretch and 4 MiB of random bytes at the end (a long QLFC stream).  The stretch's
    contexts have one successor there, but the random bytes contain some of them with other successors, which makes their whole groups
    dynamic: at k = 3 about a third of the rows head a list (714 M lists at the largest n), at k = 4 about 58 M, at k = 5 and 6 under 20 M"""
    a = np.empty(n, dtype=np.uint8)
    a[:16 * MIB] = gen.text(21, 16 * MIB)
    a[16 * MIB:20 * MIB] = 0
    a[20 * MIB:n - 4 * MIB] = period251(n - 24 * MIB)
    a[n - 4 * MIB:] = gen.rand(22, 4 * MIB)
    return a


# name -> (input, block sorter, lzpHashSize, lzpMinLen, coder) of the reference's in-place bsc_compress calls
ST_CASES = {
    "text_1G+1/m6e1": (lambda gen: tiled_text(gen, GIB + 1), 6, 0, 0, 1),      # text-heavy: about 0.6 n lists
    "mix_max/m3e1": (st_mix, 3, 0, 0, 1),
    "mix_max/m4e3": (st_mix, 4, 0, 0, 3),
    "mix_max/m5_lzp_e1": (st_mix, 5, 15, 128, 1),
    "mix_1G+1/m6e3": (lambda gen: st_mix(gen, GIB + 1), 6, 0, 0, 3),
    "zeros_max/m6e3": (lambda gen: zeros(), 6, 0, 0, 3),                        # one group of n rows, one list
}
ST_CLI_OPTS = ["-b2047", "-m6"]


def st_cli_input(gen):
    """a file larger than 2 GiB: one -b2047 block of `st_mix` and a 64 MiB text block after it"""
    return np.concatenate([st_mix(gen), gen.text(23, 64 * MIB)])
