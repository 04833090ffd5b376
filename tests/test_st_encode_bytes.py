"""The HBM bound of bsc_st_encode, bscb200_st_encode_bytes(n), without a GPU: its formula above 1 GiB, the pooled cost up to 1 GiB, its
monotonicity on each side of 1 GiB, the bad-argument returns, the exported symbol and its Python binding."""
import ctypes
import os
import subprocess

import pytest

import libbsc_b200

N_MAX = 2146435072
GIB, MIB = 1 << 30, 1 << 20
LIBPATH = os.path.join(os.path.dirname(os.path.abspath(libbsc_b200.__file__)), "libbsc_b200.so")


@pytest.fixture(scope="module")
def L():
    return libbsc_b200.lib()


@pytest.mark.parametrize("n", [GIB + 1, 1610612736, N_MAX])
def test_bound_above_1GiB(L, n):
    assert L.bscb200_st_encode_bytes(n) == 6 * n + 256 * MIB


def test_bound_at_max(L):
    """at most 6 n + 256 MiB at the largest block: about 13.1 GB, a sixth of an 80 GB card"""
    assert L.bscb200_st_encode_bytes(N_MAX) <= 6 * N_MAX + 256 * MIB
    assert L.bscb200_st_encode_bytes(N_MAX) < 13.2e9


@pytest.mark.parametrize("n", [0, 1, 29, 1 << 20, 64 * MIB, GIB])
def test_pooled_cost_up_to_1GiB(L, n):
    """the staged block in a pooled context (n + 4096) and one standard ST sort slab (30 n + 16 MiB)"""
    assert L.bscb200_st_encode_bytes(n) == n + 4096 + 30 * n + 16 * MIB


def test_monotone_on_each_side_of_1GiB(L):
    below = [0, 1, 2, 1000, 1 << 20, 100 * MIB, GIB - 1, GIB]
    above = [GIB + 1, GIB + 2, 1500 * MIB, 2 * GIB - 2 * MIB, N_MAX - 1, N_MAX]
    for side in (below, above):
        v = [L.bscb200_st_encode_bytes(n) for n in side]
        assert v == sorted(v) and len(set(v)) == len(v), (side, v)
    assert L.bscb200_st_encode_bytes(GIB + 1) < L.bscb200_st_encode_bytes(GIB)      # the bounded path needs far less than the pooled one


def test_bad_arguments(L):
    for n in (-1, -2, -(1 << 31), N_MAX + 1, (1 << 31) - 1):
        assert L.bscb200_st_encode_bytes(n) == -1, n


def test_symbol_exported_and_bound():
    p = subprocess.run(["nm", "-D", "--defined-only", LIBPATH], capture_output=True, text=True, check=True)
    assert any(line.split()[-1] == "bscb200_st_encode_bytes" for line in p.stdout.splitlines() if line.strip())
    assert libbsc_b200._SIGNATURES["bscb200_st_encode_bytes"] == ([ctypes.c_int], ctypes.c_longlong)
    f = libbsc_b200.lib().bscb200_st_encode_bytes
    assert f.restype is ctypes.c_longlong and f.argtypes == [ctypes.c_int]
