"""The HBM bound of bsc_decompress, bscb200_decompress_bytes(n, blockSorter), without a GPU: its formula above 1 GiB for every sorter,
the pooled cost up to 1 GiB, the bad-argument returns, the exported symbol and its Python binding."""
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
    assert L.bscb200_decompress_bytes(n, 1) == L.bscb200_inplace_bytes(n, 1, 1) == 18 * n + 256 * MIB
    for sorter in range(3, 9):
        v = L.bscb200_decompress_bytes(n, sorter)
        assert v == 26 * n + n // 2 + 256 * MIB, (n, sorter, v)
        assert v <= 27 * n + 256 * MIB


def test_bound_at_max_fits_an_80GB_card(L):
    assert L.bscb200_decompress_bytes(N_MAX, 6) < 58.2e9
    assert L.bscb200_decompress_bytes(N_MAX, 1) < 40e9


@pytest.mark.parametrize("n", [0, 1, 29, 1 << 20, 64 * MIB, GIB])
def test_pooled_cost_up_to_1GiB(L, n):
    for sorter in (1, 3, 4, 5, 6, 7, 8):
        want = L.bscb200_workspace_bytes(n, sorter) + L.bscb200_scratch_bytes(n, sorter)
        assert L.bscb200_decompress_bytes(n, sorter) == want, (n, sorter)


def test_bad_arguments(L):
    for n, sorter in [(-1, 1), (N_MAX + 1, 1), (N_MAX + 1, 6), (1 << 20, 0), (1 << 20, 2), (1 << 20, 9), (GIB + 1, 2), (GIB + 1, -1)]:
        assert L.bscb200_decompress_bytes(n, sorter) == -1, (n, sorter)


def test_symbol_exported_and_bound():
    p = subprocess.run(["nm", "-D", "--defined-only", LIBPATH], capture_output=True, text=True, check=True)
    assert any(line.split()[-1] == "bscb200_decompress_bytes" for line in p.stdout.splitlines() if line.strip())
    import ctypes
    assert libbsc_b200._SIGNATURES["bscb200_decompress_bytes"] == ([ctypes.c_int, ctypes.c_int], ctypes.c_longlong)
    f = libbsc_b200.lib().bscb200_decompress_bytes
    assert f.restype is ctypes.c_longlong and f.argtypes == [ctypes.c_int, ctypes.c_int]
