"""Host-side parts of blocks above 1 GiB, without a GPU: the HBM bound bscb200_inplace_bytes() and the CLI's -b range (1..2047 MiB, as
the reference CLI's), checked on the CLI source built against the unmodified reference library."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "libbsc_b200", "cli", "bsc_b200.cpp")
REFDIR = os.path.join(ROOT, "oracle", "_ref")
REFCLI = os.path.join(REFDIR, "bsc")
TESTCLI = os.path.join(ROOT, "tools", "bin", "bsc_b200_ref_limits")
N_MAX = 2146435072


def test_inplace_bytes_formula():
    import libbsc_b200
    L = libbsc_b200.lib()
    prev = -1
    for n in [0, 1, 1 << 20, 1 << 30, (1 << 30) + 1, 1610612736, N_MAX - 1, N_MAX]:
        for coder in (1, 2, 3):
            v = L.bscb200_inplace_bytes(n, 1, coder)
            assert v == 18 * n + (256 << 20), (n, coder, v)
        assert v >= prev
        prev = v
    assert L.bscb200_inplace_bytes(N_MAX, 1, 1) < 40 * 10 ** 9                 # one block at a time fits an 80 GB card twice over
    assert L.bscb200_inplace_bytes(N_MAX + 1, 1, 1) == -1
    assert L.bscb200_inplace_bytes(-1, 1, 1) == -1
    assert L.bscb200_inplace_bytes(1 << 20, 1, 0) == -1
    assert L.bscb200_inplace_bytes(1 << 20, 2, 1) == -1
    for sorter in range(3, 9):
        assert L.bscb200_inplace_bytes(N_MAX, sorter, 1) == -4


@pytest.fixture(scope="module")
def cli():
    if not (os.path.exists(REFCLI) and os.path.exists(os.path.join(REFDIR, "libbsc_ref.so"))):
        pytest.skip("oracle/_ref (reference library + CLI) not built")
    os.makedirs(os.path.dirname(TESTCLI), exist_ok=True)
    if not os.path.exists(TESTCLI) or os.path.getmtime(SRC) > os.path.getmtime(TESTCLI):
        subprocess.run(["/usr/bin/g++", "-O2", "-std=c++17", "-Wall", "-pthread", "-fopenmp", "-DBSCB200_CLI_REF", SRC, "-o", TESTCLI,
                        "-L" + REFDIR, "-lbsc_ref", "-Wl,-rpath," + REFDIR], check=True, capture_output=True)
    return TESTCLI


def test_cli_block_size_range(cli, gen, tmp_path):
    """-b2047 is accepted and writes what the reference CLI writes; -b2048 and -b0 print the usage and write nothing"""
    path = str(tmp_path / "in.bin")
    gen.text(3, 300000).tofile(path)
    for b in ("-b1024", "-b1025", "-b2047"):
        ours, theirs = str(tmp_path / "ours.bsc"), str(tmp_path / "theirs.bsc")
        subprocess.run([cli, "e", path, ours, b, "-j2"], check=True, capture_output=True)
        subprocess.run([REFCLI, "e", path, theirs, b, "-p", "-t"], check=True, capture_output=True)
        assert open(ours, "rb").read() == open(theirs, "rb").read(), b
    for b in ("-b2048", "-b0"):
        out = str(tmp_path / ("bad%s.bsc" % b))
        p = subprocess.run([cli, "e", path, out, b], capture_output=True, text=True)
        assert "Usage" in p.stdout and not os.path.exists(out), b
