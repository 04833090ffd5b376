"""Sort-transform blocks above 1 GiB, up to the reference's 2146435072 bytes: bsc_decompress runs them on a context of its own with the
lean layout of the inverse ST, in at most bscb200_decompress_bytes(n, k) = 26.5 n + 256 MiB of HBM, and returns all of it when the call
ends.  The reference compresses each input in place on the host (its blocks are first checked against
tests/golden/reference_results_st_large.json, written by tests/golden/make_reference_results_st_large.py from the inputs of
tests/large_st_inputs.py); this library must restore the input.  ST7 and ST8, which only the reference's CUDA build writes, come from
oracle/_ref/libbsc_refcuda.so where it was built.  With BSCB200_STSTATS set the library reports the list count and the st_serial time of
every block, which the test prints."""
import ctypes
import hashlib
import json
import os
import re
import subprocess
import sys
import threading
import time
import zlib

import numpy as np
import pytest

import large_st_inputs as li

pytestmark = pytest.mark.gpu

os.environ.setdefault("BSCB200_STSTATS", "1")           # read once, at the first lean inverse ST of the process

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_results_st_large.json")))
PRODUCT = os.path.join(ROOT, "libbsc_b200", "bsc_b200")
REFDIR = os.path.join(ROOT, "oracle", "_ref")
MIB, GIB = 1 << 20, 1 << 30
SLACK = 64 * MIB                        # free HBM after a call is back within this of the value before it
vp = ctypes.c_void_p


def sha(a):
    return hashlib.sha256(memoryview(np.ascontiguousarray(a, dtype=np.uint8))).hexdigest()


def host_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


@pytest.fixture(scope="module")
def lib(bsc, gen):
    """The library, after a 1 MiB ST block has gone through both directions with coders 1 and 3: kernel images load on first use and
    stay, and must not count as HBM a large block kept."""
    import torch
    L = bsc.lib
    a = gen.text(4, 1 << 20)
    for coder in (1, 3):
        z, blk = bsc.compress(a, sorter=6, coder=coder, features=3)
        q, u = bsc.decompress(blk)
        assert q == 0 and np.array_equal(u, a)
    L.bscb200_release_pools()                                           # pooled contexts and sort slabs of earlier tests
    torch.cuda.empty_cache()
    return L


def room_for(L, n, k, host_bytes):
    free, need = L.bscb200_device_free_bytes(), L.bscb200_decompress_bytes(n, k)
    if free < need:
        pytest.skip("the device has %d bytes free, a block of %d bytes needs %d" % (free, n, need))
    if host_available() < host_bytes:
        pytest.skip("the host has %d bytes available, the test needs about %d" % (host_available(), host_bytes))


class Peak:
    """lowest free HBM seen while the block runs (cudaMemGetInfo from a second thread every 10 ms)"""

    def __init__(self, L):
        self.L = L

    def __enter__(self):
        self.before = self.low = self.L.bscb200_device_free_bytes()
        self.stop = threading.Event()
        self.t = threading.Thread(target=self._poll)
        self.t.start()
        self.t0 = time.time()
        return self

    def _poll(self):
        while not self.stop.wait(0.01):
            self.low = min(self.low, self.L.bscb200_device_free_bytes())

    def __exit__(self, *exc):
        self.seconds = time.time() - self.t0
        self.stop.set()
        self.t.join()
        self.after = self.L.bscb200_device_free_bytes()
        self.low = min(self.low, self.after)

    def check(self, bound, what):
        assert self.before - self.low <= bound, (what, "peak", self.before - self.low, "bound", bound)
        assert abs(self.after - self.before) <= SLACK, (what, "free before", self.before, "after", self.after)


def ststats(capfd):
    """the [ststats] lines the library wrote to stderr since the last call"""
    err = capfd.readouterr().err
    sys.stderr.write(err)
    return re.findall(r"\[ststats\] n (\d+) k (\d) lists (\d+) st_serial ([0-9.]+) s", err)


def decode_and_check(lib, capfd, what, block, n, k, want_sha):
    bound = lib.bscb200_decompress_bytes(n, k)
    out = np.empty(n + 64, dtype=np.uint8)
    capfd.readouterr()
    with Peak(lib) as pd:
        q = lib.bsc_decompress(block.ctypes.data, block.size, out.ctypes.data, n, 3)
    stats = ststats(capfd)
    assert q == 0 and sha(out[:n]) == want_sha, (what, q)
    pd.check(bound, what)
    s = stats[-1] if stats else ("?", k, "?", "?")
    print("\n%s: n %d, %d bytes; decompress %.1f s, peak %.2f GB, bound %.2f GB; lists %s, st_serial %s s"
          % (what, n, block.size, pd.seconds, (pd.before - pd.low) / 1e9, bound / 1e9, s[2], s[3]))


@pytest.mark.parametrize("name", list(li.ST_CASES))
def test_reference_st_block_decodes(lib, ref, gen, capfd, name):
    make, sorter, lzp_hash, lzp_min, coder = li.ST_CASES[name]
    want = GOLD["inplace"][name]
    n = want["input"]["size"]
    room_for(lib, n, sorter, 3 * n)
    buf = np.empty(n + 28 + 64, dtype=np.uint8)
    buf[:n] = make(gen)
    assert sha(buf[:n]) == want["input"]["sha256"], "input generator changed"
    t0 = time.time()
    r = ref.lib.bsc_compress(vp(buf.ctypes.data), vp(buf.ctypes.data), n, lzp_hash, lzp_min, sorter, coder, 3)
    t_ref = time.time() - t0
    assert r == want["block"]["size"] and sha(buf[:r]) == want["block"]["sha256"], \
        ("the reference build differs from the one that wrote the golden file", name, r, want["block"]["size"])
    block = buf[:r].copy()
    del buf
    print("\n%s: the reference's CPU encode took %.1f s" % (name, t_ref))
    decode_and_check(lib, capfd, name, block, n, sorter, want["input"]["sha256"])


REFCUDA_CHILD = r"""
import ctypes, sys
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
from oracle import pyoracle
import large_st_inputs as li
R = ctypes.CDLL(sys.argv[1] + "/oracle/_ref/libbsc_refcuda.so")
assert R.bsc_init(1 | 2 | 8) == 0                          # FASTMODE | MULTITHREADING | CUDA (bsc.cpp -G)
R.bsc_compress.argtypes = [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 6
k, n = int(sys.argv[2]), int(sys.argv[3])
buf = np.empty(n + 28 + 64, dtype=np.uint8)
buf[:n] = li.st_mix(pyoracle.Gen(), n)
r = R.bsc_compress(buf.ctypes.data, buf.ctypes.data, n, 0, 0, k, 1, 1 | 2 | 8)
if r > 0:
    buf[:r].tofile(sys.argv[4])
print(r)
"""


@pytest.mark.parametrize("k", [7, 8])
def test_refcuda_st7_st8_block_decodes(lib, gen, capfd, tmp_path, k):
    """ST7 / ST8 blocks above 1 GiB from the reference's CUDA build, in a child process of its own (its HBM is gone when it exits)"""
    if not os.path.exists(os.path.join(REFDIR, "libbsc_refcuda.so")):
        pytest.skip("oracle/_ref/libbsc_refcuda.so not built: no ST7 / ST8 writer")
    n = GIB + 1
    room_for(lib, n, k, 3 * n)
    path = str(tmp_path / "st.blk")
    p = subprocess.run([sys.executable, "-c", REFCUDA_CHILD, ROOT, str(k), str(n), path], capture_output=True, text=True)
    r = int(p.stdout.split()[-1]) if p.returncode == 0 and p.stdout.split() else None
    if not r or r <= 0:
        pytest.skip("the reference's CUDA build did not write an ST%d block of %d bytes (exit %d, result %s): %s"
                    % (k, n, p.returncode, r, p.stderr.strip()[-300:]))
    block = np.fromfile(path, dtype=np.uint8)
    os.remove(path)
    assert block.size == r
    decode_and_check(lib, capfd, "refcuda mix_1G+1/m%de1" % k, block, n, k, sha(li.st_mix(gen, n)))


def test_not_enough_hbm_writes_nothing(lib):
    """with less free HBM than the bound the call returns LIBBSC_GPU_NOT_ENOUGH_MEMORY and leaves the output untouched"""
    import torch
    n, k = GIB + 1, 6
    h = np.zeros(28, dtype=np.uint8)
    h[0:24].view("<u4")[:] = [28 + 1000, n, k | (1 << 5), 5, 1, 1]
    h[24:28].view("<u4")[0] = zlib.adler32(h[:24].tobytes())
    block = np.concatenate([h, np.zeros(1000, dtype=np.uint8)])
    assert lib.bsc_block_info(block.ctypes.data, 28, None, None, 3) == 0
    out = np.full(n, 0xA5, dtype=np.uint8)
    free, bound = lib.bscb200_device_free_bytes(), lib.bscb200_decompress_bytes(n, k)
    hold = max(0, free - bound + GIB)
    if hold >= free:
        pytest.skip("cannot leave less than the bound free")
    x = torch.empty(hold, dtype=torch.uint8, device="cuda")
    try:
        assert lib.bscb200_device_free_bytes() < bound
        assert lib.bsc_decompress(block.ctypes.data, block.size, out.ctypes.data, n, 3) == -9
    finally:
        del x
        torch.cuda.empty_cache()
    assert (out == 0xA5).all()


def test_cli_decodes_reference_st_archive(lib, gen, tmp_path):
    """`bsc e -b2047 -m6 -p -t` of a file larger than 2 GiB (an ST6 block of 2146435072 bytes and a 64 MiB one): bsc_b200 d restores it"""
    cli = os.path.join(REFDIR, "bsc")
    if not os.path.exists(cli):
        pytest.skip("oracle/_ref/bsc (the reference CLI) not built")
    a = li.st_cli_input(gen)
    n = a.size
    room_for(lib, li.N_MAX, 6, 2 * n)
    path, arch, back = str(tmp_path / "in.bin"), str(tmp_path / "a.bsc"), str(tmp_path / "back.bin")
    assert sha(a) == GOLD["cli_input"]["sha256"], "input generator changed"
    a.tofile(path)
    del a
    t0 = time.time()
    subprocess.run([cli, "e", path, arch] + li.ST_CLI_OPTS + ["-p", "-t"], check=True, capture_output=True)
    t1 = time.time()
    theirs = np.fromfile(arch, dtype=np.uint8)
    assert {"size": int(theirs.size), "sha256": sha(theirs)} == GOLD["cli_archive"], "the reference CLI differs from the golden file's"
    del theirs
    os.remove(path)
    subprocess.run([PRODUCT, "d", arch, back], check=True, capture_output=True)
    t2 = time.time()
    assert os.path.getsize(back) == n and sha(np.fromfile(back, dtype=np.uint8)) == GOLD["cli_input"]["sha256"]
    print("\ncli -b2047 -m6: %d bytes; reference e %.1f s, bsc_b200 d %.1f s" % (n, t1 - t0, t2 - t1))
