"""Blocks above 1 GiB, up to the reference's 2146435072 bytes (its CLI's -b2047): an in-place bsc_compress sorts them with the batched
forward BWT on a context of its own, within bscb200_inplace_bytes() = 18 n + 256 MiB of HBM, and returns all of it when the call ends.
The blocks and the -b2047 archive must equal the reference's (tests/golden/reference_results_large.json, written by
tests/golden/make_reference_results_large.py from the inputs of tests/large_block_inputs.py) and decompress to the input."""
import hashlib
import json
import os
import subprocess
import threading
import time

import numpy as np
import pytest

import large_block_inputs as li

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_results_large.json")))
PRODUCT = os.path.join(ROOT, "libbsc_b200", "bsc_b200")
MIB = 1 << 20
SLACK = 64 * MIB                        # free HBM after a call is back within this of the value before it


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
    """The library, after a 1 MiB block has gone through every stage the large blocks use (batched sort, coders 1 and 3, both
    directions): kernel images load on first use and stay, and must not count as HBM a large block kept."""
    import torch
    import libbsc_b200
    a = gen.text(4, 1 << 20)
    ctx = libbsc_b200.DeviceCtx(0)
    assert ctx.set_sort_budget(1) == 0
    src = torch.from_numpy(a).cuda()
    dst = torch.zeros(a.size + 4096, dtype=torch.uint8, device="cuda")
    back = torch.zeros_like(src)
    torch.cuda.synchronize()
    for coder in (1, 3):
        r = ctx.compress(src.data_ptr(), dst.data_ptr(), a.size, 1, coder)
        assert r > 0 and ctx.decompress(dst.data_ptr(), r, back.data_ptr(), a.size) == 0
    ctx.close()
    del src, dst, back
    L = bsc.lib
    L.bscb200_release_pools()                                           # pooled contexts and sort slabs of earlier tests
    torch.cuda.empty_cache()                                            # blocks cached by torch here and in tests that ran before
    return L


def room_for(L, n, host_bytes):
    free, need = L.bscb200_device_free_bytes(), L.bscb200_inplace_bytes(n, 1, 1)
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


@pytest.mark.parametrize("name", list(li.CASES))
def test_inplace_block_matches_reference(lib, bsc, gen, name):
    make, lzp_hash, lzp_min, coder = li.CASES[name]
    want = GOLD["inplace"][name]
    n = want["input"]["size"]
    room_for(lib, n, 3 * n)
    bound = lib.bscb200_inplace_bytes(n, 1, coder)
    buf = np.empty(n + 28 + 64, dtype=np.uint8)
    buf[:n] = make(gen)
    assert sha(buf[:n]) == want["input"]["sha256"], "input generator changed"
    p = buf.ctypes.data
    with Peak(lib) as pc:
        r = lib.bsc_compress(p, p, n, lzp_hash, lzp_min, 1, coder, 3)
    assert r == want["block"]["size"] and sha(buf[:r]) == want["block"]["sha256"], (name, r, want["block"]["size"])
    pc.check(bound, "compress")
    assert bsc.block_info(buf[:28]) == (0, r, n)

    out = np.empty(n + 64, dtype=np.uint8)
    with Peak(lib) as pd:
        q = lib.bsc_decompress(p, r, out.ctypes.data, n, 3)
    assert q == 0 and sha(out[:n]) == want["input"]["sha256"], (name, q)
    pd.check(bound, "decompress")
    print("\n%s: n %d -> %d bytes; compress %.1f s, peak %.2f GB; decompress %.1f s, peak %.2f GB; bound %.2f GB"
          % (name, n, r, pc.seconds, (pc.before - pc.low) / 1e9, pd.seconds, (pd.before - pd.low) / 1e9, bound / 1e9))


def test_limits_above_1GiB(lib):
    """out of place above 1 GiB is a bad parameter and ST6 in place is not supported, as before; neither touches the buffers"""
    a = np.zeros(64, dtype=np.uint8)
    b = np.zeros(64, dtype=np.uint8)
    n = (1 << 30) + 1
    assert lib.bsc_compress(a.ctypes.data, b.ctypes.data, n, 0, 0, 1, 1, 3) == -1
    assert lib.bsc_compress(a.ctypes.data, a.ctypes.data, n, 0, 0, 6, 1, 3) == -4
    assert lib.bsc_compress(a.ctypes.data, a.ctypes.data, li.N_MAX + 1, 0, 0, 1, 1, 3) == -1
    assert lib.bscb200_inplace_bytes(n, 6, 1) == -4


def test_cli_b2047_matches_reference_cli(lib, gen, tmp_path):
    """a file larger than 2 GiB at -b2047: one in-place block of 2146435072 bytes and a 64 MiB one, byte-identical to `bsc e -b2047 -p -t`"""
    a = li.cli_input(gen)
    n = a.size
    room_for(lib, li.N_MAX, 2 * n)
    path, arch, back = str(tmp_path / "in.bin"), str(tmp_path / "a.bsc"), str(tmp_path / "back.bin")
    assert sha(a) == GOLD["cli_input"]["sha256"], "input generator changed"
    a.tofile(path)
    del a
    t0 = time.time()
    subprocess.run([PRODUCT, "e", path, arch] + li.CLI_OPTS, check=True, capture_output=True)
    t1 = time.time()
    ours = np.fromfile(arch, dtype=np.uint8)
    assert {"size": int(ours.size), "sha256": sha(ours)} == GOLD["cli_archive"]
    del ours
    subprocess.run([PRODUCT, "d", arch, back], check=True, capture_output=True)
    t2 = time.time()
    assert os.path.getsize(back) == n and sha(np.fromfile(back, dtype=np.uint8)) == GOLD["cli_input"]["sha256"]
    print("\ncli -b2047: %d bytes; e %.1f s, d %.1f s" % (n, t1 - t0, t2 - t1))
