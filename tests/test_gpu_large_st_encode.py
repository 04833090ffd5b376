"""The forward sort transform above 1 GiB: bsc_st_encode of a block above 1 GiB sorts in batches on a context of its own, in at most
bscb200_st_encode_bytes(n) = 6 n + 256 MiB of HBM, and returns all of it when the call ends.

The reference's own block layer linked against this library's stages (oracle/_ref/libbsc_dropin.so and oracle/_ref/bsc_dropin, the
drop-in of INTEGRATION.md section 1) must write exactly the reference's blocks and archive of tests/golden/reference_results_st_large.json
with this library's bsc_st_encode underneath.  ST7 and ST8, which the reference cannot write at these sizes, must equal this library's
standard sorter and decode back to the input."""
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

import large_st_inputs as li
from test_gpu_large_st_decode import GOLD, Peak, host_available, sha

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRODUCT = os.path.join(ROOT, "libbsc_b200", "bsc_b200")
REFDIR = os.path.join(ROOT, "oracle", "_ref")
MIB, GIB = 1 << 20, 1 << 30
vp = ctypes.c_void_p


@pytest.fixture(scope="module")
def lib(bsc, gen):
    """The library, after a 1 MiB block has gone through bsc_st_encode on both paths' kernels: kernel images load on first use and stay,
    and must not count as HBM a large block kept."""
    import torch
    L = bsc.lib
    a = gen.text(4, 1 << 20)
    for k in (6, 8):
        assert bsc.st_encode(a, k)[0] >= 0
    L.bscb200_release_pools()
    torch.cuda.empty_cache()
    return L


def room_for(L, hbm, host_bytes):
    free = L.bscb200_device_free_bytes()
    if free < hbm:
        pytest.skip("the device has %d bytes free, the test needs %d" % (free, hbm))
    if host_available() < host_bytes:
        pytest.skip("the host has %d bytes available, the test needs about %d" % (host_available(), host_bytes))


def coder_hbm(n):
    """what this library's bsc_coder_compress of n bytes takes on a pooled context (staged input and output, the coder stage)"""
    return 11 * n + 256 * MIB


DROPIN_CHILD = r"""
import ctypes, hashlib, json, sys, time
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
from oracle import pyoracle
import large_st_inputs as li
R = ctypes.CDLL(sys.argv[1] + "/oracle/_ref/libbsc_dropin.so")
R.bsc_init.argtypes = [ctypes.c_int]
R.bsc_compress.argtypes = [ctypes.c_void_p, ctypes.c_void_p] + [ctypes.c_int] * 6
assert R.bsc_init(3) == 0
name, path = sys.argv[2], sys.argv[3]
gen = pyoracle.Gen()
if name.startswith("st"):                                   # st<k>: the ST7 / ST8 block of st_mix(1 GiB + 1), coder 1
    k, n = int(name[2:]), (1 << 30) + 1
    a, case = li.st_mix(gen, n), (k, 0, 0, 1)
else:
    make, *case = li.ST_CASES[name]
    a = make(gen)
    n = a.size
buf = np.empty(n + 28 + 64, dtype=np.uint8)
buf[:n] = a
del a
din = hashlib.sha256(memoryview(buf[:n])).hexdigest()
t0 = time.time()
r = R.bsc_compress(buf.ctypes.data, buf.ctypes.data, n, case[1], case[2], case[0], case[3], 3)
dt = time.time() - t0
if r > 0 and path != "-":
    buf[:r].tofile(path)
print(json.dumps({"r": r, "input": din, "block": hashlib.sha256(memoryview(buf[:max(r, 0)])).hexdigest(), "seconds": dt}))
"""


def dropin(name, path="-"):
    if not os.path.exists(os.path.join(REFDIR, "libbsc_dropin.so")):
        pytest.skip("oracle/_ref/libbsc_dropin.so not built (needs the reference's sources at build time)")
    p = subprocess.run([sys.executable, "-c", DROPIN_CHILD, ROOT, name, path], capture_output=True, text=True)
    assert p.returncode == 0, (name, p.returncode, p.stderr[-2000:])
    return json.loads(p.stdout.strip().splitlines()[-1])


@pytest.mark.parametrize("name", list(li.ST_CASES))
def test_dropin_block_equals_reference(lib, name):
    """the reference's in-place bsc_compress on this library's stages writes the reference's own block"""
    want = GOLD["inplace"][name]
    n = want["input"]["size"]
    room_for(lib, max(lib.bscb200_st_encode_bytes(n), coder_hbm(n)), 2 * n)
    got = dropin(name)
    assert got["input"] == want["input"]["sha256"], "input generator changed"
    assert got["r"] == want["block"]["size"] and got["block"] == want["block"]["sha256"], (name, got["r"], want["block"]["size"])
    print("\ndrop-in %s: n %d, block %d bytes, bsc_compress %.1f s" % (name, n, got["r"], got["seconds"]))


def test_dropin_cli_archive_equals_reference(lib, gen, tmp_path):
    """`bsc e -b2047 -m6 -p -t` of a file larger than 2 GiB through the drop-in CLI equals the reference CLI's archive; bsc_b200 d
    restores the file"""
    cli = os.path.join(REFDIR, "bsc_dropin")
    if not os.path.exists(cli):
        pytest.skip("oracle/_ref/bsc_dropin not built")
    a = li.st_cli_input(gen)
    n = a.size
    room_for(lib, coder_hbm(li.N_MAX), 2 * n)
    assert sha(a) == GOLD["cli_input"]["sha256"], "input generator changed"
    path, arch, back = str(tmp_path / "in.bin"), str(tmp_path / "a.bsc"), str(tmp_path / "back.bin")
    a.tofile(path)
    del a
    t0 = time.time()
    subprocess.run([cli, "e", path, arch] + li.ST_CLI_OPTS + ["-p", "-t"], check=True, capture_output=True)
    t1 = time.time()
    ours = np.fromfile(arch, dtype=np.uint8)
    assert {"size": int(ours.size), "sha256": sha(ours)} == GOLD["cli_archive"]
    del ours
    os.remove(path)
    subprocess.run([PRODUCT, "d", arch, back], check=True, capture_output=True)
    assert os.path.getsize(back) == n and sha(np.fromfile(back, dtype=np.uint8)) == GOLD["cli_input"]["sha256"]
    print("\ndrop-in cli -b2047 -m6: %d bytes; e %.1f s" % (n, t1 - t0))


def st_encode_host(lib, a, k):
    """bsc_st_encode of a copy of `a` under Peak, checked against bscb200_st_encode_bytes; returns the index, L and the seconds"""
    n = a.size
    T = np.empty(n + 64, dtype=np.uint8)
    T[:n] = a
    with Peak(lib) as pk:
        r = lib.bsc_st_encode(T.ctypes.data, n, k, 3)
    pk.check(lib.bscb200_st_encode_bytes(n), "bsc_st_encode n %d k %d" % (n, k))
    print("\nbsc_st_encode n %d k %d: %.1f s, peak %.2f GB, bound %.2f GB"
          % (n, k, pk.seconds, (pk.before - pk.low) / 1e9, lib.bscb200_st_encode_bytes(n) / 1e9))
    return r, T[:n], pk.seconds


@pytest.mark.parametrize("k", [7, 8])
def test_st7_st8_above_1GiB(lib, gen, tmp_path, k):
    """ST7 / ST8 of 1 GiB + 1 bytes: the bounded route equals the standard sorter (about 32 GB on a device context without a budget), and
    the drop-in's block decodes back to the input"""
    import torch
    import libbsc_b200
    n = GIB + 1
    room_for(lib, 30 * n + 2 * GIB, 4 * n)
    a = li.st_mix(gen, n)
    r, L, _ = st_encode_host(lib, a, k)
    assert r >= 0, r
    want = sha(L)
    del L
    ctx = libbsc_b200.DeviceCtx(0)
    t = torch.from_numpy(a).cuda()
    torch.cuda.synchronize()
    r2 = ctx.st_encode(t.data_ptr(), n, k)
    torch.cuda.synchronize()
    L2 = t.cpu().numpy()
    del t
    ctx.close()
    lib.bscb200_release_pools()
    torch.cuda.empty_cache()
    assert r == r2 and want == sha(L2), (k, r, r2)
    del L2

    path = str(tmp_path / "st.blk")
    got = dropin("st%d" % k, path)
    assert got["r"] > 0 and got["input"] == sha(a), got
    block = np.fromfile(path, dtype=np.uint8)
    os.remove(path)
    out = np.empty(n + 64, dtype=np.uint8)
    t0 = time.time()
    q = lib.bsc_decompress(block.ctypes.data, block.size, out.ctypes.data, n, 3)
    assert q == 0 and np.array_equal(out[:n], a), (k, q)
    print("\nST%d n %d: drop-in bsc_compress %.1f s, %d bytes; bsc_decompress %.1f s" % (k, n, got["seconds"], block.size, time.time() - t0))


def test_zeros_at_max_within_bound(lib):
    """the largest block, all zeros, ST8: one key value of n entries, emitted without a sort; index 0 and L all zeros"""
    n = li.N_MAX
    room_for(lib, lib.bscb200_st_encode_bytes(n), 3 * n)
    r, L, _ = st_encode_host(lib, np.zeros(n, dtype=np.uint8), 8)
    assert r == 0 and not L.any()


def test_not_enough_hbm_leaves_T_untouched(lib):
    """with less free HBM than the bound the call returns LIBBSC_GPU_NOT_ENOUGH_MEMORY and leaves T as it was"""
    import torch
    n, k = GIB + 1, 6
    T = np.full(n, 0xA5, dtype=np.uint8)
    free, bound = lib.bscb200_device_free_bytes(), lib.bscb200_st_encode_bytes(n)
    hold = max(0, free - bound + GIB)
    if hold >= free:
        pytest.skip("cannot leave less than the bound free")
    x = torch.empty(hold, dtype=torch.uint8, device="cuda")
    try:
        assert lib.bscb200_device_free_bytes() < bound
        assert lib.bsc_st_encode(T.ctypes.data, n, k, 3) == -9
    finally:
        del x
        torch.cuda.empty_cache()
    assert (T == 0xA5).all()
