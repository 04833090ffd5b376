"""HBM of a block in flight: the per-context workspace (bscb200_workspace_bytes) holds the coder stage and the inverse BWT on every input,
a compress takes that workspace and one sort slab (bscb200_scratch_bytes), and the host-pointer entry points reserve no more than that
accounting says."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MIB = 1 << 20
SLACK = 64 * MIB              # cudaMalloc rounds every allocation up to 2 MiB; the driver keeps a little for itself


@pytest.fixture(scope="module")
def torch_cuda(bsc):
    import torch
    return torch


def round_trip_exact(torch, L, a, coder, features):
    """compress and decompress `a` on a device context whose arena is exactly bscb200_workspace_bytes(n, 1)"""
    import libbsc_b200
    n = a.size
    ctx = libbsc_b200.DeviceCtx(0)
    try:
        assert ctx.reserve(L.bscb200_workspace_bytes(n, 1)) == 0
        src = torch.from_numpy(a).cuda()
        cmp = torch.zeros(n + 28 + 4096, dtype=torch.uint8, device="cuda")
        back = torch.zeros(n + 64, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        r = ctx.compress(src.data_ptr(), cmp.data_ptr() + 4, n, 1, coder, features)
        assert r > 0, (n, coder, features, r)
        assert ctx.decompress(cmp.data_ptr() + 4, r, back.data_ptr(), n, features) == 0, (n, coder, features)
        assert torch.equal(back[:n], src), (n, coder, features)
        return r
    finally:
        ctx.close()


@pytest.mark.parametrize("coder", [1, 2, 3])
def test_exact_workspace_random_and_text(torch_cuda, bsc, gen, coder):
    """random bytes (one run per byte: the coder stage's largest buffers; the block ends stored, and the serial rules of features 1
    re-encode its sub-blocks clipped) and text (a coded block that goes through the inverse BWT)"""
    L = bsc.lib
    r = round_trip_exact(torch_cuda, L, gen.rand(1, 64 * MIB), coder, 1)
    assert r == 64 * MIB + 28
    r = round_trip_exact(torch_cuda, L, gen.text(2, 24 * MIB), coder, 3)
    assert r < 24 * MIB


@pytest.mark.parametrize("n", [t + d for t in (256 << 10, 4 << 20, 16 << 20) for d in (-1, 0, 1)])
def test_exact_workspace_at_sub_block_thresholds(torch_cuda, bsc, gen, n):
    """the number of coder streams changes at these sizes (coder.cpp:52-59)"""
    round_trip_exact(torch_cuda, bsc.lib, gen.rand(n % 7 + 1, n), 1, 1)
    round_trip_exact(torch_cuda, bsc.lib, gen.text(n % 5 + 1, n), 1, 3)


def test_exact_workspace_random_1GiB(torch_cuda, bsc, gen):
    L = bsc.lib
    n = 1 << 30
    if L.bscb200_device_free_bytes() < L.bscb200_workspace_bytes(n, 1) + L.bscb200_scratch_bytes(n, 1) + 4 * n:
        pytest.skip("not enough free HBM for a 1 GiB block")
    try:
        assert round_trip_exact(torch_cuda, L, gen.rand(3, n), 1, 1) == n + 28
    finally:
        L.bscb200_release_pools()


def test_workspace_at_bench_block_sizes(bsc):
    """at the block sizes users run, a context's workspace is at most 9 n + 64 MiB"""
    L = bsc.lib
    for n in (25 * MIB, 32 * MIB, 64 * MIB, 1 << 30):
        assert L.bscb200_workspace_bytes(n, 1) <= 9 * n + 64 * MIB, n


CHILD = r"""
import json, sys, threading, time
import numpy as np
sys.path.insert(0, %(root)r)
import torch
import libbsc_b200
from oracle import pyoracle

L = libbsc_b200.lib()
assert L.bsc_init(3) == 0
n, K = %(n)d, %(k)d


class Peak:
    def __enter__(self):
        torch.cuda.synchronize()
        self.before = self.low = L.bscb200_device_free_bytes()
        self.stop = threading.Event()
        self.t = threading.Thread(target=self.poll)
        self.t.start()
        return self

    def poll(self):
        while not self.stop.wait(0.005):
            self.low = min(self.low, L.bscb200_device_free_bytes())

    def __exit__(self, *exc):
        self.stop.set(); self.t.join()
        self.low = min(self.low, L.bscb200_device_free_bytes())


blocks = [pyoracle.Gen().text(2 + i, n) for i in range(K)]
out = {"workspace": L.bscb200_workspace_bytes(n, 1), "slab": L.bscb200_scratch_bytes(n, 1)}
if %(mode)r == "device":
    a = blocks[0]
    src = torch.from_numpy(a).cuda()
    dst = torch.zeros(n + 4096, dtype=torch.uint8, device="cuda")
    ctx = libbsc_b200.DeviceCtx(0)
    warm = torch.from_numpy(pyoracle.Gen().text(9, 1 << 20)).cuda()        # loads the kernels, then frees its slab
    assert ctx.compress(warm.data_ptr(), dst.data_ptr(), warm.numel()) > 0
    ctx.close(); L.bscb200_release_pools()
    ctx = libbsc_b200.DeviceCtx(0)
    with Peak() as p:
        r = ctx.compress(src.data_ptr(), dst.data_ptr(), n)
        torch.cuda.synchronize()
    assert r > 0
else:
    w = pyoracle.Gen().text(9, 1 << 20)                                         # loads the kernels; the pools are emptied after it
    wc, wb = np.zeros(w.size + 4096, np.uint8), np.zeros(w.size + 64, np.uint8)
    assert L.bsc_decompress(wc.ctypes.data, L.bsc_compress(w.ctypes.data, wc.ctypes.data, w.size, 0, 0, 1, 1, 3), wb.ctypes.data, w.size, 3) == 0
    L.bscb200_release_pools()
    ins = [b.copy() for b in blocks]
    cmps = [np.zeros(n + 4096, np.uint8) for _ in range(K)]
    backs = [np.zeros(n + 64, np.uint8) for _ in range(K)]
    res = [None] * K

    def work(i):
        r = L.bsc_compress(ins[i].ctypes.data, cmps[i].ctypes.data, n, 0, 0, 1, 1, 3)
        d = L.bsc_decompress(cmps[i].ctypes.data, r, backs[i].ctypes.data, n, 3) if r > 0 else None
        res[i] = (r, d)
    with Peak() as p:
        ts = [threading.Thread(target=work, args=(i,)) for i in range(K)]
        for t in ts: t.start()
        for t in ts: t.join()
        torch.cuda.synchronize()
    assert all(r > 0 and d == 0 for r, d in res), res
    assert all(np.array_equal(blocks[i], backs[i][:n]) for i in range(K))
out["peak"] = p.before - p.low
print(json.dumps(out))
"""


def child(mode, n, k=1):
    code = CHILD % {"root": ROOT, "n": n, "k": k, "mode": mode}
    p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert p.returncode == 0, p.stderr[-3000:]
    return json.loads(p.stdout.strip().splitlines()[-1])


def test_compress_peak_within_workspace_and_slab(bsc):
    """one 64 MiB compress in a fresh process: the HBM it takes is its context's workspace and one sort slab"""
    r = child("device", 64 * MIB)
    assert r["peak"] <= r["workspace"] + r["slab"] + SLACK, r


def test_host_entry_points_reserve_the_accounted_size(bsc):
    """K concurrent bsc_compress + bsc_decompress calls on pooled contexts: each context's arena is the workspace plus the staged block
    and its output, beside at most six sort slabs"""
    n, k = 64 * MIB, 4
    r = child("host", n, k)
    per_call = r["workspace"] + 2 * (n + 4096 + 512)
    assert r["peak"] <= k * per_call + min(k, 6) * r["slab"] + SLACK, r
