"""The batched forward sort transform (csrc/st_encode_batched.cu), driven through bscb200_ctx_set_sort_budget on a device context and
through bsc_st_encode above the routing threshold: for k = 3..8 it must give exactly the standard sorter's index and L, and the same
compressed blocks, with batches far smaller than the block and single key values far larger than a batch.  For k = 3..6 it must also
equal the reference's bsc_st_encode."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from test_gpu_batched_bwt import structured_inputs
from test_oracle import _sweep_inputs

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = 1                      # every budget below the fixed n gives the smallest batches: max(65536, n / 64) entries
ORDERS = (3, 4, 5, 6, 7, 8)


@pytest.fixture(scope="module")
def torch_cuda(bsc):
    import torch
    return torch


@pytest.fixture(scope="module")
def ctxs(bsc):
    import libbsc_b200
    std, small = libbsc_b200.DeviceCtx(0), libbsc_b200.DeviceCtx(0)
    assert small.set_sort_budget(TINY) == 0
    yield std, small
    std.close(); small.close()
    bsc.lib.bscb200_release_pools()


def medium_budget(n):
    """half the standard working set (30 n + 16 MiB): batches of about n / 2 entries"""
    return (30 * n + (16 << 20)) // 2


def st(torch, ctx, a, k, offset=0):
    """forward ST-k of `a` on ctx, the block at `offset` bytes into a device buffer with no padding after it"""
    t = torch.zeros(offset + a.size, dtype=torch.uint8, device="cuda")
    t[offset:] = torch.from_numpy(a)
    torch.cuda.synchronize()
    r = ctx.st_encode(t.data_ptr() + offset, a.size, k)
    return r, t[offset:].cpu().numpy()


def same_st(torch, std, ctx, a, name, k, offset=0):
    want = st(torch, std, a, k)
    got = st(torch, ctx, a, k, offset)
    assert got[0] == want[0] and want[0] >= 0, (name, k, got[0], want[0])
    assert np.array_equal(got[1], want[1]), (name, k)
    return got


def test_budget_selects_the_batched_sorter(torch_cuda, ctxs, gen):
    """an 8 MiB text block under the smallest budget (batches of n / 64 entries) is cut into many ranges and sorted in batches"""
    std, small = ctxs
    a = gen.text(5, 8 << 20)
    for ctx, batched in ((std, False), (small, True)):
        ctx.set_profile(True)
        st(torch_cuda, ctx, a, 6)
        prof = ctx.profile_report()
        ctx.set_profile(False)
        assert ("st_batch_emit" in prof) == batched and ("bb_hist16" in prof) == batched, sorted(prof)
        assert ("st_finish" in prof) != batched, sorted(prof)
        if batched:
            assert prof["st_batch_emit"][0] > 16 and prof["bb_count"][0] > 16, prof


def test_batched_st_matches_standard_tiny_batches(torch_cuda, ctxs, gen):
    std, small = ctxs
    for name, a in structured_inputs(gen):
        for k in ORDERS:
            same_st(torch_cuda, std, small, a, name, k)


def test_batched_st_matches_standard_medium_batches(torch_cuda, ctxs, gen):
    import libbsc_b200
    std, _ = ctxs
    for name, a in structured_inputs(gen):
        med = libbsc_b200.DeviceCtx(0)
        assert med.set_sort_budget(medium_budget(a.size)) == 0
        for k in ORDERS:
            same_st(torch_cuda, std, med, a, name, k)
        med.close()


def test_batched_st_matches_reference(torch_cuda, ctxs, gen, ref):
    _, small = ctxs
    for name, a in structured_inputs(gen):
        for k in (3, 4, 5, 6):
            r, L = st(torch_cuda, small, a, k)
            r2, L2 = ref.st_encode(a, k)
            assert r == r2 and np.array_equal(L, L2), (name, k, r, r2)


def test_batched_st_small_n_and_sweep(torch_cuda, ctxs, gen, checker):
    """n = 1..300 at unaligned, unpadded addresses (n < k included), and the seeded sweep of test_oracle.py, against the standard sorter
    and, for k = 3..6, the strongest checker there is (the reference where it was built)"""
    std, small = ctxs
    for n in range(1, 301):
        a = gen.text(n % 7 + 1, n)
        for k in ORDERS:
            same_st(torch_cuda, std, small, a, "text%d" % n, k, offset=n % 8)
    for name, a in _sweep_inputs(160, 20260924):
        for k in ORDERS:
            r, L = same_st(torch_cuda, std, small, a, name, k, offset=a.size % 8)
            if k <= 6 and a.size > 1:
                r2, L2 = checker.st_encode(a, k)
                if r2 >= 0:
                    assert r == r2 and np.array_equal(L, L2), (name, k, r, r2)


def test_batched_compress_matches_standard(torch_cuda, ctxs, gen):
    std, small = ctxs
    for name, a in structured_inputs(gen):
        src = torch_cuda.from_numpy(a).cuda()
        for sorter in ORDERS:
            got = []
            for ctx in (std, small):
                dst = torch_cuda.zeros(a.size + 4096, dtype=torch_cuda.uint8, device="cuda")
                torch_cuda.cuda.synchronize()
                r = ctx.compress(src.data_ptr(), dst.data_ptr(), a.size, sorter, 1)
                got.append((r, dst[:max(r, 0)].cpu().numpy()))
            assert got[0][0] == got[1][0] and got[0][0] > 0 and np.array_equal(got[0][1], got[1][1]), (name, sorter, got[0][0], got[1][0])


ROUTED_CHILD = r"""
import os, sys
import numpy as np
sys.path.insert(0, sys.argv[1])
import libbsc_b200
b = libbsc_b200.Bsc(features=3)
d = sys.argv[2]
out = {}
for f in sorted(os.listdir(d)):
    if not f.endswith(".in.npy"):
        continue
    a = np.load(os.path.join(d, f))
    for k in range(3, 9):
        r, L = b.st_encode(a, k)
        np.save(os.path.join(d, "%s.k%d.npy" % (f[:-7], k)), L)
        out["%s.k%d" % (f[:-7], k)] = int(r)
print(__import__("json").dumps(out))
"""


def routed_inputs(gen):
    mib = 1 << 20
    yield "text29", gen.text(3, 29)
    yield "text300", gen.text(4, 300)
    yield "rand5000", gen.rand(2, 5000)
    yield "text1M", gen.text(2, mib)
    yield "skew1M", gen.skew(3, mib)
    yield "zeros1M", np.zeros(mib, dtype=np.uint8)
    yield "period7_1M", np.tile(np.frombuffer(b"abcabcd", dtype=np.uint8), mib // 7 + 1)[:mib].copy()
    for name, a in list(_sweep_inputs(160, 20260924))[::8]:
        if a.size > 28:
            yield name, a


def test_routed_bsc_st_encode(torch_cuda, ctxs, gen, ref, tmp_path):
    """BSCB200_LARGE_N=28 sends every bsc_st_encode of more than 28 bytes down the path of the blocks above 1 GiB (st_encode_large, a
    context of its own, the batched sorter): it must equal the reference for k = 3..6 and the standard sorter for k = 7, 8"""
    std, _ = ctxs
    inputs = dict(routed_inputs(gen))
    for name, a in inputs.items():
        np.save(str(tmp_path / (name + ".in.npy")), a)
    env = dict(os.environ, BSCB200_LARGE_N="28")
    p = subprocess.run([sys.executable, "-c", ROUTED_CHILD, ROOT, str(tmp_path)], capture_output=True, text=True, env=env)
    assert p.returncode == 0, p.stderr[-2000:]
    got = json.loads(p.stdout.strip().splitlines()[-1])
    assert len(got) == 6 * len(inputs)
    for name, a in inputs.items():
        for k in ORDERS:
            r, L = got["%s.k%d" % (name, k)], np.load(str(tmp_path / ("%s.k%d.npy" % (name, k))))
            r2, L2 = ref.st_encode(a, k) if k <= 6 else st(torch_cuda, std, a, k)
            assert r == r2 and np.array_equal(L, L2), (name, k, r, r2)
