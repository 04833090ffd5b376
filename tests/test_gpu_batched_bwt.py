"""The batched forward BWT (csrc/bwt_encode_batched.cu), driven through bscb200_ctx_set_sort_budget on a device context: it must give
exactly the standard sorter's index, secondary indexes and L, and the same compressed blocks, with batches far smaller than the block and
groups far larger than a batch."""
import hashlib
import json
import os
import time

import numpy as np
import pytest

import reference_inputs as ri
from test_oracle import _sweep_inputs

pytestmark = pytest.mark.gpu

GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_results.json")))
TINY = 1                      # every budget below the fixed 16 n gives the smallest batches: max(65536, n / 64) entries


def digest(b):
    b = np.ascontiguousarray(b, dtype=np.uint8)
    return {"size": int(b.size), "sha256": hashlib.sha256(b.tobytes()).hexdigest()}


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
    """half the standard working set (58 n + 64 MiB): batches of about n / 2 entries"""
    return (58 * n + (64 << 20)) // 2


def bwt(torch, ctx, a, offset=0):
    """forward BWT of `a` on ctx, the block at `offset` bytes into a device buffer with no padding after it"""
    t = torch.zeros(offset + a.size, dtype=torch.uint8, device="cuda")
    t[offset:] = torch.from_numpy(a)
    torch.cuda.synchronize()
    r, aux = ctx.bwt_encode(t.data_ptr() + offset, a.size)
    return r, aux, t[offset:].cpu().numpy()


def compress(torch, ctx, a):
    src = torch.from_numpy(a).cuda()
    dst = torch.zeros(a.size + 4096, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    r = ctx.compress(src.data_ptr(), dst.data_ptr(), a.size)
    return r, dst[:max(r, 0)].cpu().numpy()


def same_bwt(torch, std, ctx, a, name, offset=0):
    want = bwt(torch, std, a)
    got = bwt(torch, ctx, a, offset)
    assert got[0] == want[0] and got[1] == want[1], (name, got[:2], want[:2])
    assert np.array_equal(got[2], want[2]), name


def structured_inputs(gen):
    rng = np.random.default_rng(5)
    mib = 1 << 20
    yield "text1M", gen.text(2, mib)
    yield "text8M", gen.text(5, 8 * mib)
    yield "skew3M", gen.skew(3, 3 * mib)
    yield "rand2M", gen.rand(1, 2 * mib)
    yield "alpha2_1M", rng.integers(0, 2, mib, dtype=np.uint8)
    yield "runs1M", np.repeat(rng.integers(0, 4, mib // 64, dtype=np.uint8), rng.integers(1, 128, mib // 64))[:mib].copy()
    yield "zeros4M", np.zeros(4 * mib, dtype=np.uint8)
    yield "period7_4M", np.tile(np.frombuffer(b"abcabcd", dtype=np.uint8), 4 * mib // 7 + 1)[:4 * mib].copy()
    yield "period8_4M", np.tile(np.frombuffer(b"abcdefgh", dtype=np.uint8), 4 * mib // 8)
    yield "text_zero_tail", np.concatenate([gen.text(4, mib), np.zeros(300000, np.uint8), gen.text(6, 5)])


def test_set_sort_budget_rejects_negative(ctxs):
    std, _ = ctxs
    assert std.set_sort_budget(-1) == -1
    assert std.set_sort_budget(0) == 0


def test_budget_selects_the_batched_sorter(torch_cuda, ctxs, gen):
    """an 8 MiB text block under the smallest budget (batches of n / 64 entries) is cut into many ranges and sorted in batches"""
    std, small = ctxs
    a = gen.text(5, 8 << 20)
    for ctx, batched in ((std, False), (small, True)):
        ctx.set_profile(True)
        bwt(torch_cuda, ctx, a)
        prof = ctx.profile_report()
        ctx.set_profile(False)
        assert ("bb_hist16" in prof) == batched, sorted(prof)
        if batched:
            assert prof["bb_count"][0] > 64 and prof["bb_find_start"][0] > 0, prof


def test_batched_bwt_matches_standard_tiny_batches(torch_cuda, ctxs, gen):
    std, small = ctxs
    for name, a in structured_inputs(gen):
        same_bwt(torch_cuda, std, small, a, name)


def test_batched_bwt_matches_standard_medium_batches(torch_cuda, ctxs, gen):
    import libbsc_b200
    std, _ = ctxs
    for name, a in structured_inputs(gen):
        med = libbsc_b200.DeviceCtx(0)
        assert med.set_sort_budget(medium_budget(a.size)) == 0
        same_bwt(torch_cuda, std, med, a, name)
        med.close()


def test_batched_bwt_small_n_and_sweep(torch_cuda, ctxs, gen, checker):
    std, small = ctxs
    for n in range(1, 301):
        a = gen.text(n % 7 + 1, n)
        same_bwt(torch_cuda, std, small, a, "text%d" % n, offset=n % 8)
    for name, a in _sweep_inputs(160, 20260924):
        same_bwt(torch_cuda, std, small, a, name)
        if a.size >= 16:
            r, aux, L = bwt(torch_cuda, small, a)
            r2, L2, aux2 = checker.bwt_encode(a)
            assert r == r2 and aux == list(aux2) and np.array_equal(L, L2), name


def test_batched_compress_matches_standard(torch_cuda, ctxs, gen):
    std, small = ctxs
    for name, a in structured_inputs(gen):
        r1, b1 = compress(torch_cuda, std, a)
        r2, b2 = compress(torch_cuda, small, a)
        assert r1 == r2 and r1 > 0 and np.array_equal(b1, b2), (name, r1, r2)


def test_batched_bwt_degenerate_64MiB(torch_cuda, ctxs):
    """the 64 MiB blocks on which every suffix stays in a large unsorted group for ~23 rounds, against the reference's digests"""
    import libbsc_b200
    for name, a in ri.degenerate_inputs().items():
        want = GOLD["degenerate"][name]
        for budget in (20 * a.size + (16 << 20), TINY):                      # batches of about n / 8 entries, then of n / 64
            ctx = libbsc_b200.DeviceCtx(0)
            assert ctx.set_sort_budget(budget) == 0
            t0 = time.time()
            r, aux, L = bwt(torch_cuda, ctx, a)
            dt = time.time() - t0
            ctx.close()
            assert r == want["index"] and aux == want["aux"] and digest(L) == want["L"], (name, budget)
            assert dt < 60, (name, budget, dt)
