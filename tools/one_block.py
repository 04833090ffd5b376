#!/usr/bin/env python3
"""tools/one_block.py -- compress + decompress ONE synthetic block through the device-resident ABI.
Small driver for one-block captures: python tools/one_block.py [MiB] [sorter]"""
import os
import sys

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import libbsc_b200
from oracle import pyoracle

mib = int(sys.argv[1]) if len(sys.argv) > 1 else 16
sorter = int(sys.argv[2]) if len(sys.argv) > 2 else 1
n = mib << 20
gen = pyoracle.Gen()
L = libbsc_b200.lib()
assert L.bsc_init(3) == 0
dev = torch.device("cuda", 0)
src = torch.from_numpy(gen.text(2, n) if sorter == 1 else gen.skew(3, n)).to(dev)
blk = torch.empty(n + 28 + 64, dtype=torch.uint8, device=dev)
back = torch.empty(n + 64, dtype=torch.uint8, device=dev)
ctx = libbsc_b200.DeviceCtx(0)
assert ctx.reserve(int(L.bscb200_workspace_bytes(n, sorter))) == 0
size = ctx.compress(src.data_ptr(), blk.data_ptr() + 4, n, sorter, 1, 3)
assert size > 0, size
if sorter == 1:
    r = ctx.decompress(blk.data_ptr() + 4, size, back.data_ptr(), n, 3)
    assert r == 0, r
    assert torch.equal(back[:n], src)
print("one block: %d -> %d bytes, kernels launched %d" % (n, size, ctx.launches()))
