#!/usr/bin/env python3
"""tools/dec_ab.py -- timing of the QLFC coder kernels on ONE block (CUDA events around every launch), round trip checked.
    python tools/dec_ab.py [MiB]
(Round 2's A/B of the decoder generations and encoder variants used this script with BSCB200_QDEC / BSCB200_QENC at commit 4a20aea:
the losers are gone and so are the switches.)"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

if len(sys.argv) > 1 and sys.argv[1] == "--child":
    os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
    import torch
    sys.path.insert(0, ROOT)
    import libbsc_b200
    from oracle import pyoracle
    mib = int(sys.argv[2])
    n = mib << 20
    L = libbsc_b200.lib()
    assert L.bsc_init(3) == 0
    dev = torch.device("cuda", 0)
    src = torch.from_numpy(pyoracle.Gen().text(2, n)).to(dev)
    blk = torch.empty(n + 28 + 64, dtype=torch.uint8, device=dev)
    back = torch.empty(n + 64, dtype=torch.uint8, device=dev)
    ctx = libbsc_b200.DeviceCtx(0)
    assert ctx.reserve(int(L.bscb200_workspace_bytes(n, 1))) == 0
    for rep in range(2):
        ctx.set_profile(rep == 1)
        size = ctx.compress(src.data_ptr(), blk.data_ptr() + 4, n, 1, 1, 3)
        assert size > 0, size
        r = ctx.decompress(blk.data_ptr() + 4, size, back.data_ptr(), n, 3)
        assert r == 0, r
        assert torch.equal(back[:n], src)
    for name, (cnt, ms, by) in ctx.profile_report().items():
        if name.startswith(("q_decode", "q_encode")):
            print("%-10s  %d launch(es)  %.1f ms  (%d MiB block, round trip bit-exact, %d bytes)" % (name, cnt, ms, mib, size), flush=True)
    sys.exit(0)

mib = sys.argv[1] if len(sys.argv) > 1 else "64"
subprocess.run([sys.executable, os.path.abspath(__file__), "--child", mib], check=False)
