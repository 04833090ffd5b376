"""Time the forward BWT of one text block on the standard sorter and on the batched sorter (bscb200_ctx_set_sort_budget).

    python tools/batched_bwt_time.py [--mib 64] [--reps 3]

Prints one JSON line: median seconds per call (after one warm-up call) for the standard sorter, for batches of about n / 8 entries
and for the smallest batches (max(65536, n / 64) entries), each checked against the standard sorter's output, plus the card's name
and power limit.  Runs from a read-only tree and writes nothing.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import libbsc_b200                       # noqa: E402
from oracle import pyoracle              # noqa: E402


def card():
    try:
        f = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        return {"gpu": f[0].strip(), "power_limit_w": float(f[1])}
    except Exception:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    n = args.mib << 20
    a = pyoracle.Gen().text(2, n)
    src = torch.from_numpy(a).cuda()
    work = torch.empty_like(src)
    arms = {"standard": 0, "batched_n_over_8": 20 * n + (16 << 20), "batched_smallest": 1}
    out, want = {}, None
    for name, budget in arms.items():
        ctx = libbsc_b200.DeviceCtx(0)
        assert ctx.set_sort_budget(budget) == 0
        times = []
        for rep in range(args.reps + 1):
            work.copy_(src)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r, aux = ctx.bwt_encode(work.data_ptr(), n)
            dt = time.perf_counter() - t0
            if rep:
                times.append(dt)
        got = (r, aux, work.cpu().numpy())
        if want is None:
            want = got
        assert got[0] == want[0] and got[1] == want[1] and np.array_equal(got[2], want[2]), name
        ctx.close()
        out[name + "_s"] = float(np.median(times))
    libbsc_b200.lib().bscb200_release_pools()
    out.update({"block_mib": args.mib, "input": "G_text(2)", "reps": args.reps, **card()})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
