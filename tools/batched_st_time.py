"""Time the forward sort transform of one text block on the standard sorter and on the batched sorter (bscb200_ctx_set_sort_budget).

    python tools/batched_st_time.py [--mib 64] [--reps 3] [--orders 6,8]

Prints one JSON line: for each order k, median seconds per call (after one warm-up call) for the standard sorter, for batches of about
n / 8 entries and for the smallest batches (max(65536, n / 64) entries), each checked against the standard sorter's output, plus the
card's name and power limit.  Runs from a read-only tree and writes nothing.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import libbsc_b200                       # noqa: E402
from oracle import pyoracle              # noqa: E402
from batched_bwt_time import card        # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--orders", default="6,8")
    args = ap.parse_args()
    n = args.mib << 20
    a = pyoracle.Gen().text(2, n)
    src = torch.from_numpy(a).cuda()
    work = torch.empty_like(src)
    arms = {"standard": 0, "batched_n_over_8": n + 28 * (n // 8) + (16 << 20), "batched_smallest": 1}
    out = {}
    for k in (int(x) for x in args.orders.split(",")):
        want = None
        for name, budget in arms.items():
            ctx = libbsc_b200.DeviceCtx(0)
            assert ctx.set_sort_budget(budget) == 0
            times = []
            for rep in range(args.reps + 1):
                work.copy_(src)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                r = ctx.st_encode(work.data_ptr(), n, k)
                dt = time.perf_counter() - t0
                if rep:
                    times.append(dt)
            got = (r, work.cpu().numpy())
            if want is None:
                want = got
            assert got[0] == want[0] and np.array_equal(got[1], want[1]), (k, name)
            ctx.close()
            out["st%d_%s_s" % (k, name)] = float(np.median(times))
        libbsc_b200.lib().bscb200_release_pools()
    out.update({"block_mib": args.mib, "input": "G_text(2)", "reps": args.reps, **card()})
    print(json.dumps(out))


if __name__ == "__main__":
    main()
