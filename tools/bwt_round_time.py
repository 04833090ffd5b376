"""Where the forward BWT's time goes: one text block through DeviceCtx.bwt_encode on the standard sorter, per switch setting.

    python tools/bwt_round_time.py [--mib 64] [--reps 5] [--seg 1024,0] [--stage default] [--alternate 2] [--root DIR] [--table]

Each pair of a BSCB200_BWT_SEG and a BSCB200_BWT_STAGE setting (staged or direct rank and L stores) runs in a child process of its
own (the library reads the switches once per process); the settings are alternated --alternate times.  A child makes one G_text(2)
block, warms up with one call, then reports
  - the device time of every kernel (set_profile / profile_report) of one call,
  - the same call split into phases from a torch.profiler trace: the initial sort and first split, each doubling round (from one
    bwt_gather_key2 to the next) and the emit, each with its device time per kernel,
  - the median wall time of --reps calls without profiling.
Every child's L, primary index and secondary indexes are checked against the first child's.  Runs are keyed "<seg>/<stage>".  --root runs another checkout's
build (an A/B against the parent commit); --table adds, computed on the host with numpy, each round's active entries m, group
count G and the share of active entries in groups of at most 32 / 256 / 1024 / 2048 / 8192 entries.  Prints one JSON line with
the card's name, power limit and maximum SM clock.  Writes nothing.
"""
import argparse
import hashlib
import json
import os
import re
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    try:
        f = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        return {"gpu": f[0].strip(), "power_limit_w": float(f[1]), "max_sm_clock_mhz": float(f[2])}
    except Exception:
        return {"gpu": None, "power_limit_w": None, "max_sm_clock_mhz": None}


def short(name):
    """a kernel's name without namespace and parameters: 'bwt_apply<false, true, true>', 'rs_onesweep<unsigned long, false, ...>'"""
    m = re.search(r"(\w+)(<.*>)?\(", name)
    return (m.group(1) + (m.group(2) or "")) if m else name


def phases(prof):
    """kernel device time (ms), launches and time per kernel per phase, in launch order"""
    from torch.autograd import DeviceType
    ev = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA), key=lambda e: e.time_range.start)
    out, cur = [], {"phase": "initial", "ms": 0.0, "kernels": 0, "per_kernel_ms": {}}
    rnd = 0
    for e in ev:
        name = e.name
        if "bwt_gather_key2" in name or ("bwt_emit" in name and not cur["phase"] == "emit"):
            out.append(cur)
            rnd += "bwt_gather_key2" in name
            cur = {"phase": "round %d" % rnd if "bwt_gather_key2" in name else "emit", "ms": 0.0, "kernels": 0, "per_kernel_ms": {}}
        ms = e.time_range.elapsed_us() / 1e3
        cur["ms"] += ms
        cur["kernels"] += 1
        k = short(name)
        cur["per_kernel_ms"][k] = cur["per_kernel_ms"].get(k, 0.0) + ms
    out.append(cur)
    for p in out:
        p["ms"] = round(p["ms"], 3)
        p["per_kernel_ms"] = {k: round(v, 3) for k, v in p["per_kernel_ms"].items()}
    return out


def child(args):
    sys.path.insert(0, args.root)
    import numpy as np
    import torch
    import libbsc_b200
    from oracle import pyoracle
    n = args.mib << 20
    src = torch.from_numpy(pyoracle.Gen().text(2, n)).cuda()
    work = torch.empty_like(src)
    ctx = libbsc_b200.DeviceCtx(0)

    def call():
        work.copy_(src)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = ctx.bwt_encode(work.data_ptr(), n)
        return r, time.perf_counter() - t0

    call()
    ctx.set_profile(True)
    (r, aux), _ = call()
    kern = {k: [c, round(ms, 3)] for k, (c, ms, b) in sorted(ctx.profile_report().items(), key=lambda x: -x[1][1])}
    ctx.set_profile(False)
    digest = hashlib.sha256(work.cpu().numpy().tobytes() + json.dumps([r, aux]).encode()).hexdigest()
    try:
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call()
            torch.cuda.synchronize()
        split = phases(prof)
    except Exception as e:                                   # the split is extra information; the rest stands without it
        split = "unavailable: %s" % e
    times = [call()[1] for _ in range(args.reps)]
    ctx.close()
    libbsc_b200.lib().bscb200_release_pools()
    print(json.dumps({"wall_s": float(np.median(times)), "wall_all_s": [round(t, 5) for t in times], "kernels_ms": kern,
                      "phases": split, "digest": digest}))


def table(mib):
    """per round of the prefix doubling: m, G and the share of the m active entries in groups of at most T entries"""
    import numpy as np
    sys.path.insert(0, ROOT)
    from oracle import pyoracle
    n = mib << 20
    p = np.concatenate([pyoracle.Gen().text(2, n), np.zeros(8, np.uint8)]).astype(np.uint64)
    key = np.zeros(n, np.uint64)
    for j in range(8):
        key = (key << np.uint64(8)) | p[j:j + n]
    order = np.argsort(key, kind="stable")
    comb = key[order]
    rank = np.empty(n + 1, np.int64)
    rank[n] = 0
    rows, h = [], 8
    while True:
        head = np.ones(n, bool)
        head[1:] = comb[1:] != comb[:-1]
        gid = np.cumsum(head) - 1
        starts = np.flatnonzero(head)
        sizes = np.diff(np.append(starts, n))
        rank[order] = starts[gid] + 1
        big = sizes[sizes > 1]
        m = int(big.sum())
        if m == 0:
            return rows
        rows.append({"h": h, "m_over_n": round(m / n, 4), "G": int(big.size),
                     "share_le": {T: round(float(big[big <= T].sum()) / m, 3) for T in (32, 256, 1024, 2048, 8192)}})
        k2 = np.where(order + h < n, rank[np.minimum(order + h, n)], 0)
        o2 = np.lexsort((k2, gid))
        order, comb = order[o2], gid[o2].astype(np.int64) * (n + 2) + k2[o2]
        h *= 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mib", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seg", default="1024,0", help="BSCB200_BWT_SEG settings, comma separated ('default': unset)")
    ap.add_argument("--stage", default="default", help="BSCB200_BWT_STAGE settings, comma separated: 0 direct, 1 staged, 'default': unset")
    ap.add_argument("--alternate", type=int, default=2)
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--table", action="store_true")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)
    out = {"block_mib": args.mib, "input": "G_text(2)", "reps": args.reps, "root": os.path.abspath(args.root), **card(), "runs": {}}
    want = None
    for _ in range(args.alternate):
        for s in args.seg.split(","):
            for g in args.stage.split(","):
                env = dict(os.environ)
                for var, val in (("BSCB200_BWT_SEG", s), ("BSCB200_BWT_STAGE", g)):
                    env.pop(var, None)
                    if val != "default":
                        env[var] = val
                key = "%s/%s" % (s, g)
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--mib", str(args.mib), "--reps", str(args.reps),
                                    "--root", args.root], env=env, capture_output=True, text=True)
                if p.returncode != 0:
                    raise SystemExit("child BSCB200_BWT_SEG/STAGE=%s failed:\n%s" % (key, p.stderr[-4000:]))
                res = json.loads(p.stdout.strip().splitlines()[-1])
                want = want or res["digest"]
                assert res["digest"] == want, "BSCB200_BWT_SEG/STAGE=%s: output differs from the first setting's" % key
                out["runs"].setdefault(key, []).append(res)
    out["median_wall_s"] = {s: [r["wall_s"] for r in rs] for s, rs in out["runs"].items()}
    if args.table:
        out["rounds"] = table(args.mib)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
