#!/usr/bin/env python3
"""tools/time_ref_cuda.py -- the reference's OWN CUDA path (libcubwt forward / inverse BWT, st.cu forward ST) against ours, same box,
same host-pointer entry points (bsc_bwt_encode / bsc_bwt_decode / bsc_st_encode: H2D + kernels + D2H inside both timings).

The reference side is oracle/_ref/libbsc_refcuda.so: the unmodified reference compiled by oracle/Makefile with -DLIBBSC_CUDA_SUPPORT for
sm_90 (SURVEY 8c "second baseline"; rows a3 / a6 / a8).  Both sides get `reps` warm calls; best and median wall times are reported,
plus our own kernel-only time (CUDA events around every launch of the stage).  Outputs are compared byte for byte.
    python tools/time_ref_cuda.py [reps] > ref_cuda.json"""
import ctypes
import json
import os
import sys
import time

os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import libbsc_b200
from oracle import pyoracle

vp, ci = ctypes.c_void_p, ctypes.c_int
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
gen = pyoracle.Gen()
R = ctypes.CDLL(os.path.join(ROOT, "oracle", "_ref", "libbsc_refcuda.so"))
FEAT = 1 | 2 | 8                                         # FASTMODE | MULTITHREADING | CUDA (bsc.cpp -G)
assert R.bsc_init(FEAT) == 0
R.bsc_bwt_encode.argtypes = [vp, ci, vp, vp, ci]
R.bsc_bwt_decode.argtypes = [vp, ci, ci, ctypes.c_ubyte, vp, ci]
R.bsc_st_encode.argtypes = [vp, ci, ci, ci]
B = libbsc_b200.Bsc(features=3)
L = B.lib


def timed(call, prep, reps):
    """prep() restores the in-place buffer (untimed); call() is ONE C entry point on preallocated, already touched buffers"""
    ts = []
    out = None
    for _ in range(reps + 1):                            # first call warms allocations / module load
        prep()
        t0 = time.perf_counter(); out = call(); ts.append(time.perf_counter() - t0)
    ts = ts[1:]
    return out, min(ts) * 1e3, float(np.median(ts)) * 1e3


def ours_kernel_ms(stage, data, **kw):
    """kernel-only time of our stage: device-resident call on a profiled context"""
    import torch
    dev = torch.device("cuda", 0)
    n = data.size
    d = torch.from_numpy(data).to(dev)
    pad = torch.empty(n + 64, dtype=torch.uint8, device=dev); pad[:n] = d
    ctx = libbsc_b200.DeviceCtx(0)
    assert ctx.reserve(int(L.bscb200_workspace_bytes(n, kw.get("sorter", 1)))) == 0
    best = None
    for rep in range(3):
        pad[:n] = d
        ctx.set_profile(True)
        if stage == "bwt_encode":
            ctx.bwt_encode(pad.data_ptr(), n)
        elif stage == "bwt_decode":
            ctx.bwt_decode(pad.data_ptr(), n, kw["index"])
        elif stage == "st_encode":
            ctx.st_encode(pad.data_ptr(), n, kw["k"])
        elif stage == "st_decode":
            ctx.st_decode(pad.data_ptr(), n, kw["k"], kw["index"])
        rep_ms = sum(ms for (_, ms, _) in ctx.profile_report().values())
        ctx.set_profile(False)
        best = rep_ms if best is None else min(best, rep_ms)
    ctx.close()
    return best


# ---- single-call mode for kernel-only sums under ncu:  TRC_SIDE=ref|ours TRC_STAGE=bwt_encode|bwt_decode|st6_encode  ncu --metrics
# gpu__time_duration.sum --csv ... python tools/time_ref_cuda.py   (one call of one entry point of one library; tools/ncu_launch_sum.py adds up)
if os.environ.get("TRC_SIDE"):
    side, stage = os.environ["TRC_SIDE"], os.environ.get("TRC_STAGE", "bwt_encode")
    lib_, feat_ = (R, FEAT) if side == "ref" else (L, 3)
    for f_, a_ in (("bsc_bwt_encode", [vp, ci, vp, vp, ci]), ("bsc_bwt_decode", [vp, ci, ci, ctypes.c_ubyte, vp, ci]), ("bsc_st_encode", [vp, ci, ci, ci])):
        getattr(lib_, f_).argtypes = a_
    ni_ = ctypes.c_ubyte(0); idx_ = (ci * 256)()
    if stage.startswith("bwt"):
        a_ = gen.text(2, 64 << 20); buf_ = np.empty(a_.size + 64, dtype=np.uint8); buf_[:a_.size] = a_
        if stage == "bwt_decode":                        # the forward transform comes from the CPU reference (no kernels in the list)
            chk_ = pyoracle.best(); r_, L_, _ = chk_.bwt_encode(a_); buf_[:a_.size] = L_
            q_ = lib_.bsc_bwt_decode(buf_.ctypes.data, a_.size, r_, 0, None, feat_)
            assert q_ == 0 and np.array_equal(buf_[:a_.size], a_)
        else:
            r_ = lib_.bsc_bwt_encode(buf_.ctypes.data, a_.size, ctypes.byref(ni_), idx_, feat_)
            assert r_ == 10745360
    else:
        a_ = gen.skew(3, 32 << 20); buf_ = np.empty(a_.size + 64, dtype=np.uint8); buf_[:a_.size] = a_
        r_ = lib_.bsc_st_encode(buf_.ctypes.data, a_.size, 6, feat_)
        assert r_ == 28690215
    print("single call done:", side, stage)
    sys.exit(0)

rows = []
text = gen.text(2, 64 << 20)
skew = gen.skew(3, 32 << 20)
ni = ctypes.c_ubyte(0); idx = (ci * 256)()
bufR = np.empty(text.size + 64, dtype=np.uint8); bufO = np.empty(text.size + 64, dtype=np.uint8)
L.bsc_bwt_encode.argtypes = [vp, ci, vp, vp, ci]
L.bsc_bwt_decode.argtypes = [vp, ci, ci, ctypes.c_ubyte, vp, ci]
L.bsc_st_encode.argtypes = [vp, ci, ci, ci]
L.bsc_st_decode.argtypes = [vp, ci, ci, ci, ci]
R.bsc_st_decode.argtypes = [vp, ci, ci, ci, ci]


def load(buf, src):
    def f():
        buf[:src.size] = src
    return f


# ---- forward BWT, 64 MiB text (a3: libcubwt_bwt_aux through bsc_bwt_encode) ----
n = text.size
r_ref, rb, rm = timed(lambda: R.bsc_bwt_encode(bufR.ctypes.data, n, ctypes.byref(ni), idx, FEAT), load(bufR, text), reps)
r_our, ob, om = timed(lambda: L.bsc_bwt_encode(bufO.ctypes.data, n, ctypes.byref(ni), idx, 3), load(bufO, text), reps)
assert r_ref == r_our and np.array_equal(bufR[:n], bufO[:n]), "forward BWT differs from the reference's CUDA path"
L_ref = bufR[:n].copy()
rows.append({"stage": "bsc_bwt_encode 64 MiB G_text", "ref_cuda_ms_best": rb, "ref_cuda_ms_median": rm, "ours_ms_best": ob, "ours_ms_median": om,
             "ours_kernels_only_ms": ours_kernel_ms("bwt_encode", text), "bit_identical": True})

# ---- inverse BWT (a6: libcubwt_unbwt through bsc_bwt_decode) ----
q_ref, rb, rm = timed(lambda: R.bsc_bwt_decode(bufR.ctypes.data, n, r_ref, 0, None, FEAT), load(bufR, L_ref), reps)
q_our, ob, om = timed(lambda: L.bsc_bwt_decode(bufO.ctypes.data, n, r_ref, 0, None, 3), load(bufO, L_ref), reps)
assert q_ref == 0 and q_our == 0 and np.array_equal(bufR[:n], text) and np.array_equal(bufO[:n], text)
rows.append({"stage": "bsc_bwt_decode 64 MiB G_text", "ref_cuda_ms_best": rb, "ref_cuda_ms_median": rm, "ours_ms_best": ob, "ours_ms_median": om,
             "ours_kernels_only_ms": ours_kernel_ms("bwt_decode", L_ref, index=r_ref), "bit_identical": True})

# ---- forward ST (a8: bsc_st_encode_cuda, k = 5..8) on 32 MiB skew ----
n = skew.size
st_out = {}
for k in (5, 6, 7, 8):
    i_ref, rb, rm = timed(lambda: R.bsc_st_encode(bufR.ctypes.data, n, k, FEAT), load(bufR, skew), reps)
    i_our, ob, om = timed(lambda: L.bsc_st_encode(bufO.ctypes.data, n, k, 3), load(bufO, skew), reps)
    assert i_ref == i_our and np.array_equal(bufR[:n], bufO[:n]), "ST%d differs from the reference's CUDA path" % k
    st_out[k] = (i_our, bufO[:n].copy())
    rows.append({"stage": "bsc_st_encode k=%d 32 MiB G_skew" % k, "ref_cuda_ms_best": rb, "ref_cuda_ms_median": rm, "ours_ms_best": ob, "ours_ms_median": om,
                 "ours_kernels_only_ms": ours_kernel_ms("st_encode", skew, k=k, sorter=k), "bit_identical": True})

# ---- inverse ST: the reference has no GPU path (st.cpp:1491, CPU only) ----
i6, S6 = st_out[6]
q_ref, rb, rm = timed(lambda: R.bsc_st_decode(bufR.ctypes.data, n, 6, i6, FEAT), load(bufR, S6), 1)
q_our, ob, om = timed(lambda: L.bsc_st_decode(bufO.ctypes.data, n, 6, i6, 3), load(bufO, S6), reps)
assert q_ref == 0 and q_our == 0 and np.array_equal(bufR[:n], skew) and np.array_equal(bufO[:n], skew)
rows.append({"stage": "bsc_st_decode k=6 32 MiB G_skew (reference: CPU, OpenMP)", "ref_cuda_ms_best": rb, "ref_cuda_ms_median": rm, "ours_ms_best": ob, "ours_ms_median": om,
             "ours_kernels_only_ms": ours_kernel_ms("st_decode", S6, k=6, index=i6, sorter=6), "bit_identical": True})

for r in rows:
    r["speedup_best"] = round(r["ref_cuda_ms_best"] / r["ours_ms_best"], 2)
    sys.stderr.write("%-58s ref %9.1f ms   ours %9.1f ms (kernels %8.1f)   x%.2f\n" % (r["stage"], r["ref_cuda_ms_best"], r["ours_ms_best"], r["ours_kernels_only_ms"], r["speedup_best"]))
print(json.dumps({"what": "reference CUDA build (libcubwt 1.6.1 / st.cu, sm_90 SASS) vs libbsc_b200, host-pointer calls, wall clock incl. H2D/D2H", "reps": reps, "rows": rows}, indent=1))
