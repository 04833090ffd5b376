#!/usr/bin/env python3
"""bench.py -- compress+decompress throughput of the block-sorting hot path on an H100.

One "step" = one pass of the hot path over this rank's batch of synthetic blocks: every block is
compressed (adler32 -> forward BWT -> QLFC static coder -> framing) and then decompressed (QLFC
decode -> inverse BWT -> adler32 check), all on the GPU through the C ABI of libbsc_b200.so.
The K timed steps flow as one pipeline (class Pipeline): W blocks are in flight per GPU, each on its own
context / stream, so the HBM-bound sorts of some blocks overlap the latency-bound coder kernels of others.

  value : whole-job MB/s (10^6 uncompressed bytes per second of compress + decompress, CLI convention bsc.cpp:427) with the
          blocks already resident in HBM (bscb200_compress_device / bscb200_decompress_device), CUDA-event timed.
  e2e   : the same steps through the reference-facing host-pointer entry points bsc_compress /
          bsc_decompress, from pinned HOST buffers to pinned HOST buffers (H2D/D2H inside the timed region);
          e2e.pageable: one step of the same from ordinary (pageable) host memory.
  compress_MBps / decompress_MBps : each direction alone, one drained pass (extra keys).
  roofline / kernels : per-kernel CUDA-event durations captured during the timed steps.
  cpu_baseline / --impl reference : the UNMODIFIED reference (oracle/_ref) driven like its CLI
          (oracle/ref_driver.c) on the box's host cores.

Workload (BASELINE.json config C3, per GPU): G_text(seed 2 + rank), 64 blocks of 64 MiB per step, sorter BWT,
coder QLFC static, LZP off.  64 blocks = 512 coder streams, more than the encoder slots of an H100 (two to four CTAs per SM on 132 SMs).
Weak scaling: every rank processes its own 4 GiB per step.

--dump-outputs DIR writes what the timed steps' last step returned to its caller (see dump_outputs), so that two builds can be
compared output for output on identical seeded inputs.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import threading
import time
from concurrent.futures import ThreadPoolExecutor

# One hardware work queue per stream: with the default of 8, streams 9..16 alias onto the queues of
# streams 1..8 and a long-running coder kernel falsely serialises the other block (measured: 2x).
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

METRIC = "compress+decompress MB/s on 64 MB blocks"


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--blocks", type=int, default=64, help="blocks per GPU and step")
    ap.add_argument("--block-mib", type=int, default=64)
    ap.add_argument("--workers", type=int, default=0, help="blocks in flight per GPU = contexts = worker threads (0 = as many as the free HBM holds, at most 96 and at most the blocks of a step)")
    ap.add_argument("--sorter", type=int, default=1)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--ref-blocks", type=int, default=16, help="blocks per step of the reference arm / cpu_baseline leg (see reference_sample_blocks)")
    ap.add_argument("--mode", default="pipeline", choices=["phased", "pipeline"], help="order of the work inside the timed steps of the device-resident leg (see class Steps); the e2e leg always flows as a pipeline")
    ap.add_argument("--no-e2e", action="store_true")
    ap.add_argument("--e2e-steps", type=int, default=12, help="the end-to-end (host buffer) leg times min(--steps, this) steps, so that a long --steps run still ends within minutes")
    ap.add_argument("--no-extras", dest="extras", action="store_false", help="skip the extra keys for BASELINE configs C2 / C3-strong / C4 / C5")
    ap.add_argument("--dump-outputs", metavar="DIR", help="write the outputs of the last timed step to DIR/<name>.npy")
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0:
        ap.error("--steps must be >= 1 and --warmup >= 0")
    return args


# ------------------------------------------------------------------------------------------------
class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region, and the card's name and power limit (part of every number)."""
    Q = "index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"

    def __init__(self, index):
        self.index, self.proc, self.lines, self.card = index, None, [], {}

    def start(self):
        try:
            f = subprocess.run(["nvidia-smi", "-i", str(self.index), "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                               capture_output=True, text=True, timeout=30).stdout.strip().split(",")
            self.card = {"gpu": f[0].strip(), "power_limit_w": float(f[1])} if len(f) == 2 else {}
        except Exception:
            pass
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q, "--format=csv,noheader,nounits", "-lms", "200"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._pump, daemon=True).start()
        except Exception:
            self.proc = None

    def _pump(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc:
            self.proc.terminate()
            self.proc.wait()
        sm, mx, reasons = [], 0, set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 8:
                continue
            try:
                sm.append(float(f[1])); mx = max(mx, float(f[2]))
            except ValueError:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), f[4:8]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        return dict(self.card, sm_mhz=float(np.median(sm)) if sm else None, sm_max_mhz=mx or None, reasons=sorted(reasons), samples=len(sm))


def make_blocks(gen, seed, nblocks, block_bytes):
    data = gen.text(seed, nblocks * block_bytes)
    return [data[i * block_bytes:(i + 1) * block_bytes] for i in range(nblocks)]


# ------------------------------------------------------------------------------------------------
def run_reference(args, rank, world):
    """--impl reference: the unmodified reference on the host cores, CLI-style block loop."""
    from oracle import pyoracle
    if rank != 0:
        return
    sample = reference_sample_blocks(args, world)
    info = reference_timing(args, steps=args.steps, warmup=args.warmup, sample_blocks=sample)
    line = {"metric": METRIC, "value": info["value"], "unit": "MB/s", "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": info["ms_per_step"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8",
            "data": "synthetic", "impl": "reference",
            "config": workload_config(args), "arm": {"host_threads": info["cores"], "blocks_per_step": sample},
            "cpu_baseline": {"value": info["value"], "unit": "MB/s", "cores": info["cores"], "kind": info["kind"], "sample": info["sample"]},
            "e2e": {"value": info["value"], "unit": "MB/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "compress_MBps": info["compress_MBps"], "decompress_MBps": info["decompress_MBps"]}
    try:
        line["cpu_baseline"]["stages"] = reference_stage_seconds(args)
    except Exception as ex:                                  # the stage table is an extra: never lose the line over it
        line["cpu_baseline"]["stages"] = {"failed": repr(ex)[:200]}
    print(json.dumps(line), flush=True)


def reference_sample_blocks(args, world=1):
    """Blocks per step of the reference arm: a BOUNDED sample of the GPU arm's workload (same generator, block size, sorter, coder).
    16 blocks of 64 MiB = BASELINE C3's 1 GiB, one block per OpenMP thread as the reference CLI does (bsc.cpp:184-199).  More blocks at
    once do not make the memory-bound suffix sorting of the reference faster, and the bounded sample keeps the leg to minutes."""
    threads = len(os.sched_getaffinity(0))
    return max(1, min(world * args.blocks, threads, args.ref_blocks))


def reference_timing(args, steps, warmup, sample_blocks=None):
    from oracle import pyoracle
    gen = pyoracle.Gen()
    nb = sample_blocks or args.blocks
    bb = args.block_mib << 20
    blocks = make_blocks(gen, 2, nb, bb)
    drv_path = os.path.join(ROOT, "oracle", "_ref", "librefdrv.so")
    if os.path.exists(drv_path):
        return _reference_native(drv_path, blocks, steps, warmup, args.sorter)
    # no compiled reference on this machine: time the oracle port, one block per Python thread
    port = pyoracle.Port()
    t0 = time.perf_counter()
    outs = [port.compress(b, args.sorter, 1, 3) for b in blocks[:1]]
    t1 = time.perf_counter()
    _ = [port.decompress(o[1]) for o in outs]
    t2 = time.perf_counter()
    mb = bb / 1e6
    return {"value": mb / (t2 - t0), "ms_per_step": (t2 - t0) * 1e3, "cores": 1, "kind": "port", "sample": "1 block of %d MiB, single thread" % args.block_mib,
            "compress_MBps": mb / (t1 - t0), "decompress_MBps": mb / (t2 - t1)}


def _reference_native(drv_path, blocks, steps, warmup, sorter):
    vp, ci = ctypes.c_void_p, ctypes.c_int
    os.environ.pop("OMP_NUM_THREADS", None)                  # torchrun exports OMP_NUM_THREADS=1 to its ranks; the baseline uses the whole host
    d = ctypes.CDLL(drv_path)
    d.refdrv_init()
    d.refdrv_set_threads(len(os.sched_getaffinity(0)))
    d.refdrv_set_nested(1 if os.environ.get("BSCB200_REF_NESTED") == "1" else 0)   # stock CLI behaviour by default (see oracle/ref_driver.c)
    nb = len(blocks)
    PP = ctypes.c_void_p * nb
    II = ci * nb
    outs = [np.empty(b.size + 28 + 64, dtype=np.uint8) for b in blocks]
    backs = [np.empty(b.size + 64, dtype=np.uint8) for b in blocks]
    inp = PP(*[b.ctypes.data for b in blocks]); sizes = II(*[b.size for b in blocks])
    outp = PP(*[o.ctypes.data for o in outs]); outsz = II()
    backp = PP(*[o.ctypes.data for o in backs]); res = II()
    d.refdrv_compress.argtypes = [vp, vp, ci, vp, vp, ci, ci]
    d.refdrv_decompress.argtypes = [vp, vp, ci, vp, vp, vp]
    tc, td, T = [], [], 1
    for it in range(warmup + steps):
        t0 = time.perf_counter()
        T = d.refdrv_compress(inp, sizes, nb, outp, outsz, sorter, 1)
        t1 = time.perf_counter()
        d.refdrv_decompress(outp, outsz, nb, backp, sizes, res)
        t2 = time.perf_counter()
        assert all(r == 0 for r in res), "reference decompress failed"
        if it >= warmup:
            tc.append(t1 - t0); td.append(t2 - t1)
    for b, o in zip(blocks, backs):
        assert np.array_equal(b, o[:b.size])
    mb = sum(b.size for b in blocks) / 1e6
    c, dd = float(np.mean(tc)), float(np.mean(td))
    return {"value": mb / (c + dd), "ms_per_step": (c + dd) * 1e3, "cores": int(T), "kind": "reference",
            "sample": "%d blocks x %d MiB G_text, CLI block loop (bsc.cpp:184-199), %d OpenMP threads of %d host threads" % (nb, blocks[0].size >> 20, T, d.refdrv_max_threads()),
            "compress_MBps": mb / c, "decompress_MBps": mb / dd, "compressed_bytes": int(sum(outsz))}


def reference_stage_seconds(args):
    """Per-stage seconds of the reference on ONE block of the workload, one host thread (what each thread of its CLI block loop does when
    there are at least as many blocks as threads, bsc.cpp:188): bsc_bwt_encode, bsc_coder_compress, bsc_coder_decompress, bsc_bwt_decode.
    SURVEY 8(d) asks for them beside the MB/s.  Only with the compiled reference (oracle/_ref)."""
    from oracle import pyoracle
    if not pyoracle.ref_available() or args.sorter != 1:
        return None
    ref = pyoracle.Ref()
    ref.features = 1                                         # LIBBSC_FEATURE_FASTMODE, no intra-block OpenMP
    a = pyoracle.Gen().text(2, args.block_mib << 20)
    t0 = time.perf_counter()
    idx, L, _ = ref.bwt_encode(a, aux=False)
    t1 = time.perf_counter()
    c, stream = ref.coder_compress(L, 1, 1)
    t2 = time.perf_counter()
    n, L2 = ref.coder_decompress(stream, a.size, 1, 1)
    t3 = time.perf_counter()
    r, back = ref.bwt_decode(L2, idx)
    t4 = time.perf_counter()
    assert idx > 0 and c > 0 and n == a.size and r == 0 and np.array_equal(back, a), "reference stage round trip failed"
    return {"block": "1 x %d MiB G_text(2), one host thread" % args.block_mib, "bwt_encode_s": round(t1 - t0, 3), "coder_compress_s": round(t2 - t1, 3),
            "coder_decompress_s": round(t3 - t2, 3), "bwt_decode_s": round(t4 - t3, 3), "compressed_bytes": int(c)}


def workload_config(args, extra=None):
    c = {"workload": "C3: G_text(seed 2+rank) %d x %d MiB blocks per GPU, BWT + QLFC static, LZP off (-b%d -m0 -e1 -p)" % (args.blocks, args.block_mib, args.block_mib),
         "blocks_per_gpu": args.blocks, "block_bytes": args.block_mib << 20, "sorter": args.sorter, "coder": 1,
         "l2": "inputs_larger_than_L2 (%d MiB per step vs 50 MB L2)" % (args.blocks * args.block_mib)}
    if extra:
        c.update(extra)
    return c


def dump_outputs(out_dir, prefix, d_cmp, csize, d_back, bb, sample_bytes):
    """The arrays the last timed step handed back for every block: its compressed block (the bytes after the 4-byte alignment pad of the
    device buffer) and its restored bytes.  Whole outputs are pinned by their size and Adler-32; their bytes by a fixed, seeded sample of
    positions, the two float32 sample arrays together at most `sample_bytes`.  Float64 / float32 .npy files."""
    import zlib
    nb = len(d_cmp)
    k = max(1, min(65536, sample_bytes // (2 * 4 * nb)))
    rng = np.random.default_rng(20240601)
    pos_back = np.sort(rng.integers(0, bb, k))
    c_adler, c_sample, b_adler, b_sample = [], [], [], []
    for i in range(nb):
        c = d_cmp[i][4:4 + csize[i]].cpu().numpy()
        c_adler.append(zlib.adler32(c.tobytes()))
        c_sample.append(c[np.sort(rng.integers(0, c.size, k))])
        b = d_back[i][:bb].cpu().numpy()
        b_adler.append(zlib.adler32(b.tobytes()))
        b_sample.append(b[pos_back])
    os.makedirs(out_dir, exist_ok=True)
    for name, arr in (("compressed_sizes", np.array(csize, np.float64)), ("compressed_adler32", np.array(c_adler, np.float64)),
                      ("compressed_sample", np.array(c_sample, np.float32)), ("restored_adler32", np.array(b_adler, np.float64)),
                      ("restored_sample", np.array(b_sample, np.float32))):
        np.save(os.path.join(out_dir, prefix + name + ".npy"), arr)


# ------------------------------------------------------------------------------------------------
class Pipeline:
    """K steps of the batch as ONE continuous flow: W worker threads (one context / one stream / one pair of output buffers each) take
    (step, block) tasks in order and run task(worker, block) on each.  Blocks are at different stages at any moment, so the HBM-bound
    sorts of some overlap the latency-bound coder kernels of others, and the SM slots a short coder stream frees are taken by the
    next block's streams.  W (blocks in flight) is independent of the number of blocks per step."""

    def __init__(self, nb, workers, task, block_buffers=False, last_task=None):
        self.nb, self.workers, self.task = nb, workers, task
        self.last_task = last_task or task                          # runs the tasks of the last step of every run()
        # block_buffers: the task writes per-BLOCK buffers (extra_configs), so a block belongs to one task at a time (step s+1 may catch up with step s)
        self.block_lock = [threading.Lock() for _ in range(nb)] if block_buffers else None

    def run(self, steps):
        lock, nxt, errs = threading.Lock(), [0], []
        total = steps * self.nb

        def loop(w):
            try:
                while True:
                    with lock:
                        t = nxt[0]; nxt[0] += 1
                    if t >= total or errs:
                        return
                    task = self.last_task if t >= total - self.nb else self.task
                    if self.block_lock:
                        with self.block_lock[t % self.nb]:
                            task(w, t % self.nb)
                    else:
                        task(w, t % self.nb)
            except BaseException as ex:                              # surface the first failure, stop the others
                errs.append(ex)
        ths = [threading.Thread(target=loop, args=(w,)) for w in range(min(self.workers, total))]
        for t in ths:
            t.start()
        for t in ths:
            t.join()
        if errs:
            raise errs[0]


def extra_configs(args, rank, local_rank, world, L, gen, torch, dist, dev):
    """The other BASELINE.json configurations as extra keys of the same line (not the headline): C2 (100 MB text, 25 MB blocks, one GPU),
    C3 as written (1 GiB text = 16 blocks of 64 MiB shared by ALL ranks: strong scaling), C4 (stage-only bsc_bwt_decode of C3's blocks),
    C5 (256 MiB high-entropy binary, 32 MiB blocks, ST6, both directions).  Host-pointer entry points, pinned buffers, blocks b -> rank
    b mod world, device-timed max over ranks; one warm pass, then `reps` timed passes."""
    from libbsc_b200 import blocks as blk
    reps = 2

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    def timed_pass(nb, task):
        if nb == 0:
            barrier(); barrier()
            ms = 0.0
        else:
            pipe = Pipeline(nb, nb, task, block_buffers=True)
            pipe.run(1)
            barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); pipe.run(reps); torch.cuda.synchronize(); e1.record(); e1.synchronize()
            ms = e0.elapsed_time(e1) / reps
            barrier()
        if dist is not None:
            t = torch.tensor([ms], device=dev, dtype=torch.float64); dist.all_reduce(t, op=dist.ReduceOp.MAX); ms = float(t[0])
        return ms

    def round_trip(data, bb, sorter, ranks):
        """compress+decompress of data cut into blocks of bb bytes, block b on rank b mod ranks (ranks beyond `ranks` idle)"""
        parts = blk.split_blocks(data.size, bb)                      # CLI-style cut (bsc.cpp:163-178)
        nblk = len(parts)
        mine = blk.assign(nblk, ranks, rank) if rank < ranks else []  # block b -> rank b mod N
        h_in = [torch.from_numpy(data[parts[b][0]:parts[b][0] + parts[b][1]]).pin_memory() for b in mine]
        h_cmp = [torch.empty(t.numel() + 28 + 64, dtype=torch.uint8).pin_memory() for t in h_in]
        h_back = [torch.zeros(t.numel() + 64, dtype=torch.uint8).pin_memory() for t in h_in]
        hsize = [0] * len(mine)

        def comp(w, i):
            torch.cuda.set_device(local_rank)
            r = L.bsc_compress(h_in[i].data_ptr(), h_cmp[i].data_ptr(), h_in[i].numel(), 0, 0, sorter, 1, 3)
            assert r > 0, r
            hsize[i] = r

        def decomp(w, i):
            torch.cuda.set_device(local_rank)
            assert L.bsc_decompress(h_cmp[i].data_ptr(), hsize[i], h_back[i].data_ptr(), h_in[i].numel(), 3) == 0

        def both(w, i):
            comp(w, i); decomp(w, i)
        ms_b = timed_pass(len(mine), both)
        ms_c = timed_pass(len(mine), comp)
        ms_d = timed_pass(len(mine), decomp)
        for a, b in zip(h_in, h_back):
            assert torch.equal(a, b[:a.numel()]), "extra config: round trip mismatch"
        mb = data.size / 1e6
        sizes = blk.gather_sizes(dist, mine, hsize, nblk, device=dev)  # what the file container needs: every block's compressed size, on every rank
        return {"value": mb / (ms_b / 1e3), "unit": "MB/s", "compress_MBps": mb / (ms_c / 1e3), "decompress_MBps": mb / (ms_d / 1e3), "blocks": nblk,
                "block_bytes": bb, "gpus": min(ranks, world), "compressed_bytes": int(sum(sizes))}, (mine, h_in)

    out = {}
    text = gen.text(2, 1 << 30)
    c2, _ = round_trip(text[:104857600], 26214400, 1, 1)
    out["C2_text_100MB_b25_1gpu"] = dict(c2, workload="G_text(2) first 104857600 bytes, 4 blocks of 26214400, BWT + QLFC static, one GPU, host buffers")
    c3, (mine, h_in) = round_trip(text, 64 << 20, 1, world)
    out["C3_text_1GiB_b64_strong"] = dict(c3, workload="G_text(2, 1 GiB) = 16 blocks of 64 MiB over all %d GPU(s) (block b -> rank b mod N): STRONG scaling, host buffers" % world, scaling="strong")
    # C4: the inverse-BWT stage alone on the L of every C3 block (bsc_bwt_decode, host pointers)
    Ls, idx = [], []
    for t in h_in:
        buf = t.clone().pin_memory()
        r = L.bsc_bwt_encode(buf.data_ptr(), buf.numel(), None, None, 3)
        assert r > 0
        Ls.append(buf); idx.append(r)
    work = [t.clone().pin_memory() for t in Ls]

    def unbwt(w, i):
        torch.cuda.set_device(local_rank)
        work[i].copy_(Ls[i])
        assert L.bsc_bwt_decode(work[i].data_ptr(), work[i].numel(), idx[i], 0, None, 3) == 0
    ms = timed_pass(len(mine), unbwt)
    for a, b in zip(h_in, work):
        assert torch.equal(a, b)
    out["C4_bwt_decode_stage_b64"] = {"value": text.size / 1e6 / (ms / 1e3), "unit": "MB/s", "blocks": 16, "gpus": world,
                                      "workload": "bsc_bwt_decode alone on the BWT of each C3 block, host buffers (H2D + kernels + D2H + one host memcpy per block inside the time)"}
    del text, Ls, work, h_in
    skew = gen.skew(3, 256 << 20)
    c5, _ = round_trip(skew, 32 << 20, 6, world)
    out["C5_skew_256MiB_b32_st6"] = dict(c5, workload="G_skew(3, 256 MiB) = 8 blocks of 32 MiB over %d GPU(s), ST6 + QLFC static (-m6), both directions, host buffers" % world, scaling="strong")
    return out


def run_b200(args, rank, local_rank, world):
    import torch
    import libbsc_b200
    from oracle import pyoracle            # generators only (tools/libbscgen.so) + the cpu_baseline leg

    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    L = libbsc_b200.lib()
    assert L.bsc_init(3) == 0, "no usable CUDA device (libbsc_b200 has no CPU path)"

    gen = pyoracle.Gen()
    nb, bb = args.blocks, args.block_mib << 20
    host_blocks = make_blocks(gen, 2 + rank, nb, bb)

    # ---- device-resident leg ------------------------------------------------------------------
    # inputs per block; compressed / restored buffers per WORKER (a task = compress block i, then decompress it, on one context),
    # plus one compressed buffer per block for the passes that run each direction alone
    d_in = [torch.from_numpy(b).to(dev) for b in host_blocks]
    d_cmp_blk = [torch.empty(bb + 28 + 64, dtype=torch.uint8, device=dev) for _ in range(nb)]
    # --dump-outputs: the last timed step restores every block into a buffer of its own, kept for dump_outputs
    d_back_blk = [torch.empty(bb + 64, dtype=torch.uint8, device=dev) for _ in range(nb)] if args.dump_outputs else None
    ws = int(L.bscb200_workspace_bytes(bb, args.sorter))
    # blocks in flight = contexts = worker threads, independent of the blocks per step.  Up to 96 (enough to keep five decoder streams per
    # SM busy at eight streams per block), as many as the free HBM holds beside the library's six shared sort slabs and 5 % headroom
    per_worker = ws + 2 * (bb + 128)
    room = int(L.bscb200_device_free_bytes()) - 6 * int(L.bscb200_scratch_bytes(bb, args.sorter))
    workers = args.workers if args.workers > 0 else max(1, min(96 if nb >= 64 else nb, int(room * 0.95) // per_worker))
    d_cmp = [torch.empty(bb + 28 + 64, dtype=torch.uint8, device=dev) for _ in range(workers)]
    d_back = [torch.empty(bb + 64, dtype=torch.uint8, device=dev) for _ in range(workers)]
    ctxs = [libbsc_b200.DeviceCtx(local_rank) for _ in range(workers)]
    for c in ctxs:
        assert c.reserve(ws) == 0, "workspace allocation failed"
    csize = [0] * nb
    last = [-1] * workers                                # block whose restored bytes sit in d_back[w]

    def dev_compress(w, i, dst=None):
        # +4: payload (offset 28) 16-byte aligned for the vectorised device adler32
        r = ctxs[w].compress(d_in[i].data_ptr(), (d_cmp[w] if dst is None else dst).data_ptr() + 4, bb, args.sorter, 1, 3)
        assert r > 0, "compress failed: %d" % r
        csize[i] = r

    def dev_decompress(w, i, src=None, dst=None):
        r = ctxs[w].decompress((d_cmp[w] if src is None else src).data_ptr() + 4, csize[i], (d_back[w] if dst is None else dst).data_ptr(), bb, 3)
        assert r == 0, "decompress failed: %d" % r
        if dst is None:
            last[w] = i

    def dev_task(w, i):
        torch.cuda.set_device(local_rank)
        dev_compress(w, i); dev_decompress(w, i)

    def dev_task_kept(w, i):                             # the same work, results left in the block's own buffers (--dump-outputs)
        torch.cuda.set_device(local_rank)
        dev_compress(w, i, d_cmp_blk[i]); dev_decompress(w, i, d_cmp_blk[i], d_back_blk[i])

    def dev_decompress_kept(w, i):
        dev_decompress(w, i, d_cmp_blk[i], d_back_blk[i])

    def dev_compress_blk(w, i):
        dev_compress(w, i, d_cmp_blk[i])

    def dev_decompress_blk(w, i):
        dev_decompress(w, i, d_cmp_blk[i])

    def dev_verify_blk(w, i):                            # every block restored once more and compared (outside every timed region)
        dev_decompress(w, i, d_cmp_blk[i])
        assert torch.equal(d_back[w][:bb], d_in[i]), "round trip mismatch in block %d" % i

    def barrier():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(fn):
        """device time of fn() between two events on the current stream, all streams drained on both sides"""
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        torch.cuda.synchronize()
        e1.record(); e1.synchronize()
        return e0.elapsed_time(e1)

    def phase(fn):
        return lambda w, i: (torch.cuda.set_device(local_rank), fn(w, i))

    class Steps:
        """--mode pipeline: compress -> decompress per block, all blocks and steps as one flow.  --mode phased: per step every block is
        compressed, then every block is decompressed (the sorts of the compress phase find the SMs free of coder CTAs)."""
        def __init__(self, task, comp, decomp, task_kept=None, decomp_kept=None):
            self.flow, self.comp, self.decomp = Pipeline(nb, workers, task, last_task=task_kept), Pipeline(nb, workers, phase(comp)), Pipeline(nb, workers, phase(decomp))
            self.decomp_last = Pipeline(nb, workers, phase(decomp_kept or decomp))

        def run(self, steps):
            if args.mode == "pipeline":
                self.flow.run(steps)
            else:
                for s in range(steps):
                    self.comp.run(1); (self.decomp_last if s == steps - 1 else self.decomp).run(1)

    pipe = Steps(dev_task, dev_compress_blk, dev_decompress_blk)
    pipe.run(args.warmup)
    if args.dump_outputs:
        pipe = Steps(dev_task, dev_compress_blk, dev_decompress_blk, dev_task_kept, dev_decompress_kept)
    for c in ctxs:
        c.set_profile(True)
    launches0 = sum(c.launches() for c in ctxs)
    sampler = ClockSampler(local_rank); sampler.start()
    barrier()
    ms_total = timed(lambda: pipe.run(args.steps))
    barrier()
    clocks = sampler.stop()
    launches = sum(c.launches() for c in ctxs) - launches0
    for w in range(workers):                             # what the timed steps left behind: each worker's last block
        assert last[w] < 0 or torch.equal(d_back[w][:bb], d_in[last[w]]), "round trip mismatch in block %d" % last[w]
    if args.dump_outputs:
        for i in range(nb):                              # the blocks of the last step were restored into buffers of their own
            assert torch.equal(d_back_blk[i][:bb], d_in[i]), "round trip mismatch in block %d" % i
        # 60 * 10^6 bytes of samples over all ranks: with the sizes and checksums the files stay within 64 MB in all
        dump_outputs(args.dump_outputs, "" if world == 1 else "rank%d_" % rank, d_cmp_blk, csize, d_back_blk, bb, 60 * 10**6 // world)
        del d_back_blk
    # per-kernel CUDA-event timings gathered during the timed steps
    kern = {}
    for c in ctxs:
        for name, (cnt, ms, by) in c.profile_report().items():
            a = kern.setdefault(name, [0, 0.0, 0.0]); a[0] += cnt; a[1] += ms; a[2] += by
        c.set_profile(False)

    # phase-separated pass (extra keys): all blocks compressed, drain, all blocks decompressed -- what each direction does alone
    ms_c = timed(lambda: Pipeline(nb, workers, phase(dev_compress_blk)).run(1))
    ms_d = timed(lambda: Pipeline(nb, workers, phase(dev_decompress_blk)).run(1))
    Pipeline(nb, workers, phase(dev_verify_blk)).run(1)

    # standalone pass: ONE block at a time on one stream, so that the per-launch durations of the
    # bandwidth-bound kernels are not stretched by the other blocks sharing HBM (roofline leg)
    alone = {}
    ctxs[0].set_profile(True)
    for i in range(min(2, nb)):
        csz_i = ctxs[0].compress(d_in[i].data_ptr(), d_cmp[0].data_ptr() + 4, bb, args.sorter, 1, 3)
        assert csz_i == csize[i]
        assert ctxs[0].decompress(d_cmp[0].data_ptr() + 4, csz_i, d_back[0].data_ptr(), bb, 3) == 0
    for name, (cnt, ms, by) in ctxs[0].profile_report().items():
        alone[name] = [cnt, ms, by]
    ctxs[0].set_profile(False)

    ms_step = ms_total / args.steps
    if dist is not None:
        t = torch.tensor([ms_step, ms_c, ms_d], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms_step, ms_c, ms_d = float(t[0]), float(t[1]), float(t[2])
    total_mb = world * nb * bb / 1e6
    value = total_mb / (ms_step / 1e3)

    # ---- end-to-end leg: HOST buffers through bsc_compress / bsc_decompress (H2D / D2H of every block inside the timed region) ----
    e2e = None
    comp_bytes = int(sum(csize))
    if not args.no_e2e:
        for c in ctxs:
            c.close()
        del d_cmp, d_back, d_in, d_cmp_blk
        torch.cuda.empty_cache()

        pin_failed = []

        def host_leg(pinned, steps, warm):
            def mk(t):
                if not pinned or pin_failed:
                    return t
                try:
                    return t.pin_memory()
                except RuntimeError as ex:                   # the host refused to lock more pages (many ranks per host): carry on pageable, say so
                    pin_failed.append(repr(ex)[:120])
                    return t
            h_in = [mk(torch.from_numpy(b)) for b in host_blocks]
            h_cmp = [mk(torch.empty(bb + 28 + 64, dtype=torch.uint8)) for _ in range(workers)]      # per worker, as in the device leg
            h_back = [mk(torch.zeros(bb + 64, dtype=torch.uint8)) for _ in range(workers)]
            hsize, hlast = [0] * nb, [-1] * workers

            def host_task(w, i):
                torch.cuda.set_device(local_rank)
                r = L.bsc_compress(h_in[i].data_ptr(), h_cmp[w].data_ptr(), bb, 0, 0, args.sorter, 1, 3)
                assert r > 0, "bsc_compress failed: %d" % r
                hsize[i] = r
                r = L.bsc_decompress(h_cmp[w].data_ptr(), hsize[i], h_back[w].data_ptr(), bb, 3)
                assert r == 0, "bsc_decompress failed: %d" % r
                hlast[w] = i
            hp = Pipeline(nb, workers, host_task)
            if warm:
                hp.run(warm)
            l0 = int(L.bscb200_total_kernel_launches())
            barrier()
            ms = timed(lambda: hp.run(steps)) / steps
            barrier()
            nl = int(L.bscb200_total_kernel_launches()) - l0
            for w in range(workers):
                assert hlast[w] < 0 or torch.equal(h_back[w][:bb], h_in[hlast[w]]), "e2e round trip mismatch in block %d" % hlast[w]
            return ms, nl, int(sum(hsize))

        e2e_steps = max(1, min(args.steps, args.e2e_steps))
        ms_e, nl, hbytes = host_leg(True, e2e_steps, max(1, min(args.warmup, 3) - 1))
        launches += nl
        ms_p, _, _ = host_leg(False, 1, 1)               # the C API takes any host pointer: the same call from PAGEABLE memory, one step
        if dist is not None:
            t = torch.tensor([ms_e, ms_p], device=dev, dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms_e, ms_p = float(t[0]), float(t[1])
        e2e = {"value": total_mb / (ms_e / 1e3), "unit": "MB/s", "h2d_bytes_per_step": nb * bb + hbytes, "d2h_bytes_per_step": hbytes + nb * bb,
               "ms_per_step": ms_e, "steps": e2e_steps, "host_memory": "pinned" if not pin_failed else "pageable for some buffers (pinning failed: %s)" % pin_failed[0],
               "pageable": {"value": total_mb / (ms_p / 1e3), "unit": "MB/s", "steps": 1}}

    extras = None
    if args.extras:
        torch.cuda.empty_cache()
        extras = extra_configs(args, rank, local_rank, world, L, gen, torch, dist, dev)

    if rank != 0:
        return

    # ---- roofline of the dominant kernel + per-kernel table ------------------------------------
    # HBM GB/s of NVIDIA's data sheets, by the name the card reports (the SXM card reports "H100 80GB HBM3"): a bound, never a measurement
    card = torch.cuda.get_device_name(dev)
    peak, model = next(((v, m) for m, v in (("H100 NVL", 3900.0), ("H100 PCIe", 2000.0), ("H100", 3350.0)) if m in card), (3350.0, None))
    peak_src = ("%s data sheet, %.0f GB/s" % (model if model != "H100" else "H100 SXM", peak)) if model else \
               "%s is not an H100: the H100 SXM data sheet's 3350 GB/s is used, the fractions do not describe this card" % card
    tot_ms = sum(v[1] for v in kern.values()) or 1.0
    table = []
    for name, (cnt, ms, by) in sorted(kern.items(), key=lambda kv: -kv[1][1]):
        row = {"kernel": name, "launches": cnt, "ms_total": round(ms, 3), "share": round(ms / tot_ms, 4)}
        if by > 0:
            row["algorithmic_GBps"] = round(by / 1e9 / (ms / 1e3), 2); row["frac_of_peak"] = round(by / 1e9 / (ms / 1e3) / peak, 5)
        table.append(row)
    dom = table[0] if table else {"kernel": None}
    dom_bytes = kern[dom["kernel"]][2] if table else 0
    dom_ms = kern[dom["kernel"]][1] if table else 1
    dom_cnt = kern[dom["kernel"]][0] if table else 1
    achieved = dom_bytes / 1e9 / (dom_ms / 1e3) if dom_bytes else 0.0
    roofline = {"kernel": dom["kernel"], "bound": "hbm", "achieved": round(achieved, 3), "peak": peak, "unit": "GB/s", "frac": round(achieved / peak, 6),
                "peak_source": peak_src,
                "bytes_per_launch": dom_bytes / max(dom_cnt, 1), "avg_launch_ms": dom_ms / max(dom_cnt, 1), "share_of_kernel_time": dom.get("share"),
                "note": "the dominant kernel is a serial recurrence per stream (<= 8 streams per block by the format): it is bound by what one warp can "
                        "issue, not by HBM; launch durations of concurrent streams overlap, shares are of summed kernel time"}
    # HBM-bound kernels, timed alone: achieved algorithmic GB/s against the data-sheet HBM bandwidth
    alone_table = []
    for name, (cnt, ms, by) in sorted(alone.items(), key=lambda kv: -kv[1][1]):
        row = {"kernel": name, "launches": cnt, "ms_total": round(ms, 3)}
        if by > 0 and ms > 0:
            row["algorithmic_GBps"] = round(by / 1e9 / (ms / 1e3), 1); row["frac_of_peak"] = round(by / 1e9 / (ms / 1e3) / peak, 4)
        alone_table.append(row)
    hbm_rows = [r for r in alone_table if r["kernel"] in ("rs_onesweep", "unbwt_lf", "rs_hist1", "adler_partial") and "algorithmic_GBps" in r]
    roofline_hbm = None
    if hbm_rows:
        r0 = hbm_rows[0]; cnt0, ms0, by0 = alone[r0["kernel"]]
        roofline_hbm = {"kernel": r0["kernel"], "bound": "hbm", "achieved": r0["algorithmic_GBps"], "peak": peak, "unit": "GB/s", "frac": r0["frac_of_peak"],
                        "bytes_per_launch": by0 / max(cnt0, 1), "avg_launch_ms": ms0 / max(cnt0, 1),
                        "how": "CUDA events around every launch, one block at a time on one stream (2 blocks), after the timed steps"}

    cpu = None
    if not args.no_cpu_baseline and world == 1:
        try:
            info = reference_timing(args, steps=1, warmup=0, sample_blocks=reference_sample_blocks(args))
            cpu = {"value": info["value"], "unit": "MB/s", "cores": info["cores"], "kind": info["kind"], "sample": info["sample"],
                   "compress_MBps": info["compress_MBps"], "decompress_MBps": info["decompress_MBps"]}
        except Exception as ex:      # never lose the GPU line because the baseline leg failed
            cpu = {"value": None, "unit": "MB/s", "cores": 0, "kind": "reference", "sample": "failed: %r" % (ex,)}
        try:
            cpu["stages"] = reference_stage_seconds(args)
        except Exception as ex:
            cpu["stages"] = {"failed": repr(ex)[:200]}

    line = {"metric": METRIC, "value": value, "unit": "MB/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
            # `config` is the workload and identical in both arms; what is specific to this arm sits in `arm`
            "config": workload_config(args),
            "arm": {"blocks_in_flight_per_gpu": workers, "mode": args.mode, "step": "phased: all blocks compressed, then all blocks decompressed; pipeline: compress -> decompress per block, "
                                                                                   "steps flow into each other; timed barrier to barrier",
                    "parallelism": "blocks round-robin over %d GPU(s), no collective" % world},
            "compress_MBps": total_mb / (ms_c / 1e3), "decompress_MBps": total_mb / (ms_d / 1e3), "phase_note": "each direction alone, one drained pass over the batch",
            "compressed_bytes_rank0": comp_bytes, "ratio": comp_bytes / float(nb * bb),
            "e2e": e2e, "gpu_launches": int(launches), "clocks": clocks, "roofline": roofline, "roofline_hbm_kernel": roofline_hbm,
            "other_configs": extras, "kernels": table, "kernels_standalone": alone_table, "cpu_baseline": cpu}
    print(json.dumps(line), flush=True)


def main():
    args = parse_args()
    rank = int(os.environ.get("RANK", "0")); world = int(os.environ.get("WORLD_SIZE", "1")); local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if args.impl == "reference":
        run_reference(args, rank, world)
    else:
        run_b200(args, rank, local_rank, world)


if __name__ == "__main__":
    main()
