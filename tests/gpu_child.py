"""One configuration of tests/test_gpu_pipeline.py, tests/test_gpu_large_paths.py or tests/test_gpu_malformed.py, run in a process of
its own: the library reads each BSCB200_* switch once per process, so every setting needs a fresh one.

    python tests/gpu_child.py <job dir>

The job dir holds jobs.json (written by the test) and the inputs it names under in/.  This script only runs the GPU: it writes every
output to out/<the job's file id>.npy and the return codes, secondary indexes and profile to results.json; the test compares them with the reference.
Before each job of a serial run it prints "[job] <name>" to stderr, so that the test can tell which [qstats ...] lines belong to which
job."""
import hashlib
import json
import os
import random
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import libbsc_b200  # noqa: E402


class Runner:
    def __init__(self, jobdir, spec):
        self.dir = jobdir
        self.spec = spec
        self.bsc = libbsc_b200.Bsc(features=3)
        self.L = self.bsc.lib
        self.results = {}
        self.lock = threading.Lock()
        self._gen = None
        self._torch = None

    # ---- inputs ---------------------------------------------------------------------------------------------------------------
    def data(self, job):
        if "in" in job:
            return np.load(os.path.join(self.dir, "in", job["in"]))
        kind, seed, n = job["gen"]
        if kind == "degenerate":
            import reference_inputs as ri
            return ri.degenerate_inputs()[seed]
        if self._gen is None:
            from oracle import pyoracle
            self._gen = pyoracle.Gen()
        return getattr(self._gen, kind)(seed, n)

    @property
    def torch(self):
        if self._torch is None:
            import torch
            self._torch = torch
        return self._torch

    def save(self, job, r, out=None, suffix="", **extra):
        """the job's return code (and secondary indexes, profile) under its name; its output in out/<the job's file id>.npy"""
        rec = dict(r=int(r), **extra)
        if out is not None:
            np.save(os.path.join(self.dir, "out", job["out"] + suffix + ".npy"), np.ascontiguousarray(out, dtype=np.uint8))
        with self.lock:
            self.results[job["name"] + suffix] = rec

    # ---- operations -----------------------------------------------------------------------------------------------------------
    def run(self, job):
        op, a = job["op"], self.data(job)
        args = job.get("args", {})
        b = self.bsc
        if op == "decode_block":
            r, out = b.decode_block(a, args["n"])
            self.save(job, r, out)
        elif op == "coder_decompress":
            r, out = b.coder_decompress(a, args["n"], 1, args.get("features", 3))
            self.save(job, r, out)
        elif op == "decompress":
            r, out = b.decompress(a, args.get("features", 3))
            self.save(job, r, out)
        elif op == "coder_compress":
            r, out = b.coder_compress(a, 1, args["features"])
            self.save(job, r, out)
        elif op == "encode_block":
            r, out = b.encode_block(a, args.get("cap"))
            self.save(job, r, out if r > 0 else None)
        elif op == "compress":
            lzp = args.get("lzp", (0, 0))
            if args.get("inplace"):
                n = a.size
                buf = np.zeros(n + 28 + 64, dtype=np.uint8)
                buf[:n] = a
                r = self.L.bsc_compress(buf.ctypes.data, buf.ctypes.data, n, lzp[0], lzp[1], args["sorter"], args["coder"], args["features"])
                out = buf[:r] if r > 0 else buf                 # on failure the whole buffer: the call must leave it as it was
            else:
                r, out = b.compress(a, args["sorter"], args["coder"], args["features"], lzp[0], lzp[1])
            self.save(job, r, out)
        elif op == "raw_decompress":                        # bsc_decompress into n + 64 bytes of 0xA5, all of which come back
            n = args["n"]
            buf = np.full(n + 64, 0xA5, dtype=np.uint8)
            r = self.L.bsc_decompress(a.ctypes.data, a.size, buf.ctypes.data, n, args.get("features", 3))
            self.save(job, r, buf)
        elif op == "inplace_decompress":                    # bsc_decompress(buf, size, buf, n) on one buffer, as the reference's CLI calls it
            n = args["n"]
            buf = np.zeros(max(n, a.size) + 64, dtype=np.uint8)
            buf[:a.size] = a
            r = self.L.bsc_decompress(buf.ctypes.data, a.size, buf.ctypes.data, n, args.get("features", 3))
            self.save(job, r, buf[:n] if r == 0 else None)
        elif op == "guarded_decompress":                    # bsc_decompress out of place and in place, with explicit sizes; both buffers whole
            n, size = args["n"], args["in_size"]
            buf = np.full(n + 64, 0xA5, dtype=np.uint8)
            r = self.L.bsc_decompress(a.ctypes.data, size, buf.ctypes.data, n, args.get("features", 3))
            self.save(job, r, buf)
            buf = np.full(max(n, a.size) + 64, 0xA5, dtype=np.uint8)
            buf[:a.size] = a
            r = self.L.bsc_decompress(buf.ctypes.data, size, buf.ctypes.data, n, args.get("features", 3))
            self.save(job, r, buf, suffix=".inplace")
        elif op == "device_guarded":
            self.device_guarded(job, a, args)
        elif op == "free_hbm":                              # free HBM once the pooled contexts and sort slabs are released
            self.L.bscb200_release_pools()
            self.save(job, 0, free=int(self.L.bscb200_device_free_bytes()))
        elif op == "compress_and_decompress":               # a block too large for a CPU reference: its known answer, then the round trip
            r, blk = b.compress(a, 1, 1, 3)
            self.save(job, r, blk)
            q, out = b.decompress(blk)
            self.save(job, q, out, suffix=".dec")
        elif op == "bwt_encode":
            r, L, aux = b.bwt_encode(a)
            self.save(job, r, L, aux=[int(x) for x in aux])
        elif op == "st_encode":
            r, L = b.st_encode(a, args["k"])
            self.save(job, r, L)
        elif op == "st_decode":
            r, T = b.st_decode(a, args["k"], args["index"])
            self.save(job, r, T)
        elif op == "bwt_batched":                           # the batched forward BWT of a device context with a tiny sort budget
            torch = self.torch
            ctx = libbsc_b200.DeviceCtx(0)
            assert ctx.set_sort_budget(args["budget"]) == 0
            t = torch.from_numpy(a).cuda()
            torch.cuda.synchronize()
            r, aux = ctx.bwt_encode(t.data_ptr(), a.size)
            self.save(job, r, t.cpu().numpy(), aux=[int(x) for x in aux])
            ctx.close()
        elif op == "bwt_profiled":                          # forward BWT on a profiling device context: which sort kernels ran
            torch = self.torch
            ctx = libbsc_b200.DeviceCtx(0)
            ctx.set_profile(True)
            t = torch.from_numpy(a).cuda()
            torch.cuda.synchronize()
            r, aux = ctx.bwt_encode(t.data_ptr(), a.size)
            prof = {k: v[0] for k, v in ctx.profile_report().items()}
            self.save(job, r, t.cpu().numpy(), aux=[int(x) for x in aux], profile=prof)
            ctx.close()
        else:
            raise ValueError(op)

    GUARD = 4096

    def guarded(self, size, fill):
        """a device buffer of exactly `size` bytes (filled with `fill`, an array or a byte) at GUARD + off bytes into a tensor whose other
        bytes hold a known pattern; returns (tensor, start) for offset `off` set by the caller through self._off"""
        torch = self.torch
        G, off = self.GUARD, self._off
        t = (torch.arange(2 * G + off + size, dtype=torch.int32, device="cuda") * 167 + 13).to(torch.uint8)
        if isinstance(fill, np.ndarray):
            t[G + off:G + off + size] = torch.from_numpy(np.ascontiguousarray(fill[:size])).cuda()
        else:
            t[G + off:G + off + size] = fill
        return t, G + off

    def guards_intact(self, t, start, size):
        want = (self.torch.arange(t.numel(), dtype=self.torch.int32, device="cuda") * 167 + 13).to(self.torch.uint8)
        return bool(self.torch.equal(t[:start], want[:start]) and self.torch.equal(t[start + size:], want[start + size:]))

    def device_guarded(self, job, a, args):
        """One device-resident entry point on caller buffers of exactly the documented size, at byte offsets 0, 1 and 7 from a 256-byte
        boundary, each between 4 KiB guards of a known pattern.  Saves the return code and output at offset 0, whether the other offsets
        gave the same, whether every guard is intact and, for the two decoders, what the host-pointer entry point returns."""
        torch = self.torch
        if not hasattr(self, "_ctx"):
            self._ctx = libbsc_b200.DeviceCtx(0)
        ctx, call = self._ctx, args["call"]
        runs = []
        for off in (0, 1, 7):
            self._off = off
            aux = None
            if call in ("decompress", "coder_decompress"):
                in_size, cap = args["in_size"], args["out_size"]
                ti, si = self.guarded(in_size, a)
                to_, so = self.guarded(cap, 0xA5)
                torch.cuda.synchronize()
                if call == "decompress":
                    r = ctx.decompress(ti.data_ptr() + si, in_size, to_.data_ptr() + so, cap, 3)
                else:
                    r = ctx.coder_decompress(ti.data_ptr() + si, in_size, to_.data_ptr() + so, cap, args["coder"], 3)
                torch.cuda.synchronize()
                ok = self.guards_intact(ti, si, in_size) and self.guards_intact(to_, so, cap) and torch.equal(ti[si:si + in_size].cpu(), torch.from_numpy(a[:in_size]))
                out = to_[so:so + cap].cpu().numpy()
            elif call == "coder_compress":
                n = a.size
                ti, si = self.guarded(n, a)
                to_, so = self.guarded(n + 4096, 0xA5)
                torch.cuda.synchronize()
                r = ctx.coder_compress(ti.data_ptr() + si, to_.data_ptr() + so, n, args["coder"], 3)
                torch.cuda.synchronize()
                ok = self.guards_intact(ti, si, n) and self.guards_intact(to_, so, n + 4096)
                out = to_[so:so + max(r, 0)].cpu().numpy()
            else:                                           # in place on d_T: bwt / st encode / decode, adler32
                n = a.size
                t, s = self.guarded(n, a)
                torch.cuda.synchronize()
                p = t.data_ptr() + s
                if call == "bwt_encode":
                    r, aux = ctx.bwt_encode(p, n)
                elif call == "bwt_decode":
                    r = ctx.bwt_decode(p, n, args["index"])
                elif call == "st_encode":
                    r = ctx.st_encode(p, n, args["k"])
                elif call == "st_decode":
                    r = ctx.st_decode(p, n, args["k"], args["index"])
                else:
                    r = ctx.adler32(p, n)
                torch.cuda.synchronize()
                ok = self.guards_intact(t, s, n)
                out = t[s:s + n].cpu().numpy()
            runs.append((int(r), out, ok, aux))
        r0, out0, _, aux0 = runs[0]
        # the output of a failed call is the entry point's working space, not a result: only codes are compared then
        same = all(r == r0 and x == aux0 and (r0 < 0 or np.array_equal(o, out0)) for r, o, _, x in runs[1:])
        extra = dict(guards=[ok for _, _, ok, _ in runs], offsets_agree=same, codes=[r for r, _, _, _ in runs], aux=aux0)
        if call in ("decompress", "coder_decompress"):       # the host entry point's code, and its output where it succeeds
            buf = np.empty(args["out_size"] + 64, dtype=np.uint8)
            if call == "decompress":
                h = int(self.L.bsc_decompress(a.ctypes.data, args["in_size"], buf.ctypes.data, args["out_size"], 3))
                size = args["out_size"] if h == 0 else -1
            else:
                h = int(self.L.bscb200_coder_decompress(a.ctypes.data, args["in_size"], buf.ctypes.data, args["out_size"], args["coder"], 3))
                size = h
            extra.update(host=h, host_sha=hashlib.sha256(buf[:size].tobytes()).hexdigest() if size >= 0 else None)
        self.save(job, r0, out0, **extra)

    # ---- modes ----------------------------------------------------------------------------------------------------------------
    def serial(self):
        for job in self.spec["jobs"]:
            sys.stderr.write("[job] %s\n" % job["name"])
            sys.stderr.flush()
            self.run(job)
            sys.stderr.flush()

    def pipeline(self):
        """T host threads start together and share one shuffled job list, as bench.py and the CLI keep many blocks in flight."""
        L = self.L
        sms = self.torch.cuda.get_device_properties(0).multi_processor_count
        biggest = self.spec["max_n"]
        per_thread = L.bscb200_workspace_bytes(biggest, 1)
        slabs = 6 * max(L.bscb200_scratch_bytes(biggest, 1), L.bscb200_scratch_bytes(self.spec["max_st_n"], 6))
        free = L.bscb200_device_free_bytes()
        threads = max(1, min(sms // 8 + 8, (free - slabs) // per_thread))
        # The list, shuffled with a seed: first the coder-only jobs on large blocks, so that every thread starts in a coder stage, then
        # the rest with the decode group spread evenly over it.  The group decodes while the coder stages of the device are loaded.
        rng = random.Random(self.spec["seed"])
        lead, rest, group = ([j for j in self.spec["jobs"] if j["args"].get("role") == role] for role in ("lead", None, "group"))
        rng.shuffle(lead)
        rng.shuffle(rest)
        step = max(1, len(rest) // max(1, len(group)))
        for i, g in enumerate(group):
            rest.insert(min(len(rest), i * (step + 1)), g)
        jobs = lead + rest
        nxt = iter(jobs)
        take = threading.Lock()
        barrier = threading.Barrier(threads)
        errors = []

        def worker():
            barrier.wait()
            while True:
                with take:
                    job = next(nxt, None)
                if job is None:
                    return
                try:
                    self.run(job)
                except Exception as e:                      # reported with the results; the test fails on it
                    errors.append("%s: %r" % (job["name"], e))

        ts = [threading.Thread(target=worker) for _ in range(threads)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        self.results["_info"] = dict(r=0, threads=threads, sms=sms, errors=errors)

    def caller_stream(self):
        """Contexts made around a torch stream S: the input reaches the device buffer only after a ~50 ms sleep kernel on S, and nothing
        synchronises the host in between.  A context that ignored S would read the zeros the buffer held before."""
        torch = self.torch
        jobs = self.spec["jobs"]
        streams = [torch.cuda.Stream() for _ in jobs]
        ctxs = [libbsc_b200.DeviceCtx(0, s.cuda_stream) for s in streams]
        barrier = threading.Barrier(len(jobs))

        def one(job, stream, ctx):
            a = self.data(job)
            args = job["args"]
            h_in = torch.from_numpy(a).pin_memory()
            d_in = torch.zeros(a.size + 64, dtype=torch.uint8, device="cuda")
            d_out = torch.zeros(args["out_size"] + 4096, dtype=torch.uint8, device="cuda")

            def call():
                if job["op"] == "compress":
                    return ctx.compress(d_in.data_ptr(), d_out.data_ptr(), a.size, args["sorter"], args["coder"], args["features"])
                return ctx.decompress(d_in.data_ptr(), a.size, d_out.data_ptr(), args["out_size"], args["features"])
            # warm-up call: the constant tables, the arena and the sort slab exist afterwards, so no allocation or first-use
            # synchronisation inside the timed call can hide a missing stream dependency
            d_in[:a.size].copy_(h_in)
            torch.cuda.synchronize()
            assert call() >= 0
            torch.cuda.synchronize()
            d_in.zero_()
            d_out.zero_()
            torch.cuda.synchronize()
            barrier.wait()
            with torch.cuda.stream(stream):
                torch.cuda._sleep(args["sleep_cycles"])
                d_in[:a.size].copy_(h_in, non_blocking=True)
            r = call()
            stream.synchronize()
            n = r if job["op"] == "compress" else args["out_size"]
            self.save(job, r, d_out[:max(n, 0)].cpu().numpy())

        ts = [threading.Thread(target=one, args=(j, s, c)) for j, s, c in zip(jobs, streams, ctxs)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        for c in ctxs:
            c.close()


def main():
    jobdir = sys.argv[1]
    spec = json.load(open(os.path.join(jobdir, "jobs.json")))
    os.makedirs(os.path.join(jobdir, "out"), exist_ok=True)
    R = Runner(jobdir, spec)
    getattr(R, spec["mode"])()
    with open(os.path.join(jobdir, "results.json"), "w") as f:
        json.dump(R.results, f)


if __name__ == "__main__":
    main()
