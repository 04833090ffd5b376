"""Every coder layout, sort switch and the many-blocks pipeline on the GPU, against the reference.

The library reads each BSCB200_* switch once per process, so every configuration runs in a child process of its own (tests/gpu_child.py).
This module computes the reference outputs on the CPU with the checker (the reference when oracle/_ref was built, else the C port), with
tests/golden/reference_results.json and with the known answers of SURVEY.md for blocks too large for that; it writes the inputs as .npy
files, the child runs the GPU and writes its outputs, and the comparison happens here.

The decoder children also prove which layout decoded: with BSCB200_QSTATS=1 the static decoder prints the rare-access count of every
stream, and for each single-stream decode it must equal the count of the host emulation (tools/qdec3_host.cpp) of the same layout.
Both count the same lane-uniform row fetches of qlfc_decoder6_stream.inc, whose number depends on how much of the counter file the
layout keeps resident."""
import ctypes
import hashlib
import json
import os
import re
import subprocess
import sys
import zlib

import numpy as np
import pytest

import reference_inputs as ri
import test_qdec3_host as tq

HERE = os.path.dirname(os.path.abspath(__file__))
CHILD = os.path.join(HERE, "gpu_child.py")
GOLD = json.load(open(os.path.join(HERE, "golden", "reference_results.json")))
K3 = dict(seed=2, n=67108864, size=12686186, adler32=0xF21848C1)     # SURVEY.md known answer: 64 MiB text, default options
CLIPPED_ZEROS = 2094        # rand(9, 600000) + this many zeros: features 1 re-encodes the 2nd sub-block with a clipped room and fails,
                            # features 3 stores a container 4 bytes below the block size (see test_battery_has_a_clipped_reencode)
GROUP_N = 200003            # decode-group size of the pipeline children: no other decode job produces a stream of this length


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint8).tobytes()).hexdigest()


# ---- the coder container (coder.cpp:111-155) and the split launch of stage_coder_decompress (qlfc.cu) ----------------------------
def container_header(c):
    """[(raw size, packed size)] of the sub-blocks of a coder container"""
    c = np.asarray(c, dtype=np.uint8)
    return [(int(c[1 + 8 * b:5 + 8 * b].view("<i4")[0]), int(c[5 + 8 * b:9 + 8 * b].view("<i4")[0])) for b in range(int(c[0]))]


def coded_streams(c):
    """packed sizes of the coded (not stored) sub-blocks in decoder launch order: longest first, stable"""
    if int(c[0]) == 1:
        return [len(c) - 1]
    return sorted([p for r, p in container_header(c) if p != r], key=lambda p: -p)


def split_point(packed):
    """coder_split_point (qlfc.cu): how many of the longest streams go to the middle-priority stream (0 = no split)"""
    n = len(packed)
    if n < 3:
        return 0
    k = 0
    while k < n and packed[k] * 20 >= packed[0] * 11:
        k += 1
    return 0 if k == n else k


# ---- host emulation of the static decoder: the per-layout fingerprint -------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    lib = tq._hostlib()
    lib.qdec6_host_decode.restype = ctypes.c_int
    lib.qdec6_host_decode.argtypes = [ctypes.c_void_p, ctypes.c_uint, ctypes.c_void_p, ctypes.c_uint, ctypes.c_void_p, ctypes.c_int]

    def rare(stream, n, per_sm):
        """rare-access count of decoding `stream` under the layout with `per_sm` streams per SM (emulation mode per_sm - 1)"""
        s = np.ascontiguousarray(stream, dtype=np.uint8)
        out = np.empty(n + 64, dtype=np.uint8)
        stats = (ctypes.c_uint * 2)()
        r = lib.qdec6_host_decode(s.ctypes.data, s.size, out.ctypes.data, n, stats, per_sm - 1)
        assert r == n
        return int(stats[0])
    return rare


# ---- inputs --------------------------------------------------------------------------------------------------------------------
def coder_inputs(gen, checker):
    """(name, coder input): the host emulation's battery, text containers of 1, 2, 4 and 8 sub-blocks, and containers built for the
    container rules"""
    def bwt(a):
        return checker.bwt_encode(a)[1]
    out = list(tq.inputs(gen, checker))
    out += [("text200k/1sub", bwt(gen.text(3, 200000))), ("text1M/2sub", bwt(gen.text(4, 1 << 20))),
            ("text5M/4sub", bwt(gen.text(5, 5 << 20))), ("text20M/8sub", bwt(gen.text(6, 20 << 20)))]
    # coded, stored, stored, coded: the random middle holds most of the sampled changes, so it gets the middle sub-blocks
    out.append(("raw between coded", np.concatenate([bwt(gen.text(7, 1 << 20)), gen.rand(2, 3 << 20), bwt(gen.text(8, 1 << 20))])))
    # one long coded stream and three short ones: a split launch
    out.append(("split", np.concatenate([gen.skew(4, 2 << 20), np.tile(np.frombuffer(b"ab", np.uint8), 5 << 19)])))
    out.append(("clipped", np.concatenate([gen.rand(9, 600000), np.zeros(CLIPPED_ZEROS, np.uint8)])))
    return out


class Battery:
    """Jobs for one kind of child: job dicts (for gpu_child.py), inputs and expected results."""

    def __init__(self, root, name):
        self.dir = os.path.join(str(root), name)
        os.makedirs(os.path.join(self.dir, "in"), exist_ok=True)
        self.jobs, self.expect, self.fingerprint, self.files = [], {}, {}, {}

    def add(self, name, op, data, expect, args=None, fingerprint=None):
        """expect: (r, output) -- output an array, a dict of size and sha256 / adler32, or None; fingerprint: {per_sm: rare-accesses}"""
        job = dict(name=name, op=op, args=args or {}, out=str(len(self.jobs)))
        self.files[name] = job["out"]
        if isinstance(data, tuple):
            job["gen"] = list(data)
        else:
            path = os.path.join(self.dir, "in", "%d.npy" % len(self.jobs))
            np.save(path, np.ascontiguousarray(data, dtype=np.uint8))
            job["in"] = path
        self.jobs.append(job)
        self.expect[name] = expect
        if fingerprint is not None:
            self.fingerprint[name] = fingerprint


def run_child(bat, config, env, mode="serial", timeout=900, **spec):
    """Run gpu_child.py with `env` on the battery; returns its results and its stderr, split by job for a serial run."""
    d = os.path.join(bat.dir, re.sub(r"[^A-Za-z0-9_.=-]+", "_", config))
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "jobs.json"), "w") as f:
        json.dump(dict(mode=mode, jobs=bat.jobs, **spec), f)
    e = dict(os.environ)
    e.update(env)
    try:
        p = subprocess.run([sys.executable, CHILD, d], env=e, capture_output=True, text=True, timeout=timeout)
    except subprocess.TimeoutExpired:
        pytest.fail("%s: the child did not finish within %d s (deadlock?)" % (config, timeout))
    assert p.returncode == 0, "%s: child failed (%d)\n%s" % (config, p.returncode, p.stderr[-4000:])
    results = json.load(open(os.path.join(d, "results.json")))
    per_job, cur = {}, None
    for line in p.stderr.splitlines():
        if line.startswith("[job] "):
            cur = line[6:]
            per_job[cur] = []
        elif cur is not None:
            per_job[cur].append(line)
    return results, p.stderr, per_job, d


def compare(bat, results, outdir, config):
    """Every job's return code and output against the expected ones; the message names the configuration, the input and the first
    differing byte."""
    bad = []
    for name in bat.expect:
        r_want, want = bat.expect[name][:2]
        rec = results.get(name)
        if rec is None:
            bad.append("%s: no result" % name)
            continue
        if rec["r"] != r_want:
            bad.append("%s: returned %d, the reference %d" % (name, rec["r"], r_want))
            continue
        if len(bat.expect[name]) > 2 and rec.get("aux") != bat.expect[name][2]:
            bad.append("%s: secondary indexes %s, the reference %s" % (name, rec.get("aux"), bat.expect[name][2]))
        if want is None:
            continue
        got = np.load(os.path.join(outdir, "out", bat.files[name] + ".npy"))
        if isinstance(want, dict):
            ok = got.size == want["size"] and (sha(got) == want["sha256"] if "sha256" in want else zlib.adler32(got.tobytes()) == want["adler32"])
            if not ok:
                bad.append("%s: %d bytes, digest differs from the reference's %s" % (name, got.size, want))
        elif got.size != want.size or not np.array_equal(got, want):
            m = min(got.size, want.size)
            diff = np.flatnonzero(got[:m] != want[:m])
            at = int(diff[0]) if diff.size else m
            bad.append("%s: %d bytes against %d, first difference at byte %d" % (name, got.size, want.size, at))
    assert not bad, "%s:\n  %s" % (config, "\n  ".join(bad[:20]))


QSTATS_DEC = re.compile(r"\[qstats dec\] sub (\d+): out (-?\d+) rare-accesses (\d+) misses (\d+)")


def check_fingerprints(bat, per_job, per_sm, config):
    checked = 0
    for name, fp in bat.fingerprint.items():
        lines = [QSTATS_DEC.match(l) for l in per_job.get(name, [])]
        lines = [m for m in lines if m]
        assert len(lines) == 1, (config, name, per_job.get(name))
        got = int(lines[0].group(3))
        assert got == fp[per_sm], "%s: %s decoded with %d rare accesses; the %d-per-SM layout makes %d (all layouts: %s)" % (
            config, name, got, per_sm, fp[per_sm], fp)
        checked += 1
    assert checked >= 10, config


# ---- the decoder battery -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def coder_battery(gen, checker):
    return coder_inputs(gen, checker)


@pytest.fixture(scope="module")
def decoder_jobs(tmp_path_factory, coder_battery, gen, checker, emu):
    bat = Battery(tmp_path_factory.mktemp("dec"), "dec")
    for name, a in coder_battery:
        r, s = checker.encode_block(a)
        if r > 0:
            bat.add(name + "/stream", "decode_block", s, (a.size, a), dict(n=a.size), {k: emu(s, a.size, k) for k in (2, 3, 4, 5)})
        r, c = checker.coder_compress(a, 1, 3)
        if r > 0:
            fp = {k: emu(c[1:], a.size, k) for k in (2, 3, 4, 5)} if c[0] == 1 else None
            bat.add(name + "/container", "coder_decompress", c, (a.size, a), dict(n=a.size), fp)
    for name, a in (("text300k", gen.text(7, 300000)), ("text1M", gen.text(2, 1 << 20)), ("skew300k", gen.skew(3, 300000)),
                    ("text5M", gen.text(9, 5 << 20)), ("allsame3000", np.full(3000, 65, np.uint8))):
        r, blk = checker.compress(a, 1, 1, 3)
        bat.add(name + "/block", "decompress", blk, (0, a))
    bat.add("K3 text 64M", "compress_and_decompress", ("text", K3["seed"], K3["n"]), (K3["size"], dict(size=K3["size"], adler32=K3["adler32"])))
    bat.expect["K3 text 64M.dec"] = (0, gen.text(K3["seed"], K3["n"]))   # the job's second output: the block restored
    bat.files["K3 text 64M.dec"] = bat.files["K3 text 64M"] + ".dec"
    return bat


def test_battery_covers_split_and_unsplit_launches(coder_battery, checker):
    """The decoder battery launches the static decoder split over both priority streams and unsplit with three or more streams."""
    split = unsplit = 0
    for name, a in coder_battery:
        r, c = checker.coder_compress(a, 1, 3)
        if r <= 0:
            continue
        packed = coded_streams(c)
        n_hi = split_point(packed)
        split += 0 < n_hi < len(packed)
        unsplit += len(packed) >= 3 and n_hi == 0
    assert split >= 1 and unsplit >= 1, (split, unsplit)


def test_battery_has_a_stored_sub_block_between_coded_ones(coder_battery, checker):
    a = dict(coder_battery)["raw between coded"]
    r, c = checker.coder_compress(a, 1, 3)
    stored = [raw == packed for raw, packed in container_header(c)]
    assert r > 0 and stored[0] is False and stored[-1] is False and any(stored), container_header(c)


def test_battery_has_a_clipped_reencode(coder_battery, checker):
    """Under features 1 (coder.cpp:111-155) the second sub-block of this block is encoded into the room left after the stored first
    one, which is smaller than the sub-block; that encode runs out of room, so the serial rules give up, while the parallel rules of
    features 3 keep a container a few bytes smaller than the block."""
    a = dict(coder_battery)["clipped"]
    r3, c3 = checker.coder_compress(a, 1, 3)
    r1, _ = checker.coder_compress(a, 1, 1)
    (raw0, packed0), (raw1, packed1) = container_header(c3)
    assert raw0 == packed0 and packed1 < raw1                    # stored, then coded
    assert a.size - (1 + 16 + raw0) < raw1                       # features 1: the room is clipped
    assert 0 < r3 < a.size and r1 == -3, (r3, r1)


def test_battery_layouts_4_and_5_leave_different_fingerprints(coder_battery, checker, emu):
    differ = 0
    for name, a in coder_battery[:13]:
        r, s = checker.encode_block(a)
        if r > 0:
            differ += emu(s, a.size, 4) != emu(s, a.size, 5)
    assert differ >= 3


# ---- 1. decoder layouts --------------------------------------------------------------------------------------------------------
DECODER_CONFIGS = [
    ("DEC_PER_SM=2", {"BSCB200_DEC_PER_SM": "2"}, 2),
    ("DEC_PER_SM=3", {"BSCB200_DEC_PER_SM": "3"}, 3),
    ("DEC_PER_SM=4", {"BSCB200_DEC_PER_SM": "4"}, 4),
    ("DEC_PER_SM=5", {"BSCB200_DEC_PER_SM": "5"}, 5),
    # priorities and the split off: the short half of a launch goes to the context's own stream
    ("DEC_PER_SM=5,PRIO=0,CODER_SPLIT=0", {"BSCB200_DEC_PER_SM": "5", "BSCB200_PRIO": "0", "BSCB200_CODER_SPLIT": "0"}, 5),
]


@pytest.mark.gpu
@pytest.mark.parametrize("config,env,per_sm", DECODER_CONFIGS, ids=[c[0] for c in DECODER_CONFIGS])
def test_decoder_layout(bsc, decoder_jobs, config, env, per_sm):
    results, _, per_job, d = run_child(decoder_jobs, config, dict(env, BSCB200_QSTATS="1"))
    compare(decoder_jobs, results, d, config)
    check_fingerprints(decoder_jobs, per_job, per_sm, config)


# ---- 2. encoder layouts --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def encoder_jobs(tmp_path_factory, coder_battery, checker):
    bat = Battery(tmp_path_factory.mktemp("enc"), "enc")
    for name, a in coder_battery:
        for f in (3, 1):
            r, c = checker.coder_compress(a, 1, f)
            bat.add("%s/f%d" % (name, f), "coder_compress", a, (r, c), dict(features=f))
        for cap in (None, a.size // 2):
            r, s = checker.encode_block(a, cap)
            bat.add("%s/cap%s" % (name, cap), "encode_block", a, (r, s if r > 0 else None), dict(cap=cap))
    return bat


ENCODER_CONFIGS = [("ENC_PER_SM=%d" % k, {"BSCB200_ENC_PER_SM": str(k)}) for k in (2, 3, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("config,env", ENCODER_CONFIGS, ids=[c[0] for c in ENCODER_CONFIGS])
def test_encoder_layout(bsc, encoder_jobs, config, env):
    results, _, _, d = run_child(encoder_jobs, config, env)
    compare(encoder_jobs, results, d, config)


# ---- 3. sort switches ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sms(bsc):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def sort_jobs(tmp_path_factory, gen, checker, port, sms):
    """RS_TILE = 4096 keys per tile; the persistent TMA grid has 2 x SMs CTAs."""
    bat = Battery(tmp_path_factory.mktemp("sort"), "sort")
    grid_n = 2 * sms * 4096
    sizes = [4095, 4096, 4097, 4098, 4099, 100001, grid_n, 8 * grid_n + 2]
    for n in sizes:
        a = gen.text(n % 97, n)
        r, L, aux = checker.bwt_encode(a)
        bat.add("bwt n=%d" % n, "bwt_encode", a, (r, L, aux))
        if n >= grid_n:
            bat.add("batched bwt n=%d" % n, "bwt_batched", a, (r, L, aux), dict(budget=1))
        if n > grid_n:
            bat.add("profiled bwt n=%d" % n, "bwt_profiled", a, (r, L, aux))
            z, blk = checker.compress(a, 1, 1, 3)
            bat.add("compress m1 n=%d" % n, "compress", a, (z, blk), dict(sorter=1, coder=1, features=3))
            continue
        for k in (3, 4, 5, 6, 7, 8):
            impl = checker if k <= 6 else port               # orders 7 and 8 exist only in the reference's CUDA build
            i, Lk = impl.st_encode(a, k)
            bat.add("st%d n=%d" % (k, n), "st_encode", a, (i, Lk), dict(k=k))
            bat.add("unst%d n=%d" % (k, n), "st_decode", Lk, (0, a), dict(k=k, index=i))
        for s in (1, 3, 4, 5, 6, 7, 8):
            impl = checker if s <= 6 else port
            z, blk = impl.compress(a, s, 1, 3)
            bat.add("compress m%d n=%d" % (s, n), "compress", a, (z, blk), dict(sorter=s, coder=1, features=3))
    for name in ("zeros", "period8"):
        want = GOLD["degenerate"][name]
        bat.add("bwt 64M " + name, "bwt_encode", ("degenerate", name, 0), (want["index"], want["L"], want["aux"]))
    return bat


SORT_CONFIGS = [("SORT_TMA=1", {"BSCB200_SORT_TMA": "1"}, "rs_onesweep_tma"), ("SORT_OCC=3", {"BSCB200_SORT_OCC": "3"}, "rs_onesweep")]


@pytest.mark.gpu
@pytest.mark.parametrize("config,env,kernel", SORT_CONFIGS, ids=[c[0] for c in SORT_CONFIGS])
def test_sort_switch(bsc, sort_jobs, config, env, kernel):
    results, _, _, d = run_child(sort_jobs, config, env)
    compare(sort_jobs, results, d, config)
    prof = [rec["profile"] for name, rec in results.items() if name.startswith("profiled")]
    assert prof and all(p.get(kernel, 0) > 0 for p in prof), (config, prof)
    if kernel != "rs_onesweep_tma":
        assert all(p.get("rs_onesweep_tma", 0) == 0 for p in prof), (config, prof)


# ---- 4. many blocks in flight --------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pipeline_jobs(tmp_path_factory, gen, checker, port, emu):
    bat = Battery(tmp_path_factory.mktemp("pipe"), "pipe")
    rng = np.random.default_rng(2024)
    sizes = [29, 100, 4097, 70000, 300000, 1 << 20, 1 << 20, 2 << 20, 5 << 20, 5 << 20, 20 << 20]   # mostly blocks that keep a coder busy
    kinds = ["text", "text", "text", "skew", "rand"]
    for j in range(80):
        n = sizes[j % len(sizes)]
        kind = kinds[int(rng.integers(len(kinds)))]
        a = getattr(gen, kind)(int(rng.integers(1, 1000)), n)
        sorter = int(rng.choice([1, 3, 4, 5, 6] + ([7, 8] if n <= (1 << 20) else [])))
        coder, f = int(rng.integers(1, 4)), int(rng.choice([1, 3]))
        impl = checker if sorter <= 6 else port
        z, blk = impl.compress(a, sorter, coder, f)
        inplace = kind == "text" and n > 4096 and j % 3 == 0    # in place, an incompressible block is NOT_COMPRESSIBLE, not stored
        bat.add("c%02d %s n=%d m%d e%d f%d%s" % (j, kind, n, sorter, coder, f, " inplace" if inplace else ""), "compress", a, (z, blk),
                dict(sorter=sorter, coder=coder, features=f, inplace=inplace))
        if j % 2 == 0:
            bat.add("d%02d %s n=%d m%d e%d" % (j, kind, n, sorter, coder), "decompress", blk, (0, a))
    for name, a in ri.lzp_inputs(gen).items():
        for f in (1, 3):
            want = GOLD["lzp"]["%s/f%d" % (name, f)]
            bat.add("lzp %s f%d" % (name, f), "compress", a, (want["size"], want), dict(sorter=1, coder=1, features=f, lzp=[15, 128]))
    # coder stages only, 8 streams each: the jobs every thread starts with
    L20 = checker.bwt_encode(gen.text(6, 20 << 20))[1]
    for f in (3, 1):
        r, c = checker.coder_compress(L20, 1, f)
        bat.add("lead coder_compress 20M f%d" % f, "coder_compress", L20, (r, c), dict(features=f, role="lead"))
    for j in range(22):
        bat.add("lead coder_decompress 20M #%d" % j, "coder_decompress", c, (L20.size, L20), dict(n=L20.size, role="lead"))
    # the decode group: one single-stream container, decoded many times; its stream length tells its [qstats dec] lines apart
    L = checker.bwt_encode(gen.text(11, GROUP_N))[1]
    r, c = checker.coder_compress(L, 1, 3)
    assert r > 0 and c[0] == 1
    bat.group = {k: emu(c[1:], GROUP_N, k) for k in (4, 5)}
    assert bat.group[4] != bat.group[5]
    for j in range(48):
        bat.add("g%02d" % j, "coder_decompress", c, (GROUP_N, L), dict(n=GROUP_N, role="group"))
    bat.max_n, bat.max_st_n = max(sizes), max(sizes)
    return bat


PIPELINE_CONFIGS = [("default", {}, True), ("SORT_SLABS=1", {"BSCB200_SORT_SLABS": "1"}, False),
                    ("CODER_SLOTS=8", {"BSCB200_CODER_SLOTS": "8"}, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("config,env,need_layout5", PIPELINE_CONFIGS, ids=[c[0] for c in PIPELINE_CONFIGS])
def test_pipeline(bsc, pipeline_jobs, config, env, need_layout5):
    bat = pipeline_jobs
    env = dict(env, CUDA_DEVICE_MAX_CONNECTIONS="32", BSCB200_QSTATS="1")
    results, stderr, _, d = run_child(bat, config, env, mode="pipeline", seed=7, max_n=bat.max_n, max_st_n=bat.max_st_n)
    info = results.pop("_info")
    assert not info["errors"], (config, info["errors"])
    assert info["threads"] >= min(info["sms"] // 8 + 8, 17), info  # more than SMs / 8 blocks can be in coder stages at once
    compare(bat, results, d, config)
    counts = [int(m.group(3)) for m in QSTATS_DEC.finditer(stderr) if int(m.group(2)) == GROUP_N]
    assert len(counts) == 48, (config, len(counts))
    assert set(counts) <= set(bat.group.values()), (config, sorted(set(counts)), bat.group)
    if need_layout5:
        assert bat.group[5] in counts, "%s: no decode ran the 5-per-SM layout (counts %s, layouts %s)" % (config, sorted(set(counts)), bat.group)


# ---- 5. contexts around the caller's stream ------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_contexts_on_caller_streams(bsc, tmp_path, gen, checker):
    bat = Battery(tmp_path, "stream")
    sleep = 100_000_000                                          # clock cycles: about 50 ms
    for j, (kind, seed, n) in enumerate((("text", 2, 5 << 20), ("skew", 3, 1 << 20))):
        a = getattr(gen, kind)(seed, n)
        z, blk = checker.compress(a, 1, 1, 3)
        bat.add("compress %s %d" % (kind, n), "compress", a, (z, blk), dict(sorter=1, coder=1, features=3, out_size=n, sleep_cycles=sleep))
        bat.add("decompress %s %d" % (kind, n), "decompress", blk, (0, a), dict(features=3, out_size=n, sleep_cycles=sleep))
    results, _, _, d = run_child(bat, "caller streams", {}, mode="caller_stream", timeout=600)
    compare(bat, results, d, "caller streams")
