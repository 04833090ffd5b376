"""Malformed blocks and corrupt streams on every decode path, against the reference's error codes.

The battery of tests/malformed_inputs.py (header fields, payloads whose Adler-32 is recomputed so that the corruption reaches the coder
kernels and the inverse transforms, and bad call arguments) runs through bsc_decompress out of place into a buffer of 0xA5 and in place,
in three child processes (tests/gpu_child.py):

  default      a lone call decodes with LayoutDiet4 (four decoder streams per SM)
  per_sm5      BSCB200_DEC_PER_SM=5: the other layout the product launches, LayoutDiet5
  routed       BSCB200_LARGE_N=28: the same blocks through the paths of blocks above 1 GiB (with_own_ctx, decompress_large_st)

Where the reference (tests/golden/reference_results_malformed.json) returns a code, the product returns the same, and on 0 the same
bytes.  Where the reference reads or writes outside its buffers ("crash"), the product returns a negative code.  On every failure the
product writes nothing: the whole output buffer, and the caller's buffer in place, are as they were before the call.

The default child also runs the device-resident entry points on caller buffers of exactly the documented size between guard regions."""
import hashlib
import json
import os
import zlib

import numpy as np
import pytest

import malformed_inputs as mi
import test_gpu_parity as tp
from test_gpu_pipeline import Battery, run_child

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_results_malformed.json")
SLACK = 64 << 20
# Cases where the product deliberately does not do what the reference does: {case: (the product's return code, reason)}.  On a negative
# code the product writes nothing; on 0 it writes the base block's data.
DIVERGENCES = {
    "stored/truncated@2514": (-6, "a stored block whose payload is shorter than dataSize: the reference copies dataSize bytes, reading "
                                  "past the end of the block (libbsc.cpp:550-555); the product returns LIBBSC_DATA_CORRUPT"),
    "stored/truncated@5026": (-6, "the same over-read of a stored block two bytes short"),
    "lzp/num_indexes=255": (0, "a count of 255 secondary indexes in a 680-byte block: the reference copies 1020 bytes from before the "
                               "start of the block (libbsc.cpp:560-564); the product never reads secondary indexes, which only speed "
                               "up the reference's CPU inverse BWT, and decodes the block"),
}
for _base in ("bwt_e1", "bwt_e2", "bwt_e3", "lzp"):
    DIVERGENCES[_base + "/index_value0+1"] = (
        0, "a secondary index off by one, its count and range valid: the reference's CPU inverse BWT starts a segment at the wrong row and "
           "writes garbage (or outside its buffer, as the sanitized build shows); the product's inverse BWT does not use secondary "
           "indexes, so it decodes the block, and the data Adler-32 confirms it.  Out-of-range values return LIBBSC_BAD_PARAMETER in both")


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint8).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def battery(gen, port):
    return mi.battery(gen, port)


@pytest.fixture(scope="module")
def fixture():
    return json.load(open(FIXTURE))


def has_lzp_bits(blk):
    return blk.size >= mi.HDR and mi.get32(blk, 8) != mi.get32(blk, 8) & 0xff


def host_jobs(bat, bases, cases):
    name0, (blk0, data0) = "bwt_e1", bases["bwt_e1"]
    bat.add("warmup", "guarded_decompress", blk0, None, dict(n=data0.size, in_size=blk0.size))
    bat.add("free/start", "free_hbm", np.zeros(1, np.uint8), None)
    for name, blk, in_size, out_size in cases:
        bat.add(name, "guarded_decompress", blk, None, dict(n=out_size, in_size=in_size))
    for name, (blk, data) in bases.items():
        bat.add("after/" + name, "guarded_decompress", blk, None, dict(n=data.size, in_size=blk.size))
    bat.add("free/end", "free_hbm", np.zeros(1, np.uint8), None)


def check_host(results, outdir, bat, bases, cases, fixture, config):
    bad = []
    for name, blk, in_size, n in cases:
        for mode, suffix in (("out", ""), ("inplace", ".inplace")):
            rec = results[name + suffix]
            buf = np.load(os.path.join(outdir, "out", bat.files[name] + suffix + ".npy"))
            before = np.full(buf.size, 0xA5, np.uint8)
            if mode == "inplace":
                before[:blk.size] = blk
            want = fixture["cases"][name][mode]
            if want == "crash" and fixture["cases"][name]["out"] != "crash":
                want = fixture["cases"][name]["out"]        # only the reference's in-place path faults; the product runs both alike
            r = rec["r"]
            tag = "%s [%s]" % (name, mode)
            if name in DIVERGENCES:
                data = bases[name.split("/")[0]][1]
                want = {"r": DIVERGENCES[name][0], "sha256": sha(data)}
            if want == "crash":
                if r >= 0:
                    bad.append("%s: returned %d where the reference crashes" % (tag, r))
            elif r != want["r"]:
                bad.append("%s: returned %d, the reference %d" % (tag, r, want["r"]))
            elif r == 0 and (sha(buf[:n]) != want["sha256"] or not np.array_equal(buf[n:], before[n:])):
                bad.append("%s: output differs from the reference's, or bytes past dataSize were written" % tag)
            if r != 0 and not np.array_equal(buf, before):
                bad.append("%s: returned %d and wrote %d bytes of the caller's buffer" % (tag, r, int(np.count_nonzero(buf != before))))
    for name, (blk, data) in bases.items():
        rec = results["after/" + name]
        buf = np.load(os.path.join(outdir, "out", bat.files["after/" + name] + ".npy"))
        if rec["r"] != 0 or not np.array_equal(buf[:data.size], data):
            bad.append("after the battery, %s no longer decodes (%d)" % (name, rec["r"]))
    drift = results["free/start"]["free"] - results["free/end"]["free"]
    if drift > SLACK:
        bad.append("free HBM after bscb200_release_pools is %d MiB below its value at the start" % (drift >> 20))
    return bad


def device_jobs(bat, gen, checker, port, cases):
    """the device-resident entry points; returns {job name: check(rec, out) -> error or None}"""
    checks = {}

    def add(name, data, args, check):
        bat.add(name, "device_guarded", data, None, args)
        checks[name] = check

    for name, blk, in_size, n in cases:
        def dec_check(rec, out, blk=blk, n=n):
            if rec["r"] != rec["host"] and not (has_lzp_bits(blk) and rec["r"] == -4):
                return "returned %d, the host entry point %d" % (rec["r"], rec["host"])
            if rec["r"] == 0 and sha(out[:n]) != rec["host_sha"]:
                return "decoded other bytes than the host entry point"
        add("dev/decompress/" + name, blk, dict(call="decompress", in_size=in_size, out_size=max(n, 0)), dec_check)
        coder = (mi.get32(blk, 8) >> 5) & 7 if blk.size > mi.HDR else 0
        if blk.size > mi.HDR + 1 and 1 <= coder <= 3 and n > 0:
            def cdec_check(rec, out):
                if rec["r"] != rec["host"]:
                    return "returned %d, the host entry point %d" % (rec["r"], rec["host"])
                if rec["r"] >= 0 and sha(out[:rec["r"]]) != rec["host_sha"]:
                    return "decoded other bytes than the host entry point"
            add("dev/coder_decompress/" + name, blk[mi.HDR:].copy(), dict(call="coder_decompress", in_size=blk.size - mi.HDR, out_size=n,
                                                                         coder=coder), cdec_check)
    for iname, a in tp.small_inputs(gen):
        idx, L, aux = checker.bwt_encode(a)

        def expect(r_want, out_want=None, aux_want=None):
            def check(rec, out):
                if rec["r"] != r_want:
                    return "returned %d, the reference %d" % (rec["r"], r_want)
                if out_want is not None and not np.array_equal(out, out_want):
                    return "output differs from the reference's"
                if aux_want is not None and rec["aux"] != aux_want:
                    return "secondary indexes %s, the reference %s" % (rec["aux"], aux_want)
            return check
        add("dev/bwt_encode/" + iname, a, dict(call="bwt_encode"), expect(idx, L, [int(x) for x in aux]))
        add("dev/bwt_decode/" + iname, L, dict(call="bwt_decode", index=idx), expect(0, a))
        for k in (4, 8):
            i, Ls = (checker if k <= 6 else port).st_encode(a, k)
            add("dev/st_encode/k%d/%s" % (k, iname), a, dict(call="st_encode", k=k), expect(i, Ls))
            add("dev/st_decode/k%d/%s" % (k, iname), Ls, dict(call="st_decode", k=k, index=i), expect(0, a))
        for c in (1, 2, 3):
            z, s = checker.coder_compress(L, c, 3)
            add("dev/coder_compress/e%d/%s" % (c, iname), L, dict(call="coder_compress", coder=c), expect(z, s))
        add("dev/adler32/" + iname, a, dict(call="adler32"), expect(zlib.adler32(a.tobytes())))
    for iname, L, index in mi.corrupt_bwt_inputs():
        add("dev/bwt_decode_corrupt/" + iname, L, dict(call="bwt_decode", index=index), expect(0))
    return checks


def check_device(results, outdir, bat, checks):
    bad = []
    for name, check in checks.items():
        rec = results[name]
        out = np.load(os.path.join(outdir, "out", bat.files[name] + ".npy"))
        err = check(rec, out)
        if not all(rec["guards"]):
            err = "a guard region was written (offsets 0, 1, 7: %s)" % rec["guards"]
        elif not rec["offsets_agree"]:
            err = err or "offsets 0, 1 and 7 from a 256-byte boundary give other results (codes %s)" % rec["codes"]
        if err:
            bad.append("%s: %s" % (name, err))
    return bad


def test_battery_matches_fixture(battery, fixture):
    """the port still makes the base blocks the fixture was recorded on, and the fixture covers the battery"""
    bases, cases = battery
    for name, (blk, data) in bases.items():
        rec = fixture["bases"][name]
        assert (sha(blk), sha(data)) == (rec["block"], rec["data"]), name
        assert fixture["cases"][name + "/valid"]["out"] == {"r": 0, "size": int(data.size), "sha256": sha(data)}, name
    assert sorted(fixture["cases"]) == sorted(c[0] for c in cases)
    assert set(DIVERGENCES) <= set(fixture["cases"])


CONFIGS = {"default": {}, "per_sm5": {"BSCB200_DEC_PER_SM": "5"}, "routed": {"BSCB200_LARGE_N": "28"}}


@pytest.mark.gpu
@pytest.mark.parametrize("config", list(CONFIGS))
def test_malformed_blocks(config, tmp_path, battery, fixture, gen, port, checker, bsc):
    bases, cases = battery
    bat = Battery(tmp_path, config)
    host_jobs(bat, bases, cases)
    checks = device_jobs(bat, gen, checker, port, cases) if config == "default" else {}
    results, _, _, outdir = run_child(bat, config, CONFIGS[config])
    bad = check_host(results, outdir, bat, bases, cases, fixture, config) + check_device(results, outdir, bat, checks)
    assert not bad, "%s: %d problems\n  %s" % (config, len(bad), "\n  ".join(bad[:40]))


def stage_call(lib, ctx, kind, args, device):
    """one stage entry point of the product on 1000 bytes of mi.stage_data(), as the fixture's generator calls the reference's"""
    import ctypes
    import torch
    n = args["n"]
    data = mi.stage_data()
    if device:
        t = torch.zeros(4096 + 2 * data.size + 4096, dtype=torch.uint8, device="cuda")
        t[:data.size] = torch.from_numpy(data).cuda()
        p, out = t.data_ptr(), t.data_ptr() + 2048
        torch.cuda.synchronize()
        r = {"bwt_decode": lambda: ctx.bwt_decode(p, n, args["index"]),
             "st_encode": lambda: ctx.st_encode(p, n, args["k"]),
             "st_decode": lambda: ctx.st_decode(p, n, args["k"], args["index"]),
             "coder_compress": lambda: ctx.coder_compress(p, out, n, args["coder"]),
             "coder_decompress": lambda: ctx.coder_decompress(p, data.size, out, data.size, args["coder"])}[kind]()
        torch.cuda.synchronize()
        return r
    a = np.zeros(max(n, 0) + data.size + 4096, np.uint8)
    a[:data.size] = data
    out = np.zeros(2 * data.size + 4096, np.uint8)
    p, o = a.ctypes.data, out.ctypes.data
    if kind == "bwt_decode":
        return lib.bsc_bwt_decode(p, n, args["index"], 0, None, 3)
    if kind == "st_encode":
        return lib.bsc_st_encode(p, n, args["k"], 3)
    if kind == "st_decode":
        return lib.bsc_st_decode(p, n, args["k"], args["index"], 3)
    if kind == "coder_compress":
        return lib.bsc_coder_compress(p, o, n, args["coder"], 3)
    if kind == "coder_decompress":
        return lib.bsc_coder_decompress(p, o, args["coder"], 3)
    bs, ds = ctypes.c_int(0), ctypes.c_int(0)
    return lib.bsc_block_info(p, n, ctypes.byref(bs), ctypes.byref(ds), 3)


@pytest.mark.gpu
def test_stage_calls_with_bad_arguments(fixture, bsc):
    """every stage entry point, host pointers and device-resident, returns the reference's code for each bad argument of the fixture
    (a negative code where the reference crashes)"""
    import libbsc_b200
    ctx = libbsc_b200.DeviceCtx(0)
    bad = []
    try:
        assert sorted(fixture["stages"]) == sorted(name for name, _, _ in mi.stage_calls())
        for name, kind, args in mi.stage_calls():
            want = fixture["stages"][name]
            for device in ((False, True) if kind != "block_info" else (False,)):
                r = stage_call(bsc.lib, ctx, kind, args, device)
                if (r >= 0) if want == "crash" else (r != want):
                    bad.append("%s%s: returned %d, the reference %s" % (name, " (device)" if device else "", r, want))
    finally:
        ctx.close()
    assert not bad, "\n".join(bad)
