#!/usr/bin/env python3
"""Generates tests/golden/reference_results_malformed.json (and the LZP base block tests/golden/rep700x900.block.lzp) from the UNMODIFIED
reference built by oracle/Makefile (oracle/_ref): its answer to every case of tests/malformed_inputs.py, out of place and in place, and
to the stage-level calls with bad arguments.

A case records the return code and, when it is 0, the size and SHA-256 of the output.  The calls run on the reference built with
AddressSanitizer (make -C oracle asan), each in a forked child: a crafted payload can make the reference read or write outside its
buffers, crash or hang, and such a case is recorded as "crash".  Without the sanitizer, whether a stray write kills the process depends
on the heap layout of the run, and the fixture would not regenerate byte for byte.  The input is followed by 1 MiB of zeros, so that
what the reference reads past a block is the same on every run; the output is followed by 1 MiB of 0xA5, which must come back unchanged.
The reference runs single-threaded (features = 1): its return codes do not depend on the threading feature, and a forked child must
not rely on an OpenMP pool.

The parent makes the blocks; a child process with the sanitizer preloaded runs them (python make_reference_results_malformed.py --run
<dir>) and imports neither torch nor oracle.pyoracle, whose build step must not run under the preload."""
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
import malformed_inputs as mi                     # noqa: E402

PAD = 1 << 20
TIMEOUT_S = 20
FEATURES = 1
vp = ctypes.c_void_p


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint8).tobytes()).hexdigest()


def in_child(fn):
    """fn() in a forked child: its JSON-able result, or "crash" when the child dies, hangs or fn raises"""
    rd, wr = os.pipe()
    pid = os.fork()
    if pid == 0:
        os.close(rd)
        try:
            msg = json.dumps(fn()).encode()
        except BaseException:
            msg = b'"crash"'
        os.write(wr, msg)
        os._exit(0)
    os.close(wr)
    import select
    chunks = []
    ready, _, _ = select.select([rd], [], [], TIMEOUT_S)
    if ready:
        while True:
            c = os.read(rd, 1 << 16)
            if not c:
                break
            chunks.append(c)
    else:
        os.kill(pid, 9)
    os.close(rd)
    _, status = os.waitpid(pid, 0)
    if not chunks or not os.WIFEXITED(status) or os.WEXITSTATUS(status) != 0:
        return "crash"
    return json.loads(b"".join(chunks))


def decompress(lib, blk, in_size, out_size, inplace):
    def run():
        if inplace:
            cap = max(blk.size, out_size, 0)
            buf = np.full(cap + PAD, 0xA5, np.uint8)
            buf[:blk.size] = blk
            buf[blk.size:blk.size + PAD] = 0          # what lies past the block reads as zeros, as out of place
            keep = buf[cap:].copy()
            r = lib.bsc_decompress(vp(buf.ctypes.data), in_size, vp(buf.ctypes.data), out_size, FEATURES)
            if not np.array_equal(buf[cap:], keep):
                return "crash"
            out = buf[:max(out_size, 0)]
        else:
            src = np.zeros(blk.size + PAD, np.uint8)
            src[:blk.size] = blk
            dst = np.full(max(out_size, 0) + PAD, 0xA5, np.uint8)
            r = lib.bsc_decompress(vp(src.ctypes.data), in_size, vp(dst.ctypes.data), out_size, FEATURES)
            if np.any(dst[max(out_size, 0):] != 0xA5):
                return "crash"
            out = dst[:max(out_size, 0)]
        rec = {"r": int(r)}
        if r == 0:
            rec.update(size=int(out.size), sha256=sha(out))
        return rec
    return in_child(run)


def stage(lib, kind, args):
    a = np.zeros(max(args["n"], 0) + PAD, np.uint8)
    a[:1000] = mi.stage_data()
    p, n = vp(a.ctypes.data), args["n"]
    out = np.zeros(PAD + 4096, np.uint8)
    if kind == "bwt_decode":
        return lib.bsc_bwt_decode(p, n, args["index"], 0, None, FEATURES)
    if kind == "st_encode":
        return lib.bsc_st_encode(p, n, args["k"], FEATURES)
    if kind == "st_decode":
        return lib.bsc_st_decode(p, n, args["k"], args["index"], FEATURES)
    if kind == "coder_compress":
        return lib.bsc_coder_compress(p, vp(out.ctypes.data), n, args["coder"], FEATURES)
    if kind == "coder_decompress":
        return lib.bsc_coder_decompress(p, vp(out.ctypes.data), args["coder"], FEATURES)
    bs, ds = ctypes.c_int(0), ctypes.c_int(0)
    return lib.bsc_block_info(p, n, ctypes.byref(bs), ctypes.byref(ds), FEATURES)


def run(d):
    """the child: every case and stage call of <d>/cases.npz on the sanitized reference; writes <d>/results.json"""
    lib = ctypes.CDLL(os.path.join(ROOT, "oracle", "_ref", "libbsc_ref_asan.so"))
    lib.bsc_init(FEATURES)
    lib.bsc_decompress.argtypes = [vp, ctypes.c_int, vp, ctypes.c_int, ctypes.c_int]
    lib.bsc_bwt_decode.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_ubyte, vp, ctypes.c_int]
    lib.bsc_coder_decompress.argtypes = [vp, vp, ctypes.c_int, ctypes.c_int]
    meta = json.load(open(os.path.join(d, "cases.json")))
    blocks = np.load(os.path.join(d, "cases.npz"))
    out = {"cases": {}, "stages": {}}
    for i, (name, in_size, out_size) in enumerate(meta):
        blk = blocks["b%d" % i]
        out["cases"][name] = {"out": decompress(lib, blk, in_size, out_size, False), "inplace": decompress(lib, blk, in_size, out_size, True)}
    for name, kind, args in mi.stage_calls():
        out["stages"][name] = in_child(lambda: int(stage(lib, kind, args)))
    json.dump(out, open(os.path.join(d, "results.json"), "w"))


def main():
    from oracle import pyoracle
    gen, port = pyoracle.Gen(), pyoracle.Port()
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "asan"], stdout=subprocess.DEVNULL)
    ref = pyoracle.Ref()
    z, lzp = ref.compress_lzp(np.tile(gen.text(3, 700), 900), 15, 128, 1, 1, FEATURES)
    assert z > 0 and mi.get32(lzp, 8) != mi.get32(lzp, 8) & 0xff
    lzp.tofile(mi.LZP_BLOCK)
    bases, cases = mi.battery(gen, port)
    with tempfile.TemporaryDirectory() as d:
        json.dump([(name, int(i), int(o)) for name, _, i, o in cases], open(os.path.join(d, "cases.json"), "w"))
        np.savez(os.path.join(d, "cases.npz"), **{"b%d" % i: c[1] for i, c in enumerate(cases)})
        asan = subprocess.run(["gcc", "-print-file-name=libasan.so"], capture_output=True, text=True, check=True).stdout.strip()
        env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0")
        subprocess.check_call([sys.executable, os.path.abspath(__file__), "--run", d], env=env, stderr=subprocess.DEVNULL)
        res = json.load(open(os.path.join(d, "results.json")))
    out = {"features": FEATURES, "seed": mi.SEED,
           "bases": {name: {"block": sha(b), "size": int(b.size), "data": sha(d)} for name, (b, d) in bases.items()}, **res}
    with open(os.path.join(HERE, "reference_results_malformed.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("ok: %d cases" % len(cases))


if __name__ == "__main__":
    if sys.argv[1:2] == ["--run"]:
        run(sys.argv[2])
    else:
        main()
