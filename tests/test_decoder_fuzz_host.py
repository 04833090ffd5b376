"""Memory safety of the single-warp QLFC decoders on corrupt streams, under AddressSanitizer and UBSan, on the CPU.

tools/qdec3_host.cpp compiles the decoders of libbsc_b200/csrc (qlfc_decoder6.cuh in all five layouts, qlfc_fast.cuh, qlfc_adaptive.cuh)
for the host, the 32 lanes one after the other.  On the GPU an access outside a decoder's shared-memory image, its cold counters or its
output slice is a sticky fault that takes the process down, or worse, goes unnoticed; here the sanitizers see every such access.

The parent makes valid streams with the C port; a child process with the sanitizer runtimes preloaded decodes them and a few thousand
seeded mutations of them: random bytes, bit flips, truncations, garbage after a valid prefix, and output capacities below the coded
size.  Every input and output lies in a malloc'd block of exactly its size, so that one byte read past the stream or written past
out_cap is a sanitizer report.  The child imports only numpy (oracle.pyoracle would run make, and nvcc, under the preload).

Each decoder may return anything in {-6, -5} and [0, out_cap], and must not touch memory outside its buffers."""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tools", "qdec3_host.cpp")
LIB = os.path.join(ROOT, "tools", "bin", "libqdec3_host_asan.so")
CASES_PER_DECODER = 400
# (name, coder whose streams it decodes, symbol, layout or None)
DECODERS = [("layout%d" % m, 1, "qdec6_host_decode", m) for m in range(5)] + [("qfast", 3, "qfast_host_decode", None),
                                                                               ("qadapt", 2, "qadapt_host_decode", None)]


def sanitizer_runtimes():
    """paths of libasan and libubsan, or None where the compiler has no AddressSanitizer runtime"""
    paths = []
    for name in ("libasan.so", "libubsan.so"):
        p = subprocess.run(["gcc", "-print-file-name=" + name], capture_output=True, text=True).stdout.strip()
        if not os.path.isabs(p) or not os.path.exists(p):
            return None if name == "libasan.so" else paths
        paths.append(p)
    return paths


def build_lib():
    deps = [SRC] + [os.path.join(ROOT, "libbsc_b200", "csrc", f) for f in os.listdir(os.path.join(ROOT, "libbsc_b200", "csrc"))
                    if f.startswith("qlfc")]
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in deps):
        subprocess.run(["g++", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-Wno-unknown-pragmas",
                        "-shared", "-fPIC", "-o", LIB, SRC], check=True)


def mutate(rng, s, kind):
    s = s.copy()
    if kind == 0:                                         # random bytes
        return rng.integers(0, 256, int(rng.integers(1, 5000)), dtype=np.uint8)
    if kind == 1:                                         # bit flips
        for _ in range(int(rng.integers(1, 20))):
            s[int(rng.integers(0, s.size))] ^= np.uint8(1 << int(rng.integers(0, 8)))
        return s
    if kind == 2:                                         # truncated
        return s[:int(rng.integers(0, s.size))]
    k = int(rng.integers(1, s.size))                      # garbage after a valid prefix
    s[k:] = rng.integers(0, 256, s.size - k, dtype=np.uint8)
    return s


def child(d):
    """decode every case under the sanitizers; writes results.json: {decoder: [return values]}"""
    libc = ctypes.CDLL(None)
    libc.malloc.restype = ctypes.c_void_p
    libc.malloc.argtypes = [ctypes.c_size_t]
    libc.free.argtypes = [ctypes.c_void_p]
    lib = ctypes.CDLL(LIB)
    vp, cu = ctypes.c_void_p, ctypes.c_uint
    base = dict(np.load(os.path.join(d, "streams.npz")))
    results = {}
    for di, (name, coder, sym, layout) in enumerate(DECODERS):
        f = getattr(lib, sym)
        f.restype = ctypes.c_int
        f.argtypes = [vp, cu, vp, cu, vp] + ([ctypes.c_int] if layout is not None else [])
        rng = np.random.default_rng([7, di])
        streams = [(k, v) for k, v in base.items() if k.startswith("c%d_" % coder)]
        out = []
        for i in range(CASES_PER_DECODER):
            key, s = streams[i % len(streams)]
            n = int(base["n_" + key])
            s = s if i < len(streams) else mutate(rng, s, i % 4)
            cap = n if i < len(streams) or i % 3 else int(rng.integers(0, n + 1))
            pin, pout = libc.malloc(max(s.size, 1)), libc.malloc(max(cap, 1))
            ctypes.memmove(pin, s.ctypes.data, s.size)
            r = f(pin, s.size, pout, cap, None, *(() if layout is None else (layout,)))
            out.append([int(r), cap, key, i])
            libc.free(pin)
            libc.free(pout)
        results[name] = out
    json.dump(results, open(os.path.join(d, "results.json"), "w"))


def test_decoders_survive_corrupt_streams_under_sanitizers(tmp_path, gen, port):
    rt = sanitizer_runtimes()
    if rt is None:
        pytest.skip("no AddressSanitizer runtime (gcc -print-file-name=libasan.so)")
    build_lib()
    streams = {}
    for tag, a in (("text", port.bwt_encode(gen.text(2, 120000))[1]), ("text5", port.bwt_encode(gen.text(5, 60000))[1]), ("runs", np.repeat(
            np.random.default_rng(3).integers(0, 200, 2000, dtype=np.uint8), np.random.default_rng(4).integers(1, 60, 2000)))):
        for coder in (1, 2, 3):
            r, s = port.encode_block(a, coder=coder)
            assert r > 0, (tag, coder)
            streams["c%d_%s" % (coder, tag)] = s
            streams["n_c%d_%s" % (coder, tag)] = np.array(a.size)
    np.savez(tmp_path / "streams.npz", **streams)
    env = dict(os.environ, LD_PRELOAD=" ".join(rt), ASAN_OPTIONS="detect_leaks=0:abort_on_error=0",
               UBSAN_OPTIONS="print_stacktrace=1:halt_on_error=1")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], env=env, capture_output=True, text=True, timeout=1800)
    report = [l for l in p.stderr.splitlines() if "Sanitizer" in l or "runtime error" in l]
    assert p.returncode == 0 and not report, "sanitizer report or child failure (%d):\n%s" % (p.returncode, p.stderr[-6000:])
    results = json.load(open(tmp_path / "results.json"))
    bad = []
    for name, recs in results.items():
        assert len(recs) == CASES_PER_DECODER, name
        for r, cap, key, i in recs:
            if not (r in (-6, -5) or 0 <= r <= cap):
                bad.append("%s case %d (%s, out_cap %d): returned %d" % (name, i, key, cap, r))
            if i < 3 and r != cap:                       # the first three cases of a decoder are its valid streams
                bad.append("%s: the valid stream %s decodes to %d bytes, not %d" % (name, key, r, cap))
    assert not bad, "\n".join(bad[:20])


if __name__ == "__main__":
    child(sys.argv[1])
