#!/usr/bin/env python3
"""Generates tests/golden/reference_results_st_large.json from the UNMODIFIED reference built by oracle/Makefile (oracle/_ref): for every
sort-transform block above 1 GiB of tests/large_st_inputs.py (ST_CASES) the size and SHA-256 of the input and of what the reference's
in-place bsc_compress returns for it, and the same for the file larger than 2 GiB and the archive the reference CLI writes for it at
`-b2047 -m6`.  The GPU test (tests/test_gpu_large_st_decode.py) compresses the same inputs with the reference on the host and checks its
blocks against these digests first, so that a different reference build shows up as such and not as a decoder bug.  Needs about 3 n
(6.5 GB) of host memory and 2.3 GB of temporary disk space; takes some minutes.
"""
import ctypes
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import pyoracle
import large_st_inputs as li


def digest(b):
    b = np.ascontiguousarray(b, dtype=np.uint8)
    return {"size": int(b.size), "sha256": hashlib.sha256(memoryview(b)).hexdigest()}


def main():
    gen, ref = pyoracle.Gen(), pyoracle.Ref()
    out = {"inplace": {}}
    for name, (make, sorter, lzp_hash, lzp_min, coder) in li.ST_CASES.items():
        a = make(gen)
        n = a.size
        buf = np.zeros(n + 28 + 64, dtype=np.uint8)
        buf[:n] = a
        t0 = time.time()
        r = ref.lib.bsc_compress(ctypes.c_void_p(buf.ctypes.data), ctypes.c_void_p(buf.ctypes.data), n, lzp_hash, lzp_min, sorter, coder, 3)
        assert r > 0, (name, r)
        out["inplace"][name] = {"input": digest(a), "block": digest(buf[:r])}
        print("%s: %d -> %d bytes in %.1f s" % (name, n, r, time.time() - t0), flush=True)
        del a, buf
    with tempfile.TemporaryDirectory() as d:
        path, arch = os.path.join(d, "in.bin"), os.path.join(d, "a.bsc")
        a = li.st_cli_input(gen)
        a.tofile(path)
        out["cli_input"] = digest(a)
        del a
        subprocess.check_call([os.path.join(ROOT, "oracle", "_ref", "bsc"), "e", path, arch] + li.ST_CLI_OPTS + ["-p", "-t"], stdout=subprocess.DEVNULL)
        out["cli_archive"] = digest(np.fromfile(arch, dtype=np.uint8))
    with open(os.path.join(HERE, "reference_results_st_large.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("ok")


if __name__ == "__main__":
    main()
