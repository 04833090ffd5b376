#!/usr/bin/env python3
"""Generates tests/golden/reference_results.json from the UNMODIFIED reference built by oracle/Makefile (oracle/_ref): the size and
SHA-256 of what the reference returns for the inputs of the GPU tests that compare against it beyond the small fixtures of
make_golden.py -- blocks made with its default LZP stage, in-place calls, 64 MiB degenerate blocks, its CLI's archive -- and the
stage entry points its own CLI and block layer import from a stage library.  The GPU tests compare with these digests, so they
need neither the reference sources nor oracle/_ref.  Inputs come from the seeded generators (tools/bscgen.c) through
tests/reference_inputs.py, the same module the tests use.
"""
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
from oracle import pyoracle
import reference_inputs as ri


def digest(b):
    b = np.ascontiguousarray(b, dtype=np.uint8)
    return {"size": int(b.size), "sha256": hashlib.sha256(b.tobytes()).hexdigest()}


def main():
    gen, ref = pyoracle.Gen(), pyoracle.Ref()
    out = {"lzp": {}, "inplace": {}, "degenerate": {}}
    for name, a in ri.lzp_inputs(gen).items():
        for feats in (3, 1):
            z, b = ref.compress_lzp(a, 15, 128, 1, 1, feats)
            assert z > 0
            out["lzp"]["%s/f%d" % (name, feats)] = digest(b)
    for name, (a, sorter) in ri.inplace_inputs(gen).items():
        n = a.size
        buf = np.zeros(n + 28 + 64, dtype=np.uint8); buf[:n] = a
        r = ref.lib.bsc_compress(ctypes.c_void_p(buf.ctypes.data), ctypes.c_void_p(buf.ctypes.data), n, 0, 0, sorter, 1, 3)
        assert r > 0
        out["inplace"][name] = digest(buf[:r])
    for name, a in ri.degenerate_inputs().items():
        r, L, aux = ref.bwt_encode(a)
        z, blk = ref.compress(a, 1, 1, 3)
        out["degenerate"][name] = {"index": int(r), "aux": [int(x) for x in aux], "L": digest(L), "block": digest(blk)}
    with tempfile.TemporaryDirectory() as d:
        path, arch = os.path.join(d, "in.bin"), os.path.join(d, "a.bsc")
        ri.cli_input(gen).tofile(path)
        subprocess.check_call([os.path.join(ROOT, "oracle", "_ref", "bsc"), "e", path, arch] + ri.CLI_OPTS + ["-p", "-t"], stdout=subprocess.DEVNULL)
        out["cli_archive"] = digest(np.fromfile(arch, dtype=np.uint8))
    nm = subprocess.run(["nm", "-u", os.path.join(ROOT, "oracle", "_ref", "bsc_dropin")], capture_output=True, text=True, check=True).stdout
    out["stage_symbols_imported_by_reference_cli"] = sorted(l.split()[-1] for l in nm.splitlines() if " U bsc" in l)
    with open(os.path.join(HERE, "reference_results.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("ok")


if __name__ == "__main__":
    main()
