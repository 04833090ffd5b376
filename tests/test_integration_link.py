"""INTEGRATION.md option 1, checked at link level: the reference's OWN CLI and block layer (bsc.cpp, libbsc.cpp) plus its host
stages (lzp, filters, adler32, platform) import from a stage library exactly the stage entry points the north star replaces --
bsc_{bwt,st,coder}_{init,encode/compress,decode/decompress} -- and libbsc_b200.so exports every one of them.  The imported set was
read with `nm -u` from the reference CLI linked against this library (tests/golden/make_reference_results.py)."""
import json
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "libbsc_b200", "libbsc_b200.so")


def test_reference_cli_links_against_the_stage_abi():
    assert os.path.exists(LIB), "run __graft_entry__.build() first"
    # what the reference's CLI, block layer and host stages left undefined when linked against this library (nm -u, stored)
    imported = set(json.load(open(os.path.join(ROOT, "tests", "golden", "reference_results.json")))["stage_symbols_imported_by_reference_cli"])
    assert imported
    nm = subprocess.run(["nm", "-D", "--defined-only", LIB], capture_output=True, text=True, check=True).stdout
    exported = {l.split()[-1] for l in nm.splitlines() if l.split()[-2:-1] == ["T"]}
    assert imported <= exported, imported - exported
