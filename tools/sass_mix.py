#!/usr/bin/env python3
"""tools/sass_mix.py -- per-kernel instruction mix of the built library's SASS (runs without a GPU): total instructions, TMA bulk copies
(UBLKCP) and mbarrier operations (SYNCS), 128- / 64-bit global loads and stores, match.any, shuffles.
    python tools/sass_mix.py > sass_instruction_mix.txt"""
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "libbsc_b200", "libbsc_b200.so")
PAT = {"total": r"^\s+/\*[0-9a-f]{4,6}\*/\s+\S", "UBLKCP": r"\bUBLKCP", "SYNCS": r"\bSYNCS", "LDG.128": r"\bLDG\.E(\.[A-Z]+)*\.128", "LDG.64": r"\bLDG\.E(\.[A-Z]+)*\.64",
       "STG.128": r"\bSTG\.E(\.[A-Z]+)*\.128", "STG.64": r"\bSTG\.E(\.[A-Z]+)*\.64", "MATCH": r"\bMATCH\.ANY", "SHFL": r"\bSHFL", "ATOMS": r"\bATOMS"}

sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
per, cur = collections.defaultdict(collections.Counter), None
for line in sass.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        cur = m.group(1)
        continue
    if cur:
        for k, p in PAT.items():
            if re.search(p, line):
                per[cur][k] += 1
names = list(per)
dem = subprocess.run(["cu++filt"] + names, capture_output=True, text=True).stdout.split("\n")
cols = ["total", "UBLKCP", "SYNCS", "LDG.128", "LDG.64", "STG.128", "STG.64", "MATCH", "SHFL", "ATOMS"]
print("SASS of libbsc_b200/libbsc_b200.so (sm_90a): instruction counts per kernel (cuobjdump -sass, tools/sass_mix.py); %d kernels" % len(names))
print("%-100s " % "kernel" + " ".join("%7s" % c for c in cols))
for n, d in sorted(zip(names, dem), key=lambda x: -per[x[0]]["total"]):
    short = re.sub(r"\((const |unsigned |<unnamed>::|void|int|short|DoneSignal|[\w\*&, ])*\)$", "", d).replace("<unnamed>::", "").replace("void ", "")[:98]
    print("%-100s " % short + " ".join("%7d" % per[n][c] for c in cols))
