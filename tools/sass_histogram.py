#!/usr/bin/env python3
"""SASS opcode histogram of libdmv_b200.so per kernel family (cuobjdump -sass), for profiles/: which memory / async /
integer instructions the shipped kernels are made of (UBLKCP = TMA bulk copy, LDG.E.256 = 256-bit loads, RED = FP64
atomics, LDGSTS = cp.async, ...).  Usage: python tools/sass_histogram.py > profiles/r02_sass_histogram.md"""
import collections
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "distributed_matvec_b200", "libdmv_b200.so")
out = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
fam = None
hist = collections.defaultdict(collections.Counter)
for line in out.splitlines():
    m = re.search(r"Function : (\S+)", line)
    if m:
        name = m.group(1)
        k = re.search(r"(k_[a-z_0-9]+?)I", name) or re.search(r"(k_[a-z_0-9]+)", name)
        fam = k.group(1) if k else "other"
        continue
    m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z][A-Z0-9_]*(?:\.[A-Z0-9_]+)*)", line)
    if m and fam:
        op = m.group(1)
        base = op.split(".")[0]
        key = op if base in ("LDG", "STG", "RED", "ATOMG", "ATOMS", "UBLKCP", "LDGSTS", "LDS", "STS", "SYNCS", "CCTL", "MEMBAR", "ST", "LD") else base
        hist[fam][key] += 1
print("# SASS opcode histogram of libdmv_b200.so (cuobjdump -sass, sm_90a), static instruction counts per kernel family\n")
interesting = ["UBLKCP", "SYNCS", "LDGSTS", "LDG", "STG", "ST", "RED", "ATOMG", "ATOMS", "LDS", "STS", "MEMBAR", "DFMA", "DMUL", "DADD",
               "IMAD", "LOP3", "SHF", "POPC", "FLO", "BREV", "ISETP", "VIMNMX", "SEL", "PRMT", "REDUX", "VOTE", "SHFL", "MATCH", "BAR"]
for f in sorted(hist):
    tot = sum(hist[f].values())
    print(f"## {f}  ({tot} instructions over all template instances)\n")
    rows = []
    for key, cnt in hist[f].most_common():
        if key.split(".")[0] in interesting:
            rows.append(f"`{key}` {cnt}")
    print(", ".join(rows[:40]) + "\n")
