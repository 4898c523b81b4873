#!/usr/bin/env python3
"""Registers / stack (spill) bytes / static shared memory of every kernel instance in libdmv_b200.so
(cuobjdump -res-usage; no GPU needed), for profiles/: the static side of the occupancy figures quoted in DESIGN.md
(k_rows at 80 registers = three CTAs of 256 threads per SM, ...).  Usage: python tools/resource_usage.py > profiles/r02_resource_usage.md"""
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "distributed_matvec_b200", "libdmv_b200.so")


def demangle(names):
    out = subprocess.run(["cu++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return out if len(out) == len(names) else names


def short(name: str) -> str:
    name = re.sub(r"^void ", "", name)
    name = re.sub(r"\(dmv::host::Projection\)|\(dmv::Projection\)|\(int\)|\(bool\)", "", name)
    name = re.sub(r"dmv::host::|dmv::|<unnamed>::|\(anonymous namespace\)::", "", name)
    name = re.sub(r"\(.*\)$", "", name)     # the argument list
    return name


def main():
    text = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    rows, fn = [], None
    for line in text.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:(\d+)", line)
        if m and fn:
            rows.append((fn, int(m.group(1)), int(m.group(2)), int(m.group(3))))
            fn = None
    names = demangle([r[0] for r in rows])
    print("# Static resources of the kernels in libdmv_b200.so (cuobjdump -res-usage, sm_90a)\n")
    print("Registers per thread, stack bytes per thread (spills + local arrays) and STATIC shared memory; the dynamic shared "
          "memory (operator / orbit tables) comes from `smem_layout` at launch. 256 threads per CTA: 80 registers = 3 CTAs "
          "per SM, 128 = 2, 64 = 4 (65 536 registers per SM).\n")
    print("Template arguments: `k_rows<CE (complex128 elements), TK (side of the square torus whose canonical form is "
          "unrolled, 0 = generic), MPH (dense index), CTAS>`, `k_rows_batch<TK, CTAS>`, `k_generate<PROJ (0 none, 1 inversion, "
          "2 group), CV (complex coefficients), CE, COUNT_ONLY>`, `k_pull / k_accumulate<PROJ, CV, CE>`, "
          "`k_gather<INV, CV, CE, NARROW, LIN, UNI, KB>`.\n")
    fam = {}
    for (mangled, reg, stack, shared), name in zip(rows, names):
        s = short(name)
        k = re.match(r"(k_\w+)", s)
        fam.setdefault(k.group(1) if k else "other", []).append((s, reg, stack, shared))
    for f in sorted(fam):
        inst = fam[f]
        print(f"## {f} ({len(inst)} instance{'s' if len(inst) != 1 else ''})\n")
        if len(inst) > 24:
            regs = sorted(i[1] for i in inst)
            stacks = sorted(i[2] for i in inst)
            print(f"registers {regs[0]} .. {regs[-1]} (median {regs[len(regs) // 2]}), stack {stacks[0]} .. {stacks[-1]} bytes "
                  f"(median {stacks[len(stacks) // 2]}), static shared {max(i[3] for i in inst)} bytes\n")
            continue
        print("| instance | registers | stack bytes | static shared |\n|---|---|---|---|")
        for s, reg, stack, shared in sorted(inst):   # by name: the tables do not follow the host's instantiation order
            print(f"| `{s}` | {reg} | {stack} | {shared} |")
        print()


if __name__ == "__main__":
    main()
