"""Build recipe of libdmv_b200.so: nvcc for sm_90a (H100), in-tree next to the package."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libdmv_b200.so")
SOURCES = ["dmv_kernels.cu", "dmv_gather.cu", "dmv_solver.cu", "dmv_group.cu", "dmv_api.cu", "dmv_exchange.cu",
           "dmv_lanczos.cu", "dmv_krylov.cu", "dmv_eigsh.cu", "dmv_observe.cu", "dmv_thermal.cu", "dmv_plugin.cu", "dmv_store.cu"]
HEADERS = ["dmv_device.cuh", "dmv_host.h", "dmv_context.h", "dmv_dense.h", "dmv_solve.h", os.path.join("..", "..", "include", "dmv_b200.h")]
ARCH = "arch=compute_90a,code=sm_90a"
NVCC_FLAGS = ["-gencode", ARCH, "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "--expt-relaxed-constexpr"]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    if os.environ.get("DMV_NO_REBUILD"):      # development runs on the GPU box: use the shipped library as it is
        return False
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    objs = []
    procs = []
    for src in SOURCES:
        obj = os.path.join(CSRC, src.replace(".cu", ".o"))
        cmd = ["nvcc", *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        procs.append((cmd, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for cmd, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stdout.write(out.decode())
        if p.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd))
    tmp = f"{LIB}.tmp{os.getpid()}"   # link into a private file, then rename: a reader never sees a half-written library
    link = ["nvcc", "-gencode", ARCH, "-shared", "-o", tmp, *objs, "-lcudart", "-ldl"]
    try:
        subprocess.run(link, check=True)
        os.replace(tmp, LIB)
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
