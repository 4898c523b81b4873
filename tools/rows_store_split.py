#!/usr/bin/env python3
"""Split the time of a product on the term store into gathers, streams and partial sums.

Times k_rows_stored on the 6x6 square at the asked column counts with three builds of the library: the shipped one,
one without the gathers (-DDMV_STORE_NO_GATHER: the entries are streamed, no x is read) and one without the partial
sums between passes (-DDMV_STORE_NO_PARTIAL).  The two measurement builds give wrong results on purpose; each runs in
its own process.  Shipped minus no-gather is the time of the gathers, shipped minus no-partial that of the partial sums.
Build the measurement libraries first: dmv_kernels.cu compiled with the macro, linked with the other objects of the
shipped build (NVCC flags of distributed_matvec_b200/build.py).
Usage: python tools/rows_store_split.py [--chunks 8,16] [--products 10] LIB_NO_GATHER LIB_NO_PARTIAL"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def run(lib, chunks, products):
    sys.path.insert(0, ROOT)
    import numpy as np
    import torch
    from distributed_matvec_b200 import build as lib_build
    if lib:
        lib_build.LIB = lib   # read by _native.lib() at the first call
    from distributed_matvec_b200 import Operator, load_config_from_yaml
    _, matrix = load_config_from_yaml(os.path.join(ROOT, "data", "heisenberg_square_6x6.yaml"))
    op = Operator(matrix)
    op.basis.build()
    n = op.basis.numberStates()
    op.use_torch_stream()
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    rng = np.random.default_rng(42)
    for dt in ("c128", "f64"):
        x = rng.random(n) - 0.5
        if dt == "c128":
            x = x + 1j * (rng.random(n) - 0.5)
        xd = torch.from_numpy(x).cuda()
        yd = torch.zeros_like(xd)
        for c in chunks:
            op.debug_rows_store(1, c)
            for _ in range(2):
                op.matvec(xd, yd)
            times = []
            for k in range(products):
                flush.fill_(k & 0xFF)
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                op.matvec(xd, yd)
                e.record()
                torch.cuda.synchronize()
                times.append(s.elapsed_time(e))
            t = np.array(times)
            print(f"  {dt:4s} C={c:3d} median {np.median(t):7.3f} ms  min {t.min():7.3f}  max {t.max():7.3f}", flush=True)
    op.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", default="8,16")
    ap.add_argument("--products", type=int, default=10)
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    ap.add_argument("libs", nargs="*")
    args = ap.parse_args()
    chunks = [int(c) for c in args.chunks.split(",")]
    if args.child is not None:
        run(args.child, chunks, args.products)
        return
    for label, lib in [("shipped", "")] + list(zip(("no gathers", "no partial sums"), args.libs)):
        print(f"== {label} {lib}", flush=True)
        subprocess.run([sys.executable, os.path.abspath(__file__), "--chunks", args.chunks, "--products",
                        str(args.products), "--child", lib], check=True)


if __name__ == "__main__":
    main()
