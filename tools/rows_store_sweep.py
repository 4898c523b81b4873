#!/usr/bin/env python3
"""Time the row kernel on its term store (k_rows_stored, csrc/dmv_store.cu) against k_rows.

Configurations: k_rows (dmv_debug_rows_store mode 0), the store at every asked column count C (capped by the basis), and
the store as the cost model chooses it (auto).  They alternate in rounds; each product is timed with CUDA events, the L2
flushed before it.  Per configuration: median and range, the store's build time (first product after the switch, less
a timed product) and size, y against k_rows by bench.py's element criterion and whether it is identical to k_rows (it
must be at C = 1).  Every store of a workload is built from the same basis, so C is switched in the outer loop and the
rounds alternate over the store built last and k_rows.
Usage: python tools/rows_store_sweep.py [--rounds R] [--products K] [--chunks 1,2,...] [workload ...]"""
import argparse
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributed_matvec_b200 import Operator, load_config_from_yaml  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError as e:
        return f"nvidia-smi unavailable ({e})"


def violations(a, b):   # bench.py's criterion_violations, on the device
    return int(((a - b).abs() > torch.clamp(1e-12 * torch.maximum(a.abs(), b.abs()), min=1e-14)).sum())


def timed(op, xd, yd, flush, k):
    flush.fill_(k & 0xFF)
    s = torch.cuda.Event(enable_timing=True)
    e = torch.cuda.Event(enable_timing=True)
    s.record()
    op.matvec(xd, yd)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--products", type=int, default=4, help="timed products per configuration and round")
    ap.add_argument("--dtypes", default="c128,f64")
    ap.add_argument("--chunks", default="1,2,4,8,12,16,24,32,64")
    ap.add_argument("workloads", nargs="*", default=["heisenberg_square_6x6", "heisenberg_chain_32_symm",
                                                     "heisenberg_chain_36_symm"])
    args = ap.parse_args()
    print("card:", card(), flush=True)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device="cuda")
    for name in args.workloads:
        basis, matrix = load_config_from_yaml(os.path.join(ROOT, "data", name + ".yaml"))
        op = Operator(matrix)
        op.basis.build()
        n = op.basis.numberStates()
        op.use_torch_stream()
        print(f"== {name}: N={n}", flush=True)
        rng = np.random.default_rng(42)
        for dt in args.dtypes.split(","):
            cplx = dt == "c128"
            x = rng.random(n) - 0.5
            if cplx:
                x = x + 1j * (rng.random(n) - 0.5)
            xd = torch.from_numpy(x).cuda()
            yd = torch.zeros_like(xd)
            op.debug_rows_store(0)
            for _ in range(2):
                op.matvec(xd, yd)
            torch.cuda.synchronize()
            ref = yd.clone()
            rows_times = []
            stores = [(f"C={c}", 1, int(c)) for c in args.chunks.split(",") if c and int(c) <= n] + [("auto", -1, 0)]
            for label, mode, chunks in stores:
                op.debug_rows_store(mode, chunks)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                op.matvec(xd, yd)
                torch.cuda.synchronize()
                first_ms = 1e3 * (time.perf_counter() - t0)
                on = op.info("rows_store")
                times = []
                for r in range(args.rounds):   # alternate: the store, then k_rows
                    op.debug_rows_store(mode, chunks)
                    times += [timed(op, xd, yd, flush, k) for k in range(args.products)]
                    y = yd.clone()
                    op.debug_rows_store(0)
                    rows_times += [timed(op, xd, yd, flush, k) for k in range(args.products)]
                bad = violations(y, ref)
                same = bool(torch.equal(y, ref))
                t = np.array(times)
                print(f"  {dt:4s} {label:6s} store={on} chunks={op.info('rows_store_chunks'):3d} "
                      f"median {np.median(t):8.3f} ms  min {t.min():8.3f}  max {t.max():8.3f}  ({len(t)} products)  "
                      f"first product {first_ms:9.1f} ms  store {op.info('rows_store_mb')} MB "
                      f"({op.info('rows_store_terms')} terms)  violations {bad}  identical {same}", flush=True)
            t = np.array(rows_times)
            print(f"  {dt:4s} k_rows {'':19s} median {np.median(t):8.3f} ms  min {t.min():8.3f}  max {t.max():8.3f}  "
                  f"({len(t)} products, alternating with every store above)", flush=True)
            del xd, yd, ref
            op.debug_rows_store(-1)
        op.close()


if __name__ == "__main__":
    main()
