#!/usr/bin/env python3
"""Product and Lanczos-step times of the 4 x 4 Hubbard torus at half filling (data/hubbard_square_4x4.yaml,
165 636 900 states) on one GPU: k_gather with sign masks, the queued k_pull ("mode" 1, "gather" 0) and the scatter form
("mode" 0) on the same context and the same seeded x, outputs compared; float64 and complex128.  The card's name and
power limit are read in the same run.  Usage: python tools/fermion_timing.py [steps]  (prints the log)"""
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from distributed_matvec_b200 import Operator, load_config_from_yaml  # noqa: E402


def timed(op, x, steps):
    op.matvec(x)   # warm-up: loads the instance, builds nothing further
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    y = None
    start.record()
    for _ in range(steps):
        y = op.matvec(x)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps, y


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"# {card}; {steps} products per figure after one warm-up, CUDA events")
    _, matrix = load_config_from_yaml(os.path.join(ROOT, "data", "hubbard_square_4x4.yaml"))
    op = Operator(matrix)
    t0 = time.perf_counter()
    op.basis.build()
    n = op.basis.numberStates()
    print(f"hubbard_square_4x4: {n} states, basis build {time.perf_counter() - t0:.2f} s, gather {op.info('gather')} "
          f"gather_signs {op.info('gather_signs')} index_mode {op.info('index_mode')} gather_narrow {op.info('gather_narrow')}")
    for cplx in (False, True):
        g = torch.Generator(device="cuda").manual_seed(5)
        x = torch.rand(n, dtype=torch.float64, device="cuda", generator=g) - 0.5
        if cplx:
            x = torch.complex(x, torch.rand(n, dtype=torch.float64, device="cuda", generator=g) - 0.5)
        op.use_torch_stream()
        results = {}
        for label, opts in (("k_gather", {}), ("k_pull", {"mode": 1, "gather": 0}), ("push", {"mode": 0})):
            for k, v in opts.items():
                op.set_option(k, v)
            ms, y = timed(op, x, steps)
            results[label] = y
            err = 0.0 if label == "k_gather" else float((y - results["k_gather"]).abs().max() /
                                                        results["k_gather"].abs().max())
            print(f"  {'complex128' if cplx else 'float64   '} {label:8s} {ms:9.2f} ms/product  {n / ms * 1e3:.3e} states/s"
                  f"  max rel diff to k_gather {err:.1e}")
            for k in opts:
                op.set_option(k, -1)
        del results
        torch.cuda.synchronize()
    for cplx in (False, True):
        for iters in (10, 40):
            t0 = time.perf_counter()
            op.lanczos(max_iters=iters, tol=0.0, complex_vectors=cplx, eigenvector=False)
            t = time.perf_counter() - t0
            if iters == 10:
                t10 = t
        print(f"  {'complex128' if cplx else 'float64   '} Lanczos: {(t - t10) / 30 * 1e3:.2f} ms per step "
              f"(difference of 40 and 10 steps)")
    op.close()


if __name__ == "__main__":
    main()
