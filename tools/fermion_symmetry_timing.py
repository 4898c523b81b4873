#!/usr/bin/env python3
"""Time per product in fermionic symmetry sectors against the unsymmetrised product, on one GPU: the 4 x 4 Hubbard torus
at half filling (data/hubbard_square_4x4_symm.yaml, momentum (0, 0), and (1, 0)) and the spinless ring of 28 sites at 14
particles (data/spinless_ring_28_symm.yaml, momentum 0, and 1).  Each sector runs the scatter form (k_generate, "mode"
0, the default) and the queued row form (k_pull, "mode" 1) on the same seeded x, outputs compared; the unsymmetrised
basis runs its default (k_gather).  float64 (real sectors) and complex128.  The card's name and power limit are read in
the same run.  Usage: python tools/fermion_symmetry_timing.py [steps] > profiles/h100_fermion_symmetry_timing.log"""
import os
import subprocess
import sys
import time

import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from distributed_matvec_b200 import Operator  # noqa: E402
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict  # noqa: E402


def timed(op, x, steps):
    op.matvec(x)   # warm-up
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    y = None
    start.record()
    for _ in range(steps):
        y = op.matvec(x)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps, y


def model(name, sectors=None):
    with open(os.path.join(ROOT, "data", name + ".yaml"), encoding="utf-8") as f:
        conf = yaml.safe_load(f)
    if sectors is not None:
        for g, k in zip(conf["basis"]["site_symmetries"], sectors):
            g["sector"] = k
    basis = basis_from_dict(conf["basis"])
    return operator_from_dict(conf["hamiltonian"], basis)


def vector(n, cplx):
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.rand(n, dtype=torch.float64, device="cuda", generator=g) - 0.5
    if cplx:
        x = torch.complex(x, torch.rand(n, dtype=torch.float64, device="cuda", generator=g) - 0.5)
    return x


def run(label, spec, steps, kinds, forms):
    op = Operator(spec)
    t0 = time.perf_counter()
    op.basis.build()
    n = op.basis.numberStates()
    print(f"{label}: {n} states, basis build {time.perf_counter() - t0:.2f} s")
    op.use_torch_stream()
    out = {}
    for cplx in kinds:
        x = vector(n, cplx)
        first = None
        for form, opts in forms:
            for k, v in opts.items():
                op.set_option(k, v)
            ms, y = timed(op, x, steps)
            err = 0.0 if first is None else float((y - first).abs().max() / first.abs().max())
            first = y if first is None else first
            print(f"  {'complex128' if cplx else 'float64   '} {form:9s} {ms:9.2f} ms/product  {n / ms * 1e3:.3e} states/s"
                  f"  max rel diff to the first form {err:.1e}")
            out[(cplx, form)] = ms
            for k in opts:
                op.set_option(k, -1)
        del first, x
        torch.cuda.synchronize()
    op.close()
    return out


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 20
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print(f"# {card}; {steps} products per figure after one warm-up, CUDA events")
    sector_forms = [("push", {"mode": 0}), ("k_pull", {"mode": 1})]
    for full, symm, real_sector, complex_sector in (("hubbard_square_4x4", "hubbard_square_4x4_symm", [0, 0], [1, 0]),
                                                    ("spinless_ring_28", "spinless_ring_28_symm", [0], [1])):
        base = run(full, model(full), steps, (False, True), [("default", {})])
        for sectors, kinds in ((real_sector, (False, True)), (complex_sector, (True,))):
            res = run(f"{symm} sector {sectors}", model(symm, sectors), steps, kinds, sector_forms)
            for cplx in kinds:
                best = min(res[(cplx, f)] for f, _ in sector_forms)
                print(f"  {'complex128' if cplx else 'float64   '} unsymmetrised / best sector form: "
                      f"{base[(cplx, 'default')] / best:.2f}x per product")


if __name__ == "__main__":
    main()
