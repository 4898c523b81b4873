#!/usr/bin/env python3
"""What dmv_reduced_density_matrix costs: chain_32_symm (sites 0 ... ℓ - 1, ℓ = 12 and 16) and the 6 x 6 square (a strip
of 12 sites, the first two rows), on a seeded random vector of the model's sector.  Per run: the time per call (CUDA
events over repeated calls of the whole entry point, after a warm-up call), its spread over the repeats, the times of
k_rdm_fill and k_rdm_gram (torch.profiler, a run of its own), the full-space amplitudes filled per second against the
off-diagonal look-ups per second of one product on the same context, and the Gram's real FP64 multiply-adds per second
(info "rdm_gram_flops" over the k_rdm_gram time) as a share of the H100 SXM data sheet's FP64 tensor-core rate
(67 TFLOP/s, 33.5e12 multiply-adds per second, for a card allowed 700 W).  The card's name and power limit are read in
the same run.

    python tools/entanglement_timing.py [--elts f64,c128] [--reps 5] [--out LOG]

Prints a few lines and one JSON line; --out also writes them to LOG.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from distributed_matvec_b200 import Operator, load_config_from_yaml  # noqa: E402
from zz_timing import card  # noqa: E402

FP64_TC_FMA_PER_S = 33.5e12
CASES = [("heisenberg_chain_32_symm", list(range(12))), ("heisenberg_chain_32_symm", list(range(16))),
         ("heisenberg_square_6x6", list(range(12)))]


def lookups_per_product(op, path):
    """off-diagonal terms of one product: antiparallel bonds of every representative, from a sample of them"""
    import yaml
    with open(path, encoding="utf-8") as f:
        d = yaml.safe_load(f)
    bonds = {tuple(s) for t in d["hamiltonian"]["terms"] if "σˣ₀" in t.get("expression", "") for s in t["sites"]}
    reps = op.basis.representatives()
    sample = reps[:: max(1, reps.shape[0] // 200000)]
    per = np.mean([sum(((int(r) >> i) ^ (int(r) >> j)) & 1 for i, j in bonds) for r in sample[:20000]])
    return per * reps.shape[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elts", default="f64,c128")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    lines = [f"card: {name}, power limit {limit}"]
    result = {"card": name, "power_limit": limit, "runs": []}
    ops = {}
    for model, sites in CASES:
        path = os.path.join(ROOT, "data", model + ".yaml")
        if model not in ops:
            _, spec = load_config_from_yaml(path)
            op = Operator(spec)
            op.basis.build()
            op.use_torch_stream()
            ops[model] = (op, lookups_per_product(op, path))
        op, lookups = ops[model]
        n = op.basis.numberStates()
        for elt in a.elts.split(","):
            dtype = torch.complex128 if elt == "c128" else torch.float64
            g = torch.Generator(device="cuda").manual_seed(5)
            x = torch.rand(n, dtype=dtype, device="cuda", generator=g) - (0.5 + 0.5j if elt == "c128" else 0.5)
            y = torch.zeros_like(x)
            op.matvec(x, y)
            torch.cuda.synchronize()
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(3):
                op.matvec(x, y)
            stop.record()
            torch.cuda.synchronize()
            product_ms = start.elapsed_time(stop) / 3
            op.reduced_density_matrix(x, sites)   # warm-up: module load, table, buffers
            torch.cuda.synchronize()
            times = []
            for _ in range(a.reps):
                start.record()
                rho = op.reduced_density_matrix(x, sites)
                stop.record()
                torch.cuda.synchronize()
                times.append(start.elapsed_time(stop))
            amplitudes, flops = op.info("rdm_amplitudes"), op.info("rdm_gram_flops")
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                op.reduced_density_matrix(x, sites)
                torch.cuda.synchronize()
            kern = {k: sum(ev.device_time for ev in prof.events() if ev.device_type.name == "CUDA" and k in ev.name) / 1e3
                    for k in ("k_rdm_fill", "k_rdm_gram", "k_rdm_reduce")}
            trace = sum(np.trace(r).real for r in rho.values())
            call_ms = float(np.median(times))
            run = {"model": model, "n_a": len(sites), "elt": elt, "n": n, "call_ms": call_ms,
                   "call_ms_min": min(times), "call_ms_max": max(times), "kernel_ms": kern,
                   "amplitudes": amplitudes, "amplitudes_per_s": amplitudes / (kern["k_rdm_fill"] * 1e-3),
                   "product_ms": product_ms, "product_lookups": lookups,
                   "product_lookups_per_s": lookups / (product_ms * 1e-3), "gram_fma": flops,
                   "gram_fma_per_s": flops / (kern["k_rdm_gram"] * 1e-3),
                   "gram_share_of_fp64_tc": flops / (kern["k_rdm_gram"] * 1e-3) / FP64_TC_FMA_PER_S, "trace": trace}
            result["runs"].append(run)
            lines.append(f"{model} |A| = {len(sites)} {elt}: n = {n}; call {call_ms:.1f} ms (min {min(times):.1f}, max "
                         f"{max(times):.1f}); k_rdm_fill {kern['k_rdm_fill']:.1f} ms = {run['amplitudes_per_s']:.3e} "
                         f"amplitudes/s ({amplitudes:.3e}); product {product_ms:.2f} ms = "
                         f"{run['product_lookups_per_s']:.3e} look-ups/s; k_rdm_gram {kern['k_rdm_gram']:.1f} ms = "
                         f"{run['gram_fma_per_s']:.3e} FMA/s = {100 * run['gram_share_of_fp64_tc']:.1f} % of the FP64 "
                         f"tensor-core data-sheet rate; k_rdm_reduce {kern['k_rdm_reduce']:.1f} ms; Tr ρ - 1 = {trace - 1:.1e}")
    for op, _ in ops.values():
        op.close()
    text = "\n".join(lines + [json.dumps(result)])
    print(text, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
