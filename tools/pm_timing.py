#!/usr/bin/env python3
"""What dmv_pm_correlations costs: the time per call (CUDA events over repeated calls of the whole entry point), the
time of its walk kernel (torch.profiler, k_pm_rows / k_pm_pairs), the antiparallel pairs it visits per second, and
beside them one product on the same operator with its off-diagonal terms per second.  The card's name and power limit
are read in the same run.

    python tools/pm_timing.py [--models heisenberg_square_6x6:f64,...] [--out LOG]

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
from zz_timing import card, event_ms  # noqa: E402

DEFAULT = ("heisenberg_square_6x6:f64,heisenberg_square_6x6:c128,heisenberg_chain_36_symm:f64,"
           "heisenberg_chain_24:f64")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default=DEFAULT)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    lines = [f"card: {name}, power limit {limit}"]
    result = {"card": name, "power_limit": limit, "runs": []}
    ops = {}
    for item in a.models.split(","):
        model, kind = item.split(":")
        if model not in ops:
            for other in ops.values():
                other.close()
            ops.clear()
            _, matrix = load_config_from_yaml(os.path.join(ROOT, "data", model + ".yaml"))
            ops[model] = Operator(matrix)
            ops[model].basis.build()
        op = ops[model]
        op.use_torch_stream()
        n, N = op.basis.numberStates(), op.spec.basis.number_sites
        dtype = torch.complex128 if kind == "c128" else torch.float64
        x = torch.rand(n, dtype=dtype, device="cuda") - (0.5 + 0.5j if kind == "c128" else 0.5)
        y = torch.zeros_like(x)
        op.pm_correlations(x)                                   # warm-up: module load, table, buffers
        call_ms = event_ms(lambda: op.pm_correlations(x), a.reps)
        op.matvec(x, y)
        product_ms = event_ms(lambda: op.matvec(x, y), 3)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                op.pm_correlations(x)
            torch.cuda.synchronize()
        walk_us = [ev.device_time for ev in prof.events() if ev.device_type.name == "CUDA" and "k_pm_" in ev.name]
        walk_ms = sum(walk_us) / a.reps / 1000.0
        reps = op.basis.representatives()
        weights = np.array([bin(int(r)).count("1") for r in reps[:: max(1, n // 100000)]])
        pairs = float(np.mean(weights * (N - weights))) * n          # antiparallel pairs of the rows
        run = {"model": model, "elt": kind, "n": n, "sites": N, "call_ms": call_ms, "walk_ms": walk_ms,
               "pairs": pairs, "pairs_per_s": pairs / (walk_ms * 1e-3) if walk_ms > 0 else None,
               "product_ms": product_ms, "walk_launches_profiled": len(walk_us)}
        result["runs"].append(run)
        lines.append(f"{model} {kind}: n = {n}, N = {N}; call {call_ms:.2f} ms, walk {walk_ms:.2f} ms, "
                     f"{pairs:.3e} pairs = {run['pairs_per_s'] or 0:.3e} pairs/s; one product {product_ms:.2f} ms "
                     f"(call / product = {call_ms / product_ms:.1f})")
    for other in ops.values():
        other.close()
    text = "\n".join(lines + [json.dumps(result)])
    print(text, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
