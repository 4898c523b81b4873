#!/usr/bin/env python3
"""What dmv_zz_correlations costs: the time of k_zz_gram per vector (CUDA events over repeated calls of the whole entry
point, and torch.profiler under the kernel's name), the bytes it has to read, n (8 + E) per vector for the
representatives and x (E = 8 float64, 16 complex128), the padded DMMA FLOPs per second 2 RP CP n (RP = N + 1 rounded up
to 16, CP = N rounded up to 8), and beside them the time of one product on the same operator.  The card's name and
power limit are read in the same run.

    python tools/zz_timing.py [--models heisenberg_square_6x6:f64,heisenberg_square_6x6:c128,...] [--out LOG]

Prints a few lines and one JSON line; --out also writes them to LOG.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from distributed_matvec_b200 import Operator, load_config_from_yaml  # noqa: E402

DEFAULT = ("heisenberg_square_6x6:f64,heisenberg_square_6x6:c128,heisenberg_chain_36_symm:f64,"
           "heisenberg_chain_24:f64")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def event_ms(fn, reps):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(reps):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default=DEFAULT)
    ap.add_argument("--reps", type=int, default=20)
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
        E = 16 if kind == "c128" else 8
        x = torch.rand(n, dtype=dtype, device="cuda") - (0.5 + 0.5j if kind == "c128" else 0.5)
        y = torch.zeros_like(x)
        op.zz_correlations(x)                                   # warm-up: module load, buffers
        call_ms = event_ms(lambda: op.zz_correlations(x), a.reps)
        op.matvec(x, y)
        product_ms = event_ms(lambda: op.matvec(x, y), 3)
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.reps):
                op.zz_correlations(x)
            torch.cuda.synchronize()
        gram_us = [ev.device_time for ev in prof.events() if ev.device_type.name == "CUDA" and "k_zz_gram" in ev.name]
        reduce_us = [ev.device_time for ev in prof.events()
                     if ev.device_type.name == "CUDA" and "k_reduce_partials" in ev.name]
        kernel_ms = sum(gram_us) / max(len(gram_us), 1) / 1000.0
        reduce_ms = sum(reduce_us) / max(len(reduce_us), 1) / 1000.0
        RP, CP = 16 * ((N + 16) // 16), 8 * ((N + 7) // 8)
        flops = 2.0 * RP * CP * n
        nbytes = n * (8 + E)
        run = {"model": model, "elt": kind, "n": n, "sites": N, "call_ms": call_ms, "k_zz_gram_ms": kernel_ms,
               "k_reduce_partials_ms": reduce_ms, "bytes": nbytes, "GBps": nbytes / (kernel_ms * 1e-3) / 1e9,
               "padded_flops": flops, "TFLOPps": flops / (kernel_ms * 1e-3) / 1e12, "product_ms": product_ms,
               "kernel_launches_profiled": len(gram_us)}
        result["runs"].append(run)
        lines.append(f"{model} {kind}: n = {n}, N = {N}; call {call_ms:.3f} ms, k_zz_gram {kernel_ms:.3f} ms "
                     f"(+ k_reduce_partials {reduce_ms:.3f} ms); {nbytes / 1e9:.3f} GB read, "
                     f"{run['GBps']:.0f} GB/s; {RP} x {CP} padded block, {flops / 1e9:.1f} GFLOP, "
                     f"{run['TFLOPps']:.1f} TFLOP/s; one product {product_ms:.2f} ms")
    for other in ops.values():
        other.close()
    text = "\n".join(lines + [json.dumps(result)])
    print(text, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
