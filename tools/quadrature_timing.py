#!/usr/bin/env python3
"""Where the time of dmv_lanczos_quadrature goes: per Lanczos step, the batched product against the two fused kernels
(k_quad_dot, k_quad_update, with their k_reduce_partials) and the host gap; the achieved bandwidth of the two kernels
(bytes from the shapes: k_quad_dot reads 2 G vectors, k_quad_update reads 3 G and writes G); and products per second
for R = 1, 2, 4, 6 start vectors (group G = min(R, the width one batched product shares)) against single
dmv_local_matvec calls.

    python tools/quadrature_timing.py [--steps 12] [--out LOG]

Runs the 6 x 6 square in float64 and complex128 and chain_24 in float64.  Wall time from CUDA events around the call;
the per-kernel split from torch.profiler (CUPTI kernel records) of one more call.  Prints a few lines and one JSON line;
--out also writes them to LOG.
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

WORKLOADS = [("heisenberg_square_6x6", False), ("heisenberg_square_6x6", True), ("heisenberg_chain_24", False)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def timed(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    out = fn()
    stop.record()
    torch.cuda.synchronize()
    return out, start.elapsed_time(stop)


def split(op, R, M, cplx):
    """per-kernel times (ms, whole call) of one call from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        op.lanczos_quadrature(R, M, complex_vectors=cplx)
        torch.cuda.synchronize()
    per = {"product": 0.0, "quad_dot": 0.0, "quad_update": 0.0, "reduce": 0.0, "other": 0.0}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        ms = ev.device_time / 1000.0
        if "k_quad_dot" in ev.name:
            per["quad_dot"] += ms
        elif "k_quad_update" in ev.name:
            per["quad_update"] += ms
        elif "k_reduce_partials" in ev.name or "k_quad_fill" in ev.name:
            per["reduce"] += ms
        elif ev.name.startswith("k_") or "dmv" in ev.name or "::" in ev.name:
            per["product"] += ms
        else:
            per["other"] += ms   # memset / memcpy
    return per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=12)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    M = a.steps
    name, limit = card()
    lines = [f"card: {name}, power limit {limit}; {M} Lanczos steps per call"]
    result = {"card": name, "power_limit": limit, "steps": M, "workloads": []}
    for model, cplx in WORKLOADS:
        _, matrix = load_config_from_yaml(os.path.join(ROOT, "data", model + ".yaml"))
        op = Operator(matrix)
        op.basis.build()
        n = op.basis.numberStates()
        elt = 2 if cplx else 1
        vec_bytes = n * 8 * elt
        dtype = torch.complex128 if cplx else torch.float64
        x = torch.ones(n, dtype=dtype, device="cuda")
        y = torch.zeros_like(x)
        op.matvec(x, y)
        _, single_ms = timed(lambda: [op.matvec(x, y) for _ in range(5)])
        single_ms /= 5
        lines.append(f"{model} {'complex128' if cplx else 'float64'}: N = {n}, one dmv_local_matvec {single_ms:.2f} ms "
                     f"({1000 / single_ms:.1f} products/s)")
        entry = {"model": model, "complex": cplx, "n": n, "single_ms": single_ms, "runs": {}}
        for R in (1, 2, 4, 6):
            op.lanczos_quadrature(R, 2, complex_vectors=cplx)   # warm-up: buffers, k_rows tables
            (_, _, _, prods), wall = timed(lambda: op.lanczos_quadrature(R, M, complex_vectors=cplx))
            G = op.info("quadrature_group")
            per = split(op, R, M, cplx)
            kernel_ms = sum(per.values())
            groups = -(-R // G)
            steps = groups * M
            dot_gbs = (2 * R * M * vec_bytes) / (per["quad_dot"] * 1e-3) / 1e9
            upd_gbs = (4 * R * (M - 1) * vec_bytes) / (per["quad_update"] * 1e-3) / 1e9
            lines += [
                f"  R = {R} (G = {G}): {prods} products in {wall:.1f} ms = {1000 * prods / wall:.1f} products/s "
                f"({1000 * prods / wall * single_ms / 1000:.2f}x single products)",
                f"    per step of a group: {wall / steps:.2f} ms = product {per['product'] / steps:.2f} + k_quad_dot "
                f"{per['quad_dot'] / steps:.3f} + k_quad_update {per['quad_update'] / steps:.3f} + reductions / fill "
                f"{per['reduce'] / steps:.3f} + copies {per['other'] / steps:.3f} + host gap "
                f"{(wall - kernel_ms) / steps:.3f} ms",
                f"    bandwidth: k_quad_dot {dot_gbs:.0f} GB/s, k_quad_update {upd_gbs:.0f} GB/s",
            ]
            entry["runs"][R] = {"group": G, "products": prods, "wall_ms": wall, "kernel_ms": per,
                                "host_gap_ms_per_step": (wall - kernel_ms) / steps, "products_per_s": 1000 * prods / wall,
                                "quad_dot_GBps": dot_gbs, "quad_update_GBps": upd_gbs}
        result["workloads"].append(entry)
        op.close()
    text = "\n".join(lines + [json.dumps(result)])
    print(text, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
