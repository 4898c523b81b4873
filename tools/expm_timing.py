#!/usr/bin/env python3
"""Where the time of dmv_expm_multiply goes: the product against orthogonalisation + combine, per Krylov step, and the
achieved bandwidth of k_block_dot / k_block_combine (bytes from the shapes: the library counts the vectors its block
kernels read or write, dmv_get_info "expm_dot_vectors" / "expm_combine_vectors").

    python tools/expm_timing.py [--model heisenberg_square_6x6] [--z -0.1j] [--krylov-dim 30] [--out LOG]

Wall time from CUDA events around the call; the per-kernel split from torch.profiler (CUPTI kernel records) of one more
call.  Prints a few lines and one JSON line; --out also writes them to LOG.
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

BLOCK = ("k_block_dot", "k_block_combine", "k_reduce_partials", "k_scale")


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="heisenberg_square_6x6")
    ap.add_argument("--z", default="-0.1j")
    ap.add_argument("--krylov-dim", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    z = complex(a.z)
    _, matrix = load_config_from_yaml(os.path.join(ROOT, "data", a.model + ".yaml"))
    op = Operator(matrix)
    op.basis.build()
    n = op.basis.numberStates()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.complex(torch.rand(n, dtype=torch.float64, device="cuda", generator=g) - 0.5,
                      torch.rand(n, dtype=torch.float64, device="cuda", generator=g) - 0.5)
    x /= torch.linalg.norm(x)
    op.expm_multiply(x, z * 0.1, krylov_dim=a.krylov_dim)          # warm-up: basis allocation, k_rows table
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(3):
        op.matvec(x)
    torch.cuda.synchronize()
    start.record()
    for _ in range(5):
        op.matvec(x)
    stop.record()
    torch.cuda.synchronize()
    product_ms = start.elapsed_time(stop) / 5
    start.record()
    y, prods, est = op.expm_multiply(x, z, krylov_dim=a.krylov_dim)
    stop.record()
    torch.cuda.synchronize()
    wall_ms = start.elapsed_time(stop)
    dot_vectors, combine_vectors = op.info("expm_dot_vectors"), op.info("expm_combine_vectors")
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        op.expm_multiply(x, z, krylov_dim=a.krylov_dim)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        key = next((b for b in BLOCK if b in ev.name), "product")
        per[key] = per.get(key, 0.0) + ev.device_time / 1000.0   # us -> ms
    orth_ms = sum(v for k, v in per.items() if k != "product")
    elt_bytes = 16
    dot_gbs = dot_vectors * n * elt_bytes / (per.get("k_block_dot", float("nan")) * 1e-3) / 1e9
    comb_gbs = combine_vectors * n * elt_bytes / (per.get("k_block_combine", float("nan")) * 1e-3) / 1e9
    name, limit = card()
    lines = [
        f"card: {name}, power limit {limit}",
        f"{a.model}: N = {n}, complex128, z = {z}, krylov_dim = {a.krylov_dim}",
        f"wall time {wall_ms:.1f} ms, {prods} products, error estimate {est:.2e}, |y| = {torch.linalg.norm(y).item():.15f}",
        f"product alone (CUDA events, 5 products): {product_ms:.2f} ms",
        f"per Krylov step (profiler kernel time): product {per.get('product', 0.0) / prods:.2f} ms, "
        f"orthogonalisation + combine {orth_ms / prods:.2f} ms "
        f"({100 * orth_ms / (orth_ms + per.get('product', 0.0)):.1f} % of the GPU time of a step)",
        "block kernels: " + ", ".join(f"{k} {per.get(k, 0.0):.1f} ms" for k in BLOCK),
        f"k_block_dot: {dot_vectors} vector reads, {dot_gbs:.0f} GB/s; "
        f"k_block_combine: {combine_vectors} vector reads + writes, {comb_gbs:.0f} GB/s",
        f"host time between kernels (wall - GPU kernel time): {wall_ms - orth_ms - per.get('product', 0.0):.1f} ms",
    ]
    result = {"model": a.model, "n": n, "z": str(z), "krylov_dim": a.krylov_dim, "wall_ms": wall_ms, "products": prods,
              "product_ms": product_ms, "kernel_ms": per, "dot_GBps": dot_gbs, "combine_GBps": comb_gbs,
              "card": name, "power_limit": limit}
    text = "\n".join(lines + [json.dumps(result)])
    print(text, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")
    op.close()


if __name__ == "__main__":
    main()
