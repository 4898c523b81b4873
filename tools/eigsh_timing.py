#!/usr/bin/env python3
"""Where the time of dmv_eigsh goes: per restart cycle, the products against the block kernels (Gram / update),
the in-place rotation and the host; the achieved bandwidth of k_block_rotate and of the R > 1 Gram / update kernels
(bytes from the shapes: the library counts the vectors its block kernels read or write, dmv_get_info
"eigsh_block_vectors" / "eigsh_rotate_vectors"); and products per second at block sizes 1, 2, 4 and 6, both inside
the solver and for dmv_matvec_batch alone.

    python tools/eigsh_timing.py [--model heisenberg_square_6x6] [--nev 4] [--out LOG]

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

GRAM = ("k_block_gram", "k_block_update", "k_reduce_partials", "k_scale", "k_fill")
ROTATE = ("k_block_rotate",)


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="heisenberg_square_6x6")
    ap.add_argument("--nev", type=int, default=4)
    ap.add_argument("--tol", type=float, default=1e-10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    _, matrix = load_config_from_yaml(os.path.join(ROOT, "data", a.model + ".yaml"))
    op = Operator(matrix)
    op.basis.build()
    n = op.basis.numberStates()
    elt_bytes = 8
    name, limit = card()
    lines = [f"card: {name}, power limit {limit}", f"{a.model}: N = {n}, float64, nev = {a.nev}, tol = {a.tol:g}"]
    result = {"model": a.model, "n": n, "nev": a.nev, "tol": a.tol, "card": name, "power_limit": limit, "blocks": {}}
    X = torch.rand((6, n), dtype=torch.float64, device="cuda") - 0.5
    for p in (1, 2, 4, 6):
        op.eigsh(a.nev, block_size=p, tol=1e-2, max_restarts=0, eigenvectors=False)   # warm-up: basis, k_rows table
        (vals, _, res, conv, prods, rst), wall = timed(lambda: op.eigsh(a.nev, block_size=p, tol=a.tol,
                                                                         eigenvectors=False))
        Y = torch.zeros((p, n), dtype=torch.float64, device="cuda")
        op.matvec_batch(X[:p], Y)
        _, batch_ms = timed(lambda: [op.matvec_batch(X[:p], Y.zero_()) for _ in range(3)])
        batch_ms /= 3
        block_vectors, rotate_vectors = op.info("eigsh_block_vectors"), op.info("eigsh_rotate_vectors")
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            op.eigsh(a.nev, block_size=p, tol=a.tol, eigenvectors=False)
            torch.cuda.synchronize()
        per = {"product": 0.0, "gram_update": 0.0, "rotate": 0.0, "other": 0.0}
        gram_update_only = 0.0
        for ev in prof.events():
            if ev.device_type.name != "CUDA":
                continue
            ms = ev.device_time / 1000.0
            if any(k in ev.name for k in ROTATE):
                per["rotate"] += ms
            elif any(k in ev.name for k in GRAM):
                per["gram_update"] += ms
                if "k_block_gram" in ev.name or "k_block_update" in ev.name:
                    gram_update_only += ms
            elif ev.name.startswith("k_") or "dmv" in ev.name or "::" in ev.name:
                per["product"] += ms
            else:
                per["other"] += ms   # memset / memcpy
        cycles = rst + 1
        kernel_ms = sum(per.values())
        host_ms = wall - kernel_ms
        rot_gbs = rotate_vectors * n * elt_bytes / (per["rotate"] * 1e-3) / 1e9 if per["rotate"] else float("nan")
        gu_gbs = block_vectors * n * elt_bytes / (gram_update_only * 1e-3) / 1e9 if gram_update_only else float("nan")
        lines += [
            f"block {p}: {conv}/{a.nev} converged, theta = {', '.join(f'{v:.9f}' for v in vals)}, {prods} products, "
            f"{rst} restarts, wall {wall:.0f} ms",
            f"  per restart cycle: {wall / cycles:.0f} ms = products {per['product'] / cycles:.0f} ms + Gram / update "
            f"{per['gram_update'] / cycles:.1f} ms + rotation {per['rotate'] / cycles:.1f} ms + copies "
            f"{per['other'] / cycles:.1f} ms + host {host_ms / cycles:.1f} ms",
            f"  bandwidth: k_block_gram + k_block_update {block_vectors} vectors, {gu_gbs:.0f} GB/s; k_block_rotate "
            f"{rotate_vectors} vectors, {rot_gbs:.0f} GB/s",
            f"  products per second: {1000 * prods / wall:.1f} in the solver, "
            f"{1000 * p / batch_ms:.1f} for dmv_matvec_batch of {p} alone ({batch_ms:.1f} ms per batch)",
        ]
        result["blocks"][p] = {"eigenvalues": list(map(float, vals)), "converged": conv, "products": prods,
                               "restarts": rst, "wall_ms": wall, "kernel_ms": per, "host_ms": host_ms,
                               "gram_update_GBps": gu_gbs, "rotate_GBps": rot_gbs,
                               "solver_products_per_s": 1000 * prods / wall, "batch_products_per_s": 1000 * p / batch_ms}
    text = "\n".join(lines + [json.dumps(result)])
    print(text, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")
    op.close()


if __name__ == "__main__":
    main()
