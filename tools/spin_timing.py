#!/usr/bin/env python3
"""What dmv_apply_spin costs on the 6 x 6 square: σᶻ_(π,π) from the k = 0 sector into the (π, π) sector of the whole
space group with odd point-group characters (sectors 3, 3, 1, 1, 2: (-1)^{x+y} changes sign under both mirrors and the
rotation) and opposite spin inversion, and σ⁻_(π,π) into that sector at weight 17, the sectors that hold all of O x.
Each run also reports |y|² / <x|O†O|x> (from zz_correlations / pm_correlations), which is 1 there.  Per element type:
the time per call (CUDA events over
repeated calls of the whole entry point), the time of k_spin_rows (torch.profiler, a run of its own), the source
look-ups per second against one product of the source; and one Lanczos step (a product) in the (π, π) target sector
against one in the source sector.  The target sector has non-trivial characters, so its products run on k_pull /
k_generate, not k_rows.  The card's name and power limit are read in the same run.

    python tools/spin_timing.py [--elts f64,c128] [--out LOG]

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
import yaml  # noqa: E402

from distributed_matvec_b200 import Operator  # noqa: E402
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict  # noqa: E402
from distributed_matvec_b200.spectral import fourier_weights  # noqa: E402
from zz_timing import card, event_ms  # noqa: E402


PIPI = (3, 3, 1, 1, 2)


def square_6x6(weight=18, sectors=(0, 0, 0, 0, 0), inversion=1):
    with open(os.path.join(ROOT, "data", "heisenberg_square_6x6.yaml"), encoding="utf-8") as f:
        d = yaml.safe_load(f)
    b = dict(d["basis"])
    b["hamming_weight"] = weight
    b["symmetries"] = [dict(g, sector=s) for g, s in zip(b["symmetries"], sectors)]
    b["spin_inversion"] = inversion
    basis = basis_from_dict(b)
    return Operator(operator_from_dict({"terms": d["hamiltonian"]["terms"]}, basis))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--elts", default="f64,c128")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    lines = [f"card: {name}, power limit {limit}"]
    result = {"card": name, "power_limit": limit, "runs": []}
    src = square_6x6()
    targets = {"z": square_6x6(sectors=PIPI, inversion=-1), "-": square_6x6(weight=17, sectors=PIPI, inversion=None)}
    for op in (src, *targets.values()):
        op.basis.build()
        op.use_torch_stream()
    n = src.basis.numberStates()
    reps = src.basis.representatives()
    w = fourier_weights(np.array([[s % 6, s // 6] for s in range(36)], dtype=float), [np.pi, np.pi]).real
    for elt in a.elts.split(","):
        dtype = torch.complex128 if elt == "c128" else torch.float64
        x = torch.rand(n, dtype=dtype, device="cuda") - (0.5 + 0.5j if elt == "c128" else 0.5)
        y = torch.zeros_like(x)
        src.matvec(x, y)
        product_ms = event_ms(lambda: src.matvec(x, y), 3)
        Cz, _ = src.zz_correlations(x)
        T = src.pm_correlations(x)
        x2 = float(torch.vdot(x, x).real)
        expect = {"z": float(w @ Cz @ w) * x2, "-": float((w @ T @ w).real) * x2}   # <x|O†O|x>
        for kind, tgt in targets.items():
            m = tgt.basis.numberStates()
            y = src.apply_spin(kind, w, x, tgt)                      # warm-up: module load, table, buffers
            captured = float(torch.vdot(y, y).real) / expect[kind]
            call_ms = event_ms(lambda: src.apply_spin(kind, w, x, tgt), a.reps)
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.reps):
                    src.apply_spin(kind, w, x, tgt)
                torch.cuda.synchronize()
            k_us = [ev.device_time for ev in prof.events() if ev.device_type.name == "CUDA" and "k_spin_rows" in ev.name]
            kernel_ms = sum(k_us) / a.reps / 1000.0
            t_reps = tgt.basis.representatives()[:: max(1, m // 100000)]
            per_row = 1.0 if kind == "z" else float(np.mean([36 - bin(int(r)).count("1") for r in t_reps]))
            lookups = per_row * m
            xt = torch.rand(m, dtype=dtype, device="cuda") - (0.5 + 0.5j if elt == "c128" else 0.5)
            yt = torch.zeros_like(xt)
            tgt.matvec(xt, yt)
            target_product_ms = event_ms(lambda: tgt.matvec(xt, yt), 3)
            run = {"kind": kind, "elt": elt, "source_n": n, "target_n": m, "call_ms": call_ms, "kernel_ms": kernel_ms,
                   "lookups": lookups, "lookups_per_s": lookups / (kernel_ms * 1e-3) if kernel_ms > 0 else None,
                   "source_product_ms": product_ms, "target_product_ms": target_product_ms,
                   "target_kernel": "rows" if tgt.info("rows") else ("gather" if tgt.info("gather") else "pull/push"),
                   "kernel_launches_profiled": len(k_us), "captured": captured}
            result["runs"].append(run)
            lines.append(f"σ{'ᶻ' if kind == 'z' else '⁻'}_(π,π) {elt}: source n = {n}, target n = {m}; call {call_ms:.2f} ms, "
                         f"k_spin_rows {kernel_ms:.2f} ms, {lookups:.3e} look-ups = {run['lookups_per_s'] or 0:.3e}/s; "
                         f"source product {product_ms:.2f} ms (call / product = {call_ms / product_ms:.2f}); "
                         f"target-sector product {target_product_ms:.2f} ms ({run['target_kernel']}, "
                         f"{target_product_ms / product_ms:.1f} x the source's); |y|² / <O†O> = {captured:.12f}")
    for op in (src, *targets.values()):
        op.close()
    text = "\n".join(lines + [json.dumps(result)])
    print(text, flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
