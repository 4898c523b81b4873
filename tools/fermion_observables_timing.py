#!/usr/bin/env python3
"""What the single-particle observables of fermionic bases cost: the time per call of dmv_one_body_density_matrix and
of dmv_apply_fermion (c† and c of a Fourier mode into the neighbouring particle sectors), each beside one product of
the same operator, CUDA events over repeated calls after a warm-up.  The card's name and power limit are read in the
same run.

    python tools/fermion_observables_timing.py [--models hubbard_square_4x4,spinless_ring_28] [--reps 10] [--out LOG]

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
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict  # noqa: E402
from distributed_matvec_b200.spectral import fourier_weights  # noqa: E402
from gen_models import fermion_models  # noqa: E402
from zz_timing import card, event_ms  # noqa: E402


def sector(conf, d):
    """the model with one particle more (d = 1) or fewer (d = -1): in the up half of a spinful basis"""
    b = dict(conf["basis"])
    b["number_particles"] += d
    if b["particle"] == "spinful-fermion":
        b["number_up"] += d
    return Operator(operator_from_dict(conf["hamiltonian"], basis_from_dict(b)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="hubbard_square_4x4,spinless_ring_28")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    lines = [f"# {name}, {limit}; {a.reps} calls per figure after one warm-up, CUDA events"]
    results = {"card": name, "power_limit": limit, "models": {}}
    print(lines[0], flush=True)
    confs = fermion_models()
    for model in a.models.split(","):
        _, matrix = load_config_from_yaml(os.path.join(ROOT, "data", model + ".yaml"))
        conf = confs[model]
        op = Operator(matrix)
        op.basis.build()
        plus, minus = sector(conf, 1), sector(conf, -1)
        plus.basis.build()
        minus.basis.build()
        n = op.basis.numberStates()
        M = matrix.basis.number_bits
        n_sites = conf["basis"]["number_sites"]
        w = np.zeros(M, dtype=np.complex128)
        w[:n_sites] = fourier_weights(np.arange(n_sites), 2 * np.pi / n_sites)
        rng = np.random.default_rng(1)
        entry = {"states": n, "plus_states": plus.basis.numberStates(), "minus_states": minus.basis.numberStates()}
        head = (f"{model}: {n} states, c+ into {entry['plus_states']}, c into {entry['minus_states']} states, "
                f"{M} modes")
        lines.append(head)
        print(head, flush=True)
        for dtype in (torch.float64, torch.complex128):
            x = torch.from_numpy(rng.random(n) - 0.5).cuda().to(dtype)
            y = torch.zeros_like(x)
            ww = w if dtype == torch.complex128 else w.real.copy()
            calls = {
                "product": lambda: op.matvec(x, y),
                "one_body_density_matrix": lambda: op.one_body_density_matrix(x),
                "apply_fermion c+": lambda: op.apply_fermion("c+", ww, x, plus),
                "apply_fermion c": lambda: op.apply_fermion("c", ww, x, minus),
            }
            times = {}
            for what, fn in calls.items():
                fn()   # warm-up
                times[what] = event_ms(fn, a.reps)
            entry[str(dtype).replace("torch.", "")] = times
            line = f"  {str(dtype).replace('torch.', ''):10s} " + "  ".join(f"{k} {v:8.2f} ms" for k, v in times.items())
            lines.append(line)
            print(line, flush=True)
            del x, y
        results["models"][model] = entry
        for o in (plus, minus, op):
            o.close()
        torch.cuda.empty_cache()
    lines.append(json.dumps(results))
    print(lines[-1], flush=True)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
