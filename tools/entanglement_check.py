#!/usr/bin/env python3
"""dmv_reduced_density_matrix across ranks (one process per rank, NCCL inside libdmv_b200) against the one-rank result.
With fewer GPUs than ranks, ranks share devices (round robin), as in tools/spin_check.py.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29563 tools/entanglement_check.py

A seeded random vector over the whole basis is cut into the ranks' hashed blocks (each rank takes the entries of its own
representatives); the collective call must give the one-rank ρ_A to 1e-12, for float64 and complex128 and for a batch
of two, and every rank must return the same ρ bit for bit.  Each line ends in OK or FAIL; used by
tests/test_entanglement.py.
"""
import numpy as np
import torch
import torch.distributed as dist

from rank_harness import Ranks
from distributed_matvec_b200 import DistributedOperator, Operator
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict


def ring(n, weight, sector, reflection=None, inversion=None, tfim=False):
    sym = [] if sector is None else [{"permutation": [(i + 1) % n for i in range(n)], "sector": sector}]
    if reflection is not None:
        sym.append({"permutation": [(n - i) % n for i in range(n)], "sector": reflection})
    d = {"number_spins": n, "hamming_weight": weight, "symmetries": sym}
    if inversion:
        d["spin_inversion"] = inversion
    basis = basis_from_dict(d)
    bonds = [[i, (i + 1) % n] for i in range(n)]
    if tfim:
        terms = [{"expression": "σᶻ₀ σᶻ₁", "sites": bonds}, {"expression": "-0.7 × σˣ₀", "sites": [[i] for i in range(n)]}]
    else:
        terms = [{"expression": f"σ{c}₀ σ{c}₁", "sites": bonds} for c in "ˣʸᶻ"]
    return operator_from_dict({"terms": terms}, basis)


# (name, model, sites): the table look-up (trivial characters), the index (a complex character), no symmetry, free weight
CASES = [("ring16 k0 r0 inv", ring(16, 8, 0, 0, 1), [0, 1, 2, 3, 4, 5, 6, 7]),
         ("ring14 k3", ring(14, 7, 3), [5, 0, 9, 2]),
         ("ring12 plain", ring(12, 6, None), [11, 3, 4]),
         ("tfim12 free k0 r0", ring(12, None, 0, 0, tfim=True), [0, 6, 1, 7, 2])]


def main():
    ranks = Ranks()
    world, local, verdict = ranks.world, ranks.local, ranks.verdict
    for name, spec, sites in CASES:
        g = Operator(spec, device=local)   # the whole basis on one rank
        g.basis.build()
        d = DistributedOperator(spec, device=local)
        d.basis.build()
        g_reps = g.basis.representatives()
        at = np.searchsorted(g_reps, d.basis.representatives())
        rng = np.random.default_rng(41)
        for dtype in (np.float64, np.complex128):
            cplx = dtype == np.complex128
            if not cplx and g.info("complex_coefficients"):
                continue
            X = rng.normal(size=(2, g_reps.shape[0])) + (1j * rng.normal(size=(2, g_reps.shape[0])) if cplx else 0)
            one = g.reduced_density_matrix(X, sites)
            many = d.op.reduced_density_matrix(np.ascontiguousarray(X[:, at]), sites)   # collective
            err = max(np.abs(many[v][w] - one[v][w]).max() for v in range(2) for w in one[v])
            flat = np.concatenate([many[v][w].ravel() for v in range(2) for w in many[v]])
            mine = torch.from_numpy(flat.view(np.float64).copy()).cuda()
            first = mine.clone()
            dist.broadcast(first, 0)
            same = bool(torch.equal(mine, first))
            verdict(err <= 1e-12 and same, f"{name:20s} P={world} {np.dtype(dtype).name} ρ {err:.1e}, ranks equal {same}")
        for o in (d.op, g):
            o.close()
    ranks.finish()


if __name__ == "__main__":
    main()
