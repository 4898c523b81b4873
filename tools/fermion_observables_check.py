#!/usr/bin/env python3
"""dmv_one_body_density_matrix and dmv_apply_fermion across ranks (one process per rank, NCCL inside libdmv_b200) against
the one-rank result.  With fewer GPUs than ranks, ranks share devices (round robin), as in tools/spin_check.py.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --standalone tools/fermion_observables_check.py

A seeded random vector over the whole source basis is cut into the ranks' hashed blocks.  The collective G must equal
the one-rank G to 1e-12 relative on every rank, and the collective c / c† must give, on every rank, the entries of the
one-rank y at that rank's representatives of the target basis to 1e-12 relative, for float64 and complex128 and for a
batch of two.  Each line ends in OK or FAIL; used by tests/test_fermion_observables.py.
"""
import math
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rank_harness import Ranks  # noqa: E402
from distributed_matvec_b200 import DistributedOperator, Operator  # noqa: E402
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict  # noqa: E402
from gen_models import _bonds_ring, hubbard, spinless_ring  # noqa: E402


def spec(conf):
    basis = basis_from_dict(conf["basis"])
    return operator_from_dict(conf["hamiltonian"], basis)


def peierls_ring(n, phi=0.3):
    c, s = math.cos(phi), math.sin(phi)
    conf = hubbard(n, _bonds_ring(n), number_up=n // 2, number_down=n // 2)
    conf["hamiltonian"]["terms"][0]["expression"] = " ".join(
        f"- {c!r} × c†₀{a} c₁{a} - {s!r}j × c†₀{a} c₁{a} - {c!r} × c†₁{a} c₀{a} + {s!r}j × c†₁{a} c₀{a}" for a in "↑↓")
    return conf


# (name, source, target, kind, modes with weights)
CASES = [("hubbard8 c+ up", hubbard(8, _bonds_ring(8)), hubbard(8, _bonds_ring(8), number_up=5), "c+", range(0, 8)),
         ("hubbard8 c down", hubbard(8, _bonds_ring(8)), hubbard(8, _bonds_ring(8), number_down=3), "c", range(8, 16)),
         ("peierls8 c+ down", peierls_ring(8), hubbard(8, _bonds_ring(8), number_down=5), "c+", range(8, 16)),
         ("spinless16 c", spinless_ring(16, 7), spinless_ring(16, 6), "c", range(16))]


def main():
    ranks = Ranks()
    world, local, verdict = ranks.world, ranks.local, ranks.verdict
    for name, src_conf, tgt_conf, kind, modes in CASES:
        src_spec, tgt_spec = spec(src_conf), spec(tgt_conf)
        gs, gt = Operator(src_spec, device=local), Operator(tgt_spec, device=local)   # whole bases on one rank
        gs.basis.build()
        gt.basis.build()
        src = DistributedOperator(src_spec, device=local)
        src.basis.build()
        tgt = DistributedOperator(tgt_spec, device=local).op
        tgt.basis.build()
        g_src, g_tgt = gs.basis.representatives(), gt.basis.representatives()
        at_src = np.searchsorted(g_src, src.basis.representatives())
        at_tgt = np.searchsorted(g_tgt, tgt.basis.representatives())
        M = src_spec.basis.number_bits
        rng = np.random.default_rng(31)
        for dtype in (np.float64, np.complex128):
            cplx = dtype == np.complex128
            n = g_src.shape[0]
            X = rng.normal(size=(2, n)) + (1j * rng.normal(size=(2, n)) if cplx else 0)
            w = np.zeros(M, dtype=np.complex128)
            w[list(modes)] = rng.normal(size=len(modes)) + (1j * rng.normal(size=len(modes)) if cplx else 0)
            G1 = gs.one_body_density_matrix(X)
            G2 = src.op.one_body_density_matrix(np.ascontiguousarray(X[:, at_src]))   # collective
            err = np.abs(G2 - G1).max() / np.abs(G1).max()
            verdict(err <= 1e-12, f"{name:18s} P={world} n={n} {np.dtype(dtype).name} G {err:.1e}")
            Y1 = gs.apply_fermion(kind, w, X, gt)
            Y2 = src.op.apply_fermion(kind, w, np.ascontiguousarray(X[:, at_src]), tgt)   # collective
            Ys = src.op.apply_fermion(kind, w, np.ascontiguousarray(X[1, at_src]), tgt)
            scale = max(np.abs(Y1).max(), 1e-300)
            err = max(np.abs(Y2 - Y1[:, at_tgt]).max(), np.abs(Ys - Y1[1, at_tgt]).max()) / scale
            verdict(err <= 1e-12, f"{name:18s} P={world} n={n} {np.dtype(dtype).name} y {err:.1e}")
        for o in (tgt, src.op, gt, gs):
            o.close()
    ranks.finish()


if __name__ == "__main__":
    main()
