#!/usr/bin/env python3
"""Products and eigsh of fermionic symmetry sectors across ranks (one process per rank, NCCL inside libdmv_b200) against
the one-rank result.  With fewer GPUs than ranks, ranks share devices (round robin), as in tools/spin_check.py.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --standalone tools/fermion_symmetry_check.py

For each sector a seeded random vector over the whole sector is cut into the ranks' hashed blocks.  The collective
product must give, on every rank, the entries of the one-rank y at that rank's representatives to 1e-12 relative, for
float64 (real sectors) and complex128; the collective eigsh must give the one-rank lowest eigenvalues to 1e-10
relative.  Each line ends in OK or FAIL; used by tests/test_fermion_symmetries.py.
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from rank_harness import Ranks  # noqa: E402
from distributed_matvec_b200 import DistributedOperator, Operator  # noqa: E402
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict  # noqa: E402
from gen_models import (_bonds_ring, _bonds_torus, hubbard, ring_reflection, ring_translation,  # noqa: E402
                        spinless_ring, torus_translations, with_site_symmetries)

# (name, model in one sector)
CASES = [("spinless12 k=5", with_site_symmetries(spinless_ring(12, 5), [ring_translation(12)], [5])),
         ("spinless12 k=6 R=1", with_site_symmetries(spinless_ring(12, 6), [ring_translation(12), ring_reflection(12)],
                                                      [6, 1])),
         ("hubbard8 k=0 R=0", with_site_symmetries(hubbard(8, _bonds_ring(8)), [ring_translation(8), ring_reflection(8)])),
         ("hubbard3x3 k=(1,2)", with_site_symmetries(hubbard(9, _bonds_torus(3, 3), number_up=5, number_down=4),
                                                     list(torus_translations(3, 3)), [1, 2]))]


def spec(conf):
    return operator_from_dict(conf["hamiltonian"], basis_from_dict(conf["basis"]))


def main():
    ranks = Ranks()
    world, local, verdict = ranks.world, ranks.local, ranks.verdict
    for name, conf in CASES:
        s = spec(conf)
        g = Operator(s, device=local)   # the whole sector on one rank
        g.basis.build()
        dop = DistributedOperator(s, device=local)
        dop.basis.build()
        reps = g.basis.representatives()
        at = np.searchsorted(reps, dop.op.basis.representatives())
        n = reps.shape[0]
        real = bool(np.all(s.basis.group.characters.imag == 0)) and s.is_real()
        rng = np.random.default_rng(17)
        for dtype in ((np.float64, np.complex128) if real else (np.complex128,)):
            x = rng.normal(size=n) + (1j * rng.normal(size=n) if dtype == np.complex128 else 0)
            y1 = g.matvec(x)
            y2 = dop.matvec(np.ascontiguousarray(x[at]))   # collective
            err = np.abs(y2 - y1[at]).max() / max(np.abs(y1).max(), 1e-300)
            verdict(err <= 1e-12, f"{name:20s} P={world} n={n} {np.dtype(dtype).name} y {err:.1e}")
        e1 = g.eigsh(2, complex_vectors=not real, eigenvectors=False)[0]
        e2 = dop.op.eigsh(2, complex_vectors=not real, eigenvectors=False)[0]   # collective
        err = np.abs(e2 - e1).max() / np.abs(e1).max()
        verdict(err <= 1e-10, f"{name:20s} P={world} n={n} eigsh {e1[0]:.10f} {err:.1e}")
        dop.op.close()
        g.close()
    ranks.finish()


if __name__ == "__main__":
    main()
