#!/usr/bin/env python3
"""dmv_lanczos_quadrature across ranks (one process per rank, NCCL inside libdmv_b200) against the one-rank result.
With fewer GPUs than ranks, ranks share devices (round robin), as in tools/multi_gpu_check.py.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29557 tools/quadrature_check.py [workload ...]

Seeded start vectors depend only on (seed, vector, representative), so every rank count starts from the same vectors.
Every rank runs the collective call on its hashed block and compares with a one-rank context over the whole basis:
log Z(beta), E and C (distributed_matvec_b200.thermal) of 30 steps to 1e-9, and the nodes of a 10-step call to 1e-9.
Each line ends in OK or FAIL; used by tests/test_quadrature.py.
"""
import sys

import numpy as np

from rank_harness import Ranks, load
from distributed_matvec_b200 import DistributedOperator, Operator
from distributed_matvec_b200.thermal import thermodynamics

DEFAULT = ["heisenberg_chain_10", "heisenberg_square_4x4", "momentum_sector", "heisenberg_chain_24"]
R, SEED = 4, 77
TEMPS = [0.25, 0.5, 1.0, 2.0, np.inf]


def main():
    ranks = Ranks()
    world, local, verdict = ranks.world, ranks.local, ranks.verdict
    for name in sys.argv[1:] or DEFAULT:
        basis, matrix = load(name)
        g = Operator(matrix, device=local)          # the whole sorted basis on one rank
        g.basis.build()
        n = g.basis.numberStates()
        dop = DistributedOperator(matrix, device=local)
        dop.basis.build()
        cplx = g.info("complex_coefficients") != 0
        for complex_vectors in sorted({cplx, True}):
            n1, w1, d1, p1 = g.lanczos_quadrature(R, 30, seed=SEED, complex_vectors=complex_vectors)
            n2, w2, d2, p2 = dop.op.lanczos_quadrature(R, 30, seed=SEED, complex_vectors=complex_vectors)   # collective
            t1 = thermodynamics([(n1, w1, 1)], TEMPS)
            t2 = thermodynamics([(n2, w2, 1)], TEMPS)
            dthermo = max(float(np.abs(a - b).max() / max(1.0, np.abs(a).max())) for a, b in zip(t1[:3], t2[:3]))
            m1 = g.lanczos_quadrature(R, 10, seed=SEED, complex_vectors=complex_vectors)[0]
            m2 = dop.op.lanczos_quadrature(R, 10, seed=SEED, complex_vectors=complex_vectors)[0]
            dnodes = float(np.abs(m1 - m2).max() / max(1.0, np.abs(m1).max()))
            verdict(dthermo <= 1e-9 and dnodes <= 1e-9 and np.array_equal(d1, d2),
                    f"{name:26s} P={world} N={n} {'complex128' if complex_vectors else 'float64'} group="
                    f"{g.info('quadrature_group')}/{dop.op.info('quadrature_group')} products={p2}/{p1} "
                    f"log Z, E, C {dthermo:.1e} nodes(10 steps) {dnodes:.1e}")
        dop.op.close()
        g.close()
    ranks.finish()


if __name__ == "__main__":
    main()
