#!/usr/bin/env python3
"""dmv_pm_correlations across ranks (one process per rank, NCCL inside libdmv_b200) against the one-rank result.
With fewer GPUs than ranks, ranks share devices (round robin), as in tools/zz_check.py.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29558 tools/pm_check.py [workload ...]

A seeded random vector (float64, and complex128) in block order is cut into the ranks' chunks and moved to the hashed
blocks (dmv_block_to_hashed); the collective call on the blocks must give the <σ⁺ᵢσ⁻ⱼ> of a one-rank context over the
whole basis to 1e-12 on every rank (the class sums add the rows in another order), for one vector and for a batch of
two.  Each line ends in OK or FAIL; used by tests/test_pm_correlations.py.
"""
import sys

import numpy as np

from rank_harness import Ranks, load
from distributed_matvec_b200 import DistributedOperator, Operator
from oracle import pyoracle as po

# spin inversion alone (pair-major walk), the torus table path, complex characters, no symmetry at all
DEFAULT = ["heisenberg_chain_10", "heisenberg_square_4x4", "momentum_sector", "heisenberg_chain_24"]


def main():
    ranks = Ranks()
    rank, world, local, verdict = ranks.rank, ranks.world, ranks.local, ranks.verdict
    for name in sys.argv[1:] or DEFAULT:
        basis, matrix = load(name)
        g = Operator(matrix, device=local)          # the whole sorted basis on one rank
        g.basis.build()
        n = g.basis.numberStates()
        dop = DistributedOperator(matrix, device=local)
        dop.basis.build()
        masks = po.locale_idx_of(g.basis.representatives(), world)
        bounds = np.linspace(0, n, world + 1).astype(int)
        m_chunk = masks[bounds[rank]:bounds[rank + 1]]
        rng = np.random.default_rng(29)
        for dtype in (np.float64, np.complex128):
            X = rng.normal(size=(2, n)) + (1j * rng.normal(size=(2, n)) if dtype == np.complex128 else 0)
            T1 = g.pm_correlations(X)
            mine = np.stack([dop.op.block_to_hashed(np.ascontiguousarray(X[v, bounds[rank]:bounds[rank + 1]]),
                                                    m_chunk) for v in range(2)])
            T2 = dop.op.pm_correlations(mine)                    # collective
            Ts = dop.op.pm_correlations(np.ascontiguousarray(mine[1]))
            err = max(np.abs(T2 - T1).max(), np.abs(Ts - T1[1]).max())
            verdict(err <= 1e-12, f"{name:26s} P={world} N={n} {np.dtype(dtype).name} T {err:.1e}")
        dop.op.close()
        g.close()
    ranks.finish()


if __name__ == "__main__":
    main()
