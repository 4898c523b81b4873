#!/usr/bin/env python3
"""dmv_eigsh across ranks (one process per rank, NCCL inside libdmv_b200) against the one-rank result.
With fewer GPUs than ranks, ranks share devices (round robin), as in tools/multi_gpu_check.py.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29551 tools/eigsh_check.py [workload ...]

Every rank runs the collective call on its hashed block, converts its eigenvectors back to block order
(dmv_hashed_to_block) and compares them with those of a one-rank context over the whole basis: the eigenvalues to 1e-9,
and for every complete eigenspace the projectors, through |P1 - P2|_F = sqrt(2) |Y2 - Y1 Y1^H Y2|_F, to 1e-8.  Each line
ends in OK or FAIL; used by tests/test_eigsh.py.
"""
import sys

import numpy as np
import torch
import torch.distributed as dist

from rank_harness import Ranks, load
from distributed_matvec_b200 import DistributedOperator, Operator
from oracle import pyoracle as po

DEFAULT = ["heisenberg_chain_10", "heisenberg_square_4x4", "momentum_sector", "heisenberg_chain_24"]
NEV = 6


def main():
    ranks = Ranks()
    rank, world, local, verdict = ranks.rank, ranks.world, ranks.local, ranks.verdict
    for name in sys.argv[1:] or DEFAULT:
        basis, matrix = load(name)
        g = Operator(matrix, device=local)          # the whole sorted basis on one rank
        g.basis.build()
        reps = g.basis.representatives()
        n = reps.shape[0]
        dop = DistributedOperator(matrix, device=local)
        dop.basis.build()
        masks = po.locale_idx_of(reps, world)
        bounds = np.linspace(0, n, world + 1).astype(int)
        m_chunk = masks[bounds[rank]:bounds[rank + 1]]
        cplx = g.info("complex_coefficients") != 0
        dtype = torch.complex128 if cplx else torch.float64
        n_mine = dop.op.basis.numberStates()
        for p in (0, 2):
            y1 = torch.empty((NEV, n), dtype=dtype, device="cuda")
            v1, _, _, c1, p1, _ = g.eigsh(NEV, block_size=p, complex_vectors=cplx, eigenvectors=y1)
            y2 = torch.empty((NEV, n_mine), dtype=dtype, device="cuda")
            v2, _, _, c2, p2, r2 = dop.op.eigsh(NEV, block_size=p, complex_vectors=cplx, eigenvectors=y2)   # collective
            torch.cuda.synchronize()
            mine = y1[:, bounds[rank]:bounds[rank + 1]]
            block = torch.stack([dop.op.hashed_to_block(y2[i].contiguous(), m_chunk) for i in range(NEV)])
            dval = float(np.abs(v1 - v2).max() / max(1.0, np.abs(v1).max()))
            # complete eigenspaces of the one-rank result (the last cluster may continue beyond NEV)
            groups, start = [], 0
            for i in range(1, NEV + 1):
                if i == NEV or v1[i] - v1[i - 1] > 1e-8 * max(1.0, abs(v1[i])):
                    groups.append((start, i))
                    start = i
            worst = 0.0
            for a, b in groups[:-1] if len(groups) > 1 else groups:
                y1c, y2c = mine[a:b].to(torch.complex128), block[a:b].to(torch.complex128)
                M = y1c.conj() @ y2c.T                        # M[i, j] = <y1_i, y2_j>, summed over the ranks
                dist.all_reduce(M)
                out = torch.tensor([float((torch.linalg.norm(y2c - M.T @ y1c) ** 2).item())], device="cuda",
                                   dtype=torch.float64)      # the part of Y2 outside span(Y1), without cancellation
                dist.all_reduce(out)
                worst = max(worst, float(np.sqrt(2.0 * out.item())))   # = |P1 - P2|_F for equal dimensions
            verdict(dval <= 1e-9 and worst <= 1e-8 and c1 == NEV and c2 == NEV,
                    f"{name:26s} P={world} N={n} block={p} {str(dtype)[6:]} products={p2}/{p1} restarts={r2} "
                    f"eigenvalues {dval:.1e} projectors {worst:.1e}")
        dop.op.close()
        g.close()
    ranks.finish()


if __name__ == "__main__":
    main()
