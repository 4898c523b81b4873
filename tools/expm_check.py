#!/usr/bin/env python3
"""dmv_expm_multiply across ranks (one process per rank, NCCL inside libdmv_b200) against the one-rank result.
With fewer GPUs than ranks, ranks share devices (round robin), as in tools/multi_gpu_check.py.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29541 tools/expm_check.py [workload ...]

Every rank evolves its hashed block of x with the collective call, converts its hashed y back to block order
(dmv_hashed_to_block) and compares its chunk with y = exp(z H) x of a one-rank context over the whole basis.  Each line
ends in OK or FAIL; used by tests/test_expm_multiply.py.
"""
import sys

import numpy as np
import torch
import torch.distributed as dist

from rank_harness import Ranks, load
from distributed_matvec_b200 import DistributedOperator, Operator
from oracle import pyoracle as po

DEFAULT = ["heisenberg_chain_10", "heisenberg_square_4x4", "heisenberg_chain_24_symm", "momentum_sector",
           "heisenberg_chain_24"]


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
        local_rows = np.flatnonzero(masks == rank)
        bounds = np.linspace(0, n, world + 1).astype(int)
        m_chunk = masks[bounds[rank]:bounds[rank + 1]]
        rng = np.random.default_rng(5)
        x = rng.random(n) - 0.5 + 1j * (rng.random(n) - 0.5)
        cases = [(-0.3j, np.complex128), (-0.5, np.complex128)]
        if not g.info("complex_coefficients"):
            cases.append((-0.5, np.float64))
        for z, dtype in cases:
            xx = (x.real if dtype == np.float64 else x).astype(dtype)
            y_one, p_one, _ = g.expm_multiply(torch.from_numpy(xx).cuda(), z)
            y_one = y_one.cpu().numpy()
            xd = torch.from_numpy(np.ascontiguousarray(xx[local_rows])).cuda()
            y_mine, prods, err = dop.op.expm_multiply(xd, z)                # collective
            y_block = dop.op.hashed_to_block(y_mine, m_chunk).cpu().numpy()
            want = y_one[bounds[rank]:bounds[rank + 1]]
            diff = float(np.linalg.norm(y_block - want)) ** 2
            total = torch.tensor([diff, float(np.linalg.norm(want)) ** 2], device="cuda", dtype=torch.float64)
            dist.all_reduce(total)
            rel = float(np.sqrt(total[0].item() / max(total[1].item(), 1e-300)))
            verdict(rel <= 1e-10,
                    f"{name:26s} P={world} N={n} z={z} {np.dtype(dtype).name} products={prods}/{p_one} "
                    f"rel_diff={rel:.1e}")
        dop.op.close()
        g.close()
    ranks.finish()


if __name__ == "__main__":
    main()
