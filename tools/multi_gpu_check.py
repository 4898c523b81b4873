#!/usr/bin/env python3
"""Parity of the real multi-GPU product (one process per rank, NCCL / NVLink inside libdmv_b200) against the CPU oracle.
With fewer GPUs than ranks, ranks share devices (round robin): the same exchanges run through CUDA IPC on one device.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 \
        --master-port 29511 tools/multi_gpu_check.py [workload ...]

Environment: DMV_EXCHANGE = -1 auto | 0 NCCL record buckets | 1 peer-direct records | 2 replicated x;
DMV_PEER_GATHER = 0 forces the NCCL all-gather in the replicated-x form.  Small models are compared element by element
with the oracle's P-locale product; models of 10^5 .. 10^7 states per rank through sampled rows (oracle_expected_rows).
Also covered: the collective block <-> hashed redistribution, Lanczos across the ranks, and the host-owned products
(HostExchangedProduct / HostReplicatedProduct) with the real Operator under the NCCL backend.  Used by
tests/test_multi_gpu.py.
"""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

from rank_harness import Ranks, load
from distributed_matvec_b200 import DistributedOperator, HostExchangedProduct, HostReplicatedProduct, Operator
from oracle import pyoracle as po

DEFAULT = ["heisenberg_chain_10", "heisenberg_chain_16", "heisenberg_square_4x4", "heisenberg_chain_24_symm",
           "heisenberg_chain_24", "heisenberg_chain_32_symm", "heisenberg_square_6x6"]


def recipe_x(n, cplx):
    rs = np.random.RandomState(42)
    x = rs.rand(n) - 0.5
    if cplx:
        x = x + 1j * (rs.rand(n) - 0.5)
    return x


def close(a, b):
    floor = 1e-14 * max(1.0, float(np.abs(b).max(initial=0.0)))
    return bool(np.all(np.abs(a - b) <= np.maximum(floor, 1e-12 * np.maximum(np.abs(a), np.abs(b)))))


def main():
    ranks = Ranks()
    rank, world, local, verdict = ranks.rank, ranks.world, ranks.local, ranks.verdict
    po.set_num_threads(max(1, len(os.sched_getaffinity(0)) // world))
    names = sys.argv[1:] or DEFAULT
    for name in names:
        basis, matrix = load(name)
        dop = DistributedOperator(matrix, device=local)
        dop.op.set_option("exchange", int(os.environ.get("DMV_EXCHANGE", "-1")))
        if os.environ.get("DMV_PEER_GATHER"):
            dop.op.set_option("peer_gather", int(os.environ["DMV_PEER_GATHER"]))
        dop.basis.build()
        mine = dop.basis.representatives()
        g = Operator(matrix, device=local)          # the whole sorted basis (one-rank context)
        g.basis.build()
        reps = g.basis.representatives()
        g.close()
        n = reps.shape[0]
        small = n <= 200000 or (n <= 3000000 and not basis.has_permutation_symmetries())
        if n <= 200000:
            o_reps, _ = po.enumerate_states(basis)
            ok_basis = bool(np.array_equal(o_reps, reps))
        else:
            ok_basis = True
        masks = po.locale_idx_of(reps, world)
        local_rows = np.flatnonzero(masks == rank)
        ok_basis &= bool(np.array_equal(mine, reps[local_rows]))
        # block <-> hashed redistribution (collective, NCCL all-to-all-v inside the library)
        bounds = np.linspace(0, n, world + 1).astype(int)
        m_chunk = masks[bounds[rank]:bounds[rank + 1]]
        for arr in (reps, (np.arange(n) * (1 + 2j)).astype(np.complex128)):
            hashed = dop.op.block_to_hashed(arr[bounds[rank]:bounds[rank + 1]], m_chunk)
            ok_basis &= bool(np.array_equal(hashed, arr[local_rows]))
            back = dop.op.hashed_to_block(torch.from_numpy(hashed).cuda(), m_chunk)
            ok_basis &= bool(np.array_equal(back.cpu().numpy(), arr[bounds[rank]:bounds[rank + 1]]))
        for cplx in (False, True):
            x = recipe_x(n, cplx)
            x_mine = np.ascontiguousarray(x[local_rows])
            if small:
                pick = np.arange(local_rows.shape[0])
                y_ref = po.matvec_global(matrix, reps, x, world)[local_rows]
            else:
                pick = np.sort(np.random.default_rng(7 + rank).choice(local_rows.shape[0], size=2048, replace=False))
                y_ref = po.expected_rows(matrix, reps, x, local_rows[pick])
            y_host = dop.matvec(x_mine)                       # host vectors through the C ABI (collective call)
            xd = torch.from_numpy(x_mine).cuda()
            yd = dop.matvec(xd)                               # device-resident vectors
            yd2 = dop.matvec(xd)                              # and again (alternating buffers of the peer-direct gather)
            torch.cuda.synchronize()
            dop.op.synchronize()
            good = ok_basis and close(y_host[pick], y_ref) and close(yd.cpu().numpy()[pick], y_ref) and \
                close(yd2.cpu().numpy()[pick], y_ref)
            scale = max(np.abs(y_ref).max(), 1e-300)
            e1 = np.abs(y_host[pick] - y_ref).max() / scale
            e2 = np.abs(yd.cpu().numpy()[pick] - y_ref).max() / scale
            exch = ("replicated-x/" + ("peer-direct gather" if dop.op.info("peer_gather") == 1 else "nccl all-gather")
                    if dop.op.info("replicated") else
                    (f"records/peer-direct in {dop.op.info('rounds')} rounds" if dop.op.info("rounds") > 1 else
                     ("records/peer-direct" if dop.op.info("peer_direct") else "records/nccl")))
            verdict(good, f"{name:26s} P={world} {'c128' if cplx else 'f64 '} N={n} rows_checked={pick.shape[0]}/rank "
                          f"basis_ok={ok_basis} err_host={e1:.1e} err_dev={e2:.1e} exchange={exch}")
        # Lanczos across the ranks (dot products reduced with NCCL): every rank must report the same energy
        if n <= 13000:
            e0, _, iters, res = dop.op.lanczos(max_iters=200, tol=1e-11, eigenvector=False)
            e_all = torch.tensor([e0], device="cuda", dtype=torch.float64)
            lst = [torch.zeros_like(e_all) for _ in range(world)]
            dist.all_gather(lst, e_all)
            same = all(abs(float(t) - e0) <= 1e-12 * abs(e0) for t in lst)
            verdict(same, f"{name:26s} P={world} lanczos E0={e0:.10f} iters={iters} residual={res:.1e}")
        # the host-owned products with the REAL Operator under NCCL (device tensors end to end)
        if n <= 20000:
            for cplx in (False, True):
                x = recipe_x(n, cplx)
                y_ref = po.matvec_global(matrix, reps, x, world)[local_rows]
                xd = torch.from_numpy(np.ascontiguousarray(x[local_rows])).cuda()
                h = Operator(matrix, device=local, rank=rank, num_ranks=world)
                h.basis.build()
                y1 = HostExchangedProduct(h).matvec(xd, torch.zeros_like(xd))
                torch.cuda.synchronize(); h.synchronize()
                y2 = HostReplicatedProduct(h).matvec(xd, torch.zeros_like(xd))
                torch.cuda.synchronize(); h.synchronize()
                good = close(y1.cpu().numpy(), y_ref) and close(y2.cpu().numpy(), y_ref)
                verdict(good, f"{name:26s} P={world} {'c128' if cplx else 'f64 '} host-owned exchange (records width "
                              f"{h.record_width(xd)}, replicated x)")
                h.close()
        dop.op.close()
    ranks.finish()


if __name__ == "__main__":
    main()
