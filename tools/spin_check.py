#!/usr/bin/env python3
"""dmv_apply_spin across ranks (one process per rank, NCCL inside libdmv_b200) against the one-rank result.
With fewer GPUs than ranks, ranks share devices (round robin), as in tools/pm_check.py.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29561 tools/spin_check.py

A seeded random vector over the whole source basis is cut into the ranks' hashed blocks (each rank takes the entries of
its own representatives); the collective call must give, on every rank, the entries of the one-rank result at that
rank's representatives of the target basis to 1e-12 relative (each row is computed the same way; only the look-up
differs), for float64 and complex128 and for a batch of two.  spectral.dynamical_correlation on the ranks must give the
one-rank S(ω) (lowest pole and total weight to 1e-10), and no poles, on every rank, where nothing of O x reaches the
target.  Each line ends in OK or FAIL; used by
tests/test_spin_operators.py.
"""
import numpy as np

from rank_harness import Ranks
from distributed_matvec_b200 import DistributedOperator, Operator
from distributed_matvec_b200.spectral import dynamical_correlation
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict


def ring(n, weight, sector, reflection=None, inversion=None):
    """Heisenberg ring; sector None: no symmetries (the plain basis)"""
    sym = [] if sector is None else [{"permutation": [(i + 1) % n for i in range(n)], "sector": sector}]
    if reflection is not None:
        sym.append({"permutation": [(n - i) % n for i in range(n)], "sector": reflection})
    d = {"number_spins": n, "hamming_weight": weight, "symmetries": sym}
    if inversion:
        d["spin_inversion"] = inversion
    basis = basis_from_dict(d)
    terms = [{"expression": f"σ{c}₀ σ{c}₁", "sites": [[i, (i + 1) % n] for i in range(n)]} for c in "ˣʸᶻ"]
    return operator_from_dict({"terms": terms}, basis)


# (name, source, target, kind): the table look-up (trivial characters), the index (a complex character), unfolding
CASES = [("ring16 k0 -> k8 z", ring(16, 8, 0, 0), ring(16, 8, 8), "z"),
         ("ring16 k0 -> k5 w7 -", ring(16, 8, 0, 0), ring(16, 7, 5), "-"),
         ("ring14 k3 -> k1 w8 +", ring(14, 7, 3), ring(14, 8, 1), "+"),
         ("ring12 k0 inv -> plain z", ring(12, 6, 0, 0, 1), ring(12, 6, None), "z")]


def main():
    ranks = Ranks()
    rank, world, local, verdict = ranks.rank, ranks.world, ranks.local, ranks.verdict
    for name, src_spec, tgt_spec, kind in CASES:
        gs, gt = Operator(src_spec, device=local), Operator(tgt_spec, device=local)   # whole bases on one rank
        gs.basis.build()
        gt.basis.build()
        src = DistributedOperator(src_spec, device=local)
        src.basis.build()
        tgt_d = DistributedOperator(tgt_spec, device=local)   # its communicator serves the Lanczos steps below
        tgt = tgt_d.op
        tgt.basis.build()
        g_src, g_tgt = gs.basis.representatives(), gt.basis.representatives()
        at_src = np.searchsorted(g_src, src.basis.representatives())
        at_tgt = np.searchsorted(g_tgt, tgt.basis.representatives())
        N = src_spec.basis.number_sites
        rng = np.random.default_rng(31)
        for dtype in (np.float64, np.complex128):
            cplx = dtype == np.complex128
            X = rng.normal(size=(2, g_src.shape[0])) + (1j * rng.normal(size=(2, g_src.shape[0])) if cplx else 0)
            w = rng.normal(size=N) + (1j * rng.normal(size=N) if cplx else 0)
            if not cplx and (gs.info("complex_coefficients") or gt.info("complex_coefficients")):
                continue
            Y1 = gs.apply_spin(kind, w, X, gt)
            Y2 = src.op.apply_spin(kind, w, np.ascontiguousarray(X[:, at_src]), tgt)   # collective
            Ys = src.op.apply_spin(kind, w, np.ascontiguousarray(X[1, at_src]), tgt)
            scale = max(np.abs(Y1).max(), 1e-300)
            err = max(np.abs(Y2 - Y1[:, at_tgt]).max(), np.abs(Ys - Y1[1, at_tgt]).max()) / scale
            verdict(err <= 1e-12, f"{name:26s} P={world} n={g_src.shape[0]} {np.dtype(dtype).name} y {err:.1e}")
            # S(ω) from the same start: the poles and residues of 12 steps, and a sector the identity cannot reach
            # (kind "1" into another sector leaves y at rounding on every rank: no poles, and no rank waits)
            x1, xr = X[0], np.ascontiguousarray(X[0, at_src])
            p1, r1 = dynamical_correlation(gs, x1, 0.0, gt, kind, w, 12)
            p2, r2 = dynamical_correlation(src.op, xr, 0.0, tgt, kind, w, 12)
            good = p1.shape == p2.shape and p1.size > 0 and np.abs(p1[0] - p2[0]) <= 1e-10 * max(1.0, abs(p1[0])) \
                and abs(r1.sum() - r2.sum()) <= 1e-10 * r1.sum()
            verdict(good, f"{name:26s} P={world} {np.dtype(dtype).name} S(ω): {p2.size} poles, lowest {p2[0] if p2.size else 0:.6f}")
            if name.startswith("ring16 k0 -> k8"):
                p0, r0 = dynamical_correlation(src.op, xr, 0.0, tgt, "1", w, 12)
                verdict(p0.size == 0 and r0.size == 0, f"{name:26s} P={world} {np.dtype(dtype).name} S(ω) of 1: "
                                                       f"{p0.size} poles")
        for o in (tgt, src.op, gt, gs):
            o.close()
    ranks.finish()


if __name__ == "__main__":
    main()
