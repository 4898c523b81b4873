#!/usr/bin/env python3
"""The record exchanges of the collective product (dmv_matvec) on 2, 3 or 4 ranks against the CPU oracle, one process
per rank.  With fewer GPUs than ranks, ranks share devices (round robin), as in tools/multi_gpu_check.py.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 3 --master-addr 127.0.0.1 \
        --master-port 29611 tools/exchange_check.py [--cases nccl,rounds2,...] [--parts mixed,switch,...] [model ...]

Every exchange of a case is set before the first product and checked through info() to be the one that ran:

    nccl        exchange = 0                  NCCL record buckets
    oneshot     exchange = 1, rounds = 1      one-shot peer-direct records
    roundsR     exchange = 1, rounds = R      peer-direct records in R overlapped rounds (R = 2, 3, 5, 64)
    rounds_auto exchange = 1, rounds = -1     the automatic number of rounds (4 from 2^18 states per rank)
    repl_peer   exchange = 2                  replicated x, peer-direct all-gather
    repl_nccl   exchange = 2, peer_gather = 0 replicated x, NCCL all-gather

Parts (each line names its case, so the caller can tell them apart):

    mixed    per model and case, one context: device products f64 f64 c128 f64 c128 c128 f64 back to back, a new x
             each and no host synchronisation in between (the alternating record buffers pass through every pair of
             element widths), then one host product; every y against the oracle afterwards.  Models with complex
             coefficients take c128 throughout.
    switch   one live context through exchange / rounds changes between products (re-setup of the rounds and the
             peer mappings), every y against the oracle
    batch    matvec_batch of 3 vectors, f64 then c128, through exchange = 1, rounds = 3
    solvers  Lanczos, eigsh and expm_multiply through exchange = 1, rounds = 2 and exchange = 0 against one rank

Models are those of data/, "momentum_sector" (complex characters) and "empty_rank": the smallest ring at Hamming
weight 1 or n - 1 in which some rank owns no state.  Small models are compared element by element with the oracle's P-locale
product, models of more than 200000 states through 2048 sampled rows per rank.  Each line ends in OK or FAIL; used by
tests/test_collective_exchange.py.
"""
import argparse
import os

import numpy as np
import torch
import torch.distributed as dist

from rank_harness import Ranks, load
from multi_gpu_check import close
from distributed_matvec_b200 import DistributedOperator, Operator
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
from oracle import pyoracle as po

# name -> (options set before the first product, info() the product must report)
CASES = {
    "nccl": ({"exchange": 0}, {"replicated": 0, "peer_direct": 0, "rounds": 0}),
    "oneshot": ({"exchange": 1, "rounds": 1}, {"replicated": 0, "peer_direct": 1, "rounds": 0}),
    **{f"rounds{R}": ({"exchange": 1, "rounds": R}, {"replicated": 0, "rounds": R}) for R in (2, 3, 5, 64)},
    "rounds_auto": ({"exchange": 1, "rounds": -1}, {"replicated": 0, "rounds": 4}),
    "repl_peer": ({"exchange": 2, "peer_gather": -1}, {"replicated": 1, "peer_gather": 1}),
    "repl_nccl": ({"exchange": 2, "peer_gather": 0}, {"replicated": 1, "peer_gather": 0}),
}
SMALL = ["heisenberg_chain_10", "heisenberg_chain_16", "heisenberg_square_4x4", "heisenberg_kagome_12_symm", "issue_01",
         "momentum_sector", "empty_rank"]
MIXED = ["f64", "f64", "c128", "f64", "c128", "c128", "f64"]   # buffer parity 0 1 0 1 0 1 0


def empty_rank_model(world):
    """Heisenberg ring of n spins at Hamming weight 1 or n - 1 (n states), the first from 3 spins on in which some
    rank owns no state (3 spins: at weight 2 on two ranks, at weight 1 on three or four)."""
    for n in range(3, 64):
        for w in (1, n - 1):
            states = np.array([((1 << n) - 1) ^ (1 << i) if w > 1 else 1 << i for i in range(n)], dtype=np.uint64)
            if np.unique(po.locale_idx_of(states, world)).shape[0] < world:
                basis = basis_from_dict({"number_spins": n, "hamming_weight": w})
                terms = [{"expression": f"σ{c}₀ σ{c}₁", "sites": [[i, (i + 1) % n] for i in range(n)]} for c in "ˣʸᶻ"]
                return basis, operator_from_dict({"terms": terms}, basis)
    raise RuntimeError(f"no ring at Hamming weight 1 or n - 1 leaves a rank of {world} empty")


def seeded_x(n, cplx, seed):
    rs = np.random.RandomState(seed)
    x = rs.rand(n) - 0.5
    return x + 1j * (rs.rand(n) - 0.5) if cplx else x


def exchange_name(op):
    if op.info("replicated"):
        return "replicated-x/" + ("peer-direct gather" if op.info("peer_gather") else "nccl all-gather")
    if op.info("rounds") > 1:
        return f"records/peer-direct in {op.info('rounds')} rounds"
    return "records/peer-direct" if op.info("peer_direct") else "records/nccl"


def ran_as(op, want):
    """(the exchange that ran is the one asked for, a description of it)"""
    got = {k: op.info(k) for k in want}
    return got == want, exchange_name(op) + ("" if got == want else f" (asked for {want}, info {got})")


class Model:
    """A model, the whole sorted basis, this rank's rows and the oracle's y for the seeded x of the checks."""

    def __init__(self, name, rank, world, local):
        self.name = name
        self.basis, self.matrix = empty_rank_model(world) if name == "empty_rank" else load(name)
        g = Operator(self.matrix, device=local)
        g.basis.build()
        self.reps = g.basis.representatives()
        self.cplx_only = g.info("complex_coefficients") != 0
        g.close()
        self.n = self.reps.shape[0]
        self.masks = po.locale_idx_of(self.reps, world)
        self.rows = np.flatnonzero(self.masks == rank)
        self.world = world
        self.small = self.n <= 200000
        if self.small:
            self.pick = np.arange(self.rows.shape[0])
        else:
            rng = np.random.default_rng(7 + rank)
            self.pick = np.sort(rng.choice(self.rows.shape[0], size=min(2048, self.rows.shape[0]), replace=False))
        self.empty = int(np.sum(np.bincount(self.masks, minlength=world) == 0))
        self._ref = {}

    def x(self, cplx, seed):
        return seeded_x(self.n, cplx or self.cplx_only, seed)

    def expected(self, cplx, seed):
        """the oracle's y on this rank's (picked) rows"""
        key = (cplx or self.cplx_only, seed)
        if key not in self._ref:
            x = self.x(cplx, seed)
            if self.small:
                self._ref[key] = po.matvec_global(self.matrix, self.reps, x, self.world)[self.rows]
            else:
                self._ref[key] = po.expected_rows(self.matrix, self.reps, x, self.rows[self.pick])
        return self._ref[key]

    def mine(self, cplx, seed, device=True):
        x = np.ascontiguousarray(self.x(cplx, seed)[self.rows])
        return torch.from_numpy(x).cuda() if device else x

    def err(self, y, cplx, seed):
        """(y equals the oracle's within multi_gpu_check.close, relative error)"""
        y = (y.cpu().numpy() if torch.is_tensor(y) else y)[self.pick]
        ref = self.expected(cplx, seed)
        return close(y, ref), float(np.abs(y - ref).max(initial=0.0) / max(np.abs(ref).max(initial=0.0), 1e-300))

    def operator(self, local, options):
        dop = DistributedOperator(self.matrix, device=local)
        for k, v in options.items():
            dop.op.set_option(k, v)
        dop.basis.build()
        return dop

    def label(self, world):
        n_mine = self.rows.shape[0]
        return f"{self.name:26s} P={world} N={self.n} mine={n_mine}" + (f" empty_ranks={self.empty}" if self.empty else "")


def check_mixed(m, case, ranks, local):
    options, want = CASES[case]
    dop = m.operator(local, options)
    ok_basis = bool(np.array_equal(dop.basis.representatives(), m.reps[m.rows]))
    widths = ["c128"] * len(MIXED) if m.cplx_only else MIXED
    xs = [m.mine(w == "c128", 100 + k) for k, w in enumerate(widths)]
    torch.cuda.synchronize()
    ys = [dop.matvec(x) for x in xs]                  # back to back on the device
    torch.cuda.synchronize()
    dop.op.synchronize()
    ran, exch = ran_as(dop.op, want)
    y_host = dop.matvec(m.mine(False, 100, device=False))   # and once more through host vectors
    results = [m.err(y, w == "c128", 100 + k) for k, (y, w) in enumerate(zip(ys, widths))]
    results.append(m.err(y_host, False, 100))
    good = ok_basis and ran and all(r[0] for r in results)
    worst = max(r[1] for r in results)
    bad = [k for k, r in enumerate(results) if not r[0]]
    ranks.verdict(good, f"case={case} mixed {m.label(ranks.world)} {'/'.join(widths)}+host basis_ok={ok_basis} "
                        f"err={worst:.1e}" + (f" wrong_products={bad}" if bad else "") + f" exchange={exch}")
    dop.op.close()


# one live context: options changed between products, and what must run after each change
SWITCH = [({"exchange": 1, "rounds": 3}, "f64", {"replicated": 0, "rounds": 3}),
          ({"rounds": 2}, "c128", {"replicated": 0, "rounds": 2}),
          ({"rounds": 0}, "f64", {"replicated": 0, "peer_direct": 1, "rounds": 0}),
          ({"exchange": 0}, "c128", {"replicated": 0, "peer_direct": 0, "rounds": 0}),
          ({"exchange": 2}, "f64", {"replicated": 1, "peer_gather": 1}),
          ({"exchange": 1, "rounds": 3}, "c128", {"replicated": 0, "rounds": 3}),
          ({"rounds": 5}, "f64", {"replicated": 0, "rounds": 5})]


def check_switch(m, ranks, local):
    dop = m.operator(local, {})
    ys, steps = [], []
    for k, (options, width, want) in enumerate(SWITCH):
        for name, v in options.items():
            dop.op.set_option(name, v)
        cplx = width == "c128" or m.cplx_only
        ys.append(dop.matvec(m.mine(cplx, 200 + k)))
        ran, exch = ran_as(dop.op, want)
        steps.append((cplx, ran, exch))
    torch.cuda.synchronize()
    dop.op.synchronize()
    for k, (y, (cplx, ran, exch)) in enumerate(zip(ys, steps)):
        good, e = m.err(y, cplx, 200 + k)
        opts = ",".join(f"{a}={b}" for a, b in SWITCH[k][0].items())
        ranks.verdict(good and ran, f"case=switch {m.label(ranks.world)} step={k} set {opts} "
                                    f"{'c128' if cplx else 'f64 '} err={e:.1e} exchange={exch}")
    dop.op.close()


def check_batch(m, ranks, local):
    options, want = {"exchange": 1, "rounds": 3}, {"replicated": 0, "rounds": 3}
    dop = m.operator(local, options)
    for cplx in (False, True):
        X = torch.stack([m.mine(cplx, 300 + k) for k in range(3)])
        Y = dop.op.matvec_batch(X)
        torch.cuda.synchronize()
        dop.op.synchronize()
        results = [m.err(Y[k], cplx, 300 + k) for k in range(3)]
        ran, exch = ran_as(dop.op, want)
        ranks.verdict(ran and all(r[0] for r in results),
                      f"case=batch {m.label(ranks.world)} 3x{'c128' if cplx or m.cplx_only else 'f64 '} "
                      f"err={max(r[1] for r in results):.1e} exchange={exch}")
    dop.op.close()


def same_on_every_rank(value):
    t = torch.tensor([value], device="cuda", dtype=torch.float64)
    lst = [torch.zeros_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(lst, t)
    return all(float(u) == value for u in lst)


def aligned_distance(a_mine, b_mine):
    """|a - phase b| over all ranks, the phase that best aligns b with a (unit vectors)"""
    ov = torch.tensor([complex(np.vdot(b_mine, a_mine))], device="cuda", dtype=torch.complex128)
    dist.all_reduce(ov)
    ov = complex(ov.item())
    phase = ov / abs(ov) if abs(ov) > 0 else 1.0
    d = torch.tensor([float(np.linalg.norm(a_mine - phase * b_mine)) ** 2], device="cuda", dtype=torch.float64)
    dist.all_reduce(d)
    return float(np.sqrt(d.item()))


def check_solvers(m, ranks, local):
    g = Operator(m.matrix, device=local)               # the same calls on one rank over the whole basis
    g.basis.build()
    e1, v1, _, _ = g.lanczos(max_iters=300, tol=1e-12)
    v1 = v1 / np.linalg.norm(v1)
    k = 4
    ev1, w1, _, c1, _, _ = g.eigsh(k)
    x = m.x(True, 400)
    xe1, _, _ = g.expm_multiply(x, -0.3j)
    xr1, _, _ = g.expm_multiply(x.real.copy(), -0.5)
    g.close()
    for case, options, want in (("solvers_rounds2", {"exchange": 1, "rounds": 2}, {"replicated": 0, "rounds": 2}),
                                ("solvers_nccl", {"exchange": 0}, {"replicated": 0, "peer_direct": 0, "rounds": 0})):
        dop = m.operator(local, options)
        label = f"case={case} {m.label(ranks.world)}"
        e2, v2, it, res = dop.op.lanczos(max_iters=300, tol=1e-12)
        ran, exch = ran_as(dop.op, want)
        n2 = torch.tensor([float(np.linalg.norm(v2)) ** 2], device="cuda", dtype=torch.float64)
        dist.all_reduce(n2)
        dv = aligned_distance(v1[m.rows], v2 / np.sqrt(n2.item()))
        de = abs(e2 - e1) / abs(e1)
        ranks.verdict(ran and de <= 1e-10 and dv <= 1e-9 and same_on_every_rank(e2),
                      f"{label} lanczos E0={e2:.12f} rel_diff={de:.1e} vector_diff={dv:.1e} iters={it} exchange={exch}")
        ev2, w2, _, c2, _, _ = dop.op.eigsh(k)
        ran, exch = ran_as(dop.op, want)
        de = float(np.abs(ev2 - ev1).max() / np.abs(ev1).max())
        gap = ev1[1] - ev1[0] > 1e-6 * abs(ev1[0])      # a non-degenerate ground state: its vector is compared
        dv = aligned_distance(w1[0][m.rows], w2[0]) if gap else 0.0
        same = all(same_on_every_rank(float(v)) for v in ev2)
        ranks.verdict(ran and de <= 1e-10 and dv <= 1e-9 and same and c2 == k and c1 == k and gap,
                      f"{label} eigsh k={k} E={np.array2string(ev2, precision=8)} rel_diff={de:.1e} "
                      f"ground_vector_diff={dv:.1e} exchange={exch}")
        for z, x1, y1 in ((-0.3j, x, xe1), (-0.5, x.real.copy(), xr1)):
            y2, prods, _ = dop.op.expm_multiply(np.ascontiguousarray(x1[m.rows]), z)
            ran, exch = ran_as(dop.op, want)
            d = torch.tensor([float(np.linalg.norm(y2 - y1[m.rows])) ** 2, float(np.linalg.norm(y1[m.rows])) ** 2],
                             device="cuda", dtype=torch.float64)
            dist.all_reduce(d)
            rel = float(np.sqrt(d[0].item() / max(d[1].item(), 1e-300)))
            ranks.verdict(ran and rel <= 1e-9, f"{label} expm_multiply z={z} {y2.dtype} products={prods} "
                                               f"rel_diff={rel:.1e} exchange={exch}")
        dop.op.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default=",".join(CASES), help="comma-separated cases of the mixed part")
    ap.add_argument("--parts", default="mixed,switch,batch,solvers")
    ap.add_argument("--switch-models", default="heisenberg_chain_16,heisenberg_kagome_12_symm,empty_rank")
    ap.add_argument("--batch-models", default="heisenberg_chain_16,momentum_sector,empty_rank")
    ap.add_argument("--solver-model", default="heisenberg_chain_16")
    ap.add_argument("models", nargs="*", default=SMALL)
    args = ap.parse_args()
    ranks = Ranks()
    po.set_num_threads(max(1, len(os.sched_getaffinity(0)) // ranks.world))
    parts = set(args.parts.split(","))
    cache = {}

    def model(name):
        if name not in cache:
            cache[name] = Model(name, ranks.rank, ranks.world, ranks.local)
        return cache[name]

    if "mixed" in parts:
        for name in args.models:
            for case in args.cases.split(","):
                check_mixed(model(name), case, ranks, ranks.local)
    if "switch" in parts:
        for name in args.switch_models.split(","):
            check_switch(model(name), ranks, ranks.local)
    if "batch" in parts:
        for name in args.batch_models.split(","):
            check_batch(model(name), ranks, ranks.local)
    if "solvers" in parts:
        check_solvers(model(args.solver_model), ranks, ranks.local)
    ranks.finish()


if __name__ == "__main__":
    main()
