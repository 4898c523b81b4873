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
import os
import socket
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from distributed_matvec_b200 import DistributedOperator, Operator, load_config_from_yaml  # noqa: E402
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict  # noqa: E402
from distributed_matvec_b200.thermal import thermodynamics  # noqa: E402

DEFAULT = ["heisenberg_chain_10", "heisenberg_square_4x4", "momentum_sector", "heisenberg_chain_24"]
R, SEED = 4, 77
TEMPS = [0.25, 0.5, 1.0, 2.0, np.inf]


def load(name):
    if name == "momentum_sector":   # translation symmetry with a complex character (momentum sector 1)
        basis = basis_from_dict({"number_spins": 10, "hamming_weight": 5,
                                 "symmetries": [{"permutation": [(i + 1) % 10 for i in range(10)], "sector": 1}]})
        terms = [{"expression": f"σ{c}₀ σ{c}₁", "sites": [[i, (i + 1) % 10] for i in range(10)]} for c in "ˣʸᶻ"]
        return basis, operator_from_dict({"terms": terms}, basis)
    return load_config_from_yaml(os.path.join(ROOT, "data", name + ".yaml"))


def main():
    rank = int(os.environ["RANK"]); world = int(os.environ["WORLD_SIZE"]); local = int(os.environ["LOCAL_RANK"])
    local %= torch.cuda.device_count()
    if torch.cuda.device_count() < world:
        os.environ["NCCL_HOSTID"] = f"{socket.gethostname()}-rank{rank}"
        os.environ.setdefault("NCCL_SOCKET_IFNAME", "lo")
        os.environ.setdefault("NCCL_IB_DISABLE", "1")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    names = sys.argv[1:] or DEFAULT
    failures = 0

    def verdict(good, text):
        nonlocal failures
        flag = torch.tensor([0 if good else 1], device="cuda")
        dist.all_reduce(flag)
        if rank == 0:
            print(f"{text} {'OK' if int(flag) == 0 else 'FAIL'}", flush=True)
        failures += int(flag)

    for name in names:
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
    dist.barrier()
    dist.destroy_process_group()
    sys.exit(1 if failures else 0)


if __name__ == "__main__":
    main()
