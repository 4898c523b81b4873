"""Shared frame of the multi-rank check tools (expm_check.py, eigsh_check.py, zz_check.py, quadrature_check.py,
multi_gpu_check.py): one process per rank under torch.distributed.run, NCCL inside libdmv_b200.

    ranks = Ranks()                 # rank, world size and device of this process; the process group
    ranks.verdict(good, text)       # one line ending in OK or FAIL, printed by rank 0, a failure on any rank counts
    ranks.finish()                  # barrier, and the exit code: 1 if any verdict failed

With fewer GPUs than ranks, ranks share devices (round robin): the same exchanges then run through CUDA IPC on one
device.  `load(name)` reads a model of data/, or the 10-site momentum sector with a complex character.
"""
import os
import socket
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from distributed_matvec_b200 import load_config_from_yaml  # noqa: E402
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict  # noqa: E402


def load(name):
    if name == "momentum_sector":   # translation symmetry with a complex character (momentum sector 1)
        basis = basis_from_dict({"number_spins": 10, "hamming_weight": 5,
                                 "symmetries": [{"permutation": [(i + 1) % 10 for i in range(10)], "sector": 1}]})
        terms = [{"expression": f"σ{c}₀ σ{c}₁", "sites": [[i, (i + 1) % 10] for i in range(10)]} for c in "ˣʸᶻ"]
        return basis, operator_from_dict({"terms": terms}, basis)
    return load_config_from_yaml(os.path.join(ROOT, "data", name + ".yaml"))


class Ranks:
    def __init__(self):
        self.rank = int(os.environ["RANK"])
        self.world = int(os.environ["WORLD_SIZE"])
        self.local = int(os.environ["LOCAL_RANK"]) % torch.cuda.device_count()
        if torch.cuda.device_count() < self.world:
            # NCCL refuses two ranks of one host on one device; as ranks of distinct hosts they talk over loopback
            # sockets (the library's own NCCL communicator reads the same variables)
            os.environ["NCCL_HOSTID"] = f"{socket.gethostname()}-rank{self.rank}"
            os.environ.setdefault("NCCL_SOCKET_IFNAME", "lo")
            os.environ.setdefault("NCCL_IB_DISABLE", "1")
        torch.cuda.set_device(self.local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", self.local))
        self.failures = 0

    def verdict(self, good, text):
        flag = torch.tensor([0 if good else 1], device="cuda")
        dist.all_reduce(flag)
        if self.rank == 0:
            print(f"{text} {'OK' if int(flag) == 0 else 'FAIL'}", flush=True)
        self.failures += int(flag)

    def finish(self):
        dist.barrier()
        dist.destroy_process_group()
        sys.exit(1 if self.failures else 0)
