"""The collective product on SEVERAL GPUs (one process per GPU, NCCL / NVLink inside libdmv_b200) against the oracle:
`matrixVectorProduct` on several locales (reference src/DistributedMatrixVector.chpl:1072-1093) with each of the three
exchanges, the collective block <-> hashed redistribution (src/BlockToHashed.chpl:87, src/HashedToBlock.chpl:67), Lanczos
across ranks and the host-owned products under NCCL.  Two ranks, on two GPUs when there are two, else both on the one GPU
(CUDA IPC mappings and flags within one device, NCCL between the ranks over loopback sockets):

    python -m pytest tests/test_multi_gpu.py -m gpu -q
"""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SMALL = ["heisenberg_chain_10", "heisenberg_chain_16", "heisenberg_square_4x4", "heisenberg_chain_24_symm"]
AT_SIZE = ["heisenberg_chain_24", "heisenberg_chain_32_symm", "heisenberg_square_6x6"]   # >= 10^6 states per rank


def _run(world, env, names, port):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.join(ROOT, "tools", "multi_gpu_check.py"),
           *names]
    out = subprocess.run(cmd, cwd=ROOT, env={**os.environ, **env}, capture_output=True, text=True, timeout=1500)
    lines = [l for l in out.stdout.splitlines() if l.rstrip().endswith(("OK", "FAIL"))]
    assert out.returncode == 0 and lines and not any(l.rstrip().endswith("FAIL") for l in lines), \
        out.stdout[-4000:] + out.stderr[-2000:]
    return lines


@pytest.mark.gpu
@pytest.mark.parametrize("exchange,peer_gather", [("-1", "-1"), ("2", "0"), ("1", "-1"), ("0", "-1")])
def test_collective_product_two_gpus(exchange, peer_gather):
    """auto (replicated x with the peer-direct gather), replicated x with the NCCL all-gather, peer-direct records,
    NCCL record buckets."""
    if not torch.cuda.is_available():
        pytest.fail("this test needs a CUDA device (no CPU fallback exists)")
    names = SMALL + (AT_SIZE if exchange in ("-1", "1") else AT_SIZE[:1])
    lines = _run(2, {"DMV_EXCHANGE": exchange, "DMV_PEER_GATHER": peer_gather}, names, 29531 + int(exchange) + 2)
    text = "\n".join(lines)
    if exchange == "-1":
        assert "replicated-x/peer-direct gather" in text
    if exchange == "2":
        assert "replicated-x/nccl all-gather" in text
    if exchange == "1":
        assert "records/peer-direct" in text
    if exchange == "0":
        assert "records/nccl" in text
