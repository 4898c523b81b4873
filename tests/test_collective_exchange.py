"""The record exchanges of the collective product on two, three and four ranks (tools/exchange_check.py, one process per
rank, NCCL / NVLink inside libdmv_b200) against the oracle: NCCL record buckets, one-shot peer-direct records, peer-direct
records in 2, 3, 5 and 64 overlapped rounds and in the automatic number, replicated x with either all-gather; a world
in which a rank owns no state; products of alternating element widths back to back on one context (the two record
buffers of the rounds); option changes between products; a batched product; and Lanczos, eigsh and expm_multiply
through the record exchanges against one rank.  With fewer GPUs than ranks the ranks share devices (CUDA IPC within a
device, NCCL between the ranks over loopback sockets):

    python -m pytest tests/test_collective_exchange.py -m gpu -q

One launch per world runs the small models through every case, a second one (two and three ranks) the at-size chain;
the tests of that world read their lines from those runs.
"""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

WORLDS = (2, 3, 4)
CASES = ("nccl", "oneshot", "rounds2", "rounds3", "rounds5", "rounds64", "repl_peer", "repl_nccl")
AT_SIZE = "heisenberg_chain_24"            # 2.7 million states: at least 2^18 per rank
PORTS = {2: 29611, 3: 29621, 4: 29631}     # (test_multi_gpu.py and the solver tests use 29511 .. 29599)
# the exchange each case must report it ran
RAN = {"nccl": "records/nccl", "oneshot": "records/peer-direct", "rounds2": "records/peer-direct in 2 rounds",
       "rounds3": "records/peer-direct in 3 rounds", "rounds5": "records/peer-direct in 5 rounds",
       "rounds64": "records/peer-direct in 64 rounds", "rounds_auto": "records/peer-direct in 4 rounds",
       "repl_peer": "replicated-x/peer-direct gather", "repl_nccl": "replicated-x/nccl all-gather"}

_runs = {}


def _run(world, args, key):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}",
           "--master-addr", "127.0.0.1", "--master-port", str(PORTS[world] + key),
           os.path.join(ROOT, "tools", "exchange_check.py"), *args]
    out = subprocess.run(cmd, cwd=ROOT, env=dict(os.environ), capture_output=True, text=True, timeout=1200)
    lines = [l.rstrip() for l in out.stdout.splitlines() if l.rstrip().endswith(("OK", "FAIL"))]
    return out.returncode, lines, out.stdout[-4000:] + out.stderr[-3000:]


def _world(world):
    if world not in _runs:
        if not torch.cuda.is_available():
            pytest.fail("this test needs a CUDA device (no CPU fallback exists)")
        runs = [_run(world, ["--cases", ",".join(CASES)], 0)]
        if world <= 3:
            runs.append(_run(world, ["--cases", "rounds_auto,nccl", "--parts", "mixed", AT_SIZE], 1))
        _runs[world] = runs
    return _runs[world]


def _lines(world, case):
    """The lines of `case` at `world` ranks, every one OK; a run that ended without a FAIL line must have exited 0."""
    runs = _world(world)
    for rc, lines, tail in runs:
        assert rc == 0 or any(l.endswith("FAIL") for l in lines), tail
    mine = [l for _, lines, _ in runs for l in lines if l.startswith(f"case={case} ")]
    assert mine, f"no line for case {case} at P={world}:\n" + "\n".join(tail for _, _, tail in runs)
    print("\n".join(mine))
    bad = [l for l in mine if l.endswith("FAIL")]
    assert not bad, "\n".join(bad)
    return mine


def _ran(line, exchange):
    return line.endswith(f" exchange={exchange} OK")


@pytest.mark.gpu
@pytest.mark.parametrize("world,case", [(w, c) for w in WORLDS for c in CASES] + [(2, "rounds_auto"), (3, "rounds_auto")])
def test_record_exchange(world, case):
    """Every small model (the at-size chain at two and three ranks) through one exchange: device products f64 f64 c128
    f64 c128 c128 f64 back to back on one context, then a host product, each y against the oracle; the exchange that
    ran is the one asked for."""
    lines = _lines(world, case)
    assert all(_ran(l, RAN[case]) for l in lines), lines
    assert all(" mixed " in l for l in lines)
    assert any("f64/f64/c128/f64/c128/c128/f64" in l for l in lines)
    if case == "rounds_auto" or (case == "nccl" and world <= 3):
        assert any(AT_SIZE + " " in l for l in lines)
    if case != "rounds_auto":
        assert any("momentum_sector" in l and "c128/c128/c128/c128/c128/c128/c128" in l for l in lines)


@pytest.mark.gpu
@pytest.mark.parametrize("world", WORLDS)
def test_empty_rank(world):
    """A ring of a few spins at Hamming weight 1 or n - 1 in which a rank owns no state: every exchange still returns
    the oracle's y, and no rank waits for ever on flags or barriers."""
    lines = [l for case in CASES for l in _lines(world, case) if "empty_rank" in l]
    assert len(lines) == len(CASES) and all("empty_ranks=" in l for l in lines), lines


@pytest.mark.gpu
@pytest.mark.parametrize("world", WORLDS)
def test_option_changes_between_products(world):
    """rounds 3 -> 2 -> 0, exchange 1 -> 0 -> 2 -> 1 and rounds 3 -> 5 on a live context (a chain, a symmetric kagome
    cluster, the empty-rank ring): every product after a change sets its exchange up again, runs the one asked for and
    equals the oracle."""
    lines = _lines(world, "switch")
    ran = ("records/peer-direct in 3 rounds", "records/peer-direct in 2 rounds", "records/peer-direct", "records/nccl",
           "replicated-x/peer-direct gather", "records/peer-direct in 3 rounds", "records/peer-direct in 5 rounds")
    assert len(lines) == len(ran) * 3
    for step, exchange in enumerate(ran):
        at = [l for l in lines if f" step={step} " in l]
        assert len(at) == 3 and all(_ran(l, exchange) for l in at), at


@pytest.mark.gpu
@pytest.mark.parametrize("world", WORLDS)
def test_batch_through_rounds(world):
    """matvec_batch of three vectors, f64 then c128, through three rounds (a chain, the momentum sector, the empty-rank
    ring), against the oracle."""
    lines = _lines(world, "batch")
    assert len(lines) == 6 and all(_ran(l, "records/peer-direct in 3 rounds") for l in lines), lines


@pytest.mark.gpu
@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("case", ("solvers_rounds2", "solvers_nccl"))
def test_solvers_through_records(world, case):
    """Lanczos, eigsh and expm_multiply (real and imaginary time) through the record exchanges equal the one-rank
    results: energies to 1e-10 relative, vectors to 1e-9, and every rank reports the same energies."""
    lines = _lines(world, case)
    exchange = "records/peer-direct in 2 rounds" if case == "solvers_rounds2" else "records/nccl"
    assert len(lines) == 4 and all(_ran(l, exchange) for l in lines), lines
