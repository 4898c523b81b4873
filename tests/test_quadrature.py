"""Finite-temperature Lanczos on the device (dmv_lanczos_quadrature / Operator.lanczos_quadrature) and the
thermodynamics built on it (distributed_matvec_b200.thermal).

References that share nothing with the library: numpy's dense eigh of the projected Hamiltonian built from Kronecker
products (oracle/dense_pin.py), scipy's eigh_tridiagonal, a numpy implementation of the same recurrence below (_ftlm),
the pinned ground-state energy and dimension of the 6 x 6 square, and dmv_expm_multiply (a separate device path with
full reorthogonalisation).  Without a GPU: the host quadrature, the thermodynamics and the numpy recurrence.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import yaml

from distributed_matvec_b200 import _native as nat
from distributed_matvec_b200.thermal import seeded_start_vectors, thermodynamics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "data")


def _quadrature(a, b):
    k = len(a)
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b if k > 1 else [0.0], dtype=np.float64)
    nodes, weights = np.zeros(k), np.zeros(k)
    nat.check(nat.lib().dmv_debug_tridiagonal_quadrature(k, a.ctypes.data, b.ctypes.data, nodes.ctypes.data,
                                                         weights.ctypes.data))
    return nodes, weights


def _ftlm(H, starts, M):
    """The library's recurrence in numpy: starts (R, n) -> (nodes [R, M], weights [R, M], steps_done [R]).  No
    normalised copies, the same breakdown rule, Gauss quadrature by scipy's eigh_tridiagonal."""
    from scipy.linalg import eigh_tridiagonal
    R, n = starts.shape
    M = min(M, n)
    Q = np.array(starts.T, dtype=np.result_type(starts, H))
    P = np.zeros_like(Q)
    b2, dots = [np.sum(np.abs(Q) ** 2, axis=0)], []
    with np.errstate(divide="ignore", invalid="ignore"):
        for j in range(M):
            W = H @ Q
            dots.append(np.real(np.sum(np.conj(Q) * W, axis=0)))
            if j + 1 == M:
                break
            bj2 = b2[j]
            dead = ~(bj2 > 0.0)
            if j > 0:
                bp2 = b2[j - 1]
                dead |= ~(bp2 > 0.0) | (np.sqrt(bj2) <= 1e-14 * np.maximum(1.0, np.abs(dots[j - 1] / bp2)))
            beta = np.sqrt(bj2)
            cw = np.where(dead, 0.0, 1.0 / beta)
            cq = np.where(dead, 0.0, dots[j] / bj2 / beta)
            cp = np.where(dead, 0.0, beta / np.sqrt(b2[j - 1])) if j > 0 else np.zeros(R)
            Rn = cw * W - cq * Q - cp * P
            Rn[:, dead] = 0.0
            Q[:, dead] = 0.0
            P, Q = Q, Rn
            b2.append(np.sum(np.abs(Q) ** 2, axis=0))
    nodes, weights, done = np.zeros((R, M)), np.zeros((R, M)), np.zeros(R, dtype=np.int64)
    for r in range(R):
        a, b = [], []
        for j in range(M):
            a.append(dots[j][r] / b2[j][r])
            if j + 1 == M:
                break
            bn2 = b2[j + 1][r]
            if not bn2 > 0.0 or np.sqrt(bn2) <= 1e-14 * max(1.0, abs(dots[j][r] / b2[j][r])):
                break
            b.append(np.sqrt(bn2))
        w, v = eigh_tridiagonal(np.array(a), np.array(b))
        k = len(a)
        nodes[r, :k], weights[r, :k], done[r] = w, b2[0][r] * v[0] ** 2, k
    return nodes, weights, done


def _load(name):
    """-> (basis spec, operator spec, term specs)"""
    from distributed_matvec_b200 import load_config_from_yaml
    from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
    if name.startswith("ring"):   # ring<n>_w<weight>_k<sector>: Heisenberg ring in a momentum sector
        n, w, k = (int(t[1:]) if i else int(t[4:]) for i, t in enumerate(name.split("_")))
        basis = basis_from_dict({"number_spins": n, "hamming_weight": w,
                                 "symmetries": [{"permutation": [(i + 1) % n for i in range(n)], "sector": k}]})
        specs = [{"expression": f"σ{c}₀ σ{c}₁", "sites": [[i, (i + 1) % n] for i in range(n)]} for c in "ˣʸᶻ"]
        return basis, operator_from_dict({"terms": specs}, basis), specs
    if name == "complex_hopping":
        basis = basis_from_dict({"number_spins": 10, "hamming_weight": 5})
        specs = [{"expression": "σ⁺₀ σ⁻₁", "sites": [[i, (i + 1) % 10] for i in range(10)]},
                 {"expression": "σ⁻₀ σ⁺₁", "sites": [[i, (i + 1) % 10] for i in range(10)]},
                 {"expression": "0.3j × σ⁺₀ σ⁻₁", "sites": [[i, (i + 2) % 10] for i in range(10)]},
                 {"expression": "-0.3j × σ⁻₀ σ⁺₁", "sites": [[i, (i + 2) % 10] for i in range(10)]}]
        return basis, operator_from_dict({"terms": specs}, basis), specs
    path = os.path.join(DATA, name + ".yaml")
    basis, matrix = load_config_from_yaml(path)
    with open(path, encoding="utf-8") as f:
        specs = yaml.safe_load(f)["hamiltonian"]["terms"]
    return basis, matrix, specs


def _dense(name):
    from oracle import dense_pin as dp
    basis, _, specs = _load(name)
    reps, _, Hp = dp.projected_hamiltonian(specs, basis, dense=True)
    return reps, Hp


TEMPS = np.array([0.25, 0.5, 1.0, 2.0, 4.0])


def _exact(w, temps):
    """(log Z, E, C, S) directly from a spectrum"""
    out = []
    for T in temps:
        beta = 0.0 if np.isinf(T) else 1.0 / T
        x = -beta * (w - w.min())
        p = np.exp(x)
        z = p.sum()
        p /= z
        e = p @ w
        log_z = np.log(z) - beta * w.min()
        out.append((log_z, e, beta ** 2 * (p @ w ** 2 - e ** 2), log_z + beta * e))
    return tuple(np.array(c) for c in zip(*out))


# ---------------------------------------------------------------------------------------------------------------- CPU
def test_tridiagonal_quadrature_matches_scipy():
    """Golub-Welsch on the host against scipy.linalg.eigh_tridiagonal: random T with k up to 400, a graded T and one
    with a split (tiny off-diagonal).  Nodes to 1e-12 relative, weights to 1e-12 absolute, sum of weights 1."""
    from scipy.linalg import eigh_tridiagonal
    rng = np.random.default_rng(5)
    cases = [(rng.normal(size=k), rng.normal(size=k - 1)) for k in (1, 2, 3, 10, 57, 200, 400)]
    cases.append((np.arange(40.0) ** 2, np.full(39, 0.5)))
    b = rng.uniform(0.5, 1.5, size=59)
    b[30] = 1e-18
    cases.append((rng.normal(size=60), b))
    for a, b in cases:
        k = len(a)
        nodes, weights = _quadrature(a, b)
        w, v = eigh_tridiagonal(a, b) if k > 1 else (a.copy(), np.ones((1, 1)))
        scale = max(1.0, np.abs(w).max())
        assert np.abs(nodes - w).max() <= 1e-12 * scale, (k, np.abs(nodes - w).max())
        assert np.abs(weights - v[0] ** 2).max() <= 1e-12, (k, np.abs(weights - v[0] ** 2).max())
        assert abs(weights.sum() - 1.0) <= 1e-12, k


def test_thermodynamics_exact_spectrum_kagome_12():
    """thermodynamics() on the exact spectrum of kagome_12 (weight 1 per level) against E, C, S computed directly, and
    against -d log Z / d beta and beta^2 d^2 log Z / d beta^2 by central differences; finite at beta = 1e3 and
    S = ln D at beta = 0."""
    _, Hp = _dense("heisenberg_kagome_12")
    w = np.linalg.eigvalsh(Hp)
    D = w.shape[0]
    sector = [(w[None, :], np.ones((1, D)), 1)]
    log_z, e, c, s = thermodynamics(sector, TEMPS)
    log_z0, e0, c0, s0 = _exact(w, TEMPS)
    assert np.allclose(log_z, log_z0, rtol=1e-13, atol=1e-12)
    assert np.allclose(e, e0, rtol=1e-12, atol=1e-12) and np.allclose(c, c0, rtol=1e-10, atol=1e-12)
    assert np.allclose(s, s0, rtol=1e-12, atol=1e-12)
    for T, ei, ci in zip(TEMPS, e, c):
        beta, h = 1.0 / T, 1e-4 / T
        lz = [thermodynamics(sector, [1.0 / (beta + d * h)])[0][0] for d in (-1, 0, 1)]
        assert abs(-(lz[2] - lz[0]) / (2 * h) - ei) <= 1e-6 * max(1.0, abs(ei)), T
        assert abs(beta ** 2 * (lz[2] - 2 * lz[1] + lz[0]) / h ** 2 - ci) <= 1e-4 * max(1.0, ci), T
    log_z, e, c, s = thermodynamics(sector, [1e-3, np.inf])
    assert np.all(np.isfinite([log_z, e, c, s]))
    assert abs(e[0] - w[0]) <= 1e-9 and s[0] >= -1e-9 and abs(log_z[0] + 1e3 * w[0]) <= 10.0
    assert abs(s[1] - np.log(D)) <= 1e-12 * np.log(D) and abs(log_z[1] - np.log(D)) <= 1e-12 * np.log(D)
    # sectors and multiplicities: two copies of the same sector double Z
    assert abs(thermodynamics([(w, np.ones(D), 2)], [np.inf])[0][0] - np.log(2 * D)) <= 1e-12


@pytest.mark.parametrize("name", ["heisenberg_chain_10", "heisenberg_kagome_12_symm"])
def test_numpy_ftlm_from_unit_vectors_is_exact(name):
    """The recurrence started from every unit vector e_i gives Tr e^{-beta H} = sum_i <e_i|e^{-beta H}|e_i> to 1e-10
    relative of dense eigh: pins the formula independently of the library."""
    _, Hp = _dense(name)
    H = np.real_if_close(Hp)
    d = H.shape[0]
    nodes, weights, done = _ftlm(H, np.eye(d), d)
    assert np.all(done >= 1) and np.allclose(weights.sum(axis=1), 1.0, rtol=0, atol=1e-13)
    w = np.linalg.eigvalsh(Hp)
    temps = np.array([np.inf, 10.0, 1.0, 0.2])
    log_z = thermodynamics([(nodes, weights, d)], temps)[0]
    assert np.abs(log_z - _exact(w, temps)[0]).max() <= 1e-10, (name, log_z - _exact(w, temps)[0])


def test_seeded_start_vectors():
    """+-1 (float64) or unit phases (complex128), |r|^2 = n, independent of the order of the representatives, and
    different for different seeds and vector indices."""
    reps = np.arange(1000, dtype=np.uint64) * np.uint64(2654435761)
    r = seeded_start_vectors(reps, 3, 42)
    assert set(np.unique(r)) == {-1.0, 1.0} and np.all((r ** 2).sum(axis=1) == 1000)
    perm = np.random.default_rng(0).permutation(1000)
    assert np.array_equal(seeded_start_vectors(reps[perm], 3, 42), r[:, perm])
    assert not np.array_equal(r[0], r[1]) and not np.array_equal(seeded_start_vectors(reps, 1, 43)[0], r[0])
    z = seeded_start_vectors(reps, 2, 42, complex_vectors=True)
    assert np.allclose(np.abs(z), 1.0, atol=1e-15) and abs(z.mean()) < 0.1


# ---------------------------------------------------------------------------------------------------------------- GPU
def _torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def need_cuda():
    if not _torch().cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


# model -> options (the queued row kernel k_pull for bases with complex characters, as in test_eigsh.py)
OPTIONS = {"issue_01": {"mode": 1}, "ring10_w5_k1": {"mode": 1}}


def _operator(name, build=True):
    from distributed_matvec_b200 import Operator
    _, matrix, _ = _load(name)
    op = Operator(matrix)
    for key, value in OPTIONS.get(name, {}).items():
        op.set_option(key, value)
    if build:
        op.basis.build()
    return op


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["heisenberg_chain_10", "heisenberg_square_4x4", "heisenberg_kagome_12_symm",
                                  "issue_01", "ring10_w5_k1"])
def test_gauss_moments(need_cuda, name):
    """M = 8 seeded steps: for every vector sum_k w_k theta_k^p = r^H H^p r for p = 0 .. 15 to 1e-10 of |H|^p |r|^2
    (Gauss exactness), with r rebuilt on the host by seeded_start_vectors (which checks the hash too)."""
    reps, Hp = _dense(name)
    op = _operator(name)
    assert np.array_equal(op.basis.representatives(), reps)
    norm = np.abs(np.linalg.eigvalsh(Hp)).max()
    for cplx in ([False, True] if op.info("complex_coefficients") == 0 else [True]):
        R = 5
        nodes, weights, done, prods = op.lanczos_quadrature(R, 8, seed=11, complex_vectors=cplx)
        assert nodes.shape == (R, 8) and prods == R * min(8, reps.shape[0])
        r = seeded_start_vectors(reps, R, 11, cplx)
        for i in range(R):
            v, r2 = r[i].copy(), np.vdot(r[i], r[i]).real
            assert abs(weights[i].sum() - r2) <= 1e-12 * r2
            for p in range(16):
                got = weights[i] @ nodes[i] ** p
                want = np.vdot(r[i], v).real
                assert abs(got - want) <= 1e-10 * norm ** p * r2, (name, cplx, i, p, got, want)
                v = Hp @ v
    op.close()


@pytest.mark.gpu
def test_unit_vectors_sum_to_the_whole_space_ring_10(need_cuda):
    """The 10-site Heisenberg ring: unit vectors as `start`, every Hamming weight x momentum sector (complex characters
    included, empty sectors skipped); the sum of the sector traces Tr e^{-beta H} is the trace over the whole 2^10 space
    from dense eigh, to 1e-10 relative for beta in {0, 0.1, 1, 5}."""
    from oracle import dense_pin as dp
    _, _, specs = _load("ring10_w5_k0")
    w_full = np.linalg.eigvalsh(dp.full_hamiltonian(specs, 10).toarray())
    betas = np.array([0.0, 0.1, 1.0, 5.0])
    shift = w_full.min()
    z = np.zeros(len(betas))
    total = 0
    for weight in range(11):
        for k in range(10):
            name = f"ring10_w{weight}_k{k}"
            reps, _ = _dense(name)
            d = reps.shape[0]
            if d == 0:
                continue
            total += d
            op = _operator(name, build=False)
            op.set_option("mode", 1)
            op.basis.build()
            nodes, weights, done, _ = op.lanczos_quadrature(d, d, start=np.eye(d, dtype=np.complex128))
            assert np.all(done >= 1) and np.allclose(weights.sum(axis=1), 1.0, rtol=0, atol=1e-12), name
            for i, beta in enumerate(betas):
                z[i] += np.sum(weights * np.exp(-beta * (nodes - shift)) * (weights > 0))
            op.close()
    assert total == 1024
    want = np.array([np.sum(np.exp(-beta * (w_full - shift))) for beta in betas])
    assert np.abs(z / want - 1.0).max() <= 1e-10, z / want - 1.0


def _jackknife(nodes, weights, temps):
    R = nodes.shape[0]
    est = np.array([thermodynamics([(np.delete(nodes, i, 0), np.delete(weights, i, 0), 1)], temps)[1:3]
                    for i in range(R)])                       # [R, 2, T]
    mean = est.mean(axis=0)
    return np.sqrt((R - 1) / R * ((est - mean) ** 2).sum(axis=0))


@pytest.mark.gpu
def test_statistics_kagome_12(need_cuda):
    """kagome_12 (924 states), R = 32, M = 60, fixed seed: E(T) and C(T) within 5 jackknife standard errors of the exact
    values; the same nodes and weights match the numpy recurrence on the same start vectors to 1e-9 in log Z, E, C."""
    reps, Hp = _dense("heisenberg_kagome_12")
    H = np.real_if_close(Hp)
    op = _operator("heisenberg_kagome_12")
    assert op.basis.numberStates() == 924
    nodes, weights, done, prods = op.lanczos_quadrature(32, 60, seed=2024)
    assert op.info("quadrature_group") == 4 and prods == 32 * 60
    log_z, e, c, _ = thermodynamics([(nodes, weights, 1)], TEMPS)
    _, e0, c0, _ = _exact(np.linalg.eigvalsh(Hp), TEMPS)
    se = _jackknife(nodes, weights, TEMPS)
    assert np.all(np.abs(e - e0) <= 5 * se[0]), (e - e0, se[0])
    assert np.all(np.abs(c - c0) <= 5 * se[1]), (c - c0, se[1])
    n2, w2, d2 = _ftlm(H, seeded_start_vectors(reps, 32, 2024), 60)
    assert np.array_equal(done, d2)
    ref = thermodynamics([(n2, w2, 1)], TEMPS)
    for got, want in zip((log_z, e, c), ref[:3]):
        assert np.abs(got - want).max() <= 1e-9 * max(1.0, np.abs(want).max()), got - want
    op.close()


def _log_z(nodes, weights, betas):
    return thermodynamics([(nodes, weights, 1)], 1.0 / np.asarray(betas))[0]


@pytest.mark.gpu
@pytest.mark.parametrize("name,group", [("heisenberg_chain_24", 4), ("heisenberg_square_4x4", 6)])
def test_batching_changes_nothing(need_cuda, name, group):
    """R = 8 in one call (chain_24: two k_gather launches of 4; square_4x4: k_rows_batch of 6 and 2) against eight
    calls with R = 1 on the same start vectors: log Z(beta) to 1e-10."""
    op = _operator(name)
    reps = op.basis.representatives()
    starts = seeded_start_vectors(reps, 8, 5)
    betas = [0.1, 0.5, 1.0, 2.0]
    nodes, weights, done, _ = op.lanczos_quadrature(8, 30, start=starts)
    assert op.info("quadrature_group") == group
    for i in range(8):
        n1, w1, d1, _ = op.lanczos_quadrature(1, 30, start=starts[i:i + 1])
        assert op.info("quadrature_group") == 1 and d1[0] == done[i]
        a, b = _log_z(nodes[i:i + 1], weights[i:i + 1], betas), _log_z(n1, w1, betas)
        assert np.abs(a - b).max() <= 1e-10, (name, i, a - b)
    op.close()


@pytest.mark.gpu
def test_square_6x6_at_size(need_cuda):
    """6 x 6 square, float64: R = 2, M = 400 seeded -- the lowest node within 1e-6 of the pinned -97.757589597 and
    Z(beta = 0) = 15 804 956 to 1e-12.  One caller-supplied vector with M = 100 (a torch tensor): sum_k w_k e^{-tau
    theta_k} = |exp(-tau H / 2) r|^2 from dmv_expm_multiply (tol 1e-12) to 1e-8 for tau in {0.1, 1}."""
    torch = _torch()
    op = _operator("heisenberg_square_6x6")
    n = op.basis.numberStates()
    assert n == 15_804_956 and op.info("rows") == 1
    nodes, weights, done, prods = op.lanczos_quadrature(2, 400, seed=42)
    assert op.info("quadrature_group") == 2 and prods == 800
    lowest = nodes[weights > 0].min()
    assert abs(lowest - (-97.757589597)) <= 1e-6, lowest
    assert abs(np.exp(thermodynamics([(nodes, weights, 1)], [np.inf])[0][0]) / n - 1.0) <= 1e-12
    r = torch.from_numpy(seeded_start_vectors(op.basis.representatives(), 1, 99)).cuda()
    nodes, weights, done, _ = op.lanczos_quadrature(1, 100, start=r)
    for tau in (0.1, 1.0):
        got = float(np.sum(weights[0] * np.exp(-tau * nodes[0]) * (weights[0] > 0)))
        y, _, _ = op.expm_multiply(r[0].contiguous(), -tau / 2, tol=1e-12)
        want = float(torch.sum(y * y).item())
        assert abs(got / want - 1.0) <= 1e-8, (tau, got, want)
    op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["heisenberg_chain_24", "heisenberg_square_4x4"])
def test_repeated_call_is_bit_identical(need_cuda, name):
    op = _operator(name)
    out = [op.lanczos_quadrature(8, 40, seed=3) for _ in range(2)]
    for a, b in zip(out[0], out[1]):
        assert np.array_equal(a, b)
    op.close()


@pytest.mark.gpu
def test_group_width(need_cuda):
    op = _operator("heisenberg_chain_24")
    op.lanczos_quadrature(8, 3)
    assert op.info("quadrature_group") == 4
    op.close()
    op = _operator("heisenberg_square_4x4")
    op.lanczos_quadrature(8, 3)
    assert op.info("quadrature_group") == 6
    op.lanczos_quadrature(8, 3, complex_vectors=True)
    assert op.info("quadrature_group") == 3
    op.close()


@pytest.mark.gpu
def test_errors(need_cuda):
    from distributed_matvec_b200 import Operator
    op = _operator("heisenberg_chain_10")
    n = op.basis.numberStates()
    for R in (0, -1):
        with pytest.raises(nat.DmvError, match="num_vectors"):
            op.lanczos_quadrature(R, 5)
    for M in (0, -3):
        with pytest.raises(nat.DmvError, match="steps"):
            op.lanczos_quadrature(2, M)
    start = np.ones((2, n))
    start[1] = 0.0
    with pytest.raises(nat.DmvError, match="zero"):
        op.lanczos_quadrature(2, 5, start=start)
    with pytest.raises(ValueError):
        op.lanczos_quadrature(3, 5, start=start)
    nodes, weights, done, prods = op.lanczos_quadrature(1, n + 50)   # steps cap at the dimension
    assert done[0] <= n and prods == n and np.all(nodes[0, n:] == 0) and np.all(weights[0, n:] == 0)
    op.close()
    op = _operator("complex_hopping")
    with pytest.raises(nat.DmvError, match="complex"):
        op.lanczos_quadrature(2, 5, complex_vectors=False)
    op.close()
    _, matrix, _ = _load("heisenberg_chain_10")
    op = Operator(matrix, rank=0, num_ranks=2)   # two ranks without a communicator
    op.basis.build()
    with pytest.raises(nat.DmvError, match="dmv_comm_init"):
        op.lanczos_quadrature(2, 5)
    op.close()
    # buffers that do not fit name the bytes they need: 128 MB free next to chain_24's 12 vectors of 21.6 MB
    torch = _torch()
    op = _operator("heisenberg_chain_24")
    op.matvec(np.zeros(op.basis.numberStates()))
    free, _ = torch.cuda.mem_get_info()
    hog = torch.empty(max(free - (128 << 20), 0), dtype=torch.uint8, device="cuda")
    try:
        with pytest.raises(nat.DmvError, match="bytes"):
            op.lanczos_quadrature(4, 5)
    finally:
        del hog
        torch.cuda.empty_cache()
    op.close()


@pytest.mark.gpu
def test_collective_quadrature_two_ranks(need_cuda):
    """Two ranks: chain_10, square_4x4, a momentum sector and chain_24 against one rank (tools/quadrature_check.py)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29557", os.path.join(ROOT, "tools", "quadrature_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    lines = [l for l in out.stdout.splitlines() if l.rstrip().endswith(("OK", "FAIL"))]
    assert out.returncode == 0 and len(lines) >= 4 and not any(l.rstrip().endswith("FAIL") for l in lines), \
        out.stdout[-4000:] + out.stderr[-2000:]
