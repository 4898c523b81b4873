"""The lowest eigenpairs on the device by block Krylov-Schur (dmv_eigsh / Operator.eigsh).

References that share nothing with the library: numpy's dense eigh of the projected Hamiltonian built from Kronecker
products (oracle/dense_pin.py), cross-checked against the oracle's dense matrix (_dense_from_oracle of test_gpu_parity);
the Bethe ansatz (tests/bethe.py) and the pinned ground-state energy of the 6 x 6 square.  The host half (the Hermitian
Jacobi eigensolver) is checked without a GPU.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import yaml

from distributed_matvec_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "data")


def _hermitian_eigen(A):
    k = A.shape[0]
    a = np.ascontiguousarray(A, dtype=np.complex128).view(np.float64)
    w, v = np.zeros(k), np.zeros((k, k), dtype=np.complex128)
    nat.check(nat.lib().dmv_debug_hermitian_eigen(k, a.ctypes.data, w.ctypes.data, v.ctypes.data))
    return w, v


def _clusters(w, gap):
    """[start, stop) ranges of eigenvalues closer than `gap` to their neighbour."""
    out, start = [], 0
    for i in range(1, len(w) + 1):
        if i == len(w) or w[i] - w[i - 1] > gap:
            out.append((start, i))
            start = i
    return out


def _projector(v):
    return v @ v.conj().T


def test_hermitian_eigen_matches_numpy():
    """Cyclic Jacobi against numpy.linalg.eigh: real and complex matrices of size 1, 2, 17, 64, exactly degenerate and
    1e-9-clustered spectra, a diagonal matrix and the arrowhead a restart leaves.  Eigenvalues to 1e-12 of the norm;
    eigenvectors through the projector onto every cluster (gap 1e-6), to 1e-12 / gap-limited accuracy."""
    rng = np.random.default_rng(17)
    cases = []
    for k in (1, 2, 17, 64):
        X = rng.normal(size=(k, k))
        cases.append(X + X.T)
        Z = rng.normal(size=(k, k)) + 1j * rng.normal(size=(k, k))
        cases.append(Z + Z.conj().T)
    for cplx in (False, True):
        Q, _ = np.linalg.qr(rng.normal(size=(30, 30)) + (1j * rng.normal(size=(30, 30)) if cplx else 0))
        lam = np.repeat([-2.0, -1.0, 0.5, 3.0, 4.0, 7.0], 5)                 # exactly degenerate, multiplicity 5
        cases.append((Q * lam) @ Q.conj().T)
        lam = np.concatenate([-1.0 + 1e-9 * np.arange(10), rng.normal(size=20)])   # clustered at 1e-9 spacing
        cases.append((Q * lam) @ Q.conj().T)
    cases.append(np.diag(rng.normal(size=20)))
    cases.append(np.diag(np.repeat([1.0, -3.0], 4)))
    for cplx in (False, True):   # arrowhead: diag(theta) bordered by a p x l coupling block, plus a dense tail
        l, p, m = 20, 4, 40
        A = np.zeros((m, m), dtype=np.complex128 if cplx else np.float64)
        A[:l, :l] = np.diag(np.sort(rng.normal(size=l)))
        B = rng.normal(size=(p, l)) * 1e-3 + (1j * rng.normal(size=(p, l)) * 1e-3 if cplx else 0)
        A[l:l + p, :l] = B
        A[:l, l:l + p] = B.conj().T
        X = rng.normal(size=(m - l, m - l)) + (1j * rng.normal(size=(m - l, m - l)) if cplx else 0)
        A[l:, l:] = X + X.conj().T
        cases.append(A)
    for A in cases:
        k = A.shape[0]
        norm = max(np.abs(np.linalg.eigvalsh(A)).max(), 1.0)
        w_ref, v_ref = np.linalg.eigh(A)
        w, v = _hermitian_eigen(A)
        assert np.all(np.diff(w) >= 0), k
        assert np.abs(w - w_ref).max() <= 1e-12 * norm, (k, np.abs(w - w_ref).max())
        assert np.abs(v.conj().T @ v - np.eye(k)).max() <= 1e-12, k
        for a, b in _clusters(w_ref, 1e-6 * norm):
            gap = min(w_ref[a] - w_ref[a - 1] if a > 0 else np.inf, w_ref[b] - w_ref[b - 1] if b < k else np.inf, norm)
            err = np.abs(_projector(v[:, a:b]) - _projector(v_ref[:, a:b])).max()
            assert err <= max(1e-12, 1e-14 * norm / gap), (k, a, b, err, gap)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def need_cuda():
    if not _torch().cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _yaml_model(name):
    from distributed_matvec_b200 import load_config_from_yaml
    path = os.path.join(DATA, name + ".yaml")
    basis, matrix = load_config_from_yaml(path)
    with open(path, encoding="utf-8") as f:
        specs = yaml.safe_load(f)["hamiltonian"]["terms"]
    return basis, matrix, specs


def _custom_model(name):
    from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
    if name == "complex_hopping":
        basis = basis_from_dict({"number_spins": 10, "hamming_weight": 5})
        specs = [{"expression": "σ⁺₀ σ⁻₁", "sites": [[i, (i + 1) % 10] for i in range(10)]},
                 {"expression": "σ⁻₀ σ⁺₁", "sites": [[i, (i + 1) % 10] for i in range(10)]},
                 {"expression": "0.3j × σ⁺₀ σ⁻₁", "sites": [[i, (i + 2) % 10] for i in range(10)]},
                 {"expression": "-0.3j × σ⁻₀ σ⁺₁", "sites": [[i, (i + 2) % 10] for i in range(10)]},
                 {"expression": "σᶻ₀", "sites": [[0], [3]]}]
    else:
        basis = basis_from_dict({"number_spins": 10, "hamming_weight": 5,
                                 "symmetries": [{"permutation": [(i + 1) % 10 for i in range(10)], "sector": 1}]})
        specs = [{"expression": f"σ{c}₀ σ{c}₁", "sites": [[i, (i + 1) % 10] for i in range(10)]} for c in "ˣʸᶻ"]
    return basis, operator_from_dict({"terms": specs}, basis), specs


# model -> options; issue_01 and momentum_sector run on the queued row kernel k_pull ("mode" 1)
SMALL = {
    "heisenberg_chain_10": {},
    "heisenberg_chain_12": {},
    "heisenberg_square_4x4": {},
    "heisenberg_kagome_12_symm": {},
    "issue_01": {"mode": 1},
    "momentum_sector": {"mode": 1},
    "complex_hopping": {},
}


def _load(name):
    return _custom_model(name) if name in ("complex_hopping", "momentum_sector") else _yaml_model(name)


def _operator(name):
    from oracle import dense_pin as dp
    from distributed_matvec_b200 import Operator
    basis, matrix, specs = _load(name)
    reps, _, Hp = dp.projected_hamiltonian(specs, basis, dense=True)
    op = Operator(matrix)
    for key, value in SMALL.get(name, {}).items():
        op.set_option(key, value)
    op.basis.build()
    assert np.array_equal(op.basis.representatives(), reps)
    return op, matrix, reps, Hp


def _check_pairs(op, Hp, nev, vals, vecs, res, conv, tol, label, p=None):
    """With a block at least as wide as every multiplicity (p None: assumed) the nev lowest eigenvalues of dense eigh
    come back with their multiplicities.  A block of p vectors finds min(multiplicity, p) copies of a degenerate
    eigenvalue: then the returned values are the lowest DISTINCT eigenvalues, each with between min(multiplicity, p) and
    multiplicity copies (the last one may be cut at nev)."""
    w_all = np.linalg.eigvalsh(Hp)
    assert conv == nev, (label, conv, res)
    close = lambda a, b: abs(a - b) <= 1e-9 * max(1.0, abs(b))   # noqa: E731
    if p is None:
        w = w_all[:nev]
        assert all(close(vals[i], w[i]) for i in range(nev)), (label, vals - w)
    else:
        levels = [(w_all[a], b - a) for a, b in _clusters(w_all, 1e-8 * max(1.0, np.abs(w_all).max()))]
        got = [(vals[a], b - a) for a, b in _clusters(vals, 1e-8 * max(1.0, np.abs(vals).max()))]
        for j, (value, copies) in enumerate(got):
            want, mult = levels[j]
            assert close(value, want), (label, j, value, want)
            assert copies <= mult and (copies >= min(mult, p) or j == len(got) - 1), (label, j, copies, mult)
    assert np.abs(vecs.conj() @ vecs.T - np.eye(nev)).max() <= 1e-10, label
    for i in range(nev):
        r = np.linalg.norm(op.matvec(np.ascontiguousarray(vecs[i])) - vals[i] * vecs[i])
        assert r <= 10 * tol * max(1.0, abs(vals[i])), (label, i, r, res[i])


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SMALL))
def test_small_models_against_dense_eigh(need_cuda, name):
    """nev = 6 at block sizes 1 and 3, float64 where the operator is real and complex128: eigenvalues to 1e-9 of dense
    eigh (a block of p vectors finds min(multiplicity, p) copies of a degenerate level), re-measured residuals
    |H y - theta y| <= 10 tol, orthonormal vectors, every pair converged."""
    from test_gpu_parity import _dense_from_oracle
    op, matrix, reps, Hp = _operator(name)
    if reps.shape[0] <= 1200:   # the oracle's dense matrix is a second, independent reference
        H2 = _dense_from_oracle(matrix, reps, True)
        assert np.abs(H2 - Hp).max() <= 1e-12 * max(1.0, np.abs(Hp).max()), name
    tol = 1e-10
    for cplx in ([False, True] if op.info("complex_coefficients") == 0 else [True]):
        for p in (1, 3):
            vals, vecs, res, conv, prods, rst = op.eigsh(6, block_size=p, tol=tol, complex_vectors=cplx)
            assert vecs.dtype == (np.complex128 if cplx else np.float64) and prods > 0
            _check_pairs(op, Hp, 6, vals, vecs, res, conv, tol, (name, cplx, p, prods, rst), p=p)
    op.close()


@pytest.mark.gpu
def test_multiplicities_chain_12(need_cuda):
    """chain_12 without projections has many degenerate levels (the +-k pairs and the SU(2) multiplets).  With block
    sizes >= 2 every eigenvalue among the 8 lowest comes back with its multiplicity, and the projector onto each complete
    eigenspace equals that of dense eigh to 1e-8."""
    op, _, reps, Hp = _operator("heisenberg_chain_12")
    w, v = np.linalg.eigh(Hp)
    nev = 8
    groups = [(a, b) for a, b in _clusters(w, 1e-8) if a < nev]
    assert any(b - a > 1 for a, b in groups)
    for p in (2, 4):
        vals, vecs, res, conv, prods, rst = op.eigsh(nev, block_size=p)
        assert conv == nev, (p, res)
        assert np.abs(vals - w[:nev]).max() <= 1e-9 * np.abs(w).max(), (p, vals, w[:nev])
        for a, b in groups:
            if b > nev:   # the last multiplet may be cut at nev
                continue
            P = _projector(vecs[a:b].T)
            err = np.abs(P - _projector(v[:, a:b])).max()
            assert err <= 1e-8, (p, a, b, err)
    op.close()


@pytest.mark.gpu
def test_whole_space_chain_4(need_cuda):
    """nev = 6, the whole dimension of chain_4: the basis spans the space and the whole spectrum comes back; nev > 6
    raises."""
    op, _, reps, Hp = _operator("heisenberg_chain_4")
    assert reps.shape[0] == 6
    for p in (0, 1, 3, 6):
        vals, vecs, res, conv, prods, rst = op.eigsh(6, block_size=p)
        _check_pairs(op, Hp, 6, vals, vecs, res, conv, 1e-10, ("chain_4", p))
    with pytest.raises(nat.DmvError, match="nev"):
        op.eigsh(7)
    op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SMALL))
def test_consistent_with_lanczos_and_lobpcg(need_cuda, name):
    """theta_0 equals dmv_lanczos to 1e-10 relative; on chain_10 and square_4x4 the three lowest equal lobpcg(k = 3)."""
    from distributed_matvec_b200.eigensolver import lobpcg
    op, _, _, _ = _operator(name)
    cplx = op.info("complex_coefficients") != 0
    vals = op.eigsh(6, tol=1e-12, complex_vectors=cplx, eigenvectors=False)[0]
    e0 = op.lanczos(max_iters=400, tol=1e-12, complex_vectors=cplx, eigenvector=False)[0]
    assert abs(vals[0] - e0) <= 1e-10 * abs(e0), (name, vals[0], e0)
    if name in ("heisenberg_chain_10", "heisenberg_square_4x4"):
        lo = np.asarray(lobpcg(op, k=3, tol=1e-10, max_iters=500)[0], dtype=np.float64)
        assert np.abs(vals[:3] - lo).max() <= 1e-8 * np.abs(lo).max(), (name, vals[:3], lo)
    op.close()


@pytest.mark.gpu
def test_square_6x6_at_size(need_cuda):
    """6 x 6 square (15.8 M states, k_rows / k_rows_batch), float64, nev = 4: theta_0 within 1e-6 of the pinned
    -97.757589597, explicit residuals <= 10 tol, and block sizes 1 and 4 agree on the four eigenvalues to 1e-9."""
    torch = _torch()
    from distributed_matvec_b200 import Operator
    _, matrix, _ = _yaml_model("heisenberg_square_6x6")
    op = Operator(matrix)
    op.basis.build()
    n = op.basis.numberStates()
    assert n > 15_000_000 and op.info("rows") == 1
    tol = 1e-10
    vecs = torch.empty((4, n), dtype=torch.float64, device="cuda")
    vals4, _, res4, conv4, prods4, rst4 = op.eigsh(4, block_size=4, tol=tol, eigenvectors=vecs)
    assert conv4 == 4, (res4, prods4, rst4)
    assert abs(vals4[0] - (-97.757589597)) <= 1e-6, vals4
    for i in range(4):
        r = torch.linalg.norm(op.matvec(vecs[i].contiguous()) - vals4[i] * vecs[i]).item()
        assert r <= 10 * tol * max(1.0, abs(vals4[i])), (i, r, res4[i])
    vals1, _, res1, conv1, prods1, rst1 = op.eigsh(4, block_size=1, tol=tol, eigenvectors=False)
    assert conv1 == 4, (res1, prods1, rst1)
    assert np.abs(vals1 - vals4).max() <= 1e-9 * np.abs(vals4).max(), (vals1, vals4)
    op.close()


@pytest.mark.gpu
def test_chain_32_symm_bethe(need_cuda):
    import bethe
    from distributed_matvec_b200 import Operator
    _, matrix, _ = _yaml_model("heisenberg_chain_32_symm")
    op = Operator(matrix)
    op.basis.build()
    want = 4.0 * bethe.heisenberg_ring_e0(32)
    vals = op.eigsh(2, tol=1e-11, eigenvectors=False)[0]
    assert abs(vals[0] - want) <= 1e-8 * abs(want), (vals[0], want)
    op.close()


@pytest.mark.gpu
def test_repeated_call_is_bit_identical_chain_24(need_cuda):
    torch = _torch()
    from distributed_matvec_b200 import Operator
    _, matrix, _ = _yaml_model("heisenberg_chain_24")
    op = Operator(matrix)
    op.basis.build()
    assert op.info("gather") == 1
    n = op.basis.numberStates()
    out = []
    for _ in range(2):
        vecs = torch.empty((4, n), dtype=torch.float64, device="cuda")
        vals, _, res, conv, prods, rst = op.eigsh(4, eigenvectors=vecs)
        torch.cuda.synchronize()
        out.append((vals, vecs, res, conv, prods, rst))
    a, b = out
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2]) and torch.equal(a[1], b[1])
    assert a[3:] == b[3:] and a[3] == 4
    assert op.info("eigsh_block_vectors") > 0 and op.info("eigsh_rotate_vectors") > 0
    op.close()


@pytest.mark.gpu
def test_errors(need_cuda):
    from distributed_matvec_b200 import Operator
    basis, matrix, _ = _yaml_model("heisenberg_chain_10")
    op = Operator(matrix)
    op.basis.build()
    n = op.basis.numberStates()
    for k in (0, -1, n + 1):
        with pytest.raises(nat.DmvError, match="nev"):
            op.eigsh(k, eigenvectors=False)
    for tol in (0.0, -1e-10, float("nan"), float("inf")):
        with pytest.raises(nat.DmvError, match="tol"):
            op.eigsh(2, tol=tol)
    for p in (-1, 7, 100):
        with pytest.raises(nat.DmvError, match="block_size"):
            op.eigsh(2, block_size=p)
    for m, p in ((-1, 0), (65, 0), (100, 0), (5, 2), (62, 4)):   # (5, 2): below nev + 2p; (62, 4): m + p > 65
        with pytest.raises(nat.DmvError, match="krylov_dim"):
            op.eigsh(2, block_size=p, krylov_dim=m)
    with pytest.raises(nat.DmvError, match="max_restarts"):
        op.eigsh(2, max_restarts=-1)
    # stopping at max_restarts is not an error: the caller reads `converged`
    vals, _, res, conv, prods, rst = op.eigsh(6, block_size=1, krylov_dim=8, max_restarts=0, eigenvectors=False)
    assert rst == 0 and 0 <= conv <= 6 and prods == 8
    op.close()
    _, cm, _ = _custom_model("complex_hopping")
    op = Operator(cm)
    op.basis.build()
    with pytest.raises(nat.DmvError, match="complex"):
        op.eigsh(2, complex_vectors=False)
    op.close()
    op = Operator(matrix, rank=0, num_ranks=2)   # two ranks without a communicator
    op.basis.build()
    with pytest.raises(nat.DmvError, match="dmv_comm_init"):
        op.eigsh(2)
    op.close()
    # a basis that does not fit names the bytes it needs: leave 256 MB free next to chain_24's 36 vectors of 21.6 MB
    torch = _torch()
    _, c24, _ = _yaml_model("heisenberg_chain_24")
    op = Operator(c24)
    op.basis.build()
    op.matvec(np.zeros(op.basis.numberStates()))
    free, _ = torch.cuda.mem_get_info()
    hog = torch.empty(max(free - (256 << 20), 0), dtype=torch.uint8, device="cuda")
    try:
        with pytest.raises(nat.DmvError, match="bytes"):
            op.eigsh(4, eigenvectors=False)
    finally:
        del hog
        torch.cuda.empty_cache()
    op.close()


@pytest.mark.gpu
def test_collective_eigsh_two_ranks(need_cuda):
    """Two ranks: chain_10, square_4x4, momentum_sector and chain_24 against one rank (tools/eigsh_check.py)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--standalone",
           os.path.join(ROOT, "tools", "eigsh_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    lines = [l for l in out.stdout.splitlines() if l.rstrip().endswith(("OK", "FAIL"))]
    assert out.returncode == 0 and len(lines) >= 4 and not any(l.rstrip().endswith("FAIL") for l in lines), \
        out.stdout[-4000:] + out.stderr[-2000:]
