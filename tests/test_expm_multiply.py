"""y = exp(z H) x on the device (dmv_expm_multiply / Operator.expm_multiply).

The references share nothing with the library: scipy.linalg.expm (and scipy.sparse.linalg.expm_multiply) of the
projected Hamiltonian built from Kronecker products (oracle/dense_pin.py), cross-checked against the oracle's dense
matrix (_dense_from_oracle of test_gpu_parity).  The host half (the tridiagonal exponential) is checked without a GPU.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.linalg
import scipy.sparse
import scipy.sparse.linalg
import yaml

from distributed_matvec_b200 import _native as nat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "data")


def _tridiagonal_expm(a, b, z):
    k = a.shape[0]
    a = np.ascontiguousarray(a, dtype=np.float64)
    b = np.ascontiguousarray(b if k > 1 else np.zeros(1), dtype=np.float64)
    c = np.zeros(2 * k)
    nat.check(nat.lib().dmv_debug_tridiagonal_expm(k, a.ctypes.data, b.ctypes.data, z.real, z.imag, c.ctypes.data))
    return c[0::2] + 1j * c[1::2]


def test_tridiagonal_expm_matches_scipy():
    """Host half of dmv_expm_multiply (implicit QL + exponential of the eigenvalues) against scipy.linalg.expm of the
    dense T, for real, imaginary and complex z up to |z| ||T|| ~ 50, decoupled blocks and clustered eigenvalues."""
    rng = np.random.default_rng(11)
    cases = [(rng.normal(size=k), rng.normal(size=max(k - 1, 0))) for k in (1, 2, 10, 64)]
    a, b = rng.normal(size=40), rng.normal(size=39)
    b[17] = 1e-13                                                    # nearly decoupled blocks
    cases.append((a, b))
    a, b = rng.normal(size=30), rng.normal(size=29)
    b[[5, 12, 20]] = 0.0                                             # exactly decoupled blocks
    cases.append((a, b))
    cases.append((np.full(30, 2.0), np.full(29, -1.0)))              # discrete Laplacian
    cases.append((np.concatenate([np.full(10, -3.0), rng.normal(size=10)]), np.full(19, 1e-9)))   # clustered
    cases.append((np.zeros(8), np.zeros(7)))                         # T = 0
    for a, b in cases:
        k = a.shape[0]
        T = np.diag(a) + (np.diag(b, 1) + np.diag(b, -1) if k > 1 else 0)
        w = np.linalg.eigvalsh(T)
        norm, mid = max(np.abs(w).max(), 1e-300), 0.5 * (w[0] + w[-1])
        for unit in (-1.0, -1j, np.exp(-0.7j), 0.3 - 1j):
            for size in (0.1, 3.0, 50.0):
                z = unit * size / max(norm, 1.0)
                # exp(z T) = exp(z mid) exp(z (T - mid)): the shift halves the norm scipy's scaling and squaring sees
                # (unshifted, its own error reaches 1.2e-12 at k = 64, z = -50 / ||T||)
                want = np.exp(z * mid) * scipy.linalg.expm(z * (T - mid * np.eye(k)))[:, 0]
                got = _tridiagonal_expm(a, b, z)
                assert np.linalg.norm(got - want) <= 1e-12 * np.linalg.norm(want), (k, z)


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
    """The two general models of test_gpu_parity.GENERAL_MODELS this file runs, with their term lists for the Kronecker
    construction (the test checks that the two definitions give the same matrix)."""
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


# model: which kernel runs the product, as info keys.  issue_01 (character -1) and momentum_sector (complex character)
# would run the scatter kernel by default; "mode" = 1 puts them on the queued row kernel k_pull.
SMALL = {
    "heisenberg_chain_10": {"gather": 1, "projection": 1},
    "heisenberg_chain_12": {"gather": 1},
    "heisenberg_square_4x4": {"rows": 1, "rows_tk": 4},
    "heisenberg_kagome_12_symm": {"rows": 1, "rows_tk": 0},
    "issue_01": {"mode": 1, "pull": 1, "gather": 0, "rows": 0},
    "momentum_sector": {"mode": 1, "pull": 1, "gather": 0, "rows": 0, "complex_coefficients": 1},
    "complex_hopping": {"gather": 1, "complex_coefficients": 1},
}
Z_VALUES = [-0.1j, -1j, -5j, -0.5, -2.0]


def _load(name):
    return _custom_model(name) if name in ("complex_hopping", "momentum_sector") else _yaml_model(name)


def _x(n, cplx, seed=3):
    rng = np.random.default_rng(seed)
    x = rng.random(n) - 0.5
    return x + 1j * (rng.random(n) - 0.5) if cplx else x


def _reference(Hp, x, z):
    if Hp.shape[0] <= 1200:
        return scipy.linalg.expm(z * Hp) @ x
    return scipy.sparse.linalg.expm_multiply(z * scipy.sparse.csr_matrix(Hp), x.astype(np.complex128))


def _check(y, y_ref, x, z):
    err = np.linalg.norm(y - y_ref)
    if z.real == 0.0:
        return err <= 1e-8 * np.linalg.norm(x), err / np.linalg.norm(x)
    return err <= 1e-8 * np.linalg.norm(y_ref), err / np.linalg.norm(y_ref)


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(SMALL))
def test_small_models_against_dense_expm(need_cuda, name):
    """exp(z H) x for real time (-0.1i, -1i, -5i) and imaginary time (-0.5, -2), float64 where allowed and complex128,
    against scipy.linalg.expm of the Kronecker-built H; host and device pointers agree, and y may alias x."""
    torch = _torch()
    from oracle import dense_pin as dp
    from distributed_matvec_b200 import Operator
    from test_gpu_parity import _dense_from_oracle
    basis, matrix, specs = _load(name)
    reps, _, Hp = dp.projected_hamiltonian(specs, basis, dense=True)
    op = Operator(matrix)
    if "mode" in SMALL[name]:
        op.set_option("mode", SMALL[name]["mode"])
    op.basis.build()
    assert np.array_equal(op.basis.representatives(), reps)
    for key, want in SMALL[name].items():
        if key != "mode":
            assert op.info(key) == want, (name, key, op.info(key))
    real_op = op.info("complex_coefficients") == 0
    if reps.shape[0] <= 1200:   # the oracle's dense matrix is a second, independent reference
        H2 = _dense_from_oracle(matrix, reps, True)
        assert np.abs(H2 - Hp).max() <= 1e-12 * max(1.0, np.abs(Hp).max()), name
    n = reps.shape[0]
    for z in Z_VALUES:
        z = complex(z)
        dtypes = [True] + ([False] if (z.imag == 0.0 and real_op) else [])
        for cplx in dtypes:
            x = _x(n, cplx)
            y_ref = _reference(Hp, x, z)
            y, prods, est = op.expm_multiply(x, z)
            assert y.dtype == x.dtype and prods >= 1
            good, rel = _check(y, y_ref, x, z)
            assert good, (name, z, cplx, rel, prods, est)
            yd, prods_d, _ = op.expm_multiply(torch.from_numpy(x).cuda(), z)
            assert prods_d == prods
            assert np.linalg.norm(yd.cpu().numpy() - y) <= 1e-12 * np.linalg.norm(y), (name, z, cplx)
            xa = x.copy()   # y aliasing x through the C ABI
            pr, e = C.c_int(), C.c_double()
            nat.check(nat.lib().dmv_expm_multiply(op._ctx, nat.DMV_C128 if cplx else nat.DMV_F64, z.real, z.imag,
                                                  xa.ctypes.data, xa.ctypes.data, 0, 1e-10, C.byref(pr), C.byref(e)))
            assert np.linalg.norm(xa - y) <= 1e-12 * np.linalg.norm(y), (name, z, cplx)
    # z = 0 returns x bit for bit; x = 0 returns 0
    x = _x(n, True)
    assert np.array_equal(op.expm_multiply(x, 0.0)[0], x)
    y0, p0, _ = op.expm_multiply(np.zeros(n, dtype=np.complex128), -1j)
    assert not np.any(y0) and p0 == 0
    op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["heisenberg_chain_10", "heisenberg_square_4x4", "momentum_sector"])
def test_krylov_dimensions(need_cuda, name):
    """krylov_dim 8, 30 and 64 meet the tolerance in real and imaginary time; with m = 2 every sub-step is one step of
    a two-vector Krylov space, and the call still converges through many small sub-steps."""
    from oracle import dense_pin as dp
    from distributed_matvec_b200 import Operator
    basis, matrix, specs = _load(name)
    reps, _, Hp = dp.projected_hamiltonian(specs, basis, dense=True)
    op = Operator(matrix)
    op.basis.build()
    x = _x(reps.shape[0], True, seed=8)
    for m in (8, 30, 64):
        for z in (-1j, -2.0):
            y, prods, est = op.expm_multiply(x, z, krylov_dim=m)
            good, rel = _check(y, _reference(Hp, x, z), x, z)
            assert good, (name, m, z, rel, prods, est)
    # m = 2: the local error of a sub-step of length h shrinks only like h^2, so it needs many sub-steps at a loose tol
    tol = 1e-4
    y, prods, est = op.expm_multiply(x, -0.1j, krylov_dim=2, tol=tol)
    err = np.linalg.norm(y - _reference(Hp, x, -0.1j))
    assert prods >= 100 and err <= 10 * tol * np.linalg.norm(x), (name, prods, err, est)
    op.close()


@pytest.mark.gpu
def test_medium_kagome_16_against_sparse_expm_multiply(need_cuda):
    """kagome_16 (12 870 states, k_gather) against scipy.sparse.linalg.expm_multiply of the sparse Kronecker-built H."""
    from oracle import dense_pin as dp
    from distributed_matvec_b200 import Operator
    basis, matrix, specs = _yaml_model("heisenberg_kagome_16")
    reps, _, Hp = dp.projected_hamiltonian(specs, basis, dense=False)
    op = Operator(matrix)
    op.basis.build()
    assert np.array_equal(op.basis.representatives(), reps) and reps.shape[0] == 12870
    for z, cplx in ((-1j, True), (-0.5, True), (-0.5, False)):
        x = _x(reps.shape[0], cplx, seed=9)
        y_ref = scipy.sparse.linalg.expm_multiply(z * Hp, x.astype(np.complex128))
        y, prods, est = op.expm_multiply(x, z)
        good, rel = _check(y, y_ref, x, complex(z))
        assert good, (z, cplx, rel, prods, est)
    op.close()


@pytest.mark.gpu
def test_single_bond_known_answer(need_cuda):
    """sigma.sigma on two sites from |up down>: the weight left on |up down> is cos^2(2 t) exactly."""
    from distributed_matvec_b200 import Operator
    from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
    basis = basis_from_dict({"number_spins": 2, "hamming_weight": None})
    matrix = operator_from_dict({"terms": [{"expression": f"σ{c}₀ σ{c}₁", "sites": [[0, 1]]} for c in "ˣʸᶻ"]}, basis)
    op = Operator(matrix)
    op.basis.build()
    reps = list(op.basis.representatives())
    assert reps == [0, 1, 2, 3]
    x = np.zeros(4, dtype=np.complex128)
    x[1] = 1.0
    for t in (0.1, 0.7, 2.5, 10.0):
        y, prods, est = op.expm_multiply(x, -1j * t)
        assert abs(abs(y[1]) ** 2 - np.cos(2 * t) ** 2) <= 1e-13, (t, y)
        assert abs(np.linalg.norm(y) - 1.0) <= 1e-13 and est == 0.0    # the Krylov space is exhausted: exact
    op.close()


@pytest.mark.gpu
def test_unitarity_and_energy_at_size(need_cuda):
    """6 x 6 square (k_rows, 15.8 M states), complex128, z = -0.05i: the norm and the energy are conserved, two steps
    compose to one, and evolving back returns x."""
    torch = _torch()
    from distributed_matvec_b200 import Operator
    _, matrix, _ = _yaml_model("heisenberg_square_6x6")
    op = Operator(matrix)
    op.basis.build()
    n = op.basis.numberStates()
    assert n > 15_000_000 and op.info("rows") == 1
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.complex(torch.rand(n, dtype=torch.float64, device="cuda", generator=g) - 0.5,
                      torch.rand(n, dtype=torch.float64, device="cuda", generator=g) - 0.5)
    nx = torch.linalg.norm(x).item()
    y, prods, est = op.expm_multiply(x, -0.05j)
    assert abs(torch.linalg.norm(y).item() - nx) <= 1e-10 * nx, (prods, est)
    ex = torch.vdot(x, op.matvec(x)).real.item()
    ey = torch.vdot(y, op.matvec(y)).real.item()
    assert abs(ey - ex) <= 1e-9 * abs(ex), (ex, ey)
    y2 = op.expm_multiply(op.expm_multiply(x, -0.02j)[0], -0.03j)[0]
    assert torch.linalg.norm(y2 - y).item() <= 1e-9 * nx
    back = op.expm_multiply(y, 0.05j)[0]
    assert torch.linalg.norm(back - x).item() <= 1e-9 * nx
    op.close()


@pytest.mark.gpu
def test_eigenvector_phase_chain_32_symm(need_cuda):
    """The Lanczos ground state of chain_32_symm only picks up the phase exp(-i E0 t) over t = 0.5."""
    torch = _torch()
    from distributed_matvec_b200 import Operator
    _, matrix, _ = _yaml_model("heisenberg_chain_32_symm")
    op = Operator(matrix)
    op.basis.build()
    e0, psi, iters, res = op.lanczos(max_iters=400, tol=1e-12)
    psi = torch.from_numpy(psi.astype(np.complex128)).cuda()
    t = 0.5
    y, prods, est = op.expm_multiply(psi, -1j * t)
    want = np.exp(-1j * e0 * t) * psi
    assert torch.linalg.norm(y - want).item() <= 1e-6, (e0, res, prods, est)
    op.close()


@pytest.mark.gpu
def test_repeated_call_is_bit_identical_chain_24(need_cuda):
    """k_gather products and the deterministic block reductions: two calls on one operator give the same bits."""
    torch = _torch()
    from distributed_matvec_b200 import Operator
    _, matrix, _ = _yaml_model("heisenberg_chain_24")
    op = Operator(matrix)
    op.basis.build()
    assert op.info("gather") == 1
    x = torch.from_numpy(_x(op.basis.numberStates(), True, seed=12)).cuda()
    y1, p1, e1 = op.expm_multiply(x, -0.3j)
    y2, p2, e2 = op.expm_multiply(x, -0.3j)
    assert torch.equal(y1, y2) and p1 == p2 and e1 == e2
    assert op.info("expm_dot_vectors") > 0 and op.info("expm_combine_vectors") > 0
    op.close()


@pytest.mark.gpu
def test_errors(need_cuda):
    from distributed_matvec_b200 import Operator
    basis, matrix, _ = _yaml_model("heisenberg_chain_10")
    op = Operator(matrix)
    op.basis.build()
    n = op.basis.numberStates()
    x = _x(n, True)
    for m in (-1, 1, 65, 100):
        with pytest.raises(nat.DmvError, match="krylov_dim"):
            op.expm_multiply(x, -1j, krylov_dim=m)
    for tol in (0.0, -1e-10, float("nan"), float("inf")):
        with pytest.raises(nat.DmvError, match="tol"):
            op.expm_multiply(x, -1j, tol=tol)
    for z in (complex(float("nan"), 0), complex(0, float("inf")), float("-inf")):
        with pytest.raises(nat.DmvError, match="finite"):
            op.expm_multiply(x, z)
    with pytest.raises(nat.DmvError, match="complex z"):
        op.expm_multiply(x.real.copy(), -1j)
    op.close()
    _, cm, _ = _custom_model("complex_hopping")
    op = Operator(cm)
    op.basis.build()
    with pytest.raises(nat.DmvError, match="complex"):
        op.expm_multiply(_x(op.basis.numberStates(), False), -0.5)
    op.close()
    op = Operator(matrix, rank=0, num_ranks=2)   # two ranks without a communicator
    op.basis.build()
    with pytest.raises(nat.DmvError, match="dmv_comm_init"):
        op.expm_multiply(_x(op.basis.numberStates(), True), -1j)
    op.close()


@pytest.mark.gpu
def test_collective_expm_two_ranks(need_cuda):
    """Two ranks (on two GPUs, or both on one): chain_10, square_4x4, chain_24_symm, momentum_sector and chain_24, the
    hashed y back in block order against the one-rank result to 1e-10 (tools/expm_check.py)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29547", os.path.join(ROOT, "tools", "expm_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    lines = [l for l in out.stdout.splitlines() if l.rstrip().endswith(("OK", "FAIL"))]
    assert out.returncode == 0 and len(lines) >= 13 and not any(l.rstrip().endswith("FAIL") for l in lines), \
        out.stdout[-4000:] + out.stderr[-2000:]
