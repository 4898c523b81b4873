"""Spin-spin correlations on the device (dmv_zz_correlations / Operator.zz_correlations).

References that share nothing with the library: the state psi = B x on the full 2^n space, with the symmetry-adapted
basis B built explicitly by oracle/dense_pin.py, where <σᶻᵢσᶻⱼ> and <σᶻᵢ> are read off |psi_s|^2 directly; the
Bethe ansatz (tests/bethe.py); the pinned ground-state energy of the 6 x 6 square; and the library's own diagonal
kernel (dmv_apply_diag), an independent path to the same sums.  The formula itself and the host half (the group
average) are checked without a GPU.
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


def _ring(n, weight, sector):
    """Heisenberg ring of n sites at a fixed Hamming weight in a momentum sector (complex characters for sector != 0,
    and a non-zero magnetisation for weight != n / 2)."""
    from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
    basis = basis_from_dict({"number_spins": n, "hamming_weight": weight,
                             "symmetries": [{"permutation": [(i + 1) % n for i in range(n)], "sector": sector}]})
    specs = [{"expression": f"σ{c}₀ σ{c}₁", "sites": [[i, (i + 1) % n] for i in range(n)]} for c in "ˣʸᶻ"]
    return basis, operator_from_dict({"terms": specs}, basis)


def _load(name):
    """-> (basis spec, operator spec)"""
    from distributed_matvec_b200 import load_config_from_yaml
    from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
    if name == "momentum_sector":
        return _ring(10, 5, 1)
    if name.startswith("ring10_w3_k"):
        return _ring(10, 3, int(name[-1]))
    if name == "complex_hopping":
        basis = basis_from_dict({"number_spins": 10, "hamming_weight": 5})
        specs = [{"expression": "σ⁺₀ σ⁻₁", "sites": [[i, (i + 1) % 10] for i in range(10)]},
                 {"expression": "σ⁻₀ σ⁺₁", "sites": [[i, (i + 1) % 10] for i in range(10)]},
                 {"expression": "0.3j × σ⁺₀ σ⁻₁", "sites": [[i, (i + 2) % 10] for i in range(10)]},
                 {"expression": "-0.3j × σ⁻₀ σ⁺₁", "sites": [[i, (i + 2) % 10] for i in range(10)]},
                 {"expression": "σᶻ₀", "sites": [[0], [3]]}]
        return basis, operator_from_dict({"terms": specs}, basis)
    return load_config_from_yaml(os.path.join(DATA, name + ".yaml"))


def _group(basis):
    """(perms [G, N], flips [G]) the correlations are averaged over: the basis group, {1} without projection"""
    n = basis.number_sites
    if not basis.requires_projection():
        return np.arange(n)[None, :], np.zeros(1, dtype=np.uint8)
    g = basis.group
    return np.asarray(g.perms), np.asarray(g.flips)


def _spins(states, n):
    """s[b, i] = +1 / -1 for bit i of states[b] set / clear"""
    bits = (states[:, None] >> np.arange(n, dtype=np.uint64)[None, :]) & np.uint64(1)
    return 2.0 * bits.astype(np.float64) - 1.0


def _full_space(basis, B, x):
    """<σᶻᵢσᶻⱼ> and <σᶻᵢ> of psi = B x, read off the full 2^n space"""
    n = basis.number_sites
    p = np.abs(B @ x) ** 2
    keep = np.nonzero(p)[0]
    s = _spins(keep.astype(np.uint64), n)
    w = p[keep] / p.sum()
    return (s * w[:, None]).T @ s, w @ s


def _gram(reps, x, n):
    """(N + 1) x N block sum_b |x_b|^2 a(r_b) s(r_b)^T with a = (s, 1)"""
    s = _spins(reps, n)
    a = np.concatenate([s, np.ones((s.shape[0], 1))], axis=1)
    return (a * (np.abs(x) ** 2)[:, None]).T @ s


def _symmetrize(gram, perms, flips):
    n = gram.shape[1]
    W = gram[0, 0]
    Cm = np.zeros((n, n))
    m = np.zeros(n)
    for p, f in zip(perms, flips):
        Cm += gram[np.ix_(p, p)]
        m += (-1.0 if f else 1.0) * gram[n, p]
    return Cm / (len(perms) * W), m / (len(perms) * W)


FORMULA = ["heisenberg_chain_10", "heisenberg_square_4x4", "heisenberg_kagome_12_symm", "issue_01", "momentum_sector",
           "ring10_w3_k0", "ring10_w3_k1", "ring10_w3_k3"]


@pytest.mark.parametrize("name", FORMULA)
def test_formula_against_full_space(name):
    """The Gram-and-average formula equals <psi|σᶻᵢσᶻⱼ|psi> and <psi|σᶻᵢ|psi> on psi = B x for random complex x, to
    1e-12: this pins the direction of the permutations and the flip convention independently of the library."""
    from oracle import dense_pin as dp
    basis, _ = _load(name)
    reps, _, B = dp.symmetry_adapted_basis(basis)
    rng = np.random.default_rng(7)
    x = rng.normal(size=reps.shape[0]) + 1j * rng.normal(size=reps.shape[0])
    C_ref, m_ref = _full_space(basis, B, x)
    perms, flips = _group(basis)
    Cf, mf = _symmetrize(_gram(reps, x, basis.number_sites), perms, flips)
    assert np.abs(Cf - C_ref).max() <= 1e-12, name
    assert np.abs(mf - m_ref).max() <= 1e-12, name
    if name.startswith("ring10_w3"):
        assert np.abs(m_ref + 0.4).max() <= 1e-12   # 3 of 10 spins up in every state: m = (3 - 7) / 10
    if basis.has_spin_inversion_symmetry() and not basis.has_permutation_symmetries():
        assert np.abs(Cf - _gram(reps, x, basis.number_sites)[:-1] / np.sum(np.abs(x) ** 2)).max() <= 1e-12
        assert np.abs(mf).max() <= 1e-15


def _basis_desc(basis):
    bd = nat.BasisDesc()
    bd.number_sites = basis.number_sites
    bd.hamming_weight = -1 if basis.hamming_weight is None else basis.hamming_weight
    bd.spin_inversion = basis.spin_inversion
    bd.has_permutations = int(basis.has_permutation_symmetries())
    keep = []
    if basis.has_permutation_symmetries():
        g = basis.group
        keep = [np.ascontiguousarray(g.perms, dtype=np.int32), np.ascontiguousarray(g.flips, dtype=np.uint8),
                np.ascontiguousarray(g.characters, dtype=np.complex128)]
        bd.group_order = len(g)
        bd.perms, bd.flips, bd.characters = (a.ctypes.data for a in keep)
    return bd, keep


@pytest.mark.parametrize("name", FORMULA + ["heisenberg_chain_12"])
def test_host_symmetrize_matches_numpy(name):
    """dmv_debug_zz_symmetrize equals the numpy group average on random Gram blocks, to 1e-14."""
    basis, _ = _load(name)
    n = basis.number_sites
    bd, keep = _basis_desc(basis)
    perms, flips = _group(basis)
    rng = np.random.default_rng(11)
    for _ in range(3):
        gram = rng.normal(size=(n + 1, n))
        gram[0, 0] = 1.0 + rng.random()
        Cd, md = np.zeros((n, n)), np.zeros(n)
        nat.check(nat.lib().dmv_debug_zz_symmetrize(C.byref(bd), gram.ctypes.data, Cd.ctypes.data, md.ctypes.data))
        Cf, mf = _symmetrize(gram, perms, flips)
        assert np.abs(Cd - Cf).max() <= 1e-14, name
        assert np.abs(md - mf).max() <= 1e-14, name
        nat.check(nat.lib().dmv_debug_zz_symmetrize(C.byref(bd), gram.ctypes.data, Cd.ctypes.data, None))
    gram[0, 0] = 0.0
    with pytest.raises(nat.DmvError, match="zero vector"):
        nat.check(nat.lib().dmv_debug_zz_symmetrize(C.byref(bd), gram.ctypes.data, Cd.ctypes.data, None))


# ---------------------------------------------------------------------------------------------------------------- GPU
def _torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def need_cuda():
    if not _torch().cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


# the queued row kernel k_pull ("mode" 1) for the eigenvectors of bases with complex characters or a non-trivial sector
OPTIONS = {"issue_01": {"mode": 1}, "momentum_sector": {"mode": 1}, "ring10_w3_k1": {"mode": 1},
           "ring10_w3_k3": {"mode": 1}}


@pytest.mark.gpu
@pytest.mark.parametrize("name", FORMULA + ["heisenberg_chain_12", "complex_hopping"])
def test_small_models_against_full_space(need_cuda, name):
    """C and m equal the full-space values to 1e-12: float64 and complex128 vectors, random vectors and eigsh
    eigenvectors, one vector and a [3, n] batch, numpy arrays and torch tensors."""
    torch = _torch()
    from oracle import dense_pin as dp
    from distributed_matvec_b200 import Operator
    basis, matrix = _load(name)
    reps, _, B = dp.symmetry_adapted_basis(basis)
    op = Operator(matrix)
    for key, value in OPTIONS.get(name, {}).items():
        op.set_option(key, value)
    op.basis.build()
    assert np.array_equal(op.basis.representatives(), reps)
    n, N = reps.shape[0], basis.number_sites
    rng = np.random.default_rng(3)
    X = {np.float64: rng.normal(size=(3, n)),
         np.complex128: rng.normal(size=(3, n)) + 1j * rng.normal(size=(3, n))}
    cplx_ops = op.info("complex_coefficients") != 0
    X["eigsh"] = op.eigsh(3, complex_vectors=True if cplx_ops else False, tol=1e-10)[1]
    for key, xs in X.items():
        ref = [_full_space(basis, B, xs[v]) for v in range(3)]
        Cb, mb = op.zz_correlations(xs)
        assert Cb.shape == (3, N, N) and mb.shape == (3, N)
        Ct, mt = op.zz_correlations(torch.from_numpy(xs).cuda())
        torch.cuda.synchronize()
        for v in range(3):
            C1, m1 = op.zz_correlations(np.ascontiguousarray(xs[v]))
            assert C1.shape == (N, N) and m1.shape == (N,)
            for Cx, mx in ((C1, m1), (Cb[v], mb[v]), (Ct[v], mt[v])):
                assert np.abs(Cx - ref[v][0]).max() <= 1e-12, (name, key, v)
                assert np.abs(mx - ref[v][1]).max() <= 1e-12, (name, key, v)
    op.close()


def _yaml_terms(name):
    with open(os.path.join(DATA, name + ".yaml"), encoding="utf-8") as f:
        return yaml.safe_load(f)["hamiltonian"]["terms"]


def _zz_bonds(name):
    return [tuple(b) for t in _yaml_terms(name) if t["expression"].startswith("σᶻ") for b in t["sites"]]


@pytest.mark.gpu
def test_square_6x6_ground_state(need_cuda):
    """6 x 6 square, ground state from eigsh: C_ii = 1, every row sums to 0 (the Sᶻ = 0 sector), m = 0, and the 72
    nearest-neighbour entries equal E0 / 216 = -0.452581433 (SU(2): <σᵢ·σⱼ> = 3 <σᶻᵢσᶻⱼ>, 72 bonds) within 1e-7."""
    torch = _torch()
    from distributed_matvec_b200 import Operator, load_config_from_yaml
    _, matrix = load_config_from_yaml(os.path.join(DATA, "heisenberg_square_6x6.yaml"))
    op = Operator(matrix)
    op.basis.build()
    n = op.basis.numberStates()
    vec = torch.empty((1, n), dtype=torch.float64, device="cuda")
    vals, _, res, conv, _, _ = op.eigsh(1, tol=1e-11, eigenvectors=vec)
    assert conv == 1 and abs(vals[0] - (-97.757589597)) <= 1e-6, (vals, res)
    Cz, m = op.zz_correlations(vec[0])
    assert np.abs(np.diag(Cz) - 1.0).max() <= 1e-10
    assert np.abs(Cz.sum(axis=1)).max() <= 1e-10
    assert np.abs(m).max() <= 1e-10
    bonds = _zz_bonds("heisenberg_square_6x6")
    assert len(bonds) == 72
    nn = np.array([Cz[i, j] for i, j in bonds])
    assert nn.max() - nn.min() <= 1e-9, nn
    assert abs(nn.mean() - (-97.757589597) / 216) <= 1e-7, nn.mean()
    assert abs(nn.mean() - vals[0] / 216) <= 1e-9
    op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n_sites", [32, 36])
def test_chain_bethe(need_cuda, n_sites):
    """chain_32_symm / chain_36_symm ground states: C_{i,i+1} = 4 E_Bethe(N) / (3N) to 1e-7 relative."""
    import bethe
    torch = _torch()
    from distributed_matvec_b200 import Operator, load_config_from_yaml
    name = f"heisenberg_chain_{n_sites}_symm"
    _, matrix = load_config_from_yaml(os.path.join(DATA, name + ".yaml"))
    op = Operator(matrix)
    op.basis.build()
    vec = torch.empty((1, op.basis.numberStates()), dtype=torch.float64, device="cuda")
    vals, _, _, conv, _, _ = op.eigsh(1, tol=1e-11, eigenvectors=vec)
    assert conv == 1
    Cz, m = op.zz_correlations(vec[0])
    want = 4.0 * bethe.heisenberg_ring_e0(n_sites) / (3 * n_sites)
    nn = np.array([Cz[i, (i + 1) % n_sites] for i in range(n_sites)])
    assert np.abs(nn - want).max() <= 1e-7 * abs(want), (nn, want)
    assert np.abs(np.diag(Cz) - 1.0).max() <= 1e-10 and np.abs(m).max() <= 1e-10
    op.close()


def _diag_energy(matrix, Cz, m):
    """sum over the diagonal terms v (-1)^popcount(a & s) (products of at most two σᶻ, each -(-1)^bit) of v times the
    expectation value of the term"""
    d = matrix.diag
    total = 0.0
    for v, mask, s in zip(d.v, d.m, d.s):
        assert int(mask) == 0
        sites = [i for i in range(64) if int(s) >> i & 1]
        assert len(sites) <= 2
        value = (1.0, -m[sites[0]] if sites else 0.0, Cz[sites[0], sites[-1]])[len(sites)]
        total += v.real * value
    return total


def _without_symmetries(name):
    """the same Hamiltonian on the basis of the same Hamming weight without symmetries (dmv_apply_diag evaluates the
    diagonal of bases that need no projection)"""
    from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
    basis, matrix = _load(name)
    if not basis.requires_projection():
        return matrix
    plain = basis_from_dict({"number_spins": basis.number_sites, "hamming_weight": basis.hamming_weight})
    return operator_from_dict({"terms": _yaml_terms(name)}, plain)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["heisenberg_chain_24", "heisenberg_chain_12", "heisenberg_kagome_12_symm",
                                  "complex_hopping"])
def test_diagonal_energy_through_apply_diag(need_cuda, name):
    """For any vector: sum over the diagonal terms of coefficient x C_ij (or m_i) equals sum_b |x_b|^2 D(r_b) / W with D
    from dmv_apply_diag on the device, an independent path through the library's diagonal code (chain_24 runs on the
    k_gather basis without symmetries; the diagonal of kagome_12_symm comes from the same terms without symmetries)."""
    from distributed_matvec_b200 import Operator
    _, matrix = _load(name)
    op = Operator(matrix)
    op.basis.build()
    reps = op.basis.representatives()
    plain = Operator(_without_symmetries(name))
    plain.basis.build()
    D = np.zeros(reps.shape[0])
    nat.check(nat.lib().dmv_apply_diag(plain._ctx, reps.shape[0], reps.ctypes.data, D.ctypes.data))
    rng = np.random.default_rng(5)
    for x in (rng.normal(size=reps.shape[0]), rng.normal(size=reps.shape[0]) + 1j * rng.normal(size=reps.shape[0])):
        Cz, m = op.zz_correlations(x)
        w = np.abs(x) ** 2
        want = float(w @ D / w.sum())
        assert abs(_diag_energy(matrix, Cz, m) - want) <= 1e-12 * max(1.0, np.abs(D).max()), name
    plain.close()
    op.close()


@pytest.mark.gpu
def test_repeated_call_is_bit_identical(need_cuda):
    torch = _torch()
    from distributed_matvec_b200 import Operator
    _, matrix = _load("heisenberg_chain_24")
    op = Operator(matrix)
    op.basis.build()
    x = torch.rand((2, op.basis.numberStates()), dtype=torch.complex128, device="cuda")
    a, b = op.zz_correlations(x), op.zz_correlations(x)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    op.close()


@pytest.mark.gpu
def test_errors(need_cuda):
    from distributed_matvec_b200 import Operator
    _, matrix = _load("heisenberg_chain_10")
    op = Operator(matrix)
    with pytest.raises(nat.DmvError, match="basis is not built"):
        nat.check(nat.lib().dmv_zz_correlations(op._ctx, nat.DMV_F64, 1, None, None, None))
    op.basis.build()
    n, N = op.basis.numberStates(), 10
    x = np.ones(n)
    out = np.zeros(N * N)
    lib = nat.lib()
    for elt in (0, 3):
        with pytest.raises(nat.DmvError, match="elt"):
            nat.check(lib.dmv_zz_correlations(op._ctx, elt, 1, x.ctypes.data, out.ctypes.data, None))
    for k in (0, -1):
        with pytest.raises(nat.DmvError, match="num_vectors"):
            nat.check(lib.dmv_zz_correlations(op._ctx, nat.DMV_F64, k, x.ctypes.data, out.ctypes.data, None))
    with pytest.raises(nat.DmvError, match="x must not be null"):
        nat.check(lib.dmv_zz_correlations(op._ctx, nat.DMV_F64, 1, None, out.ctypes.data, None))
    with pytest.raises(nat.DmvError, match="correlations must not be null"):
        nat.check(lib.dmv_zz_correlations(op._ctx, nat.DMV_F64, 1, x.ctypes.data, None, None))
    with pytest.raises(nat.DmvError, match="zero vector"):
        op.zz_correlations(np.zeros(n))
    with pytest.raises(nat.DmvError, match="zero vector"):
        op.zz_correlations(np.stack([np.ones(n), np.zeros(n)]))
    with pytest.raises(ValueError):
        op.zz_correlations(np.ones(n + 1))
    op.close()
    op = Operator(matrix, rank=0, num_ranks=2)   # two ranks without a communicator
    op.basis.build()
    with pytest.raises(nat.DmvError, match="dmv_comm_init"):
        op.zz_correlations(np.ones(op.basis.numberStates()))
    op.close()


@pytest.mark.gpu
def test_collective_zz_two_ranks(need_cuda):
    """Two ranks: chain_10, square_4x4, momentum_sector and chain_24 against one rank (tools/zz_check.py)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29557", os.path.join(ROOT, "tools", "zz_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    lines = [l for l in out.stdout.splitlines() if l.rstrip().endswith(("OK", "FAIL"))]
    assert out.returncode == 0 and len(lines) >= 4 and not any(l.rstrip().endswith("FAIL") for l in lines), \
        out.stdout[-4000:] + out.stderr[-2000:]
