"""Flip-flop correlations on the device (dmv_pm_correlations / Operator.pm_correlations / Operator.spin_correlations).

References that share nothing with the library: the state psi = B x on the full 2^n space, with the symmetry-adapted
basis B built explicitly by oracle/dense_pin.py, where <σ⁺ᵢσ⁻ⱼ> = psi[s ^ (i|j)]* psi[s] summed over the states s with
bit j set and bit i clear; the total spin S² as an operator of its own, applied by the product; the Bethe ansatz
(tests/bethe.py); the pinned ground-state energy of the 6 x 6 square.  The class-sum formula and the host half are
checked without a GPU.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from distributed_matvec_b200 import _native as nat
from oracle.dense_pin import _apply_element

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "data")
E_6X6 = -97.757589597


def _ring(n, weight, sector):
    """Heisenberg ring of n sites at a fixed Hamming weight in a momentum sector"""
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
    """(perms [G, N], flips [G], characters [G]): the basis group, {1, flip} for spin inversion alone, {1} without"""
    n = basis.number_sites
    if basis.has_permutation_symmetries():
        g = basis.group
        return np.asarray(g.perms), np.asarray(g.flips), np.asarray(g.characters)
    if basis.spin_inversion:
        return (np.stack([np.arange(n)] * 2), np.array([0, 1], dtype=np.uint8),
                np.array([1.0, float(basis.spin_inversion)], dtype=np.complex128))
    return np.arange(n)[None, :], np.zeros(1, dtype=np.uint8), np.ones(1, dtype=np.complex128)


def _full_space(B, x, n):
    """T[i, j] = <psi|σ⁺ᵢσ⁻ⱼ|psi> / <psi|psi> of psi = B x on the full 2^n space"""
    psi = B @ x
    W = np.vdot(psi, psi).real
    s = np.arange(psi.shape[0], dtype=np.uint64)
    bit = [((s >> np.uint64(i)) & np.uint64(1)).astype(bool) for i in range(n)]
    T = np.zeros((n, n), dtype=np.complex128)
    for i in range(n):
        T[i, i] = np.sum(np.abs(psi[bit[i]]) ** 2) / W
        for j in range(n):
            if i != j:
                src = s[bit[j] & ~bit[i]]
                dst = src ^ np.uint64((1 << i) | (1 << j))
                T[i, j] = np.vdot(psi[dst.astype(np.int64)], psi[src.astype(np.int64)]) / W
    return T


def _classes(n, perms, flips):
    """class of every ordered pair (row-major numbering of first pairs) and the class sizes"""
    of = -np.ones((n, n), dtype=np.int32)
    sizes = []
    for i in range(n):
        for j in range(n):
            if i == j or of[i, j] >= 0:
                continue
            c = len(sizes)
            for p, f in zip(perms, flips):
                k, l = (p[j], p[i]) if f else (p[i], p[j])
                of[k, l] = c
            sizes.append(int(np.sum(of == c)))
    return of, np.array(sizes)


def _formula(basis, reps, norms, x):
    """The class-sum formula on the representatives: K_ij = sum over rows b with bit i set and bit j clear of
    conj(x_b) / n_b chi (n x)[rep(r_b ^ (1 << i | 1 << j))], T_ij = S_c / (W |c|), T_ii = <n_i>."""
    n = basis.number_sites
    perms, flips, chars = _group(basis)
    where = {int(r): k for k, r in enumerate(reps)}
    of, sizes = _classes(n, perms, flips)
    S = np.zeros(len(sizes), dtype=np.complex128)
    for b, r in enumerate(reps):
        r = int(r)
        up = [i for i in range(n) if r >> i & 1]
        dn = [j for j in range(n) if not r >> j & 1]
        for i in up:
            for j in dn:
                a = np.array([r ^ (1 << i) ^ (1 << j)], dtype=np.uint64)
                images = np.array([_apply_element(perms[e], flips[e], n, a)[0] for e in range(len(perms))])
                e = int(np.argmin(images))
                k = where.get(int(images[e]))
                if k is not None:   # a target orbit outside the basis has a vanishing projection
                    S[of[i, j]] += np.conj(x[b]) / norms[b] * chars[e] * norms[k] * x[k]
    W = np.sum(np.abs(x) ** 2)
    T = np.where(of >= 0, S[np.maximum(of, 0)] / (W * sizes[np.maximum(of, 0)]), 0)
    occ = np.array([[int(r) >> i & 1 for i in range(n)] for r in reps], dtype=float)
    nbar = (np.abs(x) ** 2) @ occ / W   # <n_i> is the same average over the group as in test_zz_correlations
    m = np.zeros(n)
    for p, f in zip(perms, flips):
        m += (1 - nbar[p]) if f else nbar[p]
    T[np.arange(n), np.arange(n)] = m / len(perms)
    return T


FORMULA = ["heisenberg_chain_10", "heisenberg_square_4x4", "heisenberg_kagome_12_symm", "issue_01", "momentum_sector",
           "ring10_w3_k0", "ring10_w3_k1", "ring10_w3_k3", "complex_hopping"]


@pytest.mark.parametrize("name", FORMULA)
def test_formula_against_full_space(name):
    """The class-sum formula equals <psi|σ⁺ᵢσ⁻ⱼ|psi> / <psi|psi> on psi = B x for random complex x, to 1e-12: this pins
    the rows (bit i set, bit j clear), the character (chi, not conjugated), the class map of a flip (i, j) -> (p(j),
    p(i)) and the vanishing projections of the odd-inversion and momentum sectors independently of the library."""
    from oracle import dense_pin as dp
    basis, _ = _load(name)
    reps, norms, B = dp.symmetry_adapted_basis(basis)
    rng = np.random.default_rng(7)
    x = rng.normal(size=reps.shape[0]) + 1j * rng.normal(size=reps.shape[0])
    T_ref = _full_space(B, x, basis.number_sites)
    T = _formula(basis, reps, norms, x)
    assert np.abs(T - T_ref).max() <= 1e-12, name
    assert np.abs(T_ref - T_ref.conj().T).max() <= 1e-12


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


@pytest.mark.parametrize("name", FORMULA + ["heisenberg_chain_12", "heisenberg_square_6x6"])
def test_host_classes_match_numpy(name):
    """dmv_debug_pm_classes: class ids and sizes equal numpy's, and the finish from random class sums to 1e-14."""
    basis, _ = _load(name)
    n = basis.number_sites
    bd, keep = _basis_desc(basis)
    perms, flips, _ = _group(basis)
    of, sizes = _classes(n, perms, flips)
    of_d, sizes_d, count = np.zeros((n, n), dtype=np.int32), np.zeros(n * n, dtype=np.int32), C.c_int32()
    lib = nat.lib()
    nat.check(lib.dmv_debug_pm_classes(C.byref(bd), of_d.ctypes.data, sizes_d.ctypes.data, C.byref(count), None, 0.0,
                                       None, None))
    assert count.value == len(sizes) and np.array_equal(of_d, of) and np.array_equal(sizes_d[:len(sizes)], sizes)
    if name == "heisenberg_square_6x6":
        assert len(sizes) == 9   # the 6 x 6 torus: nine classes for 1260 ordered pairs
    rng = np.random.default_rng(11)
    sums = rng.normal(size=2 * len(sizes))
    m = rng.normal(size=n)
    W = 1.0 + rng.random()
    pm = np.zeros((n, n), dtype=np.complex128)
    nat.check(lib.dmv_debug_pm_classes(C.byref(bd), of_d.ctypes.data, sizes_d.ctypes.data, C.byref(count),
                                       sums.ctypes.data, W, m.ctypes.data, pm.ctypes.data))
    S = sums[0::2] + 1j * sums[1::2]
    want = np.where(of >= 0, S[np.maximum(of, 0)] / (W * sizes[np.maximum(of, 0)]), 0)
    want[np.arange(n), np.arange(n)] = 0.5 * (1.0 + m)
    assert np.abs(pm - want).max() <= 1e-14
    with pytest.raises(nat.DmvError, match="zero vector"):
        nat.check(lib.dmv_debug_pm_classes(C.byref(bd), of_d.ctypes.data, sizes_d.ctypes.data, C.byref(count),
                                           sums.ctypes.data, 0.0, m.ctypes.data, pm.ctypes.data))


# ---------------------------------------------------------------------------------------------------------------- GPU
def _torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def need_cuda():
    if not _torch().cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


# model, options, the walk it takes: k_pm_rows through k_rows' table (torus row form on the 4x4 square, ordered or
# hashed layout, generic walk with canon 0), through the index (rows 0, complex characters), k_pm_pairs on the
# identity / Lin / combinadic-rank / directory indices
CASES = [("heisenberg_square_4x4", {}), ("heisenberg_square_4x4", {"rows_table": 0}),
         ("heisenberg_square_4x4", {"canon": 0}), ("heisenberg_square_4x4", {"rows": 0}),
         ("heisenberg_kagome_12_symm", {}), ("heisenberg_kagome_16", {}), ("issue_01", {"mode": 1}),
         ("momentum_sector", {"mode": 1}), ("ring10_w3_k0", {}), ("ring10_w3_k1", {"mode": 1}),
         ("ring10_w3_k3", {"mode": 1}), ("heisenberg_chain_10", {}), ("heisenberg_chain_10", {"index": 2}),
         ("heisenberg_chain_10", {"index": 0}), ("heisenberg_chain_12", {}), ("complex_hopping", {}),
         ("complex_hopping", {"index": 3})]


@pytest.mark.gpu
@pytest.mark.parametrize("name,options", CASES, ids=[f"{n}-{'-'.join(f'{k}{v}' for k, v in o.items())}"
                                                     for n, o in CASES])
def test_small_models_against_full_space(need_cuda, name, options):
    """T equals the full-space value to 1e-12: float64 and complex128 vectors, random vectors and eigsh eigenvectors,
    one vector and a [3, n] batch, numpy arrays and torch tensors."""
    torch = _torch()
    from oracle import dense_pin as dp
    from distributed_matvec_b200 import Operator
    basis, matrix = _load(name)
    reps, _, B = dp.symmetry_adapted_basis(basis)
    op = Operator(matrix)
    for key, value in options.items():
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
        ref = [_full_space(B, xs[v], N) for v in range(3)]
        Tb = op.pm_correlations(xs)
        assert Tb.shape == (3, N, N) and Tb.dtype == np.complex128
        Tt = op.pm_correlations(torch.from_numpy(xs).cuda())
        torch.cuda.synchronize()
        for v in range(3):
            T1 = op.pm_correlations(np.ascontiguousarray(xs[v]))
            assert T1.shape == (N, N)
            for Tx in (T1, Tb[v], Tt[v]):
                assert np.abs(Tx - ref[v]).max() <= 1e-12, (name, options, key, v)
    op.close()


def _s2_operator(basis_spec, N):
    """S² - 3N/4 = 1/2 sum_{i<j} σᵢ·σⱼ as an operator on the same basis"""
    from distributed_matvec_b200 import Operator
    from distributed_matvec_b200.config import operator_from_dict
    pairs = [[i, j] for i in range(N) for j in range(i + 1, N)]
    specs = [{"expression": f"0.5 × σ{c}₀ σ{c}₁", "sites": pairs} for c in "ˣʸᶻ"]
    return Operator(operator_from_dict({"terms": specs}, basis_spec))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["heisenberg_square_4x4", "heisenberg_kagome_12_symm", "heisenberg_chain_12"])
def test_total_spin_against_operator(need_cuda, name):
    """<S²> from spin_correlations equals <x|S² x> / <x|x> with S² applied by the product, to 1e-10."""
    from distributed_matvec_b200 import Operator
    basis, matrix = _load(name)
    op = Operator(matrix)
    op.basis.build()
    N = basis.number_sites
    s2 = _s2_operator(basis, N)
    s2.basis.build()
    n = op.basis.numberStates()
    rng = np.random.default_rng(13)
    for x in (rng.normal(size=n), rng.normal(size=n) + 1j * rng.normal(size=n)):
        y = s2.matvec(np.ascontiguousarray(x))
        want = (np.vdot(x, y) / np.vdot(x, x)).real + 0.75 * N
        S, S2 = op.spin_correlations(x)
        assert abs(S2 - want) <= 1e-10 * max(1.0, abs(want)), (name, S2, want)
        assert np.abs(S - S.T).max() <= 1e-12
    s2.close()
    op.close()


@pytest.mark.gpu
def test_chain_12_multiplets(need_cuda):
    """chain_12 (no fixed Hamming weight, no symmetry): eigsh(4, block_size=3) gives the singlet ground state and the
    three vectors of the lowest triplet; <S²> = S (S + 1) = 0, 2, 2, 2 within 1e-8, whatever basis of the triplet."""
    from distributed_matvec_b200 import Operator
    _, matrix = _load("heisenberg_chain_12")
    op = Operator(matrix)
    op.basis.build()
    vals, vecs = op.eigsh(4, block_size=3, tol=1e-11)[:2]
    _, S2 = op.spin_correlations(vecs)
    assert np.abs(S2 - np.array([0.0, 2.0, 2.0, 2.0])).max() <= 1e-8, (vals, S2)
    op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["heisenberg_kagome_12_symm", "heisenberg_chain_10", "heisenberg_square_4x4"])
def test_identities(need_cuda, name):
    """Singlet ground state: Re T_ij = C_ij / 2 for i != j (SU(2)); T_ii = (1 + m_i) / 2 for any vector."""
    from distributed_matvec_b200 import Operator
    _, matrix = _load(name)
    op = Operator(matrix)
    op.basis.build()
    vecs = op.eigsh(1, tol=1e-11)[1]
    Cz, _ = op.zz_correlations(vecs[0])
    T = op.pm_correlations(vecs[0])
    off = ~np.eye(Cz.shape[0], dtype=bool)
    assert np.abs(T.real[off] - 0.5 * Cz[off]).max() <= 1e-9
    x = np.random.default_rng(17).normal(size=op.basis.numberStates())
    _, m = op.zz_correlations(x)
    assert np.abs(np.diag(op.pm_correlations(x)) - 0.5 * (1.0 + m)).max() <= 1e-13
    op.close()


def _bonds(name):
    import yaml
    with open(os.path.join(DATA, name + ".yaml"), encoding="utf-8") as f:
        terms = yaml.safe_load(f)["hamiltonian"]["terms"]
    return [tuple(b) for t in terms if t["expression"].startswith("σᶻ") for b in t["sites"]]


@pytest.mark.gpu
def test_square_6x6_ground_state(need_cuda):
    """6 x 6 square ground state from eigsh(1, tol=1e-11): the 72 bonds of C + 4 Re T sum to the pinned energy within
    1e-6, <S²> <= 1e-6, and the 72 Re T_nn agree to 1e-9 with mean E0 / 432 within 1e-7."""
    torch = _torch()
    from distributed_matvec_b200 import Operator, load_config_from_yaml
    _, matrix = load_config_from_yaml(os.path.join(DATA, "heisenberg_square_6x6.yaml"))
    op = Operator(matrix)
    op.basis.build()
    n = op.basis.numberStates()
    vec = torch.empty((1, n), dtype=torch.float64, device="cuda")
    vals, _, res, conv, _, _ = op.eigsh(1, tol=1e-11, eigenvectors=vec)
    assert conv == 1 and abs(vals[0] - E_6X6) <= 1e-6, (vals, res)
    S, S2 = op.spin_correlations(vec[0])
    T = op.pm_correlations(vec[0])
    bonds = _bonds("heisenberg_square_6x6")
    assert len(bonds) == 72
    assert abs(sum(S[i, j] for i, j in bonds) - E_6X6) <= 1e-6
    assert abs(S2) <= 1e-6
    nn = np.array([T[i, j].real for i, j in bonds])
    assert nn.max() - nn.min() <= 1e-9, nn
    assert abs(nn.mean() - E_6X6 / 432) <= 1e-7, nn.mean()
    op.close()


@pytest.mark.gpu
def test_chain_32_bethe(need_cuda):
    """chain_32_symm ground state: <σᵢ·σᵢ₊₁> = 4 E_Bethe(N) / N to 1e-7 relative for every i."""
    import bethe
    torch = _torch()
    from distributed_matvec_b200 import Operator, load_config_from_yaml
    _, matrix = load_config_from_yaml(os.path.join(DATA, "heisenberg_chain_32_symm.yaml"))
    op = Operator(matrix)
    op.basis.build()
    vec = torch.empty((1, op.basis.numberStates()), dtype=torch.float64, device="cuda")
    conv = op.eigsh(1, tol=1e-11, eigenvectors=vec)[3]
    assert conv == 1
    S, _ = op.spin_correlations(vec[0])
    want = 4.0 * bethe.heisenberg_ring_e0(32) / 32
    nn = np.array([S[i, (i + 1) % 32] for i in range(32)])
    assert np.abs(nn - want).max() <= 1e-7 * abs(want), (nn, want)
    op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["heisenberg_chain_24", "heisenberg_square_4x4", "momentum_sector"])
def test_repeated_call_is_bit_identical(need_cuda, name):
    torch = _torch()
    from distributed_matvec_b200 import Operator
    _, matrix = _load(name)
    op = Operator(matrix)
    op.basis.build()
    x = torch.rand((2, op.basis.numberStates()), dtype=torch.complex128, device="cuda")
    assert np.array_equal(op.pm_correlations(x), op.pm_correlations(x))
    op.close()


@pytest.mark.gpu
def test_errors(need_cuda):
    from distributed_matvec_b200 import Operator
    _, matrix = _load("heisenberg_chain_10")
    op = Operator(matrix)
    lib = nat.lib()
    with pytest.raises(nat.DmvError, match="basis is not built"):
        nat.check(lib.dmv_pm_correlations(op._ctx, nat.DMV_F64, 1, None, None))
    op.basis.build()
    n, N = op.basis.numberStates(), 10
    x = np.ones(n)
    out = np.zeros(2 * N * N)
    for elt in (0, 3):
        with pytest.raises(nat.DmvError, match="elt"):
            nat.check(lib.dmv_pm_correlations(op._ctx, elt, 1, x.ctypes.data, out.ctypes.data))
    for k in (0, -1):
        with pytest.raises(nat.DmvError, match="num_vectors"):
            nat.check(lib.dmv_pm_correlations(op._ctx, nat.DMV_F64, k, x.ctypes.data, out.ctypes.data))
    with pytest.raises(nat.DmvError, match="x must not be null"):
        nat.check(lib.dmv_pm_correlations(op._ctx, nat.DMV_F64, 1, None, out.ctypes.data))
    with pytest.raises(nat.DmvError, match="pm must not be null"):
        nat.check(lib.dmv_pm_correlations(op._ctx, nat.DMV_F64, 1, x.ctypes.data, None))
    with pytest.raises(nat.DmvError, match="zero vector"):
        op.pm_correlations(np.zeros(n))
    with pytest.raises(nat.DmvError, match="zero vector"):
        op.pm_correlations(np.stack([np.ones(n), np.zeros(n)]))
    with pytest.raises(ValueError):
        op.pm_correlations(np.ones(n + 1))
    with pytest.raises(ValueError):
        op.pm_correlations(np.ones((2, 2, n)))
    with pytest.raises(TypeError):
        op.pm_correlations(np.ones(n, dtype=np.float32))
    op.close()
    op = Operator(matrix, rank=0, num_ranks=2)   # two ranks without a communicator
    op.basis.build()
    with pytest.raises(nat.DmvError, match="dmv_comm_init"):
        op.pm_correlations(np.ones(op.basis.numberStates()))
    op.close()


@pytest.mark.gpu
def test_collective_pm_two_ranks(need_cuda):
    """Two ranks: chain_10, square_4x4, momentum_sector and chain_24 against one rank (tools/pm_check.py)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--standalone",
           os.path.join(ROOT, "tools", "pm_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    lines = [l for l in out.stdout.splitlines() if l.rstrip().endswith(("OK", "FAIL"))]
    assert out.returncode == 0 and len(lines) >= 8 and not any(l.rstrip().endswith("FAIL") for l in lines), \
        out.stdout[-4000:] + out.stderr[-2000:]
