"""Bipartite entanglement on the device (dmv_reduced_density_matrix / Operator.reduced_density_matrix,
Operator.entanglement_entropy) and the numpy helpers of distributed_matvec_b200.entanglement.

References that share nothing with the library: ρ_A from ψ = B x on the full space, with the symmetry-adapted basis B
built explicitly by oracle/dense_pin.py and the partial trace taken in numpy; the free-fermion spectrum of the XX ring
(tests/free_fermions.py, Peschel 2003), checked here against exact diagonalisation before any GPU test relies on it; the
library's own zz / pm correlations, an independent path to the one- and two-site ρ.
"""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import yaml

import free_fermions
from distributed_matvec_b200 import _native as nat
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
from distributed_matvec_b200.entanglement import (block_layout, entanglement_spectrum, renyi_entropy,
                                                  von_neumann_entropy)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "data")


# ------------------------------------------------------------------------------------------------------------ models
def _ring_bonds(n):
    return [[i, (i + 1) % n] for i in range(n)]


def _heisenberg(bonds):
    return [{"expression": f"σ{c}₀ σ{c}₁", "sites": bonds} for c in "ˣʸᶻ"]


def _xx(bonds):
    return [{"expression": f"σ{c}₀ σ{c}₁", "sites": bonds} for c in "ˣʸ"]


def _tfim(n, h=0.7):
    return [{"expression": "σᶻ₀ σᶻ₁", "sites": _ring_bonds(n)}, {"expression": f"-{h} × σˣ₀", "sites": [[i] for i in range(n)]}]


def _ring(n, weight, k=None, r=None, inv=None, terms=None):
    """ring of n sites: translation in sector k, reflection j -> n - j in sector r, spin inversion inv (None: absent)"""
    sym = []
    if k is not None:
        sym.append({"permutation": [(i + 1) % n for i in range(n)], "sector": k})
    if r is not None:
        sym.append({"permutation": [(n - i) % n for i in range(n)], "sector": r})
    d = {"number_spins": n, "hamming_weight": weight, "symmetries": sym}
    if inv:
        d["spin_inversion"] = inv
    basis = basis_from_dict(d)
    return basis, operator_from_dict({"terms": terms or _heisenberg(_ring_bonds(n))}, basis)


def _from_yaml(name):
    with open(os.path.join(DATA, name + ".yaml"), encoding="utf-8") as f:
        d = yaml.safe_load(f)
    basis = basis_from_dict(d["basis"])
    return basis, operator_from_dict({"terms": d["hamiltonian"]["terms"]}, basis)


MODELS = {
    "ring12_k0r0_inv": lambda: _ring(12, 6, 0, 0, 1),        # trivial characters with spin inversion
    "ring12_k0r0": lambda: _ring(12, 6, 0, 0),
    "ring10_k1": lambda: _ring(10, 5, 1),                    # a complex momentum character
    "ring10_k5r1": lambda: _ring(10, 5, 5, 1),               # real non-trivial characters
    "ring10_inv_only": lambda: _ring(10, 5, inv=-1),         # spin inversion without permutations
    "ring10_plain": lambda: _ring(10, 5),
    "ring11_w4_k0": lambda: _ring(11, 4, 0),                 # odd ring, weight off half filling
    "tfim10_free_k0r0_inv": lambda: _ring(10, None, 0, 0, 1, terms=_tfim(10)),   # free weight
    "tfim8_free_plain": lambda: _ring(8, None, terms=_tfim(8)),
    "kagome12_symm": lambda: _from_yaml("heisenberg_kagome_12_symm"),
    "torus4": lambda: _from_yaml("heisenberg_square_4x4"),
}


def _site_lists(n):
    """contiguous, scattered, permuted site lists of a model of n sites"""
    return {"one": [0], "pair": [0, 1], "half": list(range(n // 2)), "scattered": [1, 4, n - 2],
            "permuted": [n - 1, 2, 0, n // 2 + 1, 3]}


# ------------------------------------------------------------------------------------------ the numpy reference
def full_state(basis, x):
    """ψ = B x on the full 2^n space (dense), with B of oracle/dense_pin.py"""
    from oracle.dense_pin import symmetry_adapted_basis
    _, _, B = symmetry_adapted_basis(basis)
    return np.asarray(B @ np.asarray(x, dtype=np.complex128)).ravel()


def reference_rdm(psi, n, sites, weight):
    """{w: ρ_w} of the normalised ψ (full space), in the layout of dmv_reduced_density_matrix"""
    sites = [int(s) for s in sites]
    rest = [s for s in range(n) if s not in sites]
    states = np.arange(1 << n, dtype=np.int64)
    a = np.zeros_like(states)
    for k, s in enumerate(sites):
        a |= ((states >> s) & 1) << k
    b = np.zeros_like(states)
    for j, s in enumerate(rest):
        b |= ((states >> s) & 1) << j
    norm2 = np.vdot(psi, psi).real
    pop_a = np.array([bin(int(v)).count("1") for v in range(1 << len(sites))])
    out = {}
    for w, d in block_layout(n, weight, len(sites)):
        rows = np.arange(1 << len(sites)) if w is None else np.nonzero(pop_a == w)[0]
        row_of = np.full(1 << len(sites), -1)
        row_of[rows] = np.arange(rows.shape[0])
        keep = row_of[a] >= 0
        cols, col_of = np.unique(b[keep], return_inverse=True)
        M = np.zeros((d, cols.shape[0]), dtype=np.complex128)
        M[row_of[a[keep]], col_of] = psi[keep]
        out[w] = M @ M.conj().T / norm2
    return out


def _entropy(blocks):
    return von_neumann_entropy(entanglement_spectrum(blocks))


def _random_x(basis, rng, real=False):
    from oracle.dense_pin import symmetry_adapted_basis
    n = symmetry_adapted_basis(basis)[0].shape[0]
    return rng.normal(size=n) + (0 if real else 1j * rng.normal(size=n))


# ------------------------------------------------------------------------------------------- layout and refusals
def _layout(n, weight, n_a, sites=None):
    nb, wf, dims = C.c_int(-7), C.c_int(-7), np.zeros(17, dtype=np.int32)
    sp = None if sites is None else np.ascontiguousarray(np.asarray(sites, dtype=np.int32))
    nat.check(nat.lib().dmv_rdm_layout(n, -1 if weight is None else weight, n_a,
                                       None if sp is None else sp.ctypes.data, C.byref(nb), C.byref(wf),
                                       dims.ctypes.data))
    return wf.value, [int(d) for d in dims[:nb.value]]


@pytest.mark.parametrize("n,weight", [(12, 6), (12, None), (20, 3), (16, 16), (16, 0), (36, 18), (9, None), (64, 32)])
def test_layout_matches_block_layout(n, weight):
    """dmv_rdm_layout equals entanglement.block_layout for n_a = 1 ... 16, A = all sites included"""
    for n_a in range(1, min(16, n) + 1):
        want = block_layout(n, weight, n_a)
        wf, dims = _layout(n, weight, n_a)
        assert dims == [d for _, d in want], (n, weight, n_a)
        assert wf == (-1 if weight is None else want[0][0])
        if weight is not None:
            assert sum(d * math.comb(n - n_a, weight - w) for w, d in want) == math.comb(n, weight)
        else:
            assert want == [(None, 1 << n_a)]


def test_layout_refusals():
    """every refusal of the host half, with its message; block_layout refuses the same arguments"""
    cases = [((12, 6, 0), "n_a must be between 1 and 16"), ((40, 20, 17), "n_a must be between 1 and 16"),
             ((8, 4, 9), "exceeds the 8 sites"), ((0, -1, 1), "number_sites"), ((65, -1, 1), "number_sites"),
             ((12, 13, 2), "hamming_weight"), ((12, -2, 2), "hamming_weight")]
    for args, msg in cases:
        with pytest.raises(nat.DmvError, match=msg):
            _layout(*args)
        with pytest.raises(ValueError):
            block_layout(args[0], None if args[1] == -1 else args[1], args[2])
    for sites, msg in [([0, 3, 3], "site 3 appears twice"), ([0, 12], "site 12 of sites_a is outside"),
                       ([-1, 2], "site -1 of sites_a is outside")]:
        with pytest.raises(nat.DmvError, match=msg):
            _layout(12, 6, len(sites), sites)
    assert _layout(12, 6, 3, [11, 0, 5]) == (0, [1, 3, 3, 1])
    with pytest.raises(nat.DmvError, match="num_blocks"):
        nat.check(nat.lib().dmv_rdm_layout(12, 6, 2, None, None, None, None))


# ----------------------------------------------------------------------------- the numpy reference on the dense pin
CPU_MODELS = ["ring12_k0r0_inv", "ring10_k1", "ring10_k5r1", "ring10_inv_only", "ring11_w4_k0", "tfim10_free_k0r0_inv",
              "kagome12_symm", "torus4"]


@pytest.mark.parametrize("model", CPU_MODELS)
def test_reference_is_a_density_matrix(model):
    """ρ_A of the reference: Hermitian, positive semi-definite, trace 1; S(A) = S(B) for the complement; the one-site ρ
    is diag(P(σᶻ = -1), P(σᶻ = +1)) read off |ψ|² directly"""
    basis, _ = MODELS[model]()
    n = basis.number_sites
    rng = np.random.default_rng(7)
    psi = full_state(basis, _random_x(basis, rng))
    p = np.abs(psi) ** 2 / np.vdot(psi, psi).real
    for name, sites in _site_lists(n).items():
        rho = reference_rdm(psi, n, sites, basis.hamming_weight)
        assert abs(sum(np.trace(r).real for r in rho.values()) - 1.0) <= 1e-12
        for r in rho.values():
            assert np.abs(r - r.conj().T).max() <= 1e-14
            assert np.linalg.eigvalsh(r).min() >= -1e-13
        rest = [s for s in range(n) if s not in sites]
        assert abs(_entropy(rho) - _entropy(reference_rdm(psi, n, rest, basis.hamming_weight))) <= 1e-10, name
    up = p[(np.arange(1 << n) >> 3) & 1 == 1].sum()
    rho = reference_rdm(psi, n, [3], basis.hamming_weight)
    diag = np.concatenate([np.diag(r).real for r in rho.values()])
    assert np.abs(diag - [1.0 - up, up]).max() <= 1e-12 and all(np.abs(r).max() <= 1.0 for r in rho.values())


def test_reference_block_order_on_a_product_state():
    """a product state |s> (one basis state of the plain ring): ρ_A is |a><a| with a the local configuration of A,
    bit k = site sites[k], in the block of its weight at the row of its rank"""
    n, s = 8, 0b10110010
    psi = np.zeros(1 << n, dtype=complex)
    psi[s] = 1.0
    sites = [7, 1, 4]   # bits of s: 1, 1, 1 -> a = 0b111
    rho = reference_rdm(psi, n, sites, 4)
    assert set(rho) == {0, 1, 2, 3} and rho[3].shape == (1, 1) and rho[3][0, 0] == 1.0
    sites = [0, 7, 5, 2]   # bits 0, 1, 1, 0 -> a = 0b0110, weight 2, rows 0b0011, 0b0101, 0b0110 ...: row 2
    rho = reference_rdm(psi, n, sites, 4)
    assert rho[2][2, 2] == 1.0 and sum(np.abs(r).sum() for r in rho.values()) == 1.0


# ------------------------------------------------------------------------------------ free fermions (Peschel 2003)
def _xx_ground_state(n):
    import scipy.sparse.linalg as sla
    from oracle.sector_pin import sector_hamiltonian, sector_states
    states = sector_states(n, n // 2)
    H = sector_hamiltonian(_xx(_ring_bonds(n)), n, states)
    vals, vecs = (np.linalg.eigh(H.toarray()) if H.shape[0] <= 1000 else sla.eigsh(H, k=2, which="SA", tol=1e-15))
    order = np.argsort(vals)
    assert vals[order[1]] - vals[order[0]] > 1e-6   # a unique ground state
    psi = np.zeros(1 << n, dtype=complex)
    psi[states.astype(np.int64)] = vecs[:, order[0]]
    return psi


@pytest.mark.parametrize("n", [8, 10, 12, 14, 16])
def test_free_fermions_equal_exact_diagonalisation(n):
    """the block-resolved entanglement spectrum of sites 0 ... ℓ - 1 of the XX ring's ground state is the free-fermion
    one, and the entropy its closed form, for ℓ = 2, 3 and N / 2"""
    psi = _xx_ground_state(n)
    for ell in sorted({2, 3, n // 2}):
        rho = reference_rdm(psi, n, list(range(ell)), n // 2)
        got = entanglement_spectrum(rho)
        want = free_fermions.block_spectrum(n, ell)
        assert set(got) == set(want)
        for w in want:
            assert np.abs(np.sort(got[w]) - want[w]).max() <= 1e-10, (n, ell, w)
        assert abs(von_neumann_entropy(got) - free_fermions.entropy(n, ell)) <= 1e-10


# ------------------------------------------------------------------------------------------------ entropy helpers
def test_renyi_closed_forms_and_the_von_neumann_limit():
    uniform = np.full(8, 1 / 8)
    for alpha in (0, 0.5, 1, 2, 3, np.inf):
        assert abs(renyi_entropy(uniform, alpha) - np.log(8)) <= 1e-14
    p = np.array([0.7, 0.2, 0.1, 0.0])
    assert abs(renyi_entropy(p, 2) + np.log((p ** 2).sum())) <= 1e-15
    assert abs(renyi_entropy(p, 0.5) - 2 * np.log(np.sqrt(p).sum())) <= 1e-15
    assert abs(renyi_entropy(p, np.inf) + np.log(0.7)) <= 1e-15
    assert abs(renyi_entropy(p, 0) - np.log(3)) <= 1e-15
    vn = -(p[:3] * np.log(p[:3])).sum()
    assert abs(von_neumann_entropy(p) - vn) <= 1e-15 and renyi_entropy(p, 1) == von_neumann_entropy(p)
    for eps in (1e-4, -1e-4):
        assert abs(renyi_entropy(p, 1 + eps) - vn) <= 2e-4
    blocks = {0: np.diag([0.1, 0.2]), 1: np.array([[0.35, 0.05], [0.05, 0.35]])}
    spec = entanglement_spectrum(blocks)
    assert np.allclose(spec[1], [0.3, 0.4]) and abs(von_neumann_entropy(spec) - renyi_entropy([0.1, 0.2, 0.3, 0.4], 1)) \
        <= 1e-15
    assert entanglement_spectrum({None: np.diag([1.0, -1e-17])})[None].min() == 0.0
    with pytest.raises(ValueError):
        renyi_entropy(p, -1)


# ------------------------------------------------------------------------------------------------------------ GPU
def _torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def need_cuda():
    if not _torch().cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _op(model, options=None):
    from distributed_matvec_b200 import Operator
    op = Operator(model[1])
    for key, value in (options or {}).items():
        op.set_option(key, value)
    op.basis.build()
    return op


# every look-up: the dense ordered table, the ordered layout, hashed homes, the index with trivial and complex
# characters, spin inversion alone, none; the square-torus orbit minimum (and the generic walk on the torus)
COVER = [(m, {}) for m in MODELS] + [("ring12_k0r0_inv", {"rows_dense_order": 0}), ("ring12_k0r0_inv", {"rows_table": 0}),
                                     ("ring12_k0r0_inv", {"rows": 0}), ("torus4", {"rows": 0}), ("torus4", {"canon": 0}),
                                     ("torus4", {"rows_dense_order": 0})]


@pytest.mark.gpu
@pytest.mark.parametrize("model,options", COVER, ids=[f"{m}-{'-'.join(f'{k}{v}' for k, v in o.items())}" for m, o in COVER])
def test_against_numpy_reference(need_cuda, model, options):
    """float64 (real characters) and complex128, numpy and a torch batch of two, n_a = 1, 2, N / 2, scattered,
    permuted and all N sites (rank 1; up to 12 sites): every block equals the reference to 1e-12"""
    torch = _torch()
    basis, _ = MODELS[model]()
    op = _op(MODELS[model](), options)
    n, N = op.basis.numberStates(), basis.number_sites
    from oracle.dense_pin import symmetry_adapted_basis
    assert np.array_equal(op.basis.representatives(), symmetry_adapted_basis(basis)[0])
    rng = np.random.default_rng(13)
    lists = dict(_site_lists(N), **({"all": list(range(N))[::-1]} if N <= 12 else {}))
    for dtype in ([np.float64] if not op.info("complex_coefficients") else []) + [np.complex128]:
        X = rng.normal(size=(2, n)) + (1j * rng.normal(size=(2, n)) if dtype == np.complex128 else 0)
        psis = [full_state(basis, X[v]) for v in range(2)]
        for name, sites in lists.items():
            refs = [reference_rdm(psis[v], N, sites, basis.hamming_weight) for v in range(2)]
            one = op.reduced_density_matrix(np.ascontiguousarray(X[0]), sites)
            batch = op.reduced_density_matrix(torch.from_numpy(X).cuda(), sites)
            for v, got in ((0, one), (0, batch[0]), (1, batch[1])):
                assert list(got) == list(refs[v]), (model, name)
                for w in got:
                    err = np.abs(got[w] - refs[v][w]).max()
                    assert err <= 1e-12, (model, options, dtype, name, w, err)
                    if dtype == np.float64:
                        assert np.all(got[w].imag == 0.0)
            if name == "all":
                evals = np.concatenate(list(entanglement_spectrum(one).values()))
                assert abs(evals.max() - 1.0) <= 1e-12 and np.sort(evals)[-2] <= 1e-12
            assert op.info("rdm_amplitudes") > 0 and op.info("rdm_gram_flops") > 0
    op.close()


def _square_ground_state():
    torch = _torch()
    op = _op(_from_yaml("heisenberg_square_6x6"))
    vec = torch.empty((1, op.basis.numberStates()), dtype=torch.float64, device="cuda")
    vals, _, _, conv, _, _ = op.eigsh(1, tol=1e-11, eigenvectors=vec)
    assert conv == 1 and abs(vals[0] - (-97.757589597)) <= 1e-6
    return op, vec[0]


@pytest.mark.gpu
def test_square_6x6_against_correlations(need_cuda):
    """6 x 6 ground state: the one-site ρ is diag((1 - m) / 2, (1 + m) / 2); the two-site ρ of the nearest and the
    farthest pair is the matrix of C_ij, m_i, m_j and T_ij, to 1e-10; a 12-site strip is Hermitian, PSD and of trace 1"""
    op, psi = _square_ground_state()
    Cz, m = op.zz_correlations(psi)
    T = op.pm_correlations(psi)
    rho = op.reduced_density_matrix(psi, [7])
    assert abs(rho[0][0, 0] - (1 - m[7]) / 2) <= 1e-10 and abs(rho[1][0, 0] - (1 + m[7]) / 2) <= 1e-10
    for i, j in ((0, 1), (0, 21), (14, 8)):
        rho = op.reduced_density_matrix(psi, [i, j])
        c, mi, mj = Cz[i, j], m[i], m[j]
        want = {0: np.array([[(1 - mi - mj + c) / 4]]), 2: np.array([[(1 + mi + mj + c) / 4]]),
                1: np.array([[(1 + mi - mj - c) / 4, T[j, i]], [T[i, j], (1 - mi + mj - c) / 4]])}
        for w in want:
            assert np.abs(rho[w] - want[w]).max() <= 1e-10, (i, j, w, rho[w], want[w])
        assert abs(sum(np.trace(r).real for r in rho.values()) - 1.0) <= 1e-12
    strip = op.reduced_density_matrix(psi, list(range(12)))
    assert abs(sum(np.trace(r).real for r in strip.values()) - 1.0) <= 1e-10
    for r in strip.values():
        assert np.abs(r - r.conj().T).max() == 0.0 and np.linalg.eigvalsh(r).min() >= -1e-12
    op.close()


def xx_ring(n, k, r, inv):
    return _ring(n, n // 2, k, r, inv, terms=_xx(_ring_bonds(n)))


def xx_sector(n):
    """(k, r, inversion) of the sector of translations, reflection and spin inversion that holds the XX ring's ground
    state, by the dense pin over the candidate sectors k in {0, N / 2}"""
    from oracle.dense_pin import projected_hamiltonian
    best, where = None, None
    for k in (0, n // 2):
        for r in (0, 1):
            for inv in (1, -1):
                model = xx_ring(n, k, r, inv)
                _, _, Hp = projected_hamiltonian(_xx(_ring_bonds(n)), model[0])
                if Hp.shape[0] == 0:
                    continue
                e = np.linalg.eigvalsh(Hp)[0]
                if best is None or e < best - 1e-9:
                    best, where = e, (k, r, inv)
    return where


def test_xx_sector_is_the_same_on_small_rings():
    """the sector of the XX ground state is the same on rings of 8, 12 and 16 sites (N = 0 mod 4, as N = 32)"""
    assert xx_sector(8) == xx_sector(12) == xx_sector(16)


@pytest.mark.gpu
def test_xx_ring_32_against_free_fermions(need_cuda):
    """the XX ring of 32 sites in its ground state's sector (eigsh): the block-resolved spectrum of sites 0 ... ℓ - 1 is
    the free-fermion one to 1e-9 for ℓ = 4, 8, 12"""
    torch = _torch()
    k, r, inv = xx_sector(8)
    op = _op(xx_ring(32, 0 if k == 0 else 16, r, inv))
    vec = torch.empty((1, op.basis.numberStates()), dtype=torch.float64, device="cuda")
    vals, _, _, conv, _, _ = op.eigsh(1, tol=1e-12, eigenvectors=vec)
    assert conv == 1
    e_ff = 4.0 * np.cos(free_fermions.occupied_momenta(32)).sum()
    assert abs(vals[0] + abs(e_ff)) <= 1e-9 * abs(e_ff), (vals[0], e_ff)
    for ell in (4, 8, 12):
        got = entanglement_spectrum(op.reduced_density_matrix(vec[0], list(range(ell))))
        want = free_fermions.block_spectrum(32, ell)
        for w in want:
            assert np.abs(np.sort(got[w]) - want[w]).max() <= 1e-9, (ell, w)
        assert abs(op.entanglement_entropy(vec[0], list(range(ell))) - free_fermions.entropy(32, ell)) <= 1e-9
    op.close()


@pytest.mark.gpu
def test_chain_24_entropy_of_a_half_equals_its_complement(need_cuda):
    torch = _torch()
    op = _op(_from_yaml("heisenberg_chain_24_symm"))
    vec = torch.empty((1, op.basis.numberStates()), dtype=torch.float64, device="cuda")
    assert op.eigsh(1, tol=1e-12, eigenvectors=vec)[3] == 1
    rho_a = op.reduced_density_matrix(vec[0], list(range(12)))
    rho_b = op.reduced_density_matrix(vec[0], list(range(12, 24)))
    s_a, s_b = _entropy(rho_a), _entropy(rho_b)
    assert s_a > 0.5 and abs(s_a - s_b) <= 1e-10, (s_a, s_b)
    for alpha in (0.5, 2, np.inf):
        assert abs(renyi_entropy(entanglement_spectrum(rho_a), alpha) -
                   renyi_entropy(entanglement_spectrum(rho_b), alpha)) <= 1e-10
    # the complement is taken when A is the larger part
    assert abs(op.entanglement_entropy(vec[0], list(range(15))) - _entropy(
        op.reduced_density_matrix(vec[0], list(range(15, 24))))) == 0.0
    op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["ring12_k0r0_inv", "ring10_k1", "torus4", "tfim10_free_k0r0_inv"])
def test_repeated_call_is_bit_identical(need_cuda, model):
    """twice in a row, and again after products and an option set and reset on the same context"""
    torch = _torch()
    op = _op(MODELS[model]())
    x = torch.rand((2, op.basis.numberStates()), dtype=torch.complex128, device="cuda")
    sites = [3, 0, 5, 1]
    a = op.reduced_density_matrix(x, sites)
    b = op.reduced_density_matrix(x, sites)
    for _ in range(3):
        op.matvec(x[0].clone())
    op.set_option("rows_table", 0)
    op.matvec(x[1].clone())
    op.set_option("rows_table", 1)
    c = op.reduced_density_matrix(x, sites)
    for v in range(2):
        for w in a[v]:
            assert np.array_equal(a[v][w], b[v][w]) and np.array_equal(a[v][w], c[v][w]), (model, v, w)
    op.close()


@pytest.mark.gpu
def test_errors_write_nothing(need_cuda):
    """every refusal through the device entry leaves rho as it was; a ρ too large for the device names its bytes"""
    lib = nat.lib()
    op = _op(MODELS["ring12_k0r0_inv"]())
    cplx = _op(MODELS["ring10_k1"]())
    n = op.basis.numberStates()
    x = np.ones(n)
    rho = np.full(2 * 1000, 7.0)

    def call(o=op, elt=nat.DMV_F64, k=1, xp=x.ctypes.data, sites=(0, 1), rp=rho.ctypes.data):
        s = np.ascontiguousarray(np.asarray(sites, dtype=np.int32))
        nat.check(lib.dmv_reduced_density_matrix(o._ctx, elt, k, xp, len(sites), s.ctypes.data if len(sites) else None,
                                                 rp))

    zero = np.zeros(n)
    for kw, msg in [({"sites": ()}, "n_a must be between 1 and 16"), ({"sites": tuple(range(12)) + (0,) * 5},
                                                                       "n_a must be between 1 and 16"),
                    ({"sites": (0, 4, 4)}, "appears twice"), ({"sites": (0, 12)}, "outside"),
                    ({"sites": (-3,)}, "outside"), ({"xp": zero.ctypes.data}, "zero vector"),
                    ({"xp": None}, "x must not be null"), ({"rp": None}, "rho must not be null"),
                    ({"k": 0}, "num_vectors"), ({"elt": 3}, "elt"),
                    ({"o": cplx, "xp": np.ones(cplx.basis.numberStates()).ctypes.data}, "use complex vectors")]:
        with pytest.raises(nat.DmvError, match=msg):
            call(**kw)
    assert np.all(rho == 7.0)
    big = _op(_ring(18, None, terms=_tfim(18)))
    xb = np.ones(big.basis.numberStates())
    with pytest.raises(nat.DmvError, match=r"needs \d+ bytes, but only \d+ bytes are free"):
        call(o=big, xp=xb.ctypes.data, sites=tuple(range(16)))
    assert np.all(rho == 7.0)
    with pytest.raises(ValueError):
        op.reduced_density_matrix(np.ones(n + 1), [0])
    for o in (op, cplx, big):
        o.close()


@pytest.mark.gpu
def test_two_ranks_against_one(need_cuda):
    """Two ranks on one device against one rank (tools/entanglement_check.py)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29563", os.path.join(ROOT, "tools", "entanglement_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    lines = [l for l in out.stdout.splitlines() if l.rstrip().endswith(("OK", "FAIL"))]
    assert out.returncode == 0 and len(lines) >= 4 and not any(l.rstrip().endswith("FAIL") for l in lines), \
        out.stdout[-4000:] + out.stderr[-2000:]
