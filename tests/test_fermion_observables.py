"""Single-particle observables of fermionic bases: the one-body density matrix <c†ᵢcⱼ> (Operator.one_body_density_matrix)
and c, c† between particle sectors (Operator.apply_fermion), with the spectral function A(k, ω) built on them
(spectral.spectral_function).

Without a GPU: bit-level numpy references of both entries against the dense Jordan-Wigner matrices of
tests/fermion_pin.py, the canonical anticommutators through the sector matrices, and the sum rules of A(k, ω) on exact
diagonalisation of small Hubbard and free rings.
On the GPU: both entries against the references on spinless and spinful models, the zero cross-spin block, free
fermions and Hubbard sum rules at size, particle-hole symmetry on the 4 x 4 torus, determinism, every refusal, and two
ranks against one (tools/fermion_observables_check.py).
"""
from __future__ import annotations

import math
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import fermion_pin as fp  # noqa: E402
import torch  # noqa: E402
from distributed_matvec_b200 import Operator  # noqa: E402
from distributed_matvec_b200 import _native as nat  # noqa: E402
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict  # noqa: E402
from distributed_matvec_b200.spectral import fourier_weights, spectral_function  # noqa: E402
from gen_models import _bonds_ring, _bonds_torus, hubbard, spinless_ring  # noqa: E402

ONE = np.uint64(1)


# ---------------------------------------------------------------------------------------------------------------------
# numpy references, bit by bit in uint64 (the row formulas of include/dmv_b200.h)

def _parity(v) -> np.ndarray:
    return (np.bitwise_count(np.asarray(v, dtype=np.uint64)) & 1).astype(bool)


def _find(states, t):
    """indices of t in the ascending states, and whether each is there"""
    r = np.minimum(np.searchsorted(states, t), max(states.shape[0] - 1, 0))
    return r, states[r] == t


def ref_obdm(states, x, n_modes: int) -> np.ndarray:
    """G[i, j] = <x|c†ᵢcⱼ|x> / <x|x> over the ascending basis states; pairs whose target leaves the basis give 0."""
    states = np.asarray(states, dtype=np.uint64)
    x = np.asarray(x, dtype=np.complex128)
    W = float(np.vdot(x, x).real)
    G = np.zeros((n_modes, n_modes), dtype=np.complex128)
    for i in range(n_modes):
        bi = ONE << np.uint64(i)
        G[i, i] = np.sum(np.abs(x[(states & bi) != 0]) ** 2) / W
        for j in range(n_modes):
            if i == j:
                continue
            bj = ONE << np.uint64(j)
            lo, hi = min(i, j), max(i, j)
            between = ((ONE << np.uint64(hi)) - ONE) & ~((ONE << np.uint64(lo + 1)) - ONE)
            rows = np.nonzero(((states & bi) != 0) & ((states & bj) == 0))[0]
            r, ok = _find(states, states[rows] ^ bi ^ bj)
            b = rows[ok]
            sign = np.where(_parity(states[b] & between), -1.0, 1.0)
            G[i, j] = np.sum(np.conj(x[b]) * x[r[ok]] * sign) / W
    return G


def ref_apply(kind: str, w, src, tgt, x) -> np.ndarray:
    """y = Σ_k w_k c†_k x (kind "c+") or Σ_k w_k c_k x (kind "c") from the ascending src states into the tgt states."""
    src, tgt = np.asarray(src, dtype=np.uint64), np.asarray(tgt, dtype=np.uint64)
    x = np.asarray(x, dtype=np.complex128)
    y = np.zeros(tgt.shape[0], dtype=np.complex128)
    for k, wk in enumerate(np.asarray(w, dtype=np.complex128)):
        if wk == 0:
            continue
        bit = ONE << np.uint64(k)
        rows = np.nonzero(((tgt & bit) != 0) if kind == "c+" else ((tgt & bit) == 0))[0]
        r, ok = _find(src, tgt[rows] ^ bit)
        assert ok.all(), "a source state is outside the source basis"
        sign = np.where(_parity(tgt[rows] & (bit - ONE)), -1.0, 1.0)
        y[rows] += wk * sign * x[r]
    return y


def _op_text(kind: str, mode: int, n_sites: int, spinful: bool, placeholder: int) -> str:
    arrow = ("↑" if mode < n_sites else "↓") if spinful else ""
    return f"{'c†' if kind == 'c+' else 'c'}{'₀₁'[placeholder]}{arrow}"


def _site(mode: int, n_sites: int, spinful: bool) -> int:
    return mode % n_sites if spinful else mode


def pin_hop(i: int, j: int, n_sites: int, spinful: bool, states) -> sp.csr_matrix:
    """c†ᵢcⱼ on the states from fermion_pin.apply_to_states"""
    text = _op_text("c+", i, n_sites, spinful, 0) + " " + _op_text("c", j, n_sites, spinful, 1)
    return fp.apply_to_states([{"expression": text, "sites": [[_site(i, n_sites, spinful), _site(j, n_sites, spinful)]]}],
                              n_sites, spinful, states)


def pin_one(kind: str, k: int, n_sites: int, spinful: bool, src, tgt) -> sp.csr_matrix:
    """c†_k or c_k from the src states into the tgt states, from fermion_pin.apply_to_states"""
    text = _op_text(kind, k, n_sites, spinful, 0)
    return fp.apply_to_states([{"expression": text, "sites": [[_site(k, n_sites, spinful)]]}], n_sites, spinful, src,
                              targets=tgt)


def _dense_block(ops, n_modes, rows, cols) -> np.ndarray:
    return fp.monomial(n_modes, ops)[np.asarray(rows, dtype=np.int64)][:, np.asarray(cols, dtype=np.int64)].toarray()


def _rand(n, cplx, seed):
    rng = np.random.default_rng(seed)
    x = rng.normal(size=n)
    return x + 1j * rng.normal(size=n) if cplx else x


# ---------------------------------------------------------------------------------------------------------------------
# CPU: references against the dense Jordan-Wigner matrices

CPU_SECTORS = [("spinless 7 modes, 3 particles", 7, False, 3, None),
               ("spinless 6 modes, free", 6, False, None, None),
               ("spinful 4 sites, 2 up 1 down", 4, True, 2, 1),
               ("spinful 3 sites, 1 up 2 down", 3, True, 1, 2)]


def _states(n_sites, spinful, a, b):
    if spinful:
        return fp.sector_states(n_sites, a, b)
    if a is None:
        return np.arange(1 << n_sites, dtype=np.uint64)
    return fp.sector_states(n_sites, a, spinful=False)


@pytest.mark.parametrize("case", CPU_SECTORS, ids=[c[0] for c in CPU_SECTORS])
def test_reference_density_matrix_against_the_dense_pin(case):
    _, n, spinful, a, b = case
    M = 2 * n if spinful else n
    states = _states(n, spinful, a, b)
    for cplx in (False, True):
        x = _rand(states.shape[0], cplx, 7)
        G = ref_obdm(states, x, M)
        W = np.vdot(x, x).real
        for i in range(M):
            for j in range(M):
                cross = spinful and (i < n) != (j < n)
                if cross:
                    assert G[i, j] == 0   # number_up is fixed: the cross-spin block vanishes
                    continue
                pin = pin_hop(i, j, n, spinful, states)
                dense = _dense_block([("c+", i), ("c", j)], M, states, states)
                assert np.abs(pin.toarray() - dense).max() == 0, (i, j)
                assert abs(np.vdot(x, pin @ x) / W - G[i, j]) < 1e-13, (i, j)
        assert np.abs(G - G.conj().T).max() < 1e-14


@pytest.mark.parametrize("case", CPU_SECTORS, ids=[c[0] for c in CPU_SECTORS])
def test_reference_sector_operators_against_the_dense_pin(case):
    _, n, spinful, a, b = case
    M = 2 * n if spinful else n
    src = _states(n, spinful, a, b)
    rng = np.random.default_rng(3)
    x = _rand(src.shape[0], True, 9)
    for kind, d in (("c+", 1), ("c", -1)):
        halves = [(range(n), (a + d, b)), (range(n, 2 * n), (a, b + d))] if spinful else \
                 [(range(n), (None if a is None else a + d, None))]
        for modes, (ta, tb) in halves:
            if (ta is not None and not 0 <= ta <= n) or (tb is not None and not 0 <= tb <= n):
                continue
            tgt = _states(n, spinful, ta, tb)
            w = np.zeros(M, dtype=np.complex128)
            w[list(modes)] = rng.normal(size=len(modes)) + 1j * rng.normal(size=len(modes))
            y = ref_apply(kind, w, src, tgt, x)
            dense = sum(w[k] * _dense_block([(kind, k)], M, tgt, src) for k in modes)
            pin = sum(w[k] * pin_one(kind, k, n, spinful, src, tgt) for k in modes)
            assert np.abs(dense @ x - y).max() < 1e-13
            assert np.abs(pin @ x - y).max() < 1e-13


def _sector_matrix(kind, k, M, src, tgt):
    """the matrix of c†_k / c_k from the src into the tgt states, column by column through ref_apply"""
    w = np.zeros(M)
    w[k] = 1.0
    return np.stack([ref_apply(kind, w, src, tgt, e) for e in np.eye(src.shape[0])], axis=1)


@pytest.mark.parametrize("n,spinful,a,b", [(6, False, 3, None), (3, True, 1, 1)])
def test_anticommutators_through_the_sector_matrices(n, spinful, a, b):
    """{c_i, c†_j} = δ_ij on a sector, with c†c through the sector of one particle fewer and c c† through one more"""
    M = 2 * n if spinful else n
    mid = _states(n, spinful, a, b)
    for i in range(M):
        for j in range(M):
            same = not spinful or (i < n) == (j < n)
            if not same:
                continue
            up = i < n if spinful else True
            more = _states(n, spinful, a + 1 if up else a, (b + 1 if not up else b) if spinful else None)
            less = _states(n, spinful, a - 1 if up else a, (b - 1 if not up else b) if spinful else None)
            acc = _sector_matrix("c", i, M, more, mid) @ _sector_matrix("c+", j, M, mid, more) + \
                _sector_matrix("c+", j, M, less, mid) @ _sector_matrix("c", i, M, mid, less)
            assert np.abs(acc - (i == j) * np.eye(mid.shape[0])).max() < 1e-14, (i, j)


def _ground_state(conf, states):
    H = fp.sector_hamiltonian(conf["hamiltonian"]["terms"], conf["basis"]["number_sites"],
                              conf["basis"]["particle"] == "spinful-fermion", states).toarray()
    e, v = np.linalg.eigh(H)
    return e[0], v[:, 0], e[1] - e[0]


def _moments(conf, states, w, kind_states):
    """zeroth and first moments of the particle and hole parts of A(ω) for O = Σ w_j c_j, from dense sector matrices"""
    spinful = conf["basis"]["particle"] == "spinful-fermion"
    n = conf["basis"]["number_sites"]
    e0, psi, _ = _ground_state(conf, states)
    out = {}
    for part, tgt in kind_states.items():
        Ht = fp.sector_hamiltonian(conf["hamiltonian"]["terms"], n, spinful, tgt).toarray()
        y = ref_apply("c+", np.conj(w), states, tgt, psi) if part == "particle" else ref_apply("c", w, states, tgt, psi)
        m0 = np.vdot(y, y).real
        m1 = np.vdot(y, Ht @ y).real - e0 * m0
        out[part] = (m0, m1 if part == "particle" else -m1)
    return e0, psi, out


@pytest.mark.parametrize("n,u", [(4, 4.0), (6, 3.0), (6, 0.0)])
def test_hubbard_ring_sum_rules_by_exact_diagonalisation(n, u):
    """A(k, ω) of a half-filled Hubbard ring: weight 1, first moment ε_k + U <n_-σ>, hole weight n(k)"""
    conf = hubbard(n, _bonds_ring(n), u=u)
    up = dn = n // 2
    states = fp.sector_states(n, up, dn)
    coords = np.arange(n)
    for spin in (0, 1):
        for m in range(n):
            kq = 2 * np.pi * m / n
            w = np.zeros(2 * n, dtype=np.complex128)
            w[spin * n:(spin + 1) * n] = fourier_weights(coords, kq)
            more = fp.sector_states(n, up + 1, dn) if spin == 0 else fp.sector_states(n, up, dn + 1)
            less = fp.sector_states(n, up - 1, dn) if spin == 0 else fp.sector_states(n, up, dn - 1)
            _, psi, mom = _moments(conf, states, w, {"particle": more, "hole": less})
            G = ref_obdm(states, psi, 2 * n)
            nk = np.vdot(w, G @ w).real
            eps = -2.0 * np.cos(kq)
            assert abs(mom["particle"][0] + mom["hole"][0] - 1.0) < 1e-12, (n, u, spin, m)
            assert abs(mom["hole"][0] - nk) < 1e-12, (n, u, spin, m)
            first = mom["particle"][1] + mom["hole"][1]
            assert abs(first - (eps + u * (dn if spin == 0 else up) / n)) < 1e-10, (n, u, spin, m, first)


def test_free_ring_spectral_weight_by_exact_diagonalisation():
    """Free spinless ring with a closed shell: n(k) is 0 or 1, and c_k / c†_k reach one eigenstate at ε_k"""
    n, nf = 9, 3
    conf = spinless_ring(n, nf)
    states = fp.sector_states(n, nf, spinful=False)
    e0, psi, gap = _ground_state(conf, states)
    assert gap > 0.1
    occupied = {0, 1, n - 1}
    G = ref_obdm(states, psi, n)
    for m in range(n):
        w = fourier_weights(np.arange(n), 2 * np.pi * m / n)
        nk = np.vdot(w, G @ w).real
        assert abs(nk - (m in occupied)) < 1e-12, (m, nk)
        _, _, mom = _moments(conf, states, w, {"particle": fp.sector_states(n, nf + 1, spinful=False),
                                               "hole": fp.sector_states(n, nf - 1, spinful=False)})
        part = "hole" if m in occupied else "particle"
        assert abs(mom[part][0] - 1.0) < 1e-12
        assert abs(mom[part][1] - (-2.0 * np.cos(2 * np.pi * m / n))) < 1e-12


# =====================================================================================================================
# GPU


@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _model(conf):
    basis = basis_from_dict(conf["basis"])
    return basis, operator_from_dict(conf["hamiltonian"], basis)


def _peierls_chain(n, phi):
    c, s = math.cos(phi), math.sin(phi)
    conf = hubbard(n, _bonds_ring(n), number_up=n // 2, number_down=n // 2)
    conf["hamiltonian"]["terms"][0]["expression"] = " ".join(
        f"- {c!r} × c†₀{a} c₁{a} - {s!r}j × c†₀{a} c₁{a} - {c!r} × c†₁{a} c₀{a} + {s!r}j × c†₁{a} c₀{a}" for a in "↑↓")
    return conf


def _anisotropic_torus_3x4(tx=1.0, ty=0.5, u=4.0):
    bonds = _bonds_torus(3, 4)
    conf = hubbard(12, bonds, u=u, number_up=3, number_down=3)
    hop = "-{t} × c†₀↑ c₁↑ - {t} × c†₁↑ c₀↑ - {t} × c†₀↓ c₁↓ - {t} × c†₁↓ c₀↓"
    conf["hamiltonian"]["terms"][0] = {"expression": hop.format(t=tx), "sites": bonds[0::2]}
    conf["hamiltonian"]["terms"].append({"expression": hop.format(t=ty), "sites": bonds[1::2]})
    return conf


def _with_particles(conf, up=None, down=None, total=None):
    """the same Hamiltonian in another particle sector"""
    c = {"basis": dict(conf["basis"]), "hamiltonian": conf["hamiltonian"]}
    if c["basis"]["particle"] == "spinful-fermion":
        u0 = c["basis"]["number_up"]
        d0 = c["basis"]["number_particles"] - u0
        u, d = (u0 if up is None else up), (d0 if down is None else down)
        c["basis"]["number_up"], c["basis"]["number_particles"] = u, u + d
    else:
        c["basis"]["number_particles"] = total
    return c


def _hubbard_chain_8():
    return hubbard(8, _bonds_ring(8))   # the model of data/hubbard_chain_8.yaml


GPU_MODELS = {
    "spinless_ring_12_n5": lambda: spinless_ring(12, 5),
    "spinless_ring_10_free": lambda: spinless_ring(10, None),
    "hubbard_chain_8": _hubbard_chain_8,
    "hubbard_torus_3x4_anisotropic": _anisotropic_torus_3x4,
    "peierls_chain_6": lambda: _peierls_chain(6, 0.3),
}


def _states_of(conf):
    b = conf["basis"]
    if b["particle"] == "spinful-fermion":
        return fp.sector_states(b["number_sites"], b["number_up"], b["number_particles"] - b["number_up"])
    if b.get("number_particles") is None:
        return np.arange(1 << b["number_sites"], dtype=np.uint64)
    return fp.sector_states(b["number_sites"], b["number_particles"], spinful=False)


def _built(conf):
    _, matrix = _model(conf)
    op = Operator(matrix)
    op.basis.build()
    assert np.array_equal(op.basis.representatives(), _states_of(conf))
    return op


def _close(a, b, tol=1e-12):
    return np.abs(np.asarray(a) - np.asarray(b)).max() <= tol * max(1.0, np.abs(np.asarray(b)).max())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GPU_MODELS))
def test_one_body_density_matrix_against_the_reference(need_cuda, name):
    """both element types, batches, index 0 and the default index, host and device vectors; bit-identical repeats"""
    conf = GPU_MODELS[name]()
    states = _states_of(conf)
    M = conf["basis"]["number_sites"] * (2 if conf["basis"]["particle"] == "spinful-fermion" else 1)
    op = _built(conf)
    try:
        for index in (-1, 0):
            op.set_option("index", index)
            for cplx in (False, True):
                X = np.stack([_rand(states.shape[0], cplx, 20 + j) for j in range(3)])
                want = np.stack([ref_obdm(states, x, M) for x in X])
                G = op.one_body_density_matrix(X)
                assert G.shape == (3, M, M)
                assert _close(G, want), (name, index, cplx, np.abs(G - want).max())
                g1 = op.one_body_density_matrix(torch.from_numpy(X[1].copy()).cuda())
                assert np.array_equal(g1, G[1]), (name, index, cplx)
                assert np.array_equal(op.one_body_density_matrix(X), G)   # deterministic
            if conf["basis"]["particle"] == "spinful-fermion":
                n = M // 2
                assert np.all(G[:, :n, n:] == 0) and np.all(G[:, n:, :n] == 0)   # the cross-spin block
        op.set_option("index", -1)
    finally:
        op.close()


def _sectors_for(conf, kind):
    """[(weights mask, target conf)] of the sectors c† / c reach: each spin half of a spinful basis, or the spinless one"""
    b = conf["basis"]
    d = 1 if kind == "c+" else -1
    if b["particle"] == "spinful-fermion":
        n, u = b["number_sites"], b["number_up"]
        dn = b["number_particles"] - u
        out = []
        if 0 <= u + d <= n:
            out.append((np.arange(2 * n) < n, _with_particles(conf, up=u + d)))
        if 0 <= dn + d <= n:
            out.append((np.arange(2 * n) >= n, _with_particles(conf, down=dn + d)))
        return out
    nf = b.get("number_particles")
    m = np.ones(b["number_sites"], dtype=bool)
    return [(m, _with_particles(conf, total=None if nf is None else nf + d))]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GPU_MODELS))
def test_apply_fermion_against_the_reference(need_cuda, name):
    """c† and c with random complex weights (and real ones in float64) into each reachable sector, up and down halves,
    index 0 and the default index, a batch of two, torch vectors; bit-identical repeats"""
    conf = GPU_MODELS[name]()
    src_states = _states_of(conf)
    op = _built(conf)
    rng = np.random.default_rng(5)
    try:
        for kind in ("c+", "c"):
            for mask, tconf in _sectors_for(conf, kind):
                tgt = _built(tconf)
                tgt_states = _states_of(tconf)
                try:
                    for index in (-1, 0):
                        op.set_option("index", index)
                        for cplx in (False, True):
                            w = np.where(mask, rng.normal(size=mask.size) + (1j * rng.normal(size=mask.size) if cplx
                                                                             else 0), 0)
                            X = np.stack([_rand(src_states.shape[0], cplx, 40 + j) for j in range(2)])
                            want = np.stack([ref_apply(kind, w, src_states, tgt_states, x) for x in X])
                            Y = op.apply_fermion(kind, w if cplx else w.real, X, tgt)
                            assert Y.dtype == X.dtype and Y.shape == want.shape
                            assert _close(Y, want), (name, kind, index, cplx, np.abs(Y - want).max())
                            assert np.array_equal(op.apply_fermion(kind, w, X, tgt), Y)
                            yt = op.apply_fermion("c†" if kind == "c+" else kind, w,
                                                  torch.from_numpy(X[0].copy()).cuda(), tgt)
                            torch.cuda.synchronize()
                            assert np.array_equal(yt.cpu().numpy(), Y[0])
                    op.set_option("index", -1)
                finally:
                    tgt.close()
    finally:
        op.close()


@pytest.mark.gpu
def test_spinful_cross_block_is_zero_and_walks_stay_in_the_basis(need_cuda):
    """hubbard_chain_8 with index 0 and the split index: the cross-spin block is exactly 0 and nothing is reported
    outside the basis, also after an apply_fermion on each half"""
    conf = _hubbard_chain_8()
    op = _built(conf)
    try:
        x = _rand(op.basis.numberStates(), True, 1)
        for index in (-1, 0):
            op.set_option("index", index)
            G = op.one_body_density_matrix(x)
            assert np.all(G[:8, 8:] == 0) and np.all(G[8:, :8] == 0)
            assert abs(np.trace(G).real - 8.0) < 1e-12 and abs(np.trace(G[:8, :8]).real - 4.0) < 1e-12
        op.set_option("index", -1)
    finally:
        op.close()


@pytest.mark.gpu
def test_free_fermions_at_size(need_cuda):
    """spinless_ring_28 with 13 particles (37.4 M states): n(k) is 1 on the 13 occupied momenta and 0 elsewhere, and
    A(k, ω) has one pole at ε_k = -2 cos k with residue 1, in the particle part for empty k and the hole part for
    occupied k"""
    n, nf = 28, 13
    op = _built_at_size(spinless_ring(n, nf))
    plus = minus = None
    try:
        assert op.basis.numberStates() == math.comb(n, nf)
        vec = torch.zeros((1, op.basis.numberStates()), dtype=torch.float64, device="cuda")
        evals, _, _, conv, _, _ = op.eigsh(1, tol=1e-12, eigenvectors=vec)
        torch.cuda.synchronize()
        exact = np.sort(-2 * np.cos(2 * np.pi * np.arange(n) / n))[:nf].sum()
        assert conv >= 1 and abs(evals[0] - exact) < 1e-10 * abs(exact)
        x0 = vec[0].to(torch.complex128)
        x0 /= torch.linalg.vector_norm(x0)
        G = op.one_body_density_matrix(x0)
        plus = _built_at_size(spinless_ring(n, nf + 1))
        minus = _built_at_size(spinless_ring(n, nf - 1))
        occupied = {m % n for m in range(-(nf // 2), nf // 2 + 1)}
        for m in range(n):
            kq = 2 * np.pi * m / n
            w = fourier_weights(np.arange(n), kq)
            nk = np.vdot(w, G @ w).real
            assert abs(nk - (m in occupied)) < 1e-10, (m, nk)
            (pp, pr), (hp, hr) = spectral_function(op, x0, evals[0], w, 4, plus, minus)
            poles, res, other = (hp, hr, pr) if m in occupied else (pp, pr, hr)
            top = int(np.argmax(res))
            assert abs(res[top] - 1.0) < 1e-10 and abs(poles[top] - (-2 * np.cos(kq))) < 1e-8, (m, poles, res)
            assert np.all(np.delete(res, top) < 1e-10) and np.all(other < 1e-10), (m, res, other)
    finally:
        for o in (op, plus, minus):
            if o is not None:
                o.close()


def _built_at_size(conf):
    _, matrix = _model(conf)
    op = Operator(matrix)
    op.basis.build()
    return op


def _hubbard_sum_rules(conf, coords, n_sites, u, steps, ground_state):
    """particle + hole weight = 1, hole weight = n(k), first moment = ε_k + U N_-σ / N for every k and both spins;
    -> n(k) per spin [2, n_k]"""
    b = conf["basis"]
    up, dn = b["number_up"], b["number_particles"] - b["number_up"]
    op = _built_at_size(conf)
    try:
        e0, x0 = ground_state(op)
        G = op.one_body_density_matrix(x0)
        ks = _momenta(coords)
        nks = np.zeros((2, len(ks)))
        for spin in (0, 1):
            plus = _built_at_size(_with_particles(conf, up=up + 1) if spin == 0 else _with_particles(conf, down=dn + 1))
            minus = _built_at_size(_with_particles(conf, up=up - 1) if spin == 0 else _with_particles(conf, down=dn - 1))
            try:
                for a, kq in enumerate(ks):
                    w = np.zeros(2 * n_sites, dtype=np.complex128)
                    w[spin * n_sites:(spin + 1) * n_sites] = fourier_weights(coords, kq)
                    nk = np.vdot(w, G @ w).real
                    nks[spin, a] = nk
                    (pp, pr), (hp, hr) = spectral_function(op, x0, e0, w, steps, plus, minus)
                    eps = -2.0 * np.cos(np.atleast_1d(kq)).sum()
                    first = pr @ pp + hr @ hp
                    where = (spin, kq, pr.sum(), hr.sum(), nk, first)
                    assert abs(pr.sum() + hr.sum() - 1.0) < 1e-10, where
                    assert abs(hr.sum() - nk) < 1e-10, where
                    assert abs(first - (eps + u * (dn if spin == 0 else up) / n_sites)) < 1e-8, where
            finally:
                plus.close()
                minus.close()
    finally:
        op.close()
    return nks


def _momenta(coords):
    c = np.asarray(coords)
    if c.ndim == 1:
        n = c.shape[0]
        return [2 * np.pi * m / n for m in range(n)]
    lx, ly = int(c[:, 0].max()) + 1, int(c[:, 1].max()) + 1
    return [np.array([2 * np.pi * a / lx, 2 * np.pi * b / ly]) for b in range(ly) for a in range(lx)]


def _lanczos_ground_state(op):
    e, vec, _, res = op.lanczos(max_iters=600, tol=1e-12)
    x0 = torch.from_numpy(vec).cuda().to(torch.complex128)
    x0 /= torch.linalg.vector_norm(x0)
    return e, x0


@pytest.mark.gpu
def test_hubbard_chain_8_sum_rules(need_cuda):
    _hubbard_sum_rules(_hubbard_chain_8(), np.arange(8), 8, 4.0, 6, _lanczos_ground_state)


@pytest.mark.gpu
def test_hubbard_square_4x4_sum_rules_and_particle_hole_symmetry(need_cuda):
    """165 636 900 states, steps = 2 (moments below 4 are exact); the half-filled ground state is unique (Lieb), so
    n(k) + n(Q - k) = 1 with Q = (π, π)"""
    coords = np.array([[i % 4, i // 4] for i in range(16)], dtype=np.float64)
    nks = _hubbard_sum_rules(hubbard(16, _bonds_torus(4, 4), u=4.0), coords, 16, 4.0, 2, _lanczos_ground_state)
    ks = _momenta(coords)
    for a, kq in enumerate(ks):
        q = np.mod(np.array([np.pi, np.pi]) - kq, 2 * np.pi)
        b = next(i for i, k2 in enumerate(ks) if np.allclose(np.mod(k2, 2 * np.pi), q))
        for spin in (0, 1):
            assert abs(nks[spin, a] + nks[spin, b] - 1.0) < 1e-9, (spin, kq, nks[spin, a], nks[spin, b])


@pytest.mark.gpu
def test_errors(need_cuda):
    """every refusal is raised and nothing is written to y"""
    lib = nat.lib()
    spin_basis = basis_from_dict({"number_spins": 6, "hamming_weight": 3})
    spin = Operator(operator_from_dict({"terms": [{"expression": "σᶻ₀ σᶻ₁", "sites": _bonds_ring(6)}]}, spin_basis))
    conf = hubbard(4, _bonds_ring(4), number_up=2, number_down=1)
    op = Operator(_model(conf)[1])
    try:
        with pytest.raises(nat.DmvError, match="basis is not built"):
            nat.check(lib.dmv_one_body_density_matrix(op._ctx, nat.DMV_F64, 1, None, None))
        spin.basis.build()
        op.basis.build()
        n = op.basis.numberStates()
        with pytest.raises(nat.DmvError, match="spin-1/2"):
            spin.one_body_density_matrix(np.ones(spin.basis.numberStates()))
        x = np.ones(n)
        out = np.zeros(2 * 64)
        for elt in (0, 3):
            with pytest.raises(nat.DmvError, match="elt"):
                nat.check(lib.dmv_one_body_density_matrix(op._ctx, elt, 1, x.ctypes.data, out.ctypes.data))
        for k in (0, -1):
            with pytest.raises(nat.DmvError, match="num_vectors"):
                nat.check(lib.dmv_one_body_density_matrix(op._ctx, nat.DMV_F64, k, x.ctypes.data, out.ctypes.data))
        with pytest.raises(nat.DmvError, match="x must not be null"):
            nat.check(lib.dmv_one_body_density_matrix(op._ctx, nat.DMV_F64, 1, None, out.ctypes.data))
        with pytest.raises(nat.DmvError, match="out must not be null"):
            nat.check(lib.dmv_one_body_density_matrix(op._ctx, nat.DMV_F64, 1, x.ctypes.data, None))
        with pytest.raises(nat.DmvError, match="zero vector"):
            op.one_body_density_matrix(np.stack([np.ones(n), np.zeros(n)]))
        with pytest.raises(ValueError):
            op.one_body_density_matrix(np.ones(n + 1))

        # apply_fermion: each refusal leaves y as it was
        targets = {}
        for key, c in {"up+": _with_particles(conf, up=3), "down+": _with_particles(conf, down=2),
                       "up-": _with_particles(conf, up=1), "same": conf}.items():
            targets[key] = Operator(_model(c)[1])
            targets[key].basis.build()
        w_up = np.r_[np.ones(4), np.zeros(4)].astype(np.complex128)
        w_dn = np.r_[np.zeros(4), np.ones(4)].astype(np.complex128)

        def refused(match, target, kind=0, w=w_up, elt=nat.DMV_C128, k=1, xv=None, source=op):
            xx = np.ones(n, dtype=np.complex128) if xv is None else xv
            y = np.full(target.basis.numberStates() * 2, 7.0)
            with pytest.raises(nat.DmvError, match=match):
                nat.check(lib.dmv_apply_fermion(target._ctx, source._ctx, elt, kind,
                                                None if w is None else w.ctypes.data, k, xx.ctypes.data,
                                                y.ctypes.data))
            assert np.all(y == 7.0), match

        refused("spin-1/2", targets["up+"], source=spin, xv=np.ones(spin.basis.numberStates(), dtype=np.complex128))
        refused("spin-1/2", spin, xv=np.ones(n, dtype=np.complex128))
        refused("kind must be", targets["up+"], kind=5)
        refused("weights must not be null", targets["up+"], w=None)
        refused("particle numbers", targets["same"])
        refused("particle numbers", targets["down+"], w=w_up)
        refused("particle numbers", targets["up+"], kind=1)
        refused(r"both spin halves.*\(number_up 3, number_down 1\) and \(number_up 2, number_down 2\)", targets["up+"],
                w=w_up + w_dn)
        refused("real weights", targets["up+"], w=w_up * 1j, elt=nat.DMV_F64, xv=np.ones(n))
        refused("num_vectors", targets["up+"], k=0)
        refused("elt", targets["up+"], elt=3)
        y = targets["up+"].basis.numberStates()
        with pytest.raises(nat.DmvError, match="y must not be null"):
            nat.check(lib.dmv_apply_fermion(targets["up+"]._ctx, op._ctx, nat.DMV_C128, 0, w_up.ctypes.data, 1,
                                            np.ones(n, dtype=np.complex128).ctypes.data, None))
        with pytest.raises(nat.DmvError, match="x must not be null"):
            nat.check(lib.dmv_apply_fermion(targets["up+"]._ctx, op._ctx, nat.DMV_C128, 0, w_up.ctypes.data, 1, None,
                                            np.zeros(2 * y).ctypes.data))
        with pytest.raises(ValueError):
            op.apply_fermion("c-", w_up, np.ones(n), targets["up-"])
        with pytest.raises(ValueError):
            op.apply_fermion("c", np.ones(5), np.ones(n), targets["up-"])
        # accepted: all-zero weights into either half
        assert np.all(op.apply_fermion("c+", np.zeros(8), np.ones(n), targets["down+"]) == 0)
        for t in targets.values():
            t.close()
    finally:
        spin.close()
        op.close()
    op = Operator(_model(conf)[1], rank=0, num_ranks=2)   # two ranks without a communicator
    try:
        op.basis.build()
        with pytest.raises(nat.DmvError, match="dmv_comm_init"):
            op.one_body_density_matrix(np.ones(op.basis.numberStates()))
    finally:
        op.close()


@pytest.mark.gpu
def test_collective_fermion_observables_two_ranks(need_cuda):
    """Two ranks against one rank (tools/fermion_observables_check.py)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--standalone",
           os.path.join(ROOT, "tools", "fermion_observables_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    lines = [l for l in out.stdout.splitlines() if l.rstrip().endswith(("OK", "FAIL"))]
    assert out.returncode == 0 and len(lines) >= 6 and not any(l.rstrip().endswith("FAIL") for l in lines), \
        out.stdout[-4000:] + out.stderr[-2000:]
