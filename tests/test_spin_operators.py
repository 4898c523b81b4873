"""One-site operators between symmetry sectors on the device (dmv_apply_spin / Operator.apply_spin) and the dynamical
structure factors built on them (distributed_matvec_b200.spectral).

References that share nothing with the library: y_ref = B_tᴴ O B_s x with both symmetry-adapted bases built explicitly
by oracle/dense_pin.py and O assembled on the full 2^n space; the Bethe ansatz of the lowest triplet (checked here
against exact diagonalisation before any GPU test relies on it); the f-sum rule, derived below and checked against
dense matrices.  The row formula and its per-site coefficients K are pinned on the CPU against the dense construction,
and the library's host half against that statement of K.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import yaml

from distributed_matvec_b200 import _native as nat
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "data")
KINDS = {"1": 0, "z": 1, "+": 2, "-": 3}
DELTA = {"1": 0, "z": 0, "+": 1, "-": -1}


# ------------------------------------------------------------------------------------------------------------ models
def _ring_bonds(n):
    return [[i, (i + 1) % n] for i in range(n)]


def _heisenberg(bonds):
    return [{"expression": f"σ{c}₀ σ{c}₁", "sites": bonds} for c in "ˣʸᶻ"]


def _tfim(n, h=0.7):
    return [{"expression": "σᶻ₀ σᶻ₁", "sites": _ring_bonds(n)}, {"expression": f"-{h} × σˣ₀", "sites": [[i] for i in range(n)]}]


def _ring(n, weight, k=None, r=None, inv=None, terms=None, bond_mirror=False):
    """ring of n sites: translation in sector k (None: no translation), reflection in sector r (about a site, or about
    a bond, j -> n - 1 - j, as in the chain model files), spin inversion inv"""
    sym = []
    if k is not None:
        sym.append({"permutation": [(i + 1) % n for i in range(n)], "sector": k})
    if r is not None:
        sym.append({"permutation": [(n - 1 - i) if bond_mirror else (n - i) % n for i in range(n)], "sector": r})
    d = {"number_spins": n, "hamming_weight": weight, "symmetries": sym}
    if inv:
        d["spin_inversion"] = inv
    basis = basis_from_dict(d)
    return basis, operator_from_dict({"terms": terms or _heisenberg(_ring_bonds(n))}, basis)


def _from_yaml(name, weight=None, sectors=None, inv="keep", keep_generators=None):
    """a model of data/ with its basis changed: Hamming weight, generator sectors, spin inversion, generators kept"""
    with open(os.path.join(DATA, name + ".yaml"), encoding="utf-8") as f:
        d = yaml.safe_load(f)
    b = dict(d["basis"])
    if weight is not None:
        b["hamming_weight"] = weight
    sym = [dict(g) for g in b.get("symmetries") or []]
    if sectors is not None:
        for g, s in zip(sym, sectors):
            g["sector"] = s
    if keep_generators is not None:
        sym = sym[:keep_generators]
    b["symmetries"] = sym
    if inv != "keep":
        b["spin_inversion"] = inv
    basis = basis_from_dict(b)
    return basis, operator_from_dict({"terms": d["hamiltonian"]["terms"]}, basis)


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


# ------------------------------------------------------------------------------ the row formula, stated in numpy
def _np_plan(src, tgt, kind, w):
    """(k_set, k_clear, c0, walk) of dmv_apply_spin: K_k = 1/|G_t| sum_g chi_t(g) conj chi_s(g) w[p_g^-1(k)]; a flip
    negates σᶻ and swaps σ⁺ / σ⁻.  σ⁺ terms walk the set bits of a row, σ⁻ terms its clear bits."""
    ps, fs, cs = _group(src)
    pt, ft, ct = _group(tgt)
    n = src.number_sites
    k_set, k_clear = np.zeros(n, dtype=complex), np.zeros(n, dtype=complex)
    any_flip = False
    for p, f, c in zip(pt, ft, ct):
        e = [i for i in range(len(ps)) if np.array_equal(ps[i], p) and bool(fs[i]) == bool(f)]
        if not e:
            raise ValueError("not a subgroup")
        any_flip |= bool(f)
        chi = c * np.conj(cs[e[0]]) * (-1.0 if (f and kind == "z") else 1.0)
        contrib = chi * np.asarray(w)[np.argsort(p)]
        if kind in "1z" or ((kind == "+") != bool(f)):
            k_set += contrib
        else:
            k_clear += contrib
    k_set, k_clear = k_set / len(pt), k_clear / len(pt)
    c0 = 0j
    if kind == "1":
        c0, k_set = k_set.sum(), np.zeros(n, dtype=complex)
    elif kind == "z":
        k_clear = -k_set
    walk = 0 if kind in "1z" else 3 if any_flip else 2 if kind == "+" else 1
    return k_set, k_clear, c0, walk


def _np_rows(src, tgt, kind, w, x):
    """y of the row formula: y_r = 1/n_t(r) [c(r) psi(r) | sum_k K_k psi(r ^ e_k)] on psi = B_s x"""
    from oracle.dense_pin import symmetry_adapted_basis
    _, _, Bs = symmetry_adapted_basis(src)
    reps, norms, _ = symmetry_adapted_basis(tgt)
    psi = Bs @ x
    k_set, k_clear, c0, walk = _np_plan(src, tgt, kind, w)
    n = src.number_sites
    y = np.zeros(reps.shape[0], dtype=complex)
    for i, r in enumerate(int(v) for v in reps):
        bits = [(r >> k) & 1 for k in range(n)]
        if walk == 0:
            c = c0 + sum(k_set[k] if bits[k] else k_clear[k] for k in range(n)) if kind == "z" else c0
            y[i] = c * psi[r]
        else:
            for k in range(n):
                if (walk & 2 and bits[k]) or (walk & 1 and not bits[k]):
                    y[i] += (k_set[k] if bits[k] else k_clear[k]) * psi[r ^ (1 << k)]
        y[i] /= norms[i]
    return y


def _full_op(n, kind, w):
    """O = sum_j w_j o_j on the full 2^n space (sparse)"""
    s = np.arange(1 << n, dtype=np.int64)
    rows, cols, vals = [], [], []
    for j in range(n):
        b = (s >> j) & 1
        if kind in "1z":
            rows.append(s); cols.append(s); vals.append(w[j] * (np.ones(s.shape[0]) if kind == "1" else 2.0 * b - 1.0))
        else:
            m = b == (0 if kind == "+" else 1)
            rows.append(s[m] ^ (1 << j)); cols.append(s[m]); vals.append(np.full(int(m.sum()), w[j], dtype=complex))
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(1 << n, 1 << n))


def _reference(src, tgt, kind, w, x):
    from oracle.dense_pin import symmetry_adapted_basis
    _, _, Bs = symmetry_adapted_basis(src)
    _, _, Bt = symmetry_adapted_basis(tgt)
    return Bt.conj().T @ (_full_op(src.number_sites, kind, w) @ (Bs @ x))


# Sectors of the five generators of the square-torus model files (T_x, T_y, mirror x -> L - 1 - x, mirror y -> L - 1 - y,
# rotation by 90°) that hold O_(π,π)|0> for a ground state of the k = 0 sector with trivial point-group characters:
# (-1)^{x+y} is odd under both translations (sector L/2) and under the mirrors and the rotation, which all move a site to
# one of the other colour of the checkerboard (sector 1 of period 2, sector 2 of period 4); found on the 4 x 4 with the
# dense pin by test_torus_landing_sector.
TORUS4_PIPI, TORUS6_PIPI = [2, 2, 1, 1, 2], [3, 3, 1, 1, 2]


# (id, builder of (source, target) for a kind): every builder returns model specs (basis, operator)
def _pair(case, kind):
    d = DELTA[kind]
    if case == "ring12_k0r0_to_k3":
        return _ring(12, 6, 0, 0), _ring(12, 6 + d, 3)
    if case == "ring12_k0r0_to_k6r0":
        return _ring(12, 6, 0, 0), _ring(12, 6 + d, 6, 0)
    if case == "ring10_k1_to_k4":          # a complex character in the source
        return _ring(10, 5, 1), _ring(10, 5 + d, 4)
    if case == "ring8_inv_to_k4":          # the spin-inversion character changes with σᶻ; σ^± leave the inversion
        return _ring(8, 4, 0, 0, 1), (_ring(8, 4, 4, 0, -1) if d == 0 else _ring(8, 4 + d, 4, 0))
    if case == "kagome12_unfold":
        return _from_yaml("heisenberg_kagome_12_symm"), _from_yaml("heisenberg_kagome_12", weight=6 + d)
    if case == "torus4_to_translations_pipi":
        return _from_yaml("heisenberg_square_4x4"), _from_yaml("heisenberg_square_4x4", weight=8 + d, sectors=[2, 2],
                                                               inv=None, keep_generators=2)
    if case == "torus4_to_full_pipi":      # the (π, π) sector of the whole space group that holds O_(π,π)|0>
        return _from_yaml("heisenberg_square_4x4"), _from_yaml("heisenberg_square_4x4", weight=8 + d,
                                                               sectors=TORUS4_PIPI, inv=-1 if d == 0 else None)
    if case == "torus4_to_full_pipi_even":  # (π, π) with trivial point-group characters: O_(π,π)|0> does not reach it,
        # random weights do
        return _from_yaml("heisenberg_square_4x4"), _from_yaml("heisenberg_square_4x4", weight=8 + d,
                                                               sectors=[2, 2, 0, 0, 0], inv=-1 if d == 0 else None)
    if case == "tfim10_free_inv":          # free weight with spin inversion: σ^± walk both bits
        return (_ring(10, None, 0, 0, 1, terms=_tfim(10)), _ring(10, None, 5, 0, -1, terms=_tfim(10)))
    if case == "ring12_inv_unfold":
        return _ring(12, 6, 0, 0, 1), _ring(12, 6 + d)
    if case == "inversion_only":           # spin inversion without permutations (its norms are sqrt(1/2))
        return _ring(10, 5, inv=1), (_ring(10, 5, inv=-1) if d == 0 else _ring(10, 5 + d))
    if case == "plain_to_plain":
        return _ring(10, 5), _ring(10, 5 + d)
    if case == "plain_free":
        return _ring(8, None), _ring(8, None)
    raise KeyError(case)


PAIRS = ["ring12_k0r0_to_k3", "ring12_k0r0_to_k6r0", "ring10_k1_to_k4", "ring8_inv_to_k4", "kagome12_unfold",
         "torus4_to_translations_pipi", "torus4_to_full_pipi", "torus4_to_full_pipi_even", "tfim10_free_inv", "ring12_inv_unfold",
         "inversion_only", "plain_to_plain", "plain_free"]
CPU_PAIRS = ["ring12_k0r0_to_k3", "ring12_k0r0_to_k6r0", "ring10_k1_to_k4", "ring8_inv_to_k4", "tfim10_free_inv",
             "inversion_only", "plain_to_plain"]


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("case", CPU_PAIRS)
def test_row_formula_against_dense(case, kind):
    """The row formula with K (direction p_g^-1, chi_t conj chi_s, the flips) equals B_tᴴ O B_s x to 1e-12."""
    (src, _), (tgt, _) = _pair(case, kind)
    from oracle.dense_pin import symmetry_adapted_basis
    rng = np.random.default_rng(5)
    n = symmetry_adapted_basis(src)[0].shape[0]
    x = rng.normal(size=n) + 1j * rng.normal(size=n)
    w = rng.normal(size=src.number_sites) + 1j * rng.normal(size=src.number_sites)
    ref = _reference(src, tgt, kind, w, x)
    assert np.linalg.norm(ref) > 1e-3 or kind == "1"
    assert np.abs(_np_rows(src, tgt, kind, w, x) - ref).max() <= 1e-12 * max(1.0, np.linalg.norm(ref))


def _desc(basis):
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


def _debug_plan(src, tgt, kind, w, elt=nat.DMV_C128):
    bs, ks = _desc(src)
    bt, kt = _desc(tgt)
    n = src.number_sites
    wv = np.ascontiguousarray(np.asarray(w, dtype=np.complex128))
    k, c0, walk = np.zeros(2 * n, dtype=np.complex128), np.zeros(1, dtype=np.complex128), C.c_int(-1)
    nat.check(nat.lib().dmv_debug_spin_weights(C.byref(bs), C.byref(bt), elt, KINDS[kind], wv.ctypes.data, k.ctypes.data,
                                               c0.ctypes.data, C.byref(walk)))
    return k[:n], k[n:], c0[0], walk.value


@pytest.mark.parametrize("kind", list(KINDS))
@pytest.mark.parametrize("case", PAIRS + ["square6x6_pipi", "chain32_pi"])
def test_host_weights_match_numpy(case, kind):
    """dmv_debug_spin_weights: K, the constant and the walk equal the numpy statement to 1e-15 (chain, torus, kagome,
    translation sectors, flips)."""
    d = DELTA[kind]
    if case == "square6x6_pipi":
        src = _from_yaml("heisenberg_square_6x6")[0]
        tgt = _from_yaml("heisenberg_square_6x6", weight=18 + d, sectors=TORUS6_PIPI, inv=-1 if d == 0 else None)[0]
    elif case == "chain32_pi":
        src = _from_yaml("heisenberg_chain_32_symm")[0]
        tgt = _from_yaml("heisenberg_chain_32_symm", weight=16 + d, sectors=[16, 0], inv=-1 if d == 0 else None)[0]
    else:
        (src, _), (tgt, _) = _pair(case, kind)
    rng = np.random.default_rng(9)
    w = rng.normal(size=src.number_sites) + 1j * rng.normal(size=src.number_sites)
    want = _np_plan(src, tgt, kind, w)
    got = _debug_plan(src, tgt, kind, w)
    assert got[3] == want[3]
    for a, b in zip(got[:3], want[:3]):
        assert np.abs(np.asarray(a) - np.asarray(b)).max() <= 1e-15 * max(1.0, np.abs(w).sum())
    if case == "tfim10_free_inv" and kind in "+-":
        assert got[3] == 3   # both bits


def test_host_inclusion_and_refusals():
    """The subgroup check (set inclusion of (permutation, flip), characters free) and every refusal, with its message."""
    src = _ring(12, 6, 0, 0)[0]
    w = np.ones(12)
    # subgroups: translations only, plain, itself with other characters
    for tgt in (_ring(12, 6, 5)[0], _ring(12, 6)[0], _ring(12, 6, 6, 1)[0]):
        _debug_plan(src, tgt, "z", w)
    cases = [(_ring(10, 5)[0], "z", nat.DMV_C128, "same number of sites"),
             (_ring(12, 7, 0)[0], "z", nat.DMV_C128, "Hamming weights"),
             (_ring(12, 6, 0)[0], "+", nat.DMV_C128, "Hamming weights"),
             (_ring(12, None, 0)[0], "-", nat.DMV_C128, "Hamming weights"),
             (_ring(12, 6, 0, 0, 1)[0], "z", nat.DMV_C128, "not a subgroup"),
             (_ring(12, 6, 3)[0], "z", nat.DMV_F64, "DMV_F64 needs real"),
             (_ring(12, 6, 0)[0], "z", 3, "elt")]
    for tgt, kind, elt, msg in cases:
        with pytest.raises(nat.DmvError, match=msg):
            _debug_plan(src, tgt, kind, w, elt)
    with pytest.raises(nat.DmvError, match="DMV_F64 needs real"):   # complex weights
        _debug_plan(src, _ring(12, 6, 0)[0], "z", w * 1j, nat.DMV_F64)
    bs, ks = _desc(src)
    bt, kt = _desc(_ring(12, 6, 0)[0])
    wv = np.ones(12, dtype=np.complex128)
    for kind in (-1, 4):
        with pytest.raises(nat.DmvError, match="kind must be"):
            nat.check(nat.lib().dmv_debug_spin_weights(C.byref(bs), C.byref(bt), nat.DMV_C128, kind, wv.ctypes.data,
                                                       None, None, None))
    with pytest.raises(nat.DmvError, match="weights must not be null"):
        nat.check(nat.lib().dmv_debug_spin_weights(C.byref(bs), C.byref(bt), nat.DMV_C128, 1, None, None, None, None))


# ------------------------------------------------------------------------------------------ Bethe triplet, f-sum
def bethe_energy(n_sites: int, magnons: int) -> float:
    """E / J of the Bethe state with `magnons` real rapidities and the contiguous quantum numbers I_j = -(M - 1) / 2 ...
    (M - 1) / 2 of H = J sum S_i.S_{i+1} on a ring: M = N / 2 the ground state, M = N / 2 - 1 the lowest triplet (two
    holes at the edges of the quantum numbers).  N arctan(2 λ_j) = π I_j + Σ_k arctan(λ_j - λ_k)."""
    N, M = n_sites, magnons
    quantum = np.arange(M) - (M - 1) / 2.0
    lam = 0.5 * np.tan(np.pi * quantum / N)
    for _ in range(200000):
        new = 0.5 * np.tan((np.pi * quantum + np.arctan(lam[:, None] - lam[None, :]).sum(axis=1)) / N)
        done = np.abs(new - lam).max() < 1e-15
        lam = 0.5 * (new + lam)
        if done:
            break
    residual = N * np.arctan(2 * lam) - np.pi * quantum - np.arctan(lam[:, None] - lam[None, :]).sum(axis=1)
    if np.abs(residual).max() > 1e-12:
        raise RuntimeError("Bethe equations did not converge")
    return float(N / 4.0 - np.sum(2.0 / (4.0 * lam * lam + 1.0)))


def _sector_h(n, weight, bonds):
    from oracle.sector_pin import sector_hamiltonian, sector_states
    states = sector_states(n, weight)
    return states, sector_hamiltonian(_heisenberg(bonds), n, states)


@pytest.mark.parametrize("n", [8, 10, 12, 14, 16])
def test_bethe_triplet_equals_exact_diagonalisation(n):
    """The Bethe triplet (M = N/2 - 1) is the lowest S^z = 1 energy of the ring, to 1e-10 (sigma form: 4 E)."""
    import scipy.sparse.linalg as sla
    _, H = _sector_h(n, n // 2 + 1, _ring_bonds(n))
    e = np.linalg.eigvalsh(H.toarray()).min() if H.shape[0] <= 2000 else sla.eigsh(H, k=1, which="SA", tol=1e-13)[0][0]
    assert abs(e - 4.0 * bethe_energy(n, n // 2 - 1)) <= 1e-10 * abs(e), (n, e)


def _torus_bonds(L):
    return [[y * L + x, y * L + (x + 1) % L] for y in range(L) for x in range(L)] + \
           [[y * L + x, ((y + 1) % L) * L + x] for y in range(L) for x in range(L)]


def f_sum(w, bonds, T):
    """½<[O†, [H, O]]> for O = Σ_j w_j σᶻ_j and H = Σ_bonds σ_i·σ_j = Σ_bonds 2 (σ⁺_iσ⁻_j + σ⁻_iσ⁺_j) + σᶻ_iσᶻ_j: with
    [σ⁺_iσ⁻_j, σᶻ_k] = 2 (δ_jk - δ_ik) σ⁺_iσ⁻_j the σᶻσᶻ part commutes and
        ½<[O†, [H, O]]> = -8 Σ_bonds |w_i - w_j|² Re T_ij,   T_ij = <σ⁺_iσ⁻_j>."""
    return -8.0 * sum(abs(w[i] - w[j]) ** 2 * T[i, j].real for i, j in bonds)


@pytest.mark.parametrize("lattice", ["ring8", "ring10", "ring12", "torus4"])
def test_f_sum_rule_against_dense(lattice):
    """f_sum equals ½<[O†, [H, O]]> on the ground state with dense / sparse matrices, for q = π (or (π, π)) and a
    generic q."""
    import scipy.sparse.linalg as sla
    from oracle.sector_pin import Sector
    if lattice == "torus4":
        n, bonds = 16, _torus_bonds(4)
        coords = np.array([[s % 4, s // 4] for s in range(16)], dtype=float)
        qs = [np.array([np.pi, np.pi]), np.array([np.pi / 2, 0.0])]
    else:
        n = int(lattice[4:])
        bonds, coords = _ring_bonds(n), np.arange(n, dtype=float)
        qs = [np.array([np.pi]), np.array([2 * np.pi / n])]
    states, H = _sector_h(n, n // 2, bonds)
    vals, vecs = sla.eigsh(H, k=1, which="SA", tol=1e-14)
    psi = vecs[:, 0]
    sec = Sector(basis_from_dict({"number_spins": n, "hamming_weight": n // 2}), _heisenberg(bonds))
    T = sec.pm(psi)
    bits = ((states[:, None] >> np.arange(n, dtype=np.uint64)[None, :]) & np.uint64(1)).astype(float)
    from distributed_matvec_b200.spectral import fourier_weights
    for q in qs:
        w = fourier_weights(coords, q)
        O = sp.diags((2.0 * bits - 1.0) @ w)
        Od = O.conj().T
        comm = Od @ (H @ O - O @ H) - (H @ O - O @ H) @ Od
        want = 0.5 * np.vdot(psi, comm @ psi).real
        assert abs(f_sum(w, bonds, T) - want) <= 1e-10 * max(1.0, abs(want)), (lattice, q)


# ---------------------------------------------------------------------------------------------------- spectral.py
def _np_lanczos(A, y, m):
    """m Lanczos steps with full reorthogonalisation: (alpha, beta)"""
    V = [y / np.linalg.norm(y)]
    a, b = [], []
    for j in range(m):
        u = A @ V[-1]
        a.append(np.vdot(V[-1], u).real)
        for v in V:
            u = u - np.vdot(v, u) * v
        if j + 1 < m:
            b.append(np.linalg.norm(u))
            V.append(u / b[-1])
    return np.array(a), np.array(b)


def test_quadrature_poles_and_residues_against_eigendecomposition():
    """Full Lanczos from y: the Gauss nodes and weights (the continued fraction's poles and residues, from the
    library's host half) equal the distinct eigenvalues and Σ |<n|y>|² per level."""
    rng = np.random.default_rng(3)
    levels = np.array([-2.0, -1.0, -1.0, 0.5, 0.5, 0.5, 1.5, 3.0])   # degenerate levels
    Q, _ = np.linalg.qr(rng.normal(size=(8, 8)))
    A = Q @ np.diag(levels) @ Q.T
    y = rng.normal(size=8)
    distinct = np.unique(levels)
    want = np.array([np.sum(np.abs(Q[:, levels == e].T @ y) ** 2) for e in distinct])
    a, b = _np_lanczos(A, y, len(distinct))
    nodes, weights = np.zeros(len(a)), np.zeros(len(a))
    nat.check(nat.lib().dmv_debug_tridiagonal_quadrature(len(a), a.ctypes.data, b.ctypes.data, nodes.ctypes.data,
                                                         weights.ctypes.data))
    weights *= np.vdot(y, y).real
    assert np.abs(nodes - distinct).max() <= 1e-12 and np.abs(weights - want).max() <= 1e-12


@pytest.mark.parametrize("shape", ["lorentzian", "gaussian"])
def test_broaden_integrates_to_the_total_weight(shape):
    from distributed_matvec_b200.spectral import broaden
    poles, res = np.array([0.3, 1.1, 2.5]), np.array([0.5, 0.2, 0.05])
    omega = np.linspace(-2000.0, 2000.0, 4_000_001) if shape == "lorentzian" else np.linspace(-5, 8, 20001)
    s = broaden(poles, res, omega, 0.05, shape)
    assert abs(np.trapezoid(s, omega) - res.sum()) <= 1e-4 * res.sum()
    with pytest.raises(ValueError):
        broaden(poles, res, omega[:5], 0.0, shape)


class _StubSource:
    """apply_spin returns a fixed vector; one rank"""
    num_ranks, device = 1, 0

    def __init__(self, y):
        self.y = y

    def apply_spin(self, kind, weights, x, target):
        return self.y


class _StubTarget:
    def __init__(self):
        self.calls = 0

    def lanczos_quadrature(self, num_vectors, steps, start=None):
        self.calls += 1
        nodes, weights = np.zeros((1, steps)), np.zeros((1, steps))
        nodes[0, :2], weights[0, :2] = [1.0, 3.0], np.array([0.25, 0.75]) * np.vdot(start, start).real
        return nodes, weights, np.array([2]), 2


def test_dynamical_correlation_empty_sector():
    """y at rounding level relative to |x0| |w| (a sector O|0> does not reach) gives no poles and no Lanczos; a y above
    the threshold runs the quadrature, and the poles are shifted by e0."""
    from distributed_matvec_b200.spectral import dynamical_correlation
    x0, w = np.ones(50) / np.sqrt(50), np.ones(8)
    for noise in (0.0, 1e-17, 1e-13):
        tgt = _StubTarget()
        poles, res = dynamical_correlation(_StubSource(np.full(20, noise)), x0, -1.0, tgt, "z", w, 10)
        assert poles.shape == (0,) and res.shape == (0,) and tgt.calls == 0, noise
    tgt = _StubTarget()
    poles, res = dynamical_correlation(_StubSource(np.full(20, 1e-6)), x0, -1.0, tgt, "z", w, 10)
    assert tgt.calls == 1 and np.allclose(poles, [2.0, 4.0]) and np.allclose(res.sum(), 20e-12)


def test_fourier_weights_sign_follows_the_sector_convention():
    """σᶻ_q with fourier_weights moves a state of translation sector 0 into sector k with q = 2πk/N (dense pin)."""
    from distributed_matvec_b200.spectral import fourier_weights
    n = 8
    rng = np.random.default_rng(1)
    src = _ring(n, 4, 0)[0]
    from oracle.dense_pin import symmetry_adapted_basis
    x = rng.normal(size=symmetry_adapted_basis(src)[0].shape[0])
    w = fourier_weights(np.arange(n), 2 * np.pi * 3 / n)
    norms = [np.linalg.norm(_reference(src, _ring(n, 4, k)[0], "z", w, x)) for k in range(n)]
    assert np.argmax(norms) == 3 and sum(norms) - norms[3] <= 1e-12


# ------------------------------------------------------------------------------------------------------------ GPU
def _torch():
    return pytest.importorskip("torch")


@pytest.fixture(scope="module")
def need_cuda():
    if not _torch().cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _ops(src_model, tgt_model, options=None):
    from distributed_matvec_b200 import Operator
    s, t = Operator(src_model[1]), Operator(tgt_model[1])
    for key, value in (options or {}).items():
        s.set_option(key, value)
    s.basis.build()
    t.basis.build()
    return s, t


# case, source options: every look-up of a source with trivial characters (dense ordered table, ordered layout, hashed
# table, rows = 0 -> index), the square-torus orbit minimum, complex characters, spin inversion alone, no symmetry
COVER = [(c, {}) for c in PAIRS] + [("ring12_k0r0_to_k3", {"rows_dense_order": 0}),
                                     ("ring12_k0r0_to_k3", {"rows_table": 0}), ("ring12_k0r0_to_k3", {"rows": 0}),
                                     ("torus4_to_full_pipi", {"rows": 0}), ("torus4_to_full_pipi", {"canon": 0})]


@pytest.mark.gpu
@pytest.mark.parametrize("case,options", COVER, ids=[f"{c}-{'-'.join(f'{k}{v}' for k, v in o.items())}" for c, o in COVER])
def test_against_dense_pin(need_cuda, case, options):
    """Every kind, float64 (real weights and characters) and complex128, numpy and a torch [2, n] batch, equals
    B_tᴴ O B_s x to 1e-12 relative."""
    torch = _torch()
    from oracle.dense_pin import symmetry_adapted_basis
    for kind in KINDS:
        src_m, tgt_m = _pair(case, kind)
        s, t = _ops(src_m, tgt_m, options)
        reps_s, _, _ = symmetry_adapted_basis(src_m[0])
        reps_t, _, _ = symmetry_adapted_basis(tgt_m[0])
        assert np.array_equal(s.basis.representatives(), reps_s) and np.array_equal(t.basis.representatives(), reps_t)
        n, N = reps_s.shape[0], src_m[0].number_sites
        rng = np.random.default_rng(11)
        real = not (s.info("complex_coefficients") or t.info("complex_coefficients"))
        for dtype in ([np.float64] if real else []) + [np.complex128]:
            cplx = dtype == np.complex128
            X = rng.normal(size=(2, n)) + (1j * rng.normal(size=(2, n)) if cplx else 0)
            w = rng.normal(size=N) + (1j * rng.normal(size=N) if cplx else 0)
            refs = [_reference(src_m[0], tgt_m[0], kind, w, X[v]) for v in range(2)]
            y1 = s.apply_spin(kind, w, np.ascontiguousarray(X[0]), t)
            assert y1.dtype == dtype and y1.shape == (reps_t.shape[0],)
            yt = s.apply_spin(kind, w, torch.from_numpy(X).cuda(), t)
            torch.cuda.synchronize()
            yt = yt.cpu().numpy()
            for v, y in ((0, y1), (0, yt[0]), (1, yt[1])):
                scale = max(np.linalg.norm(refs[v]), 1e-4 * np.linalg.norm(X[v]) * np.linalg.norm(w))
                assert np.abs(y - refs[v]).max() <= 1e-12 * scale, (case, options, kind, dtype, v)
        s.close()
        t.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [16, 20])
def test_completeness_over_momentum_sectors(need_cuda, n):
    """Σ over every translation sector k of ‖y_k‖² = <ψ|O†O|ψ>: Σ conj(w_i) w_j C_ij (σᶻ, from zz_correlations) and
    Σ conj(w_i) w_j T_ij (σ⁻, from pm_correlations), times ‖x‖², to 1e-12."""
    from distributed_matvec_b200 import Operator
    src = Operator(_ring(n, n // 2, 0)[1])
    src.basis.build()
    rng = np.random.default_rng(23)
    x = rng.normal(size=src.basis.numberStates()) + 1j * rng.normal(size=src.basis.numberStates())
    w = rng.normal(size=n) + 1j * rng.normal(size=n)
    W = np.vdot(x, x).real
    Cz, _ = src.zz_correlations(x)
    T = src.pm_correlations(x)
    want = {"z": (np.conj(w) @ Cz @ w).real * W, "-": (np.conj(w) @ T @ w).real * W}
    for kind, d in (("z", 0), ("-", -1)):
        total = 0.0
        for k in range(n):
            t = Operator(_ring(n, n // 2 + d, k)[1])
            t.basis.build()
            y = src.apply_spin(kind, w, x, t)
            total += np.vdot(y, y).real
            t.close()
        assert abs(total - want[kind]) <= 1e-12 * want[kind], (n, kind, total, want[kind])
    src.close()


def _square_pipi_weights():
    from distributed_matvec_b200.spectral import fourier_weights
    coords = np.array([[s % 6, s // 6] for s in range(36)], dtype=float)
    return fourier_weights(coords, [np.pi, np.pi]).real   # (-1)^{x+y} / 6


@pytest.mark.gpu
def test_square_6x6_full_size(need_cuda):
    """6 x 6 ground state (eigsh): σᶻ_(π,π) into the (π, π) sector of the whole space group with odd point-group
    characters (TORUS6_PIPI) and opposite spin inversion has ‖y‖² = wᵀ C w, and σ⁻_(π,π) into that sector at weight 17
    (no spin inversion) has ‖y‖² = wᵀ T w = ½ wᵀ C w (a singlet), to 1e-10: all of O|0> lies in each target.  The
    same sector with trivial point-group characters gets nothing."""
    torch = _torch()
    from distributed_matvec_b200 import Operator
    src = Operator(_from_yaml("heisenberg_square_6x6")[1])
    src.basis.build()
    n = src.basis.numberStates()
    vec = torch.empty((1, n), dtype=torch.float64, device="cuda")
    vals, _, _, conv, _, _ = src.eigsh(1, tol=1e-11, eigenvectors=vec)
    assert conv == 1 and abs(vals[0] - (-97.757589597)) <= 1e-6
    psi = vec[0]
    w = _square_pipi_weights()
    Cz, _ = src.zz_correlations(psi)
    T = src.pm_correlations(psi)
    S_zz, S_pm = float(w @ Cz @ w), float((w @ T @ w).real)
    empty = Operator(_from_yaml("heisenberg_square_6x6", sectors=[3, 3, 0, 0, 0], inv=-1)[1])
    empty.basis.build()
    y = src.apply_spin("z", w, psi, empty)
    assert float(torch.vdot(y, y).real) <= 1e-24 * S_zz
    empty.close()
    tz = Operator(_from_yaml("heisenberg_square_6x6", sectors=TORUS6_PIPI, inv=-1)[1])
    tz.basis.build()
    y = src.apply_spin("z", w, psi, tz)
    nz = float(torch.vdot(y, y).real)
    tz.close()
    assert abs(nz - S_zz) <= 1e-10 * S_zz, (nz, S_zz)
    tm = Operator(_from_yaml("heisenberg_square_6x6", weight=17, sectors=TORUS6_PIPI, inv=None)[1])
    tm.basis.build()
    y = src.apply_spin("-", w, psi, tm)
    nm = float(torch.vdot(y, y).real)
    tm.close()
    assert abs(nm - S_pm) <= 1e-10 * S_pm and abs(nm - 0.5 * S_zz) <= 1e-9 * S_zz, (nm, S_pm, S_zz)
    src.close()


def _landing_sector(n, kind):
    """(reflection sector, spin inversion) of the k = π sector where O_π of the ring's ground state lands, found with the
    dense pin on a small ring of the same form as chain_32_symm (the mirror about a bond; N ≡ 0 mod 4: ground state at
    k = 0, r = 0, inversion +1)"""
    import scipy.sparse.linalg as sla
    from oracle.dense_pin import projected_hamiltonian
    from distributed_matvec_b200.spectral import fourier_weights
    src = _ring(n, n // 2, 0, 0, 1, bond_mirror=True)
    _, _, Hp = projected_hamiltonian(_heisenberg(_ring_bonds(n)), src[0])
    x = np.linalg.eigh(Hp)[1][:, 0]
    w = fourier_weights(np.arange(n), np.pi).real
    d = DELTA[kind]
    best, where = 0.0, None
    for r in (0, 1):
        for inv in ((1, -1) if d == 0 else (None,)):
            tgt = _ring(n, n // 2 + d, n // 2, r, inv, bond_mirror=True)[0]
            y = _reference(src[0], tgt, kind, w, x)
            if np.linalg.norm(y) > best:
                best, where = np.linalg.norm(y), (r, inv)
    return where


def _torus_landing(kind):
    """(point-group sectors, spin inversion) of the (π, π) sector of the 4 x 4 torus's whole space group that holds
    O_(π,π)|0>, by the dense pin: every consistent assignment of the mirror (period 2) and rotation (period 4) sectors"""
    import itertools
    from oracle.dense_pin import projected_hamiltonian, symmetry_adapted_basis
    src, _ = _from_yaml("heisenberg_square_4x4")
    with open(os.path.join(DATA, "heisenberg_square_4x4.yaml"), encoding="utf-8") as f:
        terms = yaml.safe_load(f)["hamiltonian"]["terms"]
    _, _, Hp = projected_hamiltonian(terms, src)
    x = np.linalg.eigh(Hp)[1][:, 0]
    w = np.array([(-1.0) ** (s % 4 + s // 4) for s in range(16)]) / 4.0
    total = np.linalg.norm(_full_op(16, kind, w) @ (symmetry_adapted_basis(src)[2] @ x))
    d = DELTA[kind]
    found = []
    for s3, s4, s5 in itertools.product((0, 1), (0, 1), range(4)):
        for inv in ((1, -1) if d == 0 else (None,)):
            try:
                tgt = _from_yaml("heisenberg_square_4x4", weight=8 + d, sectors=[2, 2, s3, s4, s5], inv=inv)[0]
                tgt.group
            except ValueError:   # not a one-dimensional representation
                continue
            part = np.linalg.norm(_reference(src, tgt, kind, w, x))
            if part > 1e-8 * total:
                found.append(([2, 2, s3, s4, s5], inv, part / total))
    return found


@pytest.mark.parametrize("kind", ["z", "-"])
def test_torus_landing_sector(kind):
    """All of O_(π,π)|0> of the 4 x 4 ground state lies in one sector of the whole space group: TORUS4_PIPI (odd under
    the mirrors and the rotation), with spin inversion -1 for σᶻ.  The generators of the 6 x 6 model file act on
    (-1)^{x+y} as those of the 4 x 4 (each one with the same sign), so TORUS6_PIPI is the 6 x 6 sector."""
    found = _torus_landing(kind)
    assert len(found) == 1, found
    sectors, inv, part = found[0]
    assert sectors == TORUS4_PIPI and inv == (-1 if kind == "z" else None) and abs(part - 1.0) <= 1e-12, found
    for name, L in (("heisenberg_square_4x4", 4), ("heisenberg_square_6x6", 6)):
        with open(os.path.join(DATA, name + ".yaml"), encoding="utf-8") as f:
            gens = [g["permutation"] for g in yaml.safe_load(f)["basis"]["symmetries"]]
        colour = np.array([(-1.0) ** (s % L + s // L) for s in range(L * L)])
        assert [int(round(colour[np.asarray(p)] @ colour / (L * L))) for p in gens] == [-1] * 5, name


@pytest.mark.parametrize("kind", ["z", "-"])
def test_landing_sector_is_the_same_on_small_rings(kind):
    """The k = π sector that holds O_π|0> is the same on the 8- and 12-site rings (the chain_32 test relies on it)."""
    assert _landing_sector(8, kind) == _landing_sector(12, kind)


@pytest.mark.gpu
def test_chain_32_structure_factor(need_cuda):
    """chain_32_symm: the lowest pole of S^zz(π, ω) is the Bethe triplet gap (1e-8 relative); S^{+-}(π, ω) into weight
    15 has the same lowest pole and half its weight (Wigner-Eckart); the zeroth moment is S(π) from zz_correlations and
    the first moment the f-sum value from pm_correlations (1e-8)."""
    torch = _torch()
    from distributed_matvec_b200 import Operator
    from distributed_matvec_b200.spectral import dynamical_correlation, fourier_weights
    n = 32
    src = Operator(_from_yaml("heisenberg_chain_32_symm")[1])
    src.basis.build()
    vec = torch.empty((1, src.basis.numberStates()), dtype=torch.float64, device="cuda")
    vals, _, _, conv, _, _ = src.eigsh(1, tol=1e-12, eigenvectors=vec)
    assert conv == 1
    e0 = float(vals[0])
    assert abs(e0 - 4.0 * bethe_energy(n, n // 2)) <= 1e-9 * abs(e0)
    gap = 4.0 * (bethe_energy(n, n // 2 - 1) - bethe_energy(n, n // 2))
    w = fourier_weights(np.arange(n), np.pi).real
    Cz, _ = src.zz_correlations(vec[0])
    T = src.pm_correlations(vec[0])
    S_pi = float(w @ Cz @ w)
    fsum = f_sum(w, _ring_bonds(n), T)
    out = {}
    for kind, weight in (("z", 16), ("-", 15)):
        r, inv = _landing_sector(12, kind)
        tgt = Operator(_from_yaml("heisenberg_chain_32_symm", weight=weight, sectors=[16, r], inv=inv)[1])
        tgt.basis.build()
        poles, res = dynamical_correlation(src, vec[0], e0, tgt, kind, w, 120)
        tgt.close()
        keep = res > 1e-10 * res.sum()
        out[kind] = (poles[keep], res[keep])
    pz, rz = out["z"]
    pm, rm = out["-"]
    assert abs(pz[0] - gap) <= 1e-8 * gap, (pz[:3], gap)
    assert abs(pm[0] - gap) <= 1e-8 * gap, (pm[:3], gap)
    assert abs(rz.sum() - S_pi) <= 1e-8 * S_pi and abs(rm.sum() - 0.5 * S_pi) <= 1e-8 * S_pi
    # without reorthogonalisation a converged pole comes back in copies whose weights add up: compare per level
    low_z, low_m = rz[np.abs(pz - gap) <= 1e-6 * gap].sum(), rm[np.abs(pm - gap) <= 1e-6 * gap].sum()
    assert abs(low_m - 0.5 * low_z) <= 1e-8 * low_z, (low_m, low_z)
    assert abs((rz * pz).sum() - fsum) <= 1e-8 * fsum, ((rz * pz).sum(), fsum)
    src.close()


@pytest.mark.gpu
def test_dynamical_correlation_sectors_of_the_4x4(need_cuda):
    """4 x 4 ground state, O = σᶻ_(π,π): the (π, π) sector with odd point-group characters gets all the weight (Σ
    residues = wᵀ C w, 1e-10) and the same sector with trivial point-group characters, whose y is rounding, no poles."""
    from distributed_matvec_b200 import Operator
    from distributed_matvec_b200.spectral import dynamical_correlation
    src = Operator(_from_yaml("heisenberg_square_4x4")[1])
    src.basis.build()
    vals, vecs = src.eigsh(1, tol=1e-12)[:2]
    psi = vecs[0]
    w = np.array([(-1.0) ** (s % 4 + s // 4) for s in range(16)]) / 4.0
    Cz, _ = src.zz_correlations(psi)
    for sectors, want in ((TORUS4_PIPI, float(w @ Cz @ w)), ([2, 2, 0, 0, 0], 0.0)):
        tgt = Operator(_from_yaml("heisenberg_square_4x4", sectors=sectors, inv=-1)[1])
        tgt.basis.build()
        poles, res = dynamical_correlation(src, psi, float(vals[0]), tgt, "z", w, 40)
        tgt.close()
        if want == 0.0:
            assert poles.shape == (0,) and res.shape == (0,), (poles, res)
        else:
            assert abs(res.sum() - want) <= 1e-10 * want and poles.min() > 0.0, (res.sum(), want)
    src.close()


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["ring12_k0r0_to_k3", "ring10_k1_to_k4", "torus4_to_full_pipi", "tfim10_free_inv"])
def test_repeated_call_is_bit_identical(need_cuda, case):
    torch = _torch()
    for kind in KINDS:
        src_m, tgt_m = _pair(case, kind)
        s, t = _ops(src_m, tgt_m)
        x = torch.rand((2, s.basis.numberStates()), dtype=torch.complex128, device="cuda")
        w = np.random.default_rng(2).normal(size=src_m[0].number_sites) * (1 + 0.5j)
        a, b = s.apply_spin(kind, w, x, t), s.apply_spin(kind, w, x, t)
        assert torch.equal(a, b), (case, kind)
        s.close()
        t.close()


@pytest.mark.gpu
def test_errors_change_nothing(need_cuda):
    """Mismatched contexts, a subgroup violation, a wrong elt and null pointers raise and leave y as it was."""
    from distributed_matvec_b200 import Operator
    lib = nat.lib()
    s, t = _ops(_ring(12, 6, 0, 0), _ring(12, 6, 3))
    n, m = s.basis.numberStates(), t.basis.numberStates()
    x = np.ones(n, dtype=np.complex128)
    w = np.ones(12, dtype=np.complex128)
    y = np.full(m, 7.0 + 7.0j)

    def call(target, source, elt=nat.DMV_C128, kind=1, weights=w.ctypes.data, k=1, xp=x.ctypes.data, yp=y.ctypes.data):
        nat.check(lib.dmv_apply_spin(target._ctx if target else None, source._ctx if source else None, elt, kind,
                                     weights, k, xp, yp))

    other = Operator(_ring(10, 5, 0)[1])
    other.basis.build()
    two = Operator(_ring(12, 6, 3)[1], rank=0, num_ranks=2)
    two.basis.build()
    bigger = Operator(_ring(12, 6, 0, 0, 1)[1])   # spin inversion: not a subgroup of the source's group
    bigger.basis.build()
    unbuilt = Operator(_ring(12, 6, 3)[1])
    for args, msg in [((other, s), "same number of sites"), ((two, s), "same rank"), ((bigger, s), "not a subgroup"),
                      ((t, s, 0), "elt"), ((t, s, 3), "elt"), ((t, s, nat.DMV_C128, 5), "kind must be"),
                      ((None, s), "must not be null"), ((unbuilt, s), "basis is not built")]:
        with pytest.raises(nat.DmvError, match=msg):
            call(*args)
    for kw, msg in [({"weights": None}, "weights must not be null"), ({"xp": None}, "x must not be null"),
                    ({"yp": None}, "y must not be null"), ({"k": 0}, "num_vectors")]:
        with pytest.raises(nat.DmvError, match=msg):
            call(t, s, **kw)
    with pytest.raises(nat.DmvError, match="DMV_F64 needs real"):
        s.apply_spin("z", w * 1j, np.ones(n), t)
    assert np.all(y == 7.0 + 7.0j)
    with pytest.raises(ValueError):
        s.apply_spin("x", w, x, t)
    with pytest.raises(ValueError):
        s.apply_spin("z", w[:5], x, t)
    with pytest.raises(ValueError):
        s.apply_spin("z", w, np.ones(n + 1, dtype=complex), t)
    for o in (s, t, other, two, bigger, unbuilt):
        o.close()


@pytest.mark.gpu
def test_collective_apply_spin_two_ranks(need_cuda):
    """Two ranks against one rank (tools/spin_check.py)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", "29561", os.path.join(ROOT, "tools", "spin_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    lines = [l for l in out.stdout.splitlines() if l.rstrip().endswith(("OK", "FAIL"))]
    assert out.returncode == 0 and len(lines) >= 6 and not any(l.rstrip().endswith("FAIL") for l in lines), \
        out.stdout[-4000:] + out.stderr[-2000:]
