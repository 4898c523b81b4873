"""Lattice symmetries of fermionic bases: momentum and point-group sectors with the fermionic exchange sign.

A basis state is |s> = c†_{a1} ... c†_{ak} |0> with a1 < ... < ak, and a group element g (output bit i takes input bit
p[i]) acts as U_g c†_{p[i]} U_g⁻¹ = c†_i, so U_g|s> = sign(g, s)|g(s)>.  The reference here is U_g built independently:
the creation operators c†_{image(a)} applied to the vacuum, as the Jordan-Wigner matrices of tests/fermion_pin.py and bit
by bit.  Sector bases are P|r>/‖P|r>‖ with P = 1/|G| Σ conj(χ(g)) U_g (oracle/dense_pin.py with the fermionic U_g).

Without a GPU: U_g is a representation, commutes with H, and the host inversion-mask sign equals it; the sectors of the
abelian groups together are the particle-number block (dimensions and spectra); every refusal, in YAML and in the ABI.
On the GPU: products against B†HB for every sector (both product paths, float64 and complex128, batches, two ranks),
enumeration, dmv_state_info, eigsh, zz_correlations, and at size spinless_ring_28 (every momentum against free fermions,
which a missing sign would turn into the twisted-boundary energies) and hubbard_square_4x4_symm.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys
from itertools import product

import numpy as np
import pytest
import scipy.sparse as sp
import yaml

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import fermion_pin as fp  # noqa: E402
from distributed_matvec_b200 import Operator  # noqa: E402
from distributed_matvec_b200 import _native as nat  # noqa: E402
from distributed_matvec_b200.config import basis_from_dict, load_config_from_yaml, operator_from_dict  # noqa: E402
from distributed_matvec_b200.symmetry import build_group, fermion_signs, widen_to_spinful  # noqa: E402
from gen_models import (_bonds_ring, _bonds_torus, hubbard, ring_reflection, ring_translation,  # noqa: E402
                        spinless_ring, torus_translations, with_site_symmetries)

DATA = os.path.join(ROOT, "data")
ONE = np.uint64(1)


# ---------------------------------------------------------------------------------------------------------------------
# the independent U_g

def _image(perm) -> np.ndarray:
    perm = np.asarray(perm, dtype=np.int64)
    image = np.empty(perm.shape[0], dtype=np.int64)
    image[perm] = np.arange(perm.shape[0])
    return image


def u_g(perm, states):
    """U_g|s> = c†_{image(a1)} ... c†_{image(ak)} |0> bit by bit: the factors act right to left, each c†_m with the
    Jordan-Wigner sign (-1)^popc(t & ((1 << m) - 1)) of the state t it acts on.  -> (g(s), sign) for uint64 states."""
    states = np.asarray(states, dtype=np.uint64)
    image = _image(perm)
    t = np.zeros_like(states)
    neg = np.zeros(states.shape, dtype=bool)
    for a in range(image.shape[0] - 1, -1, -1):
        occ = ((states >> np.uint64(a)) & ONE).astype(bool)
        m = int(image[a])
        neg ^= occ & (np.bitwise_count(t & np.uint64((1 << m) - 1)) & 1).astype(bool)
        t |= occ.astype(np.uint64) << np.uint64(m)
    return t, np.where(neg, -1, 1).astype(np.int8)


def u_g_matrix(perm) -> sp.csr_matrix:
    """U_g on the whole Fock space from the Jordan-Wigner matrices of fermion_pin: column s is the product of the creation
    operators c†_{image(a)} over the occupied a of s, ascending from the left, applied to the vacuum."""
    n = len(perm)
    image = _image(perm)
    cdag = [fp.annihilator(n, k).T.tocsr() for k in range(n)]
    cols = []
    for s in range(1 << n):
        v = np.zeros(1 << n)
        v[0] = 1.0
        for a in reversed([a for a in range(n) if (s >> a) & 1]):
            v = cdag[int(image[a])] @ v
        cols.append(sp.csr_matrix(v.reshape(-1, 1)))
    return sp.hstack(cols).tocsr()


def _compose(p, q):   # apply q first, then p
    return [q[i] for i in p]


def _terms(conf):
    return conf["hamiltonian"]["terms"]


def _spinful(conf):
    return conf["basis"]["particle"] == "spinful-fermion"


def _block_states(conf):
    b = conf["basis"]
    if _spinful(conf):
        return fp.sector_states(b["number_sites"], b["number_up"], b["number_particles"] - b["number_up"])
    return fp.sector_states(b["number_sites"], b["number_particles"], spinful=False)


def _block_hamiltonian(conf, states):
    return fp.apply_to_states(_terms(conf), conf["basis"]["number_sites"], _spinful(conf), states)


def sector_basis(group, states):
    """(representatives, norms, B) of the sector inside the block `states`: column k of B is P|r_k>/‖P|r_k>‖ over the
    rows `states`, with the independent U_g."""
    G = len(group)
    imgs, sgns = zip(*(u_g(group.perms[e], states) for e in range(G)))
    images, signs = np.stack(imgs), np.stack(sgns)
    reps_at = np.nonzero(images.min(axis=0) == states)[0]
    rows = np.searchsorted(states, images[:, reps_at])
    vals = np.conj(group.characters)[:, None] * signs[:, reps_at] / G
    cols = np.broadcast_to(np.arange(reps_at.shape[0])[None, :], rows.shape)
    B = sp.coo_matrix((vals.ravel(), (rows.ravel(), cols.ravel())), shape=(states.shape[0], reps_at.shape[0])).tocsc()
    norms = np.sqrt(np.asarray(abs(B).power(2).sum(axis=0)).ravel())
    keep = norms ** 2 > 1e-20
    B = B[:, np.nonzero(keep)[0]] @ sp.diags(1.0 / norms[keep])
    return states[reps_at[keep]], norms[keep], B.tocsr()


def _sector(conf):
    """(representatives, norms, B, B†HB dense) of a model with site_symmetries"""
    basis = basis_from_dict(conf["basis"])
    states = _block_states(conf)
    reps, norms, B = sector_basis(basis.group, states)
    H = _block_hamiltonian(conf, states)
    return reps, norms, B, (B.conj().T @ (H @ B)).toarray()


def _ring(n, particles, sectors, reflect=False):
    perms = [ring_translation(n)] + ([ring_reflection(n)] if reflect else [])
    return with_site_symmetries(spinless_ring(n, particles), perms, sectors)


def _ring_sectors(n, reflect):
    """every one-dimensional representation: momentum k alone, or with the reflection k in {0, n/2} and parity r"""
    if not reflect:
        return [[k] for k in range(n)]
    return [[k, r] for k in ([0, n // 2] if n % 2 == 0 else [0]) for r in (0, 1)]


def _torus(lx, ly, up, down, u=4.0):
    return hubbard(lx * ly, _bonds_torus(lx, ly), u=u, number_up=up, number_down=down)


# ---------------------------------------------------------------------------------------------------------------------
# CPU: U_g, the sign, completeness, refusals

def test_bit_level_u_g_equals_the_jordan_wigner_matrices():
    """u_g (bit by bit) against c†_{image(a)} products of the dense Jordan-Wigner matrices, every element of the
    dihedral group of a 6-site ring and of the spinful 3-site ring (6 modes)"""
    cases = [build_group(6, [{"permutation": ring_translation(6)}, {"permutation": ring_reflection(6)}], 0),
             widen_to_spinful(build_group(3, [{"permutation": ring_translation(3)}, {"permutation": ring_reflection(3)}],
                                          0))]
    states = np.arange(64, dtype=np.uint64)
    for g in cases:
        for p in g.perms:
            img, sgn = u_g(p, states)
            want = sp.csr_matrix((sgn.astype(float), (img.astype(np.int64), states.astype(np.int64))), shape=(64, 64))
            assert abs(u_g_matrix(p) - want).max() == 0, p


def test_u_g_is_a_representation():
    """U_g U_h = U_{gh} on the Fock space for every pair of the dihedral group of an 8-site ring, the spinful 4-site
    ring (8 modes) and the 2 x 3 torus translations (spinless, 6 modes)"""
    groups = [build_group(8, [{"permutation": ring_translation(8)}, {"permutation": ring_reflection(8)}], 0),
              widen_to_spinful(build_group(4, [{"permutation": ring_translation(4)}, {"permutation": ring_reflection(4)}],
                                           0)),
              build_group(6, [{"permutation": p} for p in torus_translations(2, 3)], 0)]
    for g in groups:
        n = g.perms.shape[1]
        states = np.arange(1 << n, dtype=np.uint64)
        for p, q in product(g.perms, repeat=2):
            s1, g1 = u_g(q, states)
            s2, g2 = u_g(p, s1)
            s3, g3 = u_g(_compose(list(p), list(q)), states)
            assert np.array_equal(s2, s3) and np.array_equal(g1 * g2, g3), (p, q)


@pytest.mark.parametrize("name", ["ring_7_3", "ring_8_4", "ring_10_5", "hubbard_chain_8", "hubbard_torus_2x3"])
def test_u_g_commutes_with_the_hamiltonian(name):
    confs = {"ring_7_3": _ring(7, 3, [0], True), "ring_8_4": _ring(8, 4, [0], True), "ring_10_5": _ring(10, 5, [0], True),
             "hubbard_chain_8": with_site_symmetries(hubbard(8, _bonds_ring(8)), [ring_translation(8), ring_reflection(8)]),
             "hubbard_torus_2x3": with_site_symmetries(_torus(2, 3, 3, 2), list(torus_translations(2, 3)))}
    conf = confs[name]
    basis = basis_from_dict(conf["basis"])
    states = _block_states(conf)
    H = _block_hamiltonian(conf, states)
    n = states.shape[0]
    for p in basis.group.perms:
        img, sgn = u_g(p, states)
        U = sp.csr_matrix((sgn.astype(float), (np.searchsorted(states, img), np.arange(n))), shape=(n, n))
        assert abs(U @ H - H @ U).max() < 1e-13, (name, p)


def test_inversion_mask_sign_equals_u_g_up_to_64_bits():
    """symmetry.fermion_signs (the inversion masks the device uses) against u_g for every element, on random states of
    64-site rings (dihedral, 128 elements), spinful 32-site rings (64 bits) and the 4 x 4 torus (translations and point
    group, spinful: 32 bits)"""
    rng = np.random.default_rng(3)
    t44 = torus_translations(4, 4)
    rot = [(3 - i // 4) + 4 * (i % 4) for i in range(16)]
    mir = [(3 - i % 4) + 4 * (i // 4) for i in range(16)]
    groups = [build_group(64, [{"permutation": ring_translation(64)}, {"permutation": ring_reflection(64)}], 0),
              widen_to_spinful(build_group(32, [{"permutation": ring_translation(32)},
                                                {"permutation": ring_reflection(32)}], 0)),
              widen_to_spinful(build_group(16, [{"permutation": p} for p in (*t44, rot, mir)], 0))]
    assert [len(g) for g in groups] == [128, 64, 128]
    for g in groups:
        n = g.perms.shape[1]
        states = rng.integers(0, 2 ** 63, size=400, dtype=np.uint64) * np.uint64(2) + rng.integers(0, 2, size=400,
                                                                                                     dtype=np.uint64)
        if n < 64:
            states &= np.uint64((1 << n) - 1)
        for p in g.perms:
            assert np.array_equal(fermion_signs(p, states), u_g(p, states)[1]), p


COMPLETE = [(f"ring_{n}_{k}", n, k) for n in range(6, 11) for k in range(n + 1)]


@pytest.mark.parametrize("name,n,k", COMPLETE)
def test_momentum_sectors_are_the_block(name, n, k):
    """the n momentum sectors of a spinless ring at k particles: dimensions sum to C(n, k), spectra together are the
    block spectrum"""
    _check_complete([_ring(n, k, [q]) for q in range(n)])


@pytest.mark.parametrize("lx,ly,up,down", [(2, 3, 3, 2), (3, 2, 2, 2), (6, 1, 3, 3)])
def test_hubbard_momentum_sectors_are_the_block(lx, ly, up, down):
    perms = list(torus_translations(lx, ly))
    orders = [lx, ly]
    confs = [with_site_symmetries(_torus(lx, ly, up, down), perms, [a, b]) for a in range(orders[0])
             for b in range(orders[1])]
    _check_complete(confs)


def _check_complete(confs):
    states = _block_states(confs[0])
    H = _block_hamiltonian(confs[0], states).toarray()
    want = np.linalg.eigvalsh(H)
    got, dims = [], 0
    for conf in confs:
        reps, _, B, Hp = _sector(conf)
        dims += reps.shape[0]
        if reps.shape[0]:
            assert abs(B.conj().T @ B - sp.identity(reps.shape[0])).max() < 1e-12
        got.append(np.linalg.eigvalsh(Hp) if reps.shape[0] else np.zeros(0))
    assert dims == states.shape[0]
    assert np.abs(np.sort(np.concatenate(got)) - want).max() < 1e-10


def test_even_particle_rings_have_vanishing_orbits():
    """a spinless ring of 4 sites at 2 particles, momentum 0: the orbit of 0b0101 has stabiliser {1, T²} and
    sign(T², 0b0101) = -1, so its signed sum vanishes and it is not a basis state (a spin basis would keep it)"""
    reps, _, _, _ = _sector(_ring(4, 2, [0]))
    assert 0b0101 not in reps.tolist()
    assert int(fermion_signs(np.array([2, 3, 0, 1]), np.array([0b0101], dtype=np.uint64))[0]) == -1


@pytest.mark.parametrize("basis,message", [
    ({"particle": "spinless-fermion", "number_sites": 4, "number_particles": 2,
      "symmetries": [{"permutation": [1, 2, 3, 0], "sector": 0}]}, "symmetries.*site_symmetries"),
    ({"particle": "spinful-fermion", "number_sites": 2, "number_particles": 2, "number_up": 1,
      "symmetries": [{"permutation": [1, 0, 3, 2], "sector": 0}]}, "site_symmetries"),
    ({"number_spins": 4, "hamming_weight": 2, "site_symmetries": [{"permutation": [1, 2, 3, 0]}]}, "site_symmetries"),
    ({"particle": "spinful-fermion", "number_sites": 4, "number_particles": 4, "number_up": 2,
      "site_symmetries": [{"permutation": [1, 2, 3, 0, 5, 6, 7, 4]}]}, "permutations of the 4 sites"),
    ({"particle": "spinless-fermion", "number_sites": 4, "number_particles": 2,
      "site_symmetries": [{"permutation": [1, 1, 3, 0]}]}, "permutations of the 4 sites"),
])
def test_yaml_refusals(basis, message):
    with pytest.raises(ValueError, match=message):
        basis_from_dict(basis)


def test_yaml_accepts_site_symmetries():
    b = basis_from_dict({"particle": "spinful-fermion", "number_sites": 4, "number_particles": 4, "number_up": 2,
                         "site_symmetries": [{"permutation": [1, 2, 3, 0], "sector": 1}]})
    assert b.has_permutation_symmetries() and b.number_states() is None and b.number_bits == 8
    assert [1, 2, 3, 0, 5, 6, 7, 4] in b.group.perms.tolist()
    assert np.all(b.group.flips == 0) and len(b.group) == 4
    for name in ("spinless_ring_28_symm", "hubbard_chain_8_symm", "hubbard_square_4x4_symm"):
        basis, _ = load_config_from_yaml(os.path.join(DATA, name + ".yaml"))
        assert basis.is_fermionic() and basis.has_permutation_symmetries() and basis.number_states() is None
        assert basis.group.perms.shape[1] == basis.number_bits


def _create(conf=None, bits=8, weight=4, particles=(nat.DMV_SPINFUL_FERMION, 4, 2), perms=None, flips=None,
            chars=None, order=None):
    bd = nat.BasisDesc()
    bd.number_sites, bd.hamming_weight, bd.spin_inversion, bd.has_permutations = bits, weight, 0, 1
    keep = []
    if perms is not None:
        perms = np.ascontiguousarray(perms, dtype=np.int32)
        flips = np.ascontiguousarray(np.zeros(perms.shape[0]) if flips is None else flips, dtype=np.uint8)
        chars = np.ascontiguousarray(np.ones(perms.shape[0]) if chars is None else chars, dtype=np.complex128)
        keep += [perms, flips, chars]
        bd.group_order = perms.shape[0] if order is None else order
        bd.perms, bd.flips, bd.characters = perms.ctypes.data, flips.ctypes.data, chars.ctypes.data
    pd = nat.ParticlesDesc()
    pd.particle_type, pd.number_particles, pd.number_up = particles
    od = nat.OperatorDesc()
    handle = C.c_void_p()
    rc = nat.lib().dmv_context_create_particles(C.byref(bd), C.byref(pd), C.byref(od), 0, 0, 1, C.byref(handle))
    if rc == 0:
        nat.lib().dmv_context_destroy(handle)
    return rc, nat.lib().dmv_last_error().decode()


def test_abi_refusals_before_any_device_work():
    """refused without a GPU: the checks run before the device look-up"""
    ident, shift = list(range(8)), [1, 2, 3, 0, 5, 6, 7, 4]
    rc, msg = _create()
    assert rc != 0 and "permutation symmetries" in msg, msg
    rc, msg = _create(perms=[ident, shift], order=0)
    assert rc != 0 and "permutation symmetries" in msg, msg
    rc, msg = _create(perms=[ident, ident], flips=[0, 1])
    assert rc != 0 and "spin flip" in msg, msg
    for bad in ([1, 2, 3, 0, 4, 5, 6, 7], [1, 2, 3, 0, 6, 7, 4, 5], [4, 5, 6, 7, 0, 1, 2, 3]):
        rc, msg = _create(perms=[ident, bad])
        assert rc != 0 and "both spin halves" in msg, (bad, msg)
    rc, msg = _create(bits=4, weight=2, particles=(nat.DMV_SPINLESS_FERMION, 2, -1), perms=[[0, 1, 2, 3]], flips=[1])
    assert rc != 0 and "spin flip" in msg, msg


# ---------------------------------------------------------------------------------------------------------------------
# GPU

@pytest.fixture(scope="module")
def need_cuda():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _op(conf):
    basis = basis_from_dict(conf["basis"])
    op = Operator(operator_from_dict(conf["hamiltonian"], basis))
    op.basis.build()
    return op


def _real(conf):
    return bool(np.all(basis_from_dict(conf["basis"]).group.characters.imag == 0))


def _check_products(conf, rng, batch=True):
    """representatives, norms and products of every path against the CPU sector; -> the operator (open)"""
    reps, norms, _, Hp = _sector(conf)
    op = _op(conf)
    n = reps.shape[0]
    assert op.basis.numberStates() == n
    assert np.array_equal(op.basis.representatives(), reps)
    if n == 0:
        return op, Hp
    assert np.abs(op.basis.norms() - norms).max() < 1e-14
    scale = max(1.0, np.abs(Hp).max())
    kinds = (np.float64, np.complex128) if _real(conf) else (np.complex128,)
    for mode in (0, 1):
        op.set_option("mode", mode)
        for dtype in kinds:
            x = rng.normal(size=n) + (1j * rng.normal(size=n) if dtype == np.complex128 else 0)
            y = op.matvec(x)
            assert np.abs(y - Hp @ x).max() < 1e-12 * scale * np.abs(x).max() * 8, (mode, dtype)
            # both forms accumulate with floating-point atomics, so a repeat may add in another order: equal to rounding
            assert np.abs(op.matvec(x) - y).max() <= 1e-14 * max(1.0, np.abs(y).max()), (mode, dtype)
            if batch:
                X = rng.normal(size=(3, n)) + (1j * rng.normal(size=(3, n)) if dtype == np.complex128 else 0)
                Y = op.matvec_batch(X)
                assert np.abs(Y - X @ Hp.T).max() < 1e-12 * scale * np.abs(X).max() * 8, (mode, dtype)
    op.set_option("mode", -1)
    return op, Hp


RINGS = [(n, k, reflect) for n in range(6, 13) for k in range(n + 1) for reflect in (False, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("n,k,reflect", RINGS)
def test_ring_sectors_against_the_projected_matrix(need_cuda, n, k, reflect):
    """every sector of spinless rings of 6 to 12 sites at every particle number: translations, and translations with
    the reflection; both product paths, both element types, batches, repeats"""
    rng = np.random.default_rng(100 * n + k)
    dims = 0
    for sec in _ring_sectors(n, reflect):
        op, _ = _check_products(_ring(n, k, sec, reflect), rng, batch=(n % 3 == 0))
        dims += op.basis.numberStates()
        op.close()
    if not reflect:
        assert dims == fp.sector_states(n, k, spinful=False).shape[0]


HUBBARD = {
    "hubbard_chain_8": (with_site_symmetries(hubbard(8, _bonds_ring(8)), [ring_translation(8), ring_reflection(8)]),
                        [[k, r] for k in (0, 4) for r in (0, 1)] + [[k] for k in range(8)]),
    "hubbard_torus_2x3": (_torus(2, 3, 3, 2), [[a, b] for a in range(2) for b in range(3)]),
    "hubbard_torus_3x3": (_torus(3, 3, 5, 4), [[a, b] for a in range(3) for b in range(3)]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(HUBBARD))
def test_hubbard_sectors_against_the_projected_matrix(need_cuda, name):
    conf, sectors = HUBBARD[name]
    rng = np.random.default_rng(11)
    for sec in sectors:
        if len(sec) == 1:   # translations alone
            c = with_site_symmetries(hubbard(8, _bonds_ring(8)), [ring_translation(8)], sec)
        elif name == "hubbard_chain_8":
            c = with_site_symmetries(hubbard(8, _bonds_ring(8)), [ring_translation(8), ring_reflection(8)], sec)
        else:
            lx, ly = (2, 3) if name.endswith("2x3") else (3, 3)
            c = with_site_symmetries(conf, list(torus_translations(lx, ly)), sec)
        op, Hp = _check_products(c, rng)
        n = op.basis.numberStates()
        if n >= 12:   # eigsh per sector against dense eigh
            evals = op.eigsh(2, complex_vectors=not _real(c), eigenvectors=False)[0]
            assert np.abs(evals - np.linalg.eigvalsh(Hp)[:2]).max() < 1e-9 * max(1.0, abs(evals[0])), (name, sec)
        op.close()


@pytest.mark.gpu
def test_state_info_and_zz_correlations(need_cuda):
    """dmv_state_info on random block states against the host reference (representative, conj(χ(g)) sign(g, s) for
    states of non-vanishing orbits, norm), and zz_correlations of a sector vector against the unfolded state B x"""
    rng = np.random.default_rng(5)
    for conf in (with_site_symmetries(hubbard(8, _bonds_ring(8)), [ring_translation(8)], [3]),
                 _ring(10, 4, [0, 1], True), _ring(9, 4, [2])):
        basis = basis_from_dict(conf["basis"])
        g = basis.group
        states = _block_states(conf)
        reps, norms, B, _ = _sector(conf)
        op = _op(conf)
        alphas = rng.choice(states, size=min(300, states.shape[0]), replace=False)
        betas, chars, got_norms = op.basis.stateInfo(alphas)
        imgs, sgns = zip(*(u_g(p, alphas) for p in g.perms))
        imgs, sgns = np.stack(imgs), np.stack(sgns)
        e = imgs.argmin(axis=0)
        cols = np.arange(alphas.shape[0])
        assert np.array_equal(betas, imgs[e, cols])
        want_norm = np.zeros(alphas.shape[0])
        at = np.searchsorted(reps, betas)
        found = (at < reps.shape[0]) & (reps[np.minimum(at, reps.shape[0] - 1)] == betas)
        want_norm[found] = norms[at[found]]
        assert np.abs(got_norms - want_norm).max() < 1e-14
        want_chars = np.conj(g.characters[e]) * sgns[e, cols]
        assert np.abs((chars - want_chars)[found]).max() < 1e-14

        x = rng.normal(size=reps.shape[0]) + 1j * rng.normal(size=reps.shape[0])
        Cz, m = op.zz_correlations(x)
        psi = B @ x
        p = np.abs(psi) ** 2 / np.sum(np.abs(psi) ** 2)
        z = 2.0 * ((states[:, None] >> np.arange(basis.number_bits, dtype=np.uint64)[None, :]) & ONE).astype(float) - 1
        assert np.abs(m - p @ z).max() < 1e-12 and np.abs(Cz - (z.T * p) @ z).max() < 1e-12
        op.close()


@pytest.mark.gpu
def test_projected_fermionic_observables_refuse(need_cuda):
    conf = _ring(8, 3, [1])
    op = _op(conf)
    other = _op(_ring(8, 4, [1]))
    try:
        x = np.ones(op.basis.numberStates(), dtype=np.complex128)
        with pytest.raises(nat.DmvError, match="projected spinless-fermion basis"):
            op.one_body_density_matrix(x)
        with pytest.raises(nat.DmvError, match="projected spinless-fermion basis"):
            op.apply_fermion("c+", np.ones(8), x, other)
        with pytest.raises(nat.DmvError, match="spinless-fermion"):
            op.reduced_density_matrix(x, [0, 1])
        with pytest.raises(nat.DmvError, match="spinless-fermion"):
            op.pm_correlations(x)
    finally:
        op.close()
        other.close()


def _free_fermion_minima(eps: np.ndarray, n_fill: int, period) -> dict:
    """{total momentum (mod period per axis): the least Σ eps over n_fill distinct momenta}; eps indexed by momentum
    tuples of the lattice, period the lattice shape"""
    period = tuple(period)
    # the momenta one by one: table[c] = {total momentum of c chosen ones: least energy}
    ks = list(np.ndindex(*period))
    table = [{(0,) * len(period): 0.0}] + [dict() for _ in range(n_fill)]
    for kv in ks:
        e = float(eps[kv])
        for c in range(min(n_fill, len(ks)) - 1, -1, -1):
            for tot, v in table[c].items():
                t2 = tuple((a + b) % p for a, b, p in zip(tot, kv, period))
                if v + e < table[c + 1].get(t2, np.inf):
                    table[c + 1][t2] = v + e
    return table[n_fill]


@pytest.mark.gpu
def test_spinless_ring_28_every_momentum_against_free_fermions(need_cuda):
    """spinless_ring_28 at 14 particles (about 1.4 M states per sector): the lowest energy of each of the 28 sectors is
    the free-fermion minimum over 14 of the momenta 2πm/28 with Σm ≡ ±sector, to 1e-9 relative.  With the exchange sign
    missing, a translation would not see the string of the bond 27-0, and the sectors would hold the twisted-boundary
    (momenta 2π(m + ½)/28) energies instead: those differ by far more than the tolerance in most sectors."""
    n = 28
    eps = -2.0 * np.cos(2 * np.pi * np.arange(n) / n)
    periodic = _free_fermion_minima(eps, 14, (n,))
    twisted = _free_fermion_minima(-2.0 * np.cos(2 * np.pi * (np.arange(n) + 0.5) / n), 14, (n,))
    assert sum(abs(periodic[(k,)] - min(twisted.values())) > 1e-3 for k in range(n)) >= n // 2
    with open(os.path.join(DATA, "spinless_ring_28_symm.yaml"), encoding="utf-8") as f:
        base = yaml.safe_load(f)
    for k in range(n):
        conf = {"basis": dict(base["basis"]), "hamiltonian": base["hamiltonian"]}
        conf["basis"]["site_symmetries"] = [{"permutation": ring_translation(n), "sector": k}]
        op = _op(conf)
        e, _, _, res = op.lanczos(max_iters=600, tol=1e-12, complex_vectors=k not in (0, n // 2), eigenvector=False)
        want = min(periodic[(k,)], periodic[((-k) % n,)])
        assert abs(e - want) < 1e-9 * abs(want), (k, e, want)
        op.close()


def _torus_conf(u, kx, ky):
    conf = with_site_symmetries(hubbard(16, _bonds_torus(4, 4), u=u), list(torus_translations(4, 4)), [kx, ky])
    return conf


# the six classes of momenta of the 4 x 4 torus under its point group, and a partner of three of them
TORUS_CLASSES = [(0, 0), (1, 0), (1, 1), (2, 0), (2, 1), (2, 2)]
TORUS_PARTNERS = [((1, 0), (0, 3)), ((2, 1), (1, 2)), ((1, 1), (3, 1))]


@pytest.mark.gpu
def test_hubbard_square_4x4_sectors_at_size(need_cuda):
    """hubbard_square_4x4 in translation sectors of about 10.4 M states.  All 16 sectors take several minutes per U, so
    the six momenta inequivalent under the point group are tested, plus three point-group partners:
    U = 0: the lowest energy equals the free-fermion minimum over 8 up and 8 down momenta of matching total momentum;
    U = 4: the minimum over the sectors equals the ground energy of the unsymmetrised 165.6 M-state basis to 1e-8, and
    partners agree.  Sampled rows of one product match a host row reference (fermion_pin.apply_to_states and the
    independent U_g)."""
    eps = np.zeros((4, 4))
    for a, b in np.ndindex(4, 4):
        eps[a, b] = -2.0 * (np.cos(2 * np.pi * a / 4) + np.cos(2 * np.pi * b / 4))
    one = _free_fermion_minima(eps, 8, (4, 4))
    free = {}
    for (ua, ub), eu in one.items():
        for (da, db), ed in one.items():
            key = ((ua + da) % 4, (ub + db) % 4)
            free[key] = min(free.get(key, np.inf), eu + ed)

    def lowest(conf, complex_vectors):
        op = _op(conf)
        e = op.lanczos(max_iters=600, tol=1e-12, complex_vectors=complex_vectors, eigenvector=False)[0]
        op.close()
        return e

    for kx, ky in TORUS_CLASSES:
        e = lowest(_torus_conf(0.0, kx, ky), (kx, ky) not in ((0, 0), (2, 0), (0, 2), (2, 2)))
        want = min(free[(kx, ky)], free[((-kx) % 4, (-ky) % 4)])
        assert abs(e - want) < 1e-9 * abs(want), ((kx, ky), e, want)
    energies = {}
    for k in TORUS_CLASSES + [p for _, p in TORUS_PARTNERS]:
        energies[k] = lowest(_torus_conf(4.0, *k), k not in ((0, 0), (2, 0), (0, 2), (2, 2)))
    for a, b in TORUS_PARTNERS:
        assert abs(energies[a] - energies[b]) < 1e-9 * abs(energies[a]), (a, b, energies[a], energies[b])
    _, full = load_config_from_yaml(os.path.join(DATA, "hubbard_square_4x4.yaml"))
    op = Operator(full)
    op.basis.build()
    e_full = op.lanczos(max_iters=600, tol=1e-12, eigenvector=False)[0]
    op.close()
    e_min = min(energies.values())
    assert abs(e_min - e_full) < 1e-8 * abs(e_full), (e_min, e_full, energies)

    # sampled rows of one product in the sector (1, 0)
    conf = _torus_conf(4.0, 1, 0)
    basis = basis_from_dict(conf["basis"])
    g = basis.group
    op = _op(conf)
    reps, norms = op.basis.representatives(), op.basis.norms()
    rng = np.random.default_rng(9)
    x = rng.normal(size=reps.shape[0]) + 1j * rng.normal(size=reps.shape[0])
    y = op.matvec(x)
    op.close()
    N = 16
    for i in rng.choice(reps.shape[0], size=64, replace=False):
        r = int(reps[i])
        targets = {r}
        for a, b in _bonds_torus(4, 4):
            for off in (0, N):
                m = (1 << (a + off)) | (1 << (b + off))
                if bin(r & m).count("1") == 1:
                    targets.add(r ^ m)
        targets = np.array(sorted(targets), dtype=np.uint64)
        col = fp.apply_to_states(_terms(conf), N, True, np.array([r], dtype=np.uint64), targets).toarray()[:, 0]
        acc = 0j
        for t, h in zip(targets, col):
            if h == 0:
                continue
            imgs, sgns = zip(*(u_g(p, np.array([t], dtype=np.uint64)) for p in g.perms))
            imgs = np.array([v[0] for v in imgs])
            e = int(imgs.argmin())
            j = int(np.searchsorted(reps, imgs[e]))
            if j >= reps.shape[0] or reps[j] != imgs[e]:
                continue   # an orbit without basis state: its component of the projected state is 0
            acc += np.conj(h) * sgns[e][0] * g.characters[e] * norms[j] * x[j]
        want = acc / norms[i]
        assert abs(y[i] - want) < 1e-11 * max(1.0, abs(want)), (i, y[i], want)


@pytest.mark.gpu
def test_two_ranks_against_one_rank(need_cuda):
    """Products and eigsh of fermionic sectors on two ranks against one rank (tools/fermion_symmetry_check.py)."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--standalone",
           os.path.join(ROOT, "tools", "fermion_symmetry_check.py")]
    out = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
    lines = [l for l in out.stdout.splitlines() if l.rstrip().endswith(("OK", "FAIL"))]
    assert out.returncode == 0 and len(lines) >= 9 and not any(l.rstrip().endswith("FAIL") for l in lines), \
        out.stdout[-4000:] + out.stderr[-2000:]
