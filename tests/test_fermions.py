"""Fermionic bases: spinless and spinful (Hubbard) models with Jordan-Wigner strings as sign masks.

Without a GPU: the compiled monomials against the dense Jordan-Wigner matrices of tests/fermion_pin.py through the C
oracle, the canonical anticommutators, spin inputs unchanged, every refusal, the basis layout and exact pins (two-site
Hubbard, atomic limit, free fermions, the attractive-repulsive mapping, spinless ring = XX ring).
On the GPU: products against the oracle at every kernel, index, split and rank count; eigenvalues at size.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as sla

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import fermion_pin as fp  # noqa: E402
import torch  # noqa: E402
from distributed_matvec_b200 import Operator  # noqa: E402
from distributed_matvec_b200 import _native as nat  # noqa: E402
from distributed_matvec_b200.config import (BasisSpec, OperatorSpec, basis_from_dict, load_config_from_yaml,  # noqa: E402
                                            operator_from_dict)
from distributed_matvec_b200.expr import FermionModes, compile_terms, parse_expression  # noqa: E402
from oracle import pyoracle as po  # noqa: E402

DATA = os.path.join(ROOT, "data")
sys.path.insert(0, os.path.join(ROOT, "tools"))
from gen_models import _bonds_ring, _bonds_torus, hubbard, spinless_ring  # noqa: E402

INDEX_LIN, INDEX_LIN_SPLIT = 3, 4


def _model(conf):
    basis = basis_from_dict(conf["basis"])
    return basis, operator_from_dict(conf["hamiltonian"], basis)


def _table_matrix(op: OperatorSpec, states: np.ndarray) -> sp.csr_matrix:
    """<β|H|α> over the ascending `states` from the compiled tables, applied term by term by the C oracle."""
    states = np.ascontiguousarray(states, dtype=np.uint64)
    n = states.shape[0]
    betas, coeffs, offsets = po.apply_off_diag(op, states)
    cols = np.repeat(np.arange(n), np.diff(offsets))
    rows = np.minimum(np.searchsorted(states, betas), n - 1)
    assert np.array_equal(states[rows], betas), "a term leaves the block"
    H = sp.coo_matrix((coeffs, (rows, cols)), shape=(n, n)).tocsr()
    return (H + sp.diags(po.apply_diag(op, states, np.ones(n, dtype=np.complex128)))).tocsr()


def _diff(a, b) -> float:
    d = a - b
    d = d.toarray() if hasattr(d, "toarray") else np.asarray(d)
    return float(np.abs(d).max()) if d.size else 0.0


def _spec(basis: BasisSpec, terms) -> OperatorSpec:
    off, diag = compile_terms(terms, basis.number_sites, basis.fermion_modes())
    return OperatorSpec(basis=basis, off_diag=off, diag=diag)


def _spinless(n, number_particles=None):
    return basis_from_dict({"particle": "spinless-fermion", "number_sites": n, "number_particles": number_particles})


# ---------------------------------------------------------------------------------------------------------------------
# compile: monomials, anticommutators, spin inputs

_OPS = {"c+": "c†", "c": "c", "n": "n"}


def test_random_monomials_equal_the_dense_jordan_wigner_matrix():
    """Every monomial of 1 to 4 operators (repeated modes included) on random modes of a 10-mode system: the compiled
    terms applied by the C oracle equal the product of the Jordan-Wigner matrices to 1e-14."""
    rng = np.random.default_rng(7)
    n = 10
    basis = _spinless(n)
    states = np.arange(1 << n, dtype=np.uint64)
    for trial in range(120):
        length = int(rng.integers(1, 5))
        kinds = [str(rng.choice(["c+", "c", "n"])) for _ in range(length)]
        modes = [int(m) for m in rng.integers(0, n, size=length)]
        distinct = sorted(set(modes), key=modes.index)
        place = {m: p for p, m in enumerate(distinct)}
        coeff = complex(rng.normal(), rng.normal())
        expr = f"({coeff.real!r}+{coeff.imag!r}j)"
        text = " ".join(f"{_OPS[k]}{place[m]}" for k, m in zip(kinds, modes))
        terms = [{"expression": f"{coeff.real!r} × {text} + {coeff.imag!r}j × {text}", "sites": [distinct]}]
        got = _table_matrix(_spec(basis, terms), states)
        want = coeff * fp.monomial(n, list(zip(kinds, modes)))
        assert _diff(got, want) < 1e-14, (trial, expr, text, distinct)


def test_anticommutators_on_the_compiled_tables():
    """{c_a, c†_b} = δ_ab and {c_a, c_b} = 0 on 8 modes, from the compiled tables."""
    n = 8
    basis = _spinless(n)
    states = np.arange(1 << n, dtype=np.uint64)
    eye = np.eye(1 << n)
    for a in range(n):
        for b in range(n):
            if a == b:
                mixed = [{"expression": "c₀ c†₀ + c†₀ c₀", "sites": [[a]]}]
                same = [{"expression": "c₀ c₀ + c₀ c₀", "sites": [[a]]}]
            else:
                mixed = [{"expression": "c₀ c†₁ + c†₁ c₀", "sites": [[a, b]]}]
                same = [{"expression": "c₀ c₁ + c₁ c₀", "sites": [[a, b]]}]
            assert _diff(_table_matrix(_spec(basis, mixed), states), eye if a == b else 0 * eye) < 1e-15, (a, b)
            op = _spec(basis, same)
            assert len(op.off_diag) == 0 and len(op.diag) == 0, (a, b)


# sha256 (first 16 hex digits) of every spin model's term tables as compiled before fermionic bases existed
SPIN_TABLES = {
    'heisenberg_chain_10': '481f6ccfaaf17365', 'heisenberg_chain_12': '69048ca951c7260d',
    'heisenberg_chain_16': 'd54dac3211a26d77', 'heisenberg_chain_20': '2ba88ec763e6ab98',
    'heisenberg_chain_24': 'c87b54cddf7ac3ae', 'heisenberg_chain_24_symm': 'c87b54cddf7ac3ae',
    'heisenberg_chain_28': 'f47f5cd698e9dca2', 'heisenberg_chain_30': 'd558aca35e7bb629',
    'heisenberg_chain_32': 'fa8eefd407be79c9', 'heisenberg_chain_32_symm': 'fa8eefd407be79c9',
    'heisenberg_chain_36_symm': '889448b97981dcc9', 'heisenberg_chain_4': 'a42923d221732e1d',
    'heisenberg_chain_40_symm': '86d01c0d92fbd920', 'heisenberg_chain_6': 'a7e86abfa5bc164e',
    'heisenberg_chain_8': '0a93edb7b2445188', 'heisenberg_kagome_12': '3d83ece17f902d07',
    'heisenberg_kagome_12_symm': '36d1ea62c7f741da', 'heisenberg_kagome_16': '1284c125d9bf1642',
    'heisenberg_square_4x4': '65866e15fef2a7d5', 'heisenberg_square_5x5': '21f7ef067126c11a',
    'heisenberg_square_6x6': 'd06c9f4de006e7e4', 'issue_01': '00f38e5e548dac8b',
}


def test_spin_models_compile_to_the_same_tables():
    import hashlib
    for name, digest in SPIN_TABLES.items():
        basis, op = load_config_from_yaml(os.path.join(DATA, name + ".yaml"))
        assert basis.particle_type == "spin-1/2" and basis.number_bits == basis.number_sites
        h = hashlib.sha256()
        for t in (op.off_diag, op.diag):
            for a in (t.v, t.m, t.r, t.x, t.s):
                h.update(a.tobytes())
        assert h.hexdigest()[:16] == digest, name


def test_hopping_groups_share_one_sign_mask():
    """Each hop and its conjugate: one flip mask, one string (the bits strictly between the two modes)."""
    _, op = load_config_from_yaml(os.path.join(DATA, "hubbard_square_4x4.yaml"))
    off = op.off_diag
    for x in np.unique(off.x):
        sel = off.x == x
        bits = [b for b in range(64) if (int(x) >> b) & 1]
        lo, hi = bits[0], bits[-1]
        between = ((1 << hi) - 1) & ~((1 << (lo + 1)) - 1)
        assert set(off.s[sel].tolist()) == {between}, hex(int(x))


# ---------------------------------------------------------------------------------------------------------------------
# refusals

@pytest.mark.parametrize("basis,message", [
    ({"particle": "majorana", "number_sites": 4}, "unknown particle type"),
    ({"particle": "spinful-fermion", "number_sites": 4, "number_particles": 4}, "both number_particles and number_up"),
    ({"particle": "spinful-fermion", "number_sites": 4, "number_particles": 4, "number_up": 5}, "number_up"),
    ({"particle": "spinful-fermion", "number_sites": 4, "number_particles": 9, "number_up": 4}, "number_up"),
    ({"particle": "spinful-fermion", "number_sites": 33, "number_particles": 2, "number_up": 1}, "between 1 and 32"),
    ({"particle": "spinless-fermion", "number_sites": 4, "number_particles": 5}, "number_particles"),
    ({"particle": "spinless-fermion", "number_sites": 4, "hamming_weight": 2}, "hamming_weight"),
    ({"particle": "spinless-fermion", "number_sites": 4, "spin_inversion": 1}, "spin_inversion"),
    ({"particle": "spinful-fermion", "number_sites": 2, "number_particles": 2, "number_up": 1,
      "symmetries": [{"permutation": [1, 0], "sector": 0}]}, "symmetries"),
])
def test_basis_refusals(basis, message):
    with pytest.raises(ValueError, match=message):
        basis_from_dict(basis)


def test_expression_refusals():
    with pytest.raises(ValueError, match="mixed"):
        parse_expression("σᶻ₀ n₀")
    spinful = basis_from_dict({"particle": "spinful-fermion", "number_sites": 2, "number_particles": 2, "number_up": 1})
    with pytest.raises(ValueError, match="spin arrow"):
        _spec(spinful, [{"expression": "c†₀ c₁", "sites": [[0, 1]]}])
    with pytest.raises(ValueError, match="spin arrow"):
        _spec(_spinless(2), [{"expression": "c†₀↑ c₁↑", "sites": [[0, 1]]}])
    with pytest.raises(ValueError, match="fermionic basis"):
        _spec(_spinless(2), [{"expression": "σᶻ₀ σᶻ₁", "sites": [[0, 1]]}])
    spin = basis_from_dict({"number_spins": 2})
    with pytest.raises(ValueError, match="fermionic basis"):
        _spec(spin, [{"expression": "c†₀ c₁", "sites": [[0, 1]]}])
    with pytest.raises(ValueError, match="matrix terms"):
        _spec(_spinless(2), [{"matrix": [[1, 0], [0, 1]], "sites": [[0]]}])
    # the arrow may stand before or after the index
    a = _spec(spinful, [{"expression": "c†₀↑ c₁↓ + n↓₀", "sites": [[0, 1]]}])
    b = _spec(spinful, [{"expression": "c†↑₀ c↓₁ + n₀↓", "sites": [[0, 1]]}])
    for ta, tb in ((a.off_diag, b.off_diag), (a.diag, b.diag)):
        for u, v in zip((ta.v, ta.m, ta.r, ta.x, ta.s), (tb.v, tb.m, tb.r, tb.x, tb.s)):
            assert np.array_equal(u, v)


def _create(bits, weight, particles, inversion=0, permutations=0):
    bd = nat.BasisDesc()
    bd.number_sites, bd.hamming_weight, bd.spin_inversion, bd.has_permutations = bits, weight, inversion, permutations
    pd = nat.ParticlesDesc()
    pd.particle_type, pd.number_particles, pd.number_up = particles
    od = nat.OperatorDesc()
    handle = C.c_void_p()
    rc = nat.lib().dmv_context_create_particles(C.byref(bd), C.byref(pd), C.byref(od), 0, 0, 1, C.byref(handle))
    return rc, nat.lib().dmv_last_error().decode()


@pytest.mark.parametrize("args,message", [
    ((8, 4, (nat.DMV_SPINFUL_FERMION, 4, 2), 1, 0), "spin inversion are not supported"),
    ((8, 4, (nat.DMV_SPINFUL_FERMION, 4, 2), 0, 1), "permutation symmetries"),
    ((9, 4, (nat.DMV_SPINFUL_FERMION, 4, 2)), "must be even"),
    ((8, 4, (nat.DMV_SPINFUL_FERMION, 4, 5)), "number_up"),
    ((8, 6, (nat.DMV_SPINFUL_FERMION, 6, 1)), "number_particles - number_up"),
    ((8, 4, (nat.DMV_SPINFUL_FERMION, 3, 1)), "must equal number_particles"),
    ((8, 9, (nat.DMV_SPINLESS_FERMION, 9, -1)), "number_particles must be -1"),
    ((8, 4, (7, 4, 2)), "particle_type must be"),
])
def test_context_refusals_before_any_device_work(args, message):
    """dmv_context_create_particles checks its input before it looks for a device or allocates."""
    rc, err = _create(*args)
    assert rc != 0 and message in err, err


# ---------------------------------------------------------------------------------------------------------------------
# basis layout

def test_spinful_dimension_and_layout():
    for n, up, down in ((4, 2, 2), (6, 1, 4), (5, 0, 3), (8, 4, 4)):
        basis = basis_from_dict({"particle": "spinful-fermion", "number_sites": n, "number_particles": up + down,
                                 "number_up": up})
        assert basis.number_bits == 2 * n
        assert basis.number_states() == math.comb(n, up) * math.comb(n, down)
        states = fp.sector_states(n, up, down)
        assert np.all(np.diff(states.astype(np.int64)) > 0)
        assert states[0] == basis.min_state_estimate() and states[-1] == basis.max_state_estimate()
        mask = (1 << n) - 1
        assert all(bin(int(s) & mask).count("1") == up and bin(int(s) >> n).count("1") == down for s in states)


# ---------------------------------------------------------------------------------------------------------------------
# exact pins on the Jordan-Wigner sector matrices

def _lowest(H):
    if H.shape[0] <= 400:
        return np.linalg.eigvalsh(H.toarray())[:1]
    return np.sort(sla.eigsh(H, k=1, which="SA", tol=1e-13)[0])


def _hubbard_sector(n, bonds, t, u, up, down):
    conf = hubbard(n, bonds, t=t, u=u, number_up=up, number_down=down)
    states = fp.sector_states(n, up, down)
    H_jw = fp.sector_hamiltonian(conf["hamiltonian"]["terms"], n, True, states)
    _, op = _model(conf)
    assert _diff(_table_matrix(op, states), H_jw) < 1e-13   # the compiled tables agree
    return H_jw


def _free_levels(n, bonds, t):
    T = np.zeros((n, n))
    for i, j in bonds:
        T[i, j] -= t
        T[j, i] -= t
    return np.linalg.eigvalsh(T)


def test_two_site_hubbard():
    for u in (0.5, 4.0, 10.0):
        e0 = _lowest(_hubbard_sector(2, [[0, 1]], 1.0, u, 1, 1))[0]
        assert abs(e0 - (u - math.sqrt(u * u + 16.0)) / 2) < 1e-12, u


def test_atomic_limit():
    for n, up, down in ((4, 2, 3), (4, 3, 3), (5, 1, 2)):
        e0 = _lowest(_hubbard_sector(n, _bonds_ring(n), 0.0, 3.0, up, down))[0]
        assert abs(e0 - 3.0 * max(0, up + down - n)) < 1e-12


@pytest.mark.parametrize("lattice", ["ring_5", "ring_6", "torus_2x3", "torus_2x4"])
def test_free_fermions(lattice):
    n, bonds = {"ring_5": (5, _bonds_ring(5)), "ring_6": (6, _bonds_ring(6)),
                "torus_2x3": (6, _bonds_torus(2, 3)), "torus_2x4": (8, _bonds_torus(2, 4))}[lattice]
    levels = _free_levels(n, bonds, 1.0)
    for up, down in ((n // 2, n // 2), (1, n // 2 + 1), (2, 1)):
        e0 = _lowest(_hubbard_sector(n, bonds, 1.0, 0.0, up, down))[0]
        assert abs(e0 - levels[:up].sum() - levels[:down].sum()) < 1e-11, (lattice, up, down)


@pytest.mark.parametrize("lattice", ["ring_6", "torus_2x4"])
def test_attractive_repulsive_mapping(lattice):
    n, bonds = {"ring_6": (6, _bonds_ring(6)), "torus_2x4": (8, _bonds_torus(2, 4))}[lattice]
    for u, up, down in ((4.0, 3, 2), (2.5, 2, 5), (4.0, n // 2, n // 2)):
        lhs = _lowest(_hubbard_sector(n, bonds, 1.0, u, up, down))[0]
        rhs = _lowest(_hubbard_sector(n, bonds, 1.0, -u, up, n - down))[0] + u * up
        assert abs(lhs - rhs) < 1e-11, (lattice, u, up, down)


def _xx_ring(n, weight, t, flip_wrap):
    basis = basis_from_dict({"number_spins": n, "hamming_weight": weight})
    terms = []
    for i, j in _bonds_ring(n):
        c = -t / 2 * (-1.0 if (flip_wrap and j == 0) else 1.0)
        terms.append({"expression": f"{c!r} × σˣ₀ σˣ₁ + {c!r} × σʸ₀ σʸ₁", "sites": [[i, j]]})
    return basis, _spec(basis, terms)


def test_spinless_ring_equals_the_xx_ring():
    """-t Σ (c†c + h.c.) on a ring: for odd N_f the spectrum of the periodic XX ring at weight N_f, for even N_f that of
    the ring with the wrap bond's sign flipped."""
    n = 9
    for nf in (2, 3, 4, 5):
        conf = spinless_ring(n, nf)
        states = fp.sector_states(n, nf, spinful=False)
        H = fp.sector_hamiltonian(conf["hamiltonian"]["terms"], n, False, states)
        _, op = _model(conf)
        assert _diff(_table_matrix(op, states), H) < 1e-13
        _, xx = _xx_ring(n, nf, 1.0, flip_wrap=nf % 2 == 0)
        spectrum = np.linalg.eigvalsh(H.toarray())
        assert np.abs(spectrum - np.linalg.eigvalsh(_table_matrix(xx, states).toarray())).max() < 1e-12
        assert abs(spectrum[0] - np.sort(-2 * np.cos(2 * np.pi * np.arange(n) / n))[:nf].sum()) < 1e-12


# =====================================================================================================================
# GPU


@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _close(y, y_ref, tol=1e-12):
    return np.abs(y - y_ref).max() <= tol * max(1.0, np.abs(y_ref).max())


def _x(n, cplx, seed=3):
    rng = np.random.default_rng(seed)
    x = rng.random(n) - 0.5
    return x + 1j * (rng.random(n) - 0.5) if cplx else x


def _peierls_chain(n, phi):
    """Hubbard ring with the hop -t e^{iφ} c†_i c_i+1 + h.c."""
    c, s = math.cos(phi), math.sin(phi)
    conf = hubbard(n, _bonds_ring(n), number_up=n // 2, number_down=n // 2)
    conf["hamiltonian"]["terms"][0]["expression"] = " ".join(
        f"- {c!r} × c†₀{a} c₁{a} - {s!r}j × c†₀{a} c₁{a} - {c!r} × c†₁{a} c₀{a} + {s!r}j × c†₁{a} c₀{a}" for a in "↑↓")
    return conf


def _vn_ring(n, nf):
    conf = spinless_ring(n, nf)
    conf["hamiltonian"]["terms"].append({"expression": "1.5 × n₀ n₁", "sites": _bonds_ring(n)})
    return conf


def _anisotropic_torus_3x4(tx=1.0, ty=0.5, u=4.0):
    """Hubbard 3 x 4 torus with hops tx along x and ty along y: a real coefficient table that is not uniform (the LUT
    build of k_gather), 48 flip-mask groups (wide rows)."""
    bonds = _bonds_torus(3, 4)   # x and y bonds alternate
    conf = hubbard(12, bonds, u=u, number_up=3, number_down=3)
    hop = "-{t} × c†₀↑ c₁↑ - {t} × c†₁↑ c₀↑ - {t} × c†₀↓ c₁↓ - {t} × c†₁↓ c₀↓"
    conf["hamiltonian"]["terms"][0] = {"expression": hop.format(t=tx), "sites": bonds[0::2]}
    conf["hamiltonian"]["terms"].append({"expression": hop.format(t=ty), "sites": bonds[1::2]})
    return conf


GPU_MODELS = {
    "hubbard_chain_8": (lambda: load_config_from_yaml(os.path.join(DATA, "hubbard_chain_8.yaml")), INDEX_LIN_SPLIT),
    "hubbard_torus_2x4": (lambda: _model(hubbard(8, _bonds_torus(2, 4))), INDEX_LIN_SPLIT),
    "hubbard_torus_3x4": (lambda: _model(hubbard(12, _bonds_torus(3, 4), number_up=3, number_down=3)), INDEX_LIN_SPLIT),
    "hubbard_torus_3x4_anisotropic": (lambda: _model(_anisotropic_torus_3x4()), INDEX_LIN_SPLIT),
    "spinless_ring_16_v": (lambda: _model(_vn_ring(16, 7)), INDEX_LIN),
    "peierls_chain_6": (lambda: _model(_peierls_chain(6, 0.3)), INDEX_LIN_SPLIT),
}


def _expected_states(basis):
    if basis.particle_type == "spinful-fermion":
        return fp.sector_states(basis.number_sites, basis.number_up, basis.number_particles - basis.number_up)
    return fp.sector_states(basis.number_sites, basis.number_particles, spinful=False)


def _dev(op, x):
    y = op.matvec(torch.from_numpy(x).cuda())
    torch.cuda.synchronize()
    return y.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GPU_MODELS))
def test_fermion_products_against_the_oracle(need_cuda, name):
    """k_gather with sign masks at every split, the directory index, k_pull and the scatter form, host and device
    vectors and matvec_batch, both element types: the oracle's product; repeated products are bit-identical."""
    load, index_mode = GPU_MODELS[name]
    basis, matrix = load()
    reps = _expected_states(basis)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        assert op.info("particle_type") == {"spinless-fermion": 1, "spinful-fermion": 2}[basis.particle_type]
        assert (op.info("gather"), op.info("gather_signs"), op.info("index_mode")) == (1, 1, index_mode)
        for cplx in ((True,) if not matrix.is_real() else (False, True)):
            x = _x(reps.shape[0], cplx)
            y_ref = po.matvec_global(matrix, reps, x, 1)
            for index in (-1, 0):
                op.set_option("index", index)
                assert op.info("index_mode") == (index_mode if index == -1 else 0)
                for split in (-1, 1, 2, 4, 8, 16, 32):
                    op.set_option("gather_split", split)
                    y = _dev(op, x)
                    where = (name, cplx, index, split)
                    assert op.info("gather") == 1, where
                    assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
                    assert np.array_equal(_dev(op, x), y), where
                    assert np.array_equal(op.matvec(x), y), where
                op.set_option("gather_split", -1)
                X = np.stack([_x(reps.shape[0], cplx, 50 + j) for j in range(4)])
                Y = op.matvec_batch(torch.from_numpy(X.copy()).cuda())
                torch.cuda.synchronize()
                for j in range(4):
                    assert _close(Y[j].cpu().numpy(), po.matvec_global(matrix, reps, X[j], 1)), (name, cplx, index, j)
                for opt, pull in (({"mode": 1, "gather": 0}, 1), ({"mode": 0}, 0)):   # k_pull, the scatter form
                    for k, v in opt.items():
                        op.set_option(k, v)
                    assert (op.info("gather"), op.info("pull")) == (0, pull)
                    assert _close(_dev(op, x), y_ref), (name, cplx, index, opt)
                    for k in opt:
                        op.set_option(k, -1)
            op.set_option("index", -1)
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("num_ranks", [2, 3])
@pytest.mark.parametrize("name", ["hubbard_chain_8", "hubbard_torus_2x4", "hubbard_torus_3x4_anisotropic",
                                  "peierls_chain_6", "spinless_ring_16_v"])
def test_fermion_products_on_several_ranks(need_cuda, name, num_ranks):
    """Records (k_generate, exchanges) and the replicated-x form (k_gather with signs on the whole-basis twin) on P
    logical ranks against the oracle's P-rank product."""
    from distributed_matvec_b200 import EmulatedCluster, block_to_hashed, hashed_to_block
    basis, matrix = GPU_MODELS[name][0]()
    reps = _expected_states(basis)
    masks, blocks = po.partition_by_hash(reps, num_ranks)
    cl = EmulatedCluster(matrix, num_ranks).build()
    try:
        for r, op in enumerate(cl.ops):
            assert np.array_equal(op.basis.representatives(), blocks[r])
        for cplx in ((True,) if not matrix.is_real() else (False, True)):
            x = _x(reps.shape[0], cplx, 31)
            y_ref = po.matvec_global(matrix, reps, x, num_ranks)
            xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, num_ranks)]
            y = hashed_to_block([t.cpu().numpy() for t in cl.matvec(xb)], masks)
            assert _close(y, y_ref), (name, num_ranks, cplx, "records")
            y = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)
            assert _close(y, y_ref), (name, num_ranks, cplx, "replicated")
            assert all(op.info("global.gather") == 1 and op.info("global.gather_signs") == 1 for op in cl.ops)
    finally:
        cl.close()


@pytest.mark.gpu
def test_fermion_observables_and_errors(need_cuda):
    """zz_correlations over the bits against the dense pin's density correlations; the spin-only observables refuse;
    c†↑ c↓ leaves the basis and is reported."""
    conf = hubbard(4, _bonds_ring(4), number_up=2, number_down=1)
    basis, matrix = _model(conf)
    states = fp.sector_states(4, 2, 1)
    op = Operator(matrix)
    try:
        op.basis.build()
        x = _x(states.shape[0], False, 5)
        Cz, m = op.zz_correlations(x)
        bits = ((states[:, None] >> np.arange(8, dtype=np.uint64)[None, :]) & np.uint64(1)).astype(float)
        sz = 2 * bits - 1
        w = x * x / (x @ x)
        assert np.abs(Cz - (sz * w[:, None]).T @ sz).max() < 1e-12
        assert np.abs(m - w @ sz).max() < 1e-12
        with pytest.raises(nat.DmvError, match="spinful-fermion"):
            op.pm_correlations(x)
        with pytest.raises(nat.DmvError, match="spinful-fermion"):
            op.reduced_density_matrix(x, [0, 1])
        with pytest.raises(nat.DmvError, match="spinful-fermion"):
            op.apply_spin("z", np.ones(8), x, op)
        # a state with the right total weight but 1 up and 2 down particles
        wrong = np.sort(np.append(states[:-1], np.uint64((0b11 << 4) | 0b1)))
        with pytest.raises(nat.DmvError, match="does not have 2 up and 1 down particles"):
            op.basis.uncheckedSetRepresentatives(wrong)
        assert np.array_equal(op.basis.representatives(), states)   # refused before anything was installed
    finally:
        op.close()
    conf["hamiltonian"]["terms"].append({"expression": "c†₀↑ c₀↓ + c†₀↓ c₀↑", "sites": [[0]]})
    basis, matrix = _model(conf)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert op.info("index_mode") == INDEX_LIN_SPLIT
        for opts in ({}, {"index": 0}, {"mode": 1, "gather": 0}, {"index": 0, "mode": 1, "gather": 0}, {"mode": 0}):
            for k, v in opts.items():
                op.set_option(k, v)
            with pytest.raises(nat.DmvError, match="invalid index"):
                op.matvec(_x(states.shape[0], False))
                op.synchronize()
            for k in opts:
                op.set_option(k, -1)
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("nf", [13, 14])
def test_spinless_ring_28_at_size(need_cuda, nf):
    """28 sites at 13 (37.4 M states) and 14 (40.1 M) particles: the lowest eigenvalue is -2t Σ cos k over the
    occupied momenta, and that of the XX ring through the spin path (periodic for odd N_f, wrap bond flipped for even)."""
    basis, matrix = _model(spinless_ring(28, nf))
    n = 28
    exact = np.sort(-2 * np.cos(2 * np.pi * np.arange(n) / n))[:nf].sum()
    op = Operator(matrix)
    try:
        op.basis.build()
        assert op.basis.numberStates() == math.comb(28, nf)
        assert op.info("gather") == 1 and op.info("gather_signs") == 1
        evals, _, _, conv, _, _ = op.eigsh(1, tol=1e-12, eigenvectors=False)
        assert conv >= 1 and abs(evals[0] - exact) < 1e-10 * abs(exact), (evals[0], exact)
    finally:
        op.close()
    _, xx = _xx_ring(n, nf, 1.0, flip_wrap=nf % 2 == 0)
    op = Operator(xx)
    try:
        op.basis.build()
        evals_xx, _, _, conv, _, _ = op.eigsh(1, tol=1e-12, eigenvectors=False)
        assert conv >= 1 and abs(evals_xx[0] - evals[0]) < 1e-10 * abs(exact)
    finally:
        op.close()


@pytest.mark.gpu
def test_hubbard_4x4_at_size(need_cuda):
    """4 x 4 torus at half filling (165 636 900 states): sampled rows of one product against the oracle; E0 = -24t at
    U = 0, and E0(4) = E0(-4) + 32 from two runs of the device solver."""
    rng = np.random.default_rng(11)
    energies = {}
    for u in (0.0, 4.0, -4.0):
        basis, matrix = _model(hubbard(16, _bonds_torus(4, 4), u=u))
        op = Operator(matrix)
        try:
            op.basis.build()
            assert op.basis.numberStates() == 165636900
            assert (op.info("gather"), op.info("gather_signs"), op.info("index_mode")) == (1, 1, INDEX_LIN_SPLIT)
            if u == 4.0:
                reps = op.basis.representatives()
                x = rng.random(reps.shape[0]) - 0.5
                y = op.matvec(torch.from_numpy(x).cuda()).cpu().numpy()
                rows = np.sort(rng.choice(reps.shape[0], 2000, replace=False))
                want = po.expected_rows(matrix, reps, x, rows)
                assert _close(y[rows], want), np.abs(y[rows] - want).max()
                del reps, x, y
            e, _, it, res = op.lanczos(max_iters=600, tol=1e-11, eigenvector=False)
            energies[u] = e
        finally:
            op.close()
    assert abs(energies[0.0] + 24.0) < 1e-9 * 24.0, energies
    assert abs(energies[4.0] - (energies[-4.0] + 32.0)) < 1e-9 * abs(energies[4.0]), energies



@pytest.mark.gpu
def test_sign_masks_with_spin_inversion_keep_to_the_queued_kernels(need_cuda):
    """A spin basis with spin inversion and an operator whose groups carry sign masks outside their supports (hops
    σ⁺ᵢ Zᵢ₊₁ Zᵢ₊₂ σ⁻ᵢ₊₃ + h.c., which commute with the global flip): k_gather has no build for both, so the product runs
    through k_pull / k_generate as before, on one rank and through the replicated-x twin, and equals the oracle's."""
    from distributed_matvec_b200 import EmulatedCluster, block_to_hashed, hashed_to_block
    from distributed_matvec_b200.expr import TermTable, fermion_monomial_terms
    n = 10
    basis = basis_from_dict({"number_spins": n, "hamming_weight": n // 2, "spin_inversion": 1})
    rows = []
    for i in range(n - 3):
        rows += fermion_monomial_terms(-1.0, [("c+", i), ("c", i + 3)])
        rows += fermion_monomial_terms(-1.0, [("c+", i + 3), ("c", i)])
    off = TermTable(*(np.array([r[k] for r in rows], dtype=np.complex128 if k == 0 else np.uint64) for k in range(5)))
    assert np.all(off.s != 0)
    _, diag = compile_terms([{"expression": "0.7 × σᶻ₀ σᶻ₁", "sites": _bonds_ring(n)}], n)
    matrix = OperatorSpec(basis=basis, off_diag=off, diag=diag)
    reps, _ = po.enumerate_states(basis)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        assert (op.info("gather"), op.info("gather_signs")) == (0, 0)
        for cplx in (False, True):
            x = _x(reps.shape[0], cplx)
            y_ref = po.matvec_global(matrix, reps, x, 1)
            for opts in ({}, {"mode": 1}, {"mode": 0}):
                for k, v in opts.items():
                    op.set_option(k, v)
                assert op.info("gather") == 0
                assert _close(_dev(op, x), y_ref), (cplx, opts)
                for k in opts:
                    op.set_option(k, -1)
    finally:
        op.close()
    masks, _ = po.partition_by_hash(reps, 2)
    cl = EmulatedCluster(matrix, 2).build()
    try:
        x = _x(reps.shape[0], False, 31)
        xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, 2)]
        y_ref = po.matvec_global(matrix, reps, x, 2)
        y = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)
        assert _close(y, y_ref)
        assert all(op.info("global.gather") == 0 for op in cl.ops)
    finally:
        cl.close()
