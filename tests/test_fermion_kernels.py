"""Every sign-mask build of k_gather, and fermionic bases past 32 bits, against a bit-level Jordan-Wigner reference.

k_gather multiplies each emitted term of a fermionic operator by (-1)^popc(b & s_out) (SG = 1): 64 instances
(CV, CE, NARROW, LIN, UNI, KB) -- complex coefficients, complex vectors, 32-bit rows, Lin-table index, one coefficient for
every emitting group, one or four vectors per launch.  The model table below reaches each of them (checked without a
GPU from the table, with a GPU from what the context reports), at every row split and walk.

The reference is fermion_pin.apply_to_states: each monomial applied to each state bit by bit, with the sign of the
Jordan-Wigner string counted on the state itself.  It shares nothing with the compiled tables that the C oracle and the
device both apply, so a wrong string -- a hop across the wrap, an exchange term whose string crosses bit N, a string
that reaches bit 63 -- fails here even where the oracle and the device agree.

Without a GPU: the reference against the dense pin, the compiled tables against the reference at 17 to 64 sites, the
BdG ground energy, build coverage.  On the GPU: the model table at every build, split and walk; bases of 34 to 64 bits
on every index and kernel; sector edges; several ranks; errors; ground energies and sampled rows at size; zz over 64
bits.  Criterion: test_fermions._close, unchanged.
"""
from __future__ import annotations

import functools
import itertools
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

import fermion_pin as fp  # noqa: E402
import torch  # noqa: E402
from distributed_matvec_b200 import Operator  # noqa: E402
from distributed_matvec_b200 import _native as nat  # noqa: E402
from distributed_matvec_b200.config import OperatorSpec, basis_from_dict  # noqa: E402
from distributed_matvec_b200.expr import compile_terms  # noqa: E402
from gen_models import _bonds_ring, _bonds_torus, hubbard, spinless_ring  # noqa: E402
from oracle import pyoracle as po  # noqa: E402
from test_fermions import _close  # noqa: E402

INDEX_DIRECTORY, INDEX_IDENTITY, INDEX_LIN, INDEX_LIN_SPLIT = 0, 1, 3, 4
SPLITS = (-1, 1, 2, 4, 8, 16, 32)   # -1: auto
WALKS = (0, 1, 2)


# ---------------------------------------------------------------------------------------------------------------------
# models

def _hop(t, arrows=("↑", "↓"), phase=0.0, scale="-"):
    """-t e^{iφ} c†₀ c₁ - t e^{-iφ} c†₁ c₀ per spin; scale "uniform": -(0.6 + 0.8i) t (c†₀ c₁ + c†₁ c₀), one complex
    coefficient with a real part in both directions (not Hermitian)."""
    c, s = t * math.cos(phase), t * math.sin(phase)
    out = []
    for a in arrows:
        if scale == "uniform":
            out.append(f"- {0.6 * t!r} × c†₀{a} c₁{a} - {0.8 * t!r}j × c†₀{a} c₁{a} - {0.6 * t!r} × c†₁{a} c₀{a} "
                       f"- {0.8 * t!r}j × c†₁{a} c₀{a}")
        elif phase:
            out.append(f"- {c!r} × c†₀{a} c₁{a} - {s!r}j × c†₀{a} c₁{a} - {c!r} × c†₁{a} c₀{a} + {s!r}j × c†₁{a} c₀{a}")
        else:
            out.append(f"- {t!r} × c†₀{a} c₁{a} - {t!r} × c†₁{a} c₀{a}")
    return " ".join(out)


def _spinful(n, up, down, terms):
    return {"basis": {"particle": "spinful-fermion", "number_sites": n, "number_particles": up + down,
                      "number_up": up}, "hamiltonian": {"terms": terms}}


def _spinless(n, nf, terms):
    basis = {"particle": "spinless-fermion", "number_sites": n}
    if nf is not None:
        basis["number_particles"] = nf
    return {"basis": basis, "hamiltonian": {"terms": terms}}


def _u(n, u=4.0):
    return {"expression": f"{u!r} × n₀↑ n₀↓", "sites": [[i] for i in range(n)]}


def _ring(n, d):
    return [[i, (i + d) % n] for i in range(n)]


def _hubbard_ring(n, up, down, t2=None, u=4.0):
    terms = [{"expression": _hop(1.0), "sites": _ring(n, 1)}, _u(n, u)]
    if t2 is not None:
        terms.append({"expression": _hop(t2), "sites": _ring(n, 2)})
    return _spinful(n, up, down, terms)


def _peierls_torus_3x4(phi=0.3):
    """Hubbard 3 x 4 torus, the x bonds with a Peierls phase: a complex LUT on 48 groups (wide)."""
    bonds = _bonds_torus(3, 4)
    return _spinful(12, 2, 2, [{"expression": _hop(1.0, phase=phi), "sites": bonds[0::2]},
                               {"expression": _hop(0.7), "sites": bonds[1::2]}, _u(12)])


def _nonhermitian_ring(n, nf, nnn):
    """-(0.6 + 0.8i) t Σ (c†_i c_j + c†_j c_i): one complex coefficient for every group, no diagonal terms."""
    terms = [{"expression": _hop(1.0, ("",), scale="uniform"), "sites": _ring(n, 1)}]
    if nnn:
        terms.append({"expression": _hop(1.0, ("",), scale="uniform"), "sites": _ring(n, 2)})
    return _spinless(n, nf, terms)


def _vn_ring(n, nf):
    conf = spinless_ring(n, nf)
    conf["hamiltonian"]["terms"].append({"expression": "1.5 × n₀ n₁", "sites": _bonds_ring(n)})
    return conf


def _bdg_chain(n, nf=None, t1=1.0, t2=0.4, d1=0.6, d2=0.25, mu=0.3):
    """Open chain: hops t1, t2 and real pairing d1, d2 on the nearest and next-nearest bonds, chemical potential mu.
    -> (config, exact ground energy of the whole Fock space): H = Σ h_ij c†_i c_j + ½ Σ (Δ_ij c†_i c†_j + h.c.) has
    E0 = ½ (Tr h - Σ_{ε > 0} ε) over the eigenvalues ε of [[h, Δ], [-Δ, -h]]."""
    h, D = -mu * np.eye(n), np.zeros((n, n))
    terms = []
    for d, t, dl in ((1, t1, d1), (2, t2, d2)):
        bonds = [[i, i + d] for i in range(n - d)]
        terms.append({"expression": f"-{t!r} × c†₀ c₁ - {t!r} × c†₁ c₀", "sites": bonds})
        terms.append({"expression": f"{dl!r} × c†₀ c†₁ + {dl!r} × c₁ c₀", "sites": bonds})
        for i, j in bonds:
            h[i, j] = h[j, i] = -t
            D[i, j], D[j, i] = dl, -dl
    terms.append({"expression": f"-{mu!r} × n₀", "sites": [[i] for i in range(n)]})
    eps = np.linalg.eigvalsh(np.block([[h, D], [-D, -h]]))
    return _spinless(n, nf, terms), 0.5 * (np.trace(h) - eps[eps > 0].sum())


def _model(conf):
    basis = basis_from_dict(conf["basis"])
    off, diag = compile_terms(conf["hamiltonian"]["terms"], basis.number_sites, basis.fermion_modes())
    return basis, OperatorSpec(basis=basis, off_diag=off, diag=diag)


# name: (config, expected build: gather_narrow, gather_uniform, complex_coefficients, index_mode, bp_words).  Every
# model runs k_gather with sign masks.  With the auto index (Lin tables, LIN = 1) and the directory (LIN = 0), both
# element types and KB = 1 and 4, each model reaches the 8 builds of its (CV, NARROW, UNI); the models below cover all
# 8 combinations, so all 64 builds.
MODELS = {
    "hubbard_chain_8": (lambda: hubbard(8, _bonds_ring(8)), (1, 1, 0, INDEX_LIN_SPLIT, 1)),
    # t != t': a real coefficient LUT on narrow rows (32 groups, 16 bits)
    "hubbard_ring_8_t_t2": (lambda: _hubbard_ring(8, 3, 3, t2=0.35), (1, 0, 0, INDEX_LIN_SPLIT, 1)),
    "hubbard_torus_3x4": (lambda: hubbard(12, _bonds_torus(3, 4), number_up=3, number_down=3),
                          (0, 1, 0, INDEX_LIN_SPLIT, 1)),
    "hubbard_torus_3x4_anisotropic": (
        lambda: _spinful(12, 3, 3, [{"expression": _hop(1.0), "sites": _bonds_torus(3, 4)[0::2]},
                                    {"expression": _hop(0.5), "sites": _bonds_torus(3, 4)[1::2]}, _u(12)]),
        (0, 0, 0, INDEX_LIN_SPLIT, 1)),
    "peierls_ring_6": (lambda: _spinful(6, 3, 3, [{"expression": _hop(1.0, phase=0.3), "sites": _ring(6, 1)}, _u(6)]),
                       (1, 0, 1, INDEX_LIN_SPLIT, 1)),
    "peierls_torus_3x4": (_peierls_torus_3x4, (0, 0, 1, INDEX_LIN_SPLIT, 1)),
    # not Hermitian: -(0.6 + 0.8i) t on every hop, a complex uniform coefficient; 12 groups (narrow) and 36 (wide)
    "nonhermitian_ring_12": (lambda: _nonhermitian_ring(12, 5, False), (1, 1, 1, INDEX_LIN, 1)),
    "nonhermitian_ring_18_nnn": (lambda: _nonhermitian_ring(18, 5, True), (0, 1, 1, INDEX_LIN, 1)),
    # no diagonal terms: y is accumulated into
    "spinless_ring_14": (lambda: spinless_ring(14, 6), (1, 1, 0, INDEX_LIN, 1)),
    "spinless_ring_16_v": (lambda: _vn_ring(16, 7), (1, 1, 0, INDEX_LIN, 1)),
    # 18 sites, 2 up and 2 down, nearest and next-nearest hops: 72 groups, two BpWords (g_base = 64 in the second)
    "hubbard_ring_18_nnn_few": (lambda: _hubbard_ring(18, 2, 2, t2=1.0), (0, 1, 0, INDEX_LIN_SPLIT, 2)),
}

# SG = 1 builds that spill where their SG = 0 twin does not (profiles/fermion_resource_usage.md):
# (CV, CE, NARROW, LIN, UNI, KB)
SPILLING = {(0, 1, 0, 0, 1, 4), (1, 0, 1, 0, 0, 4), (1, 1, 0, 0, 1, 4), (1, 1, 0, 1, 0, 1), (1, 1, 1, 0, 1, 1),
            (1, 1, 1, 1, 1, 4)}


@functools.lru_cache(maxsize=None)
def _table_model(name):
    conf = MODELS[name][0]()
    basis, matrix = _model(conf)
    return conf, basis, matrix


def _states_of(basis):
    if basis.particle_type == "spinful-fermion":
        return fp.sector_states(basis.number_sites, basis.number_up, basis.number_particles - basis.number_up)
    if basis.number_particles is None:
        return np.arange(1 << basis.number_sites, dtype=np.uint64)
    return fp.sector_states(basis.number_sites, basis.number_particles, spinful=False)


def _reference(conf, states, targets=None):
    b = conf["basis"]
    return fp.apply_to_states(conf["hamiltonian"]["terms"], b["number_sites"], b["particle"] == "spinful-fermion",
                              states, targets)


def _oracle_matrix(op: OperatorSpec, states: np.ndarray, targets: np.ndarray) -> sp.csr_matrix:
    """<β|H|α> from the compiled tables, applied term by term by the C oracle, α over `states`, β over `targets`."""
    n = states.shape[0]
    parts = []
    for lo in range(0, n, 2048):
        chunk = states[lo:lo + 2048]
        betas, coeffs, offsets = po.apply_off_diag(op, chunk)
        rows = np.minimum(np.searchsorted(targets, betas), targets.shape[0] - 1)
        assert np.array_equal(targets[rows], betas), "a compiled term leads out of the target states"
        cols = lo + np.repeat(np.arange(chunk.shape[0]), np.diff(offsets))
        parts.append(sp.coo_matrix((coeffs, (rows, cols)), shape=(targets.shape[0], n)))
    d = po.apply_diag(op, states, np.ones(n, dtype=np.complex128))
    rows = np.searchsorted(targets, states)
    keep = (rows < targets.shape[0]) & (targets[np.minimum(rows, targets.shape[0] - 1)] == states)
    assert np.all(keep[d != 0]), "a diagonal term on a state outside the targets"
    parts.append(sp.coo_matrix((d[keep], (rows[keep], np.nonzero(keep)[0])), shape=(targets.shape[0], n)))
    return functools.reduce(lambda a, b: a + b, [p.tocsr() for p in parts])


def _diff(a, b) -> float:
    d = sp.csr_matrix(a - b)
    return float(abs(d).max()) if d.nnz else 0.0


# ---------------------------------------------------------------------------------------------------------------------
# the reference against the dense pin

_KINDS = {"c+": "c†", "c": "c", "n": "n"}


def _random_monomial(rng, n_modes, spinful, n_sites):
    """One random monomial of 1 to 4 operators, repeated modes allowed -> (term spec, [(kind, mode)])."""
    length = int(rng.integers(1, 5))
    kinds = [str(rng.choice(["c+", "c", "n"])) for _ in range(length)]
    modes = [int(m) for m in rng.integers(0, n_modes, size=length)]
    return _monomial_spec(kinds, modes, complex(rng.normal(), rng.normal()), spinful, n_sites), list(zip(kinds, modes))


def _monomial_spec(kinds, modes, coeff, spinful, n_sites):
    """The spec coeff × op_1 ... op_k on concrete modes, written with placeholders and spin arrows."""
    if spinful:
        sites = [m % n_sites for m in modes]
        arrows = ["↓" if m >= n_sites else "↑" for m in modes]
    else:
        sites, arrows = list(modes), [""] * len(modes)
    distinct = sorted(set(sites), key=sites.index)
    place = {s: p for p, s in enumerate(distinct)}
    text = " ".join(f"{_KINDS[k]}{place[s]}{a}" for k, s, a in zip(kinds, sites, arrows))
    return {"expression": f"{coeff.real!r} × {text} + {coeff.imag!r}j × {text}", "sites": [distinct]}


# spin exchange, pair hopping, pairing and its conjugate, density-assisted hops on placeholders 0 and 1
NAMED_SPINFUL = ["c†₀↑ c₀↓ c†₁↓ c₁↑", "c†₀↑ c†₀↓ c₁↓ c₁↑", "c†₀↑ c†₁↓", "c₁↓ c₀↑", "c†₀↑ c†₁↑", "c₀↓ c₁↓",
                 "n₀↓ c†₀↑ c₁↑", "c†₁↓ c₀↓ n₁↑", "c†₀↓ c₀↑"]
NAMED_SPINLESS = ["c†₀ c†₁", "c₁ c₀", "n₀ c†₀ c₁", "c†₀ c₁ n₁", "c†₀ c†₁ c₁ c₀"]


def test_apply_to_states_equals_the_dense_pin():
    """Random monomials of 1 to 4 operators (pairing, repeated modes included) on 12 spinless modes and on 8 spinful
    sites (16 modes), and the named spinful and spinless terms on pairs of sites both ways round: the bit-level reference
    equals the product of the Jordan-Wigner matrices exactly."""
    rng = np.random.default_rng(2024)
    for spinful, n_sites in ((False, 12), (True, 8)):
        n_modes = 2 * n_sites if spinful else n_sites
        states = np.arange(1 << n_modes, dtype=np.uint64)
        for trial in range(40):
            spec, ops = _random_monomial(rng, n_modes, spinful, n_sites)
            got = fp.apply_to_states([spec], n_sites, spinful, states)
            want = fp.full_hamiltonian([spec], n_sites, spinful)
            assert _diff(got, want) == 0.0, (spinful, trial, spec)
        named = NAMED_SPINFUL if spinful else NAMED_SPINLESS
        pairs = [[0, n_sites - 1], [n_sites - 1, 0], [2, 5], [6, 1], [3, 4]]
        for text in named:
            spec = {"expression": f"0.7 × {text}", "sites": pairs}
            got = fp.apply_to_states([spec], n_sites, spinful, states)
            assert got.nnz > 0
            assert _diff(got, fp.full_hamiltonian([spec], n_sites, spinful)) < 1e-15, text


def test_apply_to_states_rows_and_refusal():
    """Rows other than the columns: c†c† from 1 to 3 particles; a term that leads out of the rows raises."""
    n = 6
    spec = [{"expression": "c†₀ c†₁", "sites": [[0, 5], [2, 1]]}]
    one, three = fp.sector_states(n, 1, spinful=False), fp.sector_states(n, 3, spinful=False)
    H = fp.apply_to_states(spec, n, False, one, np.sort(np.concatenate([one, three])))
    full = fp.full_hamiltonian(spec, n, False)
    rows = np.sort(np.concatenate([one, three])).astype(np.int64)
    assert _diff(H, full[rows][:, one.astype(np.int64)]) == 0.0 and H.nnz == 8
    with pytest.raises(ValueError, match="leads out"):
        fp.apply_to_states(spec, n, False, one)


def test_sector_states_vectorised():
    for n, up, down in ((5, 2, 1), (9, 0, 4), (26, 1, 2), (32, 2, 1)):
        got = fp.sector_states(n, up, down)
        want = np.array(sorted((d << n) | u for u in
                               (sum(1 << b for b in c) for c in itertools.combinations(range(n), up))
                               for d in (sum(1 << b for b in c) for c in itertools.combinations(range(n), down))),
                        dtype=np.uint64)
        assert got.dtype == np.uint64 and np.array_equal(got, want), (n, up, down)
    assert np.array_equal(fp.sector_states(64, 1, spinful=False), np.uint64(1) << np.arange(64, dtype=np.uint64))
    assert fp.sector_states(32, 3, 3).shape[0] == math.comb(32, 3) ** 2


# ---------------------------------------------------------------------------------------------------------------------
# compiled tables past 16 modes

def _wide_spinful(n, up, down, generic=True):
    """Hubbard ring of n sites with the wrap bond, next-nearest hops, hops across the ring, and (generic) spin exchange
    and pair hopping between sites far apart: Jordan-Wigner strings across bit N and, at n = 32, up to bit 63."""
    far = [[0, n - 1], [1, n // 2], [n // 3, n - 2], [n - 1, 2]]
    terms = [{"expression": _hop(1.0), "sites": _ring(n, 1)}, {"expression": _hop(0.3), "sites": _ring(n, 2)},
             {"expression": _hop(0.45), "sites": far}, _u(n)]
    if generic:
        terms += [{"expression": "0.8 × c†₀↑ c₀↓ c†₁↓ c₁↑ + 0.8 × c†₁↑ c₁↓ c†₀↓ c₀↑", "sites": far},
                  {"expression": "0.55 × c†₀↑ c†₀↓ c₁↓ c₁↑ + 0.55 × c†₁↑ c†₁↓ c₀↓ c₀↑", "sites": far + [[3, n - 3]]},
                  {"expression": "-0.2 × n₀↑ n₁↓", "sites": far}]
    return _spinful(n, up, down, terms)


def _wide_spinless(n, nf, pairing):
    """Spinless ring of n sites: nearest and next-nearest hops, hops across the whole word, a density interaction and
    (pairing) c†c† + cc on a free particle number."""
    far = [[1, n - 1], [0, n // 2], [n - 2, 3], [n // 2 + 1, n - 1]]
    terms = [{"expression": "-1.0 × c†₀ c₁ - 1.0 × c†₁ c₀", "sites": _ring(n, 1)},
             {"expression": "-0.3 × c†₀ c₁ - 0.3 × c†₁ c₀", "sites": _ring(n, 2) + far},
             {"expression": "0.9 × n₀ n₁", "sites": _ring(n, 1)}]
    if pairing:
        terms.append({"expression": "0.6 × c†₀ c†₁ + 0.6 × c₁ c₀", "sites": _ring(n, 1) + far})
    return _spinless(n, None if pairing else nf, terms)


WIDE_CPU = {
    "spinful_17": lambda: (_wide_spinful(17, 2, 2), None),
    "spinful_20": lambda: (_wide_spinful(20, 2, 1), None),
    "spinful_21": lambda: (_wide_spinful(21, 1, 2), None),
    "spinful_32": lambda: (_wide_spinful(32, 2, 1), None),
    "spinful_32_down_heavy": lambda: (_wide_spinful(32, 1, 3), None),
    "spinless_33": lambda: (_wide_spinless(33, 4, False), None),
    "spinless_40": lambda: (_wide_spinless(40, 3, False), None),
    "spinless_64": lambda: (_wide_spinless(64, 3, False), None),
    # free particle number: columns at 2 particles, rows at 0, 2 and 4
    "spinless_40_pairing": lambda: (_wide_spinless(40, None, True), 2),
    "spinless_64_pairing": lambda: (_wide_spinless(64, None, True), 2),
}


@pytest.mark.parametrize("name", sorted(WIDE_CPU))
def test_compiled_tables_equal_the_reference_past_16_modes(name):
    """The compiled tables, applied by the C oracle, equal the bit-level reference on 17 to 64 sites, strings across
    bit N, bit 32 and up to bit 63 included."""
    conf, nf = WIDE_CPU[name]()
    basis, op = _model(conf)
    n = basis.number_sites
    if nf is None:
        states = _states_of(basis)
        targets = states
    else:
        states = fp.sector_states(n, nf, spinful=False)
        targets = np.unique(np.concatenate([fp.sector_states(n, k, spinful=False) for k in (nf - 2, nf, nf + 2)]))
    top = min(32, basis.number_bits - 2)   # a string lies strictly between two modes
    assert np.any(op.off_diag.s >> np.uint64(top)), f"a string reaches bit {top}"
    if basis.number_bits == 64:
        assert np.any(op.off_diag.s >> np.uint64(62)) and np.any(states >> np.uint64(63)), "bit 63"
    got = _oracle_matrix(op, states, targets)
    want = _reference(conf, states, targets)
    assert want.nnz > states.shape[0]
    assert _diff(got, want) < 1e-13, name   # merged coefficients and the Walsh-expanded diagonal round differently


def test_bdg_ground_energy_equals_the_dense_pin():
    """Open chains of 10 and 14 sites with nn + nnn hops, pairing and μ on the whole Fock space: the dense pin's E0,
    the BdG value and the lowest eigenvalue of the compiled tables agree; the tables equal the reference."""
    for n in (10, 14):
        conf, exact = _bdg_chain(n)
        basis, op = _model(conf)
        states = np.arange(1 << n, dtype=np.uint64)
        H = fp.full_hamiltonian(conf["hamiltonian"]["terms"], n, False)
        assert _diff(fp.apply_to_states(conf["hamiltonian"]["terms"], n, False, states), H) < 1e-15
        tables = _oracle_matrix(op, states, states)
        assert _diff(tables, H) < 1e-14
        e_pin = sla.eigsh(H, k=1, which="SA", tol=1e-14)[0][0]
        e_tab = sla.eigsh(tables, k=1, which="SA", tol=1e-14)[0][0]
        assert abs(e_pin - exact) < 1e-11 * abs(exact) and abs(e_tab - exact) < 1e-11 * abs(exact), (n, e_pin, exact)


@pytest.mark.parametrize("name", sorted(MODELS))
def test_model_table_oracle_equals_the_reference(name):
    """The oracle's product on every model of the table (the GPU tests' reference) equals the bit-level reference's, in
    both element types, and the model has the build the table expects as far as the host can tell."""
    conf, basis, matrix = _table_model(name)
    narrow, _, cv, index_mode, words = MODELS[name][1]
    states = _states_of(basis)
    groups = np.unique(matrix.off_diag.x).shape[0]
    assert np.any(matrix.off_diag.s != 0)
    assert int(not matrix.is_real()) == cv
    assert int(basis.number_bits <= 32 and groups <= 32) == narrow
    assert (groups + 63) // 64 == words
    assert index_mode == (INDEX_LIN_SPLIT if basis.particle_type == "spinful-fermion" else INDEX_LIN)
    H = _reference(conf, states)
    for cplx in (False, True):
        x = _x(states.shape[0], cplx)
        want = H @ x
        if not cplx:
            want = want.real   # real vectors take the real part
        assert _close(po.matvec_global(matrix, states, x, 1), want), (name, cplx)


def test_every_signed_gather_build_is_covered():
    """The model table, expanded over element types, the auto and the directory index and KB = 1, 4, reaches all 64
    (CV, CE, NARROW, LIN, UNI, KB) builds of k_gather with sign masks, the six that spill where their twin without
    signs does not among them."""
    covered = set()
    for name, (_, (narrow, uniform, cv, index_mode, _)) in MODELS.items():
        lins = {int(index_mode in (INDEX_LIN, INDEX_LIN_SPLIT)), 0}
        for ce, lin, kb in itertools.product((0, 1), lins, (1, 4)):
            covered.add((cv, ce, narrow, lin, uniform, kb))
    every = set(itertools.product((0, 1), (0, 1), (0, 1), (0, 1), (0, 1), (1, 4)))
    assert covered == every, sorted(every - covered)
    assert SPILLING <= covered and len(covered) == 64


# =====================================================================================================================
# GPU

@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _x(n, cplx, seed=3):
    rng = np.random.default_rng(seed)
    x = rng.random(n) - 0.5
    return x + 1j * (rng.random(n) - 0.5) if cplx else x


def _dev(op, x, y0=None):
    y = op.matvec(torch.from_numpy(x).cuda(), None if y0 is None else torch.from_numpy(y0.copy()).cuda())
    torch.cuda.synchronize()
    return y.cpu().numpy()


def _set(op, **opts):
    for k, v in opts.items():
        op.set_option(k, v)


def _build_of(op):
    return (op.info("gather"), op.info("gather_signs"), op.info("gather_narrow"), op.info("gather_uniform"),
            op.info("complex_coefficients"), op.info("index_mode"), op.info("bp_words"))


def _oracle_y(matrix, reps, x, num_ranks=1, y0=None):
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    if y0 is not None:
        return po.matvec_blocks(matrix, [reps], [x], y_blocks=[y0.copy()], num_tasks=po.num_threads())[0]
    return po.matvec_global(matrix, reps, x, num_ranks, num_tasks=po.num_threads())


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MODELS))
def test_signed_gather_every_build_split_and_walk(need_cuda, name):
    """Both element types (real vectors on complex operators too) x index auto and directory x gather_split auto, 1, 2,
    4, 8, 16, 32 x gather_walk 0, 1, 2: the full vector against the oracle, host and device pointers and a repeated
    product bit-identical; matvec_batch with 4 and 9 columns bit-identical to the single products at splits 1 and 32
    under every walk.  Without diagonal terms y is accumulated into."""
    conf, basis, matrix = _table_model(name)
    narrow, uniform, cv, index_mode, words = MODELS[name][1]
    reps = _states_of(basis)
    n = reps.shape[0]
    no_diag = len(matrix.diag) == 0
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        assert _build_of(op) == (1, 1, narrow, uniform, cv, index_mode, words), (name, _build_of(op))
        for cplx in (False, True):
            x = _x(n, cplx)
            y_ref = _oracle_y(matrix, reps, x)
            y0 = _x(n, cplx, seed=9) if no_diag else None
            y0_ref = _oracle_y(matrix, reps, x, y0=y0) if no_diag else None
            X = np.stack([_x(n, cplx, 100 + j) for j in range(9)])
            for index in (-1, 0):
                _set(op, index=index)
                assert op.info("index_mode") == (index_mode if index == -1 else INDEX_DIRECTORY)
                for split in SPLITS:
                    for walk in WALKS:
                        _set(op, gather_split=split, gather_walk=walk)
                        where = (name, cplx, index, split, walk)
                        assert op.info("gather") == 1, where
                        if split > 0:
                            assert op.info("gather_split") == split, where
                        y = _dev(op, x)
                        assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
                        assert np.array_equal(_dev(op, x), y), where
                        assert np.array_equal(op.matvec(x), y), where
                        if no_diag:
                            y = _dev(op, x, y0)
                            assert _close(y, y0_ref), (where, "accumulate", np.abs(y - y0_ref).max())
                for split in (1, 32):
                    for walk in WALKS:
                        _set(op, gather_split=split, gather_walk=walk)
                        singles = np.stack([_dev(op, X[j]) for j in range(9)])
                        for k in (4, 9):
                            Y = op.matvec_batch(torch.from_numpy(X[:k].copy()).cuda())
                            torch.cuda.synchronize()
                            assert np.array_equal(Y.cpu().numpy(), singles[:k]), (name, cplx, index, split, walk, k)
                _set(op, gather_split=-1, gather_walk=0)
            _set(op, index=-1)
            for j in (0, 8):
                assert _close(singles[j], _oracle_y(matrix, reps, X[j])), (name, cplx, j)
        assert _build_of(op) == (1, 1, narrow, uniform, cv, index_mode, words)
    finally:
        op.close()


# bases past 32 bits: (config, expected index_mode, k_gather runs)
def _hubbard_wide(n, up, down):
    return _wide_spinful(n, up, down, generic=False)


WIDE = {
    "spinful_17": (lambda: _hubbard_wide(17, 2, 2), INDEX_LIN_SPLIT, 1),
    "spinful_20": (lambda: _hubbard_wide(20, 2, 2), INDEX_LIN_SPLIT, 1),
    "spinful_21": (lambda: _hubbard_wide(21, 2, 2), INDEX_DIRECTORY, 1),
    "spinful_24": (lambda: _hubbard_wide(24, 2, 2), INDEX_DIRECTORY, 1),
    "spinful_32": (lambda: _hubbard_wide(32, 2, 2), INDEX_DIRECTORY, 1),
    # exchange and pair hopping flip four bits: no bit-parallel emit test, so k_pull / the scatter form only
    "spinful_32_exchange": (lambda: _wide_spinful(32, 2, 1), INDEX_DIRECTORY, 0),
    "spinless_40": (lambda: _wide_spinless(40, 3, False), INDEX_LIN, 1),
    "spinless_64": (lambda: _wide_spinless(64, 3, False), INDEX_DIRECTORY, 1),
    "spinless_free_18_pairing": (lambda: _wide_spinless(18, None, True), INDEX_IDENTITY, 1),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(WIDE))
def test_wide_fermion_bases(need_cuda, name):
    """Spinful 17 and 20 sites (split Lin index, 64-bit rows), 21, 24 and 32 (directory; at 32 bit 63 is occupied),
    spinless 40 and 64, a free-number spinless basis with pairing (identity index): the representatives are the
    reference enumeration; k_gather at three splits and every walk, the directory index, k_pull and the scatter form in
    both element types equal the oracle, and the oracle equals the bit-level reference."""
    conf, index_mode, gather = WIDE[name]
    conf = conf()
    basis, matrix = _model(conf)
    reps = _states_of(basis)
    n = reps.shape[0]
    assert n <= 300_000
    if basis.number_bits == 64:
        assert np.any(reps >> np.uint64(63))
    H = _reference(conf, reps)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        assert (op.info("gather"), op.info("gather_signs"), op.info("index_mode")) == (gather, gather, index_mode)
        for cplx in (False, True):
            x = _x(n, cplx)
            y_ref = _oracle_y(matrix, reps, x)
            assert _close(y_ref, H @ x), (name, cplx, "oracle against the reference")
            for index in ((-1, 0) if index_mode != INDEX_DIRECTORY else (-1,)):
                _set(op, index=index)
                settings = [(s, w) for s in (-1, 1, 32) for w in WALKS] if gather else [(-1, 0)]
                for split, walk in settings:
                    _set(op, gather_split=split, gather_walk=walk)
                    assert op.info("gather") == gather
                    y = _dev(op, x)
                    assert _close(y, y_ref), (name, cplx, index, split, walk, np.abs(y - y_ref).max())
                _set(op, gather_split=-1, gather_walk=0)
                for opts, pull in (({"mode": 1, "gather": 0}, 1), ({"mode": 0}, 0)):   # k_pull, the scatter form
                    _set(op, **opts)
                    assert (op.info("gather"), op.info("pull")) == (0, pull)
                    y = _dev(op, x)
                    assert _close(y, y_ref), (name, cplx, index, opts, np.abs(y - y_ref).max())
                    _set(op, **{k: -1 for k in opts})
            _set(op, index=-1)
    finally:
        op.close()


EDGES = {
    # (number_sites, up, down): empty and full halves at 20 and 32 sites, one particle, the empty basis
    "spinful_20_no_up": (20, 0, 3), "spinful_20_all_up": (20, 20, 1), "spinful_20_no_down": (20, 3, 0),
    "spinful_32_no_up": (32, 0, 2), "spinful_32_all_up": (32, 32, 1), "spinful_32_no_down": (32, 2, 0),
    "spinful_32_one": (32, 0, 1), "spinful_20_empty": (20, 0, 0),
    "spinless_40_empty": (40, 0, None), "spinless_24_full": (24, 24, None), "spinless_64_one": (64, 1, None),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(EDGES))
def test_sector_edges(need_cuda, name):
    """Sectors at the edges: no up particle, every site up, no down particle, one particle, zero particles, a full
    spinless basis: the representatives, and the product on every index and kernel against the reference."""
    n, up, down = EDGES[name]
    conf = _hubbard_wide(n, up, down) if down is not None else _wide_spinless(n, up, False)
    basis, matrix = _model(conf)
    reps = _states_of(basis)
    H = _reference(conf, reps)
    op = Operator(matrix)
    try:
        if name == "spinful_32_all_up":
            # the enumeration walks every state of the total weight over 64 bits (C(64, 33) of them) and refuses; the
            # block is installed as it stands
            with pytest.raises(nat.DmvError, match="more than 2\\^40 states"):
                op.basis.build()
            op.basis.uncheckedSetRepresentatives(reps)
        else:
            op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        for cplx in (False, True):
            x = _x(reps.shape[0], cplx)
            y_ref = _oracle_y(matrix, reps, x)
            assert _close(y_ref, H @ x)
            for opts in ({}, {"index": 0}, {"gather_split": 32, "gather_walk": 2}, {"gather_walk": 1},
                         {"mode": 1, "gather": 0}, {"mode": 0}):
                _set(op, **opts)
                y = _dev(op, x)
                assert _close(y, y_ref), (name, cplx, opts, np.abs(y - y_ref).max())
                _set(op, **{k: (0 if k == "gather_walk" else -1) for k in opts})
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("num_ranks", [2, 3, 4])
@pytest.mark.parametrize("name", ["spinful_20", "spinful_32", "spinless_40"])
def test_wide_fermions_on_several_ranks(need_cuda, name, num_ranks):
    """Records (k_generate and the exchange) and the replicated-x form (k_gather with signs on the whole-basis twin:
    split Lin index at 20 sites, directory at 32, Lin at 40) on P logical ranks against the oracle's P-rank product; the
    twin holds the reference enumeration."""
    from distributed_matvec_b200 import EmulatedCluster, block_to_hashed, hashed_to_block
    conf = {"spinful_20": lambda: _hubbard_wide(20, 2, 2), "spinful_32": lambda: _hubbard_wide(32, 2, 1),
            "spinless_40": lambda: _wide_spinless(40, 3, False)}[name]()
    twin_index = {"spinful_20": INDEX_LIN_SPLIT, "spinful_32": INDEX_DIRECTORY, "spinless_40": INDEX_LIN}[name]
    basis, matrix = _model(conf)
    reps = _states_of(basis)
    masks, blocks = po.partition_by_hash(reps, num_ranks)
    cl = EmulatedCluster(matrix, num_ranks).build()
    try:
        for r, op in enumerate(cl.ops):
            assert np.array_equal(op.basis.representatives(), blocks[r])
        for cplx in (False, True):
            x = _x(reps.shape[0], cplx, 31)
            y_ref = _oracle_y(matrix, reps, x, num_ranks)
            xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, num_ranks)]
            y = hashed_to_block([t.cpu().numpy() for t in cl.matvec(xb)], masks)
            assert _close(y, y_ref), (name, num_ranks, cplx, "records", np.abs(y - y_ref).max())
            for split, walk in ((-1, 0), (1, 1), (32, 2)):
                for op in cl.ops:
                    _set(op, gather_split=split, gather_walk=walk)
                y = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)
                assert _close(y, y_ref), (name, num_ranks, cplx, "replicated", split, walk, np.abs(y - y_ref).max())
            for op in cl.ops:
                assert (op.info("global.gather"), op.info("global.gather_signs")) == (1, 1)
                assert op.info("global.index_mode") == twin_index
                assert op.info("global_states") == reps.shape[0]
    finally:
        cl.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n", [20, 32])
def test_wide_spin_flip_is_an_invalid_index(need_cuda, n):
    """c†↑ c↓ leaves a spinful sector of 20 and 32 sites: the product raises "invalid index" at splits 1 and 32 under
    every walk and under k_pull."""
    conf = _hubbard_wide(n, 2, 1)
    conf["hamiltonian"]["terms"].append({"expression": "c†₀↑ c₀↓ + c†₀↓ c₀↑", "sites": [[n - 1], [3]]})
    basis, matrix = _model(conf)
    reps = _states_of(basis)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert op.info("gather") == 1
        settings = [{"gather_split": s, "gather_walk": w} for s in (1, 32) for w in WALKS] + [{"mode": 1, "gather": 0}]
        for opts in settings:
            _set(op, **opts)
            with pytest.raises(nat.DmvError, match="invalid index"):
                op.matvec(_x(reps.shape[0], False))
                op.synchronize()
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("split", [1, 32])
@pytest.mark.parametrize("walk", WALKS)
def test_wide_missing_state_is_an_invalid_index(need_cuda, split, walk):
    """A 40-site spinless block with states removed through uncheckedSetRepresentatives: a hop to a removed state
    raises "invalid index"."""
    basis, matrix = _model(_wide_spinless(40, 3, False))
    reps = _states_of(basis)
    op = Operator(matrix)
    try:
        op.basis.uncheckedSetRepresentatives(reps[:-7])
        _set(op, gather_split=split, gather_walk=walk)
        assert op.info("gather") == 1 and op.info("gather_split") == split
        with pytest.raises(nat.DmvError, match="invalid index"):
            op.matvec(np.ones(reps.shape[0] - 7))
            op.synchronize()
    finally:
        op.close()


@pytest.mark.gpu
def test_bdg_chain_24_at_size(need_cuda):
    """Open chain of 24 sites with nn + nnn hops, pairing and μ on the whole Fock space (2^24 states, identity index):
    the device's lowest eigenvalue is the BdG ground energy to 1e-10."""
    conf, exact = _bdg_chain(24)
    basis, matrix = _model(conf)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert op.basis.numberStates() == 1 << 24
        assert (op.info("gather"), op.info("gather_signs"), op.info("index_mode")) == (1, 1, INDEX_IDENTITY)
        evals, _, _, conv, _, _ = op.eigsh(1, tol=1e-12, eigenvectors=False)
        assert conv >= 1 and abs(evals[0] - exact) < 1e-10 * abs(exact), (evals[0], exact)
    finally:
        op.close()


@pytest.mark.gpu
def test_hubbard_ring_32_at_size(need_cuda):
    """Hubbard ring of 32 sites with 3 up and 3 down particles (24 601 600 states, 64-bit rows, directory index): at
    U = 0 the lowest eigenvalue is the sum of the lowest ring levels of each species; at U = 4 2000 sampled rows of one
    product equal the oracle's."""
    n = 32
    levels = np.sort(-2 * np.cos(2 * np.pi * np.arange(n) / n))
    rng = np.random.default_rng(32)
    for u in (0.0, 4.0):
        basis, matrix = _model(_hubbard_ring(n, 3, 3, u=u))
        op = Operator(matrix)
        try:
            op.basis.build()
            assert op.basis.numberStates() == math.comb(32, 3) ** 2
            assert (op.info("gather"), op.info("gather_signs"), op.info("index_mode")) == (1, 1, INDEX_DIRECTORY)
            if u == 0.0:
                exact = 2 * levels[:3].sum()
                evals, _, _, conv, _, _ = op.eigsh(1, tol=1e-12, eigenvectors=False)
                assert conv >= 1 and abs(evals[0] - exact) < 1e-10 * abs(exact), (evals[0], exact)
            else:
                reps = op.basis.representatives()
                assert np.array_equal(reps, fp.sector_states(n, 3, 3))
                x = rng.random(reps.shape[0]) - 0.5
                y = op.matvec(torch.from_numpy(x).cuda()).cpu().numpy()
                rows = np.sort(rng.choice(reps.shape[0], 2000, replace=False))
                rows[-1] = reps.shape[0] - 1   # the last state: bits 63 and 31 both set
                want = po.expected_rows(matrix, reps, x, rows)
                assert _close(y[rows], want), np.abs(y[rows] - want).max()
        finally:
            op.close()


@pytest.mark.gpu
def test_zz_correlations_over_64_bits(need_cuda):
    """zz_correlations on a 32-site spinful state: the 64 x 64 matrix over the bits against numpy over the states."""
    basis, matrix = _model(_hubbard_wide(32, 2, 1))
    states = _states_of(basis)
    op = Operator(matrix)
    try:
        op.basis.build()
        for cplx in (False, True):
            x = _x(states.shape[0], cplx, 5)
            Cz, m = op.zz_correlations(x)
            assert Cz.shape == (64, 64)
            bits = ((states[:, None] >> np.arange(64, dtype=np.uint64)[None, :]) & np.uint64(1)).astype(float)
            sz = 2 * bits - 1
            w = np.abs(x) ** 2 / np.vdot(x, x).real
            assert np.abs(Cz - (sz * w[:, None]).T @ sz).max() < 1e-12, cplx
            assert np.abs(m - w @ sz).max() < 1e-12, cplx
    finally:
        op.close()
