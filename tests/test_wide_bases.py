"""Bases of 40 to 64 sites and every lattice shape the group compiler recognises, on the device.

The library takes up to 64 sites (one 64-bit word per state).  The models here reach the canonical forms and kernel
instances that the 36-site models of the other files do not: min_rotation_dihedral<uint64_t> (the __brevll branch) and
min_rotation_runs at 40 - 64 sites, the rectangular torus (orbit_min_torus, tor_mode 1), the square torus at K = 5
(tor_mode 2 outside the TK builds), the tori without a pair table (min_rotation_blocks: 8 x 8, 7 x 3), tori with
translations only, the generic walk of a torus with x-translations only, representatives at the top of the key range
(the mirror-only ring at weights 62 and 63), k_gather and the combinadic rank at 64 sites, k_zz_gram with 6 - 8 column
tiles and 4 - 5 row tiles, k_pm_rows over several passes of classes and k_pm_pairs with up to 4032 classes.

References: the CPU oracle (oracle/oracle.c) on every model, and where the sector is small enough the sector reference
of oracle/sector_pin.py (the sector-restricted twin of dense_pin: H and the symmetry-adapted basis built explicitly),
which the CPU tests below pin against dense_pin at 12 - 16 sites and then use to pin the oracle at 40 - 64 sites.
Criterion for products: _close of test_gpu_parity; correlations to 1e-12.

At 64 sites the key ~0 is a state, so it cannot mark a free slot: those bases take the dense ordered table in k_rows
and the flip-flop look-ups whatever the table options, and batched products go vector by vector (no k_rows_batch);
info("rows_dense_order_on") reports it.
"""
import ctypes as C
import functools
import os
from math import comb

import numpy as np
import pytest

from distributed_matvec_b200 import EmulatedCluster, Operator, block_to_hashed, hashed_to_block
from distributed_matvec_b200 import _native as nat
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
from oracle import pyoracle as po
from oracle import sector_pin as spin
from test_gpu_parity import _close, _x
from test_host import _torus_generators

FULL = 2**64 - 1


# ---- models ---------------------------------------------------------------------------------------------------------

def _heisenberg(bonds):
    return [{"expression": f"σ{c}₀ σ{c}₁", "sites": bonds} for c in "ˣʸᶻ"]


def _ring_bonds(n):
    return [[i, (i + 1) % n] for i in range(n)]


def _torus_bonds(k, R):
    bonds = [[k * y + x, k * y + (x + 1) % k] for y in range(R) for x in range(k)]
    return bonds + [[k * y + x, k * ((y + 1) % R) + x] for y in range(R) for x in range(k)]


def _ring_gens(n, translations=True, mirror=True, sector=0):
    gens = [{"permutation": [(i + 1) % n for i in range(n)], "sector": sector}] if translations else []
    if mirror:
        gens.append({"permutation": [n - 1 - i for i in range(n)], "sector": 0})
    return gens


# name -> (sites, weight, generators, bonds, expected branch)
# expected branch: (canon_mode, torus_mode, rows_tk) on the device; None: no permutation symmetries (k_gather)
MODELS = {}


def _add(name, n, w, gens, bonds, branch):
    MODELS[name] = (n, w, gens, bonds, branch)


for n in (40, 48, 64):
    for w in (2, 3, 4):
        _add(f"ring{n}_dihedral_w{w}", n, w, _ring_gens(n), _ring_bonds(n), (2, 0, 0))
for w in (2, 3):
    _add(f"ring64_translations_w{w}", 64, w, _ring_gens(64, mirror=False), _ring_bonds(64), (2, 0, 0))
    _add(f"ring64_momentum5_w{w}", 64, w, _ring_gens(64, mirror=False, sector=5), _ring_bonds(64), (0, 0, 0))
for k, R in ((4, 6), (6, 4), (3, 8)):
    for w in range(4, 13):
        _add(f"torus{k}x{R}_w{w}", k * R, w, _torus_generators(k, R), _torus_bonds(k, R), (1, 1, 0))
for w in (3, 4, 13):
    _add(f"torus5x5_w{w}", 25, w, _torus_generators(5, 5), _torus_bonds(5, 5), (1, 2, 0))
for w in (2, 3):
    _add(f"torus6x8_w{w}", 48, w, _torus_generators(6, 8), _torus_bonds(6, 8), (1, 1, 0))
    _add(f"torus8x8_w{w}", 64, w, _torus_generators(8, 8), _torus_bonds(8, 8), (1, 0, 0))
    _add(f"torus6x8_translations_w{w}", 48, w, _torus_generators(6, 8, False), _torus_bonds(6, 8), (1, 0, 0))
for w in (3, 5, 10):
    _add(f"torus7x3_w{w}", 21, w, _torus_generators(7, 3), _torus_bonds(7, 3), (1, 0, 0))
_add("torus4x4_translations_w8", 16, 8, _torus_generators(4, 4, False), _torus_bonds(4, 4), (1, 0, 0))
for w in (6, 8):
    _add(f"torus4x4_xtranslations_w{w}", 16, w, _torus_generators(4, 4, False)[:1], _torus_bonds(4, 4), (0, 0, 0))
for w in (62, 63):
    _add(f"ring64_mirror_w{w}", 64, w, _ring_gens(64, translations=False), _ring_bonds(64), (0, 0, 0))
for n in (44, 48, 56, 63, 64):
    for w in (2, 3):
        _add(f"plain{n}_w{w}", n, w, [], _ring_bonds(n), None)
for w in (62, 63):
    _add(f"plain64_w{w}", 64, w, [], _ring_bonds(64), None)

SYMMETRIC = [m for m in MODELS if MODELS[m][4] is not None]
PLAIN = [m for m in MODELS if MODELS[m][4] is None]


@functools.lru_cache(maxsize=None)
def _model(name):
    n, w, gens, bonds, _ = MODELS[name]
    spec = {"number_spins": n, "hamming_weight": w}
    if gens:
        spec["symmetries"] = gens
    basis = basis_from_dict(spec)
    terms = _heisenberg(bonds)
    return basis, operator_from_dict({"terms": terms}, basis), terms


def _ref_fits(name):
    basis, _, _ = _model(name)
    g = len(basis.group) if basis.requires_projection() else 1
    return g * comb(basis.number_sites, basis.hamming_weight) <= spin.MAX_IMAGES


@functools.lru_cache(maxsize=None)
def _sector(name):
    basis, _, terms = _model(name)
    return spin.Sector(basis, terms)


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """(representatives, norms, {cplx: (x, y = H x)}) from the CPU oracle"""
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    basis, matrix, _ = _model(name)
    reps, norms = po.enumerate_states(basis)
    ys = {}
    for cplx in (False, True):
        x = _x(reps.shape[0], cplx, 71)
        ys[cplx] = (x, po.matvec_global(matrix, reps, x, 1, num_tasks=po.num_threads()))
    return reps, norms, ys


def _compile_info(basis):
    """dmv_debug_compile_group's description of the orbit program: [canon mode, k, R, pair table, ..., tor_mode at 12,
    chain mirror form at 15]"""
    g = basis.group
    bd = nat.BasisDesc()
    bd.number_sites, bd.hamming_weight, bd.spin_inversion, bd.has_permutations = (
        basis.number_sites, -1 if basis.hamming_weight is None else basis.hamming_weight, basis.spin_inversion, 1)
    keep = (np.ascontiguousarray(g.perms), np.ascontiguousarray(g.flips), np.ascontiguousarray(g.characters))
    bd.group_order, bd.perms, bd.flips, bd.characters = len(g), keep[0].ctypes.data, keep[1].ctypes.data, keep[2].ctypes.data
    ext = np.zeros(16, dtype=np.int64)
    nat.check(nat.lib().dmv_debug_compile_group(C.byref(bd), ext.ctypes.data, -2, None, None, None))
    return ext


# ---- CPU: the sector reference, the oracle at width, the compiled branches ------------------------------------------

PIN_MODELS = {
    "ring14_dihedral_w5": (14, 5, _ring_gens(14), _ring_bonds(14)),
    "ring12_momentum1_w4": (12, 4, _ring_gens(12, mirror=False, sector=1), _ring_bonds(12)),
    "ring16_momentum3_w6": (16, 6, _ring_gens(16, mirror=False, sector=3), _ring_bonds(16)),
    "torus4x4_w6": (16, 6, _torus_generators(4, 4), _torus_bonds(4, 4)),
    "torus4x3_w5": (12, 5, _torus_generators(4, 3), _torus_bonds(4, 3)),
    "ring14_inversion_w7": (14, 7, _ring_gens(14), _ring_bonds(14)),
    "plain13_w4": (13, 4, [], _ring_bonds(13)),
}


@pytest.mark.parametrize("name", sorted(PIN_MODELS))
def test_sector_reference_matches_dense_pin(name):
    """The sector reference equals dense_pin (full 2^n space, Kronecker products) at 12 - 16 sites: representatives,
    norms and Hp to 1e-12, complex characters and a flip-free group included; plus a field term that leaves the
    sector (σ⁺), which the sector restriction drops like B^dagger H B does."""
    from oracle import dense_pin as dp
    n, w, gens, bonds = PIN_MODELS[name]
    spec = {"number_spins": n, "hamming_weight": w}
    if name == "ring14_inversion_w7":
        spec["spin_inversion"] = -1
    if gens:
        spec["symmetries"] = gens
    basis = basis_from_dict(spec)
    terms = _heisenberg(bonds) + [{"expression": "0.3 × σᶻ₀ σᶻ₁", "sites": [[i, (i + 2) % n] for i in range(n)]},
                                  {"expression": "0.7 × σ⁺₀", "sites": [[i] for i in range(n)]}]
    reps, norms, Hp = dp.projected_hamiltonian(terms, basis)
    S = spin.Sector(basis, terms)
    assert np.array_equal(S.reps, reps)
    assert np.allclose(S.norms, norms, rtol=0, atol=1e-14)
    assert np.abs(S.Hp.toarray() - Hp).max() <= 1e-12
    x = _x(reps.shape[0], True, 5)
    assert np.allclose(S.psi(x), dp.symmetry_adapted_basis(basis)[2][S.states.astype(np.int64)] @ x, atol=1e-14)


ORACLE_PINS = ["ring40_dihedral_w3", "ring40_dihedral_w4", "ring48_dihedral_w3", "ring64_dihedral_w3",
               "ring64_momentum5_w3", "ring64_translations_w2", "torus6x8_w3", "torus8x8_w2", "torus6x8_translations_w3",
               "ring64_mirror_w62", "ring64_mirror_w63", "plain64_w3", "plain64_w63", "plain44_w3"]


@pytest.mark.parametrize("name", ORACLE_PINS)
def test_oracle_matches_sector_reference_at_width(name):
    """The oracle's enumeration (representatives bit for bit, norms) and product (float64 and complex128) against the
    sector reference at 40 - 64 sites, where nothing else pins the oracle."""
    basis, matrix, _ = _model(name)
    S = _sector(name)
    reps, norms = po.enumerate_states(basis)
    assert np.array_equal(reps, S.reps)
    if basis.requires_projection():
        assert np.allclose(norms, S.norms, rtol=0, atol=1e-14)
    for cplx in (False, True):
        x = _x(reps.shape[0], cplx, 9)
        y = po.matvec_global(matrix, reps, x, 1)
        want = S.Hp @ x if cplx else (S.Hp @ x).real   # a real vector takes the real part of the product
        assert _close(y, want), (cplx, np.abs(y - want).max())


def test_compiled_branches():
    """Which canonical form the group compiler picks for each shape (dmv_debug_compile_group on the host):
    canon mode 2 = one block of rotations (rings), 1 = R x k blocks (tori), 0 = the walk; the pair table (2k <= 12);
    tor_mode 1 = rectangular torus, 2 = square torus (orbit_min_torus), 0 = none; the chains' zero-run search (1:
    rotations, 2: rotations and the mirror in one pass)."""
    expect = {   # (canon mode, k, R, pair table, tor_mode, chain runs form)
        "ring40_dihedral_w2": (2, 40, 1, 0, 0, 2), "ring48_dihedral_w2": (2, 48, 1, 0, 0, 2),
        "ring64_dihedral_w2": (2, 64, 1, 0, 0, 2), "ring64_translations_w2": (2, 64, 1, 0, 0, 1),
        "ring64_momentum5_w2": (0, 0, 0, 0, 0, 0),   # complex characters: the orbit scan
        "torus4x6_w4": (1, 4, 6, 1, 1, 0), "torus6x4_w4": (1, 6, 4, 1, 1, 0), "torus3x8_w4": (1, 3, 8, 1, 1, 0),
        "torus5x5_w3": (1, 5, 5, 1, 2, 0), "torus6x8_w2": (1, 6, 8, 1, 1, 0),
        "torus8x8_w2": (1, 8, 8, 0, 0, 0), "torus7x3_w3": (1, 7, 3, 0, 0, 0),   # no pair table: min_rotation_blocks
        "torus6x8_translations_w2": (1, 6, 8, 1, 0, 0), "torus4x4_translations_w8": (1, 4, 4, 1, 0, 0),
        "torus4x4_xtranslations_w6": (0, 0, 0, 0, 0, 0), "ring64_mirror_w62": (0, 0, 0, 0, 0, 0)}
    for name, want in expect.items():
        ext = _compile_info(_model(name)[0])
        got = tuple(int(v) for v in (ext[6], ext[7], ext[8], ext[9], ext[12], ext[15]))
        assert got == want, (name, got, [int(v) for v in ext])
    for name in SYMMETRIC:
        ext = _compile_info(_model(name)[0])
        assert (int(ext[6]), int(ext[12])) == MODELS[name][4][:2], (name, [int(v) for v in ext])


# ---- GPU ------------------------------------------------------------------------------------------------------------

torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _product(op, x):
    y = op.matvec(torch.from_numpy(x).cuda())
    torch.cuda.synchronize()
    return y.cpu().numpy()


def _set(op, **options):
    for k, v in options.items():
        op.set_option(k, v)


# k_rows tables: the dense ordered one (the default), the ordered layout, the hashed one; every option set each time
TABLES = {"dense_ordered": dict(rows_index=-1, rows_table=1, rows_dense_order=-1),
          "ordered": dict(rows_index=-1, rows_table=1, rows_dense_order=0),
          "hashed": dict(rows_index=-1, rows_table=0, rows_dense_order=-1)}


def _check_rows(op, name, ys):
    """k_rows in every table x rows_ctas 2 / 3 / auto x element type; bit-identity over rows_ctas on one table build"""
    n = MODELS[name][0]
    tk = MODELS[name][4][2]
    for table, options in TABLES.items():
        _set(op, **options)
        for cplx in (False, True):
            x, y_ref = ys[cplx]
            first = None
            for ctas in (2, 3, -1):
                op.set_option("rows_ctas", ctas)
                y = _product(op, x)
                where = (name, table, cplx, ctas)
                assert op.info("rows") == 1 and op.info("rows_tk") == tk, where
                # 64 sites: the dense ordered table whatever the options (~0 is a state, not a free-slot marker)
                assert op.info("rows_dense_order_on") == (1 if table == "dense_ordered" or n == 64 else 0), where
                assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
                if first is None:
                    first = y
                assert np.array_equal(y, first), (where, np.abs(y - first).max())
    _set(op, rows_ctas=-1, **TABLES["dense_ordered"])


def _check_batch(op, name, reps, matrix):
    """matvec_batch with 1 .. 6 float64 and 1 .. 3 complex128 columns, every column against the oracle"""
    n = reps.shape[0]
    for cplx, most in ((False, 6), (True, 3)):
        X = np.stack([_x(n, cplx, 600 + j) for j in range(most)])
        want = [po.matvec_global(matrix, reps, X[j], 1, num_tasks=po.num_threads()) for j in range(most)]
        for k in range(1, most + 1):
            Y = op.matvec_batch(torch.from_numpy(X[:k]).cuda())
            torch.cuda.synchronize()
            Y = Y.cpu().numpy()
            for j in range(k):
                assert _close(Y[j], want[j]), (name, cplx, k, j, np.abs(Y[j] - want[j]).max())


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(MODELS))
def test_products_on_wide_and_shaped_bases(need_cuda, name):
    """Enumeration (representatives bit for bit, norms) and the product in full vector against the oracle, and
    against Hp x of the sector reference where it is built: k_rows in every table and CTA count, k_rows_batch, the
    queued k_pull (rows = 0) and k_generate (mode = 0) on symmetric bases; k_gather with every index on the others.
    The canonical form, torus form and k_rows build each model takes are asserted."""
    basis, matrix, _ = _model(name)
    reps, norms, ys = _oracle(name)
    if _ref_fits(name):
        S = _sector(name)
        assert np.array_equal(S.reps, reps)
        for cplx in (False, True):
            x, y_ref = ys[cplx]
            assert _close(S.Hp @ x if cplx else (S.Hp @ x).real, y_ref), (name, cplx)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        branch = MODELS[name][4]
        if branch is None:
            assert op.info("gather") == 1, name
            for index in (-1, 2, 0):
                op.set_option("index", index)
                for cplx in (False, True):
                    x, y_ref = ys[cplx]
                    assert _close(_product(op, x), y_ref), (name, index, op.info("index_mode"), cplx)
                    assert _close(op.matvec(x), y_ref), (name, index, cplx)
            if basis.number_sites == 64:
                op.set_option("index", 2)
                assert op.info("index_mode") == 2   # the combinadic rank at 64 sites
            return
        assert np.allclose(op.basis.norms(), norms, rtol=0, atol=1e-15)
        assert (op.info("canon_mode"), op.info("torus_mode")) == branch[:2], (name, op.info("canon_mode"),
                                                                             op.info("torus_mode"))
        trivial = basis.group.all_characters_trivial
        assert op.info("rows_ok") == (1 if trivial else 0), name
        if trivial:
            _check_rows(op, name, ys)
            _check_batch(op, name, reps, matrix)
        for options in (dict(mode=1, rows=0), dict(mode=0, rows=-1)):
            _set(op, **options)
            assert op.info("rows") == 0
            for cplx in (False, True):
                x, y_ref = ys[cplx]
                y = _product(op, x)
                assert _close(y, y_ref), (name, options, cplx, np.abs(y - y_ref).max())
    finally:
        op.close()


THREE_RANKS = ["ring64_dihedral_w3", "ring48_dihedral_w4", "ring64_momentum5_w3", "torus4x6_w8", "torus5x5_w4",
               "torus8x8_w3", "torus7x3_w5", "torus4x4_xtranslations_w6", "ring64_mirror_w63", "plain64_w63",
               "plain56_w3"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", THREE_RANKS)
def test_three_ranks_on_wide_and_shaped_bases(need_cuda, name):
    """Three emulated ranks: the hash partition of the enumeration, and the record exchange and the replicated-x
    product against the oracle's 3-rank product, float64 and complex128."""
    P = 3
    _, matrix, _ = _model(name)
    reps, _, ys = _oracle(name)
    masks, blocks = po.partition_by_hash(reps, P)
    cl = EmulatedCluster(matrix, P).build()
    try:
        for r, blk in enumerate(cl.representatives()):
            assert np.array_equal(blk, blocks[r]), r
        for cplx in (False, True):
            x = ys[cplx][0]
            y_ref = po.matvec_global(matrix, reps, x, P, num_tasks=po.num_threads())
            xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
            y_rec = hashed_to_block([t.cpu().numpy() for t in cl.matvec(xb)], masks)
            assert _close(y_rec, y_ref), (name, cplx, np.abs(y_rec - y_ref).max())
            y_rep = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)
            assert _close(y_rep, y_ref), (name, cplx, np.abs(y_rep - y_ref).max())
    finally:
        cl.close()


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [False, True])
def test_weights_at_the_ends_of_64_sites(need_cuda, symmetric):
    """Weights 0, 1, 63 and 64 on 64 sites, with and without the dihedral group: the enumeration equals the oracle's
    (the one state of weight 64 is ~0) and the product equals the oracle's."""
    for w in (0, 1, 63, 64):
        spec = {"number_spins": 64, "hamming_weight": w}
        if symmetric:
            spec["symmetries"] = _ring_gens(64)
        basis = basis_from_dict(spec)
        matrix = operator_from_dict({"terms": _heisenberg(_ring_bonds(64))}, basis)
        reps, _ = po.enumerate_states(basis)
        op = Operator(matrix)
        try:
            op.basis.build()
            assert np.array_equal(op.basis.representatives(), reps), w
            if w == 64:
                assert reps.tolist() == [FULL]
            for cplx in (False, True):
                x = _x(reps.shape[0], cplx, 3)
                y_ref = po.matvec_global(matrix, reps, x, 1)
                assert _close(_product(op, x), y_ref), (w, symmetric, cplx)
        finally:
            op.close()


STATE_INFO_SHAPES = [(5, 1, None), (7, 1, 1), (12, 1, 1), (33, 1, 1), (40, 1, None), (64, 1, 1), (2, 2, 1), (3, 2, None),
                     (4, 3, 1), (5, 5, 1), (6, 4, None), (4, 8, 1), (6, 6, 1), (6, 6, None), (3, 3, 1), (4, 4, None),
                     (6, 8, 1), (3, 8, None), (5, 4, 1), (7, 3, 1), (8, 8, 1), (8, 2, None), (16, 2, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("k,R,inversion", STATE_INFO_SHAPES)
def test_state_info_on_device_on_random_lattices(need_cuda, k, R, inversion):
    """dmv_state_info on the device against the oracle for the chains and tori of
    test_host.test_block_rotation_canonical_form_on_random_lattices, with the same random, sparse and tied-row
    states: the device build of orbit_representative and the canonical forms it calls."""
    n = k * R
    basis = basis_from_dict({"number_spins": n, "hamming_weight": None, "spin_inversion": inversion,
                             "symmetries": _torus_generators(k, R)})
    matrix = operator_from_dict({"terms": _heisenberg(_ring_bonds(n))}, basis)
    rng = np.random.default_rng(k * 100 + R)
    hi = 2**n if n < 64 else 2**63
    mask = 2**n - 1 if n < 64 else FULL
    states = rng.integers(0, hi, size=1500, dtype=np.uint64)
    if n == 64:
        states |= rng.integers(0, 2, size=1500, dtype=np.uint64) << np.uint64(63)
    states[:6] = [0, mask, 1, 0x5555555555555555 & mask, 1 << (n - 1), 3]
    states[6:300] &= rng.integers(0, hi, size=294, dtype=np.uint64)
    if R > 1:
        bm = (1 << k) - 1
        for j in range(300, 600):
            rows = rng.integers(0, bm + 1, size=2)
            pattern = [int(rows[(y * int(rng.integers(1, 3))) % 2]) for y in range(R)]
            states[j] = sum(r << (k * y) for y, r in enumerate(pattern)) & mask
        if R == k:
            for j in range(600, 800):
                m = rng.integers(0, 2, size=(k, k))
                m = np.triu(m) | np.triu(m, 1).T
                states[j] = sum(int(m[y, a]) << (k * y + a) for y in range(R) for a in range(k))
    op = Operator(matrix)
    try:
        b, c, nrm = op.basis.stateInfo(states)
        ob, oc, on = po.state_info(basis, states)
        assert np.array_equal(b, ob), (k, R, np.nonzero(b != ob)[0][:5])
        ok = on > 0
        assert np.allclose(c[ok], oc[ok], atol=1e-15)
        assert np.allclose(nrm, on, atol=1e-15)
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["plain44_w3", "plain48_w2", "plain56_w3", "plain63_w2", "plain64_w3", "plain64_w62",
                                  "ring64_dihedral_w3", "torus8x8_w2"])
def test_zz_correlations_at_width(need_cuda, name):
    """<σᶻᵢσᶻⱼ> and <σᶻᵢ> against psi = B x of the sector reference to 1e-12, at 44 - 64 sites (k_zz_gram with 6, 7
    and 8 column tiles and 3 - 5 row tiles), real and complex x"""
    _, matrix, _ = _model(name)
    S = _sector(name)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), S.reps)
        for cplx in (False, True):
            x = _x(S.reps.shape[0], cplx, 13)
            Cz, m = op.zz_correlations(x)
            C_ref, m_ref = S.zz(x)
            assert np.abs(Cz - C_ref).max() <= 1e-12, (name, cplx, np.abs(Cz - C_ref).max())
            assert np.abs(m - m_ref).max() <= 1e-12, (name, cplx)
    finally:
        op.close()


PM_MODELS = ["torus4x4_xtranslations_w6", "torus4x4_xtranslations_w8", "ring64_translations_w2",
             "ring64_dihedral_w2", "ring64_momentum5_w2", "torus6x8_translations_w2", "plain64_w2", "plain63_w3",
             "ring64_mirror_w62"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", PM_MODELS)
def test_pm_correlations_over_several_passes(need_cuda, name):
    """<σ⁺ᵢσ⁻ⱼ> against psi = B x of the sector reference to 1e-12, float64 and complex128 x: k_pm_rows with more
    classes than one pass holds (60 on the 4 x 4 torus with x-translations only, 63 on the 64-site ring with
    translations, 32 with the dihedral group: two complex passes), complex characters, k_pm_pairs with 4032 classes
    (the 64-site ring without symmetries), and the mirror-only ring whose representatives lie at the top of the key
    range.  The 4 x 4 models are also pinned by the full-space formula of test_pm_correlations."""
    _, matrix, _ = _model(name)
    S = _sector(name)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), S.reps)
        for cplx in (False, True):
            x = _x(S.reps.shape[0], cplx, 17)
            T = op.pm_correlations(x)
            T_ref = S.pm(x)
            assert np.abs(T - T_ref).max() <= 1e-12, (name, cplx, np.abs(T - T_ref).max())
            if S.n == 16:
                from oracle import dense_pin as dp
                from test_pm_correlations import _full_space
                basis = _model(name)[0]
                T_full = _full_space(dp.symmetry_adapted_basis(basis)[2], x, 16)
                assert np.abs(T - T_full).max() <= 1e-12
    finally:
        op.close()


@pytest.mark.gpu
def test_eigsh_on_the_64_site_ring(need_cuda):
    """Operator.eigsh(3) on the 64-site dihedral ring at weight 2 against eigh of the sector reference's Hp"""
    name = "ring64_dihedral_w2"
    _, matrix, _ = _model(name)
    S = _sector(name)
    want = np.linalg.eigvalsh(S.Hp.toarray())[:3]
    op = Operator(matrix)
    try:
        op.basis.build()
        evals, vecs, res, conv, _, _ = op.eigsh(3)
        assert conv == 3
        assert np.abs(evals - want).max() <= 1e-9 * max(1.0, np.abs(want).max()), (evals, want)
    finally:
        op.close()


def _raising_ring(w, sites=64, translations=True):
    """The ring with translations (else the mirror alone) at weight w plus Σᵢ σ⁺ᵢ: at w = 63 every row also sends to ~0"""
    gens = _ring_gens(sites, mirror=not translations, translations=translations)
    basis = basis_from_dict({"number_spins": sites, "hamming_weight": w, "symmetries": gens})
    terms = _heisenberg(_ring_bonds(sites)) + [{"expression": "σ⁺₀", "sites": [[i] for i in range(sites)]}]
    return basis, operator_from_dict({"terms": terms}, basis)


PATHS = {"dense_ordered": dict(), "ordered": dict(rows_dense_order=0), "hashed": dict(rows_table=0),
         "perfect_hash": dict(rows_index=1), "pull": dict(mode=1, rows=0), "generate": dict(mode=0)}


@pytest.mark.gpu
def test_missing_all_up_state_is_an_error(need_cuda):
    """The 64-site ring with translations at weight 63 and a σ⁺ field: every row sends to ~0, which is not a basis
    state.  Every product path and table option, host and device vectors, the batched product and both three-rank
    forms (on the mirror-only ring, which has a state for every rank) raise "invalid index" -- ~0 must not be taken
    for the free-slot marker of a table."""
    basis, matrix = _raising_ring(63)
    reps, _ = po.enumerate_states(basis)
    for path, options in PATHS.items():
        op = Operator(matrix)
        try:
            _set(op, **options)
            op.basis.build()
            assert np.array_equal(op.basis.representatives(), reps)
            for cplx in (False, True):
                x = _x(reps.shape[0], cplx, 5)
                with pytest.raises(Exception, match="invalid index"):
                    op.matvec(x)
                with pytest.raises(Exception, match="invalid index"):
                    op.matvec(torch.from_numpy(x).cuda())
                    op.synchronize()
            if path == "dense_ordered":
                with pytest.raises(Exception, match="invalid index"):
                    op.matvec_batch(torch.from_numpy(np.stack([_x(reps.shape[0], False, j) for j in range(4)])).cuda())
                    op.synchronize()
        finally:
            op.close()
    # three ranks need a state each: the mirror-only ring has 32 representatives at weight 63
    basis, matrix = _raising_ring(63, translations=False)
    reps, _ = po.enumerate_states(basis)
    masks, _ = po.partition_by_hash(reps, 3)
    x = _x(reps.shape[0], False, 5)
    for form in ("matvec", "matvec_replicated"):
        cl = EmulatedCluster(matrix, 3).build()
        try:
            xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, 3)]
            with pytest.raises(Exception, match="invalid index"):
                getattr(cl, form)(xb)
                for op in cl.ops:
                    op.synchronize()
        finally:
            cl.close()


@pytest.mark.gpu
def test_all_up_state_in_the_basis(need_cuda):
    """The weight-64 sector, whose one representative is ~0: the product equals the oracle's, D x, in every path and
    table option."""
    basis = basis_from_dict({"number_spins": 64, "hamming_weight": 64, "symmetries": _ring_gens(64, mirror=False)})
    matrix = operator_from_dict({"terms": _heisenberg(_ring_bonds(64))}, basis)
    reps, _ = po.enumerate_states(basis)
    assert reps.tolist() == [FULL]
    for path, options in PATHS.items():
        op = Operator(matrix)
        try:
            _set(op, **options)
            op.basis.build()
            assert np.array_equal(op.basis.representatives(), reps)
            for cplx in (False, True):
                x = _x(1, cplx, 5)
                y_ref = po.matvec_global(matrix, reps, x, 1)
                assert _close(y_ref, 64.0 * x)   # 64 bonds of σᶻσᶻ = +1
                assert _close(_product(op, x), y_ref), (path, cplx)
        finally:
            op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n,weight", [(64, None), (63, None), (64, 32)])
def test_candidate_range_too_wide_is_an_error(need_cuda, n, weight):
    """dmv_basis_build refuses a candidate range it cannot enumerate (2^64 states at 64 sites without a fixed
    magnetisation used to wrap to an empty basis) with a message that says so"""
    basis = basis_from_dict({"number_spins": n, "hamming_weight": weight})
    matrix = operator_from_dict({"terms": _heisenberg(_ring_bonds(n))}, basis)
    op = Operator(matrix)
    try:
        with pytest.raises(Exception, match="cannot be enumerated"):
            op.basis.build()
    finally:
        op.close()
