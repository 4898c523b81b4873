"""Symmetric bases beyond the SU(2)-invariant flip-flop Hamiltonian: transverse-field Ising, anisotropic XY and J1-J2.

Every other symmetric model of the suite is a Heisenberg-like flip-flop operator at a fixed Hamming weight: k_rows then
only emits on antiparallel two-site pairs with one coefficient per group.  The models here exercise what k_rows accepts
beyond that: single-site flip masks (σˣ), emission on parallel pairs (σˣσˣ - σʸσʸ creates and annihilates pairs), a
coefficient that depends on the pair pattern within a group, single-site σᶻ terms, diagonal flip masks on the torus,
and bases that span every Hamming weight.

References that share no code with the library: the CPU oracle (oracle/pyoracle.py) for every product, the projected
Hamiltonian B^dagger H B of oracle/dense_pin.py for the solvers and observables, and two exact results for the sizes the
oracle cannot reach:
  * transverse-field Ising ring H = -sum σᶻσᶻ - h sum σˣ (Pfeuty 1970): in the sector k = 0, reflection +1, spin
    inversion +1 the lowest energy is E0 = -sum_{m=0}^{N-1} sqrt(1 + h^2 - 2 h cos(pi (2 m + 1) / N));
  * Majumdar-Ghosh H = sum σᵢ·σᵢ₊₁ + 1/2 sum σᵢ·σᵢ₊₂ at half filling: E0 = -3 N / 2, in the sector (k = 0, r = 0,
    inversion +1) for N = 0 mod 4.
Dimensions of free-weight sectors are pinned by Burnside's lemma.
"""
import functools
import os

import numpy as np
import pytest

from distributed_matvec_b200 import BatchedOperator, EmulatedCluster, Operator, block_to_hashed, hashed_to_block
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
from distributed_matvec_b200.thermal import seeded_start_vectors
from oracle import dense_pin as dp
from oracle import pyoracle as po
from test_gpu_parity import _close, _x
from test_pm_correlations import _full_space as _pm_full_space
from test_rows_kernels import CTAS, TABLES
from test_zz_correlations import _full_space as _zz_full_space

torch = pytest.importorskip("torch")

TFIM_H = 0.7


# ---- lattices and models

def _chain_group(n, k=0, r=0):
    """translations in momentum sector k, and the reflection in sector r where it commutes with them (k = 0, n / 2)"""
    out = [{"permutation": [(i + 1) % n for i in range(n)], "sector": k}]
    if 2 * k % n == 0:
        out.append({"permutation": [n - 1 - i for i in range(n)], "sector": r})
    return out


def _torus_group(side):
    """translations x, y, reflections x, y and the diagonal mirror of the side x side torus (the full space group)"""
    n = side * side
    gens = [[side * (i // side) + (i % side + 1) % side for i in range(n)], [(i + side) % n for i in range(n)],
            [side * (i // side) + side - 1 - i % side for i in range(n)],
            [side * (side - 1 - i // side) + i % side for i in range(n)], [side * (i % side) + i // side for i in range(n)]]
    return [{"permutation": p, "sector": 0} for p in gens]


def _torus_bonds(side, diagonal=False):
    out = []
    for y in range(side):
        for a in range(side):
            s = side * y + a
            up = side * ((y + 1) % side)
            out += ([[s, up + (a + 1) % side], [s, up + (a - 1) % side]] if diagonal else
                    [[s, side * y + (a + 1) % side], [s, up + a]])
    return out


def _ring(n, d=1):
    return [[i, (i + d) % n] for i in range(n)]


def _tfim_terms(n, h, bonds):
    terms = [{"expression": f"-{h} × σˣ₀", "sites": [[i] for i in range(n)]}]
    if bonds:
        terms.insert(0, {"expression": "-1 × σᶻ₀ σᶻ₁", "sites": bonds})
    return terms


def _xy_terms(n, gamma=0.4):
    return [{"expression": f"{(1 + gamma) / 2} × σˣ₀ σˣ₁", "sites": _ring(n)},
            {"expression": f"{(1 - gamma) / 2} × σʸ₀ σʸ₁", "sites": _ring(n)},
            {"expression": "0.3 × σᶻ₀ σᶻ₁", "sites": _ring(n, 2)}]


def _j1j2_terms(side, delta=0.7, j2=0.55, field=0.2):
    b1, b2 = _torus_bonds(side), _torus_bonds(side, True)
    return ([{"expression": f"σ{c}₀ σ{c}₁", "sites": b1} for c in "ˣʸ"] +
            [{"expression": f"{delta} × σᶻ₀ σᶻ₁", "sites": b1}] +
            [{"expression": f"{j2} × σ{c}₀ σ{c}₁", "sites": b2} for c in "ˣʸᶻ"] +
            [{"expression": f"{field} × σᶻ₀", "sites": [[i] for i in range(side * side)]}])


def _mg_terms(n):
    return [{"expression": f"{J} × σ{c}₀ σ{c}₁", "sites": _ring(n, d)} for d, J in ((1, 1.0), (2, 0.5)) for c in "ˣʸᶻ"]


def _spec(name):
    """-> (basis dict, term specs, expected kernel: "rows" / "push")"""
    parts = name.split("_")
    if parts[0] in ("tfim", "field") and parts[1] == "chain":     # tfim_chain_<n>_k<k>_r<r>_inv<+-1>
        n, k, r, inv = int(parts[2]), int(parts[3][1:]), int(parts[4][1:]), int(parts[5][3:])
        b = {"number_spins": n, "hamming_weight": None, "spin_inversion": inv, "symmetries": _chain_group(n, k, r)}
        terms = _tfim_terms(n, TFIM_H, _ring(n) if parts[0] == "tfim" else None)
        return b, terms, "rows" if (k, r, inv) == (0, 0, 1) else "push"
    if parts[0] == "tfim":                                            # tfim_4x4_inv<+-1>
        inv = int(parts[2][3:])
        b = {"number_spins": 16, "hamming_weight": None, "spin_inversion": inv, "symmetries": _torus_group(4)}
        return b, _tfim_terms(16, 3.0, _torus_bonds(4)), "rows" if inv == 1 else "push"
    if parts[0] == "xy":                                              # xy_chain_12_inv<+-1>
        inv = int(parts[3][3:])
        b = {"number_spins": 12, "hamming_weight": None, "spin_inversion": inv, "symmetries": _chain_group(12)}
        return b, _xy_terms(12), "rows" if inv == 1 else "push"
    if parts[0] == "j1j2":                                            # j1j2_<side>x<side>_w<weight>
        side, w = int(parts[1].split("x")[0]), int(parts[2][1:])
        b = {"number_spins": side * side, "hamming_weight": w, "symmetries": _torus_group(side)}
        if 2 * w == side * side:      # the field sums to zero at half filling: spin inversion +1 is a symmetry there
            b["spin_inversion"] = 1
        return b, _j1j2_terms(side), "rows"
    if parts[0] == "mg":                                              # mg_chain_<n>: the _symm group of the chains
        n = int(parts[2])
        b = {"number_spins": n, "hamming_weight": n // 2, "spin_inversion": 1, "symmetries": _chain_group(n)}
        return b, _mg_terms(n), "rows"
    raise KeyError(name)


@functools.lru_cache(maxsize=None)
def _model(name):
    b, terms, kernel = _spec(name)
    basis = basis_from_dict(b)
    return basis, operator_from_dict({"terms": terms}, basis), terms, kernel


def _expected_tk(name):
    """rows_tk of the default k_rows build: the torus row form on the square tori, the generic walk on the chains"""
    if name.startswith("j1j2_6x6"):
        return 6
    return 4 if ("4x4" in name) else 0


# every model the oracle computes in about a second; the expected kernel and torus form follow from the name
SMALL = (["tfim_chain_10_k0_r0_inv1", "tfim_chain_12_k0_r0_inv1", "tfim_chain_14_k0_r0_inv1",
          "tfim_chain_12_k0_r0_inv-1", "tfim_chain_12_k1_r0_inv1", "field_chain_12_k0_r0_inv1",
          "tfim_4x4_inv1", "tfim_4x4_inv-1", "xy_chain_12_inv1", "xy_chain_12_inv-1",
          "mg_chain_16", "mg_chain_24"] +
         [f"j1j2_4x4_w{w}" for w in range(17)] + [f"j1j2_6x6_w{w}" for w in (2, 3, 4, 5, 6, 30, 31, 32, 33, 34)])
ROWS = [m for m in SMALL if _spec(m)[2] == "rows"]
# models small enough for the projected Hamiltonian on the full 2^n space
DENSE = ["tfim_chain_12_k0_r0_inv1", "tfim_chain_12_k1_r0_inv1", "field_chain_12_k0_r0_inv1", "tfim_4x4_inv1",
         "xy_chain_12_inv1", "xy_chain_12_inv-1", "j1j2_4x4_w8", "j1j2_4x4_w5", "mg_chain_16"]


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """representatives and (x, y = H x) of both element types from the CPU oracle"""
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    basis, matrix, _, _ = _model(name)
    reps, _ = po.enumerate_states(basis)
    ys = {}
    for cplx in (False, True):
        x = _x(reps.shape[0], cplx, 77)
        ys[cplx] = (x, po.matvec_global(matrix, reps, x, 1, num_tasks=po.num_threads()))
    return reps, ys


@functools.lru_cache(maxsize=None)
def _dense(name):
    _, _, terms, _ = _model(name)
    basis = _model(name)[0]
    reps, _, Hp = dp.projected_hamiltonian(terms, basis)
    _, _, B = dp.symmetry_adapted_basis(basis)
    return reps, Hp, B


def _tfim_exact(n, h):
    return -sum(np.sqrt(1 + h * h - 2 * h * np.cos(np.pi * (2 * m + 1) / n)) for m in range(n))


def _free_weight_dimension(basis):
    """Burnside over all Hamming weights: a permutation fixes 2^cycles states; with the global flip every cycle must
    have even length and alternate (2 choices each)"""
    import burnside
    g = basis.group
    total = 0
    for p, f in zip(np.asarray(g.perms), np.asarray(g.flips)):
        cycles = burnside.cycle_lengths(p)
        total += 0 if (f and any(c % 2 for c in cycles)) else 1 << len(cycles)
    assert total % len(g.perms) == 0
    return total // len(g.perms)


# ---- CPU: the outside numbers

@pytest.mark.parametrize("h", [0.5, 1.5])
@pytest.mark.parametrize("n", [6, 7, 8, 9, 10, 11, 12, 13, 14])
def test_tfim_formula_against_dense_eigh(n, h):
    """Pfeuty's E0 of the periodic transverse-field Ising chain in the sector (k = 0, r = +1, inversion +1), against
    eigh of the projected Hamiltonian built on the full 2^n space."""
    b = {"number_spins": n, "hamming_weight": None, "spin_inversion": 1, "symmetries": _chain_group(n)}
    basis = basis_from_dict(b)
    _, _, Hp = dp.projected_hamiltonian(_tfim_terms(n, h, _ring(n)), basis)
    e0 = np.linalg.eigvalsh(Hp)[0]
    assert abs(e0 - _tfim_exact(n, h)) <= 1e-12 * abs(e0), (n, h, e0, _tfim_exact(n, h))


@pytest.mark.parametrize("n", [8, 12, 16])
def test_majumdar_ghosh_energy_against_dense_eigh(n):
    """E0 = -3N/2 in the (k = 0, r = 0, inversion +1) sector at half filling."""
    b = {"number_spins": n, "hamming_weight": n // 2, "spin_inversion": 1, "symmetries": _chain_group(n)}
    basis = basis_from_dict(b)
    _, _, Hp = dp.projected_hamiltonian(_mg_terms(n), basis, dense=(n < 16))
    if n < 16:
        e0 = np.linalg.eigvalsh(Hp)[0]
    else:
        import scipy.sparse.linalg as sla
        e0 = sla.eigsh(Hp.real, k=1, which="SA", tol=1e-13)[0][0]
    assert abs(e0 + 1.5 * n) <= 1e-10 * n, (n, e0)


@pytest.mark.parametrize("name", [m for m in SMALL if "6x6" not in m and not m.startswith("mg_chain_24")])
def test_free_weight_dimension_by_burnside(name):
    """The oracle's enumeration of each free-weight sector (and each fixed weight) has Burnside's dimension; sectors
    with a non-trivial character are bounded by the orbit count."""
    import burnside
    basis, _, _, _ = _model(name)
    reps, norms = po.enumerate_states(basis)
    assert np.all(np.diff(reps.astype(np.int64)) > 0) and np.all(norms > 0)
    if basis.hamming_weight is None:
        count = _free_weight_dimension(basis)
    else:
        count = burnside.dimension(basis.group.perms, basis.group.flips, basis.hamming_weight)
    if basis.group.all_characters_trivial:
        assert reps.shape[0] == count, (name, reps.shape[0], count)
    else:
        assert 0 < reps.shape[0] <= count


def test_tfim_chain_32_dimension_by_burnside():
    """The at-size TFIM sector: 33 588 234 representatives over all Hamming weights."""
    basis = basis_from_dict({"number_spins": 32, "hamming_weight": None, "spin_inversion": 1,
                             "symmetries": _chain_group(32)})
    assert _free_weight_dimension(basis) == 33588234


# ---- GPU: small models against the oracle

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


@pytest.mark.gpu
@pytest.mark.parametrize("name", SMALL)
def test_basis_against_oracle(need_cuda, name):
    """Representatives bit-exact, stateIndex / stateInfo bit-exact, computeOffDiag as a multiset."""
    basis, matrix, _, _ = _model(name)
    reps, _ = _oracle(name)
    n_sites = basis.number_sites
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        rng = np.random.default_rng(3)
        probe = np.concatenate([reps, reps ^ np.uint64(1), rng.integers(0, 2**n_sites, 3000, dtype=np.uint64)])
        assert np.array_equal(op.basis.stateIndex(probe), po.state_index(reps, probe))
        alphas = rng.integers(0, 2**n_sites, 3000, dtype=np.uint64)
        b, c, nrm = op.basis.stateInfo(alphas)
        ob, oc, on = po.state_info(basis, alphas)
        assert np.array_equal(b, ob)
        ok = on > 0
        assert np.allclose(c[ok], oc[ok], atol=1e-15) and np.allclose(nrm, on, atol=1e-15)
        m = min(reps.shape[0], 512)
        bo = BatchedOperator(op, m)
        xs = _x(m, True, 5)
        cnt, betas, coeffs, _ = bo.computeOffDiag(m, reps[:m], xs)
        obeta, ocoef, _, _ = po.compute_off_diag(matrix, 1, reps[:m], xs)
        assert cnt == obeta.shape[0]
        order, oorder = np.lexsort((coeffs.imag, coeffs.real, betas)), np.lexsort((ocoef.imag, ocoef.real, obeta))
        assert np.array_equal(betas[order], obeta[oorder])
        assert np.allclose(coeffs[order], ocoef[oorder], rtol=1e-13, atol=1e-15)
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", SMALL)
def test_every_path_against_oracle(need_cuda, name):
    """The default selection (k_rows with its torus form, or the push path), then mode push / pull / queued pull, index
    -1 / 0 / 2 and canon -1 / 0 / 1 / 2, host and device pointers, float64 and complex128.  A canonical form that cannot
    serve the basis must refuse (an error) or report itself off (canon_mode); its product is checked either way."""
    basis, matrix, _, kernel = _model(name)
    reps, ys = _oracle(name)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert op.info("rows_ok") == (1 if kernel == "rows" else 0)
        assert op.info("rows") == (1 if kernel == "rows" else 0)
        if kernel == "rows":
            assert op.info("rows_tk") == _expected_tk(name)

        def check(where):
            for cplx in (False, True):
                x, y_ref = ys[cplx]
                y = op.matvec(x)
                assert _close(y, y_ref), (name, where, cplx, "host", np.abs(y - y_ref).max())
                y = _product(op, x)
                assert _close(y, y_ref), (name, where, cplx, "device", np.abs(y - y_ref).max())

        check("default")
        for mode, gather, rows in ((0, -1, -1), (1, -1, -1), (1, 0, 0)):
            _set(op, mode=mode, gather=gather, rows=rows)
            assert op.info("pull") == (0 if mode == 0 else 1)
            assert op.info("rows") == (1 if (mode == 1 and rows == -1 and kernel == "rows") else 0)
            for index in (-1, 0, 2):
                op.set_option("index", index)
                check(("mode", mode, rows, "index", index, op.info("index_mode")))
            op.set_option("index", -1)
        _set(op, mode=-1, gather=-1, rows=-1)
        for canon in (0, 1, 2, -1):
            try:
                op.set_option("canon", canon)
            except Exception:
                continue
            check(("canon", canon, op.info("canon_mode"), op.info("rows_tk")))
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ROWS)
def test_rows_tables_and_ctas(need_cuda, name):
    """k_rows: every table layout x rows_ctas x element type in full vector against the oracle; products that differ
    only in rows_ctas are bit-identical."""
    basis, matrix, _, _ = _model(name)
    reps, ys = _oracle(name)
    op = Operator(matrix)
    try:
        op.basis.build()
        tk = _expected_tk(name)
        for cplx in (False, True):
            x, y_ref = ys[cplx]
            for table, options in TABLES.items():
                _set(op, **options)
                first = None
                for ctas in CTAS:
                    op.set_option("rows_ctas", ctas)
                    y = _product(op, x)
                    where = (name, cplx, table, ctas)
                    assert op.info("rows") == 1, where
                    want_tk = 0 if (tk == 4 and ctas == 4 and table != "perfect_hash") else tk
                    assert op.info("rows_tk") == want_tk, (where, op.info("rows_tk"))
                    assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
                    if first is None:
                        first = y
                    else:
                        assert np.array_equal(y, first), where
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["tfim_chain_12_k0_r0_inv1", "field_chain_12_k0_r0_inv1", "tfim_4x4_inv1",
                                  "xy_chain_12_inv1", "xy_chain_12_inv-1", "j1j2_4x4_w7", "j1j2_6x6_w5"])
def test_matvec_batch(need_cuda, name):
    """matvec_batch with 1, 3, 6, 9 vectors (k_rows_batch on the k_rows models) against single-vector products, and
    every column against the oracle.  The pure field has no diagonal: y accumulates into Y."""
    basis, matrix, _, _ = _model(name)
    reps, _ = _oracle(name)
    n = reps.shape[0]
    accumulate = name.startswith("field")
    op = Operator(matrix)
    try:
        op.basis.build()
        for cplx in (False, True):
            X = np.stack([_x(n, cplx, 100 + j) for j in range(9)])
            Y0 = np.stack([_x(n, cplx, 200 + j) for j in range(9)]) if accumulate else np.zeros_like(X)
            want = [po.matvec_blocks(matrix, [reps], [X[j]], y_blocks=[Y0[j].copy()])[0] for j in range(9)]
            singles = np.stack([op.matvec(torch.from_numpy(X[j]).cuda(), torch.from_numpy(Y0[j].copy()).cuda())
                                .cpu().numpy() for j in range(9)])
            for j in range(9):
                assert _close(singles[j], want[j]), (name, cplx, j)
            for k in (1, 3, 6, 9):
                Y = op.matvec_batch(torch.from_numpy(X[:k]).cuda(), torch.from_numpy(Y0[:k].copy()).cuda())
                Y = Y.cpu().numpy()
                for j in range(k):
                    assert _close(Y[j], want[j]), (name, cplx, k, j, np.abs(Y[j] - want[j]).max())
                assert _close(Y, singles[:k])
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("num_ranks", [2, 3])
@pytest.mark.parametrize("name", ["tfim_chain_12_k0_r0_inv1", "tfim_chain_12_k1_r0_inv1", "tfim_4x4_inv1",
                                  "xy_chain_12_inv1", "j1j2_4x4_w6", "j1j2_6x6_w4", "mg_chain_16"])
def test_emulated_ranks(need_cuda, name, num_ranks):
    """Record exchange and replicated-x product on P logical ranks against the oracle's P-rank product."""
    basis, matrix, _, _ = _model(name)
    reps, _ = _oracle(name)
    masks, blocks = po.partition_by_hash(reps, num_ranks)
    cl = EmulatedCluster(matrix, num_ranks).build()
    try:
        for r, blk in enumerate(cl.representatives()):
            assert np.array_equal(blk, blocks[r])
        for cplx in (False, True):
            x = _x(reps.shape[0], cplx, 31)
            y_ref = po.matvec_global(matrix, reps, x, num_ranks, num_tasks=po.num_threads())
            xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, num_ranks)]
            y_rec = hashed_to_block([t.cpu().numpy() for t in cl.matvec(xb)], masks)
            assert _close(y_rec, y_ref), (name, cplx, np.abs(y_rec - y_ref).max())
            y_rep = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)
            assert _close(y_rep, y_ref), (name, cplx, np.abs(y_rep - y_ref).max())
    finally:
        cl.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", DENSE)
def test_solvers_and_observables_against_dense(need_cuda, name):
    """eigsh (4 lowest) against eigh; <σᶻσᶻ> and <σ⁺σ⁻> of the computed ground state against the state B x on the full
    space; quadrature moments sum w theta^p against <r|H^p|r>, p <= 3; expm_multiply against scipy's expm."""
    import scipy.linalg as sla
    basis, matrix, _, _ = _model(name)
    reps, Hp, B = _dense(name)
    cplx = not basis.group.all_characters_trivial or np.iscomplexobj(Hp) and np.abs(Hp.imag).max() > 0
    Hm = Hp if cplx else Hp.real
    w = np.linalg.eigvalsh(Hm)
    scale = max(1.0, np.abs(w).max())
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        vals, vecs, res, converged, _, _ = op.eigsh(4, tol=1e-12, complex_vectors=bool(cplx))
        assert converged
        assert np.abs(np.sort(vals) - w[:4]).max() <= 1e-9 * scale, (name, vals, w[:4])
        x = vecs[int(np.argmin(vals))]
        n_sites = basis.number_sites
        Cz, m = op.zz_correlations(x)
        Cz_ref, m_ref = _zz_full_space(basis, B, x)
        assert np.abs(Cz - Cz_ref).max() <= 1e-10 and np.abs(m - m_ref).max() <= 1e-10, name
        T = op.pm_correlations(x)
        T_ref = _pm_full_space(B, x, n_sites)
        assert np.abs(T - T_ref).max() <= 1e-10, (name, np.abs(T - T_ref).max())
        R = 3
        nodes, weights, _, _ = op.lanczos_quadrature(R, 8, seed=13, complex_vectors=bool(cplx))
        r = seeded_start_vectors(reps, R, 13, bool(cplx))
        for i in range(R):
            v, r2 = r[i].copy(), np.vdot(r[i], r[i]).real
            for p in range(4):
                got, want = weights[i] @ nodes[i] ** p, np.vdot(r[i], v).real
                assert abs(got - want) <= 1e-10 * scale ** p * r2, (name, i, p, got, want)
                v = Hm @ v
        x0 = _x(reps.shape[0], True, 19)
        for z in (-0.7j, -0.3):
            y, _, _ = op.expm_multiply(x0, z, tol=1e-12)
            y_ref = sla.expm(z * Hm) @ x0
            assert np.abs(y - y_ref).max() <= 1e-9 * np.abs(y_ref).max(), (name, z, np.abs(y - y_ref).max())
    finally:
        op.close()


# ---- GPU at size: the exact energies and sampled rows on bases the oracle cannot enumerate in full

@pytest.mark.gpu
def test_tfim_chain_32_at_size(need_cuda):
    """TFIM ring of 32 sites, sector (0, 0, +1), all Hamming weights: 33 588 234 states on k_rows; Lanczos within 1e-9
    relative of Pfeuty's energy at h = 0.5 and 1.5; 1024 sampled rows of the product against the oracle."""
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    n = 32
    b = {"number_spins": n, "hamming_weight": None, "spin_inversion": 1, "symmetries": _chain_group(n)}
    basis = basis_from_dict(b)
    for h in (0.5, 1.5):
        matrix = operator_from_dict({"terms": _tfim_terms(n, h, _ring(n))}, basis)
        op = Operator(matrix)
        try:
            op.basis.build()
            assert op.basis.numberStates() == 33588234
            assert op.info("rows") == 1
            if h == 0.5:
                reps = op.basis.representatives()
                rows = np.sort(np.random.default_rng(23).choice(reps.shape[0], size=1024, replace=False))
                x = _x(reps.shape[0], False, 7)
                y = op.matvec(torch.from_numpy(x).cuda())
                got = y[torch.from_numpy(rows).cuda()].cpu().numpy()
                del y
                want = po.expected_rows(matrix, reps, x, rows)
                assert _close(got, want), np.abs(got - want).max()
                del reps, x
            e, _, _, _ = op.lanczos(eigenvector=False, tol=1e-12)
            exact = _tfim_exact(n, h)
            assert abs(e - exact) <= 1e-9 * abs(exact), (h, e, exact)
        finally:
            op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("n,states,cplx", [(32, 4707969, False), (36, 63068876, True)])
def test_majumdar_ghosh_at_size(need_cuda, n, states, cplx):
    """Majumdar-Ghosh on the chain_32_symm / chain_36_symm bases: E0 = -3N/2 within 1e-9 relative."""
    basis, matrix, _, _ = _model(f"mg_chain_{n}")
    op = Operator(matrix)
    try:
        op.basis.build()
        assert op.basis.numberStates() == states
        assert op.info("rows") == 1
        e, _, _, _ = op.lanczos(eigenvector=False, tol=1e-12, complex_vectors=cplx)
        assert abs(e + 1.5 * n) <= 1e-9 * 1.5 * n, (n, e)
    finally:
        op.close()


@pytest.mark.gpu
def test_j1j2_6x6_at_size(need_cuda):
    """J1-J2 + XXZ + field on the 6x6 torus at half filling (the bench basis, 15 804 956 states): k_rows with the 6x6 row form;
    1024 sampled rows of float64, complex128 and a three-vector batch against the oracle; the full vector against the
    product with the canonical form off (the group walk)."""
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    basis, matrix, _, _ = _model("j1j2_6x6_w18")
    op = Operator(matrix)
    try:
        op.basis.build()
        reps = op.basis.representatives()
        n = reps.shape[0]
        assert op.info("rows") == 1 and op.info("rows_tk") == 6
        rows = np.sort(np.random.default_rng(17).choice(n, size=1024, replace=False))
        rows_d = torch.from_numpy(rows).cuda()
        for cplx in (False, True):
            x = _x(n, cplx, 3)
            y = op.matvec(torch.from_numpy(x).cuda())
            got = y[rows_d].cpu().numpy()
            del y
            want = po.expected_rows(matrix, reps, x, rows)
            assert _close(got, want), (cplx, np.abs(got - want).max())
        X = np.stack([_x(n, True, 50 + j) for j in range(3)])
        Y = op.matvec_batch(torch.from_numpy(X).cuda())
        got = Y[:, rows_d].cpu().numpy()
        del Y
        for j in range(3):
            want = po.expected_rows(matrix, reps, X[j], rows)
            assert _close(got[j], want), (j, np.abs(got[j] - want).max())
        del X
        x = torch.from_numpy(_x(n, True, 4)).cuda()
        y_torus = op.matvec(x).cpu().numpy()
        op.set_option("canon", 0)
        assert op.info("canon_mode") == 0 and op.info("rows_tk") == 0
        y_walk = op.matvec(x).cpu().numpy()
        op.set_option("canon", -1)
        assert _close(y_torus, y_walk), np.abs(y_torus - y_walk).max()
    finally:
        op.close()
