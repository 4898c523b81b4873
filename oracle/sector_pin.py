"""Independent pin for wide bases: the twin of oracle/dense_pin.py restricted to one sector of fixed Hamming weight.

TEST INFRASTRUCTURE ONLY.  dense_pin builds H on the full 2^n space and stops at about 20 sites.  Here the states are
those of Hamming weight w on n <= 64 sites, a sorted uint64 array made by itertools.combinations and indexed with
np.searchsorted, so the construction goes to 64 sites as long as the sector is small.  It shares with the library only
the expression tokenizer (`parse_expression`) and the group the basis spec generates:
  - H: every product of every term applied to all sector states at once -- the 2^k output bit patterns of the k sites
    a product touches, as the "matrix" branch of dense_pin.full_hamiltonian -- in a scipy.sparse matrix of dimension
    C(n, w).  Amplitudes that leave the sector are dropped, which is H projected on the sector.
  - B: the symmetry-adapted basis of dense_pin.symmetry_adapted_basis (P = 1/|G| sum_g conj(chi(g)) U_g, column k =
    P|r_k> / ||P|r_k>||, r_k the orbit minima in ascending order) on the sector states.
  - from psi = B x: <σᶻᵢσᶻⱼ>, <σᶻᵢ> and <σ⁺ᵢσ⁻ⱼ> with the formulas of test_zz_correlations / test_pm_correlations.
The group images take |G| x C(n, w) words: keep that at about 10^7 or fewer.
"""
from __future__ import annotations

import itertools
from math import comb

import numpy as np
import scipy.sparse as sp

from distributed_matvec_b200.expr import parse_expression

from .dense_pin import _apply_element

MAX_IMAGES = 12_000_000


def sector_states(n: int, w: int) -> np.ndarray:
    """All states of Hamming weight w on n sites, ascending"""
    if comb(n, w) > 50_000_000:
        raise ValueError(f"C({n}, {w}) states are too many for the sector reference")
    states = np.fromiter((sum(1 << i for i in c) for c in itertools.combinations(range(n), w)), dtype=np.uint64,
                         count=comb(n, w))
    states.sort()
    return states


def _index(states: np.ndarray, targets: np.ndarray):
    """(positions, found): positions of targets in the sorted states, and which targets are states at all"""
    pos = np.searchsorted(states, targets)
    pos_c = np.minimum(pos, states.shape[0] - 1)
    return pos_c, states[pos_c] == targets


def _local_matrix(product, sites) -> tuple[list[int], np.ndarray]:
    """(the distinct sites a product touches, its 2^k x 2^k matrix): local index bit k - 1 - pos = bit of the site at
    position pos, as in dense_pin's "matrix" branch; factors act in the order they are written"""
    where: list[int] = []
    for f in product.factors:
        s = int(sites[f.site])
        if s not in where:
            where.append(s)
    k = len(where)
    M = np.eye(1 << k, dtype=np.complex128) * product.coeff
    for f in product.factors:
        pos = where.index(int(sites[f.site]))
        E = np.ones((1, 1), dtype=np.complex128)
        for q in range(k):
            E = np.kron(E, f.matrix() if q == pos else np.eye(2))
        M = M @ E
    return where, M


def sector_hamiltonian(term_specs: list[dict], n: int, states: np.ndarray) -> sp.csr_matrix:
    """H on the sector states (CSR, complex128)"""
    dim = states.shape[0]
    rows, cols, vals = [], [], []
    col_all = np.arange(dim)
    for spec in term_specs:
        for sites in spec["sites"]:
            for p in parse_expression(spec["expression"]):
                where, M = _local_matrix(p, sites)
                k = len(where)
                rest = np.uint64(((1 << 64) - 1) ^ sum(1 << s for s in where))
                loc_in = np.zeros(dim, dtype=np.int64)
                for pos, s in enumerate(where):
                    loc_in |= ((states >> np.uint64(s)) & np.uint64(1)).astype(np.int64) << (k - 1 - pos)
                for loc_out in range(1 << k):
                    v = M[loc_out, loc_in]
                    keep = v != 0
                    if not keep.any():
                        continue
                    out = states[keep] & rest
                    for pos, s in enumerate(where):
                        if (loc_out >> (k - 1 - pos)) & 1:
                            out |= np.uint64(1 << s)
                    at, found = _index(states, out)
                    rows.append(at[found]); cols.append(col_all[keep][found]); vals.append(v[keep][found])
    if not rows:
        return sp.csr_matrix((dim, dim), dtype=np.complex128)
    return sp.csr_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))), shape=(dim, dim),
                         dtype=np.complex128)


def symmetry_adapted_basis(basis, states: np.ndarray):
    """(representatives ascending, norms ||P r||, B sparse [C(n, w), N]) on the sector states"""
    n = basis.number_sites
    dim = states.shape[0]
    if not basis.requires_projection():
        return states, np.ones(dim), sp.identity(dim, format="csc", dtype=np.complex128)
    g = basis.group
    G = len(g)
    if G * dim > MAX_IMAGES:
        raise ValueError(f"|G| x C(n, w) = {G * dim} images are too many for the sector reference")
    images = np.stack([_apply_element(g.perms[e], g.flips[e], n, states) for e in range(G)])   # [G, S]
    is_rep = images.min(axis=0) == states
    reps_at = np.nonzero(is_rep)[0]
    R = reps_at.shape[0]
    img = images[:, reps_at]
    at, found = _index(states, img.ravel())
    if not found.all():
        raise ValueError("the group leaves the sector")
    vals = np.broadcast_to((np.conj(np.asarray(g.characters)) / G)[:, None], img.shape).ravel()
    cols = np.broadcast_to(np.arange(R)[None, :], img.shape).ravel()
    B = sp.csc_matrix((vals, (at, cols)), shape=(dim, R), dtype=np.complex128)
    B.sum_duplicates()
    nrm = np.sqrt(np.asarray(abs(B).power(2).sum(axis=0)).ravel())
    keep = nrm ** 2 >= 1e-20
    B = (B[:, np.nonzero(keep)[0]] @ sp.diags(1.0 / nrm[keep])).tocsc()
    return states[reps_at[keep]], nrm[keep], B


class Sector:
    """The sector reference of one (basis, operator) pair: states, B, Hp = B^dagger H B (sparse)"""

    def __init__(self, basis, term_specs: list[dict]):
        if basis.hamming_weight is None:
            raise ValueError("the sector reference needs a fixed Hamming weight")
        self.n = basis.number_sites
        self.states = sector_states(self.n, basis.hamming_weight)
        self.reps, self.norms, self.B = symmetry_adapted_basis(basis, self.states)
        H = sector_hamiltonian(term_specs, self.n, self.states)
        self.Hp = (self.B.conj().T @ (H @ self.B)).tocsr()

    def psi(self, x: np.ndarray) -> np.ndarray:
        return self.B @ x

    def zz(self, x: np.ndarray):
        """(<σᶻᵢσᶻⱼ>, <σᶻᵢ>) of psi = B x"""
        p = np.abs(self.psi(x)) ** 2
        p = p / p.sum()
        bits = (self.states[:, None] >> np.arange(self.n, dtype=np.uint64)[None, :]) & np.uint64(1)
        s = 2.0 * bits.astype(np.float64) - 1.0
        return (s * p[:, None]).T @ s, p @ s

    def pm(self, x: np.ndarray) -> np.ndarray:
        """T[i, j] = <psi|σ⁺ᵢσ⁻ⱼ|psi> / <psi|psi>, T[i, i] = <n_i>"""
        psi = self.psi(x)
        W = np.vdot(psi, psi).real
        n, s = self.n, self.states
        bit = [((s >> np.uint64(i)) & np.uint64(1)).astype(bool) for i in range(n)]
        T = np.zeros((n, n), dtype=np.complex128)
        for i in range(n):
            T[i, i] = np.sum(np.abs(psi[bit[i]]) ** 2) / W
            for j in range(n):
                if i != j:
                    src = np.nonzero(bit[j] & ~bit[i])[0]
                    dst, found = _index(s, s[src] ^ np.uint64((1 << i) | (1 << j)))
                    assert found.all()
                    T[i, j] = np.vdot(psi[dst], psi[src]) / W
        return T
