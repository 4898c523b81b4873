"""Independent Jordan-Wigner construction of fermionic Hamiltonians, for the tests of fermionic bases.

c_k = Z_0 ... Z_{k-1} σ⁻_k as sparse Kronecker products over the modes (bit k of a state = occupation of mode k, so
Z = +1 on an empty mode), monomials multiplied as matrices.  The expressions are read by a tokenizer of its own: nothing
of distributed_matvec_b200.expr is used.  Restricted to a particle-number block for up to 16 modes.
apply_to_states is the same construction bit by bit on given states, for any number of modes up to 64.
"""
from __future__ import annotations

import itertools
import re

import numpy as np
import scipy.sparse as sp

_SUB = {c: str(i) for i, c in enumerate("₀₁₂₃₄₅₆₇₈₉")}
_TOKEN = re.compile(r"\s*(?:(?P<num>\d+\.?\d*(?:[eE][+-]?\d+)?j?)|(?P<op>c†|c|n)(?P<idx>[↑↓]?[₀-₉0-9]+[↑↓]?)|"
                    r"(?P<mul>[×*])|(?P<sign>[+-]))")


def annihilator(n_modes: int, k: int) -> sp.csr_matrix:
    """c_k on n_modes modes; state index = integer whose bit j is the occupation of mode j."""
    z = sp.diags([1.0, -1.0])
    lower = sp.csr_matrix(np.array([[0.0, 1.0], [0.0, 0.0]]))   # |0><1|
    eye = sp.identity(2)
    out = sp.identity(1)
    for j in range(n_modes - 1, -1, -1):   # kron: the most significant bit first
        out = sp.kron(out, z if j < k else (lower if j == k else eye), format="csr")
    return out.tocsr()


def parse(text: str):
    """-> [(coeff, [(kind, placeholder, spin)])] with kind in c+, c, n and spin '', 'up' or 'down'."""
    terms, coeff, factors, sign = [], None, [], 1.0
    pos = 0
    while pos < len(text):
        m = _TOKEN.match(text, pos)
        if not m or m.end() == pos:
            if text[pos:].strip() == "":
                break
            raise ValueError(f"cannot read {text[pos:]!r}")
        pos = m.end()
        if m.group("sign"):
            if factors or coeff is not None:
                terms.append((sign * (1.0 if coeff is None else coeff), factors))
                coeff, factors, sign = None, [], 1.0
            if m.group("sign") == "-":
                sign = -sign
        elif m.group("num"):
            v = complex(m.group("num")) if m.group("num").endswith("j") else float(m.group("num"))
            coeff = v if coeff is None else coeff * v
        elif m.group("op"):
            idx = m.group("idx")
            spin = "up" if "↑" in idx else ("down" if "↓" in idx else "")
            digits = "".join(_SUB.get(ch, ch) for ch in idx if ch not in "↑↓")
            kind = {"c†": "c+", "c": "c", "n": "n"}[m.group("op")]
            factors.append((kind, int(digits), spin))
    if factors or coeff is not None:
        terms.append((sign * (1.0 if coeff is None else coeff), factors))
    return terms


def mode_of(site: int, spin: str, n_sites: int) -> int:
    return site + (n_sites if spin == "down" else 0)


def monomial(n_modes: int, ops) -> sp.csr_matrix:
    """op_1 op_2 ... op_n for ops = [(kind, mode)]."""
    out = sp.identity(1 << n_modes, format="csr", dtype=np.complex128)
    for kind, mode in ops:
        c = annihilator(n_modes, mode)
        out = out @ (c.T if kind == "c+" else (c if kind == "c" else c.T @ c))
    return out.tocsr()


def full_hamiltonian(term_specs, n_sites: int, spinful: bool) -> sp.csr_matrix:
    n_modes = 2 * n_sites if spinful else n_sites
    if n_modes > 16:
        raise ValueError("the Jordan-Wigner pin stops at 16 modes")
    H = sp.csr_matrix((1 << n_modes, 1 << n_modes), dtype=np.complex128)
    for spec in term_specs:
        for coeff, factors in parse(spec["expression"]):
            for sites in spec["sites"]:
                ops = [(kind, mode_of(int(sites[p]), spin, n_sites)) for kind, p, spin in factors]
                H = H + coeff * monomial(n_modes, ops)
    return H.tocsr()


def weight_states(n_bits: int, weight: int) -> np.ndarray:
    """Ascending n_bits-bit states with `weight` set bits."""
    if n_bits <= 24:
        s = np.arange(1 << n_bits, dtype=np.uint64)
        return s[np.bitwise_count(s) == weight]
    return np.array(sorted(sum(1 << b for b in c) for c in itertools.combinations(range(n_bits), weight)),
                    dtype=np.uint64).reshape(-1)


def sector_states(n_sites: int, number_up: int | None, number_down: int | None = None, spinful: bool = True):
    """Ascending states of the block: (down << N) | up at fixed half weights (spinful), or weight number_up (spinless).
    The spinful block is the outer product of the two halves, so sectors of 10^7 states take a fraction of a second."""
    if not spinful:
        return weight_states(n_sites, number_up)
    ups, downs = weight_states(n_sites, number_up), weight_states(n_sites, number_down)
    return ((downs[:, None] << np.uint64(n_sites)) | ups[None, :]).reshape(-1)


def apply_to_states(term_specs, n_sites: int, spinful: bool, states: np.ndarray, targets=None) -> sp.csr_matrix:
    """<β|H|α> for α over the ascending `states` (columns) and β over the ascending `targets` (rows; default the states
    themselves), bit by bit: each monomial acts on every state right to left, c_k and c†_k with the sign
    (-1)^popc(state & ((1 << k) - 1)) of the Jordan-Wigner string.  Terms need not conserve the particle number; one
    that leads out of the rows raises.  Vectorised over the states in numpy uint64, for any number of modes up to 64."""
    states = np.ascontiguousarray(states, dtype=np.uint64)
    targets = states if targets is None else np.ascontiguousarray(targets, dtype=np.uint64)
    n = states.shape[0]
    one = np.uint64(1)
    rows, cols, vals = [], [], []
    for spec in term_specs:
        for coeff, factors in parse(spec["expression"]):
            for sites in spec["sites"]:
                st = states.copy()
                neg = np.zeros(n, dtype=bool)
                alive = np.ones(n, dtype=bool)
                for kind, p, spin in reversed(factors):
                    bit = one << np.uint64(mode_of(int(sites[p]), spin, n_sites))
                    occupied = (st & bit) != 0
                    if kind == "n":
                        alive &= occupied
                        continue
                    alive &= occupied if kind == "c" else ~occupied
                    neg ^= (np.bitwise_count(st & (bit - one)) & 1).astype(bool)
                    st ^= bit
                sel = np.nonzero(alive)[0]
                if sel.size == 0:
                    continue
                r = np.minimum(np.searchsorted(targets, st[sel]), max(targets.shape[0] - 1, 0))
                if targets.shape[0] == 0 or not np.array_equal(targets[r], st[sel]):
                    raise ValueError(f"{spec['expression']!r} on {sites} leads out of the target states")
                rows.append(r)
                cols.append(sel)
                vals.append(np.where(neg[sel], -complex(coeff), complex(coeff)))
    if not rows:
        return sp.csr_matrix((targets.shape[0], n), dtype=np.complex128)
    return sp.coo_matrix((np.concatenate(vals), (np.concatenate(rows), np.concatenate(cols))),
                         shape=(targets.shape[0], n)).tocsr()


def sector_hamiltonian(term_specs, n_sites: int, spinful: bool, states: np.ndarray) -> sp.csr_matrix:
    H = full_hamiltonian(term_specs, n_sites, spinful)
    idx = states.astype(np.int64)
    return H[idx][:, idx].tocsr()
