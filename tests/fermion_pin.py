"""Independent Jordan-Wigner construction of fermionic Hamiltonians, for the tests of fermionic bases.

c_k = Z_0 ... Z_{k-1} σ⁻_k as sparse Kronecker products over the modes (bit k of a state = occupation of mode k, so
Z = +1 on an empty mode), monomials multiplied as matrices.  The expressions are read by a tokenizer of its own: nothing
of distributed_matvec_b200.expr is used.  Restricted to a particle-number block for up to 16 modes.
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


def sector_states(n_sites: int, number_up: int | None, number_down: int | None = None, spinful: bool = True):
    """Ascending states of the block: (down << N) | up at fixed half weights (spinful), or weight number_up (spinless)."""
    if not spinful:
        return np.array(sorted(sum(1 << b for b in c) for c in itertools.combinations(range(n_sites), number_up)),
                        dtype=np.uint64)
    ups = sorted(sum(1 << b for b in c) for c in itertools.combinations(range(n_sites), number_up))
    downs = sorted(sum(1 << b for b in c) for c in itertools.combinations(range(n_sites), number_down))
    return np.array([(d << n_sites) | u for d in downs for u in ups], dtype=np.uint64)


def sector_hamiltonian(term_specs, n_sites: int, spinful: bool, states: np.ndarray) -> sp.csr_matrix:
    H = full_hamiltonian(term_specs, n_sites, spinful)
    idx = states.astype(np.int64)
    return H[idx][:, idx].tocsr()
