"""Operator expressions -> non-branching terms.

Host-side mirror of what the reference obtains from the third-party
``ls_hs_load_yaml_config`` / ``ls_hs_create_operator`` calls
(reference: src/ForeignTypes.chpl:261-283, src/FFI.chpl:187-200).  The reference
only sees the compiled result through ``ls_hs_nonbranching_terms`` (src/FFI.chpl:109-119);
here the compiled result is a flat table of terms

    <beta| t |alpha> = v * [alpha & m == r] * (-1)^popcount(alpha & s),   beta = alpha ^ x

which is the contract SURVEY.md §8(a6)/(c) derives from the call sites
(src/BatchedOperator.chpl:99-106, src/DistributedMatrixVector.chpl:43-45).

Conventions (ours; irrelevant for every Heisenberg input, see DESIGN.md):
  * site i is bit i of the uint64 basis state (LSB = site 0);
  * bit = 1 means spin up (sigma^z = +1), sigma^+ turns a 0 bit into a 1 bit;
  * a ``matrix:`` term on sites (i, j) is indexed by (bit_i << 1) | bit_j.

Fermion operators (on a fermionic basis only, never mixed with σ / S in one expression):
  * ``c†₀`` creation, ``c₀`` annihilation, ``n₀`` number on placeholder site 0 (ASCII digits work too);
  * on a spinful basis each operator carries a spin arrow, before or after the index: ``c†₀↑ c₁↑``, ``n↑₀ n↓₀``;
  * they combine with the coefficient, ``×`` / ``*``, ``+`` and ``−`` grammar of the spin operators, e.g.
    ``-1.0 × c†₀↑ c₁↑ - 1.0 × c†₁↑ c₀↑`` or ``4 × n₀↑ n₀↓``.
The mode of a factor is its concrete site i (spinless; spinful up) or N + i (spinful down), and bit k of a state is the
occupation of mode k.  Modes are ordered by bit: c_k = Z_0 ... Z_{k-1} σ⁻_k (Jordan-Wigner).  Every monomial is compiled
per concrete instance: with T the set of modes it touches, its 2^|T| local matrix carries the signs of the modes inside
T, and the string of the modes outside T becomes the term's sign mask s = XOR over its c / c† factors on mode k of
(bits below k) & ~T.  A hop and its conjugate get the same x and s.
"""
from __future__ import annotations

import itertools
import re
from dataclasses import dataclass, field

import numpy as np

_SUPERSCRIPTS = {"ˣ": "x", "ʸ": "y", "ᶻ": "z", "⁺": "+", "⁻": "-", "x": "x", "y": "y", "z": "z", "+": "+", "-": "-"}
_SUBSCRIPT_DIGITS = {c: str(i) for i, c in enumerate("₀₁₂₃₄₅₆₇₈₉")}

# single-site matrices in the (|1> = up, |0> = down) basis, index = bit value
# row = outgoing bit, column = incoming bit
_SIGMA = {
    "x": np.array([[0, 1], [1, 0]], dtype=np.complex128),
    # sigma^y = [[0, -i], [i, 0]] in the (up, down) ordering; with index = bit value
    # (index 1 = up) the up<-down element (row 1, col 0) is -i.
    "y": np.array([[0, 1j], [-1j, 0]], dtype=np.complex128),
    "z": np.array([[-1, 0], [0, 1]], dtype=np.complex128),
    "+": np.array([[0, 0], [1, 0]], dtype=np.complex128),  # |1><0|
    "-": np.array([[0, 1], [0, 0]], dtype=np.complex128),  # |0><1|
    "I": np.eye(2, dtype=np.complex128),
}


_FERMION_KINDS = ("c+", "c", "n")
_ARROWS = {"↑": "up", "↓": "down"}


@dataclass(frozen=True)
class FermionModes:
    """Bit layout of a fermionic basis: mode of (site, spin) = site, or site + number_sites for spin down."""
    number_sites: int
    spinful: bool

    def mode(self, site: int, spin: str) -> int:
        if self.spinful != (spin != ""):
            raise ValueError("fermion operators need a spin arrow (↑ or ↓) on a spinful basis and none on a spinless one")
        return site + (self.number_sites if spin == "down" else 0)


@dataclass(frozen=True)
class Factor:
    """One primitive operator: kind in {'sigma','S'}, comp in x,y,z,+,-, placeholder site index; or a fermion
    operator: kind in {'c+','c','n'}, comp the spin ('up', 'down' or '' on a spinless basis)."""
    kind: str
    comp: str
    site: int

    def matrix(self) -> np.ndarray:
        m = _SIGMA[self.comp]
        if self.kind == "S" and self.comp in "xyz":
            return 0.5 * m
        return m


@dataclass
class Product:
    coeff: complex
    factors: list[Factor] = field(default_factory=list)


def _tokenize(text: str):
    i, n = 0, len(text)
    while i < n:
        ch = text[i]
        if ch.isspace():
            i += 1
        elif ch in "×*":
            yield ("mul", ch)
            i += 1
        elif ch in "+-" :
            yield ("sign", ch)
            i += 1
        elif ch in "()":
            yield (ch, ch)
            i += 1
        elif ch in "σS":
            kind = "sigma" if ch == "σ" else "S"
            i += 1
            if i >= n or text[i] not in _SUPERSCRIPTS:
                raise ValueError(f"expected component superscript after {ch!r} in {text!r}")
            comp = _SUPERSCRIPTS[text[i]]
            i += 1
            digits = ""
            while i < n and (text[i] in _SUBSCRIPT_DIGITS or text[i].isdigit()):
                digits += _SUBSCRIPT_DIGITS.get(text[i], text[i])
                i += 1
            if text[i:i + 1] == "_":
                raise ValueError("use unicode subscripts for site indices")
            if not digits:
                raise ValueError(f"missing site index in {text!r}")
            yield ("op", Factor(kind, comp, int(digits)))
        elif ch.isdigit() or ch == ".":
            m = re.match(r"(\d+\.?\d*([eE][+-]?\d+)?|\.\d+([eE][+-]?\d+)?)(j|im)?", text[i:])
            if not m:
                raise ValueError(f"bad number in {text!r}")
            val = complex(0, float(m.group(1))) if m.group(4) else complex(float(m.group(1)))
            yield ("num", val)
            i += m.end()
        elif ch == "I":
            yield ("num", 1.0 + 0j)
            i += 1
        elif ch in "cn":
            kind = "n" if ch == "n" else "c"
            i += 1
            if kind == "c" and text[i:i + 1] == "†":
                kind = "c+"
                i += 1
            spin, digits = "", ""
            while i < n and (text[i] in _SUBSCRIPT_DIGITS or text[i].isdigit() or text[i] in _ARROWS):
                if text[i] in _ARROWS:
                    if spin:
                        raise ValueError(f"two spin arrows on one operator in {text!r}")
                    spin = _ARROWS[text[i]]
                else:
                    digits += _SUBSCRIPT_DIGITS.get(text[i], text[i])
                i += 1
            if not digits:
                raise ValueError(f"missing site index in {text!r}")
            yield ("op", Factor(kind, spin, int(digits)))
        else:
            raise ValueError(f"unexpected character {ch!r} in expression {text!r}")


def parse_expression(text: str) -> list[Product]:
    """Parse a sum of products such as ``"0.8 × σˣ₀ σˣ₁"`` or ``"σ⁺₀ σ⁻₁ + σ⁻₀ σ⁺₁"``."""
    products: list[Product] = []
    cur: Product | None = None
    sign = 1.0
    for kind, val in _tokenize(text):
        if kind == "sign":
            if cur is not None and (cur.factors or cur.coeff != 1):
                products.append(cur)
                cur = None
                sign = 1.0
            if val == "-":
                sign = -sign
        elif kind == "mul":
            continue
        elif kind in "()":
            raise ValueError("parentheses are not supported in expressions")
        else:
            if cur is None:
                cur = Product(sign)
                sign = 1.0
            if kind == "num":
                cur.coeff *= val
            else:
                cur.factors.append(val)
    if cur is not None:
        products.append(cur)
    if not products:
        raise ValueError(f"empty expression {text!r}")
    kinds = {f.kind in _FERMION_KINDS for p in products for f in p.factors}
    if len(kinds) > 1:
        raise ValueError(f"spin (σ, S) and fermion (c†, c, n) operators are mixed in {text!r}")
    return products


def is_fermionic(products: list[Product]) -> bool:
    return any(f.kind in _FERMION_KINDS for p in products for f in p.factors)


def local_matrix(products: list[Product]) -> tuple[int, np.ndarray]:
    """Dense 2^k x 2^k matrix of an expression over its k placeholder sites.

    Index convention: placeholder site 0 is the MOST significant bit of the local index
    (same as ``matrix:`` terms: index = (bit_0 << (k-1)) | ... | bit_{k-1}).
    """
    k = 1 + max((f.site for p in products for f in p.factors), default=0)
    dim = 1 << k
    total = np.zeros((dim, dim), dtype=np.complex128)
    for p in products:
        per_site = [np.eye(2, dtype=np.complex128) for _ in range(k)]
        for f in p.factors:  # left-to-right product on the same site
            per_site[f.site] = per_site[f.site] @ f.matrix()
        m = np.array([[1.0 + 0j]])
        for s in range(k):
            m = np.kron(m, per_site[s])
        total += p.coeff * m
    return k, total


@dataclass
class TermTable:
    """Flat non-branching term table, all arrays of length T."""
    v: np.ndarray  # complex128
    m: np.ndarray  # uint64
    r: np.ndarray  # uint64
    x: np.ndarray  # uint64
    s: np.ndarray  # uint64

    def __len__(self) -> int:
        return int(self.v.shape[0])

    @staticmethod
    def empty() -> "TermTable":
        z = np.zeros(0, dtype=np.uint64)
        return TermTable(np.zeros(0, dtype=np.complex128), z, z.copy(), z.copy(), z.copy())

    def is_real(self) -> bool:
        return bool(np.all(self.v.imag == 0))


def _check_sites(k: int, sites: tuple[int, ...]):
    if len(set(sites)) != len(sites):
        raise ValueError(f"repeated site in {sites}")
    if len(sites) != k:
        raise ValueError(f"expression acts on {k} sites but got index tuple {sites}")


def _accumulate_instance(acc: dict, k: int, mat: np.ndarray, sites: tuple[int, ...]):
    _check_sites(k, sites)
    mask = 0
    for st in sites:
        mask |= 1 << st

    def spread(local: int) -> int:
        out = 0
        for pos, st in enumerate(sites):
            if (local >> (k - 1 - pos)) & 1:
                out |= 1 << st
        return out

    for out_idx, in_idx in itertools.product(range(1 << k), repeat=2):
        val = mat[out_idx, in_idx]
        if val == 0:
            continue
        r = spread(in_idx)
        x = r ^ spread(out_idx)
        key = (mask, r, x, 0)
        acc[key] = acc.get(key, 0j) + complex(val)


def fermion_monomial_terms(coeff: complex, ops: list[tuple[str, int]]):
    """Terms (v, m, r, x, s) of coeff * op_1 op_2 ... op_n on concrete modes, ops = [(kind, mode)] with kind in
    'c+', 'c', 'n' (the rightmost acts first).  m is the set T of touched modes, the local matrix carries the signs of
    the modes inside T, and s = XOR over the c / c† factors on mode k of (bits below k) & ~T."""
    T = sorted({mode for _, mode in ops})
    m = 0
    for mode in T:
        m |= 1 << mode
    s = 0
    for kind, mode in ops:
        if kind != "n":
            s ^= ((1 << mode) - 1) & ~m
    pos = {mode: b for b, mode in enumerate(T)}

    def spread(local: int) -> int:
        return sum(1 << T[b] for b in range(len(T)) if (local >> b) & 1)

    out = []
    for local_in in range(1 << len(T)):
        st, amp = local_in, complex(coeff)
        for kind, mode in reversed(ops):
            b = pos[mode]
            occ = (st >> b) & 1
            if kind == "n":
                if not occ:
                    amp = 0j
                    break
                continue
            if occ != (kind == "c"):   # c needs the mode occupied, c† needs it empty
                amp = 0j
                break
            if bin(st & ((1 << b) - 1)).count("1") & 1:
                amp = -amp
            st ^= 1 << b
        if amp != 0:
            r = spread(local_in)
            out.append((amp, m, r, r ^ spread(st), s))
    return out


def _accumulate_fermion_instance(acc: dict, products: list[Product], k: int, sites: tuple[int, ...],
                                 modes: FermionModes):
    _check_sites(k, sites)
    for p in products:
        ops = [(f.kind, modes.mode(sites[f.site], f.comp)) for f in p.factors]
        if not ops:
            raise ValueError("a constant term needs at least one operator on a fermionic basis")
        for v, m, r, x, s in fermion_monomial_terms(p.coeff, ops):
            key = (m, r, x, s)
            acc[key] = acc.get(key, 0j) + v


def compile_terms(term_specs: list[dict], number_sites: int,
                  fermions: FermionModes | None = None) -> tuple[TermTable, TermTable]:
    """Compile the ``hamiltonian.terms`` list of a YAML config into (off_diag, diag) tables.

    Each spec has ``sites`` (list of index tuples) and either ``expression`` (string) or
    ``matrix`` (2^k x 2^k nested list, data/old/*.yaml form).
    Equal (m, r, x, s) contributions from different expressions are summed and exact zeros
    dropped (sigma^x sigma^x + sigma^y sigma^y cancels on parallel spins), which is the
    operator-compile-time merge SURVEY.md App. A.4(2) refers to.  ``fermions``: the mode layout of a fermionic
    basis, whose expressions are compiled instance by instance (module docstring); spin terms have s = 0.
    """
    acc: dict[tuple[int, int, int, int], complex] = {}
    for spec in term_specs:
        if "expression" in spec:
            products = parse_expression(spec["expression"])
            if is_fermionic(products) != (fermions is not None):
                raise ValueError(f"{spec['expression']!r}: fermion operators (c†, c, n) need a fermionic basis, and "
                                 "a fermionic basis takes fermion operators only")
            k = 1 + max((f.site for p in products for f in p.factors), default=0)
            if fermions is not None:
                for sites in spec["sites"]:
                    sites = tuple(int(s) for s in sites)
                    if any(s < 0 or s >= number_sites for s in sites):
                        raise ValueError(f"site index out of range in {sites}")
                    _accumulate_fermion_instance(acc, products, k, sites, fermions)
                continue
            k, mat = local_matrix(products)
        elif "matrix" in spec:
            if fermions is not None:
                raise ValueError("matrix terms are not supported on a fermionic basis: use c†, c and n expressions")
            mat = np.array(spec["matrix"], dtype=np.complex128)
            k = int(mat.shape[0]).bit_length() - 1
            if mat.shape != (1 << k, 1 << k):
                raise ValueError("matrix term must be 2^k x 2^k")
        else:
            raise ValueError("term needs 'expression' or 'matrix'")
        for sites in spec["sites"]:
            sites = tuple(int(s) for s in sites)
            if any(s < 0 or s >= number_sites for s in sites):
                raise ValueError(f"site index out of range in {sites}")
            _accumulate_instance(acc, k, mat, sites)

    off, diag_groups = [], {}
    for (m, r, x, s), v in sorted(acc.items()):
        if abs(v) == 0:
            continue
        if x == 0:
            assert s == 0, "a diagonal monomial has an even number of c / c† factors on every mode, so no string"
            diag_groups.setdefault(m, {})[r] = v
        else:
            off.append((v, m, r, x, s))

    # Diagonal part: Walsh-expand each function f(r) over the bits of m so that e.g.
    # the four (m, r) entries of sigma^z sigma^z collapse into ONE term (v, m=0, r=0, s=m).
    diag = []
    for m, table in sorted(diag_groups.items()):
        bits = [b for b in range(64) if (m >> b) & 1]
        kk = len(bits)

        def expand(sub: int) -> int:
            out = 0
            for pos, b in enumerate(bits):
                if (sub >> pos) & 1:
                    out |= 1 << b
            return out

        f = np.zeros(1 << kk, dtype=np.complex128)
        for sub in range(1 << kk):
            f[sub] = table.get(expand(sub), 0j)
        for ssub in range(1 << kk):
            coef = 0j
            for sub in range(1 << kk):
                coef += f[sub] * (-1) ** bin(sub & ssub).count("1")
            coef /= (1 << kk)
            if abs(coef) > 1e-15 * max(1.0, float(np.abs(f).max())):
                diag.append((coef, 0, 0, 0, expand(ssub)))
    # merge diagonal terms with equal s coming from different bonds
    merged: dict[int, complex] = {}
    for coef, _, _, _, s in diag:
        merged[s] = merged.get(s, 0j) + coef
    diag = [(c, 0, 0, 0, s) for s, c in sorted(merged.items()) if abs(c) > 0]

    def to_table(rows) -> TermTable:
        if not rows:
            return TermTable.empty()
        return TermTable(
            np.array([t[0] for t in rows], dtype=np.complex128),
            np.array([t[1] for t in rows], dtype=np.uint64),
            np.array([t[2] for t in rows], dtype=np.uint64),
            np.array([t[3] for t in rows], dtype=np.uint64),
            np.array([t[4] for t in rows], dtype=np.uint64),
        )

    return to_table(off), to_table(diag)


def max_number_off_diag(off: TermTable) -> int:
    """Upper bound on emitted terms per row (mirror of ``ls_hs_operator_max_number_off_diag``,
    reference: src/ForeignTypes.chpl:228-229): number of distinct flip masks x."""
    return int(len(np.unique(off.x)))
