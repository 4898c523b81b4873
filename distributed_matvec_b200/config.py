"""YAML model inputs -> flat host-side descriptions of basis and operator.

Mirror of ``loadConfigFromYaml`` (reference: src/ForeignTypes.chpl:261-283), whose work is done
by the third-party ``ls_hs_load_yaml_config`` in the reference.  The YAML schema is the one of
/root/reference/data/*.yaml (and data/old/*.yaml):

    basis: {number_spins, hamming_weight, spin_inversion, symmetries: [{permutation, sector}]}
    hamiltonian: {terms: [{expression | matrix, sites}]}

plus the basis' particle type (``ls_hs_basis.particle_type``, reference src/FFI.chpl:85-99):

    basis: {particle: spin-1/2 (default) | spinless-fermion | spinful-fermion,
            number_sites, number_particles, number_up}

A spinless-fermion basis has ``number_sites`` bits, bit i the occupation of site i; with ``number_particles`` it is the
fixed-weight basis.  A spinful-fermion basis of N = ``number_sites`` <= 32 sites has 2N bits: bit i is the up occupation
of site i and bit N + i its down occupation, so a state is ``(down << N) | up``; ``number_particles`` and ``number_up``
are both required.  Fermionic bases take no spin inversion or ``hamming_weight``, and no spin ``symmetries`` (one
entry per bit, no exchange sign); their lattice symmetries are

    basis: {site_symmetries: [{permutation, sector}]}

with permutations of the ``number_sites`` sites.  A spinful permutation acts on both spin halves alike.  The state
|s> = c†_{a1} ... c†_{ak} |0> (a1 < ... < ak) goes to sign(g, s) |g(s)>, the sign of the exchanges (DESIGN.md §3).
"""
from __future__ import annotations

from dataclasses import dataclass, field
from math import comb

import numpy as np
import yaml

from .expr import FermionModes, TermTable, compile_terms, max_number_off_diag
from .symmetry import SymmetryGroup, build_group, widen_to_spinful


SPIN, SPINLESS_FERMION, SPINFUL_FERMION = "spin-1/2", "spinless-fermion", "spinful-fermion"
PARTICLE_TYPES = (SPIN, SPINLESS_FERMION, SPINFUL_FERMION)


@dataclass
class BasisSpec:
    """Flat description of a basis (what ``ls_hs_basis`` carries, src/FFI.chpl:85-105).  For fermions
    ``hamming_weight`` is the particle number, the weight over all ``number_bits`` bits."""
    number_sites: int
    hamming_weight: int | None
    spin_inversion: int            # 0 = none
    generators: list[dict] = field(default_factory=list)
    _group: SymmetryGroup | None = None
    particle_type: str = SPIN
    number_particles: int | None = None
    number_up: int | None = None   # spinful fermions only

    @property
    def number_bits(self) -> int:
        """Bits of a basis state: 2N for spinful fermions on N sites, N otherwise."""
        return 2 * self.number_sites if self.particle_type == SPINFUL_FERMION else self.number_sites

    def is_fermionic(self) -> bool:
        return self.particle_type != SPIN

    def fermion_modes(self) -> FermionModes | None:
        return FermionModes(self.number_sites, self.particle_type == SPINFUL_FERMION) if self.is_fermionic() else None

    # -- flags, named after the reference's Basis methods (src/ForeignTypes.chpl:82-100) --------
    def is_hamming_weight_fixed(self) -> bool:
        return self.hamming_weight is not None

    def has_spin_inversion_symmetry(self) -> bool:
        return self.spin_inversion != 0

    def has_permutation_symmetries(self) -> bool:
        return len(self.generators) > 0

    def requires_projection(self) -> bool:
        return self.has_permutation_symmetries() or self.has_spin_inversion_symmetry()

    def is_state_index_identity(self) -> bool:
        return not self.requires_projection() and not self.is_hamming_weight_fixed()

    @property
    def group(self) -> SymmetryGroup:
        """The group with one permutation entry per bit: a spinful site permutation p is widened to p[N + i] = N + p[i]."""
        if self._group is None:
            self._group = build_group(self.number_sites, self.generators, self.spin_inversion)
            if self.particle_type == SPINFUL_FERMION:
                self._group = widen_to_spinful(self._group)
        return self._group

    def min_state_estimate(self) -> int:
        """Smallest candidate state (mirror of ``ls_hs_min_state_estimate``, src/FFI.chpl:147)."""
        if self.hamming_weight is None:
            return 0
        if self.particle_type == SPINFUL_FERMION:
            n, up = self.number_sites, self.number_up
            return (((1 << (self.hamming_weight - up)) - 1) << n) | ((1 << up) - 1)
        return (1 << self.hamming_weight) - 1

    def max_state_estimate(self) -> int:
        """Largest candidate state (mirror of ``ls_hs_max_state_estimate``, src/FFI.chpl:148).

        With spin inversion every representative satisfies s <= s ^ mask, so the top site is
        never set (SURVEY.md App. A.2); the bound excludes it."""
        n, w = self.number_bits, self.hamming_weight
        if self.particle_type == SPINFUL_FERMION:
            up, down, half = self.number_up, w - self.number_up, self.number_sites
            return (((1 << down) - 1) << (n - down)) | (((1 << up) - 1) << (half - up))
        if w is None:
            hi = (1 << n) - 1
            if self.has_spin_inversion_symmetry():
                hi >>= 1
            return hi
        hi = ((1 << w) - 1) << (n - w)
        if self.has_spin_inversion_symmetry() and n > 0 and w > 0:
            # largest weight-w state with the top bit clear
            hi = ((1 << w) - 1) << (n - 1 - w) if n - 1 >= w else 0
        return hi

    def number_candidates(self) -> int:
        n, w = self.number_bits, self.hamming_weight
        return comb(n, w) if w is not None else 1 << n

    def number_states(self) -> int | None:
        """Dimension of a symmetry-free basis: C(N, N_up) C(N, N_down) for spinful fermions.  None for a projected
        basis: its dimension comes from enumeration."""
        if self.particle_type == SPINFUL_FERMION and not self.requires_projection():
            return comb(self.number_sites, self.number_up) * comb(self.number_sites, self.hamming_weight - self.number_up)
        if self.requires_projection():
            return None
        return self.number_candidates()


@dataclass
class OperatorSpec:
    """Flat description of an operator on a basis: compiled non-branching term tables."""
    basis: BasisSpec
    off_diag: TermTable
    diag: TermTable
    name: str = ""

    def number_diag_terms(self) -> int:       # src/ForeignTypes.chpl:222-226
        return len(self.diag)

    def number_off_diag_terms(self) -> int:   # src/ForeignTypes.chpl:228-233
        return max_number_off_diag(self.off_diag)

    def is_real(self) -> bool:                # src/ForeignTypes.chpl:258
        return self.off_diag.is_real() and self.diag.is_real()


def _generators(entries) -> list[dict]:
    return [{"permutation": [int(v) for v in g["permutation"]], "sector": int(g.get("sector", 0))}
            for g in (entries or [])]


def _fermion_basis_from_dict(d: dict, particle: str) -> BasisSpec:
    if d.get("symmetries") is not None:
        raise ValueError(f"{particle} basis: 'symmetries' is not supported: it lists spin permutations, one entry per "
                         "bit, without the fermionic exchange sign; give permutations of the sites as 'site_symmetries'")
    for key in ("spin_inversion", "hamming_weight", "number_spins"):
        if d.get(key) is not None:
            raise ValueError(f"{particle} basis: '{key}' is not supported (fermionic bases take number_sites, "
                             "number_particles, site_symmetries and, for spinful fermions, number_up)")
    if "number_sites" not in d:
        raise ValueError(f"{particle} basis needs number_sites")
    n = int(d["number_sites"])
    gens = _generators(d.get("site_symmetries"))
    for g in gens:
        if sorted(g["permutation"]) != list(range(n)):
            raise ValueError(f"{particle} basis: site_symmetries need permutations of the {n} sites "
                             f"(got {g['permutation']})")
    np_, nu = d.get("number_particles"), d.get("number_up")
    if particle == SPINLESS_FERMION:
        if not 0 < n <= 64:
            raise ValueError(f"spinless-fermion basis: number_sites must be between 1 and 64 (got {n})")
        if nu is not None:
            raise ValueError("spinless-fermion basis: 'number_up' is for spinful fermions")
        if np_ is not None and not 0 <= int(np_) <= n:
            raise ValueError(f"spinless-fermion basis: number_particles must be between 0 and {n} (got {np_})")
        w = None if np_ is None else int(np_)
        return BasisSpec(number_sites=n, hamming_weight=w, spin_inversion=0, generators=gens, particle_type=particle,
                         number_particles=w)
    if not 0 < n <= 32:
        raise ValueError(f"spinful-fermion basis: number_sites must be between 1 and 32 (got {n})")
    if np_ is None or nu is None:
        raise ValueError("spinful-fermion basis needs both number_particles and number_up")
    np_, nu = int(np_), int(nu)
    if not (0 <= nu <= n and 0 <= np_ - nu <= n):
        raise ValueError(f"spinful-fermion basis: need 0 <= number_up <= {n} and 0 <= number_particles - number_up <= "
                         f"{n} (got number_particles {np_}, number_up {nu})")
    return BasisSpec(number_sites=n, hamming_weight=np_, spin_inversion=0, generators=gens, particle_type=particle,
                     number_particles=np_, number_up=nu)


def basis_from_dict(d: dict) -> BasisSpec:
    particle = d.get("particle", SPIN)
    if particle not in PARTICLE_TYPES:
        raise ValueError(f"unknown particle type {particle!r}: expected one of {', '.join(PARTICLE_TYPES)}")
    if particle != SPIN:
        return _fermion_basis_from_dict(d, particle)
    if d.get("site_symmetries") is not None:
        raise ValueError("spin-1/2 basis: 'site_symmetries' is for fermionic bases; spin bases take 'symmetries'")
    n = int(d["number_spins"])
    if not 0 < n <= 64:
        raise ValueError("bases with more than 64 bits are not yet implemented")  # DMV:1099-1100
    hw = d.get("hamming_weight", None)
    inv = d.get("spin_inversion", None)
    return BasisSpec(
        number_sites=n,
        hamming_weight=None if hw is None else int(hw),
        spin_inversion=0 if inv is None else int(inv),
        generators=_generators(d.get("symmetries")),
    )


def operator_from_dict(d: dict, basis: BasisSpec) -> OperatorSpec:
    off, diag = compile_terms(d["terms"], basis.number_sites, basis.fermion_modes())
    return OperatorSpec(basis=basis, off_diag=off, diag=diag, name=str(d.get("name", "")))


def load_config_from_yaml(filename: str, hamiltonian: bool = True):
    """``loadConfigFromYaml(filename, hamiltonian=true)`` -> (basis, hamiltonian)."""
    with open(filename, "r", encoding="utf-8") as f:
        conf = yaml.safe_load(f)
    if "basis" not in conf:
        raise ValueError(f"failed to load Config from '{filename}'")
    basis = basis_from_dict(conf["basis"])
    if not hamiltonian:
        return basis
    if "hamiltonian" not in conf:
        raise ValueError(f"'{filename}' does not contain a Hamiltonian")
    return basis, operator_from_dict(conf["hamiltonian"], basis)
