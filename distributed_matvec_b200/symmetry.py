"""Symmetry groups of a basis: closure of the YAML generators, characters, device tables.

The reference never sees the group: it calls the third-party ``ls_hs_state_info`` /
``ls_hs_is_representative`` (reference: src/FFI.chpl:177-184, src/BatchedOperator.chpl:188-194,
src/ForeignTypes.chpl:129-143).  SURVEY.md App. A.3 states what those compute; this module is
the host-side part (group closure + compilation into bit-permutation networks for the GPU).

Convention (ours, see DESIGN.md): a permutation p acts on a state as (g.sigma)[i] = sigma[p[i]],
i.e. bit i of the result is bit p[i] of the input.
"""
from __future__ import annotations

import cmath
from dataclasses import dataclass
from fractions import Fraction

import numpy as np


def _compose(p: tuple[int, ...], q: tuple[int, ...]) -> tuple[int, ...]:
    """Permutation of 'apply q first, then p':  (p.(q.s))[i] = (q.s)[p[i]] = s[q[p[i]]]."""
    return tuple(q[i] for i in p)


def _order(p: tuple[int, ...]) -> int:
    ident = tuple(range(len(p)))
    cur, k = p, 1
    while cur != ident:
        cur = _compose(p, cur)
        k += 1
    return k


@dataclass
class SymmetryGroup:
    """All elements of the group, each with a permutation, an inversion flag and a character."""
    number_sites: int
    perms: np.ndarray       # int32 [G, n]   result bit i = input bit perms[g, i]
    flips: np.ndarray       # uint8 [G]      1 = followed by global spin inversion
    characters: np.ndarray  # complex128 [G]
    spin_inversion: int     # 0, +1, -1
    has_permutations: bool

    def __len__(self) -> int:
        return int(self.perms.shape[0])

    @property
    def all_characters_trivial(self) -> bool:
        return bool(np.all(self.characters == 1))


def build_group(number_sites: int, generators: list[dict], spin_inversion: int | None) -> SymmetryGroup:
    """Closure of ``symmetries: [{permutation, sector}]`` (+ optional spin inversion).

    The character of a generator of period T in sector k is exp(-2 pi i k / T) (SURVEY.md App. A.3);
    characters multiply under composition.  An inconsistent assignment (the same group element
    reached with two different characters) raises.
    """
    n = number_sites
    inv = int(spin_inversion or 0)
    if inv not in (0, 1, -1):
        raise ValueError("spin_inversion must be null, 1 or -1")
    ident = tuple(range(n))
    gens: list[tuple[tuple[int, ...], Fraction]] = []
    for g in generators:
        p = tuple(int(v) for v in g["permutation"])
        if sorted(p) != list(range(n)):
            raise ValueError(f"not a permutation of {n} sites: {p}")
        period = _order(p)
        sector = int(g.get("sector", 0))
        if not 0 <= sector < period:
            raise ValueError(f"sector {sector} out of range for a generator of period {period}")
        gens.append((p, Fraction(sector, period) % 1))

    # phase stored as a Fraction of a full turn so that consistency can be checked exactly
    elements: dict[tuple[int, ...], Fraction] = {ident: Fraction(0)}
    frontier = [ident]
    while frontier:
        nxt = []
        for e in frontier:
            for p, ph in gens:
                c = _compose(p, e)
                phase = (elements[e] + ph) % 1
                if c in elements:
                    if elements[c] != phase:
                        raise ValueError("sectors do not define a one-dimensional representation")
                else:
                    elements[c] = phase
                    nxt.append(c)
        frontier = nxt

    perms, flips, chars = [], [], []
    for p, phase in sorted(elements.items()):
        chi = cmath.exp(-2j * cmath.pi * float(phase))
        # snap exact values so that trivial sectors give exactly 1
        chi = complex(round(chi.real, 15), round(chi.imag, 15))
        if phase == 0:
            chi = 1 + 0j
        elif phase == Fraction(1, 2):
            chi = -1 + 0j
        perms.append(p)
        flips.append(0)
        chars.append(chi)
    if inv != 0:
        base = list(zip(perms, chars))
        for p, chi in base:
            perms.append(p)
            flips.append(1)
            chars.append(chi * inv)
    return SymmetryGroup(
        number_sites=n,
        perms=np.array(perms, dtype=np.int32).reshape(len(perms), n),
        flips=np.array(flips, dtype=np.uint8),
        characters=np.array(chars, dtype=np.complex128),
        spin_inversion=inv,
        has_permutations=len(gens) > 0,
    )


# ---------------------------------------------------------------------------------------------
# Compilation of permutations for the device
# ---------------------------------------------------------------------------------------------

def shift_mask_form(perm: np.ndarray) -> list[tuple[int, int]]:
    """Decompose a bit permutation into (mask, shift) pairs:  g(s) = OR_k rot-free shift of (s & mask_k).

    Result bit i = input bit perm[i]; input bit j = perm[i] moves by d = i - j.  Pairs are
    (mask over INPUT bits, signed shift d): out |= d >= 0 ? (s & mask) << d : (s & mask) >> -d.
    """
    groups: dict[int, int] = {}
    for i, j in enumerate(perm):
        d = i - int(j)
        groups[d] = groups.get(d, 0) | (1 << int(j))
    return sorted(groups.items(), key=lambda kv: kv[0])


def benes_masks(perm: np.ndarray, width: int = 64) -> list[tuple[int, int]]:
    """Benes network for a bit permutation as a list of (mask, delta) butterfly stages.

    Applying the stages in order with  t = ((s >> delta) ^ s) & mask;  s ^= t ^ (t << delta)
    yields the state g.s with (g.s)[i] = s[perm[i]] (bits >= len(perm) are fixed points).
    Stages whose mask is zero are dropped.  Standard recursive routing (two-colouring of the
    constraint cycles at every level).
    """
    n = len(perm)
    if n > width:
        raise ValueError("permutation wider than the network")
    src = list(range(width))  # src[i] = input position that must end up at output i
    for i in range(n):
        src[i] = int(perm[i])
    log = width.bit_length() - 1
    assert 1 << log == width

    front: list[tuple[int, int]] = []
    back: list[tuple[int, int]] = []

    # cur_src[i] : which original-input "token" must arrive at position i (w.r.t. the current
    # sub-network inputs).  We route level by level on sub-blocks.
    def route(src_of: list[int], level: int):
        """src_of: permutation on `width` positions restricted to independent blocks of size
        2*delta ... routed with butterflies of distance delta = width >> (level+1)."""
        delta = width >> (level + 1)
        if delta == 0:
            return
        blk = 2 * delta
        in_mask = 0
        out_mask = 0
        new_src = list(src_of)
        inv = [0] * width
        for i, s in enumerate(src_of):
            inv[s] = i
        # decide for every input position whether it is swapped with its partner at the input
        # stage, and for every output position whether swapped at the output stage.
        in_swap = [None] * width   # indexed by lower position of the pair
        out_swap = [None] * width
        for base in range(0, width, blk):
            for start in range(base, base + delta):
                if out_swap[start] is not None:
                    continue
                # walk the cycle: fix output pair `start` unswapped
                o = start
                o_sw = False
                while True:
                    out_swap[o] = o_sw
                    # output position o (lower) receives from the upper sub-network iff not swapped
                    # token arriving at lower-half output o comes from input position:
                    lo_pos = o if not o_sw else o + delta      # which output is fed by the "lower" subnet
                    tok = src_of[lo_pos]                        # input position of that token
                    ipair = tok if ((tok - base) % blk) < delta else tok - delta
                    # token must travel through the lower subnet => after the input stage it must sit
                    # in the lower half of its pair
                    need_swap = (tok != ipair)
                    in_swap[ipair] = need_swap
                    # partner input of that pair goes through the upper subnet
                    partner = ipair + delta if not need_swap else ipair
                    # (partner is the input position whose token goes to the upper subnet)
                    dest = inv[partner]                         # output position it must reach
                    opair = dest if ((dest - base) % blk) < delta else dest - delta
                    # it arrives via the upper subnet at the upper half of the output pair; it wants `dest`
                    nsw = (dest == opair)                       # must be swapped down if dest is the lower output
                    if out_swap[opair] is not None:
                        break
                    o, o_sw = opair, nsw
        for base in range(0, width, blk):
            for p in range(base, base + delta):
                if in_swap[p] is None:
                    in_swap[p] = False
                if in_swap[p]:
                    in_mask |= 1 << p
                if out_swap[p]:
                    out_mask |= 1 << p
        # tokens after the input stage: position p holds input token ...
        after_in = list(range(width))
        for p in range(width):
            if (in_mask >> p) & 1:
                after_in[p], after_in[p + delta] = after_in[p + delta], after_in[p]
        pos_after_in = [0] * width
        for pos, tok in enumerate(after_in):
            pos_after_in[tok] = pos
        # required sources before the output stage
        before_out = list(src_of)
        for p in range(width):
            if (out_mask >> p) & 1:
                before_out[p], before_out[p + delta] = before_out[p + delta], before_out[p]
        # inner permutation: position q (before output stage) must receive the token that sits at
        # pos_after_in[before_out[q]] after the input stage
        inner = [pos_after_in[before_out[q]] for q in range(width)]
        front.append((in_mask, delta))
        back.append((out_mask, delta))
        route(inner, level + 1)

    route(src, 0)
    # front stages in order, then the back stages in reverse; the innermost level (delta = 1)
    # appears twice back to back and can be merged only if masks are disjoint in effect, so keep both.
    stages = front + back[::-1]
    stages = [(m, d) for (m, d) in stages if m != 0]
    # verify
    for trial in (0x0123456789ABCDEF, 0xFEDCBA9876543210, 0x5555555555555555, 0x8000000000000001):
        s = trial & ((1 << width) - 1)
        out = s
        for m, d in stages:
            t = ((out >> d) ^ out) & m
            out ^= t ^ (t << d)
        expect = 0
        for i in range(width):
            if (s >> src[i]) & 1:
                expect |= 1 << i
        if out != expect:
            raise AssertionError("Benes routing failed self-check")
    return stages


def widen_to_spinful(group: SymmetryGroup) -> SymmetryGroup:
    """The group of site permutations p of a spinful-fermion basis as bit permutations: p[N + i] = N + p[i]."""
    n = group.number_sites
    return SymmetryGroup(number_sites=2 * n, perms=np.concatenate([group.perms, group.perms + n], axis=1).astype(np.int32),
                         flips=group.flips, characters=group.characters, spin_inversion=group.spin_inversion,
                         has_permutations=group.has_permutations)


def inversion_masks(perm: np.ndarray) -> np.ndarray:
    """Fermionic exchange sign of a bit permutation (result bit i = input bit perm[i]): bit j goes to image(j), the i
    with perm[i] = j, and M[i] = { j < i : image(j) > image(i) }.  sign(g, s) = (-1)^(sum over set bits i of s of
    popc(s & M[i])), the parity of the inversions of the images of the occupied modes.  -> uint64 [len(perm)]"""
    n = len(perm)
    image = np.empty(n, dtype=np.int64)
    image[np.asarray(perm, dtype=np.int64)] = np.arange(n)
    masks = np.zeros(n, dtype=np.uint64)
    for i in range(n):
        for j in range(i):
            if image[j] > image[i]:
                masks[i] |= np.uint64(1) << np.uint64(j)
    return masks


def fermion_signs(perm: np.ndarray, states: np.ndarray) -> np.ndarray:
    """sign(g, s) in {+1, -1} for an array of uint64 states, from inversion_masks (host mirror of the device's)."""
    states = np.asarray(states, dtype=np.uint64)
    parity = np.zeros(states.shape, dtype=np.uint64)
    one = np.uint64(1)
    for i, m in enumerate(inversion_masks(perm)):
        occupied = (states >> np.uint64(i)) & one
        parity ^= occupied & (np.bitwise_count(states & m).astype(np.uint64) & one)
    return np.where(parity == 0, 1, -1).astype(np.int8)


def apply_permutation_numpy(perm: np.ndarray, states: np.ndarray) -> np.ndarray:
    """(g.s)[i] = s[perm[i]] for an array of uint64 states (host helper for tests)."""
    out = np.zeros_like(states)
    for i, j in enumerate(perm):
        out |= ((states >> np.uint64(int(j))) & np.uint64(1)) << np.uint64(i)
    return out
