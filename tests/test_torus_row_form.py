"""The row form of the square-torus orbit minimum that k_rows evaluates (orbit_min_torus_sq_t: the transposed state of a
row XORed with the transposed flip mask of a term) against the single-state form orbit_min_torus_sq and the oracle,
through the device functions compiled for the host (no GPU needed)."""
import ctypes as C
import os

import numpy as np
import pytest

from distributed_matvec_b200 import _native as nat
from distributed_matvec_b200.config import basis_from_dict, load_config_from_yaml
from oracle import pyoracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "data")


def _desc(basis):
    g = basis.group
    bd = nat.BasisDesc()
    bd.number_sites, bd.hamming_weight, bd.spin_inversion, bd.has_permutations = (
        basis.number_sites, -1 if basis.hamming_weight is None else basis.hamming_weight, basis.spin_inversion or 0, 1)
    keep = (np.ascontiguousarray(g.perms), np.ascontiguousarray(g.flips), np.ascontiguousarray(g.characters))
    bd.group_order, bd.perms, bd.flips, bd.characters = len(g), keep[0].ctypes.data, keep[1].ctypes.data, keep[2].ctypes.data
    return bd, keep


def _square_torus(k, inversion):
    n = k * k
    gens = [[k * (i // k) + ((i % k + 1) % k) for i in range(n)], [(i + k) % n for i in range(n)],
            [k * (i // k) + (k - 1 - i % k) for i in range(n)], [k * (k - 1 - i // k) + i % k for i in range(n)],
            [k * (i % k) + i // k for i in range(n)]]
    return basis_from_dict({"number_spins": n, "hamming_weight": None, "spin_inversion": inversion,
                            "symmetries": [{"permutation": g, "sector": 0} for g in gens]})


def _flip_masks(k, rng):
    """Nearest-neighbour bonds of the k x k torus, and masks of other shapes: one site, diagonal pairs, whole rows and
    columns, a plaquette, random masks of every density."""
    n = k * k
    masks = []
    for y in range(k):
        for a in range(k):
            s = k * y + a
            masks.append((1 << s) | (1 << (k * y + (a + 1) % k)))          # horizontal bond
            masks.append((1 << s) | (1 << (k * ((y + 1) % k) + a)))        # vertical bond
    masks += [1, 1 << (n - 1), (1 << 0) | (1 << (k + 1)), (1 << (k - 1)) | (1 << k),   # single sites, diagonals
              (1 << k) - 1, sum(1 << (k * y) for y in range(k)),                   # a whole row, a whole column
              (1 << 0) | (1 << 1) | (1 << k) | (1 << (k + 1)), (1 << n) - 1, 0]   # plaquette, everything, nothing
    masks += [int(v) for v in rng.integers(0, 1 << n, size=16, dtype=np.uint64)]
    return np.array(masks, dtype=np.uint64)


def _check(basis, states, flips):
    bd, keep = _desc(basis)
    rows = np.zeros(states.shape[0] * flips.shape[0], dtype=np.uint64)
    single = np.zeros_like(rows)
    nat.check(nat.lib().dmv_debug_torus_sq_rows(C.byref(bd), states.shape[0], states.ctypes.data, flips.shape[0],
                                                flips.ctypes.data, rows.ctypes.data, single.ctypes.data))
    assert np.array_equal(rows, single)
    targets = (states[:, None] ^ flips[None, :]).reshape(-1) & np.uint64((1 << basis.number_sites) - 1)
    o_reps, _, _ = po.state_info(basis, targets)
    assert np.array_equal(rows, o_reps)
    return rows.shape[0]


@pytest.mark.parametrize("k", [4, 6])
@pytest.mark.parametrize("inversion", [None, 1])
def test_row_form_on_square_tori(k, inversion):
    basis = _square_torus(k, inversion)
    rng = np.random.default_rng(10 * k + (inversion or 0))
    n = k * k
    states = rng.integers(0, 1 << n, size=160 if k == 6 else 400, dtype=np.uint64)
    states[:40] &= rng.integers(0, 1 << n, size=40, dtype=np.uint64)     # sparse words: tied top pairs
    m = rng.integers(0, 2, size=(40, k, k))
    m = np.triu(m) | np.transpose(np.triu(m, 1), (0, 2, 1))                 # transpose-symmetric states
    states[40:80] = [sum(int(mm[y, a]) << (k * y + a) for y in range(k) for a in range(k)) for mm in m]
    states[80:84] = [0, (1 << n) - 1, 0x5555555555555555 & ((1 << n) - 1), sum(1 << (k * y) for y in range(k))]
    assert _check(basis, states, _flip_masks(k, rng)) > 0


@pytest.mark.parametrize("name", ["heisenberg_square_4x4", "heisenberg_square_6x6"])
def test_row_form_on_the_model_bases(name):
    """The models' own groups (the 6 x 6 square has spin inversion: 576 elements), sampled states x every bond."""
    basis, _ = load_config_from_yaml(os.path.join(DATA, name + ".yaml"))
    k = int(round(basis.number_sites ** 0.5))
    rng = np.random.default_rng(k)
    states = rng.integers(0, 1 << basis.number_sites, size=200, dtype=np.uint64)
    _check(basis, states, _flip_masks(k, rng))


def test_row_form_refuses_other_groups():
    basis, _ = load_config_from_yaml(os.path.join(DATA, "heisenberg_chain_24_symm.yaml"))
    bd, keep = _desc(basis)
    s = np.zeros(1, dtype=np.uint64)
    out = np.zeros(1, dtype=np.uint64)
    with pytest.raises(nat.DmvError, match="square-torus"):
        nat.check(nat.lib().dmv_debug_torus_sq_rows(C.byref(bd), 1, s.ctypes.data, 1, s.ctypes.data, out.ctypes.data,
                                                    out.ctypes.data))
