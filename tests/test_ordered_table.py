"""The ordered layout of the k_rows look-up table (rows_table = 1), built on the host by the library's self-check
entry with the same functions the kernels run: every representative is found, linear probing stays short, and the home
buckets follow the key prefix, which is what gives the look-ups of neighbouring rows their L2 reuse."""
import ctypes as C
import os

import numpy as np
import pytest

from distributed_matvec_b200 import _native as nat
from distributed_matvec_b200.config import load_config_from_yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "data")


def representatives(name):
    """Ascending orbit representatives of a model's S_z = 0 sector (every orbit: the characters are trivial)."""
    basis, _ = load_config_from_yaml(os.path.join(DATA, name + ".yaml"))
    n = basis.number_sites
    s = np.arange(1 << n, dtype=np.uint64)
    w = np.zeros(s.shape, dtype=np.uint8)
    for b in range(n):
        w += ((s >> np.uint64(b)) & np.uint64(1)).astype(np.uint8)
    states = np.ascontiguousarray(s[w == basis.hamming_weight])
    g = basis.group
    assert g.all_characters_trivial
    bd = nat.BasisDesc()
    bd.number_sites, bd.hamming_weight, bd.spin_inversion, bd.has_permutations = (
        n, basis.hamming_weight, basis.spin_inversion, 1)
    perms, flips, chars = (np.ascontiguousarray(g.perms), np.ascontiguousarray(g.flips),
                           np.ascontiguousarray(g.characters))
    bd.group_order, bd.perms, bd.flips, bd.characters = len(g), perms.ctypes.data, flips.ctypes.data, chars.ctypes.data
    reps = np.zeros_like(states)
    nat.check(nat.lib().dmv_debug_compile_group(C.byref(bd), None, states.shape[0], states.ctypes.data,
                                                reps.ctypes.data, None))
    return np.unique(reps)


def ordered_table(reps, bits, buckets):
    block = np.zeros(reps.shape[0], dtype=np.uint32)
    home = np.zeros_like(block)
    probes = np.zeros_like(block)
    nat.check(nat.lib().dmv_debug_ordered_table(reps.ctypes.data, reps.shape[0], bits, buckets, block.ctypes.data,
                                                home.ctypes.data, probes.ctypes.data))
    return block, home, probes


@pytest.mark.parametrize("name", ["heisenberg_square_4x4", "heisenberg_chain_24_symm"])
@pytest.mark.parametrize("bits,buckets", [(14, 8), (14, 4), (14, 2), (12, 2), (4, 2)])
def test_ordered_table_finds_every_state_in_prefix_order(name, bits, buckets):
    reps = representatives(name)
    block, home, probes = ordered_table(reps, bits, buckets)
    n_buckets = buckets * reps.shape[0]
    assert probes.min() >= 1                          # every representative is found (the entry fails otherwise)
    assert home.max() < n_buckets
    assert block.max() < 2**bits and np.all(np.diff(block.astype(np.int64)) >= 0)
    # home buckets are non-decreasing in the prefix: every home of a block lies below every home of a later block
    starts = np.flatnonzero(np.diff(block.astype(np.int64), prepend=-1))
    lo = np.minimum.reduceat(home, starts)
    hi = np.maximum.reduceat(home, starts)
    assert np.all(hi[:-1] < lo[1:])
    # linear probing at load 1 / buckets: 1.5 probes per look-up expected at load 1/2, 1.17 at 1/4, 1.07 at 1/8
    assert probes.mean() < {2: 1.8, 4: 1.3, 8: 1.15}[buckets], probes.mean()
    assert probes.max() <= 64, probes.max()


def test_ordered_table_rejects_unsorted_representatives():
    reps = np.array([5, 3, 9], dtype=np.uint64)
    block = np.zeros(3, dtype=np.uint32)
    assert nat.lib().dmv_debug_ordered_table(reps.ctypes.data, 3, 8, 2, block.ctypes.data, None, None) != 0
