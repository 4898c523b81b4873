"""Every build of k_gather that an operator can select, at every row split and walk, in full vector against the CPU oracle.

launch_gather picks one of 128 instantiations of k_gather: spin inversion (INV), complex coefficients (CV), complex
vectors (CE), 32-bit rows (NARROW: <= 32 sites and <= 32 flip-mask groups), the Lin-table index (LIN), one coefficient
for every emitting group (UNI, else the coefficient LUT) and one or four vectors per launch (KB).  On top of that sit two
run-time choices: the row split S (option "gather_split": S lanes share one row, each walks every S-th group, and S - 1
shuffles combine them; auto gives S > 1 to every basis of fewer than 16 warps per SM) and the walk over the emitting
groups (option "gather_walk": 0 per lane from the top bit, 1 group-major over the warp -- only at S = 1, else the
per-lane walk --, 2 per lane from the bottom bit).  The models here are small enough for the oracle to compute in well
under a second, except the four at size, which take the auto split S = 1.

Two of the models put more than 32 sigma^z sigma^z terms of one coupling on <= 32 sites with <= 32 flip-mask groups: the
row runs in 32-bit words, but a diagonal class holds up to 64 terms, so the class must still be evaluated in 64 bits.

Criterion: _close of test_gpu_parity (the reference's |a - b| <= max(atol, rtol max(|a|, |b|))), unchanged.  k_gather
stores every y element once from one lane, so host and device pointers, repeated products and the batched launches
(KB = 4) give bit-identical results.
"""
import functools
import os

import numpy as np
import pytest

from distributed_matvec_b200 import EmulatedCluster, Operator, block_to_hashed, hashed_to_block, load_config_from_yaml
from oracle import pyoracle as po
from test_gpu_parity import GENERAL_MODELS, _close, _custom, _x

torch = pytest.importorskip("torch")

DATA = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "data")

SPLITS = (-1, 1, 2, 8, 32)   # -1: auto
WALKS = (0, 1, 2)
INDEX_DIRECTORY, INDEX_IDENTITY, INDEX_RANK, INDEX_LIN = 0, 1, 2, 3


def _ring(n, d):
    return [[i, (i + d) % n] for i in range(n)]


def _hopping(bonds):
    return [{"expression": "σˣ₀ σˣ₁", "sites": bonds}, {"expression": "σʸ₀ σʸ₁", "sites": bonds}]


def _zz(bonds):
    return [{"expression": "σᶻ₀ σᶻ₁", "sites": bonds}]


def _heisenberg(bonds):
    return _hopping(bonds) + _zz(bonds)


# 4x4 torus, site x + 4 y: the 32 nearest-neighbour bonds and the 32 diagonal ones
TORUS_NN = [[x + 4 * y, (x + 1) % 4 + 4 * y] for y in range(4) for x in range(4)] + \
           [[x + 4 * y, x + 4 * ((y + 1) % 4)] for y in range(4) for x in range(4)]
TORUS_DIAG = [[x + 4 * y, (x + 1) % 4 + 4 * ((y + 1) % 4)] for y in range(4) for x in range(4)] + \
             [[x + 4 * y, (x + 1) % 4 + 4 * ((y + 3) % 4)] for y in range(4) for x in range(4)]


def _load(name):
    return load_config_from_yaml(os.path.join(DATA, name + ".yaml"))


def _complex_hopping(n):
    """complex_hopping of test_gpu_parity on an n-site ring at half filling."""
    return _custom(n, n // 2, [
        {"expression": "σ⁺₀ σ⁻₁", "sites": _ring(n, 1)}, {"expression": "σ⁻₀ σ⁺₁", "sites": _ring(n, 1)},
        {"expression": "0.3j × σ⁺₀ σ⁻₁", "sites": _ring(n, 2)}, {"expression": "-0.3j × σ⁻₀ σ⁺₁", "sites": _ring(n, 2)},
        {"expression": "σᶻ₀", "sites": [[0], [3]]}])


def _inversion_ring(n):
    """inversion_two_body of test_gpu_parity on an n-site ring: spin inversion, odd sector."""
    return _custom(n, n // 2, _hopping(_ring(n, 1)) + [{"expression": "0.5 × σᶻ₀ σᶻ₁", "sites": _ring(n, 2)}],
                   spin_inversion=-1)


def _narrow_diagonal_ring(n):
    """Hopping on the nearest bonds only (n groups), zz on nearest and next-nearest bonds at one coupling: one diagonal
    class of 2 n terms, more than 32 from n = 17 on, while the row still fits 32-bit words."""
    return _custom(n, n // 2, _hopping(_ring(n, 1)) + _zz(_ring(n, 1) + _ring(n, 2)))


def _many_classes():
    """XY ring of 20 sites with zz between every pair of sites at 190 distinct couplings: 190 diagonal classes, about
    150 KB of tables (the dynamic shared-memory path of launches above 48 KB)."""
    rng = np.random.default_rng(190)
    pairs = [[i, j] for i in range(20) for j in range(i + 1, 20)]
    couplings = np.round(rng.uniform(0.05, 1.0, len(pairs)), 6)
    assert len(set(couplings.tolist())) == len(pairs)
    return _custom(20, 6, _hopping(_ring(20, 1)) +
                   [{"expression": f"{c:.6f} × σᶻ₀ σᶻ₁", "sites": [p]} for c, p in zip(couplings, pairs)])


# name: (model, options set once, expected build: gather_narrow, gather_uniform, index_mode, bp_words)
MODELS = {
    "chain_16": (lambda: _load("heisenberg_chain_16"), {}, (1, 1, INDEX_LIN, 1)),
    # exactly 32 groups and one class of exactly 32 zz terms: the largest narrow operator, the control of the two below
    "torus_4x4_32_bonds": (lambda: _custom(16, 8, _heisenberg(TORUS_NN)), {}, (1, 1, INDEX_LIN, 1)),
    "kagome_16": (lambda: _load("heisenberg_kagome_16"), {}, (1, 1, INDEX_LIN, 1)),
    "chain_10_inversion": (lambda: _load("heisenberg_chain_10"), {}, (1, 1, INDEX_LIN, 1)),
    "inversion_two_body": (GENERAL_MODELS["inversion_two_body"], {}, (1, 1, INDEX_LIN, 1)),
    "anisotropic_bonds": (GENERAL_MODELS["anisotropic_bonds"], {}, (1, 0, INDEX_LIN, 1)),
    "complex_hopping": (GENERAL_MODELS["complex_hopping"], {}, (1, 0, INDEX_LIN, 1)),
    # 64-bit words on <= 32 sites (36 groups)
    "ring_18_nnn": (lambda: _custom(18, 9, _heisenberg(_ring(18, 1) + _ring(18, 2))), {}, (0, 1, INDEX_LIN, 1)),
    # 64-bit words on > 32 sites: Lin tables (34 sites), directory search (48 sites)
    "wide_two_magnon": (GENERAL_MODELS["wide_two_magnon"], {}, (0, 1, INDEX_LIN, 1)),
    "ring_48_w2": (lambda: _custom(48, 2, _heisenberg(_ring(48, 1))), {}, (0, 1, INDEX_DIRECTORY, 1)),
    # two BpWords (g_base = 64 in the second): 80 groups (Lin tables), 96 groups (directory search)
    "ring_40_w3_nnn": (lambda: _custom(40, 3, _heisenberg(_ring(40, 1) + _ring(40, 2))), {}, (0, 1, INDEX_LIN, 2)),
    "ring_48_w2_nnn": (lambda: _custom(48, 2, _heisenberg(_ring(48, 1) + _ring(48, 2))), {},
                       (0, 1, INDEX_DIRECTORY, 2)),
    # narrow rows with a diagonal class of more than 32 terms: 36 (ring), 64 (torus with its diagonal bonds)
    "narrow_diagonal_ring_18": (lambda: _narrow_diagonal_ring(18), {}, (1, 1, INDEX_LIN, 1)),
    "narrow_diagonal_torus_4x4": (lambda: _custom(16, 8, _heisenberg(TORUS_NN) + _zz(TORUS_DIAG)), {},
                                  (1, 1, INDEX_LIN, 1)),
    "chain_12_identity": (lambda: _load("heisenberg_chain_12"), {}, (1, 1, INDEX_IDENTITY, 1)),
    "chain_16_rank": (lambda: _load("heisenberg_chain_16"), {"index": 2}, (1, 1, INDEX_RANK, 1)),
    "many_diagonal_classes": (_many_classes, {}, (1, 1, INDEX_LIN, 1)),
}

AT_SIZE = {
    "chain_20": lambda: _load("heisenberg_chain_20"),
    "complex_hopping_20": lambda: _complex_hopping(20),
    "inversion_ring_20": lambda: _inversion_ring(20),
    "narrow_diagonal_ring_20": lambda: _narrow_diagonal_ring(20),
}


@functools.lru_cache(maxsize=None)
def _model(name):
    return (MODELS[name][0] if name in MODELS else AT_SIZE[name])()


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """Representatives and y = H x of both element types (x by the _x recipe), from the CPU oracle."""
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    basis, matrix = _model(name)
    reps, _ = po.enumerate_states(basis)
    ys = {}
    for cplx in (False, True):
        x = _x(reps.shape[0], cplx)
        ys[cplx] = (x, po.matvec_global(matrix, reps, x, 1, num_tasks=po.num_threads()))
    return reps, ys


@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _set(op, split, walk):
    op.set_option("gather_split", split)
    op.set_option("gather_walk", walk)


def _device(op, x, y0=None):
    y = op.matvec(torch.from_numpy(x).cuda(), None if y0 is None else torch.from_numpy(y0.copy()).cuda())
    torch.cuda.synchronize()
    return y.cpu().numpy()


def _check_build(op, name, expect):
    narrow, uniform, index_mode, words = expect
    got = (op.info("gather"), op.info("gather_narrow"), op.info("gather_uniform"), op.info("index_mode"),
           op.info("bp_words"))
    assert got == (1, narrow, uniform, index_mode, words), (name, got)


def _check_split(op, split):
    s = op.info("gather_split")
    if split > 0:
        assert s == split, (split, s)
    else:   # auto: a power of two, and never more lanes than groups
        assert s in (1, 2, 4, 8, 16, 32) and s <= max(1, op.info("n_groups")), s


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MODELS))
def test_gather_splits_and_walks(need_cuda, name):
    """float64 / complex128 x gather_split auto, 1, 2, 8, 32 x gather_walk 0, 1, 2, in full vector against the oracle;
    at every setting host and device pointers and a repeated product are bit-identical."""
    _, options, expect = MODELS[name]
    basis, matrix = _model(name)
    reps, ys = _oracle(name)
    op = Operator(matrix)
    try:
        for k, v in options.items():
            op.set_option(k, v)
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        _check_build(op, name, expect)
        for cplx in (False, True):
            x, y_ref = ys[cplx]
            for split in SPLITS:
                for walk in WALKS:
                    _set(op, split, walk)
                    _check_split(op, split)
                    y = _device(op, x)
                    where = (name, cplx, split, walk)
                    assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
                    assert np.array_equal(_device(op, x), y), where
                    assert np.array_equal(op.matvec(x), y), where
        _check_build(op, name, expect)
    finally:
        op.close()


@pytest.mark.gpu
def test_gather_without_diagonal_accumulates_into_y(need_cuda):
    """An XY ring without diagonal terms: k_gather adds to y instead of storing, at every split and walk."""
    basis, matrix = _custom(8, 4, _hopping(_ring(8, 1)))
    op = Operator(matrix)
    try:
        op.basis.build()
        _check_build(op, "xy_ring_8", (1, 1, INDEX_LIN, 1))
        reps = op.basis.representatives()
        for cplx in (False, True):
            x = _x(reps.shape[0], cplx)
            y0 = _x(reps.shape[0], cplx, seed=9)
            y_ref = po.matvec_blocks(matrix, [reps], [x], y_blocks=[y0.copy()])[0]
            assert not _close(y_ref, po.matvec_global(matrix, reps, x, 1))   # y0 does contribute
            for split in SPLITS:
                for walk in WALKS:
                    _set(op, split, walk)
                    y = _device(op, x, y0)
                    assert _close(y, y_ref), (cplx, split, walk, np.abs(y - y_ref).max())
                    assert np.array_equal(op.matvec(x, y0.copy()), y), (cplx, split, walk)
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["chain_16", "complex_hopping", "inversion_two_body", "ring_40_w3_nnn",
                                  "narrow_diagonal_torus_4x4"])
def test_gather_batch_is_bit_identical(need_cuda, name):
    """matvec_batch with 4 columns (one KB = 4 launch) and 9 (two KB = 4 launches and a single product) gives exactly
    the single products, and the oracle's, at splits 1 and 32 and every walk."""
    basis, matrix = _model(name)
    reps, _ = _oracle(name)
    n = reps.shape[0]
    op = Operator(matrix)
    try:
        op.basis.build()
        _check_build(op, name, MODELS[name][2])
        for cplx in (False, True):
            X = np.stack([_x(n, cplx, 100 + j) for j in range(9)])
            want = [po.matvec_global(matrix, reps, X[j], 1, num_tasks=po.num_threads()) for j in range(9)]
            for split in (1, 32):
                for walk in WALKS:
                    _set(op, split, walk)
                    singles = np.stack([_device(op, X[j]) for j in range(9)])
                    for j in range(9):
                        assert _close(singles[j], want[j]), (cplx, split, walk, j)
                    for k in (4, 9):
                        Y = op.matvec_batch(torch.from_numpy(X[:k].copy()).cuda())
                        torch.cuda.synchronize()
                        assert np.array_equal(Y.cpu().numpy(), singles[:k]), (cplx, split, walk, k)
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(AT_SIZE))
def test_gather_at_size_auto_split(need_cuda, name):
    """Bases of 92 378 and 184 756 states: the auto split is 1, so walk 1 runs its own group-major form; all three walks
    in full vector against the oracle."""
    basis, matrix = _model(name)
    reps, ys = _oracle(name)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        assert op.info("gather") == 1
        assert op.info("gather_narrow") == (0 if name == "complex_hopping_20" else 1)   # 40 groups
        for cplx in (False, True):
            x, y_ref = ys[cplx]
            xd = torch.from_numpy(x).cuda()
            for walk in WALKS:
                _set(op, -1, walk)
                assert op.info("gather_split") == 1
                y = op.matvec(xd).cpu().numpy()
                assert _close(y, y_ref), (name, cplx, walk, np.abs(y - y_ref).max())
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("num_ranks", [2, 3])
@pytest.mark.parametrize("name,splits", [("chain_20", (-1,)), ("inversion_two_body", (1, 32)),
                                         ("complex_hopping", (1, 32))])
def test_gather_replicated_x(need_cuda, name, splits, num_ranks):
    """The replicated-x form (k_gather over this rank's rows of the whole-basis tables, x by global index through pos)
    on P logical ranks against the oracle's P-rank product; options set on every rank before and after the whole-basis
    context exists."""
    basis, matrix = _model(name)
    reps, _ = _oracle(name)
    masks, _ = po.partition_by_hash(reps, num_ranks)
    cl = EmulatedCluster(matrix, num_ranks).build()
    try:
        for cplx in (False, True):
            x = _x(reps.shape[0], cplx, 31)
            y_ref = po.matvec_global(matrix, reps, x, num_ranks, num_tasks=po.num_threads())
            xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, num_ranks)]
            for split in splits:
                for walk in WALKS:
                    for op in cl.ops:
                        _set(op, split, walk)
                    y = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)
                    if split > 0:
                        assert all(op.info("gather_split") == split for op in cl.ops)
                    assert _close(y, y_ref), (name, num_ranks, cplx, split, walk, np.abs(y - y_ref).max())
    finally:
        cl.close()


@pytest.mark.gpu
@pytest.mark.parametrize("split", [1, 32])
@pytest.mark.parametrize("walk", WALKS)
def test_gather_missing_state_is_an_error(need_cuda, split, walk):
    """A generated state that is not in the basis halts (DMV:115-118) under every walk and split."""
    basis, matrix = _load("heisenberg_chain_16")
    reps, _ = po.enumerate_states(basis)
    op = Operator(matrix)
    try:
        op.basis.uncheckedSetRepresentatives(reps[:-7])
        _set(op, split, walk)
        assert op.info("gather") == 1 and op.info("gather_split") == split
        with pytest.raises(Exception, match="invalid index"):
            op.matvec(np.ones(reps.shape[0] - 7))
    finally:
        op.close()


@pytest.mark.gpu
def test_gather_options_out_of_range_raise(need_cuda):
    """gather_split takes -1 and the powers of two up to 32, gather_walk 0, 1, 2; anything else raises and leaves the
    option as it was."""
    basis, matrix = _load("heisenberg_chain_16")
    reps, ys = _oracle("chain_16")
    op = Operator(matrix)
    try:
        op.basis.build()
        _set(op, 4, 2)
        for key, value in (("gather_split", 0), ("gather_split", 3), ("gather_split", 64), ("gather_split", -2),
                           ("gather_walk", 3), ("gather_walk", -1)):
            with pytest.raises(Exception, match=key):
                op.set_option(key, value)
        assert op.info("gather_split") == 4
        x, y_ref = ys[True]
        assert _close(_device(op, x), y_ref)
    finally:
        op.close()
