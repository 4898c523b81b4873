"""The scatter product k_generate and the queued row product k_pull on purpose-built models, against the CPU oracle.

k_generate is the reference's own traversal: it runs for mode = 0, for every record exchange and for every counting pass
(dmv_plan).  k_pull runs for complex characters, complex operators on symmetric bases and rows = 0 / gather = 0.  Both
walk the flip-mask groups 64 at a time (word w of the emit mask), queue the emitted terms in a warp ring of 128 entries
(k_generate drains it 64 at a time, k_pull 32 at a time, with wraparound) and instantiate one build per projection (none,
spin inversion, permutation group), complex values and complex vectors.  On top of that sit:

* the row split S of k_generate (option "push_split": S lanes share one source state, each takes every S-th group, and
  only slice 0 adds the diagonal; auto picks S from the basis size, the group count and the SM count of the device);
* the index kind of k_pull (identity, Lin tables, directory search, combinadic rank, which spin inversion reverses);
* the two ways route() places a remote record: per-warp cursors from the plan up to 32 ranks, a warp-aggregated slot claim
  with global atomics on out_count from 33 to 256 ranks (and atomics in the counting pass there too).

The models have flip-mask group counts of 0, 63, 64, 65, 91, 128 and 129, rows that emit more than 64 terms, an
operator without diagonal terms (y is accumulated into, DMV:1062-1069), a 64-site basis with flips of bit 63 and a
momentum sector whose targets include zero-norm states (dropped without an error).  Each one is small enough for the
oracle to finish in about a second.

References: the CPU oracle (oracle/pyoracle.py), which shares no code with the library.  Criterion: _close of
test_gpu_parity, unchanged.  k_pull stores every y element once from one lane and, without a permutation group, sums a
row's terms in an order that does not depend on the index kind: there y is bit-identical across index kinds and calls.
"""
import functools
import os
import time

import numpy as np
import pytest

from distributed_matvec_b200 import EmulatedCluster, Operator, block_to_hashed, hashed_to_block
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
from distributed_matvec_b200.operator import BatchedOperator, _device_tensor, _elt_of
from oracle import pyoracle as po
from test_gpu_parity import _close, _x

torch = pytest.importorskip("torch")

SPLITS = (1, 2, 4, 8, 16, 32, -1)   # -1: auto
INDEX_KINDS = (-1, 0, 2, 3)         # auto, directory search, combinadic rank, Lin tables
RANKS = (2, 31, 32, 33, 64, 128, 256)


# ---- models ---------------------------------------------------------------------------------------------------------

def _pairs(n):
    """The pairs of an all-to-all graph on n sites, in order: each is its own flip-mask group."""
    return [[i, j] for i in range(n) for j in range(i + 1, n)]


def _ring(n, d):
    return [[i, (i + d) % n] for i in range(n)]


def _heisenberg(bonds):
    return [{"expression": f"σ{c}₀ σ{c}₁", "sites": bonds} for c in "ˣʸᶻ"]


def _hopping(bonds):
    return [{"expression": "σ⁺₀ σ⁻₁", "sites": bonds}, {"expression": "σ⁻₀ σ⁺₁", "sites": bonds}]


def _complex_hopping(bonds):
    """(1 + 0.3i) σ⁺σ⁻ + h.c. on every bond: one group per bond, complex coefficients."""
    return _hopping(bonds) + [{"expression": "0.3j × σ⁺₀ σ⁻₁", "sites": bonds},
                              {"expression": "-0.3j × σ⁻₀ σ⁺₁", "sites": bonds}]


def _zz(bonds, j=0.7):
    return [{"expression": f"{j} × σᶻ₀ σᶻ₁", "sites": bonds}]


def _yz(bonds):
    """σʸᵢ σᶻⱼ: Hermitian, imaginary matrix elements, invariant under spin inversion; its flip mask is bit i alone."""
    return [{"expression": "0.4 × σʸ₀ σᶻ₁", "sites": bonds}]


def _translations(n, sector, mirror=False):
    gens = [{"permutation": [(i + 1) % n for i in range(n)], "sector": sector}]
    if mirror:
        gens.append({"permutation": [n - 1 - i for i in range(n)], "sector": 0})
    return gens


def _custom(n, hw, terms, **basis_kw):
    basis = basis_from_dict({"number_spins": n, "hamming_weight": hw, **basis_kw})
    return basis, operator_from_dict({"terms": terms}, basis)


def _ring_distances(n, ds):
    return [b for d in ds for b in _ring(n, d)]


# name: (builder, flip-mask groups)
MODELS = {
    # no projection: identity index (no fixed weight), then fixed weight 8 of 17 sites on the first k pairs of the
    # all-to-all graph; from 128 groups on, rows emit more than 64 terms
    "none_12_identity_g65": (lambda: _custom(12, None, _heisenberg(_pairs(12)[:65])), 65),
    "none_17w8_g63": (lambda: _custom(17, 8, _heisenberg(_pairs(17)[:63])), 63),
    "none_17w8_g64_complex": (lambda: _custom(17, 8, _complex_hopping(_pairs(17)[:64]) + _zz(_pairs(17)[:64])), 64),
    "none_17w8_g128": (lambda: _custom(17, 8, _heisenberg(_pairs(17)[:128])), 128),
    "none_17w8_g129_complex": (lambda: _custom(17, 8, _complex_hopping(_pairs(17)[:129]) + _zz(_ring(17, 1))), 129),
    "none_14w7_no_diagonal": (lambda: _custom(14, 7, _hopping(_pairs(14))), 91),
    "none_14w7_diagonal_only": (lambda: _custom(14, 7, _zz(_pairs(14)[:40])), 0),
    # 64 sites: the ring's bond (63, 0) flips bit 63
    "none_64w3_g128": (lambda: _custom(64, 3, _heisenberg(_ring_distances(64, (1, 2)))), 128),
    # spin inversion: both characters, fixed weight and (with complex coefficients) free magnetisation
    "inversion_18w9_g129": (lambda: _custom(18, 9, _heisenberg(_pairs(18)[:129]), spin_inversion=-1), 129),
    "inversion_18w9_g64": (lambda: _custom(18, 9, _heisenberg(_pairs(18)[:64]) + _zz(_ring(18, 2)),
                                           spin_inversion=1), 64),
    "inversion_14_g65_complex": (lambda: _custom(14, None, _yz(_ring(14, 1)) + _heisenberg(_pairs(14)[:51]),
                                                 spin_inversion=1), 65),
    # permutation groups: trivial characters (real and complex operator), complex characters
    "group_ring16w8_k0_g64": (lambda: _custom(16, 8, _heisenberg(_ring_distances(16, (1, 2, 3, 4))),
                                              symmetries=_translations(16, 0, mirror=True)), 64),
    "group_ring13_k0_g65_complex": (lambda: _custom(13, None, _yz(_ring(13, 1)) +
                                                    _heisenberg(_ring_distances(13, (1, 2, 3, 4))),
                                                    symmetries=_translations(13, 0)), 65),
    # momentum 3 of 16: every state of period 8 or less has norm zero, and flips reach such states
    "group_ring16w8_k3_g64": (lambda: _custom(16, 8, _heisenberg(_ring_distances(16, (1, 2, 3, 4))),
                                              symmetries=_translations(16, 3)), 64),
    "group_ring32w3_k1_g128": (lambda: _custom(32, 3, _heisenberg(_ring_distances(32, (1, 2, 3, 4))),
                                               symmetries=_translations(32, 1)), 128),
}
# 2^17 states: a host x is copied in chunks under the k_generate launches (single rank, at least 2^16 states)
PIPELINED = {"none_17_identity_g129": (lambda: _custom(17, None, _heisenberg(_pairs(17)[:129])), 129)}

# the stepwise record routing: no symmetry, spin inversion, a group with complex characters (and zero-norm targets)
ROUTE_MODELS = {
    "none_13w6_g65": (lambda: _custom(13, 6, _heisenberg(_pairs(13)[:65])), 65),
    "inversion_12w6_g40": (lambda: _custom(12, 6, _heisenberg(_pairs(12)[:40]), spin_inversion=-1), 40),
    "group_ring12w6_k1_complex": (lambda: _custom(12, 6, _heisenberg(_ring_distances(12, (1, 2, 3))) +
                                                  _complex_hopping(_ring(12, 4)),
                                                  symmetries=_translations(12, 1)), 48),
}

ALL_MODELS = {**MODELS, **PIPELINED, **ROUTE_MODELS}


@functools.lru_cache(maxsize=None)
def _model(name):
    return ALL_MODELS[name][0]()


@functools.lru_cache(maxsize=None)
def _reps(name):
    return po.enumerate_states(_model(name)[0])[0]


@functools.lru_cache(maxsize=None)
def _oracle(name):
    """Representatives and the single-rank y of both element types.  x by the _x recipe; y0 (seed 9) is the y the
    product starts from: the operator without diagonal terms adds to it, every other one overwrites it."""
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    basis, matrix = _model(name)
    reps = _reps(name)
    ys = {}
    for cplx in (False, True):
        x, y0 = _x(reps.shape[0], cplx), _x(reps.shape[0], cplx, seed=9)
        start = y0.copy() if len(matrix.diag) == 0 else np.zeros_like(y0)
        ys[cplx] = (x, y0, po.matvec_blocks(matrix, [reps], [x], y_blocks=[start], num_tasks=po.num_threads())[0])
    return reps, ys


@functools.lru_cache(maxsize=None)
def _records(name):
    """The oracle's off-diagonal records of the whole basis (x = 1), 2048 rows at a time: their number, the most one
    row emits, and (below 2^16 states) the records themselves."""
    basis, matrix = _model(name)
    reps = _reps(name)
    total, most, betas, coeffs = 0, 0, [], []
    for lo in range(0, reps.shape[0], 2048):
        b, c, _, offsets = po.compute_off_diag(matrix, 1, reps[lo:lo + 2048], np.ones(min(2048, reps.shape[0] - lo)))
        total += b.shape[0]
        most = max(most, int(np.diff(offsets).max(initial=0)))
        if reps.shape[0] < 1 << 16:
            betas.append(b)
            coeffs.append(c)
    return total, most, (np.concatenate(betas), np.concatenate(coeffs)) if betas else None


@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


# ---- the models are what they claim (no device needed) ----------------------------------------------------------------

@pytest.mark.parametrize("name", sorted(ALL_MODELS))
def test_model_shapes(name):
    """Flip-mask group counts (distinct flip masks), rows of more than 64 terms where claimed, no diagonal / no
    off-diagonal terms, flips of bit 63, zero-norm targets of the momentum-3 sector."""
    basis, matrix = _model(name)
    assert np.unique(matrix.off_diag.x).shape[0] == ALL_MODELS[name][1], name
    if name in ("none_17w8_g128", "none_17w8_g129_complex", "inversion_18w9_g129", "none_17_identity_g129"):
        assert _records(name)[1] > 64, name
    if name == "none_14w7_no_diagonal":
        assert len(matrix.diag) == 0
    if name == "none_14w7_diagonal_only":
        assert len(matrix.off_diag) == 0 and len(matrix.diag) > 0
    if name == "none_64w3_g128":
        assert np.any(matrix.off_diag.x >> np.uint64(63))
        betas = _records(name)[2][0]
        assert np.any(betas >> np.uint64(63)) and np.any((betas >> np.uint64(63)) == 0)
    if name in ("group_ring16w8_k3_g64", "group_ring12w6_k1_complex"):
        reps = _reps(name)
        betas, coeffs = _records(name)[2]
        lost = ~np.isin(betas, reps)
        assert np.any(lost) and np.all(coeffs[lost] == 0)   # targets of norm zero: coefficient zero in the oracle


# ---- 1. k_generate at every row split -------------------------------------------------------------------------------

def _device(op, x, y0):
    y = op.matvec(torch.from_numpy(x).cuda(), torch.from_numpy(y0.copy()).cuda())
    torch.cuda.synchronize()
    return y.cpu().numpy()


def _check_split(op, split):
    s = op.info("push_split")
    if split > 0:
        assert s == split, (split, s)
    else:   # auto: a power of two, and never more lanes than groups
        assert s in (1, 2, 4, 8, 16, 32) and s <= max(1, op.info("n_groups")), s


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MODELS) + sorted(PIPELINED))
def test_generate_every_row_split(need_cuda, name):
    """mode = 0 on one rank, push_split 1 .. 32 and auto, float64 and complex128, device and host pointers: y in full
    against the oracle; info("push_split") is the forced S; the plan's count is the oracle's at every S."""
    basis, matrix = _model(name)
    reps, ys = _oracle(name)
    total = _records(name)[0]
    op = Operator(matrix)
    try:
        op.set_option("mode", 0)
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        assert op.info("n_groups") == ALL_MODELS[name][1] and op.info("pull") == 0
        for split in SPLITS:
            op.set_option("push_split", split)
            _check_split(op, split)
            assert np.array_equal(op.plan(), [total]), split
            _check_split(op, split)
            for cplx in (False, True):
                x, y0, y_ref = ys[cplx]
                where = (name, split, cplx)
                y = _device(op, x, y0)
                assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
                y = op.matvec(x, y0.copy())   # host vectors (in chunks under the kernel from 2^16 states on)
                assert _close(y, y_ref), (where, "host", np.abs(y - y_ref).max())
    finally:
        op.close()


# ---- 2. k_pull on the same models -----------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(MODELS))
def test_pull_every_index_kind(need_cuda, name):
    """mode = 1, rows = 0, gather = 0 (the queued k_pull) with every index kind the basis takes: y in full against the
    oracle, float64 and complex128; without a permutation group bit-identical across index kinds and repeated calls."""
    basis, matrix = _model(name)
    reps, ys = _oracle(name)
    op = Operator(matrix)
    try:
        for key, value in (("mode", 1), ("rows", 0), ("gather", 0)):
            op.set_option(key, value)
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        assert (op.info("pull"), op.info("gather"), op.info("rows")) == (1, 0, 0)
        assert op.info("n_groups") == ALL_MODELS[name][1]
        group = basis.has_permutation_symmetries()
        for cplx in (False, True):
            x, y0, y_ref = ys[cplx]
            got = {}
            for index in INDEX_KINDS:
                op.set_option("index", index)
                mode = op.info("index_mode")
                y = _device(op, x, y0)
                where = (name, cplx, index, mode)
                assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
                if not group:
                    assert np.array_equal(_device(op, x, y0), y), where
                    assert np.array_equal(op.matvec(x, y0.copy()), y), where
                got[mode] = y
            if not group:
                first = next(iter(got.values()))
                assert all(np.array_equal(y, first) for y in got.values()), (name, cplx, sorted(got))
            # which index kinds the basis takes: identity without a fixed weight or a projection; else the directory,
            # and for a whole fixed-weight sector the combinadic rank and (up to 40 sites) the Lin tables
            if group:
                expect = {0}
            elif basis.hamming_weight is None:
                expect = {0} if basis.spin_inversion else {1}
            else:
                expect = {0, 2} | ({3} if basis.number_sites <= 40 else set())
            assert set(got) == expect, (name, sorted(got))
    finally:
        op.close()


# ---- 3. record routing from 2 to 256 ranks --------------------------------------------------------------------------

def _global_norms(cl, masks):
    return hashed_to_block([op.basis.norms() for op in cl.ops], masks)


def _products(cl, xb):
    """One product through the stepwise API on the current plan (no dmv_plan here): generate on every rank, read every
    rank's outgoing records, then each destination accumulates what the others made for it."""
    elt = _elt_of(xb[0])
    width = 2 if (elt == 2 or cl.ops[0].info("complex_coefficients") == 1) else 1
    ys = [torch.zeros_like(x) for x in xb]
    for r, op in enumerate(cl.ops):
        op.generate(xb[r], ys[r])
    for op in cl.ops:
        op.synchronize()
    records = []
    for r, src in enumerate(cl.ops):
        b0, c0, _ = src.outgoing(0)
        regions, total = [], 0
        for q in range(cl.num_ranks):
            b, c, n = src.outgoing(q)
            assert b == b0 + 8 * total and c == c0 + 8 * width * total, (r, q)   # flat regions, `width` doubles each
            regions.append(n)
            total += n
        betas = _device_tensor(b0, total, torch.int64, src.device).cpu().numpy().view(np.uint64) if total else \
            np.zeros(0, dtype=np.uint64)
        coeffs = _device_tensor(c0, total * width, torch.float64, src.device).cpu().numpy() if total else np.zeros(0)
        coeffs = coeffs.view(np.complex128) if width == 2 else coeffs.astype(np.complex128)
        records.append((np.array(regions), betas, coeffs))
    for r, src in enumerate(cl.ops):
        for q, dst in enumerate(cl.ops):
            if q != r:
                b, c, n = src.outgoing(q)
                if n > 0:
                    dst.accumulate(elt, n, b, c, ys[q])
    for op in cl.ops:
        op.synchronize()
    return ys, records


def _sorted_records(betas, coeffs):
    order = np.lexsort((np.round(coeffs.imag, 9), np.round(coeffs.real, 9), betas))
    return betas[order], coeffs[order]


def _check_records(name, matrix, P, blocks, xb, records, norm_of):
    """Every bucket equals, as a multiset, the oracle's records of that key for the sender's block.  The library's
    records still carry 1 / norm(beta) of the target (applied by the owner): norm_of(beta) undoes it (0 for a target of
    norm zero, which the oracle's record carries as coefficient 0)."""
    for r in range(P):
        regions, betas, coeffs = records[r]
        ob, oc, ok, _ = po.compute_off_diag(matrix, P, blocks[r], xb[r].cpu().numpy())
        want = np.bincount(ok, minlength=P)
        want[r] = 0
        assert np.array_equal(regions, want), (name, P, r)
        if norm_of is not None:
            coeffs = coeffs * norm_of(betas)
        start = np.concatenate([[0], np.cumsum(regions)])
        for q in np.flatnonzero(regions):
            gb, gc = _sorted_records(betas[start[q]:start[q + 1]], coeffs[start[q]:start[q + 1]])
            wb, wc = _sorted_records(ob[ok == q], oc[ok == q])
            assert np.array_equal(gb, wb), (name, P, r, q)
            floor = 1e-14 * max(1.0, float(np.abs(wc).max(initial=0.0)))
            assert np.allclose(gc, wc, rtol=1e-12, atol=floor), (name, P, r, q, np.abs(gc - wc).max())


@pytest.mark.gpu
@pytest.mark.parametrize("P", RANKS)
@pytest.mark.parametrize("name", sorted(ROUTE_MODELS))
def test_routing_from_2_to_256_ranks(need_cuda, name, P):
    """P logical ranks on one GPU: the plan's counts per destination are the oracle's buckets; four products in a row
    on one plan (float64, complex128, float64, complex128: the record width alternates on a real operator, and out_count
    is reset before every generate) equal the oracle's P-rank product; every bucket equals the oracle's records of that
    key as a multiset (beyond 32 ranks the order inside a bucket is not defined)."""
    basis, matrix = _model(name)
    reps = _reps(name)
    masks, blocks = po.partition_by_hash(reps, P)
    t0, free0 = time.perf_counter(), torch.cuda.mem_get_info()[0]
    cl = EmulatedCluster(matrix, P).build()
    try:
        assert all(np.array_equal(op.basis.representatives(), blocks[r]) for r, op in enumerate(cl.ops))
        assert all(op.info("n_groups") == ALL_MODELS[name][1] for op in cl.ops)
        counts = np.array([op.plan() for op in cl.ops])
        for r in range(P):
            _, _, keys, _ = po.compute_off_diag(matrix, P, blocks[r], np.ones(blocks[r].shape[0]))
            assert np.array_equal(counts[r], np.bincount(keys, minlength=P)), (name, P, r)
        gnorms = _global_norms(cl, masks) if basis.has_permutation_symmetries() else None
        norm_of = None
        if gnorms is not None:
            def norm_of(b):
                i = np.minimum(np.searchsorted(reps, b), reps.shape[0] - 1)
                return np.where(reps[i] == b, gnorms[i], 0.0)
        for step, cplx in enumerate((False, True, False, True)):
            x = _x(reps.shape[0], cplx, 60 + step)
            y_ref = po.matvec_global(matrix, reps, x, P, num_tasks=po.num_threads())
            xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
            ys, records = _products(cl, xb)
            y = hashed_to_block([t.cpu().numpy() for t in ys], masks)
            assert _close(y, y_ref), (name, P, step, np.abs(y - y_ref).max())
            _check_records(name, matrix, P, blocks, xb, records, norm_of)
        assert np.array_equal(np.array([op.plan() for op in cl.ops]), counts)
        used = (free0 - torch.cuda.mem_get_info()[0]) / 2**20
    finally:
        cl.close()
    print(f"{name} P={P}: {time.perf_counter() - t0:.2f} s with the cluster, {used:.0f} MiB of device memory, "
          f"{sum(b.shape[0] == 0 for b in blocks)} ranks without a state")


@pytest.mark.gpu
@pytest.mark.parametrize("P", [3, 33])
def test_push_split_change_replans(need_cuda, P):
    """push_split changed between products on a live plan (no dmv_plan call in between): the next generate plans again
    for the new S (grid and per-warp offsets follow S up to 32 ranks), info reports it, and y stays the oracle's."""
    name = "none_13w6_g65"
    basis, matrix = _model(name)
    reps = _reps(name)
    masks, blocks = po.partition_by_hash(reps, P)
    cl = EmulatedCluster(matrix, P).build()
    try:
        counts = np.array([op.plan() for op in cl.ops])
        for step, split in enumerate((-1, 32, 1, 4, 16)):
            if split != -1:
                for op in cl.ops:
                    op.set_option("push_split", split)
                    assert op.info("push_split") == split
            for cplx in (False, True):
                x = _x(reps.shape[0], cplx, 70 + step)
                y_ref = po.matvec_global(matrix, reps, x, P, num_tasks=po.num_threads())
                xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
                ys, records = _products(cl, xb)
                y = hashed_to_block([t.cpu().numpy() for t in ys], masks)
                assert _close(y, y_ref), (P, split, cplx, np.abs(y - y_ref).max())
                _check_records(name, matrix, P, blocks, xb, records, None)
        assert np.array_equal(np.array([op.plan() for op in cl.ops]), counts)
    finally:
        cl.close()


@pytest.mark.gpu
@pytest.mark.parametrize("P", [64, 256])
@pytest.mark.parametrize("name", sorted(ROUTE_MODELS))
def test_compute_off_diag_keys_beyond_32_ranks(need_cuda, name, P):
    """dmv_compute_off_diag on a context of P ranks: every key is locale_idx_of(beta, P), and the records are the
    oracle's as a multiset, float64 and complex128."""
    basis, matrix = _model(name)
    reps = _reps(name)
    op = Operator(matrix, rank=0, num_ranks=P)
    try:
        bo = BatchedOperator(op, reps.shape[0])
        for cplx in (False, True):
            xs = _x(reps.shape[0], cplx, 5)
            n, betas, coeffs, keys = bo.computeOffDiag(reps.shape[0], reps, xs)
            ob, oc, ok, _ = po.compute_off_diag(matrix, P, reps, xs)
            assert n == ob.shape[0] and np.array_equal(keys, po.locale_idx_of(betas, P)), (name, P, cplx)
            assert keys.max() >= 32
            order, oorder = np.lexsort((coeffs.imag, coeffs.real, betas)), np.lexsort((oc.imag, oc.real, ob))
            assert np.array_equal(betas[order], ob[oorder]) and np.array_equal(keys[order], ok[oorder])
            assert np.allclose(coeffs[order], oc[oorder], rtol=1e-12, atol=1e-14)
    finally:
        op.close()


@pytest.mark.gpu
def test_forms_limited_to_32_ranks_refuse_33(need_cuda):
    """The replicated-x set-up and the device block <-> hashed redistribution hold one slot or cursor per rank in a
    warp: at 33 ranks they raise an error (and the context still computes products)."""
    name = "none_13w6_g65"
    basis, matrix = _model(name)
    reps = _reps(name)
    P = 33
    masks, blocks = po.partition_by_hash(reps, P)
    cl = EmulatedCluster(matrix, P).build()
    try:
        op = cl.ops[0]
        with pytest.raises(Exception, match="32 ranks"):
            op.replicated_setup()
        with pytest.raises(Exception, match="32 ranks"):
            op.hashed_positions(masks, P)
        chunk = _x(reps.shape[0], False)[:100]
        with pytest.raises(Exception, match="32 ranks"):
            op.block_to_hashed(chunk, masks[:100])
        with pytest.raises(Exception, match="32 ranks"):
            op.hashed_to_block(np.zeros(blocks[0].shape[0]), masks[:100])
        x = _x(reps.shape[0], True, 80)
        ys, _ = _products(cl, [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)])
        y = hashed_to_block([t.cpu().numpy() for t in ys], masks)
        assert _close(y, po.matvec_global(matrix, reps, x, P))
    finally:
        cl.close()
