"""Every build of k_rows that set_option can select, in full vector against the CPU oracle.

launch_rows picks one of about 30 instantiations of k_rows: the element type (float64 / complex128), the orbit minimum
(TK = 6 / 4: the square-torus form of the 6x6 / 4x4 lattice; 0: the generic orbit walk), the look-up table (ordered by key
prefix with 2^rows_table_bits directory blocks and rows_table_buckets buckets per state, hashed homes, or the perfect
hash) and the CTAs per SM it is compiled for (rows_ctas 2, 3 or 4; the 3- and 4-CTA builds have other register
allocations).  The bases here are the 6x6 and 4x4 tori at every Hamming weight the oracle computes in about a second:
small bases that still take the torus orbit minimum, and that hold the states with the largest stabilisers (periodic
patterns, stripes), the ones that tie in pass 1 of orbit_min_torus_sq and expand several candidates in pass 2.  Their
dimensions are pinned from outside the oracle by Burnside's lemma.

Criterion: _close of test_gpu_parity (the reference's |a - b| <= max(atol, rtol max(|a|, |b|))), unchanged.  Products on
one table build that differ only in rows_ctas are bit-identical: rows_ctas does not rebuild the table, and a lane sums its
row in program order.
"""
import functools
import os

import numpy as np
import pytest
import yaml

import burnside
from distributed_matvec_b200 import EmulatedCluster, Operator, block_to_hashed, hashed_to_block, load_config_from_yaml
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
from oracle import pyoracle as po
from test_gpu_parity import _close, _recipe_x, _x

torch = pytest.importorskip("torch")

DATA = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "data")

# (lattice, Hamming weight, spin inversion): spin inversion only at half filling, both of its sectors on the 4x4.
# Weights 0, 1, 35 and 36 of the 6x6 have one representative: the ordered directory then spans a key range of 0.
SECTORS = ([("heisenberg_square_6x6", w, None) for w in (0, 1, 2, 3, 4, 5, 6, 7, 29, 30, 31, 32, 33, 34, 35, 36)] +
           [("heisenberg_square_4x4", w, None) for w in range(17) if w != 8] +
           [("heisenberg_square_4x4", 8, 1), ("heisenberg_square_4x4", 8, -1)])
TORUS_SIDE = {"heisenberg_square_6x6": 6, "heisenberg_square_4x4": 4}
# bases of the generic orbit walk (TK = 0): a kagome cluster, a chain (block-rotation canonical form), and the lattice of
# issue_01 in the trivial sector of its one reflection (issue_01 itself has character -1, which k_rows does not take)
GENERIC = [("heisenberg_kagome_12_symm", None, None), ("heisenberg_chain_24_symm", None, None),
           ("issue_01", None, 0)]

# look-up tables of k_rows: every option is set each time, so that no setting carries over into the next
TABLES = {
    "ordered_14_8": dict(rows_index=-1, rows_table=1, rows_table_bits=14, rows_table_buckets=8),
    "ordered_14_2": dict(rows_index=-1, rows_table=1, rows_table_bits=14, rows_table_buckets=2),
    "ordered_8_4": dict(rows_index=-1, rows_table=1, rows_table_bits=8, rows_table_buckets=4),
    "ordered_1_8": dict(rows_index=-1, rows_table=1, rows_table_bits=1, rows_table_buckets=8),
    "ordered_1_2": dict(rows_index=-1, rows_table=1, rows_table_bits=1, rows_table_buckets=2),
    "hashed": dict(rows_index=-1, rows_table=0, rows_table_bits=14, rows_table_buckets=8),
    "perfect_hash": dict(rows_index=1, rows_table=1, rows_table_bits=14, rows_table_buckets=8),
}
CTAS = (2, 3, 4)


def _sector_id(s):
    name, w, inv = s
    return f"{name.replace('heisenberg_', '')}-w{w}" + ("" if inv is None else f"-inv{inv:+d}")


def _generic_id(s):
    return s[0] + ("" if s[2] is None else f"-sector{s[2]}")


@functools.lru_cache(maxsize=None)
def _model(name, weight=None, inversion=None):
    """The yaml model with its Hamming weight overridden; spin inversion dropped off half filling, else set to
    `inversion` when given.  For the generic bases `inversion` overrides the sector of the first generator instead."""
    with open(os.path.join(DATA, name + ".yaml"), encoding="utf-8") as f:
        conf = yaml.safe_load(f)
    b = dict(conf["basis"])
    if name in TORUS_SIDE:
        b["hamming_weight"] = weight
        if 2 * weight != b["number_spins"]:
            b.pop("spin_inversion", None)
        elif inversion is not None:
            b["spin_inversion"] = inversion
    elif inversion is not None:
        b["symmetries"] = [dict(g) for g in b["symmetries"]]
        b["symmetries"][0]["sector"] = inversion
    basis = basis_from_dict(b)
    return basis, operator_from_dict(conf["hamiltonian"], basis)


@functools.lru_cache(maxsize=None)
def _oracle(name, weight=None, inversion=None):
    """Representatives and y = H x of both element types (x by the _x recipe), from the CPU oracle."""
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    basis, matrix = _model(name, weight, inversion)
    reps, _ = po.enumerate_states(basis)
    ys = {}
    for cplx in (False, True):
        x = _x(reps.shape[0], cplx)
        ys[cplx] = (x, po.matvec_global(matrix, reps, x, 1, num_tasks=po.num_threads()))
    return reps, ys


def _trivial(basis):
    return basis.group.all_characters_trivial


@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _set(op, **options):
    for k, v in options.items():
        op.set_option(k, v)


def _product(op, x):
    y = op.matvec(torch.from_numpy(x).cuda())
    torch.cuda.synchronize()
    return y.cpu().numpy()


@pytest.mark.parametrize("sector", SECTORS, ids=_sector_id)
def test_sector_dimension_by_burnside(sector):
    """The oracle's enumeration of every sector used below has the dimension Burnside's lemma counts (the -1 sector of
    spin inversion has a non-trivial character: the orbit count bounds it from above)."""
    basis, _ = _model(*sector)
    reps, norms = po.enumerate_states(basis)
    g = basis.group
    count = burnside.dimension(g.perms, g.flips, basis.hamming_weight)
    assert np.all(np.diff(reps.astype(np.int64)) > 0) and np.all(norms > 0)
    if _trivial(basis):
        assert reps.shape[0] == count, (sector, reps.shape[0], count)
    else:
        assert 0 < reps.shape[0] <= count
    if sector[1] in (0, 1, 35, 36) and sector[0] == "heisenberg_square_6x6":
        assert reps.shape[0] == 1


def _matrix(op, sector, expect_tk):
    """Every table x rows_ctas x element type on one operator, against the oracle; bit-identity over rows_ctas."""
    reps, ys = _oracle(*sector)
    op.basis.build()
    assert np.array_equal(op.basis.representatives(), reps)
    for cplx in (False, True):
        x, y_ref = ys[cplx]
        for table, options in TABLES.items():
            _set(op, **options)
            first = None
            for ctas in CTAS:
                op.set_option("rows_ctas", ctas)
                y = _product(op, x)
                where = (_sector_id(sector), cplx, table, ctas)
                assert op.info("rows") == 1, where
                assert op.info("rows_tk") == expect_tk(table, ctas), (where, op.info("rows_tk"))
                assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
                if first is None:
                    first = y
                else:
                    assert np.array_equal(y, first), (where, np.abs(y - first).max())
    _set(op, rows_ctas=2, **TABLES["ordered_14_8"])


@pytest.mark.gpu
@pytest.mark.parametrize("sector", SECTORS, ids=_sector_id)
def test_rows_configurations_on_torus_sectors(need_cuda, sector):
    """Each table (ordered at 2^14 / 2^8 / 2 directory blocks and 8 / 4 / 2 buckets per state, hashed, perfect hash) x
    rows_ctas 2 / 3 / 4 x float64 / complex128, in full vector against the oracle.  TK is 6 on every 6x6 sector; on
    the 4x4 it is 4 except for the 4-CTA build of the open-addressing tables, which has no 4x4 form (TK = 0)."""
    basis, matrix = _model(*sector)
    op = Operator(matrix)
    try:
        if not _trivial(basis):
            # the -1 sector of spin inversion: k_rows does not apply, the product still matches
            assert op.info("rows_ok") == 0
            reps, ys = _oracle(*sector)
            op.basis.build()
            assert np.array_equal(op.basis.representatives(), reps)
            for cplx in (False, True):
                x, y_ref = ys[cplx]
                y = _product(op, x)
                assert op.info("rows") == 0
                assert _close(y, y_ref), (cplx, np.abs(y - y_ref).max())
            return
        assert op.info("rows_ok") == 1
        side = TORUS_SIDE[sector[0]]
        _matrix(op, sector, lambda table, ctas: 0 if (side == 4 and ctas == 4 and table != "perfect_hash") else side)
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("base", GENERIC, ids=_generic_id)
def test_rows_configurations_on_generic_walk(need_cuda, base):
    """The same matrix on bases whose orbit minimum is the generic walk (TK = 0 in every build)."""
    basis, matrix = _model(*base)
    assert _trivial(basis)
    op = Operator(matrix)
    try:
        assert op.info("rows_ok") == 1
        _matrix(op, base, lambda table, ctas: 0)
    finally:
        op.close()


@pytest.mark.gpu
def test_issue_01_keeps_off_k_rows(need_cuda):
    """issue_01 as given (character -1 of its reflection): no k_rows, and the product matches the oracle."""
    basis, matrix = _model("issue_01")
    assert not _trivial(basis)
    reps, ys = _oracle("issue_01")
    op = Operator(matrix)
    try:
        assert op.info("rows_ok") == 0
        op.basis.build()
        for cplx in (False, True):
            x, y_ref = ys[cplx]
            assert _close(_product(op, x), y_ref)
            assert op.info("rows") == 0
    finally:
        op.close()


@pytest.mark.gpu
def test_option_switching_on_one_operator(need_cuda):
    """Table layouts and element types switched back and forth on one live operator: every switch rebuilds the table
    (table_elt = 0) and, leaving the ordered layout, drops its directory; every product is checked.  Out-of-range
    values raise and leave the operator as it was."""
    sector = ("heisenberg_square_6x6", 6, None)
    basis, matrix = _model(*sector)
    reps, ys = _oracle(*sector)
    op = Operator(matrix)
    try:
        op.basis.build()
        steps = [("ordered_14_8", True), ("hashed", True), ("hashed", False), ("ordered_1_8", False),
                 ("ordered_1_8", True), ("perfect_hash", True), ("perfect_hash", False), ("ordered_14_8", False),
                 ("ordered_14_8", True), ("ordered_1_2", True), ("hashed", True), ("ordered_14_8", True)]
        for k, (table, cplx) in enumerate(steps):
            _set(op, **TABLES[table])
            x, y_ref = ys[cplx]
            y = _product(op, x)
            assert op.info("rows") == 1 and op.info("rows_tk") == 6
            assert _close(y, y_ref), (k, table, cplx, np.abs(y - y_ref).max())
        for key, value in (("rows_table", 2), ("rows_table", -1), ("rows_table_bits", 0), ("rows_table_bits", 15),
                           ("rows_table_buckets", 3), ("rows_table_buckets", 16)):
            with pytest.raises(Exception, match=key):
                op.set_option(key, value)
        x, y_ref = ys[False]
        assert _close(_product(op, x), y_ref)
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("weight", [6, 30])
def test_rows_batch_on_torus_sectors(need_cuda, weight):
    """k_rows_batch (TK = 6) with 1 .. 6 float64 and 1 .. 3 complex128 columns: every column in full against the
    oracle's product of that column (one column goes through k_rows)."""
    sector = ("heisenberg_square_6x6", weight, None)
    basis, matrix = _model(*sector)
    reps, _ = _oracle(*sector)
    n = reps.shape[0]
    op = Operator(matrix)
    try:
        op.basis.build()
        assert op.info("rows") == 1 and op.info("rows_tk") == 6
        for cplx, most in ((False, 6), (True, 3)):
            X = np.stack([_x(n, cplx, 600 + j) for j in range(most)])
            want = [po.matvec_global(matrix, reps, X[j], 1, num_tasks=po.num_threads()) for j in range(most)]
            for k in range(1, most + 1):
                Y = op.matvec_batch(torch.from_numpy(X[:k]).cuda())
                torch.cuda.synchronize()
                Y = Y.cpu().numpy()
                for j in range(k):
                    assert _close(Y[j], want[j]), (weight, cplx, k, j, np.abs(Y[j] - want[j]).max())
    finally:
        op.close()


@pytest.mark.gpu
def test_emulated_ranks_with_other_tables(need_cuda):
    """Three logical ranks on the 6x6 weight-7 sector with the hashed table and with the ordered table at 2 blocks and
    2 buckets per state, set on every rank after the replicated form has made its whole-basis context (the options are
    mirrored onto it, and its table is rebuilt): the record exchange and the replicated-x product (k_rows on the whole
    basis) against the oracle's 3-rank product."""
    P = 3
    sector = ("heisenberg_square_6x6", 7, None)
    basis, matrix = _model(*sector)
    reps, _ = _oracle(*sector)
    masks, _ = po.partition_by_hash(reps, P)
    cl = EmulatedCluster(matrix, P).build()
    try:
        assert all(op.info("rows_ok") == 1 for op in cl.ops)     # the replicated form runs k_rows on the whole basis
        xs = {}
        for cplx in (False, True):
            x = _x(reps.shape[0], cplx, 41)
            xs[cplx] = (x, po.matvec_global(matrix, reps, x, P, num_tasks=po.num_threads()))
            xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
            y = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)   # default table
            assert _close(y, xs[cplx][1])
        for options in (dict(rows_table=0), dict(rows_table=1, rows_table_bits=1, rows_table_buckets=2)):
            for op in cl.ops:
                _set(op, **options)
            for cplx in (False, True):
                x, y_ref = xs[cplx]
                xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
                y_rec = hashed_to_block([t.cpu().numpy() for t in cl.matvec(xb)], masks)
                assert _close(y_rec, y_ref), (options, cplx, np.abs(y_rec - y_ref).max())
                y_rep = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)
                assert _close(y_rep, y_ref), (options, cplx, np.abs(y_rep - y_ref).max())
    finally:
        cl.close()


# ---- at size: heisenberg_square_6x6, weight 18, spin inversion +1 (15 804 956 states)

@pytest.fixture(scope="module")
def square_6x6(need_cuda):
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    basis, matrix = load_config_from_yaml(os.path.join(DATA, "heisenberg_square_6x6.yaml"))
    op = Operator(matrix)
    op.basis.build()
    reps = op.basis.representatives()
    assert reps.shape[0] == 15804956
    yield matrix, op, reps
    op.close()


@pytest.mark.gpu
def test_torus_6x6_at_size_sampled_rows(square_6x6):
    """k_rows<float64, TK = 6> on the 4096 sampled rows against the oracle (no other test reaches it), and the
    complex128 product with the ordered table at 2 buckets per state and with the hashed table."""
    matrix, op, reps = square_6x6
    n = reps.shape[0]
    rows = np.sort(np.random.default_rng(5).choice(n, size=4096, replace=False))
    rows_d = torch.from_numpy(rows).cuda()
    for cplx, tables in ((False, ("ordered_14_8",)), (True, ("ordered_14_2", "hashed"))):
        x = _recipe_x(n, cplx)
        expect = po.expected_rows(matrix, reps, x, rows)
        xd = torch.from_numpy(x).cuda()
        for table in tables:
            _set(op, **TABLES[table])
            y = op.matvec(xd)
            got = y[rows_d].cpu().numpy()
            del y
            assert op.info("rows") == 1 and op.info("rows_tk") == 6
            assert _close(got, expect), (cplx, table, np.abs(got - expect).max())
        del xd
    _set(op, **TABLES["ordered_14_8"])


@pytest.mark.gpu
def test_torus_6x6_at_size_full_vector_against_chain_walk(square_6x6):
    """All 15.8 M elements of the default product (k_rows, torus orbit minimum) against the product with the canonical
    form switched off (canon = 0: k_rows with the group-chain walk, which shares no code with the torus tables)."""
    matrix, op, reps = square_6x6
    x = torch.from_numpy(_recipe_x(reps.shape[0], True)).cuda()
    assert op.info("rows_tk") == 6
    y_torus = op.matvec(x).cpu().numpy()
    op.set_option("canon", 0)
    try:
        assert op.info("canon_mode") == 0 and op.info("rows_tk") == 0
        y_walk = op.matvec(x).cpu().numpy()
    finally:
        op.set_option("canon", -1)
    assert _close(y_torus, y_walk), np.abs(y_torus - y_walk).max()
