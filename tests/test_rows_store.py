"""The term store of the row kernel (k_rows_stored, csrc/dmv_store.cu) against the CPU oracle and against k_rows.

The store keeps the target index and a coefficient code of every term k_rows accumulates, once per basis and rows; a
product reads it in C column blocks whose scaled x stays in L2.  Each row's sum runs block by block and within a block
in k_rows' term order with k_rows' coefficients and (n x) products, so at C = 1 the product equals k_rows' bit for bit;
at C > 1 only the order of each row's sum changes.  The small sectors here are below the size at which the store is
chosen automatically, so they force it through dmv_debug_rows_store.

Criterion: _close of test_gpu_parity, unchanged.
"""
import ctypes as C
import os

import numpy as np
import pytest

from distributed_matvec_b200 import EmulatedCluster, Operator, block_to_hashed, hashed_to_block, load_config_from_yaml
from distributed_matvec_b200 import _native as nat
from oracle import pyoracle as po
from test_gpu_parity import _close, _recipe_x, _x
from test_rows_kernels import DATA, GENERIC, SECTORS, _generic_id, _model, _oracle, _product, _sector_id, _set

torch = pytest.importorskip("torch")

F64, C128 = 1, 2
H100_L2 = 50 * 1024 * 1024
GB = 1 << 30


def _plan(n_states, n_rows, terms, elt=C128, l2=H100_L2, free=80 * GB, mode=-1, chunks=0):
    out = np.zeros(5, dtype=np.int64)
    ms = np.zeros(2)
    nat.check(nat.lib().dmv_debug_rows_store_plan(n_states, n_rows, terms, elt, l2, free, mode, chunks,
                                                  out.ctypes.data, ms.ctypes.data))
    return dict(use=bool(out[0]), chunks=int(out[1]), per_pass=int(out[2]), block=int(out[3]), bytes=int(out[4]),
                ms_store=float(ms[0]), ms_rows=float(ms[1]))


def _dictionary(lut, s_out=False, generic=False):
    lut = np.ascontiguousarray(lut, dtype=np.float64)
    coef = np.zeros(16)
    count = C.c_int(0)
    nat.check(nat.lib().dmv_debug_rows_store_coefficients(lut.ctypes.data, lut.shape[0], int(s_out), int(generic),
                                                          coef.ctypes.data, C.byref(count)))
    return coef[:max(count.value, 0)], count.value


# ---- CPU: the choice from sizes alone, and the coefficient dictionary

def test_plan_threshold_and_modes():
    """Auto needs 2^20 rows; mode 0 never builds; mode 1 builds whatever the size; forced chunks are taken as given
    (capped by the states) with one block per pass."""
    n = 1 << 20
    assert _plan(n, n, 36 * n)["use"]
    assert not _plan(n - 1, n - 1, 36 * (n - 1))["use"]
    assert not _plan(n, n, 36 * n, mode=0)["use"]
    small = _plan(1000, 1000, 36000, mode=1)
    assert small["use"] and small["chunks"] >= 1
    forced = _plan(1000, 1000, 36000, mode=1, chunks=3)
    assert forced["use"] and forced["chunks"] == 3 and forced["per_pass"] == 1 and forced["block"] == 334
    assert _plan(5, 5, 100, mode=1, chunks=64)["chunks"] == 5


def test_plan_blocks_follow_x_and_l2():
    """The column blocks depend on the sizes only: the same for both element types (float64 reads two per pass), fewer
    of them with a larger L2, one when x fits in L2."""
    n = 15804956
    c128, f64 = _plan(n, n, 585262534), _plan(n, n, 585262534, elt=F64)
    assert c128["use"] and f64["use"]
    assert c128["chunks"] == f64["chunks"] > 1 and c128["per_pass"] == 1 and f64["per_pass"] == 2
    assert c128["block"] * c128["chunks"] >= n and c128["block"] * (c128["chunks"] - 1) < n
    assert _plan(n, n, 585262534, l2=4 * H100_L2)["chunks"] < c128["chunks"]
    assert _plan(1 << 19, 1 << 19, 36 << 19, mode=1)["chunks"] == 1   # 8 MB of x
    assert c128["ms_store"] < c128["ms_rows"]


def test_plan_memory_rule_and_packing():
    """At most a quarter of the free memory, counted in full (entries, counts, offsets, diagonal, compact x and partial
    sums); a column block of more than 2^28 states does not fit the packing."""
    n = 15804956
    need = _plan(n, n, 585262534)["bytes"]
    assert need >= 585262534 * 4 + n * 16 * 2
    assert _plan(n, n, 585262534, free=4 * need)["use"]
    assert not _plan(n, n, 585262534, free=4 * need - 4)["use"]
    big = (1 << 28) + 1
    assert not _plan(big, 1 << 20, 36 << 20, mode=1, chunks=1)["use"]
    assert _plan(big, 1 << 20, 36 << 20, mode=1, chunks=2)["use"]


def test_coefficient_dictionary():
    """Distinct values in order of first appearance (bit patterns: -0.0 is its own code), their negatives with an outside
    sign mask, at most 16 codes; generic coefficients are refused."""
    coef, n = _dictionary([0.0, 2.0, 0.0, 2.0, 1.0])
    assert n == 3 and np.array_equal(coef, [0.0, 2.0, 1.0])
    coef, n = _dictionary([0.0, 2.0], s_out=True)
    assert n == 4 and list(coef[:2]) == [0.0, -0.0] and list(coef[2:]) == [2.0, -2.0]
    assert np.signbit(coef[1])
    assert _dictionary(np.arange(16.0))[1] == 16
    assert _dictionary(np.arange(17.0))[1] == -1
    assert _dictionary(np.arange(9.0), s_out=True)[1] == -1
    assert _dictionary([1.0], generic=True)[1] == -1


# ---- GPU

@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _store_matrix(op, sector):
    """k_rows and the store at C = 1, 2, 3 and 64 (capped by the basis) x float64 / complex128 on one context."""
    reps, ys = _oracle(*sector)
    op.basis.build()
    assert np.array_equal(op.basis.representatives(), reps)
    n = reps.shape[0]
    for cplx in (False, True):
        x, y_ref = ys[cplx]
        op.debug_rows_store(0)
        y_rows = _product(op, x)
        assert op.info("rows") == 1 and op.info("rows_store") == 0
        for chunks in (1, 2, 3, 64):
            op.debug_rows_store(1, chunks)
            y = _product(op, x)
            where = (sector, cplx, chunks)
            assert op.info("rows") == 1 and op.info("rows_store") == 1, where
            assert op.info("rows_store_chunks") == min(chunks, n), where
            assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
            assert np.array_equal(_product(op, x), y), where
            if chunks == 1:
                assert np.array_equal(y, y_rows), (where, np.abs(y - y_rows).max())
    op.debug_rows_store(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("sector", SECTORS, ids=_sector_id)
def test_store_on_torus_sectors(need_cuda, sector):
    basis, matrix = _model(*sector)
    op = Operator(matrix)
    try:
        if not basis.group.all_characters_trivial:   # no k_rows, no store
            reps, ys = _oracle(*sector)
            op.basis.build()
            op.debug_rows_store(1, 2)
            x, y_ref = ys[True]
            assert _close(_product(op, x), y_ref)
            assert op.info("rows") == 0 and op.info("rows_store") == 0
            return
        _store_matrix(op, sector)
    finally:
        op.close()


@pytest.mark.gpu
@pytest.mark.parametrize("base", GENERIC, ids=_generic_id)
def test_store_on_generic_walk(need_cuda, base):
    op = Operator(_model(*base)[1])
    try:
        _store_matrix(op, base)
    finally:
        op.close()


@pytest.mark.gpu
def test_fresh_context_is_bit_identical(need_cuda):
    """Two contexts with the same settings build the same store and give the same y."""
    sector = ("heisenberg_square_6x6", 7, None)
    x, _ = _oracle(*sector)[1][True]
    ys = []
    for _ in range(2):
        op = Operator(_model(*sector)[1])
        try:
            op.basis.build()
            op.debug_rows_store(1, 3)
            ys.append(_product(op, x))
            assert op.info("rows_store") == 1 and op.info("rows_store_builds") == 1
        finally:
            op.close()
    assert np.array_equal(ys[0], ys[1])


@pytest.mark.gpu
def test_store_survives_element_type_and_option_changes(need_cuda):
    """Switching between float64 and complex128 and changing the table options leave the store as it is (one build);
    a different column count rebuilds it.  Every product matches the oracle."""
    sector = ("heisenberg_square_6x6", 7, None)
    _, ys = _oracle(*sector)
    op = Operator(_model(*sector)[1])
    try:
        op.basis.build()
        op.debug_rows_store(1, 2)
        mb = None
        for options in (dict(), dict(rows_table=0), dict(rows_dense_order=0, rows_table_bits=8), dict(rows_index=1),
                        dict(canon=0), dict(rows_l2=0)):
            _set(op, **options)
            for cplx in (False, True, False):
                x, y_ref = ys[cplx]
                assert _close(_product(op, x), y_ref), (options, cplx)
                assert op.info("rows_store") == 1 and op.info("rows_store_builds") == 1, (options, cplx)
                mb = op.info("rows_store_mb") if mb is None else mb
                assert op.info("rows_store_mb") == mb
        op.debug_rows_store(1, 3)
        x, y_ref = ys[True]
        assert _close(_product(op, x), y_ref)
        assert op.info("rows_store_builds") == 2 and op.info("rows_store_chunks") == 3
    finally:
        op.close()


@pytest.mark.gpu
def test_store_rebuilt_with_the_basis(need_cuda):
    """Installing the representatives again releases the store; the next product builds a new one and matches."""
    sector = ("heisenberg_square_6x6", 6, None)
    basis, matrix = _model(*sector)
    reps, norms = po.enumerate_states(basis)
    _, ys = _oracle(*sector)
    op = Operator(matrix)
    try:
        op.basis.build()
        op.debug_rows_store(1, 2)
        x, y_ref = ys[True]
        assert _close(_product(op, x), y_ref) and op.info("rows_store_builds") == 1
        op.basis.uncheckedSetRepresentatives(reps, norms)
        assert op.info("rows_store_chunks") == 0
        assert _close(_product(op, x), y_ref) and op.info("rows_store_builds") == 2
    finally:
        op.close()


@pytest.mark.gpu
def test_host_vectors_in_row_chunks_equal_the_device_product(need_cuda):
    """A product into host memory is cut into row chunks (each its own passes over the store); it equals the product on
    device vectors bit for bit, at C = 1 and C = 5."""
    sector = ("heisenberg_square_6x6", 9, None)   # 163 k states: above the chunked path's 2^16
    op = Operator(_model(*sector)[1])
    try:
        op.basis.build()
        n = op.basis.representatives().shape[0]
        assert n >= 1 << 16
        for chunks in (1, 5):
            op.debug_rows_store(1, chunks)
            for cplx in (False, True):
                x = _x(n, cplx, 17)
                y_dev = _product(op, x)
                y_host = op.matvec(x)
                assert op.info("rows_store") == 1
                assert np.array_equal(y_host, y_dev), (chunks, cplx)
    finally:
        op.close()


@pytest.mark.gpu
def test_replicated_x_on_the_store(need_cuda):
    """Three emulated ranks: the replicated-x product on the whole-basis twin's store (rows: the rank's block, x through
    the slot table) matches the oracle at C = 1 and C = 4, and at C = 1 equals the same cluster without the store."""
    P = 3
    sector = ("heisenberg_square_6x6", 7, None)
    basis, matrix = _model(*sector)
    reps, _ = _oracle(*sector)
    masks, _ = po.partition_by_hash(reps, P)
    cl = EmulatedCluster(matrix, P).build()
    try:
        for cplx in (False, True):
            x = _x(reps.shape[0], cplx, 23)
            y_ref = po.matvec_global(matrix, reps, x, P, num_tasks=po.num_threads())
            xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
            ys = {}
            for mode, chunks in ((0, 0), (1, 1), (1, 4)):
                for op in cl.ops:
                    op.debug_rows_store(mode, chunks)
                y = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)
                assert _close(y, y_ref), (cplx, mode, chunks, np.abs(y - y_ref).max())
                assert all(op.info("global.rows_store") == mode for op in cl.ops), (cplx, mode, chunks)
                ys[(mode, chunks)] = y
            assert np.array_equal(ys[(1, 1)], ys[(0, 0)]), cplx
    finally:
        cl.close()


@pytest.mark.gpu
def test_missing_target_is_an_error_on_every_product(need_cuda):
    """A target outside the basis with a non-zero coefficient refuses the store: k_rows runs and reports it through the
    status words (DMV:115-118), on every product."""
    sector = ("heisenberg_square_6x6", 5, None)
    basis, matrix = _model(*sector)
    reps, norms = po.enumerate_states(basis)
    keep = np.ones(reps.shape[0], dtype=bool)
    keep[reps.shape[0] // 2: reps.shape[0] // 2 + 7] = False
    op = Operator(matrix)
    try:
        op.basis.uncheckedSetRepresentatives(reps[keep], norms[keep])
        op.debug_rows_store(1, 2)
        x = np.ones(int(keep.sum()), dtype=np.complex128)
        for _ in range(2):
            with pytest.raises(Exception, match="invalid index"):
                op.matvec(x)
            assert op.info("rows") == 1 and op.info("rows_store") == 0 and op.info("rows_store_chunks") == 0
    finally:
        op.close()


@pytest.mark.gpu
def test_auto_picks_the_store_on_the_6x6_square(need_cuda):
    """heisenberg_square_6x6 at size (15 804 956 states): auto builds the store, and the sampled rows of both element
    types match the oracle."""
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    _, matrix = load_config_from_yaml(os.path.join(DATA, "heisenberg_square_6x6.yaml"))
    op = Operator(matrix)
    try:
        op.basis.build()
        reps = op.basis.representatives()
        n = reps.shape[0]
        rows = np.sort(np.random.default_rng(9).choice(n, size=2048, replace=False))
        rows_d = torch.from_numpy(rows).cuda()
        for cplx in (True, False):
            x = _recipe_x(n, cplx)
            expect = po.expected_rows(matrix, reps, x, rows)
            y = op.matvec(torch.from_numpy(x).cuda())
            got = y[rows_d].cpu().numpy()
            del y
            assert op.info("rows") == 1 and op.info("rows_store") == 1 and op.info("rows_store_chunks") > 1
            assert _close(got, expect), (cplx, np.abs(got - expect).max())
        assert op.info("rows_store_builds") == 1
    finally:
        op.close()


@pytest.mark.gpu
def test_memory_rule_is_applied_before_the_build_only(need_cuda):
    """Once a store is built it stays in use while free memory drops below the rule, for device products and for the
    row chunks of a product into host memory (which follow their first chunk); a fresh context under the same pressure
    runs k_rows, and builds its store as soon as the memory is back."""
    sector = ("heisenberg_square_6x6", 9, None)   # 163 k states: above the chunked path's 2^16
    matrix = _model(*sector)[1]
    op, op2 = Operator(matrix), Operator(matrix)
    hog = None
    try:
        op.basis.build()
        op2.basis.build()
        n = op.basis.representatives().shape[0]
        x = _x(n, True, 31)
        op.debug_rows_store(0)
        y_rows = _product(op, x)
        op.debug_rows_store(1, 3)
        y_store = _product(op, x)
        assert op.info("rows_store") == 1 and op.info("rows_store_builds") == 1
        assert np.array_equal(op.matvec(x), y_store)
        need = op.info("rows_store_mb") << 20
        torch.cuda.synchronize()
        free, _ = torch.cuda.mem_get_info()
        hog = torch.empty(free - 2 * need, dtype=torch.uint8, device="cuda")   # free memory < 4 x the store
        for _ in range(2):
            assert np.array_equal(_product(op, x), y_store)
            assert np.array_equal(op.matvec(x), y_store)
            assert op.info("rows_store") == 1 and op.info("rows_store_builds") == 1
        op2.debug_rows_store(1, 3)
        for _ in range(2):
            assert np.array_equal(_product(op2, x), y_rows)
            assert np.array_equal(op2.matvec(x), y_rows)
            assert op2.info("rows") == 1 and op2.info("rows_store") == 0 and op2.info("rows_store_builds") == 0
        del hog
        hog = None
        torch.cuda.empty_cache()
        assert np.array_equal(_product(op2, x), y_store)
        assert np.array_equal(op2.matvec(x), y_store)
        assert op2.info("rows_store") == 1 and op2.info("rows_store_builds") == 1
    finally:
        del hog
        op.close()
        op2.close()


@pytest.mark.gpu
def test_operator_beyond_the_dictionary_runs_k_rows(need_cuda):
    """An XY ring whose couplings differ with the distance (1 .. 9 on 20 sites) has 18 distinct flip coefficients
    (Jx + Jy and Jx - Jy per distance), more than the 16 the store can code: with the store asked for, the product
    runs on k_rows and matches the oracle."""
    from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
    from test_symmetric_operators import _chain_group, _ring
    n = 20
    b = {"number_spins": n, "hamming_weight": None, "spin_inversion": 1, "symmetries": _chain_group(n)}
    terms = ([{"expression": f"{0.3 + 0.1 * d:.2f} × σˣ₀ σˣ₁", "sites": _ring(n, d)} for d in range(1, 10)] +
             [{"expression": f"{0.76 + 0.05 * d:.2f} × σʸ₀ σʸ₁", "sites": _ring(n, d)} for d in range(1, 10)])
    basis = basis_from_dict(b)
    matrix = operator_from_dict({"terms": terms}, basis)
    reps, _ = po.enumerate_states(basis)
    op = Operator(matrix)
    try:
        assert op.info("rows_ok") == 1
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        op.debug_rows_store(1, 2)
        for cplx in (False, True):
            x = _x(reps.shape[0], cplx, 5)
            y_ref = po.matvec_global(matrix, reps, x, 1, num_tasks=po.num_threads())
            y = _product(op, x)
            assert op.info("rows") == 1 and op.info("rows_store") == 0 and op.info("rows_store_builds") == 0
            assert _close(y, y_ref), (cplx, np.abs(y - y_ref).max())
    finally:
        op.close()
