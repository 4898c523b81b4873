"""k_rows with L2 eviction priorities on its ordered table: rows_l2 (0 none, 1 far buckets and the row's own data
evict_first, 2 and near buckets evict_last) and rows_l2_window (MB of table on either side of the row that count as near).

The priorities tell the L2 what to keep and must not change a single bit of y: neither option rebuilds the table, and a
lane still sums its row in program order.  Bases: the 6x6 torus at weight 7 (square-torus orbit minimum; its table is a
few MB, so the windows 0 / 4 / 32 MB make none, part and all of it near) and a chain with every symmetry (generic orbit
walk).  Criterion against the oracle: _close of test_gpu_parity.
"""
import numpy as np
import pytest

from distributed_matvec_b200 import EmulatedCluster, Operator, block_to_hashed, hashed_to_block
from oracle import pyoracle as po
from test_gpu_parity import _close
from test_rows_kernels import _model, _oracle, _product

torch = pytest.importorskip("torch")

BASES = {"torus_6x6_w7": ("heisenberg_square_6x6", 7, None), "chain_24_symm": ("heisenberg_chain_24_symm", None, None)}
MODES = (0, 1, 2)
WINDOWS = (0, 4, 32)
P = 3


@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(BASES))
def test_l2_priorities_do_not_change_the_product(need_cuda, name):
    """Every rows_l2 x rows_l2_window x element type: y matches the oracle and is bit-identical to rows_l2 = 0."""
    sector = BASES[name]
    reps, ys = _oracle(*sector)
    op = Operator(_model(*sector)[1])
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        for cplx in (False, True):
            x, y_ref = ys[cplx]
            first = None
            for mode in MODES:
                for window in WINDOWS:
                    op.set_option("rows_l2", mode)
                    op.set_option("rows_l2_window", window)
                    y = _product(op, x)
                    where = (name, cplx, mode, window)
                    assert op.info("rows") == 1 and op.info("rows_l2") == mode and op.info("rows_l2_window") == window, where
                    assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
                    if first is None:
                        first = y
                    assert np.array_equal(y, first), (where, np.abs(y - first).max())
    finally:
        op.close()


@pytest.mark.gpu
def test_l2_options_reject_out_of_range_values(need_cuda):
    """A rejected value raises with the option's name and changes neither the option nor the product."""
    sector = BASES["torus_6x6_w7"]
    x = _oracle(*sector)[1][True][0]
    op = Operator(_model(*sector)[1])
    try:
        op.basis.build()
        op.set_option("rows_l2", 2)
        op.set_option("rows_l2_window", 4)
        y_before = _product(op, x)
        for option, values in (("rows_l2", (-1, 3)), ("rows_l2_window", (-1, 33))):
            for value in values:
                with pytest.raises(Exception, match=option):
                    op.set_option(option, value)
        assert (op.info("rows_l2"), op.info("rows_l2_window")) == (2, 4)
        assert np.array_equal(_product(op, x), y_before)
    finally:
        op.close()


@pytest.mark.gpu
def test_l2_options_reach_the_twin(need_cuda):
    """Three logical ranks: the whole-basis twin of the replicated-x product, whose rows are a part of its table's
    basis, takes both options and computes the oracle's product with them."""
    sector = BASES["torus_6x6_w7"]
    basis, matrix = _model(*sector)
    reps, ys = _oracle(*sector)
    masks, _ = po.partition_by_hash(reps, P)
    x = ys[True][0]
    y_ref = po.matvec_global(matrix, reps, x, P, num_tasks=po.num_threads())
    cl = EmulatedCluster(matrix, P).build()
    try:
        for mode, window in ((2, 4), (1, 32), (0, 16)):
            for op in cl.ops:
                op.set_option("rows_l2", mode)
                op.set_option("rows_l2_window", window)
            xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
            y = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)
            assert _close(y, y_ref), (mode, window, np.abs(y - y_ref).max())
            for op in cl.ops:
                assert op.info("global.rows") == 1
                assert (op.info("global.rows_l2"), op.info("global.rows_l2_window")) == (mode, window)
    finally:
        cl.close()
