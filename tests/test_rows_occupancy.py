"""CTAs per SM of k_rows (option rows_ctas): -1 auto (the default), 2, 3 or 4.

Auto runs three CTAs per SM with the square-torus forms of the orbit minimum (TK = 4 / 6), whose three-CTA builds spill no
more than their two-CTA ones, and two with the generic orbit walk.  info("rows_ctas_resident") is the number of CTAs per
SM the last k_rows launch had resident, from the occupancy query of the launch.

On one table build y is bit-identical whatever the CTA count: rows_ctas does not rebuild the table, and a lane sums its
row in program order.  Criterion against the oracle: _close of test_gpu_parity.
"""
import numpy as np
import pytest

from distributed_matvec_b200 import EmulatedCluster, Operator, block_to_hashed, hashed_to_block
from oracle import pyoracle as po
from test_gpu_parity import _close
from test_rows_kernels import _model, _oracle, _product, _sector_id

torch = pytest.importorskip("torch")

# (sector, TK of its orbit minimum, CTAs per SM that auto runs)
CASES = [(("heisenberg_square_6x6", 7, None), 6, 3), (("heisenberg_square_4x4", 8, 1), 4, 3),
         (("heisenberg_chain_24_symm", None, None), 0, 2)]


@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: _sector_id(c[0]))
def test_rows_ctas_auto_and_explicit(need_cuda, case):
    """rows_ctas 2, 3 and auto on the default table (the dense ordered one) x float64 / complex128: each product matches
    the oracle, the three are bit-identical, and each launch had the CTAs per SM asked for (auto: three with a torus
    form, two with the generic walk)."""
    sector, tk, auto = case
    basis, matrix = _model(*sector)
    reps, ys = _oracle(*sector)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        assert op.info("rows_ctas_resident") == 0   # no k_rows launch yet
        for cplx in (False, True):
            x, y_ref = ys[cplx]
            first = None
            for ctas, resident in ((2, 2), (3, 3), (-1, auto)):
                op.set_option("rows_ctas", ctas)
                y = _product(op, x)
                where = (_sector_id(sector), cplx, ctas)
                assert op.info("rows") == 1 and op.info("rows_dense_order_on") == 1, where
                assert op.info("rows_tk") == tk, where
                assert op.info("rows_ctas_resident") == resident, (where, op.info("rows_ctas_resident"))
                assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
                if first is None:
                    first = y
                assert np.array_equal(y, first), (where, np.abs(y - first).max())
    finally:
        op.close()


@pytest.mark.gpu
def test_rows_ctas_values(need_cuda):
    """rows_ctas takes -1, 2, 3 and 4; any other value raises and leaves the setting as it was.  The perfect-hash index
    runs two CTAs per SM whatever the option."""
    sector = ("heisenberg_square_6x6", 5, None)
    op = Operator(_model(*sector)[1])
    try:
        op.basis.build()
        x, y_ref = _oracle(*sector)[1][True]
        op.set_option("rows_ctas", 4)
        op.set_option("rows_ctas", -1)
        for value in (-2, 0, 1, 5):
            with pytest.raises(Exception, match="rows_ctas"):
                op.set_option("rows_ctas", value)
        assert _close(_product(op, x), y_ref)
        assert op.info("rows_ctas_resident") == 3   # still auto
        op.set_option("rows_index", 1)
        assert _close(_product(op, x), y_ref)
        assert op.info("rows_dense") > 0 and op.info("rows_ctas_resident") == 2
    finally:
        op.close()


@pytest.mark.gpu
def test_rows_ctas_replicated_x_three_ranks(need_cuda):
    """Three emulated ranks under auto: the whole-basis twin of the replicated-x product runs k_rows at three CTAs per SM
    on the 6x6 torus form and computes the oracle's product."""
    P = 3
    sector = ("heisenberg_square_6x6", 7, None)
    basis, matrix = _model(*sector)
    reps, ys = _oracle(*sector)
    masks, _ = po.partition_by_hash(reps, P)
    cl = EmulatedCluster(matrix, P).build()
    try:
        for cplx in (False, True):
            x = ys[cplx][0]
            y_ref = po.matvec_global(matrix, reps, x, P, num_tasks=po.num_threads())
            xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
            y = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)
            assert _close(y, y_ref), (cplx, np.abs(y - y_ref).max())
            for op in cl.ops:
                assert op.info("global.rows") == 1 and op.info("rows_ctas_resident") == 3
    finally:
        cl.close()
