"""The dense ordered table of k_rows (option rows_dense_order = 1): one slot per state in key order, found through a
perfect hash per rank block (DenseOrder in dmv_device.cuh).

Host only: the placement the library builds is checked with its own builder and the device functions compiled for the
host -- every representative gets a distinct slot, the slots are 0 .. n - 1, a state's slot lies within its prefix
block's slot range up to the rank-block slack, and nearly every state is placed by the three hash levels.
On the GPU: products against the oracle for every directory size (one block, skewed blocks, empty blocks), both element
types and every L2 mode; bit-identity of y across rows_l2, windows and rows_ctas on one table build; the replicated-x
product of three emulated ranks; and a target outside the basis reported through the status words.
Criterion against the oracle: _close of test_gpu_parity.
"""

import numpy as np
import pytest

from distributed_matvec_b200 import EmulatedCluster, Operator, block_to_hashed, hashed_to_block
from distributed_matvec_b200 import _native as nat
from oracle import pyoracle as po
from test_gpu_parity import _close
from test_ordered_table import representatives
from test_rows_kernels import _model, _oracle, _product, _set, _sector_id

torch = pytest.importorskip("torch")

RANK_BLOCK_STATES = 40   # kDordStates
SLACK = 2 * RANK_BLOCK_STATES
BITS = (1, 8, 14)
DENSE = dict(rows_index=-1, rows_table=1, rows_dense_order=1)
# 6x6 sectors at several weights (weight 3: skewed and empty blocks at 14 bits), the 4x4 with spin inversion, and
# chains with every symmetry like chain_32_symm (generic orbit walk)
SECTORS = [("heisenberg_square_6x6", w, None) for w in (3, 5, 7, 31)] + [
    ("heisenberg_square_4x4", 8, 1), ("heisenberg_square_4x4", 6, None),
    ("heisenberg_chain_24_symm", None, None), ("heisenberg_kagome_12_symm", None, None)]


def dense_order(reps, bits):
    n = reps.shape[0]
    block = np.zeros(n, dtype=np.uint32)
    slot = np.zeros_like(block)
    probes = np.zeros_like(block)
    info = np.zeros(2, dtype=np.int64)
    nat.check(nat.lib().dmv_debug_dense_order(reps.ctypes.data, n, bits, block.ctypes.data, slot.ctypes.data,
                                              probes.ctypes.data, info.ctypes.data))
    return block, slot, probes, int(info[0]), int(info[1])


HOST_CASES = [("heisenberg_square_4x4",), ("heisenberg_chain_24_symm",), ("heisenberg_square_6x6", 5, None),
              ("heisenberg_square_6x6", 7, None)]


@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("case", HOST_CASES, ids=lambda c: "-".join(str(v) for v in c if v is not None))
def test_every_state_gets_its_own_slot_in_prefix_order(case, bits):
    if len(case) == 1:
        reps = representatives(case[0])
    else:
        reps = np.ascontiguousarray(po.enumerate_states(_model(*case)[0])[0], dtype=np.uint64)
    n = reps.shape[0]
    block, slot, probes, placed, rank_blocks = dense_order(reps, bits)
    # distinct slots 0 .. n - 1 (the entry also fails on a slot taken twice or a state not found)
    assert np.array_equal(np.sort(slot), np.arange(n, dtype=np.uint32))
    assert rank_blocks == (n + RANK_BLOCK_STATES - 1) // RANK_BLOCK_STATES
    # slot within the prefix block's range [dir[p], dir[p + 1]) up to the boundary slack: a rank block at either end
    # also holds the neighbours' keys that hash into it, about one rank block of them (at most 49 on these bases)
    assert np.all(np.diff(block.astype(np.int64)) >= 0)
    lo = np.searchsorted(block, block, side="left").astype(np.int64)
    hi = np.searchsorted(block, block, side="right").astype(np.int64)
    s = slot.astype(np.int64)
    assert np.all(s >= lo - SLACK) and np.all(s < hi + SLACK), ((lo - s).max(), (s - hi + 1).max())
    # the three levels place nearly every state (0.5 % are left over on the larger bases; the few rank blocks of the
    # 4x4 give a noisier share); the leftovers cost a short scan
    large = n > 10000
    assert placed >= (0.98 if large else 0.9) * n, placed / n
    assert probes.min() >= 1 and probes.mean() < (1.02 if large else 1.1), probes.mean()
    assert probes.max() <= 2 * RANK_BLOCK_STATES


def test_dense_order_rejects_unsorted_representatives():
    reps = np.array([5, 3, 9], dtype=np.uint64)
    assert nat.lib().dmv_debug_dense_order(reps.ctypes.data, 3, 8, None, None, None, None) != 0


@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


@pytest.mark.gpu
@pytest.mark.parametrize("sector", SECTORS, ids=_sector_id)
def test_dense_order_products(need_cuda, sector):
    """rows_table_bits 1 / 8 / 14 x float64 / complex128 x rows_l2 0 / 1 / 2 (windows 0, 1 and 32 MB) against the oracle;
    on one table build y is bit-identical across every L2 mode, window and rows_ctas."""
    basis, matrix = _model(*sector)
    reps, ys = _oracle(*sector)
    op = Operator(matrix)
    try:
        op.basis.build()
        assert np.array_equal(op.basis.representatives(), reps)
        for bits in BITS:
            _set(op, rows_table_bits=bits, **DENSE)
            for cplx in (False, True):
                x, y_ref = ys[cplx]
                first = None
                for mode, window, ctas in ((0, 0, 2), (1, 1, 2), (2, 0, 2), (2, 1, 2), (2, 32, 2), (2, 16, 3)):
                    _set(op, rows_l2=mode, rows_l2_window=window, rows_ctas=ctas)
                    y = _product(op, x)
                    where = (_sector_id(sector), bits, cplx, mode, window, ctas)
                    assert op.info("rows") == 1 and op.info("rows_dense_order_on") == 1, where
                    assert 0 < op.info("rows_dense_order_placed") <= reps.shape[0], where
                    assert op.info("rows_dense") == 0, where   # (that key counts the perfect-hash index only)
                    assert _close(y, y_ref), (where, np.abs(y - y_ref).max())
                    if first is None:
                        first = y
                    assert np.array_equal(y, first), (where, np.abs(y - first).max())
        # switched off: the ordered layout with linear probing (which auto replaces) at 8 and 2 buckets per state
        for buckets in (8, 2):
            _set(op, rows_dense_order=0, rows_l2=2, rows_l2_window=16, rows_ctas=2, rows_table_bits=14,
                 rows_table_buckets=buckets)
            for cplx in (False, True):
                x, y_ref = ys[cplx]
                assert _close(_product(op, x), y_ref), (buckets, cplx)
                assert op.info("rows") == 1 and op.info("rows_dense_order_on") == 0
                assert op.info("rows_dense_order_placed") == 0
    finally:
        op.close()


@pytest.mark.gpu
def test_dense_order_replicated_x_three_ranks(need_cuda):
    """Three emulated ranks: the whole-basis twin of the replicated-x product takes the option, builds the dense ordered
    table and computes the oracle's product, at 14 and 1 directory bits."""
    P = 3
    sector = ("heisenberg_square_6x6", 7, None)
    basis, matrix = _model(*sector)
    reps, ys = _oracle(*sector)
    masks, _ = po.partition_by_hash(reps, P)
    cl = EmulatedCluster(matrix, P).build()
    try:
        for bits in (14, 1):
            for op in cl.ops:
                _set(op, rows_table_bits=bits, **DENSE)
            for cplx in (False, True):
                x = ys[cplx][0]
                y_ref = po.matvec_global(matrix, reps, x, P, num_tasks=po.num_threads())
                xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
                y = hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)
                assert _close(y, y_ref), (bits, cplx, np.abs(y - y_ref).max())
                for op in cl.ops:
                    assert op.info("global.rows") == 1 and op.info("global.rows_dense_order") == 1
                    assert op.info("rows_dense_order_on") == 1 and op.info("rows_dense_order_placed") > 0
    finally:
        cl.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bits", (1, 14))
def test_dense_order_missing_state_is_an_error(need_cuda, bits):
    """A target outside the basis with a non-zero coefficient (states dropped from the middle of the sector) is
    reported through the status words (DMV:115-118), as with the other tables."""
    sector = ("heisenberg_square_6x6", 5, None)
    basis, matrix = _model(*sector)
    reps, norms = po.enumerate_states(basis)
    keep = np.ones(reps.shape[0], dtype=bool)
    keep[reps.shape[0] // 2: reps.shape[0] // 2 + 7] = False
    for cplx in (False, True):
        op = Operator(matrix)
        try:
            op.basis.uncheckedSetRepresentatives(reps[keep], norms[keep])
            _set(op, rows_table_bits=bits, **DENSE)
            x = np.ones(int(keep.sum()), dtype=np.complex128 if cplx else np.float64)
            with pytest.raises(Exception, match="invalid index"):
                op.matvec(x)   # host vectors: the call synchronises and reads the status words
            assert op.info("rows") == 1 and op.info("rows_dense_order_on") == 1
        finally:
            op.close()


@pytest.mark.gpu
def test_dense_order_option_values(need_cuda):
    """rows_dense_order takes -1, 0 and 1; any other value raises and changes nothing."""
    sector = ("heisenberg_square_6x6", 5, None)
    op = Operator(_model(*sector)[1])
    try:
        op.basis.build()
        op.set_option("rows_dense_order", 0)
        for value in (-2, 2):
            with pytest.raises(Exception, match="rows_dense_order"):
                op.set_option("rows_dense_order", value)
        assert op.info("rows_dense_order") == 0
        x, y_ref = _oracle(*sector)[1][True]
        assert _close(_product(op, x), y_ref)
        assert op.info("rows_dense_order_on") == 0 and op.info("rows_dense_order_placed") == 0
        # the perfect-hash index takes precedence over the dense ordered table; rows_dense counts what it places
        _set(op, rows_index=1, rows_dense_order=1)
        assert _close(_product(op, x), y_ref)
        assert op.info("rows_dense_order_on") == 0 and 0 < op.info("rows_dense") <= x.shape[0]
        _set(op, rows_index=-1)
        assert _close(_product(op, x), y_ref)
        assert op.info("rows_dense_order_on") == 1 and op.info("rows_dense") == 0
        assert 0 < op.info("rows_dense_order_placed") <= x.shape[0]
    finally:
        op.close()
