"""dmv_set_option: the accepted values of every option, and the options on the whole-basis twin of the replicated-x form.

A value outside an option's accepted set raises with the option's name in the message and changes nothing.  Every option
set on a rank also applies to its twin (the single-rank context over the whole basis that computes the rows of the
replicated-x product), whether the twin exists yet or not; info("global.<key>") answers <key> for the twin.
"""
import os

import numpy as np
import pytest

from distributed_matvec_b200 import EmulatedCluster, Operator, block_to_hashed, hashed_to_block, load_config_from_yaml
from oracle import pyoracle as po
from test_gpu_parity import _close, _x
from test_rows_kernels import _model as _torus_model

torch = pytest.importorskip("torch")

DATA = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "data")
INDEX_DIRECTORY = 0
P = 3

# every option: values it rejects (just outside its range, and between or beside the members of its set)
REJECTED = {
    "mode": (-2, 2), "index": (-2, 1, 4), "exchange": (-2, 3), "gather": (-2, 1), "rows_batch_min": (1, 7),
    "rows_batch": (-2, 2), "rows_ctas": (0, 1, 5), "rows_index": (-2, 2), "rows_table": (-1, 2),
    "rows_table_bits": (0, 15), "rows_table_buckets": (1, 3, 16), "rows_dense_order": (-2, 2), "rows_l2": (-1, 3),
    "rows_l2_window": (-1, 33), "rounds": (-2, 65), "gather_walk": (-1, 3),
    "gather_split": (-2, 0, 3, 64), "peer_gather": (-2, 1), "rows": (-2, 1), "canon": (-2, 3), "bitparallel": (-1, 2),
    "push_split": (-2, 0, 3, 64),
}

# the twin's models: k_rows (6x6 square, weight 7) and k_gather (chain of 16 sites).  Per model, each option with a
# value other than its default, and what the twin's info shows for it.  The layout of k_rows' table shows in no info
# key: for rows_table = 0 the product is the check.
TWIN_CASES = {
    "torus_6x6_w7": [("canon", 0, {"canon_mode": 0, "rows_tk": 0}), ("bitparallel", 0, {"rows": 0}),
                     ("rows", 0, {"rows": 0}), ("rows_table", 0, {"rows": 1})],
    "chain_16": [("gather", 0, {"gather": 0}), ("index", 0, {"index_mode": INDEX_DIRECTORY}),
                 ("gather_split", 4, {"gather_split": 4}), ("push_split", 2, {"push_split": 2})],
}
DEFAULTS = {"canon": -1, "bitparallel": 1, "rows": -1, "rows_table": 1, "gather": -1, "index": -1, "gather_split": -1,
            "push_split": -1}


def _matrix(name):
    if name == "torus_6x6_w7":
        return _torus_model("heisenberg_square_6x6", 7, None)
    return load_config_from_yaml(os.path.join(DATA, "heisenberg_" + name + ".yaml"))


@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _product(op, x):
    y = op.matvec(torch.from_numpy(x).cuda())
    torch.cuda.synchronize()
    return y.cpu().numpy()


@pytest.mark.gpu
def test_every_option_rejects_out_of_range_values(need_cuda):
    """Each rejected value raises with the option's name; an unknown name raises too.  Afterwards the k_gather product
    (no atomics) is bit-identical to the one before, and the selection the operator reports is unchanged."""
    basis, matrix = _matrix("chain_16")
    op = Operator(matrix)
    try:
        op.basis.build()
        x = _x(op.basis.representatives().shape[0], True)
        keys = ("gather", "rows", "pull", "index_mode", "gather_split", "push_split", "rows_tk", "canon_mode")
        before = {k: op.info(k) for k in keys}
        y_before = _product(op, x)
        for name, values in REJECTED.items():
            for value in values:
                with pytest.raises(Exception, match=name):
                    op.set_option(name, value)
        with pytest.raises(Exception, match="no_such_option"):
            op.set_option("no_such_option", 0)
        assert {k: op.info(k) for k in keys} == before
        assert np.array_equal(_product(op, x), y_before)
    finally:
        op.close()


def _replicated(cl, x, masks):
    xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
    return hashed_to_block([t.cpu().numpy() for t in cl.matvec_replicated(xb)], masks)


def _twin_info(cl, keys):
    """info("global.<key>") of rank 0; every rank's twin must agree."""
    got = [{k: op.info("global." + k) for k in keys} for op in cl.ops]
    assert all(g == got[0] for g in got), got
    return got[0]


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(TWIN_CASES))
def test_options_reach_the_twin(need_cuda, name):
    """Three logical ranks: each option, set on every rank after the twins exist, shows in the twins' info and the
    replicated-x product still matches the oracle's 3-rank product; reset, the twins' info is back to the default.  An
    option set before the twins exist is inherited by them."""
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    basis, matrix = _matrix(name)
    reps, _ = po.enumerate_states(basis)
    masks, _ = po.partition_by_hash(reps, P)
    xs = [_x(reps.shape[0], cplx, 51) for cplx in (False, True)]
    refs = [po.matvec_global(matrix, reps, x, P, num_tasks=po.num_threads()) for x in xs]

    def check(where):
        for x, y_ref in zip(xs, refs):
            y = _replicated(cl, x, masks)
            assert _close(y, y_ref), (where, x.dtype, np.abs(y - y_ref).max())

    cases = TWIN_CASES[name]
    keys = sorted({k for _, _, shown in cases for k in shown})
    cl = EmulatedCluster(matrix, P).build()
    try:
        assert all(op.info("global.canon_mode") == -1 for op in cl.ops)   # no twin yet
        check("default")
        default = _twin_info(cl, keys)
        for option, value, shown in cases:
            assert any(default[k] != v for k, v in shown.items()) or option == "rows_table", (option, default)
            for op in cl.ops:
                op.set_option(option, value)
            assert {k: v for k, v in _twin_info(cl, keys).items() if k in shown} == shown, option
            check((option, value))
            for op in cl.ops:
                op.set_option(option, DEFAULTS[option])
            check((option, "reset"))
            assert _twin_info(cl, keys) == default, option
    finally:
        cl.close()

    option, value, shown = cases[1]   # set before the twins exist: "bitparallel" / "index" (read in the basis build)
    cl = EmulatedCluster(matrix, P).build()
    try:
        for op in cl.ops:
            op.set_option(option, value)
        check((option, value, "before the twin"))
        assert {k: v for k, v in _twin_info(cl, keys).items() if k in shown} == shown, option
    finally:
        cl.close()
