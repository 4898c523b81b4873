"""Products on long-lived contexts: every option changed between products, element-type, batch and host/device switches,
observables and solvers between products, bases re-installed with dmv_set_representatives, and streams.

A context caches the k_rows tables, the k_rows_batch table, the record plan, the exchange choice, the replicated-x twin,
the orbit program, the index mode and the solvers' work space.  Each cache is refreshed either from the `stale` column
of the option table (dmv_set_option) or by install_directory (after dmv_basis_build and dmv_set_representatives).  A
stale cache gives a wrong y without an error, or a right y from a kernel or table the options no longer ask for; so
every product here is checked three ways: against the oracle (_close), bit for bit against a fresh context with the
same options and the same block where the kernel uses no floating-point atomics and its table is laid out the same
in every build (k_gather, k_pull, k_rows_batch, k_rows on its dense ordered table, and the solvers on them), and
through the info keys that show which kernel and table ran.
"""
import functools
import os
import re

import numpy as np
import pytest
import yaml

from distributed_matvec_b200 import EmulatedCluster, Operator, block_to_hashed, hashed_to_block
from distributed_matvec_b200 import _native as nat
from distributed_matvec_b200.config import basis_from_dict, operator_from_dict
from oracle import pyoracle as po
from test_gpu_parity import GENERAL_MODELS, _close, _x
from test_options import REJECTED
from test_rows_kernels import TABLES, _model as _torus, _product, _set
from test_symmetric_operators import _chain_group

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DATA = os.path.join(ROOT, "data")
INDEX_DIRECTORY = 0


# ---- models

def _yaml(name):
    with open(os.path.join(DATA, name + ".yaml"), encoding="utf-8") as f:
        return yaml.safe_load(f)


@functools.lru_cache(maxsize=None)
def _chain_16(weight=8):
    """the 16-site Heisenberg ring without symmetries (k_gather); weight None: free magnetisation"""
    conf = _yaml("heisenberg_chain_16")
    basis = basis_from_dict({**conf["basis"], "hamming_weight": weight})
    return basis, operator_from_dict(conf["hamiltonian"], basis)


@functools.lru_cache(maxsize=None)
def _ring_20(weight=None):
    """the 20-site Heisenberg ring with its translations and reflection (trivial characters, no spin flip: k_rows);
    weight None: free magnetisation.  H conserves the magnetisation, so every weight-w block of the free basis is closed
    under H and its product is the oracle's product on the fixed-weight sector."""
    conf = _yaml("heisenberg_chain_20")
    basis = basis_from_dict({"number_spins": 20, "hamming_weight": weight, "symmetries": _chain_group(20)})
    return basis, operator_from_dict(conf["hamiltonian"], basis)


MODELS = {
    "torus_6x6_w7": lambda: _torus("heisenberg_square_6x6", 7, None),    # k_rows, square-torus orbit minimum
    "chain_16": lambda: _chain_16(8),                                      # k_gather
    "momentum_10": GENERAL_MODELS["momentum_sector"],                      # complex characters: k_pull (mode 1)
    "torus_4x4_inv": lambda: _torus("heisenberg_square_4x4", 8, 1),       # k_rows, group with spin inversion
    "chain_20": lambda: _yaml_model("heisenberg_chain_20"),                # k_gather past 2^16 states: chunked D2H
}
# options every context of a model starts from: auto takes the scatter form for complex characters
BASE = {"momentum_10": {"mode": 1}}
DEFAULTS = {"mode": -1, "index": -1, "exchange": -1, "gather": -1, "rows_batch_min": 2, "rows_batch": -1, "rows_ctas": -1,
            "rows_index": -1, "rows_table": 1, "rows_table_bits": 12, "rows_table_buckets": 8, "rows_dense_order": -1,
            "rows_l2": 2, "rows_l2_window": 2, "rounds": -1, "gather_walk": 0, "gather_split": -1, "push_split": -1,
            "peer_gather": -1, "rows": -1, "canon": -1, "bitparallel": 1}


def _yaml_model(name):
    conf = _yaml(name)
    basis = basis_from_dict(conf["basis"])
    return basis, operator_from_dict(conf["hamiltonian"], basis)


# Every option of dmv_set_option, changed on a live context: (model, value, the info keys that must show it).  A model
# of the table is named once per kernel family whose caches the option touches.
OPTION_CASES = {
    "mode": [("torus_6x6_w7", 0, {"pull": 0, "rows": 0}), ("momentum_10", 0, {"pull": 0})],
    "index": [("chain_16", 2, {"index_mode": 2}), ("chain_16", 0, {"index_mode": INDEX_DIRECTORY})],
    "exchange": [("chain_16", 0, {"gather": 1})],
    "gather": [("chain_16", 0, {"gather": 0, "pull": 0})],
    "rows_batch_min": [("torus_6x6_w7", 6, {"rows": 1})],
    "rows_batch": [("torus_6x6_w7", 0, {"rows": 1}), ("torus_4x4_inv", 0, {"rows": 1})],
    "rows_ctas": [("torus_6x6_w7", 3, {"rows_tk": 6}), ("torus_4x4_inv", 4, {"rows_tk": 0})],
    "rows_index": [("torus_6x6_w7", 1, {"rows_dense_order_on": 0, "rows": 1}),
                   ("torus_4x4_inv", 1, {"rows_dense_order_on": 0, "rows_tk": 4})],
    "rows_table": [("torus_6x6_w7", 0, {"rows_dense_order_on": 0, "rows": 1})],
    "rows_table_bits": [("torus_6x6_w7", 1, {"rows_dense_order_on": 1})],
    "rows_table_buckets": [("torus_6x6_w7", 2, {"rows_dense_order_on": 1})],
    "rows_dense_order": [("torus_6x6_w7", 0, {"rows_dense_order": 0, "rows_dense_order_on": 0}),
                         ("torus_4x4_inv", 0, {"rows_dense_order": 0, "rows_dense_order_on": 0})],
    "rows_l2": [("torus_6x6_w7", 0, {"rows_l2": 0})],
    "rows_l2_window": [("torus_6x6_w7", 16, {"rows_l2_window": 16})],
    "rounds": [("chain_16", 3, {"rounds": 0})],
    "gather_walk": [("chain_16", 1, {"gather": 1})],
    "gather_split": [("chain_16", 4, {"gather_split": 4})],
    "push_split": [("chain_16", 2, {"push_split": 2}), ("momentum_10", 4, {"push_split": 4})],
    "peer_gather": [("chain_16", 0, {"gather": 1})],
    "rows": [("torus_6x6_w7", 0, {"rows": 0, "pull": 0}), ("torus_4x4_inv", 0, {"rows": 0, "pull": 0})],
    "canon": [("torus_6x6_w7", 0, {"canon_mode": 0, "rows_tk": 0}), ("momentum_10", 0, {"canon_mode": 0}),
              ("torus_4x4_inv", 0, {"canon_mode": 0, "rows_tk": 0})],
    "bitparallel": [("torus_6x6_w7", 0, {"rows": 0}), ("chain_16", 0, {"gather": 0})],
}
# the values the random walk draws from (all accepted)
ACCEPTED = {"mode": (-1, 0, 1), "index": (-1, 0, 2, 3), "exchange": (-1, 0, 1, 2), "gather": (-1, 0),
            "rows_batch_min": (2, 3, 4, 5, 6), "rows_batch": (-1, 0, 1), "rows_ctas": (-1, 2, 3, 4),
            "rows_index": (-1, 0, 1), "rows_table": (0, 1), "rows_table_bits": (1, 8, 12, 14),
            "rows_table_buckets": (2, 4, 8), "rows_dense_order": (-1, 0, 1), "rows_l2": (0, 1, 2),
            "rows_l2_window": (0, 2, 16, 32), "rounds": (-1, 0, 3, 64), "gather_walk": (0, 1, 2),
            "gather_split": (-1, 1, 2, 4, 8, 16, 32), "push_split": (-1, 1, 2, 4, 8, 16, 32), "peer_gather": (-1, 0),
            "rows": (-1, 0), "canon": (-1, 0, 1, 2), "bitparallel": (0, 1)}
# what a live context and a fresh one with the same options must agree on
INFO_KEYS = ("pull", "gather", "rows", "index_mode", "gather_split", "push_split", "rows_tk", "canon_mode", "rows_l2",
             "rows_l2_window", "rows_dense_order", "rows_dense_order_on", "rows_dense_order_placed", "rows_dense")


def _option_names_in_library():
    with open(os.path.join(ROOT, "distributed_matvec_b200", "csrc", "dmv_api.cu"), encoding="utf-8") as f:
        src = f.read()
    table = src[src.index("const OptionRow kOptionTable[]"):]
    table = table[:table.index("};")]
    return re.findall(r'\{"(\w+)", &Options::', table)


def test_option_cases_cover_every_option():
    """OPTION_CASES, ACCEPTED and DEFAULTS name exactly the options test_options rejects values of, and those are the
    rows of the library's option table: an option added to the library without a case here fails."""
    names = _option_names_in_library()
    assert len(names) == len(set(names)) and names
    assert set(OPTION_CASES) == set(REJECTED) == set(ACCEPTED) == set(DEFAULTS) == set(names)
    for option, cases in OPTION_CASES.items():
        for model, value, shown in cases:
            assert model in MODELS and value in ACCEPTED[option] and value != BASE.get(model, {}).get(option,
                                                                                                      DEFAULTS[option])
            assert set(shown) <= set(INFO_KEYS) | {"rounds"}, (option, shown)
    for option, values in ACCEPTED.items():
        assert DEFAULTS[option] in values and not set(values) & set(REJECTED[option]), option


# ---- the oracle's side

@functools.lru_cache(maxsize=None)
def _reference(name):
    """representatives, x and y = H x of both element types, and six columns of each for batches"""
    po.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    basis, matrix = MODELS[name]()
    reps, _ = po.enumerate_states(basis)
    n = reps.shape[0]
    out = {"reps": reps}
    for cplx in (False, True):
        X = np.stack([_x(n, cplx, 700 + j) for j in range(6)])
        out[cplx] = (X, np.stack([po.matvec_global(matrix, reps, X[j], 1, num_tasks=po.num_threads())
                                  for j in range(6)]))
    return out


@functools.lru_cache(maxsize=None)
def _sector(weight, symmetric=True):
    """the oracle's fixed-weight sector of the 20-site ring (or of the 16-site ring without symmetries)"""
    basis, _ = (_ring_20 if symmetric else _chain_16)(weight)
    return po.enumerate_states(basis)


@pytest.mark.parametrize("symmetric", [True, False])
def test_free_basis_by_weight_is_the_fixed_weight_sector(symmetric):
    """The reference the weight-sector blocks are checked against: the oracle's free-magnetisation basis filtered by
    popcount is, weight by weight, its fixed-weight enumeration, norms included."""
    basis, _ = (_ring_20 if symmetric else _chain_16)(None)
    reps, norms = po.enumerate_states(basis)
    weights = np.array([bin(int(s)).count("1") for s in reps])
    sites = basis.number_sites
    assert sorted(set(weights)) == list(range(sites + 1))
    for w in range(sites + 1):
        want, want_norms = _sector(w, symmetric)
        assert np.array_equal(reps[weights == w], want), w
        assert np.array_equal(norms[weights == w], want_norms), w


# ---- GPU helpers

@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


def _context(name, options=(), block=None, norms=None):
    basis, matrix = MODELS[name]() if isinstance(name, str) else name
    op = Operator(matrix)
    _set(op, **dict(BASE.get(name, {}) if isinstance(name, str) else {}, **dict(options)))
    if block is None:
        op.basis.build()
    else:
        op.basis.uncheckedSetRepresentatives(block, norms)
    return op


def _batch(op, X):
    Y = op.matvec_batch(torch.from_numpy(X).cuda())
    torch.cuda.synchronize()
    return Y.cpu().numpy()


def _fill(op, model, options):
    """One of each product on op: single float64, single complex128, a batch of six complex128 columns (two k_rows_batch
    launches of three, or k_gather's four-wide batch and two single products), a complex128 product in the scatter form (mode 0, then back to `options`') and a
    last float64 one.  The next fill starts with float64 too, so that it finds k_rows' table built for its element type
    and rebuilds it only if the option in between made it stale.
    -> (products, info after the first product)"""
    ref = _reference(model)
    out = {"f64": _product(op, ref[False][0][0])}
    info = {k: op.info(k) for k in INFO_KEYS}
    out["c128"] = _product(op, ref[True][0][0])
    out["batch"] = _batch(op, ref[True][0][:6])
    op.set_option("mode", 0)
    out["push"] = _product(op, ref[True][0][1])
    op.set_option("mode", options.get("mode", DEFAULTS["mode"]))
    out["f64 last"] = _product(op, ref[False][0][0])
    return out, info


def _reproducible(info, options):
    """which products of _fill a fresh context must reproduce bit for bit: every row kernel sums a row in its term
    order, except k_rows on an open-addressing table, which keeps two look-ups in flight and adds a retried miss after
    the newer term, so that the rounding follows the table's layout -- and that layout is not the same from build to
    build (concurrent inserts).  k_rows_batch keeps one look-up in flight, and the dense ordered table is laid out on
    the host in key order."""
    if info["pull"] != 1:
        return ()
    if info["rows"] == 1:
        singles = ("f64", "c128", "f64 last") if info["rows_dense_order_on"] == 1 else ()
        batch_by_rows = options.get("rows_batch", DEFAULTS["rows_batch"]) != 0
        return singles + (("batch",) if batch_by_rows or singles else ())
    return ("f64", "c128", "batch", "f64 last")


TABLE_KEYS = ("rows_dense_order_on", "rows_dense_order_placed", "rows_dense")   # the last k_rows table built


def _check_fill(name, options, got, fresh, where):
    (out, info), (f_out, f_info) = got, fresh
    ref = _reference(name)
    want = {"f64": ref[False][1][0], "c128": ref[True][1][0], "batch": ref[True][1][:6], "push": ref[True][1][1],
            "f64 last": ref[False][1][0]}
    for key, y in out.items():
        assert _close(y, want[key]), (where, key, np.abs(y - want[key]).max())
    for key in _reproducible(info, options):
        assert np.array_equal(out[key], f_out[key]), (where, key, "differs from a fresh context",
                                                      np.abs(out[key] - f_out[key]).max())
    keys = [k for k in INFO_KEYS if info["rows"] == 1 or k not in TABLE_KEYS]
    assert {k: info[k] for k in keys} == {k: f_info[k] for k in keys}, (where, "info differs from a fresh context",
                                                                        info, f_info)


_fresh_cache = {}


def _fresh(name, options):
    key = (name, tuple(sorted(options.items())))
    if key not in _fresh_cache:
        op = _context(name, options)
        try:
            _fresh_cache[key] = _fill(op, name, options)
        finally:
            op.close()
    return _fresh_cache[key]


OPTION_PARAMS = [(o, m, v, s) for o, cases in OPTION_CASES.items() for m, v, s in cases]


@pytest.mark.gpu
@pytest.mark.parametrize("option,model,value,shown", OPTION_PARAMS,
                         ids=[f"{o}-{m}-{v}" for o, m, v, _ in OPTION_PARAMS])
def test_option_on_live_context(need_cuda, option, model, value, shown):
    """Fill every cache (f64, c128, a batch, push once), set the option, run all of them again, reset it, run them once
    more: after each step the products match the oracle and, bit for bit, a fresh context with the same options, and
    the info keys are those of the fresh context and show what the option asks for."""
    base = dict(BASE.get(model, {}))
    default = base.get(option, DEFAULTS[option])
    op = _context(model)
    try:
        for step, opts in (("before", {}), ("set", {option: value}), ("reset", {option: default})):
            if opts:
                op.set_option(option, opts[option])
            effective = dict(base, **opts)
            got = _fill(op, model, effective)
            _check_fill(model, effective, got, _fresh(model, effective), (option, model, value, step))
            if step == "set":
                assert {k: got[1].get(k, op.info(k)) for k in shown} == shown, (option, model, step, got[1])
    finally:
        op.close()


WALK_STEPS = 40


@pytest.mark.gpu
@pytest.mark.parametrize("model", sorted(MODELS))
def test_random_walk_over_options(need_cuda, model):
    """A seeded walk of 40 steps on one context: each step changes one option (any accepted value), the element type,
    the batch width or where the vectors live (host vectors of at least 2^16 states take the row-chunked D2H path),
    and ends with a product against the oracle."""
    seed = 1000 + sorted(MODELS).index(model)
    rng = np.random.default_rng(seed)
    ref = _reference(model)
    op = _context(model)
    cplx, width, on_host = False, 0, False
    history = []
    try:
        for step in range(WALK_STEPS):
            what = rng.choice(["option", "option", "elt", "batch", "host"])
            if what == "option":
                option = sorted(ACCEPTED)[rng.integers(len(ACCEPTED))]
                value = int(rng.choice(ACCEPTED[option]))
                op.set_option(option, value)
                history.append(f"{option}={value}")
            elif what == "elt":
                cplx = not cplx
                history.append("c128" if cplx else "f64")
            elif what == "batch":
                width = int(rng.integers(0, 7))
                history.append(f"batch={width}")
            else:
                on_host = not on_host
                history.append("host" if on_host else "device")
            X, Y = ref[cplx]
            if width == 0:
                y = op.matvec(X[0]) if on_host else _product(op, X[0])
                ok = _close(y, Y[0])
            else:
                y = op.matvec_batch(X[:width]) if on_host else _batch(op, X[:width])
                ok = all(_close(y[j], Y[j]) for j in range(width))
            assert ok, f"seed {seed}, step {step}: {' '.join(history)}"
    finally:
        op.close()


# ---- observables and solvers between products, on re-installed blocks

def _session(op, n):
    """product, correlations (they refill the k_rows table), product of the other type, expm_multiply at krylov_dim
    64, eigsh with a block of 6 and the quadrature in groups of 6 (both on k_rows_batch), product"""
    xf, xc = _x(n, False, 801), _x(n, True, 802)
    out = {"y1": op.matvec(xf), "pm": op.pm_correlations(xf), "zz": np.concatenate(op.zz_correlations(xf), axis=None),
           "y2": op.matvec(xc)}
    out["expm"] = op.expm_multiply(xc, -0.3j, krylov_dim=64)[0]
    vals, vecs, _, conv, _, _ = op.eigsh(4, block_size=6, tol=1e-9)
    assert conv == 4
    out["eigsh"], out["eigvecs"] = vals, vecs
    nodes, weights, _, _ = op.lanczos_quadrature(6, 12, seed=5)
    assert op.info("quadrature_group") == 6
    out["nodes"], out["weights"] = nodes, weights
    out["y3"] = op.matvec(xf)
    return out, {"y1": xf, "y2": xc, "y3": xf}


@pytest.mark.gpu
def test_observables_and_solvers_between_products(need_cuda):
    """On one context of the free-magnetisation ring: the session above on a weight-9 block, then after re-installing
    a larger (weight 10) and a smaller (weight 6) block, so that the work space is reused after growing and after
    shrinking.  Every result is bit-identical to the same session on a fresh context with that block; the products
    match the oracle's on the fixed-weight sector."""
    free = _ring_20(None)
    op = Operator(free[1])
    try:
        for w in (9, 10, 6):
            reps, _ = _sector(w)
            op.basis.uncheckedSetRepresentatives(reps)
            got, xs = _session(op, reps.shape[0])
            fresh = Operator(free[1])
            try:
                fresh.basis.uncheckedSetRepresentatives(reps)
                want, _ = _session(fresh, reps.shape[0])
            finally:
                fresh.close()
            for key in got:
                assert np.array_equal(got[key], want[key]), (w, key, "differs from a fresh context",
                                                             np.abs(got[key] - want[key]).max())
            for key, x in xs.items():
                y_ref = po.matvec_global(_ring_20(w)[1], reps, x, 1)
                assert _close(got[key], y_ref), (w, key)
    finally:
        op.close()


# ---- re-installed bases

NORM_CASES = {
    "torus_6x6_w7": MODELS["torus_6x6_w7"],                               # trivial characters
    "momentum_10": MODELS["momentum_10"],                                 # complex characters
    "torus_4x4_inv+1": MODELS["torus_4x4_inv"],                           # spin flips in the group
    "torus_4x4_inv-1": lambda: _torus("heisenberg_square_4x4", 8, -1),    # spin flips, character -1
    "ring_20_free": lambda: _ring_20(None),                               # free magnetisation
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(NORM_CASES))
def test_set_representatives_computes_norms(need_cuda, name):
    """dmv_set_representatives without norms (k_compute_norms) gives dmv_basis_build's norms bit for bit and the
    oracle's to 1e-15 relative; the products on that context then match the oracle."""
    basis, matrix = NORM_CASES[name]()
    reps, o_norms = po.enumerate_states(basis)
    built = Operator(matrix)
    try:
        built.basis.build()
        assert np.array_equal(built.basis.representatives(), reps)
        b_norms = built.basis.norms()
    finally:
        built.close()
    op = Operator(matrix)
    try:
        if name == "momentum_10":
            op.set_option("mode", 1)
        op.basis.uncheckedSetRepresentatives(reps)
        norms = op.basis.norms()
        assert np.array_equal(norms, b_norms), np.abs(norms - b_norms).max()
        assert np.all(np.abs(norms - o_norms) <= 1e-15 * o_norms), np.abs(norms - o_norms).max()
        for cplx in (False, True):
            x = _x(reps.shape[0], cplx, 811)
            y_ref = po.matvec_global(matrix, reps, x, 1, num_tasks=po.num_threads())
            assert _close(op.matvec(x), y_ref), (name, cplx)
            assert _close(_product(op, x), y_ref), (name, cplx)
    finally:
        op.close()


def _probe(reps, sites, seed):
    rng = np.random.default_rng(seed)
    absent = rng.integers(0, 1 << sites, 2000, dtype=np.uint64)
    return np.concatenate([reps, absent, np.array([0, (1 << sites) - 1], dtype=np.uint64)])


def _weight_blocks(sites):
    full = np.array([(1 << sites) - 1], dtype=np.uint64)     # all up: closed under H, the only state of its weight
    return [("w", None), ("w'", None), ("w''", None), ("empty", np.zeros(0, dtype=np.uint64)), ("single", full),
            ("w again", None)]


def _check_weight_block(op, reps, matrix_w, sites, where, products):
    n = reps.shape[0]
    assert op.basis.numberStates() == n, where
    if n:                              # (every mode indexes an empty block alike)
        assert op.info("index_mode") == INDEX_DIRECTORY, (where, op.info("index_mode"))
    probe = _probe(reps, sites, 5)
    assert np.array_equal(op.basis.stateIndex(probe), po.state_index(reps, probe)), where
    xs = {cplx: _x(n, cplx, 820) for cplx in (False, True)}
    refs = {cplx: po.matvec_global(matrix_w, reps, xs[cplx], 1) if n else np.zeros(0, xs[cplx].dtype)
            for cplx in (False, True)}
    X = np.stack([_x(n, True, 830 + j) for j in range(3)])
    Y = [po.matvec_global(matrix_w, reps, X[j], 1) if n else np.zeros(0, complex) for j in range(3)]
    for label, options in products:
        _set(op, **options)
        for cplx in (False, True):
            y = _product(op, xs[cplx])
            assert y.shape == (n,) and _close(y, refs[cplx]), (where, label, cplx)
            assert _close(op.matvec(xs[cplx]), refs[cplx]), (where, label, cplx, "host")
        Yb = _batch(op, X)
        assert Yb.shape == (3, n) and all(_close(Yb[j], Y[j]) for j in range(3)), (where, label, "batch")


# k_rows under every table layout (the dense ordered one on and off), k_rows_batch, k_pull and the scatter form
ROWS_PRODUCTS = ([(t, dict(o, rows_dense_order=d)) for t, o in TABLES.items() for d in (0, 1) if not (d and t == "hashed")]
                 + [("k_pull", dict(TABLES["ordered_14_8"], rows=0, mode=1)), ("push", dict(rows=-1, mode=0)),
                    ("default", dict(TABLES["ordered_14_8"], rows_dense_order=-1, mode=-1))])
GATHER_PRODUCTS = [("k_gather", dict(mode=-1)), ("k_gather split 4", dict(gather_split=4)),
                   ("push", dict(gather_split=-1, mode=0)), ("k_pull", dict(mode=1, gather=0)),
                   ("default", dict(mode=-1, gather=-1))]


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [True, False], ids=["ring_20_k_rows", "chain_16_k_gather"])
def test_weight_blocks_in_free_context(need_cuda, symmetric):
    """Weight-sector blocks installed one after the other into one free-magnetisation context: w, a larger w', a
    smaller w'', an empty block, the single all-up state, w again.  n grows and shrinks and the largest representative
    (the directory shift) moves.  After each install the index is the directory (no other mode indexes such a block),
    dmv_state_index equals the oracle's on the block and on absent states, and every product kernel matches the
    oracle's fixed-weight sector; the empty block gives empty products."""
    sites = 20 if symmetric else 16
    weights = {"w": 9, "w'": 10, "w''": 6, "w again": 9} if symmetric else {"w": 7, "w'": 8, "w''": 5, "w again": 7}
    model = _ring_20 if symmetric else _chain_16
    op = Operator(model(None)[1])
    try:
        for label, block in _weight_blocks(sites):
            w = weights.get(label, 0 if block is None or block.shape[0] == 0 else sites)
            reps = _sector(w, symmetric)[0] if block is None else block
            op.basis.uncheckedSetRepresentatives(reps)
            if symmetric and reps.shape[0]:
                assert np.array_equal(op.basis.norms(), _sector(w, True)[1]), label
            _check_weight_block(op, reps, model(w)[1], sites, (label, w),
                                ROWS_PRODUCTS if symmetric else GATHER_PRODUCTS)
    finally:
        op.close()


@pytest.mark.gpu
def test_rank_indices_reject_a_block_of_the_mirror_weight(need_cuda):
    """A fixed-weight context (16 sites, weight 5) holding the block of weight 11, which has as many states: the
    combinadic rank and the Lin tables pass the count check and must be rejected by k_verify_rank, whatever the index
    option asks; the product matches the oracle's weight-11 sector."""
    reps, _ = _sector(11, False)
    assert reps.shape[0] == _sector(5, False)[0].shape[0]
    matrix = _chain_16(11)[1]
    x = _x(reps.shape[0], True, 840)
    y_ref = po.matvec_global(matrix, reps, x, 1)
    op = Operator(_chain_16(5)[1])
    try:
        for index in (-1, 2, 3, 0):
            op.set_option("index", index)
            op.basis.uncheckedSetRepresentatives(reps)
            assert op.info("index_mode") == INDEX_DIRECTORY, (index, op.info("index_mode"))
            probe = _probe(reps, 16, 6)
            assert np.array_equal(op.basis.stateIndex(probe), po.state_index(reps, probe)), index
            assert _close(_product(op, x), y_ref), index
        op.basis.build()               # the context's own sector: the option applies again
        op.set_option("index", 2)
        assert op.info("index_mode") == 2
    finally:
        op.close()


P = 3


def _hashed(cl, x, masks, replicated):
    xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
    yb = cl.matvec_replicated(xb) if replicated else cl.matvec(xb)
    return hashed_to_block([t.cpu().numpy() for t in yb], masks)


@pytest.mark.gpu
def test_emulated_ranks_reinstall_blocks(need_cuda):
    """Three logical ranks of the 6x6 square at weight 7: once the replicated-x twin and a record plan exist, the same
    hash blocks are installed again (without norms).  That deletes the twin and resets the plan; both forms of the
    product still match the oracle's 3-rank product, and each rank's plan counts the oracle's records."""
    basis, matrix = MODELS["torus_6x6_w7"]()
    reps = _reference("torus_6x6_w7")["reps"]
    masks, blocks = po.partition_by_hash(reps, P)
    x = _x(reps.shape[0], True, 850)
    y_ref = po.matvec_global(matrix, reps, x, P, num_tasks=po.num_threads())
    cl = EmulatedCluster(matrix, P).build()
    try:
        assert _close(_hashed(cl, x, masks, True), y_ref) and _close(_hashed(cl, x, masks, False), y_ref)
        assert all(op.info("global_states") == reps.shape[0] for op in cl.ops)
        cl.set_representatives(blocks)
        assert all(op.info("global_states") == -1 and op.info("replicated") == 0 for op in cl.ops)
        for replicated in (False, True, False):
            y = _hashed(cl, x, masks, replicated)
            assert _close(y, y_ref), (replicated, np.abs(y - y_ref).max())
        for r, op in enumerate(cl.ops):
            _, _, keys, _ = po.compute_off_diag(matrix, P, blocks[r], np.ones(blocks[r].shape[0]))
            assert np.array_equal(op.plan(), np.bincount(keys, minlength=P)), r
    finally:
        cl.close()


@pytest.mark.gpu
def test_emulated_ranks_weight_blocks_in_free_context(need_cuda):
    """Three logical ranks of the free-magnetisation ring holding the hash blocks of its weight-9 sector.  The record
    exchange matches the oracle's 3-rank product on the sector.  The replicated-x form enumerates its twin over the
    whole free basis: it must raise that the blocks are not the hash partition of that basis, or be correct -- never a
    silently wrong y."""
    reps, _ = _sector(9)
    matrix_w = _ring_20(9)[1]
    masks, blocks = po.partition_by_hash(reps, P)
    cl = EmulatedCluster(_ring_20(None)[1], P)
    try:
        cl.set_representatives(blocks)
        for cplx in (False, True):
            x = _x(reps.shape[0], cplx, 860)
            y_ref = po.matvec_global(matrix_w, reps, x, P)
            assert _close(_hashed(cl, x, masks, False), y_ref), cplx
            try:
                y = _hashed(cl, x, masks, True)
            except nat.DmvError as e:
                assert "not the hash partition of the full basis" in str(e), e
            else:
                assert _close(y, y_ref), (cplx, "replicated-x form silently wrong")
            assert _close(_hashed(cl, x, masks, False), y_ref), (cplx, "after the replicated form")
        # a larger sector: generate plans by itself, since the plan of the last block does not fit this one
        reps, _ = _sector(10)
        masks, blocks = po.partition_by_hash(reps, P)
        cl.set_representatives(blocks)
        x = _x(reps.shape[0], True, 870)
        xb = [torch.from_numpy(b).cuda() for b in block_to_hashed(x, masks, P)]
        ys = [torch.zeros_like(t) for t in xb]
        for r, op in enumerate(cl.ops):
            op.generate(xb[r], ys[r])
            op.synchronize()
        for r, src in enumerate(cl.ops):
            _, _, keys, _ = po.compute_off_diag(_ring_20(10)[1], P, blocks[r], np.ones(blocks[r].shape[0]))
            want = np.bincount(keys, minlength=P)
            for q, dst in enumerate(cl.ops):
                betas, coeffs, n = src.outgoing(q)
                assert q == r or n == want[q], (r, q, n, want[q])
                if q != r and n:
                    dst.accumulate(nat.DMV_C128, n, betas, coeffs, ys[q])
        for op in cl.ops:
            op.synchronize()
        y = hashed_to_block([t.cpu().numpy() for t in ys], masks)
        y_ref = po.matvec_global(_ring_20(10)[1], reps, x, P)
        assert _close(y, y_ref), np.abs(y - y_ref).max()
    finally:
        cl.close()


# ---- streams

def _stream_run(op, name):
    """a product, a batch of four and expm_multiply with x written by a torch kernel on the current stream just before"""
    ref = _reference(name)
    X = torch.from_numpy(ref[True][0][:4]).cuda()
    scale = torch.full((1,), 2.0, dtype=torch.float64, device="cuda")
    x = X[0] * scale                            # written on the current stream, no synchronisation
    y = op.matvec(x)
    Xs = X * scale
    Yb = op.matvec_batch(Xs)
    ye = op.expm_multiply(X[1] * scale, -0.2j, krylov_dim=16)[0]
    return y.cpu().numpy(), Yb.cpu().numpy(), ye.cpu().numpy()


def _stream_expected(name):
    ref = _reference(name)
    expm = _context(name)
    try:
        ye = expm.expm_multiply(2.0 * ref[True][0][1], -0.2j, krylov_dim=16)[0]
    finally:
        expm.close()
    return 2.0 * ref[True][1][0], 2.0 * ref[True][1][:4], ye


def _check_stream(got, want, where):
    y, Yb, ye = got
    assert _close(y, want[0]), (where, "product")
    assert all(_close(Yb[j], want[1][j]) for j in range(4)), (where, "batch")
    assert _close(ye, want[2]), (where, "expm_multiply")


@pytest.mark.gpu
def test_streams(need_cuda):
    """On a side torch stream, then the default stream, then the context's own stream (dmv_set_stream(ctx, NULL, 1),
    host vectors), then two contexts on two side streams interleaved: every result matches the oracle (expm_multiply:
    a fresh context on its own stream)."""
    names = ("chain_16", "torus_6x6_w7")
    want = {name: _stream_expected(name) for name in names}
    ops = {name: _context(name) for name in names}
    try:
        torch.cuda.synchronize()
        for name, op in ops.items():
            side = torch.cuda.Stream()
            with torch.cuda.stream(side):
                got = _stream_run(op, name)
            _check_stream(got, want[name], (name, "side stream"))
            _check_stream(_stream_run(op, name), want[name], (name, "default stream"))
            nat.check(nat.lib().dmv_set_stream(op._ctx, None, 1))
            # Operator.use_torch_stream skips the call when torch's stream is the one it set last: forget that one, so
            # that the next torch product moves the context back to a torch stream whichever stream that is
            op._stream_handle = None
            ref = _reference(name)
            X = 2.0 * ref[True][0][:4]
            got = (op.matvec(X[0]), op.matvec_batch(X), op.expm_multiply(X[1], -0.2j, krylov_dim=16)[0])
            _check_stream(got, want[name], (name, "own stream"))
        streams = {name: torch.cuda.Stream() for name in names}
        results = {name: [] for name in names}
        ref = {name: _reference(name) for name in names}
        for k in range(2):
            for name in names:
                with torch.cuda.stream(streams[name]):
                    x = torch.from_numpy(ref[name][True][0][0]).cuda() * 2.0
                    results[name].append(ops[name].matvec(x))
        torch.cuda.synchronize()
        for name in names:
            for y in results[name]:
                assert _close(y.cpu().numpy(), want[name][0]), (name, "two side streams")
    finally:
        for op in ops.values():
            op.close()
