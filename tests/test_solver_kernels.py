"""The vector kernels of the device solvers (csrc/dmv_solver.cu), one launcher at a time, against exact references.

dmv_lanczos, dmv_expm_multiply, dmv_eigsh and dmv_lanczos_quadrature run these kernels between products.  Through the
solvers an error hides: dmv_eigsh re-orthogonalises and re-measures every residual, so a Gram entry that is slightly
wrong costs products, not answers.  Here dmv_debug_solver_kernel runs one launcher on a host arena of doubles laid out
by the test -- stored vectors in any order with gaps, W blocks with w_stride > n, out aliasing w -- with every gap and
guard band filled with sentinel NaNs, and the partials and small outputs poisoned with NaN before the launch.

Exact references: vector entries, coefficients and rotation matrices are small integers (real and imaginary parts in
[-7, 7]).  Every product and every partial sum is then an integer far below 2^53, exact in float64 whatever the
summation order, grid or atomics, so the kernel must equal numpy's float64 result exactly (as values: +0 and -0 agree).
k_quad_update takes b2 values that are powers of four and integer dot values: 1 / beta, alpha / beta and beta / beta_prev
are then exact binary fractions and the recurrence is exact too.  A second pass runs the same launchers on Gaussian
data against a long-double reference within a derived rounding bound, twice, and requires bit-identical repeats of
every partials-based kernel (k_dot and k_lanczos_update add with atomics and are exempt).

Without a GPU: the references check themselves (int64 against float64, the quadrature step against a plain Lanczos
step, the hashes against the splitmix64 known answers) and the entry's argument checks run.
"""
import ctypes as C
import math

import numpy as np
import pytest

from distributed_matvec_b200 import _native as nat
from distributed_matvec_b200.thermal import _hash64_01, _hash64_01_int, seeded_start_vectors

torch = pytest.importorskip("torch")

# ---- constants copied from csrc/dmv_solver.cu and csrc/dmv_host.h ------------------------------------------------
K_THREADS = 256                  # kThreads: threads per CTA of every solver kernel
K_MAX_BLOCK_VECTORS = 65         # kMaxBlockVectors: stored vectors a block launcher accepts
K_MAX_BLOCK_RHS = 6              # kMaxBlockRhs: W vectors of k_block_gram / k_block_update, G of the quadrature
K_ROT_WORDS = 64                 # kRotWords: 8-byte words of every vector in a k_block_rotate tile
GRAM_CHUNK = {1: 8, 2: 4, 3: 2, 4: 2, 5: 1, 6: 1}   # gram_chunk<CE, R>() = 8 / R: stored vectors per pass

# Elements of one vector a CTA covers per pass of its grid-stride loop ("tile"), by launcher and instance:
#   block_dot:  kThreads * dot_elems<CE>(),     dot_elems = CE ? 2 : 4
#   block_gram: kThreads * gram_elems<CE, R>(), gram_elems = CE ? (R <= 3 ? 4 : 2) : (R <= 3 ? 8 : 4)
#   block_rotate: kRotWords words, 64 real or 32 complex elements
#   lanczos_update: one 8-byte word per thread (real and imaginary parts alike), kThreads words
#   every other launcher: one element per thread, kThreads ("scale" and "fill" count words)
TILE = {
    "lanczos_update": {False: 256, True: 128},
    "block_dot": {False: 1024, True: 512},
    "block_gram": {False: {1: 2048, 2: 2048, 3: 2048, 4: 1024, 5: 1024, 6: 1024},
                   True: {1: 1024, 2: 1024, 3: 1024, 4: 512, 5: 512, 6: 512}},
    "block_rotate": {False: 64, True: 32},
}


def tile(kernel, ce, width=1):
    t = TILE.get(kernel)
    if t is None:
        return K_THREADS
    t = t[ce]
    return t[width] if isinstance(t, dict) else t


def lengths(kernel, ce, width=1):
    """n in {0, 1, 31, 33, tile - 1, tile, tile + 1}"""
    t = tile(kernel, ce, width)
    return sorted({0, 1, 31, 33, t - 1, t, t + 1})


# A quiet NaN with a payload no arithmetic produces: every gap and guard band of the arena holds it.
SENTINEL_BITS = np.uint64(0x7FF8DEAD5E7711E1)
SENTINEL = np.array([SENTINEL_BITS], dtype=np.uint64).view(np.float64)[0]
EPS = 2.0 ** -53   # unit roundoff of float64


@pytest.fixture(scope="module")
def need_cuda():
    if not torch.cuda.is_available():
        pytest.fail("these tests need a CUDA device (no CPU fallback exists)")


# ---- the arena --------------------------------------------------------------------------------------------------
def words_of(v, ce):
    v = np.asarray(v, dtype=np.complex128 if ce else np.float64)
    return np.ascontiguousarray(v).view(np.float64).ravel()


def vec_of(words, ce):
    return np.ascontiguousarray(words).view(np.complex128) if ce else np.array(words)


class Arena:
    """Vectors placed one after another, each behind a band of sentinels (an even number of words, so every complex
    vector starts on 16 bytes)."""

    def __init__(self, ce, gap=6):
        self.ce, self.gap, self.parts, self.size = ce, gap, [], gap
        self.c = 2 if ce else 1

    def put(self, v):
        w = words_of(v, self.ce)
        off = self.size
        self.parts.append((off, w))
        self.size += w.size + self.gap
        return off

    def put_block(self, vs, stride):
        """the vectors vs[r] at r * stride elements apart (sentinels between them when stride > n)"""
        n = vs[0].shape[0]
        w = np.full(((len(vs) - 1) * stride + n) * self.c, SENTINEL)
        for r, v in enumerate(vs):
            w[r * stride * self.c:(r * stride + n) * self.c] = words_of(v, self.ce)
        return self.put_words(w)

    def put_words(self, w):
        off = self.size
        self.parts.append((off, np.asarray(w, dtype=np.float64)))
        self.size += len(w) + self.gap
        return off

    def build(self):
        a = np.full(self.size, SENTINEL)
        for off, w in self.parts:
            a[off:off + w.size] = w
        return a

    def get(self, a, off, n):
        return vec_of(a[off:off + n * self.c], self.ce)


def same_bits(a, b):
    return np.array_equal(np.asarray(a, dtype=np.float64).view(np.uint64), np.asarray(b, dtype=np.float64).view(np.uint64))


def put_vec(a, off, v, ce):
    w = words_of(v, ce)
    a[off:off + w.size] = w


def run(kernel, ce, n, args, arena, coef=(), out_words=0, out=None, scalar=0.0):
    """dmv_debug_solver_kernel -> (arena after, small outputs, grid)"""
    arena = np.array(arena, dtype=np.float64)
    coef = np.ascontiguousarray(coef, dtype=np.float64)
    out = np.zeros(out_words) if out is None else np.array(out, dtype=np.float64)
    a = np.array([int(x) & ((1 << 64) - 1) for x in args], dtype=np.uint64).view(np.int64)
    grid = C.c_int(-1)
    nat.check(nat.lib().dmv_debug_solver_kernel(
        kernel.encode(), nat.DMV_C128 if ce else nat.DMV_F64, n, a.ctypes.data if a.size else None, a.size, scalar,
        arena.ctypes.data, arena.size, coef.ctypes.data if coef.size else None, coef.size,
        out.ctypes.data if out.size else None, out.size, C.byref(grid)))
    return arena, out, grid.value


def rejects(kernel, ce, n, args, arena_words, coef_words=0, out_words=0, match=""):
    arena = np.zeros(arena_words)
    coef = np.zeros(max(coef_words, 1))
    out = np.zeros(max(out_words, 1))
    a = np.asarray(args, dtype=np.int64)
    grid = C.c_int(-1)
    rc = nat.lib().dmv_debug_solver_kernel(kernel.encode(), nat.DMV_C128 if ce else nat.DMV_F64, n,
                                          a.ctypes.data if a.size else None, a.size, 0.0, arena.ctypes.data,
                                          arena.size, coef.ctypes.data, coef_words, out.ctypes.data, out_words,
                                          C.byref(grid))
    assert rc != 0, (kernel, args)
    msg = nat.lib().dmv_last_error().decode()
    assert match in msg, msg


# ---- data -------------------------------------------------------------------------------------------------------
def ints(rng, shape, ce, lo=-7, hi=7):
    x = rng.integers(lo, hi + 1, size=shape).astype(np.float64)
    if ce:
        x = x + 1j * rng.integers(lo, hi + 1, size=shape).astype(np.float64)
    return x


def gauss(rng, shape, ce):
    x = rng.standard_normal(shape)
    if ce:
        x = x + 1j * rng.standard_normal(shape)
    return x


def cplx_pairs(c, ce):
    """J coefficients as the launchers read them: interleaved (re, im); real vectors read the real parts"""
    c = np.asarray(c, dtype=np.complex128).ravel()
    return np.ascontiguousarray(c).view(np.float64)


def as_out(h):
    """complex results as (re, im) pairs, the layout of the small outputs"""
    return np.ascontiguousarray(np.asarray(h, dtype=np.complex128).ravel()).view(np.float64)


def exact_dot(a, b):
    """sum conj(a) b in int64 arithmetic (integer-valued data only)"""
    ar, ai, br, bi = (np.rint(t).astype(np.int64) for t in (np.real(a), np.imag(a), np.real(b), np.imag(b)))
    return complex(int(ar @ br + ai @ bi), int(ar @ bi - ai @ br))


def ld_dot(a, b):
    """sum conj(a) b in long double, and sum |a_i| |b_i| (the scale of its rounding error)"""
    a, b = np.asarray(a), np.asarray(b)
    ar, ai = np.real(a).astype(np.longdouble), np.imag(a).astype(np.longdouble)
    br, bi = np.real(b).astype(np.longdouble), np.imag(b).astype(np.longdouble)
    re = np.sum(ar * br + ai * bi)
    im = np.sum(ar * bi - ai * br)
    scale = float(np.sum(np.abs(ar * br) + np.abs(ai * bi) + np.abs(ar * bi) + np.abs(ai * br)))
    return complex(float(re), float(im)), scale


# Rounding bound of a reduction.  Each result is one sum of the m = n (real) or 2 n (complex) products p_i, computed
# by a tree: a per-thread chain over its elements (at most ceil(n / (grid kThreads)) of them), a warp butterfly (5 adds),
# 8 warps in order, and k_reduce_partials (ceil(grid / kThreads) per thread, 5 + 8 more).  Every add and product rounds
# once with relative error <= eps, so the computed sum is sum p_i (1 + d_i) with |d_i| <= (D + 1) eps / (1 - (D + 1) eps)
# where D is the depth of the tree; D <= ceil(n / (grid kThreads)) + ceil(grid / kThreads) + 26 (two-level chains of
# k_block_dot / k_block_gram, E elements then the tiles of a CTA, never exceed the elements of a thread), so
# |error| <= 2 (D + 2) eps sum |p_i|.  The long-double reference adds < 1e-3 of that.
def reduce_bound(n, grid, scale):
    depth = -(-max(n, 1) // (max(grid, 1) * K_THREADS)) + -(-max(grid, 1) // K_THREADS) + 26
    return 2.0 * (depth + 2) * EPS * scale


# Rounding bound of an updated element out_i = a w_i - sum_{k < J} c_k V_{k,i}: J + 1 products and J subtractions in
# one chain, each rounding once (complex: two real products per term), so |error| <= 2 (J + 2) eps (|a w_i| +
# sum |c_k| |V_{k,i}|) with |c| the modulus.
def update_bound(J, scale):
    return 2.0 * (J + 2) * EPS * scale


# ---- host-only: the references check themselves -------------------------------------------------------------------
@pytest.mark.parametrize("ce", [False, True])
def test_integer_references_are_exact(ce):
    """The integer cases up to the largest the GPU tests use: the int64 reference equals numpy's float64 dot and matrix products bit for bit."""
    rng = np.random.default_rng(1)
    for n in (1, 33, 2049, 1 << 22):
        a, b = ints(rng, n, ce), ints(rng, n, ce)
        assert exact_dot(a, b) == np.vdot(a, b)
        assert abs(exact_dot(a, b).real) < 2 ** 40
        assert ld_dot(a, b)[0] == exact_dot(a, b)
    V, W = ints(rng, (65, 2049), ce), ints(rng, (6, 2049), ce)
    G = V.conj() @ W.T
    for k in (0, 31, 64):
        for r in range(6):
            assert exact_dot(V[k], W[r]) == G[k, r]
    c = ints(rng, (65, 6), ce)
    upd = W - c.T @ V
    for r in range(6):
        want = W[r].astype(np.complex128) - sum(c[k, r] * V[k] for k in range(65))
        assert np.array_equal(upd[r], want)


def quad_reference(P, Q, W, dot, b2, j):
    """Step j of the quadrature recurrence, independently of the library: alpha_j = dot_j / b2_j, beta_t = sqrt(b2_t),
    r_{j+1} = (W - alpha_j Q) / beta_j - (beta_j / beta_{j-1}) P, P = Q = 0 for a vector whose recurrence broke down
    (b2_j = 0, b2_{j-1} = 0, or sqrt(b2_j) <= 1e-14 max(1, |dot_{j-1} / b2_{j-1}|)).  P, Q, W: (G, n); dot, b2: (j + 1, G).
    -> (P', Q', |r_{j+1}|^2 per vector)"""
    G = P.shape[0]
    Pn, Qn, nrm = P.copy(), Q.copy(), np.zeros(G)
    for g in range(G):
        bj2 = b2[j][g]
        dead = not bj2 > 0.0
        if not dead and j > 0:
            bp2 = b2[j - 1][g]
            dead = not bp2 > 0.0 or math.sqrt(bj2) <= 1e-14 * max(1.0, abs(dot[j - 1][g] / bp2))
        if dead:
            Pn[g] = 0.0
            Qn[g] = 0.0
            continue
        alpha, beta = dot[j][g] / bj2, math.sqrt(bj2)
        r = (W[g] - alpha * Q[g]) / beta
        if j > 0:
            r = r - (beta / math.sqrt(b2[j - 1][g])) * P[g]
        Pn[g] = r
        nrm[g] = float(np.sum(np.abs(r) ** 2))
    return Pn, Qn, nrm


def test_quadrature_reference_is_a_lanczos_step():
    """quad_reference on a small dense Hermitian matrix: the unnormalised vectors r_t are the Lanczos vectors times
    |r_t| (scipy-free: q_{t+1} beta_{t+1} = H q_t - alpha_t q_t - beta_t q_{t-1} with normalised q)."""
    rng = np.random.default_rng(2)
    for ce in (False, True):
        n = 12
        A = gauss(rng, (n, n), ce)
        H = A + A.conj().T
        r0 = gauss(rng, n, ce)
        # the plain normalised Lanczos recurrence
        q, q_prev, beta_prev, alphas, betas, qs = r0 / np.linalg.norm(r0), np.zeros(n), 0.0, [], [], []
        for _ in range(4):
            qs.append(q)
            w = H @ q
            alpha = np.vdot(q, w).real
            w = w - alpha * q - beta_prev * q_prev
            beta = np.linalg.norm(w)
            alphas.append(alpha)
            betas.append(beta)
            q_prev, q, beta_prev = q, w / beta, beta
        # the unnormalised recurrence, one quad_reference step at a time; r_t = |r_0| q_t
        P, Q = np.full((1, n), np.nan, dtype=r0.dtype), r0[None, :].copy()
        dots, b2s = [], []
        for j in range(4):
            Wv = (H @ Q[0])[None, :]
            dots.append([np.vdot(Q[0], Wv[0]).real])
            b2s.append([np.vdot(Q[0], Q[0]).real])
            assert np.allclose(Q[0], math.sqrt(b2s[j][0]) * qs[j], atol=1e-10)   # r_j = |r_j| q_j
            assert abs(dots[j][0] / b2s[j][0] - alphas[j]) < 1e-10
            Pn, Qn, nrm = quad_reference(P, Q, Wv, dots, b2s, j)
            assert abs(math.sqrt(nrm[0]) - betas[j]) <= 1e-10 * betas[j]           # |r_{j+1}| = beta_{j+1}
            P, Q = Q, Pn
    # breakdown rules: b2 = 0, a previous b2 = 0, and the quad_breakdown threshold on both sides
    z = np.zeros((1, 3))
    one = np.ones((1, 3))
    assert not quad_reference(z, one, one, [[0.0]], [[0.0]], 0)[0].any()
    assert not quad_reference(z, one, one, [[1.0], [1.0]], [[0.0], [1.0]], 1)[0].any()
    assert not quad_reference(z, one, one, [[128.0], [1.0]], [[1.0], [4.0 ** -40]], 1)[0].any()   # 2^-40 <= 1.28e-12
    assert quad_reference(z, one, one, [[64.0], [1.0]], [[1.0], [4.0 ** -40]], 1)[0].all()        # 2^-40 > 6.4e-13


def fill_reference(m, seed, offset):
    """k_fill: x[i] = (h >> 11) 2^-53 - 0.5 with h = hash64_01(seed 0x9e3779b97f4a7c15 + offset + i + 1) mod 2^64"""
    base = (int(seed) * 0x9E3779B97F4A7C15 + int(offset) + 1) & ((1 << 64) - 1)
    keys = np.uint64(base) + np.arange(m, dtype=np.uint64)   # wraps modulo 2^64
    h = _hash64_01(keys)
    return (h >> np.uint64(11)).astype(np.float64) * 2.0 ** -53 - 0.5


def test_hash_references_reproduce_splitmix64():
    """fill_reference and seeded_start_vectors hash the splitmix64 sequence: with the key k 0x9e3779b97f4a7c15 they
    give the published first outputs of splitmix64 seeded with 0 (test_oracle_pins)."""
    known = [0xe220a8397b1dcdaf, 0x6e789e6aa1b965f4, 0x06c45d188009454f, 0xf88bb8a8724c81ec]
    M = (1 << 64) - 1
    for k, h in enumerate(known, start=1):
        assert _hash64_01_int((k * 0x9E3779B97F4A7C15) & M) == h
        # seed k, offset 2^64 - 1, element 0: the key is k * golden
        assert fill_reference(1, k, M)[0] == (h >> 11) * 2.0 ** -53 - 0.5
    # the key of vector r of seeded_start_vectors with seed 0 is hash64_01((r + 1) golden) = known[r]; rep 0 hashes it
    x = seeded_start_vectors(np.zeros(1, dtype=np.uint64), 4, 0)
    for r, h in enumerate(known):
        assert x[r, 0] == (1.0 if _hash64_01_int(h) >> 63 == 0 else -1.0)
    # offsets with the high bits set wrap like the device's uint64 arithmetic
    off = (0xFFFFFF << 40) & M
    got = fill_reference(3, 5, off)
    want = [((_hash64_01_int((5 * 0x9E3779B97F4A7C15 + off + i + 1) & M) >> 11) * 2.0 ** -53 - 0.5) for i in range(3)]
    assert np.array_equal(got, want)


def test_entry_rejects_bad_arguments():
    """Argument checks of dmv_debug_solver_kernel that come before any device work: unknown kernel, element type,
    offsets past the arena, odd offsets for complex elements, too few offsets, short coefficient or output arrays."""
    rejects("no_such_kernel", False, 4, [0, 0], 16, match="unknown kernel")
    rejects("block_dot", False, -1, [0, 0], 16, out_words=2, match="n must be")
    rejects("dot", False, 8, [0, 9], 16, out_words=2, match="past the arena")
    rejects("dot", False, 8, [-2, 0], 16, out_words=2, match="past the arena")
    rejects("dot", True, 4, [0, 3], 16, out_words=2, match="odd word offset")
    rejects("block_dot", True, 4, [1, 0, 9], 32, out_words=4, match="odd word offset")
    rejects("block_gram", True, 4, [1, 1, 0, 4, 11], 64, out_words=4, match="odd word offset")
    rejects("block_gram", False, 4, [0, 2, 0, 3], 64, out_words=8, match="w_stride")
    rejects("block_gram", False, 4, [0, 2, 60, 4], 64, out_words=8, match="past the arena")
    rejects("block_dot", False, 4, [2, 0, 4], 16, out_words=6, match="offsets")
    rejects("block_dot", False, 4, [1, 0, 4], 16, out_words=2, match="outputs")
    rejects("block_combine", False, 4, [2, 0, 4, 8, 12], 32, coef_words=2, out_words=2, match="coefficients")
    rejects("lanczos_update", False, 4, [0, 4, -1], 16, coef_words=1, out_words=1, match="coefficients")
    rejects("block_dot", False, 4, [1, -1, 4], 16, out_words=4, match="past the arena")   # w must not be null
    rejects("quad_update", False, 4, [1, 0, 4, 8, -1, 2], 16, coef_words=4, out_words=2, match="j must be")
    rejects("quad_update", False, 4, [1, 0, 4, 8, 1, 3], 16, coef_words=6, out_words=2, match="coefficients")
    rejects("quad_dot", True, 4, [2, 0, 16], 24, out_words=4, match="past the arena")
    rejects("dot", False, 8, [0, 0], 8, out_words=1, match="outputs")


# ---- GPU: one checker per launcher --------------------------------------------------------------------------------
# exact=True: integer data, results equal to numpy's float64 (exact) values.  exact=False: Gaussian data, results within
# the rounding bounds above of a long-double reference, and a second identical call that must repeat every output bit
# (partials-based launchers).  Every checker also requires the arena outside its outputs to keep its bits.

def check_arena(after, before, regions):
    """regions: (offset, expected words, bound or None); everything else keeps its bits"""
    keep = np.ones(before.size, dtype=bool)
    for off, want, bound in regions:
        got = after[off:off + want.size]
        keep[off:off + want.size] = False
        if bound is None:
            assert np.array_equal(got, want), np.flatnonzero(got != want)[:8]
        else:
            assert np.all(np.abs(got - want) <= bound), np.flatnonzero(~(np.abs(got - want) <= bound))[:8]
    assert same_bits(after[keep], before[keep]), np.flatnonzero(after[keep].view(np.uint64) != before[keep].view(np.uint64))[:8]


def check_values(got, want, bound):
    got, want = np.asarray(got), np.asarray(want)
    if bound is None:
        assert np.array_equal(got, want), (got, want)
    else:
        assert np.all(np.abs(got - want) <= bound), (got, want, bound)


def repeat_identical(call, first):
    """a second call on the same inputs gives the same bits (arena and outputs)"""
    after, out, grid = call()
    assert same_bits(after, first[0]) and same_bits(out, first[1]) and grid == first[2]


def gen_of(exact):
    return ints if exact else gauss


def pair_scale(a, b):
    """sum over i of (|Re a_i| + |Im a_i|) (|Re b_i| + |Im b_i|), the scale of a complex product's rounding"""
    return (np.abs(np.real(a)) + np.abs(np.imag(a))) * (np.abs(np.real(b)) + np.abs(np.imag(b)))


def reductions(pairs, n, grid, exact):
    """expected (re, im) words and bounds of <a, b> for the (a, b) pairs"""
    want, bound = [], []
    for a, b in pairs:
        if exact:
            want.append(np.vdot(a, b))
            continue
        v, scale = ld_dot(a, b)
        want.append(v)
        bound += [reduce_bound(n, grid, scale)] * 2
    return as_out(want), None if exact else np.array(bound)


def elementwise(terms, ce, nterms, exact):
    """expected words and bounds of sum_t coef_t vec_t (coef complex scalars; real vectors use real parts)"""
    if exact:
        acc = sum(c * v for c, v in terms)
        return words_of(acc, ce), None
    acc = sum(np.asarray(c, dtype=np.clongdouble if ce else np.longdouble) * np.asarray(v, dtype=np.clongdouble if ce else np.longdouble) for c, v in terms)
    scale = sum(pair_scale(c, v) for c, v in terms)
    # each of the <= 4 nterms + 2 roundings of an element (two products, their difference and the accumulation per
    # complex term) errs by at most eps times a partial sum bounded by `scale`
    b = (4 * nterms + 4) * EPS * scale
    w = words_of(np.asarray(acc, dtype=np.complex128 if ce else np.float64), ce)
    return w, np.repeat(b, 2) if ce else b


def real_if(c, ce):
    return c if ce else np.real(c)


def check_block_dot(rng, ce, n, J, exact=True):
    gen = gen_of(exact)
    V = [gen(rng, n, ce) for _ in range(J)]
    w = gen(rng, n, ce)
    A, offs = Arena(ce), {}
    for i in rng.permutation(J + 1):
        offs[i] = A.put(V[i] if i < J else w)
    arena = A.build()
    args = [J, offs[J]] + [offs[k] for k in range(J)]
    call = lambda: run("block_dot", ce, n, args, arena, out_words=2 * (J + 1))
    after, out, grid = res = call()
    want, bound = reductions([(v, w) for v in V] + [(w, w)], n, grid, exact)
    check_values(out, want, bound)
    check_arena(after, arena, [])
    if not exact:
        repeat_identical(call, res)
    return grid


def check_block_combine(rng, ce, n, J, a, mode, exact=True):
    """mode: "separate" (out its own vector), "alias" (out = w), "null" (w = null, a = 0)"""
    gen = gen_of(exact)
    V = [gen(rng, n, ce) for _ in range(J)]
    w = gen(rng, n, ce)
    c = ints(rng, J, True) if exact else gauss(rng, J, True)   # real vectors read only the real parts
    A, offs = Arena(ce), {}
    for i in rng.permutation(J + 1):
        offs[i] = A.put(V[i] if i < J else w)
    o = offs[J] if mode == "alias" else A.put_words(np.full(n * A.c, SENTINEL))
    arena = A.build()
    w_at = -1 if mode == "null" else offs[J]
    a = 0.0 if mode == "null" else a
    args = [J, w_at, o] + [offs[k] for k in range(J)]
    call = lambda: run("block_combine", ce, n, args, arena, coef=cplx_pairs(c, ce), out_words=2, scalar=a)
    after, out, grid = res = call()
    terms = [(-real_if(c[k], ce), V[k]) for k in range(J)] + ([] if mode == "null" else [(a, w)])
    want, bound = elementwise(terms if terms else [(0.0, np.zeros(n))], ce, J + 1, exact)
    check_arena(after, arena, [(o, want, bound)])
    got = A.get(after, o, n)
    check_values(out, *reductions([(got, got)], n, grid, exact))
    if not exact:
        repeat_identical(call, res)
    return grid


def w_block(rng, ce, n, R, gen):
    return [gen(rng, n, ce) for _ in range(R)], n + 3   # w_stride > n: sentinels between the W vectors


def check_block_gram(rng, ce, n, J, R, exact=True):
    """W between the stored vectors in memory, and (J >= 2) V_1 = W_0 and V_{J-1} = W_{R-1}: W inside the V list"""
    gen = gen_of(exact)
    V = [gen(rng, n, ce) for _ in range(J)]
    Wv, stride = w_block(rng, ce, n, R, gen)
    A, offs = Arena(ce), {}
    order = list(rng.permutation(J))
    order.insert(len(order) // 2, "W")
    for i in order:
        offs[i] = A.put_block(Wv, stride) if i == "W" else A.put(V[i])
    vo = [offs[k] for k in range(J)]
    if J >= 2:
        V[1], vo[1] = Wv[0], offs["W"]
        V[J - 1], vo[J - 1] = Wv[R - 1], offs["W"] + (R - 1) * stride * A.c
    arena = A.build()
    args = [J, R, offs["W"], stride] + vo
    call = lambda: run("block_gram", ce, n, args, arena, out_words=2 * (J * R + R * R))
    after, out, grid = res = call()
    pairs = [(V[k], Wv[r]) for k in range(J) for r in range(R)] + [(Wv[r], Wv[s]) for r in range(R) for s in range(R)]
    check_values(out, *reductions(pairs, n, grid, exact))
    check_arena(after, arena, [])
    if not exact:
        repeat_identical(call, res)
    return grid


def check_block_update(rng, ce, n, J, R, exact=True):
    gen = gen_of(exact)
    V = [gen(rng, n, ce) for _ in range(J)]
    Wv, stride = w_block(rng, ce, n, R, gen)
    c = ints(rng, (J, R), True) if exact else gauss(rng, (J, R), True)
    A, offs = Arena(ce), {}
    order = list(rng.permutation(J))
    order.insert(len(order) // 2, "W")
    for i in order:
        offs[i] = A.put_block(Wv, stride) if i == "W" else A.put(V[i])
    arena = A.build()
    args = [J, R, offs["W"], stride] + [offs[k] for k in range(J)]
    call = lambda: run("block_update", ce, n, args, arena, coef=cplx_pairs(c, ce), out_words=2 * R)
    after, out, grid = res = call()
    regions = []
    for r in range(R):
        terms = [(1.0, Wv[r])] + [(-real_if(c[k, r], ce), V[k]) for k in range(J)]
        want, bound = elementwise(terms, ce, J + 1, exact)
        regions.append((offs["W"] + r * stride * A.c, want, bound))
    check_arena(after, arena, regions)
    got = [A.get(after, offs["W"] + r * stride * A.c, n) for r in range(R)]
    want, bound = reductions([(g, g) for g in got], n, grid, exact)
    check_values(out, want, bound)
    if not exact:
        repeat_identical(call, res)
    return grid


def check_block_rotate(rng, ce, n, k, l, exact=True):
    """V in a permuted order in memory, with gaps: V_j <- sum_i S_ij V_i for j < l, in place"""
    gen = gen_of(exact)
    V = [gen(rng, n, ce) for _ in range(k)]
    S = ints(rng, (k, l), True) if exact else gauss(rng, (k, l), True) / math.sqrt(k)
    A, offs = Arena(ce), {}
    for i in rng.permutation(k):
        offs[i] = A.put(V[i])
    arena = A.build()
    args = [k, l] + [offs[i] for i in range(k)]
    after, out, grid = run("block_rotate", ce, n, args, arena, coef=cplx_pairs(S, ce))
    regions = []
    for j in range(l):
        want, bound = elementwise([(real_if(S[i, j], ce), V[i]) for i in range(k)], ce, k, exact)
        regions.append((offs[j], want, bound))
    check_arena(after, arena, regions)
    return grid


def check_quad_dot(rng, ce, n, G, same=False, exact=True):
    gen = gen_of(exact)
    Av = [gen(rng, n, ce) for _ in range(G)]
    Bv = Av if same else [gen(rng, n, ce) for _ in range(G)]
    A = Arena(ce)
    a_at = A.put(np.concatenate(Av) if n else np.zeros(0))
    b_at = a_at if same else A.put(np.concatenate(Bv) if n else np.zeros(0))
    arena = A.build()
    call = lambda: run("quad_dot", ce, n, [G, a_at, b_at], arena, out_words=2 * G)
    after, out, grid = res = call()
    check_values(out, *reductions(list(zip(Av, Bv)), n, grid, exact))
    check_arena(after, arena, [])
    if not exact:
        repeat_identical(call, res)
    return grid


def quad_coefficients(rng, G, j, kinds, exact):
    """dot, b2 of steps 0 .. j, shape (j + 1, G); kinds[g]: "live", "b2_zero" (b2_j = 0), "prev_zero" (b2_{j-1} = 0)
    or "breakdown" (quad_breakdown: sqrt(b2_j) = 2^-40 <= 1e-14 |dot_{j-1} / b2_{j-1}| = 1.28e-12)"""
    if exact:   # powers of four and integers: every coefficient of the step is an exact binary fraction
        b2 = 4.0 ** rng.integers(0, 3, size=(j + 1, G))
        dot = rng.integers(-20, 21, size=(j + 1, G)).astype(np.float64)
    else:
        b2 = rng.uniform(0.5, 2.0, size=(j + 1, G))
        dot = rng.standard_normal((j + 1, G))
    for g, kind in enumerate(kinds):
        if kind == "b2_zero":
            b2[j, g] = 0.0
        elif kind == "prev_zero":
            b2[j - 1, g] = 0.0
        elif kind == "breakdown":
            b2[j, g], b2[j - 1, g], dot[j - 1, g] = 4.0 ** -40, 1.0, 128.0
    return dot, b2


def check_quad_update(rng, ce, n, G, j, kinds=None, exact=True):
    """P = r_{j-1} (all sentinels at j = 0: it must not be read), Q = r_j, W = H r_j as G vectors n apart; the
    imaginary slots of dot and b2 are sentinels (never read)"""
    kinds = kinds or ["live"] * G
    gen = gen_of(exact)
    P = np.array([gen(rng, n, ce) for _ in range(G)]).reshape(G, n)
    Q = np.array([gen(rng, n, ce) for _ in range(G)]).reshape(G, n)
    Wm = np.array([gen(rng, n, ce) for _ in range(G)]).reshape(G, n)
    dot, b2 = quad_coefficients(rng, G, j, kinds, exact)
    A = Arena(ce)
    p_at = A.put_words(np.full(G * n * A.c, SENTINEL)) if j == 0 else A.put(P.ravel())
    q_at, w_at = A.put(Q.ravel()), A.put(Wm.ravel())
    arena = A.build()
    coef = np.full(4 * (j + 1) * G, SENTINEL)
    coef[0:2 * (j + 1) * G:2] = dot.ravel()
    coef[2 * (j + 1) * G::2] = b2.ravel()
    args = [G, p_at, q_at, w_at, j, 2 * (j + 1) * G]
    call = lambda: run("quad_update", ce, n, args, arena, coef=coef, out_words=2 * G)
    after, out, grid = res = call()
    if exact:
        Pn, Qn, nrm = quad_reference(P, Q, Wm, dot, b2, j)
        pb = qb = None
    else:
        ld = np.clongdouble if ce else np.longdouble
        Pn, Qn, _ = quad_reference(P.astype(ld), Q.astype(ld), Wm.astype(ld), dot.astype(np.longdouble),
                                   b2.astype(np.longdouble), j)
        Pn, Qn = Pn.astype(P.dtype), Qn.astype(Q.dtype)
        # r = cw W - cq Q - cp P with cw = 1 / beta, cq = dot / b2 / beta, cp = beta / beta_prev: each coefficient
        # carries <= 3 roundings (sqrt and divisions), each term one product and one accumulation, so every term is off
        # by a factor within (1 + eps)^5 and the element by <= 16 eps (|cw W| + |cq Q| + |cp P|)
        scale = np.zeros((G, n))
        for g in range(G):
            if kinds[g] != "live":
                continue
            beta = math.sqrt(b2[j, g])
            cp = beta / math.sqrt(b2[j - 1, g]) if j > 0 and b2[j - 1, g] > 0 else 0.0
            scale[g] = (np.abs(Wm[g]) + abs(dot[j, g] / b2[j, g]) * np.abs(Q[g]) + (cp * np.abs(P[g]) if j > 0 else 0)) / beta
        pb = np.repeat(16 * EPS * scale.ravel(), 2) if ce else 16 * EPS * scale.ravel()
        qb = None
    regions = [(p_at, words_of(Pn.ravel(), ce), pb), (q_at, words_of(Qn.ravel(), ce), qb)]
    check_arena(after, arena, regions)
    got = A.get(after, p_at, G * n).reshape(G, n)
    check_values(out, *reductions([(got[g], got[g]) for g in range(G)], n, grid, exact))
    for g, kind in enumerate(kinds):
        if kind != "live":
            assert not np.any(got[g]) and not np.any(A.get(after, q_at, G * n).reshape(G, n)[g])
            assert out[2 * g] == 0.0 and out[2 * g + 1] == 0.0
    if not exact:
        repeat_identical(call, res)
    return grid


def check_dot(rng, ce, n, exact=True):
    """k_dot adds <a, b> to its output (real vectors leave out[1] alone)"""
    gen = gen_of(exact)
    a, b = gen(rng, n, ce), gen(rng, n, ce)
    A = Arena(ce)
    a_at, b_at = A.put(a), A.put(b)
    arena = A.build()
    after, out, grid = run("dot", ce, n, [a_at, b_at], arena, out=[3.0, -5.0])
    want, bound = reductions([(a, b)], n, grid, exact)
    want = want + np.array([3.0, -5.0 if ce else 0.0])
    if not ce:
        want[1] = -5.0
        bound = None if exact else np.array([bound[0], 0.0])
    check_values(out, want, bound)
    check_arena(after, arena, [])
    return grid


def check_lanczos_update(rng, ce, n, with_u, exact=True):
    """w -= alpha v + beta u (alpha, beta real), out[0] += |w|^2 after"""
    gen = gen_of(exact)
    w, v, u = gen(rng, n, ce), gen(rng, n, ce), gen(rng, n, ce)
    alpha, beta = (float(rng.integers(-7, 8)), float(rng.integers(-7, 8))) if exact else tuple(rng.standard_normal(2))
    A = Arena(ce)
    w_at, v_at = A.put(w), A.put(v)
    u_at = A.put(u) if with_u else -1
    arena = A.build()
    after, out, grid = run("lanczos_update", ce, n, [w_at, v_at, u_at], arena, coef=[alpha, beta], out=[2.0])
    terms = [(1.0, w), (-alpha, v)] + ([(-beta, u)] if with_u else [])
    want, bound = elementwise(terms, ce, 2, exact)
    check_arena(after, arena, [(w_at, want, bound)])
    got = A.get(after, w_at, n)
    want, bound = reductions([(got, got)], n, grid, exact)
    check_values(out, want[:1] + 2.0, None if exact else bound[:1])
    return grid


def check_scale(rng, words, s, alias, accumulate):
    """y = s x (y may be x) or y += s x, over words"""
    x, y = ints(rng, words, False), ints(rng, words, False)
    A = Arena(False)
    x_at = A.put(x)
    y_at = x_at if alias else A.put(y)
    arena = A.build()
    after, _, grid = run("scale", False, words, [x_at, y_at, int(accumulate)], arena, scalar=s)
    base = x if alias else y
    want = base + s * x if accumulate else s * x
    check_arena(after, arena, [(y_at, want, None)])
    return grid


def check_fill(words, seed, offset):
    A = Arena(False)
    x_at = A.put_words(np.full(words, SENTINEL))
    arena = A.build()
    after, _, grid = run("fill", False, words, [x_at, seed, offset], arena)
    check_arena(after, arena, [(x_at, fill_reference(words, seed, offset), None)])
    return grid


def check_quad_fill(rng, ce, n, seed, first, G):
    """x[g n + i] = seeded start value of vector first + g at reps[i]: float64 bit for bit; complex128 to 2 ulp of
    libm (device sincos)"""
    reps = rng.integers(0, 2 ** 63, size=n, dtype=np.uint64) | (rng.integers(0, 2, size=n, dtype=np.uint64) << np.uint64(63))
    A = Arena(ce)
    x_at = A.put_words(np.full(G * n * A.c, SENTINEL))
    arena = A.build()
    after, _, grid = run("quad_fill", ce, n, [x_at, seed, first, G], arena, coef=reps.view(np.float64))
    want = seeded_start_vectors(reps, first + G, seed, complex_vectors=ce)[first:].ravel()
    if ce:
        ww = words_of(want, True)
        bound = 2.0 * np.spacing(np.abs(ww))
        check_arena(after, arena, [(x_at, ww, bound)])
    else:
        check_arena(after, arena, [(x_at, want, None)])
    return grid


# ---- GPU: integer cases, exact ------------------------------------------------------------------------------------
CE = [pytest.param(False, id="float64"), pytest.param(True, id="complex128")]


@pytest.mark.gpu
@pytest.mark.parametrize("R", range(1, K_MAX_BLOCK_RHS + 1))
@pytest.mark.parametrize("ce", CE)
def test_block_gram_and_update_exact(need_cuda, ce, R):
    """k_block_gram<CE, R> and k_block_update<CE, R> at J in {0, 1, KC - 1, KC, KC + 1, 59, 64, 65} (KC = gram_chunk,
    stored vectors per pass; complex R = 6 with J >= 59 takes the shared-memory opt-in above 48 KB) and n in {0, 1, 31,
    33, tile - 1, tile, tile + 1}; W with w_stride > n between the stored vectors, and inside the V list for the Gram."""
    rng = np.random.default_rng(100 + 10 * R + ce)
    KC = GRAM_CHUNK[R]
    for J in sorted({0, 1, KC - 1, KC, KC + 1, 59, 64, 65}):
        for n in lengths("block_gram", ce, R):
            assert check_block_gram(rng, ce, n, J, R) >= 1   # an empty rank still writes its partials
        for n in lengths("block_update", ce):
            assert check_block_update(rng, ce, n, J, R) >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("ce", CE)
def test_block_dot_and_combine_exact(need_cuda, ce):
    """k_block_dot and k_block_combine at J in {0, 1, 7, 8, 9, 64, 65} (kDotChunk = 8 vectors per register chunk) and
    n in {0, 1, 31, 33, tile - 1, tile, tile + 1}; combine into its own vector, over w (out aliasing w), and with w null
    and a = 0 (the restart of dmv_expm_multiply)."""
    rng = np.random.default_rng(200 + ce)
    for J in (0, 1, 7, 8, 9, 64, 65):
        for n in lengths("block_dot", ce):
            assert check_block_dot(rng, ce, n, J) >= 1
        for n in lengths("block_combine", ce):
            for mode, a in (("separate", 3.0), ("alias", -2.0), ("null", 0.0)):
                assert check_block_combine(rng, ce, n, J, a, mode) >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("ce", CE)
def test_block_rotate_exact(need_cuda, ce):
    """k_block_rotate at k in {1, 2, 7, 64, 65}, l in {1, k - 1, k}, n in {0, 1, 31, 33, tile - 1, tile, tile + 1},
    in place over stored vectors in a permuted order with gaps: outputs j < l exact, j >= l and the gaps untouched."""
    rng = np.random.default_rng(300 + ce)
    for k in (1, 2, 7, 64, 65):
        for l in sorted({1, k - 1, k} - {0}):
            for n in lengths("block_rotate", ce):
                grid = check_block_rotate(rng, ce, n, k, l)
                assert (grid >= 1) == (n > 0)


QUAD_KINDS = ["live", "b2_zero", "prev_zero", "breakdown"]


@pytest.mark.gpu
@pytest.mark.parametrize("G", range(1, K_MAX_BLOCK_RHS + 1))
@pytest.mark.parametrize("ce", CE)
def test_quad_dot_and_update_exact(need_cuda, ce, G):
    """k_quad_dot<CE, G> (A = B too) and k_quad_update<CE, G> at n in {0, 1, 31, 33, tile - 1, tile, tile + 1}: step
    j = 0 with P all NaN (never read), steps with every vector live, and groups that mix live vectors with vectors dead
    by b2 = 0, by a zero previous b2 and by quad_breakdown; dead vectors get P = Q = 0 and norm 0."""
    rng = np.random.default_rng(400 + 10 * G + ce)
    for n in lengths("quad_dot", ce):
        assert check_quad_dot(rng, ce, n, G) >= 1
        assert check_quad_dot(rng, ce, n, G, same=True) >= 1
        check_quad_update(rng, ce, n, G, 0)
        check_quad_update(rng, ce, n, G, 0, ["live" if g % 2 else "b2_zero" for g in range(G)])
        check_quad_update(rng, ce, n, G, 3)
        for shift in range(len(QUAD_KINDS)):
            check_quad_update(rng, ce, n, G, 2, [QUAD_KINDS[(g + shift) % 4] for g in range(G)])


@pytest.mark.gpu
@pytest.mark.parametrize("ce", CE)
def test_dot_lanczos_update_and_scale_exact(need_cuda, ce):
    """k_dot (adds to its output; real vectors leave the imaginary slot alone), k_lanczos_update with and without u,
    k_scale into another vector, over x itself, and accumulating; n = 0 launches nothing and leaves the outputs."""
    rng = np.random.default_rng(500 + ce)
    for n in lengths("dot", ce):
        assert (check_dot(rng, ce, n) >= 1) == (n > 0)
        for with_u in (False, True):
            assert (check_lanczos_update(rng, ce, n, with_u) >= 1) == (n > 0)
        words = n * (2 if ce else 1)
        for s, alias, acc in ((3.0, False, False), (-0.5, True, False), (2.0, False, True), (-4.0, True, True)):
            assert (check_scale(rng, words, s, alias, acc) >= 1) == (words > 0)


@pytest.mark.gpu
@pytest.mark.parametrize("ce", CE)
def test_fill_and_quad_fill_match_the_host_hash(need_cuda, ce):
    """k_fill bit for bit against fill_reference, with rank offsets whose high bits are set (rank << 40); k_quad_fill
    against seeded_start_vectors (thermal.py): float64 bit for bit, complex128 phases to 2 ulp."""
    rng = np.random.default_rng(600 + ce)
    for n in lengths("fill", ce):
        words = n * (2 if ce else 1)
        for seed, offset in ((0, 0), (12345, 3 << 40), ((1 << 64) - 1, (0xFFFFFF << 40) & ((1 << 64) - 1))):
            check_fill(words, seed, offset)
        for seed, first, G in ((0, 0, 1), (987654321, 5, 3), ((1 << 64) - 7, 2, 6)):
            check_quad_fill(rng, ce, n, seed, first, G)


# ---- GPU: several tiles per CTA ------------------------------------------------------------------------------------
MULTI_TILE = {   # launcher -> (checker, width R / G of the instance)
    "block_dot": (lambda rng, ce, n: check_block_dot(rng, ce, n, 2), 1),
    "block_combine": (lambda rng, ce, n: check_block_combine(rng, ce, n, 2, 3.0, "alias"), 1),
    "block_gram": (lambda rng, ce, n: check_block_gram(rng, ce, n, 1, 2), 2),
    "block_update": (lambda rng, ce, n: check_block_update(rng, ce, n, 1, 2), 2),
    "block_rotate": (lambda rng, ce, n: check_block_rotate(rng, ce, n, 3, 2), 1),
    "quad_dot": (lambda rng, ce, n: check_quad_dot(rng, ce, n, 2), 2),
    "quad_update": (lambda rng, ce, n: check_quad_update(rng, ce, n, 2, 1), 2),
    "dot": (lambda rng, ce, n: check_dot(rng, ce, n), 1),
    "lanczos_update": (lambda rng, ce, n: check_lanczos_update(rng, ce, n, True), 1),
    "scale": (lambda rng, ce, n: check_scale(rng, n, 3.0, False, True), 1),
    "fill": (lambda rng, ce, n: check_fill(n, 77, 5 << 40), 1),
    "quad_fill": (lambda rng, ce, n: check_quad_fill(rng, ce, n, 31, 1, 2), 1),
}


def multi_tile_length(kernel, ce, width):
    """more than two tiles for every CTA one wave can hold (at most 8 CTAs of 256 threads per SM), and a ragged last
    tile"""
    t = tile(kernel, ce, width)
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return 2 * 8 * sms * t + t // 2 + 3, t


@pytest.mark.gpu
@pytest.mark.parametrize("kernel", sorted(MULTI_TILE))
@pytest.mark.parametrize("ce", CE)
def test_several_tiles_per_cta_exact(need_cuda, ce, kernel):
    """Each launcher at a length where the grid it reports covers at least two tiles per CTA, with a ragged last tile
    (integer data, exact): the grid-stride loops and k_reduce_partials over more than 256 CTAs."""
    if kernel in ("scale", "fill") and ce:
        pytest.skip("word kernels: no element type")
    check, width = MULTI_TILE[kernel]
    n, t = multi_tile_length(kernel, ce, width)
    grid = check(np.random.default_rng(700 + ce), ce, n)
    assert grid >= 1 and -(-n // t) >= 2 * grid and n % t != 0, (n, t, grid)


# ---- GPU: Gaussian data, rounding bounds and repeatability ----------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("ce", CE)
def test_gaussian_data_within_rounding_bounds_and_repeatable(need_cuda, ce):
    """The same launchers on Gaussian data against long-double references within the bounds derived above; every
    partials-based launcher called twice gives bit-identical outputs and vectors."""
    rng = np.random.default_rng(800 + ce)
    for kernel, width in (("block_dot", 1), ("block_gram", 3), ("block_gram", 6), ("quad_dot", 4)):
        t = tile(kernel, ce, width)
        for n in (t + 1, 5 * t + 17, multi_tile_length(kernel, ce, width)[0] if width == 1 else 3 * t):
            if kernel == "block_dot":
                check_block_dot(rng, ce, n, 9, exact=False)
            elif kernel == "block_gram":
                check_block_gram(rng, ce, n, 9, width, exact=False)
            else:
                check_quad_dot(rng, ce, n, width, exact=False)
    for n in (K_THREADS + 1, 7 * K_THREADS + 3):
        check_block_combine(rng, ce, n, 9, 1.0, "alias", exact=False)
        check_block_combine(rng, ce, n, 5, 0.0, "null", exact=False)
        for R in (1, 4, 6):
            check_block_update(rng, ce, n, 9, R, exact=False)
        for G in (1, 5):
            check_quad_update(rng, ce, n, G, 0, exact=False)
            check_quad_update(rng, ce, n, G, 2, exact=False)
        check_dot(rng, ce, n, exact=False)
        check_lanczos_update(rng, ce, n, True, exact=False)
    for n in (K_ROT_WORDS + 1, 9 * K_ROT_WORDS + 5):
        check_block_rotate(rng, ce, n, 12, 7, exact=False)


@pytest.mark.gpu
def test_launchers_reject_bad_shapes(need_cuda):
    """The launchers' own shape checks, reached through the entry: J > 65, R and G outside 1 .. 6, k_block_rotate's
    1 <= l <= k <= 65."""
    big = 4096
    for ce in (False, True):
        rejects("block_dot", ce, 4, [66, 0] + [8] * 66, big, out_words=2 * 67, match="bad number of vectors")
        rejects("block_combine", ce, 4, [66, 0, 0] + [8] * 66, big, coef_words=2 * 66, out_words=2,
                match="bad number of vectors")
        for J, R in ((66, 1), (1, 0), (1, 7)):
            args = [J, R, 0, 4] + [64] * J
            rejects("block_gram", ce, 4, args, big, out_words=2 * (J * 7 + 49), match="bad number of vectors")
            rejects("block_update", ce, 4, args, big, coef_words=2 * J * 7, out_words=14, match="bad number of vectors")
        for k, l in ((66, 1), (2, 0), (2, 3)):
            rejects("block_rotate", ce, 4, [k, l] + [8] * k, big, coef_words=2 * k * max(l, 1), match="bad shape")
        for G in (0, 7):
            rejects("quad_dot", ce, 4, [G, 0, 64], big, out_words=14, match="bad number of vectors")
            rejects("quad_update", ce, 4, [G, 0, 64, 128, 0, 14], big, coef_words=28, out_words=14,
                    match="bad number of vectors")
