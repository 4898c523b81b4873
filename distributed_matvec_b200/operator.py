"""Host-side mirror of the reference's operator interface for the hot path.

Names follow the reference (src/ForeignTypes.chpl, src/BatchedOperator.chpl,
src/DistributedMatrixVector.chpl) so that tests read like the reference's own:

    basis, matrix = load_config_from_yaml(path)            # loadConfigFromYaml (FT:261)
    op = Operator(matrix)                                   # one GPU context
    op.basis.build()                                        # Basis.build / enumerateStates
    y = local_matrix_vector(op, x)                          # localMatrixVector (DMV:1055)

Vectors may be numpy arrays (host; copied through the library) or torch CUDA tensors (used in place,
on torch's current stream).  Everything that computes runs in libdmv_b200.so on the GPU.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _native as nat
from .config import SPINFUL_FERMION, SPINLESS_FERMION, BasisSpec, OperatorSpec


def _is_torch(a) -> bool:
    return type(a).__module__.startswith("torch")


def _elt_of(a) -> int:
    if _is_torch(a):
        import torch
        if a.dtype == torch.float64:
            return nat.DMV_F64
        if a.dtype == torch.complex128:
            return nat.DMV_C128
        raise TypeError("vectors must be float64 or complex128")
    if a.dtype == np.float64:
        return nat.DMV_F64
    if a.dtype == np.complex128:
        return nat.DMV_C128
    raise TypeError("vectors must be float64 or complex128")


def _ptr(a) -> int:
    if a is None:
        return None
    if _is_torch(a):
        if not a.is_contiguous():
            raise ValueError("tensors must be contiguous")
        return a.data_ptr()
    if not a.flags["C_CONTIGUOUS"]:
        raise ValueError("arrays must be C-contiguous")
    return a.ctypes.data


class Basis:
    """``Basis`` record of the reference (src/ForeignTypes.chpl:8-117) bound to a GPU context."""

    def __init__(self, spec: BasisSpec, owner: "Operator"):
        self.spec = spec
        self._op = owner

    # flags (src/ForeignTypes.chpl:82-100)
    def isStateIndexIdentity(self): return self.spec.is_state_index_identity()
    def requiresProjection(self): return self.spec.requires_projection()
    def isHammingWeightFixed(self): return self.spec.is_hamming_weight_fixed()
    def hasSpinInversionSymmetry(self): return self.spec.has_spin_inversion_symmetry()
    def hasPermutationSymmetries(self): return self.spec.has_permutation_symmetries()
    def numberSites(self): return self.spec.number_sites
    @property
    def spinInversion(self): return self.spec.spin_inversion
    # particle type (src/ForeignTypes.chpl:79-98)
    def isSpinBasis(self): return not self.spec.is_fermionic()
    def isSpinfulFermionicBasis(self): return self.spec.particle_type == SPINFUL_FERMION
    def isSpinlessFermionicBasis(self): return self.spec.particle_type == SPINLESS_FERMION
    def numberParticles(self): return self.spec.number_particles
    def numberUp(self): return self.spec.number_up

    def build(self):
        """``Basis.build()`` (FT:72): enumerate this rank's representatives on the GPU."""
        nat.check(nat.lib().dmv_basis_build(self._op._ctx))
        return self

    def uncheckedSetRepresentatives(self, representatives, norms=None):
        """``uncheckedSetRepresentatives`` (FT:74-77): install an ascending block owned by this rank."""
        reps = representatives
        if not _is_torch(reps):
            reps = np.ascontiguousarray(reps, dtype=np.uint64)
        if norms is not None and not _is_torch(norms):
            norms = np.ascontiguousarray(norms, dtype=np.float64)
        n = int(reps.shape[0])
        nat.check(nat.lib().dmv_set_representatives(self._op._ctx, _ptr(reps), n, _ptr(norms)))
        return self

    def numberStates(self) -> int:
        n = int(nat.lib().dmv_number_states(self._op._ctx))
        if n < 0:
            raise nat.DmvError("basis is not built")   # FT:113-114
        return n

    def representatives(self) -> np.ndarray:
        n = self.numberStates()
        out = np.zeros(n, dtype=np.uint64)
        nat.check(nat.lib().dmv_get_representatives(self._op._ctx, out.ctypes.data, None))
        return out

    def norms(self) -> np.ndarray:
        n = self.numberStates()
        out = np.zeros(n, dtype=np.float64)
        nat.check(nat.lib().dmv_get_representatives(self._op._ctx, None, out.ctypes.data))
        return out

    def stateIndex(self, spins) -> np.ndarray:
        """``ls_hs_state_index`` (FFI:173-175)."""
        spins = np.ascontiguousarray(spins, dtype=np.uint64)
        out = np.zeros(spins.shape[0], dtype=np.int64)
        nat.check(nat.lib().dmv_state_index(self._op._ctx, spins.shape[0], spins.ctypes.data, out.ctypes.data))
        return out

    def stateInfo(self, alphas):
        """``ls_hs_state_info`` (FFI:181-184): (representatives, characters, norms)."""
        alphas = np.ascontiguousarray(alphas, dtype=np.uint64)
        n = alphas.shape[0]
        betas = np.zeros(n, dtype=np.uint64)
        chars = np.zeros(n, dtype=np.complex128)
        norms = np.zeros(n, dtype=np.float64)
        nat.check(nat.lib().dmv_state_info(self._op._ctx, n, alphas.ctypes.data, betas.ctypes.data,
                                           chars.ctypes.data, norms.ctypes.data))
        return betas, chars, norms


class Operator:
    """``Operator`` record of the reference (src/ForeignTypes.chpl:154-259) + its per-GPU context.

    rank / num_ranks define the hash partition owner(s) = hash64_01(s) % num_ranks
    (src/StatesEnumeration.chpl:122-136)."""

    def __init__(self, spec: OperatorSpec, device: int = 0, rank: int = 0, num_ranks: int = 1):
        self.spec = spec
        self.rank, self.num_ranks, self.device = rank, num_ranks, device
        b = spec.basis
        self._keep = []
        bd = nat.BasisDesc()
        bd.number_sites = b.number_bits
        bd.hamming_weight = -1 if b.hamming_weight is None else b.hamming_weight
        bd.spin_inversion = b.spin_inversion
        bd.has_permutations = int(b.has_permutation_symmetries())
        if b.has_permutation_symmetries():
            g = b.group
            perms = np.ascontiguousarray(g.perms, dtype=np.int32)
            flips = np.ascontiguousarray(g.flips, dtype=np.uint8)
            chars = np.ascontiguousarray(g.characters, dtype=np.complex128)
            self._keep += [perms, flips, chars]
            bd.group_order = len(g)
            bd.perms, bd.flips, bd.characters = perms.ctypes.data, flips.ctypes.data, chars.ctypes.data
        else:
            bd.group_order = 0
        od = nat.OperatorDesc()
        off, diag = spec.off_diag, spec.diag
        arrs = [np.ascontiguousarray(a) for a in (off.v, off.m, off.r, off.x, off.s, diag.v, diag.m, diag.r, diag.s)]
        self._keep += arrs
        od.n_off = len(off)
        od.off_v, od.off_m, od.off_r, od.off_x, od.off_s = (a.ctypes.data for a in arrs[:5])
        od.n_diag = len(diag)
        od.diag_v, od.diag_m, od.diag_r, od.diag_s = (a.ctypes.data for a in arrs[5:])
        pd = nat.ParticlesDesc()
        pd.particle_type = {SPINLESS_FERMION: nat.DMV_SPINLESS_FERMION,
                            SPINFUL_FERMION: nat.DMV_SPINFUL_FERMION}.get(b.particle_type, nat.DMV_SPIN)
        pd.number_particles = -1 if b.number_particles is None else b.number_particles
        pd.number_up = -1 if b.number_up is None else b.number_up
        handle = C.c_void_p()
        nat.check(nat.lib().dmv_context_create_particles(C.byref(bd), C.byref(pd), C.byref(od), device, rank, num_ranks,
                                                         C.byref(handle)))
        self._ctx = handle
        self.basis = Basis(b, self)

    def close(self):
        if getattr(self, "_ctx", None):
            nat.lib().dmv_context_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- reference accessors ---------------------------------------------------------------------
    def numberDiagTerms(self) -> int: return self.spec.number_diag_terms()          # FT:222
    def numberOffDiagTerms(self) -> int:                                             # FT:228
        return int(nat.lib().dmv_max_number_off_diag(self._ctx))
    def numberTerms(self) -> int:
        """emitted off-diagonal terms of this rank in one product (from the last plan)"""
        return int(nat.lib().dmv_number_terms(self._ctx))

    # -- block <-> hashed redistribution (arrFromBlockToHashed / arrFromHashedToBlock) ----------------------
    def hashed_positions(self, masks: np.ndarray, num_ranks: int):
        """-> (counts[num_ranks], positions): slot of every chunk element in "grouped by owner, stable" order."""
        masks = np.ascontiguousarray(masks, dtype=np.uint8)
        counts = np.zeros(num_ranks, dtype=np.int64)
        pos = np.zeros(masks.shape[0], dtype=np.uint32)
        nat.check(nat.lib().dmv_hashed_positions(self._ctx, masks.shape[0], masks.ctypes.data, num_ranks,
                                                 counts.ctypes.data, pos.ctypes.data))
        return counts, pos

    def permute(self, arr: np.ndarray, positions: np.ndarray, gather: bool) -> np.ndarray:
        arr = np.ascontiguousarray(arr)
        assert arr.dtype.itemsize in (8, 16)
        out = np.zeros_like(arr)
        positions = np.ascontiguousarray(positions, dtype=np.uint32)
        nat.check(nat.lib().dmv_permute(self._ctx, arr.dtype.itemsize // 8, arr.shape[0], positions.ctypes.data,
                                        arr.ctypes.data, out.ctypes.data, 1 if gather else 0))
        return out

    def block_to_hashed(self, block_chunk, masks_chunk: np.ndarray, hashed_count: int | None = None):
        """arrFromBlockToHashed (src/BlockToHashed.chpl:87): this rank's chunk of a vector in sorted-state order ->
        this rank's hashed block.  Collective when num_ranks > 1.  numpy or torch CUDA arrays."""
        masks_chunk = np.ascontiguousarray(masks_chunk, dtype=np.uint8)
        n_out = self.basis.numberStates() if hashed_count is None else hashed_count
        if _is_torch(block_chunk):
            import torch
            self.use_torch_stream()
            out = torch.zeros(n_out, dtype=block_chunk.dtype, device=block_chunk.device)
            itemsize = block_chunk.element_size()
        else:
            block_chunk = np.ascontiguousarray(block_chunk)
            out = np.zeros(n_out, dtype=block_chunk.dtype)
            itemsize = block_chunk.dtype.itemsize
        nat.check(nat.lib().dmv_block_to_hashed(self._ctx, itemsize // 8, masks_chunk.shape[0], masks_chunk.ctypes.data,
                                                _ptr(block_chunk), _ptr(out), n_out))
        return out

    def hashed_to_block(self, hashed, masks_chunk: np.ndarray):
        """arrFromHashedToBlock (src/HashedToBlock.chpl:67): inverse of block_to_hashed."""
        masks_chunk = np.ascontiguousarray(masks_chunk, dtype=np.uint8)
        n_out = masks_chunk.shape[0]
        if _is_torch(hashed):
            import torch
            self.use_torch_stream()
            out = torch.zeros(n_out, dtype=hashed.dtype, device=hashed.device)
            itemsize = hashed.element_size()
        else:
            hashed = np.ascontiguousarray(hashed)
            out = np.zeros(n_out, dtype=hashed.dtype)
            itemsize = hashed.dtype.itemsize
        nat.check(nat.lib().dmv_hashed_to_block(self._ctx, itemsize // 8, n_out, masks_chunk.ctypes.data, _ptr(hashed),
                                                int(hashed.shape[0]), _ptr(out)))
        return out

    def set_option(self, name: str, value: int):
        """dmv_set_option: the options and their values are listed in include/dmv_b200.h."""
        nat.check(nat.lib().dmv_set_option(self._ctx, name.encode(), int(value)))
        return self

    def debug_rows_store(self, mode: int, chunks: int = 0):
        """dmv_debug_rows_store: the term store of the row kernel -1 auto, 0 never, 1 whenever it can be built; chunks
        0 the cost model's column blocks, else 1 .. 64."""
        nat.check(nat.lib().dmv_debug_rows_store(self._ctx, int(mode), int(chunks)))
        return self

    def info(self, name: str) -> int:
        return int(nat.lib().dmv_get_info(self._ctx, name.encode()))

    # -- streams ---------------------------------------------------------------------------------
    def use_torch_stream(self):
        """Launch on torch's current stream (so torch tensors and CUDA events order correctly)."""
        import torch
        handle = torch.cuda.current_stream(self.device).cuda_stream
        if getattr(self, "_stream_handle", -1) != handle:
            nat.check(nat.lib().dmv_set_stream(self._ctx, C.c_void_p(handle), 0))
            self._stream_handle = handle

    def synchronize(self):
        nat.check(nat.lib().dmv_synchronize(self._ctx))

    # -- hot path ----------------------------------------------------------------------------------
    def _check_vec(self, a, name):
        n = self.basis.numberStates()
        if int(a.shape[0]) != n or a.ndim != 1:
            raise ValueError(f"{name} must have shape ({n},)")

    def matvec(self, x, y=None):
        """``localMatrixVector`` (num_ranks == 1) / ``matrixVectorProduct`` (collective)."""
        elt = _elt_of(x)
        self._check_vec(x, "x")
        if _is_torch(x):
            self.use_torch_stream()
        if y is None:
            if _is_torch(x):
                import torch
                y = torch.zeros_like(x)
            else:
                y = np.zeros_like(x)     # `similar(x)`: test/TestMatrixVectorProduct.chpl:37
        else:
            self._check_vec(y, "y")
            if _elt_of(y) != elt:
                raise TypeError("x and y must have the same element type")
        fn = nat.lib().dmv_local_matvec if self.num_ranks == 1 else nat.lib().dmv_matvec
        nat.check(fn(self._ctx, elt, _ptr(x), _ptr(y)))
        return y

    def matvec_batch(self, X, Y=None):
        """Several vectors per call: X, Y of shape (num_vectors, number_states), C-contiguous (dmv_matvec_batch)."""
        assert X.ndim == 2 and int(X.shape[1]) == self.basis.numberStates()
        if _is_torch(X):
            import torch
            self.use_torch_stream()
            X = X.contiguous()
            Y = torch.zeros_like(X) if Y is None else Y
        else:
            X = np.ascontiguousarray(X)
            Y = np.zeros_like(X) if Y is None else Y
        nat.check(nat.lib().dmv_matvec_batch(self._ctx, _elt_of(X), int(X.shape[0]), _ptr(X), _ptr(Y)))
        if not _is_torch(X):
            self.synchronize()
        return Y

    def lanczos(self, max_iters: int = 300, tol: float = 1e-10, seed: int = 42, complex_vectors: bool = False,
                eigenvector: bool = True):
        """Lowest eigenpair by Lanczos on the device (dmv_lanczos): -> (energy, vector or None, iterations, residual)."""
        elt = nat.DMV_C128 if complex_vectors else nat.DMV_F64
        n = self.basis.numberStates()
        vec = np.zeros(n, dtype=np.complex128 if complex_vectors else np.float64) if eigenvector else None
        e, it, res = C.c_double(), C.c_int(), C.c_double()
        nat.check(nat.lib().dmv_lanczos(self._ctx, elt, max_iters, tol, seed, C.byref(e),
                                        vec.ctypes.data if eigenvector else None, C.byref(it), C.byref(res)))
        return float(e.value), vec, int(it.value), float(res.value)

    def expm_multiply(self, x, z, krylov_dim: int = 0, tol: float = 1e-10):
        """y = exp(z H) x on the device (dmv_expm_multiply): real time is z = -1j * t, imaginary time z = -tau.
        x: numpy array or torch CUDA tensor (float64 only for a real z and a real operator); y has the same kind.
        Collective when num_ranks > 1.  -> (y, products of H applied, sum of the local error estimates)"""
        elt = _elt_of(x)
        self._check_vec(x, "x")
        z = complex(z)
        if _is_torch(x):
            import torch
            self.use_torch_stream()
            y = torch.empty_like(x)
        else:
            y = np.empty_like(x)
        prods, err = C.c_int(), C.c_double()
        nat.check(nat.lib().dmv_expm_multiply(self._ctx, elt, z.real, z.imag, _ptr(x), _ptr(y), int(krylov_dim),
                                              float(tol), C.byref(prods), C.byref(err)))
        return y, int(prods.value), float(err.value)

    def eigsh(self, k, block_size: int = 0, krylov_dim: int = 0, tol: float = 1e-10, max_restarts: int = 1000,
              seed: int = 42, complex_vectors: bool = False, eigenvectors=True):
        """The k lowest eigenpairs by block Krylov-Schur on the device (dmv_eigsh).  eigenvectors: True -> a numpy array
        (k, n); False -> none; or a C-contiguous torch CUDA tensor (k, n) of the vector type, filled in place on torch's
        current stream.  Collective when num_ranks > 1.
        -> (eigenvalues[k], vectors or None, residuals[k], converged, products, restarts)"""
        elt = nat.DMV_C128 if complex_vectors else nat.DMV_F64
        n = self.basis.numberStates()
        k = int(k)
        vec, ptr = None, None
        if _is_torch(eigenvectors):
            import torch
            want = torch.complex128 if complex_vectors else torch.float64
            if (tuple(eigenvectors.shape) != (k, n) or eigenvectors.dtype != want or not eigenvectors.is_cuda
                    or not eigenvectors.is_contiguous()):
                raise ValueError(f"eigenvectors must be a C-contiguous CUDA tensor of shape ({k}, {n}) and dtype {want}")
            self.use_torch_stream()
            vec, ptr = eigenvectors, _ptr(eigenvectors)
        elif eigenvectors is True:
            vec = np.zeros((max(k, 0), n), dtype=np.complex128 if complex_vectors else np.float64)
            ptr = vec.ctypes.data
        elif eigenvectors is not False and eigenvectors is not None:
            raise TypeError("eigenvectors must be True, False or a torch CUDA tensor")
        evals, res = np.zeros(max(k, 1)), np.zeros(max(k, 1))
        conv, prods, rst = C.c_int(), C.c_int(), C.c_int()
        nat.check(nat.lib().dmv_eigsh(self._ctx, elt, k, int(block_size), int(krylov_dim), float(tol),
                                      int(max_restarts), int(seed), evals.ctypes.data, ptr, res.ctypes.data,
                                      C.byref(conv), C.byref(prods), C.byref(rst)))
        return evals[:k], vec, res[:k], int(conv.value), int(prods.value), int(rst.value)

    def zz_correlations(self, x):
        """Spin-spin correlations C[i, j] = <x|σᶻᵢσᶻⱼ|x> / <x|x> and magnetisation m[i] = <x|σᶻᵢ> / <x|x> on the device
        (dmv_zz_correlations), with σᶻ = +1 on a set bit.  x: shape (n,) or (k, n), float64 or complex128, a numpy
        array or a torch CUDA tensor (used in place on torch's current stream).  Collective when num_ranks > 1.
        On a fermionic basis i, j run over the bits (modes) and σᶻᵢ = 2nᵢ - 1.
        -> numpy (C, m) of shapes (N, N), (N,), or (k, N, N), (k, N) for a batch, N the number of bits."""
        elt = _elt_of(x)
        n, N = self.basis.numberStates(), self.spec.basis.number_bits
        if x.ndim not in (1, 2) or int(x.shape[-1]) != n:
            raise ValueError(f"x must have shape ({n},) or (k, {n})")
        k = 1 if x.ndim == 1 else int(x.shape[0])
        if _is_torch(x):
            self.use_torch_stream()
        else:
            x = np.ascontiguousarray(x)
        C_out, m_out = np.zeros((k, N, N)), np.zeros((k, N))
        nat.check(nat.lib().dmv_zz_correlations(self._ctx, elt, k, _ptr(x), C_out.ctypes.data, m_out.ctypes.data))
        return (C_out[0], m_out[0]) if x.ndim == 1 else (C_out, m_out)

    def pm_correlations(self, x):
        """Flip-flop correlations T[i, j] = <x|σ⁺ᵢσ⁻ⱼ|x> / <x|x> on the device (dmv_pm_correlations), with σ⁺ turning a
        0 bit into a 1 bit.  x as for zz_correlations.  -> numpy complex128 of shape (N, N), or (k, N, N) for a batch."""
        elt = _elt_of(x)
        n, N = self.basis.numberStates(), self.spec.basis.number_bits
        if x.ndim not in (1, 2) or int(x.shape[-1]) != n:
            raise ValueError(f"x must have shape ({n},) or (k, {n})")
        k = 1 if x.ndim == 1 else int(x.shape[0])
        if _is_torch(x):
            self.use_torch_stream()
        else:
            x = np.ascontiguousarray(x)
        out = np.zeros((k, N, N), dtype=np.complex128)
        nat.check(nat.lib().dmv_pm_correlations(self._ctx, elt, k, _ptr(x), out.ctypes.data))
        return out[0] if x.ndim == 1 else out

    def spin_correlations(self, x):
        """<σᵢ·σⱼ> = <σᶻᵢσᶻⱼ> + 4 Re <σ⁺ᵢσ⁻ⱼ> (3 on the diagonal) and the total spin <S²> = ¼ Σᵢⱼ <σᵢ·σⱼ>, from
        zz_correlations and pm_correlations.  -> numpy (S [N, N], S2 float), or (S [k, N, N], S2 [k]) for a batch."""
        Cz, _ = self.zz_correlations(x)
        T = self.pm_correlations(x)
        S = Cz + 4.0 * T.real
        N = S.shape[-1]
        S[..., np.arange(N), np.arange(N)] = 3.0
        S2 = 0.25 * S.sum(axis=(-2, -1))
        return (S, float(S2)) if S.ndim == 2 else (S, S2)

    _SPIN_KINDS = {"1": 0, "z": 1, "+": 2, "-": 3}

    def apply_spin(self, kind: str, weights, x, target: "Operator"):
        """y = B_targetᴴ O B_this x with O = sum_j weights[j] o_j, o_j = 1, σᶻ_j, σ⁺_j or σ⁻_j for kind "1", "z", "+",
        "-" (dmv_apply_spin): the projection of O psi onto the target's sector.  `target` is another Operator on the
        same device and sites whose group is a subgroup of this one's (a target without symmetries unfolds x into the
        plain basis).  x: shape (n,) or (k, n), float64 (real weights and characters only) or complex128, a numpy array
        or a torch CUDA tensor (then y is a torch tensor on torch's current stream).  Collective when num_ranks > 1.
        -> y of shape (n_target,) or (k, n_target), of x's kind and type."""
        if kind not in self._SPIN_KINDS:
            raise ValueError(f"kind must be one of {sorted(self._SPIN_KINDS)}, got {kind!r}")
        elt = _elt_of(x)
        n, N = self.basis.numberStates(), self.spec.basis.number_bits
        if x.ndim not in (1, 2) or int(x.shape[-1]) != n:
            raise ValueError(f"x must have shape ({n},) or (k, {n})")
        w = np.ascontiguousarray(np.asarray(weights, dtype=np.complex128).reshape(-1))
        if w.shape[0] != N:
            raise ValueError(f"weights must have {N} entries")
        k = 1 if x.ndim == 1 else int(x.shape[0])
        m = target.basis.numberStates()
        shape = (m,) if x.ndim == 1 else (k, m)
        if _is_torch(x):
            import torch
            if not x.is_cuda:
                raise ValueError("a torch x must be a CUDA tensor")
            self.use_torch_stream()
            target.use_torch_stream()
            x = x.contiguous()
            y = torch.empty(shape, dtype=x.dtype, device=x.device)
        else:
            x = np.ascontiguousarray(x)
            y = np.empty(shape, dtype=x.dtype)
        nat.check(nat.lib().dmv_apply_spin(target._ctx, self._ctx, elt, self._SPIN_KINDS[kind], w.ctypes.data, k,
                                           _ptr(x), _ptr(y)))
        return y

    def one_body_density_matrix(self, x):
        """The one-body density matrix G[i, j] = <x|c†ᵢ cⱼ|x> / <x|x> of a fermionic basis on the device
        (dmv_one_body_density_matrix), i, j over the modes (spinful: site, then site + N for down).  A spinful basis
        fixes number_up, so its cross-spin block is exactly 0.  x as for zz_correlations.
        -> numpy complex128 of shape (M, M), or (k, M, M) for a batch, M the number of modes."""
        elt = _elt_of(x)
        n, M = self.basis.numberStates(), self.spec.basis.number_bits
        if x.ndim not in (1, 2) or int(x.shape[-1]) != n:
            raise ValueError(f"x must have shape ({n},) or (k, {n})")
        k = 1 if x.ndim == 1 else int(x.shape[0])
        if _is_torch(x):
            self.use_torch_stream()
        else:
            x = np.ascontiguousarray(x)
        out = np.zeros((k, M, M), dtype=np.complex128)
        nat.check(nat.lib().dmv_one_body_density_matrix(self._ctx, elt, k, _ptr(x), out.ctypes.data))
        return out[0] if x.ndim == 1 else out

    _FERMION_KINDS = {"c+": 0, "c†": 0, "c": 1}

    def apply_fermion(self, kind: str, weights, x, target: "Operator"):
        """y = O x with O = sum_j weights[j] c†_j (kind "c+" or "c†") or sum_j weights[j] c_j (kind "c") on the device
        (dmv_apply_fermion), from this fermionic basis into `target`'s particle sector (one particle more for c†, one
        fewer for c; on a spinful basis the non-zero weights lie in one spin half, whose count changes).  x, weights
        and y as for apply_spin, with one weight per mode.  Collective when num_ranks > 1.
        -> y of shape (n_target,) or (k, n_target), of x's kind and type."""
        if kind not in self._FERMION_KINDS:
            raise ValueError(f"kind must be one of {sorted(self._FERMION_KINDS)}, got {kind!r}")
        elt = _elt_of(x)
        n, M = self.basis.numberStates(), self.spec.basis.number_bits
        if x.ndim not in (1, 2) or int(x.shape[-1]) != n:
            raise ValueError(f"x must have shape ({n},) or (k, {n})")
        w = np.ascontiguousarray(np.asarray(weights, dtype=np.complex128).reshape(-1))
        if w.shape[0] != M:
            raise ValueError(f"weights must have {M} entries")
        k = 1 if x.ndim == 1 else int(x.shape[0])
        m = target.basis.numberStates()
        shape = (m,) if x.ndim == 1 else (k, m)
        if _is_torch(x):
            import torch
            if not x.is_cuda:
                raise ValueError("a torch x must be a CUDA tensor")
            self.use_torch_stream()
            target.use_torch_stream()
            x = x.contiguous()
            y = torch.empty(shape, dtype=x.dtype, device=x.device)
        else:
            x = np.ascontiguousarray(x)
            y = np.empty(shape, dtype=x.dtype)
        nat.check(nat.lib().dmv_apply_fermion(target._ctx, self._ctx, elt, self._FERMION_KINDS[kind], w.ctypes.data, k,
                                              _ptr(x), _ptr(y)))
        return y

    def reduced_density_matrix(self, x, sites):
        """ρ_A = Tr_B |ψ><ψ| of ψ = B x / ‖x‖ for the sites A = `sites` (1 to 16 distinct sites; bit k of a row of ρ_A is
        site sites[k]) on the device (dmv_reduced_density_matrix).  x as for zz_correlations.  Collective when
        num_ranks > 1.  -> {w: complex128 ndarray (d_w, d_w)} by the weight w of A (key None at free weight; see
        entanglement.block_layout), or a list of such dicts for a batch."""
        from .entanglement import block_layout
        elt = _elt_of(x)
        n, N = self.basis.numberStates(), self.spec.basis.number_bits
        if x.ndim not in (1, 2) or int(x.shape[-1]) != n:
            raise ValueError(f"x must have shape ({n},) or (k, {n})")
        sites_a = np.ascontiguousarray(np.asarray(sites, dtype=np.int32).reshape(-1))
        layout = block_layout(N, self.spec.basis.hamming_weight, int(sites_a.shape[0]))
        k = 1 if x.ndim == 1 else int(x.shape[0])
        if _is_torch(x):
            self.use_torch_stream()
            x = x.contiguous()
        else:
            x = np.ascontiguousarray(x)
        out = np.zeros((k, sum(d * d for _, d in layout)), dtype=np.complex128)
        nat.check(nat.lib().dmv_reduced_density_matrix(self._ctx, elt, k, _ptr(x), int(sites_a.shape[0]),
                                                       sites_a.ctypes.data, out.ctypes.data))
        result = []
        for v in range(k):
            blocks, off = {}, 0
            for w, d in layout:
                blocks[w] = out[v, off:off + d * d].reshape(d, d)
                off += d * d
            result.append(blocks)
        return result[0] if x.ndim == 1 else result

    def entanglement_entropy(self, x, sites, alpha=1):
        """The Rényi entropy S_α(A) (α = 1: von Neumann, natural logarithm) of ψ = B x / ‖x‖ for the sites A, from
        reduced_density_matrix and entanglement.renyi_entropy.  When A has more sites than its complement B, ρ_B is
        computed instead: for a pure state ρ_A and ρ_B have the same non-zero spectrum, so S(A) = S(B).  -> float, or
        an ndarray for a batch."""
        from .entanglement import entanglement_spectrum, renyi_entropy
        N = self.spec.basis.number_bits
        sites = [int(s) for s in np.asarray(sites).reshape(-1)]
        rest = [s for s in range(N) if s not in set(sites)]
        if 0 < len(rest) < len(sites):
            sites = rest
        rho = self.reduced_density_matrix(x, sites)
        if isinstance(rho, dict):
            return renyi_entropy(entanglement_spectrum(rho), alpha)
        return np.array([renyi_entropy(entanglement_spectrum(r), alpha) for r in rho])

    def lanczos_quadrature(self, num_vectors: int, steps: int, seed: int = 42, start=None,
                           complex_vectors: bool = False):
        """Finite-temperature Lanczos (stochastic Lanczos quadrature) on the device (dmv_lanczos_quadrature): for each
        start vector r, `steps` Lanczos steps give Gauss nodes and weights with <r|f(H)|r> ~ sum_k w_k f(theta_k).
        start: None for the seeded vectors of `seed` (distributed_matvec_b200.thermal.seeded_start_vectors mirrors them),
        else a numpy array or a torch CUDA tensor of shape (num_vectors, n), float64 or complex128 (then
        complex_vectors follows its type).  Collective when num_ranks > 1.
        -> numpy (nodes [R, steps], weights [R, steps], steps_done [R], products); slots past steps_done hold zeros."""
        R, M = int(num_vectors), int(steps)
        n = self.basis.numberStates()
        ptr = None
        if start is not None:
            if _is_torch(start):
                if not start.is_cuda:
                    raise ValueError("a torch start must be a CUDA tensor")
                self.use_torch_stream()
                start = start.contiguous()
            else:
                start = np.ascontiguousarray(start)
            complex_vectors = _elt_of(start) == nat.DMV_C128
            if tuple(start.shape) != (R, n):
                raise ValueError(f"start must have shape ({R}, {n})")
            ptr = _ptr(start)
        elt = nat.DMV_C128 if complex_vectors else nat.DMV_F64
        nodes, weights = np.zeros((max(R, 1), max(M, 1))), np.zeros((max(R, 1), max(M, 1)))
        done, prods = np.zeros(max(R, 1), dtype=np.int32), C.c_int()
        nat.check(nat.lib().dmv_lanczos_quadrature(self._ctx, elt, R, M, int(seed), ptr, nodes.ctypes.data,
                                                   weights.ctypes.data, done.ctypes.data, C.byref(prods)))
        return nodes, weights, done.astype(np.int64), int(prods.value)

    # -- replicated-x form of the distributed product (dmv_replicated_*), for hosts that own the all-gather -------
    def replicated_setup(self) -> int:
        """Build the whole basis and the slot table on this rank; returns the slot size (elements per rank)."""
        nat.check(nat.lib().dmv_replicated_setup(self._ctx))
        return self.info("replicated_block")

    def replicated_block(self) -> int:
        return self.info("replicated_block")

    def replicated_rows(self, x_cat, y):
        """y <- this rank's rows of H applied to the gathered x (torch CUDA tensors)."""
        self.use_torch_stream()
        nat.check(nat.lib().dmv_replicated_product(self._ctx, _elt_of(y), _ptr(x_cat), _ptr(y)))
        return y

    def plan(self) -> np.ndarray:
        counts = np.zeros(self.num_ranks, dtype=np.int64)
        nat.check(nat.lib().dmv_plan(self._ctx, counts.ctypes.data))
        return counts

    def generate(self, x, y):
        if _is_torch(x):
            self.use_torch_stream()
        nat.check(nat.lib().dmv_generate(self._ctx, _elt_of(x), _ptr(x), _ptr(y)))

    def outgoing(self, dest: int):
        b, c, n = C.c_void_p(), C.c_void_p(), C.c_int64()
        nat.check(nat.lib().dmv_outgoing(self._ctx, dest, C.byref(b), C.byref(c), C.byref(n)))
        return b.value, c.value, int(n.value)

    def accumulate(self, elt: int, count: int, betas_ptr, coeffs_ptr, y):
        nat.check(nat.lib().dmv_accumulate(self._ctx, elt, count, C.c_void_p(betas_ptr), C.c_void_p(coeffs_ptr), _ptr(y)))

    # -- tensor views for hosts that own the exchange (HostExchangedProduct) ----------------------
    def record_width(self, x) -> int:
        """doubles per coefficient of the records generated for vectors like x: 2 for complex vectors or when a
        coefficient / character has a non-zero imaginary part (the library's own rule, dmv_get_info), else 1"""
        return 2 if (_elt_of(x) == nat.DMV_C128 or self.info("complex_coefficients") == 1) else 1

    def outgoing_tensors(self, width: int):
        """(betas int64, coeffs float64) torch views of all outgoing buckets, concatenated by destination."""
        import torch
        first = None
        total = 0
        for q in range(self.num_ranks):
            b, c, n = self.outgoing(q)
            if q != self.rank:
                if first is None:
                    first = (b, c)
                total += n
        if total == 0:
            dev = torch.device("cuda", self.device)
            return torch.empty(0, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.float64, device=dev)
        betas = _device_tensor(first[0], total, torch.int64, self.device)
        coeffs = _device_tensor(first[1], total * width, torch.float64, self.device)
        return betas, coeffs

    def accumulate_tensors(self, x, betas, coeffs, y):
        if betas.numel() > 0:
            self.accumulate(_elt_of(x), int(betas.numel()), betas.data_ptr(), coeffs.data_ptr(), y)

    def timings(self) -> dict:
        buf = (C.c_double * 8)()
        n = nat.lib().dmv_last_timings(self._ctx, buf, 8)
        return {nat.lib().dmv_timing_name(i).decode(): buf[i] for i in range(n)}


def _device_tensor(ptr: int, count: int, dtype, device: int):
    """Zero-copy torch view of library-owned device memory (valid until the next generate)."""
    import torch
    itemsize = torch.empty(0, dtype=dtype).element_size()

    class _Holder:
        __cuda_array_interface__ = {"shape": (count,), "typestr": "<i8" if dtype == torch.int64 else "<f8",
                                    "data": (ptr, False), "version": 2, "strides": (itemsize,)}
    return torch.as_tensor(_Holder(), device=torch.device("cuda", device))


class BatchedOperator:
    """``BatchedOperator`` (src/BatchedOperator.chpl:40-213)."""

    def __init__(self, matrix: Operator, batchSize: int):
        self.matrix, self.batchSize = matrix, batchSize

    def computeOffDiag(self, count: int, alphas, xs):
        """-> (n, betas, coeffs, keys); entry order unspecified (see include/dmv_b200.h)."""
        assert count <= self.batchSize                                           # BO:87
        alphas = np.ascontiguousarray(alphas[:count], dtype=np.uint64)
        xs = np.ascontiguousarray(xs[:count])
        elt = _elt_of(xs)
        cap = max(1, count * max(1, self.matrix.numberOffDiagTerms()))
        betas = np.zeros(cap, dtype=np.uint64)
        coeffs = np.zeros(cap, dtype=np.complex128)
        keys = np.zeros(cap, dtype=np.uint8)
        n = C.c_int64()
        nat.check(nat.lib().dmv_compute_off_diag(self.matrix._ctx, count, alphas.ctypes.data, xs.ctypes.data, elt,
                                                 C.byref(n), betas.ctypes.data, coeffs.ctypes.data, keys.ctypes.data))
        n = int(n.value)
        return n, betas[:n], coeffs[:n], keys[:n]


def _take(arr, ctype, dtype):
    """Copy a callee-allocated chpl_external_array out and release it through its freer (BO:232 contract)."""
    n = int(arr.num_elts)
    if n == 0 or not arr.elts:
        return np.zeros(0, dtype=dtype)
    out = np.ctypeslib.as_array(C.cast(arr.elts, C.POINTER(ctype)), shape=(n,)).copy()
    if arr.freer:
        arr.freer(arr.elts)
    return out.view(dtype) if dtype is not None and out.dtype != np.dtype(dtype) else out


class ChapelKernels:
    """The reference's plugin table ``ls_chpl_kernels`` (src/FFI.chpl:233-239) on top of one Operator: the four
    entry points take the opaque ``ls_hs_operator*`` / ``ls_hs_basis*`` handle, which is bound to the context
    with dmv_bind_operator (any unique address works as the handle here)."""

    def __init__(self, matrix: Operator):
        self.matrix = matrix
        self._handle = C.c_void_p(id(self))          # stands in for the ls_hs_operator* / ls_hs_basis*
        nat.check(nat.lib().dmv_bind_operator(self._handle, matrix._ctx))

    def close(self):
        nat.lib().dmv_bind_operator(self._handle, None)

    def operator_apply_diag(self, alphas, num_tasks: int = 1) -> np.ndarray:
        """ls_chpl_operator_apply_diag (BO:217-234)."""
        alphas = np.ascontiguousarray(alphas, dtype=np.uint64)
        out = nat.ExternalArray()
        nat.lib().ls_chpl_operator_apply_diag(self._handle, alphas.shape[0], alphas.ctypes.data, C.byref(out), num_tasks)
        return _take(out, C.c_double, np.float64)

    def operator_apply_off_diag(self, alphas, num_tasks: int = 1):
        """ls_chpl_operator_apply_off_diag (BO:236-275) -> (betas, coeffs, offsets); entries [0, offsets[-1]) used."""
        alphas = np.ascontiguousarray(alphas, dtype=np.uint64)
        b, c, o = nat.ExternalArray(), nat.ExternalArray(), nat.ExternalArray()
        nat.lib().ls_chpl_operator_apply_off_diag(self._handle, alphas.shape[0], alphas.ctypes.data, C.byref(b),
                                                  C.byref(c), C.byref(o), num_tasks)
        offsets = _take(o, C.c_int64, np.int64)
        betas = _take(b, C.c_uint64, np.uint64)
        coeffs = _take(c, C.c_double, np.float64).view(np.complex128)
        return betas, coeffs, offsets

    def enumerate_representatives(self, lower: int = 0, upper: int = 2**64 - 1) -> np.ndarray:
        """ls_chpl_enumerate_representatives (SE:588-603)."""
        out = nat.ExternalArray()
        nat.lib().ls_chpl_enumerate_representatives(self._handle, lower, upper, C.byref(out))
        return _take(out, C.c_uint64, np.uint64)

    def primme_matvec(self, X: np.ndarray, ldy: int | None = None) -> np.ndarray:
        """ls_chpl_primme_matvec (src/Diagonalize.chpl:134-162): X is column-major [ldx, blockSize] as PRIMME hands it
        over, i.e. a C-contiguous array of shape (blockSize, ldx) here; returns Y of shape (blockSize, ldy)."""
        X = np.ascontiguousarray(X, dtype=np.float64)
        block, ldx = X.shape
        ldy = ldx if ldy is None else ldy
        Y = np.zeros((block, ldy), dtype=np.float64)
        ierr = C.c_int(-1)
        nat.lib().ls_chpl_primme_matvec(X.ctypes.data, C.byref(C.c_int64(ldx)), Y.ctypes.data, C.byref(C.c_int64(ldy)),
                                        C.byref(C.c_int(block)), self._handle, C.byref(ierr))
        assert ierr.value == 0
        return Y

    def matrix_vector_product(self, x: np.ndarray) -> np.ndarray:
        """ls_chpl_matrix_vector_product (DMV:1095-1110): real(64), one vector."""
        x = np.ascontiguousarray(x, dtype=np.float64)
        y = np.zeros_like(x)
        nat.lib().ls_chpl_matrix_vector_product(self._handle, 1, x.ctypes.data, y.ctypes.data)
        return y


def local_matrix_vector(matrix: Operator, x, y=None):
    """``localMatrixVector(matrix, x, y, representatives)`` (DMV:1055-1070)."""
    return matrix.matvec(x, y)


def locale_idx_of(matrix: Operator, states, num_locales: int) -> np.ndarray:
    """``localeIdxOf`` (src/StatesEnumeration.chpl:129-136) evaluated on the GPU."""
    states = np.ascontiguousarray(states, dtype=np.uint64)
    keys = np.zeros(states.shape[0], dtype=np.uint8)
    nat.check(nat.lib().dmv_locale_idx_of(matrix._ctx, states.shape[0], states.ctypes.data, num_locales,
                                          keys.ctypes.data))
    return keys
