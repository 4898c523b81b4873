"""Dynamical spin structure factors by Lanczos quadrature (Operator.apply_spin + Operator.lanczos_quadrature): numpy only.

    S^{ab}(q, ω) = Σ_n |<n| S^b_q |0>|² δ(ω - (E_n - E_0))

With y = O|0> (apply_spin: the projection onto one target sector), M Lanczos steps from y give the tridiagonal T_M =
Q diag(θ) Qᵀ and the Gauss quadrature <y|f(H)|y> ≈ Σ_k w_k f(θ_k), w_k = |y|² Q₀ₖ².  For f(H) = (z - H)⁻¹ this is the
M-level continued fraction of <y|(z - H)⁻¹|y>: its poles are the nodes θ_k and its residues the weights w_k.  So
dmv_lanczos_quadrature with start = y already returns the continued fraction in pole form, and no separate continued
fraction is needed; `broaden` turns the poles into a spectrum.  The moments Σ_k w_k ω_k^m are exact for m < 2 M.

Momentum convention.  A translation generator of the model files moves site j + a onto site j ((g.s)[j] = s[j + a],
the permutation [a, a + 1, ..., a - 1] of a chain), and `sector: k` of a generator of period T gives it the character
exp(-2πik/T): a state of sector k has momentum q·a = 2πk/T.  σ_q = Σ_j e^{-i q·r_j} σ_j / √N (fourier_weights) adds q
to the momentum: from sector k_s it reaches sector k_s + k with q·a = 2πk/T.
"""
from __future__ import annotations

import numpy as np


def fourier_weights(coords, q) -> np.ndarray:
    """w_j = exp(-i q·r_j) / √N for site positions coords (N,) or (N, d) and wave vector q (scalar or (d,)); the sign
    matches the sector convention of the module docstring."""
    r = np.asarray(coords, dtype=np.float64)
    if r.ndim == 1:
        r = r[:, None]
    qv = np.atleast_1d(np.asarray(q, dtype=np.float64))
    if qv.shape[0] != r.shape[1]:
        raise ValueError("q and the coordinates must have the same dimension")
    return np.exp(-1j * (r @ qv)) / np.sqrt(r.shape[0])


ZERO_WEIGHT = 1e-20   # |y|² / (|x0|² |w|²) below which a target sector holds nothing of O|0>


def _norm2(v) -> float:
    """|v|² of this rank's block (numpy array or torch tensor)"""
    if hasattr(v, "detach"):
        return float((v.detach().abs() ** 2).sum().item())
    return float(np.vdot(v, v).real)


def dynamical_correlation(source_op, x0, e0: float, target_op, kind: str, weights, steps: int):
    """Poles and residues of S(q, ω) = <0|O† δ(ω - (H - E_0)) O|0> restricted to the target sector:
    y = source_op.apply_spin(kind, weights, x0, target_op), then `steps` Lanczos steps of target_op from y.
    x0: the state |0> in the source basis (numpy or torch CUDA, normalised), e0 its energy.
    -> (poles ω_k = θ_k - e0, residues w_k) as numpy arrays, Σ_k w_k = |y|²; empty arrays when nothing of O|0> lies in
    the target sector: |y|² <= ZERO_WEIGHT |x0|² |w|², where the per-site coefficients of a sector that O|0> does not
    reach cancel to rounding and leave y at about 1e-16 |x0| |w|.  On several ranks (source_op.num_ranks > 1) the two
    norms are summed over the ranks with torch.distributed, so every rank takes the same branch; the process group must
    be the one of the DistributedOperator (NCCL: the sums travel through the operator's device)."""
    y = source_op.apply_spin(kind, weights, x0, target_op)
    w2 = float(np.sum(np.abs(np.asarray(weights, dtype=np.complex128)) ** 2))
    norms = np.array([_norm2(y), _norm2(x0)])
    if source_op.num_ranks > 1:
        import torch
        import torch.distributed as dist
        t = torch.tensor(norms, dtype=torch.float64, device=torch.device("cuda", source_op.device))
        dist.all_reduce(t)
        norms = t.cpu().numpy()
    if norms[0] <= ZERO_WEIGHT * norms[1] * w2:
        return np.zeros(0), np.zeros(0)
    start = y.reshape(1, -1)
    nodes, wts, done, _ = target_op.lanczos_quadrature(1, steps, start=start)
    m = int(done[0])
    return nodes[0, :m] - e0, wts[0, :m]


def broaden(poles, residues, omega, eta: float, shape: str = "lorentzian") -> np.ndarray:
    """S(ω) = Σ_k w_k L(ω - ω_k) on the grid omega with a Lorentzian (half width eta) or a Gaussian (standard deviation
    eta) of unit area, so that ∫ S dω = Σ_k w_k on a grid that covers the poles with room for the tails."""
    p = np.asarray(poles, dtype=np.float64)[None, :]
    w = np.asarray(residues, dtype=np.float64)[None, :]
    om = np.asarray(omega, dtype=np.float64)[:, None]
    if not eta > 0.0:
        raise ValueError("eta must be positive")
    if shape == "lorentzian":
        kern = (eta / np.pi) / ((om - p) ** 2 + eta * eta)
    elif shape == "gaussian":
        kern = np.exp(-0.5 * ((om - p) / eta) ** 2) / (eta * np.sqrt(2.0 * np.pi))
    else:
        raise ValueError("shape must be 'lorentzian' or 'gaussian'")
    return (kern * w).sum(axis=1)
