"""Entanglement spectra and entropies from the reduced density matrices of Operator.reduced_density_matrix.

Numpy only.  A reduced density matrix comes as {w: ρ_w}: at a fixed Hamming weight the blocks of the weight w of the
sites of A (ascending), at free weight one block under the key None (block_layout gives the layout).
"""
from __future__ import annotations

import math

import numpy as np


def block_layout(n_sites: int, weight, n_a: int):
    """[(w, d_w)] of the blocks of ρ_A for n_a sites of A (dmv_rdm_layout): at weight W the weights w = max(0, W - (N -
    n_a)) ... min(n_a, W) of A with d_w = C(n_a, w); at free weight (weight None or -1) [(None, 2^n_a)]."""
    if not 1 <= n_sites <= 64:
        raise ValueError("n_sites must be between 1 and 64")
    if not 1 <= n_a <= 16:
        raise ValueError(f"n_a must be between 1 and 16 (got {n_a})")
    if n_a > n_sites:
        raise ValueError(f"n_a = {n_a} exceeds the {n_sites} sites")
    if weight is None or weight == -1:
        return [(None, 1 << n_a)]
    if not 0 <= weight <= n_sites:
        raise ValueError(f"weight must be None, -1 or between 0 and {n_sites}")
    return [(w, math.comb(n_a, w)) for w in range(max(0, weight - (n_sites - n_a)), min(n_a, weight) + 1)]


def entanglement_spectrum(blocks):
    """{w: eigenvalues of ρ_w, ascending, clipped at 0} (the entanglement spectrum, resolved by the weight of A)."""
    return {w: np.clip(np.linalg.eigvalsh(np.asarray(rho)), 0.0, None) for w, rho in blocks.items()}


def _probabilities(spectrum) -> np.ndarray:
    p = np.concatenate([np.asarray(v, dtype=float).ravel() for v in spectrum.values()]) \
        if isinstance(spectrum, dict) else np.asarray(spectrum, dtype=float).ravel()
    return p[p > 0.0]


def von_neumann_entropy(spectrum) -> float:
    """S = -Σ p log p (natural logarithm) of a spectrum: a dict of entanglement_spectrum or an array."""
    p = _probabilities(spectrum)
    return float(-(p * np.log(p)).sum())


def renyi_entropy(spectrum, alpha) -> float:
    """S_α = log(Σ p^α) / (1 - α) for α > 0; α = 1 is the von Neumann entropy (the limit α -> 1), α = inf gives
    -log max p, α = 0 the logarithm of the number of non-zero eigenvalues."""
    alpha = float(alpha)
    p = _probabilities(spectrum)
    if alpha < 0.0:
        raise ValueError("alpha must not be negative")
    if alpha == 1.0:
        return von_neumann_entropy(p)
    if alpha == 0.0:
        return float(np.log(p.size))
    if math.isinf(alpha):
        return float(-np.log(p.max()))
    return float(np.log((p ** alpha).sum()) / (1.0 - alpha))
