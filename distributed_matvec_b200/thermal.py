"""Thermodynamics from the finite-temperature Lanczos method (Operator.lanczos_quadrature): numpy only.

For each symmetry sector, R start vectors r and M Lanczos steps give Gauss nodes theta_rk and weights w_rk with
Tr_sector f(H) ~ (1/R) sum_r sum_k w_rk f(theta_rk).  `thermodynamics` sums such estimates over sectors and returns
log Z, E, C and S per temperature (k_B = 1, energies in the unit of the Hamiltonian); `seeded_start_vectors` rebuilds on
the host the start vectors the library draws from a seed (include/dmv_b200.h, dmv_lanczos_quadrature).
"""
from __future__ import annotations

import numpy as np

_MASK = (1 << 64) - 1
_GOLDEN = 0x9E3779B97F4A7C15


def _hash64_01_int(x: int) -> int:
    x &= _MASK
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _MASK
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _MASK
    return x ^ (x >> 31)


def _hash64_01(x: np.ndarray) -> np.ndarray:
    """hash64_01 of csrc/dmv_device.cuh on a uint64 array (products wrap modulo 2^64)"""
    x = np.asarray(x, dtype=np.uint64)
    x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return x ^ (x >> np.uint64(31))


def seeded_start_vectors(representatives, num_vectors: int, seed: int, complex_vectors: bool = False) -> np.ndarray:
    """The start vectors of dmv_lanczos_quadrature with start = NULL, shape (num_vectors, len(representatives)):
    h = hash64_01(s ^ hash64_01(seed + 0x9e3779b97f4a7c15 (r + 1))) for representative s of vector r; float64: +1 if
    bit 63 of h is clear, else -1; complex128: exp(i phi) with phi = 2 pi (h >> 11) 2^-53."""
    reps = np.asarray(representatives, dtype=np.uint64)
    out = np.empty((num_vectors, reps.shape[0]), dtype=np.complex128 if complex_vectors else np.float64)
    for r in range(num_vectors):
        key = np.uint64(_hash64_01_int(int(seed) + _GOLDEN * (r + 1)))
        h = _hash64_01(reps ^ key)
        if complex_vectors:
            phi = (2.0 * np.pi) * ((h >> np.uint64(11)).astype(np.float64) * 2.0 ** -53)
            out[r] = np.cos(phi) + 1j * np.sin(phi)
        else:
            out[r] = np.where((h >> np.uint64(63)) == 0, 1.0, -1.0)
    return out


def thermodynamics(sectors, temperatures):
    """Thermodynamics of the sum of sectors, each given as (nodes, weights, multiplicity): nodes and weights of shape
    (R, M) (or (M,) for one vector) from lanczos_quadrature; multiplicity counts degenerate sectors that were not run
    (the other sign of a momentum, the other spin-inversion sector).  Z = sum_s multiplicity_s / R_s sum_rk w e^{-beta
    theta}.  temperatures: T > 0 (np.inf for beta = 0).  Computed in log space, shifted by the lowest node, so
    beta |E_0| ~ 1e3 neither overflows nor loses Z.
    -> (log Z, E, C, S) arrays over the temperatures: E = <H>, C = beta^2 (<H^2> - <H>^2), S = log Z + beta E."""
    parts = []
    for nodes, weights, multiplicity in sectors:
        th = np.atleast_2d(np.asarray(nodes, dtype=np.float64))
        w = np.atleast_2d(np.asarray(weights, dtype=np.float64))
        if th.shape != w.shape:
            raise ValueError("nodes and weights must have the same shape")
        keep = w > 0.0
        parts.append((th[keep], w[keep] * (float(multiplicity) / th.shape[0])))
    theta = np.concatenate([p[0] for p in parts])
    wts = np.concatenate([p[1] for p in parts])
    if theta.size == 0:
        raise ValueError("no node carries weight")
    e0 = theta.min()
    temps = np.atleast_1d(np.asarray(temperatures, dtype=np.float64))
    out = np.zeros((4, temps.shape[0]))
    log_w = np.log(wts)
    for i, T in enumerate(temps):
        if not T > 0.0:
            raise ValueError("temperatures must be positive (np.inf for beta = 0)")
        beta = 0.0 if np.isinf(T) else 1.0 / T
        x = log_w - beta * (theta - e0)
        top = x.max()
        p = np.exp(x - top)
        s = p.sum()
        log_z = top + np.log(s) - beta * e0
        p /= s
        energy = float(p @ theta)
        heat = beta * beta * float(p @ (theta - energy) ** 2)
        out[:, i] = (log_z, energy, heat, log_z + beta * energy)
    return out[0], out[1], out[2], out[3]
