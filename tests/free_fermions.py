"""Entanglement spectrum of the XX ring at half filling from free fermions (Peschel 2003) -- an exact, independent
algorithm that shares nothing with the product, the oracle or the reference.  Test infrastructure.

H = Σ_i σˣ_iσˣ_{i+1} + σʸ_iσʸ_{i+1} = 2 Σ_i (σ⁺_iσ⁻_{i+1} + h.c.) on N sites, periodic.  Jordan-Wigner maps it to free
fermions with hopping 2 (a set bit is an occupied site).  With N / 2 fermions the boundary condition of the fermions is
antiperiodic when N / 2 is even, k = 2π (n + ½) / N, and periodic when N / 2 is odd, k = 2π n / N.  The ground state
fills the N / 2 momenta of one side of the band; the spectrum below does not depend on which contiguous half it is, so
the N / 2 momenta closest to 0 are taken.

For a block A of ℓ contiguous sites the reduced density matrix is Gaussian: with ν_m the eigenvalues of the restricted
correlation matrix C_ij = <c†_i c_j> = (1 / N) Σ_{k occupied} e^{ik(i - j)}, i, j in A, the eigenvalues of ρ_A are the
products Π_{m in S} ν_m Π_{m not in S} (1 - ν_m) over the subsets S of modes, and |S| is the number of fermions, that is
the Hamming weight w of A.  The Jordan-Wigner string of a contiguous block stays inside it, so ρ_A of the spins has the
same spectrum.
"""
import itertools

import numpy as np


def occupied_momenta(n_sites: int) -> np.ndarray:
    if n_sites < 2 or n_sites % 2:
        raise ValueError("even number of sites")
    half = n_sites // 2
    shift = 0.5 if half % 2 == 0 else 0.0
    k = 2.0 * np.pi * (np.arange(-n_sites // 2, n_sites // 2) + shift) / n_sites
    return np.sort(k[np.argsort(np.abs(k), kind="stable")[:half]])


def correlation_matrix(n_sites: int, ell: int) -> np.ndarray:
    """C_ij = (1 / N) Σ_{k occupied} e^{ik(i - j)} for i, j < ℓ"""
    k = occupied_momenta(n_sites)
    d = np.arange(ell)[:, None] - np.arange(ell)[None, :]
    return (np.exp(1j * k[None, None, :] * d[:, :, None]).sum(axis=2) / n_sites)


def block_spectrum(n_sites: int, ell: int) -> dict:
    """{w: the eigenvalues of block w of ρ_A, ascending} for A = sites 0 ... ℓ - 1 of the XX ring's ground state"""
    nu = np.clip(np.linalg.eigvalsh(correlation_matrix(n_sites, ell)), 0.0, 1.0)
    out = {w: [] for w in range(ell + 1)}
    for occ in itertools.product((0, 1), repeat=ell):
        p = np.prod([nu[m] if o else 1.0 - nu[m] for m, o in enumerate(occ)])
        out[sum(occ)].append(p)
    return {w: np.sort(np.array(v)) for w, v in out.items()}


def entropy(n_sites: int, ell: int) -> float:
    """S(A) = -Σ_m ν_m log ν_m + (1 - ν_m) log (1 - ν_m)"""
    nu = np.linalg.eigvalsh(correlation_matrix(n_sites, ell))
    nu = nu[(nu > 1e-300) & (nu < 1.0 - 1e-16)]
    return float(-(nu * np.log(nu) + (1.0 - nu) * np.log(1.0 - nu)).sum())
