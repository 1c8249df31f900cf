"""Exact references for the Magnus propagator (integrators 1 and 2) on Hamiltonians that are constant in time.

With H constant, every Magnus scheme the step controller can choose (CF4, order 2, Richardson-extrapolated,
step-doubled, steps cut anywhere) gives exactly ``exp(-i H T) psi0``: what remains is the truncation of the Chebyshev /
Lanczos exponentials and rounding, whatever steps the controller takes.

``constant_spec`` builds specs whose samples hold the same value at every sampling time, the last one included (the
workload builders end on a zero sample, over which a cubic spline rings).  H is assembled by the oracle
(``oracle.ref_hamiltonian``, the reference's term list) from the first sample and exponentiated by a dense ``eigh``:

- ``dense_evolve``: the whole register, for D <= 4096 (d = 3 / 4, XY, any coupling);
- ``ClusterReference``: d = 2 registers whose couplings are block-diagonal over clusters of at most 10 atoms.  The
  state stays a product of per-cluster states, so any N is in reach: the full vector up to N ~ 20, single amplitudes
  and the norm beyond.  ``interleaved_clusters`` spreads every cluster over all qudit positions (qudit 0 is the most
  significant bit), so that each cluster has atoms in the tile bits, in the second-pass bits and in the bits loaded as
  extra partners.
"""
from __future__ import annotations

import numpy as np

from helpers import random_state
from pulser_b200.spec import DriveTable, HamiltonianSpec

EIGENBASIS = {("ising", 2): ["r", "g"], ("ising", 3): ["r", "g", "h"], ("ising", 4): ["r", "g", "h", "x"],
              ("XY", 2): ["u", "d"]}


def constant_spec(drives, imat, n_samples: int = 64, dt_ns: int = 1, dim: int = 2,
                  interaction_type: str = "ising", basis_name: str | None = None) -> HamiltonianSpec:
    """``drives``: ``[(basis, coef[N], det[N])]``, constant in time; ``imat``: ``[N, N]`` (Ising) or ``[2, N, N]`` (XY:
    exchange, van der Waals).  ``n_samples`` intervals of ``dt_ns``."""
    imat = np.asarray(imat, dtype=float)
    if imat.ndim == 2:
        imat = imat[None]
    n = imat.shape[-1]
    nt = n_samples + 1
    tables = []
    for basis, coef, det in drives:
        coef = np.broadcast_to(np.asarray(coef, dtype=complex), (n,))
        det = np.broadcast_to(np.asarray(det, dtype=float), (n,))
        uniform = bool(np.all(coef == coef[0]) and np.all(det == det[0]))
        tables.append(DriveTable(basis, np.repeat(coef[:, None], nt, axis=1), np.repeat(det[:, None], nt, axis=1),
                                 uniform))
    if basis_name is None:
        basis_name = "XY" if interaction_type == "XY" else ("ground-rydberg" if len(drives) == 1 else "all")
    return HamiltonianSpec(
        n_qudits=n, dim=dim, eigenbasis=list(EIGENBASIS[(interaction_type, dim)]), basis_name=basis_name,
        interaction_type=interaction_type,
        sampling_times=np.arange(nt, dtype=float) * dt_ns / 1000, total_duration_ns=n_samples * dt_ns,
        interaction_matrix=imat, bad_atoms=np.zeros(n, dtype=bool), drives=tables,
        collapse_ops=np.zeros((0, dim, dim), dtype=complex), qubit_ids=[f"q{i}" for i in range(n)],
    )


def interleaved_clusters(n: int, n_clusters: int | None = None, shift: int = 0) -> list[list[int]]:
    """atom k in cluster (k + shift) % C, C = ceil(n / 10) unless given"""
    c = n_clusters or -(-n // 10)
    out = [[k for k in range(n) if (k + shift) % c == j] for j in range(c)]
    if max(len(a) for a in out) > 10:
        raise ValueError("clusters of more than 10 atoms")
    return out


def cluster_couplings(n: int, clusters, seed: int, lo: float = 0.5, hi: float = 4.0) -> np.ndarray:
    """symmetric ``[N, N]`` couplings, random in [lo, hi] inside a cluster and exactly 0 between clusters"""
    rng = np.random.default_rng(seed)
    U = np.zeros((n, n))
    for atoms in clusters:
        for a, i in enumerate(atoms):
            for j in atoms[a + 1:]:
                U[i, j] = U[j, i] = rng.uniform(lo, hi)
    return U


def dense_hamiltonian(spec) -> np.ndarray:
    """H at the (constant) first sample, as the oracle assembles it"""
    from oracle.ref_hamiltonian import OracleHamiltonian

    H = None
    for a, c in OracleHamiltonian.from_spec(spec).terms:
        m = a.toarray() * (1.0 if c is None else complex(c[0]))
        H = m if H is None else H + m
    return H


def expm_apply(H: np.ndarray, psi: np.ndarray, T: float) -> np.ndarray:
    w, V = np.linalg.eigh(H)
    return V @ (np.exp(-1j * w * T) * (V.conj().T @ psi))


def dense_evolve(spec, psi0: np.ndarray, T: float) -> np.ndarray:
    if spec.hilbert_dim > 4096:
        raise ValueError("dense reference limited to D <= 4096")
    return expm_apply(dense_hamiltonian(spec), np.asarray(psi0, dtype=complex), T)


class ClusterReference:
    """``exp(-i H T)`` of a d = 2 Ising register whose couplings vanish between the given clusters, as the product of
    the per-cluster exponentials (dense ``eigh`` of each cluster's oracle Hamiltonian)"""

    def __init__(self, spec, clusters) -> None:
        if spec.dim != 2 or spec.interaction_type != "ising":
            raise ValueError("cluster reference covers d = 2 Ising registers")
        n = spec.n_qudits
        self.n, self.clusters = n, [list(a) for a in clusters]
        if sorted(k for a in self.clusters for k in a) != list(range(n)):
            raise ValueError("clusters must partition the atoms")
        U = spec.pair_matrix()
        inside = np.zeros((n, n), dtype=bool)
        for a in self.clusters:
            inside[np.ix_(a, a)] = True
        if np.any(U[~inside] != 0.0):
            raise ValueError("couplings between clusters")
        self.H = [dense_hamiltonian(self._sub(spec, a)) for a in self.clusters]

    @staticmethod
    def _sub(spec, atoms) -> HamiltonianSpec:
        import copy

        s = copy.copy(spec)
        s.n_qudits = len(atoms)
        s.interaction_matrix = spec.interaction_matrix[:, atoms][:, :, atoms]
        s.bad_atoms = spec.bad_atoms[atoms]
        s.drives = [DriveTable(d.basis, d.coef[atoms], d.det[atoms], d.uniform) for d in spec.drives]
        s.qubit_ids = [spec.qubit_ids[k] for k in atoms]
        return s

    def initial(self, seed: int) -> list[np.ndarray]:
        """random per-cluster states"""
        return [random_state(2 ** len(a), seed + 7 * c) for c, a in enumerate(self.clusters)]

    def ground(self) -> list[np.ndarray]:
        """the all-ground product state (|g> is digit 1 of the eigenbasis r, g)"""
        out = []
        for a in self.clusters:
            v = np.zeros(2 ** len(a), dtype=complex)
            v[-1] = 1.0
            out.append(v)
        return out

    def evolve(self, parts, T: float) -> list[np.ndarray]:
        return [expm_apply(H, p, T) for H, p in zip(self.H, parts)]

    def full(self, parts) -> np.ndarray:
        """the product state as one vector of 2^N amplitudes"""
        out, order = np.ones(1, dtype=complex), []
        for p, a in zip(parts, self.clusters):
            out = np.multiply.outer(out, p).reshape(-1)
            order += a
        t = out.reshape([2] * self.n).transpose(np.argsort(order))
        return np.ascontiguousarray(t).reshape(-1)

    def amplitudes(self, parts, idx) -> np.ndarray:
        """amplitudes of the product state at the given indices of the full vector"""
        idx = np.asarray(idx, dtype=np.int64)
        out = np.ones(idx.shape, dtype=complex)
        for p, a in zip(parts, self.clusters):
            sub = np.zeros(idx.shape, dtype=np.int64)
            for m, k in enumerate(a):
                sub |= ((idx >> (self.n - 1 - k)) & 1) << (len(a) - 1 - m)
            out *= p[sub]
        return out

    @staticmethod
    def norm(parts) -> float:
        return float(np.prod([np.linalg.norm(p) for p in parts]))


def probe_indices(n: int, count: int = 4000, seed: int = 0, tile_bits: int = 11) -> np.ndarray:
    """all-Rydberg (0), all-ground (2^N - 1), the indices that set exactly the bits of the tile, of the next
    ``tile_bits`` bits and of those above (and their complements), and ``count`` random ones"""
    full = (1 << n) - 1
    lo = (1 << min(tile_bits, n)) - 1
    mid = ((1 << min(2 * tile_bits, n)) - 1) & ~lo
    hi = full & ~(lo | mid)
    fixed = [0, full]
    for m in (lo, mid, hi, lo | hi, mid | hi, lo | mid):
        fixed += [m, full & ~m]
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([np.array(fixed, dtype=np.int64), rng.integers(0, full + 1, count)]))
