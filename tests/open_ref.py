"""Exact references for open-system evolution (numpy / scipy, no GPU), for the master-equation and quantum-jump tests.

Conventions follow ``pulser_b200/lindblad.py``: qudit 0 is the most significant digit of a basis index and a density
matrix is vectorised row-major, ``vec(rho)[i*D + j] = rho[i, j]``; for one qudit ``vec(rho_k)[a*d + b]``.
``H = sum_k [coef_k(t) |g><r|_k + h.c.] - sum_k det_k(t) n_k + sum_{i<j} U_ij n_i n_j`` with ``n_k = |r><r|_k``, the
assembly of ``oracle/ref_hamiltonian.py``; the sample tables are interpolated as the oracle does (QuTiP's cubic
not-a-knot spline, ``make_interp_spline(k=3)``).

Each function is exact for the case its docstring names, and none calls into ``pulser_b200``.
"""
from __future__ import annotations

import numpy as np
from scipy.integrate import solve_ivp
from scipy.interpolate import make_interp_spline
from scipy.linalg import expm


def random_ops(d: int, count: int, scale: float, seed: int) -> np.ndarray:
    """``count`` dense complex collapse operators; their ``L^+ L`` are far from diagonal."""
    rng = np.random.default_rng(seed)
    return scale * (rng.normal(size=(count, d, d)) + 1j * rng.normal(size=(count, d, d))) / np.sqrt(2 * d)


def random_diag_ops(d: int, count: int, scale: float, seed: int) -> np.ndarray:
    """``count`` diagonal complex collapse operators (dephasing type)."""
    rng = np.random.default_rng(seed)
    return np.array([np.diag(scale * (rng.normal(size=d) + 1j * rng.normal(size=d)) / np.sqrt(2)) for _ in range(count)])


def relaxation(eigenbasis, gamma: float) -> np.ndarray:
    """``sqrt(gamma) |g><r|``."""
    d = len(eigenbasis)
    L = np.zeros((d, d), dtype=np.complex128)
    L[list(eigenbasis).index("g"), list(eigenbasis).index("r")] = np.sqrt(gamma)
    return L


def random_density(D: int, rank: int, seed: int) -> np.ndarray:
    """A random mixed state ``A A^+ / Tr`` with ``A`` of shape ``D x rank``."""
    rng = np.random.default_rng(seed)
    A = rng.normal(size=(D, rank)) + 1j * rng.normal(size=(D, rank))
    rho = A @ A.conj().T
    return rho / np.trace(rho).real


def single_qudit_generator(ops) -> np.ndarray:
    """``G`` with ``vec(D(rho)) = G vec(rho)`` for ``D(rho) = sum_L L rho L^+ - 1/2 {L^+ L, rho}``, built column by
    column from the definition (basis matrices ``|a><b|``)."""
    ops = np.asarray(ops, dtype=np.complex128)
    d = ops.shape[-1]
    K = sum(L.conj().T @ L for L in ops)
    G = np.zeros((d * d, d * d), dtype=np.complex128)
    for a in range(d):
        for b in range(d):
            E = np.zeros((d, d), dtype=np.complex128)
            E[a, b] = 1.0
            out = sum(L @ E @ L.conj().T for L in ops) - 0.5 * (K @ E + E @ K)
            G[:, a * d + b] = out.reshape(-1)
    return G


def pair_expm_apply(rho: np.ndarray, G_k, T: float) -> np.ndarray:
    """``(prod_k expm(T G_k)) vec(rho)`` on a ``D x D`` matrix: qudit ``k``'s map acts on its (row, column) digit pair.
    Exact solution of the master equation with ``H = 0``."""
    n = len(G_k)
    d = int(round(np.sqrt(G_k[0].shape[0])))
    D = d**n
    x = np.asarray(rho, dtype=np.complex128).reshape([d] * (2 * n))
    for k in range(n):
        M = expm(T * np.asarray(G_k[k])).reshape(d, d, d, d)
        x = np.moveaxis(np.tensordot(M, x, axes=([2, 3], [k, n + k])), (0, 1), (k, n + k))
    return x.reshape(D, D)


def _digits(n: int, d: int) -> np.ndarray:
    """``[D, n]``: digit of qudit k in basis index i (qudit 0 most significant)."""
    idx = np.arange(d**n)
    return np.stack([(idx // d ** (n - 1 - k)) % d for k in range(n)], axis=1)


def _spline_integral(times: np.ndarray, y: np.ndarray, T: float, points: int = 4) -> complex:
    """``int_0^T`` of the cubic not-a-knot interpolant of ``y`` by Gauss-Legendre per sampling interval (exact for the
    cubic pieces)."""
    f = make_interp_spline(times, y, k=3)
    x, w = np.polynomial.legendre.leggauss(points)
    acc = 0.0
    for a, b in zip(times[:-1], times[1:]):
        if a >= T:
            break
        b = min(b, T)
        acc = acc + 0.5 * (b - a) * np.sum(w * f(0.5 * (b - a) * x + 0.5 * (a + b)))
    return acc


def diagonal_phases(spec, T: float) -> np.ndarray:
    """``Phi_a = int_0^T E_a(t) dt`` for a diagonal ``H`` (detuning + interaction, no drive), ``[D]``."""
    n, d = spec.n_qudits, spec.dim
    r = list(spec.eigenbasis).index("r")
    nk = (_digits(n, d) == r).astype(float)
    det_int = np.zeros(n)
    for drv in spec.drives:
        assert not np.any(drv.coef != 0), "diagonal_phases: the drive must be off"
        det_int += np.array([_spline_integral(spec.sampling_times, drv.det[k], T).real for k in range(n)])
    U = np.array(spec.interaction_matrix[-1], dtype=float) if spec.has_interaction() else np.zeros((n, n))
    iu = np.triu_indices(n, 1)
    pair = np.einsum("si,sj->sij", nk, nk)[:, iu[0], iu[1]] @ U[iu]
    return pair * T - nk @ det_int


def diagonal_lindblad(rho0: np.ndarray, spec, ops, T: float) -> np.ndarray:
    """Exact ``rho(T)`` for a diagonal ``H`` and diagonal collapse operators ``ops`` (every ``L`` acts on every qudit):
    ``rho_ab(T) = rho_ab(0) exp(-i (Phi_a - Phi_b)) prod_k exp(T g(a_k, b_k))``."""
    ops = np.asarray(ops, dtype=np.complex128)
    assert all(np.allclose(L, np.diag(np.diag(L)), atol=0.0) for L in ops)
    n, d = spec.n_qudits, spec.dim
    l = np.array([np.diag(L) for L in ops])  # [n_ops, d]
    g = (l[:, :, None] * l[:, None, :].conj() - 0.5 * np.abs(l[:, :, None]) ** 2
         - 0.5 * np.abs(l[:, None, :]) ** 2).sum(axis=0)  # [d, d]
    dig = _digits(n, d)
    logdec = np.zeros((d**n, d**n), dtype=np.complex128)
    for k in range(n):
        logdec += g[dig[:, k][:, None], dig[:, k][None, :]]
    phi = diagonal_phases(spec, T)
    return np.asarray(rho0) * np.exp(-1j * (phi[:, None] - phi[None, :]) + T * logdec)


def product_lindblad(spec, ops, rho_k0, T: float, rtol: float = 1e-13, atol: float = 1e-15) -> list[np.ndarray]:
    """``[rho_k(T)]`` of a non-interacting register: each qudit's ``d x d`` master equation with its own interpolated
    drive and detuning, integrated by DOP853 interval by interval (all qudits in one ODE).  ``rho_k0``: ``[n, d, d]``
    or one ``d x d`` for every qudit.  The register's ``rho(T)`` is ``kron`` of the list."""
    n, d = spec.n_qudits, spec.dim
    eig = list(spec.eigenbasis)
    r, gi = eig.index("r"), eig.index("g")
    ops = np.asarray(ops, dtype=np.complex128)
    K = sum(L.conj().T @ L for L in ops)
    times = spec.sampling_times
    coef_f, det_f = [], []
    for drv in spec.drives:
        assert drv.basis == "ground-rydberg"
        coef_f.append([make_interp_spline(times, drv.coef[k], k=3) for k in range(n)])
        det_f.append([make_interp_spline(times, drv.det[k], k=3) for k in range(n)])
    sgr = np.zeros((d, d), dtype=np.complex128); sgr[gi, r] = 1.0
    srr = np.zeros((d, d), dtype=np.complex128); srr[r, r] = 1.0

    def hams(t):
        H = np.zeros((n, d, d), dtype=np.complex128)
        for cf, df in zip(coef_f, det_f):
            for k in range(n):
                c = complex(cf[k](t))
                H[k] += c * sgr + np.conj(c) * sgr.T - float(df[k](t)) * srr
        return H

    def f(t, y):
        rho = y.reshape(n, d, d)
        H = hams(t)
        Hr = H @ rho
        out = -1j * (Hr - rho @ H)
        for L in ops:
            out = out + L @ rho @ L.conj().T
        Kr = K @ rho
        out = out - 0.5 * (Kr + rho @ K)
        return out.reshape(-1)

    rho = np.broadcast_to(np.asarray(rho_k0, dtype=np.complex128), (n, d, d)).copy()
    y = rho.reshape(-1)
    for a, b in zip(times[:-1], times[1:]):
        if a >= T:
            break
        b = min(b, T)
        sol = solve_ivp(f, (a, b), y, method="DOP853", rtol=rtol, atol=atol)
        assert sol.success, sol.message
        y = sol.y[:, -1]
    return list(y.reshape(n, d, d))


def kron_all(mats) -> np.ndarray:
    out = np.asarray(mats[0])
    for m in mats[1:]:
        out = np.kron(out, m)
    return out


def apply_local(psi: np.ndarray, M: np.ndarray, n: int) -> np.ndarray:
    """``(M (x) ... (x) M) psi`` for one state ``[D]`` or a batch ``[B, D]``."""
    d = M.shape[0]
    psi = np.asarray(psi, dtype=np.complex128)
    batch = psi.reshape(-1, d**n)
    x = batch.reshape([batch.shape[0]] + [d] * n)
    for k in range(n):
        x = np.moveaxis(np.tensordot(M, x, axes=([1], [k + 1])), 0, k + 1)
    return x.reshape(psi.shape)


def no_jump_state(psi0: np.ndarray, K: np.ndarray, T: float) -> np.ndarray:
    """``normalise(prod_k expm(-T/2 K)_k psi0)``: the no-jump trajectory of ``H = 0`` with ``K = sum L^+ L`` (any
    ``d x d`` Hermitian matrix); ``psi0`` is ``[D]`` or ``[B, D]``."""
    K = np.asarray(K, dtype=np.complex128)
    psi0 = np.asarray(psi0, dtype=np.complex128)
    n = int(round(np.log(psi0.shape[-1]) / np.log(K.shape[0])))
    out = apply_local(psi0, expm(-0.5 * T * K), n)
    return out / np.linalg.norm(out, axis=-1, keepdims=True)
