"""Exact reference for the Taylor propagator: the Schroedinger evolution of a d = 2 register with one drive under
QobjEvo's interpolated coefficients, to ~1e-15 of the state norm (numpy / scipy only).

Inside one piece of the not-a-knot cubic spline every coefficient row is an exact cubic, so that
``H(t) = Dint + sum_j H_j (t - x_i)^j`` holds exactly on ``[x_i, x_{i+1}]``. ``PiecewiseCubicHamiltonian.evolve`` walks the
pieces of a window, cuts each one into sub-steps of ``h ||H - gamma|| <= 1`` and sums the Taylor series of every
sub-step in its own local time, with the full polynomial history, until the terms fall below 1e-17 of the norm. Nothing
here comes from the library: the coefficients are scipy's (``make_interp_spline`` + ``PPoly.from_spline``, real and
imaginary parts of the drive rows splined separately), the roles are ``oracle.matfree.BASIS_ROLES`` and the interaction
is ``spec.pair_matrix()``. The rows may differ from qubit to qubit in any way (uniform drives, noise trajectories,
detuning maps of any number of shapes); the drive history is applied through the singular value decomposition of the
per-step coefficient matrix, so rows that share one time shape cost one flip pass per term.
"""
from __future__ import annotations

from math import comb

import numpy as np
from scipy.interpolate import PPoly, make_interp_spline

from oracle.matfree import BASIS_ROLES

_BINOM = np.array([[comb(l, j) for j in range(4)] for l in range(4)], dtype=float)   # [l, j] = C(l, j)


class PiecewiseCubicHamiltonian:
    def __init__(self, spec) -> None:
        if spec.dim != 2 or len(spec.drives) != 1:
            raise ValueError("the reference covers d = 2 registers with one drive")
        n = spec.n_qudits
        self.n, self.D = n, 2**n
        drv = spec.drives[0]
        to, frm = BASIS_ROLES[drv.basis]
        self.ito, self.ifr = spec.eigenbasis.index(to), spec.eigenbasis.index(frm)
        t = np.asarray(spec.sampling_times, dtype=float)
        coef = np.asarray(drv.coef, dtype=complex)
        rows = np.concatenate([coef.real, coef.imag, np.asarray(drv.det, dtype=float)])
        x, cs = None, []
        for r in rows:
            pp = PPoly.from_spline(make_interp_spline(t, r, k=3))
            keep = np.diff(pp.x) > 0          # from_spline also returns the zero-length pieces of the end knots
            if x is None:
                x = np.append(pp.x[:-1][keep], pp.x[1:][keep][-1])
            cs.append(pp.c[::-1][:, keep])    # ascending powers of (t - x_i): [4, pieces]
        c = np.stack(cs, axis=-1)             # [4, pieces, 3N]
        self.x = x
        self.drive = c[:, :, :n] + 1j * c[:, :, n:2 * n]
        self.det = c[:, :, 2 * n:]
        # Ising interaction on the Rydberg digit, sum_{i<j} U_ij n_i n_j
        dint = np.zeros([2] * n)
        if spec.has_interaction():
            r = spec.eigenbasis.index("r")
            U = spec.pair_matrix()
            for i in range(n):
                for j in range(i + 1, n):
                    if U[i, j] != 0.0:
                        idx = [slice(None)] * n
                        idx[i] = idx[j] = r
                        dint[tuple(idx)] += U[i, j]
        self.dint = dint.reshape(-1)

    # ---------------------------------------------------------------- pieces and terms
    def _view(self, v: np.ndarray, k: int) -> np.ndarray:
        return v.reshape(2**k, 2, 2 ** (self.n - 1 - k))

    def _piece(self, t: float) -> int:
        return int(np.clip(np.searchsorted(self.x, t, side="right") - 1, 0, len(self.x) - 2))

    def _diag(self, det: np.ndarray) -> np.ndarray:
        """``-sum_k det[k] [digit_k = from]`` as a vector"""
        out = np.zeros(self.D)
        for k in range(self.n):
            self._view(out, k)[:, self.ifr, :] -= det[k]
        return out

    def _flip(self, u: np.ndarray, y1: np.ndarray, y2: np.ndarray, out: np.ndarray) -> None:
        """``out += sum_k u_k |to><from|_k y1 + conj(u_k) |from><to|_k y2``"""
        for k in range(self.n):
            o, a, b = self._view(out, k), self._view(y1, k), self._view(y2, k)
            o[:, self.ito, :] += u[k] * a[:, self.ifr, :]
            o[:, self.ifr, :] += np.conj(u[k]) * b[:, self.ito, :]

    def apply(self, t: float, v: np.ndarray) -> np.ndarray:
        """``H(t) v`` from the exact cubics of the piece that holds ``t``"""
        i = self._piece(t)
        tau = t - self.x[i]
        pw = tau ** np.arange(4)
        v = np.asarray(v, dtype=complex)
        out = (self.dint + self._diag(pw @ self.det[:, i, :])) * v
        c = pw @ self.drive[:, i, :]
        self._flip(c, v, v, out)
        return out

    # ---------------------------------------------------------------- evolution
    def evolve(self, psi: np.ndarray, t0: float, t1: float, split: int = 1) -> np.ndarray:
        """``psi(t1)`` from ``psi(t0)``; windows may start and end anywhere inside a piece.  ``split`` cuts every sub-step
        into that many (a self-check of the series)"""
        psi = np.array(psi, dtype=complex).reshape(-1)
        lo, hi = float(self.dint.min()), float(self.dint.max())
        gamma, half = 0.5 * (lo + hi), 0.5 * (hi - lo)
        t = float(t0)
        while t < t1:
            i = self._piece(t)
            if self.x[i + 1] <= t:        # t on the last breakpoint of the table
                break
            e = min(float(self.x[i + 1]), float(t1))
            psi = self._evolve_piece(psi, i, t - self.x[i], e - self.x[i], gamma, half, split)
            t = e
        return psi

    def _evolve_piece(self, psi, i, ta, tb, gamma, half, split):
        a_det, a_drive = self.det[:, i, :], self.drive[:, i, :]
        diag_l = [self._diag(a_det[l]) for l in range(4)]
        tm = max(abs(ta), abs(tb))
        pw = tm ** np.arange(4)
        bound = half + float(np.sum(np.abs(a_det) * pw[:, None]) + np.sum(np.abs(a_drive) * pw[:, None]))
        nsub = split * max(1, int(np.ceil((tb - ta) * bound)))    # h ||H - gamma|| <= 1
        hs = (tb - ta) / nsub
        scale = np.linalg.norm(psi)
        for q in range(nsub):
            tau0 = ta + q * hs
            # sum_l a_l tau^l = sum_j (sum_l w[j, l] a_l) u^j  with  tau = tau0 + hs u;  the series is in u
            w = np.zeros((4, 4))
            for j in range(4):
                for l in range(j, 4):
                    w[j, l] = _BINOM[l, j] * tau0 ** (l - j) * hs**j
            diag = [hs * sum(w[j, l] * diag_l[l] for l in range(j, 4) if w[j, l] != 0.0) for j in range(4)]
            diag[0] = diag[0] + hs * (self.dint - gamma)
            cm = hs * (w @ a_drive).T                          # [N, 4]: the drive rows in u, times hs
            U, S, Vh = np.linalg.svd(cm, full_matrices=False)
            keep = S > 1e-15 * S[0] if S[0] > 0.0 else np.zeros(len(S), dtype=bool)
            terms = [psi]
            out = psi.copy()
            m = 0
            while True:
                hist = terms[-4:][::-1]                       # chi_m, chi_{m-1}, ...
                y = np.zeros(self.D, dtype=complex)
                for j, v in enumerate(hist):
                    y += diag[j] * v
                for r in np.nonzero(keep)[0]:
                    y1 = sum(Vh[r, j] * v for j, v in enumerate(hist))
                    y2 = sum(np.conj(Vh[r, j]) * v for j, v in enumerate(hist))
                    self._flip(S[r] * U[:, r], y1, y2, y)
                nxt = (-1j / (m + 1)) * y
                terms.append(nxt)
                out += nxt
                m += 1
                if m > 200:
                    raise RuntimeError("Taylor series of a sub-step did not converge")
                if m >= 4 and all(np.linalg.norm(v) < 1e-17 * scale for v in terms[-4:]):
                    break
                terms = terms[-4:]
            psi = out
        return psi * np.exp(-1j * gamma * (tb - ta))
