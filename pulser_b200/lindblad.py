"""Lindblad master equation on the CUDA path (replaces ``qutip.mesolve``).

Reference: ``QutipEmulator._run_solver`` hands ``c_ops`` built by
``Hamiltonian._build_collapse_operators``
(``pulser-simulation/pulser_simulation/hamiltonian.py:97-124``) to
``qutip.mesolve`` / ``mcsolve`` (``simulation.py:705-735``).

Here the density matrix is vectorised row-major, ``vec(rho)[i*D + j] = rho[i,j]``,
i.e. it is the state of 2N qudits: row digits evolve under ``H``, column digits
under ``-H^T``.  For the Pulser Hamiltonian that is again a Pulser-shaped
Hamiltonian (drive ``-conj(c)``, detuning ``-det``, interaction ``-U`` on the
column qudits; in XY mode the real symmetric exchange couplings become ``-U^xy``
there as well), so the unitary part reuses the Schroedinger kernels unchanged;
the dissipator of single-qudit collapse operators factorises into one
``d^2 x d^2`` matrix per (row digit, column digit) pair (``pair_op_kernel``).
Where every atom's generator is the same and has no entry that flips exactly
one bit of the (row, column) pair -- dephasing, relaxation, depolarizing, any
set of collapse operators each diagonal or off-diagonal -- and the drive keeps
one phase, ``pb200_propagate`` runs the time-dependent Taylor propagator with
the dissipator inside the series (no splitting error; default tolerance 1e-10).
Otherwise, or with ``integrator=1 / 2``, the two are combined by symmetric
splitting + Richardson extrapolation (see include/pulser_b200.h).
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np

from ._lib import check, lib
from .engine import DevicePlan, _p
from .spec import DriveTable, HamiltonianSpec


def dissipator_generator(collapse_ops: np.ndarray) -> np.ndarray:
    """``sum_L  L (x) conj(L) - 1/2 L^+L (x) 1 - 1/2 1 (x) (L^+L)^T`` on ``vec(rho_k)[a*d+b]``."""
    ops = np.asarray(collapse_ops, dtype=np.complex128)
    d = ops.shape[-1]
    eye = np.eye(d)
    gen = np.zeros((d * d, d * d), dtype=np.complex128)
    for L in ops:
        ldl = L.conj().T @ L
        gen += np.kron(L, L.conj()) - 0.5 * np.kron(ldl, eye) - 0.5 * np.kron(eye, ldl.T)
    return gen


def doubled_spec(spec: HamiltonianSpec) -> HamiltonianSpec:
    """The 2N-qudit description whose Schroedinger evolution is ``-i[H, rho]``."""
    n = spec.n_qudits
    K = spec.interaction_matrix.shape[0]
    imat = np.zeros((K, 2 * n, 2 * n))
    imat[:, :n, :n] = spec.interaction_matrix
    imat[:, n:, n:] = -spec.interaction_matrix
    drives = []
    for d in spec.drives:
        coef = np.concatenate([d.coef, -np.conj(d.coef)], axis=0)
        det = np.concatenate([d.det, -d.det], axis=0)
        drives.append(DriveTable(d.basis, coef, det, False))
    return HamiltonianSpec(
        n_qudits=2 * n,
        dim=spec.dim,
        eigenbasis=list(spec.eigenbasis),
        basis_name=spec.basis_name,
        interaction_type=spec.interaction_type,
        sampling_times=spec.sampling_times,
        total_duration_ns=spec.total_duration_ns,
        interaction_matrix=imat,
        bad_atoms=np.concatenate([spec.bad_atoms, spec.bad_atoms]),
        drives=drives,
        collapse_ops=np.zeros((0, spec.dim, spec.dim), dtype=np.complex128),
        qubit_ids=[f"row{i}" for i in range(n)] + [f"col{i}" for i in range(n)],
        # XY + SLM mask: the masked pairs of the row block and of the column block switch on together
        slm_end=spec.slm_end,
        slm_targets=list(spec.slm_targets) + [t + n for t in spec.slm_targets],
    )


class LindbladPlan:
    """A batch of density matrices of one sequence resident on one GPU."""

    def __init__(self, specs: HamiltonianSpec | Sequence[HamiltonianSpec], interp_order: int = 3,
                 device: int = 0) -> None:
        if isinstance(specs, HamiltonianSpec):
            specs = [specs]
        self.specs = list(specs)
        s0 = self.specs[0]
        if s0.dim > 3:
            raise NotImplementedError("Lindblad path: d <= 3")
        if len(s0.collapse_ops) == 0:
            raise ValueError("no collapse operators: use DevicePlan")
        # a non-interacting original must not acquire an interaction through has_interaction()
        self.n = s0.n_qudits
        self.D = s0.hilbert_dim
        doubled = [doubled_spec(s) for s in self.specs]
        if not s0.has_interaction():
            for d in doubled:
                d.interaction_matrix = np.zeros_like(d.interaction_matrix)
        self.plan = DevicePlan(doubled, interp_order, device)
        gen = dissipator_generator(s0.collapse_ops)
        gens = np.ascontiguousarray(np.repeat(gen[None], self.n, axis=0))
        check(lib.pb200_plan_set_dissipator(self.plan._handle, self.n, _p(gens.view(np.float64))))

    def close(self) -> None:
        self.plan.close()

    def __enter__(self) -> "LindbladPlan":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def set_state(self, state: np.ndarray) -> None:
        """A ket (D) or a density matrix (D x D), shared by all trajectories."""
        state = np.asarray(state, dtype=np.complex128)
        if state.size == self.D:
            v = state.reshape(-1)
            rho = np.outer(v, v.conj())
        else:
            rho = state.reshape(self.D, self.D)
        self.plan.set_state(np.ascontiguousarray(rho).reshape(-1))

    def propagate(self, t_start: float, t_stop: float, **opts) -> dict:
        return self.plan.propagate(t_start, t_stop, **opts)

    def get_rho(self) -> np.ndarray:
        """[n_traj, D, D]"""
        return self.plan.get_state().reshape(-1, self.D, self.D)

    # --- reductions on the device (pb200_density_*): not divided by the trace --------------------------------------
    @property
    def n_traj(self) -> int:
        return self.plan.n_traj

    def _count(self, traj0: int, count: int | None) -> int:
        return self.plan.n_traj - traj0 if count is None else count

    def density_trace(self, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``Re Tr rho_b``, ``[count]``."""
        count = self._count(traj0, count)
        out = np.empty(count, dtype=np.float64)
        check(lib.pb200_density_trace(self.plan._handle, traj0, count, _p(out)))
        return out

    def density_occupation(self, digit: int, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``Tr(|digit><digit|_k rho_b)``, ``[count, N]``."""
        count = self._count(traj0, count)
        out = np.empty((count, self.n), dtype=np.float64)
        check(lib.pb200_density_occupation(self.plan._handle, traj0, count, int(digit), _p(out)))
        return out

    def density_correlation(self, digit: int, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``Tr(n_i n_j rho_b)`` with ``n_k = |digit><digit|_k``, ``[count, N, N]``."""
        count = self._count(traj0, count)
        out = np.empty((count, self.n, self.n), dtype=np.float64)
        check(lib.pb200_density_correlation(self.plan._handle, traj0, count, int(digit), _p(out)))
        return out

    def density_expect(self, terms, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``Tr(O rho_b)`` (complex) of an operator given as monomial terms (``pulser_b200.opterms.OpTerms``)."""
        count = self._count(traj0, count)
        if (terms.n, terms.d) != (self.n, self.plan.dim):
            raise ValueError(f"operator on {terms.n} qudits of dimension {terms.d}, the plan holds {self.n} of "
                             f"{self.plan.dim}")
        out = np.empty((count, 2), dtype=np.float64)
        check(lib.pb200_density_expect(self.plan._handle, traj0, count, C.byref(terms.c_desc()), _p(out)))
        return out[:, 0] + 1j * out[:, 1]

    def density_energy(self, ham_plan: DevicePlan, t_us: float, traj0: int = 0,
                       count: int | None = None) -> tuple[np.ndarray, np.ndarray]:
        """``(Tr(H rho_b), Tr(H^2 rho_b))`` with ``H = H(t_us)`` of the single-state plan ``ham_plan``."""
        count = self._count(traj0, count)
        e = np.empty(count, dtype=np.float64)
        e2 = np.empty(count, dtype=np.float64)
        check(lib.pb200_density_energy(self.plan._handle, ham_plan._handle, float(t_us), traj0, count, _p(e), _p(e2)))
        return e, e2

    def density_overlap(self, phi: np.ndarray, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``<phi|rho_b|phi>`` (complex) for a host ket ``phi`` of D amplitudes."""
        count = self._count(traj0, count)
        v = np.ascontiguousarray(np.asarray(phi, dtype=np.complex128).reshape(-1))
        if v.shape[0] != self.D:
            raise ValueError(f"state of length {v.shape[0]}, expected {self.D}")
        out = np.empty((count, 2), dtype=np.float64)
        check(lib.pb200_density_overlap(self.plan._handle, traj0, count, _p(v.view(np.float64)), _p(out)))
        return out[:, 0] + 1j * out[:, 1]

    def density_sample(self, n_samples: int, one_state: str, traj: int = 0) -> "Counter[str]":
        """Bitstring shots from ``diag rho`` drawn on the device with the uniforms of the global ``np.random`` stream
        (the recipe of ``DevicePlan.sample``)."""
        from collections import Counter

        u = np.ascontiguousarray(np.random.rand(n_samples), dtype=np.float64)
        idx = np.empty(n_samples, dtype=np.int64)
        check(lib.pb200_density_sample(self.plan._handle, traj, self.specs[0].eigenbasis.index(one_state), _p(u),
                                       n_samples, idx.ctypes.data_as(C.POINTER(C.c_int64))))
        return Counter(np.binary_repr(int(i), self.n) for i in idx)
