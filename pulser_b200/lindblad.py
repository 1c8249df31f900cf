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
