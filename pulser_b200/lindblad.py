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
set of collapse operators each diagonal or off-diagonal -- and the drive is one
global shape (per-qubit static factors allowed) whose phase may move in time
(phase shifts, phase jumps between pulses, Ramsey pairs, EOM drift correction:
the column qudits then drive ``-conj(omega(t))``, which the stage forms from the
same partner loads), ``pb200_propagate`` runs the time-dependent Taylor
propagator with the dissipator inside the series (no splitting error; default
tolerance 1e-10).  Otherwise, or with ``integrator=1 / 2``, the two are combined
by symmetric splitting + Richardson extrapolation (see include/pulser_b200.h).

``ShardedLindbladPlan`` splits vec(rho) of one sequence over 2, 4 or 8 state-vector shards
(``pulser_b200.sharded``): the top bits of the 2N-qubit index are the top row bits, so a shard
holds complete rows of rho and every density reduction is a sum of per-shard shares.
"""
from __future__ import annotations

import ctypes as C
from typing import Sequence

import numpy as np

from ._lib import PB200Error, check, lib
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


def _rho_of(state: np.ndarray, D: int) -> np.ndarray:
    """A ket (D) or a density matrix (D x D) as the D x D density matrix."""
    state = np.asarray(state, dtype=np.complex128)
    if state.size == D:
        v = state.reshape(-1)
        return np.outer(v, v.conj())
    return state.reshape(D, D)


def _doubled_specs(specs: Sequence[HamiltonianSpec]) -> list[HamiltonianSpec]:
    """``doubled_spec`` of each; a non-interacting original must not acquire an interaction through has_interaction()."""
    doubled = [doubled_spec(s) for s in specs]
    if not specs[0].has_interaction():
        for d in doubled:
            d.interaction_matrix = np.zeros_like(d.interaction_matrix)
    return doubled


def _set_dissipator(plan: DevicePlan, spec: HamiltonianSpec) -> None:
    """The generator of ``spec``'s collapse operators on every atom (``pb200_plan_set_dissipator``)."""
    gen = dissipator_generator(spec.collapse_ops)
    gens = np.ascontiguousarray(np.repeat(gen[None], spec.n_qudits, axis=0))
    check(lib.pb200_plan_set_dissipator(plan._handle, spec.n_qudits, _p(gens.view(np.float64))))


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
        self.n = s0.n_qudits
        self.D = s0.hilbert_dim
        self.plan = DevicePlan(_doubled_specs(self.specs), interp_order, device)
        _set_dissipator(self.plan, s0)

    def close(self) -> None:
        self.plan.close()

    def __enter__(self) -> "LindbladPlan":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def set_state(self, state: np.ndarray) -> None:
        """A ket (D) or a density matrix (D x D), shared by all trajectories."""
        self.plan.set_state(np.ascontiguousarray(_rho_of(state, self.D)).reshape(-1))

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


class ShardedLindbladPlan:
    """vec(rho) of one sequence split over ``len(devices)`` state-vector shards; ``devices[i]`` is shard i's device.

    vec(rho) is the state of 2N qubits whose top ``log2(G)`` bits are the top row bits: shard i holds the rows
    ``[i D / G, (i + 1) D / G)`` of rho.  Every shard is a plan of the doubled register with the dissipator, linked into
    one group (``pb200_shards_link``) and advanced by ``pb200_shards_propagate``, whose schedule is the unsharded plan's.
    The reductions are the ``pb200_density_*`` of each shard, i.e. its rows' share, summed here.  The methods mirror
    those of ``LindbladPlan`` that ``B200Backend._stream_density`` and ``DeviceDensityView`` call (one trajectory).

    Scope: d = 2, a drive of one phase (a phase that moves in time runs on an unsharded ``LindbladPlan``), a dissipator
    without single-bit-flip entries, Ising interaction, no SLM mask; anything else raises ``NotImplementedError`` with
    its reason.
    """

    def __init__(self, specs: HamiltonianSpec | Sequence[HamiltonianSpec], devices: Sequence[int],
                 interp_order: int = 3) -> None:
        from .sharded import MAX_LOCAL_BITS, MIN_LOCAL_BITS, shard_bits_of, validate_devices

        devices = validate_devices(devices)
        if isinstance(specs, HamiltonianSpec):
            specs = [specs]
        if len(specs) != 1:
            raise NotImplementedError("a sharded density matrix holds one trajectory (no stochastic noise)")
        s0 = specs[0]
        self.specs = list(specs)
        if s0.dim != 2:
            raise NotImplementedError(f"density-matrix shards need a d = 2 register (this one has d = {s0.dim}: leakage)")
        if s0.interaction_type == "XY":
            raise NotImplementedError("density-matrix shards take the Ising interaction, not XY")
        if s0.slm_coefficient() is not None:
            raise NotImplementedError("density-matrix shards take no SLM mask")
        if len(s0.collapse_ops) == 0:
            raise ValueError("no collapse operators: use ShardedPlan")
        self.n = s0.n_qudits
        self.D = s0.hilbert_dim
        self.G = len(devices)
        self.bits = shard_bits_of(self.G)
        self.L = 2 * self.n - self.bits
        if not MIN_LOCAL_BITS <= self.L <= MAX_LOCAL_BITS:
            raise ValueError(
                f"{self.G} shards of the density matrix of {self.n} atoms hold 2^{self.L} entries each; a shard holds "
                f"2^{MIN_LOCAL_BITS} to 2^{MAX_LOCAL_BITS}"
            )
        self.rows = self.D >> self.bits
        self.devices = devices
        self.interp_order = interp_order
        doubled = _doubled_specs(self.specs)
        self.shards: list[DevicePlan] = []
        self._arr = None
        self._ham: dict[tuple[int, int], DevicePlan] = {}
        try:
            for i, dev in enumerate(devices):
                self.shards.append(DevicePlan(doubled, interp_order, dev, shard=(self.bits, i)))
                _set_dissipator(self.shards[-1], s0)
            self._arr = (C.c_void_p * self.G)(*[s._handle for s in self.shards])
            check(lib.pb200_shards_link(self._arr, self.G))
        except PB200Error as e:
            self.close()
            if e.code == -3:  # PB200_ERR_UNSUPPORTED: a moving drive phase, single-bit-flip collapse operators, ...
                raise NotImplementedError(str(e)) from e
            raise
        except Exception:
            self.close()
            raise

    def close(self) -> None:
        for p in list(self.shards) + list(self._ham.values()):
            p.close()
        self.shards = []
        self._ham = {}
        self._arr = None

    def __del__(self) -> None:  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self) -> "ShardedLindbladPlan":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def set_state(self, state: np.ndarray) -> None:
        """A ket (D) or a density matrix (D x D); each shard takes its rows."""
        rho = _rho_of(state, self.D)
        for i, s in enumerate(self.shards):
            part = np.ascontiguousarray(rho[i * self.rows:(i + 1) * self.rows]).reshape(-1)
            check(lib.pb200_state_set(s._handle, 0, 1, _p(part.view(np.float64)), -1, 1))

    def propagate(self, t_start: float, t_stop: float, **opts) -> dict:
        """Advance rho from ``t_start`` to ``t_stop`` (us): ``ShardedPlan.propagate`` on the linked shards."""
        from .sharded import ShardedPlan

        return ShardedPlan.propagate(self, t_start, t_stop, **opts)

    def get_rho(self) -> np.ndarray:
        """[1, D, D]"""
        return np.concatenate([s.get_state()[0] for s in self.shards]).reshape(1, self.D, self.D)

    # --- reductions: each shard's rows' share (pb200_density_*), summed; not divided by the trace ---------------------
    @property
    def n_traj(self) -> int:
        return 1

    @staticmethod
    def _one(traj0: int, count: int | None) -> None:
        if traj0 != 0 or count not in (None, 1):
            raise ValueError("a sharded density matrix holds one trajectory")

    def density_trace(self, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``Re Tr rho``, ``[1]``."""
        self._one(traj0, count)
        return np.array([sum(self._shard_traces())])

    def _shard_traces(self) -> list[float]:
        out = []
        for s in self.shards:
            t = np.empty(1, dtype=np.float64)
            check(lib.pb200_density_trace(s._handle, 0, 1, _p(t)))
            out.append(float(t[0]))
        return out

    def density_occupation(self, digit: int, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``Tr(|digit><digit|_k rho)``, ``[1, N]``."""
        self._one(traj0, count)
        total = np.zeros((1, self.n), dtype=np.float64)
        for s in self.shards:
            out = np.empty((1, self.n), dtype=np.float64)
            check(lib.pb200_density_occupation(s._handle, 0, 1, int(digit), _p(out)))
            total += out
        return total

    def density_correlation(self, digit: int, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``Tr(n_i n_j rho)`` with ``n_k = |digit><digit|_k``, ``[1, N, N]``."""
        self._one(traj0, count)
        total = np.zeros((1, self.n, self.n), dtype=np.float64)
        for s in self.shards:
            out = np.empty((1, self.n, self.n), dtype=np.float64)
            check(lib.pb200_density_correlation(s._handle, 0, 1, int(digit), _p(out)))
            total += out
        return total

    def density_expect(self, terms, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``Tr(O rho)`` (complex) of an operator given as monomial terms, ``[1]``."""
        self._one(traj0, count)
        if (terms.n, terms.d) != (self.n, 2):
            raise ValueError(f"operator on {terms.n} qudits of dimension {terms.d}, the plan holds {self.n} of 2")
        total = 0j
        for s in self.shards:
            out = np.empty(2, dtype=np.float64)
            check(lib.pb200_density_expect(s._handle, 0, 1, C.byref(terms.c_desc()), _p(out)))
            total += complex(out[0], out[1])
        return np.array([total])

    def _ham_on(self, ham_plan: DevicePlan, device: int) -> DevicePlan:
        """``ham_plan`` itself on its own device, else a copy of it on ``device`` (made once)."""
        if getattr(ham_plan, "device", None) == device:
            return ham_plan
        key = (id(ham_plan), device)
        if key not in self._ham:
            self._ham[key] = DevicePlan(ham_plan.specs, ham_plan.interp_order, device)
        return self._ham[key]

    def density_energy(self, ham_plan: DevicePlan, t_us: float, traj0: int = 0,
                       count: int | None = None) -> tuple[np.ndarray, np.ndarray]:
        """``(Tr(H rho), Tr(H^2 rho))`` with ``H = H(t_us)`` of the single-state plan ``ham_plan`` (copied once to every
        other device that holds a shard)."""
        self._one(traj0, count)
        e_tot, e2_tot = 0.0, 0.0
        for s, dev in zip(self.shards, self.devices):
            e = np.empty(1, dtype=np.float64)
            e2 = np.empty(1, dtype=np.float64)
            check(lib.pb200_density_energy(s._handle, self._ham_on(ham_plan, dev)._handle, float(t_us), 0, 1, _p(e),
                                           _p(e2)))
            e_tot += float(e[0]); e2_tot += float(e2[0])
        return np.array([e_tot]), np.array([e2_tot])

    def density_overlap(self, phi: np.ndarray, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``<phi|rho|phi>`` (complex) for a host ket ``phi`` of D amplitudes, ``[1]``."""
        self._one(traj0, count)
        v = np.ascontiguousarray(np.asarray(phi, dtype=np.complex128).reshape(-1))
        if v.shape[0] != self.D:
            raise ValueError(f"state of length {v.shape[0]}, expected {self.D}")
        total = 0j
        for s in self.shards:
            out = np.empty(2, dtype=np.float64)
            check(lib.pb200_density_overlap(s._handle, 0, 1, _p(v.view(np.float64)), _p(out)))
            total += complex(out[0], out[1])
        return np.array([total])

    def density_sample(self, n_samples: int, one_state: str, traj: int = 0) -> "Counter[str]":
        """Bitstring shots from ``diag rho`` with the recipe of ``LindbladPlan.density_sample``: one
        ``np.random.rand(n)`` call, each shot routed to a shard by the shards' partial traces in bitstring order
        (``sharded.route_shots``), then searched in that shard's cumulative weights."""
        from collections import Counter

        from .sharded import global_bitstring, route_shots

        self._one(traj, None)
        u = np.random.rand(n_samples)
        one = self.specs[0].eigenbasis.index(one_state)
        shard, block, local_u = route_shots(u, np.array(self._shard_traces()), reverse=(one == 0))
        local_b = np.zeros(n_samples, dtype=np.int64)
        for i, s in enumerate(self.shards):
            sel = np.nonzero(shard == i)[0]
            if sel.size == 0:
                continue
            ui = np.ascontiguousarray(local_u[sel], dtype=np.float64)
            idx = np.empty(sel.size, dtype=np.int64)
            check(lib.pb200_density_sample(s._handle, 0, one, _p(ui), int(sel.size),
                                           idx.ctypes.data_as(C.POINTER(C.c_int64))))
            local_b[sel] = idx
        b = global_bitstring(block, local_b, self.n - self.bits)
        return Counter(np.binary_repr(int(i), self.n) for i in b)
