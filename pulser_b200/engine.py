"""Python face of the C-ABI plan: one ``HamiltonianSpec`` (or a batch of
trajectories sharing its structure) -> device plan -> propagate.

This is the host-side replacement of ``Hamiltonian(...)`` construction
(reference ``pulser-simulation/pulser_simulation/simulation.py:299-311``) and
of the ``qutip.sesolve`` call (``simulation.py:729-735``).  All arithmetic
happens in ``libpulser_b200.so`` on the GPU; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
from typing import TYPE_CHECKING, Sequence

import numpy as np

from . import _lib
from ._lib import PlanDesc, RunOpts, RunStats, check, lib
from .spec import BASIS_ROLES, DriveTable, HamiltonianSpec

if TYPE_CHECKING:
    from .opterms import OpTerms

_dp = C.POINTER(C.c_double)


def _p(a: np.ndarray):
    return a.ctypes.data_as(_dp)


def all_ground_index(spec: HamiltonianSpec) -> int:
    """Index of the all-ground product state (``simulation.py:498-505``)."""
    eig = spec.eigenbasis
    g = eig.index("u") if spec.interaction_type == "XY" else eig.index("g")
    idx = 0
    for _ in range(spec.n_qudits):
        idx = idx * spec.dim + g
    return idx


def _with_common_drives(specs: list[HamiltonianSpec]) -> list[HamiltonianSpec]:
    """Give every trajectory of a batch the same ordered list of addressed bases.

    ``spec_from_pulser`` only creates a table for a basis whose samples are non-zero in that trajectory (the
    reference skips all-zero terms the same way, ``hamiltonian.py:353-395``), so a state-preparation error that
    removes the only atoms a channel addresses leaves that trajectory with fewer drives than its batch mates.  A
    missing basis is an all-zero table: the Hamiltonian is unchanged and the batch shares one kernel geometry.
    """
    import copy

    order: list[str] = []
    for s in specs:
        for d in s.drives:
            if d.basis not in order:
                order.append(d.basis)
    if all([d.basis for d in s.drives] == order for s in specs):
        return specs
    out = []
    for s in specs:
        have = {d.basis: d for d in s.drives}
        nt = len(s.sampling_times)
        drives = [
            have.get(b) or DriveTable(b, np.zeros((s.n_qudits, nt), dtype=np.complex128),
                                      np.zeros((s.n_qudits, nt), dtype=np.float64), True)
            for b in order
        ]
        s2 = copy.copy(s)
        s2.drives = drives
        out.append(s2)
    return out


class DevicePlan:
    """A batch of trajectories of one sequence resident on one GPU.

    ``shard=(bits, index)``: the plan holds shard ``index`` of ``2**bits`` of one state
    (``pb200_plan_create_shard``): the ``D = 2**(N - bits)`` amplitudes whose top ``bits`` qubits
    equal ``index``.  Shards are driven together by ``pulser_b200.sharded.ShardedPlan``.
    """

    def __init__(
        self,
        specs: HamiltonianSpec | Sequence[HamiltonianSpec],
        interp_order: int = 3,
        device: int = 0,
        shard: tuple[int, int] | None = None,
    ) -> None:
        if isinstance(specs, HamiltonianSpec):
            specs = [specs]
        specs = _with_common_drives(list(specs))
        s0 = specs[0]
        self._xy = s0.interaction_type == "XY"
        self._slm = s0.slm_coefficient()
        for s in specs[1:]:
            c = s.slm_coefficient()
            if (c is None) != (self._slm is None) or (
                c is not None and (not np.array_equal(c, self._slm) or list(s.slm_targets) != list(s0.slm_targets))
            ):
                raise ValueError("trajectories must share the SLM mask")
        for s in specs[1:]:
            if (
                s.n_qudits != s0.n_qudits
                or s.eigenbasis != s0.eigenbasis
                or len(s.drives) != len(s0.drives)
                or [d.basis for d in s.drives] != [d.basis for d in s0.drives]
                or not np.array_equal(s.sampling_times, s0.sampling_times)
            ):
                raise ValueError("trajectories must share basis, drives, times")
        self.specs = specs
        self.spec = s0
        self.n_traj = len(specs)
        self.n = s0.n_qudits
        self.dim = s0.dim
        self.shard = None if shard is None else (int(shard[0]), int(shard[1]))
        self.D = s0.hilbert_dim if shard is None else s0.hilbert_dim >> self.shard[0]
        self.interp_order = interp_order
        self.device = device
        self._handle = C.c_void_p()
        times = np.ascontiguousarray(s0.sampling_times, dtype=np.float64)
        desc = PlanDesc()
        desc.n_qudits = self.n
        desc.dim = self.dim
        desc.n_times = len(times)
        desc.interp_order = interp_order
        desc.n_drives = len(s0.drives)
        any_inter = any(s.has_interaction() for s in specs)
        # XY mode: the |uu><uu| van der Waals term sits on |u> (hamiltonian.py:276-294)
        ryd = "u" if self._xy else "r"
        desc.rydberg_state = s0.eigenbasis.index(ryd) if any_inter else -1
        desc.n_traj = self.n_traj
        desc.device = device
        desc.sampling_times = _p(times)
        self._uniform = []
        for q, d in enumerate(s0.drives):
            to, frm = BASIS_ROLES[d.basis]
            desc.drives[q].state_to = s0.eigenbasis.index(to)
            desc.drives[q].state_from = s0.eigenbasis.index(frm)
            uni = all(s.drives[q].uniform for s in specs)
            desc.drives[q].uniform = int(uni)
            self._uniform.append(uni)
        if self.shard is None:
            check(lib.pb200_plan_create(C.byref(self._handle), C.byref(desc)))
        else:
            check(lib.pb200_plan_create_shard(C.byref(self._handle), C.byref(desc), *self.shard))
        try:
            self._upload(any_inter)
        except Exception:
            self.close()
            raise

    # ------------------------------------------------------------------
    def _upload(self, any_inter: bool) -> None:
        specs = self.specs
        n, nt = self.n, len(self.spec.sampling_times)
        if self._slm is not None and any_inter:
            # XY + SLM mask (hamiltonian.py:399-424): must precede the interaction matrices, which it splits
            masked = np.zeros(n, dtype=np.uint8)
            masked[list(self.spec.slm_targets)] = 1
            coeff = np.ascontiguousarray(self._slm, dtype=np.float64)
            check(lib.pb200_plan_set_slm_mask(self._handle, masked.ctypes.data_as(C.POINTER(C.c_uint8)), _p(coeff)))
        if any_inter:
            mats = [s.pair_matrix() for s in specs]
            shared = all(np.array_equal(m, mats[0]) for m in mats[1:])
            if shared:
                U = np.ascontiguousarray(mats[0], dtype=np.float64)
                check(lib.pb200_plan_set_interaction(self._handle, 0, 1, _p(U), None, 1))
            else:
                U = np.ascontiguousarray(np.stack(mats), dtype=np.float64)
                check(
                    lib.pb200_plan_set_interaction(
                        self._handle, 0, self.n_traj, _p(U), None, 0
                    )
                )
        if any_inter and self._xy:
            mats = [s.xy_matrix() for s in specs]
            iu, idn = self.spec.eigenbasis.index("u"), self.spec.eigenbasis.index("d")
            shared = all(np.array_equal(m, mats[0]) for m in mats[1:])
            U = np.ascontiguousarray(mats[0] if shared else np.stack(mats), dtype=np.float64)
            check(
                lib.pb200_plan_set_xy(
                    self._handle, 0, 1 if shared else self.n_traj, _p(U), None, int(shared), iu, idn
                )
            )
        for q, uni in enumerate(self._uniform):
            rows = 1 if uni else n
            # chunk the upload to bound host memory
            chunk = max(1, (64 << 20) // (rows * nt * 24))
            for b0 in range(0, self.n_traj, chunk):
                part = specs[b0 : b0 + chunk]
                coef = np.ascontiguousarray(
                    np.stack([s.drives[q].coef[:rows] for s in part]),
                    dtype=np.complex128,
                )
                det = np.ascontiguousarray(
                    np.stack([s.drives[q].det[:rows] for s in part]),
                    dtype=np.float64,
                )
                check(
                    lib.pb200_plan_set_drive(
                        self._handle, q, b0, len(part),
                        _p(coef.view(np.float64)), _p(det),
                    )
                )

    # ------------------------------------------------------------------
    def close(self) -> None:
        if self._handle:
            lib.pb200_plan_destroy(self._handle)
            self._handle = C.c_void_p()

    def __del__(self) -> None:  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self) -> "DevicePlan":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def set_collapse(self, ops: np.ndarray, seed: int = 0) -> None:
        """Switch the plan to wave-function Monte Carlo with single-qudit collapse
        operators ``ops[n_ops, d, d]`` acting on every qudit (``pb200_plan_set_collapse``)."""
        ops = np.ascontiguousarray(ops, dtype=np.complex128)
        check(lib.pb200_plan_set_collapse(self._handle, ops.shape[0], _p(ops.view(np.float64)), C.c_uint64(seed)))

    def jump_counts(self) -> np.ndarray:
        out = np.zeros(self.n_traj, dtype=np.int64)
        check(lib.pb200_plan_jump_counts(self._handle, out.ctypes.data_as(C.POINTER(C.c_int64))))
        return out

    def set_stream(self, cuda_stream: int) -> None:
        check(lib.pb200_plan_set_stream(self._handle, C.c_void_p(cuda_stream)))

    # ------------------------------------------------------------------
    def set_state(self, psi: np.ndarray | str = "all-ground") -> None:
        """Same state for every trajectory, or ``psi[n_traj, D]``."""
        if isinstance(psi, str):
            if psi != "all-ground":
                raise ValueError(psi)
            check(
                lib.pb200_state_set(
                    self._handle, 0, self.n_traj, None, all_ground_index(self.spec), 0
                )
            )
            return
        psi = np.ascontiguousarray(psi, dtype=np.complex128)
        if psi.size == self.D:
            check(
                lib.pb200_state_set(
                    self._handle, 0, self.n_traj, _p(psi.reshape(-1).view(np.float64)), -1, 1
                )
            )
        elif psi.size == self.D * self.n_traj:
            check(
                lib.pb200_state_set(
                    self._handle, 0, self.n_traj, _p(psi.reshape(-1).view(np.float64)), -1, 0
                )
            )
        else:
            raise ValueError(
                "Incompatible shape of initial state."
                + f"Expected {self.D}, got {psi.shape[0]}."
            )

    def get_state(self, traj0: int = 0, count: int | None = None) -> np.ndarray:
        count = self.n_traj - traj0 if count is None else count
        out = np.empty((count, self.D), dtype=np.complex128)
        check(lib.pb200_state_get(self._handle, traj0, count, _p(out.view(np.float64))))
        return out

    def probabilities(self, traj0: int = 0, count: int | None = None) -> np.ndarray:
        count = self.n_traj - traj0 if count is None else count
        out = np.empty((count, self.D), dtype=np.float64)
        check(lib.pb200_state_probabilities(self._handle, traj0, count, _p(out)))
        return out

    def norm2(self) -> np.ndarray:
        out = np.empty(self.n_traj, dtype=np.float64)
        check(lib.pb200_state_norm2(self._handle, 0, self.n_traj, _p(out)))
        return out

    def occupation(self, digit: int, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """Per-qudit population of eigenstate ``digit``, ``[count, N]`` (device reduction)."""
        count = self.n_traj - traj0 if count is None else count
        out = np.empty((count, self.n), dtype=np.float64)
        check(lib.pb200_state_occupation(self._handle, traj0, count, int(digit), _p(out)))
        return out

    def correlation(self, digit: int, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``<n_i n_j>`` with ``n_k = |digit><digit|``, ``[count, N, N]`` (device reduction;
        CorrelationMatrix observable, ``pulser/backend/default_observables.py:331-394``)."""
        count = self.n_traj - traj0 if count is None else count
        out = np.empty((count, self.n, self.n), dtype=np.float64)
        check(lib.pb200_state_correlation(self._handle, traj0, count, int(digit), _p(out)))
        return out

    def energy(self, t_us: float) -> tuple[np.ndarray, np.ndarray]:
        """``(<H(t)>, <H(t)^2>)`` of every trajectory, one H-apply + one fused dot on the
        device (Energy / EnergyVariance / EnergySecondMoment, ``default_observables.py:431-561``)."""
        e = np.empty(self.n_traj, dtype=np.float64)
        e2 = np.empty(self.n_traj, dtype=np.float64)
        check(lib.pb200_state_energy(self._handle, float(t_us), _p(e), _p(e2)))
        return e, e2

    def overlap(self, phi: np.ndarray, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``<phi|psi_b>`` (complex) for the selected trajectories (Fidelity observable)."""
        count = self.n_traj - traj0 if count is None else count
        v = np.ascontiguousarray(np.asarray(phi, dtype=np.complex128).reshape(-1))
        if v.shape[0] != self.D:
            raise ValueError(f"state of length {v.shape[0]}, expected {self.D}")
        out = np.empty((count, 2), dtype=np.float64)
        check(lib.pb200_state_overlap(self._handle, traj0, count, _p(v.view(np.float64)), _p(out)))
        return out[:, 0] + 1j * out[:, 1]

    def expect_terms(self, terms: "OpTerms", traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``<psi_b|O|psi_b>`` (complex, not normalised) for the selected trajectories, with ``O`` given as monomial
        terms (``pulser_b200.opterms.OpTerms``), matrix-free on the device (``pb200_state_expect``)."""
        count = self.n_traj - traj0 if count is None else count
        if (terms.n, terms.d) != (self.n, self.dim):
            raise ValueError(f"operator on {terms.n} qudits of dimension {terms.d}, the plan holds {self.n} of {self.dim}")
        out = np.empty((count, 2), dtype=np.float64)
        check(lib.pb200_state_expect(self._handle, traj0, count, C.byref(terms.c_desc()), _p(out)))
        return out[:, 0] + 1j * out[:, 1]

    def copy_state_from(self, other: "DevicePlan", src_traj: int = 0, dst_traj: int = 0) -> None:
        """Device-to-device copy of one trajectory's current state of ``other`` into this plan
        (``pb200_state_copy``)."""
        check(lib.pb200_state_copy(self._handle, dst_traj, other._handle, src_traj))

    def sample(self, n_samples: int, one_state: str, traj: int = 0) -> "Counter[str]":
        """Bitstring samples of trajectory ``traj`` drawn on the device with the
        reference's recipe and the global ``np.random`` stream
        (``qutip_result.py:101-158`` + ``pulser/math/multinomial.py:17-36``)."""
        from collections import Counter

        u = np.ascontiguousarray(np.random.rand(n_samples), dtype=np.float64)
        idx = np.empty(n_samples, dtype=np.int64)
        check(
            lib.pb200_state_sample(
                self._handle, traj, self.spec.eigenbasis.index(one_state), _p(u), n_samples,
                idx.ctypes.data_as(C.POINTER(C.c_int64)),
            )
        )
        return Counter(np.binary_repr(int(i), self.n) for i in idx)

    def device_ptr(self) -> int:
        ptr = C.c_void_p()
        check(lib.pb200_state_device_ptr(self._handle, C.byref(ptr)))
        return int(ptr.value)

    # ------------------------------------------------------------------
    def propagate(
        self,
        t_start: float,
        t_stop: float,
        max_step: int = 0,
        refine_window: int = -1,
        cheb_tol: float = 0.0,
        rough_tol: float = 0.0,
        magnus_order: int = 4,
        tol: float = 0.0,
        check_every: int = 0,
        extrapolate: int = 0,
        integrator: int = 0,
    ) -> dict:
        """Advance all trajectories from ``t_start`` to ``t_stop`` (us).

        ``tol > 0`` (default 1e-9): adaptive Magnus steps with step-doubling
        error control; ``tol < 0``: fixed steps of ``max_step`` samples.
        """
        opts = RunOpts(max_step, refine_window, cheb_tol, rough_tol, magnus_order, check_every, tol, extrapolate, integrator)
        st = RunStats()
        check(
            lib.pb200_propagate(
                self._handle, float(t_start), float(t_stop), C.byref(opts), C.byref(st)
            )
        )
        return {f: getattr(st, f) for f, _ in RunStats._fields_}

    def apply_h(self, t_us: float, vec: np.ndarray, traj: int = 0) -> np.ndarray:
        vec = np.ascontiguousarray(vec, dtype=np.complex128).reshape(-1)
        if vec.size != self.D:
            raise ValueError("vector has the wrong dimension")
        out = np.empty(self.D, dtype=np.complex128)
        check(
            lib.pb200_apply_h(
                self._handle, traj, float(t_us), _p(vec.view(np.float64)), _p(out.view(np.float64))
            )
        )
        return out

    def coefficients_at(self, t_us: float, drive: int = 0, row: int = 0, traj: int = 0):
        out = np.empty(3)
        check(lib.pb200_coefficients_at(self._handle, traj, drive, row, float(t_us), _p(out)))
        return complex(out[0], out[1]), float(out[2])

    def bench_apply(self, t_us: float, reps: int) -> tuple[float, int]:
        ms = C.c_double()
        n = C.c_int64()
        check(lib.pb200_bench_apply(self._handle, float(t_us), reps, C.byref(ms), C.byref(n)))
        return ms.value, n.value


def device_count() -> int:
    return int(_lib.lib.pb200_device_count())
