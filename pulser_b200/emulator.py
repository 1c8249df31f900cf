"""``B200Emulator``: the ``QutipEmulator`` surface on top of the CUDA path.

Drop-in for ``pulser_simulation.QutipEmulator``
(reference ``pulser-simulation/pulser_simulation/simulation.py:84-1051``):
same constructor / ``from_sequence`` / ``run`` / ``set_initial_state`` /
``set_evaluation_times`` / ``get_hamiltonian`` / properties, same validation
messages, same evaluation-time and trajectory semantics.  Everything upstream
of the Hamiltonian (sampling, noise trajectories, interaction matrix) is the
reference's own pulser-core code; ``Hamiltonian(...)`` construction
(``simulation.py:299-311``) and ``_run_solver`` (``:689-766``) are replaced by
``HamiltonianSpec`` -> ``DevicePlan`` -> ``pb200_propagate``.

Collapse operators (``simulation.py:705-735``) run as a master equation on the
vectorised density matrix (``lindblad.py``, registers with dim^(2N) <= 2^26) and
as Monte-Carlo wave functions beyond that (``n_trajectories`` set).  XY mode runs
the same paths (SLM mask included: ``pb200_plan_set_slm_mask``).
"""
from __future__ import annotations

import warnings
from collections import Counter
from enum import Enum
from typing import Any, Iterator, Optional, Union

import numpy as np

from ._compat import ensure_pulser
from .results import (
    B200Result,
    CoherentResults,
    DensityMatrix,
    NoisyResults,
    SampledCounts,
    StateVector,
)
from .spec import HamiltonianSpec, spec_from_pulser

if not ensure_pulser():  # pragma: no cover
    raise ImportError(
        "pulser_b200.emulator needs pulser-core (set PULSER_B200_PULSER_PATH or "
        "install pulser-core); the plain-array path is pulser_b200.engine."
    )

import pulser.sampler as sampler  # noqa: E402
from pulser import Sequence  # noqa: E402
from pulser._hamiltonian_data import (  # noqa: E402
    HamiltonianData,
    has_shot_to_shot_except_spam,
)
from pulser.devices._device_datacls import BaseDevice  # noqa: E402
from pulser.noise_model import NoiseModel  # noqa: E402
from pulser.register.base_register import BaseRegister  # noqa: E402
from pulser.sampler.samples import ChannelSamples, SequenceSamples  # noqa: E402


def _has_stochastic_noise(noise_model: NoiseModel) -> bool:
    """simulation.py:61-64."""
    return has_shot_to_shot_except_spam(noise_model) or (
        "SPAM" in noise_model.noise_types and noise_model.state_prep_error != 0
    )


class Solver(str, Enum):
    """simulation.py:67-81 (kept for signature compatibility)."""

    DEFAULT = "default"
    MESOLVER = "MasterEquation"
    MCSOLVER = "MonteCarlo"


# QuTiP solver options the reference forwards (simulation.py:800-845); they
# have no meaning for the fixed-order propagator and are accepted and ignored.
_QUTIP_OPTIONS = {
    "max_step", "nsteps", "atol", "rtol", "method", "order", "min_step",
    "first_step", "store_states", "store_final_state", "normalize_output",
    "progress_kwargs", "keep_runs_results", "map", "num_cpus", "timeout",
    "norm_steps", "norm_t_tol", "norm_tol", "mc_corr_eps", "improved_sampling",
}
# options of this backend
_B200_OPTIONS = {"b200_max_step", "b200_cheb_tol", "b200_refine_window", "b200_batch", "b200_tol"}


class _PendingTrajectories:
    """Lazy list of ``(HamiltonianSpec, reps)`` of a noisy run: entry ``k`` is built from noise trajectory
    ``entries[k][0]`` the way ``HamiltonianData.noisy_samples`` builds it
    (``pulser/_hamiltonian_data/hamiltonian_data.py:536-545``) when it is indexed, and not before."""

    def __init__(self, sim: "B200Emulator", hd: Any, entries: list) -> None:
        self._sim, self._hd, self._entries = sim, hd, entries
        self._last: tuple[int, HamiltonianSpec] | None = None

    def __len__(self) -> int:
        return len(self._entries)

    def _make(self, k: int) -> tuple[HamiltonianSpec, int]:
        index, reps = self._entries[k]
        if self._last is None or self._last[0] != index:
            traj = self._hd.noise_trajectories[index].trajectory
            self._last = (index, self._sim._spec_of(self._hd, traj, self._hd._sample_with_trajectory(traj)))
        return self._last[1], reps

    def __getitem__(self, key: Any) -> Any:
        if isinstance(key, slice):
            return [self._make(k) for k in range(*key.indices(len(self._entries)))]
        return self._make(key if key >= 0 else len(self._entries) + key)

    def __iter__(self) -> Iterator[tuple[HamiltonianSpec, int]]:
        return (self._make(k) for k in range(len(self._entries)))

    def batches(self, batch: int) -> Iterator[list]:
        """Chunks of ``batch`` entries; the specs of the NEXT chunk are assembled by a helper thread while the
        caller's current chunk is on the GPU (``pb200_propagate`` runs without the GIL), so the per-trajectory host
        work -- pulser-core's sample rebuilding and the spec extraction, ~20 ms per 16-atom trajectory -- is off
        the critical path (SURVEY section 8f row 1).  Building a spec draws no random numbers."""
        from concurrent.futures import ThreadPoolExecutor

        n = len(self._entries)
        if n == 0:
            return
        build = lambda b0: [self._make(k) for k in range(b0, min(b0 + batch, n))]  # noqa: E731
        with ThreadPoolExecutor(max_workers=1) as pool:
            pending = pool.submit(build, 0)
            for b0 in range(0, n, batch):
                chunk = pending.result()
                if b0 + batch < n:
                    pending = pool.submit(build, b0 + batch)
                yield chunk


class _NoiseModelConfig:
    """Minimal SimConfig stand-in (``noise``, ``supported_noises``, ``to_noise_model``) used by ``add_config`` /
    ``reset_config`` when ``pulser_simulation.simconfig`` (QuTiP) cannot be imported."""

    def __init__(self, noise_model: NoiseModel, like: Any) -> None:
        self._nm = noise_model
        self.noise = tuple(noise_model.noise_types)
        from pulser._hamiltonian_data.hamiltonian_data import SUPPORTED_NOISES  # type: ignore

        self.supported_noises = getattr(like, "supported_noises", None) or SUPPORTED_NOISES

    def to_noise_model(self) -> NoiseModel:
        return self._nm


class B200Emulator:
    r"""Emulator of a pulse sequence on an H100 GPU.

    Args: identical to ``QutipEmulator`` (simulation.py:84-141), plus
        ``interp_order`` (QobjEvo coefficient interpolation order, 3 = QuTiP 5
        default) and ``gpu`` (CUDA device ordinal).
    """

    def __init__(
        self,
        sampled_seq: SequenceSamples,
        register: BaseRegister,
        device: BaseDevice,
        sampling_rate: float = 1.0,
        config: Any = None,
        evaluation_times: Union[float, str, Any] = "Full",
        noise_model: NoiseModel | None = None,
        solver: Solver = Solver.DEFAULT,
        n_trajectories: int | None = None,
        *,
        interp_order: int = 3,
        gpu: int = 0,
    ) -> None:
        if not isinstance(sampled_seq, SequenceSamples):
            raise TypeError(
                "The provided sequence has to be a valid "
                "SequenceSamples instance."
            )
        if sampled_seq.max_duration == 0:
            raise ValueError("SequenceSamples is empty.")
        self._sampling_rate = sampling_rate
        device.validate_register(register)
        self._register = register
        self.solver = Solver(solver)
        if sampled_seq._slm_mask.end > 0 and not device.supports_slm_mask:
            raise ValueError("Samples use SLM mask but device does not have one.")
        if not sampled_seq.used_bases <= device.supported_bases:
            raise ValueError("Bases used in samples should be supported by device.")
        if not sampled_seq._slm_mask.targets <= set(register.qubit_ids):
            raise ValueError(
                "The ids of qubits targeted in SLM mask"
                " should be defined in register."
            )
        self._tot_duration = sampled_seq.max_duration
        self.samples_obj = sampled_seq.extend_duration(self._tot_duration + 1)
        self._n_trajectories = n_trajectories
        if not (0 < sampling_rate <= 1.0):
            raise ValueError(
                "The sampling rate (`sampling_rate` = "
                f"{sampling_rate}) must be greater than 0 and "
                "less than or equal to 1."
            )
        if int(self._tot_duration * sampling_rate) < 4:
            raise ValueError("`sampling_rate` is too small, less than 4 data points.")
        if noise_model is not None and config is not None:
            raise ValueError(
                "'noise_model' and 'config' cannot both be provided to "
                "'QutipEmulator'. Please provide just a 'noise_model'."
            )
        if config is not None:
            warnings.warn(
                "Supplying a 'SimConfig' to QutipEmulator has been "
                "deprecated. Please instantiate with a 'NoiseModel' "
                "instead.",
                DeprecationWarning,
                stacklevel=2,
            )
            noise_model = config.to_noise_model()
        if not noise_model:
            noise_model = NoiseModel()
        self._interp_order = interp_order
        self._gpu = gpu
        self._noise_trajectories_used = False
        self._hamiltonian_data = HamiltonianData(
            self.samples_obj,
            register,
            device,
            noise_model,
            self._get_n_trajectories(noise_model, check_value=True),
        )
        self._current_spec = next(self._specs)[0]
        self._noiseless_cache: dict[bool, HamiltonianSpec] = {}
        self._eval_times_array: np.ndarray
        self.set_evaluation_times(evaluation_times)
        if self.samples_obj._measurement:
            self._meas_basis = self.samples_obj._measurement
        else:
            if "all" in self.basis_name:
                self._meas_basis = "digital"
            else:
                self._meas_basis = self.basis_name.replace("_with_error", "")
        self.set_initial_state("all-ground")
        self.last_run_stats: dict = {}

    # ------------------------------------------------------------------
    def _get_n_trajectories(self, noise_model: NoiseModel, check_value: bool) -> int | None:
        n_trajectories = (
            self._n_trajectories if self._n_trajectories is not None else noise_model.runs
        )
        if check_value and _has_stochastic_noise(noise_model) and n_trajectories is None:
            raise ValueError(
                "'n_trajectories' must be defined when the NoiseModel contains"
                " stochastic noise, which is the case for the given noise "
                f"model: {noise_model!r}"
            )
        return n_trajectories

    @property
    def n_trajectories(self) -> int | None:
        return self._get_n_trajectories(self.noise_model, check_value=False)

    @property
    def device(self) -> BaseDevice:
        return self._hamiltonian_data.device

    def _spec_of(self, hd: HamiltonianData, traj: Any, noisy_samples: Any) -> HamiltonianSpec:
        return spec_from_pulser(
            noisy_samples, traj, hd.basis_data, hd.lindblad_data,
            self._sampling_rate, self._tot_duration,
        )

    @property
    def _specs(self) -> Iterator[tuple[HamiltonianSpec, int]]:
        """One spec per noise trajectory (replaces ``_hamiltonians``, :299-311)."""
        hd = self._hamiltonian_data
        for traj, noisy_samples, reps in hd.noisy_samples:
            yield self._spec_of(hd, traj, noisy_samples), reps

    def _noiseless_spec(self, leakage: bool = False) -> HamiltonianSpec:
        """Spec of the noiseless Hamiltonian handed to observables (``_get_noiseless_hamiltonian``,
        simulation.py:266-297): with ``leakage`` the operator lives in the 3-level basis of the leakage run, which
        the reference obtains from a NoiseModel carrying a zero effective-noise operator."""
        leakage = bool(leakage)
        if leakage not in self._noiseless_cache:
            if leakage:
                dim = self._hamiltonian_data.basis_data.dim
                noise = NoiseModel(eff_noise_opers=(np.zeros((dim, dim)),), eff_noise_rates=(0.0,), with_leakage=True)
            else:
                noise = NoiseModel()
            hd = HamiltonianData(self.samples_obj, self._register, self.device, noise, n_trajectories=1)
            self._noiseless_cache[leakage] = self._spec_of(hd, hd.noise_trajectories[0].trajectory, hd.samples)
        return self._noiseless_cache[leakage]

    @property
    def sampling_times(self) -> np.ndarray:
        return self._noiseless_spec().sampling_times

    @property
    def dim(self) -> int:
        return self._hamiltonian_data.basis_data.dim

    @property
    def basis_name(self) -> str:
        return self._hamiltonian_data.basis_data.basis_name

    @property
    def basis(self) -> dict[str, StateVector]:
        eig = self._hamiltonian_data.basis_data.eigenbasis
        return {s: StateVector(np.eye(len(eig))[i]) for i, s in enumerate(eig)}

    @property
    def noise_model(self) -> NoiseModel:
        return self._hamiltonian_data.noise_model

    @property
    def total_duration_ns(self) -> int:
        return self._tot_duration

    # ---- deprecated SimConfig interface (simulation.py:338-477) ---------------------------------
    @staticmethod
    def _simconfig_class() -> Any:
        """``pulser_b200.simconfig.SimConfig``: the reference class without its qutip import."""
        from .simconfig import SimConfig

        return SimConfig

    @property
    def config(self) -> Any:
        """The current configuration, as a SimConfig instance (``simulation.py:338-341``)."""
        return self._simconfig_class().from_noise_model(self._hamiltonian_data.noise_model)

    def _noise_model_of_config(self, cfg: Any, invalid_suffix: str, list_prefix: str) -> NoiseModel:
        """Common front door of the deprecated SimConfig setters: deprecation warning, duck-type check
        (``noise`` / ``supported_noises`` / ``to_noise_model``) and the interaction-mode support check, with the
        reference's messages (``simulation.py:359-382`` and ``:431-451`` differ only in punctuation)."""
        warnings.warn(
            "Supplying a 'SimConfig' to QutipEmulator has been deprecated."
            " Please instantiate with a 'NoiseModel' instead.",
            DeprecationWarning,
            stacklevel=3,
        )
        if not all(hasattr(cfg, a) for a in ("to_noise_model", "supported_noises", "noise")):
            raise ValueError(f"Object {cfg} is not a valid `SimConfig`{invalid_suffix}")
        mode = self._hamiltonian_data.basis_data.interaction_type
        unsupported = set(cfg.noise) - cfg.supported_noises[mode]
        if unsupported:
            raise NotImplementedError(
                f"Interaction mode '{mode}' does not support simulation of noise types:"
                f"{list_prefix}{', '.join(unsupported)}."
            )
        return cfg.to_noise_model()

    def _adopt_noise_model(self, noise_model: NoiseModel) -> None:
        """Rebuild the Hamiltonian data under a new noise model and keep or reset the initial state
        (``simulation.py:383-412``)."""
        dim_before = self.dim
        self._noise_trajectories_used = False
        self._hamiltonian_data = HamiltonianData(
            self.samples_obj, self._register, self.device, noise_model,
            self._get_n_trajectories(noise_model, check_value=True),
        )
        self._current_spec = next(self._specs)[0]
        self._noiseless_cache = {}
        if self.dim != dim_before:
            if not self._initial_is_ground:
                warnings.warn(
                    "Current initial state's dimension does not match new"
                    " dimensions. Setting it to 'all-ground'."
                )
            self.set_initial_state("all-ground")
        else:
            self.set_initial_state(self._initial_state)

    def set_config(self, cfg: Any) -> None:
        """Sets current config to cfg and updates simulation parameters (``simulation.py:348-412``; deprecated
        since v1.6 like the original).  ``cfg`` is duck-typed."""
        self._adopt_noise_model(self._noise_model_of_config(cfg, ".", ""))

    def add_config(self, config: Any) -> None:
        """Updates the current configuration with parameters of another one (``simulation.py:414-469``): noise
        types that are new get their parameters from ``config``, the ones already present keep theirs."""
        import dataclasses as _dc

        incoming = self._noise_model_of_config(config, "", " ")
        current = self._hamiltonian_data.noise_model
        added = set(incoming.noise_types) - set(current.noise_types)
        params = _dc.asdict(current)
        params.pop("noise_types")
        for name in NoiseModel._find_relevant_params(
            added, incoming.state_prep_error, incoming.amp_sigma, incoming.laser_waist
        ):
            params[name] = getattr(incoming, name)
        self._adopt_noise_model(NoiseModel(**params))

    def show_config(self, solver_options: bool = False) -> None:
        """Shows current configuration (``simulation.py:471-473``)."""
        print(self.config.__str__(solver_options))

    def reset_config(self) -> None:
        """Resets configuration to default (``simulation.py:475-477``)."""
        self.set_config(_NoiseModelConfig(NoiseModel(), None))

    # ---- operators (hamiltonian.py:145-244, simulation.py:601-623) -------------------------------
    @property
    def op_matrix(self) -> dict[str, Any]:
        """``"I"`` and the projectors ``sigma_ab = |a><b|`` of the eigenbasis, as sparse matrices."""
        import scipy.sparse as sp

        eig = list(self._hamiltonian_data.basis_data.eigenbasis)
        d = len(eig)
        ops: dict[str, Any] = {"I": sp.identity(d, dtype=complex, format="csr")}
        for i, a in enumerate(eig):
            for j, b in enumerate(eig):
                m = sp.lil_matrix((d, d), dtype=complex)
                m[i, j] = 1.0
                ops["sigma_" + a + b] = m.tocsr()
        return ops

    def build_operator(self, operations: Union[list, tuple]) -> Any:
        """Creates an operator with non-trivial actions on some qubits: ``[(operator_1, qubits_1), ...]`` gives the
        tensor product of ``operator_i`` on ``qubits_i`` and the identity elsewhere; ``(operator, 'global')`` the sum
        over all qubits.  ``operator``: a key of ``op_matrix``, an array or anything with ``full()``/``toarray()``.
        Returns a ``scipy.sparse`` matrix (accepted by ``SimulationResults.expect``)."""
        import scipy.sparse as sp

        qids = list(self._register.qubit_ids)
        qindex = {q: i for i, q in enumerate(qids)}
        op_matrix = self.op_matrix
        op_list = [op_matrix["I"] for _ in qids]
        if not isinstance(operations, list):
            operations = [operations]
        for operator, qubits in operations:
            if isinstance(qubits, str) and qubits == "global":
                total = None
                for q_id in qids:
                    term = self.build_operator([(operator, [q_id])])
                    total = term if total is None else total + term
                return total
            qubits_set = set(qubits)
            if len(qubits_set) < len(qubits):
                raise ValueError("Duplicate atom ids in argument list.")
            if not qubits_set.issubset(qindex.keys()):
                v = qubits_set - qindex.keys()
                raise ValueError("Invalid qubit names: " f"{v}")
            if isinstance(operator, str):
                try:
                    operator = op_matrix[operator]
                except KeyError:
                    raise ValueError(f"{operator} is not a valid operator")
            elif hasattr(operator, "full"):
                operator = sp.csr_matrix(np.asarray(operator.full(), dtype=complex))
            else:
                operator = sp.csr_matrix(operator, dtype=complex)
            for qubit in qubits:
                op_list[qindex[qubit]] = operator
        out = op_list[0]
        for m in op_list[1:]:
            out = sp.kron(out, m, format="csr")
        return sp.csr_matrix(out)

    def draw(
        self,
        draw_phase_area: bool = False,
        draw_phase_shifts: bool = False,
        draw_phase_curve: bool = False,
        fig_name: str | None = None,
        kwargs_savefig: dict = {},
    ) -> None:
        """Draws the samples of the sequence used for the emulation (``simulation.py:917-953``); needs matplotlib."""
        try:
            import matplotlib.pyplot as plt
            from pulser._seq_drawer import draw_samples
        except Exception as exc:  # pragma: no cover - plotting stack absent
            raise ImportError("draw() needs matplotlib and pulser's sequence drawer") from exc
        if type(getattr(plt, "__loader__", None)).__name__ == "_StubLoader":
            raise ImportError("draw() needs matplotlib (pulser_b200._compat installed a stub because it is absent)")
        draw_samples(
            self.samples_obj,
            self._register,
            self._sampling_rate,
            draw_phase_area=draw_phase_area,
            draw_phase_shifts=draw_phase_shifts,
            draw_phase_curve=draw_phase_curve,
        )
        if fig_name is not None:
            plt.savefig(fig_name, **kwargs_savefig)
        plt.show()

    # ------------------------------------------------------------------
    @property
    def initial_state(self) -> StateVector:
        return self._initial_state

    def _all_ground(self) -> StateVector:
        hd = self._hamiltonian_data
        eig = hd.basis_data.eigenbasis
        g = eig.index("u" if hd.basis_data.interaction_type == "XY" else "g")
        d, n = hd.basis_data.dim, hd.n_qudits
        idx = 0
        for _ in range(n):
            idx = idx * d + g
        psi = np.zeros(d**n, dtype=complex)
        psi[idx] = 1.0
        return StateVector(psi, [[d] * n, [1] * n])

    def set_initial_state(self, state: Union[str, np.ndarray, Any]) -> None:
        """simulation.py:484-525."""
        hd = self._hamiltonian_data
        if isinstance(state, str) and state == "all-ground":
            self._initial_state = self._all_ground()
            self._initial_is_ground = True
            return
        arr = state.full() if hasattr(state, "full") else np.asarray(state)
        shape = arr.shape[0]
        legal_shape = hd.basis_data.dim**hd.n_qudits
        if shape != legal_shape:
            raise ValueError(
                "Incompatible shape of initial state."
                + f"Expected {legal_shape}, got {shape}."
            )
        d, n = hd.basis_data.dim, hd.n_qudits
        self._initial_state = StateVector(arr.reshape(-1), [[d] * n, [1] * n]).unit()
        self._initial_is_ground = self._initial_state == self._all_ground()

    @property
    def evaluation_times(self) -> np.ndarray:
        return np.array(self._eval_times_array)

    def set_evaluation_times(self, value: Union[str, Any, float]) -> None:
        """simulation.py:532-599."""
        times = self.sampling_times
        if isinstance(value, str):
            if value == "Full":
                eval_times = np.copy(times)
            elif value == "Minimal":
                eval_times = np.array([])
            else:
                raise ValueError(
                    "Wrong evaluation time label. It should "
                    "be `Full`, `Minimal`, an array of times or"
                    + " a float between 0 and 1."
                )
        elif isinstance(value, float):
            if value > 1 or value <= 0:
                raise ValueError("evaluation_times float must be between 0 and 1.")
            indices = np.linspace(0, len(times) - 1, int(value * len(times)), dtype=int)
            eval_times = times[indices]
        elif isinstance(value, (list, tuple, np.ndarray)):
            if np.max(value, initial=0) > self._tot_duration * 1e-3:
                raise ValueError(
                    "Provided evaluation-time list extends "
                    "further than sequence duration."
                )
            if np.min(value, initial=0) < 0:
                raise ValueError(
                    "Provided evaluation-time list contains negative values."
                )
            eval_times = np.array(value)
        else:
            raise ValueError(
                "Wrong evaluation time label. It should "
                "be `Full`, `Minimal`, an array of times or a "
                + "float between 0 and 1."
            )
        self._eval_times_array = np.union1d(eval_times, [0.0, self._tot_duration * 1e-3])
        self._eval_times_instruction = value

    # ------------------------------------------------------------------
    def get_hamiltonian(self, time: float, noiseless: bool = False) -> np.ndarray:
        """Dense H(t) in rad/us (simulation.py:625-661); small systems only.

        Built on the device by applying H(t) to the basis vectors (``pb200_apply_h``).
        """
        if time > self._tot_duration:
            raise ValueError(
                f"Provided time (`time` = {time}) must be "
                "less than or equal to the sequence duration "
                f"({self._tot_duration})."
            )
        if time < 0:
            raise ValueError(
                f"Provided time (`time` = {time}) must be "
                "greater than or equal to 0."
            )
        from .engine import DevicePlan

        spec = self._noiseless_spec() if noiseless else self._current_spec
        D = spec.hilbert_dim
        if D > 4096:
            raise ValueError("get_hamiltonian: dense matrix limited to 4096 states")
        H = np.zeros((D, D), dtype=complex)
        with DevicePlan(spec, self._interp_order, self._gpu) as plan:
            eye = np.eye(D, dtype=complex)
            for j in range(D):
                H[:, j] = plan.apply_h(time / 1000, eye[j])
        return H

    @staticmethod
    def _get_min_variation(ch_sample: ChannelSamples) -> int:
        """simulation.py:663-687 (only used to report ``max_step``)."""
        end_point = ch_sample.duration - 1
        mv = []
        for sample in (ch_sample.amp.as_array(detach=True), ch_sample.det.as_array(detach=True)):
            mv.append(
                int(np.min(np.diff(np.nonzero(np.diff(sample)), prepend=-1, append=end_point)))
            )
        return min(mv)

    # ------------------------------------------------------------------
    def _has_collapse_ops(self) -> bool:
        return len(self._hamiltonian_data.lindblad_data.local_collapse_ops) > 0

    def _density_matrix_fits(self) -> bool:
        hd = self._hamiltonian_data
        return hd.basis_data.dim <= 3 and hd.basis_data.dim ** (2 * hd.n_qudits) <= (1 << 26)

    def _use_mcwf(self) -> bool:
        return self._has_collapse_ops() and not self._density_matrix_fits()

    def _check_supported(self) -> None:
        """Collapse operators run as a master equation on the vectorised density
        matrix (``pulser_b200/lindblad.py``): deterministic where the reference uses
        ``mesolve`` and, for ``mcsolve`` requests, the exact ensemble average that the
        Monte-Carlo trajectories estimate (``simulation.py:705-718``)."""
        if self._has_collapse_ops() and not self._density_matrix_fits():
            # wave-function Monte Carlo (pb200_plan_set_collapse): needs a trajectory count
            if self.n_trajectories is None:
                raise ValueError(
                    "'n_trajectories' must be defined to emulate collapse operators on a register "
                    "whose density matrix does not fit on the device (Monte-Carlo wave function)."
                )

    def _validate_options(self, options: dict) -> dict:
        unknown = set(options) - _QUTIP_OPTIONS - _B200_OPTIONS
        if unknown:
            raise TypeError(f"Unknown solver options: {sorted(unknown)}")
        if "SPAM" in self.noise_model.noise_types:
            if self.noise_model.state_prep_error > 0 and not self._initial_is_ground:
                raise NotImplementedError(
                    "Can't combine state preparation errors with an initial "
                    "state different from the ground."
                )
        return {
            "max_step": int(options.get("b200_max_step", 0)),
            "cheb_tol": float(options.get("b200_cheb_tol", 0.0)),
            "refine_window": int(options.get("b200_refine_window", -1)),
            "tol": float(options.get("b200_tol", 0.0)),
        }

    def _run_batch(self, specs: list[HamiltonianSpec], opts: dict) -> list[list[np.ndarray]]:
        """States [n_eval][n_traj, D] of a batch of trajectories (replaces
        ``_run_solver``'s ``qutip.sesolve`` call, simulation.py:729-735)."""
        from . import engine, lindblad

        times = self._eval_times_array
        out = []
        stats: dict = {}
        lind = self._has_collapse_ops()
        plan_cm = (
            lindblad.LindbladPlan(specs, self._interp_order, self._gpu)
            if lind
            else engine.DevicePlan(specs, self._interp_order, self._gpu)
        )
        with plan_cm as plan:
            plan.set_state(self._initial_state.full().reshape(-1))
            fetch = plan.get_rho if lind else plan.get_state
            out.append(fetch())
            for t0, t1 in zip(times[:-1], times[1:]):
                st = plan.propagate(t0, t1, **opts)
                for k, v in st.items():
                    stats[k] = max(stats.get(k, 0), v) if k == "max_rho" else stats.get(k, 0) + v
                out.append(fetch())
        self.last_run_stats = stats
        return out

    def _wrap(self, states: list[np.ndarray]) -> CoherentResults:
        hd = self._hamiltonian_data
        d, n = hd.basis_data.dim, hd.n_qudits
        results = [
            B200Result(
                tuple(hd.register.qubits),
                self._meas_basis,
                (
                    DensityMatrix(s, [[d] * n, [d] * n])
                    if np.ndim(s) == 2
                    else StateVector(s, [[d] * n, [1] * n])
                ),
                self._meas_basis in self.basis_name,
                evaluation_time=t / (self._tot_duration * 1e-3),
            )
            for s, t in zip(states, self._eval_times_array)
        ]
        meas_errors = (
            {
                "epsilon": self.noise_model.p_false_pos,
                "epsilon_prime": self.noise_model.p_false_neg,
            }
            if "SPAM" in self.noise_model.noise_types
            else None
        )
        return CoherentResults(
            results, n, self.basis_name, self._eval_times_array, self._meas_basis, meas_errors
        )

    def run(self, progress_bar: bool = False, print_progress: bool = False, **options: Any):
        """Simulate the sequence (simulation.py:800-883).

        Returns ``CoherentResults``, or ``NoisyResults`` when the noise model
        has stochastic noise.
        """
        if not (progress_bar is True or progress_bar is False or progress_bar is None):  # 1 == True is not a bool
            raise ValueError("`progress_bar` must be a bool.")
        opts = self._validate_options(options)
        self._check_supported()
        if not _has_stochastic_noise(self.noise_model) and not self._use_mcwf():
            if print_progress:
                print("Emulating Trajectory 1/1")
            states = self._run_batch([self._current_spec], opts)
            return self._wrap([s[0] for s in states])

        total_count = np.array([Counter() for _ in self._eval_times_array])
        if self._has_collapse_ops() and not self._use_mcwf():
            for cleanres, reps in self._noisy_runs(
                print_progress=print_progress, batch=int(options.get("b200_batch", 0)), opts=opts
            ):
                total_count += np.array(
                    [
                        cleanres.sample_state(t, n_samples=self.noise_model.samples_per_run * reps)
                        for t in self._eval_times_array
                    ]
                )
        else:
            total_count += self._noisy_counts(
                print_progress=print_progress, batch=int(options.get("b200_batch", 0)), opts=opts
            )
        # one process per GPU: every rank evolved its stripe of the trajectories; the Counters are additive
        # (simulation.py:848-861), so ONE all-reduce of the histograms merges them (parallel.py)
        from . import parallel

        if parallel.world_size() > 1:
            total_count = np.array(
                parallel.merge_trajectory_counts(list(total_count), self._hamiltonian_data.n_qudits)
            )
            parallel.sync_numpy_random()  # the ranks consumed different numbers of sampling uniforms
        n_measures = int(self.n_trajectories) * self.noise_model.samples_per_run
        hd = self._hamiltonian_data
        results = [
            SampledCounts(
                tuple(hd.register.qubits), self._meas_basis, total_count[ind],
                evaluation_time=t / (self._tot_duration * 1e-3),
            )
            for ind, t in enumerate(self._eval_times_array)
        ]
        return NoisyResults(
            results, hd.n_qudits, self.basis_name, self._eval_times_array, n_measures
        )

    def _pending_trajectories(self) -> list:
        """(spec, reps) of this rank's stripe; redraws the trajectories on repeated runs (:892-902)."""
        from . import parallel

        if parallel.world_size() > 1:
            # every rank must draw the same trajectory list before taking its stripe (ADVICE r01): common seed,
            # then a fresh draw on every rank
            parallel.sync_numpy_random()
            self._noise_trajectories_used = True
        if self._noise_trajectories_used:
            nm = self._hamiltonian_data.noise_model
            self._hamiltonian_data = HamiltonianData(
                self.samples_obj, self._register, self.device, nm,
                self._get_n_trajectories(nm, check_value=True),
            )
        self._noise_trajectories_used = True
        # (index into hd.noise_trajectories, reps): the specs themselves are built when a batch asks for them, so
        # a thousand trajectories never sit in host memory as per-atom sample tables at once
        hd = self._hamiltonian_data
        entries = [(i, int(reps)) for i, (_, reps) in enumerate(hd.noise_trajectories)]
        if self._use_mcwf():
            # every Monte-Carlo trajectory is its own random realisation: no merging by `reps`
            if not _has_stochastic_noise(self.noise_model):
                entries = [(entries[0][0], 1)] * int(self.n_trajectories)
            else:
                entries = [(i, 1) for i, reps in entries for _ in range(reps)]
        if parallel.world_size() > 1:  # trajectory j -> rank j mod world (same list on every rank, see above)
            entries = [entries[j] for j in parallel.stripe(len(entries), parallel.rank(), parallel.world_size())]
        return _PendingTrajectories(self, hd, entries)

    def _noisy_counts(self, print_progress: bool, batch: int, opts: dict) -> np.ndarray:
        """Bitstring Counters per evaluation time of all noise trajectories, sampled ON THE DEVICE
        (``pb200_state_sample``): only the shots travel to the host, never the states.
        Replaces the per-trajectory ``sample_state`` loop of simulation.py:850-861."""
        from . import engine
        from .results import CoherentResults

        times = self._eval_times_array
        counts = np.array([Counter() for _ in times])
        pending = self._pending_trajectories()
        if not pending:
            return counts
        hd = self._hamiltonian_data
        n = hd.n_qudits
        D = pending[0][0].hilbert_dim
        if batch <= 0:
            batch = self._auto_batch(D, len(pending), stored_states=False)
        one_state = {"ground-rydberg": "r", "digital": "h", "XY": "d"}[self._meas_basis]
        matching = self._meas_basis in self.basis_name
        spr = self.noise_model.samples_per_run
        flipper = None
        if "SPAM" in self.noise_model.noise_types and (
            self.noise_model.p_false_pos > 0 or self.noise_model.p_false_neg > 0
        ):
            flipper = CoherentResults(
                [], n, self.basis_name, times, self._meas_basis,
                {"epsilon": self.noise_model.p_false_pos, "epsilon_prime": self.noise_model.p_false_neg},
            )
        traj_nb = 0
        n_trajectories = self.n_trajectories

        def sample_all(plan, chunk, t_index):
            for i, (_, reps) in enumerate(chunk):
                if hd.basis_data.dim == 2 and not matching:
                    c = Counter({"0" * n: spr * reps})  # only 000...0 is measured (qutip_result.py:120-123)
                else:
                    c = plan.sample(spr * reps, one_state, traj=i)
                if flipper is not None:
                    c = flipper._flip(c)
                counts[t_index] += c

        for chunk in pending.batches(batch):
            if print_progress:
                for _, reps in chunk:
                    if reps == 1:
                        print(f"Emulating Trajectory {traj_nb+1}/{n_trajectories}")
                    else:
                        print("Emulating Trajectories " f"[{traj_nb+1} - {traj_nb+reps}]/{n_trajectories}")
                    traj_nb += reps
            with engine.DevicePlan([s for s, _ in chunk], self._interp_order, self._gpu) as plan:
                if self._use_mcwf():
                    plan.set_collapse(chunk[0][0].collapse_ops, seed=int(np.random.randint(0, 2**31 - 1)))
                plan.set_state(self._initial_state.full().reshape(-1))
                sample_all(plan, chunk, 0)
                for k, (t0, t1) in enumerate(zip(times[:-1], times[1:])):
                    plan.propagate(t0, t1, **opts)
                    sample_all(plan, chunk, k + 1)
            self._current_spec = chunk[-1][0]
        return counts

    def _auto_batch(self, D: int, n_pending: int, stored_states: bool = True) -> int:
        """Trajectories per device batch.  Device side: 3 state buffers + 6 step-doubling buffers + per-trajectory
        Dint of ``D`` (wave functions) or ``D*D`` (the vectorised density matrix of the master equation) amplitudes
        within 8 GiB; host side (``_run_batch`` keeps every evaluation-time state of the batch): 4 GiB."""
        amps = D * D if (self._has_collapse_ops() and not self._use_mcwf()) else D
        dev = (8 << 30) // (amps * (9 * 16 + 8))
        host = dev
        if stored_states:
            host = (4 << 30) // max(1, len(self._eval_times_array) * amps * 16)
        return int(max(1, min(n_pending, dev, host, 1024)))

    def _noisy_runs(self, print_progress: bool, batch: int, opts: dict):
        """simulation.py:885-915, trajectories evolved in device batches."""
        n_trajectories = self.n_trajectories
        pending = self._pending_trajectories()
        if not pending:
            return
        D = pending[0][0].hilbert_dim
        if batch <= 0:
            batch = self._auto_batch(D, len(pending))
        traj_nb = 0
        for chunk in pending.batches(batch):
            states = self._run_batch([s for s, _ in chunk], opts)
            for i, (spec, reps) in enumerate(chunk):
                if print_progress:
                    if reps == 1:
                        print(f"Emulating Trajectory {traj_nb+1}/{n_trajectories}")
                    else:
                        print(
                            "Emulating Trajectories "
                            f"[{traj_nb+1} - {traj_nb+reps}]/{n_trajectories}"
                        )
                self._current_spec = spec
                traj_nb += reps
                yield self._wrap([s[i] for s in states]), reps

    # ------------------------------------------------------------------
    @classmethod
    def from_sequence(
        cls,
        sequence: Sequence,
        sampling_rate: float = 1.0,
        config: Any = None,
        evaluation_times: Union[float, str, Any] = "Full",
        with_modulation: bool = False,
        noise_model: NoiseModel | None = None,
        solver: Solver = Solver.DEFAULT,
        n_trajectories: int | None = None,
        **kwargs: Any,
    ) -> "B200Emulator":
        """simulation.py:955-1051."""
        if not isinstance(sequence, Sequence):
            raise TypeError(
                "The provided sequence has to be a valid "
                "pulser.Sequence instance."
            )
        if sequence.is_parametrized() or sequence.is_register_mappable():
            raise ValueError(
                "The provided sequence needs to be built to be simulated. Call"
                " `Sequence.build()` with the necessary parameters."
            )
        if not sequence._schedule:
            raise ValueError("The provided sequence has no declared channels.")
        if all(sequence._schedule[x][-1].tf == 0 for x in sequence.declared_channels):
            raise ValueError("No instructions given for the channels in the sequence.")
        if with_modulation and sequence._slm_mask_targets:
            raise NotImplementedError(
                "Simulation of sequences combining an SLM mask and output "
                "modulation is not supported."
            )
        return cls(
            sampler.sample(
                sequence,
                modulation=with_modulation,
                extended_duration=sequence.get_duration(include_fall_time=with_modulation),
            ),
            sequence.register,
            sequence.device,
            sampling_rate,
            config,
            evaluation_times,
            noise_model=noise_model,
            solver=solver,
            n_trajectories=n_trajectories,
            **kwargs,
        )
