"""Result objects of the GPU emulator: qutip-free mirrors of the reference's.

* ``StateVector``    -- the minimal ``qutip.Qobj`` surface the reference's
  result classes and its users touch (``full()``, ``isket``, ``shape``,
  ``dims``, ``norm()``, ``unit()``, ``overlap()``).
* ``B200Result``     -- ``pulser_simulation.qutip_result.QutipResult``
  (``qutip_result.py:31-242``): one state at one evaluation time, bitstring
  weights incl. the 3/4-level marginalisation, ``get_state`` post-processing.
* ``CoherentResults`` / ``NoisyResults`` -- ``pulser_simulation.simresults``
  (``simresults.py:38-568``): ``states``, ``get_state``, ``get_final_state``,
  ``expect`` (pseudo-density with SPAM errors), ``sample_state`` with the
  epsilon / epsilon' bit flips, ``sample_final_state``.

Sampling draws from the global ``np.random`` stream with the reference's own
``multinomial`` recipe (``pulser-core/pulser/math/multinomial.py:17-36``), so a
given state + seed yields the reference's Counter.
"""
from __future__ import annotations

from collections import Counter
from typing import Any, Mapping, Optional, Sequence

import numpy as np

EIGENSTATES = {
    "ground-rydberg": ["r", "g"],
    "digital": ["g", "h"],
    "XY": ["u", "d"],
}
STATES_RANK = ("u", "d", "r", "g", "h", "x")


def states_from_bases(bases: Sequence[str]) -> list[str]:
    """``pulser.channels.base_channel.get_states_from_bases``."""
    all_states = set().union(*(set(EIGENSTATES[b]) for b in bases))
    return [s for s in STATES_RANK if s in all_states]


class StateVector:
    """A ket as a numpy array with the slice of the Qobj API that matters."""

    isket = True
    isoper = False

    def __init__(self, data: np.ndarray, dims: Optional[list] = None) -> None:
        self._data = np.asarray(data, dtype=np.complex128).reshape(-1)
        n = self._data.size
        self.dims = dims if dims is not None else [[n], [1]]

    def full(self) -> np.ndarray:
        return self._data.reshape(-1, 1).copy()

    @property
    def shape(self) -> tuple[int, int]:
        return (self._data.size, 1)

    def copy(self) -> "StateVector":
        return StateVector(self._data.copy(), self.dims)

    def norm(self) -> float:
        return float(np.linalg.norm(self._data))

    def unit(self) -> "StateVector":
        return StateVector(self._data / self.norm(), self.dims)

    def overlap(self, other: "StateVector") -> complex:
        return complex(np.vdot(other._data, self._data))

    def tidyup(self, atol: float = 1e-12) -> "StateVector":
        d = self._data.copy()
        d.real[np.abs(d.real) < atol] = 0.0
        d.imag[np.abs(d.imag) < atol] = 0.0
        return StateVector(d, self.dims)

    def __mul__(self, scalar: complex) -> "StateVector":
        return StateVector(self._data * scalar, self.dims)

    __rmul__ = __mul__

    def __eq__(self, other: object) -> bool:
        if not isinstance(other, StateVector):
            return NotImplemented
        return self.shape == other.shape and bool(
            np.allclose(self._data, other._data, atol=1e-12, rtol=0)
        )

    def __repr__(self) -> str:
        return f"StateVector(dims={self.dims}, data={self._data!r})"


class DensityMatrix:
    """A density operator with the slice of the Qobj API the result classes use."""

    isket = False
    isoper = True

    def __init__(self, data: np.ndarray, dims: Optional[list] = None) -> None:
        data = np.asarray(data, dtype=np.complex128)
        n = int(np.rint(np.sqrt(data.size)))
        self._data = data.reshape(n, n)
        self.dims = dims if dims is not None else [[n], [n]]

    def full(self) -> np.ndarray:
        return self._data.copy()

    def diag(self) -> np.ndarray:
        return np.diagonal(self._data).copy()

    @property
    def shape(self) -> tuple[int, int]:
        return self._data.shape

    def copy(self) -> "DensityMatrix":
        return DensityMatrix(self._data.copy(), self.dims)

    def tr(self) -> complex:
        return complex(np.trace(self._data))

    def tidyup(self, atol: float = 1e-12) -> "DensityMatrix":
        d = self._data.copy()
        d.real[np.abs(d.real) < atol] = 0.0
        d.imag[np.abs(d.imag) < atol] = 0.0
        return DensityMatrix(d, self.dims)

    def __repr__(self) -> str:
        return f"DensityMatrix(dims={self.dims}, shape={self.shape})"


def multinomial(n_samples: int, probabilities: np.ndarray) -> np.ndarray:
    """``pulser.math.multinomial`` (same RNG consumption)."""
    rnd = np.random.rand(n_samples)
    cumsums = np.cumsum(probabilities)
    return np.searchsorted(cumsums, rnd)


class B200Result:
    """One state at one evaluation time (mirror of ``QutipResult``)."""

    def __init__(
        self,
        atom_order: tuple,
        meas_basis: str,
        state: StateVector,
        matching_meas_basis: bool,
        evaluation_time: float = 1.0,
    ) -> None:
        self.atom_order = tuple(atom_order)
        self.meas_basis = meas_basis
        self.state = state
        self.matching_meas_basis = matching_meas_basis
        self.evaluation_time = evaluation_time

    @property
    def _size(self) -> int:
        return len(self.atom_order)

    @property
    def _dim(self) -> int:  # qutip_result.py:57-65
        return int(np.rint(self.state.shape[0] ** (1 / self._size)))

    @property
    def _basis_name(self) -> str:  # qutip_result.py:67-91
        if self.meas_basis == "XY":
            return "XY_with_error" if self._dim == 3 else "XY"
        if self._dim == 4:
            return "all_with_error"
        if self._dim == 3:
            if self.matching_meas_basis:
                return self.meas_basis + "_with_error"
            return "all"
        if not self.matching_meas_basis:
            return "digital" if self.meas_basis == "ground-rydberg" else "ground-rydberg"
        return self.meas_basis

    @property
    def _eigenbasis(self) -> list[str]:  # qutip_result.py:93-100
        bases = self._basis_name.split("_with_error")
        states = states_from_bases(
            ["ground-rydberg", "digital"] if bases[0] == "all" else [bases[0]]
        )
        states += ["x"] if len(bases) == 2 else []
        return states

    def _weights(self) -> np.ndarray:  # qutip_result.py:101-158
        size = self._size
        if not self.state.isket:
            probs = np.abs(self.state.diag())
        else:
            probs = (np.abs(self.state.full()) ** 2).flatten()
        if self._dim == 2:
            if self.matching_meas_basis:
                weights = probs[::-1] if self.meas_basis == "ground-rydberg" else probs
            else:
                weights = np.zeros(probs.size)
                weights[0] = 1.0
        elif self._dim in (3, 4):
            one_state = {"ground-rydberg": "r", "digital": "h", "XY": "d"}
            if self.meas_basis not in one_state:
                raise RuntimeError(f"Unknown measurement basis '{self.meas_basis}'.")
            one_idx = self._eigenbasis.index(one_state[self.meas_basis])
            # marginalise every qudit onto {not one, one}: the reference's
            # python loop over 2^N bitstrings, vectorised
            t = probs.reshape([self._dim] * size)
            for ax in range(size):
                one = np.take(t, [one_idx], axis=ax)
                rest = np.sum(t, axis=ax, keepdims=True) - one
                t = np.concatenate([rest, one], axis=ax)
            weights = t.reshape(-1)
        else:
            raise NotImplementedError(
                "Cannot sample system with single-atom state vectors of "
                "dimension > 4."
            )
        return weights / sum(weights)

    @property
    def sampling_dist(self) -> dict[str, float]:
        n = self._size
        return {
            np.binary_repr(ind, width=n): prob
            for ind, prob in enumerate(self._weights())
            if prob != 0
        }

    def get_samples(self, n_samples: int) -> Counter:
        return Counter(
            np.binary_repr(i, self._size)
            for i in multinomial(n_samples, self._weights())
        )

    def get_state(
        self,
        reduce_to_basis: Optional[str] = None,
        ignore_global_phase: bool = True,
        tol: float = 1e-6,
        normalize: bool = True,
    ) -> StateVector:  # qutip_result.py:160-242
        state = self.state.copy()
        is_density_matrix = not state.isket
        if is_density_matrix and self._dim != 2 and reduce_to_basis is not None:
            raise NotImplementedError(
                "Reduce to basis not implemented for density matrix"
                " states."
            )
        if ignore_global_phase and not is_density_matrix:
            full = state.full()
            global_ph = float(np.angle(full[np.argmax(np.abs(full))])[0])
            state = state * np.exp(-1j * global_ph)
        if self._dim == 2:
            if reduce_to_basis not in [None, self._basis_name]:
                raise TypeError(
                    f"Can't reduce a system in {self._basis_name}"
                    + f" to the {reduce_to_basis} basis."
                )
        elif reduce_to_basis is not None:
            if reduce_to_basis not in EIGENSTATES:
                raise ValueError(
                    "'reduce_to_basis' must be 'ground-rydberg', "
                    f"'XY', or 'digital', not '{reduce_to_basis}'."
                )
            basis_states = set(self._eigenbasis)
            target_states = set(EIGENSTATES[reduce_to_basis])
            if not target_states.issubset(basis_states):
                raise ValueError(
                    f"Can't reduce a state expressed in {self._basis_name}"
                    f" into {reduce_to_basis}"
                )
            ex_states = basis_states - target_states
            d, n = self._dim, self._size
            idx = np.arange(d**n)
            excluded = np.zeros(d**n, dtype=bool)
            for ex in ex_states:
                e = self._eigenbasis.index(ex)
                for k in range(n):
                    excluded |= (idx // d**k) % d == e
            arr = state.full().reshape(-1)
            if not np.all(np.isclose(np.abs(arr[excluded]) ** 2, 0, atol=tol)):
                raise TypeError(
                    "Can't reduce to chosen basis because the population of a "
                    "state to eliminate is above the allowed tolerance."
                )
            state = StateVector(arr[~excluded])
            if normalize:
                state = state.unit()
        return state.tidyup()


class SampledCounts:
    """``pulser.result.SampledResult`` surface used by ``NoisyResults``."""

    def __init__(self, atom_order: tuple, meas_basis: str, bitstring_counts: Mapping[str, int], evaluation_time: float = 1.0):
        self.atom_order = tuple(atom_order)
        self.meas_basis = meas_basis
        self.bitstring_counts = dict(bitstring_counts)
        self.evaluation_time = evaluation_time
        self.n_samples = sum(self.bitstring_counts.values())

    @property
    def _size(self) -> int:
        return len(self.atom_order)

    def _weights(self) -> np.ndarray:
        w = np.zeros(2**self._size)
        for bitstr, c in self.bitstring_counts.items():
            w[int(bitstr, 2)] = c / self.n_samples
        return w / np.sum(w)

    @property
    def sampling_dist(self) -> dict[str, float]:
        return {b: c / self.n_samples for b, c in self.bitstring_counts.items()}

    def get_samples(self, n_samples: int) -> Counter:
        return Counter(
            np.binary_repr(i, self._size)
            for i in multinomial(n_samples, self._weights())
        )


def _as_dense(obs: Any) -> np.ndarray:
    if hasattr(obs, "full"):
        return np.asarray(obs.full())
    if hasattr(obs, "toarray"):
        return np.asarray(obs.toarray())
    return np.asarray(obs)


class SimulationResults:
    """Common part of ``simresults.SimulationResults`` (``:38-229``)."""

    _use_pseudo_dens = False

    def __init__(self, size: int, basis_name: str, sim_times: np.ndarray) -> None:
        self._size = size
        bases = ["ground-rydberg", "digital", "all", "XY"]
        bases += [b + "_with_error" for b in bases]
        if basis_name not in bases:
            raise ValueError(f"`basis_name` must be in {bases}")
        self._basis_name = basis_name
        self._dim = 3 if basis_name.startswith("all") else 2
        if "_with_error" in basis_name:
            self._dim += 1
        self._sim_times = np.asarray(sim_times)
        self._results_seq: tuple = ()

    def __len__(self) -> int:
        return len(self._results_seq)

    def __getitem__(self, i: Any) -> Any:
        return self._results_seq[i]

    def __iter__(self):
        return iter(self._results_seq)

    def _get_index_from_time(self, t_float: float, tol: float = 1.0e-3) -> int:
        try:
            return int(np.where(abs(t_float - self._sim_times) < tol)[0][0])
        except IndexError:
            raise IndexError(
                f"Given time {t_float} is absent from simulation times within"
                + f" tolerance {tol}."
            )

    # -- measurement model -------------------------------------------------
    def _meas_matrix(self) -> np.ndarray:
        """M[state_index, measured_bit] of ``_meas_projector`` (``:219-229, 500-520``)."""
        gr = "ground-rydberg" in self._basis_name
        M = np.zeros((2, 2))
        errs = getattr(self, "_meas_errors", None) or {"epsilon": 0.0, "epsilon_prime": 0.0}
        for bit, err in ((0, errs["epsilon"]), (1, errs["epsilon_prime"])):
            good = 1 - bit if gr else bit
            M[good, bit] += 1 - err
            M[1 - good, bit] += err
        return M

    def _calc_pseudo_density_diag(self, t_index: int) -> np.ndarray:
        """Diagonal of the pseudo-density matrix (``simresults.py:192-217``)."""
        w = self[t_index]._weights().reshape([2] * self._size)
        M = self._meas_matrix()
        for ax in range(self._size):
            w = np.moveaxis(np.tensordot(M, w, axes=([1], [ax])), 0, ax)
        return w.reshape(-1)

    def expect(self, obs_list: Sequence[Any]) -> list[np.ndarray]:
        if not isinstance(obs_list, (list, np.ndarray)):
            raise TypeError("`obs_list` must be a list of operators.")
        dim = self._dim if not self._use_pseudo_dens else 2
        legal_shape = (dim**self._size, dim**self._size)
        out = []
        for obs in obs_list:
            if not (
                isinstance(obs, np.ndarray)
                or hasattr(obs, "full")
                or hasattr(obs, "toarray")
            ):
                raise TypeError(
                    f"Incompatible type {type(obs)} of "
                    + "observable. Type must be ArrayLike or "
                    + "qutip.Qobj."
                )
            if tuple(obs.shape) != legal_shape:
                raise ValueError(
                    "Incompatible shape of observable."
                    + f"Expected {legal_shape}, got {obs.shape}."
                )
            if self._use_pseudo_dens:
                dense = _as_dense(obs)
                if np.count_nonzero(dense - np.diag(np.diagonal(dense))) != 0:
                    raise ValueError(f"Observable {obs!r} is non-diagonal.")
                diag = np.diagonal(dense)
                vals = [
                    np.dot(diag, self._calc_pseudo_density_diag(i))
                    for i in range(len(self))
                ]
            else:
                sparse = hasattr(obs, "toarray") and not hasattr(obs, "full")
                mat = obs if sparse else _as_dense(obs)
                vals = []
                for res in self:
                    if res.state.isket:
                        v = res.state.full().reshape(-1)
                        vals.append(np.vdot(v, mat @ v))
                    else:
                        vals.append(np.trace(mat @ res.state.full()))
            arr = np.array(vals)
            if np.allclose(arr.imag, 0.0, atol=1e-12):
                arr = arr.real
            out.append(arr)
        return out

    def sample_state(self, t: float, n_samples: int = 1000, t_tol: float = 1.0e-3) -> Counter:
        return self[self._get_index_from_time(t, t_tol)].get_samples(n_samples)

    def sample_final_state(self, N_samples: int = 1000) -> Counter:
        return self.sample_state(self._sim_times[-1], N_samples)


class CoherentResults(SimulationResults):
    """Mirror of ``simresults.CoherentResults`` (``:370-568``)."""

    def __init__(
        self,
        run_output: Sequence[B200Result],
        size: int,
        basis_name: str,
        sim_times: np.ndarray,
        meas_basis: str,
        meas_errors: Optional[Mapping[str, float]] = None,
    ) -> None:
        super().__init__(size, basis_name, sim_times)
        if "all" in self._basis_name:
            if meas_basis not in {"ground-rydberg", "digital"}:
                raise ValueError("`meas_basis` must be 'ground-rydberg' or 'digital'.")
        else:
            expected = self._basis_name.replace("_with_error", "")
            if meas_basis != expected:
                raise ValueError(
                    f"`meas_basis` associated to basis_name '"
                    f"{self._basis_name}' must be '{expected}'."
                )
        self._meas_basis = meas_basis
        self._results_seq = tuple(run_output)
        if meas_errors is not None:
            if set(meas_errors) != {"epsilon", "epsilon_prime"}:
                raise ValueError(
                    "When defining measurement errors, only values of "
                    "'epsilon' and 'epsilon_prime' must be given."
                )
            self._use_pseudo_dens = True
        self._meas_errors = meas_errors

    @property
    def states(self) -> list[StateVector]:
        return [res.state for res in self]

    def get_state(self, t: float, reduce_to_basis=None, ignore_global_phase=True,
                  tol: float = 1e-6, normalize: bool = True, t_tol: float = 1.0e-3) -> StateVector:
        return self[self._get_index_from_time(t, t_tol)].get_state(
            reduce_to_basis, ignore_global_phase, tol, normalize
        )

    def get_final_state(self, reduce_to_basis=None, ignore_global_phase=True,
                        tol: float = 1e-6, normalize: bool = True) -> StateVector:
        return self.get_state(
            self._sim_times[-1], reduce_to_basis, ignore_global_phase, tol, normalize
        )

    def sample_state(self, t: float, n_samples: int = 1000, t_tol: float = 1.0e-3) -> Counter:
        return self._flip(super().sample_state(t, n_samples, t_tol))

    def _flip(self, sampled: Counter) -> Counter:
        """Detection errors epsilon / epsilon' applied to sampled bitstrings (simresults.py:522-568)."""
        if self._meas_errors is None or (
            self._meas_errors["epsilon"] == 0.0 and self._meas_errors["epsilon_prime"] == 0
        ):
            return sampled
        eps, eps_p = self._meas_errors["epsilon"], self._meas_errors["epsilon_prime"]
        shots = list(sampled.keys())
        n_detects = list(sampled.values())
        shot_arr = np.array([list(s) for s in shots], dtype=int)
        flip_probs = np.where(shot_arr == 1, eps_p, eps)
        flip_rep = np.repeat(flip_probs, n_detects, axis=0)
        rnd = np.random.uniform(size=(np.sum(n_detects), len(shot_arr[0])))
        new_shots = shot_arr.repeat(n_detects, axis=0) ^ (rnd < flip_rep)
        detected: Counter = Counter(map(tuple, new_shots))
        return Counter({"".join(map(str, k)): v for k, v in detected.items()})


class NoisyResults(SimulationResults):
    """Mirror of ``simresults.NoisyResults`` (``:232-367``)."""

    _use_pseudo_dens = True

    def __init__(self, run_output: Sequence[SampledCounts], size: int, basis_name: str,
                 sim_times: np.ndarray, n_measures: int) -> None:
        basis = basis_name.replace("_with_error", "")  # simresults.py:281-282: bitstrings carry no leakage level
        basis_name_ = "digital" if basis == "all" else basis
        super().__init__(size, basis_name_, sim_times)
        self.n_measures = n_measures
        self._results_seq = tuple(run_output)

    @property
    def states(self) -> list[np.ndarray]:
        return [self._calc_pseudo_density_diag(i) for i in range(len(self))]

    @property
    def results(self) -> list[Counter]:
        """Probability distribution of the bitstrings (``simresults.py:290-293``)."""
        return [Counter(res.sampling_dist) for res in self]

    def get_state(self, t: float, t_tol: float = 1.0e-3) -> np.ndarray:
        return self._calc_pseudo_density_diag(self._get_index_from_time(t, t_tol))

    def get_final_state(self) -> np.ndarray:
        return self.get_state(self._sim_times[-1])
