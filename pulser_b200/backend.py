"""``B200Backend``: the ``pulser.backend.EmulatorBackend`` plugin (seam S2).

Mirrors ``pulser_simulation.qutip_backend.QutipBackendV2``
(``pulser-simulation/pulser_simulation/qutip_backend.py:121-325``) with
``B200Config`` / ``B200State`` / ``B200Operator`` in place of
``QutipConfig`` / ``QutipState`` / ``QutipOperator``
(``qutip_config.py:28-192``, ``qutip_state.py:35-281``, ``qutip_op.py:30-259``).
States come from the CUDA path (``B200Emulator``); the Hamiltonian handed to the
observables applies ``H(t)`` on the device (``pb200_apply_h``), so ``Energy`` &
co. never build a matrix.
"""
from __future__ import annotations

import math
import warnings
from collections import Counter, defaultdict
from typing import Any, Literal, Mapping, Sequence, Type

import numpy as np
import scipy.sparse as sp

from ._compat import ensure_pulser

if not ensure_pulser():  # pragma: no cover
    raise ImportError("pulser_b200.backend needs pulser-core")

import pulser  # noqa: E402
from pulser.backend.abc import EmulatorBackend  # noqa: E402
from pulser.backend.config import EmulationConfig  # noqa: E402
from pulser.backend.default_observables import BitStrings, StateResult  # noqa: E402
from pulser.backend.operator import Operator  # noqa: E402
from pulser.backend.results import Results  # noqa: E402
from pulser.backend.state import State  # noqa: E402

from .emulator import B200Emulator, Solver, _has_stochastic_noise  # noqa: E402
from .opterms import OpTerms  # noqa: E402
from .results import multinomial  # noqa: E402


class B200State(State[complex, float]):
    """A state vector or density matrix as a numpy array (``QutipState`` mirror)."""

    def __init__(self, state: np.ndarray, *, eigenstates: Sequence[str]):
        super().__init__(eigenstates=eigenstates)
        arr = np.asarray(state.full() if hasattr(state, "full") else state, dtype=np.complex128)
        if arr.ndim == 2 and arr.shape[1] == 1:
            arr = arr.reshape(-1)
        if arr.ndim == 2 and arr.shape[0] == 1:
            arr = arr.reshape(-1).conj()  # a bra
        if arr.ndim not in (1, 2) or (arr.ndim == 2 and arr.shape[0] != arr.shape[1]):
            raise TypeError("'state' must be a ket (1-D) or a density matrix (square 2-D).")
        self._state = arr
        n = math.log(arr.shape[0], self.qudit_dim)
        if not np.isclose(n, round(n)):
            raise ValueError(
                f"A state with shape {arr.shape} is incompatible with "
                f"a system of {self.qudit_dim}-level qudits."
            )

    @property
    def is_ket(self) -> bool:
        return self._state.ndim == 1

    @property
    def n_qudits(self) -> int:
        return round(math.log(self._state.shape[0], self.qudit_dim))

    def to_array(self) -> np.ndarray:
        return self._state.copy()

    def overlap(self, other: "B200State") -> float:
        if not isinstance(other, B200State):
            raise TypeError(
                "'B200State.overlap()' expects another 'B200State', not " f"{type(other)}."
            )
        if self.n_qudits != other.n_qudits or self.qudit_dim != other.qudit_dim:
            raise ValueError(
                "Can't calculate the overlap between a state with "
                f"{self.n_qudits} {self.qudit_dim}-dimensional qudits and "
                f"another with {other.n_qudits} {other.qudit_dim}-dimensional "
                "qudits."
            )
        if self.eigenstates != other.eigenstates:
            msg = (
                "Can't calculate the overlap between states with eigenstates "
                f"{self.eigenstates} and {other.eigenstates}."
            )
            if set(self.eigenstates) != set(other.eigenstates):
                raise ValueError(msg)
            raise NotImplementedError(msg)
        if isinstance(other, DeviceDensityView) and not isinstance(self, _DeviceResident) and self.is_ket:
            return other.overlap(self)  # <phi|rho|phi> on the device (Fidelity.apply calls target.overlap(state))
        a, b = self._state, other._state
        if a.ndim == 1 and b.ndim == 1:
            return float(np.abs(np.vdot(a, b)) ** 2)
        if a.ndim == 1:
            return float(np.vdot(a, b @ a).real)
        if b.ndim == 1:
            return float(np.vdot(b, a @ b).real)
        return float(np.trace(a @ b).real)

    def probabilities(self, *, cutoff: float = 1e-12) -> dict[str, float]:
        probs = (np.abs(self._state) ** 2) if self.is_ket else np.abs(np.diagonal(self._state))
        non_zero = np.argwhere(probs > cutoff).flatten()
        probs = probs[non_zero]
        probs = probs / np.sum(probs)
        return dict(zip(map(self.get_basis_state_from_index, non_zero), probs))

    def bitstring_probabilities(self, *, one_state: str | None = None, cutoff: float = 1e-12) -> Mapping[str, float]:
        one_state = one_state or self.infer_one_state()
        zero_states = set(self.eigenstates) - {one_state}
        probs = self.probabilities(cutoff=cutoff)
        out: dict[str, float] = defaultdict(float)
        for state_str, p in probs.items():
            bitstring = state_str.replace(one_state, "1")
            for s_ in zero_states:
                bitstring = bitstring.replace(s_, "0")
            out[bitstring] += p
        return dict(out)

    def sample(self, *, num_shots: int, one_state: str | None = None, p_false_pos: float = 0.0,
               p_false_neg: float = 0.0) -> Counter:
        """qutip_state.py:169-218 (same RNG consumption)."""
        bitstring_probs = self.bitstring_probabilities(one_state=one_state, cutoff=1 / (1000 * num_shots))
        bitstrings = np.array(list(bitstring_probs))
        probs = np.array(list(map(float, bitstring_probs.values())))
        indices = multinomial(num_shots, probs)
        if p_false_pos == 0.0 and p_false_neg == 0.0:
            return Counter(bitstrings[indices].tolist())
        bitstr_arr = np.array([list(bs) for bs in bitstrings[indices]], dtype=int)
        flip_probs = np.where(bitstr_arr == 1, p_false_neg, p_false_pos)
        flips = np.random.uniform(size=flip_probs.shape) < flip_probs
        new_counts: Counter = Counter(map(tuple, bitstr_arr ^ flips))
        return Counter({"".join(map(str, k)): v for k, v in new_counts.items()})

    @classmethod
    def _from_state_amplitudes(cls, *, eigenstates: Sequence[str], n_qudits: int,
                               amplitudes: Mapping[str, complex]):
        d = len(eigenstates)
        vec = np.zeros(d**n_qudits, dtype=np.complex128)
        amps = {k: complex(v) for k, v in amplitudes.items()}
        for basis_state, amp in amps.items():
            idx = 0
            for s in basis_state:
                idx = idx * d + eigenstates.index(s)
            vec[idx] += amp
        return cls(vec, eigenstates=eigenstates), amps

    def __repr__(self) -> str:
        return f"B200State(eigenstates={self.eigenstates}, shape={self._state.shape})"

    def __eq__(self, other: Any) -> bool:
        return (
            isinstance(other, B200State)
            and self.eigenstates == other.eigenstates
            and self._state.shape == other._state.shape
            and bool(np.allclose(self._state, other._state, atol=1e-12, rtol=0))
        )


class _DeviceResident:
    """Marker + protocol of states whose data lives in a ``DevicePlan``."""

    def _projector_expect(self, coeff: complex, letter: str | None, targets: frozenset) -> complex | None:
        raise NotImplementedError

    def _terms_expect(self, terms: OpTerms) -> complex | None:
        """``<O>`` of an operator given as monomial terms, or ``None`` when this state cannot reduce it on the device."""
        return None


class DeviceStateView(_DeviceResident, B200State):
    """The current state of one trajectory of a ``DevicePlan``, left on the GPU.

    Handed to the observables by ``B200Backend`` while it steps through the
    evaluation times: ``Occupation`` / ``CorrelationMatrix`` (number-operator
    expectations), ``Energy*`` (with ``DeviceHamiltonian``), ``Fidelity`` and
    ``BitStrings`` reduce on the device (``pb200_state_occupation / _correlation /
    _energy / _overlap / _sample``), and so does ``Expectation`` of an operator with
    monomial terms (``pb200_state_expect``); anything else falls back to a host copy
    (``to_array``), fetched once.  Replaces the replay of stored ``QutipState``s of
    ``qutip_backend.py:254-280``, which cannot hold one state per step at N >= 20.
    """

    def __init__(self, plan: Any, *, eigenstates: Sequence[str], traj: int = 0, norm2: float | None = None):
        State.__init__(self, eigenstates=eigenstates)
        self._plan = plan
        self._traj = int(traj)
        self._host: np.ndarray | None = None
        self._norm2 = float(plan.norm2()[self._traj]) if norm2 is None else float(norm2)
        self._corr: dict[int, np.ndarray] = {}
        self._energy: dict[tuple[int, float], tuple[float, float]] = {}

    @property
    def _state(self) -> np.ndarray:  # host copy, normalised like qutip_backend.py:268-272
        if self._host is None:
            self._host = self._plan.get_state()[self._traj] / math.sqrt(self._norm2)
        return self._host

    @property
    def is_ket(self) -> bool:
        return True

    @property
    def n_qudits(self) -> int:
        return int(self._plan.n)

    def _correlations(self, letter: str) -> np.ndarray:
        digit = self.eigenstates.index(letter)
        if digit not in self._corr:
            self._corr[digit] = self._plan.correlation(digit, self._traj, 1)[0] / self._norm2
        return self._corr[digit]

    def _projector_expect(self, coeff, letter, targets):
        if len(targets) == 0:
            return complex(coeff)
        if len(targets) > 2:
            return None
        idx = sorted(targets)
        return complex(coeff) * float(self._correlations(letter)[idx[0], idx[-1]])

    def _terms_expect(self, terms: OpTerms) -> complex | None:
        expect_terms = getattr(self._plan, "expect_terms", None)
        if expect_terms is None:
            return None
        return complex(expect_terms(terms, self._traj, 1)[0]) / self._norm2

    def _energy_moments(self, plan: Any, t_us: float) -> tuple[float, float] | None:
        """``<H>``, ``<H^2>`` of this state under the Hamiltonian of ``plan``.  ``plan`` is either the plan that
        holds the state or the single-trajectory plan of the NOISELESS sequence (the operator handed to the
        observables of a noisy run): then the state is copied device to device first (``pb200_state_copy``)."""
        key = (id(plan), t_us)
        if key not in self._energy:
            if plan is self._plan:
                e, e2 = plan.energy(t_us)
                k = self._traj
            elif hasattr(plan, "copy_state_from") and getattr(plan, "n_traj", 1) == 1:
                plan.copy_state_from(self._plan, self._traj, 0)
                e, e2 = plan.energy(t_us)
                k = 0
            else:
                return None
            self._energy[key] = (float(e[k]) / self._norm2, float(e2[k]) / self._norm2)
        return self._energy[key]

    def overlap(self, other: "B200State") -> float:
        if isinstance(other, B200State) and not isinstance(other, _DeviceResident) and other.is_ket \
                and other.eigenstates == self.eigenstates and other.n_qudits == self.n_qudits:
            return float(abs(self._plan.overlap(other._state, self._traj, 1)[0]) ** 2 / self._norm2)
        return B200State.overlap(self, other)

    def sample(self, *, num_shots: int, one_state: str | None = None, p_false_pos: float = 0.0,
               p_false_neg: float = 0.0) -> Counter:
        """Shots drawn on the device (``pb200_state_sample``: cumulative sum + searchsorted of the uniforms of
        the global ``np.random`` stream, the recipe of ``qutip_result.py:101-158``); same distribution as
        ``B200State.sample`` without the host-side probability dictionary."""
        one_state = one_state or self.infer_one_state()
        return _spam_flips(self._plan.sample(int(num_shots), one_state, self._traj), p_false_pos, p_false_neg)

    def __repr__(self) -> str:
        return f"DeviceStateView(eigenstates={self.eigenstates}, n_qudits={self.n_qudits})"


def _spam_flips(counts: Counter, p_false_pos: float, p_false_neg: float) -> Counter:
    """Measurement errors on device-drawn shots: every bit of every shot flips with ``p_false_neg`` (a 1) or
    ``p_false_pos`` (a 0), with the uniforms of ``B200State.sample`` (qutip_state.py:169-218)."""
    if p_false_pos == 0.0 and p_false_neg == 0.0:
        return counts
    keys = list(counts)
    bitstr_arr = np.repeat(np.array([list(k) for k in keys], dtype=int), [counts[k] for k in keys], axis=0)
    flip_probs = np.where(bitstr_arr == 1, p_false_neg, p_false_pos)
    flips = np.random.uniform(size=flip_probs.shape) < flip_probs
    new_counts: Counter = Counter(map(tuple, bitstr_arr ^ flips))
    return Counter({"".join(map(str, k)): v for k, v in new_counts.items()})


class DeviceDensityView(_DeviceResident, B200State):
    """The current density matrix of one trajectory of a ``LindbladPlan``, left on the GPU.

    The master-equation counterpart of ``DeviceStateView``: ``Occupation`` / ``CorrelationMatrix``, ``Expectation``
    of an operator with monomial terms, ``Energy*`` (with ``DeviceHamiltonian``), ``Fidelity`` and ``BitStrings``
    reduce on the device (``pb200_density_*``), every value divided by the device trace.  Anything else reads a host
    copy (``to_array``), fetched once.  ``copy.deepcopy`` (``StateResult``) gives a plain ``B200State``, so a stored
    state never follows the plan as it moves on.
    """

    def __init__(self, plan: Any, *, eigenstates: Sequence[str], traj: int = 0, trace: float | None = None):
        State.__init__(self, eigenstates=eigenstates)
        self._plan = plan
        self._traj = int(traj)
        self._host: np.ndarray | None = None
        self._trace = float(plan.density_trace(self._traj, 1)[0]) if trace is None else float(trace)
        self._corr: dict[int, np.ndarray] = {}
        self._energy: dict[tuple[int, float], tuple[float, float]] = {}

    @property
    def _state(self) -> np.ndarray:  # host copy, normalised like qutip_backend.py:268-272
        if self._host is None:
            self._host = self._plan.get_rho()[self._traj] / self._trace
        return self._host

    @property
    def is_ket(self) -> bool:
        return False

    @property
    def n_qudits(self) -> int:
        return int(self._plan.n)

    def _projector_expect(self, coeff, letter, targets):
        if len(targets) == 0:
            return complex(coeff)
        if len(targets) > 2:
            return None
        digit = self.eigenstates.index(letter)
        if digit not in self._corr:
            self._corr[digit] = self._plan.density_correlation(digit, self._traj, 1)[0] / self._trace
        idx = sorted(targets)
        return complex(coeff) * float(self._corr[digit][idx[0], idx[-1]])

    def _terms_expect(self, terms: OpTerms) -> complex | None:
        return complex(self._plan.density_expect(terms, self._traj, 1)[0]) / self._trace

    def _energy_moments(self, plan: Any, t_us: float) -> tuple[float, float]:
        """``Tr(H rho)``, ``Tr(H^2 rho)`` over the trace, ``H = H(t_us)`` of the single-state plan ``plan``."""
        key = (id(plan), t_us)
        if key not in self._energy:
            e, e2 = self._plan.density_energy(plan, t_us, self._traj, 1)
            self._energy[key] = (float(e[0]) / self._trace, float(e2[0]) / self._trace)
        return self._energy[key]

    def overlap(self, other: "B200State") -> float:
        if isinstance(other, B200State) and not isinstance(other, _DeviceResident) and other.is_ket \
                and other.eigenstates == self.eigenstates and other.n_qudits == self.n_qudits:
            return float(self._plan.density_overlap(other._state, self._traj, 1)[0].real / self._trace)
        return B200State.overlap(self, other)

    def sample(self, *, num_shots: int, one_state: str | None = None, p_false_pos: float = 0.0,
               p_false_neg: float = 0.0) -> Counter:
        """Shots drawn on the device from ``diag rho`` (``pb200_density_sample``, the recipe of
        ``DeviceStateView.sample``), then the same measurement errors."""
        one_state = one_state or self.infer_one_state()
        return _spam_flips(self._plan.density_sample(int(num_shots), one_state, self._traj), p_false_pos, p_false_neg)

    def __deepcopy__(self, memo: dict) -> B200State:
        return B200State(self._state.copy(), eigenstates=self.eigenstates)

    def __repr__(self) -> str:
        return f"DeviceDensityView(eigenstates={self.eigenstates}, n_qudits={self.n_qudits})"


class _HPsiView(_DeviceResident, B200State):
    """``H(t)|psi>`` (or ``H(t) rho H(t)``) of a device-resident state: its squared norm (trace) is known from the
    fused device reduction, the state itself is only formed (more H-applies, fetched to the host) if somebody asks
    for it."""

    def __init__(self, source: DeviceStateView | DeviceDensityView, ham: "DeviceHamiltonian", norm2: float):
        State.__init__(self, eigenstates=source.eigenstates)
        self._source, self._ham, self._weight = source, ham, norm2
        self._host: np.ndarray | None = None

    @property
    def _state(self) -> np.ndarray:
        if self._host is None:
            out = self._ham._matvec(self._source._state)
            self._host = out if self._source.is_ket else self._ham._matvec(out.conj().T).conj().T
        return self._host

    @property
    def is_ket(self) -> bool:
        return self._source.is_ket

    @property
    def n_qudits(self) -> int:
        return self._source.n_qudits

    def _projector_expect(self, coeff, letter, targets):
        return complex(coeff) * self._weight if len(targets) == 0 else None


class B200Operator(Operator[complex, complex, B200State]):
    """An operator as a scipy sparse matrix (``QutipOperator`` mirror)."""

    def __init__(self, operator: Any, eigenstates: Sequence[str], *, pattern: tuple | None = None,
                 terms: OpTerms | None = None):
        """``operator``: a matrix, or a zero-argument callable building it on first use.

        ``pattern = (coeff, state, frozenset(qudits))`` marks ``coeff * prod_k |state><state|_k`` (identity for an
        empty set): its expectation on a device-resident state is a reduction on the GPU, the matrix is never built.
        ``terms``: the same operator as monomial terms (``pulser_b200.opterms``); its expectation on a device-resident
        state is computed matrix-free on the GPU.
        """
        super().__init__()
        B200State._validate_eigenstates(eigenstates)
        self._eigenstates = eigenstates
        self._pattern = pattern
        self._terms = terms
        if callable(operator):
            self._builder, self._matrix = operator, None
        else:
            self._builder, self._matrix = None, self._as_matrix(operator)
            # qutip_op.py:57 (QutipState._validate_shape): the dimension must be a power of the qudit dimension
            d = len(eigenstates)
            n = math.log(self._matrix.shape[0], d)
            if self._matrix.shape[0] != self._matrix.shape[1] or not np.isclose(n, round(n)):
                raise ValueError(
                    f"A state with shape {tuple(self._matrix.shape)} is incompatible with "
                    f"a system of {d}-level qudits."
                )

    @staticmethod
    def _as_matrix(operator: Any) -> sp.csr_matrix:
        mat = sp.csr_matrix(operator.full() if hasattr(operator, "full") else operator, dtype=np.complex128)
        if mat.shape[0] != mat.shape[1]:
            raise TypeError("'operator' must be a square matrix.")
        return mat

    @property
    def _operator(self) -> sp.csr_matrix:
        if self._matrix is None:
            self._matrix = self._as_matrix(self._builder())
        return self._matrix

    @property
    def eigenstates(self) -> tuple[str, ...]:
        return tuple(self._eigenstates)

    def to_array(self) -> np.ndarray:
        return self._operator.toarray()

    def _validate_other(self, other: Any, expected_type: Type, op_name: str) -> None:
        if not isinstance(other, expected_type):
            raise TypeError(f"'{op_name}' expects a '{expected_type.__name__}' instance, not {type(other)}.")
        if self.eigenstates != other.eigenstates:
            msg = (
                f"Can't apply {op_name} between a {self.__class__.__name__} "
                f"with eigenstates {self.eigenstates} and a "
                f"{other.__class__.__name__} with {other.eigenstates}."
            )
            if set(self.eigenstates) != set(other.eigenstates):
                raise ValueError(msg)
            raise NotImplementedError(msg)

    def _matvec(self, arr: np.ndarray) -> np.ndarray:
        return self._operator @ arr

    def apply_to(self, state: B200State, /) -> B200State:
        self._validate_other(state, B200State, "B200Operator.apply_to()")
        out = self._matvec(state._state)
        if not state.is_ket:
            out = self._matvec(out.conj().T).conj().T  # O rho O^+
        cls = B200State if isinstance(state, _DeviceResident) else type(state)
        return cls(out, eigenstates=state.eigenstates)

    @property
    def _isherm(self) -> bool:
        if not hasattr(self, "_herm_cache") and self._terms is not None and self._terms.adjoint_matches():
            self._herm_cache = True
        if not hasattr(self, "_herm_cache"):
            m = self._operator
            self._herm_cache = bool(abs(m - m.getH()).max() < 1e-12) if m.nnz else True
        return self._herm_cache

    def expect(self, state: B200State, /) -> complex:
        """``qutip.expect`` semantics: a real number for a Hermitian operator."""
        self._validate_other(state, B200State, "B200Operator.expect()")
        if self._pattern is not None and isinstance(state, _DeviceResident):
            val = state._projector_expect(*self._pattern)
            if val is not None:
                return val.real if val.imag == 0.0 else val
        if self._terms is not None and isinstance(state, _DeviceResident):
            val = state._terms_expect(self._terms)
            if val is not None:
                return val.real if self._isherm else val
        if state.is_ket:
            val = complex(np.vdot(state._state, self._matvec(state._state)))
        else:
            val = complex(np.trace(self._matvec(state._state)))
        return val.real if self._isherm else val

    def __add__(self, other: "B200Operator", /) -> "B200Operator":
        self._validate_other(other, B200Operator, "__add__")
        a, b = self._terms, getattr(other, "_terms", None)
        # operators on different registers have no compiled sum: the matrices report the mismatch, as they always did
        terms = a + b if a is not None and b is not None and a.compatible(b) else None
        if terms is None:
            return B200Operator(self._operator + other._operator, eigenstates=self.eigenstates)
        return B200Operator(lambda: self._operator + other._operator, eigenstates=self.eigenstates, terms=terms)

    def __rmul__(self, scalar: complex) -> "B200Operator":
        pat = self._pattern
        if pat is not None:
            pat = (complex(scalar) * pat[0], pat[1], pat[2])
        terms = None if self._terms is None else self._terms.scaled(scalar)
        return B200Operator(lambda: complex(scalar) * self._operator, eigenstates=self.eigenstates, pattern=pat,
                            terms=terms)

    def __matmul__(self, other: "B200Operator") -> "B200Operator":
        self._validate_other(other, B200Operator, "__matmul__")
        pat = None
        a, b = self._pattern, getattr(other, "_pattern", None)
        if a is not None and b is not None and (a[1] == b[1] or not a[2] or not b[2]):
            # projectors on one eigenstate commute and are idempotent: the product is the projector on the union
            pat = (a[0] * b[0], a[1] if a[2] else b[1], a[2] | b[2])
        a, b = self._terms, getattr(other, "_terms", None)
        terms = a @ b if a is not None and b is not None and a.compatible(b) else None
        return B200Operator(lambda: self._operator @ other._operator, eigenstates=self.eigenstates, pattern=pat,
                            terms=terms)

    @classmethod
    def _from_operator_repr(cls, *, eigenstates: Sequence[str], n_qudits: int, operations: Any):
        """qutip_op.py:150-220 with scipy.sparse Kronecker products."""
        d = len(eigenstates)

        def qudit_op(qop: Mapping[str, complex]) -> sp.csr_matrix:
            m = sp.lil_matrix((d, d), dtype=np.complex128)
            for proj_str, coeff in qop.items():
                m[eigenstates.index(proj_str[0]), eigenstates.index(proj_str[1])] += complex(coeff)
            return m.tocsr()

        reconstructed = []
        for coeff, tensor_op in operations:
            re_tensor = [({k: complex(v) for k, v in qop.items()}, set(inds)) for qop, inds in tensor_op]
            for qop, inds in re_tensor:
                for key in qop:
                    if len(key) != 2 or key[0] not in eigenstates or key[1] not in eigenstates:
                        raise ValueError(f"Invalid projector '{key}' for eigenstates {tuple(eigenstates)}.")
                if any(ind < 0 or ind >= n_qudits for ind in inds):
                    raise ValueError("Qudit index out of range in the operator representation.")
            reconstructed.append((complex(coeff), re_tensor))

        def build() -> sp.csr_matrix:
            full = sp.csr_matrix((d**n_qudits, d**n_qudits), dtype=np.complex128)
            for coeff, re_tensor in reconstructed:
                factors = [sp.identity(d, format="csr", dtype=np.complex128) for _ in range(n_qudits)]
                for qop, inds in re_tensor:
                    for ind in inds:
                        factors[ind] = qudit_op(qop)
                term = factors[0]
                for f in factors[1:]:
                    term = sp.kron(term, f, format="csr")
                full = full + coeff * term
            return full

        # one term made of |a><a| projectors of a single eigenstate (number operators, identity)?
        pattern = None
        if len(reconstructed) == 1:
            coeff, re_tensor = reconstructed[0]
            letters, targets, scale, ok = set(), set(), complex(1.0), True
            for qop, inds in re_tensor:
                if len(qop) != 1 or targets & inds:
                    ok = False
                    break
                (key, val), = qop.items()
                if key[0] != key[1]:
                    ok = False
                    break
                letters.add(key[0])
                targets |= inds
                scale *= val ** len(inds)
            if ok and len(letters) <= 1:
                pattern = (coeff * scale, next(iter(letters)) if letters else None, frozenset(targets))
        terms = OpTerms.from_operations(reconstructed, eigenstates, n_qudits)
        return B200Operator(build, eigenstates=eigenstates, pattern=pattern, terms=terms), reconstructed

    def __repr__(self) -> str:
        return f"B200Operator(eigenstates={self.eigenstates}, shape={self._operator.shape})"

    def __eq__(self, other: Any) -> bool:
        return (
            isinstance(other, B200Operator)
            and self.eigenstates == other.eigenstates
            and abs(self._operator - other._operator).max() < 1e-12
        )


class DeviceHamiltonian(B200Operator):
    """``H(t)`` of the noiseless sequence, applied matrix-free on the GPU.

    Stands for the ``QutipOperator(noiseless H(t))`` the reference hands to every
    observable (``qutip_backend.py:258-264``)."""

    def __init__(self, plan: Any, t_us: float, eigenstates: Sequence[str]):
        Operator.__init__(self)
        self._eigenstates = eigenstates
        self._plan = plan
        self._t = t_us
        self._pattern = None
        self._terms = None
        self._builder, self._matrix = None, None  # never materialised
        self._herm_cache = True

    @property
    def _operator(self):
        raise NotImplementedError("DeviceHamiltonian is matrix-free")

    def expect(self, state: B200State, /) -> complex:
        if isinstance(state, (DeviceStateView, DeviceDensityView)):
            self._validate_other(state, B200State, "B200Operator.expect()")
            mom = state._energy_moments(self._plan, self._t)
            if mom is not None:
                return mom[0]
        return super().expect(state)

    def apply_to(self, state: B200State, /) -> B200State:
        if isinstance(state, (DeviceStateView, DeviceDensityView)):
            self._validate_other(state, B200State, "B200Operator.apply_to()")
            mom = state._energy_moments(self._plan, self._t)
            if mom is not None:
                return _HPsiView(state, self, mom[1])
        return super().apply_to(state)

    def _matvec(self, arr: np.ndarray) -> np.ndarray:
        if arr.ndim == 1:
            return self._plan.apply_h(self._t, arr)
        return np.stack([self._plan.apply_h(self._t, np.ascontiguousarray(arr[:, j])) for j in range(arr.shape[1])], axis=1)

    def __add__(self, other, /):  # pragma: no cover - not needed by the default observables
        raise NotImplementedError("DeviceHamiltonian is matrix-free")

    __rmul__ = __matmul__ = __add__


class B200Config(EmulationConfig[B200State]):
    """``QutipConfig`` mirror (``qutip_config.py:28-192``): same options, plus

    ``devices``: CUDA ordinals of the shards of the state (2, 4 or 8 entries; the same ordinal may repeat).
    A noiseless single-state run is then split over ``len(devices)`` plans (``pulser_b200.sharded.ShardedPlan``), so
    registers larger than one GPU's memory can run; so is the density matrix of a master equation whose noise is
    dephasing, relaxation, depolarizing or eff_noise only (``pulser_b200.lindblad.ShardedLindbladPlan``), exact where
    one device would need Monte-Carlo trajectories, under a drive of one phase (a master equation whose drive phase
    moves runs on one device, on the Taylor propagator as well).  Default ``None``: one plan on one device.
    """

    _enforce_expected_kwargs = True
    sampling_rate: float
    _state_type = B200State
    _operator_type = B200Operator
    solver: Solver

    def __init__(self, *, sampling_rate: float = 1.0,
                 solver: Solver | Literal["default", "MasterEquation", "MonteCarlo"] = Solver.DEFAULT,
                 print_progress: bool = False, progress_bar: bool = False, **backend_options: Any):
        if backend_options.setdefault("interaction_matrix") is not None:
            raise NotImplementedError("'B200Backend' does not handle custom interaction matrices.")
        if not (0 < sampling_rate <= 1.0):
            raise ValueError(
                f"The sampling rate (`sampling_rate` = {sampling_rate}) must"
                " be greater than 0 and less than or equal to 1."
            )
        initial_state = backend_options.setdefault("initial_state")
        if initial_state is not None and not isinstance(initial_state, B200State):
            raise TypeError(
                "If provided, `initial_state` must be an instance of "
                f"`B200State`, not {type(initial_state)}."
            )
        devices = backend_options.setdefault("devices")
        if devices is not None:
            from .sharded import validate_devices

            backend_options["devices"] = validate_devices(devices)
        noise_model = backend_options.get("noise_model")
        if noise_model is not None and noise_model.samples_per_run not in [None, 1]:
            warnings.warn(  # qutip_config.py:114-123: the V2 protocol samples through its observables
                f"The number of samples per run (`samples_per_run` = {noise_model.samples_per_run}) "
                "is ignored when using B200Backend.",
                stacklevel=2,
            )
        try:
            solver = Solver(solver)
        except ValueError:
            allowed_str = ", ".join(s.value for s in Solver)
            raise ValueError(f"Invalid solver '{solver}'. Allowed solvers are: {allowed_str}.")
        super().__init__(sampling_rate=sampling_rate, solver=Solver(solver), print_progress=print_progress,
                         progress_bar=progress_bar, **backend_options)

    def _expected_kwargs(self) -> set[str]:
        return super()._expected_kwargs() | {"sampling_rate", "solver", "print_progress", "progress_bar", "devices"}

    def _get_legacy_evaluation_times(self, total_duration_ns: int):
        """qutip_config.py:169-192: relative observable times -> microseconds."""
        extra: set[float] = set()
        if self.callbacks:
            return "Full"
        for obs in self.observables:
            if obs.evaluation_times is not None:
                extra.update(obs.evaluation_times)
        rel = self.default_evaluation_times
        if isinstance(rel, str) and rel == "Full":
            if not extra:
                return "Full"
            idx = np.linspace(0, total_duration_ns - 1, int(self.sampling_rate * total_duration_ns), dtype=int)
            rel = idx / total_duration_ns
        rel = np.union1d(np.asarray(rel, dtype=float), np.array(sorted(extra), dtype=float))
        # two requests that differ by a rounding error (0.493 vs 0.49299999999999994) are ONE evaluation: the
        # observables match their times up to pulser's TIME_TOLERANCE, so evaluating both would store twice
        from pulser.backend.observable import TIME_TOLERANCE

        keep = np.concatenate(([True], np.diff(rel) >= TIME_TOLERANCE)) if len(rel) else np.zeros(0, dtype=bool)
        return np.asarray(rel)[keep] * total_duration_ns * 1e-3


def density_matrix_aggregator(values: list) -> "B200State":
    """Average the states of the noise trajectories into a mixed state (each with probability 1/n): the custom
    aggregator the reference attaches to its ``StateResult`` tag (``pulser_simulation/aggregators.py:20-39``)."""
    acc = None
    for value in values:
        arr = np.asarray(value._state)
        rho = np.outer(arr, arr.conj()) if value.is_ket else arr
        acc = rho.astype(complex) if acc is None else acc + rho
    return B200State(acc / len(values), eigenstates=values[0].eigenstates)


def _state_aggregators(results: list) -> dict:
    """``qutip_backend.py:37-42, 322-325``: the tag of the StateResult observable, if any, gets the aggregator."""
    if not results:
        return {}
    for tag in results[0].get_result_tags():
        if tag.startswith(StateResult()._base_tag):
            return {tag: density_matrix_aggregator}
    return {}


class B200Backend(EmulatorBackend):
    """Emulate a sequence on an H100 through the generic ``pulser.backend`` API."""

    default_config = B200Config(observables=[BitStrings(evaluation_times=[1.0]), StateResult()])
    _config: B200Config

    def __init__(self, sequence: pulser.Sequence, *, config: EmulationConfig | None = None,
                 mimic_qpu: bool = False) -> None:
        super().__init__(sequence, config=config, mimic_qpu=mimic_qpu)
        noise_model = None
        if self._config.prefer_device_noise_model:
            noise_model = sequence.device.noise_model
        noise_model = noise_model or self._config.noise_model
        self._sim_obj = B200Emulator.from_sequence(
            sequence,
            sampling_rate=self._config.sampling_rate,
            noise_model=noise_model,
            with_modulation=self._config.with_modulation,
            solver=self._config.solver,
            n_trajectories=self._config.n_trajectories,
        )
        self._sim_obj.set_evaluation_times(
            self._config._get_legacy_evaluation_times(self._sim_obj.total_duration_ns)
        )
        if self._config.initial_state is not None:
            self._sim_obj.set_initial_state(self._config.initial_state.to_array())

    @staticmethod
    def run_from_sequence_samples(sequence_samples: Any, register: Any, device: Any, *,
                                  config: EmulationConfig | None = None) -> Results:
        """Executes an already sampled sequence (``QutipBackendV2.run_from_sequence_samples``,
        ``qutip_backend.py:193-232``): same emulator construction as ``__init__`` minus the ``Sequence`` checks."""
        cfg = B200Backend.validate_config(config or B200Backend.default_config)
        noise_model = device.noise_model if cfg.prefer_device_noise_model else None
        sim = B200Emulator(
            sequence_samples, register, device,
            sampling_rate=cfg.sampling_rate,
            config=None,
            noise_model=noise_model or cfg.noise_model,
            solver=cfg.solver,
            n_trajectories=cfg.n_trajectories,
        )
        sim.set_evaluation_times(cfg._get_legacy_evaluation_times(sim.total_duration_ns))
        if cfg.initial_state is not None:
            sim.set_initial_state(cfg.initial_state.to_array())
        runner = object.__new__(B200Backend)  # run() only needs the emulator and the validated config
        runner._sim_obj, runner._config = sim, cfg
        return runner.run()

    def _replay(self, plan: Any, coherent: Any, res: Results) -> None:
        """Feed the stored states to callbacks / observables (qutip_backend.py:254-280)."""
        sim, config = self._sim_obj, self._config
        eig = sim._hamiltonian_data.basis_data.eigenbasis
        for r in coherent:
            t = float(r.evaluation_time)
            raw = r.state.full()
            raw = raw.reshape(-1) if r.state.isket else raw
            nrm = np.linalg.norm(raw) if r.state.isket else np.trace(raw).real
            state = B200State(raw / nrm, eigenstates=eig)
            ham = DeviceHamiltonian(plan, t * res.total_duration / 1000, eig)
            for callback in config.callbacks:
                callback(config=config, t=t, state=state, hamiltonian=ham, result=res)
            for obs in config.observables:
                obs(config=config, t=t, state=state, hamiltonian=ham, result=res)

    def _stream(self, plan: Any, res: Results) -> None:
        """Noiseless sequence: step the device plan through the evaluation times and hand the observables a
        view of the state that stays on the GPU (no per-time state on the host; SURVEY section 8(f) row 2)."""
        sim, config = self._sim_obj, self._config
        eig = sim._hamiltonian_data.basis_data.eigenbasis
        opts = sim._validate_options({})
        if config.print_progress:
            print("Emulating Trajectory 1/1")
        plan.set_state(sim._initial_state.full().reshape(-1))
        times = sim._eval_times_array
        stats: dict = {}
        prev = float(times[0])
        for t_us in times:
            t_us = float(t_us)
            if t_us > prev:
                st = plan.propagate(prev, t_us, **opts)
                for k, v in st.items():
                    stats[k] = max(stats.get(k, 0), v) if k == "max_rho" else stats.get(k, 0) + v
                prev = t_us
            t = t_us / (sim._tot_duration * 1e-3)
            state = DeviceStateView(plan, eigenstates=eig)
            ham = DeviceHamiltonian(plan, t_us, eig)
            for callback in config.callbacks:
                callback(config=config, t=t, state=state, hamiltonian=ham, result=res)
            for obs in config.observables:
                obs(config=config, t=t, state=state, hamiltonian=ham, result=res)
        sim.last_run_stats = stats

    def _stream_noisy(self, hplan: Any, atom_order: tuple) -> list[Results]:
        """Stochastic noise on pure states (noisy Hamiltonians, Monte-Carlo wave functions): the trajectories are
        evolved in device batches through the evaluation times and every observable sees a ``DeviceStateView`` of
        its trajectory; the Hamiltonian handed over is the noiseless one (``qutip_backend.py:258-264``), its
        expectation on a noisy state goes through ``pb200_state_copy``.  One ``Results`` per trajectory repetition,
        like the replay path; within a batch the observables are visited time-major (as ``_noisy_counts`` does)."""
        from . import engine

        sim, config = self._sim_obj, self._config
        eig = sim._hamiltonian_data.basis_data.eigenbasis
        opts = {"max_step": 0, "cheb_tol": 0.0, "refine_window": -1, "tol": 0.0}
        times = sim._eval_times_array
        pending = sim._pending_trajectories()
        out: list[Results] = []
        if not pending:
            return out
        D = pending[0][0].hilbert_dim
        batch = max(1, min(len(pending), int((8 << 30) // (D * 56)), 1024))
        traj_nb, n_trajectories = 0, sim.n_trajectories
        for chunk in pending.batches(batch):
            if config.print_progress:
                for _, reps in chunk:
                    if reps == 1:
                        print(f"Emulating Trajectory {traj_nb+1}/{n_trajectories}")
                    else:
                        print("Emulating Trajectories " f"[{traj_nb+1} - {traj_nb+reps}]/{n_trajectories}")
                    traj_nb += reps
            per_traj = [[Results(atom_order=atom_order, total_duration=sim.total_duration_ns) for _ in range(reps)]
                        for _, reps in chunk]
            with engine.DevicePlan([s for s, _ in chunk], sim._interp_order, sim._gpu) as plan:
                if sim._use_mcwf():
                    plan.set_collapse(chunk[0][0].collapse_ops, seed=int(np.random.randint(0, 2**31 - 1)))
                plan.set_state(sim._initial_state.full().reshape(-1))
                prev = float(times[0])
                for t_us in times:
                    t_us = float(t_us)
                    if t_us > prev:
                        plan.propagate(prev, t_us, **opts)
                        prev = t_us
                    t = t_us / (sim._tot_duration * 1e-3)
                    ham = DeviceHamiltonian(hplan, t_us, eig)
                    norms = plan.norm2()
                    for i, results in enumerate(per_traj):
                        state = DeviceStateView(plan, eigenstates=eig, traj=i, norm2=float(norms[i]))
                        for res in results:
                            for callback in config.callbacks:
                                callback(config=config, t=t, state=state, hamiltonian=ham, result=res)
                            for obs in config.observables:
                                obs(config=config, t=t, state=state, hamiltonian=ham, result=res)
            sim._current_spec = chunk[-1][0]
            for results in per_traj:
                out.extend(results)
        return out

    def _streams_density(self) -> bool:
        """A master-equation run whose density matrices stay on the device (``_stream_density``): the plan class
        provides the density reductions, and the register is not XY (``pb200_density_energy`` has no exchange
        term).  Otherwise the stored density matrices are replayed."""
        from . import lindblad

        sim = self._sim_obj
        return (sim._has_collapse_ops() and not sim._use_mcwf() and hasattr(lindblad.LindbladPlan, "density_trace")
                and sim._hamiltonian_data.basis_data.interaction_type != "XY")

    def _stream_density(self, hplan: Any, atom_order: tuple, devices: list[int] | None = None) -> list[Results]:
        """Master equation: the density matrices of the trajectories (one without stochastic noise) are evolved in
        device batches through the evaluation times, and every observable sees a ``DeviceDensityView`` of its
        trajectory, so no density matrix is stored per evaluation time.  The Hamiltonian handed over is the noiseless
        one (``qutip_backend.py:258-264``).  One ``Results`` per trajectory repetition, like the replay path; within a
        batch the observables are visited time-major, as in ``_stream_noisy``.  ``devices``: the one density matrix
        is split over these shards (``lindblad.ShardedLindbladPlan``) instead of one ``LindbladPlan``."""
        from . import lindblad

        sim, config = self._sim_obj, self._config
        eig = sim._hamiltonian_data.basis_data.eigenbasis
        opts = {"max_step": 0, "cheb_tol": 0.0, "refine_window": -1, "tol": 0.0}
        times = sim._eval_times_array
        if _has_stochastic_noise(sim.noise_model):
            pending = sim._pending_trajectories()
            if not pending:
                return []
            chunks = pending.batches(sim._auto_batch(pending[0][0].hilbert_dim, len(pending), stored_states=False))
            n_trajectories = sim.n_trajectories
        else:
            chunks, n_trajectories = [[(sim._current_spec, 1)]], 1
        out: list[Results] = []
        traj_nb = 0
        for chunk in chunks:
            if config.print_progress:
                for _, reps in chunk:
                    if reps == 1:
                        print(f"Emulating Trajectory {traj_nb+1}/{n_trajectories}")
                    else:
                        print("Emulating Trajectories " f"[{traj_nb+1} - {traj_nb+reps}]/{n_trajectories}")
                    traj_nb += reps
            per_traj = [[Results(atom_order=atom_order, total_duration=sim.total_duration_ns) for _ in range(reps)]
                        for _, reps in chunk]
            stats: dict = {}
            specs = [s for s, _ in chunk]
            if devices is None:
                plan = lindblad.LindbladPlan(specs, sim._interp_order, sim._gpu)
            else:
                plan = lindblad.ShardedLindbladPlan(specs, devices, sim._interp_order)
            with plan:
                plan.set_state(sim._initial_state.full().reshape(-1))
                prev = float(times[0])
                for t_us in times:
                    t_us = float(t_us)
                    if t_us > prev:
                        st = plan.propagate(prev, t_us, **opts)
                        for k, v in st.items():
                            stats[k] = max(stats.get(k, 0), v) if k == "max_rho" else stats.get(k, 0) + v
                        prev = t_us
                    t = t_us / (sim._tot_duration * 1e-3)
                    ham = DeviceHamiltonian(hplan, t_us, eig)
                    traces = plan.density_trace()
                    for i, results in enumerate(per_traj):
                        state = DeviceDensityView(plan, eigenstates=eig, traj=i, trace=float(traces[i]))
                        for res in results:
                            for callback in config.callbacks:
                                callback(config=config, t=t, state=state, hamiltonian=ham, result=res)
                            for obs in config.observables:
                                obs(config=config, t=t, state=state, hamiltonian=ham, result=res)
            sim.last_run_stats = stats
            sim._current_spec = chunk[-1][0]
            for results in per_traj:
                out.extend(results)
        return out

    def _run_sharded(self, devices: list[int]) -> Results:
        """A state split over ``devices`` (``B200Config(devices=...)``), streamed through the evaluation times like the
        single-plan runs: the state vector of a noiseless sequence, or the density matrix of a master equation whose
        noise is collapse operators only (``_sharded_master_equation``)."""
        from . import engine, sharded
        from ._lib import PB200Error

        sim = self._sim_obj
        master = _sharded_master_equation(sim.noise_model)
        sim._validate_options({})
        if not master:
            # the master equation runs exactly at any size here: no Monte-Carlo fallback needs a trajectory count
            sim._check_supported()
        n_dev = engine.device_count()
        missing = sorted({d for d in devices if d >= n_dev})
        if missing:
            raise ValueError(f"`devices` names CUDA device(s) {missing}, but {n_dev} are visible")
        atom_order = tuple(sim._register.qubit_ids)
        if master:
            with engine.DevicePlan(sim._noiseless_spec(), sim._interp_order, devices[0]) as hplan:
                return self._stream_density(hplan, atom_order, devices)[0]
        res = Results(atom_order=atom_order, total_duration=sim.total_duration_ns)
        try:
            plan = sharded.ShardedPlan(sim._noiseless_spec(), devices, sim._interp_order)
        except PB200Error as e:
            if e.code == -3:  # PB200_ERR_UNSUPPORTED: outside what the sharded Taylor propagator covers
                raise NotImplementedError(str(e)) from e
            raise
        with plan:
            self._stream(plan, res)
        return res

    def run(self) -> Results:
        from . import engine

        sim = self._sim_obj
        devices = getattr(self._config, "_backend_options", {}).get("devices")
        if devices is not None:
            return self._run_sharded(devices)
        opts = {"print_progress": self._config.print_progress, "progress_bar": self._config.progress_bar}
        atom_order = tuple(sim._register.qubit_ids)
        with engine.DevicePlan(sim._noiseless_spec(sim.noise_model.with_leakage), sim._interp_order, sim._gpu) as hplan:
            if not sim.noise_model.noise_types:
                # no noise at all: the evolved Hamiltonian IS the noiseless one handed to the observables
                sim._validate_options({})
                sim._check_supported()
                res = Results(atom_order=atom_order, total_duration=sim.total_duration_ns)
                self._stream(hplan, res)
                return res
            if not _has_stochastic_noise(sim.noise_model):
                if self._streams_density():
                    sim._validate_options({})
                    sim._check_supported()
                    return self._stream_density(hplan, atom_order)[0]
                with warnings.catch_warnings():
                    warnings.simplefilter("ignore", DeprecationWarning)
                    single = sim.run(**opts)
                res = Results(atom_order=atom_order, total_duration=sim.total_duration_ns)
                self._replay(hplan, single, res)
                return res
            results: list[Results] = []
            sim._validate_options({})
            sim._check_supported()
            if not sim._has_collapse_ops() or sim._use_mcwf():
                # pure states: observables reduce on the device, nothing is stored per evaluation time
                streamed = self._stream_noisy(hplan, atom_order)
                return Results.aggregate(streamed, **_state_aggregators(streamed))
            if self._streams_density():
                # density matrices: observables reduce on the device, nothing is stored per evaluation time
                streamed = self._stream_density(hplan, atom_order)
                return Results.aggregate(streamed, **_state_aggregators(streamed))
            for cleanres, reps in sim._noisy_runs(print_progress=self._config.print_progress, batch=0,
                                                  opts={"max_step": 0, "cheb_tol": 0.0, "refine_window": -1, "tol": 0.0}):
                for _ in range(reps):
                    res = Results(atom_order=atom_order, total_duration=sim.total_duration_ns)
                    self._replay(hplan, cleanres, res)
                    results.append(res)
            return Results.aggregate(results, **_state_aggregators(results))


# noise types that are collapse operators of the master equation, with no stochastic part
_COLLAPSE_NOISE = frozenset({"dephasing", "relaxation", "depolarizing", "eff_noise"})


def _sharded_master_equation(noise_model: Any) -> bool:
    """Does a run with ``devices`` split a density matrix (True) or a state vector (False, no noise)?  Raises
    ``NotImplementedError`` with the reason for any noise model that neither covers."""
    types = set(noise_model.noise_types)
    if not types:
        return False
    if "leakage" in types:
        raise NotImplementedError(
            "a density matrix split over `devices` needs a d = 2 register; leakage (d = 3) is not sharded"
        )
    if not types <= _COLLAPSE_NOISE or _has_stochastic_noise(noise_model):
        raise NotImplementedError(
            "a state split over `devices` runs noiseless sequences and master equations without stochastic noise "
            f"(dephasing, relaxation, depolarizing, eff_noise); this one has the noise types {sorted(types)}"
        )
    return True


class B200LegacyBackend(pulser.backend.abc.Backend):
    """Mirror of the deprecated V1 backend ``pulser_simulation.QutipBackend``
    (``pulser-simulation/pulser_simulation/qutip_backend.py:44-118``): takes an
    ``EmulatorConfig`` and returns ``CoherentResults`` / ``NoisyResults`` from
    ``B200Emulator.run``.  Same checks, messages and deprecation warning."""

    def __init__(self, sequence: pulser.Sequence, config: Any = None, mimic_qpu: bool = False):
        from pulser.backend.config import EmulatorConfig

        with warnings.catch_warnings():
            warnings.simplefilter("once")
            warnings.warn(
                "'QutipBackend' is deprecated. Please use "
                "'pulser_simulation.QutipBackendV2' instead.",
                DeprecationWarning,
                stacklevel=2,
            )
        super().__init__(sequence, mimic_qpu=mimic_qpu)
        if config is None:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore", DeprecationWarning)
                config = EmulatorConfig()
        if not isinstance(config, EmulatorConfig):
            raise TypeError(
                "'config' must be of type 'EmulatorConfig', "
                f"not {type(config)}."
            )
        self._config = config
        noise_model = None
        if self._config.prefer_device_noise_model:
            noise_model = sequence.device.noise_model
        self._sim_obj = B200Emulator.from_sequence(
            sequence,
            sampling_rate=self._config.sampling_rate,
            noise_model=noise_model or self._config.noise_model,
            evaluation_times=self._config.evaluation_times,
            with_modulation=self._config.with_modulation,
        )
        self._sim_obj.set_initial_state(self._config.initial_state)

    def run(self, progress_bar: bool = False, **options: Any) -> Any:
        """Emulates the sequence on the GPU (``QutipBackend.run``, ``qutip_backend.py:89-118``); QuTiP solver
        options are accepted and ignored like in ``B200Emulator.run``."""
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", DeprecationWarning)
            return self._sim_obj.run(progress_bar=progress_bar, **options)
