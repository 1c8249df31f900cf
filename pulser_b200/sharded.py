"""One state split over several plans: registers larger than one GPU.

``ShardedPlan(spec, devices=[...])`` splits the ``2**N`` amplitudes of one state over
``G = len(devices)`` shards (2, 4 or 8).  Shard ``i`` holds the global indices
``[i 2**L, (i+1) 2**L)``, ``L = N - log2(G)``: the top qubits select the shard.  Each shard is
an ordinary plan on ``devices[i]`` (several shards may share a device), and one process drives
them all: ``pb200_shards_propagate`` runs every order of the time-dependent Taylor series on every
shard, whose partners across the shard bits are read from the peers' slices.

Scope: what the Taylor propagator takes with one state -- d = 2, one global drive (its phase may
change in time: phase shifts, phase jumps between pulses, EOM drift correction), per-qubit detuning
of up to 4 time shapes (detuning maps), Ising interaction.  The methods mirror the single-state methods of ``DevicePlan`` that
``B200Backend._stream``, ``DeviceStateView`` and ``DeviceHamiltonian`` call, with the same shapes
(a leading trajectory axis of 1).
"""
from __future__ import annotations

import ctypes as C
from collections import Counter
from typing import Sequence

import numpy as np

from ._lib import RunOpts, RunStats, check, lib
from .engine import DevicePlan, _p, all_ground_index
from .spec import HamiltonianSpec

MIN_LOCAL_BITS, MAX_LOCAL_BITS = 13, 29


def shard_bits_of(n_shards: int) -> int:
    """``log2(n_shards)`` for 2, 4 or 8 shards; ``ValueError`` otherwise."""
    if n_shards not in (2, 4, 8):
        raise ValueError(f"a state splits into 2, 4 or 8 shards, not {n_shards}")
    return n_shards.bit_length() - 1


def validate_devices(devices) -> list[int]:
    """The ``devices`` option: a list of ``G`` CUDA ordinals (G = 2, 4 or 8), ``devices[i]`` = shard i's."""
    if isinstance(devices, (str, bytes)) or not isinstance(devices, Sequence):
        raise TypeError(f"`devices` must be a list of CUDA device ordinals, not {type(devices).__name__}")
    out = []
    for d in devices:
        if isinstance(d, bool) or not isinstance(d, (int, np.integer)) or d < 0:
            raise TypeError(f"`devices` holds CUDA device ordinals (ints >= 0), got {d!r}")
        out.append(int(d))
    shard_bits_of(len(out))
    return out


def route_shots(u: np.ndarray, shard_weights: np.ndarray, reverse: bool) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Route uniforms ``u`` to shards by their cumulative weights in global bitstring order.

    In bitstring order the shards are blocks of ``2**L`` bitstrings; ``reverse`` when the bitstring is the complement
    of the state index (ground-rydberg basis: bit = [digit == r], r is digit 0), i.e. shard ``G - 1`` comes first.
    Returns, per shot, the shard, its block in bitstring order (the top bits of the bitstring) and the uniform
    rescaled into that shard's weight, so that a search of the shard's own cumulative weights with it finds the
    bitstring the search over the concatenated weights finds.
    """
    w = np.asarray(shard_weights, dtype=np.float64)
    g = len(w)
    order = np.arange(g)[::-1] if reverse else np.arange(g)
    wo = w[order]
    cum = np.cumsum(wo)
    target = np.asarray(u, dtype=np.float64) * cum[-1]
    pos = np.minimum(np.searchsorted(cum, target, side="left"), g - 1)
    # only u = 0 can land on an empty leading block: move it to the first block that has weight
    empty = wo[pos] <= 0.0
    if np.any(empty):
        pos[empty] = int(np.argmax(wo > 0.0))
    prev = cum[pos] - wo[pos]
    local_u = np.clip((target - prev) / wo[pos], 0.0, 1.0)
    return order[pos], pos, local_u


def global_bitstring(block: np.ndarray, local_b: np.ndarray, local_bits: int) -> np.ndarray:
    """Bitstring index from a shard's block in bitstring order and the low ``local_bits`` bits it sampled."""
    return (np.asarray(block, dtype=np.int64) << local_bits) | np.asarray(local_b, dtype=np.int64)


class ShardedPlan:
    """One state of ``spec`` split over ``len(devices)`` shards; ``devices[i]`` is shard i's CUDA device."""

    def __init__(self, spec: HamiltonianSpec, devices: Sequence[int], interp_order: int = 3) -> None:
        devices = validate_devices(devices)
        if isinstance(spec, (list, tuple)):
            if len(spec) != 1:
                raise NotImplementedError("a sharded plan holds one state (no trajectory batches)")
            spec = spec[0]
        self.spec = spec
        self.n_traj = 1
        self.n = spec.n_qudits
        self.dim = spec.dim
        self.G = len(devices)
        self.bits = shard_bits_of(self.G)
        self.L = self.n - self.bits
        self.devices = devices
        self.interp_order = interp_order
        if self.dim != 2:
            raise NotImplementedError(f"state-vector shards need a d = 2 register (this one has d = {self.dim})")
        if not MIN_LOCAL_BITS <= self.L <= MAX_LOCAL_BITS:
            raise ValueError(
                f"{self.G} shards of a {self.n}-qubit state hold 2^{self.L} amplitudes each; a shard holds "
                f"2^{MIN_LOCAL_BITS} to 2^{MAX_LOCAL_BITS}"
            )
        # per-qubit detuning (detuning maps) is the library's to accept or refuse; the drive rows must be identical
        # (one global drive, whatever its phase does in time)
        coef = np.asarray(spec.drives[0].coef) if len(spec.drives) == 1 else None
        if spec.interaction_type == "XY" or coef is None or not (coef == coef[:1]).all():
            raise NotImplementedError(
                "state-vector shards need one global drive (no XY interaction, per-qubit drive amplitudes or several "
                "bases)"
            )
        self.D = spec.hilbert_dim
        self.Dl = 1 << self.L
        self.shards: list[DevicePlan] = []
        self._arr = None
        try:
            for i, dev in enumerate(devices):
                self.shards.append(DevicePlan(spec, interp_order, dev, shard=(self.bits, i)))
            self._arr = (C.c_void_p * self.G)(*[s._handle for s in self.shards])
            check(lib.pb200_shards_link(self._arr, self.G))
        except Exception:
            self.close()
            raise

    # ------------------------------------------------------------------
    def close(self) -> None:
        for s in self.shards:
            s.close()
        self.shards = []
        self._arr = None

    def __del__(self) -> None:  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self) -> "ShardedPlan":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    # ------------------------------------------------------------------
    def set_state(self, psi: np.ndarray | str = "all-ground") -> None:
        """The all-ground state, or the full state vector ``psi[D]`` (each shard takes its slice)."""
        if isinstance(psi, str):
            if psi != "all-ground":
                raise ValueError(psi)
            idx = all_ground_index(self.spec)
            for s in self.shards:
                check(lib.pb200_state_set(s._handle, 0, 1, None, idx, 0))
            return
        psi = np.ascontiguousarray(psi, dtype=np.complex128).reshape(-1)
        if psi.size != self.D:
            raise ValueError(f"Incompatible shape of initial state.Expected {self.D}, got {psi.size}.")
        for i, s in enumerate(self.shards):
            part = np.ascontiguousarray(psi[i * self.Dl:(i + 1) * self.Dl])
            check(lib.pb200_state_set(s._handle, 0, 1, _p(part.view(np.float64)), -1, 1))

    def get_state(self, traj0: int = 0, count: int | None = None) -> np.ndarray:
        return np.concatenate([s.get_state()[0] for s in self.shards])[None, :]

    def norm2(self) -> np.ndarray:
        return np.array([sum(float(s.norm2()[0]) for s in self.shards)])

    def occupation(self, digit: int, traj0: int = 0, count: int | None = None) -> np.ndarray:
        return sum(s.occupation(digit) for s in self.shards)

    def correlation(self, digit: int, traj0: int = 0, count: int | None = None) -> np.ndarray:
        return sum(s.correlation(digit) for s in self.shards)

    def overlap(self, phi: np.ndarray, traj0: int = 0, count: int | None = None) -> np.ndarray:
        v = np.asarray(phi, dtype=np.complex128).reshape(-1)
        if v.shape[0] != self.D:
            raise ValueError(f"state of length {v.shape[0]}, expected {self.D}")
        return sum(s.overlap(v[i * self.Dl:(i + 1) * self.Dl]) for i, s in enumerate(self.shards))

    def expect_terms(self, terms, traj0: int = 0, count: int | None = None) -> np.ndarray:
        """``<psi|O|psi>`` of the whole state, ``O`` as monomial terms (``pb200_shards_expect``); shape ``[1]``."""
        if (terms.n, terms.d) != (self.n, self.dim):
            raise ValueError(f"operator on {terms.n} qudits of dimension {terms.d}, the plan holds {self.n} of {self.dim}")
        out = np.empty(2, dtype=np.float64)
        check(lib.pb200_shards_expect(self._arr, self.G, C.byref(terms.c_desc()), _p(out)))
        return np.array([complex(out[0], out[1])])

    def energy(self, t_us: float) -> tuple[np.ndarray, np.ndarray]:
        e = np.empty(1, dtype=np.float64)
        e2 = np.empty(1, dtype=np.float64)
        check(lib.pb200_shards_energy(self._arr, self.G, float(t_us), _p(e), _p(e2)))
        return e, e2

    def apply_h(self, t_us: float, vec: np.ndarray, traj: int = 0) -> np.ndarray:
        vec = np.ascontiguousarray(vec, dtype=np.complex128).reshape(-1)
        if vec.size != self.D:
            raise ValueError("vector has the wrong dimension")
        out = np.empty(self.D, dtype=np.complex128)
        check(lib.pb200_shards_apply_h(self._arr, self.G, float(t_us), _p(vec.view(np.float64)), _p(out.view(np.float64))))
        return out

    def sample(self, n_samples: int, one_state: str, traj: int = 0) -> "Counter[str]":
        """Bitstring samples with the single-plan recipe: one ``np.random.rand(n)`` call, each shot routed to a shard
        by the cumulative shard weights in bitstring order, then searched in that shard's cumulative weights."""
        u = np.random.rand(n_samples)
        one = self.spec.eigenbasis.index(one_state)
        weights = np.array([float(s.norm2()[0]) for s in self.shards])
        shard, block, local_u = route_shots(u, weights, reverse=(one == 0))
        local_b = np.zeros(n_samples, dtype=np.int64)
        for i, s in enumerate(self.shards):
            sel = np.nonzero(shard == i)[0]
            if sel.size == 0:
                continue
            ui = np.ascontiguousarray(local_u[sel], dtype=np.float64)
            idx = np.empty(sel.size, dtype=np.int64)
            check(lib.pb200_state_sample(s._handle, 0, one, _p(ui), int(sel.size), idx.ctypes.data_as(C.POINTER(C.c_int64))))
            local_b[sel] = idx
        b = global_bitstring(block, local_b, self.L)
        return Counter(np.binary_repr(int(i), self.n) for i in b)

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
        """Advance the state from ``t_start`` to ``t_stop`` (us) with the Taylor propagator; ``tol > 0`` sets the
        error budget, options that steer the Magnus controller are refused (``pb200_shards_propagate``)."""
        opts = RunOpts(max_step, refine_window, cheb_tol, rough_tol, magnus_order, check_every, tol, extrapolate, integrator)
        st = RunStats()
        check(lib.pb200_shards_propagate(self._arr, self.G, float(t_start), float(t_stop), C.byref(opts), C.byref(st)))
        return {f: getattr(st, f) for f, _ in RunStats._fields_}
