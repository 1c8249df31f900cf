"""Shared builders of seeded test inputs (no pulser needed)."""
from __future__ import annotations

import numpy as np

from pulser_b200 import workloads as W
from pulser_b200.spec import DriveTable, HamiltonianSpec


def chain_coords(n: int, spacing: float = 7.0, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    pts = np.array([[i * spacing, 0.0] for i in range(n)], dtype=float)
    return pts + rng.uniform(-0.8, 0.8, size=pts.shape)


def random_local_spec(
    n: int, T: int = 200, seed: int = 1, phase: bool = True, c6: float = W.C6_LEVEL_60
) -> HamiltonianSpec:
    """Per-qubit smooth random amp/det/phase tables (a noisy-trajectory look-alike)."""
    rng = np.random.default_rng(seed)
    t = np.arange(T + 1) / T
    base_amp = 8.0 * np.sin(np.pi * t) ** 2
    base_det = -10.0 + 25.0 * t
    coef = np.zeros((n, T + 1), dtype=complex)
    det = np.zeros((n, T + 1))
    for k in range(n):
        a = base_amp * rng.uniform(0.7, 1.1)
        ph = (rng.uniform(-1, 1) + rng.uniform(-2, 2) * t) if phase else 0.0
        coef[k] = 0.5 * a * np.exp(-1j * ph)
        det[k] = base_det + rng.normal(0, 2.0)
        det[k, -1] = 0.0
        coef[k, -1] = 0.0
    coords = chain_coords(n, 7.0, seed)
    return HamiltonianSpec(
        n_qudits=n, dim=2, eigenbasis=["r", "g"], basis_name="ground-rydberg",
        interaction_type="ising",
        sampling_times=np.arange(T + 1, dtype=float) / 1000,
        total_duration_ns=T,
        interaction_matrix=W.interaction_matrix(coords, c6),
        bad_atoms=np.zeros(n, dtype=bool),
        drives=[DriveTable("ground-rydberg", coef, det, False)],
        collapse_ops=np.zeros((0, 2, 2), dtype=complex),
        qubit_ids=[f"q{i}" for i in range(n)],
    )


OPEN_EIGENBASIS = {2: ["r", "g"], 3: ["r", "g", "x"], 4: ["r", "g", "h", "x"]}


def open_spec(
    n: int, d: int = 2, T: int = 40, seed: int = 0, drive: bool = True, detuning: bool = True,
    interaction: bool = True, ops=None, step_ns: int = 1,
) -> HamiltonianSpec:
    """Ground-rydberg register of ``d`` levels (``r, g`` first) with per-qudit smooth random tables on ``T`` sampling
    intervals of ``step_ns``: a complex drive (or none), a time-dependent detuning (or none) and a chain interaction
    (or none), plus collapse operators."""
    rng = np.random.default_rng(seed)
    t = np.arange(T + 1) / T
    coef = np.zeros((n, T + 1), dtype=complex)
    det = np.zeros((n, T + 1))
    for k in range(n):
        if drive:
            ph = rng.uniform(-1, 1) + rng.uniform(-2, 2) * t
            coef[k] = 0.5 * rng.uniform(6.0, 10.0) * np.sin(np.pi * t) ** 2 * np.exp(-1j * ph)
        if detuning:
            det[k] = rng.uniform(-8, 8) + rng.uniform(-10, 10) * t + rng.uniform(-5, 5) * np.sin(3 * np.pi * t)
    imat = W.interaction_matrix(chain_coords(n, 7.0, seed), W.C6_LEVEL_60)
    if not interaction:
        imat = np.zeros_like(imat)
    return HamiltonianSpec(
        n_qudits=n, dim=d, eigenbasis=list(OPEN_EIGENBASIS[d]), basis_name="ground-rydberg",
        interaction_type="ising",
        sampling_times=np.arange(T + 1, dtype=float) * step_ns / 1000,
        total_duration_ns=T * step_ns,
        interaction_matrix=imat,
        bad_atoms=np.zeros(n, dtype=bool),
        drives=[DriveTable("ground-rydberg", coef, det, False)],
        collapse_ops=np.zeros((0, d, d), dtype=complex) if ops is None else np.asarray(ops, dtype=complex),
        qubit_ids=[f"q{i}" for i in range(n)],
    )


def curved_spec(n: int, T: int = 300, phase: float = 0.0, seed: int = 3, radius: float = 20.0,
                min_dist: float = 6.0, swing: float = 14.0) -> HamiltonianSpec:
    """Global drive with a Blackman amplitude (peak ~8 rad/us whatever T) and a sin^2 detuning of amplitude ``swing``:
    smooth curved waveforms, so that a polynomial of degree above 3 spans several sampling intervals"""
    t = np.arange(T)
    amp = W.blackman(T, 2.2 * np.pi * T / 600)
    det = -6.0 + swing * np.sin(1.3 * np.pi * t / T) ** 2
    coords = W.disc_register(n, radius, min_dist, seed)
    return W.ising_global_spec(coords, W.C6_LEVEL_60, amp, det, phase=phase)


def dmm_waveforms(T: int) -> list[np.ndarray]:
    """four detuning-map waveforms of different time shapes (negative, as a DMM allows)"""
    t = np.arange(T)
    return [
        -4.0 * np.sin(np.pi * t / T) ** 2,
        -np.concatenate([np.linspace(0.0, 5.0, T // 2), np.full(T - T // 2, 5.0)]),
        -2.0 * (1.0 + np.sin(5.0 * np.pi * t / T)),
        -1.5 * np.cos(3.0 * np.pi * t / T) ** 2,
    ]


def with_dmm(base: HamiltonianSpec, n_maps: int, seed: int = 0) -> HamiltonianSpec:
    """``base`` plus ``n_maps`` detuning maps with random weights on different subsets of the atoms"""
    n = base.n_qudits
    rng = np.random.default_rng(seed)
    wfs = dmm_waveforms(base.total_duration_ns)
    maps = [(rng.uniform(0.2, 1.0, n) * (np.arange(n) % (s + 2) != 0), wfs[s]) for s in range(n_maps)]
    return W.detuning_map_spec(base, maps)


def random_state(D: int, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    v = rng.normal(size=D) + 1j * rng.normal(size=D)
    return v / np.linalg.norm(v)
