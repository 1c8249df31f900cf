"""Synthetic workloads of BASELINE.json ``configs`` as plain-array specs.

pulser is an optional dependency, so the benchmark and
the GPU parity tests build their inputs here with numpy only, restating what
``pulser.sampler.sample`` + ``HamiltonianData`` produce for these sequences
(waveform formulas: reference ``pulser-core/pulser/waveforms.py:584`` constant,
``:661-674`` ramp, ``:740-743`` Blackman; C6 coefficients:
``pulser-core/pulser/devices/interaction_coefficients/``; interaction matrix
``pulser-core/pulser/_hamiltonian_data/hamiltonian_data.py:607-611``; the
zero-padded extra sample ``pulser-simulation/pulser_simulation/simulation.py:172-173``).
``tests/test_oracle_cpu.py`` checks the builders against what the real
pulser objects produce (stored in ``tests/golden/pulser_*.npz``).

Definitions follow SURVEY.md section 8(d).
"""
from __future__ import annotations

import numpy as np

from .spec import DriveTable, HamiltonianSpec

# device.interaction_coeff (rad/us * um^6)
C6_LEVEL_70 = 5420158.53  # MockDevice, DigitalAnalogDevice
C6_LEVEL_60 = 865723.02  # AnalogDevice


# ---------------------------------------------------------------- waveforms
def ramp(duration: int, start: float, stop: float) -> np.ndarray:
    slope = (stop - start) / (duration - 1)
    lo, hi = sorted([float(start), float(stop)])
    return np.clip(slope * np.arange(duration, dtype=float) + start, lo, hi)


def constant(duration: int, value: float) -> np.ndarray:
    return value * np.ones(duration)


def blackman(duration: int, area: float) -> np.ndarray:
    norm = np.clip(np.blackman(duration), 0, np.inf)
    return norm * (area / np.sum(norm) * 1e3)


# ---------------------------------------------------------------- registers
def disc_register(
    n: int, radius: float, min_dist: float, seed: int
) -> np.ndarray:
    """n points uniform in a disc with rejection on the minimum distance."""
    rng = np.random.default_rng(seed)
    pts: list[np.ndarray] = []
    while len(pts) < n:
        p = rng.uniform(-radius, radius, size=2)
        if np.hypot(*p) > radius:
            continue
        if all(np.hypot(*(p - q)) >= min_dist for q in pts):
            pts.append(np.round(p, 6))
    return np.array(pts)


def square_register(side: int, spacing: float) -> np.ndarray:
    """``Register.square(side, spacing)`` coordinates (centred, row-major).

    Reference ``pulser-core/pulser/register/register.py`` (rectangle:
    ``coords = [(x, y) for y in rows for x in columns] * spacing``, centred).
    """
    coords = (
        np.array(
            [(x, y) for y in range(side) for x in range(side)], dtype=float
        )
        * spacing
    )
    return coords - np.mean(coords, axis=0)


def interaction_matrix(coords: np.ndarray, c6: float) -> np.ndarray:
    """(1, N, N) C6/r^6 as ``HamiltonianData._interaction_matrix``."""
    from scipy.spatial.distance import cdist

    pts = np.round(np.asarray(coords, dtype=float), 6)
    d = np.round(cdist(pts, pts), 6)  # COORD_PRECISION = 6
    n = len(pts)
    out = np.zeros((1, n, n))
    iu = np.triu_indices(n, 1)
    out[0][iu] = c6 / d[iu] ** 6
    out[0] = out[0] + out[0].T
    return out


# ---------------------------------------------------------------- spec
def ising_global_spec(
    coords: np.ndarray,
    c6: float,
    amp: np.ndarray,
    det: np.ndarray,
    phase: np.ndarray | float = 0.0,
    basis_name: str = "ground-rydberg",
) -> HamiltonianSpec:
    """Global ground-rydberg drive over ``len(amp)`` ns, sampling_rate 1.

    Adds the zero-padded extra sample of ``extend_duration(T+1)``
    (amp, det -> 0; phase -> edge value; reference ``samples.py:152-200``).
    """
    n = len(coords)
    T = len(amp)
    phase = np.broadcast_to(np.asarray(phase, dtype=float), (T,))
    amp_e = np.append(amp, 0.0)
    det_e = np.append(det, 0.0)
    phase_e = np.append(phase, phase[-1])
    coef = 0.5 * amp_e * np.exp(-1j * phase_e)
    return HamiltonianSpec(
        n_qudits=n,
        dim=2,
        eigenbasis=["r", "g"],
        basis_name=basis_name,
        interaction_type="ising",
        sampling_times=np.arange(T + 1, dtype=np.double) / 1000,
        total_duration_ns=T,
        interaction_matrix=interaction_matrix(coords, c6),
        bad_atoms=np.zeros(n, dtype=bool),
        drives=[
            DriveTable(
                "ground-rydberg",
                np.repeat(coef[None, :], n, axis=0),
                np.repeat(det_e[None, :], n, axis=0),
                True,
            )
        ],
        collapse_ops=np.zeros((0, 2, 2), dtype=np.complex128),
        qubit_ids=[f"q{i}" for i in range(n)],
    )


def blockade_sweep_waveforms(
    omega: float = 2 * np.pi * 1.5,
    t_rise: int = 500,
    t_sweep: int = 2500,
    t_fall: int = 1000,
) -> tuple[np.ndarray, np.ndarray]:
    """Rise / detuning sweep / fall of SURVEY 8(d) C2 (ends at Omega = 0)."""
    U = omega / 2
    d0, df = -6 * U, 2 * U
    amp = np.concatenate(
        [ramp(t_rise, 0.0, omega), constant(t_sweep, omega), ramp(t_fall, omega, 0.0)]
    )
    det = np.concatenate(
        [constant(t_rise, d0), ramp(t_sweep, d0, df), constant(t_fall, df)]
    )
    return amp, det


def config_c1() -> HamiltonianSpec:
    """C1: 4-atom square, constant Omega/delta pulse, 1000 ns (MockDevice)."""
    coords = square_register(2, 6.0)
    return ising_global_spec(
        coords, C6_LEVEL_70, constant(1000, 2 * np.pi), constant(1000, np.pi)
    )


def config_c2(n: int = 20, seed: int | None = None, **kw) -> HamiltonianSpec:
    """C2: n-atom random 2D register (AnalogDevice limits), blockade sweep."""
    coords = disc_register(n, 38.0, 5.0, n if seed is None else seed)
    amp, det = blockade_sweep_waveforms(**kw)
    return ising_global_spec(coords, C6_LEVEL_60, amp, det)


def config_c5(n: int = 24, t_total: int = 4000) -> HamiltonianSpec:
    """C5: n-atom adiabatic anneal 0 -> Omega -> 0 with a detuning ramp."""
    coords = disc_register(n, 38.0, 5.0, n)
    omega = 2 * np.pi * 1.5
    U = omega / 2
    t_edge = t_total // 4
    amp = np.concatenate(
        [
            ramp(t_edge, 0.0, omega),
            constant(t_total - 2 * t_edge, omega),
            ramp(t_edge, omega, 0.0),
        ]
    )
    det = ramp(t_total, -6 * U, 2 * U)
    return ising_global_spec(coords, C6_LEVEL_60, amp, det)


# ---------------------------------------------------------------- noisy trajectories (C4)
KEFF = 8.7  # rad/us per (um/us), pulser-core/pulser/constants.py (conversion in noise_model._doppler_sigma)


def doppler_sigma(temperature_uK: float) -> float:
    """``pulser.noise_model._doppler_sigma`` (CORE/noise_model.py:127-133):
    KEFF * sqrt(KB * T / MASS) with T in K."""
    KB = 1.38e-23
    MASS = 1.45e-25
    return KEFF * float(np.sqrt(KB * temperature_uK * 1e-6 / MASS))


def waist_amp_fraction(coords: np.ndarray, waist: float, prop_dir=(0.0, 1.0, 0.0)) -> np.ndarray:
    """Gaussian-beam amplitude loss per atom for a global channel
    (``HamiltonianData._finite_waist_amp_fraction``, hamiltonian_data.py:758-780):
    exp(-(distance to the optical axis / waist)^2), axis along ``prop_dir``."""
    pts = np.zeros((len(coords), 3))
    pts[:, : coords.shape[1]] = coords
    u = np.asarray(prop_dir, dtype=float)
    u = u / np.linalg.norm(u)
    perp = pts - np.outer(pts @ u, u)
    return np.exp(-(np.linalg.norm(perp, axis=1) / waist) ** 2)


def noisy_trajectory_spec(base: HamiltonianSpec, coords: np.ndarray, doppler: np.ndarray, amp_fluct: float,
                          waist: float | None, slot_mask: np.ndarray | None = None) -> HamiltonianSpec:
    """One noise trajectory of a global ground-rydberg sequence (doppler + amplitude noise),
    restating ``HamiltonianData._sample_with_trajectory`` (hamiltonian_data.py:408-534): inside the pulse
    slots det_k += doppler_k and amp_k *= amp_fluct * waist_fraction_k; all samples become Local."""
    import copy

    n = base.n_qudits
    d0 = base.drives[0]
    nt = d0.coef.shape[1]
    mask = np.ones(nt) if slot_mask is None else slot_mask
    if slot_mask is None:
        mask[-1] = 0.0  # the zero-padded extra sample lies outside every slot
    frac = amp_fluct * (waist_amp_fraction(coords, waist) if waist is not None else np.ones(n))
    coef = d0.coef * np.where(mask[None, :] > 0, frac[:, None], 1.0)
    det = d0.det + np.asarray(doppler)[:, None] * mask[None, :]
    spec = copy.copy(base)
    spec.drives = [DriveTable(d0.basis, coef, det, False)]
    return spec


def detuning_map_spec(base: HamiltonianSpec, maps) -> HamiltonianSpec:
    """Detuning maps on a ground-rydberg sequence: ``maps`` is a list of ``(weights, waveform)``, one per detuning map
    modulator (``Sequence.config_detuning_map`` + ``add_dmm_detuning``); atom k's detuning gains
    ``sum weights[k] * waveform(t)``, as the reference samples it (``samples.py:560-601``: det += cs.det * weight).
    A waveform has one sample per ns; the zero-padded extra sample gets 0.  All samples become Local."""
    import copy

    d0 = base.drives[0]
    nt = d0.det.shape[1]
    det = np.array(d0.det, dtype=float)
    for weights, waveform in maps:
        wf = np.zeros(nt)
        wf[: len(waveform)] = waveform
        det = det + np.outer(np.asarray(weights, dtype=float), wf)
    spec = copy.copy(base)
    spec.drives = [DriveTable(d0.basis, np.array(d0.coef), det, False)]
    return spec


def config_c4_stream(n_traj: int = 1024, seed: int = 4, side: int = 4, temperature: float = 50.0,
                     amp_sigma: float = 0.05, laser_waist: float = 175.0, keep=None):
    """Generator over the C4 trajectories in order: yields ``(j, spec)``; with ``keep`` (a set of indices) the other
    trajectories only advance the random stream, so that every rank of a striped run draws the same list without
    materialising the 1.5 MB of per-atom sample tables of the trajectories it does not own."""
    coords = square_register(side, 6.0)
    amp, det = blockade_sweep_waveforms()
    base = ising_global_spec(coords, C6_LEVEL_70, amp, det)
    rng = np.random.default_rng(seed)
    sig = doppler_sigma(temperature)
    for j in range(n_traj):
        dop = rng.normal(0.0, sig, size=len(coords))
        fl = max(0.0, rng.normal(1.0, amp_sigma))
        if keep is None or j in keep:
            yield j, noisy_trajectory_spec(base, coords, dop, fl, laser_waist)


def config_c4(n_traj: int = 1024, seed: int = 4, side: int = 4, temperature: float = 50.0,
              amp_sigma: float = 0.05, laser_waist: float = 175.0) -> list[HamiltonianSpec]:
    """C4: 16-atom 4x4 square (6 um), blockade sweep, doppler + amplitude noise trajectories."""
    return [s for _, s in config_c4_stream(n_traj, seed, side, temperature, amp_sigma, laser_waist)]


# ---------------------------------------------------------------- 3-level "all" basis (C3)
def config_c3(n: int = 14, seed: int | None = None, t_raman: int = 500, t_ryd: int = 1000) -> HamiltonianSpec:
    """C3: n atoms, basis "all" (eigenbasis r, g, h): raman_global Blackman pi/2, then
    rydberg_global Blackman pi, then raman_global Blackman pi/2 again (MockDevice)."""
    coords = disc_register(n, 22.0, 6.0, (100 + n) if seed is None else seed)
    T = 2 * t_raman + t_ryd
    amp_dig = np.zeros(T)
    amp_dig[:t_raman] = blackman(t_raman, np.pi / 2)
    amp_dig[t_raman + t_ryd:] = blackman(t_raman, np.pi / 2)
    amp_ryd = np.zeros(T)
    amp_ryd[t_raman:t_raman + t_ryd] = blackman(t_ryd, np.pi)

    def table(basis: str, amp: np.ndarray) -> DriveTable:
        coef = 0.5 * np.append(amp, 0.0).astype(np.complex128)
        return DriveTable(basis, np.repeat(coef[None, :], n, axis=0), np.zeros((n, T + 1)), True)

    return HamiltonianSpec(
        n_qudits=n, dim=3, eigenbasis=["r", "g", "h"], basis_name="all", interaction_type="ising",
        sampling_times=np.arange(T + 1, dtype=np.double) / 1000, total_duration_ns=T,
        interaction_matrix=interaction_matrix(coords, C6_LEVEL_70), bad_atoms=np.zeros(n, dtype=bool),
        drives=[table("ground-rydberg", amp_ryd), table("digital", amp_dig)],
        collapse_ops=np.zeros((0, 3, 3), dtype=np.complex128), qubit_ids=[f"q{i}" for i in range(n)],
    )


# ---------------------------------------------------------------- XY mode (microwave channel)
C3_XY = 36288.3559282823  # device.interaction_coeff_xy at Rydberg level 70 (MockDevice), rad/us * um^3


def xy_interaction_matrix(coords: np.ndarray, c3: float, c6: float, magnetic_field=(0.0, 0.0, 30.0)) -> np.ndarray:
    """(2, N, N): [0] = C3 (1 - 3 cos^2 theta) / r^3, [1] = C6 / r^6
    (``HamiltonianData._interaction_matrix``, hamiltonian_data.py:585-611)."""
    n = len(coords)
    pts = np.zeros((n, 3))
    pts[:, : coords.shape[1]] = np.round(np.asarray(coords, dtype=float), 6)
    mag = np.asarray(magnetic_field, dtype=float)
    out = np.zeros((2, n, n))
    out[1] = interaction_matrix(coords, c6)[0]
    for i in range(n):
        for j in range(i + 1, n):
            diff = pts[i] - pts[j]
            r = np.round(np.linalg.norm(diff), 6)
            cosine = diff @ mag / (np.linalg.norm(diff) * np.linalg.norm(mag))
            out[0, i, j] = out[0, j, i] = c3 * (1 - 3 * cosine**2) / r**3
    return out


def config_xy(n: int = 8, seed: int = 7, t_total: int = 600, local_rows: bool = False,
              magnetic_field=(0.0, 0.0, 30.0)) -> HamiltonianSpec:
    """n-atom XY-mode register driven by a global microwave pulse (Blackman envelope, constant detuning)."""
    coords = disc_register(n, 30.0, 8.0, seed)
    amp = np.append(blackman(t_total, 1.5 * np.pi), 0.0)
    det = np.append(constant(t_total, 0.8), 0.0)
    coef = np.repeat((0.5 * amp.astype(np.complex128))[None, :], n, axis=0)
    dets = np.repeat(det[None, :], n, axis=0)
    if local_rows:  # per-atom amplitude / detuning spread, as a noise trajectory would have
        rng = np.random.default_rng(seed + 1)
        coef = coef * rng.normal(1.0, 0.05, size=(n, 1))
        dets = dets + rng.normal(0.0, 0.3, size=(n, 1)) * (np.arange(t_total + 1) < t_total)
    return HamiltonianSpec(
        n_qudits=n, dim=2, eigenbasis=["u", "d"], basis_name="XY", interaction_type="XY",
        sampling_times=np.arange(t_total + 1, dtype=np.double) / 1000, total_duration_ns=t_total,
        interaction_matrix=xy_interaction_matrix(coords, C3_XY, C6_LEVEL_70, magnetic_field),
        bad_atoms=np.zeros(n, dtype=bool), drives=[DriveTable("XY", coef, dets, not local_rows)],
        collapse_ops=np.zeros((0, 2, 2), dtype=np.complex128), qubit_ids=[f"q{i}" for i in range(n)],
    )
