"""The exact piecewise-cubic reference of tests/taylor_ref.py, pinned on the CPU: its ``H(t) v`` against the matrix-free
oracle, its evolution against dense ``expm`` where H is constant and against the DOP853 oracle where it is not, and
against itself with halved sub-steps."""
import numpy as np
import pytest
from scipy.linalg import expm

from helpers import curved_spec, random_state, with_dmm
from pulser_b200 import workloads as W
from taylor_ref import PiecewiseCubicHamiltonian


def _noisy(base, n_traj=2, seed=1):
    coords = W.disc_register(base.n_qudits, 20.0, 6.0, 3)
    rng = np.random.default_rng(seed)
    return [W.noisy_trajectory_spec(base, coords, rng.normal(0, 1.5, base.n_qudits), 1.0 + 0.05 * rng.normal(), 60.0)
            for _ in range(n_traj)]


def _specs(n):
    c2 = W.config_c2(n=n, seed=2, t_rise=40, t_sweep=100, t_fall=40)
    curved = curved_spec(n, T=160, phase=0.83)
    return {
        "c2": c2,
        "blackman": curved,
        "dmm1": with_dmm(c2, 1),
        "dmm4": with_dmm(curved_spec(n, T=160), 4, seed=5),
        "noisy": _noisy(curved)[1],
    }


@pytest.mark.parametrize("name", ["c2", "blackman", "dmm1", "dmm4", "noisy"])
def test_apply_matches_matfree(name):
    from oracle.matfree import MatFreeHamiltonian

    spec = _specs(7)[name]
    ref, mf = PiecewiseCubicHamiltonian(spec), MatFreeHamiltonian(spec)
    rng = np.random.default_rng(1)
    v = random_state(spec.hilbert_dim, 2)
    tf = spec.sampling_times[-1]
    for t in list(rng.uniform(0.0, tf, 6)) + [0.0, 0.0013, tf - 3e-4, tf]:
        a, b = ref.apply(t, v), mf.apply(t, v)
        assert np.linalg.norm(a - b) <= 1e-13 * np.linalg.norm(b), t


@pytest.mark.parametrize("n", [3, 6, 8])
def test_constant_hamiltonian_against_expm(n):
    """constant samples (per-qubit complex drives and detunings, Ising interaction): H is constant and the reference
    equals ``expm(-i H T) psi`` on any window"""
    from oracle.matfree import MatFreeHamiltonian

    rng = np.random.default_rng(n)
    T = 40
    spec = W.ising_global_spec(W.disc_register(n, 10.0, 5.0, n), W.C6_LEVEL_60, np.full(T, 9.0), np.full(T, -4.0))
    d = spec.drives[0]
    nt = spec.n_times
    d.coef = np.repeat((rng.uniform(2, 6, n) * np.exp(1j * rng.uniform(-3, 3, n)))[:, None], nt, axis=1)
    d.det = np.repeat(rng.uniform(-8, 8, n)[:, None], nt, axis=1)
    d.uniform = False
    ref = PiecewiseCubicHamiltonian(spec)
    D = spec.hilbert_dim
    H = np.stack([MatFreeHamiltonian(spec).apply(0.01, e) for e in np.eye(D)], axis=1)
    psi = random_state(D, 3)
    for a, b in ((0.0, 0.04), (0.0031, 0.0207), (0.0123, 0.0124)):
        got = ref.evolve(psi, a, b)
        want = expm(-1j * H * (b - a)) @ psi
        assert np.linalg.norm(got - want) <= 1e-13, (a, b)


@pytest.mark.parametrize("name", ["c2", "blackman", "dmm1", "dmm4", "noisy"])
def test_against_dop853_and_halved_substeps(name):
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    spec = _specs(6)[name]
    ref = PiecewiseCubicHamiltonian(spec)
    psi = random_state(spec.hilbert_dim, 7)
    a, b = 0.0123, spec.sampling_times[-1] - 0.0077      # off-grid ends, across the kinks of the C2 waveforms
    got = ref.evolve(psi, a, b)
    # DOP853 stopped at every sampling time, so that none of its steps straddles a knot of the splines
    cuts = [a] + [t for t in spec.sampling_times if a < t < b] + [b]
    want = evolve.sesolve(OracleHamiltonian.from_spec(spec), psi, cuts, rtol=1e-13, atol=1e-15)[-1]
    assert np.linalg.norm(got - want) <= 1e-11
    assert np.linalg.norm(got - ref.evolve(psi, a, b, split=2)) <= 1e-14
