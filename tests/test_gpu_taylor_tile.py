"""GPU tests of the 2^13-amplitude tile of the Taylor stage kernel (``stage_d2_taylor_kernel``): a register of 13
qubits is one tile, larger ones add out-of-tile partner loads; 16 amplitudes per thread are worked through in two
chunks of 8, the top tile bit flipping between them.  Each drive kind the kernel instantiates is covered: a uniform
drive of phase 0 (real unit) and of phase != 0 (complex unit), and per-qubit static factors (trajectory batches)."""
import numpy as np
import pytest

from helpers import random_state
from pulser_b200 import workloads as W

pytestmark = pytest.mark.gpu

STATE_TOL = 1e-8


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


def _smooth_spec(n, phase, T):
    amp = W.blackman(T, 2.2 * np.pi)
    det = -8.0 + 20.0 * np.sin(np.linspace(0.0, 1.3, T)) ** 2
    coords = W.disc_register(n, 16.0, 5.0, 3)
    return W.ising_global_spec(coords, W.C6_LEVEL_60, amp, det, phase=phase)


@pytest.mark.parametrize("phase", [0.0, -2.1])
def test_one_tile_vs_oracle(engine, phase):
    """N = 13: the whole register is one tile (no partner loads), against the DOP853 oracle."""
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    spec = _smooth_spec(13, phase, T=200)
    psi0 = random_state(spec.hilbert_dim, 5)
    tf = spec.sampling_times[-1]
    ref = evolve.sesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf], rtol=1e-13, atol=1e-15)[-1]
    with engine.DevicePlan(spec) as plan:
        plan.set_state(psi0)
        st = plan.propagate(0.0, tf, integrator=3)
        got = plan.get_state()[0]
    assert st["integrator"] == 3
    assert np.max(np.abs(got - ref)) < STATE_TOL


@pytest.mark.parametrize("n,phase", [(15, 0.0), (15, 0.83)])
def test_partner_bits_vs_magnus(engine, n, phase):
    """N = 15: two bits outside the tile; the Taylor run agrees with the Richardson-CF4 run at a 100x tighter
    tolerance."""
    spec = _smooth_spec(n, phase, T=300)
    psi0 = random_state(spec.hilbert_dim, 7)
    tf = spec.sampling_times[-1]
    with engine.DevicePlan(spec) as plan:
        plan.set_state(psi0)
        st3 = plan.propagate(0.0, tf, integrator=3)
        got = plan.get_state()[0]
        plan.set_state(psi0)
        plan.propagate(0.0, tf, integrator=1, tol=1e-10)
        ref = plan.get_state()[0]
    assert st3["integrator"] == 3
    assert np.max(np.abs(got - ref)) < STATE_TOL


def test_trajectory_batch_vs_lanczos(engine):
    """N = 14 noise batch (per-qubit amplitude factors and doppler offsets, phase != 0): one bit outside the tile,
    blockIdx.y = trajectory; against the Magnus-Lanczos path trajectory by trajectory."""
    amp, det = W.blockade_sweep_waveforms(t_rise=60, t_sweep=150, t_fall=60)
    n = 14
    coords = W.disc_register(n, 14.0, 5.0, 5)
    base = W.ising_global_spec(coords, W.C6_LEVEL_60, amp, det, phase=0.4)
    rng = np.random.default_rng(n)
    specs = [W.noisy_trajectory_spec(base, coords, rng.normal(0, 1.5, n), max(0.0, rng.normal(1.0, 0.05)), 60.0)
             for _ in range(3)]
    tf = base.sampling_times[-1]
    with engine.DevicePlan(specs) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf, integrator=3)
        got = plan.get_state().copy()
        plan.set_state("all-ground")
        st2 = plan.propagate(0.0, tf, integrator=2, tol=1e-10)
        lan = plan.get_state().copy()
    assert st["integrator"] == 3 and st2["integrator"] == 2
    assert np.max(np.abs(got - lan)) < STATE_TOL
