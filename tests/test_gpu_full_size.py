"""BASELINE configurations at their configured sizes (VERDICT r01 items 3 and 6).

* ``pb200_apply_h`` against the matrix-free numpy oracle (``oracle/matfree.py``) on the production geometry of every
  configuration: C2 (N = 20, d = 2), C3 (N = 14, d = 3), C5 (N = 24, d = 2, 13 bits outside the tile);
* C5 end to end (reference call replaced: ``qutip.sesolve``, simulation.py:729-735): unit norm, Lanczos against
  Chebyshev, default controller against a 1000x tighter one;
* the C5 code path (auto rule -> Lanczos) at a size the DOP853 oracle can follow.
"""
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


@pytest.mark.parametrize("name", ["c2_n20", "c3_n14", "c5_n24"])
def test_apply_h_at_configured_size_vs_matrix_free_oracle(engine, name):
    from oracle.matfree import MatFreeHamiltonian

    spec = {"c2_n20": lambda: W.config_c2(n=20), "c3_n14": lambda: W.config_c3(n=14),
            "c5_n24": lambda: W.config_c5(n=24)}[name]()
    v = random_state(spec.hilbert_dim, 11)
    t = 0.4 * spec.sampling_times[-1] + 1.7e-4
    ref = MatFreeHamiltonian(spec).apply(t, v)
    with engine.DevicePlan(spec) as plan:
        got = plan.apply_h(t, v)
    assert np.max(np.abs(got - ref)) < 1e-12 * max(1.0, np.max(np.abs(ref)))


def test_c5_whole_sequence(engine):
    """configs[4]: 24 atoms, 4000 ns.  The Taylor run (what the auto rule picks for a global drive of constant phase),
    the Lanczos (Krylov) run, the Chebyshev run and a 1000x tighter Krylov run agree to the north-star 1e-8."""
    spec = W.config_c5(n=24)
    tf = spec.sampling_times[-1]
    outs = {}
    with engine.DevicePlan(spec) as plan:
        for key, kw in (("auto", {}), ("lanczos", {"integrator": 2}), ("cheb", {"integrator": 1}),
                        ("tight", {"integrator": 2, "tol": 1e-11})):
            plan.set_state("all-ground")
            st = plan.propagate(0.0, tf, **kw)
            assert abs(plan.norm2()[0] - 1.0) < 1e-9
            outs[key] = (plan.get_state()[0], st)
    assert outs["auto"][1]["integrator"] == 3          # global drive of constant phase: the time-dependent Taylor propagator
    assert outs["lanczos"][1]["integrator"] == 2 and outs["cheb"][1]["integrator"] == 1
    for key in ("lanczos", "cheb", "tight"):
        assert np.max(np.abs(outs["auto"][0] - outs[key][0])) < STATE_TOL, key
    assert outs["lanczos"][1]["n_applies"] < outs["cheb"][1]["n_applies"]
    assert outs["auto"][1]["n_applies"] < 0.5 * outs["lanczos"][1]["n_applies"]


def test_c5_lanczos_path_vs_oracle(engine):
    """The Magnus / Krylov path C5 takes when the Taylor propagator does not apply, at N = 10 against the DOP853
    oracle."""
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    spec = W.config_c5(n=10, t_total=800)
    psi0 = evolve.all_ground_state(spec)
    tf = spec.sampling_times[-1]
    ref = evolve.sesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf], rtol=1e-13, atol=1e-15)[-1]
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf, integrator=2)
        got = plan.get_state()[0]
    assert st["integrator"] == 2
    assert np.max(np.abs(got - ref)) < STATE_TOL


def test_c3_configured_size_self_convergence(engine):
    """configs[2] at N = 14 (3^14 amplitudes): both integrators and a 100x tighter controller agree to 1e-8 on a
    shortened sequence (the apply-level parity at this size is the test above)."""
    spec = W.config_c3(n=14, t_raman=60, t_ryd=120)
    tf = spec.sampling_times[-1]
    outs = []
    with engine.DevicePlan(spec) as plan:
        for kw in ({"integrator": 1}, {"integrator": 2}, {"tol": 1e-10}):
            plan.set_state("all-ground")
            plan.propagate(0.0, tf, **kw)
            assert abs(plan.norm2()[0] - 1.0) < 1e-9
            outs.append(plan.get_state()[0])
    assert np.max(np.abs(outs[0] - outs[1])) < STATE_TOL
    assert np.max(np.abs(outs[0] - outs[2])) < STATE_TOL


def test_c4_configured_size_batch(engine):
    """configs[3] at N = 16: a device batch of noise trajectories, the batched Taylor propagator (what integrator 0
    picks: per-qubit static amplitude factors and doppler offsets) against Lanczos and Chebyshev, unit norms, and the
    device-side shot + density reductions bench.py uses."""
    amp, det = W.blockade_sweep_waveforms(t_rise=60, t_sweep=160, t_fall=60)
    base = W.ising_global_spec(W.square_register(4, 6.0), W.C6_LEVEL_70, amp, det)
    rng = np.random.default_rng(3)
    coords = W.square_register(4, 6.0)
    specs = [W.noisy_trajectory_spec(base, coords, rng.normal(0, W.doppler_sigma(50.0), 16),
                                     max(0.0, rng.normal(1.0, 0.05)), 175.0) for _ in range(6)]
    tf = base.sampling_times[-1]
    outs = {}
    with engine.DevicePlan(specs) as plan:
        for integ in (1, 2, 0):
            plan.set_state("all-ground")
            st = plan.propagate(0.0, tf, integrator=integ)
            assert np.max(np.abs(plan.norm2() - 1.0)) < 1e-9
            outs[integ] = plan.get_state().copy()
        assert st["integrator"] == 3
        occ = plan.occupation(base.eigenbasis.index("r"))
        np.random.seed(0)
        shots = plan.sample(50, "r", traj=3)
    assert np.max(np.abs(outs[1] - outs[2])) < STATE_TOL
    assert np.max(np.abs(outs[0] - outs[2])) < STATE_TOL
    idx = np.arange(base.hilbert_dim)
    p = np.abs(outs[2][3]) ** 2
    ref_occ = np.array([p[((idx >> (15 - k)) & 1) == 0].sum() for k in range(16)])
    assert np.max(np.abs(occ[3] - ref_occ)) < 1e-10
    assert sum(shots.values()) == 50
