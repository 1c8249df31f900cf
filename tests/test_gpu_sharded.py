"""GPU tests of state-vector sharding (``ShardedPlan``, ``pb200_shards_*``): the state of one register split over
2, 4 or 8 plans -- here all on device 0, which runs the same kernels, streams and events as shards on distinct
devices -- against the unsharded plan and the oracles."""
from collections import Counter

import numpy as np
import pytest

from helpers import random_state
from pulser_b200 import HAVE_PULSER
from pulser_b200 import workloads as W

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


@pytest.fixture(scope="module")
def sharded(engine):
    from pulser_b200 import sharded

    return sharded


def _curved_spec(n, phase, T):
    """Blackman amplitude, sin^2 detuning: polynomial steps of degree up to 8 (history and G ring across shards)."""
    amp = W.blackman(T, 2.2 * np.pi)
    det = -8.0 + 20.0 * np.sin(np.linspace(0.0, 1.3, T)) ** 2
    coords = W.disc_register(n, 16.0, 5.0, 3)
    return W.ising_global_spec(coords, W.C6_LEVEL_60, amp, det, phase=phase)


@pytest.mark.parametrize("G", [2, 4])
@pytest.mark.parametrize("phase", [0.0, 0.83])
def test_apply_h_vs_matfree(sharded, G, phase):
    from oracle.matfree import MatFreeHamiltonian

    spec = _curved_spec(15, phase, T=200)
    v = random_state(spec.hilbert_dim, G)
    with sharded.ShardedPlan(spec, [0] * G) as plan:
        for t in (0.0371, 0.1234):
            got = plan.apply_h(t, v)
            ref = MatFreeHamiltonian(spec).apply(t, v)
            assert np.max(np.abs(got - ref)) <= 1e-12 * np.max(np.abs(ref))


def test_apply_h_c2_eight_shards(sharded):
    from oracle.matfree import MatFreeHamiltonian

    spec = W.config_c2(n=20)
    v = random_state(spec.hilbert_dim, 3)
    with sharded.ShardedPlan(spec, [0] * 8) as plan:
        got = plan.apply_h(1.7, v)
    ref = MatFreeHamiltonian(spec).apply(1.7, v)
    assert np.max(np.abs(got - ref)) <= 1e-12 * np.max(np.abs(ref))


@pytest.fixture(scope="module")
def c2_unsharded(engine):
    spec = W.config_c2(n=20)
    tf = spec.sampling_times[-1]
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf)
        psi = plan.get_state()[0]
    assert st["integrator"] == 3
    return spec, st, psi


def _same_schedule(a, b):
    assert a["n_steps"] == b["n_steps"] and a["n_applies"] == b["n_applies"]
    assert a["err_estimate"] == b["err_estimate"]


@pytest.mark.parametrize("G", [2, 4, 8])
def test_c2_whole_sequence(sharded, c2_unsharded, G):
    """Same host schedule (steps, orders, error estimate), same state up to the reordered partner sums."""
    spec, st1, psi1 = c2_unsharded
    with sharded.ShardedPlan(spec, [0] * G) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, spec.sampling_times[-1])
        psi = plan.get_state()[0]
    assert st["integrator"] == 3
    _same_schedule(st, st1)
    assert np.max(np.abs(psi - psi1)) <= 1e-9


@pytest.mark.parametrize("n,G,phase", [(14, 2, 0.0), (15, 4, -2.1)])
def test_curved_sequence_vs_oracle(sharded, n, G, phase):
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    spec = _curved_spec(n, phase, T=300)
    psi0 = random_state(spec.hilbert_dim, 11)
    tf = spec.sampling_times[-1]
    ref = evolve.sesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf], rtol=1e-13, atol=1e-15)[-1]
    with sharded.ShardedPlan(spec, [0] * G) as plan:
        plan.set_state(psi0)
        # two calls: the ring and the events carry over a call boundary
        plan.propagate(0.0, 0.4 * tf)
        st = plan.propagate(0.4 * tf, tf)
        got = plan.get_state()[0]
    assert st["integrator"] == 3
    assert np.max(np.abs(got - ref)) < 1e-8


def test_observables_vs_device_plan(engine, sharded):
    spec = W.config_c2(n=16, t_rise=100, t_sweep=400, t_fall=150)
    tf = spec.sampling_times[-1]
    phi = random_state(spec.hilbert_dim, 2)
    out = {}
    for kind in ("plan", "shards"):
        plan = engine.DevicePlan(spec) if kind == "plan" else sharded.ShardedPlan(spec, [0] * 4)
        with plan:
            plan.set_state("all-ground")
            plan.propagate(0.0, 0.6 * tf)
            r = {
                "norm2": plan.norm2(), "occ": plan.occupation(0), "corr": plan.correlation(0),
                "energy": np.array(plan.energy(0.6 * tf)), "overlap": plan.overlap(phi), "psi": plan.get_state()[0],
            }
            for one in ("r", "g"):
                np.random.seed(77)
                r["sample_" + one] = plan.sample(2000, one)
            out[kind] = r
    a, b = out["plan"], out["shards"]
    assert np.max(np.abs(a["psi"] - b["psi"])) < 1e-10
    for k in ("norm2", "occ", "corr", "energy", "overlap"):
        assert a[k].shape == b[k].shape, k
        assert np.max(np.abs(a[k] - b[k])) <= 1e-10 * max(1.0, np.max(np.abs(a[k]))), k
    for one in ("r", "g"):
        assert isinstance(b["sample_" + one], Counter)
        assert a["sample_" + one] == b["sample_" + one]


def test_refusals(engine, sharded):
    from pulser_b200._lib import PB200Error

    amp, det = W.blockade_sweep_waveforms(t_rise=60, t_sweep=150, t_fall=60)
    coords = W.disc_register(14, 14.0, 5.0, 5)
    base = W.ising_global_spec(coords, W.C6_LEVEL_60, amp, det)
    # per-qubit drive rows (doppler offsets, amplitude factors)
    per_qubit = W.noisy_trajectory_spec(base, coords, np.linspace(-1.0, 1.0, 14), 0.97, 60.0)
    with pytest.raises((NotImplementedError, PB200Error), match="per-qubit|global drive"):
        sharded.ShardedPlan(per_qubit, [0, 0])
    with pytest.raises(NotImplementedError, match="d = 2"):
        sharded.ShardedPlan(W.config_c3(n=14), [0, 0])
    with pytest.raises(ValueError, match="2\\^12"):
        sharded.ShardedPlan(W.config_c2(n=14), [0] * 4)
    with sharded.ShardedPlan(base, [0, 0]) as plan:
        plan.set_state("all-ground")
        with pytest.raises(PB200Error, match="Taylor propagator only"):
            plan.propagate(0.0, 0.1, integrator=1)
        with pytest.raises(PB200Error, match="shard 0 of 2"):
            plan.shards[0].propagate(0.0, 0.1)


def _pulser_sequence(n):
    import pulser
    from pulser.waveforms import BlackmanWaveform, RampWaveform

    coords = W.disc_register(n, 30.0, 5.0, n)
    reg = pulser.Register.from_coordinates(coords, prefix="q")
    seq = pulser.Sequence(reg, pulser.MockDevice)
    seq.declare_channel("ryd", "rydberg_global")
    seq.add(pulser.Pulse(BlackmanWaveform(400, 3 * np.pi), RampWaveform(400, -8.0, 6.0), 0.0), "ryd")
    return seq


@pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable")
def test_backend_devices_option(engine):
    from pulser.backend.default_observables import (
        BitStrings, CorrelationMatrix, Energy, EnergyVariance, Fidelity, Occupation)
    from pulser.noise_model import NoiseModel
    from pulser_b200.backend import B200Backend, B200Config, B200State

    n = 14
    seq = _pulser_sequence(n)
    eig = ("r", "g")
    target = B200State(random_state(1 << n, 4), eigenstates=eig)
    times = [0.5, 1.0]

    def cfg(**kw):
        return B200Config(observables=[
            Occupation(evaluation_times=times), CorrelationMatrix(evaluation_times=times),
            Energy(evaluation_times=times), EnergyVariance(evaluation_times=times),
            Fidelity(target, evaluation_times=times), BitStrings(evaluation_times=[1.0], num_shots=500)], **kw)

    res = {}
    for kind, kw in (("one", {}), ("shards", {"devices": [0, 0]})):
        np.random.seed(9)
        res[kind] = B200Backend(seq, config=cfg(**kw)).run()
    for t in times:
        for tag in ("occupation", "correlation_matrix", "energy", "energy_variance", "fidelity"):
            a = np.asarray(res["one"].get_result(tag, t), dtype=complex)
            b = np.asarray(res["shards"].get_result(tag, t), dtype=complex)
            # the unsharded run may take the Magnus path at the same 1e-8 state tolerance: agreement to that level,
            # scaled by |H| for the energies
            assert np.max(np.abs(a - b)) <= 1e-6 * max(1.0, float(np.max(np.abs(a)))), tag
    assert res["one"].final_bitstrings == res["shards"].final_bitstrings
    noisy = cfg(devices=[0, 0], noise_model=NoiseModel(temperature=50.0, runs=2, samples_per_run=1))
    with pytest.raises(NotImplementedError, match="noiseless"):
        B200Backend(seq, config=noisy).run()


def test_two_devices(engine, sharded, c2_unsharded):
    if engine.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    spec, st1, psi1 = c2_unsharded
    with sharded.ShardedPlan(spec, [0, 1]) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, spec.sampling_times[-1])
        psi = plan.get_state()[0]
    _same_schedule(st, st1)
    assert np.max(np.abs(psi - psi1)) <= 1e-9
