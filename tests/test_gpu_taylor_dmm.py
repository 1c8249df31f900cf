"""GPU tests of detuning maps on the Taylor propagator: a global drive with per-qubit detuning of up to four time shapes
(detuning map modulators, masks, doppler noise), on single plans (the uniform-gather kernel with local detuning),
trajectory batches and state-vector shards, against the DOP853 oracle, the Krylov path and the matrix-free oracle."""
import numpy as np
import pytest

from helpers import random_state
from pulser_b200 import HAVE_PULSER
from pulser_b200 import workloads as W

pytestmark = pytest.mark.gpu

STATE_TOL = 1e-8


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


def _oracle(spec, psi0, times):
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    return evolve.sesolve(OracleHamiltonian.from_spec(spec), psi0, times, rtol=1e-13, atol=1e-15)


def _waveforms(T):
    """negative DMM waveforms of different time shapes; the fifth only serves the refusal"""
    t = np.arange(T)
    return [
        -np.concatenate([np.linspace(0.0, 6.0, T // 2), np.full(T - T // 2, 6.0)]),
        -4.0 * np.sin(np.pi * t / T) ** 2,
        -np.where(t > 0.7 * T, 3.0, 0.0),            # an SLM-like step
        -2.0 * (1.0 + np.sin(7.0 * np.pi * t / T)),
        -1.5 * np.cos(3.0 * np.pi * t / T) ** 2,
    ]


def _dmm(n, n_maps, T=300, seed=3, scale=1.0, phase=0.0, first=0):
    amp, det = W.blockade_sweep_waveforms(t_rise=60, t_sweep=T - 120, t_fall=60)
    coords = W.disc_register(n, 14.0, 5.0, seed)
    base = W.ising_global_spec(coords, W.C6_LEVEL_60, amp, det, phase=phase)
    rng = np.random.default_rng(100 + n_maps)
    maps = [(scale * rng.uniform(0.2, 1.0, n) * (np.arange(n) % (s + 2) != 0), wf)
            for s, wf in enumerate(_waveforms(T)[first:first + n_maps])]
    return coords, base, W.detuning_map_spec(base, maps)


@pytest.mark.parametrize("n_maps", [1, 3])
@pytest.mark.parametrize("n", [6, 12, 13, 14])
def test_dmm_vs_oracle(engine, n, n_maps):
    """N < 13: the one-thread-per-amplitude stage; N >= 13: the tiled uniform-gather stage with local detuning"""
    from oracle import evolve

    _, _, spec = _dmm(n, n_maps)
    psi0 = evolve.all_ground_state(spec)
    tf = spec.sampling_times[-1]
    ref = _oracle(spec, psi0, [0.0, tf])[-1]
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf)
        got = plan.get_state()[0]
        plan.set_state("all-ground")
        st2 = plan.propagate(0.0, tf, integrator=2)
        lan = plan.get_state()[0]
    assert st["integrator"] == 3 and st2["integrator"] == 2
    assert np.max(np.abs(got - ref)) < STATE_TOL
    assert np.max(np.abs(got - lan)) < STATE_TOL
    assert st["err_estimate"] < 1e-8


@pytest.mark.parametrize("n", [5, 12, 14])
def test_noisy_dmm_batch_vs_oracle(engine, n):
    """DMM + doppler + amplitude noise (two to four shapes per batch): the batched Taylor stage with several shapes"""
    from oracle import evolve

    coords, _, spec = _dmm(n, 2, phase=0.4)
    rng = np.random.default_rng(n)
    specs = [W.noisy_trajectory_spec(spec, coords, rng.normal(0, 1.5, n), max(0.0, rng.normal(1.0, 0.05)), 60.0)
             for _ in range(3)]
    tf = spec.sampling_times[-1]
    psi0 = evolve.all_ground_state(spec)
    with engine.DevicePlan(specs) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf)
        got = plan.get_state().copy()
    assert st["integrator"] == 3
    for b, s in enumerate(specs):
        ref = _oracle(s, psi0, [0.0, tf])[-1]
        assert np.max(np.abs(got[b] - ref)) < STATE_TOL, b


@pytest.mark.parametrize("n,phase", [(13, 0.0), (14, 0.83)])
def test_single_plan_against_batch_kernel(engine, n, phase):
    """the uniform-gather stage with local detuning (one state) against the batched stage (the same spec twice); both
    converged far below the default tolerance, so that only the kernels' rounding separates them"""
    _, _, spec = _dmm(n, 1, phase=phase)
    tf = spec.sampling_times[-1]
    psi0 = random_state(spec.hilbert_dim, 9)
    with engine.DevicePlan(spec) as plan:
        plan.set_state(psi0)
        st1 = plan.propagate(0.0, tf, tol=1e-12)
        one = plan.get_state()[0]
    with engine.DevicePlan([spec, spec]) as plan:
        plan.set_state(np.stack([psi0, psi0]))
        st2 = plan.propagate(0.0, tf, tol=1e-12)
        two = plan.get_state()
    assert st1["integrator"] == 3 and st2["integrator"] == 3
    assert np.array_equal(two[0], two[1])
    assert np.max(np.abs(one - two[0])) < 1e-10
    # the single plan's per-excitation-number bound is at least as tight as the batch's per-trajectory bound
    assert st1["n_applies"] <= st2["n_applies"]


def test_weak_map_costs_what_the_plain_sequence_costs(engine):
    """with the per-excitation-number bound, a DMM of weights 1e-3 costs no more than 5 % over the plain sequence (a
    smooth map waveform: a kink the plain sequence does not have would cost steps of its own)"""
    _, base, spec = _dmm(12, 1, T=600, scale=1e-3, first=1)
    tf = spec.sampling_times[-1]
    applies = []
    for s in (base, spec):
        with engine.DevicePlan(s) as plan:
            plan.set_state("all-ground")
            st = plan.propagate(0.0, tf)
            assert st["integrator"] == 3
            applies.append(st["n_applies"])
    assert applies[1] <= 1.05 * applies[0], applies


def test_c2_dmm_against_magnus(engine):
    """N = 20, DMM on half the atoms: Taylor against the Richardson-CF4 path at tol = 1e-10"""
    spec = W.config_c2(n=20)
    T = spec.total_duration_ns
    w = np.where(np.arange(20) % 2 == 0, 1.0, 0.0)
    spec = W.detuning_map_spec(spec, [(w, _waveforms(T)[0])])
    tf = spec.sampling_times[-1]
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st3 = plan.propagate(0.0, tf)
        got = plan.get_state()[0]
        plan.set_state("all-ground")
        st1 = plan.propagate(0.0, tf, integrator=1, tol=1e-10)
        ref = plan.get_state()[0]
    assert st3["integrator"] == 3 and st1["integrator"] == 1
    assert np.max(np.abs(got - ref)) < STATE_TOL


def test_five_shapes_fall_back_or_raise(engine):
    _, _, spec = _dmm(8, 5)
    tf = spec.sampling_times[-1]
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf)
        assert st["integrator"] in (1, 2)
        with pytest.raises(Exception, match="Taylor.*more than 4 time shapes"):
            plan.propagate(0.0, tf, integrator=3)


@pytest.fixture(scope="module")
def sharded(engine):
    from pulser_b200 import sharded

    return sharded


@pytest.mark.parametrize("n_maps", [1, 2])
@pytest.mark.parametrize("G", [2, 4, 8])
def test_shards_vs_unsharded(engine, sharded, G, n_maps):
    """same host schedule as the unsharded plan, same state up to the reordered partner sums, same observables (the
    unsharded plan is held to Taylor: at 200 ns the sin^2 map is too curved for the auto rule, shards always take it)"""
    _, _, spec = _dmm(16, n_maps, T=200)
    tf = spec.sampling_times[-1]
    out = {}
    for kind in ("plan", "shards"):
        plan = engine.DevicePlan(spec) if kind == "plan" else sharded.ShardedPlan(spec, [0] * G)
        with plan:
            plan.set_state("all-ground")
            st = plan.propagate(0.0, tf, integrator=3)
            out[kind] = (st, plan.get_state()[0], plan.occupation(0), np.array(plan.energy(0.5 * tf)))
    (s1, p1, o1, e1), (s2, p2, o2, e2) = out["plan"], out["shards"]
    assert s1["integrator"] == 3 and s2["integrator"] == 3
    assert s1["n_steps"] == s2["n_steps"] and s1["n_applies"] == s2["n_applies"]
    assert s1["err_estimate"] == s2["err_estimate"]
    assert np.max(np.abs(p1 - p2)) < 1e-10
    assert np.max(np.abs(o1 - o2)) < 1e-10
    assert np.max(np.abs(e1 - e2)) <= 1e-10 * max(1.0, np.max(np.abs(e1)))


@pytest.mark.parametrize("n_maps,phase", [(1, 0.0), (2, 0.83)])
def test_shards_apply_h_vs_matfree(sharded, n_maps, phase):
    from oracle.matfree import MatFreeHamiltonian

    _, _, spec = _dmm(15, n_maps, T=200, phase=phase)
    v = random_state(spec.hilbert_dim, 4)
    with sharded.ShardedPlan(spec, [0] * 4) as plan:
        for t in (0.0371, 0.1234):
            got = plan.apply_h(t, v)
            ref = MatFreeHamiltonian(spec).apply(t, v)
            assert np.max(np.abs(got - ref)) <= 1e-12 * np.max(np.abs(ref))


@pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable")
def test_pulser_sequence_with_dmm(engine):
    """a real Sequence with a detuning map (MockDevice: a virtual device with a DMM channel) runs through B200Backend,
    on one plan and on two shards of device 0: the same occupations and bitstrings"""
    import pulser
    from pulser.backend.default_observables import BitStrings, Occupation
    from pulser.waveforms import BlackmanWaveform, RampWaveform

    from pulser_b200.backend import B200Backend, B200Config

    n = 14
    coords = W.disc_register(n, 30.0, 5.0, n)
    reg = pulser.Register.from_coordinates(coords, prefix="q")
    seq = pulser.Sequence(reg, pulser.MockDevice)
    seq.declare_channel("ryd", "rydberg_global")
    dmap = reg.define_detuning_map({f"q{i}": (1.0 if i % 2 else 0.4) for i in range(n)})
    seq.config_detuning_map(dmap, "dmm_0")
    seq.add(pulser.Pulse(BlackmanWaveform(400, 3 * np.pi), RampWaveform(400, -8.0, 6.0), 0.0), "ryd")
    seq.add_dmm_detuning(RampWaveform(400, 0.0, -5.0), "dmm_0")
    times = [0.5, 1.0]

    def cfg(**kw):
        return B200Config(observables=[Occupation(evaluation_times=times),
                                       BitStrings(evaluation_times=[1.0], num_shots=500)], **kw)

    res = {}
    for kind, kw in (("one", {}), ("shards", {"devices": [0, 0]})):
        np.random.seed(9)
        res[kind] = B200Backend(seq, config=cfg(**kw)).run()
    for t in times:
        a = np.asarray(res["one"].get_result("occupation", t), dtype=float)
        b = np.asarray(res["shards"].get_result("occupation", t), dtype=float)
        assert np.max(np.abs(a - b)) <= 1e-6
    assert res["one"].final_bitstrings == res["shards"].final_bitstrings
