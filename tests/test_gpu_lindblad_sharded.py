"""The master equation on state-vector shards (``lindblad.ShardedLindbladPlan``, ``stage_d2_taylor_kernel<..., SHARD,
..., DISS>``): vec(rho) split by its top row bits over 2, 4 and 8 shards (all on device 0 unless a test says otherwise)
against the unsharded ``LindbladPlan`` (same schedule, same rho), the exact piecewise-cubic Liouvillian evolution held to
the propagator's own bound, the density reductions, ``B200Backend`` with ``devices``, and the refusals."""
from __future__ import annotations

import numpy as np
import pytest

import open_ref as R
from helpers import curved_spec, open_spec
from pulser_b200 import HAVE_PULSER

pytestmark = pytest.mark.gpu

EIG = ["r", "g"]
SIGMA = {"x": np.array([[0, 1], [1, 0]], dtype=complex), "y": np.array([[0, -1j], [1j, 0]]),
         "z": np.array([[1, 0], [0, -1]], dtype=complex)}


def _ops(kind: str) -> np.ndarray:
    """Collapse operators of one qualifying channel: Pulser's dephasing + relaxation and depolarizing, and effective
    noise whose operators are each diagonal or each off-diagonal."""
    if kind == "dephasing+relaxation":
        return np.array([np.sqrt(2 * 1.5) * np.diag([1.0, 0.0]), R.relaxation(EIG, 2.0)], dtype=complex)
    if kind == "depolarizing":
        return np.array([np.sqrt(1.0 / 4) * SIGMA[a] for a in "xyz"])
    if kind == "eff-diagonal":
        return R.random_diag_ops(2, 2, 1.5, 4)
    if kind == "eff-offdiagonal":
        rng = np.random.default_rng(5)
        z = rng.normal(size=(2, 2)) + 1j * rng.normal(size=(2, 2))
        return np.array([[[0, z[i, 0]], [z[i, 1], 0]] for i in range(2)], dtype=complex)
    raise ValueError(kind)


def _spec(n: int, kind: str, T: int = 300):
    spec = curved_spec(n, T=T, phase=0.4)   # a curved drive of one constant phase
    spec.collapse_ops = _ops(kind)
    return spec


@pytest.fixture(scope="module")
def mods(lib):
    from pulser_b200 import engine, lindblad

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine, lindblad


def _same_schedule(a, b):
    assert a["n_steps"] == b["n_steps"] and a["n_applies"] == b["n_applies"]
    assert a["err_estimate"] == b["err_estimate"]
    assert a["integrator"] == b["integrator"] == 3


def _sum_stats(stats):
    out = {}
    for st in stats:
        for k, v in st.items():
            out[k] = max(out.get(k, 0), v) if k in ("max_rho", "integrator") else out.get(k, 0) + v
    return out


def _run(plan, rho0, times, **opts):
    """Shards run the Taylor propagator only; the unsharded plan is held to it too (integrator 3), where the automatic
    choice could take the Magnus path for a curved drive."""
    plan.set_state(rho0)
    stats = [plan.propagate(a, b, integrator=3, **opts) for a, b in zip(times[:-1], times[1:])]
    return plan.get_rho()[0], _sum_stats(stats)


# ---------------------------------------------------------------------------------------------------------------
# 1. against the unsharded plan: the same schedule, rho to 1e-11, whole runs and runs split into two calls
@pytest.mark.parametrize("kind", ["dephasing+relaxation", "depolarizing", "eff-diagonal", "eff-offdiagonal"])
@pytest.mark.parametrize("n,G", [(8, 2), (8, 4), (8, 8), (10, 2), (10, 4), (10, 8)])
def test_against_unsharded(mods, n, G, kind):
    _, lindblad = mods
    spec = _spec(n, kind)
    tf = spec.sampling_times[-1]
    rho0 = R.random_density(2**n, 3, n + G)
    for times in ([0.0, tf], [0.0, 0.37 * tf, tf]):
        with lindblad.LindbladPlan(spec) as lp:
            ref, st1 = _run(lp, rho0, times)
        with lindblad.ShardedLindbladPlan(spec, [0] * G) as sp:
            got, st = _run(sp, rho0, times)
        err = float(np.max(np.abs(got - ref)))
        print(f"\n[unsharded] N={n} G={G} {kind} calls={len(times) - 1}: max |d rho| = {err:.2e}, "
              f"steps {st['n_steps']}, applies {st['n_applies']}")
        _same_schedule(st, st1)
        assert err <= 1e-11


# ---------------------------------------------------------------------------------------------------------------
# 2. against the exact piecewise-cubic evolution under the sparse Liouvillian, held to the propagator's own bound
@pytest.mark.parametrize("n,G,window", [(7, 2, (0.05, 0.2)), (8, 4, (0.1213, 0.1218))])
def test_own_error_bound(mods, n, G, window):
    from test_gpu_taylor_lindblad import PiecewiseCubicLiouvillian

    _, lindblad = mods
    spec = _spec(n, "dephasing+relaxation")
    rho0 = R.random_density(2**n, 3, n)
    ref = PiecewiseCubicLiouvillian(spec).evolve(rho0.reshape(-1), *window).reshape(2**n, 2**n)
    with lindblad.ShardedLindbladPlan(spec, [0] * G) as sp:
        got, st = _run(sp, rho0, list(window), tol=1e-10)
    err = float(np.linalg.norm((got - ref).reshape(-1)))
    print(f"\n[bound] N={n} G={G} window={window}: |d| = {err:.2e}, err_estimate = {st['err_estimate']:.2e}")
    assert st["err_estimate"] <= 1e-10
    assert err <= 2.0 * st["err_estimate"] + 1e-14 * float(np.linalg.norm(rho0))


# ---------------------------------------------------------------------------------------------------------------
# 3. the density reductions of the shards against those of the unsharded plan
def _operators(n: int):
    from pulser_b200.opterms import OpTerms

    ops = [
        [(1.0, [({"rg": 1.0, "gr": 1.0}, {0})])],                      # flips atom 0: the top row bit, a shard bit
        [(0.5, [({"rr": 1.0}, {1}), ({"rg": 1.0j, "gr": -1.0j}, {n - 1})])],
        [(1.0, [({"rg": 1.0}, {0, 2})]), (0.3 - 0.2j, [({"gg": 1.0, "rr": -1.0}, {1, n - 2})])],
        [(1.0, [({"rr": -1.0, "gg": 1.0}, set(range(n)))])],          # parity: sign and care masks, no flip
    ]
    return [OpTerms.from_operations(o, EIG, n) for o in ops]


@pytest.mark.parametrize("n,G", [(8, 2), (8, 8), (10, 4)])
def test_reductions(mods, n, G):
    engine, lindblad = mods
    spec = _spec(n, "dephasing+relaxation")
    tf = spec.sampling_times[-1]
    rho0 = R.random_density(2**n, 4, 3 * n)
    phi = R.random_density(2**n, 1, 7)[:, 0]
    phi = phi / np.linalg.norm(phi)
    noiseless = curved_spec(n, T=300, phase=0.4)
    with lindblad.LindbladPlan(spec) as lp, lindblad.ShardedLindbladPlan(spec, [0] * G) as sp, \
            engine.DevicePlan(noiseless) as hplan:
        for p in (lp, sp):
            _run(p, rho0, [0.0, 0.6 * tf])

        def close(a, b, what):
            a, b = np.asarray(a), np.asarray(b)
            assert np.max(np.abs(a - b)) <= 1e-10 * max(1.0, float(np.max(np.abs(a)))), what

        close(lp.density_trace(), sp.density_trace(), "trace")
        for digit in (0, 1):
            close(lp.density_occupation(digit), sp.density_occupation(digit), "occupation")
            close(lp.density_correlation(digit), sp.density_correlation(digit), "correlation")
        for terms in _operators(n):
            close(lp.density_expect(terms), sp.density_expect(terms), "expect")
        for t_us in (0.2 * tf, 0.6 * tf):
            for a, b in zip(lp.density_energy(hplan, t_us), sp.density_energy(hplan, t_us)):
                close(a, b, "energy")
        close(lp.density_overlap(phi), sp.density_overlap(phi), "overlap")
        for one in ("r", "g"):
            np.random.seed(11)
            c1 = lp.density_sample(3000, one)
            np.random.seed(11)
            c2 = sp.density_sample(3000, one)
            assert c1 == c2, one


# ---------------------------------------------------------------------------------------------------------------
# 4. B200Backend with `devices` and a collapse-operator noise model, against the same run on one plan
def _pulser_sequence(n):
    """Linear ramps: splines smooth enough that the run on one plan takes the Taylor propagator too, as the shards do
    (a curved waveform at the master equation's 1e-10 tolerance may send it to the Magnus path)."""
    import pulser
    from pulser.waveforms import ConstantWaveform, RampWaveform
    from pulser_b200 import workloads as W

    reg = pulser.Register.from_coordinates(W.disc_register(n, 30.0, 7.0, n), prefix="q")
    seq = pulser.Sequence(reg, pulser.MockDevice)
    seq.declare_channel("ryd", "rydberg_global")
    om = 2 * np.pi * 1.5
    seq.add(pulser.Pulse(RampWaveform(100, 0.0, om), ConstantWaveform(100, -3 * om), 0.0), "ryd")
    seq.add(pulser.Pulse(ConstantWaveform(200, om), RampWaveform(200, -3 * om, om), 0.0), "ryd")
    seq.add(pulser.Pulse(RampWaveform(100, om, 0.0), ConstantWaveform(100, om), 0.0), "ryd")
    return seq


@pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable")
def test_backend_devices_master_equation(mods):
    from pulser.backend.default_observables import (
        BitStrings, CorrelationMatrix, Energy, EnergySecondMoment, EnergyVariance, Expectation, Fidelity, Occupation)
    from pulser.noise_model import NoiseModel
    from pulser_b200.backend import B200Backend, B200Config, B200Operator, B200State

    n = 9
    seq = _pulser_sequence(n)
    eig = ("r", "g")
    rng = np.random.default_rng(3)
    target = B200State(rng.normal(size=2**n) + 1j * rng.normal(size=2**n), eigenstates=eig)
    sx = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=n, operations=[
        (1.0, [({"rg": 1.0, "gr": 1.0}, {0})]), (0.5, [({"rr": 1.0}, {2, n - 1})])])
    times = [0.5, 1.0]
    noise = NoiseModel(dephasing_rate=0.8, relaxation_rate=0.3)

    def cfg(**kw):
        return B200Config(noise_model=noise, observables=[
            Occupation(evaluation_times=times), CorrelationMatrix(evaluation_times=times),
            Expectation(sx, evaluation_times=times), Energy(evaluation_times=times),
            EnergyVariance(evaluation_times=times), EnergySecondMoment(evaluation_times=times),
            Fidelity(target, evaluation_times=times), BitStrings(evaluation_times=[0.5, 1.0], num_shots=800)], **kw)

    res = {}
    for kind, kw in (("one", {}), ("shards", {"devices": [0, 0]})):
        np.random.seed(9)
        be = B200Backend(seq, config=cfg(**kw))
        res[kind] = be.run()
        calls = len(be._sim_obj._eval_times_array) - 1
        assert be._sim_obj.last_run_stats["integrator"] == 3 * calls, kind
    tags = res["one"].get_result_tags()
    assert tags == res["shards"].get_result_tags() and len(tags) == 8
    for tag in tags:
        for t in times:
            a, b = res["one"].get_result(tag, t), res["shards"].get_result(tag, t)
            if tag.startswith("bitstrings"):
                assert a == b and sum(a.values()) == 800, tag
            else:
                a, b = np.asarray(a, dtype=complex), np.asarray(b, dtype=complex)
                assert np.max(np.abs(a - b)) <= 1e-9 * max(1.0, float(np.max(np.abs(a)))), tag


# ---------------------------------------------------------------------------------------------------------------
# 5. refusals, with their reasons
def _refusal(lindblad, spec, G=2, exc=NotImplementedError) -> str:
    with pytest.raises(exc) as e:
        with lindblad.ShardedLindbladPlan(spec, [0] * G):
            pass
    return str(e.value)


def test_refusals(mods):
    _, lindblad = mods
    # single-bit-flip entries: a collapse operator mixing diagonal and off-diagonal elements
    spec = _spec(8, "dephasing+relaxation")
    spec.collapse_ops = np.array([[[0.5, 0.0], [1.0, 0.0]]], dtype=complex)
    assert "single-bit-flip entries" in _refusal(lindblad, spec)
    # a moving drive phase (open_spec's phases move in time)
    spec = open_spec(8, 2, T=40, interaction=False, ops=_ops("dephasing+relaxation"))
    spec.drives[0].coef[:] = spec.drives[0].coef[:1]
    assert "drive phase moves" in _refusal(lindblad, spec)
    # leakage: three levels
    spec = open_spec(8, 3, T=40, interaction=False, ops=R.random_diag_ops(3, 1, 2.0, 0))
    assert "d = 2" in _refusal(lindblad, spec)
    # XY
    spec = _spec(8, "dephasing+relaxation")
    spec.interaction_type = "XY"
    assert "XY" in _refusal(lindblad, spec)
    # stochastic noise: a batch of trajectories
    spec = _spec(8, "dephasing+relaxation")
    with pytest.raises(NotImplementedError, match="one trajectory"):
        lindblad.ShardedLindbladPlan([spec, spec], [0, 0])
    # a shard of fewer than 2^13 entries
    assert "2^13" in _refusal(lindblad, _spec(7, "dephasing+relaxation"), G=4, exc=ValueError)


@pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable")
def test_backend_refusals(mods):
    from pulser.noise_model import NoiseModel
    from pulser_b200.backend import B200Backend, B200Config

    seq = _pulser_sequence(9)
    cases = [
        (NoiseModel(temperature=50.0, runs=2, samples_per_run=1), "noiseless"),
        (NoiseModel(amp_sigma=0.1, runs=2, samples_per_run=1), "without stochastic noise"),
        (NoiseModel(eff_noise_opers=(np.diag([0.0, 0.0, 1.0]),), eff_noise_rates=(0.5,), with_leakage=True),
         "leakage"),
    ]
    for noise, needle in cases:
        with pytest.raises(NotImplementedError, match=needle):
            B200Backend(seq, config=B200Config(devices=[0, 0], noise_model=noise)).run()


# ---------------------------------------------------------------------------------------------------------------
# 6. two devices: peer loads across the shard bits, a Hamiltonian plan per device for the energy
def test_two_devices(mods):
    engine, lindblad = mods
    if engine.device_count() < 2:
        pytest.skip("needs 2 CUDA devices")
    spec = _spec(8, "dephasing+relaxation")
    tf = spec.sampling_times[-1]
    rho0 = R.random_density(2**8, 3, 2)
    with lindblad.LindbladPlan(spec) as lp:
        ref, st1 = _run(lp, rho0, [0.0, tf])
        with engine.DevicePlan(curved_spec(8, T=300, phase=0.4)) as hplan:
            e1 = lp.density_energy(hplan, 0.5 * tf)
            with lindblad.ShardedLindbladPlan(spec, [0, 1]) as sp:
                got, st = _run(sp, rho0, [0.0, tf])
                e2 = sp.density_energy(hplan, 0.5 * tf)
    _same_schedule(st, st1)
    assert np.max(np.abs(got - ref)) <= 1e-11
    for a, b in zip(e1, e2):
        assert abs(a[0] - b[0]) <= 1e-10 * max(1.0, abs(a[0]))
