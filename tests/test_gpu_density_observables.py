"""The density-matrix reductions (``pb200_density_*``) against dense numpy, and ``B200Backend``'s streamed master
equation (``DeviceDensityView``) against the replay of the density matrices ``B200Emulator.run`` stores."""
from __future__ import annotations

import copy
import warnings

import numpy as np
import pytest

from density_ref import number_masks, terms_matrix
from helpers import curved_spec, open_spec, with_dmm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def mods(lib):
    from pulser_b200 import engine, lindblad

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine, lindblad


def _dephasing(d: int) -> np.ndarray:
    return np.array([np.sqrt(2.0) * np.diag([1.0] + [0.0] * (d - 1))], dtype=complex)


def _noiseless(spec):
    s = copy.copy(spec)
    s.collapse_ops = np.zeros((0, spec.dim, spec.dim), dtype=complex)
    return s


def _random_rhos(D: int, count: int, seed: int) -> np.ndarray:
    rng = np.random.default_rng(seed)
    out = []
    for b in range(count):
        a = rng.normal(size=(D, D)) + 1j * rng.normal(size=(D, D))
        rho = a @ a.conj().T
        out.append(rho * (0.5 + b) / np.trace(rho).real)  # traces 0.5, 1.5, 2.5
    return np.stack(out)


def _operators(n: int, eig: list[str]):
    from pulser_b200.opterms import OpTerms

    a, b = eig[0], eig[1]
    ops = {
        "sum_sx": [(1.0, [({a + b: 1.0, b + a: 1.0}, {k})]) for k in range(n)],
        "sp_sm_pair": [(0.7, [({a + b: 1.0}, {0}), ({b + a: 1.0}, {n - 1})])],
        "parity": [(1.0, [({a + a: -1.0, b + b: 1.0}, set(range(n)))])],
        "sp0": [(1.0, [({a + b: 1.0}, {0})])],
    }
    return {k: OpTerms.from_operations(v, eig, n) for k, v in ops.items()}


def _close(got, ref, scale, rtol=1e-12):
    assert np.all(np.abs(np.asarray(got) - np.asarray(ref)) <= rtol * scale), (got, ref)


def _check_plan(mods, spec, seed=0):
    """Every export on a batch of 3 random density matrices against the dense formulas."""
    from oracle.ref_hamiltonian import OracleHamiltonian

    engine, lindblad = mods
    n, d, eig = spec.n_qudits, spec.dim, list(spec.eigenbasis)
    D = d**n
    rhos = _random_rhos(D, 3, seed)
    with lindblad.LindbladPlan([spec] * 3) as lp, engine.DevicePlan(_noiseless(spec)) as hp:
        lp.plan.set_state(rhos.reshape(3, -1))
        traces = np.trace(rhos, axis1=1, axis2=2).real
        _close(lp.density_trace(), traces, traces)
        diag = np.diagonal(rhos, axis1=1, axis2=2).real
        for digit in range(d):
            m = number_masks(n, d, digit)
            corr = np.einsum("ir,jr,br->bij", m, m, diag)
            _close(lp.density_occupation(digit), np.einsum("ir,br->bi", m, diag), traces[:, None])
            _close(lp.density_correlation(digit), corr, traces[:, None, None])
            _close(lp.density_occupation(digit, 1, 2), np.einsum("ir,br->bi", m, diag)[1:], traces[1:, None])
        for name, terms in _operators(n, eig).items():
            O = terms_matrix(terms)
            ref = np.einsum("rs,bsr->b", O, rhos)
            scale = np.einsum("rs,bsr->b", np.abs(O), np.abs(rhos))
            _close(lp.density_expect(terms), ref, scale)
        phi = np.random.default_rng(seed + 1).normal(size=D) + 1j * np.random.default_rng(seed + 2).normal(size=D)
        ref = np.einsum("r,brc,c->b", phi.conj(), rhos, phi)
        _close(lp.density_overlap(phi), ref, np.einsum("r,brc,c->b", np.abs(phi), np.abs(rhos), np.abs(phi)))
        ham = OracleHamiltonian.from_spec(_noiseless(spec))
        for t in (0.3 * spec.sampling_times[-1], 0.77 * spec.sampling_times[-1]):
            H = ham.matrix_at(t).toarray()
            e, e2 = lp.density_energy(hp, t)
            _close(e, np.einsum("rs,bsr->b", H, rhos).real, np.einsum("rs,bsr->b", np.abs(H), np.abs(rhos)))
            H2 = H @ H
            _close(e2, np.einsum("rs,bsr->b", H2, rhos).real,
                   np.einsum("rs,bsr->b", np.abs(H) @ np.abs(H), np.abs(rhos)))


@pytest.mark.parametrize("n", [2, 3, 4, 5, 6, 7])
def test_exports_match_numpy_qubits(mods, n):
    _check_plan(mods, open_spec(n, 2, T=30, seed=n, ops=_dephasing(2)), seed=n)


@pytest.mark.parametrize("n", [2, 3, 4, 5])
def test_exports_match_numpy_leakage_basis(mods, n):
    _check_plan(mods, open_spec(n, 3, T=30, seed=n, ops=_dephasing(3)), seed=10 + n)


def test_exports_match_numpy_detuning_maps(mods):
    spec = with_dmm(curved_spec(5, T=120), 2, seed=1)
    spec.collapse_ops = _dephasing(2)
    _check_plan(mods, spec, seed=7)


def test_refusals(mods):
    import pulser_b200.workloads as W
    from pulser_b200._lib import PB200Error

    engine, lindblad = mods
    spec = open_spec(3, 2, T=20, ops=_dephasing(2))
    with engine.DevicePlan(_noiseless(spec)) as plan:
        plan.set_state("all-ground")
        fake = lindblad.LindbladPlan.__new__(lindblad.LindbladPlan)  # the reductions on a state-vector plan
        fake.plan, fake.n, fake.D, fake.specs = plan, 3, 8, [spec]
        for call in (lambda: fake.density_trace(), lambda: fake.density_occupation(0),
                     lambda: fake.density_correlation(0), lambda: fake.density_overlap(np.ones(8)),
                     lambda: fake.density_expect(_operators(3, ["r", "g"])["sp0"]),
                     lambda: fake.density_energy(plan, 0.01), lambda: fake.density_sample(10, "r")):
            with pytest.raises(PB200Error, match="no dissipator") as e:
                call()
            assert e.value.code == -3
    xy = W.config_xy(n=3, t_total=40)
    xy.collapse_ops = _dephasing(2)
    with lindblad.LindbladPlan(xy) as lp, engine.DevicePlan(_noiseless(xy)) as hp:
        lp.set_state(np.eye(8)[0])
        with pytest.raises(PB200Error, match="XY") as e:
            lp.density_energy(hp, 0.01)
        assert e.value.code == -3


def test_sampling_draws_n_uniforms_and_follows_the_diagonal(mods):
    engine, lindblad = mods
    n, shots = 4, 20000
    spec = open_spec(n, 2, T=20, ops=_dephasing(2))
    rho = _random_rhos(16, 1, 3)[0] * 3.0
    with lindblad.LindbladPlan(spec) as lp:
        lp.set_state(rho)
        np.random.seed(9)
        counts = lp.density_sample(shots, "r")
        after = np.random.rand()
    np.random.seed(9)
    np.random.rand(shots)
    assert after == np.random.rand()
    assert sum(counts.values()) == shots
    p = np.diagonal(rho).real / np.trace(rho).real
    is_r = number_masks(n, 2, 0)
    for r in range(16):
        key = "".join("1" if is_r[k, r] else "0" for k in range(n))
        sigma = np.sqrt(shots * p[r] * (1 - p[r]))
        assert abs(counts.get(key, 0) - shots * p[r]) <= 5 * sigma + 1, key


# ---- B200Backend: streamed against the replay of stored density matrices ---------------------------------------------
def _sweep(n: int = 6, duration: int = 400):
    import pulser
    from pulser.waveforms import BlackmanWaveform, RampWaveform

    radius = 6.0 * n / (2 * np.pi)  # neighbours 6 um apart on a ring
    reg = pulser.Register.from_coordinates([(radius * np.cos(2 * np.pi * k / n), radius * np.sin(2 * np.pi * k / n))
                                            for k in range(n)], prefix="q")
    seq = pulser.Sequence(reg, pulser.MockDevice)
    seq.declare_channel("ryd", "rydberg_global")
    seq.add(pulser.Pulse(BlackmanWaveform(duration, 2.5 * np.pi), RampWaveform(duration, -8.0, 6.0), 0.3), "ryd")
    return seq


def _backend_observables(n: int, eig: tuple, times: list):
    from pulser.backend.default_observables import (
        BitStrings, CorrelationMatrix, Energy, EnergySecondMoment, EnergyVariance, Expectation, Fidelity,
        Occupation, StateResult)
    from pulser_b200.backend import B200Operator, B200State

    a, b = eig[0], eig[1]
    target = B200State.from_state_amplitudes(eigenstates=eig, amplitudes={a + b * (n - 1): 1.0, b * n: 0.5j})
    sx = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=n, operations=[
        (1.0, [({a + b: 1.0, b + a: 1.0}, {k})]) for k in range(n)])
    sp0 = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=n, operations=[(1.0, [({a + b: 1.0}, {0})])])
    return [Occupation(evaluation_times=times), CorrelationMatrix(evaluation_times=times),
            Energy(evaluation_times=times), EnergyVariance(evaluation_times=times),
            EnergySecondMoment(evaluation_times=times), Fidelity(target, evaluation_times=times),
            Expectation(sx, evaluation_times=times, tag_suffix="sx"),
            Expectation(sp0, evaluation_times=times, tag_suffix="sp0"),
            StateResult(evaluation_times=times), BitStrings(evaluation_times=[1.0], num_shots=4000)]


TAGS = ("occupation", "correlation_matrix", "energy", "energy_variance", "energy_second_moment", "fidelity",
        "expectation_sx", "expectation_sp0")


def _compare_backend(seq, noise, eig, n_trajectories=None):
    import pulser
    from pulser_b200 import B200Backend, B200Config

    times = [0.2, 0.4, 0.6, 0.8, 1.0]
    out = {}
    for stream in (True, False):
        np.random.seed(21)
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            cfg = B200Config(observables=_backend_observables(len(seq.register.qubits), eig, times),
                             noise_model=pulser.NoiseModel(**noise), n_trajectories=n_trajectories)
            be = B200Backend(seq, config=cfg)
            assert be._streams_density()
            if not stream:
                be._streams_density = lambda: False  # the replay of the density matrices B200Emulator.run stores
            out[stream] = be.run()
    a, b = out[True], out[False]
    assert set(a.get_result_tags()) == set(b.get_result_tags())
    for tag in TAGS:
        if tag not in a.get_result_tags():  # not averaged over trajectories by Results.aggregate
            continue
        # the evaluation times as stored (t_us / duration, within pulser's time tolerance of the requested ones)
        stored = a.get_result_times(tag)
        assert stored == b.get_result_times(tag) and len(stored) == len(times)
        for t in stored:
            x, y = np.asarray(a.get_result(tag, t), dtype=complex), np.asarray(b.get_result(tag, t), dtype=complex)
            assert np.max(np.abs(x - y)) <= 1e-10 * max(1.0, np.max(np.abs(y))), (tag, t, x, y)
    for t in a.get_result_times("state"):
        np.testing.assert_allclose(a.get_result("state", t).to_array(), b.get_result("state", t).to_array(), atol=1e-10)
    fa, fb = a.final_bitstrings, b.final_bitstrings
    shots = sum(fb.values())
    assert sum(fa.values()) == shots
    for key in set(fa) | set(fb):  # two samples of one distribution
        pa, pb = fa.get(key, 0) / shots, fb.get(key, 0) / shots
        p = 0.5 * (pa + pb)
        assert abs(pa - pb) <= 5 * np.sqrt(2 * p * (1 - p) / shots) + 2 / shots, key


def test_backend_streams_like_the_replay(mods):
    _compare_backend(_sweep(), {"dephasing_rate": 0.5, "relaxation_rate": 0.3}, ("r", "g"))


def test_backend_streams_like_the_replay_with_leakage(mods):
    leak = np.zeros((3, 3)); leak[2, 0] = 1.0  # |x><r|
    noise = {"eff_noise_opers": (leak,), "eff_noise_rates": (0.3,), "with_leakage": True}
    _compare_backend(_sweep(5, 300), noise, ("r", "g", "x"))


def test_backend_trajectory_batch_aggregates_like_the_replay(mods):
    noise = {"temperature": 50.0, "dephasing_rate": 0.5}
    _compare_backend(_sweep(5, 300), noise, ("r", "g"), n_trajectories=4)


def test_no_density_matrix_travels_to_the_host(mods, monkeypatch):
    import pulser
    from pulser.backend.default_observables import Occupation
    from pulser_b200 import B200Backend, B200Config

    _, lindblad = mods
    calls = []
    orig = lindblad.LindbladPlan.get_rho
    monkeypatch.setattr(lindblad.LindbladPlan, "get_rho", lambda self: (calls.append(1), orig(self))[1])
    times = list(np.linspace(0.0, 1.0, 101))
    cfg = B200Config(observables=[Occupation(evaluation_times=times)],
                     noise_model=pulser.NoiseModel(dephasing_rate=0.5, relaxation_rate=0.3))
    res = B200Backend(_sweep(11, 300), config=cfg).run()
    assert calls == []
    occ = np.asarray(res.get_result("occupation", 1.0), dtype=float)
    assert occ.shape == (11,) and np.all((occ > 0) & (occ < 1))
