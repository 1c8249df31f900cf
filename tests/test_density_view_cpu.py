"""CPU tests of the streamed master-equation path of ``B200Backend``: a numpy stand-in for ``LindbladPlan`` that
provides the density reductions (``density_*``) decides the routing, and the observables it feeds through
``DeviceDensityView`` must equal the replay of the stored density matrices."""
import copy
import types
import warnings

import numpy as np
import pytest

from pulser_b200 import HAVE_PULSER

pytestmark = pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable here")

from density_ref import number_masks, terms_matrix  # noqa: E402
from fake_device import FakeDevicePlan, FakeLindbladPlan  # noqa: E402


class NumpyDensityPlan(FakeLindbladPlan):
    """The oracle-backed master equation with the device reductions restated in numpy.  The density matrices carry a
    trace of ``SCALE``, so every value the view reports must have been divided by the trace."""

    SCALE = 2.5
    get_rho_calls = 0

    def set_state(self, psi):
        super().set_state(psi)
        self.states = [self.SCALE * s for s in self.states]

    def get_rho(self):
        NumpyDensityPlan.get_rho_calls += 1
        return super().get_rho()

    def _rhos(self, traj0, count):
        return self.states[traj0: len(self.states) if count is None else traj0 + count]

    def density_trace(self, traj0=0, count=None):
        return np.array([np.trace(r).real for r in self._rhos(traj0, count)])

    def density_correlation(self, digit, traj0=0, count=None):
        m = number_masks(self.n, self.specs[0].dim, digit)
        return np.stack([[[np.diagonal(r).real[m[i] & m[j]].sum() for j in range(self.n)] for i in range(self.n)]
                         for r in self._rhos(traj0, count)])

    def density_occupation(self, digit, traj0=0, count=None):
        return np.stack([np.diagonal(c) for c in self.density_correlation(digit, traj0, count)])

    def density_expect(self, terms, traj0=0, count=None):
        return np.array([np.trace(terms_matrix(terms) @ r) for r in self._rhos(traj0, count)])

    def density_energy(self, ham_plan, t_us, traj0=0, count=None):
        h = ham_plan.hams[0].matrix_at(t_us, ham_plan.order)
        rhos = self._rhos(traj0, count)
        return (np.array([np.trace(h @ r).real for r in rhos]), np.array([np.trace(h @ h @ r).real for r in rhos]))

    def density_overlap(self, phi, traj0=0, count=None):
        return np.array([np.vdot(phi, r @ phi) for r in self._rhos(traj0, count)])

    def density_sample(self, n_samples, one_state, traj=0):
        from pulser_b200.backend import B200State

        r = self.states[traj]
        return B200State(r / np.trace(r).real, eigenstates=self.specs[0].eigenbasis).sample(
            num_shots=n_samples, one_state=one_state)


@pytest.fixture
def modules(monkeypatch):
    from pulser_b200 import backend, engine, lindblad

    monkeypatch.setattr(engine, "DevicePlan", FakeDevicePlan)
    NumpyDensityPlan.get_rho_calls = 0
    return types.SimpleNamespace(backend=backend, lindblad=lindblad, monkeypatch=monkeypatch)


def _seq(n=3, duration=200):
    from pulser import Pulse, Register, Sequence
    from pulser.devices import MockDevice
    from pulser.waveforms import BlackmanWaveform

    reg = Register.from_coordinates([(7.0 * i, 0.0) for i in range(n)], prefix="q")
    seq = Sequence(reg, MockDevice)
    seq.declare_channel("ch", "rydberg_global")
    seq.add(Pulse.ConstantDetuning(BlackmanWaveform(duration, np.pi), -1.0, 0.3), "ch")
    return seq


def _observables(times):
    from pulser.backend.default_observables import (
        BitStrings, CorrelationMatrix, Energy, EnergySecondMoment, EnergyVariance, Expectation, Fidelity,
        Occupation, StateResult)
    from pulser_b200.backend import B200Operator, B200State

    eig = ("r", "g")
    target = B200State.from_state_amplitudes(eigenstates=eig, amplitudes={"rgg": 1.0, "grg": 1.0j})
    sx = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=3, operations=[
        (1.0, [({"rg": 1.0, "gr": 1.0}, {k})]) for k in range(3)])
    sp0 = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=3, operations=[(1.0, [({"rg": 1.0}, {0})])])
    return [Occupation(evaluation_times=times), CorrelationMatrix(evaluation_times=times),
            Energy(evaluation_times=times), EnergyVariance(evaluation_times=times),
            EnergySecondMoment(evaluation_times=times), Fidelity(target, evaluation_times=times),
            Expectation(sx, evaluation_times=times, tag_suffix="sx"),
            Expectation(sp0, evaluation_times=times, tag_suffix="sp0"),
            StateResult(evaluation_times=times), BitStrings(evaluation_times=[1.0], num_shots=40)]


def _run(m, plan_cls, noise, n_trajectories=None, times=(0.5, 1.0)):
    import pulser

    m.monkeypatch.setattr(m.lindblad, "LindbladPlan", plan_cls)
    np.random.seed(3)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        cfg = m.backend.B200Config(observables=_observables(list(times)), noise_model=pulser.NoiseModel(**noise),
                                   n_trajectories=n_trajectories)
        be = m.backend.B200Backend(_seq(), config=cfg)
        return be, be.run()


def _assert_same(a, b, times=(0.5, 1.0)):
    assert set(a.get_result_tags()) == set(b.get_result_tags())
    for tag in ("occupation", "correlation_matrix", "energy", "energy_variance", "energy_second_moment", "fidelity",
                "expectation_sx", "expectation_sp0"):
        if tag not in a.get_result_tags():  # Results.aggregate skips what it cannot average
            continue
        for t in times:
            np.testing.assert_allclose(np.asarray(a.get_result(tag, t), dtype=complex),
                                       np.asarray(b.get_result(tag, t), dtype=complex), atol=1e-8, err_msg=f"{tag} {t}")
    for t in times:
        np.testing.assert_allclose(a.get_result("state", t).to_array(), b.get_result("state", t).to_array(), atol=1e-8)
    assert sum(a.final_bitstrings.values()) == sum(b.final_bitstrings.values())


def test_master_equation_streams_when_the_plan_reduces_on_the_device(modules):
    """With the density reductions the run never downloads a density matrix for the observables (StateResult's
    deepcopy is the one host copy) and gives what the replay of stored matrices gives, normalised by the trace."""
    noise = {"dephasing_rate": 0.8, "relaxation_rate": 0.5}
    be, streamed = _run(modules, NumpyDensityPlan, noise)
    assert be._streams_density()
    assert NumpyDensityPlan.get_rho_calls == 2  # the two StateResult copies
    assert be._sim_obj.last_run_stats["n_steps"] == 2
    be, replayed = _run(modules, FakeLindbladPlan, noise)
    assert not be._streams_density()
    _assert_same(streamed, replayed)
    assert streamed.get_result("state", 1.0).to_array().trace() == pytest.approx(1.0)


def test_xy_registers_and_plain_fakes_keep_the_replay(modules):
    be, _ = _run(modules, NumpyDensityPlan, {"dephasing_rate": 0.8}, times=(1.0,))
    assert be._streams_density()
    hd = be._sim_obj._hamiltonian_data
    xy = types.SimpleNamespace(lindblad_data=hd.lindblad_data, n_qudits=hd.n_qudits,
                               basis_data=types.SimpleNamespace(interaction_type="XY", dim=hd.basis_data.dim))
    modules.monkeypatch.setattr(be._sim_obj, "_hamiltonian_data", xy)
    assert not be._streams_density()
    modules.monkeypatch.setattr(modules.lindblad, "LindbladPlan", FakeLindbladPlan)
    be, _ = _run(modules, FakeLindbladPlan, {"dephasing_rate": 0.8}, times=(1.0,))
    assert not be._streams_density()


def test_deepcopy_of_a_view_is_a_host_state(modules):
    from pulser_b200.backend import B200State, DeviceDensityView

    sim = modules.backend.B200Emulator.from_sequence(_seq())
    plan = NumpyDensityPlan([sim._noiseless_spec()])
    plan.set_state(sim._initial_state.full().reshape(-1))
    plan.propagate(0.0, 0.1)
    view = DeviceDensityView(plan, eigenstates=("r", "g"))
    assert not view.is_ket and view.n_qudits == 3
    stored = copy.deepcopy(view)
    assert type(stored) is B200State
    rho = plan.get_rho()[0] / NumpyDensityPlan.SCALE
    np.testing.assert_allclose(stored.to_array(), rho, atol=1e-14)
    plan.propagate(0.1, 0.2)
    np.testing.assert_allclose(stored.to_array(), rho, atol=1e-14)


def test_trajectories_aggregate_like_the_replay(modules):
    """Stochastic noise on top of the master equation: one Results per trajectory repetition, aggregated with the
    density-matrix aggregator for StateResult."""
    noise = {"dephasing_rate": 0.8, "amp_sigma": 0.1, "temperature": 50.0, "laser_waist": 175.0}
    _, streamed = _run(modules, NumpyDensityPlan, noise, n_trajectories=3)
    assert NumpyDensityPlan.get_rho_calls == 2 * 3
    _, replayed = _run(modules, FakeLindbladPlan, noise, n_trajectories=3)
    _assert_same(streamed, replayed)
