"""CPU side of global drives whose phase moves: the exact reference of tests/taylor_ref.py on phase-jump and phase-ramp
inputs against DOP853 (the GPU tests rest on it), Pulser sequences with phase changes reach one global drive row whose
phase moves, and ShardedPlan's checks accept them before any device call."""
import numpy as np
import pytest

from helpers import curved_spec, random_state, with_dmm
from phase_sequences import KINDS, moving_phase_rows, phase_sequence
from pulser_b200 import HAVE_PULSER
from pulser_b200 import workloads as W
from taylor_ref import PiecewiseCubicHamiltonian


def _jump(n, T=160, at=80):
    amp, det = W.blockade_sweep_waveforms(t_rise=40, t_sweep=T - 80, t_fall=40)
    ph = np.where(np.arange(len(amp)) < at, 0.0, np.pi / 2)
    return W.ising_global_spec(W.disc_register(n, 14.0, 6.0, n), W.C6_LEVEL_60, amp, det, phase=ph)


def _specs(n):
    ramp = curved_spec(n, T=160, phase=0.2 + 1.5 * np.arange(160) / 160)
    coords = W.disc_register(n, 14.0, 6.0, n)
    return {
        "jump": _jump(n),
        "ramp": ramp,
        "jump_dmm2": with_dmm(_jump(n), 2, seed=4),
        "jump_noisy": W.noisy_trajectory_spec(_jump(n), coords, np.linspace(-1.0, 1.0, n), 0.97, 60.0),
    }


@pytest.mark.parametrize("name", ["jump", "ramp", "jump_dmm2", "jump_noisy"])
def test_reference_against_dop853(name):
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    spec = _specs(6)[name]
    ref = PiecewiseCubicHamiltonian(spec)
    psi = random_state(spec.hilbert_dim, 7)
    a, b = 0.0123, spec.sampling_times[-1] - 0.0077
    got = ref.evolve(psi, a, b)
    cuts = [a] + [t for t in spec.sampling_times if a < t < b] + [b]
    want = evolve.sesolve(OracleHamiltonian.from_spec(spec), psi, cuts, rtol=1e-13, atol=1e-15)[-1]
    assert np.linalg.norm(got - want) <= 1e-11
    assert np.linalg.norm(got - ref.evolve(psi, a, b, split=2)) <= 1e-14


@pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable here")
@pytest.mark.parametrize("kind", KINDS)
def test_pulser_sequences_reach_moving_phase(kind):
    from pulser_b200 import sharded
    from pulser_b200.emulator import B200Emulator

    spec = B200Emulator.from_sequence(phase_sequence(kind))._current_spec
    assert moving_phase_rows(spec)
    with pytest.raises(Exception) as e:
        sharded.ShardedPlan(spec, [63, 63])
    assert not isinstance(e.value, NotImplementedError)


@pytest.mark.parametrize("name", ["jump", "ramp", "jump_dmm2"])
def test_sharded_plan_validation(name):
    """a moving phase passes the Python checks of ShardedPlan (it fails only on creating the plans: no device here or
    no such device); per-qubit drive rows are still refused before any device call"""
    from pulser_b200 import sharded

    spec = _specs(14)[name]
    assert moving_phase_rows(spec)
    with pytest.raises(Exception) as e:
        sharded.ShardedPlan(spec, [63, 63])
    assert not isinstance(e.value, NotImplementedError)
    with pytest.raises(NotImplementedError, match="per-qubit"):
        sharded.ShardedPlan(_specs(14)["jump_noisy"], [63, 63])
