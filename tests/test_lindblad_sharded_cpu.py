"""CPU tests of the master equation on state-vector shards: which noise models ``B200Backend`` sends with ``devices`` to
the sharded density matrix (``lindblad.ShardedLindbladPlan``, here a numpy stand-in) and which it refuses, with what
message; and the shot routing of ``ShardedLindbladPlan.density_sample`` over the diagonal blocks of rho."""
import numpy as np
import pytest

from pulser_b200 import HAVE_PULSER


def _device_search(cum: np.ndarray, u: np.ndarray) -> np.ndarray:
    """search_sorted_kernel: first j with cum[j] >= u * cum[-1]"""
    return np.minimum(np.searchsorted(cum, u * cum[-1], side="left"), len(cum) - 1)


@pytest.mark.parametrize("n,G,one_digit", [(5, 2, 0), (5, 4, 1), (6, 8, 0), (6, 2, 1)])
def test_shot_routing_over_row_blocks(n, G, one_digit):
    """Shard i holds the rows [i D / G, (i + 1) D / G) of rho: routing each shot by the shards' partial traces, then
    searching the diagonal of the shard's block, picks the bitstring the search over the whole diagonal picks."""
    from pulser_b200.sharded import global_bitstring, route_shots

    rng = np.random.default_rng(n * 10 + G + one_digit)
    D, bits = 1 << n, G.bit_length() - 1
    rows, L = D >> bits, n - bits
    a = rng.normal(size=(D, 3)) + 1j * rng.normal(size=(D, 3))
    a[rows: 2 * rows] = 0.0                   # an empty block of rows
    rho = a @ a.conj().T
    diag = np.diagonal(rho).real
    idx = np.arange(D)
    b_of = idx if one_digit == 1 else (~idx) & (D - 1)
    weights = np.zeros(D)
    weights[b_of] = diag
    u = rng.random(3000)
    ref = _device_search(np.cumsum(weights), u)

    traces = np.array([np.trace(rho[i * rows:(i + 1) * rows, i * rows:(i + 1) * rows]).real for i in range(G)])
    shard, block, local_u = route_shots(u, traces, reverse=(one_digit == 0))
    local_b = np.zeros(len(u), dtype=np.int64)
    for i in range(G):
        sel = shard == i
        if not np.any(sel):
            continue
        lidx = np.arange(rows)
        lb = lidx if one_digit == 1 else (~lidx) & (rows - 1)
        w = np.zeros(rows)
        w[lb] = diag[i * rows:(i + 1) * rows]   # bitstring_weights_kernel on the block: weights[b mod rows]
        local_b[sel] = _device_search(np.cumsum(w), local_u[sel])
    assert np.array_equal(global_bitstring(block, local_b, L), ref)
    assert not np.any(shard == 1)


# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture
def modules(monkeypatch):
    if not HAVE_PULSER:
        pytest.skip("pulser-core not importable here")
    from fake_device import FakeDevicePlan
    from pulser_b200 import backend, engine, lindblad
    from test_density_view_cpu import NumpyDensityPlan

    class FakeShardedLindbladPlan(NumpyDensityPlan):
        """One numpy density matrix standing in for its shards; records the devices it was given."""

        made: list = []

        def __init__(self, specs, devices, interp_order=3):
            super().__init__(specs, interp_order)
            FakeShardedLindbladPlan.made.append(list(devices))

    monkeypatch.setattr(engine, "DevicePlan", FakeDevicePlan)
    monkeypatch.setattr(engine, "device_count", lambda: 2)
    monkeypatch.setattr(lindblad, "LindbladPlan", NumpyDensityPlan)
    monkeypatch.setattr(lindblad, "ShardedLindbladPlan", FakeShardedLindbladPlan)
    FakeShardedLindbladPlan.made = []
    return backend, FakeShardedLindbladPlan


def _seq(n=3):
    from pulser import Pulse, Register, Sequence
    from pulser.devices import MockDevice
    from pulser.waveforms import BlackmanWaveform

    reg = Register.from_coordinates([(7.0 * i, 0.0) for i in range(n)], prefix="q")
    seq = Sequence(reg, MockDevice)
    seq.declare_channel("ch", "rydberg_global")
    seq.add(Pulse.ConstantDetuning(BlackmanWaveform(200, np.pi), 1.0, 0.0), "ch")
    return seq


@pytest.mark.parametrize("kw", [
    {"dephasing_rate": 0.5},
    {"dephasing_rate": 0.5, "relaxation_rate": 0.2},
    {"depolarizing_rate": 0.3},
    {"eff_noise_opers": (np.diag([1.0, 0.0]),), "eff_noise_rates": (0.4,)},
])
def test_collapse_noise_runs_sharded_master_equation(modules, kw):
    """A noise model of collapse operators only goes to the sharded density matrix on `devices`, and its observables are
    those of the same run on one plan."""
    from pulser.backend.default_observables import Occupation
    from pulser.noise_model import NoiseModel

    backend, fake = modules
    noise = NoiseModel(**kw)
    times = [0.5, 1.0]
    res = {}
    for key, extra in (("one", {}), ("shards", {"devices": [0, 1]})):
        cfg = backend.B200Config(noise_model=noise, observables=[Occupation(evaluation_times=times)], **extra)
        res[key] = backend.B200Backend(_seq(), config=cfg).run()
    assert fake.made == [[0, 1]]
    for t in times:
        assert np.allclose(res["one"].get_result("occupation", t), res["shards"].get_result("occupation", t),
                           rtol=0, atol=1e-12)


@pytest.mark.parametrize("kw,needle", [
    ({"temperature": 50.0, "runs": 2, "samples_per_run": 1}, "noiseless"),
    ({"amp_sigma": 0.1, "runs": 2, "samples_per_run": 1}, "without stochastic noise"),
    ({"dephasing_rate": 0.5, "temperature": 50.0, "runs": 2, "samples_per_run": 1}, "noise types"),
    ({"eff_noise_opers": (np.diag([0.0, 0.0, 1.0]),), "eff_noise_rates": (0.5,), "with_leakage": True}, "leakage"),
])
def test_refused_noise_models(modules, kw, needle):
    from pulser.noise_model import NoiseModel

    backend, fake = modules
    cfg = backend.B200Config(devices=[0, 0], noise_model=NoiseModel(**kw))
    with pytest.raises(NotImplementedError, match=needle):
        backend.B200Backend(_seq(), config=cfg).run()
    assert fake.made == []


def test_noiseless_keeps_state_vector_shards(modules):
    """Without noise `devices` still splits the state vector: the routing says so before any plan is made."""
    from pulser.noise_model import NoiseModel

    backend, _ = modules
    assert backend._sharded_master_equation(NoiseModel()) is False
    assert backend._sharded_master_equation(NoiseModel(relaxation_rate=0.1)) is True
