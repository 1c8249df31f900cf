"""GPU tests of ``Expectation`` on device states: ``pb200_state_expect`` / ``pb200_shards_expect`` (the monomial-term
kernels ``expect_terms_d2_kernel`` / ``expect_terms_kernel``) against the scipy matrices and the numpy restatement of
the kernel formula, and the backend's three streaming paths (single plan, shards, noisy batches)."""
import warnings

import numpy as np
import pytest

import opterms_ref
from helpers import random_local_spec, random_state
from pulser_b200 import HAVE_PULSER
from pulser_b200 import workloads as W

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable here")]

EIGS = {2: ("r", "g"), 3: ("r", "g", "h"), 4: ("r", "g", "h", "x")}


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


def _op(eig, n, ops):
    from pulser_b200.backend import B200Operator

    op = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=n, operations=ops)
    assert op._terms is not None
    return op


def _spec(n, d):
    if d == 2:
        return random_local_spec(n, T=20, seed=n)
    spec = W.config_c3(n=n, t_raman=20, t_ryd=40)
    if d == 4:
        spec.eigenbasis = list(spec.eigenbasis) + ["x"]
        spec.dim = 4
    assert tuple(spec.eigenbasis) == EIGS[d]
    return spec


def _named_ops(n):
    """The four operators of experiments/expect_cost.py."""
    x = {"rg": 1.0, "gr": 1.0}
    z = {"rr": 1.0, "gg": -1.0}
    return {
        "sum_x": [(1.0, [(x, {i})]) for i in range(n)],
        "staggered_z": [((-1.0) ** i, [(z, {i})]) for i in range(n)],
        "pairs_pm": [(1.0, [({"rg": 1.0}, {i}), ({"gr": 1.0}, {j})]) for i in range(n) for j in range(n) if i != j],
        "parity": [(1.0, [(z, set(range(n)))])],
    }


def _close(got, ref, rtol=1e-12):
    assert abs(got - ref) <= rtol * max(1.0, abs(ref)), (got, ref)


@pytest.mark.parametrize("d,n", [(2, 5), (2, 8), (2, 12), (2, 13), (2, 16), (3, 5), (4, 4)])
def test_expect_vs_matrix(engine, d, n):
    rng = np.random.default_rng(100 * d + n)
    eig = EIGS[d]
    ops = opterms_ref.random_operations(rng, eig, n, 6)
    z = {eig[0] * 2: 1.0, eig[1] * 2: -1.0}
    ops += [(0.3, [(z, set(range(n)))]), (-0.2j, [({eig[0] + eig[1]: 1.0, eig[1] + eig[0]: 1.0}, set(range(n)))])]
    op = _op(eig, n, ops)
    psi = random_state(d**n, n)
    with engine.DevicePlan(_spec(n, d)) as plan:
        plan.set_state(psi)
        got = plan.expect_terms(op._terms)
    assert got.shape == (1,)
    _close(got[0], complex(np.vdot(psi, op.to_array() @ psi)))


@pytest.mark.parametrize("d,n", [(2, 10), (3, 5), (4, 4)])
def test_expect_several_chunks_vs_matrix(engine, d, n):
    """More than 256 terms and 256 site entries: the term table is staged through shared memory in several chunks."""
    rng = np.random.default_rng(7 * d + n)
    eig = EIGS[d]
    op = _op(eig, n, opterms_ref.random_operations(rng, eig, n, 60))
    assert len(op._terms) > 256 and sum(len(s) for _, s in op._terms.terms) > 256
    psi = random_state(d**n, d)
    with engine.DevicePlan(_spec(n, d)) as plan:
        plan.set_state(psi)
        got = plan.expect_terms(op._terms)[0]
    _close(got, complex(np.vdot(psi, op.to_array() @ psi)))


def test_expect_batch_with_offset(engine):
    n = 9
    eig = EIGS[2]
    op = _op(eig, n, opterms_ref.random_operations(np.random.default_rng(3), eig, n, 8))
    m = op.to_array()
    psis = np.stack([random_state(2**n, s) for s in range(4)])
    with engine.DevicePlan([random_local_spec(n, T=20, seed=s) for s in range(4)]) as plan:
        plan.set_state(psis)
        got = plan.expect_terms(op._terms, traj0=1, count=3)
    assert got.shape == (3,)
    for c in range(3):
        _close(got[c], complex(np.vdot(psis[1 + c], m @ psis[1 + c])))


@pytest.mark.parametrize("n", [20, 24])
def test_expect_large_registers(engine, n):
    psi = random_state(2**n, n)
    named = _named_ops(n)
    if n == 24:
        named.pop("pairs_pm")  # the numpy restatement takes minutes for its 552 terms at this size
    with engine.DevicePlan(random_local_spec(n, T=20, seed=1)) as plan:
        plan.set_state(psi)
        for name, ops in named.items():
            op = _op(EIGS[2], n, ops)
            _close(plan.expect_terms(op._terms)[0], opterms_ref.expect(op._terms, psi))


@pytest.mark.parametrize("G", [2, 4, 8])
def test_sharded_equals_single_plan(engine, G):
    from pulser_b200 import sharded

    n = 16
    eig = EIGS[2]
    rng = np.random.default_rng(G)
    x = {"rg": 1.0, "gr": 1.0}
    cases = {
        "one shard bit": [(1.0, [(x, {i})]) for i in range(n)],
        "several shard bits": [(0.5, [({"rg": 1.0}, {0}), ({"gr": 1.0}, {1}), (x, {n - 1})]),
                               (1.0, [(x, set(range(n)))])],
        "none": [(1.0, [({"rr": 1.0, "gg": -1.0}, set(range(n)))]), (2.0, [({"rr": 1.0}, {0, 5})])],
        "random": opterms_ref.random_operations(rng, eig, n, 10),
    }
    spec = W.config_c2(n=n, seed=2)
    psi = random_state(2**n, G)
    with engine.DevicePlan(spec) as single, sharded.ShardedPlan(spec, [0] * G) as plan:
        single.set_state(psi)
        plan.set_state(psi)
        for name, ops in cases.items():
            op = _op(eig, n, ops)
            got = plan.expect_terms(op._terms)
            assert got.shape == (1,)
            _close(got[0], single.expect_terms(op._terms)[0])


def _sequence(n=14, duration=300):
    from pulser import Pulse, Register, Sequence
    from pulser.devices import MockDevice
    from pulser.waveforms import BlackmanWaveform

    reg = Register.from_coordinates([(6.0 * (i % 7), 6.0 * (i // 7)) for i in range(n)], prefix="q")
    seq = Sequence(reg, MockDevice)
    seq.declare_channel("ch", "rydberg_global")
    seq.add(Pulse.ConstantDetuning(BlackmanWaveform(duration, np.pi), -1.0, 0.0), "ch")
    return seq


@pytest.mark.parametrize("mode", ["single", "shards", "doppler"])
def test_backend_expectation_on_device(engine, monkeypatch, mode):
    """``Expectation`` in a ``B200Backend`` run equals the host evaluation of the same run's states, without a matrix."""
    import pulser
    from pulser.backend.default_observables import Expectation
    from pulser.backend.observable import Callback

    from pulser_b200 import backend

    n = 14
    eig = ("r", "g")
    named = _named_ops(n)
    ops = {k: _op(eig, n, v) for k, v in named.items()}
    mats = {k: _op(eig, n, v).to_array() for k, v in named.items()}  # separate instances: the run's never build one
    times = [0.5, 1.0]
    seen: dict = {}

    class HostExpect(Callback):
        def __call__(self, config, t, state, hamiltonian, result):
            hit = [s for s in times if abs(t - s) < 1e-6]
            if hit:
                psi = state.to_array()
                for k, m in mats.items():
                    seen.setdefault((k, hit[0]), []).append(complex(np.vdot(psi, m @ psi)))

    kw = {}
    if mode == "shards":
        kw["devices"] = [0, 0]
    if mode == "doppler":
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            kw["noise_model"] = pulser.NoiseModel(temperature=50.0)
        kw["n_trajectories"] = 3
    obs = [Expectation(op, evaluation_times=times, tag_suffix=k) for k, op in ops.items()]
    cfg = backend.B200Config(observables=obs, callbacks=[HostExpect()], default_evaluation_times=times, **kw)
    built = []
    orig = backend.B200Operator._as_matrix
    monkeypatch.setattr(backend.B200Operator, "_as_matrix", staticmethod(lambda x: (built.append(1), orig(x))[1]))
    np.random.seed(11)
    res = backend.B200Backend(_sequence(n), config=cfg).run()
    monkeypatch.undo()
    assert len(built) == 0
    # the config's operators went through the C ABI and still copy (Pulser deep-copies observables)
    import copy

    copy.deepcopy(cfg)
    assert cfg.with_changes(sampling_rate=0.5).observables[0].operator._terms.terms == cfg.observables[0].operator._terms.terms
    for k in ops:
        for t in times:
            ref = np.mean(seen[(k, t)])
            assert len(seen[(k, t)]) == (3 if mode == "doppler" else 1)
            got = res.get_result(f"expectation_{k}", t)
            assert isinstance(got, float)  # Hermitian: real, like qutip.expect
            assert abs(got - ref.real) <= 1e-10 * max(1.0, abs(ref)) and abs(ref.imag) < 1e-10 * max(1.0, abs(ref))


def test_refusals(engine):
    import ctypes as C

    from pulser_b200 import sharded
    from pulser_b200._lib import PB200Error, lib

    n = 14
    op = _op(EIGS[2], n, _named_ops(n)["sum_x"])
    with sharded.ShardedPlan(W.config_c2(n=n, seed=2), [0, 0]) as plan:
        plan.set_state("all-ground")
        out = np.zeros(2)
        assert lib.pb200_state_expect(plan.shards[0]._handle, 0, 1, C.byref(op._terms.c_desc()),
                                      out.ctypes.data_as(C.POINTER(C.c_double))) != 0
        assert b"pb200_shards_expect" in lib.pb200_last_error()
    wide = _op(EIGS[2], n + 1, _named_ops(n + 1)["sum_x"])._terms
    wide.n = n  # an operator whose site n lies outside an n-qudit register
    with engine.DevicePlan(random_local_spec(n, T=20)) as plan:
        plan.set_state("all-ground")
        with pytest.raises(PB200Error, match="names qudit 14 of a 14-qudit register") as e:
            plan.expect_terms(wide)
        assert e.value.code == -1


def test_density_matrix_plan_refused(engine):
    from pulser_b200._lib import PB200Error
    from pulser_b200.lindblad import LindbladPlan

    n = 3
    spec = random_local_spec(n, T=20)
    spec.collapse_ops = np.array([np.sqrt(0.3) * np.array([[1, 0], [0, 0]], dtype=complex)])
    with LindbladPlan(spec) as lp:
        lp.set_state(random_state(2**n, 1))
        op = _op(EIGS[2], 2 * n, _named_ops(2 * n)["sum_x"])  # the plan holds the vectorised density matrix: 2N qudits
        with pytest.raises(PB200Error, match="density matrix") as e:
            lp.plan.expect_terms(op._terms)
        assert e.value.code == -3
