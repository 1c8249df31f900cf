"""Global drives whose phase changes in time on the Taylor propagator: phase jumps between pulses, phase ramps and
stretches of one phase other than the reference row's, on every stage-kernel variant.

Each case is held to the propagator's own bound against the exact piecewise-cubic reference (tests/taylor_ref.py, which
splines the real and imaginary drive parts separately, so it is exact for a moving phase):

    ||psi_dev - psi_ref||_2 <= (2 err_estimate + 1e-14) ||psi0||_2

The step log shows which drive kind each step ran: ``real`` (the plan's own phase), ``rot`` (one other phase over the
step: the constant-phase kernels with the step's unit) and ``cplx`` (the phase moves inside the step: the complex-drive
kernels, two gathers per order).
"""
from __future__ import annotations

import dataclasses
import functools
import re
from typing import Callable

import numpy as np
import pytest

from helpers import curved_spec, random_state, with_dmm
from phase_sequences import KINDS, moving_phase_rows, phase_sequence
from pulser_b200 import HAVE_PULSER
from pulser_b200 import workloads as W
from taylor_ref import PiecewiseCubicHamiltonian

pytestmark = pytest.mark.gpu

A = 2.0
FLOOR = 1e-14
TIGHT = 1e-11
STATE_TOL = 1e-8

STEP_RE = re.compile(r"taylor step t=\S+ h_ns=\S+ p_om=(\d+) p_th=\d+ p_m=\d+ K=(\d+) ring=(\d+) .* drive=(\w+)")


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


# ---------------------------------------------------------------- inputs
def _phase_steps(T: int, edges, phases) -> np.ndarray:
    """phase samples: phases[i] from edges[i - 1] on (edges in ns)"""
    t = np.arange(T)
    return np.asarray(phases, dtype=float)[np.searchsorted(np.asarray(edges), t, side="right")]


@functools.lru_cache(maxsize=None)
def _jump(n: int):
    """C2 shape (rise, sweep, fall; 500 ns): phase 0 until 250 ns, then pi/2 under full amplitude.  The largest sample
    (the reference row's phase) lies in the first half, so the second half runs the constant-phase kernels rotated"""
    amp, det = W.blockade_sweep_waveforms(t_rise=100, t_sweep=300, t_fall=100)
    ph = _phase_steps(len(amp), [250], [0.0, np.pi / 2])
    return W.ising_global_spec(W.disc_register(n, 22.0, 6.0, n), W.C6_LEVEL_60, amp, det, phase=ph)


@functools.lru_cache(maxsize=None)
def _ramp(n: int):
    """Blackman / sin^2 over 8 us with a slow linear phase ramp: multi-interval complex steps of high degree"""
    return curved_spec(n, T=8000, phase=0.2 + 0.6 * np.arange(8000) / 8000, seed=n, swing=4.0)


def _base(kind: str, n: int):
    return _jump(n) if kind == "jump" else _ramp(n)


@functools.lru_cache(maxsize=None)
def _dmm(kind: str, n: int, n_maps: int):
    return with_dmm(_base(kind, n), n_maps, seed=n + n_maps)


@functools.lru_cache(maxsize=None)
def _noisy(kind: str, n: int, n_traj: int, n_maps: int = 0):
    base = _base(kind, n)
    if n_maps:
        base = with_dmm(base, n_maps, seed=n)
    coords = W.disc_register(n, 22.0, 6.0, n)
    rng = np.random.default_rng(10 * n + n_traj)
    return tuple(W.noisy_trajectory_spec(base, coords, rng.normal(0, 1.5, n), 1.0 + 0.05 * rng.normal(), 60.0)
                 for _ in range(n_traj))


def _interval(i: int, f0: float = 0.0, f1: float = 1.0):
    def window(spec):
        t = spec.sampling_times
        return t[i] + f0 * (t[i + 1] - t[i]), t[i] + f1 * (t[i + 1] - t[i])
    return window


def _span(a: float, b: float):
    return lambda spec: (a, b)


JUMP = _interval(249)              # the sampling interval of the jump: both drive parts move
ROT = _interval(320, 0.2, 0.9)     # a stretch of phase pi/2: one phase, not the reference row's
RAMP = _span(3.0500, 3.2500)       # 200 ns of the slow ramp


@dataclasses.dataclass(frozen=True)
class Case:
    id: str
    variant: str
    specs: Callable
    window: Callable
    drive: str                     # the drive kind every step of the case runs
    shards: int = 0


CASES = [
    # stage_d2_taylor_small_kernel<true> (N < 13)
    Case("small_jump_n12", "small", lambda: _jump(12), JUMP, "cplx"),
    Case("small_rot_n12", "small", lambda: _jump(12), ROT, "rot"),
    Case("small_ramp_n12", "small", lambda: _ramp(12), RAMP, "cplx"),
    Case("small_batch_jump_n6", "small", lambda: _noisy("jump", 6, 3), JUMP, "cplx"),
    Case("small_dmm_batch_rot_n6", "small", lambda: _noisy("jump", 6, 2, n_maps=2), ROT, "rot"),
    # uniform
    Case("uniform_jump_n13", "uniform", lambda: _jump(13), JUMP, "cplx"),
    Case("uniform_rot_n14", "uniform", lambda: _jump(14), ROT, "rot"),
    Case("uniform_ramp_n13", "uniform", lambda: _ramp(13), RAMP, "cplx"),
    # batch, one detuning shape
    Case("batch_jump_n13", "batch", lambda: _noisy("jump", 13, 2), JUMP, "cplx"),
    Case("batch_rot_n14", "batch", lambda: _noisy("jump", 14, 2), ROT, "rot"),
    Case("batch_ramp_n13", "batch", lambda: _noisy("ramp", 13, 2), RAMP, "cplx"),
    # uniform drive with detuning shapes (NS = PB200_TAYLOR_SMAX)
    Case("dmm1_jump_n13", "dmm_single", lambda: _dmm("jump", 13, 1), JUMP, "cplx"),
    Case("dmm4_rot_n13", "dmm_single", lambda: _dmm("jump", 13, 4), ROT, "rot"),
    Case("dmm1_ramp_n13", "dmm_single", lambda: _dmm("ramp", 13, 1), RAMP, "cplx"),
    # batch with several shapes
    Case("dmm_batch_jump_n14", "dmm_batch", lambda: _noisy("jump", 14, 2, n_maps=2), JUMP, "cplx"),
    Case("dmm_batch_rot_n14", "dmm_batch", lambda: _noisy("jump", 14, 2, n_maps=2), ROT, "rot"),
    Case("dmm_batch_ramp_n14", "dmm_batch", lambda: _noisy("ramp", 14, 2, n_maps=2), RAMP, "cplx"),
    # shards of device 0
    Case("shard_g2_jump_n16", "shard", lambda: _jump(16), JUMP, "cplx", shards=2),
    Case("shard_g4_rot_n16", "shard", lambda: _jump(16), ROT, "rot", shards=4),
    Case("shard_g8_ramp_n16", "shard", lambda: _ramp(16), RAMP, "cplx", shards=8),
    Case("shard_dmm1_jump_n16", "shard_dmm", lambda: _dmm("jump", 16, 1), JUMP, "cplx", shards=2),
    Case("shard_dmm4_rot_n16", "shard_dmm", lambda: _dmm("jump", 16, 4), ROT, "rot", shards=8),
    Case("shard_dmm1_ramp_n16", "shard_dmm", lambda: _dmm("ramp", 16, 1), RAMP, "cplx", shards=4),
]

_REFS: dict = {}
_RESULTS: dict = {}


def _run(case, engine, capfd, monkeypatch):
    if case.id in _RESULTS:
        return _RESULTS[case.id]
    from pulser_b200 import sharded

    specs = case.specs()
    specs = list(specs) if isinstance(specs, tuple) else [specs]
    a, b = case.window(specs[0])
    psi0 = [random_state(specs[0].hilbert_dim, 31 + k) for k in range(len(specs))]
    monkeypatch.setenv("PB200_TAYLOR_LOG", "1")
    capfd.readouterr()
    plan = sharded.ShardedPlan(specs[0], [0] * case.shards) if case.shards else \
        engine.DevicePlan(specs if len(specs) > 1 else specs[0])
    with plan:
        plan.set_state(np.stack(psi0) if len(specs) > 1 else psi0[0])
        st = plan.propagate(a, b, integrator=3, tol=TIGHT)
        got = plan.get_state()
    steps = [(int(m[1]), int(m[2]), int(m[3]), m[4]) for m in STEP_RE.finditer(capfd.readouterr().err)]
    errs = []
    for k, (s, p) in enumerate(zip(specs, psi0)):
        key = (case.id, k)
        if key not in _REFS:
            _REFS[key] = PiecewiseCubicHamiltonian(s).evolve(p, a, b)
        errs.append(float(np.linalg.norm(got[k] - _REFS[key])))
    _RESULTS[case.id] = {"st": st, "steps": steps, "errs": errs}
    return _RESULTS[case.id]


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_within_own_error_bound(engine, case, capfd, monkeypatch):
    r = _run(case, engine, capfd, monkeypatch)
    st = r["st"]
    assert st["integrator"] == 3
    assert len(r["steps"]) == st["n_steps"] > 0
    assert {s[3] for s in r["steps"]} == {case.drive}, r["steps"]
    assert st["err_estimate"] <= TIGHT
    bound = A * st["err_estimate"] + FLOOR
    for k, e in enumerate(r["errs"]):
        assert e <= bound, (k, e, st["err_estimate"])


def test_step_log_reach(engine, capfd, monkeypatch):
    """every variant runs both drive kinds; the ramps reach p_om >= 4 with the doubled G history (ring of a complex
    step = chi ring + 2 (p_om + 1))"""
    for case in CASES:
        _run(case, engine, capfd, monkeypatch)
    for variant in {c.variant for c in CASES}:
        kinds = {s[3] for c in CASES if c.variant == variant for s in _RESULTS[c.id]["steps"]}
        assert kinds == {"rot", "cplx"}, variant
    cplx = [s for r in _RESULTS.values() for s in r["steps"] if s[3] == "cplx"]
    assert max(s[0] for s in cplx) >= 4
    assert any(s[2] >= 2 * (s[0] + 1) + 2 for s in cplx if s[0] >= 4)
    with capfd.disabled():
        print("\nmax ||error|| / err_estimate per stage variant (moving phase):")
        for variant in dict.fromkeys(c.variant for c in CASES):
            ratios = [max(_RESULTS[c.id]["errs"]) / _RESULTS[c.id]["st"]["err_estimate"]
                      for c in CASES if c.variant == variant and _RESULTS[c.id]["st"]["err_estimate"] > FLOOR]
            print(f"  {variant:12s} {max(ratios):.3f}" if ratios else f"  {variant:12s} -")


def test_constant_phase_logs_real(engine, capfd, monkeypatch):
    """a constant-phase sequence of any phase runs every step as `real`"""
    monkeypatch.setenv("PB200_TAYLOR_LOG", "1")
    spec = W.config_c2(n=14)
    spec2 = curved_spec(13, T=600, phase=0.83)
    for s in (spec, spec2):
        capfd.readouterr()
        with engine.DevicePlan(s) as plan:
            plan.set_state("all-ground")
            st = plan.propagate(0.0, s.sampling_times[-1], integrator=3)
        kinds = {m[4] for m in STEP_RE.finditer(capfd.readouterr().err)}
        assert st["integrator"] == 3 and kinds == {"real"}


# ---------------------------------------------------------------- whole sequences
def _oracle(spec, psi0, tf):
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    return evolve.sesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf], rtol=1e-13, atol=1e-15)[-1]


def _ramsey(n: int, phi: float = 1.1):
    """pi/2 (100 ns) at phase 0, 300 ns of free evolution, pi/2 at phase phi"""
    T = 500
    t = np.arange(T)
    amp = np.where((t < 100) | ((t >= 400) & (t < 500)), np.pi / 0.2, 0.0)
    det = np.full(T, -2.0)
    ph = _phase_steps(T, [250], [0.0, phi])
    return W.ising_global_spec(W.disc_register(n, 14.0, 6.0, n), W.C6_LEVEL_60, amp, det, phase=ph)


def _back_to_back(n: int):
    """three 150 ns square pulses back to back, phases 0, 0.7, -1.3: two jumps under full amplitude"""
    T = 450
    amp = np.full(T, 2 * np.pi * 1.5)
    det = np.linspace(-6.0, 4.0, T)
    ph = _phase_steps(T, [150, 300], [0.0, 0.7, -1.3])
    return W.ising_global_spec(W.disc_register(n, 14.0, 6.0, n), W.C6_LEVEL_60, amp, det, phase=ph)


@pytest.mark.parametrize("n", [8, 13])
@pytest.mark.parametrize("kind", ["ramsey", "back_to_back"])
def test_sequences_vs_oracle(engine, kind, n):
    from oracle import evolve

    spec = _ramsey(n) if kind == "ramsey" else _back_to_back(n)
    tf = spec.sampling_times[-1]
    psi0 = evolve.all_ground_state(spec)
    ref = _oracle(spec, psi0, tf)
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf)
        got = plan.get_state()[0]
    assert st["integrator"] == 3           # the auto rule takes the Taylor propagator
    assert st["err_estimate"] < 1e-8
    assert np.max(np.abs(got - ref)) < STATE_TOL


def test_noisy_ramsey_batch_vs_oracle(engine):
    from oracle import evolve

    n = 8
    base = _ramsey(n)
    coords = W.disc_register(n, 14.0, 6.0, n)
    rng = np.random.default_rng(5)
    specs = [W.noisy_trajectory_spec(base, coords, rng.normal(0, 1.5, n), 1.0 + 0.05 * rng.normal(), 60.0)
             for _ in range(3)]
    tf = base.sampling_times[-1]
    psi0 = evolve.all_ground_state(base)
    with engine.DevicePlan(specs) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf)
        got = plan.get_state().copy()
    assert st["integrator"] == 3
    for b, s in enumerate(specs):
        assert np.max(np.abs(got[b] - _oracle(s, psi0, tf))) < STATE_TOL, b


def test_n20_jump_vs_cf4(engine):
    """N = 20, phase jump mid-sweep: Taylor against Richardson-CF4 (what ran before), far fewer H-applies"""
    spec = _jump(20)
    tf = spec.sampling_times[-1]
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf, tol=1e-10)
        tay = plan.get_state()[0].copy()
        plan.set_state("all-ground")
        st1 = plan.propagate(0.0, tf, integrator=1, tol=1e-10)
        cf4 = plan.get_state()[0]
    assert st["integrator"] == 3 and st1["integrator"] == 1
    assert np.max(np.abs(tay - cf4)) < STATE_TOL
    assert st["n_applies"] < 0.5 * st1["n_applies"]


@pytest.mark.parametrize("G", [2, 4, 8])
def test_shards_match_unsharded(engine, G):
    from pulser_b200 import sharded

    spec = _jump(16)
    tf = spec.sampling_times[-1]
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st1 = plan.propagate(0.0, tf)
        one = plan.get_state()[0].copy()
    with sharded.ShardedPlan(spec, [0] * G) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf)
        psi = plan.get_state()[0]
    for k in ("n_steps", "n_applies", "integrator"):
        assert st[k] == st1[k], k
    assert st["err_estimate"] == pytest.approx(st1["err_estimate"], rel=1e-12)
    assert np.max(np.abs(psi - one)) < 1e-12


# ---------------------------------------------------------------- through the public API
def _taylor_forced(engine, spec):
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, spec.sampling_times[-1], integrator=3)
        return st, plan.get_state()[0].copy()


@pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable")
@pytest.mark.parametrize("kind", KINDS)
def test_pulser_sequences(engine, kind):
    """real Pulser sequences through B200Emulator: the auto rule takes the Taylor propagator for the two smooth
    sequences (and for the EOM block where taylor_worthwhile accepts it; otherwise Taylor is forced on the same
    spec), and the result agrees with the Magnus path"""
    from pulser_b200.emulator import B200Emulator

    emu = B200Emulator.from_sequence(phase_sequence(kind), evaluation_times="Minimal")
    assert moving_phase_rows(emu._current_spec)
    auto = emu.run().states[-1].full().ravel()
    integrator = emu.last_run_stats["integrator"]
    mag = emu.run(b200_max_step=20).states[-1].full().ravel()
    assert emu.last_run_stats["integrator"] in (1, 2)
    if kind != "eom":
        assert integrator == 3
    tay = auto
    if integrator != 3:
        st, tay = _taylor_forced(engine, emu._current_spec)
        assert st["integrator"] == 3
    assert np.max(np.abs(tay - mag)) < STATE_TOL


@pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable")
@pytest.mark.parametrize("kind", ["phases", "phase_shift"])
def test_pulser_sequences_on_shards(engine, kind):
    """B200Backend with devices=[0, 0] runs what it refused while the phase had to be constant, and agrees with one
    plan"""
    from pulser.backend.default_observables import Occupation
    from pulser_b200.backend import B200Backend, B200Config

    seq = phase_sequence(kind, n=14)   # 2 shards of 2^13 amplitudes
    occ = {}
    for key, kw in (("one", {}), ("shards", {"devices": [0, 0]})):
        res = B200Backend(seq, config=B200Config(observables=[Occupation(evaluation_times=[1.0])], **kw)).run()
        occ[key] = np.asarray(res.get_result("occupation", 1.0), dtype=float)
    assert np.max(np.abs(occ["one"] - occ["shards"])) < 1e-7
