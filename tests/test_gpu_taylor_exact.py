"""Every variant of the Taylor stage kernel against the exact piecewise-cubic reference (tests/taylor_ref.py), held to
the propagator's own a-priori bound:

    ||psi_dev - psi_ref||_2 <= (A * err_estimate + 1e-14) * ||psi0||_2        (every trajectory / the whole sharded state)

``err_estimate`` is what ``propagate`` returns: fit residuals + Taylor remainders (bounds) + the rounding estimate
0.05 eps e^rho per step (DESIGN 3a). Only the rounding part is an estimate, hence A > 1. The tight cases run at
``tol = 1e-11``, so that each check is at least 1000x tighter than the 1e-8 of the whole-sequence tests.

One-interval calls (the facade's "Full" evaluation times) are one exact cubic step: only truncation and rounding remain.
Multi-interval windows of 60-300 ns on slow Blackman / sin^2 waveforms reach polynomial degrees 4-8, the stored-gather
(``G``) history and the fit residuals. The step log (``PB200_TAYLOR_LOG``) shows that the cases reach what they are
meant to reach.
"""
from __future__ import annotations

import dataclasses
import functools
import re
from typing import Callable

import numpy as np
import pytest

from helpers import curved_spec, random_state, with_dmm
from pulser_b200 import workloads as W
from taylor_ref import PiecewiseCubicHamiltonian

pytestmark = pytest.mark.gpu

# ||error|| / err_estimate allowed: only the rounding part of the bound is an estimate.  Measured on an H100 80GB HBM3
# (700 W): at most 0.49 where err_estimate exceeds the floor (small kernel, N = 6 batch over 200 ns), 0.11 on N >= 13.
A = 2.0
FLOOR = 1e-14    # relative to ||psi0||: the rounding of one short step and of the reference
TIGHT = 1e-11

STEP_RE = re.compile(r"taylor step t=\S+ h_ns=\S+ p_om=(\d+) p_th=(\d+) p_m=\d+ K=(\d+) ring=(\d+) rho=(\S+)")


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


# ---------------------------------------------------------------- inputs
@functools.lru_cache(maxsize=None)
def _c2(n: int, phase: float = 0.0):
    """C2-shaped (rise, sweep, fall; 500 ns) on a register spread enough to keep the reference cheap"""
    amp, det = W.blockade_sweep_waveforms(t_rise=100, t_sweep=300, t_fall=100)
    return W.ising_global_spec(W.disc_register(n, 22.0, 6.0, n), W.C6_LEVEL_60, amp, det, phase=phase)


@functools.lru_cache(maxsize=None)
def _curved(n: int, phase: float = 0.0):
    """Blackman amplitude and sin^2 detuning over 8 us: at tol = 1e-11 the splines of 1 ns samples are then smooth
    enough (4th differences / 384 below the fit budget) for steps of degree 4-8 over tens of sampling intervals"""
    return curved_spec(n, T=8000, phase=phase, seed=n, swing=4.0)


@functools.lru_cache(maxsize=None)
def _weak(n: int):
    """weak drive and detuning, far-apart atoms: a 1e-6 us window then needs only K = 2 orders"""
    amp, det = np.full(200, 2.0), np.linspace(-2.0, 1.0, 200)
    return W.ising_global_spec(W.disc_register(n, 40.0, 14.0, n), W.C6_LEVEL_60, amp, det)


@functools.lru_cache(maxsize=None)
def _strong(n: int):
    """strong drive and detuning sampled every 40 ns: one interval spans rho > 14 and takes several steps"""
    T = 12
    t = np.arange(T)
    amp = 2 * np.pi * (6.0 + 2.0 * np.sin(0.5 * t))
    det = -30.0 + 4.0 * t
    spec = W.ising_global_spec(W.disc_register(n, 22.0, 6.0, n), W.C6_LEVEL_60, amp, det)
    spec.sampling_times = np.arange(T + 1, dtype=float) * 40.0 / 1000
    spec.total_duration_ns = 40 * T
    return spec


@functools.lru_cache(maxsize=None)
def _dmm(base: str, n: int, n_maps: int, phase: float = 0.0):
    return with_dmm((_c2 if base == "c2" else _curved)(n, phase), n_maps, seed=n + n_maps)


@functools.lru_cache(maxsize=None)
def _noisy(kind: str, n: int, n_traj: int, phase: float = 0.4, n_maps: int = 0):
    """C4-shaped batch (doppler offsets + per-atom amplitude factors) of a C2-shaped or curved sequence, optionally with
    detuning maps (then 1 + n_maps detuning shapes)"""
    base = (_c2 if kind == "c2" else _curved)(n, phase)
    if n_maps:
        base = with_dmm(base, n_maps, seed=n)
    coords = W.disc_register(n, 22.0, 6.0, n)
    rng = np.random.default_rng(10 * n + n_traj)
    return tuple(W.noisy_trajectory_spec(base, coords, rng.normal(0, 1.5, n), 1.0 + 0.05 * rng.normal(), 60.0)
                 for _ in range(n_traj))


def _interval(i: int, f0: float = 0.0, f1: float = 1.0):
    """window inside sampling interval i (i < 0: counted from the end, -1 = the last, zero-padded one)"""
    def window(spec):
        t = spec.sampling_times
        j = i % (len(t) - 1)
        return t[j] + f0 * (t[j + 1] - t[j]), t[j] + f1 * (t[j + 1] - t[j])
    return window


def _tiny(i: int):
    def window(spec):
        a = spec.sampling_times[i] + 0.4e-3
        return a, a + 1e-6
    return window


def _span(a: float, b: float):
    return lambda spec: (a, b)


@dataclasses.dataclass(frozen=True)
class Case:
    id: str
    variant: str                   # the stage-kernel instantiation the case runs
    specs: Callable                # () -> spec or tuple of specs (a batch)
    window: Callable               # spec -> (a, b)
    one_interval: bool
    one_step: bool = False         # the interval's rho is below the cap: exactly one step
    tol: float = TIGHT
    shards: int = 0                # G > 0: ShardedPlan on G shards of device 0
    norm: float = 1.0

    @property
    def tight(self) -> bool:
        return self.tol <= TIGHT


CASES = [
    # stage_d2_taylor_small_kernel (N < 13)
    Case("small_real_tiny_n6", "small", lambda: _weak(6), _tiny(100), True, True),
    Case("small_complex_offgrid_n12", "small", lambda: _c2(12, 0.83), _interval(250, 0.3, 0.8), True, True),
    Case("small_batch_last_n6", "small", lambda: _noisy("c2", 6, 3), _interval(-1), True, True),
    Case("small_dmm1_ramp_n6", "small", lambda: _dmm("c2", 6, 1), _interval(50), True, True),
    Case("small_dmm4_plateau_n12", "small", lambda: _dmm("c2", 12, 4), _interval(250), True, True),
    Case("small_dmm_batch_n6", "small", lambda: _noisy("c2", 6, 3, n_maps=2), _interval(300), True, True),
    Case("small_real_multi_n6", "small", lambda: _curved(6), _span(3.0123, 3.2877), False),
    Case("small_complex_multi_n12", "small", lambda: _curved(12, 0.83), _span(3.1003, 3.2003), False),
    Case("small_batch_multi_n6", "small", lambda: _noisy("curved", 6, 3), _span(3.0500, 3.2500), False),
    Case("small_dmm4_multi_n12", "small", lambda: _dmm("curved", 12, 4), _span(3.1000, 3.2000), False),
    Case("small_dmm_batch_multi_n6", "small", lambda: _noisy("curved", 6, 3, n_maps=2), _span(3.1000, 3.2500), False),
    # <UNIFORM=true, REAL_G=true>: C2 shape, phase 0
    Case("uniform_real_ramp_n13", "uniform_real", lambda: _c2(13), _interval(50), True, True),
    Case("uniform_real_plateau_n14", "uniform_real", lambda: _c2(14), _interval(250), True, True),
    Case("uniform_real_last_n16", "uniform_real", lambda: _c2(16), _interval(-1), True, True),
    Case("uniform_real_plateau_n20", "uniform_real", lambda: _c2(20), _interval(250), True, True),
    Case("uniform_real_ramp_n22", "uniform_real", lambda: _c2(22), _interval(450), True, True),
    Case("uniform_real_tiny_n13", "uniform_real", lambda: _c2(13), _tiny(250), True, True),
    Case("uniform_real_strong_n13", "uniform_real", lambda: _strong(13), _interval(5), True, tol=1e-8),
    Case("uniform_real_multi_n13", "uniform_real", lambda: _curved(13), _span(3.0500, 3.2500), False),
    Case("uniform_real_multi_unnormalised_n14", "uniform_real", lambda: _curved(14), _span(3.1201, 3.1801), False,
         norm=2.5),
    # <true, false>: phase != 0
    Case("uniform_complex_offgrid_n16", "uniform_complex", lambda: _c2(16, 0.83), _interval(120, 0.3, 0.8), True, True),
    Case("uniform_complex_multi_n13", "uniform_complex", lambda: _curved(13, 0.83), _span(3.0877, 3.2377), False),
    # <false, false>: C4-shaped batch
    Case("batch_plateau_n16", "batch", lambda: _noisy("c2", 16, 2), _interval(250), True, True),
    Case("batch_multi_n13", "batch", lambda: _noisy("curved", 13, 3), _span(3.1000, 3.2000), False),
    # <true, true / false, SHARD=false, NS=4>: DMM single state
    Case("dmm1_real_ramp_n16", "dmm_single", lambda: _dmm("c2", 16, 1), _interval(50), True, True),
    Case("dmm4_complex_offgrid_n13", "dmm_single", lambda: _dmm("c2", 13, 4, 0.83), _interval(200, 0.3, 0.8), True,
         True),
    Case("dmm1_complex_multi_n13", "dmm_single", lambda: _dmm("curved", 13, 1, 0.83), _span(3.1000, 3.2000), False),
    Case("dmm4_real_multi_n13", "dmm_single", lambda: _dmm("curved", 13, 4), _span(3.1000, 3.2000), False),
    # <false, false, false, NS=4>: noisy DMM batch (2 maps + doppler = 3 shapes)
    Case("dmm_batch_last_n14", "dmm_batch", lambda: _noisy("c2", 14, 3, n_maps=2), _interval(-1), True, True),
    Case("dmm_batch_multi_n14", "dmm_batch", lambda: _noisy("curved", 14, 2, n_maps=2), _span(3.1200, 3.1800), False),
    # <true, true / false, SHARD=true>: ShardedPlan on one device
    Case("shard_g2_real_n16", "shard", lambda: _c2(16), _interval(250), True, True, shards=2),
    Case("shard_g4_complex_n16", "shard", lambda: _c2(16, 0.83), _interval(120, 0.3, 0.8), True, True, shards=4),
    Case("shard_g8_real_n16", "shard", lambda: _c2(16), _interval(250), True, True, shards=8),
    Case("shard_g8_real_n20", "shard", lambda: _c2(20), _interval(250), True, True, shards=8),
    Case("shard_g2_real_multi_n16", "shard", lambda: _curved(16), _span(3.1200, 3.1800), False, shards=2),
    Case("shard_g4_complex_multi_n16", "shard", lambda: _curved(16, 0.83), _span(3.1200, 3.1800), False, shards=4),
    # <true, true / false, SHARD=true, NS=4>: sharded DMM
    Case("shard_dmm1_real_n16", "shard_dmm", lambda: _dmm("c2", 16, 1), _interval(50), True, True, shards=2),
    Case("shard_dmm4_complex_n16", "shard_dmm", lambda: _dmm("c2", 16, 4, 0.83), _interval(250), True, True,
         shards=4),
    Case("shard_dmm1_real_multi_n16", "shard_dmm", lambda: _dmm("curved", 16, 1), _span(3.1200, 3.1800), False,
         shards=4),
    Case("shard_dmm4_complex_multi_n16", "shard_dmm", lambda: _dmm("curved", 16, 4, 0.83), _span(3.1200, 3.1800), False,
         shards=8),
]


# ---------------------------------------------------------------- running a case
_REFS: dict = {}
_RESULTS: dict = {}


def _states(case, D, n_traj):
    return [case.norm * random_state(D, 31 + b) for b in range(n_traj)]


def _reference(spec, psi0, a, b):
    key = (id(spec), psi0.tobytes(), a, b)
    if key not in _REFS:
        _REFS[key] = PiecewiseCubicHamiltonian(spec).evolve(psi0, a, b)
    return _REFS[key]


def _run(case, engine, capfd, monkeypatch):
    if case.id in _RESULTS:
        return _RESULTS[case.id]
    from pulser_b200 import sharded

    specs = case.specs()
    specs = list(specs) if isinstance(specs, tuple) else [specs]
    a, b = case.window(specs[0])
    psi0 = _states(case, specs[0].hilbert_dim, len(specs))
    monkeypatch.setenv("PB200_TAYLOR_LOG", "1")
    capfd.readouterr()
    if case.shards:
        plan = sharded.ShardedPlan(specs[0], [0] * case.shards)
    else:
        plan = engine.DevicePlan(specs if len(specs) > 1 else specs[0])
    with plan:
        plan.set_state(np.stack(psi0) if len(specs) > 1 else psi0[0])
        st = plan.propagate(a, b, integrator=3, tol=case.tol)
        got = plan.get_state()
    steps = [tuple(float(x) for x in m.groups()) for m in STEP_RE.finditer(capfd.readouterr().err)]
    errs = [float(np.linalg.norm(got[i] - _reference(s, p, a, b))) for i, (s, p) in enumerate(zip(specs, psi0))]
    res = {"st": st, "steps": steps, "errs": errs, "norm": case.norm, "window": (a, b)}
    _RESULTS[case.id] = res
    return res


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_within_own_error_bound(engine, case, capfd, monkeypatch):
    r = _run(case, engine, capfd, monkeypatch)
    st = r["st"]
    assert st["integrator"] == 3
    assert len(r["steps"]) == st["n_steps"] > 0
    if case.tight:
        assert st["err_estimate"] <= TIGHT
    if case.one_step:
        assert st["n_steps"] == 1
    bound = (A * st["err_estimate"] + FLOOR) * case.norm
    for b, e in enumerate(r["errs"]):
        assert e <= bound, (b, e, st["err_estimate"])


def test_step_log_reach(engine, capfd, monkeypatch):
    """the cases as a whole reach high polynomial degrees of both coefficient functions, both parities of the order,
    long steps and a deep ring; the strong one-interval case is split into several steps near the cap"""
    for case in CASES:
        _run(case, engine, capfd, monkeypatch)
    steps = np.array([s for r in _RESULTS.values() for s in r["steps"]])
    p_om, p_th, K, ring, rho = steps.T
    assert p_om.max() >= 4 and p_th.max() >= 4
    assert set(K.astype(int) % 2) == {0, 1}
    assert rho.max() >= 10 and ring.max() >= 8
    assert _RESULTS["small_real_tiny_n6"]["steps"][0][2] == 2      # a 1e-6 us window: K = 2
    strong = _RESULTS["uniform_real_strong_n13"]
    assert strong["st"]["n_steps"] >= 2 and max(s[4] for s in strong["steps"]) >= 10
    for variant in {c.variant for c in CASES}:
        kinds = {c.one_interval for c in CASES if c.variant == variant}
        assert kinds == {True, False}, variant
    with capfd.disabled():   # the ratios where the estimate is above the rounding floor of one short step
        print("\nmax ||error|| / (err_estimate ||psi0||) per stage variant, cases with err_estimate > 1e-14:")
        for variant in dict.fromkeys(c.variant for c in CASES):
            ratios = [(max(_RESULTS[c.id]["errs"]) / c.norm / _RESULTS[c.id]["st"]["err_estimate"], c.id)
                      for c in CASES if c.variant == variant and _RESULTS[c.id]["st"]["err_estimate"] > FLOOR]
            print(f"  {variant:16s} {max(ratios)[0]:.3f} ({max(ratios)[1]})" if ratios else f"  {variant:16s} -")
