"""Every stage kernel of the Magnus propagator (integrators 1 and 2: Chebyshev-Clenshaw and Lanczos exponentials)
against the exact references of tests/magnus_ref.py, held to a bound taken from the run's own stats:

    ||psi_dev - psi_ref||_2 <= A * (n_exponentials * cheb_tol + C * eps * n_applies) + FLOOR      (every trajectory)

With H constant in time every Magnus scheme is exact, so only the exponentials' truncation (Chebyshev degree or Lanczos
stop, both set by ``cheb_tol``) and rounding remain, whatever steps the controller takes.  Every bound comes out below
1e-10, at least 100x tighter than the 1e-8 of the whole-sequence tests.  At N = 27 / 28 the error norm is estimated from
4000 random amplitudes, and the device norm and the largest error of the probed amplitudes (all-ground, all-Rydberg, the
indices that set the bits of each pass, the random ones) are held to the bound too.  That estimate is statistical: a
defect confined to a few thousand amplitudes that no probe hits would escape it, which the full-vector cases up to
N = 20 and the per-kernel signatures below are there to catch.

Each case also asserts what its stats show about the kernel it ran: dual-chain launches (fewer launches than applies),
one launch per Lanczos iteration (fused) or more (unfused), one or two launches per stage (one-pass / two-pass
geometries), and on the forwarding kernel one logged forwarding stage per H-apply (``PB200_MAGNUS_LOG``).

Lanczos at N = 28 is left out: its basis needs at least 11 state vectors (47 GB) there.  The unfused Lanczos iteration
runs at N = 9 instead.

The last tests compare partner-sum forwarding (stage_d2_fwd_kernel, one state of uniform drives at 17 <= N <= 19)
with the table path on sequences whose drive phase goes 0 -> phi -> 0 -> phi: a complex stage must not read forwarded
sums that a real stage produced (the real kernel writes only their first plane).  The stage log shows that the runs
reach that hand-off from a real to a complex stage.
"""
from __future__ import annotations

import dataclasses
import functools
import os
import re
import time
from typing import Callable

import numpy as np
import pytest

from helpers import random_state
from magnus_ref import (ClusterReference, cluster_couplings, constant_spec, dense_evolve, interleaved_clusters,
                        probe_indices)
from pulser_b200 import workloads as W

pytestmark = pytest.mark.gpu

CHEB_TOL = 1e-14
EPS = np.finfo(float).eps
# Measured on an H100 80GB HBM3 (700 W): err / (eps * n_applies) reaches 3.9 (multilevel_d4_n4_order2), hence C = 4;
# err / (n_exponentials * cheb_tol + C * eps * n_applies) then reaches 0.54 (same case), 0.22 elsewhere, so that
# err / bound stays below 0.27.  test_reach_and_ratios prints both ratios per case.
A = 2.0
C = 4.0
FLOOR = 1e-15
MAX_BOUND = 1e-10
FULL_MAX_N = 22          # above: sampled amplitudes


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


# ---------------------------------------------------------------- inputs
def _dt_ns(coef, det, U, rho_per_sample):
    """sampling interval that gives each sample about ``rho_per_sample`` of spectral half-width"""
    w = 0.5 * (np.triu(U, 1).sum() + np.abs(det).sum()) + np.abs(coef).sum()
    return max(1, int(round(rho_per_sample / (w * 1e-3))))


@functools.lru_cache(maxsize=None)
def _ising(n: int, kind: str, seed: int = 0, n_clusters: int = 0, shift: int = 0, n_samples: int = 20,
           rho_per_sample: float = 0.5):
    """d = 2 register of interleaved clusters; kind: real / complex (uniform drive, phase 0 / 0.83) or local (complex
    per-atom drive and detuning)"""
    clusters = interleaved_clusters(n, n_clusters or None, shift)
    rng = np.random.default_rng(1000 * n + seed)
    U = cluster_couplings(n, clusters, seed=rng.integers(1 << 30))
    if kind == "local":
        coef = rng.uniform(1.5, 4.0, n) * np.exp(1j * rng.uniform(-np.pi, np.pi, n))
        det = rng.uniform(-8.0, 4.0, n)
    else:
        coef = np.full(n, 3.0 * np.exp(-0.83j if kind == "complex" else 0.0))
        det = np.full(n, -4.0)
    dt = _dt_ns(coef, det, U, rho_per_sample)
    spec = constant_spec([("ground-rydberg", coef, det)], U, n_samples=n_samples, dt_ns=dt)
    return spec, clusters


@functools.lru_cache(maxsize=None)
def _dense(kind: str, n: int, seed: int = 0, n_samples: int = 20, rho_per_sample: float = 0.5):
    """d = 3 (one drive), d = 4 (two drives, a leakage level no drive touches) or XY registers with dense couplings"""
    rng = np.random.default_rng(2000 * n + seed)
    U = rng.uniform(0.2, 2.0, (n, n))
    U = np.triu(U, 1) + np.triu(U, 1).T
    c = lambda s: s * rng.uniform(1.0, 3.0, n) * np.exp(1j * rng.uniform(-np.pi, np.pi, n))   # noqa: E731
    d = lambda: rng.uniform(-5.0, 5.0, n)                                                      # noqa: E731
    if kind == "d3":
        drives, kw = [("ground-rydberg", c(1), d())], dict(dim=3)
    elif kind == "d4":
        drives, kw = [("ground-rydberg", c(1), d()), ("digital", c(0.7), d())], dict(dim=4)
    else:
        Uxy = rng.uniform(-3.0, 3.0, (n, n))
        Uxy = np.triu(Uxy, 1) + np.triu(Uxy, 1).T
        drives, kw = [("XY", c(1), d())], dict(interaction_type="XY")
        U = np.stack([Uxy, U])
    w = sum(np.abs(x[1]).sum() + 0.5 * np.abs(x[2]).sum() for x in drives) + 0.5 * np.abs(U).sum()
    return constant_spec(drives, U, n_samples=n_samples, dt_ns=max(1, int(round(rho_per_sample / (w * 1e-3)))), **kw)


def _batch(n: int, n_clusters=(2, 3, 4), kind: str = "local"):
    """trajectories that differ in drive and in how the couplings split into clusters (per-trajectory Dint)"""
    out = [_ising(n, kind, seed=b, n_clusters=c, shift=b) for b, c in enumerate(n_clusters)]
    first = out[0][0]   # one time grid for the batch
    return [(dataclasses.replace(s, sampling_times=first.sampling_times, total_duration_ns=first.total_duration_ns), c)
            for s, c in out]


@dataclasses.dataclass(frozen=True)
class Case:
    id: str
    variant: str
    build: Callable               # () -> [(spec, clusters or None)]
    opts: dict
    cuts: tuple = ()              # call boundaries inside (0, T), as fractions of T
    ground: bool = False          # all-ground initial state (the N >= 27 registers)
    dual: bool = False            # extrapolated steps sharing launches: n_launches < n_applies
    lanczos_fused: bool | None = None
    per_apply: int = 0            # fixed steps without extrapolation: exactly this many launches per H-apply


FIXED = dict(tol=-1.0, max_step=16)
SINGLE = dict(tol=-1.0, max_step=16, extrapolate=-1)
CUTS = (0.2373, 0.5519, 0.8061)

CASES = [
    # stage_d2_kernel (N < 11): one chain per launch
    Case("d2_real_n6", "stage_d2", lambda: [_ising(6, "real")], dict(integrator=1)),
    Case("d2_complex_n8_fixed", "stage_d2", lambda: [_ising(8, "complex")], dict(integrator=1, **FIXED)),
    Case("d2_table_n9_nocheck", "stage_d2", lambda: [_ising(9, "local")], dict(integrator=1, extrapolate=-1)),
    Case("d2_table_n9_order2", "stage_d2", lambda: [_ising(9, "local", seed=1)],
         dict(integrator=1, magnus_order=2, tol=1e-9)),
    Case("d2_batch_n6", "stage_d2", lambda: _batch(6, (1, 2, 3)), dict(integrator=1)),
    # stage_d2_rb_kernel, one pass
    Case("rb_real_n11", "stage_d2_rb", lambda: [_ising(11, "real")], dict(integrator=1), dual=True),
    Case("rb_complex_n14_substeps", "stage_d2_rb", lambda: [_ising(14, "complex", n_samples=4, rho_per_sample=6.0)],
         dict(integrator=1), cuts=CUTS, dual=True),
    Case("rb_table_n14_order2", "stage_d2_rb", lambda: [_ising(14, "local")],
         dict(integrator=1, magnus_order=2, extrapolate=-1, tol=1e-9)),
    Case("rb_real_n20_fixed", "stage_d2_rb", lambda: [_ising(20, "real")], dict(integrator=1, **FIXED), dual=True),
    Case("rb_table_n20_cuts", "stage_d2_rb", lambda: [_ising(20, "local")], dict(integrator=1), cuts=CUTS, dual=True),
    Case("rb_table_n27", "stage_d2_rb", lambda: [_ising(27, "local", n_samples=12)], dict(integrator=1, **SINGLE),
         ground=True, per_apply=1),
    # stage_d2_rb_kernel, two passes
    Case("rb2_table_n28", "stage_d2_rb_2pass", lambda: [_ising(28, "local", n_samples=12)],
         dict(integrator=1, **SINGLE), ground=True, per_apply=2),
    Case("rb2_complex_n28_order2", "stage_d2_rb_2pass", lambda: [_ising(28, "complex", n_samples=12)],
         dict(integrator=1, magnus_order=2, **SINGLE), ground=True, per_apply=2),
    # stage_d2_fwd_kernel: one state of uniform drives, 17 <= N <= 19
    Case("fwd_real_n17_single", "stage_d2_fwd", lambda: [_ising(17, "real")],
         dict(integrator=1, **SINGLE), per_apply=1),
    Case("fwd_complex_n18_dual", "stage_d2_fwd", lambda: [_ising(18, "complex")],
         dict(integrator=1), cuts=CUTS, dual=True),
    Case("fwd_real_n19_dual_fixed", "stage_d2_fwd", lambda: [_ising(19, "real")],
         dict(integrator=1, **FIXED), dual=True),
    Case("fwd_complex_n19_order2", "stage_d2_fwd", lambda: [_ising(19, "complex")],
         dict(integrator=1, magnus_order=2, **SINGLE), per_apply=1),
    # table path of a batch with per-trajectory Dint
    Case("batch_dint_n14", "stage_d2_rb_batch", lambda: _batch(14), dict(integrator=1), dual=True),
    Case("batch_dint_n14_order2", "stage_d2_rb_batch", lambda: _batch(14, (3, 2, 4)),
         dict(integrator=1, magnus_order=2, **SINGLE), per_apply=1),
    # Lanczos: one launch per iteration on the one-pass register-blocked and the tiled multilevel kernels
    Case("lanczos_fused_real_n12", "lanczos_fused", lambda: [_ising(12, "real")], dict(integrator=2),
         lanczos_fused=True),
    Case("lanczos_fused_table_n20", "lanczos_fused", lambda: [_ising(20, "local")], dict(integrator=2),
         lanczos_fused=True),
    Case("lanczos_fused_d3_n6", "lanczos_fused", lambda: [(_dense("d3", 6), None)], dict(integrator=2),
         lanczos_fused=True),
    Case("lanczos_fused_d4_n4", "lanczos_fused", lambda: [(_dense("d4", 4), None)], dict(integrator=2),
         lanczos_fused=True),
    Case("lanczos_unfused_n9", "lanczos_unfused", lambda: [_ising(9, "local")], dict(integrator=2),
         lanczos_fused=False),
    Case("lanczos_unfused_n9_fixed", "lanczos_unfused", lambda: [_ising(9, "complex")],
         dict(integrator=2, **SINGLE), lanczos_fused=False),
    # stage_multilevel_rb_kernel (Chebyshev)
    Case("multilevel_d3_n6", "stage_multilevel", lambda: [(_dense("d3", 6, seed=1), None)], dict(integrator=1)),
    Case("multilevel_d4_n4_order2", "stage_multilevel", lambda: [(_dense("d4", 4, seed=1), None)],
         dict(integrator=1, magnus_order=2, **FIXED)),
    Case("multilevel_d3_n5_substeps", "stage_multilevel",
         lambda: [(_dense("d3", 5, n_samples=4, rho_per_sample=6.0), None)], dict(integrator=1), cuts=CUTS),
    # stage_generic_kernel: XY
    Case("generic_xy_n6", "stage_generic", lambda: [(_dense("xy", 6), None)], dict(integrator=1)),
    Case("generic_xy_n7_order2", "stage_generic", lambda: [(_dense("xy", 7), None)],
         dict(integrator=1, magnus_order=2, extrapolate=-1, tol=1e-9)),
    Case("generic_xy_n9_lanczos", "stage_generic", lambda: [(_dense("xy", 9), None)], dict(integrator=2), cuts=CUTS),
    Case("generic_xy_n8_fixed", "stage_generic", lambda: [(_dense("xy", 8), None)], dict(integrator=1, **SINGLE),
         per_apply=1),
]


# ---------------------------------------------------------------- running a case
_RESULTS: dict = {}
FWD_RE = re.compile(r"magnus fwd stage chain=(\d+) exp_real=(\d) launch_real=(\d) role=(\d)")


def _fwd_stages(err: str):
    """the logged forwarding stages, (chain, exponential real, launch real, role) each, one list per run_chains call"""
    calls = []
    for line in err.splitlines():
        if line.startswith("magnus fwd chains="):
            calls.append([])
        elif (m := FWD_RE.match(line)):
            calls[-1].append(tuple(int(x) for x in m.groups()))
    return calls


def _handoffs(calls):
    """(complex stages that follow a real stage of their chain, those of them that read forwarded sums)"""
    after_real = reads = 0
    for stages in calls:
        prev = {}
        for chain, _, real, role in stages:
            if not real and prev.get(chain) == 1:
                after_real += 1
                reads += role > 0
            prev[chain] = real
    return after_real, reads


def _logged(capfd, fn):
    """fn() with the forwarding stage log on; returns (fn(), the logged stages)"""
    capfd.readouterr()
    os.environ["PB200_MAGNUS_LOG"] = "1"
    try:
        out = fn()
    finally:
        del os.environ["PB200_MAGNUS_LOG"]
    return out, _fwd_stages(capfd.readouterr().err)


def _initial(spec, clusters, b, ground):
    if clusters is None:
        return None, random_state(spec.hilbert_dim, 40 + b)
    ref = ClusterReference(spec, clusters)
    parts = ref.ground() if ground else ref.initial(40 + b)
    return (ref, parts), (None if ground else ref.full(parts))


def _krylov_launches(st, per_apply):
    """launches of a default (adaptive, extrapolated) Lanczos run: per exponential dot2 + normalize_copy +
    krylov_combine, `per_apply` per iteration, one Richardson axpby per step, three per check"""
    return (3 * st["n_exponentials"] + per_apply * st["n_applies"] + st["n_steps"] + st["n_rejected"]
            + 3 * st["n_checks"])


def _run(case, engine, capfd, det_scale: float = 1.0):
    key = (case.id, det_scale)
    if key in _RESULTS:
        return _RESULTS[key]
    built = case.build()
    specs = [s for s, _ in built]
    T = float(specs[0].sampling_times[-1])
    inits = [_initial(s, c, b, case.ground) for b, (s, c) in enumerate(built)]

    def run():
        with engine.DevicePlan(specs) as plan:
            if case.ground:
                plan.set_state("all-ground")
            else:
                plan.set_state(np.stack([v for _, v in inits]))
            bounds = [0.0] + [f * T for f in case.cuts] + [T]
            calls = [plan.propagate(a, b, cheb_tol=CHEB_TOL, **case.opts) for a, b in zip(bounds[:-1], bounds[1:])]
            return calls, np.sqrt(plan.norm2()), plan.get_state()

    t0 = time.perf_counter()
    (calls, norms, got), fwd = _logged(capfd, run)
    wall = time.perf_counter() - t0
    st = {k: sum(c[k] for c in calls) for k in ("n_steps", "n_exponentials", "n_applies", "n_launches", "n_checks",
                                                  "n_rejected")}
    st["max_rho"] = max(c["max_rho"] for c in calls)
    st["min_step_samples"] = min(c["mean_step_samples"] for c in calls)
    errs = []
    for b, ((spec, clusters), (cl, v0)) in enumerate(zip(built, inits)):
        if det_scale != 1.0:   # the self-check: a reference whose detuning is off by a relative det_scale - 1
            drives = [dataclasses.replace(d, det=d.det * det_scale) for d in spec.drives]
            spec = dataclasses.replace(spec, drives=drives)
            if cl is not None:
                cl = (ClusterReference(spec, clusters), cl[1])
        if cl is None:
            errs.append(float(np.linalg.norm(got[b] - dense_evolve(spec, v0, T))))
            continue
        ref, parts = cl
        out = ref.evolve(parts, T)
        n = spec.n_qudits
        if n <= FULL_MAX_N:
            errs.append(float(np.linalg.norm(got[b] - ref.full(out))))
        else:
            idx = probe_indices(n, 4000, seed=n)
            d = np.abs(got[b][idx] - ref.amplitudes(out, idx))
            rand = np.random.default_rng(n).integers(0, 1 << n, 4000)
            dr = np.abs(got[b][rand] - ref.amplitudes(out, rand))
            est = float(np.sqrt((1 << n) * np.mean(dr**2)))
            errs.append(max(est, float(d.max()), abs(float(norms[b]) - ref.norm(out))))
    del got
    res = {"calls": calls, "st": st, "errs": errs, "wall": wall, "fwd_stages": sum(len(c) for c in fwd),
           "norm_err": max(abs(float(x) - 1.0) for x in norms)}
    _RESULTS[key] = res
    return res


def _bound(st):
    return A * (st["n_exponentials"] * CHEB_TOL + C * EPS * st["n_applies"]) + FLOOR


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_within_own_error_bound(engine, case, capfd):
    r = _run(case, engine, capfd)
    st = r["st"]
    integ = case.opts["integrator"]
    assert all(c["integrator"] == integ for c in r["calls"])
    assert st["n_applies"] > 0 and st["n_exponentials"] > 0
    bound = _bound(st)
    assert bound <= MAX_BOUND, bound
    for b, e in enumerate(r["errs"]):
        assert e <= bound, (b, e, bound, st)
    assert r["norm_err"] <= bound
    if case.dual:
        assert st["n_launches"] < st["n_applies"], st
    if case.lanczos_fused is True:
        for c in r["calls"]:
            assert c["n_launches"] == _krylov_launches(c, 1), c
    elif case.lanczos_fused is False:
        assert st["n_launches"] >= 3 * st["n_exponentials"] + 2 * st["n_applies"], st
    if case.per_apply:
        assert st["n_launches"] == case.per_apply * st["n_applies"], st
    # the forwarding kernel runs every stage of the stage_d2_fwd cases and no stage elsewhere
    assert r["fwd_stages"] == (st["n_applies"] if case.variant == "stage_d2_fwd" else 0), (r["fwd_stages"], st)


def test_bound_sees_a_relative_detuning_error_of_1e_8(engine, capfd):
    """the same run held to a reference whose detuning is off by a relative 1e-8 fails the bound"""
    case = next(c for c in CASES if c.id == "rb_table_n20_cuts")
    r = _run(case, engine, capfd, det_scale=1.0 + 1e-8)
    assert min(r["errs"]) > _bound(r["st"]), (r["errs"], _bound(r["st"]))


def test_reach_and_ratios(engine, capfd):
    """every kernel reaches a Chebyshev / Lanczos half-width of at least 3 in some case; sub-sample steps occur; the
    table of err / bound and of the rounding ratio err / (eps n_applies) per case"""
    for case in CASES:
        _run(case, engine, capfd)
    with capfd.disabled():
        lines = ["\ncase                              err        bound      err/bound  err/(eps*n_app)  n_exp  n_app  "
                 "max_rho  step   wall_s"]
        for c in CASES:
            r = _RESULTS[(c.id, 1.0)]
            st, e = r["st"], max(r["errs"])
            lines.append(f"{c.id:32s} {e:.3e}  {_bound(st):.3e}  {e / _bound(st):.2e}   "
                         f"{e / (EPS * st['n_applies']):.3e}        {st['n_exponentials']:5d}  {st['n_applies']:5d}  "
                         f"{st['max_rho']:6.2f}  {st['min_step_samples']:5.2f}  {r['wall']:6.2f}")
        print("\n".join(lines))
    for variant in {c.variant for c in CASES}:
        assert max(_RESULTS[(c.id, 1.0)]["st"]["max_rho"] for c in CASES if c.variant == variant) >= 3.0, variant
    assert min(r["st"]["min_step_samples"] for r in _RESULTS.values()) < 1.0


# ---------------------------------------------------------------- phase changes on the forwarding path
def _phase_spec(n: int):
    """global drive whose phase goes 0 -> 0.9 -> 0 -> 0.9 in 40 ns segments, over a detuning ramp"""
    T = 160
    amp = np.full(T, 2 * np.pi * 1.2)
    det = np.linspace(-6.0, 4.0, T)
    phase = np.where((np.arange(T) // 40) % 2 == 1, 0.9, 0.0)
    return W.ising_global_spec(W.disc_register(n, 38.0, 5.0, 3), W.C6_LEVEL_60, amp, det, phase=phase)


PHASE_MODES = {"single": dict(tol=-1.0, max_step=2, extrapolate=-1), "dual": dict(tol=-1.0, max_step=2)}


@pytest.mark.parametrize("n", [17, 19])
@pytest.mark.parametrize("order", [1, 3])
@pytest.mark.parametrize("mode", list(PHASE_MODES))
def test_forwarding_across_phase_changes(engine, n, order, mode, capfd):
    """one state (forwarded partner sums) against the same spec as a batch of two (table path, no forwarding): same
    fixed steps and degrees, states equal to rounding.  The stage log of the forwarding run shows every stage on the
    forwarding kernel and, at linear interpolation (exactly real drive on the phase-0 segments), complex stages that
    follow a real one; none of those may read the forwarded sums"""
    spec = _phase_spec(n)
    tf = spec.sampling_times[-1]
    psi0 = random_state(spec.hilbert_dim, 9)
    out = {}
    for batch in ([spec], [spec, spec]):
        def run():
            with engine.DevicePlan(batch, interp_order=order) as plan:
                plan.set_state(psi0)
                st = plan.propagate(0.0, tf, integrator=1, **PHASE_MODES[mode])
                return plan.get_state().copy(), st
        out[len(batch)], stages = _logged(capfd, run)
        if len(batch) == 1:
            fwd_calls = stages
        else:
            assert stages == []
    fwd, table = out[1][0][0], out[2][0]
    assert out[1][1]["n_applies"] == out[2][1]["n_applies"] == sum(len(c) for c in fwd_calls)
    after_real, reads = _handoffs(fwd_calls)
    err = max(np.max(np.abs(fwd - table[0])), np.max(np.abs(fwd - table[1])))
    assert err < 5e-13 and reads == 0, (err, after_real, reads)
    if order == 1 and mode == "single":   # one chain over the whole call: the phase changes fall inside it
        assert after_real > 0
    if n == 17 and order == 1 and mode == "dual":
        with engine.DevicePlan(spec, interp_order=order) as plan:
            plan.set_state(psi0)
            plan.propagate(0.0, tf, integrator=2, tol=1e-11)
            assert np.max(np.abs(fwd - plan.get_state()[0])) < 1e-8
