"""The master equation under a drive whose phase moves, on the Taylor propagator (``LindbladPlan``, ``integrator = 3``):
``stage_d2_taylor_kernel<..., CPLX = true, DISS = true>`` (NS = 1 and NS = 4) and ``stage_d2_taylor_small_kernel<true,
true>``, with the steps of one other phase (``rot``) on the constant-phase DISS kernels and a table that conjugates on
the column bits.  Checked against an exact piecewise-cubic evolution under the sparse Liouvillian (held to the
propagator's own ``err_estimate``), the product of single-qubit master equations, the dense-Lindblad oracle, separate
runs of a SPAM batch, the splitting path, and through ``B200Emulator`` / ``B200Backend`` on Pulser sequences with phase
changes.
"""
from __future__ import annotations

import re

import numpy as np
import pytest

import open_ref as R
from helpers import curved_spec, with_dmm
from phase_sequences import KINDS, moving_phase_rows, phase_sequence
from pulser_b200 import HAVE_PULSER
from pulser_b200 import workloads as W
from test_gpu_taylor_lindblad import PiecewiseCubicLiouvillian

pytestmark = pytest.mark.gpu

STEP_RE = re.compile(r"taylor step t=\S+ h_ns=\S+ p_om=(\d+) .* drive=(\w+)")
EIG = ["r", "g"]


def _ops(scale: float = 1.0) -> np.ndarray:
    """dephasing + relaxation"""
    return scale * np.concatenate([np.sqrt(2 * 3.0) * np.diag([1.0, 0.0])[None], R.relaxation(EIG, 4.0)[None]])


def _fro(x) -> float:
    return float(np.linalg.norm(np.asarray(x).reshape(-1)))


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


def _lindblad(specs, rho0, t0=0.0, t1=None, **opts):
    from pulser_b200.lindblad import LindbladPlan

    with LindbladPlan(specs) as lp:
        if np.asarray(rho0).ndim == 3:
            lp.plan.set_state(np.ascontiguousarray(rho0).reshape(len(rho0), -1))
        else:
            lp.set_state(rho0)
        st = lp.propagate(t0, lp.specs[0].sampling_times[-1] if t1 is None else t1, **opts)
        return lp.get_rho(), st


# ---------------------------------------------------------------- inputs
def _phase_steps(T: int, edges, phases) -> np.ndarray:
    t = np.arange(T)
    return np.asarray(phases, dtype=float)[np.searchsorted(np.asarray(edges), t, side="right")]


def _jump(n: int, T: int = 160):
    """rise, sweep, fall; phase 0, then pi/2 under full amplitude from T/2 on (the largest sample lies before it, so
    the second half runs rotated)"""
    amp, det = W.blockade_sweep_waveforms(t_rise=T // 4, t_sweep=T // 2, t_fall=T // 4)
    ph = _phase_steps(len(amp), [T // 2], [0.0, np.pi / 2])
    return W.ising_global_spec(W.disc_register(n, 14.0, 6.0, n), W.C6_LEVEL_60, amp, det, phase=ph)


def _ramp(n: int, T: int = 160):
    """Blackman / sin^2 with a linear phase ramp over the whole sequence: every step complex"""
    return curved_spec(n, T=T, phase=0.2 + 1.5 * np.arange(T) / T, seed=n, swing=4.0)


def _ramsey(n: int, phi: float = 1.1):
    """pi/2 (40 ns) at phase 0, 80 ns of free evolution, pi/2 at phase phi"""
    T = 160
    t = np.arange(T)
    amp = np.where((t < 40) | (t >= 120), np.pi / 0.08, 0.0)
    det = np.full(T, -2.0)
    ph = _phase_steps(T, [80], [0.0, phi])
    return W.ising_global_spec(W.disc_register(n, 14.0, 6.0, n), W.C6_LEVEL_60, amp, det, phase=ph)


SEQS = {"jump": _jump, "ramp": _ramp, "ramsey": _ramsey}
# windows (us) around what moves: the jump at 80 ns from where the splines still ring at the plan's phase (real steps)
# to where they ring at the new one (complex steps), 60 ns of the ramp, the Ramsey pair's second pulse and its edge
WINDOWS = {"jump": (0.030, 0.100), "ramp": (0.050, 0.110), "ramsey": (0.110, 0.135)}


def _spec(kind: str, variant: str):
    n = {"small": 4, "tiled": 7, "dmm": 7}[variant]
    spec = SEQS[kind](n)
    if variant == "dmm":
        spec = with_dmm(spec, 2, seed=3)
    spec.collapse_ops = _ops(0.5)
    return spec


CASES = [(k, v) for v in ("small", "tiled", "dmm") for k in SEQS]
_RESULTS: dict = {}


def _run_case(kind, variant, capfd, monkeypatch):
    key = (kind, variant)
    if key in _RESULTS:
        return _RESULTS[key]
    spec = _spec(kind, variant)
    assert (spec.drives[0].coef == spec.drives[0].coef[:1]).all()
    n = spec.n_qudits
    rho0 = R.random_density(2**n, 3, n)
    a, b = WINDOWS[kind]
    monkeypatch.setenv("PB200_TAYLOR_LOG", "1")
    capfd.readouterr()
    rho, st = _lindblad(spec, rho0, a, b, integrator=3, tol=1e-11)
    kinds = [m[2] for m in STEP_RE.finditer(capfd.readouterr().err)]
    ref = PiecewiseCubicLiouvillian(spec).evolve(rho0.reshape(-1), a, b).reshape(2**n, 2**n)
    _RESULTS[key] = {"st": st, "kinds": kinds, "err": _fro(rho[0] - ref), "scale": _fro(rho0)}
    return _RESULTS[key]


@pytest.mark.parametrize("kind,variant", CASES, ids=[f"{v}-{k}" for k, v in CASES])
def test_own_error_bound(engine, kind, variant, capfd, monkeypatch):
    r = _run_case(kind, variant, capfd, monkeypatch)
    st = r["st"]
    print(f"\n[bound] {variant} {kind}: |d| = {r['err']:.2e}, err_estimate = {st['err_estimate']:.2e}, "
          f"steps {st['n_steps']} ({', '.join(sorted(set(r['kinds'])))})")
    assert st["integrator"] == 3
    assert len(r["kinds"]) == st["n_steps"] > 0
    assert st["err_estimate"] <= 1e-10
    assert r["err"] <= 2.0 * st["err_estimate"] + 1e-14 * r["scale"]


def test_step_log_reach(engine, capfd, monkeypatch):
    """the cases run every drive kind: real (the plan's phase), rot (one other phase) and cplx (a moving phase); each
    kernel runs rot and cplx steps (which phase is the plan's follows the largest drive sample, so a detuning map's
    jump case may keep its real steps outside the window)"""
    for kind, variant in CASES:
        _run_case(kind, variant, capfd, monkeypatch)
    for variant in ("small", "tiled", "dmm"):
        kinds = {k for (kd, v), r in _RESULTS.items() if v == variant for k in r["kinds"]}
        assert {"rot", "cplx"} <= kinds, (variant, kinds)
    assert {k for r in _RESULTS.values() for k in r["kinds"]} == {"real", "rot", "cplx"}
    assert set(_RESULTS[("ramp", "tiled")]["kinds"]) == {"cplx"}


# ---------------------------------------------------------------- product reference
@pytest.mark.parametrize("n", [4, 10, 12])
def test_driven_product_moving_phase(engine, n):
    """a non-interacting register under a global drive whose phase ramps: the product of single-qubit master
    equations"""
    ops = _ops()
    spec = _ramp(n, T=40)
    spec.interaction_matrix = np.zeros_like(spec.interaction_matrix)
    spec.collapse_ops = ops
    T = spec.sampling_times[-1]
    rho_k0 = [R.random_density(2, 2, 20 + k) for k in range(n)]
    ref = R.kron_all(R.product_lindblad(spec, ops, rho_k0, T))
    rho, st = _lindblad(spec, R.kron_all(rho_k0), integrator=3, tol=1e-10)
    err = float(np.max(np.abs(rho[0] - ref)))
    print(f"\n[product] N={n}: max |rho - ref| = {err:.2e}, steps {st['n_steps']}, applies {st['n_applies']}")
    assert st["integrator"] == 3
    assert err < 1e-10


# ---------------------------------------------------------------- oracle
@pytest.mark.parametrize("n", [2, 3, 4, 5])
@pytest.mark.parametrize("kind", ["jump", "ramsey"])
def test_interacting_against_mesolve(engine, kind, n):
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    spec = SEQS[kind](n)
    spec.collapse_ops = _ops(0.3)
    tf = spec.sampling_times[-1]
    psi0 = evolve.all_ground_state(spec)
    ref = evolve.mesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf], rtol=1e-12, atol=1e-14)[-1]
    for integrator in (0, 3):
        rho, st = _lindblad(spec, np.outer(psi0, psi0.conj()), tol=1e-10, integrator=integrator)
        err = float(np.max(np.abs(rho[0] - ref)))
        print(f"\n[mesolve] N={n} {kind} integrator={integrator}->{st['integrator']}: max |rho - ref| = {err:.2e}")
        assert st["integrator"] == 3 and err < 1e-8


# ---------------------------------------------------------------- SPAM batch
def test_spam_batch_against_separate_runs(engine):
    """per-trajectory factors (bad atoms: a = 0) under a moving phase"""
    n = 8
    specs = []
    for bad in ([], [1], [2, 5]):
        s = _jump(n)
        s.collapse_ops = _ops(0.1)
        s.bad_atoms = np.isin(np.arange(n), bad)
        for d in s.drives:
            d.coef[list(bad)] = 0.0
            d.det[list(bad)] = 0.0
            d.uniform = not bad
        specs.append(s)
    rho0 = R.random_density(2**n, 2, 1)
    batch, st = _lindblad(specs, rho0, integrator=3, tol=1e-10)
    assert st["integrator"] == 3
    for b, s in enumerate(specs):
        one, _ = _lindblad(s, rho0, integrator=3, tol=1e-10)
        err = float(np.max(np.abs(batch[b] - one[0])))
        print(f"\n[spam] trajectory {b}: max |batch - single| = {err:.2e}")
        assert err < 1e-10


# ---------------------------------------------------------------- the splitting path
def test_taylor_against_splitting_n12(engine):
    """N = 12, a phase jump of pi/2 mid-sweep: Taylor against Chebyshev splitting"""
    n = 12
    amp, det = W.blockade_sweep_waveforms(t_rise=50, t_sweep=100, t_fall=50)
    ph = _phase_steps(len(amp), [100], [0.0, np.pi / 2])
    spec = W.ising_global_spec(W.disc_register(n, 16.0, 5.0, 3), W.C6_LEVEL_60, amp, det, phase=ph)
    spec.collapse_ops = np.concatenate([np.sqrt(2 * 0.05) * np.diag([1.0, 0.0])[None], R.relaxation(EIG, 0.01)[None]])
    psi0 = np.zeros(2**n, dtype=complex)
    psi0[-1] = 1.0
    rho_t, st_t = _lindblad(spec, psi0, tol=1e-10)
    rho_s, st_s = _lindblad(spec, psi0, integrator=1, tol=1e-10)
    err = float(np.max(np.abs(rho_t[0] - rho_s[0])))
    print(f"\n[split] N={n} phase jump: max |taylor - splitting| = {err:.2e}; integrator {st_t['integrator']}: "
          f"{st_t['gpu_ms']:.0f} ms, {st_t['n_applies']} applies; integrator {st_s['integrator']}: "
          f"{st_s['gpu_ms']:.0f} ms, {st_s['n_applies']} applies")
    assert st_t["integrator"] == 3 and st_s["integrator"] == 1
    assert err < 1e-8


# ---------------------------------------------------------------- the facade
def _oracle_rho(spec):
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    psi0 = evolve.all_ground_state(spec)
    return evolve.mesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, spec.sampling_times[-1]], rtol=1e-12,
                          atol=1e-14)[-1]


@pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable")
@pytest.mark.parametrize("kind", KINDS)
def test_emulator_noisy_phase_sequences(engine, kind):
    """B200Emulator with a dephasing + relaxation noise model: the auto rule takes the Taylor propagator for the two
    smooth sequences (the EOM block's square pulses may be too rough for it: then Taylor is forced on the same spec)"""
    from pulser.noise_model import NoiseModel
    from pulser_b200 import B200Emulator

    emu = B200Emulator.from_sequence(phase_sequence(kind, n=3), evaluation_times="Minimal",
                                     noise_model=NoiseModel(dephasing_rate=0.5, relaxation_rate=0.2))
    res = emu.run()
    spec = emu._current_spec
    assert len(spec.collapse_ops) > 0 and moving_phase_rows(spec)
    ref = _oracle_rho(spec)
    calls = len(emu._eval_times_array) - 1
    print(f"\n[emulator] {kind}: stats {emu.last_run_stats}")
    if kind != "eom":
        assert emu.last_run_stats["integrator"] == 3 * calls
    got = np.asarray(res.get_final_state().full())
    assert float(np.max(np.abs(got - ref))) < 1e-8
    psi0 = np.zeros(spec.dim**spec.n_qudits, dtype=complex)
    psi0[-1] = 1.0   # all ground (g is the last digit)
    rho, st = _lindblad(spec, psi0, integrator=3)
    assert st["integrator"] == 3
    assert float(np.max(np.abs(rho[0] - ref))) < 1e-8


@pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable")
@pytest.mark.parametrize("kind", ["phases", "phase_shift"])
def test_backend_streams_noisy_phase_sequences(engine, kind, monkeypatch):
    """B200Backend keeps the density matrix on the device (DeviceDensityView: no host copy of rho) and every call
    runs the Taylor propagator"""
    import pulser
    from pulser.backend.default_observables import Occupation
    from pulser_b200 import B200Backend, B200Config, lindblad

    fetched, integrators = [], []
    get_rho, propagate = lindblad.LindbladPlan.get_rho, lindblad.LindbladPlan.propagate
    monkeypatch.setattr(lindblad.LindbladPlan, "get_rho", lambda self: (fetched.append(1), get_rho(self))[1])

    def recording(self, *args, **opts):
        st = propagate(self, *args, **opts)
        integrators.append(st["integrator"])
        return st

    monkeypatch.setattr(lindblad.LindbladPlan, "propagate", recording)
    cfg = B200Config(observables=[Occupation(evaluation_times=[0.5, 1.0])],
                     noise_model=pulser.NoiseModel(dephasing_rate=0.5, relaxation_rate=0.2))
    be = B200Backend(phase_sequence(kind, n=3), config=cfg)
    assert be._streams_density()
    res = be.run()
    print(f"\n[backend] {kind}: integrators {integrators}")
    assert fetched == []
    assert integrators and set(integrators) == {3}
    spec = be._sim_obj._current_spec
    rho = _oracle_rho(spec)
    n = spec.n_qudits
    nr = [R.kron_all([np.diag([1.0, 0.0]) if j == k else np.eye(2) for j in range(n)]) for k in range(n)]
    occ_ref = np.array([np.real(np.trace(rho @ m)) for m in nr])
    occ = np.asarray(res.get_result("occupation", 1.0), dtype=float)
    assert np.max(np.abs(occ - occ_ref)) < 1e-8
