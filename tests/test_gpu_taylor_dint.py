"""The tiled Taylor stage forms the interaction diagonal Dint = sum_{i<j} U_ij n_i n_j itself, from per-CTA, per-thread
and per-register-bit factors of the coupling matrix. These cases use random signed couplings between every pair of
atoms (not a van der Waals decay), so that pairs link every class of index bits: thread bits, register bits, the chunk
bit, bits above the tile and shard bits. Each case is held to the propagator's own error bound against the exact
piecewise-cubic reference, the criterion of test_gpu_taylor_exact.py."""
from __future__ import annotations

import dataclasses

import numpy as np
import pytest

from helpers import random_state
from pulser_b200 import workloads as W
from taylor_ref import PiecewiseCubicHamiltonian

pytestmark = pytest.mark.gpu

A = 2.0
FLOOR = 1e-14
TOL = 1e-11


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


def _couplings(n: int, seed: int, scale: float = 3.0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    u = rng.normal(0.0, scale, (n, n))
    u = np.triu(u, 1)
    return u + u.T


def _spec(n: int, seed: int = 0, phase: float = 0.0, moving: bool = False, bad=None):
    amp, det = W.blockade_sweep_waveforms(t_rise=100, t_sweep=300, t_fall=100)
    spec = W.ising_global_spec(W.disc_register(n, 22.0, 6.0, n), W.C6_LEVEL_60, amp, det, phase=phase)
    spec = dataclasses.replace(spec, interaction_matrix=_couplings(n, seed)[None])
    if bad is not None:
        spec = dataclasses.replace(spec, bad_atoms=np.asarray(bad, dtype=bool))
    if moving:   # a drive phase that changes inside every step: the complex-drive (CPLX) stage
        d = spec.drives[0]
        ramp = np.exp(-1j * 2.0 * np.arange(d.coef.shape[1]) / d.coef.shape[1])
        spec.drives[0] = dataclasses.replace(d, coef=np.asarray(d.coef) * ramp[None, :])
    return spec


def _window(spec, i: int = 250):
    t = spec.sampling_times
    return t[i], t[i + 3]


def _check(specs, got, psi0, a, b, st):
    assert st["integrator"] == 3
    assert st["err_estimate"] <= TOL
    bound = A * st["err_estimate"] + FLOOR
    for s, g, p in zip(specs, got, psi0):
        err = float(np.linalg.norm(g - PiecewiseCubicHamiltonian(s).evolve(p, a, b)))
        assert err <= bound * np.linalg.norm(p), (err, st["err_estimate"])


@pytest.mark.parametrize("n", [14, 20])
def test_single_plan(engine, n):
    spec = _spec(n, seed=n)
    a, b = _window(spec)
    psi0 = random_state(spec.hilbert_dim, n)
    with engine.DevicePlan(spec) as plan:
        plan.set_state(psi0)
        st = plan.propagate(a, b, integrator=3, tol=TOL)
        got = plan.get_state()
    _check([spec], got, [psi0], a, b, st)


def test_batch_per_trajectory_couplings(engine):
    n = 14
    rng = np.random.default_rng(5)
    specs = [_spec(n, seed=40 + k, bad=rng.random(n) < 0.2) for k in range(3)]
    a, b = _window(specs[0])
    psi0 = [random_state(specs[0].hilbert_dim, 60 + k) for k in range(3)]
    with engine.DevicePlan(specs) as plan:
        plan.set_state(np.stack(psi0))
        st = plan.propagate(a, b, integrator=3, tol=TOL)
        got = plan.get_state()
    _check(specs, got, psi0, a, b, st)


def test_moving_phase(engine):
    spec = _spec(14, seed=7, moving=True)
    a, b = _window(spec)
    psi0 = random_state(spec.hilbert_dim, 7)
    with engine.DevicePlan(spec) as plan:
        plan.set_state(psi0)
        st = plan.propagate(a, b, integrator=3, tol=TOL)
        got = plan.get_state()
    _check([spec], got, [psi0], a, b, st)


def test_four_shards(engine):
    from pulser_b200 import sharded

    spec = _spec(15, seed=15, phase=0.4)
    a, b = _window(spec)
    psi0 = random_state(spec.hilbert_dim, 15)
    with sharded.ShardedPlan(spec, [0] * 4) as plan:
        plan.set_state(psi0)
        st = plan.propagate(a, b, integrator=3, tol=TOL)
        got = plan.get_state()
    _check([spec], got, [psi0], a, b, st)


def test_master_equation(engine):
    """2N = 14 bits of vec(rho): the stage sees the block coupling matrix diag(U, -U)"""
    import open_ref as R
    from test_gpu_taylor_lindblad import PiecewiseCubicLiouvillian, _lindblad, _ops

    n = 7
    spec = _spec(n, seed=3)
    spec.collapse_ops = _ops("dephasing+relaxation") * 0.5
    a, b = _window(spec, 200)
    rho0 = R.random_density(2**n, 3, n)
    ref = PiecewiseCubicLiouvillian(spec).evolve(rho0.reshape(-1), a, b).reshape(2**n, 2**n)
    rho, st = _lindblad(spec, rho0, a, b, integrator=3, tol=TOL)
    assert st["integrator"] == 3
    err = float(np.linalg.norm((rho[0] - ref).reshape(-1)))
    assert err <= A * st["err_estimate"] + FLOOR * float(np.linalg.norm(rho0.reshape(-1)))
