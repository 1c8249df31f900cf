"""Magnus step controller (integrator = 1 / 2) under the options the default
runs leave alone, each held to the DOP853 oracle:

- plain step doubling (``extrapolate = -1``) on Chebyshev and on Lanczos;
- second-order Magnus steps, with and without Richardson extrapolation;
- a non-default check interval, refinement window and roughness threshold;
- a fixed Chebyshev truncation tolerance;
- runs cut into several calls at off-grid times, where each call inherits the
  step length the previous one ended with.

A call inherits that step length only when its options are those of the call
before; the last tests pin that the options are compared exactly.
"""
import numpy as np
import pytest

from pulser_b200 import workloads as W

pytestmark = pytest.mark.gpu

STATE_TOL = 1e-8
CUTS = (0.0, 0.0371, 0.2093, 0.3514)   # off the 1 ns sampling grid


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


@pytest.fixture(scope="module")
def sweep():
    """An 8-atom blockade sweep of 500 ns and its oracle final state."""
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    spec = W.config_c2(n=8, seed=20, t_rise=100, t_sweep=300, t_fall=100)
    psi0 = evolve.all_ground_state(spec)
    tf = spec.sampling_times[-1]
    ref = evolve.sesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf], rtol=1e-13, atol=1e-15)[-1]
    return spec, ref


def _run(engine, spec, cuts=(0.0,), **opts):
    """Final state of a run from the ground state, one call per [cuts[i], cuts[i + 1]], and each call's stats."""
    bounds = list(cuts) + [spec.sampling_times[-1]]
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        stats = [plan.propagate(a, b, **opts) for a, b in zip(bounds[:-1], bounds[1:])]
        return plan.get_state()[0], stats


def _err(got, ref):
    return float(np.max(np.abs(got - ref)))


@pytest.mark.parametrize("integrator", [1, 2])
def test_plain_step_doubling(engine, sweep, integrator):
    """extrapolate = -1: CF4 steps checked by one step of h against two of h/2."""
    spec, ref = sweep
    got, (st,) = _run(engine, spec, extrapolate=-1, tol=1e-9, integrator=integrator)
    assert st["integrator"] == integrator and st["n_checks"] > 0
    assert _err(got, ref) < STATE_TOL, _err(got, ref)


@pytest.mark.parametrize("extrapolate", [0, -1])
def test_second_order_magnus(engine, sweep, extrapolate):
    """magnus_order = 2: the midpoint exponential; extrapolated it is a 4th-order scheme."""
    spec, ref = sweep
    tol = 1e-9 if extrapolate == 0 else 1e-7
    got, (st,) = _run(engine, spec, magnus_order=2, extrapolate=extrapolate, tol=tol, integrator=1)
    assert st["n_checks"] > 0
    assert _err(got, ref) < 10 * tol, _err(got, ref)


def test_check_every_refine_window_rough_tol(engine, sweep):
    spec, ref = sweep
    got, (st,) = _run(engine, spec, check_every=4, refine_window=3, rough_tol=1e-3, integrator=1)
    _, (st_default,) = _run(engine, spec, integrator=1)
    assert st["n_checks"] > st_default["n_checks"]
    assert _err(got, ref) < STATE_TOL, _err(got, ref)


def test_user_cheb_tol(engine, sweep):
    """A fixed Chebyshev truncation tolerance replaces the per-step share of the budget."""
    spec, ref = sweep
    got, (st,) = _run(engine, spec, cheb_tol=1e-14, integrator=1)
    _, (st_loose,) = _run(engine, spec, cheb_tol=1e-10, integrator=1)
    assert st["n_applies"] > st_loose["n_applies"]
    assert _err(got, ref) < STATE_TOL, _err(got, ref)


@pytest.mark.parametrize("integrator", [1, 2])
def test_cut_run_equals_whole(engine, sweep, integrator):
    """A run cut at off-grid times (evaluation times) equals the whole run."""
    spec, ref = sweep
    whole, _ = _run(engine, spec, integrator=integrator)
    pieces, stats = _run(engine, spec, CUTS, integrator=integrator)
    assert all(s["integrator"] == integrator for s in stats)
    assert _err(pieces, whole) < STATE_TOL, _err(pieces, whole)
    assert _err(pieces, ref) < STATE_TOL, _err(pieces, ref)


# (options of the first call, options of the second, start of the first call).  The second pair differs in tol and
# extrapolate only, and 1e-17 * 1e3 + 1 + 2 * 4 + 16 * 32 == 1e-3 * 1e3 + 0 + 2 * 4 + 16 * 32 in double precision: a
# key that sums the options cannot tell these calls apart.  The tight first call ends on a short step, which the loose
# second call must not start from.
OPTION_CHANGES = [
    (dict(tol=1e-8), dict(tol=1e-9), 0.0),
    (dict(tol=1e-17, max_step=32), dict(tol=1e-3, extrapolate=-1, max_step=32), 0.4602),
]


@pytest.mark.parametrize("first,second,t0", OPTION_CHANGES, ids=["tol", "tol-extrapolate"])
def test_changed_options_start_afresh(engine, sweep, first, second, t0):
    """A call whose options differ from the previous call's, continuing where that call stopped, runs exactly as the
    same call on a fresh plan from the same state."""
    spec, _ = sweep
    t1, t2 = 0.4811, 0.4995
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        plan.propagate(t0, t1, integrator=1, **first)
        mid = plan.get_state()[0]
        plan.propagate(t1, t2, integrator=1, **second)
        continued = plan.get_state()[0]
    with engine.DevicePlan(spec) as plan:
        plan.set_state(mid)
        plan.propagate(t1, t2, integrator=1, **second)
        fresh = plan.get_state()[0]
    assert _err(continued, fresh) < 1e-12, _err(continued, fresh)
