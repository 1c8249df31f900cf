"""The single-precision tail orders of the Taylor propagator (TaylorStep::k_lo) on C2-shaped sequences, N = 13-16:
ramp and plateau steps and multi-step windows against the exact piecewise-cubic reference (tests/taylor_ref.py),
held to the propagator's own error estimate, which includes the bound on the rounding of the stored tail orders.

The switch order is chosen after the step, its order K and its ring are fixed, so the schedule is the one of the
all-fp64 propagator: the step count, K of every step and the launch count below are those of the commit before the
single-precision orders (H100 80GB HBM3).
"""
from __future__ import annotations

import dataclasses
import functools
import os
import re
import tempfile

import numpy as np
import pytest

from helpers import random_state
from pulser_b200 import workloads as W
from taylor_ref import PiecewiseCubicHamiltonian

pytestmark = pytest.mark.gpu

A = 2.0          # ||error|| / err_estimate allowed: the rounding part of the estimate is not a bound (DESIGN 3a)
FLOOR = 1e-14

STEP_RE = re.compile(r"taylor step .* K=(\d+) ring=.* k_lo=(\d+)")


@functools.lru_cache(maxsize=None)
def c2(n: int):
    """C2-shaped (rise, sweep, fall; 500 ns) on a register spread enough to keep the reference cheap"""
    amp, det = W.blockade_sweep_waveforms(t_rise=100, t_sweep=300, t_fall=100)
    return W.ising_global_spec(W.disc_register(n, 22.0, 6.0, n), W.C6_LEVEL_60, amp, det)


@dataclasses.dataclass(frozen=True)
class Case:
    id: str
    n: int
    a: float
    b: float
    tol: float


CASES = [
    Case("rise_interval_n13", 13, 0.050, 0.051, 1e-8),          # amplitude ramp: p_om = 1, G_k stored
    Case("plateau_interval_n14", 14, 0.250, 0.251, 1e-8),       # constant drive, detuning ramp
    Case("rise_to_sweep_n15", 15, 0.040, 0.180, 1e-8),
    Case("sweep_n16", 16, 0.150, 0.350, 1e-8),
    Case("sweep_tight_n16", 16, 0.150, 0.350, 1e-10),
    Case("whole_n13", 13, 0.0, 0.500, 1e-8),
]

# (steps, K of every step, launches) of the all-fp64 propagator
EXPECTED = {
    'rise_interval_n13': (1, [9], 9),
    'plateau_interval_n14': (1, [8], 8),
    'rise_to_sweep_n15': (27, [58, 14, 10, 10, 10, 10, 10, 10, 10, 10, 11, 12, 12, 12, 11, 10, 10, 10, 10, 10, 10, 10, 10, 12, 20,
         61, 29], 412),
    'sweep_n16': (4, [61, 62, 62, 47], 232),
    'sweep_tight_n16': (4, [65, 66, 67, 51], 249),
    'whole_n13': (65, [63, 32, 13, 12, 9, 9, 9, 9, 9, 10, 10, 11, 12, 11, 11, 10, 9, 9, 9, 9, 9, 9, 12, 16, 61, 62, 61, 73,
         10, 10, 7, 7, 7, 8, 8, 8, 9, 10, 10, 11, 11, 9, 9, 8, 8, 8, 7, 7, 11, 12, 48, 9, 9, 7, 7, 7, 7, 7,
         7, 8, 9, 10, 12, 13, 25], 959),
}


def run_case(engine, case: Case):
    """(stats, [(K, k_lo)] from the step log, final state, initial state), the step log read from stderr"""
    spec = c2(case.n)
    psi0 = random_state(spec.hilbert_dim, 7 + case.n)
    os.environ["PB200_TAYLOR_LOG"] = "1"
    with tempfile.TemporaryFile(mode="w+") as f:
        fd = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            with engine.DevicePlan(spec) as plan:
                plan.set_state(psi0)
                st = plan.propagate(case.a, case.b, integrator=3, tol=case.tol)
                got = plan.get_state()[0]
        finally:
            os.dup2(fd, 2)
            os.close(fd)
            del os.environ["PB200_TAYLOR_LOG"]
        f.seek(0)
        steps = [(int(m[1]), int(m[2])) for m in STEP_RE.finditer(f.read())]
    return st, steps, got, psi0


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_tail_orders_within_error_estimate(engine, case):
    st, steps, got, psi0 = run_case(engine, case)
    assert st["integrator"] == 3 and len(steps) == st["n_steps"] > 0
    # the tail orders ran in single precision, the head of every step in fp64
    assert all(0 < k_lo <= K for K, k_lo in steps) and any(k_lo < K for K, k_lo in steps)
    ref = PiecewiseCubicHamiltonian(c2(case.n)).evolve(psi0, case.a, case.b)
    err = float(np.linalg.norm(got - ref))
    assert err <= A * st["err_estimate"] + FLOOR, (err, st["err_estimate"])
    # the schedule of the all-fp64 propagator
    n_steps, ks, launches = EXPECTED[case.id]
    assert (st["n_steps"], [K for K, _ in steps], st["n_launches"]) == (n_steps, ks, launches)
