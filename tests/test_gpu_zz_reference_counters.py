"""GPU master-equation path against the reference's own Counter goldens (runs last: file name sorts after the
other GPU tests).

``tests/golden/ref_counter_*.npz`` <- the hard-coded Counters of the reference's
``tests/pulser_simulation/test_simulation.py:978-1046`` (test_noises_rydberg), ``:1079-1171``
(test_noises_digital) -- real QuTiP ``mesolve`` outputs -- and ``:2594-2650`` (test_eom_limit_det, ``sesolve``),
all sampled with ``np.random.seed(123)``.  The CPU oracle reproduces
all 14 exactly (``tests/golden/make_golden.py --counters`` asserts it, ``tests/test_oracle_cpu.py`` re-checks); here the
CUDA Lindblad path must land on the same density matrix (north-star tolerance 1e-4) and -- sampled with the
reference's recipe from the same stream position -- on the same Counter, up to the two shots a 1e-4 shift of a
cumulative boundary can move.
"""
import glob
import os
from collections import Counter

import numpy as np
import pytest

from pulser_b200.spec import HamiltonianSpec

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
NAMES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLD, "ref_counter_*.npz")))


def load(name):
    with np.load(os.path.join(GOLD, name + ".npz"), allow_pickle=False) as data:
        return HamiltonianSpec.from_npz(data), {k: data[k] for k in data.files}


def sample_like_the_reference(spec, state, extra):
    from pulser_b200.results import B200Result, CoherentResults, DensityMatrix, StateVector

    n, d = spec.n_qudits, spec.dim
    meas = str(extra["meas_basis"])
    wrapped = DensityMatrix(state, [[d] * n, [d] * n]) if np.ndim(state) == 2 else StateVector(state, [[d] * n, [1] * n])
    res = CoherentResults(
        [B200Result(tuple(spec.qubit_ids), meas, wrapped, True, evaluation_time=1.0)],
        n, spec.basis_name, np.array([spec.sampling_times[-1]]), meas)
    np.random.seed(int(extra["seed"]))
    np.random.rand(int(extra["pre_draws"]))  # what the reference's constructor drew before the run
    return res.sample_final_state()


@pytest.mark.parametrize("name", [n for n in NAMES if "_eom_" in n])
def test_schroedinger_reference_counters(lib, name):
    """reference test_simulation.py:2594-2650 (test_eom_limit_det): noiseless three-atom sesolve runs in EOM mode at
    the detuning limits, through the stage kernels."""
    from pulser_b200 import engine

    spec, extra = load(name)
    expected = Counter(dict(zip((str(k) for k in extra["counter_keys"]), (int(v) for v in extra["counter_values"]))))
    with engine.DevicePlan(spec) as plan:
        plan.set_state(extra["psi0"])
        plan.propagate(0.0, spec.sampling_times[-1])
        psi = plan.get_state()[0]
    # EOM detunings of +-1000 rad/us held for microseconds: the stiffest sequence of the suite; north-star bound,
    # the measured error is printed (pytest -s)
    err = float(np.max(np.abs(psi - extra["orc_final"])))
    print(f"{name}: max |psi_gpu - psi_oracle| = {err:.3e}")
    assert err < 1e-8
    got = sample_like_the_reference(spec, psi, extra)
    assert got == expected  # a 1e-8 shift of a cumulative boundary moves no shot


@pytest.mark.parametrize("name", [n for n in NAMES if "_eom_" not in n])
def test_master_equation_reference_counters(lib, name):
    from pulser_b200 import engine
    from pulser_b200.lindblad import LindbladPlan

    assert engine.device_count() > 0
    spec, extra = load(name)
    expected = Counter(dict(zip((str(k) for k in extra["counter_keys"]), (int(v) for v in extra["counter_values"]))))
    with LindbladPlan(spec) as lp:
        lp.set_state(extra["psi0"])
        lp.propagate(0.0, spec.sampling_times[-1])
        rho = lp.get_rho()[0]
    assert abs(np.trace(rho).real - 1.0) < 1e-6
    assert np.max(np.abs(rho - extra["orc_rho"])) < 1e-4
    got = sample_like_the_reference(spec, rho, extra)
    moved = sum(abs(got.get(k, 0) - expected.get(k, 0)) for k in set(got) | set(expected)) // 2
    assert moved <= 2, (got, expected)


def test_expect_leakage_reference_value(lib):
    """reference tests/pulser_simulation/test_simresults.py:339-361: <|r><r|>(T) = 0.7804005 (atol 1e-6, a QuTiP
    mesolve output) for a single atom with the collapse operator |x><g|, on the CUDA master-equation path."""
    from pulser_b200.lindblad import LindbladPlan

    spec, extra = load("ref_expect_leakage")
    with LindbladPlan(spec) as lp:
        lp.set_state(extra["psi0"])
        lp.propagate(0.0, spec.sampling_times[-1], tol=1e-9)
        rho = lp.get_rho()[0]
    assert np.isclose(rho[0, 0].real, float(extra["ref_value"]), atol=1e-6)  # the reference's own tolerance
    assert np.max(np.abs(rho - extra["orc_rho"])) < 1e-6
