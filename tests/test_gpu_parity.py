"""GPU parity tests: CUDA path (through the C ABI) against the CPU oracle.

Tolerances (BASELINE.json north_star): rtol 1e-8 on Schroedinger state
amplitudes, measured as max |psi_gpu - psi_oracle| (states have unit norm).
"""
import numpy as np
import pytest

from helpers import random_local_spec, random_state
from pulser_b200 import workloads as W

pytestmark = pytest.mark.gpu

STATE_TOL = 1e-8


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


def _oracle_final(spec, psi0, t_end=None, order=3):
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    H = OracleHamiltonian.from_spec(spec)
    t_end = spec.sampling_times[-1] if t_end is None else t_end
    return evolve.sesolve(H, psi0, [0.0, t_end], order=order, rtol=1e-13, atol=1e-15)[-1]


@pytest.mark.parametrize("n", [1, 2, 4, 7, 10, 11, 12, 13, 15, 16])
def test_apply_h_uniform(engine, n):
    """H(t) psi on the device == matrix-free oracle (global drive)."""
    from oracle.matfree import MatFreeHamiltonian

    spec = W.config_c2(n=n, seed=5) if n > 1 else W.ising_global_spec(
        np.zeros((1, 2)), W.C6_LEVEL_60, *W.blockade_sweep_waveforms())
    mf = MatFreeHamiltonian(spec)
    v = random_state(spec.hilbert_dim, n)
    with engine.DevicePlan(spec) as plan:
        for t in (0.1234, 1.7, 3.9995):
            got = plan.apply_h(t, v)
            ref = mf.apply(t, v)
            assert np.max(np.abs(got - ref)) < 1e-12 * max(1.0, np.max(np.abs(ref)))


@pytest.mark.parametrize("n", [3, 6, 11, 12, 14, 16])
def test_apply_h_local_complex(engine, n):
    """Per-qubit complex drives (noisy-trajectory shape)."""
    from oracle.matfree import MatFreeHamiltonian

    spec = random_local_spec(n, T=64, seed=n)
    mf = MatFreeHamiltonian(spec)
    v = random_state(spec.hilbert_dim, n)
    with engine.DevicePlan(spec) as plan:
        for t in (0.0031, 0.0405):
            got = plan.apply_h(t, v)
            ref = mf.apply(t, v)
            assert np.max(np.abs(got - ref)) < 1e-12 * max(1.0, np.max(np.abs(ref)))


def test_c1_four_atom_square(engine):
    """BASELINE config C1 end to end against the tight-tolerance oracle."""
    from oracle import evolve

    spec = W.config_c1()
    psi0 = evolve.all_ground_state(spec)
    ref = _oracle_final(spec, psi0)
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, spec.sampling_times[-1])
        got = plan.get_state()[0]
    assert st["n_applies"] > 0 and st["n_launches"] > 0
    assert np.max(np.abs(got - ref)) < STATE_TOL
    assert abs(np.linalg.norm(got) - 1.0) < 1e-9


@pytest.mark.parametrize("n,max_step,tol", [(6, 1, -1.0), (8, 2, -1.0), (8, 0, 0.0), (10, 0, 0.0), (12, 0, 0.0)])
def test_blockade_sweep_vs_oracle(engine, n, max_step, tol):
    """C2-shaped sequence (4000 ns) at oracle-sized registers; fixed steps
    (tol < 0) and the default adaptive step-doubling controller (tol = 0)."""
    from oracle import evolve

    spec = W.config_c2(n=n, seed=20)
    psi0 = evolve.all_ground_state(spec)
    ref = _oracle_final(spec, psi0)
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, spec.sampling_times[-1], max_step=max_step, tol=tol, integrator=1)
        got = plan.get_state()[0]
    assert np.max(np.abs(got - ref)) < STATE_TOL
    assert (st["n_checks"] > 0) == (tol >= 0)


def test_dense_strongly_interacting_register(engine):
    """Closely packed atoms (U ~ 100 rad/us): the controller must shorten the steps."""
    from oracle import evolve

    amp, det = W.blockade_sweep_waveforms(t_rise=100, t_sweep=400, t_fall=100)
    spec = W.ising_global_spec(W.square_register(3, 6.0)[:8], W.C6_LEVEL_70, amp, det)
    psi0 = evolve.all_ground_state(spec)
    ref = _oracle_final(spec, psi0)
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, spec.sampling_times[-1])
        got = plan.get_state()[0]
    assert np.max(np.abs(got - ref)) < STATE_TOL
    assert st["mean_step_samples"] < 8.0  # dense register: the spectral-radius cap shortens the steps


def test_local_noisy_trajectory_vs_oracle(engine):
    from oracle import evolve

    spec = random_local_spec(6, T=300, seed=3)
    psi0 = random_state(spec.hilbert_dim, 9)
    ref = _oracle_final(spec, psi0)
    with engine.DevicePlan(spec) as plan:
        plan.set_state(psi0)
        plan.propagate(0.0, spec.sampling_times[-1])
        got = plan.get_state()[0]
    assert np.max(np.abs(got - ref)) < STATE_TOL


def test_batch_of_trajectories(engine):
    """Three different trajectories evolved in one batch == one by one."""
    specs = [random_local_spec(5, T=120, seed=s) for s in (11, 12, 13)]
    psi0 = random_state(specs[0].hilbert_dim, 2)
    singles = []
    for s in specs:
        with engine.DevicePlan(s) as plan:
            plan.set_state(psi0)
            plan.propagate(0.0, s.sampling_times[-1], max_step=2, tol=-1.0)
            singles.append(plan.get_state()[0])
    with engine.DevicePlan(specs) as plan:
        plan.set_state(psi0)
        plan.propagate(0.0, specs[0].sampling_times[-1], max_step=2, tol=-1.0)
        got = plan.get_state()
    for a, b in zip(got, singles):
        assert np.max(np.abs(a - b)) < 1e-11
    ref = _oracle_final(specs[1], psi0)
    assert np.max(np.abs(got[1] - ref)) < STATE_TOL


def test_intermediate_times_and_restart(engine):
    """Propagating in pieces equals propagating at once (evaluation times)."""
    spec = W.config_c2(n=7, seed=3)
    tf = spec.sampling_times[-1]
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        plan.propagate(0.0, tf)
        whole = plan.get_state()[0]
        plan.set_state("all-ground")
        for a, b in [(0.0, 0.4567), (0.4567, 1.2), (1.2, 3.0005), (3.0005, tf)]:
            plan.propagate(a, b)
        pieces = plan.get_state()[0]
    assert np.max(np.abs(whole - pieces)) < STATE_TOL


@pytest.mark.parametrize("n", [18, 20])
def test_full_size_properties(engine, n):
    """BASELINE-size properties: unitarity and step-size self-convergence."""
    spec = W.config_c2(n=n, t_rise=100, t_sweep=200, t_fall=100)
    tf = spec.sampling_times[-1]
    outs = {}
    with engine.DevicePlan(spec) as plan:
        for tol in (0.0, 1e-11):  # default controller against a 100x tighter one
            plan.set_state("all-ground")
            plan.propagate(0.0, tf, tol=tol)
            n2 = plan.norm2()[0]
            assert abs(n2 - 1.0) < 1e-9
            outs[tol] = plan.get_state()[0]
    assert np.max(np.abs(outs[0.0] - outs[1e-11])) < STATE_TOL


def _sparse_apply_h(spec, t, states, amps):
    """H(t) v for v = sum_i amps[i] |states[i]> (d = 2, one drive, Ising), from the coefficient functions and role
    table of oracle/matfree.py: O(N^2) per basis state, for registers whose dense vectors the oracle cannot build."""
    from scipy.interpolate import make_interp_spline
    from oracle.matfree import BASIS_ROLES

    n = spec.n_qudits
    drv = spec.drives[0]
    to, frm = (spec.eigenbasis.index(x) for x in BASIS_ROLES[drv.basis])
    assert {to, frm} == {0, 1}
    c = make_interp_spline(spec.sampling_times, drv.coef.T, k=3)(t)
    det = make_interp_spline(spec.sampling_times, drv.det.T, k=3)(t)
    r = spec.eigenbasis.index("r")
    U = spec.pair_matrix()
    out = {}
    for s, a in zip(states, amps):
        dig = [(s >> (n - 1 - k)) & 1 for k in range(n)]     # qudit 0 is the most significant bit
        ryd = [k for k in range(n) if dig[k] == r]
        diag = sum(U[i, j] for x, i in enumerate(ryd) for j in ryd[x + 1:]) - sum(det[k] for k in range(n) if dig[k] == frm)
        out[s] = out.get(s, 0.0) + diag * a
        for k in range(n):   # c |to><from| + conj(c) |from><to| on qudit k
            s2 = s ^ (1 << (n - 1 - k))
            out[s2] = out.get(s2, 0.0) + (c[k] if dig[k] == frm else np.conj(c[k])) * a
    return out


@pytest.mark.parametrize("n,kind", [(17, "uniform"), (16, "local"), (27, "local"), (28, "uniform"), (28, "local")])
def test_pass_geometries(engine, n, kind):
    """H psi on the pass decompositions production takes, uniform and local drives: one pass of the 2^11 tile with
    partner loads for the bits above it (N <= 27), and from N = 28 a second pass over the next 9 bits with the rest as
    partner loads.  N >= 27 against the sparse oracle, for a sparse input with partners in every pass and extra bit."""
    spec = W.config_c2(n=n, seed=2) if kind == "uniform" else random_local_spec(n, T=32, seed=5)
    if n < 27:
        from oracle.matfree import MatFreeHamiltonian

        v = random_state(spec.hilbert_dim, 4)
        with engine.DevicePlan(spec) as plan:
            got = plan.apply_h(0.0123, v)
        ref = MatFreeHamiltonian(spec).apply(0.0123, v)
        assert np.max(np.abs(got - ref)) < 1e-12 * max(1.0, np.max(np.abs(ref)))
        return
    rng = np.random.default_rng(4)
    states = [(1 << n) - 1, 1 << (n - 1)] + [int(x) for x in rng.integers(0, 1 << n, size=6)]
    states = list(dict.fromkeys(states))
    amps = rng.normal(size=len(states)) + 1j * rng.normal(size=len(states))
    t = 0.0123
    ref = _sparse_apply_h(spec, t, states, amps)
    v = np.zeros(1 << n, dtype=np.complex128)
    v[states] = amps
    with engine.DevicePlan(spec) as plan:
        got = plan.apply_h(t, v)
    del v
    idx = np.array(sorted(ref))
    want = np.array([ref[i] for i in idx])
    assert len(idx) <= len(states) * (n + 1)
    assert np.max(np.abs(got[idx] - want)) < 1e-12 * max(1.0, np.max(np.abs(want)))
    got[idx] = 0.0
    assert not np.any(got)


# ---------------------------------------------------------------------------
# Lindblad master equation (mesolve replacement); north_star tolerance 1e-4
LINDBLAD_TOL = 1e-4


def _lindblad_spec(n, T, ops, seed=0):
    from pulser_b200.spec import HamiltonianSpec

    amp, det = W.blockade_sweep_waveforms(t_rise=T // 4, t_sweep=T // 2, t_fall=T // 4)
    coords = W.disc_register(n, 12.0, 5.0, seed + 3)
    spec = W.ising_global_spec(coords, W.C6_LEVEL_60, amp, det)
    spec.collapse_ops = np.asarray(ops, dtype=complex)
    return spec


@pytest.mark.parametrize("n,kind", [(2, "dephasing+relaxation"), (4, "dephasing+relaxation"), (3, "depolarizing")])
def test_lindblad_vs_oracle_mesolve(engine, n, kind):
    """Density-matrix evolution against the dense-Lindblad oracle (qutip.mesolve restatement)."""
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian
    from pulser_b200.lindblad import LindbladPlan

    if kind == "depolarizing":  # sqrt(G/4) X, Y, Z (hamiltonian_data.py:699-716)
        g = np.sqrt(0.4 / 4)
        ops = [g * np.array([[0, 1], [1, 0]]), g * np.array([[0, -1j], [1j, 0]]), g * np.array([[1, 0], [0, -1]])]
    else:  # sqrt(2 G_d)|r><r| and sqrt(G_rel)|g><r| in the [r, g] eigenbasis
        ops = [np.sqrt(2 * 0.3) * np.array([[1, 0], [0, 0]]), np.sqrt(0.2) * np.array([[0, 0], [1, 0]])]
    spec = _lindblad_spec(n, 400, ops)
    tf = spec.sampling_times[-1]
    H = OracleHamiltonian.from_spec(spec)
    psi0 = evolve.all_ground_state(spec)
    ref = evolve.mesolve(H, psi0, [0.0, tf])[-1]
    with LindbladPlan(spec) as lp:
        lp.set_state(psi0)
        st = lp.propagate(0.0, tf)
        rho = lp.get_rho()[0]
    assert st["n_launches"] > 0
    assert abs(np.trace(rho).real - 1.0) < 1e-6
    assert np.max(np.abs(rho - rho.conj().T)) < 1e-8
    assert np.max(np.abs(rho - ref)) < LINDBLAD_TOL
    # populations decohered: purity below one
    assert np.trace(rho @ rho).real < 0.999


@pytest.mark.parametrize("masked", [False, True])
def test_lindblad_xy_vs_oracle_mesolve(engine, masked):
    """XY master equation (exchange couplings doubled onto the column qudits with the opposite sign), with and
    without an SLM mask, against the dense-Lindblad oracle."""
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian
    from pulser_b200.lindblad import LindbladPlan

    spec = W.config_xy(n=3, seed=4, t_total=300, magnetic_field=(0.3, 1.0, 0.5))
    # sqrt(2 G_d)|u><u| (dephasing) and sqrt(G)|d><u| (decay) in the [u, d] eigenbasis
    spec.collapse_ops = np.asarray([np.sqrt(2 * 0.25) * np.array([[1, 0], [0, 0]]),
                                    np.sqrt(0.3) * np.array([[0, 0], [1, 0]])], dtype=complex)
    if masked:
        spec.slm_end, spec.slm_targets = 120, [1]
    tf = spec.sampling_times[-1]
    H = OracleHamiltonian.from_spec(spec)
    psi0 = random_state(spec.hilbert_dim, 6)
    ref = evolve.mesolve(H, psi0, [0.0, tf])[-1]
    with LindbladPlan(spec) as lp:
        lp.set_state(psi0)
        lp.propagate(0.0, tf)
        rho = lp.get_rho()[0]
    assert abs(np.trace(rho).real - 1.0) < 1e-6
    assert np.max(np.abs(rho - ref)) < LINDBLAD_TOL
    assert np.trace(rho @ rho).real < 0.999


# ---------------------------------------------------------------------------
# 3-level "all" basis (BASELINE config C3) and noisy trajectories (C4)
def test_c3_all_basis_vs_oracle(engine):
    from oracle import evolve

    spec = W.config_c3(n=5, t_raman=200, t_ryd=400)
    psi0 = evolve.all_ground_state(spec)
    ref = _oracle_final(spec, psi0)
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        plan.propagate(0.0, spec.sampling_times[-1])
        got = plan.get_state()[0]
    assert np.max(np.abs(got - ref)) < STATE_TOL


def test_c3_larger_register_properties(engine):
    """3^11 = 177147 amplitudes: unitarity and agreement with a 100x tighter controller."""
    spec = W.config_c3(n=11, t_raman=100, t_ryd=200)
    tf = spec.sampling_times[-1]
    outs = []
    with engine.DevicePlan(spec) as plan:
        for tol in (0.0, 1e-10):
            plan.set_state("all-ground")
            plan.propagate(0.0, tf, tol=tol)
            assert abs(plan.norm2()[0] - 1.0) < 1e-9
            outs.append(plan.get_state()[0])
    assert np.max(np.abs(outs[0] - outs[1])) < STATE_TOL


def _multilevel_spec(n, dim, seed=0, T=48):
    """'all'-basis register (digital + ground-rydberg drives) with per-atom complex tables; dim 4 adds a leakage
    level |x> that no drive touches."""
    base = W.config_c3(n=n, t_raman=T // 3, t_ryd=T - 2 * (T // 3))
    rng = np.random.default_rng(seed)
    nt = len(base.sampling_times)
    for d in base.drives:  # make the rows differ (noisy-trajectory shape) and the drives complex
        d.coef = d.coef * rng.normal(1.0, 0.1, size=(n, 1)) * np.exp(1j * rng.uniform(-1, 1, size=(n, 1)))
        d.det = d.det + rng.normal(0.0, 0.5, size=(n, 1)) * (np.arange(nt) < nt - 1)
        d.uniform = False
    if dim == 4:
        base.eigenbasis = list(base.eigenbasis) + ["x"]
        base.dim = 4
    return base


@pytest.mark.parametrize("n,dim", [(1, 3), (2, 3), (3, 3), (7, 3), (8, 3), (9, 3), (10, 3), (1, 4), (5, 4), (7, 4)])
def test_tiled_multilevel_kernel_apply_h(engine, n, dim):
    """stage_multilevel_rb_kernel (d = 3 / 4) == matrix-free oracle; (1, 3) runs the one-thread-per-amplitude generic
    kernel instead."""
    from oracle.matfree import MatFreeHamiltonian

    spec = _multilevel_spec(n, dim, seed=n)
    mf = MatFreeHamiltonian(spec)
    v = random_state(spec.hilbert_dim, n)
    with engine.DevicePlan(spec) as plan:
        for t in (0.0071, 0.0302):
            got = plan.apply_h(t, v)
            ref = mf.apply(t, v)
            assert np.max(np.abs(got - ref)) < 1e-12 * max(1.0, np.max(np.abs(ref)))


def test_c4_noisy_trajectories_batch_vs_oracle(engine):
    """Doppler + amplitude noise trajectories (C4 shape, 2x2 register so that the oracle can follow)."""
    from oracle import evolve

    coords = W.square_register(2, 6.0)
    amp, det = W.blockade_sweep_waveforms(t_rise=100, t_sweep=300, t_fall=100)
    base = W.ising_global_spec(coords, W.C6_LEVEL_70, amp, det)
    rng = np.random.default_rng(0)
    specs = [W.noisy_trajectory_spec(base, coords, rng.normal(0, 0.6, 4), max(0.0, rng.normal(1, 0.05)), 175.0)
             for _ in range(5)]
    psi0 = evolve.all_ground_state(base)
    with engine.DevicePlan(specs) as plan:
        plan.set_state("all-ground")
        plan.propagate(0.0, base.sampling_times[-1])
        got = plan.get_state()
    for g, s in zip(got, specs):
        assert np.max(np.abs(g - _oracle_final(s, psi0))) < STATE_TOL


# ---------------------------------------------------------------------------
# Lanczos (Krylov) exponentials
@pytest.mark.parametrize("builder", [
    lambda: W.config_c1(),
    lambda: W.config_c2(n=9, seed=20, t_rise=100, t_sweep=400, t_fall=100),
    lambda: random_local_spec(6, T=200, seed=4),
    lambda: W.config_c3(n=4, t_raman=100, t_ryd=200),
])
def test_krylov_integrator_vs_oracle(engine, builder):
    from oracle import evolve

    spec = builder()
    psi0 = evolve.all_ground_state(spec)
    ref = _oracle_final(spec, psi0)
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, spec.sampling_times[-1], integrator=2)
        got = plan.get_state()[0]
    assert st["integrator"] == 2 and st["n_applies"] > 0
    # d = 2 below the 2^11 tile: stage_d2_kernel + dot2 + the separate vector update per iteration; d = 3: fused
    assert st["n_launches"] == _krylov_launches(st, 3 if spec.dim == 2 else 1)
    assert np.max(np.abs(got - ref)) < STATE_TOL
    assert abs(np.linalg.norm(got) - 1.0) < 1e-9


def test_lanczos_needs_fewer_applies_on_blockaded_register(engine):
    """Dense 3x3 array at 6 um (U = 116 rad/us): wide spectrum, narrow populated band."""
    from oracle import evolve

    amp, det = W.blockade_sweep_waveforms(t_rise=100, t_sweep=300, t_fall=100)
    spec = W.ising_global_spec(W.square_register(3, 6.0), W.C6_LEVEL_70, amp, det)
    psi0 = evolve.all_ground_state(spec)
    ref = _oracle_final(spec, psi0)
    out = {}
    with engine.DevicePlan(spec) as plan:
        for integ in (0, 1, 2):
            plan.set_state("all-ground")
            st = plan.propagate(0.0, spec.sampling_times[-1], integrator=integ)
            out[integ] = (st, plan.get_state()[0])
    assert out[2][0]["integrator"] == 2 and out[1][0]["integrator"] == 1 and out[0][0]["integrator"] in (1, 2, 3)
    for st, got in out.values():
        assert np.max(np.abs(got - ref)) < STATE_TOL
    assert out[2][0]["n_applies"] < out[1][0]["n_applies"]


def _krylov_launches(st, per_apply):
    """Kernel launches of a default (adaptive, extrapolated) Lanczos run without dissipator: per exponential dot2 +
    normalize_copy + krylov_combine, `per_apply` per Lanczos iteration; per step one Richardson axpby, and a checked
    step runs three extrapolated steps and one diffnorm2 (rejected steps included)."""
    return (3 * st["n_exponentials"] + per_apply * st["n_applies"] + st["n_steps"] + st["n_rejected"]
            + 3 * st["n_checks"])


@pytest.mark.parametrize("kind", ["d2-uniform", "d2-batch", "d3", "d4-leak"])
def test_fused_lanczos_one_launch_per_iteration(engine, kind):
    """The one-launch Lanczos iteration (normalisation / orthogonalisation folded into the next stage's own-element
    operands, LanczosFuse in kernels.cuh): one launch per iteration, and the oracle's state.  The stage + vector-update
    pair runs below the register-blocked tile (test_krylov_integrator_vs_oracle)."""
    from oracle import evolve

    if kind == "d2-uniform":
        spec = W.config_c2(n=12, seed=20, t_rise=100, t_sweep=300, t_fall=100)
    elif kind == "d2-batch":
        spec = [random_local_spec(11, T=120, seed=s) for s in (41, 42, 43)]
    elif kind == "d3":
        spec = W.config_c3(n=6, t_raman=100, t_ryd=200)
    else:
        spec = _multilevel_spec(4, 4, seed=2, T=150)
    first = spec[0] if isinstance(spec, list) else spec
    tf = first.sampling_times[-1]
    psi0 = evolve.all_ground_state(first)
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        st = plan.propagate(0.0, tf, integrator=2)
        got = plan.get_state().copy()
    assert st["integrator"] == 2
    assert st["n_launches"] == _krylov_launches(st, 1)
    specs = spec if isinstance(spec, list) else [spec]
    for g, s1 in zip(got, specs):
        assert np.max(np.abs(g - _oracle_final(s1, psi0))) < STATE_TOL


def _uniform_spec(kind, n):
    if kind == "real":
        return W.config_c2(n=n, seed=3, t_rise=40, t_sweep=80, t_fall=40)
    amp, det = W.blockade_sweep_waveforms(t_rise=40, t_sweep=80, t_fall=40)
    phase = 0.3 + 0.004 * np.arange(len(amp))
    return W.ising_global_spec(W.disc_register(n, 38.0, 5.0, 3), W.C6_LEVEL_60, amp, det, phase=phase)


@pytest.mark.parametrize("kind,n", [("real", 17), ("complex", 17), ("real", 18), ("real", 19), ("complex", 19)])
def test_partner_sum_forwarding_equals_single_pass(engine, kind, n):
    """stage_d2_fwd_kernel (alternating tile geometries, forwarded partner sums; one state of uniform drives at
    17 <= N <= 19) against the same spec as a batch of two identical trajectories, which runs the same Chebyshev chains
    on the single-pass stage kernel: same H-applies, same launches, states equal to rounding.  At N = 17 it is also
    held to the Lanczos path at a tight tolerance."""
    spec = _uniform_spec(kind, n)
    tf = spec.sampling_times[-1]
    psi0 = random_state(spec.hilbert_dim, 5)
    out = {}
    for batch in ([spec], [spec, spec]):
        with engine.DevicePlan(batch) as plan:
            plan.set_state(psi0)
            st = plan.propagate(0.0, tf, integrator=1)
            out[len(batch)] = (plan.get_state().copy(), st)
    fwd, single = out[1][0][0], out[2][0]
    assert np.max(np.abs(fwd - single[0])) < 5e-13 and np.max(np.abs(fwd - single[1])) < 5e-13
    assert out[1][1]["n_applies"] == out[2][1]["n_applies"]
    assert out[1][1]["n_launches"] == out[2][1]["n_launches"]  # one launch per stage either way
    if n == 17:
        with engine.DevicePlan(spec) as plan:
            plan.set_state(psi0)
            plan.propagate(0.0, tf, integrator=2, tol=1e-11)
            assert np.max(np.abs(fwd - plan.get_state()[0])) < STATE_TOL


# ---------------------------------------------------------------------------
# measurement on the device
def test_device_sampling_equals_reference_recipe(engine):
    """Same state + same np.random seed -> the Counter the reference's host recipe gives
    (QutipResult._weights + multinomial), for d = 2 (reversed order) and the 3-level marginalisation."""
    from pulser_b200.results import B200Result, StateVector

    for spec, meas, one, matching in (
        (W.config_c2(n=9, seed=2, t_rise=50, t_sweep=100, t_fall=50), "ground-rydberg", "r", True),
        (W.config_c3(n=5, t_raman=100, t_ryd=150), "digital", "h", False),
        (W.config_c3(n=5, t_raman=100, t_ryd=150), "ground-rydberg", "r", False),
    ):
        with engine.DevicePlan(spec) as plan:
            plan.set_state("all-ground")
            plan.propagate(0.0, spec.sampling_times[-1])
            psi = plan.get_state()[0]
            np.random.seed(77)
            dev = plan.sample(2000, one)
            occ = plan.occupation(spec.eigenbasis.index(one))[0]
        np.random.seed(77)
        host = B200Result(tuple(range(spec.n_qudits)), meas, StateVector(psi), matching).get_samples(2000)
        assert dev == host
        d, n = spec.dim, spec.n_qudits
        probs = (np.abs(psi) ** 2).reshape([d] * n)
        ref_occ = [np.take(probs, spec.eigenbasis.index(one), axis=k).sum() for k in range(n)]
        np.testing.assert_allclose(occ, ref_occ, atol=1e-12)


def test_mcwf_average_matches_master_equation(engine):
    """Quantum-jump trajectories (mcsolve replacement): the ensemble average of the populations agrees with
    the Lindblad oracle within the statistical error of 3000 trajectories."""
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    ops = [np.sqrt(2 * 1.5) * np.array([[1, 0], [0, 0]]), np.sqrt(2.0) * np.array([[0, 0], [1, 0]])]
    spec = _lindblad_spec(2, 300, ops)
    tf = spec.sampling_times[-1]
    psi0 = evolve.all_ground_state(spec)
    rho = evolve.mesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf])[-1]
    ref = np.real(np.diag(rho))
    B = 3000
    with engine.DevicePlan([spec] * B) as plan:
        plan.set_collapse(np.asarray(ops, dtype=complex), seed=12345)
        plan.set_state("all-ground")
        plan.propagate(0.0, 0.5 * tf)   # thresholds persist across calls
        plan.propagate(0.5 * tf, tf)
        probs = plan.probabilities()
        jumps = plan.jump_counts()
        n2 = plan.norm2()
    np.testing.assert_allclose(n2, 1.0, atol=1e-9)
    assert jumps.sum() > B // 20
    mean = probs.mean(axis=0)
    sigma = np.sqrt(np.maximum(ref * (1 - ref), 1e-4) / B)
    assert np.all(np.abs(mean - ref) < 5 * sigma + 2e-3)


def test_mcwf_general_collapse_operators(engine):
    """Collapse operators whose L^+L is NOT diagonal (general effective noise, hamiltonian.py:97-124): the no-jump
    evolution applies exp(-tau sum L^+L) qudit by qudit and the jump weights come from the single-qudit reduced
    density matrices.  Ensemble average against the Lindblad oracle."""
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    plus = np.array([1.0, 1.0]) / np.sqrt(2.0)
    ops = [np.sqrt(1.8) * np.outer([0.0, 1.0], plus),            # |g><+| : L^+L = 1.8 |+><+|
           np.sqrt(0.9) * np.array([[0.0, 1.0], [1.0, 0.0]]) * np.array([[1.0, 1.0], [1.0, -1.0]]) / np.sqrt(2.0)]
    assert abs((ops[0].conj().T @ ops[0])[0, 1]) > 0.1           # genuinely non-diagonal
    spec = _lindblad_spec(2, 300, ops)
    tf = spec.sampling_times[-1]
    psi0 = evolve.all_ground_state(spec)
    rho = evolve.mesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf])[-1]
    ref = np.real(np.diag(rho))
    B = 3000
    with engine.DevicePlan([spec] * B) as plan:
        plan.set_collapse(np.asarray(ops, dtype=complex), seed=4321)
        plan.set_state("all-ground")
        plan.propagate(0.0, 0.4 * tf)
        plan.propagate(0.4 * tf, tf)
        probs = plan.probabilities()
        jumps = plan.jump_counts()
        n2 = plan.norm2()
    np.testing.assert_allclose(n2, 1.0, atol=1e-9)
    assert jumps.sum() > B // 20
    mean = probs.mean(axis=0)
    sigma = np.sqrt(np.maximum(ref * (1 - ref), 1e-4) / B)
    assert np.all(np.abs(mean - ref) < 5 * sigma + 2e-3)


@pytest.mark.parametrize("n,local_rows", [(2, False), (5, False), (9, True), (12, False), (13, True)])
def test_xy_apply_h(engine, n, local_rows):
    """XY mode: exchange term U_ij (|ud><du| + h.c.) + |uu><uu| van der Waals + microwave drive vs the oracle."""
    from oracle.matfree import MatFreeHamiltonian

    spec = W.config_xy(n=n, seed=n, t_total=80, local_rows=local_rows, magnetic_field=(0.3, 1.0, 0.5))
    mf = MatFreeHamiltonian(spec)
    v = random_state(spec.hilbert_dim, n)
    with engine.DevicePlan(spec) as plan:
        for t in (0.0123, 0.0551):
            got = plan.apply_h(t, v)
            ref = mf.apply(t, v)
            assert np.max(np.abs(got - ref)) < 1e-12 * max(1.0, np.max(np.abs(ref)))


@pytest.mark.parametrize("n,integrator", [(4, 1), (7, 1), (7, 2), (9, 0)])  # 0 auto, 1 Chebyshev, 2 Lanczos
def test_xy_evolution_vs_oracle(engine, n, integrator):
    from oracle import evolve

    spec = W.config_xy(n=n, seed=40 + n, t_total=300)
    psi0 = evolve.all_ground_state(spec)
    assert abs(psi0[0]) == 1.0  # all-|u>
    ref = _oracle_final(spec, psi0)
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        plan.propagate(0.0, spec.sampling_times[-1], integrator=integrator)
        got = plan.get_state()[0]
    assert np.max(np.abs(got - ref)) < STATE_TOL


def test_xy_batch_with_missing_atoms(engine):
    """Trajectories with different bad atoms: per-trajectory exchange couplings."""
    import copy
    from oracle import evolve

    base = W.config_xy(n=6, seed=3, t_total=200)
    specs = []
    for bad in ([], [2], [0, 5]):
        s = copy.copy(base)
        s.bad_atoms = np.zeros(6, dtype=bool)
        s.bad_atoms[bad] = True
        s.interaction_matrix = base.interaction_matrix.copy()
        s.interaction_matrix[:, bad, :] = 0.0
        s.interaction_matrix[:, :, bad] = 0.0
        d0 = base.drives[0]
        coef, det = d0.coef.copy(), d0.det.copy()
        coef[bad] = 0.0
        det[bad] = 0.0
        from pulser_b200.spec import DriveTable
        s.drives = [DriveTable(d0.basis, coef, det, False)]
        specs.append(s)
    psi0 = evolve.all_ground_state(base)
    with engine.DevicePlan(specs) as plan:
        plan.set_state("all-ground")
        plan.propagate(0.0, base.sampling_times[-1])
        got = plan.get_state()
    for b, s in enumerate(specs):
        assert np.max(np.abs(got[b] - _oracle_final(s, psi0))) < STATE_TOL


@pytest.mark.parametrize("builder", [
    lambda: W.config_c2(n=10, seed=4),
    lambda: W.config_c3(n=5),
    lambda: random_local_spec(9, T=80, seed=3),
    lambda: W.config_xy(n=7, seed=1, t_total=80),
])
def test_device_observable_reductions(engine, builder):
    """pb200_state_correlation / _energy / _overlap against the plain formulas on the downloaded state
    (CorrelationMatrix, Energy*, Fidelity of pulser/backend/default_observables.py)."""
    from oracle.matfree import MatFreeHamiltonian

    spec = builder()
    D, n, d = spec.hilbert_dim, spec.n_qudits, spec.dim
    mf = MatFreeHamiltonian(spec)
    psi = random_state(D, 11) * 1.3          # not normalised on purpose
    phi = random_state(D, 12)
    idx = np.arange(D)
    digits = [(idx // d ** (n - 1 - k)) % d for k in range(n)]
    t = float(spec.sampling_times[len(spec.sampling_times) // 3]) + 1e-4
    with engine.DevicePlan(spec) as plan:
        plan.set_state(psi)
        p = np.abs(psi) ** 2
        for digit in range(d):
            corr = plan.correlation(digit)[0]
            ref = np.array([[p[(digits[i] == digit) & (digits[j] == digit)].sum() for j in range(n)] for i in range(n)])
            assert np.max(np.abs(corr - ref)) < 1e-12 * p.sum()
            assert np.max(np.abs(np.diag(corr) - plan.occupation(digit)[0])) < 1e-12 * p.sum()
        e, e2 = plan.energy(t)
        hpsi = mf.apply(t, psi)
        assert abs(e[0] - np.vdot(psi, hpsi).real) < 1e-11 * max(1.0, abs(np.vdot(hpsi, hpsi).real) ** 0.5)
        assert abs(e2[0] - np.vdot(hpsi, hpsi).real) < 1e-11 * max(1.0, np.vdot(hpsi, hpsi).real)
        ov = plan.overlap(phi)[0]
        assert abs(ov - np.vdot(phi, psi)) < 1e-12
        assert np.max(np.abs(plan.get_state()[0] - psi)) == 0.0   # the reductions leave the state untouched


def test_device_observables_full_size(engine):
    """N = 20: no oracle matrix; consistency of the device reductions among themselves."""
    spec = W.config_c2(n=20)
    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        plan.propagate(0.0, 0.4)
        corr = plan.correlation(0)[0]
        occ = plan.occupation(0)[0]
        nrm = plan.norm2()[0]
        assert np.max(np.abs(np.diag(corr) - occ)) < 1e-12
        assert np.all(corr <= np.minimum.outer(occ, occ) + 1e-12) and np.all(corr >= -1e-15)
        assert np.allclose(corr, corr.T, atol=0)
        e, e2 = plan.energy(0.4)
        assert e2[0] >= e[0] ** 2 / nrm - 1e-9           # Cauchy-Schwarz: <H^2> >= <H>^2
        psi = plan.get_state()[0]
        assert abs(plan.overlap(psi)[0] - nrm) < 1e-11
        hpsi = plan.apply_h(0.4, psi)
        assert abs(e[0] - np.vdot(psi, hpsi).real) < 1e-9 and abs(e2[0] - np.vdot(hpsi, hpsi).real) < 1e-8


def test_xy_with_leakage_level(engine):
    """XY eigenbasis (u, d, x): d = 3 with the flip-flop term (leakage NoiseModel shape, hamiltonian_data.py:927-931)."""
    from oracle import evolve
    from oracle.matfree import MatFreeHamiltonian

    spec = W.config_xy(n=5, seed=2, t_total=150, local_rows=True)
    spec.dim = 3
    spec.eigenbasis = ["u", "d", "x"]
    spec.basis_name = "XY_with_error"
    spec.collapse_ops = np.zeros((0, 3, 3), dtype=np.complex128)
    mf = MatFreeHamiltonian(spec)
    v = random_state(spec.hilbert_dim, 8)
    psi0 = evolve.all_ground_state(spec)
    ref = _oracle_final(spec, psi0)
    with engine.DevicePlan(spec) as plan:
        got = plan.apply_h(0.0313, v)
        assert np.max(np.abs(got - mf.apply(0.0313, v))) < 1e-12 * np.max(np.abs(got))
        plan.set_state("all-ground")
        plan.propagate(0.0, spec.sampling_times[-1])
        assert np.max(np.abs(plan.get_state()[0] - ref)) < STATE_TOL


# ---------------------------------------------------------------------------
# Partner-sum forwarding between Clenshaw stages (kernels.cuh FWD, DESIGN.md section 4): the alternating-geometry
# stages must reproduce the single-pass stages bit for bit up to rounding.
def test_state_copy_between_plans(engine):
    """pb200_state_copy: the state of one noisy trajectory evaluated under the NOISELESS Hamiltonian of another plan
    (what the generic backend's Energy observables need for stochastic-noise runs), no host round trip."""
    from oracle.matfree import MatFreeHamiltonian

    noisy = [random_local_spec(9, T=80, seed=s) for s in (31, 32, 33)]
    clean = W.config_c2(n=9, seed=5, t_rise=20, t_sweep=40, t_fall=20)
    assert clean.hilbert_dim == noisy[0].hilbert_dim
    psi0 = random_state(clean.hilbert_dim, 8)
    t = 0.0413
    with engine.DevicePlan(noisy) as plan, engine.DevicePlan(clean) as hplan:
        plan.set_state(psi0)
        plan.propagate(0.0, 0.05)
        states = plan.get_state()
        for traj in (2, 0):
            hplan.copy_state_from(plan, traj, 0)
            np.testing.assert_array_equal(hplan.get_state()[0], states[traj])
            e, e2 = hplan.energy(t)
            hpsi = MatFreeHamiltonian(clean).apply(t, states[traj])
            assert abs(e[0] - np.vdot(states[traj], hpsi).real) < 1e-10 * max(1.0, np.linalg.norm(hpsi))
            assert abs(e2[0] - np.vdot(hpsi, hpsi).real) < 1e-10 * max(1.0, np.vdot(hpsi, hpsi).real)
        np.testing.assert_array_equal(plan.get_state(), states)  # the source is untouched
        with pytest.raises(Exception, match="different Hilbert spaces"):
            with engine.DevicePlan(W.config_c2(n=8, seed=5, t_rise=20, t_sweep=40, t_fall=20)) as small:
                small.copy_state_from(plan, 0, 0)
