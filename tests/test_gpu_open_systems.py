"""GPU tests of the dissipative paths against the exact references of ``tests/open_ref.py``.

Master equation (``LindbladPlan``: ``pair_op_kernel`` and the symmetric splitting of the Chebyshev and Lanczos chains)
on cases with closed-form or product solutions, at the sizes the facade sends there (d = 2 up to N = 12, d = 3 up to
N = 8).  Monte-Carlo wave function (``mcwf_decay_kernel``, ``qudit_op_kernel``, ``reduced_density_kernel``, the jump
channel choice) on deterministic properties of single trajectories, and on jump statistics at N = 14 against the
analytic decay law.  Measured errors are printed (``-s``) next to the bounds chosen from them.
"""
import numpy as np
import pytest

import open_ref as R
from helpers import open_spec

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


def _lindblad(engine, specs, rho0, **opts):
    """Final density matrices ``[B, D, D]`` and the run statistics; ``rho0`` is one matrix or ``[B, D, D]``."""
    from pulser_b200.lindblad import LindbladPlan

    with LindbladPlan(specs) as lp:
        if np.asarray(rho0).ndim == 3:
            lp.plan.set_state(np.ascontiguousarray(rho0).reshape(len(rho0), -1))
        else:
            lp.set_state(rho0)
        T = lp.specs[0].sampling_times[-1]
        st = lp.propagate(0.0, T, **opts)
        return lp.get_rho(), st


def _fro(x):
    return float(np.linalg.norm(np.asarray(x).reshape(-1)))


# ---------------------------------------------------------------------------------------------------------------
# 1. H = 0, general collapse operators: exp(T sum_k G_k) exactly
@pytest.mark.parametrize("d,n,B", [(2, 1, 1), (2, 2, 1), (2, 5, 1), (2, 9, 1), (2, 12, 1),
                                   (3, 1, 1), (3, 3, 1), (3, 6, 1), (3, 8, 1), (2, 5, 3)])
def test_lindblad_zero_hamiltonian(engine, d, n, B):
    ops = R.random_ops(d, 3, 8.0, 100 * d + n)
    spec = open_spec(n, d, T=20, drive=False, detuning=False, interaction=False, ops=ops)
    T = spec.sampling_times[-1]
    G = [R.single_qudit_generator(ops)] * n
    rho0 = np.stack([R.random_density(d**n, 4, 7 * n + b) for b in range(B)])
    refs = [R.pair_expm_apply(r, G, T) for r in rho0]
    assert min(_fro(r - r0) for r, r0 in zip(refs, rho0)) > 1e-2 * _fro(rho0[0])  # the dissipator acts
    for integrator in (1, 2):
        rho, st = _lindblad(engine, [spec] * B, rho0 if B > 1 else rho0[0], integrator=integrator)
        assert st["integrator"] == integrator
        err = max(np.max(np.abs(rho[b] - refs[b])) / _fro(refs[b]) for b in range(B))
        print(f"\n[zero-H] d={d} N={n} B={B} integrator={integrator}: max |rho - ref| / |ref| = {err:.2e}")
        assert err < 1e-12


# ---------------------------------------------------------------------------------------------------------------
# 2. diagonal H (time-dependent detuning + interaction) with diagonal dephasing: they commute, CF4 is exact
@pytest.mark.parametrize("d,n", [(2, 3), (2, 10), (2, 12), (3, 4), (3, 8)])
def test_lindblad_diagonal(engine, d, n):
    ops = R.random_diag_ops(d, 2, 4.0, 10 + d + n)
    spec = open_spec(n, d, T=40, seed=n, drive=False, ops=ops)
    T = spec.sampling_times[-1]
    rho0 = R.random_density(d**n, 3, n)
    ref = R.diagonal_lindblad(rho0, spec, ops, T)
    rho, st = _lindblad(engine, spec, rho0)
    err = float(np.max(np.abs(rho[0] - ref)))
    print(f"\n[diagonal] d={d} N={n} integrator={st['integrator']}: max |rho - ref| = {err:.2e}")
    assert err < 1e-10


# ---------------------------------------------------------------------------------------------------------------
# 3. driven, non-interacting register at production size: the product of single-qudit master equations
TIGHT_PRODUCT = 1e-10  # ~10x the largest error measured on an H100 (6.9e-12, d = 2, N = 4)


@pytest.mark.parametrize("d,n", [(2, 4), (2, 10), (2, 12), (3, 3), (3, 7)])
def test_lindblad_driven_product(engine, d, n):
    import torch

    eig = open_spec(1, d).eigenbasis
    ops = np.concatenate([R.random_diag_ops(d, 1, 2.0, 3), [R.relaxation(eig, 3.0)], R.random_ops(d, 1, 2.0, 4)])
    spec = open_spec(n, d, T=40, seed=n + 2, interaction=False, ops=ops)
    T = spec.sampling_times[-1]
    rho_k0 = [R.random_density(d, 2, 20 + k) for k in range(n)]
    ref = R.kron_all(R.product_lindblad(spec, ops, rho_k0, T))
    rho0 = R.kron_all(rho_k0)
    for tol, bound in ((0.0, 1e-4), (1e-10, TIGHT_PRODUCT)):
        rho, st = _lindblad(engine, spec, rho0, tol=tol)
        free, total = torch.cuda.mem_get_info()
        err = float(np.max(np.abs(rho[0] - ref)))
        # the buffer pool keeps what the plan allocated, so the card's used memory after the run bounds its peak
        print(f"\n[product] d={d} N={n} tol={tol or 'default'} integrator={st['integrator']} steps={st['n_steps']}: "
              f"max |rho - ref| = {err:.2e} (bound {bound:.0e}); card memory in use {(total - free) / 2**30:.1f} GiB")
        if d == 2 and n == 12:
            assert st["integrator"] == 2  # 2^24 amplitudes: Lanczos by the automatic choice
        assert err < bound


# ---------------------------------------------------------------------------------------------------------------
# 4. interacting register at a tight tolerance against the dense-Lindblad oracle
TIGHT_MESOLVE = 1e-8  # ~10x the largest error measured on an H100 (7.3e-10, N = 2)


@pytest.mark.parametrize("n,kind", [(2, "dephasing+relaxation"), (4, "dephasing+relaxation"), (3, "depolarizing")])
def test_lindblad_interacting_tight(engine, n, kind):
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian
    from pulser_b200 import workloads as W

    if kind == "depolarizing":
        g = np.sqrt(0.4 / 4)
        ops = [g * np.array([[0, 1], [1, 0]]), g * np.array([[0, -1j], [1j, 0]]), g * np.array([[1, 0], [0, -1]])]
    else:
        ops = [np.sqrt(2 * 0.3) * np.array([[1, 0], [0, 0]]), np.sqrt(0.2) * np.array([[0, 0], [1, 0]])]
    amp, det = W.blockade_sweep_waveforms(t_rise=100, t_sweep=200, t_fall=100)
    spec = W.ising_global_spec(W.disc_register(n, 12.0, 5.0, 3), W.C6_LEVEL_60, amp, det)
    spec.collapse_ops = np.asarray(ops, dtype=complex)
    tf = spec.sampling_times[-1]
    psi0 = evolve.all_ground_state(spec)
    ref = evolve.mesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf], rtol=1e-12, atol=1e-14)[-1]
    rho, st = _lindblad(engine, spec, np.outer(psi0, psi0.conj()), tol=1e-10)
    err = float(np.max(np.abs(rho[0] - ref)))
    print(f"\n[interacting] N={n} {kind} tol=1e-10 steps={st['n_steps']}: max |rho - ref| = {err:.2e} "
          f"(bound {TIGHT_MESOLVE:.0e})")
    assert err < TIGHT_MESOLVE


# ---------------------------------------------------------------------------------------------------------------
# 5. MCWF no-jump evolution: exact for H = 0 with any K = sum L^+L, and for diagonal H with diagonal K
def _basis_ops(d, kind, n, T):
    """Collapse operators whose total norm loss over ``T`` on ``n`` qudits stays below 1e-3."""
    ops = R.random_ops(d, 2, 1.0, 5 * d + n) if kind == "general" else R.random_diag_ops(d, 2, 1.0, 5 * d + n)
    K = sum(L.conj().T @ L for L in ops)
    scale = np.sqrt(1e-3 / (n * T * np.linalg.norm(K, 2)))
    return ops * scale


@pytest.mark.parametrize("kind", ["general", "diagonal"])
@pytest.mark.parametrize("d,n", [(2, 3), (2, 14), (2, 18), (3, 5), (3, 9), (4, 4), (4, 7)])
def test_mcwf_no_jump_exact(engine, d, n, kind):
    B = 3
    spec = open_spec(n, d, T=20, seed=n, drive=False, detuning=kind == "diagonal", interaction=kind == "diagonal")
    T = spec.sampling_times[-1]
    ops = _basis_ops(d, kind, n, T)
    K = sum(L.conj().T @ L for L in ops)
    assert (np.max(np.abs(K - np.diag(np.diag(K)))) > 1e-6) == (kind == "general")
    rng = np.random.default_rng(n)
    psi0 = rng.normal(size=(B, d**n)) + 1j * rng.normal(size=(B, d**n))
    psi0 /= np.linalg.norm(psi0, axis=1, keepdims=True)
    ref = R.no_jump_state(psi0, K, T)
    if kind == "diagonal":
        ref = ref * np.exp(-1j * R.diagonal_phases(spec, T))[None, :]
    with engine.DevicePlan([spec] * B) as plan:
        plan.set_collapse(ops, seed=2024)
        plan.set_state(psi0)
        # thresholds and the renormalisation carry over between calls; a tight Chebyshev tolerance keeps the
        # unitary part of the diagonal case exact to rounding
        plan.propagate(0.0, 0.45 * T, cheb_tol=1e-15)
        plan.propagate(0.45 * T, T, cheb_tol=1e-15)
        got = plan.get_state()
        jumps = plan.jump_counts()
    assert np.all(jumps == 0)
    err = float(np.max(np.abs(got - ref)))
    print(f"\n[no-jump] d={d} N={n} {kind}: max |psi - ref| = {err:.2e}, 1 - |<psi0|ref>| = "
          f"{1 - np.min(np.abs(np.sum(psi0.conj() * R.no_jump_state(psi0, K, T), axis=1))):.1e}")
    assert err < 1e-12


# ---------------------------------------------------------------------------------------------------------------
# 6. jump structure: from a basis state under diagonal H and relaxation, every trajectory stays a basis state
def _basis_index(n, d, digits):
    idx = 0
    for a in digits:
        idx = idx * d + a
    return idx


@pytest.mark.parametrize("d,n,S", [(2, 14, (0, 3, 4, 9, 13)), (4, 9, (0, 3, 4, 8))])
def test_mcwf_jump_structure(engine, d, n, S):
    B = 256
    spec = open_spec(n, d, T=60, seed=3, drive=False)
    eig = spec.eigenbasis
    r, g = eig.index("r"), eig.index("g")
    ops = [R.relaxation(eig, 12.0)]
    if d == 4:  # sqrt(g') |g><phi|, phi = (|h> + |x>)/sqrt 2: L^+L non-diagonal, but no weight on r / g states
        phi = np.zeros(d); phi[eig.index("h")] = phi[eig.index("x")] = 1 / np.sqrt(2)
        Lx = np.zeros((d, d), dtype=complex); Lx[g] = np.sqrt(6.0) * phi
        assert abs((Lx.conj().T @ Lx)[eig.index("h"), eig.index("x")]) > 1.0
        ops.append(Lx)
    ops = np.asarray(ops, dtype=complex)
    digits0 = [r if k in S else g for k in range(n)]
    psi0 = np.zeros(d**n, dtype=complex)
    psi0[_basis_index(n, d, digits0)] = 1.0
    T = spec.sampling_times[-1]
    with engine.DevicePlan([spec] * B) as plan:
        plan.set_collapse(ops, seed=77)
        plan.set_state(psi0)
        plan.propagate(0.0, 0.5 * T)
        plan.propagate(0.5 * T, T)
        psi = plan.get_state()
        jumps = plan.jump_counts()
    top = np.argmax(np.abs(psi), axis=1)
    amp = np.abs(psi[np.arange(B), top])
    rest = np.abs(psi).copy()
    rest[np.arange(B), top] = 0.0
    assert np.all(np.isfinite(psi))
    assert np.max(np.abs(amp - 1.0)) < 1e-12
    assert np.max(rest) < 1e-12
    for b in range(B):
        dig = [(top[b] // d ** (n - 1 - k)) % d for k in range(n)]
        rset = {k for k in range(n) if dig[k] == r}
        assert all(dig[k] in (r, g) for k in range(n)), dig
        assert rset <= set(S), (b, rset)
        assert len(S) - len(rset) == jumps[b], (b, rset, jumps[b])
    assert 0 < jumps.mean() < len(S) and np.any(jumps >= 2)


# ---------------------------------------------------------------------------------------------------------------
# 7. jump statistics at N = 14 against the analytic decay law (no absolute slack)
def _decay_run(engine, spec, ops, B, seed):
    n, d = spec.n_qudits, spec.dim
    with engine.DevicePlan([spec] * B) as plan:
        plan.set_collapse(np.asarray(ops, dtype=complex), seed=seed)
        plan.set_state(np.eye(1, d**n, 0, dtype=complex)[0])  # |r...r>
        T = spec.sampling_times[-1]
        st = plan.propagate(0.0, T)
        psi = plan.get_state()
        jumps = plan.jump_counts()
    pops = np.abs(psi.reshape([B] + [d] * n)) ** 2
    # per-trajectory single-qudit populations [B, n, d]
    occ = np.stack([np.stack([pops.sum(axis=tuple(j + 1 for j in range(n) if j != k))[:, a] for a in range(d)], axis=1)
                    for k in range(n)], axis=1)
    return occ, jumps, st


@pytest.mark.parametrize("gamma,step_ns,T", [(20.0, 4, 25), (5.0, 1, 300)])
def test_mcwf_decay_statistics(engine, gamma, step_ns, T):
    n, B = 14, 1024
    spec = open_spec(n, 2, T=T, drive=False, detuning=False, interaction=False, step_ns=step_ns)
    t_end = spec.sampling_times[-1]
    occ, jumps, st = _decay_run(engine, spec, [R.relaxation(spec.eigenbasis, gamma)], B, seed=31)
    f = 1.0 - occ[:, :, 0].mean(axis=1)  # decayed fraction of each trajectory
    np.testing.assert_allclose(f * n, jumps, atol=1e-9)
    exact = 1.0 - np.exp(-gamma * t_end)
    sigma = f.std(ddof=1) / np.sqrt(B)
    print(f"\n[decay] gamma={gamma}/us interval={step_ns} ns T={t_end * 1e3:.0f} ns: decayed {f.mean():.4f} vs exact "
          f"{exact:.4f}, diff {f.mean() - exact:+.4f}, 5 sigma = {5 * sigma:.4f}, steps = {st['n_steps']}")
    assert abs(f.mean() - exact) < 5 * sigma


def test_mcwf_population_statistics(engine):
    """Relaxation, dephasing and a general operator (non-diagonal L^+L): ensemble single-qudit populations against
    the product of single-qudit master equations."""
    n, B, T = 14, 1024, 300
    spec = open_spec(n, 2, T=T, drive=False, detuning=False, interaction=False)
    eig = spec.eigenbasis
    ops = np.concatenate([[R.relaxation(eig, 3.0)], [np.diag([np.sqrt(2 * 1.0), 0.0])], R.random_ops(2, 1, 1.5, 9)])
    t_end = spec.sampling_times[-1]
    occ, jumps, st = _decay_run(engine, spec, ops, B, seed=5)
    rho_r = np.zeros((2, 2), dtype=complex); rho_r[0, 0] = 1.0
    ref = np.real(np.diag(R.product_lindblad(spec, ops, rho_r, t_end)[0]))
    x = occ.mean(axis=1)  # [B, d]: qudit-averaged populations of each trajectory
    sigma = x.std(axis=0, ddof=1) / np.sqrt(B)
    print(f"\n[populations] mean {x.mean(axis=0)} vs ref {ref}, diff {x.mean(axis=0) - ref}, 5 sigma {5 * sigma}, "
          f"steps = {st['n_steps']}, jumps/trajectory = {jumps.mean():.2f}")
    assert np.all(np.abs(x.mean(axis=0) - ref) < 5 * sigma)


def test_mcwf_realistic_rates_keep_sampling_steps(engine):
    """At Pulser's default dephasing (0.05/us) and relaxation (0.01/us) rates with 1 ns sampling on 14 atoms the jump
    bound does not shorten the sampling interval: one step per interval."""
    n, T = 14, 200
    spec = open_spec(n, 2, T=T, seed=1, interaction=False)
    eig = spec.eigenbasis
    ops = [np.diag([np.sqrt(2 * 0.05), 0.0]), R.relaxation(eig, 0.01)]
    with engine.DevicePlan([spec] * 4) as plan:
        plan.set_collapse(np.asarray(ops, dtype=complex), seed=1)
        plan.set_state("all-ground")
        st = plan.propagate(0.0, spec.sampling_times[-1])
    print(f"\n[realistic] N={n}, {T} intervals of 1 ns: steps = {st['n_steps']}")
    assert st["n_steps"] <= T + 16  # pulse-edge sub-steps only
