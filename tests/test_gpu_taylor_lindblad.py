"""The master equation on the Taylor propagator (``LindbladPlan``, ``integrator = 3``): the dissipator inside the series
(``stage_d2_taylor_kernel<..., DISS = true>`` and ``stage_d2_taylor_small_kernel<false, true>``) against the exact
references of ``tests/open_ref.py``, the dense-Lindblad oracle, an exact piecewise-cubic evolution under the sparse
Liouvillian (held to the propagator's own ``err_estimate``) and the splitting path; and the refusals, with their reasons.
"""
from __future__ import annotations

import numpy as np
import pytest

import open_ref as R
from helpers import curved_spec, open_spec, with_dmm
from taylor_ref import PiecewiseCubicHamiltonian

pytestmark = pytest.mark.gpu

EIG = ["r", "g"]
SIGMA = {"x": np.array([[0, 1], [1, 0]], dtype=complex), "y": np.array([[0, -1j], [1j, 0]]),
         "z": np.array([[1, 0], [0, -1]], dtype=complex)}


def _ops(kind: str, seed: int = 0) -> np.ndarray:
    """Collapse operators of one qualifying channel (each L diagonal or each L off-diagonal)."""
    rng = np.random.default_rng(seed)
    if kind == "dephasing":
        return np.array([np.sqrt(2 * 3.0) * np.diag([1.0, 0.0])], dtype=complex)
    if kind == "relaxation":
        return np.array([R.relaxation(EIG, 4.0)])
    if kind == "dephasing+relaxation":
        return np.concatenate([_ops("dephasing"), _ops("relaxation")])
    if kind == "depolarizing":
        return np.array([np.sqrt(2.0 / 4) * SIGMA[a] for a in "xyz"])
    if kind == "random-diagonal":
        return R.random_diag_ops(2, 2, 3.0, seed)
    if kind == "random-offdiagonal":
        z = 2.0 * (rng.normal(size=(2, 2)) + 1j * rng.normal(size=(2, 2)))
        return np.array([[[0, z[i, 0]], [z[i, 1], 0]] for i in range(2)], dtype=complex)
    raise ValueError(kind)


def _fro(x) -> float:
    return float(np.linalg.norm(np.asarray(x).reshape(-1)))


def _lindblad(specs, rho0, t0=0.0, t1=None, **opts):
    from pulser_b200.lindblad import LindbladPlan

    with LindbladPlan(specs) as lp:
        if np.asarray(rho0).ndim == 3:
            lp.plan.set_state(np.ascontiguousarray(rho0).reshape(len(rho0), -1))
        else:
            lp.set_state(rho0)
        st = lp.propagate(t0, lp.specs[0].sampling_times[-1] if t1 is None else t1, **opts)
        return lp.get_rho(), st


def _const_phase(spec, seed: int = 0):
    """``spec`` with each qubit's drive at one constant phase (a moving phase is refused under a dissipator)"""
    rng = np.random.default_rng(seed)
    d = spec.drives[0]
    for k in range(spec.n_qudits):
        d.coef[k] = np.abs(d.coef[k]) * np.exp(1j * rng.uniform(-1, 1))
    return spec


@pytest.fixture(scope="module")
def engine(lib):
    from pulser_b200 import engine

    assert engine.device_count() > 0, "GPU tests need a CUDA device"
    return engine


# ---------------------------------------------------------------------------------------------------------------
# 1. H = 0: exp(T sum_k G_k) exactly, every qualifying channel, small and tiled kernels
@pytest.mark.parametrize("kind", ["dephasing", "relaxation", "depolarizing", "random-diagonal", "random-offdiagonal"])
@pytest.mark.parametrize("n,B", [(1, 1), (5, 1), (9, 1), (12, 1), (5, 3)])
def test_zero_hamiltonian(engine, kind, n, B):
    ops = _ops(kind, n)
    _zero_h_case(n, B, ops, f"{kind}")


def test_zero_hamiltonian_n13(engine):
    _zero_h_case(13, 1, _ops("dephasing+relaxation"), "dephasing+relaxation")


def _zero_h_case(n, B, ops, label):
    spec = open_spec(n, 2, T=20, drive=False, detuning=False, interaction=False, ops=ops)
    T = spec.sampling_times[-1]
    G = [R.single_qudit_generator(ops)] * n
    rho0 = np.stack([R.random_density(2**n, 4, 7 * n + b) for b in range(B)])
    refs = [R.pair_expm_apply(r, G, T) for r in rho0]
    assert min(_fro(r - r0) for r, r0 in zip(refs, rho0)) > 1e-3 * _fro(rho0[0])  # the dissipator acts
    rho, st = _lindblad([spec] * B, rho0 if B > 1 else rho0[0], integrator=3, tol=1e-12)
    assert st["integrator"] == 3
    err = max(np.max(np.abs(rho[b] - refs[b])) / _fro(refs[b]) for b in range(B))
    print(f"\n[zero-H] {label} N={n} B={B}: max |rho - ref| / |ref| = {err:.2e}, K total {st['n_applies']}")
    assert err < 1e-12


# ---------------------------------------------------------------------------------------------------------------
# 2. diagonal H (detuning + interaction) with dephasing: closed form
@pytest.mark.parametrize("n", [3, 10, 12])
def test_diagonal_dephasing(engine, n):
    ops = R.random_diag_ops(2, 2, 4.0, 10 + n)
    spec = open_spec(n, 2, T=40, seed=n, drive=False, ops=ops)
    rho0 = R.random_density(2**n, 3, n)
    ref = R.diagonal_lindblad(rho0, spec, ops, spec.sampling_times[-1])
    rho, st = _lindblad(spec, rho0, integrator=3)
    err = float(np.max(np.abs(rho[0] - ref)))
    print(f"\n[diagonal] N={n}: max |rho - ref| = {err:.2e}, err_estimate {st['err_estimate']:.1e}")
    assert st["integrator"] == 3 and err < 1e-10


# ---------------------------------------------------------------------------------------------------------------
# 3. driven non-interacting register: product of single-qubit master equations (per-qubit amplitudes, phases and
#    detunings: the several-shape DISS kernel)
@pytest.mark.parametrize("n", [4, 10, 12])
def test_driven_product(engine, n):
    ops = _ops("dephasing+relaxation")
    spec = _const_phase(open_spec(n, 2, T=40, seed=n + 2, interaction=False, ops=ops), n)
    T = spec.sampling_times[-1]
    rho_k0 = [R.random_density(2, 2, 20 + k) for k in range(n)]
    ref = R.kron_all(R.product_lindblad(spec, ops, rho_k0, T))
    rho, st = _lindblad(spec, R.kron_all(rho_k0), integrator=3, tol=1e-10)
    err = float(np.max(np.abs(rho[0] - ref)))
    print(f"\n[product] N={n}: max |rho - ref| = {err:.2e}, steps {st['n_steps']}, applies {st['n_applies']}")
    assert err < 1e-10


# ---------------------------------------------------------------------------------------------------------------
# 4. interacting registers against the dense-Lindblad oracle
@pytest.mark.parametrize("n,kind", [(2, "dephasing+relaxation"), (3, "dephasing+relaxation"), (4, "dephasing+relaxation"),
                                    (5, "dephasing+relaxation"), (3, "depolarizing")])
def test_interacting_against_mesolve(engine, n, kind):
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian
    from pulser_b200 import workloads as W

    amp, det = W.blockade_sweep_waveforms(t_rise=100, t_sweep=200, t_fall=100)
    spec = W.ising_global_spec(W.disc_register(n, 12.0, 5.0, 3), W.C6_LEVEL_60, amp, det)
    spec.collapse_ops = _ops(kind) * 0.3
    tf = spec.sampling_times[-1]
    psi0 = evolve.all_ground_state(spec)
    ref = evolve.mesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, tf], rtol=1e-12, atol=1e-14)[-1]
    for integrator in (0, 3):
        rho, st = _lindblad(spec, np.outer(psi0, psi0.conj()), tol=1e-10, integrator=integrator)
        err = float(np.max(np.abs(rho[0] - ref)))
        print(f"\n[mesolve] N={n} {kind} integrator={integrator}->{st['integrator']}: max |rho - ref| = {err:.2e}")
        assert st["integrator"] == 3 and err < 1e-8


# ---------------------------------------------------------------------------------------------------------------
# 5. the propagator's own error bound against an exact piecewise-cubic evolution under the sparse Liouvillian
class PiecewiseCubicLiouvillian(PiecewiseCubicHamiltonian):
    """``taylor_ref``'s exact cubic pieces on the doubled register, plus the static dissipator ``sum_k Gen_k`` on the
    (row k, column k) bit pairs: each sub-step's series gets ``h D chi_m`` at history 0."""

    def __init__(self, spec) -> None:
        from pulser_b200.lindblad import doubled_spec

        super().__init__(doubled_spec(spec))
        self.natoms = spec.n_qudits
        self.gen = R.single_qudit_generator(spec.collapse_ops).reshape(2, 2, 2, 2)
        self.gnorm = float(np.linalg.norm(R.single_qudit_generator(spec.collapse_ops), 2)) * self.natoms

    def dissipate(self, v: np.ndarray) -> np.ndarray:
        n = self.natoms
        x = v.reshape([2] * (2 * n))
        out = np.zeros_like(x)
        for k in range(n):
            out += np.moveaxis(np.tensordot(self.gen, x, axes=([2, 3], [k, n + k])), (0, 1), (k, n + k))
        return out.reshape(-1)

    def _evolve_piece(self, psi, i, ta, tb, gamma, half, split):
        from taylor_ref import _BINOM

        a_det, a_drive = self.det[:, i, :], self.drive[:, i, :]
        diag_l = [self._diag(a_det[l]) for l in range(4)]
        tm = max(abs(ta), abs(tb))
        pw = tm ** np.arange(4)
        bound = half + self.gnorm + float(np.sum(np.abs(a_det) * pw[:, None]) + np.sum(np.abs(a_drive) * pw[:, None]))
        nsub = split * max(1, int(np.ceil((tb - ta) * bound)))
        hs = (tb - ta) / nsub
        scale = np.linalg.norm(psi)
        for q in range(nsub):
            tau0 = ta + q * hs
            w = np.zeros((4, 4))
            for j in range(4):
                for l in range(j, 4):
                    w[j, l] = _BINOM[l, j] * tau0 ** (l - j) * hs**j
            diag = [hs * sum(w[j, l] * diag_l[l] for l in range(j, 4) if w[j, l] != 0.0) for j in range(4)]
            diag[0] = diag[0] + hs * (self.dint - gamma)
            cm = hs * (w @ a_drive).T
            terms = [psi]
            out = psi.copy()
            m = 0
            while True:
                hist = terms[-4:][::-1]
                y = np.zeros(self.D, dtype=complex)
                for j, v in enumerate(hist):
                    y += diag[j] * v
                for j, v in enumerate(hist):
                    if np.any(cm[:, j] != 0.0):
                        self._flip(cm[:, j], v, v, y)
                nxt = (-1j * y + hs * self.dissipate(hist[0])) / (m + 1)
                terms.append(nxt)
                out += nxt
                m += 1
                if m > 300:
                    raise RuntimeError("Taylor series of a sub-step did not converge")
                if m >= 4 and all(np.linalg.norm(v) < 1e-17 * scale for v in terms[-4:]):
                    break
                terms = terms[-4:]
            psi = out
        return psi * np.exp(-1j * gamma * (tb - ta))


@pytest.mark.parametrize("n,window", [(4, (0.0, 0.25)), (4, (0.1217, 0.1225)), (7, (0.05, 0.2)), (7, (0.1213, 0.1218))])
def test_own_error_bound(engine, n, window):
    spec = curved_spec(n, T=300, phase=0.4)
    spec.collapse_ops = _ops("dephasing+relaxation") * 0.5
    rho0 = R.random_density(2**n, 3, n)
    ref = PiecewiseCubicLiouvillian(spec).evolve(rho0.reshape(-1), *window).reshape(2**n, 2**n)
    rho, st = _lindblad(spec, rho0, *window, integrator=3, tol=1e-11)
    err = _fro(rho[0] - ref)
    print(f"\n[bound] N={n} window={window}: |d| = {err:.2e}, err_estimate = {st['err_estimate']:.2e}, "
          f"steps {st['n_steps']}, max rho {st['max_rho']:.1f}")
    assert st["err_estimate"] <= 1e-10
    assert err <= 2.0 * st["err_estimate"] + 1e-14 * _fro(rho0)


# ---------------------------------------------------------------------------------------------------------------
# 6. variants: detuning map, SPAM batch, Taylor against the splitting path
def test_detuning_map_with_dissipation(engine):
    n = 7
    spec = with_dmm(curved_spec(n, T=200), 2, seed=3)
    spec.collapse_ops = _ops("dephasing+relaxation") * 0.5
    rho0 = R.random_density(2**n, 2, 5)
    t1 = 0.12
    ref = PiecewiseCubicLiouvillian(spec).evolve(rho0.reshape(-1), 0.0, t1).reshape(2**n, 2**n)
    rho, st = _lindblad(spec, rho0, 0.0, t1, integrator=3, tol=1e-11)
    err = _fro(rho[0] - ref)
    print(f"\n[dmm] N={n}: |d| = {err:.2e}, err_estimate = {st['err_estimate']:.2e}")
    assert err <= 2.0 * st["err_estimate"] + 1e-14 * _fro(rho0)


def test_spam_batch_against_separate_runs(engine):
    from pulser_b200 import workloads as W

    n = 8
    amp, det = W.blockade_sweep_waveforms(t_rise=60, t_sweep=120, t_fall=60)
    base = W.ising_global_spec(W.disc_register(n, 12.0, 5.0, 3), W.C6_LEVEL_60, amp, det)
    base.collapse_ops = _ops("dephasing+relaxation") * 0.1
    specs = []
    for bad in ([], [1], [2, 5]):
        s = W.ising_global_spec(W.disc_register(n, 12.0, 5.0, 3), W.C6_LEVEL_60, amp, det)
        s.collapse_ops = base.collapse_ops
        s.bad_atoms = np.isin(np.arange(n), bad)
        for d in s.drives:   # a bad atom is neither driven nor detuned
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


def test_taylor_against_splitting_n12(engine):
    from pulser_b200 import workloads as W

    n = 12
    amp, det = W.blockade_sweep_waveforms(t_rise=50, t_sweep=100, t_fall=50)
    spec = W.ising_global_spec(W.disc_register(n, 16.0, 5.0, 3), W.C6_LEVEL_60, amp, det)
    spec.collapse_ops = np.concatenate([np.sqrt(2 * 0.05) * np.diag([1.0, 0.0])[None], R.relaxation(EIG, 0.01)[None]])
    psi0 = np.zeros(2**n, dtype=complex)
    psi0[-1] = 1.0
    rho_t, st_t = _lindblad(spec, psi0, tol=1e-10)
    rho_s, st_s = _lindblad(spec, psi0, integrator=1, tol=1e-10)
    err = float(np.max(np.abs(rho_t[0] - rho_s[0])))
    print(f"\n[split] N={n}: max |taylor - splitting| = {err:.2e}; {st_t['gpu_ms']:.0f} ms against {st_s['gpu_ms']:.0f} ms")
    assert st_t["integrator"] == 3 and st_s["integrator"] == 1
    assert err < 1e-8


# ---------------------------------------------------------------------------------------------------------------
# 7. refusals, with their reasons
def _refusal(spec) -> str:
    from pulser_b200._lib import PB200Error

    with pytest.raises(PB200Error) as e:
        _lindblad(spec, np.eye(1, spec.dim**spec.n_qudits)[0], integrator=3)
    return str(e.value)


def test_refuses_mixed_collapse_operator(engine):
    spec = open_spec(3, 2, T=40, interaction=False, ops=[np.array([[0.5, 0.0], [1.0, 0.0]])])
    assert "single-bit-flip entries" in _refusal(_const_phase(spec))
    spec.collapse_ops = R.random_ops(2, 2, 2.0, 1)
    assert "single-bit-flip entries" in _refusal(spec)


def test_refuses_moving_phase(engine):
    spec = open_spec(3, 2, T=40, interaction=False, ops=_ops("dephasing"))   # open_spec's phases move in time
    assert "drive phase moves" in _refusal(spec)


def test_refuses_three_levels(engine):
    spec = open_spec(3, 3, T=40, interaction=False, ops=R.random_diag_ops(3, 1, 2.0, 0))
    assert "d = 3" in _refusal(spec)


# ---------------------------------------------------------------------------------------------------------------
# 8. the facade: B200Emulator.run() with a dephasing + relaxation noise model reaches the Taylor path
def test_facade_noise_model_run(engine):
    from pulser_b200 import HAVE_PULSER

    if not HAVE_PULSER:
        pytest.skip("pulser-core not importable")
    import pulser
    from pulser.noise_model import NoiseModel
    from pulser.waveforms import ConstantWaveform, RampWaveform
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian
    from pulser_b200 import B200Emulator

    reg = pulser.Register.square(2, 6.0, prefix="q")
    seq = pulser.Sequence(reg, pulser.MockDevice)
    seq.declare_channel("ryd", "rydberg_global")
    om = 2 * np.pi * 1.5   # linear ramps: splines smooth enough for multi-interval polynomial steps
    seq.add(pulser.Pulse(RampWaveform(100, 0.0, om), ConstantWaveform(100, -3 * om), 0.0), "ryd")
    seq.add(pulser.Pulse(ConstantWaveform(200, om), RampWaveform(200, -3 * om, om), 0.0), "ryd")
    seq.add(pulser.Pulse(RampWaveform(100, om, 0.0), ConstantWaveform(100, om), 0.0), "ryd")
    noise = NoiseModel(dephasing_rate=0.5, relaxation_rate=0.2)
    emu = B200Emulator.from_sequence(seq, noise_model=noise, evaluation_times="Minimal")
    res = emu.run()
    spec = emu._current_spec
    assert len(spec.collapse_ops) > 0
    psi0 = evolve.all_ground_state(spec)
    ref = evolve.mesolve(OracleHamiltonian.from_spec(spec), psi0, [0.0, spec.sampling_times[-1]], rtol=1e-12,
                         atol=1e-14)[-1]
    got = np.asarray(res.get_final_state().full())
    err = float(np.max(np.abs(got - ref)))
    calls = len(emu._eval_times_array) - 1   # last_run_stats sums the calls' statistics
    print(f"\n[facade] max |rho - ref| = {err:.2e}, stats {emu.last_run_stats}")
    assert emu.last_run_stats["integrator"] == 3 * calls
    assert err < 1e-8
