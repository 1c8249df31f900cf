"""The open-system references of ``tests/open_ref.py`` against the dense-Lindblad oracle (``oracle.evolve.mesolve``)
and dense matrix exponentials, at N <= 3 with d = 2 and d = 3.  The GPU tests of the master-equation and quantum-jump
paths rest on these references."""
import numpy as np
import pytest
from scipy.linalg import expm

import open_ref as R
from helpers import open_spec

TOL = 1e-9


def _mesolve(spec, rho0, T):
    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    return evolve.mesolve(OracleHamiltonian.from_spec(spec), rho0, [0.0, T], rtol=1e-12, atol=1e-14)[-1]


def test_generator_matches_definition():
    """``vec(G rho) = vec(L rho L^+ - 1/2 {L^+L, rho})`` on random matrices, row-major vectorisation."""
    ops = R.random_ops(3, 2, 1.0, 0)
    G = R.single_qudit_generator(ops)
    rng = np.random.default_rng(1)
    rho = rng.normal(size=(3, 3)) + 1j * rng.normal(size=(3, 3))
    K = sum(L.conj().T @ L for L in ops)
    ref = sum(L @ rho @ L.conj().T for L in ops) - 0.5 * (K @ rho + rho @ K)
    np.testing.assert_allclose((G @ rho.reshape(-1)).reshape(3, 3), ref, atol=1e-14)


@pytest.mark.parametrize("d,n", [(2, 1), (2, 3), (3, 2)])
def test_pair_expm_apply_vs_mesolve(d, n):
    ops = R.random_ops(d, 2, 2.0, 10 * d + n)
    spec = open_spec(n, d, T=20, seed=n, drive=False, detuning=False, interaction=False, ops=ops)
    rho0 = R.random_density(d**n, 3, n)
    T = spec.sampling_times[-1]
    got = R.pair_expm_apply(rho0, [R.single_qudit_generator(ops)] * n, T)
    ref = _mesolve(spec, rho0, T)
    assert np.max(np.abs(got - ref)) < TOL
    assert np.max(np.abs(got - rho0)) > 1e-2  # the dissipator acted


@pytest.mark.parametrize("d,n", [(2, 2), (2, 3), (3, 2)])
def test_diagonal_lindblad_vs_mesolve(d, n):
    ops = R.random_diag_ops(d, 2, 3.0, 7 + d)
    spec = open_spec(n, d, T=30, seed=n + 1, drive=False, ops=ops)
    rho0 = R.random_density(d**n, 2, n + 5)
    T = spec.sampling_times[-1]
    got = R.diagonal_lindblad(rho0, spec, ops, T)
    ref = _mesolve(spec, rho0, T)
    assert np.max(np.abs(got - ref)) < TOL
    # the interaction and the detuning both rotate the coherences
    assert np.max(np.abs(np.angle(got[np.abs(got) > 1e-3] / rho0[np.abs(got) > 1e-3]))) > 0.1


@pytest.mark.parametrize("d,n", [(2, 1), (2, 3), (3, 2)])
def test_product_lindblad_vs_mesolve(d, n):
    eig = open_spec(1, d).eigenbasis
    ops = np.concatenate([R.random_diag_ops(d, 1, 2.0, 3), [R.relaxation(eig, 4.0)], R.random_ops(d, 1, 1.5, 4)])
    spec = open_spec(n, d, T=40, seed=n + 2, interaction=False, ops=ops)
    rho_k0 = [R.random_density(d, 2, 20 + k) for k in range(n)]
    T = spec.sampling_times[-1]
    got = R.kron_all(R.product_lindblad(spec, ops, rho_k0, T))
    ref = _mesolve(spec, R.kron_all(rho_k0), T)
    assert np.max(np.abs(got - ref)) < TOL
    # stopping early stops at the right time
    T2 = 0.37 * T
    got2 = R.kron_all(R.product_lindblad(spec, ops, rho_k0, T2))
    assert np.max(np.abs(got2 - _mesolve(spec, R.kron_all(rho_k0), T2))) < TOL


@pytest.mark.parametrize("d,n", [(2, 3), (3, 2)])
def test_no_jump_state_vs_dense(d, n):
    ops = R.random_ops(d, 2, 1.0, d + n)
    K = sum(L.conj().T @ L for L in ops)
    Ktot = sum(R.kron_all([K if j == k else np.eye(d) for j in range(n)]) for k in range(n))
    rng = np.random.default_rng(0)
    psi0 = rng.normal(size=(3, d**n)) + 1j * rng.normal(size=(3, d**n))
    T = 0.13
    ref = expm(-0.5 * T * Ktot) @ psi0.T
    ref = (ref / np.linalg.norm(ref, axis=0)).T
    np.testing.assert_allclose(R.no_jump_state(psi0, K, T), ref, atol=1e-13)
