"""CPU tests of the single-precision tail orders of the Taylor propagator: the host rule that picks a step's switch
order k_lo (pb200_host_taylor_lowprec) and its error bound, against the recurrence of stage_d2_taylor_kernel restated
in numpy with chi_{k+1} and G_k rounded to complex64 from order k_lo on, as the kernel stores them."""
import ctypes as C

import numpy as np
import pytest

from pulser_b200 import workloads as W

dp = C.POINTER(C.c_double)


def P(a):
    return a.ctypes.data_as(dp)


def order(lib, h, m, tol):
    k, tail = C.c_int32(), C.c_double()
    assert lib.pb200_host_taylor_order(h, P(m), len(m) - 1, tol, C.byref(k), C.byref(tail)) == 0
    return k.value


def lowprec(lib, h, m, K, g_stored, tol):
    k_lo, bound = C.c_int32(), C.c_double()
    assert lib.pb200_host_taylor_lowprec(h, P(m), len(m) - 1, K, int(g_stored), tol, C.byref(k_lo), C.byref(bound)) == 0
    return k_lo.value, bound.value


def taylor_step(h, diag, om, X, psi, K, k_lo=None):
    """psi(1) of (k+1) chi_{k+1} = -i h sum_j (D_j chi_{k-j} + om_j G_{k-j}),  G_k = X chi_k: every order k >= k_lo
    stores chi_{k+1} and G_k in single precision, and every later read (the next order's source, the history terms,
    the sum) sees the stored copy"""
    p = len(om) - 1
    store = lambda v, k: v.astype(np.complex64).astype(np.complex128) if k_lo is not None and k >= k_lo else v
    chi, G = [psi], []
    for k in range(K):
        G.append(store(X @ chi[k], k))
        s = diag[0] * chi[k] + om[0] * (X @ chi[k])
        for j in range(1, min(p, k) + 1):
            s = s + diag[j] * chi[k - j] + om[j] * G[k - j]
        chi.append(store(-1j * h / (k + 1) * s, k))
    return np.sum(chi, axis=0)


def random_problem(rng, n, p, rho):
    """a Hermitian X (the drive), diagonal D_j and drive coefficients om_j, scaled to h sum_j m_j / (j + 1) = rho"""
    A = rng.normal(size=(n, n)) + 1j * rng.normal(size=(n, n))
    X = (A + A.conj().T) / 2
    diag = rng.normal(size=(p + 1, n))
    om = rng.normal(size=p + 1)
    m = np.abs(diag).max(axis=1) + np.abs(om) * np.linalg.norm(X, 2)
    h = rho / np.sum(m / np.arange(1, p + 2))
    psi = rng.normal(size=n) + 1j * rng.normal(size=n)
    return h, diag, om, X, psi / np.linalg.norm(psi), m


@pytest.mark.parametrize("p,rho,tol", [(0, 14.0, 1e-9), (1, 10.0, 1e-10), (1, 14.0, 1e-7), (3, 6.0, 1e-6), (8, 4.0, 1e-8)])
def test_rounding_stays_within_the_bound(lib, p, rho, tol):
    rng = np.random.default_rng(100 + 10 * p + int(rho))
    h, diag, om, X, psi, m = random_problem(rng, 24, p, rho)
    K = order(lib, h, m, 1e-14)
    k_lo, bound = lowprec(lib, h, m, K, p >= 1, tol)
    assert 0 < k_lo < K and 0.0 < bound <= tol
    exact = taylor_step(h, diag, om, X, psi, K)
    low = taylor_step(h, diag, om, X, psi, K, k_lo)
    dev = np.linalg.norm(low - exact)
    assert 0.0 < dev <= bound


def test_switch_order_is_monotone_in_the_tolerance(lib):
    m = np.array([12.0, 3.0])
    K = order(lib, 1.0, m, 1e-13)
    prev = K
    for tol in (0.0, 1e-16, 1e-13, 1e-11, 1e-9, 1e-7, 1e-5, 1e-3):
        k_lo, bound = lowprec(lib, 1.0, m, K, True, tol)
        assert k_lo <= prev and bound <= tol
        prev = k_lo
    assert lowprec(lib, 1.0, m, K, True, 0.0) == (K, 0.0)
    assert lowprec(lib, 1.0, np.array([12.0]), K, False, 0.0) == (K, 0.0)


def test_c2_shaped_step_sends_fewer_orders_low_at_a_tighter_tolerance(lib):
    """a plateau step of C2 (rho = 14, the propagator's cap) and a ramp step (linear detuning: p = 1, G stored), with
    the scheduler's per-step share 0.1 rate h of the truncation and of the rounding"""
    spec = W.config_c2(n=20)
    T = spec.sampling_times[-1] - spec.sampling_times[0]
    h = 0.05
    for m, g in ((np.array([14.0 / h]), False), (np.array([12.0 / h, 4.0 / h]), True)):
        low = {}
        for gtol in (1e-8, 1e-12):
            rate = gtol / T
            K = order(lib, h, m, max(1e-15, 0.1 * rate * h))
            k_lo, bound = lowprec(lib, h, m, K, g, 0.1 * rate * h)
            assert bound <= 0.1 * rate * h
            low[gtol] = K - k_lo
        assert 0 < low[1e-12] < low[1e-8]
