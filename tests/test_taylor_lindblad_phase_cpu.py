"""The master equation under a moving drive phase, as the Taylor stage computes it
(``stage_d2_taylor_kernel<..., CPLX = true, DISS = true>`` and ``stage_d2_taylor_small_kernel<true, true>``), checked in
numpy against the dense Liouvillian.

On vec(rho) of N atoms, ``s = (r << N) | c``, atom k owns row bit 2N-1-k and column bit N-1-k.  With the drive of
atom k written as ``a_k unit omega(t)``, ``omega = x + i y``, ``lindblad.doubled_spec`` gives row qudit k the
coefficient ``a_k unit omega`` and column qudit k ``-conj(a_k unit omega)``.  The stage's per-bit table holds
``f = a_k unit`` on row bits and ``-conj(a_k unit)`` on column bits, and the drive part of H_j is ``x_j A + y_j B``:
    A chi[s] = sum_p f_p^(s) chi[s ^ 2^p]                       (f_p, or conj(f_p) where bit p of s is not to_bit)
    B chi[s] = i sum_p sg_p(s) f_p^(s) chi[s ^ 2^p],  sg_p(s) = +1 iff (bit p of s == to_bit) XOR (p < N)
i.e. the complex-drive signed sum whose sign changes on the column bits.  A step of one phase other than the plan's
(``rot``) runs A alone with the table of its own unit, which must conjugate on the column bits.
"""
from __future__ import annotations

import numpy as np
import pytest

from helpers import open_spec
from pulser_b200.lindblad import doubled_spec

TO_BIT = 0   # the drive's |to> digit (r = 0 in the r, g eigenbasis)


def flip(nbits: int, p: int, to_bit: int = TO_BIT) -> np.ndarray:
    """|to><from| on bit position p of an nbits register"""
    s = np.arange(2**nbits)
    m = np.zeros((2**nbits, 2**nbits))
    on = ((s >> p) & 1) == to_bit
    m[s[on], s[on] ^ (1 << p)] = 1.0
    return m


def drive_hamiltonian(coef: np.ndarray) -> np.ndarray:
    """sum_q (coef_q |to><from|_q + h.c.), qudit q at bit position n - 1 - q"""
    n = len(coef)
    h = np.zeros((2**n, 2**n), dtype=complex)
    for q, z in enumerate(coef):
        f = flip(n, n - 1 - q)
        h += z * f + np.conj(z) * f.T
    return h


def liouvillian_drive(coef: np.ndarray) -> np.ndarray:
    """H (x) I - I (x) H^T on row-major vec(rho): i times the drive part of the generator of -i [H, rho]"""
    h = drive_hamiltonian(coef)
    eye = np.eye(h.shape[0])
    return np.kron(h, eye) - np.kron(eye, h.T)


def stage_table(a: np.ndarray, unit: complex) -> np.ndarray:
    """per-bit factors of the stage's table on vec(rho) (taylor_table with the conjugating column rule):
    a unit on the row bit of atom k, -conj(a unit) on its column bit"""
    n = len(a)
    f = np.zeros(2 * n, dtype=complex)
    for k in range(n):
        f[2 * n - 1 - k] = a[k] * unit
        f[n - 1 - k] = -np.conj(a[k] * unit)
    return f


def stage_gathers(f: np.ndarray, chi: np.ndarray, n: int, to_bit: int = TO_BIT, col_sign: bool = True):
    """the stage's two partner sums from one set of partner loads: G = A chi and G' = B chi (the kernel's loop)"""
    nbits = 2 * n
    s = np.arange(2**nbits)
    p_sum = np.zeros(2**nbits, dtype=complex)
    q_sum = np.zeros(2**nbits, dtype=complex)
    for p in range(nbits):
        bit = (s >> p) & 1
        gx, gyt = f[p].real, f[p].imag
        gy = np.where(bit == to_bit, gyt, -gyt)
        z = (gx + 1j * gy) * chi[s ^ (1 << p)]
        sg = np.where((bit == to_bit) != (col_sign and p < n), 1.0, -1.0)
        p_sum += z
        q_sum += sg * z
    return p_sum, 1j * q_sum


def _omegas(rng, count):
    return rng.normal(size=count) + 1j * rng.normal(size=count)


@pytest.mark.parametrize("n", [1, 2, 3])
def test_doubled_spec_is_the_liouvillian(n):
    """doubled_spec's drive rows are the commutator's: column row k = -conj(row k) (what taylor_prepare recognises)"""
    spec = open_spec(n, 2, T=6, seed=n, interaction=False)
    d = doubled_spec(spec).drives[0].coef
    np.testing.assert_array_equal(d[n:], -np.conj(d[:n]))
    for i in range(d.shape[1]):
        np.testing.assert_allclose(drive_hamiltonian(d[:, i]), liouvillian_drive(spec.drives[0].coef[:, i]),
                                   atol=1e-14)


@pytest.mark.parametrize("kind", ["real", "rot", "cplx"])
@pytest.mark.parametrize("n", [1, 2, 3])
def test_xa_plus_yb_is_the_drive(kind, n):
    """x A + y B with the column-signed B equals the Liouvillian drive of a unit omega, for random complex omega.
    real: the table of the plan's unit; rot: the table of the step's own unit, omega real along it; cplx: the plan's
    unit, omega complex"""
    rng = np.random.default_rng(10 * n + len(kind))
    plan_unit = np.exp(1j * rng.uniform(-np.pi, np.pi))
    a = np.ones(n)
    for trial in range(4):
        if kind == "rot":
            unit = plan_unit * np.exp(1j * rng.uniform(-np.pi, np.pi))
            om = complex(rng.normal())
        else:
            unit = plan_unit
            om = _omegas(rng, 1)[0] if kind == "cplx" else complex(rng.normal())
        f = stage_table(a, unit)
        ref = liouvillian_drive(a * unit * om)
        chi = rng.normal(size=4**n) + 1j * rng.normal(size=4**n)
        g, g2 = stage_gathers(f, chi, n)
        np.testing.assert_allclose(om.real * g + om.imag * g2, ref @ chi, atol=1e-12 * np.linalg.norm(ref @ chi))


@pytest.mark.parametrize("n", [2, 3])
def test_batch_per_trajectory_factors(n):
    """SPAM batches: per-trajectory complex factors a_k (a bad atom has a_k = 0) keep their factors under the
    conjugating rule"""
    rng = np.random.default_rng(n)
    unit = np.exp(0.7j)
    for a in (rng.normal(size=n) + 1j * rng.normal(size=n), np.where(np.arange(n) == 1, 0.0, 1.0)):
        om = _omegas(rng, 1)[0]
        f = stage_table(a, unit)
        ref = liouvillian_drive(a * unit * om)
        chi = rng.normal(size=4**n) + 1j * rng.normal(size=4**n)
        g, g2 = stage_gathers(f, chi, n)
        np.testing.assert_allclose(om.real * g + om.imag * g2, ref @ chi, atol=1e-12 * np.linalg.norm(ref @ chi))


def test_column_sign_is_needed():
    """without the sign change on the column bits, B is not the drive's y-part"""
    n = 2
    rng = np.random.default_rng(5)
    f = stage_table(np.ones(n), np.exp(0.3j))
    chi = rng.normal(size=4**n) + 1j * rng.normal(size=4**n)
    _, g2 = stage_gathers(f, chi, n)
    _, g2_plain = stage_gathers(f, chi, n, col_sign=False)   # the single-state signed sum
    ref = liouvillian_drive(np.exp(0.3j) * np.full(n, 1j)) @ chi
    np.testing.assert_allclose(g2, ref, atol=1e-12 * np.linalg.norm(ref))
    assert np.linalg.norm(g2_plain - ref) > 0.1 * np.linalg.norm(ref)


def test_rot_table_conjugates():
    """the table of a rotated unit u_s: -conj(a u_s) on the column bits.  The constant-phase rule (the fit's column
    factor a_col = -conj(unit)^2 conj(a) / ..., times the unit it is uploaded with) holds for the plan's unit only"""
    n = 2
    rng = np.random.default_rng(7)
    unit = np.exp(0.4j)
    a = rng.normal(size=n) + 1j * rng.normal(size=n)
    # the fit's factor of column qudit k against the reference row a_0 unit omega: -conj(a_k unit) / (a_0 unit) a_0
    a_col = -np.conj(a * unit) / unit
    for u_s in (unit, unit * np.exp(1.1j), unit * np.exp(-2.5j)):
        f = stage_table(a, u_s)
        np.testing.assert_allclose(f[:n][::-1], -np.conj(a * u_s), atol=1e-15)
        old = a_col * u_s
        if u_s == unit:
            np.testing.assert_allclose(f[:n][::-1], old, atol=1e-15)
        else:
            assert np.max(np.abs(f[:n][::-1] - old)) > 1e-3
        om = complex(rng.normal())
        ref = liouvillian_drive(a * u_s * om)
        chi = rng.normal(size=4**n) + 1j * rng.normal(size=4**n)
        g, _ = stage_gathers(f, chi, n)
        np.testing.assert_allclose(om.real * g, ref @ chi, atol=1e-12 * np.linalg.norm(ref @ chi))
