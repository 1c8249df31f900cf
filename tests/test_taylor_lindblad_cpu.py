"""The dissipator as the Taylor stage applies it (``stage_d2_taylor_kernel<..., DISS = true>``), checked in numpy against
the dense Liouvillian of ``lindblad.dissipator_generator`` and against the definition of the master equation.

On vec(rho) of N atoms, ``s = (r << N) | c``, atom k owns row bit 2N-1-k and column bit N-1-k.  When every atom carries
the same generator ``Gen`` and no entry of ``Gen`` flips exactly one bit of the pair, the dissipator is
    diagonal   w0 + wr popc(r) + wc popc(c) + wrc popc(r & c)
    both-flip  sum_k f[i_k(s)] chi[s ^ 2^(2N-1-k) ^ 2^(N-1-k)],   i_k = 2 row bit + column bit,  f[i] = Gen[i, 3 - i]
which is what the kernel computes.  Its 2-norm is at most N max(row sum, column sum) of Gen (the step-length bound).
"""
from __future__ import annotations

import numpy as np
import pytest

import open_ref as R
from pulser_b200.lindblad import dissipator_generator

X = np.array([[0, 1], [1, 0]], dtype=complex)
Y = np.array([[0, -1j], [1j, 0]])
Z = np.diag([1.0, -1.0]).astype(complex)


def _offdiag_ops(seed):
    rng = np.random.default_rng(seed)
    z = rng.normal(size=(2, 2)) + 1j * rng.normal(size=(2, 2))
    return np.array([[[0, z[i, 0]], [z[i, 1], 0]] for i in range(2)])


CHANNELS = {
    "dephasing": np.sqrt(0.05 / 2) * Z[None],
    "relaxation": R.relaxation(["r", "g"], 0.3)[None],
    "dephasing+relaxation": np.concatenate([np.sqrt(0.05 / 2) * Z[None], R.relaxation(["r", "g"], 0.3)[None]]),
    "depolarizing": np.array([np.sqrt(0.4 / 4) * P for P in (X, Y, Z)]),
    "random-diagonal": R.random_diag_ops(2, 2, 1.5, 3),
    "random-offdiagonal": _offdiag_ops(4),
}


def single_bit_entries(gen: np.ndarray) -> float:
    """largest |Gen[i, j]| over the entries that flip exactly one bit of the (row, column) pair"""
    i, j = np.meshgrid(np.arange(4), np.arange(4), indexing="ij")
    return float(np.max(np.abs(gen[((i ^ j) == 1) | ((i ^ j) == 2)])))


def qualifies(gen: np.ndarray) -> bool:
    return single_bit_entries(gen) <= 1e-15 * np.max(np.abs(gen))


def decomposed_apply(gen: np.ndarray, n: int, v: np.ndarray) -> np.ndarray:
    """the kernel's popcount diagonal + both-flip gather on vec(rho) of n atoms"""
    g = np.diag(gen)
    f = np.array([gen[i, 3 - i] for i in range(4)])
    w0, wr, wc, wrc = n * g[0], g[2] - g[0], g[1] - g[0], g[0] - g[1] - g[2] + g[3]
    s = np.arange(4**n)
    r, c = s >> n, s & ((1 << n) - 1)
    popc = np.vectorize(lambda x: bin(int(x)).count("1"))
    out = (w0 + wr * popc(r) + wc * popc(c) + wrc * popc(r & c)) * v
    for k in range(n):
        pr, pc = 2 * n - 1 - k, n - 1 - k
        i = 2 * ((s >> pr) & 1) + ((s >> pc) & 1)
        out = out + f[i] * v[s ^ (1 << pr) ^ (1 << pc)]
    return out


def dense_dissipator(ops: np.ndarray, n: int, rho: np.ndarray) -> np.ndarray:
    """sum_k sum_L L_k rho L_k^+ - 1/2 {L_k^+ L_k, rho} with L_k = L on atom k (atom 0 most significant)"""
    out = np.zeros_like(rho)
    for k in range(n):
        for L in ops:
            Lk = R.kron_all([L if j == k else np.eye(2) for j in range(n)])
            K = Lk.conj().T @ Lk
            out += Lk @ rho @ Lk.conj().T - 0.5 * (K @ rho + rho @ K)
    return out


@pytest.mark.parametrize("kind", sorted(CHANNELS))
@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_decomposition_matches_dense_liouvillian(kind, n):
    ops = CHANNELS[kind]
    gen = dissipator_generator(ops)
    assert qualifies(gen)
    rng = np.random.default_rng(n)
    rho = rng.normal(size=(2**n, 2**n)) + 1j * rng.normal(size=(2**n, 2**n))
    got = decomposed_apply(gen, n, rho.reshape(-1)).reshape(2**n, 2**n)
    ref = dense_dissipator(ops, n, rho)
    np.testing.assert_allclose(got, ref, atol=1e-13 * np.max(np.abs(ref)))


@pytest.mark.parametrize("kind", sorted(CHANNELS))
def test_norm_bound(kind):
    gen = dissipator_generator(CHANNELS[kind])
    n = 3
    dense = np.stack([decomposed_apply(gen, n, e) for e in np.eye(4**n)], axis=1)
    rows = max(abs(gen[i, i]) + abs(gen[i, 3 - i]) for i in range(4))
    cols = max(abs(gen[i, i]) + abs(gen[3 - i, i]) for i in range(4))
    assert np.linalg.norm(dense, 2) <= n * max(rows, cols) * (1 + 1e-12)


def test_qualification_rule():
    # an operator that mixes diagonal and off-diagonal elements, and a general random one, flip single bits
    mixed = np.array([[[0.5, 0.0], [1.0, 0.0]]], dtype=complex)
    assert single_bit_entries(dissipator_generator(mixed)) > 0.1
    assert not qualifies(dissipator_generator(mixed))
    assert not qualifies(dissipator_generator(R.random_ops(2, 2, 1.0, 7)))
    # the same operators split into a diagonal and an off-diagonal one qualify
    assert qualifies(dissipator_generator(np.array([np.diag([0.5, 0.0]), [[0.0, 0.0], [1.0, 0.0]]], dtype=complex)))
