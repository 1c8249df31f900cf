"""numpy restatement of the expectation kernels' formula, shared by the CPU and GPU tests of ``pulser_b200.opterms``:

    <psi|O|psi> = sum_terms c sum_s conj(psi_s) prod_k w_k[s_k] psi_{s'},  s' = s with digit (s_k + m_k) mod d on S.
"""
from __future__ import annotations

from collections import defaultdict

import numpy as np


def expect(terms, psi: np.ndarray) -> complex:
    psi = np.asarray(psi, dtype=np.complex128).reshape(-1)
    n, d = terms.n, terms.d
    idx = np.arange(d**n, dtype=np.int64)
    strides = [d ** (n - 1 - k) for k in range(n)]
    digits: dict = {}

    def digit(k):
        if k not in digits:
            digits[k] = ((idx // strides[k]) % d).astype(np.int8)
        return digits[k]

    # group the terms by their digit shifts, so that each partner vector is gathered once
    groups: dict = defaultdict(list)
    for c, sites in terms.terms:
        groups[tuple((k, m) for k, m, _ in sites if m)].append((c, sites))
    total = 0j
    for shifts, members in groups.items():
        partner = idx.copy()
        for k, m in shifts:
            a = digit(k).astype(np.int64)
            partner += (((a + m) % d) - a) * strides[k]
        q = psi.conj() * psi[partner]
        for c, sites in members:
            w = np.full(idx.shape, complex(c))
            for k, _, wk in sites:
                w *= np.asarray(wk, dtype=np.complex128)[digit(k)]
            total += complex(np.dot(w, q))
    return total


def random_operations(rng, eig, n, n_terms=4):
    """Random ``(coeff, [(qudit_op, qudits)])`` entries: 0-3 groups of 1-4 distinct qudits, random complex site matrices."""
    ops = []
    for _ in range(n_terms):
        groups = []
        free = list(rng.permutation(n))
        for _ in range(rng.integers(0, 4)):
            size = int(rng.integers(1, min(4, n) + 1))
            if len(free) < size:
                break
            groups.append((random_qudit_op(rng, eig), {int(k) for k in free[:size]}))
            free = free[size:]
        ops.append((complex(rng.normal(), rng.normal()), groups))
    return ops


def random_qudit_op(rng, eig, density=0.6):
    out = {}
    for a in eig:
        for b in eig:
            if rng.random() < density:
                out[a + b] = complex(rng.normal(), rng.normal())
    return out or {eig[0] + eig[0]: 1.0}
