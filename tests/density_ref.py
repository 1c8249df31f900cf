"""Dense numpy forms shared by the CPU and GPU tests of the density-matrix reductions (``pb200_density_*``)."""
from __future__ import annotations

import numpy as np


def terms_matrix(terms) -> np.ndarray:
    """The D x D matrix of an operator given as monomial terms: term t puts c prod_k w_k[r_k] at (r, shift_t(r))."""
    n, d = terms.n, terms.d
    idx = np.arange(d**n, dtype=np.int64)
    out = np.zeros((d**n, d**n), dtype=np.complex128)
    for c, sites in terms.terms:
        partner = idx.copy()
        w = np.full(idx.shape, complex(c))
        for k, m, wk in sites:
            st = d ** (n - 1 - k)
            a = (idx // st) % d
            partner += (((a + m) % d) - a) * st
            w *= np.asarray(wk, dtype=np.complex128)[a]
        np.add.at(out, (idx, partner), w)
    return out


def number_masks(n: int, d: int, digit: int) -> np.ndarray:
    """``[N, D]`` booleans: digit k of basis state r equals ``digit``."""
    idx = np.arange(d**n)
    return np.stack([(idx // d ** (n - 1 - k)) % d == digit for k in range(n)])
