"""Operators of Pulser's operator representation as lists of monomial terms: expectations without the matrix.

Every single-qudit ``d x d`` matrix ``O`` splits into at most ``d`` monomial matrices by digit shift ``m``:
``M_m[a, (a + m) mod d] = O[a, (a + m) mod d]``, kept when non-zero.  A term ``c prod_{k in S} O_k`` therefore
expands into ``prod_k (#non-zero shifts of O_k)`` monomial terms ``c (x)_{k in S} (w_k, m_k)``, and

    <psi| c (x)_k (w_k, m_k) |psi> = c sum_s conj(psi_s) prod_k w_k[s_k] psi_{s'},

where ``s'`` has the digit ``(s_k + m_k) mod d`` at every ``k in S`` (qudit 0 = most significant digit).  Pauli
strings, sigma+-, projectors, parity (Z) and X strings over all sites are one monomial term each.

This module owns that format.  ``B200Operator`` carries an ``OpTerms`` beside its lazily built matrix, and
``OpTerms.c_desc()`` packs it for ``pb200_state_expect`` / ``pb200_shards_expect`` (``include/pulser_b200.h``).
"""
from __future__ import annotations

import ctypes as C
import itertools
import math
from typing import Any, Mapping, Sequence

import numpy as np

# largest number of monomial terms after expansion; an operator above it has no compiled form (its matrix is used)
MAX_TERMS = 1 << 14

# one monomial term: (coeff, ((site, shift, weights), ...)) with the sites in increasing order, weights a tuple of d
Term = tuple[complex, tuple[tuple[int, int, tuple[complex, ...]], ...]]


def _monomials(mat: np.ndarray) -> list[tuple[int, tuple[complex, ...]]] | None:
    """The non-zero shifts of a site matrix, ``[(m, w)]``; ``[]`` for the identity, ``None`` for the zero matrix."""
    d = mat.shape[0]
    if np.array_equal(mat, np.eye(d)):
        return []
    out = []
    for m in range(d):
        w = tuple(complex(mat[a, (a + m) % d]) for a in range(d))
        if any(w):
            out.append((m, w))
    return out or None


def _site_product(d: int, x: tuple[int, tuple], y: tuple[int, tuple]) -> tuple[int, tuple] | None:
    """``(w1, m1) @ (w2, m2)``: shift ``m1 + m2``, ``w[a] = w1[a] w2[a + m1]``; ``None`` when it vanishes."""
    (m1, w1), (m2, w2) = x, y
    w = tuple(w1[a] * w2[(a + m1) % d] for a in range(d))
    return ((m1 + m2) % d, w) if any(w) else None


class OpTerms:
    """``sum_t c_t (x)_{k in S_t} (w_k, m_k)`` over ``n`` qudits of dimension ``d``."""

    __slots__ = ("n", "d", "terms", "_packed")

    def __init__(self, n: int, d: int, terms: Sequence[Term]):
        self.n, self.d = int(n), int(d)
        self.terms: tuple[Term, ...] = tuple(terms)
        self._packed: tuple[np.ndarray, ...] | None = None

    def __len__(self) -> int:
        return len(self.terms)

    @classmethod
    def from_operations(cls, operations: Sequence[tuple[complex, Sequence[tuple[Mapping[str, complex], set]]]],
                        eigenstates: Sequence[str], n_qudits: int) -> "OpTerms | None":
        """The monomial terms of Pulser's operator representation (validated ``(coeff, [(qudit_op, qudits)])``
        entries), or ``None`` above ``MAX_TERMS``.  A qudit named by several groups of one term takes the last one,
        like the matrix ``B200Operator._from_operator_repr`` builds (``qutip_op.py:148-218``)."""
        d = len(eigenstates)
        terms: list[Term] = []
        for coeff, tensor_op in operations:
            factors: dict[int, np.ndarray] = {}
            for qop, inds in tensor_op:
                mat = np.zeros((d, d), dtype=np.complex128)
                for key, val in qop.items():
                    mat[eigenstates.index(key[0]), eigenstates.index(key[1])] += complex(val)
                for k in inds:
                    factors[int(k)] = mat
            per_site = []
            for k in sorted(factors):
                monos = _monomials(factors[k])
                if monos is None:  # a zero factor: the term vanishes
                    break
                if monos:
                    per_site.append([(k, m, w) for m, w in monos])
            else:
                if complex(coeff) == 0:
                    continue
                if len(terms) + math.prod(len(p) for p in per_site) > MAX_TERMS:
                    return None
                terms.extend((complex(coeff), combo) for combo in itertools.product(*per_site))
        return cls(n_qudits, d, terms)

    # ---- arithmetic: the compiled form of +, scalar * and @ -------------------------------------------------------
    def compatible(self, other: "OpTerms") -> bool:
        """Both act on the same number of qudits of the same dimension."""
        return (self.n, self.d) == (other.n, other.d)

    def _check_compatible(self, other: "OpTerms", op: str) -> None:
        if not self.compatible(other):
            raise ValueError(f"Can't apply {op} between operators on {self.n} and {other.n} qudits of dimensions "
                             f"{self.d} and {other.d}.")

    def __add__(self, other: "OpTerms") -> "OpTerms | None":
        self._check_compatible(other, "+")
        if len(self) + len(other) > MAX_TERMS:
            return None
        return OpTerms(self.n, self.d, self.terms + other.terms)

    def scaled(self, scalar: complex) -> "OpTerms":
        s = complex(scalar)
        return OpTerms(self.n, self.d, [(s * c, sites) for c, sites in self.terms])

    def __matmul__(self, other: "OpTerms") -> "OpTerms | None":
        self._check_compatible(other, "@")
        if len(self) * len(other) > MAX_TERMS:
            return None
        d = self.d
        out: list[Term] = []
        for (c1, s1), (c2, s2) in itertools.product(self.terms, other.terms):
            sites = {k: (m, w) for k, m, w in s1}
            for k, m, w in s2:
                if k not in sites:
                    sites[k] = (m, w)
                    continue
                prod = _site_product(d, sites[k], (m, w))
                if prod is None:
                    break
                sites[k] = prod
            else:
                ident = (0, (1.0,) * d)
                out.append((c1 * c2, tuple((k, m, w) for k, (m, w) in sorted(sites.items()) if (m, w) != ident)))
        return OpTerms(self.n, self.d, out)

    # ---- Hermiticity without the matrix -----------------------------------------------------------------------------
    def adjoint(self) -> "OpTerms":
        """Site by site, the adjoint of ``(w, m)`` is shift ``-m mod d`` with ``w'[b] = conj(w[(b - m) mod d])``."""
        d = self.d
        return OpTerms(self.n, d, [
            (complex(c).conjugate(),
             tuple((k, (-m) % d, tuple(complex(w[(b - m) % d]).conjugate() for b in range(d))) for k, m, w in sites))
            for c, sites in self.terms])

    def _canonical(self) -> dict:
        """Terms keyed by their sites, each site scaled so that its first non-zero weight is 1 (the scale moves into
        the coefficient), terms with identical sites merged: ``{key: coeff}``.  The keys hold the exact weights, so
        only identical terms merge (complex division and products are exact under conjugation, so the adjoint of a
        canonical list closed under adjoints reproduces its keys bit for bit)."""
        out: dict = {}
        for c, sites in self.terms:
            key = []
            for k, m, w in sites:
                w = np.asarray(w, dtype=np.complex128)
                lead = w[np.flatnonzero(w)[0]]
                c = c * lead
                key.append((k, m, tuple(complex(x) for x in w / lead)))
            key = tuple(key)
            out[key] = out.get(key, 0j) + c
        return out

    def adjoint_matches(self, rtol: float = 1e-12) -> bool:
        """True when the canonical term list equals the one of the adjoint to ``rtol``: the operator is Hermitian.
        False decides nothing (the same operator may be Hermitian in another decomposition)."""
        a, b = self._canonical(), self.adjoint()._canonical()
        scale = max([abs(c) for c in a.values()] + [abs(c) for c in b.values()] + [0.0])
        if scale == 0.0:
            return True
        tol = rtol * scale
        a = {k: c for k, c in a.items() if abs(c) > tol}
        b = {k: c for k, c in b.items() if abs(c) > tol}
        return a.keys() == b.keys() and all(abs(c - b[k]) <= tol for k, c in a.items())

    # ---- the C-ABI form -----------------------------------------------------------------------------------------------
    def arrays(self) -> tuple[np.ndarray, np.ndarray, np.ndarray, np.ndarray, np.ndarray]:
        """``coeff[T]`` (complex), ``site_start[T + 1]``, ``site[E]``, ``shift[E]`` (int32), ``weight[E, d]``."""
        coeff = np.array([c for c, _ in self.terms], dtype=np.complex128)
        site_start = np.zeros(len(self.terms) + 1, dtype=np.int32)
        site_start[1:] = np.cumsum([len(s) for _, s in self.terms])
        flat = [e for _, sites in self.terms for e in sites]
        site = np.array([k for k, _, _ in flat], dtype=np.int32)
        shift = np.array([m for _, m, _ in flat], dtype=np.int32)
        weight = np.array([w for _, _, w in flat], dtype=np.complex128).reshape(len(flat), self.d)
        return coeff, site_start, site, shift, weight

    def c_desc(self) -> Any:
        """``pb200_op_terms`` pointing into arrays owned by this object (packed once; keep the object alive while the
        descriptor is in use).  The descriptor itself is built per call: an object holding ctypes pointers could not
        be deep-copied, and Pulser deep-copies the observables of a config."""
        from ._lib import OpTermsDesc

        if self._packed is None:
            self._packed = tuple(np.ascontiguousarray(a) for a in self.arrays())
        coeff, site_start, site, shift, weight = self._packed
        i32 = C.POINTER(C.c_int32)
        dp = C.POINTER(C.c_double)
        return OpTermsDesc(len(self.terms), coeff.ctypes.data_as(dp), site_start.ctypes.data_as(i32),
                           site.ctypes.data_as(i32), shift.ctypes.data_as(i32), weight.ctypes.data_as(dp))
