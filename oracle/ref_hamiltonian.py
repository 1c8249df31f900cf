"""ORACLE (test infrastructure, never on the product path).

CPU restatement of ``pulser_simulation.hamiltonian.Hamiltonian`` with
scipy.sparse in place of qutip (qutip >= 5 is the pinned third-party
dependency that holds the arithmetic and is absent from this image,
``pulser-simulation/requirements.txt:1``).

PARITY PIN STATUS: Hamiltonian *assembly* is pinned against the reference's
own golden matrices (tests/test_oracle_golden.py <- reference
``tests/pulser_simulation/test_simulation.py:476-588``).  Evolved-state parity
against real QuTiP is pinned only at the loose tolerances of the reference's
own tests (rtol 1e-2 / atol 1e-5); at 1e-8 it is **parity unpinned** because
QuTiP cannot be executed here (see DESIGN.md).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline
legs may import this package.

Every function cites the reference lines it follows; paths are relative to
``pulser-simulation/pulser_simulation/`` of the Pulser repository.
"""
from __future__ import annotations

import itertools
from typing import Any, Sequence

import numpy as np
import scipy.sparse as sp

# hamiltonian.py:340-345
_OP_IDS = {
    "ground-rydberg": ("sigma_gr", "sigma_rr"),
    "digital": ("sigma_hg", "sigma_gg"),
    "XY": ("sigma_ud", "sigma_dd"),
}


def basis_op_matrices(eigenbasis: Sequence[str]) -> dict[str, sp.csr_matrix]:
    """hamiltonian.py:231-244 -- ``sigma_ab = |a><b|`` and ``I``."""
    d = len(eigenbasis)
    ops: dict[str, sp.csr_matrix] = {"I": sp.identity(d, format="csr", dtype=complex)}
    for i, a in enumerate(eigenbasis):
        for j, b in enumerate(eigenbasis):
            m = sp.lil_matrix((d, d), dtype=complex)
            m[i, j] = 1.0
            ops[f"sigma_{a}{b}"] = m.tocsr()
    return ops


def build_operator(
    n_qudits: int,
    op_matrix: dict[str, sp.csr_matrix],
    operations: Sequence[tuple[Any, Any]],
) -> sp.csr_matrix:
    """hamiltonian.py:145-200 -- tensor product, qubit 0 leftmost.

    ``operations`` = ``[(op_name_or_matrix, [qubit indices] | "global")]``.
    """
    op_list = [op_matrix["I"]] * n_qudits
    for operator, qubits in operations:
        if isinstance(qubits, str) and qubits == "global":
            return sum(
                build_operator(n_qudits, op_matrix, [(operator, [q])])
                for q in range(n_qudits)
            )
        if isinstance(operator, str):
            operator = op_matrix[operator]
        else:
            operator = sp.csr_matrix(np.asarray(operator, dtype=complex))
        op_list = list(op_list)
        for q in qubits:
            op_list[q] = operator
    out = op_list[0]
    for m in op_list[1:]:
        out = sp.kron(out, m, format="csr")
    return sp.csr_matrix(out)


class OracleHamiltonian:
    """``H(t) = sum_k coeff_k(t) A_k`` exactly as the reference assembles it.

    ``terms`` is the QobjEvo list *after* ``ham + ham.dag()``
    (hamiltonian.py:436-438): each entry is ``(csr, coeff)`` where ``coeff`` is
    ``None`` for a constant term or an array over ``sampling_times``.
    """

    def __init__(
        self,
        n_qudits: int,
        eigenbasis: Sequence[str],
        sampling_times: np.ndarray,
        terms: list[tuple[sp.csr_matrix, np.ndarray | None]],
        collapse_ops: list[sp.csr_matrix],
    ) -> None:
        self.n_qudits = n_qudits
        self.eigenbasis = list(eigenbasis)
        self.dim = len(eigenbasis)
        self.sampling_times = np.asarray(sampling_times, dtype=float)
        self.terms = terms
        self.collapse_ops = collapse_ops

    # ------------------------------------------------------------------
    @classmethod
    def from_spec(cls, spec: Any) -> "OracleHamiltonian":
        """Assemble from a plain-array ``HamiltonianSpec``.

        Follows hamiltonian.py:246-439 term by term (make_vdw_term :260-274,
        build_coeffs_ops :333-389, ``+ dag`` :437).
        """
        n = spec.n_qudits
        ops = basis_op_matrices(spec.eigenbasis)
        qobj_list: list[tuple[sp.csr_matrix, np.ndarray | None]] = []
        bad = np.asarray(spec.bad_atoms, dtype=bool)
        effective_size = n - int(bad.sum())
        if "digital" not in spec.basis_name and effective_size > 1:
            slm = set(int(t) for t in spec.slm_targets)

            def make_interaction_term(masked: bool = False) -> sp.csr_matrix:
                # hamiltonian.py:296-331
                inter = sp.csr_matrix((spec.dim**n, spec.dim**n), dtype=complex)
                if masked:
                    eff = n - int(bad.sum()) - sum(1 for q in slm if not bad[q])
                    if eff < 2:
                        return inter
                for q1, q2 in itertools.combinations(range(n), 2):
                    if bad[q1] or bad[q2]:
                        continue
                    if masked and spec.interaction_type == "XY" and (q1 in slm or q2 in slm):
                        continue
                    if spec.interaction_type == "XY":  # make_xy_term, hamiltonian.py:276-294
                        u_xy = spec.interaction_matrix[0, q1, q2]
                        u_ryd = spec.interaction_matrix[1, q1, q2]
                        inter = inter + u_xy * build_operator(
                            n, ops, [("sigma_ud", [q1]), ("sigma_du", [q2])]
                        ) + 0.5 * u_ryd * build_operator(n, ops, [("sigma_uu", [q1, q2])])
                    else:  # make_vdw_term, hamiltonian.py:260-274
                        u = 0.5 * spec.interaction_matrix[-1, q1, q2]
                        inter = inter + u * build_operator(
                            n, ops, [("sigma_rr", [q1, q2])]
                        )
                return sp.csr_matrix(inter)

            if spec.interaction_type == "XY" and spec.slm_end > 0:
                # hamiltonian.py:399-424: binary coefficient arrays for the two interaction terms
                duration = int(spec.total_duration_ns) + 1
                coeff = np.ones(duration - 1)
                coeff[0 : spec.slm_end] = 0
                idx = np.linspace(0, len(coeff) - 1, len(spec.sampling_times), dtype=int)
                qobj_list.append((make_interaction_term(), coeff[idx]))
                qobj_list.append(
                    (make_interaction_term(masked=True), np.logical_not(coeff).astype(int)[idx].astype(float))
                )
            else:
                qobj_list.append((make_interaction_term(), None))
        for drv in spec.drives:
            op_ids = _OP_IDS[drv.basis]
            if drv.uniform:
                coeffs = [drv.coef[0], -0.5 * drv.det[0]]
                for op_id, coeff in zip(op_ids, coeffs):
                    if np.any(coeff != 0):
                        qobj_list.append(
                            (build_operator(n, ops, [(op_id, "global")]), coeff)
                        )
            else:
                for q in range(n):
                    coeffs = [drv.coef[q], -0.5 * drv.det[q]]
                    for op_id, coeff in zip(op_ids, coeffs):
                        if np.any(coeff != 0):
                            qobj_list.append(
                                (build_operator(n, ops, [(op_id, [q])]), coeff)
                            )
        if not qobj_list:
            qobj_list = [
                (sp.csr_matrix((spec.dim**n, spec.dim**n), dtype=complex), None)
            ]
        # ham + ham.dag()  (hamiltonian.py:437)
        terms = list(qobj_list)
        for a, c in qobj_list:
            terms.append(
                (sp.csr_matrix(a.conj().T), None if c is None else np.conj(c))
            )
        c_ops = []
        for m in spec.collapse_ops:  # hamiltonian.py:121-124
            for q in range(n):
                c_ops.append(build_operator(n, ops, [(m, [q])]))
        return cls(n, spec.eigenbasis, spec.sampling_times, terms, c_ops)

    @classmethod
    def from_pulser(
        cls,
        samples: Any,
        noise_trajectory: Any,
        basis_data: Any,
        lindblad_data: Any,
        sampling_rate: float,
    ) -> "OracleHamiltonian":
        """Assemble directly from the reference constructor's arguments.

        Independent of ``pulser_b200.spec`` on purpose: walks
        ``samples.to_nested_dict()`` itself the way hamiltonian.py:426-431
        does, so that it also checks the product's spec extraction.
        """
        register = noise_trajectory.register
        qids = list(register.qubits)
        qidx = {q: i for i, q in enumerate(qids)}
        n = len(qids)
        eig = list(basis_data.eigenbasis)
        d = len(eig)
        ops = basis_op_matrices(eig)
        duration = samples.max_duration

        def adapt(arr: np.ndarray) -> np.ndarray:  # hamiltonian.py:87-95
            idx = np.linspace(
                0, len(arr) - 1, int(sampling_rate * duration), dtype=int
            )
            return np.asarray(arr)[idx]

        times = adapt(np.arange(duration, dtype=np.double) / 1000)
        qobj_list: list[tuple[sp.csr_matrix, np.ndarray | None]] = []
        bad = {q: bool(noise_trajectory.bad_atoms[q]) for q in qids}
        effective_size = n - sum(bad.values())
        imat = noise_trajectory.interaction_matrix.as_array(detach=True)
        if "digital" not in basis_data.basis_name and effective_size > 1:
            slm = set(samples._slm_mask.targets)

            def make_interaction_term(masked: bool = False) -> sp.csr_matrix:
                inter = sp.csr_matrix((d**n, d**n), dtype=complex)
                if masked:
                    eff = n - sum(bad.values()) - sum(1 for q in slm if not bad[q])
                    if eff < 2:
                        return inter
                for q1, q2 in itertools.combinations(qids, 2):
                    if bad[q1] or bad[q2]:
                        continue
                    if masked and basis_data.interaction_type == "XY" and (q1 in slm or q2 in slm):
                        continue
                    i1, i2 = qidx[q1], qidx[q2]
                    if basis_data.interaction_type == "XY":
                        inter = inter + imat[0, i1, i2] * build_operator(
                            n, ops, [("sigma_ud", [i1]), ("sigma_du", [i2])]
                        ) + 0.5 * imat[1, i1, i2] * build_operator(n, ops, [("sigma_uu", [i1, i2])])
                    else:
                        inter = inter + 0.5 * imat[-1, i1, i2] * build_operator(
                            n, ops, [("sigma_rr", [i1, i2])]
                        )
                return sp.csr_matrix(inter)

            if basis_data.interaction_type == "XY" and samples._slm_mask.end > 0:
                coeff = np.ones(duration - 1)  # hamiltonian.py:405-407
                coeff[0 : samples._slm_mask.end] = 0
                qobj_list.append((make_interaction_term(), adapt(coeff)))
                qobj_list.append(
                    (make_interaction_term(masked=True), adapt(np.logical_not(coeff).astype(int)).astype(float))
                )
            else:
                qobj_list.append((make_interaction_term(), None))
        nested = samples.to_nested_dict()
        for addr in nested:
            for basis in nested[addr]:
                if not nested[addr][basis]:
                    continue
                op_ids = _OP_IDS[basis]
                if addr == "Global":
                    s = nested[addr][basis]
                    coeffs = [
                        0.5 * s["amp"] * np.exp(-1j * s["phase"]),
                        -0.5 * s["det"],
                    ]
                    for op_id, coeff in zip(op_ids, coeffs):
                        if np.any(coeff != 0):
                            qobj_list.append(
                                (
                                    build_operator(n, ops, [(op_id, "global")]),
                                    adapt(coeff),
                                )
                            )
                else:
                    for qid, s in nested[addr][basis].items():
                        coeffs = [
                            0.5 * s["amp"] * np.exp(-1j * s["phase"]),
                            -0.5 * s["det"],
                        ]
                        for coeff, op_id in zip(coeffs, op_ids):
                            if np.any(coeff != 0):
                                qobj_list.append(
                                    (
                                        build_operator(
                                            n, ops, [(op_id, [qidx[qid]])]
                                        ),
                                        adapt(coeff),
                                    )
                                )
        if not qobj_list:
            qobj_list = [(sp.csr_matrix((d**n, d**n), dtype=complex), None)]
        terms = list(qobj_list)
        for a, c in qobj_list:
            terms.append(
                (sp.csr_matrix(a.conj().T), None if c is None else np.conj(c))
            )
        # collapse operators, hamiltonian.py:97-124
        c_ops = []
        for coeff, cop in lindblad_data.local_collapse_ops:
            if isinstance(cop, str):
                if cop not in ops:
                    m = sum(
                        coeff * pc * ops[pn]
                        for pc, pn in lindblad_data.depolarizing_pauli_2ds[cop]
                    )
                else:
                    m = coeff * ops[cop]
                m = m.toarray()
            else:
                m = coeff * np.asarray(cop, dtype=complex)
            for q in range(n):
                c_ops.append(build_operator(n, ops, [(m, [q])]))
        return cls(n, eig, times, terms, c_ops)

    # ------------------------------------------------------------------
    def coefficient_functions(self, order: int = 3) -> list[Any]:
        """Interpolants of the array coefficients over ``sampling_times``.

        QuTiP 5 ``coefficient(array, tlist=..., order=3)`` (third-party, from
        its public documentation): order 0 = previous-value step, 1 = linear,
        >= 2 = ``scipy.interpolate.make_interp_spline(tlist, arr, k=order)``
        (not-a-knot for cubic).  Kept switchable (SURVEY Appendix C.3).
        """
        from scipy.interpolate import make_interp_spline

        t = self.sampling_times
        fns = []
        for _, c in self.terms:
            if c is None:
                fns.append(None)
            elif order == 0:
                cc = np.asarray(c)

                def f(x, cc=cc, t=t):
                    i = np.clip(np.searchsorted(t, x, side="right") - 1, 0, len(t) - 1)
                    return cc[i]

                fns.append(f)
            else:
                fns.append(make_interp_spline(t, np.asarray(c), k=order))
        return fns

    def matrix_at(self, t_us: float, order: int = 3, fns: list | None = None) -> sp.csr_matrix:
        """``QobjEvo.__call__(t)`` -- used by ``get_hamiltonian``
        (simulation.py:656-661)."""
        fns = fns if fns is not None else self.coefficient_functions(order)
        out = None
        for (a, _), f in zip(self.terms, fns):
            m = a if f is None else a * complex(f(t_us))
            out = m if out is None else out + m
        return sp.csr_matrix(out)
