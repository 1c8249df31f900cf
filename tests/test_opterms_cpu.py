"""CPU tests of the compiled form of operators (``pulser_b200.opterms``): monomial terms against the matrices
``B200Operator`` builds, the arithmetic, the Hermiticity decision, and the backend's device path run on a fake plan."""
import numpy as np
import pytest
import scipy.sparse as sp

import opterms_ref
from fake_device import FakeDevicePlan
from pulser_b200 import HAVE_PULSER

pytestmark = pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable here")

EIGS = {2: ("r", "g"), 3: ("u", "d", "x"), 4: ("g", "r", "h", "x")}


class FakeTermsPlan(FakeDevicePlan):
    """The oracle-backed plan with ``expect_terms`` answered by the numpy restatement of the kernel."""

    def expect_terms(self, terms, traj0=0, count=None):
        count = len(self.states) - traj0 if count is None else count
        return np.array([opterms_ref.expect(terms, self.states[traj0 + c]) for c in range(count)])


@pytest.fixture
def backend(monkeypatch):
    from fake_device import FakeLindbladPlan
    from pulser_b200 import backend, engine, lindblad

    monkeypatch.setattr(engine, "DevicePlan", FakeTermsPlan)
    monkeypatch.setattr(lindblad, "LindbladPlan", FakeLindbladPlan)
    return backend


def _psi(rng, dim):
    v = rng.normal(size=dim) + 1j * rng.normal(size=dim)
    return v / np.linalg.norm(v)


def _check(op, psi):
    ref = np.vdot(psi, op.to_array() @ psi)
    got = opterms_ref.expect(op._terms, psi)
    assert abs(got - ref) <= 1e-12 * max(1.0, abs(ref))


@pytest.mark.parametrize("d", [2, 3, 4])
@pytest.mark.parametrize("seed", range(4))
def test_random_operations_match_matrix(d, seed):
    from pulser_b200.backend import B200Operator

    rng = np.random.default_rng(10 * d + seed)
    eig = EIGS[d]
    n = {2: 5, 3: 4, 4: 3}[d]
    ops = opterms_ref.random_operations(rng, eig, n)
    # identity terms, Z / X strings over all sites
    ops.append((1.3 - 0.2j, []))
    z = {eig[0] * 2: 1.0, eig[1] * 2: -1.0}
    x = {eig[0] + eig[1]: 1.0, eig[1] + eig[0]: 1.0}
    ops.append((0.4, [(z, set(range(n)))]))
    ops.append((-0.9, [(x, set(range(n)))]))
    op = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=n, operations=ops)
    assert op._terms is not None
    psi = _psi(rng, d**n)
    _check(op, psi)
    # a qudit named by several groups of one term (the public constructor refuses it): the last group wins
    ops = [(0.7, [({eig[0] * 2: 1.0}, {0, 1}), (opterms_ref.random_qudit_op(rng, eig), {1, 2})]),
           (0.2j, [(opterms_ref.random_qudit_op(rng, eig), {0}), (opterms_ref.random_qudit_op(rng, eig), {0})])]
    op, _ = B200Operator._from_operator_repr(eigenstates=eig, n_qudits=n, operations=ops)
    _check(op, psi)


def test_monomial_counts():
    from pulser_b200.backend import B200Operator

    eig = EIGS[2]
    z = {"rr": 1.0, "gg": -1.0}
    x = {"rg": 1.0, "gr": 1.0}
    y = {"rg": -1j, "gr": 1j}
    for qop in (z, x, y, {"rg": 1.0}, {"rr": 1.0}):
        op = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=6, operations=[(1.0, [(qop, set(range(6)))])])
        assert len(op._terms) == 1  # one monomial term over all sites
    # a general site matrix has d shifts: a product over 3 sites expands into 2^3 terms
    gen = {"rr": 1.0, "rg": 2.0, "gr": 3.0, "gg": 4.0}
    op = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=4, operations=[(1.0, [(gen, {0, 1, 2})])])
    assert len(op._terms) == 8
    # the identity adds no site
    ident = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=4, operations=[(2.0, [({"rr": 1.0, "gg": 1.0}, {1})])])
    assert ident._terms.terms == ((2.0, ()),)


@pytest.mark.parametrize("d", [2, 3])
def test_arithmetic_keeps_compiled_form(d):
    from pulser_b200.backend import B200Operator, B200State

    rng = np.random.default_rng(7 + d)
    eig = EIGS[d]
    n = 4 if d == 2 else 3
    A = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=n, operations=opterms_ref.random_operations(rng, eig, n, 3))
    B = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=n, operations=opterms_ref.random_operations(rng, eig, n, 3))
    psi = _psi(rng, d**n)
    for op in (A + B, (0.3 - 2j) * A, A @ B, B @ A @ B, 2.0 * (A @ B) + B):
        assert op._terms is not None
        _check(op, psi)
    # host states still use the matrices
    st = B200State(psi, eigenstates=eig)
    assert (A + B).expect(st) == pytest.approx(complex(np.vdot(psi, (A.to_array() + B.to_array()) @ psi)))


def _hermiticity_cases():
    eig = EIGS[2]
    herm = [
        [(1.0, [({"rg": 1.0, "gr": 1.0}, {i})]) for i in range(4)],                      # sum sigma_x
        [((-1) ** i, [({"rr": 1.0, "gg": -1.0}, {i})]) for i in range(4)],               # staggered Z
        [(1.0, [({"rg": 1.0}, {i}), ({"gr": 1.0}, {j})]) for i in range(4) for j in range(4) if i != j],  # s+ s- + h.c.
        [(1.0, [({"rg": -1j, "gr": 1j}, {0, 2})])],                                     # Y Y
        [(2.0, [({"rg": 1 + 1j, "gr": 1 - 1j, "rr": 0.3}, {1})])],                      # general Hermitian site
        [(1.0, [({"rr": 1.0, "gg": -1.0}, {0, 1, 2, 3})])],                             # parity
    ]
    non = [
        [(1.0, [({"rg": 1.0}, {0})])],
        [(1j, [({"rg": 1.0, "gr": 1.0}, {1})])],
        [(1.0, [({"rg": 1.0}, {0}), ({"gr": 1.0}, {2})])],
        [(1.0, [({"rg": 1 + 1j, "gr": 1 + 1j}, {3})])],
    ]
    return eig, herm, non


def test_hermiticity_without_matrix(monkeypatch):
    from pulser_b200 import backend

    eig, herm, non = _hermiticity_cases()
    O = backend.B200Operator
    for ops, expected in [(o, True) for o in herm] + [(o, False) for o in non]:
        op = O.from_operator_repr(eigenstates=eig, n_qudits=4, operations=ops)
        m = op.to_array()
        assert bool(np.max(np.abs(m - m.conj().T)) < 1e-12) == expected
        fresh = O.from_operator_repr(eigenstates=eig, n_qudits=4, operations=ops)
        built = []
        orig = O._as_matrix
        monkeypatch.setattr(O, "_as_matrix", staticmethod(lambda x: (built.append(1), orig(x))[1]))
        assert fresh._isherm == expected
        monkeypatch.undo()
        assert (len(built) == 0) == expected  # the matrix is only needed when the adjoint lists differ
    # Hermitian in an unusual decomposition, i X - 2i |g><r|: the adjoint lists differ, the matrix decides
    odd = O.from_operator_repr(eigenstates=eig, n_qudits=2,
                               operations=[(1j, [({"rg": 1.0, "gr": 1.0}, {0})]), (-2j, [({"gr": 1.0}, {0})])])
    assert not odd._terms.adjoint_matches()
    built = []
    monkeypatch.setattr(O, "_as_matrix", staticmethod(lambda x: (built.append(1), orig(x))[1]))
    assert odd._isherm and len(built) == 1


def test_no_compiled_form_for_matrices_and_over_the_cap():
    from pulser_b200 import opterms
    from pulser_b200.backend import B200Operator

    eig = EIGS[2]
    assert B200Operator(np.eye(4), eigenstates=eig)._terms is None
    gen = {"rr": 1.0, "rg": 2.0, "gr": 3.0, "gg": 4.0}
    n = 15  # 2^15 monomial terms > MAX_TERMS
    assert 2**n > opterms.MAX_TERMS
    op = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=n, operations=[(1.0, [(gen, set(range(n)))])])
    assert op._terms is None
    ok = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=n, operations=[(1.0, [(gen, set(range(14)))])])
    assert ok._terms is not None and len(ok._terms) == opterms.MAX_TERMS
    assert ok._terms + ok._terms is None and ok._terms @ ok._terms is None
    small = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=2, operations=[(1.0, [(gen, {0})])])
    assert (small + B200Operator(sp.identity(4, format="csr"), eigenstates=eig))._terms is None


def test_c_arrays_layout():
    from pulser_b200.backend import B200Operator

    op = B200Operator.from_operator_repr(eigenstates=EIGS[3], n_qudits=3,
                                         operations=[(2.0, [({"ud": 1.0}, {2}), ({"xx": 3.0}, {0})]), (1.0, [])])
    coeff, site_start, site, shift, weight = op._terms.arrays()
    assert list(coeff) == [2.0, 1.0] and list(site_start) == [0, 2, 2]
    assert list(site) == [0, 2] and list(shift) == [0, 1]
    np.testing.assert_array_equal(weight, [[0, 0, 3], [1, 0, 0]])


def test_operators_on_different_registers_do_not_combine():
    """``+`` still fails at once on the matrices; ``@`` keeps no compiled form, so its matrix reports the mismatch."""
    from pulser_b200.backend import B200Operator

    eig = EIGS[2]
    x = {"rg": 1.0, "gr": 1.0}
    a3 = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=3, operations=[(1.0, [(x, {0})])])
    a4 = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=4, operations=[(1.0, [(x, {0})])])
    with pytest.raises(ValueError):
        a3 + a4
    prod = a3 @ a4
    assert prod._terms is None
    with pytest.raises(ValueError):
        prod.to_array()
    with pytest.raises(ValueError, match="3 and 4 qudits"):
        a3._terms + a4._terms
    with pytest.raises(ValueError, match="3 and 4 qudits"):
        a3._terms @ a4._terms


def test_nearly_equal_terms_do_not_merge(monkeypatch):
    """X - (|r><g| + (1 + 1e-10)|g><r|) = -1e-10 |g><r| is not Hermitian: terms whose weights differ are not merged."""
    from pulser_b200.backend import B200Operator

    eig = EIGS[2]
    op = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=2, operations=[
        (1.0, [({"rg": 1.0, "gr": 1.0}, {0})]), (-1.0, [({"rg": 1.0, "gr": 1.0 + 1e-10}, {0})])])
    assert not op._terms.adjoint_matches()
    assert not op._isherm


def test_deepcopy_after_packing():
    """Pulser deep-copies the observables of a config (``with_changes``): an operator packed for the C ABI still copies."""
    import copy

    from pulser.backend.default_observables import Expectation

    from pulser_b200.backend import B200Config, B200Operator

    eig = EIGS[2]
    op = B200Operator.from_operator_repr(eigenstates=eig, n_qudits=3, operations=[(1.0, [({"rg": 1.0, "gr": 1.0}, {1})])])
    cfg = B200Config(observables=[Expectation(op, evaluation_times=[1.0])])
    packed = cfg.observables[0].operator._terms
    desc = packed.c_desc()
    assert desc.n_terms == 1 and desc.coeff[0] == 1.0 and desc.site[0] == 1
    twin = copy.deepcopy(cfg.observables[0].operator)
    assert twin._terms.terms == packed.terms
    cfg2 = cfg.with_changes(sampling_rate=0.5)
    assert cfg2.observables[0].operator._terms.terms == packed.terms


def _seq(n=3, duration=240):
    from pulser import Pulse, Register, Sequence
    from pulser.devices import MockDevice
    from pulser.waveforms import BlackmanWaveform

    reg = Register.from_coordinates([(7.0 * i, 0.0) for i in range(n)], prefix="q")
    seq = Sequence(reg, MockDevice)
    seq.declare_channel("ch", "rydberg_global")
    seq.add(Pulse.ConstantDetuning(BlackmanWaveform(duration, np.pi), 1.0, 0.0), "ch")
    return seq


def test_backend_expectations_through_expect_terms(backend, monkeypatch):
    """A plan with ``expect_terms`` answers ``Expectation`` without a matrix: same values as the host formulas."""
    from pulser.backend.default_observables import Expectation

    from oracle import evolve
    from oracle.ref_hamiltonian import OracleHamiltonian

    seq = _seq()
    eig = ("r", "g")
    O = backend.B200Operator
    n = 3
    sx = O.from_operator_repr(eigenstates=eig, n_qudits=n, operations=[(1.0, [({"rg": 1.0, "gr": 1.0}, {i})]) for i in range(n)])
    flip = O.from_operator_repr(eigenstates=eig, n_qudits=n, operations=[(1.0, [({"rg": 1.0}, {0}), ({"gr": 0.5j}, {2})])])
    times = [0.25, 1.0]
    cfg = backend.B200Config(observables=[Expectation(sx, evaluation_times=times, tag_suffix="sx"),
                                          Expectation(flip, evaluation_times=times, tag_suffix="flip")])
    built = []
    orig = O._as_matrix
    monkeypatch.setattr(O, "_as_matrix", staticmethod(lambda x: (built.append(1), orig(x))[1]))
    res = backend.B200Backend(seq, config=cfg).run()
    assert len(built) == 1  # only the Hermiticity decision of the non-Hermitian operator needs its matrix
    monkeypatch.setattr(O, "_as_matrix", staticmethod(orig))
    sim = backend.B200Emulator.from_sequence(seq)
    spec = sim._noiseless_spec()
    T = spec.sampling_times[-1]
    states = evolve.sesolve(OracleHamiltonian.from_spec(spec), evolve.all_ground_state(spec), [0.0, 0.25 * T, T],
                            rtol=1e-11, atol=1e-13)[1:]
    for t_rel, st in zip(times, states):
        st = st / np.linalg.norm(st)
        got = res.get_result("expectation_sx", t_rel)
        assert isinstance(got, float)
        assert got == pytest.approx(np.vdot(st, sx.to_array() @ st).real, abs=1e-7)
        got = res.get_result("expectation_flip", t_rel)
        assert isinstance(got, complex)
        assert got == pytest.approx(complex(np.vdot(st, flip.to_array() @ st)), abs=1e-7)
