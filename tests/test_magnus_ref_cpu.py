"""The exact references of tests/magnus_ref.py on the CPU: the product of per-cluster exponentials equals the dense
exponential of the whole register, sampled amplitudes equal the full product vector, and the specs are constant under
the library's own interpolation at every order the plan offers."""
import ctypes as C

import numpy as np
import pytest

from magnus_ref import (ClusterReference, cluster_couplings, constant_spec, dense_evolve, interleaved_clusters,
                        probe_indices)


def _ising(n, clusters, seed, local=True, phase=0.0):
    rng = np.random.default_rng(seed)
    if local:
        coef = rng.uniform(1.0, 4.0, n) * np.exp(1j * rng.uniform(-np.pi, np.pi, n))
        det = rng.uniform(-6.0, 6.0, n)
    else:
        coef, det = 2.5 * np.exp(-1j * phase), -3.0
    return constant_spec([("ground-rydberg", coef, det)], cluster_couplings(n, clusters, seed + 1), n_samples=8)


@pytest.mark.parametrize("n,n_clusters,local", [(7, 3, True), (9, 2, False), (10, 2, True), (10, 4, False)])
def test_cluster_product_equals_dense_exponential(n, n_clusters, local):
    clusters = interleaved_clusters(n, n_clusters)
    spec = _ising(n, clusters, seed=n, local=local, phase=0.7)
    ref = ClusterReference(spec, clusters)
    parts = ref.initial(seed=3)
    T = 0.37
    got = ref.full(ref.evolve(parts, T))
    want = dense_evolve(spec, ref.full(parts), T)
    assert np.linalg.norm(got - want) < 1e-13
    assert abs(ref.norm(ref.evolve(parts, T)) - 1.0) < 1e-13
    # the evolution is far from trivial: the state moved by O(1)
    assert np.linalg.norm(want - ref.full(parts)) > 0.3


def test_couplings_between_clusters_are_refused():
    clusters = interleaved_clusters(6, 2)
    spec = _ising(6, clusters, seed=1)
    # atoms 0 and 1 sit in different clusters
    spec.interaction_matrix[0, 0, 1] = spec.interaction_matrix[0, 1, 0] = 1.0
    with pytest.raises(ValueError):
        ClusterReference(spec, clusters)


@pytest.mark.parametrize("n,n_clusters", [(14, 2), (16, 3)])
def test_sampled_amplitudes_equal_full_vector(n, n_clusters):
    clusters = interleaved_clusters(n, n_clusters, shift=1)
    ref = ClusterReference(_ising(n, clusters, seed=n), clusters)
    parts = ref.evolve(ref.initial(seed=5), 0.21)
    full = ref.full(parts)
    idx = probe_indices(n, 500, seed=n)
    assert np.max(np.abs(ref.amplitudes(parts, idx) - full[idx])) < 1e-15
    assert abs(ref.norm(parts) - np.linalg.norm(full)) < 1e-13
    ground = ref.full(ref.ground())
    assert ground[-1] == 1.0 and np.linalg.norm(ground) == 1.0


def test_interleaved_clusters_reach_every_pass():
    """at N = 27 / 28 every cluster has atoms in the 11 tile bits, in the next 11 and above them"""
    for n in (20, 27, 28):
        for atoms in interleaved_clusters(n):
            bits = {n - 1 - k for k in atoms}
            assert min(bits) < 11 and any(11 <= b < 22 for b in bits)
            assert n <= 22 or max(bits) >= 22


def _constant_specs():
    rng = np.random.default_rng(0)
    n = 5
    yield constant_spec([("ground-rydberg", 1.5, 2.0)], np.zeros((n, n)), n_samples=30)
    yield constant_spec([("ground-rydberg", rng.normal(size=n) + 1j * rng.normal(size=n), rng.normal(size=n))],
                        np.zeros((n, n)), n_samples=7, dt_ns=20)
    yield constant_spec([("ground-rydberg", 1.0 + 0.5j, -1.0), ("digital", 0.3 - 0.2j, 0.4)], np.zeros((n, n)),
                        n_samples=12, dim=4)


@pytest.mark.parametrize("order", [0, 1, 3])
def test_specs_are_constant_under_interpolation(lib, order):
    """``pb200_host_interpolate`` (the plan's interpolant) returns the sample value at random times"""
    P = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))   # noqa: E731
    for spec in _constant_specs():
        x = np.ascontiguousarray(spec.sampling_times)
        tq = np.random.default_rng(order).uniform(x[0], x[-1], 200)
        tq[:2] = x[0], x[-1]
        for d in spec.drives:
            for row in list(d.coef) + list(d.det.astype(complex)):
                y = np.ascontiguousarray(row, dtype=complex)
                out = np.empty(2 * len(tq))
                assert lib.pb200_host_interpolate(P(x), P(y.view(np.float64)), len(x), order, P(tq), len(tq),
                                                  P(out)) == 0
                assert np.max(np.abs(out.view(np.complex128) - y[0])) <= 1e-15 * max(1.0, abs(y[0]))
