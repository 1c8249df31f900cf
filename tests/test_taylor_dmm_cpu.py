"""Host side of detuning maps on the Taylor propagator: the separable structure with several detuning time shapes
(``pb200_host_taylor_shapes``) and the validation of sharded plans with per-qubit detuning.  No GPU needed."""
import ctypes as C

import numpy as np
import pytest

from pulser_b200 import workloads as W

SMAX = 4


def P(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


@pytest.fixture(scope="module")
def lib():
    from pulser_b200._lib import lib

    return lib


def _shapes(lib, coef, det, max_shapes=SMAX):
    B, N, nt = det.shape
    ns = C.c_int32(-2)
    a = np.zeros((B, N), dtype=np.complex128)
    c = np.zeros((B, N, max(max_shapes, 1)))
    m = np.zeros((max(max_shapes, 1), nt))
    coef = np.ascontiguousarray(coef, dtype=np.complex128)
    det = np.ascontiguousarray(det, dtype=np.float64)
    assert lib.pb200_host_taylor_shapes(P(coef.view(np.float64)), P(det), B, N, nt, max_shapes, C.byref(ns),
                                        P(a.view(np.float64)), P(c), P(m)) == 0
    return ns.value, a, c, m


def _tables(specs):
    return (np.array([s.drives[0].coef for s in specs]), np.array([s.drives[0].det for s in specs]))


def _rebuilt(coef, det, a, c, m, S):
    b, k, _ = np.unravel_index(np.argmax(np.abs(coef)), coef.shape)
    ce = np.max(np.abs(coef - a[:, :, None] * coef[b, k][None, None, :]))
    de = np.max(np.abs(det - det[0, 0][None, None, :] - np.einsum("bks,st->bkt", c[:, :, :S], m[:S])))
    return ce, de


def _base(n=8, T=400, seed=3):
    amp, det = W.blockade_sweep_waveforms(t_rise=80, t_sweep=T - 160, t_fall=80)
    coords = W.disc_register(n, 14.0, 5.0, seed)
    return coords, W.ising_global_spec(coords, W.C6_LEVEL_60, amp, det)


def _dmm_waveforms(T):
    """negative DMM waveforms of different time shapes (a ramp, a Blackman-like bump, a late step, a sine)"""
    t = np.arange(T)
    return [
        -np.concatenate([np.linspace(0.0, 6.0, T // 2), np.full(T - T // 2, 6.0)]),
        -4.0 * np.sin(np.pi * t / T) ** 2,
        -np.where(t > 0.7 * T, 3.0, 0.0),
        -2.0 * (1.0 + np.sin(7.0 * np.pi * t / T)),
        -np.where((t > 0.2 * T) & (t < 0.4 * T), 1.5, 0.0),
    ]


def _dmm_specs(n_maps, noisy=False, n=8, T=400, B=3):
    coords, base = _base(n, T)
    rng = np.random.default_rng(n_maps)
    maps = [(rng.uniform(0.0, 1.0, n) * (rng.uniform(size=n) < 0.6), wf) for wf in _dmm_waveforms(T)[:n_maps]]
    spec = W.detuning_map_spec(base, maps)
    if not noisy:
        return [spec]
    return [W.noisy_trajectory_spec(spec, coords, rng.normal(0, 1.5, n), max(0.0, rng.normal(1.0, 0.05)), 60.0)
            for _ in range(B)]


@pytest.mark.parametrize("n_maps,noisy,expect", [(1, False, 1), (1, True, 2), (2, True, 3), (3, False, 3),
                                                 (4, False, 4), (3, True, 4)])
def test_shape_counts_and_rebuild(lib, n_maps, noisy, expect):
    """one DMM: S = 1; with doppler noise one more shape (the slot mask); DMM + an SLM-like step: 3; up to 4"""
    coef, det = _tables(_dmm_specs(n_maps, noisy))
    S, a, c, m = _shapes(lib, coef, det)
    assert S == expect
    ce, de = _rebuilt(coef, det, a, c, m, S)
    assert ce < 1e-11 and de < 1e-11
    assert np.allclose(np.max(np.abs(m[:S]), axis=1), 1.0, rtol=0, atol=1e-15)   # max |M_s| = 1
    assert np.all(m[S:] == 0.0) and np.all(c[:, :, S:] == 0.0)
    if not noisy:
        assert np.all(a == 1.0)      # identical drive rows: a uniform drive


def test_too_many_shapes_and_non_rank1_drive_are_refused(lib):
    coef, det = _tables(_dmm_specs(5))
    assert _shapes(lib, coef, det)[0] == -1
    assert _shapes(lib, coef, det, max_shapes=5 - 1)[0] == -1
    coef4, det4 = _tables(_dmm_specs(4))
    assert _shapes(lib, coef4, det4, max_shapes=3)[0] == -1
    assert _shapes(lib, coef4, det4, max_shapes=4)[0] == 4
    bad = coef4.copy()
    bad[0, 3, 100:200] *= 1.0 + 1e-9              # one qubit's amplitude changes shape
    assert _shapes(lib, bad, det4)[0] == -1
    # no shape at all: a plain global sequence
    _, base = _base()
    assert _shapes(lib, *_tables([base]))[0] == 0
    assert _shapes(lib, *_tables([base]), max_shapes=0)[0] == 0
    assert _shapes(lib, coef4, det4, max_shapes=0)[0] == -1


def test_bad_arguments(lib):
    coef, det = _tables(_dmm_specs(1))
    for ms in (-1, SMAX + 1):
        ns = C.c_int32(0)
        assert lib.pb200_host_taylor_shapes(P(np.ascontiguousarray(coef).view(np.float64)), P(det), 1, det.shape[1],
                                            det.shape[2], ms, C.byref(ns), None, None, None) != 0


def test_c4_batches_match_the_one_shape_export(lib):
    """on the striped C4 batches (doppler + amplitude noise) the shapes export finds S = 1 with the factors of
    pb200_host_taylor_separable"""
    from pulser_b200 import parallel

    mine = set(parallel.stripe(1024, 3, 8))
    chunk = [s for _, s in W.config_c4_stream(1024, keep=mine)][:64]
    coef, det = _tables(chunk)
    B, N, nt = det.shape
    ok = C.c_int32(-1)
    a1 = np.zeros((B, N), dtype=np.complex128)
    c1 = np.zeros((B, N))
    m1 = np.zeros(nt)
    coefc = np.ascontiguousarray(coef, dtype=np.complex128)
    detc = np.ascontiguousarray(det, dtype=np.float64)
    assert lib.pb200_host_taylor_separable(P(coefc.view(np.float64)), P(detc), B, N, nt, C.byref(ok),
                                           P(a1.view(np.float64)), P(c1), P(m1)) == 0
    assert ok.value == 1
    S, a, c, m = _shapes(lib, coef, det)
    assert S == 1
    assert np.array_equal(a, a1) and np.array_equal(c[:, :, 0], c1) and np.array_equal(m[0], m1)


def test_old_export_still_refuses_two_shapes(lib):
    coef, det = _tables(_dmm_specs(1, noisy=True))
    B, N, nt = det.shape
    ok = C.c_int32(-1)
    coefc = np.ascontiguousarray(coef, dtype=np.complex128)
    assert lib.pb200_host_taylor_separable(P(coefc.view(np.float64)), P(np.ascontiguousarray(det)), B, N, nt,
                                           C.byref(ok), None, None, None) == 0
    assert ok.value == 0
    assert _shapes(lib, coef, det)[0] == 2


def test_sharded_plan_validation():
    """a DMM spec passes the Python checks of ShardedPlan (it fails only on creating the plans: no device here or
    no such device), per-qubit drive amplitudes are refused before any device call"""
    from pulser_b200 import sharded

    coords, base = _base(n=14, T=200)
    spec = W.detuning_map_spec(base, [(np.linspace(0.0, 1.0, 14), _dmm_waveforms(200)[0])])
    with pytest.raises(Exception) as e:
        sharded.ShardedPlan(spec, [63, 63])
    assert not isinstance(e.value, NotImplementedError)
    amp = W.noisy_trajectory_spec(spec, coords, np.zeros(14), 0.97, 60.0)
    with pytest.raises(NotImplementedError, match="per-qubit"):
        sharded.ShardedPlan(amp, [63, 63])
