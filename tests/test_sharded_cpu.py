"""CPU tests of state-vector sharding: argument checks of ``pb200_plan_create_shard`` (made before any device call),
the ``devices`` option of ``B200Config`` and the shot routing of ``ShardedPlan.sample``."""
import ctypes as C

import numpy as np
import pytest

from pulser_b200 import HAVE_PULSER


def _desc(n, times):
    from pulser_b200._lib import PlanDesc

    d = PlanDesc()
    d.n_qudits, d.dim, d.n_times, d.interp_order = n, 2, len(times), 3
    d.n_drives, d.rydberg_state, d.n_traj, d.device = 1, 0, 1, 0
    d.sampling_times = times.ctypes.data_as(C.POINTER(C.c_double))
    d.drives[0].state_to, d.drives[0].state_from, d.drives[0].uniform = 1, 0, 1
    return d


@pytest.mark.parametrize(
    "n,bits,index,needle",
    [
        (20, 0, 0, b"shard_bits"),
        (20, 4, 0, b"shard_bits"),
        (20, 1, 2, b"shard_index"),
        (20, 2, -1, b"shard_index"),
        (14, 2, 0, b"N - shard_bits = 12"),     # L = 12: below one 2^13 tile
        (33, 3, 0, b"N - shard_bits = 30"),     # L = 30: above 2^29
        (31, 1, 1, b"N - shard_bits = 30"),
    ],
)
def test_create_shard_argument_checks(lib, n, bits, index, needle):
    times = np.linspace(0.0, 1.0, 11)
    h = C.c_void_p()
    assert lib.pb200_plan_create_shard(C.byref(h), C.byref(_desc(n, times)), bits, index) == -1
    assert needle in lib.pb200_last_error()
    assert not h.value


def test_create_shard_scope_checks(lib):
    """d = 3 and trajectory batches are refused before a device is needed."""
    times = np.linspace(0.0, 1.0, 11)
    h = C.c_void_p()
    d = _desc(16, times)
    d.dim = 3
    assert lib.pb200_plan_create_shard(C.byref(h), C.byref(d), 1, 0) == -3
    assert b"d = 2" in lib.pb200_last_error()
    d = _desc(16, times)
    d.n_traj = 4
    assert lib.pb200_plan_create_shard(C.byref(h), C.byref(d), 1, 0) == -3


def test_group_calls_need_a_linked_group(lib):
    arr = (C.c_void_p * 2)()
    assert lib.pb200_shards_link(arr, 3) == -1
    assert b"2, 4 or 8" in lib.pb200_last_error()
    assert lib.pb200_shards_propagate(arr, 1, 0.0, 1.0, None, None) == -1


@pytest.mark.parametrize("devices", [[0, 0], [0, 1, 2, 3], (1,) * 8, [np.int64(0), 1]])
def test_validate_devices_accepts(devices):
    from pulser_b200.sharded import validate_devices

    assert validate_devices(devices) == [int(d) for d in devices]


@pytest.mark.parametrize(
    "devices,exc",
    [([0], ValueError), ([0, 0, 0], ValueError), ([0] * 16, ValueError), ("01", TypeError), (0, TypeError),
     ([0, -1], TypeError), ([0, 1.0], TypeError), ([True, False], TypeError)],
)
def test_validate_devices_rejects(devices, exc):
    from pulser_b200.sharded import validate_devices

    with pytest.raises(exc):
        validate_devices(devices)


@pytest.mark.skipif(not HAVE_PULSER, reason="pulser-core not importable here")
def test_config_devices_option():
    from pulser_b200.backend import B200Config

    assert B200Config().devices is None
    assert B200Config(devices=(0, 0, 1, 1)).devices == [0, 0, 1, 1]
    with pytest.raises(ValueError, match="2, 4 or 8"):
        B200Config(devices=[0, 1, 2])
    with pytest.raises(TypeError):
        B200Config(devices="0,1")


def _device_search(cum_local, u_local):
    # what pb200_state_sample does with a shard's weights: first j with cum[j] >= u * cum[-1]
    return np.minimum(np.searchsorted(cum_local, u_local * cum_local[-1], side="left"), len(cum_local) - 1)


@pytest.mark.parametrize("G,L", [(2, 3), (4, 2), (8, 3)])
@pytest.mark.parametrize("one_digit", [0, 1])
def test_shot_routing_matches_global_search(G, L, one_digit):
    """Routing by shard weights, then searching the shard, picks the bitstring a search over all 2^N weights picks.
    one_digit = 0: the bitstring is the complement of the state index (ground-rydberg), 1: the index itself."""
    from pulser_b200.sharded import global_bitstring, route_shots

    rng = np.random.default_rng(G * 10 + L + one_digit)
    n = L + (G.bit_length() - 1)
    probs = rng.random(1 << n) ** 3
    probs[rng.random(1 << n) < 0.3] = 0.0
    probs[(1 << L) : (2 << L)] = 0.0        # an empty shard
    probs /= probs.sum()
    idx = np.arange(1 << n)
    b_of = idx if one_digit == 1 else (~idx) & ((1 << n) - 1)
    weights = np.zeros(1 << n)
    weights[b_of] = probs                    # global bitstring weights
    u = rng.random(4000)
    ref = np.minimum(np.searchsorted(np.cumsum(weights), u * weights.sum(), side="left"), (1 << n) - 1)

    slices = [probs[i << L : (i + 1) << L] for i in range(G)]
    shard, block, local_u = route_shots(u, np.array([s.sum() for s in slices]), reverse=(one_digit == 0))
    local_b = np.zeros(len(u), dtype=np.int64)
    for i in range(G):
        sel = shard == i
        if not np.any(sel):
            continue
        lidx = np.arange(1 << L)
        lb = lidx if one_digit == 1 else (~lidx) & ((1 << L) - 1)
        w = np.zeros(1 << L)
        w[lb] = slices[i]                    # the shard's weights by the low L bits of the bitstring
        local_b[sel] = _device_search(np.cumsum(w), local_u[sel])
    got = global_bitstring(block, local_b, L)
    assert np.array_equal(got, ref)
    assert not np.any(shard == 1)            # the empty shard never draws a shot
