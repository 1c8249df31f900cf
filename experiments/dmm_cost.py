"""Experiment (GPU): cost of detuning maps (DMM) on the Taylor propagator.

(a) C2 (N = 20), plain and with a detuning map on half the atoms (weights 1, a ramp to -6 rad/us over the first half,
    then constant): device time per Taylor order, H-applies per ns and steps, best of 3.
(b) A 64-trajectory C4-shaped batch (N = 16, doppler + amplitude noise) with the same map: trajectories/s on the
    Taylor propagator (two detuning shapes) against the Krylov path (``integrator=2``), and max |dpsi| between them.
(c) The DMM C2 on 1 / 2 / 4 / 8 shards of device 0: device time per order, max |dpsi| against the unsharded plan.

The card name and power limit are recorded in the same run.  Prints one JSON object.

Usage: python experiments/dmm_cost.py [--out FILE]
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from experiments.shard_scaling import gpu_info  # noqa: E402
from pulser_b200 import engine, sharded, workloads as W  # noqa: E402


def dmm_waveform(T: int) -> np.ndarray:
    return -np.concatenate([np.linspace(0.0, 6.0, T // 2), np.full(T - T // 2, 6.0)])


def with_map(spec, n):
    w = np.where(np.arange(n) % 2 == 0, 1.0, 0.0)
    return W.detuning_map_spec(spec, [(w, dmm_waveform(spec.total_duration_ns))])


def best_run(make, spec, reps=3, **kw):
    best = None
    for _ in range(reps):
        with make() as plan:
            plan.set_state("all-ground")
            st = plan.propagate(0.0, spec.sampling_times[-1], **kw)
            psi = plan.get_state().copy()
        if best is None or st["gpu_ms"] < best[0]["gpu_ms"]:
            best = (st, psi)
    return best


def row(st, T):
    return {"integrator": st["integrator"], "gpu_ms": st["gpu_ms"], "n_steps": st["n_steps"],
            "n_applies": st["n_applies"], "us_per_order": 1e3 * st["gpu_ms"] / max(st["n_applies"], 1),
            "applies_per_ns": st["n_applies"] / T}


def main() -> None:
    out: dict = {"gpus": gpu_info()}
    # (a)
    plain = W.config_c2(n=20)
    T = plain.total_duration_ns
    dmm = with_map(plain, 20)
    out["c2"] = {}
    for name, spec in (("plain", plain), ("dmm", dmm)):
        st, _ = best_run(lambda: engine.DevicePlan(spec), spec)
        out["c2"][name] = row(st, T)
    # (b)
    specs = [with_map(s, 16) for s in W.config_c4(64)]
    T4 = specs[0].total_duration_ns
    out["c4_dmm_batch64"] = {}
    states = {}
    for name, integ in (("taylor", 0), ("krylov", 2)):
        st, psi = best_run(lambda: engine.DevicePlan(specs), specs[0], reps=2, integrator=integ)
        states[name] = psi
        r = row(st, T4)
        r["trajectories_per_s"] = 64 / (st["gpu_ms"] * 1e-3)
        out["c4_dmm_batch64"][name] = r
    out["c4_dmm_batch64"]["max_abs_dpsi"] = float(np.max(np.abs(states["taylor"] - states["krylov"])))
    # (c)
    rows = []
    ref = None
    for G in (1, 2, 4, 8):
        st, psi = best_run(lambda: engine.DevicePlan(dmm) if G == 1 else sharded.ShardedPlan(dmm, [0] * G), dmm)
        ref = psi if G == 1 else ref
        r = row(st, T)
        r["shards"] = G
        r["max_abs_dpsi"] = float(np.max(np.abs(psi - ref)))
        rows.append(r)
    out["c2_dmm_shards"] = rows
    text = json.dumps(out, indent=1)
    print(text)
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
