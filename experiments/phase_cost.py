"""Experiment (GPU): cost of a moving drive phase on the Taylor propagator.

Sequences:
  c2_jump   C2 (N = 20) with the drive phase switched from 0 to pi/2 under full amplitude mid-sweep;
  c2_ramsey the same register running a Ramsey pair (pi/2 at phase 0, free evolution, pi/2 at phase 1.1);
  c5_jump   C5 (N = 24) with one phase jump (0 -> pi/2 at mid-sequence).
Reference points: c2_plain (C2, every step on the real kernel) and c2_ramp (C2 under a phase ramp over the whole
sequence, every step on the complex kernel) give the microseconds per order of the two kernels.

Per sequence: H-applies per ns, device time per order, the share of orders that ran complex (step log), the largest
ring R (state-sized vectors including the state; sets the shard capacity), the same sequence on the Magnus path
(``integrator=1``, what ran before), and for c2_jump 2 / 4 / 8 shards of device 0.  Best of 3.  The card name and
power limit are recorded in the same run.  Prints one JSON object.

Usage: python experiments/phase_cost.py [--out FILE]
"""
from __future__ import annotations

import dataclasses
import json
import os
import re
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from experiments.shard_scaling import gpu_info  # noqa: E402
from pulser_b200 import engine, sharded, workloads as W  # noqa: E402

STEP_RE = re.compile(r"taylor step .* K=(\d+) ring=(\d+) .* drive=(\w+)")


def with_phase(spec, phase):
    """the spec's drive with the phase samples `phase` (ns grid) instead of its own"""
    d = spec.drives[0]
    coef = np.array(d.coef, dtype=complex)
    T = coef.shape[1] - 1
    ph = np.append(phase[:T], phase[T - 1])
    coef = np.abs(coef) * np.exp(-1j * ph)[None, :]
    return dataclasses.replace(spec, drives=[dataclasses.replace(d, coef=coef)])


def jump(spec, at=None):
    T = spec.total_duration_ns
    at = T // 2 if at is None else at
    return with_phase(spec, np.where(np.arange(T) < at, 0.0, np.pi / 2))


def ramsey(n):
    T = 500
    t = np.arange(T)
    amp = np.where((t < 100) | (t >= 400), np.pi / 0.2, 0.0)
    ph = np.where(t < 250, 0.0, 1.1)
    return W.ising_global_spec(W.disc_register(n, 22.0, 6.0, n), W.C6_LEVEL_60, amp, np.full(T, -2.0), phase=ph)


def logged(make, spec, reps=3, **kw):
    """best of `reps` runs; the step log of the last one, read from stderr through a temporary file"""
    best = None
    steps = []
    for _ in range(reps):
        with tempfile.TemporaryFile(mode="w+") as f:
            fd = os.dup(2)
            os.dup2(f.fileno(), 2)
            try:
                with make() as plan:
                    plan.set_state("all-ground")
                    st = plan.propagate(0.0, spec.sampling_times[-1], **kw)
                    psi = plan.get_state().copy()
            finally:
                os.dup2(fd, 2)
                os.close(fd)
            f.seek(0)
            steps = [(int(m[1]), int(m[2]), m[3]) for m in STEP_RE.finditer(f.read())]
        if best is None or st["gpu_ms"] < best[0]["gpu_ms"]:
            best = (st, psi)
    return best[0], best[1], steps


def row(st, T, steps=()):
    r = {"integrator": st["integrator"], "gpu_ms": st["gpu_ms"], "n_steps": st["n_steps"],
         "n_applies": st["n_applies"], "us_per_order": 1e3 * st["gpu_ms"] / max(st["n_applies"], 1),
         "applies_per_ns": st["n_applies"] / T, "err_estimate": st["err_estimate"]}
    if steps:
        orders = sum(k for k, _, _ in steps)
        r["complex_order_share"] = sum(k for k, _, d in steps if d == "cplx") / max(orders, 1)
        r["max_ring"] = max(g for _, g, _ in steps)
    return r


def main() -> None:
    os.environ["PB200_TAYLOR_LOG"] = "1"
    out: dict = {"gpus": gpu_info()}
    c2 = W.config_c2(n=20)
    T2 = c2.total_duration_ns
    seqs = {
        "c2_plain": c2,
        "c2_ramp": with_phase(c2, np.linspace(0.0, 2.0, T2)),
        "c2_jump": jump(c2),
        "c2_ramsey": ramsey(20),
        "c5_jump": jump(W.config_c5()),
    }
    for name, spec in seqs.items():
        T = spec.total_duration_ns
        st, psi, steps = logged(lambda: engine.DevicePlan(spec), spec)
        r = {"taylor": row(st, T, steps)}
        st1, psi1, _ = logged(lambda: engine.DevicePlan(spec), spec, reps=1, integrator=1)
        r["magnus_cf4"] = row(st1, T)
        r["max_abs_dpsi_taylor_magnus"] = float(np.max(np.abs(psi - psi1)))
        if name == "c2_jump":
            r["shards"] = []
            for G in (2, 4, 8):
                stg, psig, _ = logged(lambda: sharded.ShardedPlan(spec, [0] * G), spec)
                rg = row(stg, T)
                rg["shards"] = G
                rg["max_abs_dpsi"] = float(np.max(np.abs(psig - psi)))
                r["shards"].append(rg)
        out[name] = r
        print(name, json.dumps(r), file=sys.stderr)
    text = json.dumps(out, indent=1)
    print(text)
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
