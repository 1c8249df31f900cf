"""Experiment (GPU): cost and reach of state-vector sharding (``pulser_b200.sharded.ShardedPlan``).

(a) One device, C2 (N = 20) split into 1 / 2 / 4 / 8 shards that all live on device 0: time per Taylor order and
    steps/s of the whole sequence (device time, CUDA events), and max |dpsi| against the unsharded plan.  This is the
    cost of splitting -- more launches, streams and events, and the same-device "peer" loads.
(b) With G >= 2 visible devices: a C5-shaped anneal at the largest N that fits G shards (N = 29 .. 32), timed over
    its first 200 ns, with the inter-GPU bytes per order from the shapes (16 B x 2^L x log2(G) per shard).
(c) The ring R (state-sized vectors of the largest step, read from the PB200_TAYLOR_LOG step log) of C2 and C5, and
    the per-shard bytes (R 16 + 8) 2^L it implies for N = 28 .. 32 on 1 / 2 / 4 / 8 GPUs.

The card name and power limit are recorded in the same run.  Prints one JSON object.

Usage: python experiments/shard_scaling.py [--out FILE]
"""
from __future__ import annotations

import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pulser_b200 import engine, sharded, workloads as W  # noqa: E402


def gpu_info() -> list[dict]:
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout
    except Exception as e:  # pragma: no cover - machine dependent
        return [{"error": str(e)}]
    rows = []
    for line in out.strip().splitlines():
        name, power, clk = [x.strip() for x in line.split(",")]
        rows.append({"name": name, "power_limit_w": power, "sm_clock_max_mhz": clk})
    return rows


def run(plan, spec, t_stop=None):
    plan.set_state("all-ground")
    tf = spec.sampling_times[-1] if t_stop is None else t_stop
    st = plan.propagate(0.0, tf)
    return st, plan.get_state()[0] if spec.n_qudits <= 24 else None


def ring_of(spec) -> int:
    """Largest ring of a whole-sequence run, from the step log of the propagator (stderr of the library)."""
    with tempfile.TemporaryFile(mode="w+") as tmp:
        saved = os.dup(2)
        os.environ["PB200_TAYLOR_LOG"] = "1"
        try:
            os.dup2(tmp.fileno(), 2)
            with engine.DevicePlan(spec) as plan:
                run(plan, spec)
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            os.environ.pop("PB200_TAYLOR_LOG", None)
        tmp.seek(0)
        rings = [int(m) for m in re.findall(r"ring=(\d+)", tmp.read())]
    return max(rings)


def main() -> None:
    out: dict = {"gpus": gpu_info(), "device_count": engine.device_count()}
    # (a)
    spec = W.config_c2(n=20)
    rows = []
    ref = None
    for G in (1, 2, 4, 8):
        best = None
        for _ in range(3):
            plan = engine.DevicePlan(spec) if G == 1 else sharded.ShardedPlan(spec, [0] * G)
            with plan:
                st, psi = run(plan, spec)
            if best is None or st["gpu_ms"] < best[0]["gpu_ms"]:
                best = (st, psi)
        st, psi = best
        if G == 1:
            ref = psi
        rows.append({
            "shards": G, "gpu_ms": st["gpu_ms"], "n_steps": st["n_steps"], "n_applies": st["n_applies"],
            "us_per_order": 1e3 * st["gpu_ms"] / st["n_applies"], "steps_per_s": st["n_steps"] / (st["gpu_ms"] * 1e-3),
            "max_abs_dpsi": float(np.max(np.abs(psi - ref))),
        })
    out["c2_one_device"] = rows
    # (c)
    rings = {"C2": ring_of(W.config_c2(n=20)), "C5": ring_of(W.config_c5(n=20))}
    R = max(rings.values())
    out["ring"] = rings
    out["bytes_per_shard_GiB"] = {
        f"N={n}": {f"G={G}": round((R * 16 + 8) * 2.0 ** (n - (G.bit_length() - 1)) / 2**30, 1) for G in (1, 2, 4, 8)}
        for n in range(28, 33)
    }
    # (b)
    G = engine.device_count()
    G = 8 if G >= 8 else 4 if G >= 4 else 2 if G >= 2 else 1
    if G < 2:
        out["multi_gpu"] = "not measured: one device visible"
    else:
        res = None
        for n in range(32, 28, -1):
            L = n - (G.bit_length() - 1)
            if L > sharded.MAX_LOCAL_BITS:
                continue
            spec = W.config_c5(n=n)
            try:
                with sharded.ShardedPlan(spec, list(range(G))) as plan:
                    st, _ = run(plan, spec, t_stop=0.2)
            except Exception as e:
                out.setdefault("multi_gpu_skipped", []).append({"N": n, "error": str(e)[:200]})
                continue
            res = {"N": n, "shards": G, "window_us": 0.2, "gpu_ms": st["gpu_ms"], "n_steps": st["n_steps"],
                   "steps_per_s": st["n_steps"] / (st["gpu_ms"] * 1e-3), "us_per_order": 1e3 * st["gpu_ms"] / st["n_applies"],
                   "peer_bytes_per_order_per_shard": 16 * 2**L * (G.bit_length() - 1)}
            break
        out["multi_gpu"] = res if res is not None else "no size fitted"
    text = json.dumps(out, indent=1)
    print(text)
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
