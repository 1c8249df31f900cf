"""Experiment (GPU): the single-precision tail orders of the Taylor propagator on C2 and C5.

Per workload: the fraction of orders at or after each step's switch order k_lo (from the step log,
``PB200_TAYLOR_LOG``), and the device time per order of each precision combination of the stage kernel
(fp64 -> fp64, fp64 -> fp32 at k_lo, fp32 -> fp32): the interval between its completion and the previous order's in
the ``torch.profiler`` kernel records of one whole sequence after a warm-up run.  The card name and power limit are
recorded in the same run.  Prints one JSON object.

Usage: python experiments/taylor_lowprec_cost.py [--out FILE]
"""
from __future__ import annotations

import json
import os
import re
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from experiments.shard_scaling import gpu_info  # noqa: E402
from pulser_b200 import engine, workloads as W  # noqa: E402

STEP_RE = re.compile(r"taylor step .* K=(\d+) ring=.* k_lo=(\d+)")
KERNEL_RE = re.compile(r"stage_d2_taylor_kernel<([^>]*)>")
COMBOS = {(False, False): "fp64->fp64", (False, True): "fp64->fp32", (True, True): "fp32->fp32"}


def step_log(spec):
    """(K, k_lo) of every step of one whole sequence, read from stderr through a temporary file"""
    os.environ["PB200_TAYLOR_LOG"] = "1"
    with tempfile.TemporaryFile(mode="w+") as f:
        fd = os.dup(2)
        os.dup2(f.fileno(), 2)
        try:
            with engine.DevicePlan(spec) as plan:
                plan.set_state("all-ground")
                plan.propagate(0.0, spec.sampling_times[-1])
        finally:
            os.dup2(fd, 2)
            os.close(fd)
            del os.environ["PB200_TAYLOR_LOG"]
        f.seek(0)
        return [(int(m[1]), int(m[2])) for m in STEP_RE.finditer(f.read())]


def kernel_times(spec):
    """device time per order of each precision combination over one profiled sequence (after a warm-up run)"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    with engine.DevicePlan(spec) as plan:
        plan.set_state("all-ground")
        plan.propagate(0.0, spec.sampling_times[-1])
        plan.set_state("all-ground")
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            st = plan.propagate(0.0, spec.sampling_times[-1])
            torch.cuda.synchronize()
    recs = []
    for ev in prof.events():
        m = KERNEL_RE.search(ev.name)
        if not m or ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        args = [x.strip() for x in m.group(1).split(",")]
        key = COMBOS.get((args[8] == "true", args[9] == "true"), "other") if len(args) == 10 else "fp64->fp64"
        recs.append((ev.time_range.start, ev.time_range.end, key))
    # programmatic dependent launch starts an order while the previous one drains, so a kernel record also holds its
    # wait on the previous order: an order's time is the interval between its completion and the previous one's
    recs.sort()
    per = {}
    for i, (t0, t1, key) in enumerate(recs):
        n, us = per.get(key, (0, 0.0))
        per[key] = (n + 1, us + (t1 - (recs[i - 1][1] if i else t0)))
    total = sum(n for n, _ in per.values())
    return {
        "orders": int(st["n_applies"]), "kernel_records": total,
        "per_combination": {k: {"orders": n, "us_per_order": us / n, "share": n / total} for k, (n, us) in sorted(per.items())},
        "us_per_order_all": sum(us for _, us in per.values()) / max(total, 1),
    }


def main():
    out = {"gpu": gpu_info()}
    for name, spec in (("c2", W.config_c2(n=20)), ("c5", W.config_c5(n=24))):
        steps = step_log(spec)
        orders = sum(k for k, _ in steps)
        low = sum(k - lo for k, lo in steps)
        out[name] = {"steps": len(steps), "orders": orders, "orders_at_or_after_k_lo": low,
                     "fraction_low": low / max(orders, 1), **kernel_times(spec)}
    text = json.dumps(out, indent=1)
    print(text)
    if "--out" in sys.argv:
        with open(sys.argv[sys.argv.index("--out") + 1], "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
