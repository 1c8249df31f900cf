"""Experiment (GPU): cost of ``Expectation`` of general operators on device states (``pb200_state_expect`` /
``pb200_shards_expect``) against the host fallback it replaces.

Four operators: sum_i sigma^x_i, sum_i (-1)^i sigma^z_i, all pairs sigma^+_i sigma^-_j + h.c. and the all-site Z
parity.  For each, the device call (term table upload, kernel, the 16-byte result back) is timed with CUDA events over
``--reps`` calls after ``--warmup`` calls, at N = 20 and N = 24 on one plan and on 4 shards of N = 20 that all live on
device 0.  Beside each time: the bytes the kernel must move, 16 D (1 + #distinct non-zero flip masks), and that figure
over the time.  At N = 20 the host fallback is timed too (not for the pairs, whose matrix has 1e8 non-zeros): the
matrix build (once per operator), and per evaluation the state copied to the host plus the CSR matvec.  The card name and power limit are recorded in the same run.  Prints one
JSON object.

Usage: python experiments/expect_cost.py [--reps R] [--warmup W] [--out FILE]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pulser_b200 import engine, sharded, workloads as W  # noqa: E402
from pulser_b200.backend import B200Operator  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__))))
from shard_scaling import gpu_info  # noqa: E402


def operators(n: int) -> dict:
    x = {"rg": 1.0, "gr": 1.0}
    z = {"rr": 1.0, "gg": -1.0}
    return {
        "sum_x": [(1.0, [(x, {i})]) for i in range(n)],
        "staggered_z": [((-1.0) ** i, [(z, {i})]) for i in range(n)],
        "pairs_pm": [(1.0, [({"rg": 1.0}, {i}), ({"gr": 1.0}, {j})]) for i in range(n) for j in range(n) if i != j],
        "parity": [(1.0, [(z, set(range(n)))])],
    }


def distinct_masks(terms) -> int:
    return len({sum(1 << (terms.n - 1 - k) for k, m, _ in sites if m) for _, sites in terms.terms} - {0})


def time_device(call, reps: int, warmup: int) -> float:
    import torch

    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        call()  # each call ends in a stream synchronise (the result is on the host)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps * 1e3  # us


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert engine.device_count() > 0, "expect_cost.py needs a CUDA device"
    rng = np.random.default_rng(0)
    report = {"gpus": gpu_info(), "reps": args.reps, "warmup": args.warmup, "rows": []}
    for n, G in ((20, 1), (24, 1), (20, 4)):
        spec = W.config_c2(n=n, seed=1)
        D = 1 << n
        psi = rng.normal(size=D) + 1j * rng.normal(size=D)
        psi /= np.linalg.norm(psi)
        plan = engine.DevicePlan(spec) if G == 1 else sharded.ShardedPlan(spec, [0] * G)
        with plan:
            plan.set_state(psi)
            for name, ops in operators(n).items():
                op = B200Operator.from_operator_repr(eigenstates=("r", "g"), n_qudits=n, operations=ops)
                terms = op._terms
                us = time_device(lambda: plan.expect_terms(terms), args.reps, args.warmup)
                masks = distinct_masks(terms)
                nbytes = 16 * D * (1 + masks)
                row = {"n": n, "shards": G, "operator": name, "terms": len(terms), "distinct_masks": masks,
                       "device_us": round(us, 2), "bytes": nbytes, "bytes_per_s": nbytes / (us * 1e-6),
                       "value": complex(plan.expect_terms(terms)[0]).real}
                if n == 20 and G == 1 and name != "pairs_pm":  # pairs_pm: 1e8 non-zeros, minutes of Kronecker products
                    t0 = time.perf_counter()
                    mat = op._operator  # the CSR matrix of the host fallback
                    row["host_build_s"] = round(time.perf_counter() - t0, 3)
                    t0 = time.perf_counter()
                    for _ in range(3):
                        host = plan.get_state()[0]
                        val = np.vdot(host, mat @ host)
                    row["host_eval_ms"] = round((time.perf_counter() - t0) / 3 * 1e3, 2)
                    row["host_value"] = complex(val).real
                report["rows"].append(row)
                print(json.dumps(row), flush=True)
    print(json.dumps(report))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
