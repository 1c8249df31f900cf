"""Experiment (GPU): the master equation on state-vector shards against one plan.

Case: the N = 13 dephasing + relaxation sweep of ``experiments/lindblad_cost.py`` ("Minimal" evaluation times: one call
over the sequence, tol = 1e-10) on one ``LindbladPlan`` and on 2, 4 and 8 shards of one device
(``ShardedLindbladPlan``), which adds the peer loads across the shard bits and one launch per shard and order.  Per run:
device time, microseconds per order, the schedule (steps, H-applies, err_estimate: equal across the runs) and
max |rho_shards - rho_one|.  Best of `--reps`.

Ring: the largest Taylor ring R (state-sized buffers per step, from the ``PB200_TAYLOR_LOG`` step log) of the unsharded
plan at N = 10 .. 13, for both channels; a shard of vec(rho) needs (R 16 + 8) 2^L bytes, L = 2N - log2(G).

The card name and power limit are recorded in the same run.  Prints one JSON object.

Usage: python experiments/lindblad_shards_cost.py [--reps R] [--out FILE]
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from experiments.lindblad_cost import RING_RE, spec_of  # noqa: E402
from experiments.shard_scaling import gpu_info  # noqa: E402
from pulser_b200.lindblad import LindbladPlan, ShardedLindbladPlan  # noqa: E402


def run(make, spec, reps: int):
    """Best of `reps` whole-sequence runs of the plan `make()`; the step log's largest ring with it."""
    tf = float(spec.sampling_times[-1])
    ground = np.eye(1, 2**spec.n_qudits, 2**spec.n_qudits - 1)[0]   # all atoms in g
    best = None
    for _ in range(reps):
        with tempfile.TemporaryFile(mode="w+") as f:
            fd = os.dup(2)
            os.dup2(f.fileno(), 2)
            try:
                with make() as plan:
                    plan.set_state(ground)
                    st = plan.propagate(0.0, tf, tol=1e-10, integrator=3)
                    rho = plan.get_rho()[0]
            finally:
                os.dup2(fd, 2)
                os.close(fd)
            f.seek(0)
            rings = [int(m[1]) for m in RING_RE.finditer(f.read())]
        st = {k: st[k] for k in ("gpu_ms", "n_steps", "n_applies", "err_estimate", "integrator")}
        st["max_ring"] = max(rings) if rings else None
        st["us_per_order"] = 1e3 * st["gpu_ms"] / max(st["n_applies"], 1)
        if best is None or st["gpu_ms"] < best[0]["gpu_ms"]:
            best = (st, rho)
    return best


def main() -> None:
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    os.environ["PB200_TAYLOR_LOG"] = "1"
    out = {"gpu": gpu_info(), "n13": {}, "ring": []}
    spec = spec_of(13, "dephasing+relaxation")
    one, rho1 = run(lambda: LindbladPlan(spec), spec, args.reps)
    out["n13"]["one"] = one
    print(json.dumps({"one": one}), flush=True)
    for G in (2, 4, 8):
        st, rho = run(lambda: ShardedLindbladPlan(spec, [0] * G), spec, args.reps)
        st["max_diff_to_one"] = float(np.max(np.abs(rho - rho1)))
        st["time_ratio"] = st["gpu_ms"] / one["gpu_ms"]
        out["n13"][f"shards_{G}"] = st
        print(json.dumps({f"shards_{G}": st}), flush=True)
    for n in (10, 11, 12, 13):
        for kind in ("dephasing+relaxation", "depolarizing"):
            s = spec_of(n, kind)
            st, _ = (one, None) if (n, kind) == (13, "dephasing+relaxation") else run(lambda: LindbladPlan(s), s, 1)
            out["ring"].append({"n": n, "noise": kind, "max_ring": st["max_ring"]})
            print(json.dumps(out["ring"][-1]), flush=True)
    text = json.dumps(out)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
