"""Experiment (GPU): the master equation on the Taylor propagator against the splitting path.

Cases: C2's blockade sweep (SURVEY 8d, shortened to 50 / 200 / 50 ns so that the splitting path at N = 13 stays
affordable) on N = 8, 10, 12, 13 disc registers, with dephasing 0.05 and relaxation 0.01 rad/us (C4's noise rates) and
with depolarizing 0.05 rad/us; "Minimal" evaluation times (one call over the sequence) and "Full" ones (one call per
sampling interval, N <= 10).  Each case runs on the Taylor propagator (integrator 3) and on the Richardson-CF4 + Strang
splitting path with Chebyshev (1) and Lanczos (2) exponentials, all at tol = 1e-10.

Per run: device time, H-applies per ns, microseconds per order (Taylor; dephasing alone has no both-flip loads), the
largest ring R from the step log, the card's memory in use after the run (the buffer pool keeps what a plan took, so it
bounds the peak), and max |rho_taylor - rho_splitting|.  Best of `--reps`.  The card name and power limit are recorded
in the same run.  Prints one JSON object.

Usage: python experiments/lindblad_cost.py [--reps R] [--out FILE]
"""
from __future__ import annotations

import json
import os
import re
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from experiments.shard_scaling import gpu_info  # noqa: E402
from pulser_b200 import workloads as W  # noqa: E402
from pulser_b200.lindblad import LindbladPlan  # noqa: E402

RING_RE = re.compile(r"taylor step .* ring=(\d+) ")
SIGMA = [np.array([[0, 1], [1, 0]], dtype=complex), np.array([[0, -1j], [1j, 0]]), np.array([[1, 0], [0, -1]], dtype=complex)]


def channel(kind: str) -> np.ndarray:
    deph = np.sqrt(2 * 0.05) * np.diag([1.0, 0.0])[None].astype(complex)   # Pulser: sqrt(rate / 2) Z = this up to a phase
    relax = np.zeros((1, 2, 2), dtype=complex)
    relax[0, 1, 0] = np.sqrt(0.01)                                          # sqrt(rate) |g><r|, r = digit 0
    if kind == "dephasing":
        return deph
    if kind == "dephasing+relaxation":
        return np.concatenate([deph, relax])
    if kind == "depolarizing":
        return np.array([np.sqrt(0.05 / 4) * s for s in SIGMA])
    raise ValueError(kind)


def spec_of(n: int, kind: str):
    amp, det = W.blockade_sweep_waveforms(t_rise=50, t_sweep=200, t_fall=50)
    spec = W.ising_global_spec(W.disc_register(n, 38.0, 5.0, n), W.C6_LEVEL_60, amp, det)
    spec.collapse_ops = channel(kind)
    return spec


def run(spec, full: bool, integrator: int, reps: int):
    import torch

    times = spec.sampling_times if full else spec.sampling_times[[0, -1]]
    best = None
    for _ in range(reps):
        with tempfile.TemporaryFile(mode="w+") as f:
            fd = os.dup(2)
            os.dup2(f.fileno(), 2)
            try:
                tot = {"gpu_ms": 0.0, "n_applies": 0, "n_steps": 0, "err_estimate": 0.0, "integrator": 0}
                with LindbladPlan(spec) as lp:
                    lp.set_state(np.eye(1, 2**spec.n_qudits, 2**spec.n_qudits - 1)[0])   # all atoms in g
                    for t0, t1 in zip(times[:-1], times[1:]):
                        st = lp.propagate(float(t0), float(t1), integrator=integrator, tol=1e-10)
                        for k in ("gpu_ms", "n_applies", "n_steps", "err_estimate"):
                            tot[k] += st[k]
                        tot["integrator"] = st["integrator"]
                    rho = lp.get_rho()[0]
                    free, total = torch.cuda.mem_get_info()
            finally:
                os.dup2(fd, 2)
                os.close(fd)
            f.seek(0)
            rings = [int(m[1]) for m in RING_RE.finditer(f.read())]
        tot["max_ring"] = max(rings) if rings else None
        tot["mem_in_use_gib"] = (total - free) / 2**30
        if best is None or tot["gpu_ms"] < best[0]["gpu_ms"]:
            best = (tot, rho)
    st, rho = best
    T = spec.total_duration_ns
    st["applies_per_ns"] = st["n_applies"] / T
    st["us_per_order"] = 1e3 * st["gpu_ms"] / max(st["n_applies"], 1)
    return st, rho


def main() -> None:
    import argparse

    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--sizes", default="8,10,12,13")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    os.environ["PB200_TAYLOR_LOG"] = "1"
    out = {"gpu": gpu_info(), "cases": []}
    for n in [int(x) for x in args.sizes.split(",")]:
        for kind in ("dephasing", "dephasing+relaxation", "depolarizing"):
            for full in (False, True):
                if full and n > 10:
                    continue
                spec = spec_of(n, kind)
                case = {"n": n, "noise": kind, "eval": "Full" if full else "Minimal"}
                st3, rho3 = run(spec, full, 3, args.reps)
                case["taylor"] = st3
                for integ in (1, 2):
                    if n == 13 and integ == 1:
                        continue   # Chebyshev at 2^26 amplitudes: Lanczos is the automatic choice there
                    st, rho = run(spec, full, integ, 1 if n >= 12 else args.reps)
                    st["max_diff_to_taylor"] = float(np.max(np.abs(rho - rho3)))
                    case[f"splitting_{integ}"] = st
                out["cases"].append(case)
                print(json.dumps(case), flush=True)
    text = json.dumps(out)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
