"""Experiment (GPU): the master equation under a moving drive phase on the Taylor propagator against the splitting path.

Cases: the 300 ns blockade sweep of experiments/lindblad_cost.py (50 / 200 / 50 ns) with dephasing 0.05 and relaxation
0.01 rad/us on N = 8, 10, 12 (and 13, Taylor alone), at tol = 1e-10, "Minimal" evaluation times, in four variants:
  constant  the sweep at one phase (real orders only: the reference for the cost of a real order)
  jump      a phase jump of pi/2 under full amplitude mid-sweep (150 ns)
  ramsey    a Ramsey pair: pi/2 pulses of 50 ns at phases 0 and 1.1 around 200 ns of free evolution under the sweep's
            detuning
  ramp      the sweep under a phase ramp of 2 rad over the whole sequence: every step complex (the worst case)
Each variant runs on the Taylor propagator (integrator 3) and on the Richardson-CF4 + Strang splitting path with
Chebyshev (1) and Lanczos (2) exponentials.

Per run: device time, H-applies per ns, microseconds per order, and from the step log (PB200_TAYLOR_LOG) the share of
complex orders (steps with drive=cplx, weighted by their K) and the largest ring R; for splitting, max |rho - rho_taylor|.
The microseconds of a real order are those of `constant`, those of a complex order those of `ramp`.  Best of `--reps`
for Taylor, one run for splitting at N >= 12.  The card name and power limit are recorded in the same run.  Prints one
JSON line per case and one JSON object at the end.

Usage: python experiments/lindblad_phase_cost.py [--reps R] [--sizes 8,10,12,13] [--out FILE]
"""
from __future__ import annotations

import json
import os
import re
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from experiments.lindblad_cost import channel  # noqa: E402
from experiments.shard_scaling import gpu_info  # noqa: E402
from pulser_b200 import workloads as W  # noqa: E402
from pulser_b200.lindblad import LindbladPlan  # noqa: E402

STEP_RE = re.compile(r"taylor step .* K=(\d+) ring=(\d+) .* drive=(\w+)")
VARIANTS = ("constant", "jump", "ramsey", "ramp")


def spec_of(n: int, variant: str):
    amp, det = W.blockade_sweep_waveforms(t_rise=50, t_sweep=200, t_fall=50)
    T = len(amp)
    t = np.arange(T)
    phase = np.zeros(T)
    if variant == "jump":
        phase = np.where(t < T // 2, 0.0, np.pi / 2)
    elif variant == "ramsey":
        amp = np.where((t < 50) | (t >= T - 50), np.pi / 0.1, 0.0)   # pi/2 in 50 ns at Omega = 10 pi rad/us
        phase = np.where(t < T // 2, 0.0, 1.1)
    elif variant == "ramp":
        phase = 2.0 * t / T
    spec = W.ising_global_spec(W.disc_register(n, 38.0, 5.0, n), W.C6_LEVEL_60, amp, det, phase=phase)
    spec.collapse_ops = channel("dephasing+relaxation")
    return spec


def run(spec, integrator: int, reps: int):
    best = None
    for _ in range(reps):
        with tempfile.TemporaryFile(mode="w+") as f:
            fd = os.dup(2)
            os.dup2(f.fileno(), 2)
            try:
                with LindbladPlan(spec) as lp:
                    lp.set_state(np.eye(1, 2**spec.n_qudits, 2**spec.n_qudits - 1)[0])   # all atoms in g
                    st = lp.propagate(0.0, float(spec.sampling_times[-1]), integrator=integrator, tol=1e-10)
                    rho = lp.get_rho()[0]
            finally:
                os.dup2(fd, 2)
                os.close(fd)
            f.seek(0)
            steps = [(int(m[1]), int(m[2]), m[3]) for m in STEP_RE.finditer(f.read())]
        st = {k: st[k] for k in ("gpu_ms", "n_applies", "n_steps", "err_estimate", "integrator")}
        if steps:
            orders = sum(k for k, _, _ in steps)
            st["cplx_order_share"] = sum(k for k, _, d in steps if d == "cplx") / max(orders, 1)
            st["steps_by_kind"] = {d: sum(1 for _, _, e in steps if e == d) for d in ("real", "rot", "cplx")}
            st["max_ring"] = max(r for _, r, _ in steps)
        if best is None or st["gpu_ms"] < best[0]["gpu_ms"]:
            best = (st, rho)
    st, rho = best
    st["applies_per_ns"] = st["n_applies"] / spec.total_duration_ns
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
        for variant in VARIANTS:
            spec = spec_of(n, variant)
            case = {"n": n, "variant": variant}
            st3, rho3 = run(spec, 3, args.reps)
            assert st3["integrator"] == 3
            case["taylor"] = st3
            if n <= 12 and variant != "constant":   # constant-phase splitting: experiments/lindblad_cost.py
                for integ in (1, 2):
                    st, rho = run(spec, integ, 1 if n >= 12 else args.reps)
                    st["max_diff_to_taylor"] = float(np.max(np.abs(rho - rho3)))
                    case[f"splitting_{integ}"] = st
            out["cases"].append(case)
            print(json.dumps(case), flush=True)
    text = json.dumps(out)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
